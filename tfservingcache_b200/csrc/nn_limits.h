// Shapes the transformer kernels of nn_kernels.cu can run. Host-only (no CUDA headers): the manifest loader (model.cc)
// rejects a bundle with the same rule the launchers apply, so a model that pages in can always be served.
#pragma once
#include <cfloat>
#include <cstddef>

namespace tfsc {

constexpr size_t kAttnSmemCap = 200 * 1024;  // dynamic shared memory the attention kernels opt in to

// CUDA's cap on gridDim.y (and z). Launchers whose y extent grows with the batch split the batch on the host above it.
constexpr int kMaxGridY = 65535;

// row-at-a-time attention kernel: K [S][d+1], V [S][d], P [8][S], Q [8][d] and the mask [S] of one head
inline size_t attention_smem_bytes(int S, int H, int heads) {
  const int d = H / heads;
  return ((size_t)S * (d + 1) + (size_t)S * d + (size_t)8 * S + 8 * d + S) * sizeof(float);
}

// Head width d = H / heads with d % 4 == 0 and d <= 128 runs at every S (tiled kernels up to S = 256, the key-block kernel
// above) on 16-byte aligned qkv / ctx; every other width runs on the row kernel while its shared memory fits.
inline bool attention_supported(int S, int H, int heads, bool aligned16) {
  if (S < 1 || heads < 1 || H < heads || H % heads) return false;
  const int d = H / heads;
  if (d % 4 == 0 && H % 4 == 0 && d <= 128 && aligned16) return true;
  return attention_smem_bytes(S, H, heads) <= kAttnSmemCap;
}

// Causal attention (query i sees keys j <= i) runs on the tiled and key-block kernels only: d % 4 == 0, d <= 128, 16-byte
// aligned qkv / ctx, every S.
inline bool attention_causal_supported(int S, int H, int heads, bool aligned16) {
  if (S < 1 || heads < 1 || H < heads || H % heads) return false;
  const int d = H / heads;
  return d % 4 == 0 && H % 4 == 0 && d <= 128 && aligned16;
}

// LayerNorm stages one row of H floats in dynamic shared memory next to its 64-byte reduction scratch, within the 48 KB a
// kernel gets without opting in: H <= 12272
inline bool layernorm_supported(int H) { return H >= 1 && (size_t)H * sizeof(float) + 64 <= 48 * 1024; }

// Classification head (head.cu): one CTA stages a row of N logits in shared memory (128 KB at N = 32768, a BERT-vocab head
// of 30522 fits) and selects the top k of them by k block-wide argmax rounds. A head without top-k outputs runs as k = 1.
constexpr int kHeadMaxN = 32768, kHeadMaxK = 32;
inline bool head_supported(int N, int k) { return N >= 1 && N <= kHeadMaxN && k >= 1 && k <= kHeadMaxK && k <= N; }

// Span head (span.cu): one CTA stages the start and end logits of a row of S tokens and the best end of every start in
// shared memory (64 KB at S = 4096) and selects the k best (start, end) pairs with end - start < L by k warp argmax
// rounds. A head with start / end logits only runs as L = k = 1.
constexpr int kSpanMaxS = 4096, kSpanMaxK = 32;
inline bool span_supported(int S, int L, int k) { return S >= 1 && S <= kSpanMaxS && L >= 1 && L <= S && k >= 1 && k <= kSpanMaxK; }

// Encoder head (encoder_head.cu): a cluster of up to 8 CTAs per row streams the [S, H] hidden states once; each CTA keeps
// fp32 partial sums of its tokens for H columns in shared memory (32 KB at H = 8192), and in-row offsets p * H + c are
// 32-bit (S * H <= 2^26).
constexpr int kEncoderMaxS = 8192, kEncoderMaxH = 8192;
inline bool encoder_head_supported(int S, int H) { return S >= 1 && S <= kEncoderMaxS && H >= 1 && H <= kEncoderMaxH; }

// Fill-mask (mlm.cu). The gather: one CTA per row scans S tokens for [MASK] and copies the hidden states of up to M of them
// (1 <= M <= S <= 8192, H <= 8192, M positions in shared memory). The head: one CTA per (row, slot) stages the first `vocab`
// logits of its slot like the classification head (128 KB at vocab = 32768) and selects the top k of them. A head with
// masked_positions only runs as k = 1.
constexpr int kMaskGatherMaxS = 8192, kMaskGatherMaxH = 8192;
inline bool mask_gather_supported(int S, int H, int M) {
  return S >= 1 && S <= kMaskGatherMaxS && H >= 1 && H <= kMaskGatherMaxH && M >= 1 && M <= S;
}
inline bool fill_mask_supported(int M, int vocab, int k) {
  return M >= 1 && M <= kMaskGatherMaxS && vocab >= 1 && vocab <= kHeadMaxN && k >= 1 && k <= kHeadMaxK && k <= vocab;
}

// Next-token head (mlm.cu): the fill-mask head's kernel with one slot per row. Its CTA stages a row of `vocab` fp32 logits
// in dynamic shared memory beside about 0.4 KB of static shared memory, within the 227 KB a CTA may opt in to on an H100:
// vocab <= 57344 (224 KB), which holds GPT-2's 50257. A head with next_token_position only runs as k = 1.
constexpr int kNextTokenMaxVocab = 57344;
inline bool next_token_supported(int vocab, int k) {
  return vocab >= 1 && vocab <= kNextTokenMaxVocab && k >= 1 && k <= kHeadMaxK && k <= vocab;
}

// Scoring (score.cu): the token_score op projects at most kScoreChunkTokens token rows of the flattened [rows x S] batch at a
// time into one chunk-sized logits region (206 MB at Vp = 50272), and its score kernel stages a row of `vocab` logits like the
// next-token head (vocab <= 57344). The score head walks the S positions of a row.
constexpr int kScoreChunkTokens = 1024, kScoreMaxS = 16384;
inline bool score_supported(int S, int vocab) { return S >= 1 && S <= kScoreMaxS && vocab >= 1 && vocab <= kNextTokenMaxVocab; }

// Decode attention (generate.cu): one query per row over L cached keys, split into blocks of kDecodeKeys keys, one CTA per
// (row, head, block). A CTA stages its block's keys in shared memory (34 KB at d = 128, within the 48 KB a kernel gets
// without opting in) and the last CTA of a (row, head) combines the blocks in order. Head width d % 4 == 0, d <= 128.
constexpr int kDecodeKeys = 64, kDecodeMaxKeys = 16384;
inline int decode_attention_splits(int L) { return (L + kDecodeKeys - 1) / kDecodeKeys; }
inline bool decode_attention_supported(int L, int H, int heads) {
  if (L < 1 || L > kDecodeMaxKeys || heads < 1 || H < heads || H % heads) return false;
  const int d = H / heads;
  return d % 4 == 0 && d <= 128;
}
// The work buffer a launch over keys [0, L) needs: an int32 counter per (row, head), which must be zero before the first
// launch and is left zero by each, then each block's running max, sum and unnormalised context.
inline size_t decode_attention_work_bytes(long long rows, int L, int H, int heads) {
  const size_t rh = (size_t)rows * heads, parts = rh * decode_attention_splits(L);
  return ((rh * 4 + 255) & ~(size_t)255) + parts * (2 + (size_t)(H / heads)) * sizeof(float);
}

// Greedy generation (generate.cu): the select step stages a row of `vocab` logits like the next-token head (vocab <= 57344)
// and writes max_new_tokens = N ids and log-probabilities per row; the decode steps' keys are bounded by decode attention's.
inline bool generate_supported(int vocab, int N) {
  return vocab >= 1 && vocab <= kNextTokenMaxVocab && N >= 1 && N <= kDecodeMaxKeys;
}
// Sampled generation (generate.cu): a temperature whose fp32 value and fp32 reciprocal are finite and > 0 (the kernel
// weighs (z - m) * (1 / temperature): a subnormal temperature's reciprocal is inf), 0 <= top_k <= vocab (0: off) and
// 0 < top_p <= 1 (1: off).
inline bool sampling_temperature_ok(double temperature) {
  const float t = (float)temperature;
  return temperature > 0 && temperature <= FLT_MAX && t > 0.f && 1.f / t <= FLT_MAX;
}
inline bool sampling_supported(int vocab, double temperature, int top_k, double top_p) {
  return sampling_temperature_ok(temperature) && top_k >= 0 && top_k <= vocab && top_p > 0 && top_p <= 1;
}
// Repetition control (generate.cu): a repetition penalty whose fp32 value is finite, > 0 and normal (the kernel multiplies
// and divides by it in fp32, as torch does), a no-repeat n-gram size n >= 0 (0: off) and a minimum length m >= 0 (0: off).
inline bool repetition_penalty_ok(double p) {
  const float f = (float)p;
  return p > 0 && p <= FLT_MAX && f >= FLT_MIN && f <= FLT_MAX;
}
inline bool processing_supported(double penalty, int ngram, int min_new) {
  return repetition_penalty_ok(penalty) && ngram >= 0 && min_new >= 0;
}

// Depthwise convolution (depthwise.cu): a thread runs the kh x kw taps of one output pixel for 4 channels (1 on the scalar
// path). Kernels up to 7 x 7, stride 1 or 2 and padding up to k / 2 cover MobileNetV2 and EfficientNet B0-B7 (3 x 3 and
// 5 x 5, stride <= 2) with margin; offsets within an image are 32-bit (H * W * C < 2^31).
constexpr int kDepthwiseMaxK = 7, kDepthwiseMaxStride = 2;
inline bool depthwise_supported(int H, int W, int C, int KH, int KW, int stride, int pad) {
  return H >= 1 && W >= 1 && C >= 1 && KH >= 1 && KH <= kDepthwiseMaxK && KW >= 1 && KW <= kDepthwiseMaxK && stride >= 1 &&
         stride <= kDepthwiseMaxStride && pad >= 0 && pad <= KH / 2 && pad <= KW / 2 && H + 2 * pad >= KH && W + 2 * pad >= KW &&
         (long long)H * W * C <= 0x7fffffffLL;
}

// Shifted-window attention (swin.cu): one CTA per (image, window, head) stages K [N][d+1] and V [N][d] of its window
// (N = ws^2 tokens) and a query row and a probability row per warp in shared memory, within the 48 KB a kernel gets without
// opting in; a lane holds ceil(N / 32) <= 8 scores. ws = 7 and 12 at d = 32 (every torchvision Swin V1) fit, ws = 12 up to
// d = 39, ws = 7 up to d = 64. C is the context width (the source holds 3C values per token); offsets within an image are
// 32-bit (H * W * 3C < 2^31).
constexpr int kWindowMaxWs = 16, kWindowMaxD = 64, kWindowWarps = 4;
inline size_t window_attention_smem_bytes(int ws, int d) {
  const size_t N = (size_t)ws * ws;
  return (N * (2 * d + 1) + (size_t)kWindowWarps * (N + d)) * sizeof(float);
}
inline bool window_attention_supported(int H, int W, int C, int heads, int ws, int shift) {
  if (H < 1 || W < 1 || C < 1 || heads < 1 || C % heads || ws < 1 || ws > kWindowMaxWs || H % ws || W % ws || shift < 0 ||
      shift >= ws)
    return false;
  const int d = C / heads;
  return d <= kWindowMaxD && window_attention_smem_bytes(ws, d) <= 48 * 1024 && (long long)H * W * 3 * C <= 0x7fffffffLL;
}

// Patch merging (swin.cu): a 2 x 2 space-to-depth gather, [h, w, c] -> [h/2, w/2, 4c]; offsets within an image are 32-bit.
inline bool patch_merge_supported(int h, int w, int c) {
  return h >= 2 && w >= 2 && h % 2 == 0 && w % 2 == 0 && c >= 1 && (long long)h * w * c <= 0x7fffffffLL;
}

}  // namespace tfsc
