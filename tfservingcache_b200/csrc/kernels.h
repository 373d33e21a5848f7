// Device kernels of the executor (SURVEY.md section 8a row X). All fp32, sm_90a.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "nn_limits.h"

namespace tfsc {

constexpr int kMaxRowsPerLaunch = 8;  // rows handled by one streaming pass over W (SIMT path)

// X1: y = a*x + b (a, b device scalars). half_plus_two (deploy/docker-compose/readme.md:40-42).
cudaError_t launch_affine(const float* x, float* y, int64_t n, const float* a, const float* b, cudaStream_t s);

// X2: y[rows,n] = act(x[rows,k] W[k,n] + bias[n]); W row-major [k,n]. Streams W exactly once per
// group of <= kMaxRowsPerLaunch rows. workspace: dense_workspace_bytes(rows,k,n), zero-initialised
// counters are maintained by the kernel itself (self-resetting).
size_t dense_workspace_bytes(int rows, int k, int n);
cudaError_t launch_dense(const float* x, const float* w, const float* bias, float* y, int rows, int k, int n,
                         bool relu, void* workspace, size_t workspace_bytes, cudaStream_t s, int variant = 0);
// variant: 0 auto (TFSC_DENSE_VARIANT, default LDG stream for <= 8 rows + tensor cores above), 1 LDG stream only,
// 2 / 4 bulk-copy (TMA) ring for the <= 8-row passes (tensor cores above, as in auto), 3 tensor cores for every row count,
// 5 cluster-pair kernel for the <= 8-row passes (experimental)

// X3: wgmma 3xTF32 path for 9..64 rows per pass (dense_tc.cu)
bool dense_tc_supported(int rows, int k, int n, const float* w, const float* x, const float* bias, const float* y);
// output columns per tensor-core strip: one arrival counter each at the start of a dense workspace (tc::STRIP)
constexpr int kTcStripCols = 256;
size_t dense_tc_workspace_bytes(int k, int n);
cudaError_t launch_dense_tc(const float* x, const float* w, const float* bias, float* y, int rows, int k, int n,
                            bool relu, void* workspace, size_t workspace_bytes, cudaStream_t s);

// X2, cluster-pair kernel (dense_cluster.cu, default for <= 8 rows): two CTAs of a cluster split K and meet in
// distributed shared memory -- no split-K workspace, no atomics. rows <= 8, n % 4 == 0, k % 4 == 0, k >= 128.
bool dense_cluster_supported(int rows, int k, int n, const float* w, const float* x, const float* bias, const float* y);
cudaError_t launch_dense_cluster(const float* x, const float* w, const float* bias, float* y, int rows, int k, int n, bool relu,
                                 cudaStream_t s);
// grid of the cluster kernel on the current device: co-resident 2-CTA clusters and the strip width chosen for n columns
cudaError_t dense_cluster_grid(int rows, int n, int* active_clusters, int* strip_cols);

// X4/X5 building blocks (nn_kernels.cu): act 0 none / 1 relu / 2 gelu(erf) / 3 tanh / 4 relu6 / 5 silu / 6 sigmoid /
// 7 gelu_tanh
cudaError_t launch_gemm(const float* A, const float* B, const float* bias, const float* R, float* C, int M, int N, int K,
                        int lda, int act, cudaStream_t s);
cudaError_t launch_im2col(const float* x, float* col, int Bn, int H, int W, int C, int KH, int KW, int stride, int pad,
                          int OH, int OW, int ldc, cudaStream_t s);
cudaError_t launch_maxpool(const float* x, float* y, int Bn, int H, int W, int C, int KH, int KW, int stride, int pad, int OH,
                           int OW, cudaStream_t s);
cudaError_t launch_avgpool(const float* x, float* y, int Bn, int HW, int C, cudaStream_t s);
// MobileNet / EfficientNet blocks (depthwise.cu). y[b, oy, ox, ch] = act(sum_ij x[b, oy*stride - pad + i, ox*stride - pad +
// j, ch] * w[i, j, ch] + bias[ch]), w [KH, KW, C], act 0 none / 1 relu / 4 relu6 / 5 silu / 6 sigmoid; cudaErrorInvalidValue
// outside depthwise_supported (nn_limits.h), for another act or a null pointer.
cudaError_t launch_depthwise_conv(const float* x, const float* w, const float* bias, float* y, int Bn, int H, int W, int C, int KH,
                                  int KW, int stride, int pad, int act, cudaStream_t s);
// y[b, p, ch] = x[b, p, ch] * gate[b, ch] over HW positions p (the squeeze-and-excitation gate)
cudaError_t launch_channel_scale(const float* x, const float* gate, float* y, int Bn, int HW, int C, cudaStream_t s);
// Swin blocks (swin.cu). Shifted-window attention over the packed q | k | v [H, W, 3C] of each image, writing ctx [H, W, C]:
// heads of d = C / heads columns, ws x ws windows of the map rolled by -shift, bias [heads, ws^2, ws^2] added to the
// scores, -100 between tokens of different shift regions (shift > 0). cudaErrorInvalidValue outside
// window_attention_supported (nn_limits.h) or for a null pointer.
cudaError_t launch_window_attention(const float* qkv, const float* bias, float* ctx, int Bn, int H, int W, int C, int heads, int ws,
                                    int shift, cudaStream_t s);
// y[b, oy, ox, q*C + c] = x[b, 2oy + (q & 1), 2ox + (q >> 1), c] (patch merging), [H, W, C] -> [H/2, W/2, 4C]
cudaError_t launch_patch_merge(const float* x, float* y, int Bn, int H, int W, int C, cudaStream_t s);
// y = LayerNorm(x (+res)) or, with ids != nullptr, LayerNorm(word[id] + pos[s] + type[t]) (BERT embeddings): token
// b*S + s reads ids[b*stride + s] and, unless types is nullptr (segment 0), t = clamp(types[b*stride + s], 0, 1)
cudaError_t launch_layernorm(const float* x, const float* res, const int* ids, const int* types, int stride, const float* word,
                             const float* pos, const float* type, const float* gamma, const float* beta, float* y, int tokens,
                             int S, int H, int vocab, float eps, cudaStream_t s);
// multi-head self-attention: qkv[B, S, 3H] (q | k | v), ctx[B, S, H]; key j of sequence b is masked when
// mask[b*mask_stride + j] == 0 (an attention-mask input, or the token ids with stride S: [PAD] = 0); mask may be nullptr.
// Both launchers return cudaErrorInvalidValue for shapes outside attention_supported / layernorm_supported (nn_limits.h).
cudaError_t launch_attention(const float* qkv, const int* mask, int mask_stride, float* ctx, int Bn, int S, int H, int heads,
                             cudaStream_t s);
// The same under the causal rule: query i sees keys j <= i, a hidden key gets exactly zero weight, and the mask (may be
// nullptr) hides keys as above. cudaErrorInvalidValue outside attention_causal_supported (nn_limits.h).
cudaError_t launch_attention_causal(const float* qkv, const int* mask, int mask_stride, float* ctx, int Bn, int S, int H, int heads,
                                    cudaStream_t s);

// Classification head (head.cu): from logits[rows, n] writes, for each non-null pointer, row r of that output at
// ptr + r * ld (ld in 32-bit words): a copy of the logits [n], softmax probabilities [n], the argmax class as a
// little-endian int64 (two words: index, 0), the top k indices [k] (descending logit, ties to the lower index) and their
// probabilities [k] (the same bits as probabilities[index]). k counts only when a top-k pointer is set.
// cudaErrorInvalidValue outside head_supported (nn_limits.h).
struct HeadOutputs {
  float* logits = nullptr;
  int64_t logits_ld = 0;
  float* probs = nullptr;
  int64_t probs_ld = 0;
  int* classes = nullptr;
  int64_t classes_ld = 0;
  int* topk_idx = nullptr;
  int64_t topk_idx_ld = 0;
  float* topk_prob = nullptr;
  int64_t topk_prob_ld = 0;
};
cudaError_t launch_classify_head(const float* logits, int rows, int n, int k, const HeadOutputs& o, cudaStream_t s);

// Span head (span.cu): from per-token logits[rows, S, 2] (start, end interleaved) writes, for each non-null pointer, row r
// of that output at ptr + r * ld (ld in 32-bit words): start logits [S], end logits [S], and the k best answer spans --
// start indices [k], end indices [k] (int32) and scores start[i] + end[j] [k] (fp32) -- over the pairs of eligible tokens
// with i <= j < i + L, ordered by score descending, then i, then j ascending. Token p of row r is eligible when
// mask[q] != 0 (no mask: ids[q] != 0), types[q] == 1 and, with sep_id >= 0, ids[q] != sep_id, q = r * stride + p. Slots
// past the last candidate hold (-1, -1, -FLT_MAX). k and the inputs count only when a span pointer is set.
// cudaErrorInvalidValue outside span_supported (nn_limits.h).
struct SpanInputs {
  const int* ids = nullptr;
  const int* mask = nullptr;
  const int* types = nullptr;
  int64_t stride = 0;
  int sep_id = -1;
};
struct SpanOutputs {
  float* start_logits = nullptr;
  int64_t start_ld = 0;
  float* end_logits = nullptr;
  int64_t end_ld = 0;
  int* starts = nullptr;
  int64_t starts_ld = 0;
  int* ends = nullptr;
  int64_t ends_ld = 0;
  float* scores = nullptr;
  int64_t scores_ld = 0;
};
cudaError_t launch_span_head(const float* logits, const SpanInputs& in, int rows, int S, int L, int k, const SpanOutputs& o,
                             cudaStream_t s);

// Encoder head (encoder_head.cu): from the last hidden states hidden[rows, S, H] (and the pooler's pooled[rows, H]) writes,
// for each non-null pointer, row r of that output at ptr + r * ld (ld in 32-bit words): a copy of the hidden states [S, H],
// a copy of the pooler output [H], the hidden state of token 0 [H], and the masked mean sum_p m[p] h[p] / max(sum_p m[p],
// 1e-9) [H] with m[p] = mask[q] != 0 (no mask: ids[q] != 0), q = r * stride + p. normalize_cls / normalize_mean divide
// that output by max(||x||_2, 1e-12). The hidden states are read once; the sums run in an order fixed by S and H alone.
// cudaErrorInvalidValue outside encoder_head_supported (nn_limits.h).
struct EncoderInputs {
  const int* ids = nullptr;
  const int* mask = nullptr;
  int64_t stride = 0;
};
struct EncoderOutputs {
  float* sequence = nullptr;
  int64_t sequence_ld = 0;
  float* pooled = nullptr;
  int64_t pooled_ld = 0;
  float* cls = nullptr;
  int64_t cls_ld = 0;
  float* mean = nullptr;
  int64_t mean_ld = 0;
  bool normalize_cls = false, normalize_mean = false;
};
cudaError_t launch_encoder_head(const float* hidden, const float* pooled, const EncoderInputs& in, int rows, int S, int H,
                                const EncoderOutputs& o, cudaStream_t s);

// Fill-mask gather (mlm.cu): for each row r, the candidates are the tokens p < S with ids[q] == mask_token_id and, unless
// mask is nullptr, mask[q] != 0, q = r * stride + p. The first M of them in ascending p fill slots 0, 1, ...: positions[r * M
// + s] = p and gathered[r, s, :] = hidden[r, p, :] (a bit-exact copy); empty slots get -1 and zeros. Either output may be
// nullptr. cudaErrorInvalidValue outside mask_gather_supported (nn_limits.h).
cudaError_t launch_mask_gather(const float* hidden, const int* ids, const int* mask, int64_t stride, int rows, int S, int H,
                               int M, int mask_token_id, int* positions, float* gathered, cudaStream_t s);

// Fill-mask head (mlm.cu): slot s of row r reads the first `vocab` of the logits row logits + (r * M + s) * ld and, when
// positions[r * M + s] >= 0, writes at ptr + r * ld_out + s * k (ld_out in 32-bit words) the top k ids (descending logit,
// ties to the lower id), their softmax probabilities over the vocab logits (the same bits as launch_classify_head on that
// row) and their logits; an empty slot writes -1, 0 and -FLT_MAX. `positions_out` receives a copy of the positions [M] per
// row. k counts only when a top-k pointer is set. cudaErrorInvalidValue outside fill_mask_supported (nn_limits.h).
struct FillMaskOutputs {
  int* positions = nullptr;
  int64_t positions_ld = 0;
  int* ids = nullptr;
  int64_t ids_ld = 0;
  float* probs = nullptr;
  int64_t probs_ld = 0;
  float* logits = nullptr;
  int64_t logits_ld = 0;
};
// max_vocab is the cap to check: kHeadMaxN (fill_mask_supported), or kNextTokenMaxVocab with M = 1 (next_token_supported).
cudaError_t launch_fill_mask_head(const float* logits, int64_t ld, const int* positions, int rows, int M, int vocab, int k,
                                  int max_vocab, const FillMaskOutputs& o, cudaStream_t s);

// GPT-2 (gpt2.cu). Embedding without LayerNorm: y[b*S + s, :] = word[id, :] + pos[s, :], id = ids[b*stride + s] clamped to
// 0..vocab-1, one fp32 add. cudaErrorInvalidValue for stride < S or a null pointer.
cudaError_t launch_embed_positions(const int* ids, int64_t stride, const float* word, const float* pos, float* y, int rows, int S,
                                   int H, int vocab, cudaStream_t s);
// Last attended token: p = the largest position with mask[r*stride + p] != 0 (mask nullptr: S - 1; none: -1);
// positions[r] = p and gathered[r, :] = hidden[r, p, :] (a bit-exact copy; zeros for p = -1). Either output may be nullptr.
cudaError_t launch_last_token(const float* hidden, const int* mask, int64_t stride, int rows, int S, int H, int* positions,
                              float* gathered, cudaStream_t s);

// Greedy generation (generate.cu). KV cache write: kc[r, s, :] = qkv[r, s, H:2H] and vc[r, s, :] = qkv[r, s, 2H:3H] for
// s < S, caches [rows, T, H] (bit-exact copies).
cudaError_t launch_kv_cache_write(const float* qkv, float* kc, float* vc, int rows, int S, int T, int H, cudaStream_t s);
// Decode attention of one query per row: qkv [rows, 3H] is the step's q | k | v of the token at slot
// q_r = pos[r] + 1 + t. The query sees the cached keys j < q_r and its own key, except that a key j <= pos[r] whose prompt mask
// mask[r * mask_stride + j] is 0 gets the additive -10000 (mask may be nullptr). Writes ctx [rows, H] and appends this k and
// v at slot q_r of kc / vc [rows, T, H]. The keys are split over decode_attention_splits(S + t + 1) blocks, a function of S
// and t only, and combined in block order, so a row's bits do not depend on its batch. `work` holds
// decode_attention_work_bytes(rows, S + t + 1, H, heads) (nn_limits.h). cudaErrorInvalidValue outside
// decode_attention_supported(S + t + 1, H, heads), for S + t + 1 > T or mask_stride < S.
cudaError_t launch_decode_attention(const float* qkv, float* kc, float* vc, const int* pos, int t, const int* mask,
                                    int64_t mask_stride, int S, int T, float* ctx, int rows, int H, int heads, void* work,
                                    cudaStream_t s);
// One greedy step per row: from logits[r, :vocab] (ld >= vocab) the argmax g (ties to the lower id) and its log-probability
// logit[g] - logsumexp(logits[:vocab]). A row is live at t = 0 when pos[r] >= 0, later while done[r] == 0. A live row
// writes ids[t] = g, log_probs[t] and length = t + 1, and is done after g == eos (eos < 0: none); any other row writes
// -1 and 0 (and length 0 at t = 0). Unless `last`, every row writes the next step's input y[r, :] = word[g] + pos_table[
// pos[r] + 1 + t] (one fp32 add, as launch_embed_positions). Any output pointer may be nullptr; lds count 32-bit words.
struct GenerateOutputs {
  int* ids = nullptr;
  int64_t ids_ld = 0;
  float* log_probs = nullptr;
  int64_t log_probs_ld = 0;
  int* length = nullptr;
  int64_t length_ld = 0;
};
cudaError_t launch_generate_select(const float* logits, int64_t ld, int vocab, const int* pos, int t, bool last, int eos,
                                   int* done, const GenerateOutputs& o, const float* word, const float* pos_table, float* y,
                                   int rows, int H, cudaStream_t s);
// One sampled step per row: launch_generate_select with g drawn from the row's logits at temperature, top_k and top_p with
// the seed seeds[r * seed_stride] (DESIGN §3); top_k = 1 is the greedy token. The log-probability is the model's,
// logit[g] - logsumexp(logits[:vocab]), the bits launch_generate_select gives for the same g. A row's token depends on its
// logits' bits, seed and t only. cudaErrorInvalidValue outside sampling_supported (nn_limits.h) or for seed_stride < 1.
cudaError_t launch_generate_sample(const float* logits, int64_t ld, int vocab, const int* pos, int t, bool last, int eos,
                                   int* done, const GenerateOutputs& o, const float* word, const float* pos_table, float* y,
                                   int rows, int H, const int* seeds, int64_t seed_stride, float temperature, int top_k,
                                   float top_p, cudaStream_t s);
// One step of a processing bundle (DESIGN §3): launch_generate_select (seeds null) or launch_generate_sample with g chosen
// from the row's logits after the repetition penalty over its history, the no-repeat n-gram bans (ngram: 0 off) and the
// EOS ban while t < min_new. The history is the row's attended prompt ids, ids / mask [r * stride + j] for j <= pos[r]
// (mask null: every position), written to hist [r * hist_ld ..] and its length to hist_len0[r] at t = 0, then g_0 .. g_{t-1};
// the step appends g at hist[r * hist_ld + hist_len0[r] + t], so pos[r] + N <= hist_ld is the caller's to keep. The
// log-probability is the raw row's, the bits launch_generate_select gives for the same g. cudaErrorInvalidValue outside
// processing_supported (nn_limits.h), for min_new > 0 without an EOS id below vocab or, with seeds, outside sampling_supported.
cudaError_t launch_generate_process(const float* logits, int64_t ld, int vocab, const int* pos, int t, bool last, int eos,
                                    int* done, const GenerateOutputs& o, const float* word, const float* pos_table, float* y,
                                    int rows, int H, const int* ids, const int* mask, int64_t stride, int* hist, int64_t hist_ld,
                                    int* hist_len0, float penalty, int ngram, int min_new, const int* seeds, int64_t seed_stride,
                                    float temperature, int top_k, float top_p, cudaStream_t s);

// Scoring (score.cu). Token row i < n of logits[i * ld, +vocab) (ld >= vocab) is token g = first + i of a [rows, S] batch:
// row r = g / S, position p = g % S. When p is attended (mask[r * stride + p] != 0; mask nullptr: every position) and
// s = the smallest attended position above p exists, it writes, with t = ids[r * stride + s] clamped to [0, vocab),
// log_probs[r * S + s] = (z[t] - max z) - (float)log(sum_j expf(z[j] - max z)) (the sum in fp64, the select step's
// helpers and block size, so the bits of launch_generate_select's log-probability for g = t) and
// ranks[r * S + s] = #{j : z[j] > z[t]} + #{j < t : z[j] == z[t]}; it writes nothing else. cudaErrorInvalidValue outside
// score_supported (nn_limits.h), for stride < S or a null pointer.
cudaError_t launch_token_score(const float* logits, int64_t ld, int64_t first, int n, const int* ids, const int* mask,
                               int64_t stride, int S, int vocab, float* log_probs, int* ranks, cudaStream_t s);
// Score head: for each row r and position s of [rows, S], scored when s is attended and an attended position lies below it,
// writes at ptr + r * ld (ld in 32-bit words) token_log_probs[s] = log_probs[r * S + s] (0 unscored), token_ranks[s] =
// ranks[r * S + s] (-1 unscored), the fp64 sum of the scored log-probabilities in an order fixed by S, rounded once to fp32,
// and the number of scored positions. Reads log_probs / ranks at scored positions only. Any output pointer may be nullptr.
struct ScoreOutputs {
  float* log_probs = nullptr;
  int64_t log_probs_ld = 0;
  int* ranks = nullptr;
  int64_t ranks_ld = 0;
  float* sum = nullptr;
  int64_t sum_ld = 0;
  int* count = nullptr;
  int64_t count_ld = 0;
};
cudaError_t launch_score_head(const float* log_probs, const int* ranks, const int* mask, int64_t stride, int rows, int S,
                              const ScoreOutputs& o, cudaStream_t s);

// wgmma 3xTF32 version of launch_gemm (gemm_tc.cu) for M >= 64, N % 32 == 0, K >= 32, lda % 4 == 0
bool gemm_tc_supported(const float* A, const float* B, const float* bias, const float* R, const float* C, int M, int N, int K,
                       int lda);
cudaError_t launch_gemm_tc(const float* A, const float* B, const float* bias, const float* R, float* C, int M, int N, int K,
                           int lda, int act, cudaStream_t s);

// X6 (+ X7): batch gather / scatter as ONE kernel over a table of (src, dst, bytes) segments. A source / destination may be
// pinned host memory (zero-copy over PCIe: the client thread wrote it, no batcher-side memcpy, no staging copy), local HBM,
// or another GPU's forward window mapped through CUDA IPC (the forward hop a6: NVLink loads / stores inside this kernel).
struct CopySeg {
  const void* src;
  void* dst;
  uint64_t bytes;
};
cudaError_t launch_copy_segments(const CopySeg* segs, int n, cudaStream_t s);

// X4: implicit-GEMM convolution on the tensor cores (gemm_tc.cu): y[B,OH,OW,N] = act(conv(x[B,H,W,C], w[KH,KW,C,N]) + bias (+ R)); the A
// tiles are gathered from the NHWC activations by TMA im2col tensor maps -- no patch matrix in HBM. C % 32 == 0, N % 32 == 0.
bool conv_tc_supported(const float* x, const float* w, const float* bias, const float* R, const float* y, int Bn, int H, int W,
                       int C, int KH, int KW, int stride, int pad, int OH, int OW, int N);
cudaError_t launch_conv_tc(const float* x, const float* w, const float* bias, const float* R, float* y, int Bn, int H, int W, int C,
                           int KH, int KW, int stride, int pad, int OH, int OW, int N, int act, cudaStream_t s);

int64_t kernel_launch_count();

// streaming multiprocessors of the current device (132 on an H100 SXM), queried once per device
int device_sm_count();

}  // namespace tfsc
