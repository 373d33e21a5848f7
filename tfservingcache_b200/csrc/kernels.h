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

// X4/X5 building blocks (nn_kernels.cu): act 0 none / 1 relu / 2 gelu(erf) / 3 tanh / 4 relu6 / 5 silu / 6 sigmoid
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
cudaError_t launch_fill_mask_head(const float* logits, int64_t ld, const int* positions, int rows, int M, int vocab, int k,
                                  const FillMaskOutputs& o, cudaStream_t s);

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
