// Model bundle description ("tfsc-b200-v1"): what the provider hands to the cache manager and
// what the executor runs. A bundle is <baseDir>/<name>/<version>/{tfsc_model.json, weights.bin};
// weights.bin is copied verbatim into pinned host memory and from there into the HBM arena, so
// offsets in the manifest are valid in all three places (256-byte aligned tensors).
#pragma once
#include <memory>
#include <string>
#include <vector>

#include "common.h"
#include "json.h"

namespace tfsc {

enum class Template { Affine, Mlp, Graph };

// One node of a "graph" bundle: activations are NHWC fp32, `src`/`dst`/`res` index scratch activation buffers (-1 = the
// request tensor, -2 = the response tensor). What each kind computes, its manifest name, shape rule, activations,
// residual and weights are in the op kind table (model.cc).
enum class OpKind { Conv, MaxPool, AvgPool, Dense, Embed, LayerNorm, Attention, MaskGather, DepthwiseConv, ChannelScale,
                    WindowAttention, PatchMerge, LastToken, TokenScore };
constexpr OpKind kLastOpKind = OpKind::TokenScore;
struct GraphOp {
  OpKind kind = OpKind::Conv;
  int src = -1, dst = 0, res = -100;  // res = -100: no residual input
  int gate = -100;                    // ChannelScale: the buffer holding the [c] gate of each image
  int window = 0, shift = 0;          // WindowAttention
  int h = 1, w = 1, c = 1;            // input H, W, C per image
  int kh = 1, kw = 1, stride = 1, pad = 0, cout = 1, oh = 1, ow = 1;
  int act = 0;                        // 0 none, 1 relu, 2 gelu(erf), 3 tanh, 4 relu6, 5 silu, 6 sigmoid, 7 gelu_tanh
  size_t w_off = 0, b_off = 0;        // kernel / bias; LayerNorm + Embed: gamma / beta
  // transformer ops (a "image" is a sequence: h = S tokens, w = 1, c = hidden width)
  int heads = 1, vocab = 0, max_pos = 0;
  size_t word_off = 0, pos_off = 0, type_off = 0;  // Embed tables [vocab,c], [max_pos,c], [2,c]
  float eps = 1e-12f;
  int64_t lda = 0;                    // Dense: elements per image of the source (> c selects the first token)
  int mask_token_id = 0;              // MaskGather (slots = oh)
  bool causal = false;                // Attention: query i sees keys j <= i
  bool norm = true;                   // Embed: LayerNorm after the sum (false: word + position only)
};

struct DenseLayer {
  int in = 0, out = 0;
  bool relu = false;
  size_t w_off = 0, b_off = 0;  // bytes into the blob; W row-major [in,out] fp32, b[out]
};

// classify / regress signatures of a model (tensorflow/serving/{classify,regress}): their input is a list of tf.Example,
// `feature` names the float feature that holds one input row per example (half_plus_two: "x")
struct ExtraSignature {
  std::string name;     // e.g. "regress_x_to_y"
  int method = 0;       // 1 = classify, 2 = regress
  std::string feature;
};

// One declared input of a multi-input graph bundle (signature.inputs): BERT's input_ids / input_mask / segment_ids, and a
// sampling generate bundle's per-request seed. New roles go at the end: the forward hop sends the enum's numbers.
enum class InputRole { Ids, Mask, TypeIds, Seed };
struct ModelInput {
  std::string name;
  InputRole role = InputRole::Ids;
  int64_t offset = 0;  // elements into the packed request row (inputs in byte-wise sorted name order, `width` values each)
  int64_t width = 0;   // values per row: input_width
};
// The one rule for how many int32 values per row an input of `role` holds in a bundle of S tokens: S, or 1 for a seed
inline int64_t input_width(InputRole role, int64_t S) { return role == InputRole::Seed ? 1 : S; }
// Sets the width (input_width) and offset of every input, in packed order, and returns the packed row's width
int64_t place_inputs(std::vector<ModelInput>* inputs, int64_t S);

// The head that computes a bundle's signature.outputs; every output of a bundle belongs to the same one (None: no outputs).
// Classify: the last op's N logits (head.cu). Span (question answering): the last op's [S, 1, 2] per-token start / end
// logits (span.cu). Encoder (embeddings): the last hidden states [S, 1, H] and the pooler's [H] (encoder_head.cu).
// FillMask (masked-language-model prediction): the [M, 1, Vp] vocabulary logits of the M [MASK] slots a mask_gather op
// selected (mlm.cu). NextToken (causal language-model prediction): the [1, 1, Vp] vocabulary logits of the one token a
// last_token op selected per row (the fill-mask head's kernel with one slot). Generate (greedy generation): a next-token
// bundle's graph run once on the prompt and then once per new token on a KV cache (generate.cu). Score (scoring the input):
// the log-probability and rank of every attended token under the logits of the attended position before it, which a
// token_score op computes in chunks of the vocabulary projection over all S tokens (score.cu).
enum class HeadKind { None, Classify, Span, Encoder, FillMask, NextToken, Generate, Score };

// One declared output of a multi-output bundle (signature.outputs). Its name, head, dtype and per-row shape are in the
// kind table (model.cc). New kinds go at the end: the forward hop sends the enum's numbers.
enum class OutputKind {
  Logits, Probabilities, Classes, TopKClasses, TopKProbabilities,
  StartLogits, EndLogits, SpanStarts, SpanEnds, SpanScores,
  SequenceOutput, PooledOutput, ClsEmbedding, MeanEmbedding,
  MaskedPositions, MaskedTopKIds, MaskedTopKProbabilities, MaskedTopKLogits,
  NextTokenPosition, NextTokenTopKIds, NextTokenTopKProbabilities, NextTokenTopKLogits,
  GeneratedIds, GeneratedLogProbs, GeneratedLength,
  TokenLogProbs, TokenRanks, TokenLogProbSum, TokenCount
};
constexpr OutputKind kLastOutputKind = OutputKind::TokenCount;
struct ModelOutput {
  std::string name;
  OutputKind kind = OutputKind::Logits;
  int64_t offset = 0;  // elements (32-bit words) into the packed response row (outputs in byte-wise sorted name order)
  int64_t width = 0;   // words per row (output_form)
};
const char* output_kind_name(OutputKind k);
int output_dtype(OutputKind k);  // TFSC_DT_FLOAT / TFSC_DT_INT64 / TFSC_DT_INT32
// What one row of an output kind looks like, the one rule behind the packed layout, every response writer and the
// metadata: `width` 32-bit words holding a scalar (rank 0: classes, one int64 in 2 words), a vector of dims[0] values
// (rank 1) or a dims[0] x dims[1] matrix (rank 2), in terms of the bundle's head_n / head_k (ModelDesc).
struct OutputForm {
  int64_t width = 0;
  int dtype = TFSC_DT_FLOAT;
  int rank = 1;
  int64_t dims[2] = {0, 0};
};
OutputForm output_form(OutputKind k, int head_n, int head_k);
constexpr int kMaxOutputs = 5;

struct ModelDesc {
  Template tmpl = Template::Mlp;
  std::vector<ExtraSignature> extra_sigs;
  std::vector<DenseLayer> layers;  // Mlp
  size_t a_off = 0, b_off = 0;     // Affine scalars
  size_t weights_bytes = 0;
  std::string input_name = "x", output_name = "y";
  // elements per batch row; 0 = elementwise / any shape (Affine)
  int64_t in_dim = 0, out_dim = 0;
  int max_width = 0;  // widest activation (for scratch sizing)
  // Graph
  std::vector<GraphOp> ops;
  int n_buffers = 0;
  int64_t buf_elems = 0;  // largest activation, elements per image
  int64_t col_elems = 0;  // largest im2col matrix, elements per image
  std::vector<int64_t> input_shape;   // per image, e.g. [224,224,3]
  std::vector<int64_t> output_shape;  // per image, e.g. [1000]
  int input_dtype = TFSC_DT_FLOAT;    // TFSC_DT_INT32 for token-id inputs (BERT)
  // signature.inputs, sorted by name (= packed row order); empty for single-input bundles (input_name, in_dim elements)
  std::vector<ModelInput> inputs;
  const ModelInput* input(InputRole r) const {
    for (auto& i : inputs)
      if (i.role == r) return &i;
    return nullptr;
  }
  // signature.outputs, sorted by name (= packed response row order); empty for single-output bundles (output_name, out_dim
  // elements). With outputs, out_dim is the packed row width, `head` the head that computes them, and head_n / head_k
  // the two numbers every output's row shape is given in (output_form), which the forward hop carries:
  //   Classify: head_n = N logits, head_k = the top-k k (0: no top-k output).
  //   Span:     head_n = S, head_k = the number of spans (0: logits only).
  //   Encoder:  head_n = H, head_k = S.
  //   FillMask: head_n = M (the mask_gather op's slots), head_k = k (0: masked_positions only).
  //   NextToken: head_n = vocab (the embed op's), head_k = k (0: next_token_position only).
  //   Generate: head_n = vocab (the embed op's), head_k = N (max_new_tokens).
  //   Score:    head_n = S, head_k = 0.
  // The rest is known to the owner only, the kernels' business: a span head's span_max_len = max_answer_length and
  // span_sep_id = sep_id (-1: none); an encoder head's encoder_pooler (the last op is the pooler: it writes pooled_output,
  // and the hidden states are its source buffer) and normalize_cls / normalize_mean; a fill-mask head's mlm_vocab (the
  // embed op's vocab, the logits the head reads of each Vp-wide row) and mlm_mask_token_id; a generate head's gen_eos
  // (eos_token_id, -1: none) and, on a sampling bundle (gen_sampling: a generate entry gave temperature, top_k or top_p),
  // gen_temperature (1), gen_top_k (0: off) and gen_top_p (1: off), and on a processing bundle (gen_processing: a generate
  // entry gave repetition_penalty, no_repeat_ngram_size or min_new_tokens) gen_repetition_penalty (1), gen_no_repeat_ngram
  // (0: off) and gen_min_new_tokens (0: off).
  std::vector<ModelOutput> outputs;
  HeadKind head = HeadKind::None;
  int head_n = 0, head_k = 0;
  int span_max_len = 0, span_sep_id = -1;
  bool encoder_pooler = false, normalize_cls = false, normalize_mean = false;
  int mlm_vocab = 0, mlm_mask_token_id = 0;
  int gen_eos = -1;
  bool gen_sampling = false;
  float gen_temperature = 1.f, gen_top_p = 1.f;
  int gen_top_k = 0;
  bool gen_processing = false;
  float gen_repetition_penalty = 1.f;
  int gen_no_repeat_ngram = 0, gen_min_new_tokens = 0;
  const ModelOutput* output(OutputKind k) const {
    for (auto& o : outputs)
      if (o.kind == k) return &o;
    return nullptr;
  }
  const ModelOutput* output(const std::string& name) const {
    for (auto& o : outputs)
      if (o.name == name) return &o;
    return nullptr;
  }
  // bytes of executor scratch (activation buffers + im2col) for `rows` images / batch rows
  size_t scratch_bytes(int64_t rows) const;
  // stride of the graph activation buffers in that scratch: rounded up to 256 bytes, so every buffer (and the im2col
  // matrix after them) starts 256-byte aligned whatever rows * buf_elems is
  size_t graph_buf_bytes(int64_t rows) const;
  // offset of the head's logits in that scratch (graph bundles with outputs: after the buffers and the im2col matrix)
  size_t head_scratch_offset(int64_t rows) const;
  // fill-mask and next-token bundles: offset of the mask_gather op's int32 positions [rows, M] (the last_token op's
  // [rows]) in that scratch, after the head's logits
  size_t mlm_positions_offset(int64_t rows) const;
  // generate bundles: the regions after the positions, for T = S + N - 1 cache slots. Attention op i (in op order) keeps
  // its K cache [rows, T, H] at kv + 2 i cache_bytes and its V cache right after it; then the decode attention work buffer
  // (decode_attention_work_bytes at T keys) and the int32 [rows] done flags; a processing bundle's int32 token histories
  // hist [rows, S + N] and their prompt lengths hist_len0 [rows] follow (0 on other bundles).
  // counter_bytes: the work buffer's leading int32 counters, the part that must be zero before a request's first step
  struct GenerateScratch {
    size_t kv = 0, cache_bytes = 0, work = 0, counter_bytes = 0, done = 0, hist = 0, hist_len0 = 0, end = 0;
  };
  GenerateScratch generate_scratch(int64_t rows) const;
  // score bundles: after the buffers, the token_score op's logits region for min(kScoreChunkTokens, rows * S) token rows of
  // Vp columns, then the fp32 log-probabilities and int32 ranks [rows, S] its score kernel writes and the head reads
  struct ScoreScratch {
    size_t logits = 0, log_probs = 0, ranks = 0, end = 0;
  };
  ScoreScratch score_scratch(int64_t rows) const;
};

// Set d->head from the first output's kind, sort d->outputs by name, set their offsets and widths from d->head_n / d->head_k
// and d->out_dim to the packed row width. Fails on a shape the head kernel cannot run (head_supported and its kin).
bool layout_outputs(ModelDesc* d, std::string* err);
// "'classes' (int64), 'logits' (float), ..." for error messages
std::string expected_outputs(const ModelDesc& d);

bool parse_manifest(const Json& j, ModelDesc* d, std::string* err);
ModelDesc make_mlp_desc(const std::vector<int>& dims, const std::vector<std::string>& activations);
ModelDesc make_affine_desc();
std::string manifest_json(const ModelDesc& d);

// A model held in the host tier (pinned memory when a CUDA device is present).
struct HostModel {
  ModelId id;
  ModelDesc desc;
  void* data = nullptr;
  size_t bytes = 0;
  std::function<void(void*, size_t)> release;  // returns the block to its pool
  ~HostModel() {
    if (data && release) release(data, bytes);
  }
};

}  // namespace tfsc
