#include "model.h"

#include <algorithm>

#include "nn_limits.h"

namespace tfsc {

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

size_t ModelDesc::scratch_bytes(int64_t rows) const {
  // an mlp's head reads the last layer's logits from the activation buffer that layer would have used, so only graph
  // bundles with outputs need more: the last op's rows after the buffers and the im2col matrix (N logits per row for a
  // classify head, 2S per-token start / end logits for a span head)
  if (tmpl == Template::Mlp) return 2 * (((size_t)rows * (size_t)(max_width > 0 ? max_width : 1) * 4 + 255) & ~(size_t)255);
  if (tmpl == Template::Graph) {
    size_t last = 1;
    for (auto v : output_shape) last *= (size_t)v;
    // a fill-mask bundle's int32 [rows, M] positions follow the head's logits
    return head_scratch_offset(rows) + (outputs.empty() ? 0 : align256((size_t)rows * last * 4)) +
           (head == HeadKind::FillMask ? align256((size_t)rows * (size_t)head_n * 4) : 0);
  }
  return 256;
}

size_t ModelDesc::graph_buf_bytes(int64_t rows) const { return align256((size_t)rows * (size_t)buf_elems * 4); }

size_t ModelDesc::head_scratch_offset(int64_t rows) const {
  return (size_t)n_buffers * graph_buf_bytes(rows) + align256((size_t)rows * (size_t)col_elems * 4);
}

size_t ModelDesc::mlm_positions_offset(int64_t rows) const {
  size_t last = 1;
  for (auto v : output_shape) last *= (size_t)v;
  return head_scratch_offset(rows) + align256((size_t)rows * last * 4);
}

// ------------------------------------------------------------------------------------------------ output kinds ----
// A row of an output kind in the bundle's head_n / head_k (ModelDesc): one int64 scalar (2 words), a vector of head_n or
// head_k values, or a head_k x head_n / head_n x head_k matrix
enum class Rows { Int64, N, K, KxN, NxK };
// The entry fields a kind takes besides name and kind: "k"; "k", "max_answer_length" and "sep_id"; or "normalize"
enum class Fields { None, K, Span, Normalize };
struct OutputKindInfo {
  const char* name;
  HeadKind head;
  int dtype;
  Rows rows;
  Fields fields;
};
// One row per OutputKind, in enum order. head_n / head_k per head: see ModelDesc::outputs.
static constexpr OutputKindInfo kOutputKinds[] = {
    {"logits", HeadKind::Classify, TFSC_DT_FLOAT, Rows::N, Fields::None},
    {"probabilities", HeadKind::Classify, TFSC_DT_FLOAT, Rows::N, Fields::None},
    {"classes", HeadKind::Classify, TFSC_DT_INT64, Rows::Int64, Fields::None},
    {"top_k_classes", HeadKind::Classify, TFSC_DT_INT32, Rows::K, Fields::K},
    {"top_k_probabilities", HeadKind::Classify, TFSC_DT_FLOAT, Rows::K, Fields::K},
    {"start_logits", HeadKind::Span, TFSC_DT_FLOAT, Rows::N, Fields::None},
    {"end_logits", HeadKind::Span, TFSC_DT_FLOAT, Rows::N, Fields::None},
    {"span_starts", HeadKind::Span, TFSC_DT_INT32, Rows::K, Fields::Span},
    {"span_ends", HeadKind::Span, TFSC_DT_INT32, Rows::K, Fields::Span},
    {"span_scores", HeadKind::Span, TFSC_DT_FLOAT, Rows::K, Fields::Span},
    {"sequence_output", HeadKind::Encoder, TFSC_DT_FLOAT, Rows::KxN, Fields::None},
    {"pooled_output", HeadKind::Encoder, TFSC_DT_FLOAT, Rows::N, Fields::None},
    {"cls_embedding", HeadKind::Encoder, TFSC_DT_FLOAT, Rows::N, Fields::Normalize},
    {"mean_embedding", HeadKind::Encoder, TFSC_DT_FLOAT, Rows::N, Fields::Normalize},
    {"masked_positions", HeadKind::FillMask, TFSC_DT_INT32, Rows::N, Fields::None},
    {"masked_top_k_ids", HeadKind::FillMask, TFSC_DT_INT32, Rows::NxK, Fields::K},
    {"masked_top_k_probabilities", HeadKind::FillMask, TFSC_DT_FLOAT, Rows::NxK, Fields::K},
    {"masked_top_k_logits", HeadKind::FillMask, TFSC_DT_FLOAT, Rows::NxK, Fields::K},
};
static_assert(sizeof(kOutputKinds) / sizeof(kOutputKinds[0]) == (size_t)kLastOutputKind + 1, "one row per OutputKind");

static const OutputKindInfo& kind_info(OutputKind k) { return kOutputKinds[(int)k]; }
static bool takes_k(OutputKind k) { return kind_info(k).fields == Fields::K || kind_info(k).fields == Fields::Span; }

const char* output_kind_name(OutputKind k) { return kind_info(k).name; }
int output_dtype(OutputKind k) { return kind_info(k).dtype; }

OutputForm output_form(OutputKind k, int head_n, int head_k) {
  OutputForm f;
  f.dtype = kind_info(k).dtype;
  switch (kind_info(k).rows) {
    case Rows::Int64: f.width = 2, f.rank = 0, f.dims[0] = 1; break;
    case Rows::N: f.width = f.dims[0] = head_n; break;
    case Rows::K: f.width = f.dims[0] = head_k; break;
    case Rows::KxN: f.rank = 2, f.dims[0] = head_k, f.dims[1] = head_n, f.width = (int64_t)head_k * head_n; break;
    case Rows::NxK: f.rank = 2, f.dims[0] = head_n, f.dims[1] = head_k, f.width = (int64_t)head_n * head_k; break;
  }
  return f;
}

// the head of a bundle's outputs is the first one's (the loader refuses a mix)
static void set_head(ModelDesc* d) { d->head = d->outputs.empty() ? HeadKind::None : kind_info(d->outputs.front().kind).head; }

// a top-k or span result output: without one, a bundle's head_k must be 0
static bool declares_k(const ModelDesc& d) {
  for (auto& o : d.outputs)
    if (takes_k(o.kind)) return true;
  return false;
}

// Each head's limits on a row, checked by the loader on the bundle and by layout_outputs on what the forward hop carries
static bool classify_fits(int n, int k, bool with_k) { return head_supported(n, with_k ? k : 1) && (with_k || k == 0); }
static bool span_fits(int S, int L, int k, bool with_k) { return span_supported(S, with_k ? L : 1, with_k ? k : 1) && (with_k || k == 0); }
static bool fill_mask_fits(int M, int V, int k, bool with_k) { return fill_mask_supported(M, V, with_k ? k : 1) && (with_k || k == 0); }
static bool encoder_fits(int S, int H, std::string* err) {
  if (encoder_head_supported(S, H)) return true;
  *err = "signature.outputs: no encoder head kernel for S = " + std::to_string(S) + " and H = " + std::to_string(H) +
         " (1 <= S <= " + std::to_string(kEncoderMaxS) + ", 1 <= H <= " + std::to_string(kEncoderMaxH) + ")";
  return false;
}

bool layout_outputs(ModelDesc* d, std::string* err) {
  set_head(d);
  const bool with_k = declares_k(*d);
  switch (d->head) {
    case HeadKind::FillMask:  // vocab is the owner's business, so only M and k decide whether a row can be laid out
      if (!fill_mask_fits(d->head_n, kHeadMaxN, d->head_k, with_k)) {
        *err = "signature.outputs: no fill-mask head for M = " + std::to_string(d->head_n) + " slots and k = " +
               std::to_string(d->head_k) + " (1 <= M <= " + std::to_string(kMaskGatherMaxS) + ", 1 <= k <= " +
               std::to_string(kHeadMaxK) + ")";
        return false;
      }
      break;
    case HeadKind::Encoder:
      if (!encoder_fits(d->head_k, d->head_n, err)) return false;
      break;
    case HeadKind::Span:  // max_answer_length is the owner's business, so only S and k decide whether a row can be laid out
      if (!span_fits(d->head_n, 1, d->head_k, with_k)) {
        *err = "signature.outputs: no span kernel for S = " + std::to_string(d->head_n) + " and k = " + std::to_string(d->head_k) +
               " (1 <= S <= " + std::to_string(kSpanMaxS) + ", 1 <= k <= " + std::to_string(kSpanMaxK) + ")";
        return false;
      }
      break;
    default:
      if (!classify_fits(d->head_n, d->head_k, with_k)) {
        *err = "signature.outputs: no head kernel for " + std::to_string(d->head_n) + " logits and k = " + std::to_string(d->head_k) +
               " (1 <= N <= " + std::to_string(kHeadMaxN) + ", 1 <= k <= min(N, " + std::to_string(kHeadMaxK) + "))";
        return false;
      }
  }
  // the packed row holds the outputs in byte-wise name order, so a rank can split a response without the manifest
  std::sort(d->outputs.begin(), d->outputs.end(), [](const ModelOutput& a, const ModelOutput& b) { return a.name < b.name; });
  int64_t off = 0;
  for (auto& o : d->outputs) {
    o.offset = off;
    o.width = output_form(o.kind, d->head_n, d->head_k).width;
    off += o.width;
  }
  d->out_dim = off;
  return true;
}

std::string expected_outputs(const ModelDesc& d) {
  std::string s;
  for (auto& o : d.outputs) {
    if (!s.empty()) s += ", ";
    const int dt = output_dtype(o.kind);
    s += "'" + o.name + "' (" + (dt == TFSC_DT_INT64 ? "int64" : dt == TFSC_DT_INT32 ? "int32" : "float") + ")";
  }
  return s;
}

static void finish(ModelDesc* d) {
  if (d->tmpl == Template::Graph) {
    d->in_dim = 1;
    for (auto v : d->input_shape) d->in_dim *= v;
    if (!d->inputs.empty()) d->in_dim *= (int64_t)d->inputs.size();  // the packed row: S values per declared input
    d->out_dim = 1;
    for (auto v : d->output_shape) d->out_dim *= v;
    return;
  }
  if (d->tmpl == Template::Mlp) {
    d->in_dim = d->layers.front().in;
    d->out_dim = d->layers.back().out;
    d->max_width = 0;
    for (auto& l : d->layers) {
      if (l.in > d->max_width) d->max_width = l.in;
      if (l.out > d->max_width) d->max_width = l.out;
    }
  } else {
    d->in_dim = d->out_dim = 0;
  }
}

ModelDesc make_mlp_desc(const std::vector<int>& dims, const std::vector<std::string>& activations) {
  ModelDesc d;
  d.tmpl = Template::Mlp;
  size_t off = 0;
  for (size_t l = 0; l + 1 < dims.size(); ++l) {
    DenseLayer L;
    L.in = dims[l];
    L.out = dims[l + 1];
    if (!activations.empty()) L.relu = activations[l] == "relu";
    else L.relu = (l + 2 < dims.size());  // relu on all but the last layer
    L.w_off = off;
    off = align256(off + (size_t)L.in * L.out * 4);
    L.b_off = off;
    off = align256(off + (size_t)L.out * 4);
    d.layers.push_back(L);
  }
  d.weights_bytes = off;
  finish(&d);
  return d;
}

ModelDesc make_affine_desc() {
  ModelDesc d;
  d.tmpl = Template::Affine;
  d.a_off = 0;
  d.b_off = 256;
  d.weights_bytes = 512;
  finish(&d);
  return d;
}

// signature.outputs, one entry at a time. An entry is refused for, in this order: an unknown kind, no name, a duplicate, a
// mix of heads (fill-mask, then encoder, then span: the message names the later entry's head), a 'normalize' on a kind
// without one, and then the fields its head takes. Sets d->head.
static bool parse_outputs(const Json& outs, ModelDesc* d, std::string* err) {
  int k = -1, max_len = -1, sep_id = -1;
  bool span_seen = false;  // a span_starts / span_ends / span_scores entry set max_len and sep_id
  // an integer field of an output entry: 0 absent, 1 read into *v, -1 present but not an integer
  auto int_field = [](const Json& oj, const char* key, int* v) {
    const Json* f = oj.get(key);
    if (!f) return 0;
    if (f->type != Json::Num || f->num != (double)(int)f->num) return -1;
    *v = (int)f->num;
    return 1;
  };
  for (auto& oj : outs.arr) {
    ModelOutput mo;
    mo.name = oj.type == Json::Obj ? oj.get_str("name", "") : "";
    const std::string kind = oj.type == Json::Obj ? oj.get_str("kind", "") : "";
    const OutputKindInfo* ki = nullptr;
    for (auto& i : kOutputKinds)
      if (kind == i.name) ki = &i;
    if (!ki) {
      *err = "signature.outputs: unknown kind '" + kind + "' (";
      for (auto& i : kOutputKinds) *err += std::string(&i == kOutputKinds ? "" : ", ") + i.name;
      *err += ")";
      return false;
    }
    mo.kind = (OutputKind)(ki - kOutputKinds);
    if (mo.name.empty()) {
      *err = "signature.outputs: every output needs a name";
      return false;
    }
    for (auto& o : d->outputs)
      if (o.name == mo.name || o.kind == mo.kind) {
        *err = "signature.outputs: duplicate " + std::string(o.name == mo.name ? "name '" + mo.name + "'" : "kind '" + kind + "'");
        return false;
      }
    const HeadKind h = ki->head, first = d->outputs.empty() ? h : kind_info(d->outputs.front().kind).head;
    const std::string is = " ('" + mo.name + "' is " + kind + ")";
    if ((h == HeadKind::FillMask) != (first == HeadKind::FillMask)) {
      *err = "signature.outputs: fill-mask outputs (masked_positions, masked_top_k_ids, masked_top_k_probabilities,"
             " masked_top_k_logits) cannot be mixed with classification, span or encoder outputs" + is;
      return false;
    }
    if (h != HeadKind::FillMask) {
      if ((h == HeadKind::Encoder) != (first == HeadKind::Encoder)) {
        *err = "signature.outputs: encoder outputs (sequence_output, pooled_output, cls_embedding, mean_embedding) cannot be mixed"
               " with classification or span outputs" + is;
        return false;
      }
      if (const Json* nj = oj.get("normalize")) {
        if (ki->fields != Fields::Normalize) {
          *err = "signature.outputs: 'normalize' belongs to cls_embedding and mean_embedding" + is;
          return false;
        }
        if (nj->type != Json::Bool) {
          *err = "signature.outputs: '" + mo.name + "' has a 'normalize' that is not true or false";
          return false;
        }
        (mo.kind == OutputKind::ClsEmbedding ? d->normalize_cls : d->normalize_mean) = nj->b;
      }
      if (h != HeadKind::Encoder && (h == HeadKind::Span) != (first == HeadKind::Span)) {
        *err = "signature.outputs: span outputs (start_logits, end_logits, span_starts, span_ends, span_scores) cannot be mixed"
               " with classification outputs" + is;
        return false;
      }
    }
    const bool span_fields = oj.get("max_answer_length") || oj.get("sep_id");
    int v = 0;
    switch (h) {
      case HeadKind::FillMask:
        if (oj.get("normalize") || span_fields) {
          *err = "signature.outputs: 'normalize', 'max_answer_length' and 'sep_id' do not apply to fill-mask outputs" + is;
          return false;
        }
        if (!takes_k(mo.kind) && oj.get("k")) {
          *err = "signature.outputs: 'k' belongs to masked_top_k_ids, masked_top_k_probabilities and masked_top_k_logits" + is;
          return false;
        }
        if (takes_k(mo.kind) && (int_field(oj, "k", &v) != 1 || v < 1 || (k >= 0 && v != k))) {
          *err = "signature.outputs: '" + mo.name + "' needs an integer 'k' >= 1, the same for every fill-mask top-k output";
          return false;
        }
        if (takes_k(mo.kind)) k = v;
        break;
      case HeadKind::Encoder:
        if (oj.get("k") || span_fields) {
          *err = "signature.outputs: 'k', 'max_answer_length' and 'sep_id' do not apply to encoder outputs" + is;
          return false;
        }
        break;
      case HeadKind::Span:
        if (!takes_k(mo.kind)) {
          if (oj.get("k") || span_fields) {
            *err = "signature.outputs: 'k', 'max_answer_length' and 'sep_id' belong to span_starts, span_ends and span_scores" + is;
            return false;
          }
          break;
        }
        if (int_field(oj, "k", &v) != 1 || (span_seen && v != k)) {
          *err = "signature.outputs: '" + mo.name + "' needs an integer 'k', the same for every span output";
          return false;
        }
        k = v;
        if (int_field(oj, "max_answer_length", &v) != 1 || (span_seen && v != max_len)) {
          *err = "signature.outputs: '" + mo.name + "' needs an integer 'max_answer_length', the same for every span output";
          return false;
        }
        max_len = v;
        v = -1;
        if (const int r = int_field(oj, "sep_id", &v); r < 0 || (r == 1 && v < 0) || (span_seen && v != sep_id)) {
          *err = "signature.outputs: '" + mo.name + "' has a 'sep_id' that is not a token id >= 0 or differs from the other"
                 " span outputs' (give the same sep_id to every span output, or to none)";
          return false;
        }
        sep_id = v;
        span_seen = true;
        break;
      default:  // classification: 'k' on the top-k kinds only; max_answer_length and sep_id are ignored
        if (!takes_k(mo.kind) && oj.get("k")) {
          *err = "signature.outputs: 'k' belongs to the top-k outputs only" + is;
          return false;
        }
        if (takes_k(mo.kind) && (int_field(oj, "k", &v) != 1 || (k >= 0 && v != k))) {
          *err = "signature.outputs: '" + mo.name + "' needs an integer 'k', the same for both top-k outputs";
          return false;
        }
        if (takes_k(mo.kind)) k = v;
    }
    d->outputs.push_back(mo);
  }
  d->head_k = span_seen ? k : k < 0 ? 0 : k;  // a span k is always given, and a negative one is refused by span_fits
  d->span_max_len = span_seen ? max_len : 0;
  d->span_sep_id = sep_id;
  set_head(d);
  return true;
}

// ------------------------------------------------------------------- the bundle each head's outputs need ----
// The span, encoder and fill-mask heads read the request's ids / mask / segment ids where the embedding reads them
static bool embed_graph(const ModelDesc& d, const std::string& outputs, const char* bundle, std::string* err) {
  if (d.tmpl != Template::Graph) {
    *err = "signature.outputs: " + outputs + " outputs need a graph bundle (" + bundle + ")";
    return false;
  }
  if (d.ops.front().kind != OpKind::Embed) {
    *err = "signature.outputs: " + outputs + " outputs need a graph bundle whose first op is 'embed'";
    return false;
  }
  return true;
}

// the classify head reads the last op's (or the mlp's last layer's) N logits: head_n = N
static bool check_classify_bundle(ModelDesc* d, std::string* err) {
  if (d->tmpl == Template::Affine) {
    *err = "signature.outputs needs an mlp or graph bundle (an affine bundle has no logits row)";
    return false;
  }
  if (d->tmpl == Template::Graph && d->output_shape.size() != 1) {
    *err = "signature.outputs needs a graph whose output is one vector of logits per row (output_shape has rank " +
           std::to_string(d->output_shape.size()) + ")";
    return false;
  }
  d->head_n = d->out_dim > 0x7fffffff ? 0 : (int)d->out_dim;
  return true;
}

// the span head reads the per-token start / end logits [S, 1, 2] of the last op: head_n = S
static bool check_span_bundle(ModelDesc* d, std::string* err) {
  if (!embed_graph(*d, "span", "a BERT encoder ending in per-token start / end logits", err)) return false;
  if (!d->input(InputRole::TypeIds)) {
    *err = "signature.outputs: span outputs need a 'type_ids' input (the passage is segment 1)";
    return false;
  }
  const int S = d->ops.front().h;
  const GraphOp& last = d->ops.back();
  if (last.oh != S || last.ow != 1 || last.cout != 2) {
    *err = "signature.outputs: span outputs need a last op that writes [" + std::to_string(S) +
           ", 1, 2] start / end logits per token (it writes [" + std::to_string(last.oh) + ", " + std::to_string(last.ow) +
           ", " + std::to_string(last.cout) + "])";
    return false;
  }
  if (!span_fits(S, d->span_max_len, d->head_k, declares_k(*d))) {
    *err = "signature.outputs: no span kernel for S = " + std::to_string(S) + ", max_answer_length = " +
           std::to_string(d->span_max_len) + " and k = " + std::to_string(d->head_k) + " (1 <= S <= " +
           std::to_string(kSpanMaxS) + ", 1 <= max_answer_length <= S, 1 <= k <= " + std::to_string(kSpanMaxK) + ")";
    return false;
  }
  d->head_n = S;
  return true;
}

// the encoder head reads the last hidden states [S, 1, H]: what the last op writes, or, when the last op is the pooler (a
// tanh dense over token 0), its source buffer: head_n = H, head_k = S
static bool check_encoder_bundle(ModelDesc* d, std::string* err) {
  if (!embed_graph(*d, "encoder", "a BERT encoder ending in its hidden states or pooler", err)) return false;
  const int S = d->ops.front().h, H = d->ops.front().c;
  const GraphOp& last = d->ops.back();
  const GraphOp* prev = d->ops.size() >= 2 ? &d->ops[d->ops.size() - 2] : nullptr;
  const bool hidden = last.oh == S && last.ow == 1 && last.cout == H;
  const bool pooler = last.kind == OpKind::Dense && last.act == 3 && last.c == H && last.cout == H && last.src >= 0 &&
                      last.lda == (int64_t)S * H && prev && prev->dst == last.src && prev->oh == S && prev->ow == 1 &&
                      prev->cout == H;
  if (!hidden && !pooler) {
    const std::string sh = "[" + std::to_string(S) + ", 1, " + std::to_string(H) + "]";
    *err = "signature.outputs: encoder outputs need a last op that writes the " + sh + " hidden states, or a tanh pooler"
           " dense over token 0 of the " + sh + " hidden states the op before it writes (it writes [" +
           std::to_string(last.oh) + ", " + std::to_string(last.ow) + ", " + std::to_string(last.cout) + "])";
    return false;
  }
  d->encoder_pooler = pooler;
  if (d->output(OutputKind::PooledOutput) && !pooler) {
    *err = "signature.outputs: pooled_output needs a bundle whose last op is the pooler (a tanh dense over token 0)";
    return false;
  }
  if (!encoder_fits(S, H, err)) return false;
  d->head_n = H, d->head_k = S;
  return true;
}

// the fill-mask head: one mask_gather op reads the encoder's [S, 1, H] hidden states, the ops after it run on its M slots
// and the last one writes [M, 1, Vp] vocabulary logits: head_n = M
static bool check_fill_mask_bundle(ModelDesc* d, int gathers, std::string* err) {
  if (!embed_graph(*d, "fill-mask", "a BERT encoder, a mask_gather op and the MLM head", err)) return false;
  if (gathers != 1) {
    *err = "signature.outputs: fill-mask outputs need exactly one mask_gather op (the bundle has " + std::to_string(gathers) + ")";
    return false;
  }
  const GraphOp& emb = d->ops.front();
  const int S = emb.h, H = emb.c, V = emb.vocab;
  const GraphOp* g = nullptr;
  for (auto& o : d->ops)
    if (o.kind == OpKind::MaskGather) g = &o;
  const int M = g->oh;
  if (g->src < 0 || g->h != S || g->w != 1 || g->c != H) {
    *err = "signature.outputs: the mask_gather op needs the [" + std::to_string(S) + ", 1, " + std::to_string(H) +
           "] hidden states of a scratch buffer (it reads [" + std::to_string(g->h) + ", " + std::to_string(g->w) + ", " +
           std::to_string(g->c) + "] of buffer " + std::to_string(g->src) + ")";
    return false;
  }
  if (g->mask_token_id < 1 || g->mask_token_id >= V) {
    *err = "signature.outputs: mask_token_id " + std::to_string(g->mask_token_id) + " is not a token id in [1, " +
           std::to_string(V) + ")";
    return false;
  }
  const GraphOp& last = d->ops.back();
  if (last.oh != M || last.ow != 1 || last.cout < V) {
    *err = "signature.outputs: fill-mask outputs need a last op that writes [" + std::to_string(M) + ", 1, Vp] logits, Vp >= " +
           std::to_string(V) + " (it writes [" + std::to_string(last.oh) + ", " + std::to_string(last.ow) + ", " +
           std::to_string(last.cout) + "])";
    return false;
  }
  if (!mask_gather_supported(S, H, M) || !fill_mask_fits(M, V, d->head_k, declares_k(*d))) {
    *err = "signature.outputs: no fill-mask kernels for S = " + std::to_string(S) + ", H = " + std::to_string(H) + ", M = " +
           std::to_string(M) + ", vocab = " + std::to_string(V) + " and k = " + std::to_string(d->head_k) + " (1 <= M <= S <= " +
           std::to_string(kMaskGatherMaxS) + ", H <= " + std::to_string(kMaskGatherMaxH) + ", 1 <= vocab <= " +
           std::to_string(kHeadMaxN) + ", 1 <= k <= min(vocab, " + std::to_string(kHeadMaxK) + "))";
    return false;
  }
  d->mlm_vocab = V;
  d->mlm_mask_token_id = g->mask_token_id;
  d->head_n = M;
  return true;
}

bool parse_manifest(const Json& j, ModelDesc* d, std::string* err) {
  if (j.type != Json::Obj) {
    *err = "manifest is not a JSON object";
    return false;
  }
  if (j.get_str("format", "") != "tfsc-b200-v1") {
    *err = "unsupported manifest format '" + j.get_str("format", "") + "'";
    return false;
  }
  if (j.get_str("dtype", "float32") != "float32") {
    *err = "only float32 bundles are supported";
    return false;
  }
  if (const Json* sig = j.get("signature")) {
    d->input_name = sig->get_str("input", "x");
    d->output_name = sig->get_str("output", "y");
    if (const Json* ins = sig->get("inputs")) {
      if (sig->get("input")) {
        *err = "signature: 'inputs' and 'input' are mutually exclusive";
        return false;
      }
      if (ins->type != Json::Arr || ins->arr.empty() || ins->arr.size() > 3) {
        *err = "signature.inputs must list 1 to 3 inputs";
        return false;
      }
      for (auto& ij : ins->arr) {
        ModelInput mi;
        mi.name = ij.get_str("name", "");
        const std::string role = ij.get_str("role", "");
        if (role == "ids") mi.role = InputRole::Ids;
        else if (role == "mask") mi.role = InputRole::Mask;
        else if (role == "type_ids") mi.role = InputRole::TypeIds;
        else {
          *err = "signature.inputs: unknown role '" + role + "' (ids, mask, type_ids)";
          return false;
        }
        if (mi.name.empty()) {
          *err = "signature.inputs: every input needs a name";
          return false;
        }
        for (auto& o : d->inputs)
          if (o.name == mi.name || o.role == mi.role) {
            *err = "signature.inputs: duplicate " + std::string(o.name == mi.name ? "name '" + mi.name + "'" : "role '" + role + "'");
            return false;
          }
        d->inputs.push_back(mi);
      }
      if (!d->input(InputRole::Ids)) {
        *err = "signature.inputs: no input has the role 'ids'";
        return false;
      }
      // the packed row holds the inputs in byte-wise name order, so a rank can pack a request without the manifest
      std::sort(d->inputs.begin(), d->inputs.end(), [](const ModelInput& a, const ModelInput& b) { return a.name < b.name; });
      d->input_name = d->input(InputRole::Ids)->name;
    }
    if (const Json* outs = sig->get("outputs")) {
      if (sig->get("output")) {
        *err = "signature: 'outputs' and 'output' are mutually exclusive";
        return false;
      }
      if (outs->type != Json::Arr || outs->arr.empty() || outs->arr.size() > (size_t)kMaxOutputs) {
        *err = "signature.outputs must list 1 to " + std::to_string(kMaxOutputs) + " outputs";
        return false;
      }
      if (!parse_outputs(*outs, d, err)) return false;
    }
  }
  if (const Json* ex = j.get("extra_signatures")) {
    for (auto& e : ex->arr) {
      ExtraSignature g;
      g.name = e.get_str("name", "");
      const std::string m = e.get_str("method", "");
      g.method = m == "classify" ? 1 : m == "regress" ? 2 : 0;
      g.feature = e.get_str("feature", d->input_name);
      if (g.name.empty() || g.method == 0) {
        *err = "extra_signatures entries need a name and method classify|regress";
        return false;
      }
      d->extra_sigs.push_back(g);
    }
  }
  d->weights_bytes = (size_t)j.get_int("weights_bytes", 0);
  std::string t = j.get_str("template", "");
  if (t == "affine") {
    d->tmpl = Template::Affine;
    d->a_off = (size_t)j.get_int("a_offset", 0);
    d->b_off = (size_t)j.get_int("b_offset", 256);
    if (d->a_off + 4 > d->weights_bytes || d->b_off + 4 > d->weights_bytes || (d->a_off & 3) || (d->b_off & 3)) {
      *err = "affine offsets out of range";
      return false;
    }
  } else if (t == "mlp") {
    d->tmpl = Template::Mlp;
    const Json* layers = j.get("layers");
    if (!layers || layers->type != Json::Arr || layers->arr.empty()) {
      *err = "mlp manifest needs a non-empty 'layers' array";
      return false;
    }
    int prev_out = -1;
    for (auto& lj : layers->arr) {
      DenseLayer L;
      L.in = (int)lj.get_int("in", 0);
      L.out = (int)lj.get_int("out", 0);
      L.relu = lj.get_str("activation", "linear") == "relu";
      L.w_off = (size_t)lj.get_int("w_offset", -1);
      L.b_off = (size_t)lj.get_int("b_offset", -1);
      if (L.in <= 0 || L.out <= 0 || (L.w_off & 255) || (L.b_off & 255) ||
          L.w_off + (size_t)L.in * L.out * 4 > d->weights_bytes || L.b_off + (size_t)L.out * 4 > d->weights_bytes) {
        *err = "mlp layer out of range or misaligned";
        return false;
      }
      if (prev_out >= 0 && prev_out != L.in) {
        *err = "mlp layer dims do not chain";
        return false;
      }
      prev_out = L.out;
      d->layers.push_back(L);
    }
  } else if (t == "graph") {
    d->tmpl = Template::Graph;
    const Json* ops = j.get("ops");
    const Json* ish = j.get("input_shape");
    if (!ops || ops->type != Json::Arr || ops->arr.empty() || !ish || ish->type != Json::Arr) {
      *err = "graph manifest needs 'ops' and 'input_shape'";
      return false;
    }
    for (auto& v : ish->arr) d->input_shape.push_back(v.integer());
    d->input_dtype = j.get_str("input_dtype", "float32") == "int32" ? TFSC_DT_INT32 : TFSC_DT_FLOAT;
    d->n_buffers = (int)j.get_int("n_buffers", 0);
    if (d->n_buffers < 1 || d->n_buffers > 16) {
      *err = "graph manifest: n_buffers out of range";
      return false;
    }
    int64_t in_elems = 1;
    for (auto v : d->input_shape) in_elems *= v;
    std::vector<int64_t> written(d->n_buffers, -1);  // elements per image held by each scratch buffer
    int64_t out_elems = -1;
    for (auto& oj : ops->arr) {
      GraphOp o;
      const std::string kind = oj.get_str("op", "");
      if (kind == "conv") o.kind = OpKind::Conv;
      else if (kind == "maxpool") o.kind = OpKind::MaxPool;
      else if (kind == "avgpool") o.kind = OpKind::AvgPool;
      else if (kind == "dense") o.kind = OpKind::Dense;
      else if (kind == "embed") o.kind = OpKind::Embed;
      else if (kind == "layernorm") o.kind = OpKind::LayerNorm;
      else if (kind == "attention") o.kind = OpKind::Attention;
      else if (kind == "mask_gather") o.kind = OpKind::MaskGather;
      else if (kind == "depthwise_conv") o.kind = OpKind::DepthwiseConv;
      else if (kind == "channel_scale") o.kind = OpKind::ChannelScale;
      else if (kind == "window_attention") o.kind = OpKind::WindowAttention;
      else if (kind == "patch_merge") o.kind = OpKind::PatchMerge;
      else {
        *err = "graph manifest: unknown op '" + kind + "'";
        return false;
      }
      o.src = (int)oj.get_int("src", -1);
      o.dst = (int)oj.get_int("dst", 0);
      o.res = (int)oj.get_int("res", -100);
      o.h = (int)oj.get_int("h", 1);
      o.w = (int)oj.get_int("w", 1);
      o.c = (int)oj.get_int("c", 1);
      o.kh = (int)oj.get_int("kh", 1);
      o.kw = (int)oj.get_int("kw", 1);
      o.stride = (int)oj.get_int("stride", 1);
      o.pad = (int)oj.get_int("pad", 0);
      o.cout = (int)oj.get_int("cout", o.c);
      const std::string act = oj.get_str("act", "none");
      o.act = act == "relu" ? 1 : act == "gelu" ? 2 : act == "tanh" ? 3 : act == "relu6" ? 4 : act == "silu" ? 5 : act == "sigmoid" ? 6 : 0;
      // the older ops read an unknown act string as none; the depthwise and gate ops refuse it
      if (o.kind == OpKind::DepthwiseConv && !(act == "none" || o.act == 1 || o.act >= 4)) {
        *err = "graph manifest: depthwise_conv act '" + act + "' is not none, relu, relu6, silu or sigmoid";
        return false;
      }
      if ((o.kind == OpKind::ChannelScale || o.kind == OpKind::WindowAttention || o.kind == OpKind::PatchMerge) && act != "none") {
        *err = "graph manifest: " + kind + " takes no activation (act '" + act + "')";
        return false;
      }
      o.heads = (int)oj.get_int("heads", 1);
      o.vocab = (int)oj.get_int("vocab", 0);
      o.max_pos = (int)oj.get_int("max_pos", 0);
      o.word_off = (size_t)oj.get_int("word_offset", 0);
      o.pos_off = (size_t)oj.get_int("pos_offset", 0);
      o.type_off = (size_t)oj.get_int("type_offset", 0);
      o.eps = (float)oj.get_num("eps", 1e-12);
      o.w_off = (size_t)oj.get_int("w_offset", 0);
      o.b_off = (size_t)oj.get_int("b_offset", 0);
      if (o.kind == OpKind::MaskGather) {
        o.oh = (int)oj.get_int("slots", 0);
        o.mask_token_id = (int)oj.get_int("mask_token_id", 0);
      }
      if (o.h < 1 || o.w < 1 || o.c < 1 || o.kh < 1 || o.kw < 1 || o.stride < 1 || o.pad < 0 || o.cout < 1) {
        *err = "graph manifest: bad op geometry";
        return false;
      }
      if (o.kind == OpKind::Embed || o.kind == OpKind::LayerNorm) {
        o.oh = o.h;
        o.ow = o.w;
        o.cout = o.c;
        if (!layernorm_supported(o.c)) {
          *err = "graph manifest: no LayerNorm kernel for hidden " + std::to_string(o.c) + " (at most 12272)";
          return false;
        }
      } else if (o.kind == OpKind::Attention) {
        o.oh = o.h;
        o.ow = o.w;
        o.cout = o.c / 3;
        if (o.c % 3 || o.heads < 1 || o.cout % o.heads || o.w != 1) {
          *err = "graph manifest: attention expects a packed [S,1,3H] qkv source";
          return false;
        }
        // the executor's scratch buffers are 256-byte aligned (graph_buf_bytes); the request input (src -1) and the response
        // (dst -2) may be any caller pointer, so an op that reads or writes those must run without the aligned kernels
        if (!attention_supported(o.h, o.cout, o.heads, o.src >= 0 && o.dst >= 0)) {
          *err = "graph manifest: no attention kernel for S = " + std::to_string(o.h) + ", hidden " + std::to_string(o.cout) + ", " +
                 std::to_string(o.heads) + " heads (head width d % 4 == 0 and d <= 128 runs at every S; other widths only while"
                 " K and V of a head fit in shared memory)";
          return false;
        }
      } else if (o.kind == OpKind::MaskGather) {
        // [S, 1, H] -> [M, 1, H]; the shapes are checked with the fill-mask outputs below
        o.ow = 1;
        o.cout = o.c;
        if (o.oh < 1 || o.oh > o.h) {
          *err = "graph manifest: mask_gather needs 1 <= slots <= h (slots = " + std::to_string(o.oh) + ", h = " +
                 std::to_string(o.h) + ")";
          return false;
        }
      } else if (o.kind == OpKind::AvgPool) {
        o.oh = o.ow = 1;
        o.cout = o.c;
      } else if (o.kind == OpKind::ChannelScale) {
        o.oh = o.h;
        o.ow = o.w;
        o.cout = o.c;
        o.gate = (int)oj.get_int("gate", -100);
        if (o.res != -100) {
          *err = "graph manifest: channel_scale takes no residual input";
          return false;
        }
      } else if (o.kind == OpKind::DepthwiseConv) {
        if (o.cout != o.c) {
          *err = "graph manifest: depthwise_conv writes its c = " + std::to_string(o.c) + " channels (cout " + std::to_string(o.cout) + ")";
          return false;
        }
        if (o.res != -100) {
          *err = "graph manifest: depthwise_conv takes no residual input";
          return false;
        }
        if (!depthwise_supported(o.h, o.w, o.c, o.kh, o.kw, o.stride, o.pad)) {
          *err = "graph manifest: no depthwise_conv kernel for " + std::to_string(o.h) + " x " + std::to_string(o.w) + " x " +
                 std::to_string(o.c) + ", kernel " + std::to_string(o.kh) + " x " + std::to_string(o.kw) + ", stride " +
                 std::to_string(o.stride) + ", pad " + std::to_string(o.pad) + " (kernel <= " + std::to_string(kDepthwiseMaxK) +
                 ", stride <= " + std::to_string(kDepthwiseMaxStride) + ", pad <= kernel / 2, h * w * c < 2^31)";
          return false;
        }
        o.oh = (o.h + 2 * o.pad - o.kh) / o.stride + 1;
        o.ow = (o.w + 2 * o.pad - o.kw) / o.stride + 1;
      } else if (o.kind == OpKind::WindowAttention) {
        o.oh = o.h;
        o.ow = o.w;
        o.cout = o.c / 3;
        o.window = (int)oj.get_int("window", 0);
        o.shift = (int)oj.get_int("shift", 0);
        o.b_off = (size_t)oj.get_int("bias_offset", 0);
        const std::string at = " (h x w = " + std::to_string(o.h) + " x " + std::to_string(o.w) + ", window " + std::to_string(o.window);
        if (o.c % 3) {
          *err = "graph manifest: window_attention expects a packed [h, w, 3C] qkv source (c = " + std::to_string(o.c) + ")";
          return false;
        }
        if (o.heads < 1 || o.cout % o.heads) {
          *err = "graph manifest: window_attention needs heads that divide C = " + std::to_string(o.cout) + " (heads " +
                 std::to_string(o.heads) + ")";
          return false;
        }
        // torchvision zero-pads a map that is not a multiple of the window before the qkv projection, so its padded
        // tokens are keys with k = the qkv bias: not served
        if (o.window >= 1 && (o.h % o.window || o.w % o.window)) {
          *err = "graph manifest: window_attention needs a feature map that is a multiple of the window" + at + ")";
          return false;
        }
        if (o.window >= 1 && (o.shift < 0 || o.shift >= o.window)) {
          *err = "graph manifest: window_attention shift " + std::to_string(o.shift) + " is outside [0, window)" + at + ")";
          return false;
        }
        if (!window_attention_supported(o.h, o.w, o.cout, o.heads, o.window, o.shift)) {
          *err = "graph manifest: no window_attention kernel for C = " + std::to_string(o.cout) + ", " + std::to_string(o.heads) +
                 " heads" + at + ", shift " + std::to_string(o.shift) + ") (window <= " + std::to_string(kWindowMaxWs) +
                 ", head width <= " + std::to_string(kWindowMaxD) + ", K and V of a window within 48 KB, h * w * 3C < 2^31)";
          return false;
        }
        if (o.res != -100) {
          *err = "graph manifest: window_attention takes no residual input";
          return false;
        }
        const size_t n = (size_t)o.window * o.window;
        if ((o.b_off & 255) || o.b_off + (size_t)o.heads * n * n * 4 > d->weights_bytes) {
          *err = "graph manifest: window_attention bias table out of range or not 256-byte aligned";
          return false;
        }
      } else if (o.kind == OpKind::PatchMerge) {
        o.oh = o.h / 2;
        o.ow = o.w / 2;
        if (o.h % 2 || o.w % 2) {
          *err = "graph manifest: patch_merge needs an even h and w (h x w = " + std::to_string(o.h) + " x " + std::to_string(o.w) + ")";
          return false;
        }
        if (oj.get("cout") && o.cout != 4 * o.c) {
          *err = "graph manifest: patch_merge writes 4c = " + std::to_string(4 * o.c) + " channels (cout " + std::to_string(o.cout) + ")";
          return false;
        }
        o.cout = 4 * o.c;
        if (o.res != -100) {
          *err = "graph manifest: patch_merge takes no residual input";
          return false;
        }
        if (!patch_merge_supported(o.h, o.w, o.c)) {
          *err = "graph manifest: no patch_merge kernel for " + std::to_string(o.h) + " x " + std::to_string(o.w) + " x " +
                 std::to_string(o.c) + " (h * w * c < 2^31)";
          return false;
        }
      } else if (o.kind == OpKind::Dense) {
        o.oh = o.ow = 1;
        o.kh = o.kw = 1;
      } else {
        o.oh = (o.h + 2 * o.pad - o.kh) / o.stride + 1;
        o.ow = (o.w + 2 * o.pad - o.kw) / o.stride + 1;
        if (o.kind == OpKind::MaxPool) o.cout = o.c;
      }
      const int64_t in_e = o.kind == OpKind::Embed ? (int64_t)o.h * o.w : (int64_t)o.h * o.w * o.c;
      const int64_t out_e = (int64_t)o.oh * o.ow * o.cout;
      auto buf_ok = [&](int b) { return b == -1 || (b >= 0 && b < d->n_buffers); };
      if (!buf_ok(o.src) || !(o.dst == -2 || (o.dst >= 0 && o.dst < d->n_buffers)) || (o.res != -100 && !buf_ok(o.res)) ||
          o.dst == o.src || o.dst == o.res) {
        *err = "graph manifest: bad buffer index";
        return false;
      }
      const int64_t have = o.src == -1 ? in_elems : written[o.src];
      o.lda = have;
      if (o.kind == OpKind::ChannelScale) {
        if (o.gate == o.dst) {
          *err = "graph manifest: channel_scale cannot write its gate buffer (gate == dst == " + std::to_string(o.dst) + ")";
          return false;
        }
        if (o.gate < 0 || o.gate >= d->n_buffers || written[o.gate] != o.c) {
          *err = "graph manifest: channel_scale needs a gate that an earlier op wrote to a scratch buffer with c = " +
                 std::to_string(o.c) + " values per image (gate " + std::to_string(o.gate) + ")";
          return false;
        }
        if (have != in_e) {
          *err = "graph manifest: channel_scale reads " + std::to_string(have) + " values per image, not h * w * c = " +
                 std::to_string(in_e);
          return false;
        }
      }
      const bool size_ok = o.kind == OpKind::Dense ? have >= in_e : have == in_e;  // Dense may read the first token only
      if (o.kind == OpKind::Embed && (o.src != -1 || o.vocab < 1 || o.max_pos < o.h || (o.word_off & 255) || (o.pos_off & 255) ||
                                      (o.type_off & 255) || o.word_off + (size_t)o.vocab * o.c * 4 > d->weights_bytes ||
                                      o.pos_off + (size_t)o.max_pos * o.c * 4 > d->weights_bytes ||
                                      o.type_off + (size_t)2 * o.c * 4 > d->weights_bytes)) {
        *err = "graph manifest: bad embed op";
        return false;
      }
      if ((o.kind == OpKind::Embed || o.kind == OpKind::LayerNorm) &&
          ((o.w_off & 255) || (o.b_off & 255) || o.w_off + (size_t)o.c * 4 > d->weights_bytes || o.b_off + (size_t)o.c * 4 > d->weights_bytes)) {
        *err = "graph manifest: LayerNorm gamma/beta out of range";
        return false;
      }
      if (!size_ok || (o.res != -100 && (o.res == -1 ? in_elems : written[o.res]) != out_e)) {
        *err = "graph manifest: op input size does not match its producer";
        return false;
      }
      if (o.kind == OpKind::Conv || o.kind == OpKind::Dense || o.kind == OpKind::DepthwiseConv) {
        const size_t wbytes = (size_t)o.kh * o.kw * o.c * (o.kind == OpKind::DepthwiseConv ? 1 : o.cout) * 4;
        if ((o.w_off & 255) || (o.b_off & 255) || o.w_off + wbytes > d->weights_bytes || o.b_off + (size_t)o.cout * 4 > d->weights_bytes) {
          *err = "graph manifest: weights out of range or misaligned";
          return false;
        }
        const bool direct = o.kh == 1 && o.kw == 1 && o.stride == 1 && o.pad == 0;
        if (!direct && o.kind != OpKind::DepthwiseConv) {
          const int64_t ldc = ((int64_t)o.kh * o.kw * o.c + 3) / 4 * 4;
          d->col_elems = std::max<int64_t>(d->col_elems, (int64_t)o.oh * o.ow * ldc);
        }
      }
      if (o.dst == -2) out_elems = out_e;
      else {
        written[o.dst] = out_e;
        d->buf_elems = std::max<int64_t>(d->buf_elems, out_e);
      }
      d->ops.push_back(o);
    }
    if (out_elems < 0 || d->ops.back().dst != -2) {
      *err = "graph manifest: the last op must write the response (dst = -2)";
      return false;
    }
    d->output_shape.clear();
    const GraphOp& last = d->ops.back();
    if (last.oh * last.ow > 1) {
      d->output_shape.push_back(last.oh);
      d->output_shape.push_back(last.ow);
    }
    d->output_shape.push_back(last.cout);
  } else {
    *err = "unknown template '" + t + "'";
    return false;
  }
  if (!d->inputs.empty()) {
    // several inputs feed the embedding (ids, segment ids) and attention (mask) only: every other op reads scratch buffers
    bool ok = d->tmpl == Template::Graph && d->ops.front().kind == OpKind::Embed;
    for (size_t i = 1; ok && i < d->ops.size(); ++i) ok = d->ops[i].src != -1 && d->ops[i].res != -1;
    if (!ok) {
      *err = "signature.inputs needs a graph bundle whose first op is 'embed' and the only op that reads the request";
      return false;
    }
    if (d->input_dtype != TFSC_DT_INT32) {
      *err = "signature.inputs needs input_dtype int32";
      return false;
    }
    const int64_t S = d->ops.front().h;
    for (size_t i = 0; i < d->inputs.size(); ++i) d->inputs[i].offset = (int64_t)i * S;
  }
  finish(d);
  int gathers = 0;
  for (auto& o : d->ops) gathers += o.kind == OpKind::MaskGather;
  if (gathers && d->head != HeadKind::FillMask) {
    *err = "graph manifest: a mask_gather op needs fill-mask outputs (masked_positions, masked_top_k_ids, "
           "masked_top_k_probabilities, masked_top_k_logits)";
    return false;
  }
  if (d->outputs.empty()) return true;
  bool ok = false;
  switch (d->head) {
    case HeadKind::FillMask: ok = check_fill_mask_bundle(d, gathers, err); break;
    case HeadKind::Encoder: ok = check_encoder_bundle(d, err); break;
    case HeadKind::Span: ok = check_span_bundle(d, err); break;
    default: ok = check_classify_bundle(d, err);
  }
  if (!ok) return false;
  for (auto& o : d->outputs) {
    bool clash = d->inputs.empty() && o.name == d->input_name;
    for (auto& i : d->inputs) clash = clash || o.name == i.name;
    if (clash) {
      *err = "signature.outputs: '" + o.name + "' is also an input name";
      return false;
    }
  }
  return layout_outputs(d, err);
}

}  // namespace tfsc

// Offline manifest check (no device): the loader's verdict on a tfsc_model.json and the packed row layout it derives.
extern "C" int tfsc_manifest_check(const char* manifest_json, char* buf, size_t cap) {
  using namespace tfsc;
  Json j;
  ModelDesc d;
  std::string err;
  if (!manifest_json || !json_parse(manifest_json, &j, &err) || !parse_manifest(j, &d, &err))
    return fail(TFSC_E_INVALID, "%s", err.empty() ? "manifest_check: no manifest" : err.c_str());
  std::string s = "{\"in_dim\": " + std::to_string(d.in_dim) + ", \"out_dim\": " + std::to_string(d.out_dim) +
                  ", \"head_n\": " + std::to_string(d.head_n) + ", \"head_k\": " + std::to_string(d.head_k) + ", \"outputs\": [";
  for (size_t i = 0; i < d.outputs.size(); ++i) {
    const ModelOutput& o = d.outputs[i];
    const int dt = output_dtype(o.kind);
    s += i ? ", {\"name\": " : "{\"name\": ";
    json_escape(o.name, &s);
    s += ", \"kind\": \"" + std::string(output_kind_name(o.kind)) + "\", \"offset\": " + std::to_string(o.offset) +
         ", \"width\": " + std::to_string(o.width) + ", \"dtype\": \"" +
         (dt == TFSC_DT_INT64 ? "int64" : dt == TFSC_DT_INT32 ? "int32" : "float32") + "\"}";
  }
  s += "]}";
  return copy_out(s, buf, cap);
}

namespace tfsc {

std::string manifest_json(const ModelDesc& d) {
  std::string s = "{\"format\":\"tfsc-b200-v1\",\"dtype\":\"float32\",\"signature\":{\"input\":";
  json_escape(d.input_name, &s);
  s += ",\"output\":";
  json_escape(d.output_name, &s);
  s += "},\"weights_bytes\":" + std::to_string(d.weights_bytes);
  if (d.tmpl == Template::Affine) {
    s += ",\"template\":\"affine\",\"a_offset\":" + std::to_string(d.a_off) + ",\"b_offset\":" + std::to_string(d.b_off);
  } else {
    s += ",\"template\":\"mlp\",\"layers\":[";
    for (size_t i = 0; i < d.layers.size(); ++i) {
      auto& L = d.layers[i];
      if (i) s += ",";
      s += "{\"in\":" + std::to_string(L.in) + ",\"out\":" + std::to_string(L.out) + ",\"activation\":\"" +
           (L.relu ? "relu" : "linear") + "\",\"w_offset\":" + std::to_string(L.w_off) +
           ",\"b_offset\":" + std::to_string(L.b_off) + "}";
    }
    s += "]";
  }
  s += "}";
  return s;
}

}  // namespace tfsc
