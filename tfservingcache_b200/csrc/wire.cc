#include "wire.h"

#include <cmath>

#include "parse.h"

namespace tfsc {

static void put_varint(std::string* s, uint64_t v) {
  while (v >= 0x80) {
    s->push_back((char)(v | 0x80));
    v >>= 7;
  }
  s->push_back((char)v);
}
static void put_tag(std::string* s, uint32_t field, uint32_t wt) { put_varint(s, (field << 3) | wt); }
static void put_ld(std::string* s, uint32_t field, const std::string& payload) {
  put_tag(s, field, 2);
  put_varint(s, payload.size());
  s->append(payload);
}

static bool decode_shape(const uint8_t* d, size_t n, std::vector<int64_t>* shape) {
  PbReader r(d, n);
  uint32_t f, wt;
  uint64_t v;
  const uint8_t* p;
  size_t l;
  while (!r.done()) {
    if (!r.next(&f, &wt, &v, &p, &l)) return false;
    if (f == 2 && wt == 2) {  // dim
      int64_t size = 0;
      PbReader r2(p, l);
      while (!r2.done()) {
        uint32_t f2, wt2;
        uint64_t v2;
        const uint8_t* p2;
        size_t l2;
        if (!r2.next(&f2, &wt2, &v2, &p2, &l2)) return false;
        if (f2 == 1 && wt2 == 0) size = (int64_t)v2;
      }
      shape->push_back(size);
    }
  }
  return true;
}

static bool decode_tensor(const uint8_t* d, size_t n, TensorView* t) {
  PbReader r(d, n);
  uint32_t f, wt;
  uint64_t v;
  const uint8_t* p;
  size_t l;
  while (!r.done()) {
    if (!r.next(&f, &wt, &v, &p, &l)) return false;
    switch (f) {
      case 1: t->dtype = (int)v; break;
      case 2:
        if (wt == 2 && !decode_shape(p, l, &t->shape)) return false;
        break;
      case 4:
        if (wt == 2) {
          t->content = p;
          t->content_len = l;
        }
        break;
      case 5:  // float_val: packed (wt 2) or one fixed32 per entry (wt 5)
        if (wt == 2) {
          if (!t->packed_f32 && t->loose_f32.empty()) {
            t->packed_f32 = p;
            t->packed_f32_len = l;
          } else {  // several packed chunks: concatenate
            if (t->packed_f32) {
              t->loose_f32.resize(t->packed_f32_len / 4);
              memcpy(t->loose_f32.data(), t->packed_f32, t->packed_f32_len / 4 * 4);
              t->packed_f32 = nullptr;
            }
            size_t old = t->loose_f32.size();
            t->loose_f32.resize(old + l / 4);
            memcpy(t->loose_f32.data() + old, p, l / 4 * 4);
          }
        } else if (wt == 5) {
          float fv;
          uint32_t u = (uint32_t)v;
          memcpy(&fv, &u, 4);
          if (t->packed_f32) {
            t->loose_f32.resize(t->packed_f32_len / 4);
            memcpy(t->loose_f32.data(), t->packed_f32, t->packed_f32_len / 4 * 4);
            t->packed_f32 = nullptr;
          }
          t->loose_f32.push_back(fv);
        }
        break;
      case 7:  // int_val: packed varints (wt 2) or one varint per entry (wt 0)
        if (wt == 0) t->ints.push_back((int32_t)(int64_t)v);
        else if (wt == 2) {
          PbReader r2(p, l);
          uint64_t vv;
          while (!r2.done()) {
            if (!r2.varint(&vv)) return false;
            t->ints.push_back((int32_t)(int64_t)vv);
          }
        }
        break;
      default: break;  // other typed value fields are rejected later by dtype
    }
  }
  return true;
}

bool decode_predict_request(const void* data, size_t len, PredictRequestView* out, std::string* err) {
  PbReader r(data, len);
  uint32_t f, wt;
  uint64_t v;
  const uint8_t* p;
  size_t l;
  while (!r.done()) {
    if (!r.next(&f, &wt, &v, &p, &l)) {
      *err = "malformed PredictRequest";
      return false;
    }
    if (f == 1 && wt == 2) {
      // model_spec: re-wrap as a one-field message for the shared scanner
      std::string wrapped;
      put_ld(&wrapped, 1, std::string((const char*)p, l));
      if (!scan_model_spec(wrapped.data(), wrapped.size(), &out->model_name, &out->has_version, &out->version,
                           &out->signature_name)) {
        *err = "malformed ModelSpec";
        return false;
      }
    } else if (f == 2 && wt == 2) {  // map<string, TensorProto> entry
      TensorView t;
      PbReader r2(p, l);
      while (!r2.done()) {
        uint32_t f2, wt2;
        uint64_t v2;
        const uint8_t* p2;
        size_t l2;
        if (!r2.next(&f2, &wt2, &v2, &p2, &l2)) {
          *err = "malformed inputs entry";
          return false;
        }
        if (f2 == 1 && wt2 == 2) t.name.assign((const char*)p2, l2);
        else if (f2 == 2 && wt2 == 2 && !decode_tensor(p2, l2, &t)) {
          *err = "malformed TensorProto";
          return false;
        }
      }
      out->inputs.push_back(std::move(t));
    } else if (f == 3 && wt == 2) {
      out->output_filter.emplace_back((const char*)p, l);
    }
  }
  return true;
}

// 16 Mi elements = 64 MB = 4x the reference's 16 MiB gRPC message limit (cachemanager.go:230-233)
static constexpr int64_t kMaxBroadcastElements = (int64_t)16 << 20;

bool tensor_f32(const TensorView& t, const float** data, int64_t* n, std::vector<float>* scratch, std::string* err) {
  if (t.dtype != TFSC_DT_FLOAT) {
    *err = "input '" + t.name + "' has dtype " + std::to_string(t.dtype) + "; only DT_FLOAT (1) is supported";
    return false;
  }
  for (auto d : t.shape)
    if (d < 0) {
      *err = "input '" + t.name + "' has an unknown dimension";
      return false;
    }
  const int64_t want = t.num_elements();
  if (want < 0) {
    *err = "input '" + t.name + "': tensor_shape is too large";
    return false;
  }
  if (t.content_len) {
    if ((int64_t)(t.content_len / 4) != want || t.content_len % 4) {
      *err = "tensor_content size does not match tensor_shape";
      return false;
    }
    if (reinterpret_cast<uintptr_t>(t.content) % 4 == 0) {
      *data = reinterpret_cast<const float*>(t.content);
    } else {  // protobuf payloads are byte-aligned
      scratch->resize(want);
      memcpy(scratch->data(), t.content, t.content_len);
      *data = scratch->data();
    }
    *n = want;
    return true;
  }
  const uint8_t* src = t.packed_f32;
  int64_t have = (int64_t)(t.packed_f32_len / 4);
  if (!src) {
    src = reinterpret_cast<const uint8_t*>(t.loose_f32.data());
    have = (int64_t)t.loose_f32.size();
  }
  if (have == want) {
    if (reinterpret_cast<uintptr_t>(src) % 4 == 0) {
      *data = reinterpret_cast<const float*>(src);
    } else {
      scratch->resize(want);
      memcpy(scratch->data(), src, (size_t)want * 4);
      *data = scratch->data();
    }
    *n = want;
    return true;
  }
  if (have == 1 && want > 1) {  // TF semantics: a single value fills the tensor
    if (want > kMaxBroadcastElements) {  // the only path where a few request bytes size a large allocation
      *err = "input '" + t.name + "': scalar broadcast to " + std::to_string(want) + " elements exceeds the limit of " +
             std::to_string(kMaxBroadcastElements);
      return false;
    }
    float fv;
    memcpy(&fv, src, 4);
    scratch->assign(want, fv);
    *data = scratch->data();
    *n = want;
    return true;
  }
  *err = "float_val count " + std::to_string(have) + " does not match tensor_shape (" + std::to_string(want) + ")";
  return false;
}

bool tensor_i32(const TensorView& t, const int32_t** data, int64_t* n, std::vector<int32_t>* scratch, std::string* err) {
  if (t.dtype != TFSC_DT_INT32) {
    *err = "input '" + t.name + "' has dtype " + std::to_string(t.dtype) + "; expected DT_INT32 (3)";
    return false;
  }
  for (auto d : t.shape)
    if (d < 0) {
      *err = "input '" + t.name + "' has an unknown dimension";
      return false;
    }
  const int64_t want = t.num_elements();
  if (want < 0) {
    *err = "input '" + t.name + "': tensor_shape is too large";
    return false;
  }
  if (t.content_len) {
    if ((int64_t)(t.content_len / 4) != want || t.content_len % 4) {
      *err = "tensor_content size does not match tensor_shape";
      return false;
    }
    scratch->resize(want);
    memcpy(scratch->data(), t.content, t.content_len);
  } else if ((int64_t)t.ints.size() == want) {
    *scratch = t.ints;
  } else if (t.ints.size() == 1 && want > 1) {
    if (want > kMaxBroadcastElements) {
      *err = "input '" + t.name + "': scalar broadcast to " + std::to_string(want) + " elements exceeds the limit of " +
             std::to_string(kMaxBroadcastElements);
      return false;
    }
    scratch->assign(want, t.ints[0]);
  } else {
    *err = "int_val count " + std::to_string(t.ints.size()) + " does not match tensor_shape (" + std::to_string(want) + ")";
    return false;
  }
  *data = scratch->data();
  *n = want;
  return true;
}

// ------------------------------------------------------------------ Classify / Regress / SessionRun ----
static bool decode_model_spec_field(const uint8_t* p, size_t l, std::string* name, bool* has_version, int64_t* version,
                                    std::string* signature) {
  std::string wrapped;
  put_ld(&wrapped, 1, std::string((const char*)p, l));
  return scan_model_spec(wrapped.data(), wrapped.size(), name, has_version, version, signature);
}

static bool decode_feature(const uint8_t* d, size_t n, std::vector<float>* vals, bool* numeric) {
  PbReader r(d, n);
  uint32_t f, wt;
  uint64_t v;
  const uint8_t* p;
  size_t l;
  *numeric = false;
  while (!r.done()) {
    if (!r.next(&f, &wt, &v, &p, &l)) return false;
    if (f == 2 && wt == 2) {  // FloatList
      *numeric = true;
      PbReader r2(p, l);
      while (!r2.done()) {
        uint32_t f2, wt2;
        uint64_t v2;
        const uint8_t* p2;
        size_t l2;
        if (!r2.next(&f2, &wt2, &v2, &p2, &l2)) return false;
        if (f2 != 1) continue;
        if (wt2 == 2) {
          for (size_t i = 0; i + 4 <= l2; i += 4) {
            float fv;
            memcpy(&fv, p2 + i, 4);
            vals->push_back(fv);
          }
        } else if (wt2 == 5) {
          float fv;
          uint32_t u = (uint32_t)v2;
          memcpy(&fv, &u, 4);
          vals->push_back(fv);
        }
      }
    } else if (f == 3 && wt == 2) {  // Int64List
      *numeric = true;
      PbReader r2(p, l);
      while (!r2.done()) {
        uint32_t f2, wt2;
        uint64_t v2;
        const uint8_t* p2;
        size_t l2;
        if (!r2.next(&f2, &wt2, &v2, &p2, &l2)) return false;
        if (f2 != 1) continue;
        if (wt2 == 0) vals->push_back((float)(int64_t)v2);
        else if (wt2 == 2) {
          PbReader r3(p2, l2);
          uint64_t vv;
          while (!r3.done()) {
            if (!r3.varint(&vv)) return false;
            vals->push_back((float)(int64_t)vv);
          }
        }
      }
    }
  }
  return true;
}

// tf.Example -> numeric features
static bool decode_example(const uint8_t* d, size_t n, ExampleView* ex) {
  PbReader r(d, n);
  uint32_t f, wt;
  uint64_t v;
  const uint8_t* p;
  size_t l;
  while (!r.done()) {
    if (!r.next(&f, &wt, &v, &p, &l)) return false;
    if (f != 1 || wt != 2) continue;  // Features
    PbReader r2(p, l);
    while (!r2.done()) {
      uint32_t f2, wt2;
      uint64_t v2;
      const uint8_t* p2;
      size_t l2;
      if (!r2.next(&f2, &wt2, &v2, &p2, &l2)) return false;
      if (f2 != 1 || wt2 != 2) continue;  // map entry
      std::string key;
      std::vector<float> vals;
      bool numeric = false;
      PbReader r3(p2, l2);
      while (!r3.done()) {
        uint32_t f3, wt3;
        uint64_t v3;
        const uint8_t* p3;
        size_t l3;
        if (!r3.next(&f3, &wt3, &v3, &p3, &l3)) return false;
        if (f3 == 1 && wt3 == 2) key.assign((const char*)p3, l3);
        else if (f3 == 2 && wt3 == 2 && !decode_feature(p3, l3, &vals, &numeric)) return false;
      }
      if (numeric) ex->features.emplace_back(std::move(key), std::move(vals));
    }
  }
  return true;
}

bool decode_example_request(const void* data, size_t len, ExampleRequestView* out, std::string* err) {
  PbReader r(data, len);
  uint32_t f, wt;
  uint64_t v;
  const uint8_t* p;
  size_t l;
  while (!r.done()) {
    if (!r.next(&f, &wt, &v, &p, &l)) {
      *err = "malformed request";
      return false;
    }
    if (f == 1 && wt == 2) {
      if (!decode_model_spec_field(p, l, &out->model_name, &out->has_version, &out->version, &out->signature_name)) {
        *err = "malformed ModelSpec";
        return false;
      }
    } else if (f == 2 && wt == 2) {  // Input
      PbReader r2(p, l);
      while (!r2.done()) {
        uint32_t f2, wt2;
        uint64_t v2;
        const uint8_t* p2;
        size_t l2;
        if (!r2.next(&f2, &wt2, &v2, &p2, &l2)) {
          *err = "malformed Input";
          return false;
        }
        if ((f2 != 1 && f2 != 2) || wt2 != 2) continue;
        ExampleView context;
        const size_t first = out->examples.size();
        PbReader r3(p2, l2);
        while (!r3.done()) {
          uint32_t f3, wt3;
          uint64_t v3;
          const uint8_t* p3;
          size_t l3;
          if (!r3.next(&f3, &wt3, &v3, &p3, &l3)) {
            *err = "malformed ExampleList";
            return false;
          }
          if (f3 == 1 && wt3 == 2) {
            ExampleView ex;
            if (!decode_example(p3, l3, &ex)) {
              *err = "malformed tf.Example";
              return false;
            }
            out->examples.push_back(std::move(ex));
          } else if (f3 == 2 && wt3 == 2 && f2 == 2) {
            if (!decode_example(p3, l3, &context)) {
              *err = "malformed context tf.Example";
              return false;
            }
          }
        }
        for (size_t i = first; i < out->examples.size(); ++i)  // the context's features belong to every example
          for (auto& cf : context.features)
            if (!out->examples[i].find(cf.first)) out->examples[i].features.push_back(cf);
      }
    }
  }
  return true;
}

static std::string spec_bytes(const std::string& model_name, int64_t version, const std::string& signature) {
  std::string spec;
  if (!model_name.empty()) put_ld(&spec, 1, model_name);
  std::string ver;
  if (version != 0) {
    put_tag(&ver, 1, 0);
    put_varint(&ver, (uint64_t)version);
  }
  put_ld(&spec, 2, ver);
  if (!signature.empty()) put_ld(&spec, 3, signature);
  return spec;
}

static void put_f32(std::string* s, uint32_t field, float v) {
  put_tag(s, field, 5);
  s->append(reinterpret_cast<const char*>(&v), 4);
}

std::string encode_classification_response(const std::string& model_name, int64_t version, const std::string& signature,
                                           const float* scores, int64_t n, int64_t c) {
  std::string result;
  for (int64_t i = 0; i < n; ++i) {
    std::string cls;
    for (int64_t k = 0; k < c; ++k) {
      std::string one;  // Class{label = "" (omitted), score}
      if (scores[i * c + k] != 0.f || std::signbit(scores[i * c + k])) put_f32(&one, 2, scores[i * c + k]);
      put_ld(&cls, 1, one);
    }
    put_ld(&result, 1, cls);
  }
  std::string out;
  put_ld(&out, 1, result);
  put_ld(&out, 2, spec_bytes(model_name, version, signature));
  return out;
}

std::string encode_regression_response(const std::string& model_name, int64_t version, const std::string& signature,
                                       const float* values, int64_t n) {
  std::string result;
  for (int64_t i = 0; i < n; ++i) {
    std::string one;
    if (values[i] != 0.f || std::signbit(values[i])) put_f32(&one, 1, values[i]);
    put_ld(&result, 1, one);
  }
  std::string out;
  put_ld(&out, 1, result);
  put_ld(&out, 2, spec_bytes(model_name, version, signature));
  return out;
}

bool decode_session_run_request(const void* data, size_t len, SessionRunView* out, std::string* err) {
  PbReader r(data, len);
  uint32_t f, wt;
  uint64_t v;
  const uint8_t* p;
  size_t l;
  while (!r.done()) {
    if (!r.next(&f, &wt, &v, &p, &l)) {
      *err = "malformed SessionRunRequest";
      return false;
    }
    if (f == 1 && wt == 2) {
      if (!decode_model_spec_field(p, l, &out->model_name, &out->has_version, &out->version, &out->signature_name)) {
        *err = "malformed ModelSpec";
        return false;
      }
    } else if (f == 2 && wt == 2) {  // NamedTensorProto
      TensorView t;
      PbReader r2(p, l);
      while (!r2.done()) {
        uint32_t f2, wt2;
        uint64_t v2;
        const uint8_t* p2;
        size_t l2;
        if (!r2.next(&f2, &wt2, &v2, &p2, &l2)) {
          *err = "malformed feed";
          return false;
        }
        if (f2 == 1 && wt2 == 2) t.name.assign((const char*)p2, l2);
        else if (f2 == 2 && wt2 == 2 && !decode_tensor(p2, l2, &t)) {
          *err = "malformed TensorProto";
          return false;
        }
      }
      out->feeds.push_back(std::move(t));
    } else if (f == 3 && wt == 2) {
      out->fetch.emplace_back((const char*)p, l);
    } else if (f == 4 && wt == 2) {
      out->target.emplace_back((const char*)p, l);
    }
  }
  return true;
}

// ------------------------------------------------------------------ Predict / SessionRun responses ----
// TensorProto up to its values: dtype, tensor_shape
static std::string tensor_header(int dtype, const std::vector<int64_t>& shape) {
  std::string s;
  put_tag(&s, 1, 0);
  put_varint(&s, (uint64_t)dtype);
  std::string sh;
  for (auto d : shape) {
    std::string dim;
    if (d != 0) {
      put_tag(&dim, 1, 0);
      put_varint(&dim, (uint64_t)d);
    }
    put_ld(&sh, 2, dim);
  }
  put_ld(&s, 2, sh);
  return s;
}

static std::string tensor_proto(const OutTensor& t) {
  std::string s = tensor_header(t.dtype, t.shape);
  if (t.n > 0) {
    std::string vals;
    if (t.dtype == TFSC_DT_FLOAT) {
      vals.assign(static_cast<const char*>(t.data), (size_t)t.n * 4);  // packed float_val = little-endian fp32
      put_ld(&s, 5, vals);
    } else if (t.dtype == TFSC_DT_INT64) {
      const int64_t* v = static_cast<const int64_t*>(t.data);
      for (int64_t i = 0; i < t.n; ++i) put_varint(&vals, (uint64_t)v[i]);
      put_ld(&s, 10, vals);  // packed int64_val
    } else {
      const int32_t* v = static_cast<const int32_t*>(t.data);
      for (int64_t i = 0; i < t.n; ++i) put_varint(&vals, (uint64_t)(int64_t)v[i]);  // int32 varints sign-extend
      put_ld(&s, 7, vals);  // packed int_val
    }
  }
  return s;
}

std::string encode_predict_response(const std::string& model_name, int64_t version, const std::string& signature_name,
                                    const std::vector<OutTensor>& outs) {
  std::string s;
  for (auto& t : outs) {
    std::string entry;
    put_ld(&entry, 1, t.name);
    put_ld(&entry, 2, tensor_proto(t));
    put_ld(&s, 1, entry);
  }
  put_ld(&s, 2, spec_bytes(model_name, version, signature_name));
  return s;
}

std::string encode_session_run_response(const std::string& model_name, int64_t version, const std::string& signature_name,
                                        const OutTensor& t) {
  std::string named, s;
  if (!t.name.empty()) put_ld(&named, 1, t.name);
  put_ld(&named, 2, tensor_proto(t));
  put_ld(&s, 1, named);
  put_ld(&s, 3, spec_bytes(model_name, version, signature_name));
  return s;
}

// The bytes of a response whose field 1 is one {name_field, tensor = 2} entry holding a DT_FLOAT tensor of `shape`, and
// whose field `spec_field` is the model spec, split around the packed float_val payload: the encoders' bytes, with the
// values left for the executor to write in between.
static void float_frame(const std::string& name_field, const std::vector<int64_t>& shape, uint32_t spec_field,
                        const std::string& spec, std::string* prefix, std::string* suffix) {
  int64_t n = 1;
  for (auto d : shape) n *= d;
  const size_t payload = (size_t)n * 4;
  std::string thead = tensor_header(TFSC_DT_FLOAT, shape);
  if (payload) {
    put_tag(&thead, 5, 2);
    put_varint(&thead, payload);
  }
  std::string entry = name_field;
  put_tag(&entry, 2, 2);
  put_varint(&entry, thead.size() + payload);
  prefix->clear();
  put_tag(prefix, 1, 2);
  put_varint(prefix, entry.size() + thead.size() + payload);
  *prefix += entry + thead;
  suffix->clear();
  put_ld(suffix, spec_field, spec);
}

void predict_response_frame(const std::string& model_name, int64_t version, const std::string& signature_name,
                            const std::string& output_name, const std::vector<int64_t>& shape, std::string* prefix,
                            std::string* suffix) {
  std::string key;  // a map entry always carries its key
  put_ld(&key, 1, output_name);
  float_frame(key, shape, 2, spec_bytes(model_name, version, signature_name), prefix, suffix);
}

void session_run_response_frame(const std::string& model_name, int64_t version, const std::string& signature_name,
                                const std::string& tensor_name, const std::vector<int64_t>& shape, std::string* prefix,
                                std::string* suffix) {
  std::string name;
  if (!tensor_name.empty()) put_ld(&name, 1, tensor_name);
  float_frame(name, shape, 3, spec_bytes(model_name, version, signature_name), prefix, suffix);
}

}  // namespace tfsc
