// Robustness harness for the host-side parsers of libtfsc_b200 (no CUDA): compiled with
// -fsanitize=address,undefined by tests/test_native_fuzz.py and fed random / mutated inputs. A server must survive
// malformed PredictRequest bytes, URLs, JSON bodies and manifests without reading out of bounds.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../../tfservingcache_b200/csrc/arena.h"
#include "../../tfservingcache_b200/csrc/json.h"
#include "../../tfservingcache_b200/csrc/lru.h"
#include "../../tfservingcache_b200/csrc/model.h"
#include "../../tfservingcache_b200/csrc/parse.h"
#include "../../tfservingcache_b200/csrc/provider.h"
#include "../../tfservingcache_b200/csrc/ring.h"
#include "../../tfservingcache_b200/csrc/savedmodel.h"
#include "../../tfservingcache_b200/csrc/wire.h"

using namespace tfsc;

static std::mt19937_64 rng(12345);
static std::string random_bytes(size_t n) {
  std::string s(n, 0);
  for (auto& c : s) c = (char)(rng() & 0xFF);
  return s;
}
static std::string mutate(std::string s) {
  if (s.empty()) return s;
  int n = 1 + (int)(rng() % 4);
  for (int i = 0; i < n; ++i) {
    size_t p = rng() % s.size();
    switch (rng() % 4) {
      case 0: s[p] = (char)(rng() & 0xFF); break;
      case 1: s.erase(p, 1 + rng() % 3); break;
      case 2: s.insert(p, random_bytes(1 + rng() % 3)); break;
      default: s.resize(p); break;
    }
    if (s.empty()) break;
  }
  return s;
}

// a well-formed PredictRequest built by hand (model_spec{name, version}, inputs{"x": float tensor})
static std::string good_request() {
  auto varint = [](std::string* o, uint64_t v) {
    while (v >= 0x80) { o->push_back((char)(v | 0x80)); v >>= 7; }
    o->push_back((char)v);
  };
  auto ld = [&](std::string* o, int f, const std::string& p) { varint(o, (f << 3) | 2); varint(o, p.size()); o->append(p); };
  std::string ver; varint(&ver, 8); varint(&ver, 42);
  std::string spec; ld(&spec, 1, "foobar"); ld(&spec, 2, ver);
  std::string dim; varint(&dim, 8); varint(&dim, 2);
  std::string shape; ld(&shape, 2, dim); ld(&shape, 2, dim);
  std::string tensor; varint(&tensor, 8); varint(&tensor, 1); ld(&tensor, 2, shape); ld(&tensor, 4, std::string(16, '\x01'));
  std::string entry; ld(&entry, 1, "x"); ld(&entry, 2, tensor);
  std::string req; ld(&req, 1, spec); ld(&req, 2, entry); ld(&req, 3, "y");
  return req;
}

int main(int argc, char** argv) {
  const int iters = argc > 1 ? atoi(argv[1]) : 20000;
  const std::string good = good_request();
  {  // the good request decodes as expected
    PredictRequestView v; std::string err;
    if (!decode_predict_request(good.data(), good.size(), &v, &err) || v.model_name != "foobar" || v.version != 42 ||
        v.inputs.size() != 1 || v.inputs[0].shape.size() != 2 || v.output_filter.size() != 1) { fprintf(stderr, "good request failed\n"); return 1; }
    const float* d; int64_t n; std::vector<float> sc;
    if (!tensor_f32(v.inputs[0], &d, &n, &sc, &err) || n != 4) { fprintf(stderr, "good tensor failed\n"); return 1; }
  }
  {  // a response frame around its float payload is byte for byte what the encoders write for the same DT_FLOAT tensor
    const std::vector<std::vector<int64_t>> shapes = {{3}, {2, 4}, {0}, {}, {5, 40}};
    for (auto& shape : shapes)
      for (int64_t version : {(int64_t)0, (int64_t)123456789})
        for (const char* sig : {"", "serving_default"})
          for (const char* name : {"", "y:0"}) {
            int64_t n = 1;
            for (auto dim : shape) n *= dim;
            std::vector<float> vals((size_t)n + 1);
            for (int64_t k = 0; k < n; ++k) vals[k] = 0.25f * (float)k - 1.f;
            const std::string payload(reinterpret_cast<const char*>(vals.data()), (size_t)n * 4);
            OutTensor t;
            t.name = name;
            t.shape = shape;
            t.data = vals.data();
            t.n = n;
            std::string prefix, suffix;
            predict_response_frame("half_plus_two", version, sig, name, shape, &prefix, &suffix);
            if (prefix + payload + suffix != encode_predict_response("half_plus_two", version, sig, {t})) {
              fprintf(stderr, "predict_response_frame differs from encode_predict_response (rank %zu, version %lld, sig '%s', name '%s')\n",
                      shape.size(), (long long)version, sig, name);
              return 1;
            }
            session_run_response_frame("half_plus_two", version, sig, name, shape, &prefix, &suffix);
            if (prefix + payload + suffix != encode_session_run_response("half_plus_two", version, sig, t)) {
              fprintf(stderr, "session_run_response_frame differs from encode_session_run_response (rank %zu, version %lld, sig '%s', name '%s')\n",
                      shape.size(), (long long)version, sig, name);
              return 1;
            }
          }
  }
  const std::string good_json = "{\"instances\": [[1.0, 2.5e3, -3], [4, 5, 6]], \"signature_name\": \"serving_default\", \"x\": {\"a\": [true, null, \"s\\u00e9\"]}}";
  const std::string good_manifest = "{\"format\":\"tfsc-b200-v1\",\"template\":\"mlp\",\"dtype\":\"float32\",\"weights_bytes\":1280,\"layers\":[{\"in\":8,\"out\":16,\"activation\":\"relu\",\"w_offset\":0,\"b_offset\":512},{\"in\":16,\"out\":4,\"activation\":\"linear\",\"w_offset\":768,\"b_offset\":1024}]}";
  long decoded = 0, jsons = 0, manifests = 0;
  for (int i = 0; i < iters; ++i) {
    std::string in = (i % 3 == 0) ? random_bytes(rng() % 200) : mutate(good);
    PredictRequestView v; std::string err;
    if (decode_predict_request(in.data(), in.size(), &v, &err)) {
      ++decoded;
      for (auto& t : v.inputs) {
        const float* d; int64_t n; std::vector<float> sc;
        if (tensor_f32(t, &d, &n, &sc, &err)) { volatile float s = 0; for (int64_t k = 0; k < n; ++k) s += d[k]; (void)s; }
        const int32_t* di; std::vector<int32_t> si;
        if (tensor_i32(t, &di, &n, &si, &err)) { volatile int s = 0; for (int64_t k = 0; k < n; ++k) s += di[k]; (void)s; }
      }
    }
    std::string name; bool has; int64_t ver;
    scan_model_spec(in.data(), in.size(), &name, &has, &ver, nullptr);
    std::string url = (i % 2) ? mutate("/v1/models/foobar/versions/42:predict") : random_bytes(rng() % 60), n2, v2;
    match_rest_url(url, &n2, &v2);
    int64_t pv; parse_int64(mutate("9223372036854775807"), &pv);
    Json j; std::string js = (i % 2) ? mutate(good_json) : random_bytes(rng() % 100);
    if (json_parse(js, &j, &err)) ++jsons;
    Json mj; std::string ms = mutate(good_manifest);
    if (json_parse(ms, &mj, &err)) { ModelDesc d; if (parse_manifest(mj, &d, &err)) ++manifests; }
  }
  // ring + LRU under churn
  Ring ring; std::vector<std::string> members;
  LRUCache lru("", 1000);
  for (int i = 0; i < 2000; ++i) {
    if (rng() % 10 == 0) { members.clear(); int n = rng() % 12; for (int k = 0; k < n; ++k) members.push_back("h" + std::to_string(rng() % 20) + ":1:2"); ring.set(members); }
    std::vector<std::string> out; ring.get_n("key" + std::to_string(rng() % 100), 1 + rng() % 4, &out);
    ModelId id{"m" + std::to_string(rng() % 30), (int64_t)(rng() % 3)};
    if (rng() % 2) lru.put(id, CachedModel{id, "p", (int64_t)(rng() % 400)}); else lru.get(id, nullptr);
    if (lru.current_size() < 0) { fprintf(stderr, "negative LRU size\n"); return 1; }
  }
  // HBM arena allocator: random alloc / release, blocks never overlap, accounting exact, full coalescing at the end
  {
    Arena a; a.init(1 << 20, 1024);
    std::vector<std::pair<size_t, size_t>> live;  // offset, rounded length
    for (int i = 0; i < 20000; ++i) {
      if (live.empty() || rng() % 3) {
        size_t bytes = 1 + rng() % (96 << 10), off = 0;
        if (a.alloc(bytes, &off)) {
          size_t len = (bytes + 1023) / 1024 * 1024;
          if (off % 1024 || off + len > a.capacity()) { fprintf(stderr, "arena: bad block\n"); return 1; }
          for (auto& b : live)
            if (off < b.first + b.second && b.first < off + len) { fprintf(stderr, "arena: overlap\n"); return 1; }
          live.push_back({off, len});
        } else if (a.largest_free() >= (bytes + 1023) / 1024 * 1024) { fprintf(stderr, "arena: refused a fitting block\n"); return 1; }
      } else {
        size_t k = rng() % live.size();
        a.release(live[k].first);
        a.release(live[k].first);  // double release is ignored
        live[k] = live.back(); live.pop_back();
      }
      size_t sum = 0; for (auto& b : live) sum += b.second;
      if (sum != a.used() || live.size() != a.blocks()) { fprintf(stderr, "arena: accounting\n"); return 1; }
    }
    for (auto& b : live) a.release(b.first);
    if (a.used() != 0 || a.largest_free() != a.capacity()) { fprintf(stderr, "arena: not coalesced\n"); return 1; }
  }
  // SavedModel importer: argv[2] = a well-formed fixture directory written by the pytest wrapper; every file is mutated in a
  // scratch copy (argv[3]) and re-imported: errors are fine, out-of-bounds access is not
  long sm_ok = 0, sm_runs = 0;
  if (argc > 3) {
    const std::string src = argv[2], dst = argv[3];
    auto slurp = [](const std::string& p) { std::string o; FILE* f = fopen(p.c_str(), "rb"); if (f) { char b[4096]; size_t n; while ((n = fread(b, 1, sizeof b, f)) > 0) o.append(b, n); fclose(f); } return o; };
    auto spit = [](const std::string& p, const std::string& d) { FILE* f = fopen(p.c_str(), "wb"); if (f) { fwrite(d.data(), 1, d.size(), f); fclose(f); } };
    const char* files[3] = {"/saved_model.pb", "/variables/variables.index", "/variables/variables.data-00000-of-00001"};
    std::string good_f[3];
    for (int k = 0; k < 3; ++k) { good_f[k] = slurp(src + files[k]); spit(dst + files[k], good_f[k]); }
    SavedModelBundle sb; std::string err;
    if (!savedmodel_import(dst, &sb, &err)) { fprintf(stderr, "savedmodel fixture failed: %s\n", err.c_str()); return 1; }
    // the disk provider imports the same directory on the fly when it holds no tfsc_model.json (argv[4] = base dir
    // with the fixture linked as <base>/m/00000007)
    if (argc > 4) {
      DiskModelProvider prov(argv[4]);
      HostAllocFn alloc = [](size_t n, std::function<void(void*, size_t)>* rel) { *rel = [](void* q, size_t) { free(q); }; return malloc(n); };
      std::string perr;
      auto hm = prov.load_model("m", 7, alloc, &perr);
      if (!hm || hm->desc.tmpl != Template::Mlp || hm->desc.layers.size() != 2 || hm->desc.layers[0].in != 12 || hm->desc.layers[1].out != 5 ||
          hm->bytes != sb.weights.size() || memcmp(hm->data, sb.weights.data(), hm->bytes) != 0) {
        fprintf(stderr, "disk provider SavedModel import failed: %s\n", perr.c_str());
        return 1;
      }
      if (prov.load_model("m", 8, alloc, &perr) || perr != "No matching model found") { fprintf(stderr, "expected no match\n"); return 1; }
    }
    for (int i = 0; i < 1500; ++i) {
      const int k = i % 3;
      spit(dst + files[k], (i % 5 == 0) ? random_bytes(rng() % 300) : mutate(good_f[k]));
      SavedModelBundle b2; ++sm_runs;
      if (savedmodel_import(dst, &b2, &err)) ++sm_ok;
      spit(dst + files[k], good_f[k]);
    }
  }
  // Classify / Regress / SessionRun codecs against bytes serialized from the reference's own schema (argv[5] = directory the
  // pytest wrapper filled from tests/golden/examples_golden.json), then the same decoders under mutation
  long ex_ok = 0, ex_runs = 0;
  if (argc > 5) {
    const std::string dir = argv[5];
    auto slurp = [](const std::string& p) { std::string o; FILE* f = fopen(p.c_str(), "rb"); if (f) { char b[4096]; size_t n; while ((n = fread(b, 1, sizeof b, f)) > 0) o.append(b, n); fclose(f); } return o; };
    const float ys[3] = {2.5f, 3.0f, 4.5f};
    std::string err;
    for (const char* kind : {"regress", "classify"}) {
      const std::string req = slurp(dir + "/" + kind + "_request.bin"), resp = slurp(dir + "/" + kind + "_response.bin");
      ExampleRequestView v;
      if (req.empty() || !decode_example_request(req.data(), req.size(), &v, &err) || v.model_name != "half_plus_two" || v.version != 123 ||
          v.signature_name != std::string(kind) + "_x_to_y" || v.examples.size() != 3) { fprintf(stderr, "%s golden request: decode failed\n", kind); return 1; }
      const float xs[3] = {1.f, 2.f, 5.f};
      for (int i = 0; i < 3; ++i) {
        const std::vector<float>* f = v.examples[i].find("x");
        if (!f || f->size() != 1 || (*f)[0] != xs[i] || v.examples[i].find("ignored_bytes")) { fprintf(stderr, "%s golden request: features\n", kind); return 1; }
      }
      const std::string got = std::string(kind) == "regress" ? encode_regression_response("half_plus_two", 123, "regress_x_to_y", ys, 3)
                                                              : encode_classification_response("half_plus_two", 123, "classify_x_to_y", ys, 3, 1);
      if (got != resp) { fprintf(stderr, "%s golden response: bytes differ (%zu vs %zu)\n", kind, got.size(), resp.size()); return 1; }
    }
    {  // ExampleListWithContext: the context feature reaches every example
      const std::string req = slurp(dir + "/regress_with_context_request.bin");
      ExampleRequestView v;
      if (!decode_example_request(req.data(), req.size(), &v, &err) || v.examples.size() != 3) { fprintf(stderr, "context request\n"); return 1; }
      for (auto& e : v.examples) { const std::vector<float>* f = e.find("x"); if (!f || f->size() != 1 || (*f)[0] != 2.f) { fprintf(stderr, "context feature\n"); return 1; } }
    }
    const std::string sreq = slurp(dir + "/session_run_request.bin"), sresp = slurp(dir + "/session_run_response.bin");
    {
      SessionRunView v;
      if (!decode_session_run_request(sreq.data(), sreq.size(), &v, &err) || v.model_name != "half_plus_two" || v.version != 123 ||
          v.feeds.size() != 1 || v.feeds[0].name != "x:0" || v.fetch != std::vector<std::string>{"y:0"}) { fprintf(stderr, "session_run golden request\n"); return 1; }
      const float* d; int64_t n; std::vector<float> sc;
      if (!tensor_f32(v.feeds[0], &d, &n, &sc, &err) || n != 3 || d[0] != 1.f || d[2] != 5.f) { fprintf(stderr, "session_run feed tensor\n"); return 1; }
      std::string prefix, suffix;
      session_run_response_frame("half_plus_two", 123, "", "y:0", {3}, &prefix, &suffix);
      const std::string got = prefix + std::string(reinterpret_cast<const char*>(ys), 12) + suffix;
      if (got != sresp) { fprintf(stderr, "session_run golden response: bytes differ\n"); return 1; }
    }
    const std::string good_ex = slurp(dir + "/regress_with_context_request.bin");
    for (int i = 0; i < iters; ++i) {
      std::string in = (i % 4 == 0) ? random_bytes(rng() % 200) : mutate((i & 1) ? good_ex : sreq);
      ExampleRequestView ev; ++ex_runs;
      if (decode_example_request(in.data(), in.size(), &ev, &err)) {
        ++ex_ok;
        volatile float acc = 0;
        for (auto& e : ev.examples) for (auto& f : e.features) for (float x : f.second) acc += x;
        (void)acc;
      }
      SessionRunView sv;
      if (decode_session_run_request(in.data(), in.size(), &sv, &err))
        for (auto& t : sv.feeds) { const float* d; int64_t n; std::vector<float> sc; if (tensor_f32(t, &d, &n, &sc, &err)) { volatile float a2 = 0; for (int64_t k = 0; k < n; ++k) a2 += d[k]; (void)a2; } }
    }
  }
  printf("examples: %ld of %ld mutated Classify/Regress requests decoded\n", ex_ok, ex_runs);
  printf("savedmodel: %ld of %ld mutated imports accepted\n", sm_ok, sm_runs);
  printf("fuzz ok: %d iterations, %ld requests decoded, %ld json parsed, %ld manifests accepted\n", iters, decoded, jsons, manifests);
  return 0;
}
