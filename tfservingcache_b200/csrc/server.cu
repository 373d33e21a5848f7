// The server object behind the C ABI: cmd/taskhandler/main.go:45-113 (serveCache + serveProxy)
// for the GPUs of this process. Proxy tier = ring lookup + replica pick (taskhandler.go:84-92);
// cache tier = one Node per GPU (node.h); the forward hop between them is a function call (host
// buffers are staged straight into the owner GPU) or NVLink peer access (device buffers).
#include <cuda_runtime.h>

#include <chrono>
#include <cmath>
#include <map>
#include <memory>
#include <mutex>
#include <new>
#include <stdexcept>

#include "forward.h"
#include "inputs.h"
#include "json.h"
#include "kernels.h"
#include "node.h"
#include "parse.h"
#include "provider.h"
#include "ring.h"
#include "wire.h"

using namespace tfsc;

struct tfsc_server {
  Json cfg;
  std::unique_ptr<ModelProvider> provider;
  std::vector<std::unique_ptr<Node>> nodes;
  std::vector<std::string> local_members;  // member string of nodes[i]
  std::mutex ring_mu;
  Ring ring;
  std::map<std::string, int> member_node;
  std::vector<std::string> member_list;    // current members in the order given (index = member id of tfsc_predict_member)
  std::map<std::string, int> member_rank;  // member string -> rank of the process that serves it (cluster.endpoints index)
  int replicas = 1;
  std::mutex pick_mu;
  std::unique_ptr<ReplicaPicker> picker;
  std::atomic<int64_t> req_rest{0}, req_grpc{0}, fail_rest{0}, fail_grpc{0};
  std::unique_ptr<Forwarder> fwd;  // declared last: destroyed first (it hands requests to nodes[0])
};

static int route(tfsc_server* s, const std::string& name, const std::string& version, std::vector<int>* nodes,
                 int* picked, std::vector<int>* ranks = nullptr) {
  std::vector<std::string> members;
  const std::string key = name + "##" + version;
  int n_members = 0;
  {
    std::lock_guard<std::mutex> lk(s->ring_mu);
    // FindNodeForKey: GetN(key, max(replicasPerModel, 1)), cluster.go:117
    if (!s->ring.get_n(key, s->replicas < 1 ? 1 : s->replicas, &members)) return fail(TFSC_E_EMPTY_RING, "empty circle");
    n_members = s->ring.members();
    nodes->clear();
    for (auto& m : members) {
      auto it = s->member_node.find(m);
      nodes->push_back(it == s->member_node.end() ? -1 : it->second);
      if (ranks) {
        auto rt = s->member_rank.find(m);
        ranks->push_back(rt == s->member_rank.end() ? -1 : rt->second);
      }
    }
  }
  // "Pick random node", taskhandler.go:91 (policy "random"), or the primary / hot-spread / balanced variants
  std::vector<int> ids;
  for (auto& m : members) ids.push_back((int)(crc32_ieee(m.data(), m.size()) & 0x7FFFFFFF));  // stable id per member
  std::lock_guard<std::mutex> lk(s->pick_mu);
  *picked = s->picker->pick_ids(key, ids.data(), (int)nodes->size(), n_members);
  return (int)nodes->size();
}

static void set_members(tfsc_server* s, const std::vector<std::string>& members) {
  std::lock_guard<std::mutex> lk(s->ring_mu);
  s->ring.set(members);
  s->member_list = members;
  s->member_node.clear();
  for (size_t i = 0; i < s->local_members.size(); ++i) s->member_node[s->local_members[i]] = (int)i;
  // with cluster.endpoints the i-th member is served by the process listening on endpoints[i] (one rank per GPU)
  s->member_rank.clear();
  if (s->fwd)
    for (size_t i = 0; i < members.size() && (int)i < s->fwd->world(); ++i)
      if (!s->member_node.count(members[i])) s->member_rank[members[i]] = (int)i;
}

// No exception may cross the C ABI (a cgo / ctypes caller would see std::terminate): allocation failures and
// anything else thrown below the entry points become error codes.
template <typename F>
static int guarded(const char* what, F&& f) {
  try {
    return f();
  } catch (const std::bad_alloc&) {
    return fail(TFSC_E_EXHAUSTED, "%s: out of host memory", what);
  } catch (const std::length_error&) {
    return fail(TFSC_E_EXHAUSTED, "%s: request too large", what);
  } catch (const std::exception& e) {
    return fail(TFSC_E_INTERNAL, "%s: %s", what, e.what());
  } catch (...) {
    return fail(TFSC_E_INTERNAL, "%s: unknown exception", what);
  }
}

extern "C" {

static tfsc_server* server_create_impl(const char* config_json) {
  auto s = std::make_unique<tfsc_server>();
  std::string err;
  if (!config_json || !json_parse(config_json, &s->cfg, &err) || s->cfg.type != Json::Obj) {
    fail(TFSC_E_INVALID, "config: %s", err.empty() ? "expected a JSON object" : err.c_str());
    return nullptr;
  }
  int n_dev = 0;
  cudaError_t ce = cudaGetDeviceCount(&n_dev);
  if (ce != cudaSuccess || n_dev == 0) {
    cudaGetLastError();
    fail(TFSC_E_NO_DEVICE, "no CUDA device available (%s): this library has no CPU fallback",
         ce == cudaSuccess ? "device count is 0" : cudaGetErrorString(ce));
    return nullptr;
  }
  s->provider = create_provider(s->cfg, &err);
  if (!s->provider) {
    fail(TFSC_E_INVALID, "%s", err.c_str());
    return nullptr;
  }
  std::vector<int> devices;
  if (const Json* d = s->cfg.get("gpu.devices")) {
    for (auto& v : d->arr) devices.push_back((int)v.integer());
  }
  if (devices.empty())
    for (int i = 0; i < n_dev; ++i) devices.push_back(i);
  for (int d : devices) {
    cudaDeviceProp prop;
    if (d < 0 || d >= n_dev || cudaGetDeviceProperties(&prop, d) != cudaSuccess) {
      fail(TFSC_E_NO_DEVICE, "gpu.devices: device %d not present", d);
      return nullptr;
    }
    if (prop.major != 9 || prop.minor != 0) {
      fail(TFSC_E_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", d, prop.major,
           prop.minor);
      return nullptr;
    }
  }
  if (s->cfg.get_int("gpu.blockingSync", 1)) {
    // a serving process must not burn host cores spin-waiting on the GPU (the box's CPU quota is shared by all
    // ranks): make cudaEventSynchronize / cudaStreamSynchronize block. Applies to the primary context, i.e. also
    // to other CUDA users in this process (torch).
    for (int d : devices) {
      DeviceGuard g(d);
      if (cudaSetDeviceFlags(cudaDeviceScheduleBlockingSync) != cudaSuccess) cudaGetLastError();
    }
  }
  s->replicas = (int)std::max(s->cfg.get_num("proxy.replicasPerModel", 1), 1.0);
  const std::string policy = s->cfg.get_str("proxy.replicaPick", "random");
  if (policy != "random" && policy != "first" && policy != "hot-spread" && policy != "balanced" && policy != "hash") {
    fail(TFSC_E_INVALID, "unknown proxy.replicaPick '%s'", policy.c_str());
    return nullptr;
  }
  int64_t seed = s->cfg.get_int("proxy.seed", -1);
  // rand.Seed(time.Now().UnixNano()), taskhandler.go:49, unless pinned for reproducible tests
  s->picker = std::make_unique<ReplicaPicker>(
      policy, seed >= 0 ? (uint64_t)seed : (uint64_t)std::chrono::steady_clock::now().time_since_epoch().count(),
      s->cfg.get_num("proxy.hotFraction", 0.5));
  if (const Json* lm = s->cfg.get("gpu.localMembers"))
    for (auto& v : lm->arr) s->local_members.push_back(v.string());
  for (size_t i = 0; i < devices.size(); ++i) {
    NodeConfig nc;
    nc.device = devices[i];
    nc.host_cache_bytes = s->cfg.get_int("modelCache.size", (int64_t)1 << 40);
    nc.max_concurrent_models = (int)s->cfg.get_int("serving.maxConcurrentModels", 1 << 30);
    nc.arena_bytes = s->cfg.get_int("gpu.arenaBytes", 0);
    nc.max_batch = (int)s->cfg.get_int("gpu.maxBatch", 8);
    nc.max_request_rows = (int)s->cfg.get_int("gpu.maxRequestRows", 1024);
    nc.fetch_timeout_s = s->cfg.get_num("serving.modelFetchTimeout", 10.0);
    nc.slots = (int)s->cfg.get_int("gpu.stagingSlots", 4);
    nc.tick_us = (int)s->cfg.get_int("gpu.tickMicros", 0);
    auto node = std::make_unique<Node>(nc, s->provider.get());
    if (!node->init(&err)) {
      fail(TFSC_E_NO_DEVICE, "node %zu (device %d): %s", i, devices[i], err.c_str());
      return nullptr;
    }
    s->nodes.push_back(std::move(node));
    if (s->local_members.size() <= i) s->local_members.push_back("gpu" + std::to_string(devices[i]) + ":0:0");
  }
  // a6, the forward hop: every local GPU may read/write every other local GPU's memory over NVLink, so a
  // request tensor that sits on GPU i is consumed by the owner GPU j's kernels in place (peer loads/stores)
  for (int a : devices)
    for (int b : devices) {
      if (a == b) continue;
      int can = 0;
      if (cudaDeviceCanAccessPeer(&can, a, b) == cudaSuccess && can) {
        DeviceGuard g(a);
        cudaError_t pe = cudaDeviceEnablePeerAccess(b, 0);
        if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
        else if (pe == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
      }
    }
  std::vector<std::string> members;
  if (const Json* m = s->cfg.get("gpu.members"))
    for (auto& v : m->arr) members.push_back(v.string());
  if (members.empty()) members = s->local_members;
  if (const Json* eps = s->cfg.get("cluster.endpoints")) {
    // one process per GPU: requests whose ring owner is another rank are forwarded there (a6), tensors over NVLink
    FwdConfig fc;
    for (auto& v : eps->arr) fc.endpoints.push_back(v.string());
    fc.rank = (int)s->cfg.get_int("cluster.rank", 0);
    fc.slot_bytes = (size_t)s->cfg.get_int("cluster.slotBytes", 1 << 20);
    fc.slots = (int)s->cfg.get_int("cluster.windowSlots", 128);
    fc.timeout_s = s->cfg.get_num("proxy.grpcTimeout", 10.0);
    fc.workers = (int)s->cfg.get_int("cluster.forwardWorkers", 8);
    if (fc.endpoints.size() != members.size()) {
      fail(TFSC_E_INVALID, "cluster.endpoints must list one endpoint per entry of gpu.members (%zu vs %zu)", fc.endpoints.size(),
           members.size());
      return nullptr;
    }
    s->fwd = std::make_unique<Forwarder>(fc, s->nodes[0].get());
    if (!s->fwd->init(&err)) {
      fail(TFSC_E_INVALID, "%s", err.c_str());
      return nullptr;
    }
  }
  set_members(s.get(), members);
  return s.release();
}

void tfsc_server_destroy(tfsc_server* s) { delete s; }
int tfsc_server_num_nodes(const tfsc_server* s) { return s ? (int)s->nodes.size() : 0; }

int tfsc_server_set_members(tfsc_server* s, const char* const* members, int n) {
  if (!s || n < 0) return fail(TFSC_E_INVALID, "set_members: bad arguments");
  std::vector<std::string> v;
  for (int i = 0; i < n; ++i) v.emplace_back(members[i]);
  set_members(s, v);
  return n;
}

int tfsc_route(tfsc_server* s, const char* model_name, const char* version, int* nodes, int cap, int* picked) {
  if (!s || !model_name || !version) return fail(TFSC_E_INVALID, "route: bad arguments");
  std::vector<int> v;
  int p = 0;
  int rc = route(s, model_name, version, &v, &p);
  if (rc < 0) return rc;
  for (int i = 0; i < rc && i < cap; ++i) nodes[i] = v[i];
  if (picked) *picked = p;
  return rc;
}

static int check_device() {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
    cudaGetLastError();
    return fail(TFSC_E_NO_DEVICE, "no CUDA device available: this library has no CPU fallback");
  }
  return 0;
}

static Node* node_at(tfsc_server* s, int node) {
  if (!s || node < 0 || node >= (int)s->nodes.size()) {
    fail(TFSC_E_INVALID, "node index %d out of range", node);
    return nullptr;
  }
  return s->nodes[node].get();
}

int tfsc_model_ensure(tfsc_server* s, int node, const char* model_name, int64_t version) {
  Node* n = node_at(s, node);
  if (!n || !model_name) return TFSC_E_INVALID;
  std::string err;
  int rc = n->fetch({model_name, version}, nullptr, &err);
  if (rc < 0) return fail(rc, "%s", err.c_str());
  return rc;
}

int tfsc_model_ensure_async(tfsc_server* s, int node, const char* model_name, int64_t version) {
  Node* n = node_at(s, node);
  if (!n || !model_name) return TFSC_E_INVALID;
  std::string err;
  std::shared_ptr<DeviceModel> dm;
  int rc = n->fetch({model_name, version}, &dm, &err);
  if (rc < 0) return fail(rc, "%s", err.c_str());
  n->unpin(dm);
  return rc;
}

int tfsc_model_status(tfsc_server* s, int node, const char* model_name, int64_t version) {
  Node* n = node_at(s, node);
  if (!n || !model_name) return TFSC_E_INVALID;
  return n->status({model_name, version});
}

int tfsc_resident_list(tfsc_server* s, int node, char* buf, size_t cap) {
  Node* n = node_at(s, node);
  if (!n) return TFSC_E_INVALID;
  std::string l = n->resident_lines();
  int rc = copy_out(l, buf, cap);
  if (rc < 0) return rc;
  int c = 0;
  for (char ch : l) c += ch == '\n';
  return c;
}

int tfsc_host_list(tfsc_server* s, int node, char* buf, size_t cap) {
  Node* n = node_at(s, node);
  if (!n) return TFSC_E_INVALID;
  std::string l = n->host_lines();
  int rc = copy_out(l, buf, cap);
  if (rc < 0) return rc;
  int c = 0;
  for (char ch : l) c += ch == '\n';
  return c;
}

// route -> parse version -> owner. The owner is a node of this process (*node) or another rank (*remote >= 0, a6).
// Shared by the three Predict entry points.
static int resolve(tfsc_server* s, const std::string& name, const std::string& version, Node** node, ModelId* id,
                   int* remote = nullptr) {
  std::vector<int> nodes, ranks;
  int picked = 0;
  int rc = route(s, name, version, &nodes, &picked, &ranks);
  if (rc < 0) return rc;
  int local = nodes[picked];
  if (remote) *remote = -1;
  if (local < 0) {
    if (!remote || ranks[picked] < 0)
      return fail(TFSC_E_NOT_FOUND, "owner of %s##%s is not a GPU of this process", name.c_str(), version.c_str());
    *remote = ranks[picked];
  }
  int64_t v;
  if (!parse_int64(version, &v))  // handleModelRequest, cachemanager.go:297
    return fail(TFSC_E_INVALID, "strconv.ParseInt: parsing \"%s\": invalid syntax", version.c_str());
  *node = local >= 0 ? s->nodes[local].get() : nullptr;
  *id = {name, v};
  return 0;
}

// ensure-resident -> predict on the owner: a node of this process, or another rank through the forward hop
// (taskhandler.go:95-147: the request goes to whichever node the ring names, tensors stay in device memory here)
static int run_predict(tfsc_server* s, Node* node, int remote, const ModelId& id, const std::vector<InTensor>& ts,
                       const InputLayout& l, const Node::OutAllocFn& alloc, std::string* err, int64_t deadline_ns = 0) {
  if (node) return node->predict_host(id, ts, l, alloc, nullptr, nullptr, err, deadline_ns);
  return s->fwd->forward(remote, id.name, id.version, ts, l, alloc, nullptr, deadline_ns, err);
}
static int run_predict_one(tfsc_server* s, Node* node, int remote, const ModelId& id, const void* x, int64_t n, int dtype,
                           const Node::OutAllocFn& alloc, std::string* err, int64_t deadline_ns = 0) {
  std::vector<InTensor> ts(1);
  ts[0].dtype = dtype;
  ts[0].data = x;
  ts[0].n = n;
  const InputLayout l = layout_inputs(&ts);
  return run_predict(s, node, remote, id, ts, l, alloc, err, deadline_ns);
}

// The C ABI's input tensors: per-tensor argument checks (before residency, as always), then sorted by name into `ts`.
// Whether they fit the model is checked once it is resident (Node::prepare, check_layout).
static int abi_inputs(const tfsc_tensor* in, int n_in, bool need_data, std::vector<InTensor>* ts, InputLayout* l) {
  for (int i = 0; i < n_in; ++i) {
    const tfsc_tensor& x = in[i];
    if ((x.dtype != TFSC_DT_FLOAT && x.dtype != TFSC_DT_INT32) || x.rank < 0 || x.rank > 8)
      return fail(TFSC_E_INVALID, "predict: input must be DT_FLOAT or DT_INT32, rank <= 8");
    if (n_in > 1 && !x.name) return fail(TFSC_E_INVALID, "predict: every input needs a name when n_in > 1 (got %d inputs)", n_in);
    InTensor t;
    t.name = x.name ? x.name : "";
    t.dtype = x.dtype;
    t.data = x.data;
    t.shape.assign(x.shape, x.shape + x.rank);
    int64_t n = 1;
    for (auto d : t.shape) {
      if (d < 0 || (d != 0 && n > ((int64_t)1 << 40) / d)) return fail(TFSC_E_INVALID, "predict: bad input shape");
      n *= d;
    }
    if ((size_t)n * 4 != x.nbytes || (need_data && !x.data)) return fail(TFSC_E_INVALID, "predict: input nbytes does not match shape");
    t.n = x.data ? n : 0;
    ts->push_back(std::move(t));
  }
  *l = layout_inputs(ts);
  return 0;
}

// ---- Predict responses: the executor writes packed rows (model.h; a single-output model's row is its one output), and
// every front-end answers the outputs of one plan with the same rule, for local and forwarded requests alike.

// The selected outputs of one response, in the order they are answered, with their dtypes and full shapes (batch dims +
// per row). A model without signature.outputs answers one float output, d.output_name.
struct OutputPlan {
  std::vector<ModelOutput> sel;
  std::vector<int> dtypes;
  std::vector<std::vector<int64_t>> shapes;
  int64_t out_dim = 0, rows = 0;  // out_dim: words per packed row
  bool declared = false;          // the model declares signature.outputs
  // the packed rows are exactly the one output's values, so the executor can write them into the final buffer
  bool whole_row() const { return sel.size() == 1 && sel[0].offset == 0 && sel[0].width == out_dim; }
};

static int64_t product(const std::vector<int64_t>& v) {
  int64_t n = 1;
  for (auto x : v) n *= x;
  return n;
}

// The batch dims of a request with input shape `in_shape` that the executor will run as `rows` rows: an affine model
// answers in the input's shape, a graph keeps what precedes the per-image input shape ([B, H, W, C] -> [B, ...]), an mlp
// the leading dims of the input ([B, in] -> [B, out]; [in] -> [out]). Returns false (with a message) unless they account
// for exactly `rows` rows: the client's tensor_shape must never be the only thing that sizes a response buffer (e.g.
// [1, 2*in_dim] is two rows, not one).
static bool batch_dims(const ModelDesc& d, int64_t rows, const std::vector<int64_t>& in_shape, std::vector<int64_t>* dims,
                       std::string* why) {
  dims->clear();
  if (d.tmpl == Template::Affine) {
    *dims = in_shape;
  } else if (d.tmpl == Template::Graph) {
    if (in_shape.size() > d.input_shape.size())
      for (size_t i = 0; i + d.input_shape.size() < in_shape.size(); ++i) dims->push_back(in_shape[i]);
  } else if (in_shape.size() <= 1) {
    if (rows != 1 || in_shape.empty()) dims->push_back(rows);
  } else {
    for (size_t i = 0; i + 1 < in_shape.size(); ++i) dims->push_back(in_shape[i]);
  }
  int64_t on = 1;
  for (auto v : *dims) {
    if (v < 0 || (v != 0 && on > ((int64_t)1 << 40) / v)) {
      on = -1;
      break;
    }
    on *= v;
  }
  if (on != rows) {
    std::string sh = "[";
    for (size_t i = 0; i < in_shape.size(); ++i) sh += (i ? "," : "") + std::to_string(in_shape[i]);
    *why = "input shape " + sh + "] does not match the model signature: the trailing dimensions must hold exactly " +
           std::to_string(d.tmpl == Template::Affine ? 1 : d.in_dim) + " elements per row";
    return false;
  }
  return true;
}

// `names` (empty = every output, in packed order) must name declared outputs, each once; a single-output model answers its
// one output whatever they name. p->declared is set even when planning fails, for the front-ends' own name checks.
static bool plan_outputs(const ModelDesc& d, int64_t rows, const std::vector<int64_t>& in_shape, const std::vector<std::string>& names,
                         OutputPlan* p, std::string* why) {
  p->declared = !d.outputs.empty();
  std::vector<int64_t> dims;
  if (!batch_dims(d, rows, in_shape, &dims, why)) return false;
  p->sel.clear();
  p->dtypes.clear();
  p->shapes.clear();
  p->out_dim = d.tmpl == Template::Affine ? 1 : d.out_dim;
  p->rows = rows;
  if (!p->declared) {
    ModelOutput o;
    o.name = d.output_name;
    o.width = p->out_dim;
    p->sel.push_back(o);
    p->dtypes.push_back(TFSC_DT_FLOAT);
    if (d.tmpl == Template::Graph) dims.insert(dims.end(), d.output_shape.begin(), d.output_shape.end());
    else if (d.tmpl == Template::Mlp) dims.push_back(d.out_dim);
    p->shapes.push_back(dims);
    return true;
  }
  std::vector<std::string> want = names;
  if (want.empty())
    for (auto& o : d.outputs) want.push_back(o.name);
  for (size_t i = 0; i < want.size(); ++i) {
    const ModelOutput* o = d.output(want[i]);
    for (size_t j = 0; o && j < i; ++j)
      if (want[j] == want[i]) {
        *why = "output '" + want[i] + "' is requested twice; model outputs: " + expected_outputs(d);
        return false;
      }
    if (!o) {
      *why = "unknown output '" + want[i] + "'; model outputs: " + expected_outputs(d);
      return false;
    }
    p->sel.push_back(*o);
    p->dtypes.push_back(output_dtype(o->kind));
    std::vector<int64_t> sh = dims;
    const OutputForm f = output_form(o->kind, d.head_n, d.head_k);
    for (int r = 0; r < f.rank; ++r) sh.push_back(f.dims[r]);
    p->shapes.push_back(sh);
  }
  return true;
}

// the values of output i of the plan, cut out of `rows` packed rows (fp32 and int32: one word each, int64: two)
static void split_output(const OutputPlan& p, size_t i, const void* packed, void* dst) {
  const ModelOutput& o = p.sel[i];
  const char* src = static_cast<const char*>(packed);
  char* out = static_cast<char*>(dst);
  for (int64_t r = 0; r < p.rows; ++r)
    memcpy(out + (size_t)(r * o.width) * 4, src + (size_t)(r * p.out_dim + o.offset) * 4, (size_t)o.width * 4);
}

static std::string dtype_name(int dt) { return dt == TFSC_DT_INT64 ? "DT_INT64" : dt == TFSC_DT_INT32 ? "DT_INT32" : "DT_FLOAT"; }

// A single-input model's signature check: the one input, when the request names it, must carry the model's input name.
static bool input_matches(const ModelDesc& d, const std::string* name, std::string* bad) {
  if (!d.inputs.empty() || !name || *name == d.input_name) return true;
  *bad = "input '" + *name + "' does not match the model signature (expects '" + d.input_name + "')";
  return false;
}

// The outputs of one C ABI request, synchronous, asynchronous or forwarded: out[i].name selects the outputs of a model
// that declares them (any order, no repeats). A whole-row plan is written straight into out[0].data, any other into
// `packed`, which deliver() cuts into out[i].
struct AbiOutputs {
  tfsc_tensor* out = nullptr;
  int n_out = 0;
  std::vector<int64_t> in_shape;  // of the first input in name order: the response's batch dims
  bool in_named = false;          // the caller's in[0] has a name, in_name
  std::string in_name;
  OutputPlan plan;
  std::vector<float> packed;
  std::string bad;  // why the request does not fit the model

  AbiOutputs() = default;
  AbiOutputs(const tfsc_tensor& in0, const std::vector<int64_t>& shape, tfsc_tensor* o, int n)
      : out(o), n_out(n), in_shape(shape), in_named(in0.name != nullptr), in_name(in0.name ? in0.name : "") {}

  // the executor's destination for `rows` rows: nullptr with `bad` set when the request does not fit the model, nullptr
  // alone when an output buffer is too small
  void* alloc(const ModelDesc& d, int64_t rows) {
    if (!input_matches(d, in_named ? &in_name : nullptr, &bad)) return nullptr;
    std::vector<std::string> names;
    bool all_named = true;
    for (int i = 0; i < n_out; ++i) {
      all_named = all_named && out[i].name;
      names.push_back(out[i].name ? out[i].name : "");
    }
    const bool planned = plan_outputs(d, rows, in_shape, names, &plan, &bad);
    if (plan.declared && !all_named) {  // reported ahead of the plan's own errors
      bad = "predict: the model has several outputs, every out[i].name must name one of " + expected_outputs(d);
      return nullptr;
    }
    if (!planned) return nullptr;
    for (size_t i = 0; i < plan.sel.size(); ++i)
      if (!out[i].data || out[i].nbytes < (size_t)(rows * plan.sel[i].width) * 4 || plan.shapes[i].size() > 8) return nullptr;
    if (plan.whole_row()) return out[0].data;
    packed.assign((size_t)(rows * plan.out_dim), 0.f);
    return packed.data();
  }

  // fills out[i] (data, dtype, shape, nbytes) once the executor has written the rows
  void deliver() {
    for (size_t i = 0; i < plan.sel.size(); ++i) {
      if (!plan.whole_row()) split_output(plan, i, packed.data(), out[i].data);
      out[i].dtype = plan.dtypes[i];
      out[i].rank = (int32_t)plan.shapes[i].size();
      for (size_t j = 0; j < plan.shapes[i].size(); ++j) out[i].shape[j] = plan.shapes[i][j];
      out[i].nbytes = (size_t)(plan.rows * plan.sel[i].width) * 4;
    }
  }
};

// owner = member `member` of the current member list (the cache tier of that member, cachemanager.ServeRest/ServeGrpc: no
// ring lookup -- the caller already routed, e.g. with tfsc_route), local node or another rank
static int resolve_member(tfsc_server* s, int member, const std::string& name, const std::string& version, Node** node,
                          ModelId* id, int* remote) {
  std::string m;
  {
    std::lock_guard<std::mutex> lk(s->ring_mu);
    if (member < 0 || member >= (int)s->member_list.size()) return fail(TFSC_E_INVALID, "member index %d out of range", member);
    m = s->member_list[member];
    auto it = s->member_node.find(m);
    *node = it == s->member_node.end() ? nullptr : s->nodes[it->second].get();
    auto rt = s->member_rank.find(m);
    *remote = rt == s->member_rank.end() ? -1 : rt->second;
  }
  if (!*node && *remote < 0) return fail(TFSC_E_NOT_FOUND, "member %s is not served by this process and has no cluster endpoint", m.c_str());
  int64_t v;
  if (!parse_int64(version, &v)) return fail(TFSC_E_INVALID, "strconv.ParseInt: parsing \"%s\": invalid syntax", version.c_str());
  *id = {name, v};
  return 0;
}

static int predict_impl(tfsc_server* s, const char* model_name, const char* version, const tfsc_tensor* in, int n_in,
                        tfsc_tensor* out, int n_out, int64_t deadline_ns, int member = -1) {
  if (!s || !model_name || !version || !in || n_in < 1 || !out || n_out < 1)
    return fail(TFSC_E_INVALID, "predict: bad arguments");
  Node* node;
  ModelId id;
  int remote = -1;
  int rc = member >= 0 ? resolve_member(s, member, model_name, version, &node, &id, &remote)
                       : resolve(s, model_name, version, &node, &id, &remote);
  if (rc < 0) return rc;
  std::vector<InTensor> ts;
  InputLayout layout;
  if ((rc = abi_inputs(in, n_in, false, &ts, &layout)) < 0) return rc;
  AbiOutputs outs(in[0], ts[0].shape, out, n_out);
  std::string err;
  auto alloc = [&](const ModelDesc& d, int64_t rows) { return outs.alloc(d, rows); };
  rc = run_predict(s, node, remote, id, ts, layout, alloc, &err, deadline_ns);
  if (rc < 0 && !outs.bad.empty()) return fail(TFSC_E_INVALID, "%s", outs.bad.c_str());
  if (rc < 0) return fail(rc, "%s", err.c_str());
  outs.deliver();
  return 0;
}

static void set_resp(const std::string& body, void** resp, size_t* resp_len) {
  char* b = (char*)malloc(body.size() + 1);
  memcpy(b, body.data(), body.size());
  b[body.size()] = 0;
  *resp = b;
  *resp_len = body.size();
}

// A request tensor as an executor input: DT_INT32 (token ids) or else DT_FLOAT. tensor_content and packed float_val stay
// zero-copy views into the request; values stored any other way are gathered in `fs` / `is`.
static bool tensor_input(const TensorView& v, InTensor* t, std::vector<float>* fs, std::vector<int32_t>* is, std::string* err) {
  t->shape = v.shape;
  if (v.dtype == TFSC_DT_INT32) {
    const int32_t* p = nullptr;
    const bool ok = tensor_i32(v, &p, &t->n, is, err);
    t->data = p;
    t->dtype = TFSC_DT_INT32;
    return ok;
  }
  const float* p = nullptr;
  const bool ok = tensor_f32(v, &p, &t->n, fs, err);
  t->data = p;
  t->dtype = TFSC_DT_FLOAT;
  return ok;
}

// A gRPC response with a hole of `payload` bytes between prefix and suffix, for the executor to write the values into
static void* frame_hole(const std::string& prefix, size_t payload, const std::string& suffix, char** buf, size_t* len) {
  *len = prefix.size() + payload + suffix.size();
  *buf = (char*)malloc(*len ? *len : 1);
  if (!*buf) return nullptr;
  memcpy(*buf, prefix.data(), prefix.size());
  memcpy(*buf + prefix.size() + payload, suffix.data(), suffix.size());
  return *buf + prefix.size();
}

// output i of the plan as a response tensor, its values cut out of the packed rows into `vals`
static OutTensor out_tensor(const OutputPlan& p, size_t i, const void* packed, std::vector<char>* vals) {
  vals->resize((size_t)(p.rows * p.sel[i].width) * 4);
  split_output(p, i, packed, vals->data());
  OutTensor t;
  t.name = p.sel[i].name;
  t.dtype = p.dtypes[i];
  t.shape = p.shapes[i];
  t.data = vals->data();
  t.n = product(p.shapes[i]);
  return t;
}

static int grpc_predict_impl(tfsc_server* s, const void* req, size_t req_len, void** resp, size_t* resp_len) {
  if (!s || !req || !resp || !resp_len) return fail(TFSC_E_INVALID, "grpc_predict: bad arguments");
  s->req_grpc++;  // promRequestsTotal{grpc}, tfservingproxy.go:202
  PredictRequestView view;
  std::string err;
  if (!decode_predict_request(req, req_len, &view, &err)) {
    s->fail_grpc++;
    return fail(TFSC_E_INVALID, "%s", err.c_str());
  }
  // clientForSpec: version string = FormatInt(GetVersion().GetValue()) -> "0" when absent (:246-250)
  const std::string version = std::to_string(view.version);
  Node* node;
  ModelId id;
  int remote = -1;
  int rc = resolve(s, view.model_name, version, &node, &id, &remote);
  if (rc < 0) {
    s->fail_grpc++;
    return rc;
  }
  if (view.inputs.empty()) {
    // the reference forwards even an empty request; residency is still ensured first (on the owner, when it is local)
    rc = node ? node->fetch(id, nullptr, &err) : 0;
    s->fail_grpc++;
    if (rc < 0) return fail(rc, "%s", err.c_str());
    return fail(TFSC_E_INVALID, "PredictRequest has no inputs");
  }
  // every named input; tensor_content stays a zero-copy view into the request, packing is the only copy
  const size_t n_in = view.inputs.size();
  std::vector<InTensor> ts(n_in);
  std::vector<std::vector<float>> scratch(n_in);
  std::vector<std::vector<int32_t>> iscratch(n_in);
  bool input_ok = true;
  for (size_t i = 0; i < n_in && input_ok; ++i) {
    ts[i].name = view.inputs[i].name;
    input_ok = tensor_input(view.inputs[i], &ts[i], &scratch[i], &iscratch[i], &err);
  }
  const InputLayout layout = layout_inputs(&ts);
  const TensorView& tv = view.inputs[0];
  const std::string sig = view.signature_name.empty() ? "serving_default" : view.signature_name;
  char* buf = nullptr;
  size_t total = 0;
  std::string bad_sig;
  OutputPlan plan;
  std::vector<float> packed;
  auto alloc = [&](const ModelDesc& d, int64_t rows) -> void* {
    if (d.inputs.empty() && (n_in != 1 || tv.name != d.input_name)) {
      bad_sig = "input keys do not match the model signature (expects '" + d.input_name + "')";
      return nullptr;
    }
    // output_filter selects declared outputs (empty: all); the response map lists them in sorted name order. The two
    // messages follow TF-Serving's predict_util.cc as far as they are known (wording unverified against its source), and
    // are reported ahead of the plan's own errors.
    std::set<std::string> sel;
    std::string bad_filter;
    for (auto& a : view.output_filter) {
      if (!d.output(a)) {
        std::string set;
        for (auto& o : d.outputs) set += (set.empty() ? "" : ",") + o.name;
        bad_filter = "output tensor alias not found in signature: " + a + " Outputs expected to be in the set {" + set + "}.";
        break;
      }
      if (!sel.insert(a).second) {
        bad_filter = "duplicate output tensor alias: " + a;
        break;
      }
    }
    const bool planned = plan_outputs(d, rows, ts[0].shape, std::vector<std::string>(sel.begin(), sel.end()), &plan, &bad_sig);
    if (plan.declared && !bad_filter.empty()) {
      bad_sig = bad_filter;
      return nullptr;
    }
    if (!planned) return nullptr;
    if (plan.whole_row() && plan.dtypes[0] == TFSC_DT_FLOAT) {  // the executor's result goes straight into the response
      std::string prefix, suffix;
      predict_response_frame(view.model_name, id.version, sig, plan.sel[0].name, plan.shapes[0], &prefix, &suffix);
      return frame_hole(prefix, (size_t)(rows * plan.out_dim) * 4, suffix, &buf, &total);
    }
    packed.assign((size_t)(rows * plan.out_dim), 0.f);
    return packed.data();
  };
  if (!input_ok) {
    std::string e2;
    rc = node ? node->fetch(id, nullptr, &e2) : 0;  // residency first, like the reference; then reject the tensor
    s->fail_grpc++;
    if (rc < 0) return fail(rc, "%s", e2.c_str());
    return fail(TFSC_E_INVALID, "%s", err.c_str());
  }
  rc = run_predict(s, node, remote, id, ts, layout, alloc, &err);
  if (rc < 0) {
    free(buf);
    s->fail_grpc++;
    if (!bad_sig.empty()) return fail(TFSC_E_INVALID, "%s", bad_sig.c_str());
    return fail(rc, "%s", err.c_str());
  }
  if (buf) {
    *resp = buf;
    *resp_len = total;
    return 0;
  }
  std::vector<std::vector<char>> vals(plan.sel.size());
  std::vector<OutTensor> outs;
  for (size_t i = 0; i < plan.sel.size(); ++i) outs.push_back(out_tensor(plan, i, packed.data(), &vals[i]));
  set_resp(encode_predict_response(view.model_name, id.version, sig, outs), resp, resp_len);
  return 0;
}

// ---- Classify / Regress (tfservingproxy.go:173-198): tf.Example inputs -> one row per example -> the predict path.
// method: 1 = classify, 2 = regress. Fills scores [n, per] (classify: per = outputs per example; regress: per == 1).
static int run_examples(tfsc_server* s, const ExampleRequestView& view, int method, std::vector<float>* scores, int64_t* n_out,
                        int64_t* per_out, ModelId* id_out, std::string* sig_out, std::string* err) {
  const std::string version = std::to_string(view.version);  // clientForSpec: "0" when absent
  Node* node;
  ModelId id;
  int remote = -1;
  int rc = resolve(s, view.model_name, version, &node, &id, &remote);
  if (rc < 0) {
    *err = tfsc_last_error();
    return rc;
  }
  if (!node) {
    *err = "model " + view.model_name + " is owned by rank " + std::to_string(remote) + "; Classify / Regress are served by the owner";
    return TFSC_E_NOT_FOUND;
  }
  ModelDesc d;
  rc = node->describe(id, &d, nullptr, err);  // fetchModel first, like every request of the reference
  if (rc < 0) return rc;
  if (!d.inputs.empty()) {
    *err = std::string(method == 1 ? "Classify" : "Regress") + " serves single-input models; " + view.model_name + " has inputs " +
           expected_inputs(d) + " (use Predict)";
    return TFSC_E_INVALID;
  }
  if (!d.outputs.empty()) {
    *err = std::string(method == 1 ? "Classify" : "Regress") + " serves single-output models; " + view.model_name + " has outputs " +
           expected_outputs(d) + " (use Predict)";
    return TFSC_E_INVALID;
  }
  const std::string want = view.signature_name.empty() ? "serving_default" : view.signature_name;
  const ExtraSignature* sg = nullptr;
  for (auto& e : d.extra_sigs)
    if (e.name == want) sg = &e;
  const char* mname = method == 1 ? "tensorflow/serving/classify" : "tensorflow/serving/regress";
  if (!sg) {
    // TF-Serving's answers: an unknown signature key, or a signature of the wrong method (classifier.cc / regressor.cc)
    if (want == "serving_default")
      *err = std::string("Expected ") + (method == 1 ? "classification" : "regression") + " signature method_name to be " + mname +
             ". Was: tensorflow/serving/predict";
    else
      *err = "Serving signature name: \"" + want + "\" not found in signature def";
    return TFSC_E_INVALID;
  }
  if (sg->method != method) {
    *err = std::string("Expected ") + (method == 1 ? "classification" : "regression") + " signature method_name to be " + mname +
           ". Was: " + (sg->method == 1 ? "tensorflow/serving/classify" : "tensorflow/serving/regress");
    return TFSC_E_INVALID;
  }
  if (view.examples.empty()) {
    *err = "Input is empty";  // TF-Serving: InvalidArgument("Input is empty.")
    return TFSC_E_INVALID;
  }
  const int64_t per_row = d.tmpl == Template::Affine ? 1 : d.in_dim;
  if (d.input_dtype != TFSC_DT_FLOAT) {
    *err = "the model's input is not a float tensor: no tf.Example signature";
    return TFSC_E_INVALID;
  }
  std::vector<float> x;
  x.reserve((size_t)view.examples.size() * per_row);
  for (size_t i = 0; i < view.examples.size(); ++i) {
    const std::vector<float>* f = view.examples[i].find(sg->feature);
    if (!f || (int64_t)f->size() != per_row) {
      *err = "example " + std::to_string(i) + ": feature '" + sg->feature + "' must hold " + std::to_string(per_row) +
             " float value(s), found " + (f ? std::to_string(f->size()) : std::string("none"));
      return TFSC_E_INVALID;
    }
    x.insert(x.end(), f->begin(), f->end());
  }
  const int64_t n = (int64_t)view.examples.size();
  const int64_t per = d.tmpl == Template::Affine ? 1 : d.out_dim;
  if (method == 2 && per != 1) {
    *err = "Expected output Tensor shape to be either [batch_size] or [batch_size, 1] but got [" + std::to_string(n) + "," +
           std::to_string(per) + "]";  // regressor.cc
    return TFSC_E_INVALID;
  }
  scores->assign((size_t)(n * per), 0.f);
  auto alloc = [&](const ModelDesc&, int64_t rows) -> void* { return rows == n ? scores->data() : nullptr; };
  rc = node->predict_host(id, x.data(), (int64_t)x.size(), TFSC_DT_FLOAT, alloc, nullptr, nullptr, err);
  if (rc < 0) return rc;
  *n_out = n;
  *per_out = per;
  *id_out = id;
  *sig_out = want;
  return 0;
}

static int grpc_examples_impl(tfsc_server* s, int method, const void* req, size_t req_len, void** resp, size_t* resp_len) {
  if (!s || !req || !resp || !resp_len) return fail(TFSC_E_INVALID, "grpc_classify/regress: bad arguments");
  s->req_grpc++;  // promRequestsTotal{grpc}, tfservingproxy.go:174,188
  ExampleRequestView view;
  std::string err;
  if (!decode_example_request(req, req_len, &view, &err)) {
    s->fail_grpc++;
    return fail(TFSC_E_INVALID, "%s", err.c_str());
  }
  std::vector<float> scores;
  int64_t n = 0, per = 0;
  ModelId id;
  std::string sig;
  int rc = run_examples(s, view, method, &scores, &n, &per, &id, &sig, &err);
  if (rc < 0) {
    s->fail_grpc++;
    return fail(rc, "%s", err.c_str());
  }
  const std::string out = method == 1 ? encode_classification_response(view.model_name, id.version, sig, scores.data(), n, per)
                                      : encode_regression_response(view.model_name, id.version, sig, scores.data(), n);
  set_resp(out, resp, resp_len);
  return 0;
}

static int grpc_session_run_impl(tfsc_server* s, const void* req, size_t req_len, void** resp, size_t* resp_len) {
  if (!s || !req || !resp || !resp_len) return fail(TFSC_E_INVALID, "grpc_session_run: bad arguments");
  s->req_grpc++;  // tfservingproxy.go:234
  SessionRunView view;
  std::string err;
  if (!decode_session_run_request(req, req_len, &view, &err)) {
    s->fail_grpc++;
    return fail(TFSC_E_INVALID, "%s", err.c_str());
  }
  Node* node;
  ModelId id;
  int remote = -1;
  int rc = resolve(s, view.model_name, std::to_string(view.version), &node, &id, &remote);
  if (rc < 0) {
    s->fail_grpc++;
    return rc;
  }
  auto strip = [](const std::string& t) { return t.size() > 2 && t.compare(t.size() - 2, 2, ":0") == 0 ? t.substr(0, t.size() - 2) : t; };
  if (view.feeds.size() != 1 || view.fetch.size() != 1 || !view.target.empty()) {
    ModelDesc d;
    const bool known = node && node->describe(id, &d, nullptr, &err) >= 0;
    s->fail_grpc++;
    if (known && !d.inputs.empty())
      return fail(TFSC_E_INVALID, "SessionRun serves single-input models; %s has inputs %s (use Predict)", view.model_name.c_str(),
                  expected_inputs(d).c_str());
    return fail(TFSC_E_INVALID, "SessionRun on a model template takes exactly one feed (the signature input) and one fetch (its output)");
  }
  const TensorView& tv = view.feeds[0];
  std::vector<InTensor> ts(1);  // unnamed: the feed's name is checked against the signature below
  std::vector<float> scratch;
  std::vector<int32_t> iscratch;
  if (!tensor_input(tv, &ts[0], &scratch, &iscratch, &err)) {
    s->fail_grpc++;
    return fail(TFSC_E_INVALID, "%s", err.c_str());
  }
  const InputLayout layout = layout_inputs(&ts);
  char* buf = nullptr;
  size_t total = 0;
  std::string bad;
  OutputPlan plan;
  std::vector<float> packed;
  auto alloc = [&](const ModelDesc& d, int64_t rows) -> void* {
    const std::string fetch = strip(view.fetch[0]);
    const bool planned = plan_outputs(d, rows, tv.shape, {fetch}, &plan, &bad);
    // the feed names the model's input and the fetch its output, or any one of its declared outputs (reported ahead of the
    // plan's own errors)
    if (strip(tv.name) != d.input_name || (plan.declared ? !d.output(fetch) : fetch != d.output_name)) {
      bad = "feed / fetch do not name the model's tensors (feed '" + d.input_name + ":0', fetch " +
            (plan.declared ? "one of " + expected_outputs(d) : "'" + d.output_name + ":0'") + ")";
      return nullptr;
    }
    if (!planned) return nullptr;
    if (plan.whole_row() && plan.dtypes[0] == TFSC_DT_FLOAT) {  // the executor's result goes straight into the response
      std::string prefix, suffix;
      session_run_response_frame(view.model_name, id.version, view.signature_name, view.fetch[0], plan.shapes[0], &prefix, &suffix);
      return frame_hole(prefix, (size_t)(rows * plan.out_dim) * 4, suffix, &buf, &total);
    }
    packed.assign((size_t)(rows * plan.out_dim), 0.f);
    return packed.data();
  };
  rc = run_predict(s, node, remote, id, ts, layout, alloc, &err);
  if (rc < 0) {
    free(buf);
    s->fail_grpc++;
    if (!bad.empty()) return fail(TFSC_E_INVALID, "%s", bad.c_str());
    return fail(rc, "%s", err.c_str());
  }
  if (buf) {
    *resp = buf;
    *resp_len = total;
    return 0;
  }
  std::vector<char> vals;
  OutTensor t = out_tensor(plan, 0, packed.data(), &vals);
  t.name = view.fetch[0];
  set_resp(encode_session_run_response(view.model_name, id.version, view.signature_name, t), resp, resp_len);
  return 0;
}

// ------------------------------------------------------------------------------ REST ------
static const char* state_name(int st) {
  switch (st) {
    case TFSC_STATE_START: return "START";
    case TFSC_STATE_LOADING: return "LOADING";
    case TFSC_STATE_AVAILABLE: return "AVAILABLE";
    case TFSC_STATE_UNLOADING: return "UNLOADING";
    case TFSC_STATE_END: return "END";
    default: return "UNKNOWN";
  }
}

static int http_for(int rc) {
  switch (rc) {
    case TFSC_E_INVALID: return 400;
    case TFSC_E_NOT_FOUND: return 404;
    case TFSC_E_TIMEOUT: return 504;
    case TFSC_E_EXHAUSTED: return 507;
    case TFSC_E_EMPTY_RING: return 503;
    default: return 500;
  }
}

static std::string error_json(const std::string& msg) {
  std::string s = "{ \"error\": ";
  json_escape(msg, &s);
  s += " }";
  return s;
}

// flatten a (nested, rectangular) JSON array of numbers
static bool flatten(const Json& j, size_t depth, std::vector<int64_t>* shape, std::vector<float>* out, std::string* err) {
  if (j.type == Json::Num) {
    if (shape->size() > depth) {
      *err = "ragged tensor";
      return false;
    }
    out->push_back((float)j.num);
    return true;
  }
  if (j.type != Json::Arr) {
    *err = "tensor values must be numbers or nested arrays of numbers";
    return false;
  }
  if (shape->size() == depth) shape->push_back((int64_t)j.arr.size());
  else if ((*shape)[depth] != (int64_t)j.arr.size()) {
    *err = "ragged tensor";
    return false;
  }
  for (auto& e : j.arr)
    if (!flatten(e, depth + 1, shape, out, err)) return false;
  return true;
}

static void write_tensor_json(const float* v, const std::vector<int64_t>& shape, size_t dim, size_t* idx, std::string* s) {
  if (dim == shape.size()) {
    json_float(v[(*idx)++], s);
    return;
  }
  *s += "[";
  for (int64_t i = 0; i < shape[dim]; ++i) {
    if (i) *s += ", ";
    write_tensor_json(v, shape, dim + 1, idx, s);
  }
  *s += "]";
}

// one value of a packed row as JSON: fp32 as json_float, int32 / int64 as integers
static void json_word_value(OutputKind k, const uint32_t* w, std::string* s) {
  const int dt = output_dtype(k);
  if (dt == TFSC_DT_INT64) {
    *s += std::to_string((int64_t)((uint64_t)w[0] | ((uint64_t)w[1] << 32)));
  } else if (dt == TFSC_DT_INT32) {
    *s += std::to_string((int32_t)w[0]);
  } else {
    float f;
    memcpy(&f, w, 4);
    json_float(f, s);
  }
}

// values [dims...] of one output, row-major, `step` words per value
static void json_nested(OutputKind k, const uint32_t* w, const std::vector<int64_t>& dims, size_t dim, int64_t* idx, int step,
                        std::string* s) {
  if (dim == dims.size()) {
    json_word_value(k, w + *idx * step, s);
    ++*idx;
    return;
  }
  *s += "[";
  for (int64_t i = 0; i < dims[dim]; ++i) {
    if (i) *s += ", ";
    json_nested(k, w, dims, dim + 1, idx, step, s);
  }
  *s += "]";
}

// TF-Serving's multi-output REST shapes: row format {"predictions": [{"<output>": value, ...} per row]}, columnar format
// {"outputs": {"<output>": tensor, ...}}; keys in packed (sorted name) order
static std::string rest_multi_output_json(const OutputPlan& p, const float* packed, bool row_format) {
  const uint32_t* words = reinterpret_cast<const uint32_t*>(packed);
  std::string b = std::string("{\n    \"") + (row_format ? "predictions" : "outputs") + "\": " + (row_format ? "[" : "{");
  if (row_format) {
    for (int64_t r = 0; r < p.rows; ++r) {
      b += r ? ", {" : "{";
      for (size_t i = 0; i < p.sel.size(); ++i) {
        const ModelOutput& o = p.sel[i];
        if (i) b += ", ";
        json_escape(o.name, &b);
        b += ": ";
        const uint32_t* w = words + r * p.out_dim + o.offset;
        const size_t rank = (size_t)output_form(o.kind, 0, 0).rank;
        if (rank == 0) {
          json_word_value(o.kind, w, &b);
        } else {
          // one row's value: the trailing `rank` dims of the plan's shape ([N], [k], [H] or sequence_output's [S, H])
          const std::vector<int64_t>& sh = p.shapes[i];
          int64_t idx = 0;
          json_nested(o.kind, w, std::vector<int64_t>(sh.end() - (ptrdiff_t)rank, sh.end()), 0, &idx, 1, &b);
        }
      }
      b += "}";
    }
    b += "]\n}";
    return b;
  }
  for (size_t i = 0; i < p.sel.size(); ++i) {
    const ModelOutput& o = p.sel[i];
    std::vector<uint32_t> vals((size_t)(p.rows * o.width));
    split_output(p, i, packed, vals.data());
    if (i) b += ", ";
    json_escape(o.name, &b);
    b += ": ";
    int64_t idx = 0;
    json_nested(o.kind, vals.data(), p.shapes[i], 0, &idx, output_dtype(o.kind) == TFSC_DT_INT64 ? 2 : 1, &b);
  }
  b += "}\n}";
  return b;
}

static int rest_handle_impl(tfsc_server* s, const char* method, const char* url, const void* body, size_t body_len,
                            int* http_status, void** resp, size_t* resp_len) {
  if (!s || !method || !url || !http_status || !resp || !resp_len) return fail(TFSC_E_INVALID, "rest_handle: bad arguments");
  s->req_rest++;  // promRequestsTotal{rest}, tfservingproxy.go:96
  std::string name, version;
  const std::string u(url);
  int st = match_rest_url(u, &name, &version);
  if (st != 200) {  // :99-124
    s->fail_rest++;
    *http_status = st;
    set_resp(rest_error_body(st), resp, resp_len);
    return 0;
  }
  // what follows "/versions/<v>" selects the TF-Serving verb
  size_t vpos = u.find(version, u.find('/', 11));
  std::string tail = u.substr(vpos + version.size());
  size_t qpos = tail.find('?');
  if (qpos != std::string::npos) tail.resize(qpos);
  Node* node;
  ModelId id;
  int remote = -1;
  int rc = resolve(s, name, version, &node, &id, &remote);
  auto fail_http = [&](int code, const std::string& msg) {
    s->fail_rest++;
    *http_status = code;
    set_resp(error_json(msg), resp, resp_len);
    return 0;
  };
  if (rc < 0) return fail_http(http_for(rc), tfsc_last_error());
  std::string err;
  const std::string m(method);
  if (!node && !(m == "POST" && tail == ":predict"))
    // only Predict takes the forward hop; status / metadata of a model are answered by the rank that owns it
    return fail_http(404, "model " + name + " is owned by rank " + std::to_string(remote) + "; ask that rank for " + tail);
  if (m == "GET" && (tail.empty() || tail == "/")) {
    // the request passes through handleModelRequest (fetchModel) before TF-Serving answers
    rc = node->fetch(id, nullptr, &err);
    if (rc < 0) return fail_http(http_for(rc), err);
    int stt = node->status(id);
    std::string b = "{\n \"model_version_status\": [\n  {\n   \"version\": \"" + std::to_string(id.version) +
                    "\",\n   \"state\": \"" + state_name(stt) +
                    "\",\n   \"status\": {\n    \"error_code\": \"OK\",\n    \"error_message\": \"\"\n   }\n  }\n ]\n}\n";
    *http_status = 200;
    set_resp(b, resp, resp_len);
    return 0;
  }
  if (m == "POST" && tail == ":predict") {
    Json req;
    bool parsed = json_parse(std::string((const char*)body, body_len), &req, &err) && req.type == Json::Obj;
    const Json* instances = parsed ? req.get("instances") : nullptr;
    const Json* inputs = parsed ? req.get("inputs") : nullptr;
    std::vector<int64_t> shape;
    std::vector<float> flat;
    std::string input_key;
    // several named inputs (multi-input models, e.g. BERT's input_ids / input_mask / segment_ids): one column per key
    std::vector<std::pair<std::string, Json>> columns;
    bool ok = parsed && ((instances != nullptr) != (inputs != nullptr));
    if (parsed && !ok) err = "JSON body must contain exactly one of 'instances' (row format) or 'inputs' (columnar)";
    if (ok && instances && instances->type == Json::Arr && !instances->arr.empty() && instances->arr[0].type == Json::Obj &&
        instances->arr[0].obj.size() > 1) {
      // row format, {"instances": [{"input_ids": [...], "input_mask": [...]}, ...]}: every instance names the same keys
      for (auto& kv : instances->arr[0].obj) {
        columns.emplace_back(kv.first, Json());
        columns.back().second.type = Json::Arr;
      }
      for (auto& inst : instances->arr) {
        if (inst.type != Json::Obj || inst.obj.size() != columns.size()) {
          ok = false;
          err = "every instance object must name the same inputs";
          break;
        }
        for (auto& col : columns) {
          const Json* v = inst.get(col.first);
          if (!v) {
            ok = false;
            err = "every instance object must name the same inputs (one lacks '" + col.first + "')";
            break;
          }
          col.second.arr.push_back(*v);
        }
        if (!ok) break;
      }
    } else if (ok && inputs && inputs->type == Json::Obj && inputs->obj.size() > 1) {
      // columnar format, {"inputs": {"input_ids": [[...]], "input_mask": [[...]], ...}}
      for (auto& kv : inputs->obj) columns.emplace_back(kv.first, kv.second);
    } else if (ok && instances) {
      const Json* src = instances;
      Json unwrapped;
      // row format: a list of instances; an instance may be {"<input>": value}
      if (instances->type == Json::Arr && !instances->arr.empty() && instances->arr[0].type == Json::Obj) {
        unwrapped.type = Json::Arr;
        for (auto& inst : instances->arr) {
          if (inst.type != Json::Obj || inst.obj.size() != 1) {
            ok = false;
            err = "each instance object must name exactly one input";
            break;
          }
          input_key = inst.obj[0].first;
          unwrapped.arr.push_back(inst.obj[0].second);
        }
        src = &unwrapped;
      }
      if (ok) ok = flatten(*src, 0, &shape, &flat, &err);
    } else if (ok) {
      const Json* src = inputs;
      if (inputs->type == Json::Obj) {
        if (inputs->obj.size() != 1) {
          ok = false;
          err = "'inputs' object must name exactly one input";
        } else {
          input_key = inputs->obj[0].first;
          src = &inputs->obj[0].second;
        }
      }
      if (ok) ok = flatten(*src, 0, &shape, &flat, &err);
    }
    std::vector<std::vector<int64_t>> col_shape(columns.size());
    std::vector<std::vector<int32_t>> col_ints(columns.size());
    for (size_t i = 0; ok && i < columns.size(); ++i) {
      std::vector<float> vals;
      ok = flatten(columns[i].second, 0, &col_shape[i], &vals, &err);
      if (ok && vals.empty()) {
        ok = false;
        err = "input '" + columns[i].first + "' is empty";
      }
      // JSON numbers carry no dtype: the inputs of a multi-input model are int32 (token ids, mask, segment ids)
      col_ints[i].resize(vals.size());
      for (size_t k = 0; k < vals.size(); ++k) col_ints[i][k] = (int32_t)llround((double)vals[k]);
    }
    if (!ok || (flat.empty() && columns.empty())) {
      std::string e2;
      rc = node ? node->fetch(id, nullptr, &e2) : 0;  // residency is ensured before the body is looked at
      if (rc < 0) return fail_http(http_for(rc), e2);
      return fail_http(400, err.empty() ? "empty request" : err);
    }
    std::vector<float> y;
    std::string bad_sig;
    OutputPlan plan;
    std::vector<InTensor> ts(columns.size());
    for (size_t i = 0; i < columns.size(); ++i) {
      ts[i].name = columns[i].first;
      ts[i].dtype = TFSC_DT_INT32;
      ts[i].data = col_ints[i].data();
      ts[i].shape = col_shape[i];
      ts[i].n = (int64_t)col_ints[i].size();
    }
    const InputLayout layout = layout_inputs(&ts);
    if (!ts.empty()) shape = ts[0].shape;  // the batch dimension of the response
    auto alloc = [&](const ModelDesc& d, int64_t rows) -> void* {
      if (!input_matches(d, input_key.empty() ? nullptr : &input_key, &bad_sig)) return nullptr;
      // every output (REST has no output filter), answered in packed order below
      if (!plan_outputs(d, rows, shape, {}, &plan, &bad_sig)) return nullptr;
      y.assign((size_t)(rows * plan.out_dim), 0.f);
      return y.data();
    };
    if (!ts.empty()) rc = run_predict(s, node, remote, id, ts, layout, alloc, &err);
    else rc = run_predict_one(s, node, remote, id, flat.data(), (int64_t)flat.size(), TFSC_DT_FLOAT, alloc, &err);
    if (ts.empty() && rc == TFSC_E_INVALID && err.find("input dtype") == 0) {
      // JSON numbers carry no dtype: the signature wants int32 (token ids) -> resend the same values as integers
      std::vector<int32_t> ints(flat.size());
      for (size_t i = 0; i < flat.size(); ++i) ints[i] = (int32_t)llround((double)flat[i]);
      err.clear();
      rc = run_predict_one(s, node, remote, id, ints.data(), (int64_t)ints.size(), TFSC_DT_INT32, alloc, &err);
    }
    if (rc < 0) return fail_http(bad_sig.empty() ? http_for(rc) : 400, bad_sig.empty() ? err : bad_sig);
    if (plan.declared) {
      *http_status = 200;
      set_resp(rest_multi_output_json(plan, y.data(), instances != nullptr), resp, resp_len);
      return 0;
    }
    // TF-Serving's writer: 4-space indent, arrays on one line, closing bracket on its own line
    const std::vector<int64_t>& oshape = plan.shapes[0];
    std::string b = std::string("{\n    \"") + (instances ? "predictions" : "outputs") + "\": ";
    size_t idx = 0;
    if (oshape.empty()) {
      json_float(y[0], &b);
      b += "\n}";
    } else {
      std::string t;
      write_tensor_json(y.data(), oshape, 0, &idx, &t);
      t.pop_back();  // drop the final ']' and re-emit it TF-Serving style
      b += t + "\n    ]\n}";
    }
    *http_status = 200;
    set_resp(b, resp, resp_len);
    return 0;
  }
  if (m == "GET" && tail == "/metadata") {
    ModelDesc d;
    rc = node->describe(id, &d, nullptr, &err);
    if (rc < 0) return fail_http(http_for(rc), err);
    std::string dim = d.tmpl == Template::Affine ? "" : std::to_string(d.in_dim);
    std::string odim = d.tmpl == Template::Affine ? "" : std::to_string(d.out_dim);
    // the batch dimension -1, then `dims` (none for a scalar per row)
    auto tensor_info = [](const std::string& key, const std::vector<std::string>& dims, const char* dtype) {
      std::string t = "\"" + key + "\": {\"dtype\": \"" + dtype + "\", \"tensor_shape\": {\"dim\": [{\"size\": \"-1\", \"name\": \"\"}";
      for (auto& dim : dims) t += ", {\"size\": \"" + dim + "\", \"name\": \"\"}";
      t += "], \"unknown_rank\": false}, \"name\": \"" + key + ":0\"}";
      return t;
    };
    // every declared input of a multi-input model is DT_INT32 [-1, width]: [-1, S], a seed [-1, 1]
    std::string ins;
    for (auto& mi : d.inputs) ins += (ins.empty() ? "" : ", ") + tensor_info(mi.name, {std::to_string(mi.width)}, "DT_INT32");
    if (d.inputs.empty())
      ins = tensor_info(d.input_name, dim.empty() ? std::vector<std::string>{} : std::vector<std::string>{dim},
                        d.input_dtype == TFSC_DT_INT32 ? "DT_INT32" : "DT_FLOAT");
    // a multi-output model lists every output: logits / probabilities [-1, N], classes [-1] (int64), top-k [-1, k],
    // start / end logits [-1, S], spans [-1, k], sequence_output [-1, S, H], the other encoder outputs [-1, H],
    // masked_positions [-1, M], the fill-mask top-k outputs [-1, M, k]
    std::string outs;
    for (auto& mo : d.outputs) {
      const OutputForm f = output_form(mo.kind, d.head_n, d.head_k);
      std::vector<std::string> dims;
      for (int r = 0; r < f.rank; ++r) dims.push_back(std::to_string(f.dims[r]));
      outs += (outs.empty() ? "" : ", ") + tensor_info(mo.name, dims, dtype_name(f.dtype).c_str());
    }
    if (d.outputs.empty())
      outs = tensor_info(d.output_name, odim.empty() ? std::vector<std::string>{} : std::vector<std::string>{odim}, "DT_FLOAT");
    std::string b = "{\n\"model_spec\": {\"name\": ";
    json_escape(name, &b);
    b += ", \"signature_name\": \"\", \"version\": \"" + std::to_string(id.version) + "\"},\n\"metadata\": {\"signature_def\": {\"signature_def\": {\"serving_default\": {\"inputs\": {" +
         ins + "}, \"outputs\": {" + outs + "}, \"method_name\": \"tensorflow/serving/predict\"}}}}\n}\n";
    *http_status = 200;
    set_resp(b, resp, resp_len);
    return 0;
  }
  if (m == "POST" && (tail == ":classify" || tail == ":regress")) {
    // TF-Serving REST: {"signature_name": ..., "context": {feature: value}, "examples": [{feature: value | [values]}, ...]}
    const int method = tail == ":classify" ? 1 : 2;
    Json req;
    bool parsed = json_parse(std::string((const char*)body, body_len), &req, &err) && req.type == Json::Obj;
    const Json* examples = parsed ? req.get("examples") : nullptr;
    if (!parsed || !examples || examples->type != Json::Arr) {
      std::string e2;
      rc = node->fetch(id, nullptr, &e2);
      if (rc < 0) return fail_http(http_for(rc), e2);
      return fail_http(400, parsed ? "JSON body must contain an 'examples' list" : err);
    }
    ExampleRequestView view;
    view.model_name = name;
    view.version = id.version;
    view.has_version = true;
    view.signature_name = req.get_str("signature_name", "");
    auto add_features = [&](const Json& obj, ExampleView* ex) {
      if (obj.type != Json::Obj) return false;
      for (auto& kv : obj.obj) {
        std::vector<float> vals;
        if (kv.second.type == Json::Num) vals.push_back((float)kv.second.num);
        else if (kv.second.type == Json::Arr) {
          for (auto& e : kv.second.arr)
            if (e.type == Json::Num) vals.push_back((float)e.num);
            else return false;
        } else continue;  // string features are not numeric inputs
        if (!ex->find(kv.first)) ex->features.emplace_back(kv.first, vals);
      }
      return true;
    };
    bool ok = true;
    for (auto& e : examples->arr) {
      ExampleView ex;
      ok = ok && add_features(e, &ex);
      if (const Json* ctx = req.get("context")) ok = ok && add_features(*ctx, &ex);
      view.examples.push_back(std::move(ex));
    }
    if (!ok) return fail_http(400, "examples must be objects mapping feature names to numbers or lists of numbers");
    std::vector<float> scores;
    int64_t n = 0, per = 0;
    ModelId rid;
    std::string sig;
    rc = run_examples(s, view, method, &scores, &n, &per, &rid, &sig, &err);
    if (rc < 0) return fail_http(rc == TFSC_E_INVALID ? 400 : http_for(rc), err);
    std::string b = "{\n    \"results\": [";
    for (int64_t i = 0; i < n; ++i) {
      if (i) b += ", ";
      if (method == 2) {
        json_float(scores[(size_t)i], &b);
      } else {
        b += "[";
        for (int64_t k = 0; k < per; ++k) {
          if (k) b += ", ";
          b += "[\"\", ";
          json_float(scores[(size_t)(i * per + k)], &b);
          b += "]";
        }
        b += "]";
      }
    }
    b += "]\n}";
    *http_status = 200;
    set_resp(b, resp, resp_len);
    return 0;
  }
  return fail_http(400, "Malformed request: " + m + " " + u);
}

tfsc_server* tfsc_server_create(const char* config_json) {
  tfsc_server* out = nullptr;
  guarded("server_create", [&] {
    out = server_create_impl(config_json);
    return 0;
  });
  return out;
}
int tfsc_predict(tfsc_server* s, const char* model_name, const char* version, const tfsc_tensor* in, int n_in,
                 tfsc_tensor* out, int n_out) {
  return guarded("predict", [&] { return predict_impl(s, model_name, version, in, n_in, out, n_out, 0); });
}
int tfsc_predict_deadline(tfsc_server* s, const char* model_name, const char* version, const tfsc_tensor* in, int n_in,
                          tfsc_tensor* out, int n_out, int64_t deadline_ns) {
  return guarded("predict", [&] { return predict_impl(s, model_name, version, in, n_in, out, n_out, deadline_ns); });
}
int tfsc_predict_member(tfsc_server* s, int member, const char* model_name, const char* version, const tfsc_tensor* in, int n_in,
                        tfsc_tensor* out, int n_out, int64_t deadline_ns) {
  return guarded("predict", [&] { return predict_impl(s, model_name, version, in, n_in, out, n_out, deadline_ns, member); });
}
int64_t tfsc_now_ns(void) { return Node::now_ns(); }
int tfsc_grpc_predict(tfsc_server* s, const void* req, size_t req_len, void** resp, size_t* resp_len) {
  return guarded("grpc_predict", [&] { return grpc_predict_impl(s, req, req_len, resp, resp_len); });
}
int tfsc_grpc_classify(tfsc_server* s, const void* req, size_t req_len, void** resp, size_t* resp_len) {
  return guarded("grpc_classify", [&] { return grpc_examples_impl(s, 1, req, req_len, resp, resp_len); });
}
int tfsc_grpc_regress(tfsc_server* s, const void* req, size_t req_len, void** resp, size_t* resp_len) {
  return guarded("grpc_regress", [&] { return grpc_examples_impl(s, 2, req, req_len, resp, resp_len); });
}
int tfsc_grpc_session_run(tfsc_server* s, const void* req, size_t req_len, void** resp, size_t* resp_len) {
  return guarded("grpc_session_run", [&] { return grpc_session_run_impl(s, req, req_len, resp, resp_len); });
}
int tfsc_rest_handle(tfsc_server* s, const char* method, const char* url, const void* body, size_t body_len,
                     int* http_status, void** resp, size_t* resp_len) {
  return guarded("rest_handle", [&] { return rest_handle_impl(s, method, url, body, body_len, http_status, resp, resp_len); });
}

// ---- asynchronous Predict (SURVEY 8b: tfsc_predict_submit / _wait / _release): a cgo handler does not park an OS
// thread per in-flight request. submit = route + ensure-resident + signature checks + staging of the input rows (the
// caller's input buffer is free again when submit returns); the output buffer is written by wait().
struct tfsc_ticket {
  tfsc_server* srv = nullptr;
  Node* node = nullptr;
  PredictRequest req;
  char* staging = nullptr;
  size_t staging_bytes = 0, in_al = 0, out_bytes = 0;
  AbiOutputs outs;
  void* y = nullptr;  // where wait() copies the staged result: outs' destination
  // requests owned by another rank take the (synchronous) forward hop on a helper thread
  std::thread remote_thread;
  std::mutex mu;
  std::condition_variable cv;
  int remote_rc = 1;
  std::string remote_err;
  std::vector<std::vector<char>> remote_x;  // copies of the inputs, so the caller's buffers are free when submit returns
  std::vector<InTensor> remote_ts;
  InputLayout remote_l;
  bool delivered = false;
};

static int submit_impl(tfsc_server* s, const char* model_name, const char* version, const tfsc_tensor* in, int n_in,
                       tfsc_tensor* out, int n_out, int64_t deadline_ns, tfsc_ticket** ticket) {
  if (!s || !model_name || !version || !in || n_in < 1 || !out || n_out < 1 || !ticket)
    return fail(TFSC_E_INVALID, "predict_submit: bad arguments");
  *ticket = nullptr;
  Node* node;
  ModelId id;
  int remote = -1;
  int rc = resolve(s, model_name, version, &node, &id, &remote);
  if (rc < 0) return rc;
  std::vector<InTensor> ts;
  InputLayout layout;
  if ((rc = abi_inputs(in, n_in, true, &ts, &layout)) < 0) return rc;
  auto t = std::make_unique<tfsc_ticket>();
  t->srv = s;
  t->node = node;
  t->outs = AbiOutputs(in[0], ts[0].shape, out, n_out);
  std::string err;
  if (!node) {
    // another rank owns the model: the forward hop is synchronous, run it beside the caller
    for (auto& c : ts) {
      const char* p = static_cast<const char*>(c.data);
      t->remote_x.emplace_back(p, p + (size_t)c.n * 4);
      c.data = t->remote_x.back().data();
    }
    t->remote_ts = ts;
    t->remote_l = layout;
    tfsc_ticket* tp = t.get();
    t->remote_thread = std::thread([tp, s, remote, id, deadline_ns] {
      std::string e2;
      auto alloc = [tp](const ModelDesc& d, int64_t rows) { return tp->outs.alloc(d, rows); };
      int r = s->fwd->forward(remote, id.name, id.version, tp->remote_ts, tp->remote_l, alloc, nullptr, deadline_ns, &e2);
      const std::string& bad = tp->outs.bad;
      std::lock_guard<std::mutex> lk(tp->mu);
      tp->remote_rc = r < 0 && !bad.empty() ? TFSC_E_INVALID : r;
      tp->remote_err = !bad.empty() ? bad : e2;
      tp->cv.notify_all();
    });
    *ticket = t.release();
    return 0;
  }
  rc = node->prepare(id, layout, &t->req, nullptr, &err);
  if (rc < 0) return fail(rc, "%s", err.c_str());
  t->y = t->outs.alloc(t->req.dm->desc, t->req.rows);
  if (!t->y) {
    node->abandon(&t->req);
    if (!t->outs.bad.empty()) return fail(TFSC_E_INVALID, "%s", t->outs.bad.c_str());
    return fail(TFSC_E_BUFFER, "output buffer too small");
  }
  t->out_bytes = (size_t)(t->req.rows * t->outs.plan.out_dim) * 4;
  t->in_al = ((size_t)layout.n_elems * 4 + 255) & ~(size_t)255;
  t->staging_bytes = t->in_al + t->out_bytes;
  t->staging = static_cast<char*>(node->staging_alloc(t->staging_bytes));
  if (!t->staging) {
    node->abandon(&t->req);
    return fail(TFSC_E_EXHAUSTED, "cannot pin %zu bytes of request staging", t->staging_bytes);
  }
  pack_rows(ts, layout, t->req.rows, t->staging);  // one tensor: the same bytes as a memcpy of it
  t->req.x = t->staging;
  t->req.y = t->staging + t->in_al;
  t->req.host_staged = true;
  t->req.deadline_ns = deadline_ns;
  node->enqueue(&t->req);
  *ticket = t.release();
  return 0;
}

static int wait_impl(tfsc_ticket* t, int64_t timeout_ns) {
  if (!t) return fail(TFSC_E_INVALID, "predict_wait: null ticket");
  int rc;
  std::string err;
  if (!t->node) {
    std::unique_lock<std::mutex> lk(t->mu);
    auto pred = [&] { return t->remote_rc != 1; };
    if (timeout_ns < 0) t->cv.wait(lk, pred);
    else if (!t->cv.wait_for(lk, std::chrono::nanoseconds(timeout_ns), pred))
      return fail(TFSC_E_TIMEOUT, "predict_wait: request still in flight");
    rc = t->remote_rc;
    err = t->remote_err;
  } else {
    std::unique_lock<std::mutex> lk(t->req.mu);
    auto pred = [&] { return t->req.rc != 1; };
    if (timeout_ns < 0) t->req.cv.wait(lk, pred);
    else if (!t->req.cv.wait_for(lk, std::chrono::nanoseconds(timeout_ns), pred))
      return fail(TFSC_E_TIMEOUT, "predict_wait: request still in flight");
    rc = t->req.rc;
    err = t->req.err;
  }
  if (rc < 0) return fail(rc, "%s", err.c_str());
  if (!t->delivered) {
    if (t->node) memcpy(t->y, t->staging + t->in_al, t->out_bytes);  // a forwarded result is already in place
    t->outs.deliver();
    t->delivered = true;
  }
  return 0;
}

int tfsc_predict_submit(tfsc_server* s, const char* model_name, const char* version, const tfsc_tensor* in, int n_in,
                        tfsc_tensor* out, int n_out, int64_t deadline_ns, tfsc_ticket** ticket) {
  return guarded("predict_submit", [&] { return submit_impl(s, model_name, version, in, n_in, out, n_out, deadline_ns, ticket); });
}
int tfsc_predict_wait(tfsc_ticket* t, int64_t timeout_ns) {
  return guarded("predict_wait", [&] { return wait_impl(t, timeout_ns); });
}
void tfsc_predict_release(tfsc_ticket* t) {
  if (!t) return;
  if (t->node) {
    {  // the batcher / kernels may still use the staging buffer: wait for the request to retire
      std::unique_lock<std::mutex> lk(t->req.mu);
      t->req.cv.wait(lk, [&] { return t->req.rc != 1; });
    }
    t->node->staging_free(t->staging, t->staging_bytes);
  } else if (t->remote_thread.joinable()) {
    t->remote_thread.join();
  }
  delete t;
}

// ---- forward window (a6 / X7 across processes) ----
int tfsc_fwd_window(tfsc_server* s, void** dev_ptr, size_t* bytes, size_t* slot_bytes) {
  if (!s || !s->fwd) return fail(TFSC_E_INVALID, "fwd_window: the server has no cluster.endpoints");
  if (dev_ptr) *dev_ptr = s->fwd->window();
  if (bytes) *bytes = s->fwd->window_bytes();
  if (slot_bytes) *slot_bytes = s->fwd->slot_bytes();
  return s->fwd->rank();
}
int tfsc_device_memcpy(void* dst, const void* src, size_t nbytes) {
  cudaError_t e = cudaMemcpy(dst, src, nbytes, cudaMemcpyDefault);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(TFSC_E_INTERNAL, "device_memcpy: %s", cudaGetErrorString(e));
  }
  return 0;
}
int tfsc_fwd_peer_window(tfsc_server* s, int peer_rank, void** dev_ptr, size_t* bytes) {
  if (!s || !s->fwd || !dev_ptr) return fail(TFSC_E_INVALID, "fwd_peer_window: bad arguments / no cluster.endpoints");
  return guarded("fwd_peer_window", [&] {
    std::string err;
    char* p = s->fwd->peer_window(peer_rank, bytes, &err);
    if (!p) return fail(TFSC_E_INTERNAL, "%s", err.c_str());
    *dev_ptr = p;
    return 0;
  });
}

int tfsc_predict_device(tfsc_server* s, int node, const char* model_name, int64_t version, const void* x,
                        int64_t rows, void* y, void* stream) {
  Node* n = node_at(s, node);
  if (!n || !model_name) return TFSC_E_INVALID;
  std::string err;
  int rc = n->predict_device({model_name, version}, x, rows, y, (cudaStream_t)stream, &err);
  if (rc < 0) return fail(rc, "%s", err.c_str());
  return 0;
}

int tfsc_node_set_max_resident(tfsc_server* s, int node, int max_concurrent_models) {
  Node* n = node_at(s, node);
  if (!n) return TFSC_E_INVALID;
  if (max_concurrent_models < 1) return fail(TFSC_E_INVALID, "serving.maxConcurrentModels must be >= 1");
  n->set_max_concurrent_models(max_concurrent_models);
  return 0;
}

int tfsc_k_copy_segments(const tfsc_copy_seg* segs, int n, void* stream) {
  if (int rc = check_device()) return rc;
  if (!segs || n < 0) return fail(TFSC_E_INVALID, "copy_segments: bad arguments");
  static_assert(sizeof(tfsc_copy_seg) == sizeof(CopySeg), "ABI struct mirrors the kernel's segment");
  cudaError_t e = launch_copy_segments(reinterpret_cast<const CopySeg*>(segs), n, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "copy_segments: %s", cudaGetErrorString(e));
}

int tfsc_node_sync(tfsc_server* s, int node) {
  Node* n = node_at(s, node);
  if (!n) return TFSC_E_INVALID;
  return n->sync();
}

int tfsc_get_stats(tfsc_server* s, int node, tfsc_stats* out) {
  if (!s || !out) return fail(TFSC_E_INVALID, "get_stats: bad arguments");
  memset(out, 0, sizeof *out);
  if (node >= 0) {
    Node* n = node_at(s, node);
    if (!n) return TFSC_E_INVALID;
    n->stats(out);
  } else {
    for (auto& n : s->nodes) n->stats(out);
  }
  out->proxy_requests_rest = s->req_rest;
  out->proxy_requests_grpc = s->req_grpc;
  out->proxy_failures_rest = s->fail_rest;
  out->proxy_failures_grpc = s->fail_grpc;
  out->kernel_launches = kernel_launch_count();
  if (s->fwd) {
    const FwdStats& f = s->fwd->stats();
    out->fwd_out_requests = f.out_requests;
    out->fwd_in_requests = f.in_requests;
    out->fwd_out_failures = f.out_failures;
    out->fwd_peer_bytes_read = f.peer_bytes_read;
    out->fwd_peer_bytes_written = f.peer_bytes_written;
    out->fwd_rtt_seconds_sum = (double)f.rtt_ns_sum * 1e-9;
  }
  return 0;
}

// ------------------------------------------------------------------ raw kernel entries ------
int tfsc_k_affine(const float* x, float* y, int64_t n, const float* a, const float* b, void* stream) {
  if (int rc = check_device()) return rc;
  cudaError_t e = launch_affine(x, y, n, a, b, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "affine: %s", cudaGetErrorString(e));
}

int tfsc_k_dense(const float* x, const float* w, const float* b, float* y, int rows, int k, int n, int relu,
                 float* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = check_device()) return rc;
  cudaError_t e = launch_dense(x, w, b, y, rows, k, n, relu != 0, workspace, workspace_bytes, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "dense: %s", cudaGetErrorString(e));
}

size_t tfsc_k_dense_workspace(int rows, int k, int n) { return dense_workspace_bytes(rows, k, n); }

int tfsc_k_dense_variant(int variant, const float* x, const float* w, const float* b, float* y, int rows, int k, int n,
                         int relu, float* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = check_device()) return rc;
  if (variant < 0 || variant > 5) return fail(TFSC_E_INVALID, "dense: variant %d not in 0..5", variant);
  cudaError_t e = launch_dense(x, w, b, y, rows, k, n, relu != 0, workspace, workspace_bytes, (cudaStream_t)stream, variant);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "dense(variant %d): %s", variant, cudaGetErrorString(e));
}

int tfsc_k_dense_cluster_grid(int rows, int n, int* active_clusters, int* strip_cols) {
  if (int rc = check_device()) return rc;
  if (rows < 1 || rows > 8 || n < 1 || !active_clusters || !strip_cols) return fail(TFSC_E_INVALID, "dense_cluster_grid: rows in 1..8, n >= 1");
  cudaError_t e = dense_cluster_grid(rows, n, active_clusters, strip_cols);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "dense_cluster_grid: %s", cudaGetErrorString(e));
}

int tfsc_k_dense_tc(const float* x, const float* w, const float* b, float* y, int rows, int k, int n, int relu,
                    float* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = check_device()) return rc;
  if (!dense_tc_supported(rows, k, n, w, x, b, y))
    return fail(TFSC_E_INVALID, "dense_tc: unsupported shape/alignment (rows<=64, n%%32==0, k%%4==0, 16B-aligned)");
  cudaError_t e = launch_dense_tc(x, w, b, y, rows, k, n, relu != 0, workspace, workspace_bytes, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "dense_tc: %s", cudaGetErrorString(e));
}

int tfsc_k_gemm(const float* a, const float* b, const float* bias, const float* r, float* c, int m, int n, int k, int lda,
                int act, void* stream) {
  if (int rc = check_device()) return rc;
  cudaError_t e = launch_gemm(a, b, bias, r, c, m, n, k, lda, act, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "gemm: %s", cudaGetErrorString(e));
}
int tfsc_k_gemm_tc(const float* a, const float* b, const float* bias, const float* r, float* c, int m, int n, int k, int lda,
                   int act, void* stream) {
  if (int rc = check_device()) return rc;
  if (!gemm_tc_supported(a, b, bias, r, c, m, n, k, lda))
    return fail(TFSC_E_INVALID, "gemm_tc: unsupported shape/alignment (m>=64, n>=64, n%%32==0, k>=32, lda%%4==0, 16B-aligned)");
  cudaError_t e = launch_gemm_tc(a, b, bias, r, c, m, n, k, lda, act, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "gemm_tc: %s", cudaGetErrorString(e));
}
int tfsc_k_conv_tc(const float* x, const float* w, const float* bias, const float* r, float* y, int batch, int h, int wd, int c,
                   int kh, int kw, int stride, int pad, int cout, int act, void* stream) {
  if (int rc = check_device()) return rc;
  const int oh = (h + 2 * pad - kh) / stride + 1, ow = (wd + 2 * pad - kw) / stride + 1;
  if (!conv_tc_supported(x, w, bias, r, y, batch, h, wd, c, kh, kw, stride, pad, oh, ow, cout))
    return fail(TFSC_E_INVALID, "conv_tc: unsupported shape/alignment (c %% 32 == 0, cout >= 64 and %% 32 == 0, batch*oh*ow >= 64, 16B-aligned)");
  cudaError_t e = launch_conv_tc(x, w, bias, r, y, batch, h, wd, c, kh, kw, stride, pad, oh, ow, cout, act, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "conv_tc: %s", cudaGetErrorString(e));
}
int tfsc_k_im2col(const float* x, float* col, int batch, int h, int w, int c, int kh, int kw, int stride, int pad, int ldc,
                  void* stream) {
  if (int rc = check_device()) return rc;
  const int oh = (h + 2 * pad - kh) / stride + 1, ow = (w + 2 * pad - kw) / stride + 1;
  cudaError_t e = launch_im2col(x, col, batch, h, w, c, kh, kw, stride, pad, oh, ow, ldc, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "im2col: %s", cudaGetErrorString(e));
}
int tfsc_k_maxpool(const float* x, float* y, int batch, int h, int w, int c, int kh, int kw, int stride, int pad, void* stream) {
  if (int rc = check_device()) return rc;
  const int oh = (h + 2 * pad - kh) / stride + 1, ow = (w + 2 * pad - kw) / stride + 1;
  cudaError_t e = launch_maxpool(x, y, batch, h, w, c, kh, kw, stride, pad, oh, ow, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "maxpool: %s", cudaGetErrorString(e));
}
int tfsc_k_avgpool(const float* x, float* y, int batch, int hw, int c, void* stream) {
  if (int rc = check_device()) return rc;
  cudaError_t e = launch_avgpool(x, y, batch, hw, c, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "avgpool: %s", cudaGetErrorString(e));
}
int tfsc_k_depthwise_conv(const float* x, const float* w, const float* bias, float* y, int batch, int h, int wd, int c, int kh, int kw,
                          int stride, int pad, int act, void* stream) {
  if (int rc = check_device()) return rc;
  if (!x || !w || !bias || !y || batch < 0 || !depthwise_supported(h, wd, c, kh, kw, stride, pad))
    return fail(TFSC_E_INVALID, "depthwise_conv: no kernel for batch %d, %d x %d x %d, kernel %d x %d, stride %d, pad %d (kernel <= %d, "
                "stride <= %d, pad <= kernel / 2, h * w * c < 2^31)", batch, h, wd, c, kh, kw, stride, pad, kDepthwiseMaxK,
                kDepthwiseMaxStride);
  if (!(act == 0 || act == 1 || (act >= 4 && act <= 6)))
    return fail(TFSC_E_INVALID, "depthwise_conv: act %d is not 0 none, 1 relu, 4 relu6, 5 silu or 6 sigmoid", act);
  cudaError_t e = launch_depthwise_conv(x, w, bias, y, batch, h, wd, c, kh, kw, stride, pad, act, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "depthwise_conv: %s", cudaGetErrorString(e));
}
int tfsc_k_channel_scale(const float* x, const float* gate, float* y, int batch, int hw, int c, void* stream) {
  if (int rc = check_device()) return rc;
  if (!x || !gate || !y || batch < 0 || hw < 1 || c < 1 || (int64_t)hw * c > 0x7fffffff)
    return fail(TFSC_E_INVALID, "channel_scale: no kernel for batch %d, hw %d, c %d (hw * c < 2^31)", batch, hw, c);
  cudaError_t e = launch_channel_scale(x, gate, y, batch, hw, c, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "channel_scale: %s", cudaGetErrorString(e));
}
int tfsc_k_window_attention(const float* qkv, const float* bias, float* ctx, int batch, int h, int w, int c, int heads, int window,
                            int shift, void* stream) {
  if (int rc = check_device()) return rc;
  if (!qkv || !bias || !ctx || batch < 0 || !window_attention_supported(h, w, c, heads, window, shift))
    return fail(TFSC_E_INVALID, "window_attention: no kernel for batch %d, %d x %d, c %d, %d heads, window %d, shift %d (h, w multiples "
                "of window <= %d, 0 <= shift < window, head width <= %d, K and V of a window within 48 KB, h * w * 3c < 2^31)",
                batch, h, w, c, heads, window, shift, kWindowMaxWs, kWindowMaxD);
  cudaError_t e = launch_window_attention(qkv, bias, ctx, batch, h, w, c, heads, window, shift, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "window_attention: %s", cudaGetErrorString(e));
}
int tfsc_k_patch_merge(const float* x, float* y, int batch, int h, int w, int c, void* stream) {
  if (int rc = check_device()) return rc;
  if (!x || !y || batch < 0 || !patch_merge_supported(h, w, c))
    return fail(TFSC_E_INVALID, "patch_merge: no kernel for batch %d, %d x %d x %d (even h and w, h * w * c < 2^31)", batch, h, w, c);
  cudaError_t e = launch_patch_merge(x, y, batch, h, w, c, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "patch_merge: %s", cudaGetErrorString(e));
}
int tfsc_k_attention(const float* qkv, const int* ids, float* ctx, int batch, int seq, int hidden, int heads, void* stream) {
  if (int rc = check_device()) return rc;
  const bool al = ((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(ctx)) & 15) == 0;
  if (!qkv || !ctx || batch < 1 || (int64_t)batch * heads > 0x7fffffff || !attention_supported(seq, hidden, heads, al))
    return fail(TFSC_E_INVALID, "attention: no kernel for batch %d, seq %d, hidden %d, heads %d", batch, seq, hidden, heads);
  cudaError_t e = launch_attention(qkv, ids, seq, ctx, batch, seq, hidden, heads, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "attention: %s", cudaGetErrorString(e));
}
int tfsc_k_attention_mask(const float* qkv, const int* mask, int mask_stride, float* ctx, int batch, int seq, int hidden, int heads,
                          void* stream) {
  if (int rc = check_device()) return rc;
  const bool al = ((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(ctx)) & 15) == 0;
  if (!qkv || !ctx || batch < 1 || (int64_t)batch * heads > 0x7fffffff || !attention_supported(seq, hidden, heads, al))
    return fail(TFSC_E_INVALID, "attention_mask: no kernel for batch %d, seq %d, hidden %d, heads %d", batch, seq, hidden, heads);
  if (mask && mask_stride < seq) return fail(TFSC_E_INVALID, "attention_mask: mask_stride %d is below seq %d", mask_stride, seq);
  cudaError_t e = launch_attention(qkv, mask, mask_stride, ctx, batch, seq, hidden, heads, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "attention_mask: %s", cudaGetErrorString(e));
}
int tfsc_k_embed(const int* ids, const int* types, int stride, const float* word, const float* pos, const float* type,
                 const float* gamma, const float* beta, float* y, int batch, int seq, int hidden, int vocab, float eps, void* stream) {
  if (int rc = check_device()) return rc;
  if (!ids || !word || !pos || !type || !gamma || !beta || !y || batch < 0 || seq < 1 || vocab < 1 ||
      (int64_t)batch * seq > 0x7fffffff || !layernorm_supported(hidden))
    return fail(TFSC_E_INVALID, "embed: no kernel for batch %d, seq %d, hidden %d, vocab %d (hidden in 1..12272)", batch, seq, hidden,
                vocab);
  if (stride < seq) return fail(TFSC_E_INVALID, "embed: stride %d is below seq %d", stride, seq);
  cudaError_t e = launch_layernorm(nullptr, nullptr, ids, types, stride, word, pos, type, gamma, beta, y, batch * seq, seq, hidden,
                                   vocab, eps, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "embed: %s", cudaGetErrorString(e));
}
int tfsc_k_layernorm(const float* x, const float* res, const float* gamma, const float* beta, float* y, int tokens, int hidden,
                     float eps, void* stream) {
  if (int rc = check_device()) return rc;
  if (!x || !gamma || !beta || !y || tokens < 0 || !layernorm_supported(hidden))
    return fail(TFSC_E_INVALID, "layernorm: no kernel for %d tokens of hidden %d (hidden in 1..12272)", tokens, hidden);
  cudaError_t e = launch_layernorm(x, res, nullptr, nullptr, 0, nullptr, nullptr, nullptr, gamma, beta, y, tokens, 1, hidden, 0, eps,
                                   (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "layernorm: %s", cudaGetErrorString(e));
}
int tfsc_k_classify_head(const float* logits, int rows, int n, int k, float* probs, int64_t* classes, int32_t* topk_idx,
                         float* topk_prob, void* stream) {
  if (int rc = check_device()) return rc;
  if (!logits || rows < 0 || !head_supported(n, k))
    return fail(TFSC_E_INVALID, "classify_head: no kernel for %d rows of %d logits, k = %d (1 <= n <= %d, 1 <= k <= min(n, %d))", rows,
                n, k, kHeadMaxN, kHeadMaxK);
  HeadOutputs o;
  o.probs = probs;
  o.probs_ld = n;
  o.classes = reinterpret_cast<int*>(classes);
  o.classes_ld = 2;
  o.topk_idx = topk_idx;
  o.topk_idx_ld = k;
  o.topk_prob = topk_prob;
  o.topk_prob_ld = k;
  cudaError_t e = launch_classify_head(logits, rows, n, k, o, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "classify_head: %s", cudaGetErrorString(e));
}
int tfsc_k_span_head(const float* logits, const int32_t* ids, const int32_t* mask, const int32_t* types, int stride, int rows, int S,
                     int max_answer_length, int k, int sep_id, float* start_logits, float* end_logits, int32_t* span_starts,
                     int32_t* span_ends, float* span_scores, void* stream) {
  if (int rc = check_device()) return rc;
  const bool spans = span_starts || span_ends || span_scores;
  if (!logits || rows < 0 || !span_supported(S, spans ? max_answer_length : 1, spans ? k : 1))
    return fail(TFSC_E_INVALID, "span_head: no kernel for %d rows of S = %d, max_answer_length = %d, k = %d (1 <= S <= %d, "
                "1 <= max_answer_length <= S, 1 <= k <= %d)", rows, S, max_answer_length, k, kSpanMaxS, kSpanMaxK);
  if (spans && (!ids || !types || stride < S))
    return fail(TFSC_E_INVALID, "span_head: spans need the ids and the segment ids, stride >= S (%d < %d)", stride, S);
  SpanInputs in;
  in.ids = ids;
  in.mask = mask;
  in.types = types;
  in.stride = stride;
  in.sep_id = sep_id < 0 ? -1 : sep_id;
  SpanOutputs o;
  o.start_logits = start_logits;
  o.start_ld = S;
  o.end_logits = end_logits;
  o.end_ld = S;
  o.starts = span_starts;
  o.starts_ld = k;
  o.ends = span_ends;
  o.ends_ld = k;
  o.scores = span_scores;
  o.scores_ld = k;
  cudaError_t e = launch_span_head(logits, in, rows, S, max_answer_length, k, o, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "span_head: %s", cudaGetErrorString(e));
}
int tfsc_k_encoder_head(const float* hidden, const float* pooled, const int32_t* ids, const int32_t* mask, int stride, int rows, int S,
                        int H, int normalize_cls, int normalize_mean, float* sequence_output, float* pooled_output,
                        float* cls_embedding, float* mean_embedding, void* stream) {
  if (int rc = check_device()) return rc;
  if (rows < 0 || !encoder_head_supported(S, H))
    return fail(TFSC_E_INVALID, "encoder_head: no kernel for %d rows of S = %d, H = %d (1 <= S <= %d, 1 <= H <= %d)", rows, S, H,
                kEncoderMaxS, kEncoderMaxH);
  if (!hidden && (sequence_output || cls_embedding || mean_embedding))
    return fail(TFSC_E_INVALID, "encoder_head: sequence_output, cls_embedding and mean_embedding need the hidden states");
  if (!pooled && pooled_output) return fail(TFSC_E_INVALID, "encoder_head: pooled_output needs the pooler output");
  if (mean_embedding && (!ids || stride < S))
    return fail(TFSC_E_INVALID, "encoder_head: mean_embedding needs the ids, stride >= S (%d < %d)", stride, S);
  EncoderInputs in;
  in.ids = ids;
  in.mask = mask;
  in.stride = stride;
  EncoderOutputs o;
  o.sequence = sequence_output;
  o.sequence_ld = (int64_t)S * H;
  o.pooled = pooled_output;
  o.pooled_ld = H;
  o.cls = cls_embedding;
  o.cls_ld = H;
  o.mean = mean_embedding;
  o.mean_ld = H;
  o.normalize_cls = normalize_cls != 0;
  o.normalize_mean = normalize_mean != 0;
  cudaError_t e = launch_encoder_head(hidden, pooled, in, rows, S, H, o, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "encoder_head: %s", cudaGetErrorString(e));
}
int tfsc_k_mask_gather(const float* hidden, const int32_t* ids, const int32_t* mask, int stride, int rows, int S, int H, int slots,
                       int mask_token_id, int32_t* positions, float* gathered, void* stream) {
  if (int rc = check_device()) return rc;
  if (rows < 0 || !mask_gather_supported(S, H, slots))
    return fail(TFSC_E_INVALID, "mask_gather: no kernel for %d rows of S = %d, H = %d, M = %d (1 <= M <= S <= %d, 1 <= H <= %d)",
                rows, S, H, slots, kMaskGatherMaxS, kMaskGatherMaxH);
  if (!ids || stride < S) return fail(TFSC_E_INVALID, "mask_gather: needs the ids, stride >= S (%d < %d)", stride, S);
  if (gathered && !hidden) return fail(TFSC_E_INVALID, "mask_gather: the gathered rows need the hidden states");
  cudaError_t e = launch_mask_gather(hidden, ids, mask, stride, rows, S, H, slots, mask_token_id, positions, gathered,
                                     (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "mask_gather: %s", cudaGetErrorString(e));
}
int tfsc_k_fill_mask_head(const float* logits, int64_t ld, const int32_t* positions, int rows, int slots, int vocab, int k,
                          int32_t* top_ids, float* top_probs, float* top_logits, void* stream) {
  if (int rc = check_device()) return rc;
  if (rows < 0 || !fill_mask_supported(slots, vocab, k))
    return fail(TFSC_E_INVALID, "fill_mask_head: no kernel for %d rows of M = %d, vocab = %d, k = %d (1 <= M <= %d, 1 <= vocab <= %d, "
                "1 <= k <= min(vocab, %d))", rows, slots, vocab, k, kMaskGatherMaxS, kHeadMaxN, kHeadMaxK);
  if (!positions || ((top_ids || top_probs || top_logits) && (!logits || ld < vocab)))
    return fail(TFSC_E_INVALID, "fill_mask_head: needs the positions and the logits, ld >= vocab (%lld < %d)", (long long)ld, vocab);
  FillMaskOutputs o;
  o.ids = top_ids;
  o.ids_ld = (int64_t)slots * k;
  o.probs = top_probs;
  o.probs_ld = (int64_t)slots * k;
  o.logits = top_logits;
  o.logits_ld = (int64_t)slots * k;
  cudaError_t e = launch_fill_mask_head(logits, ld, positions, rows, slots, vocab, k, kHeadMaxN, o, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "fill_mask_head: %s", cudaGetErrorString(e));
}
int tfsc_k_attention_causal(const float* qkv, const int* mask, int mask_stride, float* ctx, int batch, int seq, int hidden, int heads,
                            void* stream) {
  if (int rc = check_device()) return rc;
  const bool al = ((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(ctx)) & 15) == 0;
  if (!qkv || !ctx || batch < 1 || (int64_t)batch * heads > 0x7fffffff || !attention_causal_supported(seq, hidden, heads, al))
    return fail(TFSC_E_INVALID, "attention_causal: no kernel for batch %d, seq %d, hidden %d, heads %d (d %% 4 == 0, d <= 128, "
                "16-byte aligned qkv / ctx)", batch, seq, hidden, heads);
  if (mask && mask_stride < seq) return fail(TFSC_E_INVALID, "attention_causal: mask_stride %d is below seq %d", mask_stride, seq);
  cudaError_t e = launch_attention_causal(qkv, mask, mask_stride, ctx, batch, seq, hidden, heads, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "attention_causal: %s", cudaGetErrorString(e));
}
int tfsc_k_embed_positions(const int32_t* ids, int stride, const float* word, const float* pos, float* y, int batch, int seq, int hidden,
                           int vocab, void* stream) {
  if (int rc = check_device()) return rc;
  if (!ids || !word || !pos || !y || batch < 0 || seq < 1 || hidden < 1 || vocab < 1)
    return fail(TFSC_E_INVALID, "embed_positions: no kernel for batch %d, seq %d, hidden %d, vocab %d", batch, seq, hidden, vocab);
  if (stride < seq) return fail(TFSC_E_INVALID, "embed_positions: stride %d is below seq %d", stride, seq);
  cudaError_t e = launch_embed_positions(ids, stride, word, pos, y, batch, seq, hidden, vocab, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "embed_positions: %s", cudaGetErrorString(e));
}
int tfsc_k_last_token(const float* hidden, const int32_t* mask, int stride, int rows, int S, int H, int32_t* positions, float* gathered,
                      void* stream) {
  if (int rc = check_device()) return rc;
  if (rows < 0 || S < 1 || H < 1 || (gathered && !hidden))
    return fail(TFSC_E_INVALID, "last_token: no kernel for %d rows of S = %d, H = %d (the gathered rows need the hidden states)",
                rows, S, H);
  if (mask && stride < S) return fail(TFSC_E_INVALID, "last_token: stride %d is below S %d", stride, S);
  cudaError_t e = launch_last_token(hidden, mask, stride, rows, S, H, positions, gathered, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "last_token: %s", cudaGetErrorString(e));
}
int tfsc_k_next_token_head(const float* logits, int64_t ld, const int32_t* positions, int rows, int vocab, int k, int32_t* top_ids,
                           float* top_probs, float* top_logits, void* stream) {
  if (int rc = check_device()) return rc;
  if (rows < 0 || !next_token_supported(vocab, k))
    return fail(TFSC_E_INVALID, "next_token_head: no kernel for %d rows of vocab = %d, k = %d (1 <= vocab <= %d, 1 <= k <= min(vocab, %d))",
                rows, vocab, k, kNextTokenMaxVocab, kHeadMaxK);
  if (!positions || ((top_ids || top_probs || top_logits) && (!logits || ld < vocab)))
    return fail(TFSC_E_INVALID, "next_token_head: needs the positions and the logits, ld >= vocab (%lld < %d)", (long long)ld, vocab);
  FillMaskOutputs o;
  o.ids = top_ids;
  o.ids_ld = k;
  o.probs = top_probs;
  o.probs_ld = k;
  o.logits = top_logits;
  o.logits_ld = k;
  cudaError_t e = launch_fill_mask_head(logits, ld, positions, rows, 1, vocab, k, kNextTokenMaxVocab, o, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "next_token_head: %s", cudaGetErrorString(e));
}
int tfsc_k_kv_cache_write(const float* qkv, float* kc, float* vc, int rows, int S, int T, int H, void* stream) {
  if (int rc = check_device()) return rc;
  if (!qkv || !kc || !vc || rows < 0 || S < 1 || T < S || H < 1)
    return fail(TFSC_E_INVALID, "kv_cache_write: no kernel for %d rows of S = %d, T = %d, H = %d", rows, S, T, H);
  cudaError_t e = launch_kv_cache_write(qkv, kc, vc, rows, S, T, H, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "kv_cache_write: %s", cudaGetErrorString(e));
}
int64_t tfsc_k_decode_attention_work_bytes(int rows, int L, int H, int heads) {
  if (rows < 0 || !decode_attention_supported(L, H, heads)) return -1;
  return (int64_t)decode_attention_work_bytes(rows, L, H, heads);
}
int tfsc_k_decode_attention(const float* qkv, float* kc, float* vc, const int32_t* pos, int t, const int32_t* mask, int mask_stride,
                            int S, int T, float* ctx, int rows, int H, int heads, void* work, int64_t work_bytes, void* stream) {
  if (int rc = check_device()) return rc;
  const int L = S + t + 1;
  if (!qkv || !kc || !vc || !pos || !ctx || !work || rows < 0 || t < 0 || S < 1 || L > T || !decode_attention_supported(L, H, heads))
    return fail(TFSC_E_INVALID, "decode_attention: no kernel for %d rows, S = %d, t = %d, T = %d, hidden %d, heads %d (1 <= S + t + 1"
                " <= min(T, %d), d %% 4 == 0, d <= 128)", rows, S, t, T, H, heads, kDecodeMaxKeys);
  if (mask && mask_stride < S) return fail(TFSC_E_INVALID, "decode_attention: mask_stride %d is below S %d", mask_stride, S);
  if (work_bytes < (int64_t)decode_attention_work_bytes(rows, L, H, heads))
    return fail(TFSC_E_INVALID, "decode_attention: work_bytes %lld is below %lld", (long long)work_bytes,
                (long long)decode_attention_work_bytes(rows, L, H, heads));
  cudaError_t e = launch_decode_attention(qkv, kc, vc, pos, t, mask, mask_stride, S, T, ctx, rows, H, heads, work, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "decode_attention: %s", cudaGetErrorString(e));
}
int tfsc_k_generate_select(const float* logits, int64_t ld, int vocab, const int32_t* pos, int t, int last, int eos, int32_t* done,
                           int32_t* ids, int64_t ids_ld, float* log_probs, int64_t lp_ld, int32_t* length, int64_t length_ld,
                           const float* word, const float* pos_table, float* y, int rows, int H, void* stream) {
  if (int rc = check_device()) return rc;
  if (!logits || !pos || !done || rows < 0 || t < 0 || vocab < 1 || vocab > kNextTokenMaxVocab || ld < vocab || H < 1 ||
      (!last && (!word || !pos_table || !y)))
    return fail(TFSC_E_INVALID, "generate_select: no kernel for %d rows of vocab = %d, ld = %lld, H = %d (1 <= vocab <= %d, ld >= vocab,"
                " the tables and y unless last)", rows, vocab, (long long)ld, H, kNextTokenMaxVocab);
  GenerateOutputs o;
  o.ids = ids;
  o.ids_ld = ids_ld;
  o.log_probs = log_probs;
  o.log_probs_ld = lp_ld;
  o.length = length;
  o.length_ld = length_ld;
  cudaError_t e = launch_generate_select(logits, ld, vocab, pos, t, last != 0, eos, done, o, word, pos_table, y, rows, H,
                                         (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "generate_select: %s", cudaGetErrorString(e));
}
int tfsc_k_generate_sample(const float* logits, int64_t ld, int vocab, const int32_t* pos, int t, int last, int eos, int32_t* done,
                           int32_t* ids, int64_t ids_ld, float* log_probs, int64_t lp_ld, int32_t* length, int64_t length_ld,
                           const float* word, const float* pos_table, float* y, int rows, int H, const int32_t* seeds,
                           int64_t seed_stride, float temperature, int top_k, float top_p, void* stream) {
  if (int rc = check_device()) return rc;
  if (!logits || !pos || !done || rows < 0 || t < 0 || vocab < 1 || vocab > kNextTokenMaxVocab || ld < vocab || H < 1 ||
      (!last && (!word || !pos_table || !y)) || !seeds || seed_stride < 1)
    return fail(TFSC_E_INVALID, "generate_sample: no kernel for %d rows of vocab = %d, ld = %lld, H = %d, seed_stride = %lld (1 <="
                " vocab <= %d, ld >= vocab, seeds and seed_stride >= 1, the tables and y unless last)", rows, vocab, (long long)ld, H,
                (long long)seed_stride, kNextTokenMaxVocab);
  if (!sampling_supported(vocab, temperature, top_k, top_p))
    return fail(TFSC_E_INVALID, "generate_sample: temperature = %g, top_k = %d, top_p = %g (a finite temperature > 0 with a finite"
                " reciprocal, 0 <= top_k <= vocab = %d, 0 < top_p <= 1)", (double)temperature, top_k, (double)top_p, vocab);
  GenerateOutputs o;
  o.ids = ids;
  o.ids_ld = ids_ld;
  o.log_probs = log_probs;
  o.log_probs_ld = lp_ld;
  o.length = length;
  o.length_ld = length_ld;
  cudaError_t e = launch_generate_sample(logits, ld, vocab, pos, t, last != 0, eos, done, o, word, pos_table, y, rows, H, seeds,
                                         seed_stride, temperature, top_k, top_p, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "generate_sample: %s", cudaGetErrorString(e));
}
int tfsc_k_generate_process(const float* logits, int64_t ld, int vocab, const int32_t* pos, int t, int last, int eos, int32_t* done,
                            int32_t* ids, int64_t ids_ld, float* log_probs, int64_t lp_ld, int32_t* length, int64_t length_ld,
                            const float* word, const float* pos_table, float* y, int rows, int H, const int32_t* prompt_ids,
                            const int32_t* mask, int64_t stride, int32_t* hist, int64_t hist_ld, int32_t* hist_len0,
                            float repetition_penalty, int no_repeat_ngram_size, int min_new_tokens, const int32_t* seeds,
                            int64_t seed_stride, float temperature, int top_k, float top_p, void* stream) {
  if (int rc = check_device()) return rc;
  if (!logits || !pos || !done || rows < 0 || t < 0 || vocab < 1 || vocab > kNextTokenMaxVocab || ld < vocab || H < 1 ||
      (!last && (!word || !pos_table || !y)) || !prompt_ids || stride < 1 || !hist || hist_ld <= t || !hist_len0)
    return fail(TFSC_E_INVALID, "generate_process: no kernel for %d rows of vocab = %d, ld = %lld, H = %d, stride = %lld, hist_ld ="
                " %lld at t = %d (1 <= vocab <= %d, ld >= vocab, prompt ids, hist and hist_len0, stride >= 1, hist_ld > t, the tables"
                " and y unless last)", rows, vocab, (long long)ld, H, (long long)stride, (long long)hist_ld, t, kNextTokenMaxVocab);
  if (!processing_supported(repetition_penalty, no_repeat_ngram_size, min_new_tokens) ||
      (min_new_tokens > 0 && (eos < 0 || eos >= vocab)))
    return fail(TFSC_E_INVALID, "generate_process: repetition_penalty = %g, no_repeat_ngram_size = %d, min_new_tokens = %d, eos = %d"
                " (a finite, normal fp32 penalty > 0, n >= 0, m >= 0, an eos below vocab = %d when m > 0)", (double)repetition_penalty,
                no_repeat_ngram_size, min_new_tokens, eos, vocab);
  if (seeds && (seed_stride < 1 || !sampling_supported(vocab, temperature, top_k, top_p)))
    return fail(TFSC_E_INVALID, "generate_process: seed_stride = %lld, temperature = %g, top_k = %d, top_p = %g (seed_stride >= 1,"
                " a finite temperature > 0 with a finite reciprocal, 0 <= top_k <= vocab = %d, 0 < top_p <= 1)", (long long)seed_stride,
                (double)temperature, top_k, (double)top_p, vocab);
  GenerateOutputs o;
  o.ids = ids;
  o.ids_ld = ids_ld;
  o.log_probs = log_probs;
  o.log_probs_ld = lp_ld;
  o.length = length;
  o.length_ld = length_ld;
  cudaError_t e = launch_generate_process(logits, ld, vocab, pos, t, last != 0, eos, done, o, word, pos_table, y, rows, H, prompt_ids,
                                          mask, stride, hist, hist_ld, hist_len0, repetition_penalty, no_repeat_ngram_size,
                                          min_new_tokens, seeds, seed_stride, temperature, top_k, top_p, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "generate_process: %s", cudaGetErrorString(e));
}
int tfsc_k_token_score(const float* logits, int64_t ld, int64_t first, int n, const int32_t* ids, const int32_t* mask, int64_t stride,
                       int rows, int S, int vocab, float* log_probs, int32_t* ranks, void* stream) {
  if (int rc = check_device()) return rc;
  if (n < 0 || first < 0 || rows < 0 || !score_supported(S, vocab) || first + n > (int64_t)rows * S)
    return fail(TFSC_E_INVALID, "token_score: no kernel for tokens [%lld, %lld) of %d rows of S = %d, vocab = %d (1 <= S <= %d, 1 <="
                " vocab <= %d, the tokens within rows * S)", (long long)first, (long long)first + n, rows, S, vocab, kScoreMaxS,
                kNextTokenMaxVocab);
  if (!logits || !ids || !log_probs || !ranks || ld < vocab || stride < S)
    return fail(TFSC_E_INVALID, "token_score: needs the logits, ids and outputs, ld >= vocab and stride >= S (ld = %lld, stride = %lld)",
                (long long)ld, (long long)stride);
  cudaError_t e = launch_token_score(logits, ld, first, n, ids, mask, stride, S, vocab, log_probs, ranks, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "token_score: %s", cudaGetErrorString(e));
}
int tfsc_k_score_head(const float* log_probs, const int32_t* ranks, const int32_t* mask, int64_t stride, int rows, int S,
                      float* token_log_probs, int64_t lp_ld, int32_t* token_ranks, int64_t ranks_ld, float* sum, int64_t sum_ld,
                      int32_t* count, int64_t count_ld, void* stream) {
  if (int rc = check_device()) return rc;
  if (rows < 0 || S < 1 || S > kScoreMaxS || stride < S)
    return fail(TFSC_E_INVALID, "score_head: no kernel for %d rows of S = %d, stride = %lld (1 <= S <= %d, stride >= S)", rows, S,
                (long long)stride, kScoreMaxS);
  if (((token_log_probs || sum) && !log_probs) || (token_ranks && !ranks))
    return fail(TFSC_E_INVALID, "score_head: its outputs need the log-probabilities and ranks they copy");
  ScoreOutputs o;
  o.log_probs = token_log_probs;
  o.log_probs_ld = lp_ld;
  o.ranks = token_ranks;
  o.ranks_ld = ranks_ld;
  o.sum = sum;
  o.sum_ld = sum_ld;
  o.count = count;
  o.count_ld = count_ld;
  cudaError_t e = launch_score_head(log_probs, ranks, mask, stride, rows, S, o, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : fail(TFSC_E_INTERNAL, "score_head: %s", cudaGetErrorString(e));
}
int tfsc_debug_gemm_trace(long long*) {
  return fail(TFSC_E_UNIMPLEMENTED, "no GEMM clock trace: the persistent GEMM kernel it timed is not part of the sm_90a build");
}

}  // extern "C"
