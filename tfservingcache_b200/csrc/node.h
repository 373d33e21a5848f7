// One ring member = one GPU: the cache tier of the reference (pkg/cachemanager) rebuilt around
// device memory. Holds
//   * the LRU host tier (lrucache.go semantics, entries live in pinned host memory),
//   * the HBM arena + residency table (the "loaded in TF-Serving" set of
//     cachemanager.go:167-195 / servingcontroller.go, same six states),
//   * a copy stream paging weights in with cudaMemcpyAsync from pinned memory,
//   * the batcher: concurrent Predict calls for the same resident model are gathered into one
//     contiguous [rows, in] device buffer and run with one pass over the weights.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <condition_variable>
#include <deque>
#include <memory>
#include <mutex>
#include <set>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "arena.h"
#include "inputs.h"
#include "lru.h"
#include "model.h"
#include "provider.h"

namespace tfsc {

struct DeviceModel {
  ModelId id;
  std::shared_ptr<HostModel> host;
  ModelDesc desc;
  int state = TFSC_STATE_START;
  size_t off = 0, bytes = 0;
  char* dptr = nullptr;
  cudaEvent_t ready = nullptr;  // recorded on the copy stream after the H2D page-in
  std::atomic<bool> ready_seen{false};  // event known complete: consumers skip the stream wait
  int inflight = 0;             // pins: launches that still read dptr
  bool draining = false;        // unloaded while its page-in was still in flight: parked in Node::drain_
};

struct NodeConfig {
  int device = 0;
  int64_t host_cache_bytes = 0;     // modelCache.size
  int max_concurrent_models = 2;    // serving.maxConcurrentModels
  int64_t arena_bytes = 0;          // gpu.arenaBytes (0 = 85% of free HBM)
  int max_batch = 8;                // gpu.maxBatch: rows gathered across requests per launch
  int max_request_rows = 1024;      // largest single request
  double fetch_timeout_s = 10.0;    // ModelFetchTimeout (main.go:122)
  int slots = 4;                    // staging slots in flight
  int tick_us = 0;                  // gpu.tickMicros: hold a partial batch up to this long for more rows (0 = launch at once)
  int64_t staging_pool_bytes = (int64_t)2 << 30;  // pinned request-staging buffers kept for reuse
};

// One Predict request inside the node. `x` / `y` are DEVICE-ACCESSIBLE addresses: a pinned host staging buffer (host
// callers: the client thread copied its rows there, the gather kernel reads them over PCIe), local HBM, or a peer GPU's
// forward window (requests forwarded by another rank, a6: read / written over NVLink). Completion is a condition variable
// (synchronous callers) or the `on_done` callback (tickets, forwarded requests).
struct PredictRequest {
  std::shared_ptr<DeviceModel> dm;
  const void* x = nullptr;
  void* y = nullptr;
  int64_t rows = 0;
  bool host_staged = true;   // x / y are pinned host memory (h2d / d2h byte counters), else device / peer memory
  uint64_t seq = 0;          // global arrival order (the batcher serves oldest-request-first)
  int64_t arrival_ns = 0;    // steady clock
  int64_t deadline_ns = 0;   // steady clock (CLOCK_MONOTONIC); 0 = none. Checked while the request is still queued
  int rc = 1;                // 1 = pending
  std::string err;
  std::mutex mu;
  std::condition_variable cv;
  std::function<void(PredictRequest*)> on_done;  // if set: called once (completer / batcher thread) instead of the notify
};

class Node {
 public:
  Node(const NodeConfig& cfg, ModelProvider* provider);
  ~Node();
  bool init(std::string* err);

  // fetchModel (cachemanager.go:91-152). On success returns TFSC_FETCH_* and, if `pinned` is
  // given, a pinned handle the caller must unpin().
  int fetch(const ModelId& id, std::shared_ptr<DeviceModel>* pinned, std::string* err);
  void unpin(const std::shared_ptr<DeviceModel>& dm);
  int status(const ModelId& id);  // GetModelStatus: TFSC_STATE_* or TFSC_E_NOT_FOUND
  std::string resident_lines();
  std::string host_lines();

  // host-buffer predict through the batcher (blocks the caller). `ts` are the request tensors sorted and described by
  // layout_inputs (inputs.h); one tensor of n_elems values is split into rows by the model (n_elems / in_dim), several
  // are packed row by row. y_alloc(desc, rows) supplies the output buffer once the model is known (return nullptr to
  // reject, e.g. caller buffer too small).
  using OutAllocFn = std::function<void*(const ModelDesc&, int64_t rows)>;
  int predict_host(const ModelId& id, const std::vector<InTensor>& ts, const InputLayout& l, const OutAllocFn& y_alloc, int* outcome,
                   ModelDesc* desc_out, std::string* err, int64_t deadline_ns = 0);
  int predict_host(const ModelId& id, const void* x, int64_t n_elems, int in_dtype, const OutAllocFn& y_alloc, int* outcome,
                   ModelDesc* desc_out, std::string* err, int64_t deadline_ns = 0);  // one unnamed tensor
  // The two halves of predict_host for asynchronous callers (tickets, forwarded requests):
  // prepare = fetchModel + input checks (the layout against the model), fills req->dm (pinned) and req->rows; on error
  // nothing stays pinned.
  int prepare(const ModelId& id, const InputLayout& l, PredictRequest* req, int* outcome, std::string* err);
  // enqueue = hand the request to the batcher; req->x / req->y must be set and the request must stay alive until it
  // completes (rc != 1 / on_done called). The pin taken by prepare() is released on completion.
  void enqueue(PredictRequest* req);
  void abandon(PredictRequest* req);  // after a successful prepare() that will not be enqueued: drop the pin
  // pinned, device-accessible request staging (size-class pool); nullptr when the host cannot pin more memory
  void* staging_alloc(size_t bytes);
  void staging_free(void* p, size_t bytes);
  static size_t row_in_bytes(const ModelDesc& d);
  static size_t row_out_bytes(const ModelDesc& d);
  static int64_t now_ns();
  // describe a model (triggers fetch): needed to size outputs before predict
  int describe(const ModelId& id, ModelDesc* desc, int* outcome, std::string* err);
  // device-buffer predict on `stream` (nullptr = compute stream), asynchronous
  int predict_device(const ModelId& id, const void* x, int64_t rows, void* y, cudaStream_t stream, std::string* err);
  int sync();
  void stats(tfsc_stats* s);
  int device() const { return cfg_.device; }
  // serving.maxConcurrentModels at run time (the reference re-reads viper keys per call, cluster.go:117): the resident
  // prefix shrinks at once (models beyond it are unloaded) and grows with the following reloads
  void set_max_concurrent_models(int n);

 private:
  struct Slot {
    char *d_in = nullptr, *d_out = nullptr, *scratch = nullptr;
    void* ws = nullptr;
    size_t io_cap = 0, scratch_cap = 0, ws_cap = 0;
    cudaEvent_t in_done = nullptr, k_done = nullptr, done = nullptr;
    std::vector<PredictRequest*> reqs;
    std::shared_ptr<DeviceModel> dm;
    bool busy = false;
  };
  struct Retire {
    cudaEvent_t ev;
    std::shared_ptr<DeviceModel> dm;
  };
  struct StreamScratch {  // activation buffers + split-K workspace of one caller stream
    char* base = nullptr;
    size_t act_bytes = 0, ws_bytes = 0;
  };

  // all *_locked functions require mu_
  std::vector<CachedModel> resident_prefix_locked();
  int reload_locked(std::unique_lock<std::mutex>& lk, const ModelId& want, std::string* err);
  void begin_unload_locked(const std::shared_ptr<DeviceModel>& d);
  void release_locked(const std::shared_ptr<DeviceModel>& d);
  void reap_locked();
  bool compact_locked();  // slide idle resident blocks together (D2D) when the arena is fragmented; true if anything moved
  void on_host_evict_locked(const CachedModel& m);
  void refresh_state_locked(DeviceModel* d);
  void* host_alloc(size_t bytes, std::function<void(void*, size_t)>* release);
  bool ensure_slot(Slot* s, const ModelDesc& d, int64_t rows, std::string* err);
  cudaError_t run_model(const DeviceModel& dm, const char* x, int64_t rows, char* y, char* scratch, void* ws, size_t ws_cap,
                        cudaStream_t st);
  static size_t model_ws_bytes(const ModelDesc& d);
  void batcher_loop();
  void completer_loop();
  void complete(PredictRequest* r, int rc, const std::string& err);
  cudaEvent_t get_event();
  void put_event(cudaEvent_t e);

  NodeConfig cfg_;
  ModelProvider* provider_;
  cudaStream_t compute_ = nullptr, copy_ = nullptr;  // kernels / weight page-in
  cudaStream_t in_ = nullptr, out_ = nullptr;         // request inputs H2D / results D2H
  char* slab_ = nullptr;
  Arena arena_;

  std::mutex mu_;
  std::condition_variable cv_;
  LRUCache lru_;
  std::unordered_map<ModelId, std::shared_ptr<HostModel>, ModelIdHash> host_;
  std::unordered_map<ModelId, std::shared_ptr<DeviceModel>, ModelIdHash> dev_;
  std::unordered_map<ModelId, int, ModelIdHash> loading_;  // provider loads in flight (1) / failed (-1)
  std::deque<Retire> retire_;
  std::vector<std::shared_ptr<DeviceModel>> drain_;  // UNLOADING blocks waiting for their page-in event (never under a sync)
  std::unordered_set<ModelId, ModelIdHash> ended_;   // ids of recently unloaded models (status END), bounded FIFO
  std::deque<ModelId> ended_fifo_;
  static constexpr int kRefetch = 1 << 20;           // reload_locked: model left the host tier meanwhile
  std::vector<cudaEvent_t> event_pool_;

  std::mutex scratch_mu_;
  std::unordered_map<cudaStream_t, StreamScratch> stream_scratch_;

  // pinned block pool (exact-size reuse)
  std::mutex pool_mu_;
  std::unordered_map<size_t, std::vector<void*>> pool_;
  // pinned request staging, power-of-two size classes
  std::mutex stage_mu_;
  std::unordered_map<size_t, std::vector<void*>> stage_pool_;
  size_t stage_pooled_bytes_ = 0;

  // batcher
  std::mutex q_mu_;
  std::condition_variable q_cv_, slot_cv_;
  std::unordered_map<DeviceModel*, std::deque<PredictRequest*>> pending_;
  std::set<std::pair<uint64_t, DeviceModel*>> order_;  // (seq of the model's oldest request, model)
  uint64_t seq_ = 0;
  std::deque<Slot*> inflight_;
  std::vector<Slot> slots_;
  std::thread batcher_, completer_;
  bool stop_ = false, batcher_done_ = false;

  // stats (guarded by mu_ unless atomic)
  int64_t total_ = 0, hits_ = 0, misses_ = 0, ev_host_ = 0, ev_hbm_ = 0, h2d_weights_ = 0, compactions_ = 0, compacted_bytes_ = 0;
  std::atomic<int64_t> h2d_inputs_{0}, d2h_outputs_{0}, batches_{0}, batched_rows_{0};
  double cache_dur_ = 0, fetch_dur_ = 0;
};

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

}  // namespace tfsc
