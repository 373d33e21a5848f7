#include "node.h"

#include <chrono>
#include <cstdlib>
#include <set>

#include "kernels.h"

namespace tfsc {

using Clock = std::chrono::steady_clock;
static double secs_since(Clock::time_point t0) { return std::chrono::duration<double>(Clock::now() - t0).count(); }

#define CU_OK(expr, errp, code)                                                        \
  do {                                                                                 \
    cudaError_t _e = (expr);                                                           \
    if (_e != cudaSuccess) {                                                           \
      if (errp) *(errp) = std::string(#expr) + ": " + cudaGetErrorString(_e);          \
      return code;                                                                     \
    }                                                                                  \
  } while (0)

Node::Node(const NodeConfig& cfg, ModelProvider* provider)
    : cfg_(cfg), provider_(provider), lru_("", cfg.host_cache_bytes) {
  lru_.on_evict = [this](const CachedModel& m) { on_host_evict_locked(m); };
}

bool Node::init(std::string* err) {
  DeviceGuard g(cfg_.device);
  CU_OK(cudaStreamCreateWithFlags(&compute_, cudaStreamNonBlocking), err, false);
  CU_OK(cudaStreamCreateWithFlags(&copy_, cudaStreamNonBlocking), err, false);
  CU_OK(cudaStreamCreateWithFlags(&in_, cudaStreamNonBlocking), err, false);
  CU_OK(cudaStreamCreateWithFlags(&out_, cudaStreamNonBlocking), err, false);
  size_t bytes = (size_t)cfg_.arena_bytes;
  if (bytes == 0) {
    size_t fr = 0, tot = 0;
    CU_OK(cudaMemGetInfo(&fr, &tot), err, false);
    bytes = (size_t)(fr * 0.85);
  }
  CU_OK(cudaMalloc(&slab_, bytes), err, false);
  arena_.init(bytes, 1024);
  slots_.resize(cfg_.slots > 0 ? cfg_.slots : 1);
  for (auto& s : slots_) {
    CU_OK(cudaEventCreateWithFlags(&s.in_done, cudaEventDisableTiming), err, false);
    CU_OK(cudaEventCreateWithFlags(&s.k_done, cudaEventDisableTiming), err, false);
    CU_OK(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming), err, false);
  }
  batcher_ = std::thread([this] { batcher_loop(); });
  completer_ = std::thread([this] { completer_loop(); });
  return true;
}

Node::~Node() {
  {
    std::lock_guard<std::mutex> lk(q_mu_);
    stop_ = true;
  }
  q_cv_.notify_all();
  slot_cv_.notify_all();
  if (batcher_.joinable()) batcher_.join();
  {
    std::lock_guard<std::mutex> lk(q_mu_);
    batcher_done_ = true;  // only now may the completer stop: the batcher can no longer hand it a batch
  }
  q_cv_.notify_all();
  if (completer_.joinable()) completer_.join();
  DeviceGuard g(cfg_.device);
  cudaDeviceSynchronize();
  for (auto& s : slots_) {
    if (s.d_in) cudaFree(s.d_in);
    if (s.d_out) cudaFree(s.d_out);
    if (s.scratch) cudaFree(s.scratch);
    if (s.ws) cudaFree(s.ws);
    if (s.done) cudaEventDestroy(s.done);
    if (s.in_done) cudaEventDestroy(s.in_done);
    if (s.k_done) cudaEventDestroy(s.k_done);
  }
  for (auto& kv : stream_scratch_) cudaFree(kv.second.base);
  for (auto& r : retire_) cudaEventDestroy(r.ev);
  // every reference to a DeviceModel / HostModel must go while the pinned-block pool still exists: HostModel's release
  // functor returns the block to pool_ (a member destroyed BEFORE retire_ / dev_ / host_ in reverse declaration order)
  retire_.clear();
  drain_.clear();
  for (auto& kv : dev_)
    if (kv.second->ready) cudaEventDestroy(kv.second->ready);
  dev_.clear();
  host_.clear();  // returns pinned blocks to the pool
  for (auto e : event_pool_) cudaEventDestroy(e);
  for (auto& kv : pool_)
    for (void* p : kv.second) cudaFreeHost(p);
  for (auto& kv : stage_pool_)
    for (void* p : kv.second) cudaFreeHost(p);
  if (slab_) cudaFree(slab_);
  if (compute_) cudaStreamDestroy(compute_);
  if (copy_) cudaStreamDestroy(copy_);
  if (in_) cudaStreamDestroy(in_);
  if (out_) cudaStreamDestroy(out_);
}

cudaEvent_t Node::get_event() {
  if (!event_pool_.empty()) {
    cudaEvent_t e = event_pool_.back();
    event_pool_.pop_back();
    return e;
  }
  cudaEvent_t e = nullptr;
  cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
  return e;
}
void Node::put_event(cudaEvent_t e) { event_pool_.push_back(e); }

void* Node::host_alloc(size_t bytes, std::function<void(void*, size_t)>* release) {
  void* p = nullptr;
  {
    std::lock_guard<std::mutex> lk(pool_mu_);
    auto it = pool_.find(bytes);
    if (it != pool_.end() && !it->second.empty()) {
      p = it->second.back();
      it->second.pop_back();
    }
  }
  if (!p) {
    DeviceGuard g(cfg_.device);
    if (cudaHostAlloc(&p, bytes, cudaHostAllocPortable) != cudaSuccess) {
      // the host cannot pin more memory (shared box): keep the model in pageable memory; page-ins of this
      // blob then go through the driver's staging buffers (slower, still correct)
      cudaGetLastError();
      p = malloc(bytes);
      if (!p) return nullptr;
      *release = [](void* q, size_t) { free(q); };
      return p;
    }
  }
  *release = [this](void* q, size_t n) {
    std::lock_guard<std::mutex> lk(pool_mu_);
    auto& v = pool_[n];
    if (v.size() < 8) v.push_back(q);  // exact-size reuse: pinning 1 GB costs ~100 ms, reuse is free
    else cudaFreeHost(q);
  };
  return p;
}

// ------------------------------------------------------------------ residency machine ------
std::vector<CachedModel> Node::resident_prefix_locked() {
  // cachemanager.go:168-169: first min(len, MaxConcurrentModels) of the MRU list, additionally
  // cut where the HBM arena byte budget would be exceeded.
  std::vector<CachedModel> all = lru_.list_models();
  std::vector<CachedModel> out;
  size_t used = 0;
  for (auto& m : all) {
    if ((int)out.size() >= cfg_.max_concurrent_models) break;
    size_t need = ((size_t)m.size_on_disk + 1023) / 1024 * 1024;
    if (used + need > arena_.capacity()) break;
    used += need;
    out.push_back(m);
  }
  return out;
}

void Node::refresh_state_locked(DeviceModel* d) {
  if (d->state == TFSC_STATE_LOADING && d->ready && cudaEventQuery(d->ready) == cudaSuccess) {
    d->state = TFSC_STATE_AVAILABLE;
    d->ready_seen = true;
  } else {
    cudaGetLastError();  // clear cudaErrorNotReady
  }
}

void Node::release_locked(const std::shared_ptr<DeviceModel>& d_in) {
  const std::shared_ptr<DeviceModel> d = d_in;  // the dev_ entry (possibly the caller's reference) is erased below
  if (!d->dptr) return;
  if (!d->ready_seen && d->ready) {
    // the page-in DMA must not outlive its source / its arena block. Never wait for it under mu_ (a multi-GB copy would
    // stall every fetch / status call of the node): park the block as "draining", reap_locked() frees it once the
    // copy-stream event has completed.
    if (cudaEventQuery(d->ready) != cudaSuccess) {
      cudaGetLastError();
      if (!d->draining) {
        d->draining = true;
        drain_.push_back(d);
      }
      return;
    }
    d->ready_seen = true;
  }
  d->draining = false;
  arena_.release(d->off);
  d->dptr = nullptr;
  d->state = TFSC_STATE_END;
  d->host.reset();
  if (d->ready) {
    put_event(d->ready);
    d->ready = nullptr;
  }
  ++ev_hbm_;
  // END entries keep no DeviceModel (desc + op list): only the id survives, in a bounded FIFO, so GetModelStatus can
  // still answer END for a recently unloaded servable
  auto it = dev_.find(d->id);
  if (it != dev_.end() && it->second == d) dev_.erase(it);
  if (ended_.insert(d->id).second) {
    ended_fifo_.push_back(d->id);
    if (ended_fifo_.size() > 65536) {
      ended_.erase(ended_fifo_.front());
      ended_fifo_.pop_front();
    }
  }
  cv_.notify_all();
}

void Node::begin_unload_locked(const std::shared_ptr<DeviceModel>& d_in) {
  const std::shared_ptr<DeviceModel> d = d_in;
  d->state = TFSC_STATE_UNLOADING;
  if (d->inflight == 0) release_locked(d);
}

void Node::on_host_evict_locked(const CachedModel& m) {
  ++ev_host_;
  host_.erase(m.id);
  auto it = dev_.find(m.id);
  if (it != dev_.end() && (it->second->state == TFSC_STATE_AVAILABLE || it->second->state == TFSC_STATE_LOADING))
    begin_unload_locked(it->second);
}

void Node::reap_locked() {
  for (size_t i = 0; i < drain_.size();) {  // blocks whose page-in was still in flight when they were unloaded
    std::shared_ptr<DeviceModel> d = drain_[i];
    if (cudaEventQuery(d->ready) != cudaSuccess) {
      cudaGetLastError();
      ++i;
      continue;
    }
    d->ready_seen = true;
    d->draining = false;
    drain_.erase(drain_.begin() + i);
    if (d->state == TFSC_STATE_UNLOADING && d->inflight == 0) release_locked(d);
  }
  while (!retire_.empty()) {
    cudaError_t q = cudaEventQuery(retire_.front().ev);
    if (q != cudaSuccess) {
      cudaGetLastError();
      break;
    }
    auto r = retire_.front();
    retire_.pop_front();
    put_event(r.ev);
    if (--r.dm->inflight == 0 && r.dm->state == TFSC_STATE_UNLOADING) release_locked(r.dm);
  }
}

void Node::unpin(const std::shared_ptr<DeviceModel>& dm) {
  std::lock_guard<std::mutex> lk(mu_);
  if (--dm->inflight == 0 && dm->state == TFSC_STATE_UNLOADING) {
    DeviceGuard g(cfg_.device);
    release_locked(dm);
  }
}

bool Node::compact_locked() {
  std::map<size_t, std::shared_ptr<DeviceModel>> by_off;
  for (auto& kv : dev_)
    if (kv.second->dptr) by_off[kv.second->off] = kv.second;
  std::map<size_t, size_t> layout;
  size_t cursor = 0;
  bool moved = false;
  for (auto& kv : by_off) {
    const std::shared_ptr<DeviceModel>& d = kv.second;
    const size_t len = arena_.aligned(d->bytes);
    refresh_state_locked(d.get());
    const bool idle = d->state == TFSC_STATE_AVAILABLE && d->inflight == 0 && d->ready_seen && d->ready;
    const size_t delta = d->off > cursor ? d->off - cursor : 0;
    // a block slides down by `delta`; source and destination overlap when delta < len, so the copy goes forward in chunks of
    // at most delta bytes (each chunk's destination lies below everything not copied yet). Tiny deltas are not worth it.
    if (idle && delta > 0 && delta >= len / 64) {
      cudaError_t e = cudaSuccess;
      for (size_t done = 0; done < d->bytes && e == cudaSuccess; done += delta) {
        const size_t n = d->bytes - done < delta ? d->bytes - done : delta;
        e = cudaMemcpyAsync(slab_ + cursor + done, slab_ + d->off + done, n, cudaMemcpyDeviceToDevice, copy_);
      }
      if (e == cudaSuccess) e = cudaEventRecord(d->ready, copy_);
      if (e != cudaSuccess) {
        cudaGetLastError();
        layout[d->off] = len;  // keep it where it is (a partially issued copy only wrote below the block's own start)
        cursor = d->off + len;
        continue;
      }
      d->off = cursor;
      d->dptr = slab_ + cursor;
      d->state = TFSC_STATE_LOADING;  // launches wait for the copy-stream event, exactly as after a page-in
      d->ready_seen = false;
      compacted_bytes_ += (int64_t)d->bytes;
      moved = true;
    }
    layout[d->off] = len;
    cursor = d->off + len;
  }
  if (moved) {
    arena_.relayout(layout);
    ++compactions_;
  }
  return moved;
}

int Node::reload_locked(std::unique_lock<std::mutex>& lk, const ModelId& want, std::string* err) {
  const auto deadline = Clock::now() + std::chrono::duration<double>(cfg_.fetch_timeout_s);
  for (;;) {
    reap_locked();
    std::vector<CachedModel> prefix = resident_prefix_locked();
    std::set<std::pair<std::string, int64_t>> keep;
    bool want_in = false;
    for (auto& m : prefix) {
      keep.insert({m.id.name, m.id.version});
      if (m.id == want) want_in = true;
    }
    if (!want_in) {
      CachedModel cm;
      if (!lru_.peek(want, &cm)) return kRefetch;  // evicted from the host tier while mu_ was dropped: back to the miss path
      *err = "model " + want.name + ":" + std::to_string(want.version) + " does not fit the HBM arena (" +
             std::to_string(arena_.capacity()) + " bytes) / serving.maxConcurrentModels";
      return TFSC_E_EXHAUSTED;
    }
    // unload what fell out of the resident prefix (TF-Serving drops models absent from the new config)
    std::vector<std::shared_ptr<DeviceModel>> drop;  // release_locked erases from dev_: collect first
    for (auto& kv : dev_) {
      auto& d = kv.second;
      if ((d->state == TFSC_STATE_AVAILABLE || d->state == TFSC_STATE_LOADING) &&
          !keep.count({d->id.name, d->id.version}))
        drop.push_back(d);
    }
    for (auto& d : drop) begin_unload_locked(d);
    // page in what is missing, MRU first
    for (auto& m : prefix) {
      auto it = dev_.find(m.id);
      std::shared_ptr<DeviceModel> d = it == dev_.end() ? nullptr : it->second;
      if (d && (d->state == TFSC_STATE_AVAILABLE || d->state == TFSC_STATE_LOADING)) continue;
      if (d && d->state == TFSC_STATE_UNLOADING && d->dptr) {  // still pinned by in-flight work: revive in place
        d->state = d->ready_seen ? TFSC_STATE_AVAILABLE : TFSC_STATE_LOADING;
        continue;
      }
      auto hit = host_.find(m.id);
      if (hit == host_.end()) continue;
      size_t off;
      if (!arena_.alloc(hit->second->bytes, &off)) {
        // enough free bytes in total but no hole large enough (mixed 102 MB / 438 MB / 1 GB models): pack the idle
        // resident blocks together with device-to-device copies (~3 TB/s) instead of evicting down the LRU and paying
        // PCIe reloads (~55 GB/s) later
        const bool fragmented = arena_.capacity() - arena_.used() >= arena_.aligned(hit->second->bytes);
        if (!(m.id == want && fragmented && compact_locked() && arena_.alloc(hit->second->bytes, &off))) {
          if (m.id == want) break;  // must wait for space
          continue;                 // other prefix members are paged in opportunistically
        }
      }
      auto nd = std::make_shared<DeviceModel>();
      nd->id = m.id;
      nd->host = hit->second;
      nd->desc = hit->second->desc;
      nd->off = off;
      nd->bytes = hit->second->bytes;
      nd->dptr = slab_ + off;
      nd->state = TFSC_STATE_LOADING;
      nd->ready = get_event();
      cudaError_t e = cudaMemcpyAsync(nd->dptr, nd->host->data, nd->bytes, cudaMemcpyHostToDevice, copy_);
      if (e == cudaSuccess) e = cudaEventRecord(nd->ready, copy_);
      if (e != cudaSuccess) {
        arena_.release(off);
        put_event(nd->ready);
        *err = std::string("page-in failed: ") + cudaGetErrorString(e);
        return TFSC_E_INTERNAL;
      }
      h2d_weights_ += (int64_t)nd->bytes;
      dev_[m.id] = nd;
    }
    auto wit = dev_.find(want);
    if (wit != dev_.end() && (wit->second->state == TFSC_STATE_AVAILABLE || wit->second->state == TFSC_STATE_LOADING))
      return 0;
    // blocked on arena space: wait for pinned victims to retire, else evict further (fragmentation)
    bool pending_release = !retire_.empty();
    for (auto& kv : dev_)
      if (kv.second->state == TFSC_STATE_UNLOADING && kv.second->dptr) pending_release = true;
    if (!pending_release) {
      std::shared_ptr<DeviceModel> victim;
      for (auto rit = prefix.rbegin(); rit != prefix.rend(); ++rit) {
        if (rit->id == want) continue;
        auto it = dev_.find(rit->id);
        if (it != dev_.end() && it->second->dptr && it->second->inflight == 0 &&
            (it->second->state == TFSC_STATE_AVAILABLE || it->second->state == TFSC_STATE_LOADING)) {
          victim = it->second;
          break;
        }
      }
      if (victim) {
        begin_unload_locked(victim);
        continue;
      }
    }
    if (Clock::now() >= deadline) {
      *err = "Timeout: Model did not load in time";  // cachemanager.go:191-193
      return TFSC_E_TIMEOUT;
    }
    if (!retire_.empty()) {
      cudaEvent_t ev = retire_.front().ev;
      lk.unlock();
      cudaEventSynchronize(ev);
      lk.lock();
    } else {
      cv_.wait_for(lk, std::chrono::milliseconds(2));
    }
  }
}

int Node::fetch(const ModelId& id, std::shared_ptr<DeviceModel>* pinned, std::string* err) {
  DeviceGuard g(cfg_.device);
  const auto t0 = Clock::now();
  std::unique_lock<std::mutex> lk(mu_);
  ++total_;
  reap_locked();
  int outcome = -1;
  std::shared_ptr<DeviceModel> d;
  for (;;) {
    CachedModel cm;
    if (!lru_.get(id, &cm)) {  // tryGetModelFromCache, cachemanager.go:154-165 (Get touches recency)
      if (outcome < 0) {
        outcome = TFSC_FETCH_MISS;
        ++misses_;
      }
      if (loading_.count(id)) {  // coalesce concurrent misses of one model (fixes the duplicate download)
        cv_.wait(lk, [&] { return loading_.count(id) == 0; });
        continue;
      }
      loading_[id] = 1;
      lk.unlock();
      const auto tf = Clock::now();
      std::string perr;
      std::shared_ptr<HostModel> hm;
      int64_t size = provider_->model_size(id.name, id.version, &perr);  // :116
      if (size >= 0)
        hm = provider_->load_model(
            id.name, id.version,
            [this](size_t n, std::function<void(void*, size_t)>* rel) { return host_alloc(n, rel); }, &perr);  // :122
      lk.lock();
      loading_.erase(id);
      fetch_dur_ += secs_since(tf);
      if (!hm) {
        cv_.notify_all();
        cache_dur_ += secs_since(t0);
        *err = perr;
        return perr == "No matching model found" || size < 0 ? TFSC_E_NOT_FOUND : TFSC_E_INTERNAL;
      }
      size = (int64_t)hm->bytes > size ? (int64_t)hm->bytes : size;
      lru_.ensure_free_bytes(size);  // :121
      CachedModel nm{id, id.name + "/" + std::to_string(id.version), size};
      lru_.put(id, nm);  // :127
      host_[id] = hm;
      cv_.notify_all();
      continue;  // now present: falls into the reload branch below (:128)
    }
    auto dit = dev_.find(id);
    if (dit != dev_.end()) refresh_state_locked(dit->second.get());
    const int st = dit == dev_.end() ? -1 : dit->second->state;
    if (st == TFSC_STATE_AVAILABLE || st == TFSC_STATE_LOADING) {
      d = dit->second;
      if (outcome < 0) {
        outcome = TFSC_FETCH_HIT;  // :144-150
        ++hits_;
      }
      break;
    }
    if (outcome < 0) outcome = TFSC_FETCH_RELOAD;  // :133-143: cached but not resident
    int rc = reload_locked(lk, id, err);
    if (rc == kRefetch) continue;
    if (rc < 0) {
      cache_dur_ += secs_since(t0);
      return rc;
    }
    d = dev_[id];
    break;
  }
  d->inflight++;
  cache_dur_ += secs_since(t0);
  lk.unlock();
  if (pinned) {
    *pinned = d;
  } else {
    // synchronous ensure: the poll-until-AVAILABLE loop of :175-193 becomes one event wait
    cudaError_t e = d->ready_seen ? cudaSuccess : cudaEventSynchronize(d->ready);
    {
      std::lock_guard<std::mutex> l2(mu_);
      if (e == cudaSuccess) refresh_state_locked(d.get());
    }
    unpin(d);
    if (e != cudaSuccess) {
      *err = std::string("page-in failed: ") + cudaGetErrorString(e);
      return TFSC_E_INTERNAL;
    }
  }
  return outcome;
}

void Node::set_max_concurrent_models(int n) {
  DeviceGuard g(cfg_.device);
  std::lock_guard<std::mutex> lk(mu_);
  cfg_.max_concurrent_models = n;
  reap_locked();
  // what TF-Serving does when a reload config lists fewer models: everything outside the new resident prefix unloads
  std::set<std::pair<std::string, int64_t>> keep;
  for (auto& m : resident_prefix_locked()) keep.insert({m.id.name, m.id.version});
  std::vector<std::shared_ptr<DeviceModel>> drop;
  for (auto& kv : dev_)
    if ((kv.second->state == TFSC_STATE_AVAILABLE || kv.second->state == TFSC_STATE_LOADING) &&
        !keep.count({kv.second->id.name, kv.second->id.version}))
      drop.push_back(kv.second);
  for (auto& d : drop) begin_unload_locked(d);
}

int Node::status(const ModelId& id) {
  DeviceGuard g(cfg_.device);
  std::lock_guard<std::mutex> lk(mu_);
  reap_locked();
  auto it = dev_.find(id);
  if (it == dev_.end()) {
    if (loading_.count(id)) return TFSC_STATE_START;
    if (ended_.count(id)) return TFSC_STATE_END;
    return fail(TFSC_E_NOT_FOUND, "Model not found");  // servingcontroller.go:137
  }
  refresh_state_locked(it->second.get());
  return it->second->state;
}

std::string Node::resident_lines() {
  DeviceGuard g(cfg_.device);
  std::lock_guard<std::mutex> lk(mu_);
  std::string s;
  for (auto& m : lru_.list_models()) {
    auto it = dev_.find(m.id);
    if (it == dev_.end() || !it->second->dptr) continue;
    refresh_state_locked(it->second.get());
    s += m.id.name + "\t" + std::to_string(m.id.version) + "\t" + std::to_string(it->second->bytes) + "\t" +
         std::to_string(it->second->state) + "\n";
  }
  return s;
}

std::string Node::host_lines() {
  std::lock_guard<std::mutex> lk(mu_);
  std::string s;
  for (auto& m : lru_.list_models())
    s += m.id.name + "\t" + std::to_string(m.id.version) + "\t" + std::to_string(m.size_on_disk) + "\t" + m.path + "\n";
  return s;
}

void Node::stats(tfsc_stats* s) {
  std::lock_guard<std::mutex> lk(mu_);
  s->cache_total += total_;
  s->cache_hits_total += hits_;
  s->cache_misses_total += misses_;
  s->evictions_host += ev_host_;
  s->evictions_hbm += ev_hbm_;
  s->h2d_weight_bytes += h2d_weights_;
  s->arena_compactions += compactions_;
  s->arena_compacted_bytes += compacted_bytes_;
  s->h2d_input_bytes += h2d_inputs_.load();
  s->d2h_output_bytes += d2h_outputs_.load();
  s->batches += batches_.load();
  s->batched_rows += batched_rows_.load();
  s->arena_bytes_used += (int64_t)arena_.used();
  s->arena_bytes_capacity += (int64_t)arena_.capacity();
  s->resident_models += (int64_t)arena_.blocks();
  s->host_models += (int64_t)lru_.size();
  s->cache_duration_seconds_sum += cache_dur_;
  s->cache_fetch_duration_seconds_sum += fetch_dur_;
}

// ------------------------------------------------------------------------- execution ------
size_t Node::model_ws_bytes(const ModelDesc& d) {
  size_t m = 256;
  for (auto& L : d.layers) {
    size_t w = dense_workspace_bytes(kMaxRowsPerLaunch, L.in, L.out);
    if (w > m) m = w;
  }
  bool after_gather = false;
  for (auto& o : d.ops) {  // graph bundles: plain dense heads (ResNet fc) run on the weight-streaming dense kernels
    // and so does a fill-mask bundle's vocabulary projection on a few rows, and a score bundle's on a chunk of a few tokens
    // (run_model)
    if (o.kind == OpKind::Dense || o.kind == OpKind::TokenScore || (after_gather && o.kind == OpKind::Conv)) {
      size_t w = dense_workspace_bytes(kMaxRowsPerLaunch, o.c, o.cout);
      if (w > m) m = w;
    }
    after_gather = after_gather || o.kind == OpKind::MaskGather || o.kind == OpKind::LastToken;
  }
  return m;
}

static bool conv_tc_enabled() {  // TFSC_CONV_TC=0: explicit im2col + GEMM (the round-1 path) for A/B comparisons
  static bool v = [] {
    const char* e = getenv("TFSC_CONV_TC");
    return !e || atoi(e) != 0;
  }();
  return v;
}

// multi-output bundles: one launch of the bundle's head writes every declared output of a row at its offset in the packed
// row (out_dim words). `out` is what the last op (or the mlp's last layer) wrote: N logits (classify), [S, 2] start / end
// logits (span), the [S, H] hidden states or, under a pooler, its [H] output (encoder), [M, Vp] vocabulary logits
// (fill-mask), [1, Vp] vocabulary logits (next-token). The graph heads read the request's ids / mask / segment ids where the embedding reads them (`in`), an
// encoder under a pooler its source buffer (`hidden`), a fill-mask head the mask_gather op's [rows, M] `positions`, a
// next-token head the last_token op's [rows] `positions`.
static cudaError_t run_head(const ModelDesc& d, const float* out, const SpanInputs& in, const float* hidden, const int* positions,
                            int64_t rows, char* y, cudaStream_t st) {
  float* yf = reinterpret_cast<float*>(y);
  const int64_t ld = d.out_dim;
  switch (d.head) {
    case HeadKind::Span: {
      SpanOutputs o;
      for (const ModelOutput& m : d.outputs) {
        float* p = yf + m.offset;
        switch (m.kind) {
          case OutputKind::StartLogits: o.start_logits = p, o.start_ld = ld; break;
          case OutputKind::EndLogits: o.end_logits = p, o.end_ld = ld; break;
          case OutputKind::SpanStarts: o.starts = reinterpret_cast<int*>(p), o.starts_ld = ld; break;
          case OutputKind::SpanEnds: o.ends = reinterpret_cast<int*>(p), o.ends_ld = ld; break;
          case OutputKind::SpanScores: o.scores = p, o.scores_ld = ld; break;
          default: break;
        }
      }
      return launch_span_head(out, in, (int)rows, d.head_n, d.span_max_len, d.head_k, o, st);
    }
    case HeadKind::Encoder: {
      EncoderOutputs o;
      for (const ModelOutput& m : d.outputs) {
        float* p = yf + m.offset;
        switch (m.kind) {
          case OutputKind::SequenceOutput: o.sequence = p, o.sequence_ld = ld; break;
          case OutputKind::PooledOutput: o.pooled = p, o.pooled_ld = ld; break;
          case OutputKind::ClsEmbedding: o.cls = p, o.cls_ld = ld; break;
          case OutputKind::MeanEmbedding: o.mean = p, o.mean_ld = ld; break;
          default: break;
        }
      }
      o.normalize_cls = d.normalize_cls;
      o.normalize_mean = d.normalize_mean;
      EncoderInputs e;
      e.ids = in.ids;
      e.mask = in.mask;
      e.stride = in.stride ? in.stride : d.ops.front().h;
      return launch_encoder_head(d.encoder_pooler ? hidden : out, d.encoder_pooler ? out : nullptr, e, (int)rows, d.head_k,
                                 d.head_n, o, st);
    }
    case HeadKind::FillMask: {
      FillMaskOutputs o;
      for (const ModelOutput& m : d.outputs) {
        float* p = yf + m.offset;
        switch (m.kind) {
          case OutputKind::MaskedPositions: o.positions = reinterpret_cast<int*>(p), o.positions_ld = ld; break;
          case OutputKind::MaskedTopKIds: o.ids = reinterpret_cast<int*>(p), o.ids_ld = ld; break;
          case OutputKind::MaskedTopKProbabilities: o.probs = p, o.probs_ld = ld; break;
          case OutputKind::MaskedTopKLogits: o.logits = p, o.logits_ld = ld; break;
          default: break;
        }
      }
      return launch_fill_mask_head(out, d.ops.back().cout, positions, (int)rows, d.head_n, d.mlm_vocab, d.head_k, kHeadMaxN, o, st);
    }
    case HeadKind::NextToken: {  // the fill-mask head with one slot per row, up to the next-token vocabulary cap
      FillMaskOutputs o;
      for (const ModelOutput& m : d.outputs) {
        float* p = yf + m.offset;
        switch (m.kind) {
          case OutputKind::NextTokenPosition: o.positions = reinterpret_cast<int*>(p), o.positions_ld = ld; break;
          case OutputKind::NextTokenTopKIds: o.ids = reinterpret_cast<int*>(p), o.ids_ld = ld; break;
          case OutputKind::NextTokenTopKProbabilities: o.probs = p, o.probs_ld = ld; break;
          case OutputKind::NextTokenTopKLogits: o.logits = p, o.logits_ld = ld; break;
          default: break;
        }
      }
      return launch_fill_mask_head(out, d.ops.back().cout, positions, (int)rows, 1, d.head_n, d.head_k, kNextTokenMaxVocab, o, st);
    }
    case HeadKind::Classify: {
      HeadOutputs o;
      for (const ModelOutput& m : d.outputs) {
        float* p = yf + m.offset;
        switch (m.kind) {
          case OutputKind::Logits: o.logits = p, o.logits_ld = ld; break;
          case OutputKind::Probabilities: o.probs = p, o.probs_ld = ld; break;
          case OutputKind::Classes: o.classes = reinterpret_cast<int*>(p), o.classes_ld = ld; break;
          case OutputKind::TopKClasses: o.topk_idx = reinterpret_cast<int*>(p), o.topk_idx_ld = ld; break;
          case OutputKind::TopKProbabilities: o.topk_prob = p, o.topk_prob_ld = ld; break;
          default: break;
        }
      }
      return launch_classify_head(out, (int)rows, d.head_n, d.head_k, o, st);
    }
    default: return cudaSuccess;  // a single-output bundle: the last op wrote y
  }
}

cudaError_t Node::run_model(const DeviceModel& dm, const char* x, int64_t rows, char* y, char* scratch, void* ws,
                            size_t ws_cap, cudaStream_t st) {
  const ModelDesc& d = dm.desc;
  if (d.tmpl == Template::Affine) {
    return launch_affine((const float*)x, (float*)y, rows, (const float*)(dm.dptr + d.a_off),
                         (const float*)(dm.dptr + d.b_off), st);
  }
  if (d.tmpl == Template::Graph) {
    // conv net: NHWC activations in `n_buffers` scratch buffers, conv = (im2col +) GEMM with fused bias /
    // residual / ReLU epilogue (BN is folded into the kernel + bias when the bundle is written)
    const size_t buf_bytes = d.graph_buf_bytes(rows);  // 256-byte aligned buffers: the loader's kernel checks rely on it
    char* col = scratch + (size_t)d.n_buffers * buf_bytes;
    // with signature.outputs the op that writes the response (-2) writes the logits to scratch, and the head writes y
    char* out = d.outputs.empty() ? y : scratch + d.head_scratch_offset(rows);
    auto buf = [&](int i) -> char* { return i == -1 ? const_cast<char*>(x) : i == -2 ? out : scratch + (size_t)i * buf_bytes; };
    const int B = (int)rows;
    // token-id inputs: single-input bundles read ids [B, S] and derive the attention mask from them ([PAD] = 0, stride S);
    // multi-input bundles read each declared input at its offset in the packed row, stride in_dim (inputs.h)
    const int* ids = (const int*)x;
    const int* mask = d.input_dtype == TFSC_DT_INT32 ? ids : nullptr;
    const int* types = nullptr;
    int stride = 0;  // single-input: each op's own S
    if (!d.inputs.empty()) {
      const ModelInput* mi = d.input(InputRole::Mask);
      const ModelInput* ti = d.input(InputRole::TypeIds);
      ids = (const int*)x + d.input(InputRole::Ids)->offset;
      mask = mi ? (const int*)x + mi->offset : ids;  // no mask input: [PAD] = 0 of the ids, as single-input bundles
      types = ti ? (const int*)x + ti->offset : nullptr;
      stride = (int)d.in_dim;
    }
    // fill-mask bundles: the mask_gather op writes the [MASK] positions here, next-token bundles the last_token op its
    // positions, and the head reads them
    int* positions = d.head == HeadKind::FillMask || d.head == HeadKind::NextToken || d.head == HeadKind::Generate
                         ? reinterpret_cast<int*>(scratch + d.mlm_positions_offset(rows))
                         : nullptr;
    // the request's attention-mask input, or nullptr: what the causal attention and last_token ops read (GPT-2's id 0 is a
    // token, not [PAD], so they never derive a mask from the ids)
    const int* mask_input = d.input(InputRole::Mask) ? mask : nullptr;
    bool after_gather = false;
    auto exec = [&](const GraphOp& o) -> cudaError_t {
      const float* src = (const float*)buf(o.src);
      float* dst = (float*)buf(o.dst);
      cudaError_t e = cudaSuccess;
      switch (o.kind) {
        case OpKind::Conv:
        case OpKind::Dense: {
          const float* W = (const float*)(dm.dptr + o.w_off);
          const float* bias = (const float*)(dm.dptr + o.b_off);
          const float* res = o.res == -100 ? nullptr : (const float*)buf(o.res);
          const int K = o.kh * o.kw * o.c;
          if (o.kind == OpKind::Dense && !res && o.act <= 1 && (int)o.lda == K && B < 64) {
            // a classifier head on a handful of rows is the tenant-MLP problem (HBM-bound weight streaming), not a GEMM tile
            return launch_dense(src, W, bias, dst, B, K, o.cout, o.act == 1, ws, ws_cap, st);
          }
          if (after_gather && o.kind == OpKind::Conv && o.dst == -2 && !res && o.act <= 1 && o.kh == 1 && o.kw == 1 &&
              o.stride == 1 && o.pad == 0 && o.cout % 32 == 0 && B * o.oh * o.ow < 64) {
            // a fill-mask vocabulary projection, padded to Vp % 32 == 0, on fewer than 64 slots (one [MASK] per row at the
            // default batch of 8): too few rows for the tensor-core GEMM, so it streams the [H, Vp] weights once (DESIGN §4);
            // an unpadded decoder keeps the GEMM path
            return launch_dense(src, W, bias, dst, B * o.oh * o.ow, K, o.cout, o.act == 1, ws, ws_cap, st);
          }
          const bool direct = o.kh == 1 && o.kw == 1 && o.stride == 1 && o.pad == 0;
          if (o.kind == OpKind::Conv && !direct && conv_tc_enabled() &&
              conv_tc_supported(src, W, bias, res, dst, B, o.h, o.w, o.c, o.kh, o.kw, o.stride, o.pad, o.oh, o.ow, o.cout)) {
            // implicit GEMM: TMA im2col gathers the patch tiles straight from the NHWC activations (no col buffer)
            return launch_conv_tc(src, W, bias, res, dst, B, o.h, o.w, o.c, o.kh, o.kw, o.stride, o.pad, o.oh, o.ow, o.cout, o.act, st);
          }
          const float* A = src;
          int lda = o.kind == OpKind::Dense ? (int)o.lda : K;  // Dense over a [S,H] source reads token 0 of every sequence
          if (!direct) {
            lda = (K + 3) / 4 * 4;
            e = launch_im2col(src, (float*)col, B, o.h, o.w, o.c, o.kh, o.kw, o.stride, o.pad, o.oh, o.ow, lda, st);
            if (e != cudaSuccess) return e;
            A = (const float*)col;
          }
          e = launch_gemm(A, W, bias, res, dst, B * o.oh * o.ow, o.cout, K, lda, o.act, st);
          break;
        }
        case OpKind::MaxPool: e = launch_maxpool(src, dst, B, o.h, o.w, o.c, o.kh, o.kw, o.stride, o.pad, o.oh, o.ow, st); break;
        case OpKind::AvgPool: e = launch_avgpool(src, dst, B, o.h * o.w, o.c, st); break;
        case OpKind::Embed:
          if (!o.norm) {
            e = launch_embed_positions(ids, stride ? stride : o.h, (const float*)(dm.dptr + o.word_off), (const float*)(dm.dptr + o.pos_off),
                                       dst, B, o.h, o.c, o.vocab, st);
            break;
          }
          e = launch_layernorm(nullptr, nullptr, ids, types, stride ? stride : o.h, (const float*)(dm.dptr + o.word_off),
                               (const float*)(dm.dptr + o.pos_off), (const float*)(dm.dptr + o.type_off),
                               (const float*)(dm.dptr + o.w_off), (const float*)(dm.dptr + o.b_off), dst, B * o.h, o.h, o.c, o.vocab,
                               o.eps, st);
          break;
        case OpKind::LayerNorm:
          e = launch_layernorm(src, o.res == -100 ? nullptr : (const float*)buf(o.res), nullptr, nullptr, 0, nullptr, nullptr, nullptr,
                               (const float*)(dm.dptr + o.w_off), (const float*)(dm.dptr + o.b_off), dst, B * o.h, o.h, o.c, 0, o.eps, st);
          break;
        case OpKind::Attention:
          if (o.causal) e = launch_attention_causal(src, mask_input, stride ? stride : o.h, dst, B, o.h, o.cout, o.heads, st);
          else e = launch_attention(src, mask, stride ? stride : o.h, dst, B, o.h, o.cout, o.heads, st);
          break;
        case OpKind::MaskGather:
          e = launch_mask_gather(src, ids, d.input(InputRole::Mask) ? mask : nullptr, stride ? stride : o.h, B, o.h, o.c, o.oh,
                                 o.mask_token_id, positions, dst, st);
          after_gather = true;
          break;
        case OpKind::DepthwiseConv:
          e = launch_depthwise_conv(src, (const float*)(dm.dptr + o.w_off), (const float*)(dm.dptr + o.b_off), dst, B, o.h, o.w, o.c,
                                    o.kh, o.kw, o.stride, o.pad, o.act, st);
          break;
        case OpKind::ChannelScale: e = launch_channel_scale(src, (const float*)buf(o.gate), dst, B, o.h * o.w, o.c, st); break;
        case OpKind::WindowAttention:
          e = launch_window_attention(src, (const float*)(dm.dptr + o.b_off), dst, B, o.h, o.w, o.cout, o.heads, o.window, o.shift, st);
          break;
        case OpKind::PatchMerge: e = launch_patch_merge(src, dst, B, o.h, o.w, o.c, st); break;
        case OpKind::LastToken:
          e = launch_last_token(src, mask_input, stride ? stride : o.h, B, o.h, o.c, positions, dst, st);
          after_gather = true;  // the vocabulary projection below 64 rows streams its weights, as fill-mask's
          break;
        case OpKind::TokenScore: {
          // the [B * S, Vp] logits would take B * S * Vp * 4 bytes (26 GB at 128 x 1024 tokens), so the projection runs on
          // chunks of kScoreChunkTokens token rows, each into the same region and then scored (DESIGN §4). A chunk takes the
          // route a next-token projection of that many rows takes: the weight-streaming dense kernels below 64 rows (the
          // cluster kernel up to 8, dense_tc from 9), the tensor-core GEMM from 64. Every route waits for the previous
          // chunk's score kernel (griddepcontrol.wait) before it writes the region.
          const ModelDesc::ScoreScratch ss = d.score_scratch(rows);
          float* logits = (float*)(scratch + ss.logits);
          const float* W = (const float*)(dm.dptr + o.w_off);
          const float* bias = (const float*)(dm.dptr + o.b_off);
          const int64_t tokens = (int64_t)B * o.h;
          for (int64_t first = 0; e == cudaSuccess && first < tokens; first += kScoreChunkTokens) {
            const int n = (int)std::min<int64_t>(kScoreChunkTokens, tokens - first);
            const float* xc = src + first * o.c;
            e = n < 64 && o.cout % 32 == 0 ? launch_dense(xc, W, bias, logits, n, o.c, o.cout, false, ws, ws_cap, st)
                                           : launch_gemm(xc, W, bias, nullptr, logits, n, o.cout, o.c, o.c, 0, st);
            if (e == cudaSuccess)
              e = launch_token_score(logits, o.cout, first, n, ids, mask_input, stride ? stride : o.h, o.h, o.vocab,
                                     (float*)(scratch + ss.log_probs), (int*)(scratch + ss.ranks), st);
          }
          break;
        }
      }
      return e;
    };
    // generate bundles: each attention op's K and V caches [rows, T, H], T = S + N - 1 slots
    const ModelDesc::GenerateScratch gs = d.head == HeadKind::Generate ? d.generate_scratch(rows) : ModelDesc::GenerateScratch();
    auto cache = [&](int attn, int v) { return (float*)(scratch + gs.kv + (2 * (size_t)attn + v) * gs.cache_bytes); };
    const int T = d.ops.front().h + d.head_k - 1;
    int attn = 0;
    for (const GraphOp& o : d.ops) {
      cudaError_t e = exec(o);
      if (e == cudaSuccess && d.head == HeadKind::Generate && o.kind == OpKind::Attention) {  // the prompt's keys and values
        e = launch_kv_cache_write((const float*)buf(o.src), cache(attn, 0), cache(attn, 1), B, o.h, T, o.cout, st);
        ++attn;
      }
      if (e != cudaSuccess) return e;
    }
    if (d.head == HeadKind::Generate) {
      // decoding: the prefill above left each row's logits at its last attended token p_b (positions); each step picks
      // (greedy) or draws (sampling) a token, embeds it at slot p_b + 1 + t into the embed op's buffer and runs the decoder
      // on that one token per row against the caches (DESIGN §4). A fixed N - 1 steps, no host synchronisation.
      const GraphOp& emb = d.ops.front();
      GenerateOutputs go;
      for (const ModelOutput& m : d.outputs) {
        float* p = reinterpret_cast<float*>(y) + m.offset;
        switch (m.kind) {
          case OutputKind::GeneratedIds: go.ids = reinterpret_cast<int*>(p), go.ids_ld = d.out_dim; break;
          case OutputKind::GeneratedLogProbs: go.log_probs = p, go.log_probs_ld = d.out_dim; break;
          case OutputKind::GeneratedLength: go.length = reinterpret_cast<int*>(p), go.length_ld = d.out_dim; break;
          default: break;
        }
      }
      int* done = reinterpret_cast<int*>(scratch + gs.done);
      // the decode attention counters start at zero and every launch leaves them so; the partials after them are written
      // before they are read
      cudaError_t e = cudaMemsetAsync(scratch + gs.work, 0, gs.counter_bytes, st);
      for (int t = 0; e == cudaSuccess && t < d.head_k; ++t) {
        after_gather = false;
        attn = 0;
        for (size_t i = 1; t > 0 && e == cudaSuccess && i < d.ops.size(); ++i) {
          GraphOp o = d.ops[i];
          if (o.kind == OpKind::LastToken) {  // a copy of each row's one token; the prompt's positions stay
            e = launch_last_token((const float*)buf(o.src), nullptr, 1, B, 1, o.c, nullptr, (float*)buf(o.dst), st);
            after_gather = true;
          } else if (o.kind == OpKind::Attention) {
            e = launch_decode_attention((const float*)buf(o.src), cache(attn, 0), cache(attn, 1), positions, t - 1, mask_input,
                                        stride ? stride : emb.h, emb.h, T, (float*)buf(o.dst), B, o.cout, o.heads,
                                        scratch + gs.work, st);
            ++attn;
          } else {
            if (!after_gather) o.h = o.oh = 1;  // the decoder's LayerNorms and 1x1 convs on one token per row
            e = exec(o);
          }
        }
        const int* seeds = d.gen_sampling ? (const int*)x + d.input(InputRole::Seed)->offset : nullptr;
        if (e == cudaSuccess && d.gen_processing)  // repetition control over each row's history of attended prompt and generated ids
          e = launch_generate_process((const float*)out, d.ops.back().cout, d.head_n, positions, t, t == d.head_k - 1, d.gen_eos,
                                      done, go, (const float*)(dm.dptr + emb.word_off), (const float*)(dm.dptr + emb.pos_off),
                                      (float*)buf(emb.dst), B, emb.c, ids, mask_input, stride ? stride : emb.h,
                                      reinterpret_cast<int*>(scratch + gs.hist), emb.h + d.head_k,
                                      reinterpret_cast<int*>(scratch + gs.hist_len0), d.gen_repetition_penalty, d.gen_no_repeat_ngram,
                                      d.gen_min_new_tokens, seeds, d.in_dim, d.gen_temperature, d.gen_top_k, d.gen_top_p, st);
        else if (e == cudaSuccess && d.gen_sampling)  // a sampling bundle draws each row's token with its seed (the loader's checks)
          e = launch_generate_sample((const float*)out, d.ops.back().cout, d.head_n, positions, t, t == d.head_k - 1, d.gen_eos,
                                     done, go, (const float*)(dm.dptr + emb.word_off), (const float*)(dm.dptr + emb.pos_off),
                                     (float*)buf(emb.dst), B, emb.c, seeds, d.in_dim, d.gen_temperature, d.gen_top_k, d.gen_top_p, st);
        else if (e == cudaSuccess)
          e = launch_generate_select((const float*)out, d.ops.back().cout, d.head_n, positions, t, t == d.head_k - 1, d.gen_eos,
                                     done, go, (const float*)(dm.dptr + emb.word_off), (const float*)(dm.dptr + emb.pos_off),
                                     (float*)buf(emb.dst), B, emb.c, st);
      }
      return e;
    }
    if (d.head == HeadKind::Score) {  // the token_score op left each scored token's log-probability and rank in scratch
      const ModelDesc::ScoreScratch ss = d.score_scratch(rows);
      ScoreOutputs so;
      for (const ModelOutput& m : d.outputs) {
        float* p = reinterpret_cast<float*>(y) + m.offset;
        switch (m.kind) {
          case OutputKind::TokenLogProbs: so.log_probs = p, so.log_probs_ld = d.out_dim; break;
          case OutputKind::TokenRanks: so.ranks = reinterpret_cast<int*>(p), so.ranks_ld = d.out_dim; break;
          case OutputKind::TokenLogProbSum: so.sum = p, so.sum_ld = d.out_dim; break;
          case OutputKind::TokenCount: so.count = reinterpret_cast<int*>(p), so.count_ld = d.out_dim; break;
          default: break;
        }
      }
      return launch_score_head((const float*)(scratch + ss.log_probs), (const int*)(scratch + ss.ranks), mask_input,
                               stride ? stride : d.head_n, B, d.head_n, so, st);
    }
    SpanInputs in;
    in.ids = ids;
    in.mask = d.input(InputRole::Mask) ? mask : nullptr;
    in.types = types;
    in.stride = stride;
    in.sep_id = d.span_sep_id;
    // with a pooler the hidden states are the pooler's source buffer and `out` holds its [rows, H] output
    const float* hidden = d.encoder_pooler ? (const float*)buf(d.ops.back().src) : nullptr;
    return run_head(d, (const float*)out, in, hidden, positions, rows, y, st);
  }
  char* act0 = scratch;
  char* act1 = scratch + d.scratch_bytes(rows) / 2;
  const char* in = x;
  for (size_t l = 0; l < d.layers.size(); ++l) {
    const DenseLayer& L = d.layers[l];
    // with signature.outputs the last layer writes its logits to the next activation buffer, and the head writes y
    char* out = (l + 1 == d.layers.size() && d.outputs.empty()) ? y : ((l & 1) ? act1 : act0);
    cudaError_t e = launch_dense((const float*)in, (const float*)(dm.dptr + L.w_off), (const float*)(dm.dptr + L.b_off),
                                 (float*)out, (int)rows, L.in, L.out, L.relu, ws, ws_cap, st);
    if (e != cudaSuccess) return e;
    in = out;
  }
  return run_head(d, (const float*)in, SpanInputs(), nullptr, nullptr, rows, y, st);
}

size_t Node::row_in_bytes(const ModelDesc& d) { return d.tmpl == Template::Affine ? 4 : (size_t)d.in_dim * 4; }
size_t Node::row_out_bytes(const ModelDesc& d) { return d.tmpl == Template::Affine ? 4 : (size_t)d.out_dim * 4; }
int64_t Node::now_ns() { return std::chrono::duration_cast<std::chrono::nanoseconds>(Clock::now().time_since_epoch()).count(); }

// ---- pinned request staging: power-of-two size classes, reused (cudaHostAlloc costs ~100 us + a page-table walk) ----
static size_t stage_class(size_t bytes) {
  size_t c = 4096;
  while (c < bytes) c <<= 1;
  return c;
}

void* Node::staging_alloc(size_t bytes) {
  const size_t c = stage_class(bytes ? bytes : 1);
  {
    std::lock_guard<std::mutex> lk(stage_mu_);
    auto it = stage_pool_.find(c);
    if (it != stage_pool_.end() && !it->second.empty()) {
      void* p = it->second.back();
      it->second.pop_back();
      stage_pooled_bytes_ -= c;
      return p;
    }
  }
  DeviceGuard g(cfg_.device);
  void* p = nullptr;
  // portable + mapped: under unified addressing the host pointer is valid in kernels of every device of the process
  if (cudaHostAlloc(&p, c, cudaHostAllocPortable | cudaHostAllocMapped) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  return p;
}

void Node::staging_free(void* p, size_t bytes) {
  if (!p) return;
  const size_t c = stage_class(bytes ? bytes : 1);
  {
    std::lock_guard<std::mutex> lk(stage_mu_);
    if (stage_pooled_bytes_ + c <= (size_t)cfg_.staging_pool_bytes) {
      stage_pool_[c].push_back(p);
      stage_pooled_bytes_ += c;
      return;
    }
  }
  cudaFreeHost(p);
}

bool Node::ensure_slot(Slot* s, const ModelDesc& d, int64_t rows, std::string* err) {
  int64_t cap_rows = rows > cfg_.max_batch ? rows : cfg_.max_batch;
  size_t io = (size_t)cap_rows * std::max(row_in_bytes(d), row_out_bytes(d));
  size_t act = d.scratch_bytes(cap_rows);
  size_t ws = model_ws_bytes(d);
  if (io > s->io_cap) {
    cudaStreamSynchronize(compute_);
    if (s->d_in) cudaFree(s->d_in);
    if (s->d_out) cudaFree(s->d_out);
    s->d_in = s->d_out = nullptr;
    s->io_cap = 0;
    CU_OK(cudaMalloc((void**)&s->d_in, io), err, false);
    CU_OK(cudaMalloc((void**)&s->d_out, io), err, false);
    s->io_cap = io;
  }
  if (act > s->scratch_cap) {
    cudaStreamSynchronize(compute_);
    if (s->scratch) cudaFree(s->scratch);
    s->scratch = nullptr;
    s->scratch_cap = 0;
    CU_OK(cudaMalloc((void**)&s->scratch, act), err, false);
    s->scratch_cap = act;
  }
  if (ws > s->ws_cap) {
    cudaStreamSynchronize(compute_);
    if (s->ws) cudaFree(s->ws);
    s->ws = nullptr;
    s->ws_cap = 0;
    CU_OK(cudaMalloc(&s->ws, ws), err, false);
    CU_OK(cudaMemsetAsync(s->ws, 0, ws, compute_), err, false);
    s->ws_cap = ws;
  }
  return true;
}

int Node::describe(const ModelId& id, ModelDesc* desc, int* outcome, std::string* err) {
  std::shared_ptr<DeviceModel> dm;
  int rc = fetch(id, &dm, err);
  if (rc < 0) return rc;
  if (outcome) *outcome = rc;
  *desc = dm->desc;
  unpin(dm);
  return 0;
}

int Node::prepare(const ModelId& id, const InputLayout& l, PredictRequest* req, int* outcome, std::string* err) {
  int rc = fetch(id, &req->dm, err);  // handleModelRequest -> fetchModel, before any input validation (as the reference)
  if (rc < 0) return rc;
  if (outcome) *outcome = rc;
  const ModelDesc& d = req->dm->desc;
  const int64_t per_row = d.tmpl == Template::Affine ? 1 : d.in_dim;
  auto reject = [&](const std::string& msg) {
    unpin(req->dm);
    req->dm.reset();
    *err = msg;
    return TFSC_E_INVALID;
  };
  std::string why;
  if (!check_layout(d, l, &why)) return reject(why);
  const int64_t n_elems = l.n_elems;
  const int in_dtype = l.dtype;
  if (l.multi()) {
    if (l.rows > cfg_.max_request_rows)
      return reject("request has " + std::to_string(l.rows) + " rows; gpu.maxRequestRows is " + std::to_string(cfg_.max_request_rows));
    req->rows = l.rows;
    return 0;
  }
  if (in_dtype != d.input_dtype)
    return reject("input dtype " + std::to_string(in_dtype) + " does not match the model signature (expects dtype " +
                  std::to_string(d.input_dtype) + ")");
  if (n_elems <= 0 || n_elems % per_row != 0)
    return reject("input has " + std::to_string(n_elems) + " elements; model " + id.name + " expects a multiple of " +
                  std::to_string(per_row));
  const int64_t rows = n_elems / per_row;
  if (rows > cfg_.max_request_rows)
    return reject("request has " + std::to_string(rows) + " rows; gpu.maxRequestRows is " + std::to_string(cfg_.max_request_rows));
  req->rows = rows;
  return 0;
}

void Node::abandon(PredictRequest* req) {
  if (req->dm) {
    unpin(req->dm);
    req->dm.reset();
  }
}

void Node::enqueue(PredictRequest* req) {
  req->rc = 1;
  req->arrival_ns = now_ns();
  {
    std::lock_guard<std::mutex> lk(q_mu_);
    req->seq = ++seq_;
    auto& q = pending_[req->dm.get()];
    if (q.empty()) order_.insert({req->seq, req->dm.get()});
    q.push_back(req);
  }
  q_cv_.notify_all();
}

// completion: release the model pin, then hand the result over. Nothing of `r` may be touched after the hand-over (a
// synchronous caller destroys the request as soon as it sees rc != 1; on_done owns the request's lifetime).
void Node::complete(PredictRequest* r, int rc, const std::string& err) {
  std::shared_ptr<DeviceModel> dm = std::move(r->dm);
  if (dm) unpin(dm);
  if (r->on_done) {
    r->err = err;
    r->rc = rc;
    auto fn = std::move(r->on_done);
    fn(r);
    return;
  }
  std::lock_guard<std::mutex> l(r->mu);
  r->err = err;
  r->rc = rc;
  r->cv.notify_all();
}

int Node::predict_host(const ModelId& id, const void* x, int64_t n_elems, int in_dtype, const OutAllocFn& y_alloc,
                       int* outcome, ModelDesc* desc_out, std::string* err, int64_t deadline_ns) {
  std::vector<InTensor> ts(1);
  ts[0].dtype = in_dtype;
  ts[0].data = x;
  ts[0].n = x ? n_elems : 0;
  const InputLayout l = layout_inputs(&ts);
  return predict_host(id, ts, l, y_alloc, outcome, desc_out, err, deadline_ns);
}

int Node::predict_host(const ModelId& id, const std::vector<InTensor>& ts, const InputLayout& l, const OutAllocFn& y_alloc,
                       int* outcome, ModelDesc* desc_out, std::string* err, int64_t deadline_ns) {
  PredictRequest req;
  int rc = prepare(id, l, &req, outcome, err);
  if (rc < 0) return rc;
  const ModelDesc& d = req.dm->desc;
  if (desc_out) *desc_out = d;
  void* y = y_alloc(d, req.rows);
  if (!y) {
    abandon(&req);
    *err = "output buffer too small";
    return TFSC_E_BUFFER;
  }
  // the client thread stages its own rows (pinned, device-accessible): the batcher thread never touches request payloads,
  // the gather kernel pulls the rows over PCIe straight into the batch buffer
  const size_t in_b = (size_t)req.rows * row_in_bytes(d), out_b = (size_t)req.rows * row_out_bytes(d);
  const size_t in_al = (in_b + 255) & ~(size_t)255;
  char* st = static_cast<char*>(staging_alloc(in_al + out_b));
  if (!st) {
    abandon(&req);
    *err = "cannot pin " + std::to_string(in_al + out_b) + " bytes of request staging";
    return TFSC_E_EXHAUSTED;
  }
  pack_rows(ts, l, req.rows, st);  // one tensor: the same bytes as a memcpy of it
  req.x = st;
  req.y = st + in_al;
  req.host_staged = true;
  req.deadline_ns = deadline_ns;
  enqueue(&req);
  {
    std::unique_lock<std::mutex> lk(req.mu);
    req.cv.wait(lk, [&] { return req.rc != 1; });
  }
  if (req.rc == 0) memcpy(y, st + in_al, out_b);
  staging_free(st, in_al + out_b);
  if (req.rc < 0) *err = req.err;
  return req.rc;
}

void Node::batcher_loop() {
  cudaSetDevice(cfg_.device);
  std::vector<CopySeg> segs;
  for (;;) {
    std::unique_lock<std::mutex> lk(q_mu_);
    q_cv_.wait(lk, [&] { return stop_ || !order_.empty(); });
    if (order_.empty()) {
      if (stop_) break;
      continue;
    }
    // oldest-request-first: requests are served in arrival order, and every request of the same
    // model that is already queued rides along (up to gpu.maxBatch rows) in the same pass over W
    DeviceModel* m = order_.begin()->second;
    auto& q = pending_[m];
    if (cfg_.tick_us > 0 && !stop_) {
      // batching window (gpu.tickMicros): a partial batch waits for more rows until its oldest request is tick old
      int64_t queued = 0;
      for (auto* r : q) queued += r->rows;
      const int64_t due = q.front()->arrival_ns + (int64_t)cfg_.tick_us * 1000;
      const int64_t now = now_ns();
      if (queued < cfg_.max_batch && now < due) {
        q_cv_.wait_for(lk, std::chrono::nanoseconds(due - now));
        continue;  // re-evaluate: more rows may have arrived, or another model is now the oldest
      }
    }
    order_.erase(order_.begin());
    std::vector<PredictRequest*> batch, expired;
    int64_t rows = 0;
    const int64_t now = now_ns();
    while (!q.empty()) {
      PredictRequest* r = q.front();
      if (r->deadline_ns > 0 && now > r->deadline_ns) {  // still queued past its deadline: never launched
        expired.push_back(r);
        q.pop_front();
        continue;
      }
      if (!batch.empty() && rows + r->rows > cfg_.max_batch) break;
      batch.push_back(r);
      rows += r->rows;
      q.pop_front();
      if (rows >= cfg_.max_batch) break;
    }
    if (!q.empty()) order_.insert({q.front()->seq, m});
    else pending_.erase(m);
    if (!expired.empty()) {
      lk.unlock();
      for (auto* r : expired) complete(r, TFSC_E_TIMEOUT, "deadline exceeded while queued");
      lk.lock();
    }
    if (batch.empty()) continue;
    Slot* s = nullptr;
    slot_cv_.wait(lk, [&] {
      for (auto& c : slots_)
        if (!c.busy) {
          s = &c;
          return true;
        }
      return stop_;
    });
    if (!s) {  // shutting down
      lk.unlock();
      for (auto* r : batch) complete(r, TFSC_E_INTERNAL, "server shutting down");
      continue;
    }
    s->busy = true;
    lk.unlock();

    std::shared_ptr<DeviceModel> dm = batch[0]->dm;
    const ModelDesc& d = dm->desc;
    std::string err;
    cudaError_t e = cudaSuccess;
    if (!ensure_slot(s, d, rows, &err)) e = cudaErrorMemoryAllocation;
    const size_t rin = row_in_bytes(d), rout = row_out_bytes(d);
    if (e == cudaSuccess) {
      // three streams: gather | kernels | scatter, chained by events, so the transfers of neighbouring batches overlap
      // the weight-streaming kernels instead of serialising with them. Gather and scatter are one kernel each over a
      // segment table (X6): sources / destinations are pinned host staging (PCIe), local HBM or peer windows (NVLink, X7).
      segs.clear();
      size_t off = 0;
      int64_t h2d = 0;
      for (auto* r : batch) {
        segs.push_back({r->x, s->d_in + off, (uint64_t)r->rows * rin});
        if (r->host_staged) h2d += (int64_t)((size_t)r->rows * rin);
        off += (size_t)r->rows * rin;
      }
      e = launch_copy_segments(segs.data(), (int)segs.size(), in_);
      h2d_inputs_ += h2d;
      if (e == cudaSuccess) e = cudaEventRecord(s->in_done, in_);
      if (e == cudaSuccess) e = cudaStreamWaitEvent(compute_, s->in_done, 0);
      if (e == cudaSuccess && !dm->ready_seen) e = cudaStreamWaitEvent(compute_, dm->ready, 0);
      if (e == cudaSuccess) e = run_model(*dm, s->d_in, rows, s->d_out, s->scratch, s->ws, s->ws_cap, compute_);
      if (e == cudaSuccess) e = cudaEventRecord(s->k_done, compute_);
      if (e == cudaSuccess) e = cudaStreamWaitEvent(out_, s->k_done, 0);
      segs.clear();
      off = 0;
      int64_t d2h = 0;
      for (auto* r : batch) {
        segs.push_back({s->d_out + off, r->y, (uint64_t)r->rows * rout});
        if (r->host_staged) d2h += (int64_t)((size_t)r->rows * rout);
        off += (size_t)r->rows * rout;
      }
      if (e == cudaSuccess) e = launch_copy_segments(segs.data(), (int)segs.size(), out_);
      d2h_outputs_ += d2h;
      if (e == cudaSuccess) e = cudaEventRecord(s->done, out_);
    }
    batches_++;
    batched_rows_ += rows;
    if (e != cudaSuccess) {
      if (err.empty()) err = std::string("launch failed: ") + cudaGetErrorString(e);
      cudaGetLastError();
      cudaDeviceSynchronize();  // nothing of this batch may still write into the requests' buffers
      cudaGetLastError();
      for (auto* r : batch) complete(r, TFSC_E_INTERNAL, err);
      lk.lock();
      s->busy = false;
      lk.unlock();
      slot_cv_.notify_all();
      continue;
    }
    s->reqs = std::move(batch);
    s->dm = dm;
    lk.lock();
    inflight_.push_back(s);
    lk.unlock();
    q_cv_.notify_all();
  }
  // shutting down: whatever is still queued fails
  std::vector<PredictRequest*> rest;
  {
    std::lock_guard<std::mutex> lk(q_mu_);
    for (auto& kv : pending_)
      for (auto* r : kv.second) rest.push_back(r);
    pending_.clear();
    order_.clear();
  }
  for (auto* r : rest) complete(r, TFSC_E_INTERNAL, "server shutting down");
}

void Node::completer_loop() {
  cudaSetDevice(cfg_.device);
  for (;;) {
    Slot* s = nullptr;
    {
      std::unique_lock<std::mutex> lk(q_mu_);
      q_cv_.wait(lk, [&] { return !inflight_.empty() || batcher_done_; });
      if (inflight_.empty()) {
        if (batcher_done_) break;
        continue;
      }
      s = inflight_.front();
      inflight_.pop_front();
    }
    cudaError_t e = cudaEventSynchronize(s->done);
    const std::string msg = e == cudaSuccess ? std::string() : std::string("execution failed: ") + cudaGetErrorString(e);
    std::vector<PredictRequest*> reqs = std::move(s->reqs);
    s->reqs.clear();
    s->dm.reset();
    {
      std::lock_guard<std::mutex> lk(q_mu_);
      s->busy = false;  // the slot's device buffers are free again (results already sit in the requests' own buffers)
    }
    slot_cv_.notify_all();
    for (auto* r : reqs) complete(r, e == cudaSuccess ? 0 : TFSC_E_INTERNAL, msg);
  }
}

int Node::predict_device(const ModelId& id, const void* x, int64_t rows, void* y, cudaStream_t stream,
                         std::string* err) {
  DeviceGuard g(cfg_.device);
  if (rows <= 0) return 0;
  std::shared_ptr<DeviceModel> dm;
  cudaEvent_t ev;
  {
    std::lock_guard<std::mutex> lk(mu_);
    reap_locked();
    auto it = dev_.find(id);
    if (it != dev_.end()) refresh_state_locked(it->second.get());
    if (it == dev_.end() || !(it->second->state == TFSC_STATE_AVAILABLE || it->second->state == TFSC_STATE_LOADING)) {
      *err = "model " + id.name + ":" + std::to_string(id.version) + " is not HBM-resident (call tfsc_model_ensure)";
      return TFSC_E_NOT_FOUND;
    }
    dm = it->second;
    dm->inflight++;
    ev = get_event();
  }
  cudaStream_t st = stream ? stream : compute_;
  const ModelDesc& d = dm->desc;
  cudaError_t e = cudaSuccess;
  StreamScratch* sc = nullptr;
  if (d.tmpl != Template::Affine) {
    const size_t act = d.scratch_bytes(rows);
    const size_t ws = model_ws_bytes(d);
    std::lock_guard<std::mutex> lk(scratch_mu_);
    sc = &stream_scratch_[st];
    if (sc->act_bytes < act || sc->ws_bytes < ws) {
      if (sc->base) {
        cudaStreamSynchronize(st);
        cudaFree(sc->base);
        sc->base = nullptr;
      }
      size_t a = act > sc->act_bytes ? act : sc->act_bytes, w = ws > sc->ws_bytes ? ws : sc->ws_bytes;
      e = cudaMalloc((void**)&sc->base, a + w);
      if (e == cudaSuccess) e = cudaMemsetAsync(sc->base + a, 0, w, st);
      sc->act_bytes = a;
      sc->ws_bytes = w;
    }
  }
  if (e == cudaSuccess && !dm->ready_seen) e = cudaStreamWaitEvent(st, dm->ready, 0);
  if (e == cudaSuccess) {
    char* a0 = sc ? sc->base : nullptr;
    void* ws = sc ? sc->base + sc->act_bytes : nullptr;
    e = run_model(*dm, (const char*)x, rows, (char*)y, a0, ws, sc ? sc->ws_bytes : 0, st);
  }
  if (e == cudaSuccess) e = cudaEventRecord(ev, st);
  {
    std::lock_guard<std::mutex> lk(mu_);
    if (e == cudaSuccess) retire_.push_back({ev, dm});
    else {
      put_event(ev);
      if (--dm->inflight == 0 && dm->state == TFSC_STATE_UNLOADING) release_locked(dm);
    }
  }
  if (e != cudaSuccess) {
    cudaGetLastError();
    *err = std::string("predict_device: ") + cudaGetErrorString(e);
    return TFSC_E_INTERNAL;
  }
  return 0;
}

int Node::sync() {
  DeviceGuard g(cfg_.device);
  cudaError_t e = cudaDeviceSynchronize();
  std::lock_guard<std::mutex> lk(mu_);
  reap_locked();
  return e == cudaSuccess ? 0 : TFSC_E_INTERNAL;
}

}  // namespace tfsc
