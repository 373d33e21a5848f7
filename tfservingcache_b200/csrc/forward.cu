#include "forward.h"

#include <errno.h>
#include <poll.h>
#include <sys/socket.h>
#include <sys/time.h>
#include <sys/un.h>
#include <unistd.h>

#include <chrono>
#include <cstring>

namespace tfsc {

namespace {

enum : uint8_t { MSG_HELLO = 1, MSG_HELLO_ACK = 2, MSG_FWD = 3, MSG_DONE = 4 };

struct Writer {
  std::string b;
  void u32(uint32_t v) { b.append(reinterpret_cast<const char*>(&v), 4); }
  void i32(int32_t v) { b.append(reinterpret_cast<const char*>(&v), 4); }
  void u64(uint64_t v) { b.append(reinterpret_cast<const char*>(&v), 8); }
  void i64(int64_t v) { b.append(reinterpret_cast<const char*>(&v), 8); }
  void str(const std::string& s) {
    u32((uint32_t)s.size());
    b.append(s);
  }
  void raw(const void* p, size_t n) { b.append(static_cast<const char*>(p), n); }
  void vec(const std::vector<int64_t>& v) {
    u32((uint32_t)v.size());
    for (auto x : v) i64(x);
  }
};

struct Reader {
  const char* p;
  size_t n;
  bool ok = true;
  Reader(const std::string& s) : p(s.data()), n(s.size()) {}
  bool take(void* out, size_t k) {
    if (!ok || k > n) {
      ok = false;
      memset(out, 0, k);
      return false;
    }
    memcpy(out, p, k);
    p += k;
    n -= k;
    return true;
  }
  uint32_t u32() { uint32_t v; take(&v, 4); return v; }
  int32_t i32() { int32_t v; take(&v, 4); return v; }
  uint64_t u64() { uint64_t v; take(&v, 8); return v; }
  int64_t i64() { int64_t v; take(&v, 8); return v; }
  std::string str() {
    uint32_t k = u32();
    if (!ok || k > n) {
      ok = false;
      return {};
    }
    std::string s(p, k);
    p += k;
    n -= k;
    return s;
  }
  std::vector<int64_t> vec() {
    uint32_t k = u32();
    std::vector<int64_t> v;
    if (k > 64) ok = false;
    for (uint32_t i = 0; ok && i < k; ++i) v.push_back(i64());
    return v;
  }
};

bool write_all(int fd, const void* buf, size_t n) {
  const char* p = static_cast<const char*>(buf);
  while (n > 0) {
    ssize_t w = ::send(fd, p, n, MSG_NOSIGNAL);
    if (w < 0) {
      if (errno == EINTR) continue;
      return false;
    }
    p += w;
    n -= (size_t)w;
  }
  return true;
}

bool read_all(int fd, void* buf, size_t n) {
  char* p = static_cast<char*>(buf);
  while (n > 0) {
    ssize_t r = ::recv(fd, p, n, 0);
    if (r == 0) return false;
    if (r < 0) {
      if (errno == EINTR) continue;
      return false;
    }
    p += r;
    n -= (size_t)r;
  }
  return true;
}

bool read_msg(int fd, uint8_t* type, std::string* payload) {
  uint32_t len = 0;
  if (!read_all(fd, &len, 4) || len < 1 || len > (1u << 20)) return false;
  std::string buf(len, '\0');
  if (!read_all(fd, &buf[0], len)) return false;
  *type = (uint8_t)buf[0];
  payload->assign(buf, 1, std::string::npos);
  return true;
}

// bound a blocking handshake read (a peer that accepted but never answers must not hang the caller forever)
void set_rcv_timeout(int fd, double seconds) {
  timeval tv;
  tv.tv_sec = (time_t)seconds;
  tv.tv_usec = (suseconds_t)((seconds - (double)tv.tv_sec) * 1e6);
  setsockopt(fd, SOL_SOCKET, SO_RCVTIMEO, &tv, sizeof tv);
}

bool make_addr(const std::string& endpoint, sockaddr_un* addr, socklen_t* len, std::string* path_out) {
  std::string path = endpoint.rfind("unix:", 0) == 0 ? endpoint.substr(5) : endpoint;
  if (path.empty() || path.size() >= sizeof(addr->sun_path)) return false;
  memset(addr, 0, sizeof *addr);
  addr->sun_family = AF_UNIX;
  memcpy(addr->sun_path, path.data(), path.size());
  *len = (socklen_t)(offsetof(sockaddr_un, sun_path) + path.size() + 1);
  if (path[0] == '@') {  // abstract namespace: no file to clean up
    addr->sun_path[0] = '\0';
    *len = (socklen_t)(offsetof(sockaddr_un, sun_path) + path.size());
  }
  if (path_out) *path_out = path;
  return true;
}

void write_sig(Writer* w, const FwdSignature& s) {
  w->i32(s.tmpl);
  w->i64(s.in_dim);
  w->i64(s.out_dim);
  w->i32(s.input_dtype);
  w->str(s.input_name);
  w->str(s.output_name);
  w->vec(s.input_shape);
  w->vec(s.output_shape);
  w->u32((uint32_t)s.input_names.size());
  for (size_t i = 0; i < s.input_names.size(); ++i) {
    w->str(s.input_names[i]);
    w->i32(s.input_roles[i]);
  }
  w->u32((uint32_t)s.output_names.size());
  for (size_t i = 0; i < s.output_names.size(); ++i) {
    w->str(s.output_names[i]);
    w->i32(s.output_kinds[i]);
  }
  w->i32(s.head_n);
  w->i32(s.head_k);
}

FwdSignature read_sig(Reader* r) {
  FwdSignature s;
  s.tmpl = r->i32();
  s.in_dim = r->i64();
  s.out_dim = r->i64();
  s.input_dtype = r->i32();
  s.input_name = r->str();
  s.output_name = r->str();
  s.input_shape = r->vec();
  s.output_shape = r->vec();
  const uint32_t k = r->u32();
  if (k > 3) r->ok = false;
  for (uint32_t i = 0; r->ok && i < k; ++i) {
    s.input_names.push_back(r->str());
    s.input_roles.push_back(r->i32());
  }
  const uint32_t m = r->u32();
  if (m > (uint32_t)kMaxOutputs) r->ok = false;
  for (uint32_t i = 0; r->ok && i < m; ++i) {
    s.output_names.push_back(r->str());
    const int32_t kind = r->i32();
    if (kind < 0 || kind > (int32_t)kLastOutputKind) r->ok = false;
    s.output_kinds.push_back(kind);
  }
  s.head_n = r->i32();
  s.head_k = r->i32();
  return s;
}

// one mapping per peer window and process (a handle must not be opened twice in one context)
std::mutex g_map_mu;
std::map<std::string, std::pair<char*, int>> g_mapped;  // handle bytes -> (ptr, refs)

char* map_window(const cudaIpcMemHandle_t& h, int device, std::string* err) {
  std::lock_guard<std::mutex> lk(g_map_mu);
  std::string key(reinterpret_cast<const char*>(&h), sizeof h);
  auto it = g_mapped.find(key);
  if (it != g_mapped.end()) {
    it->second.second++;
    return it->second.first;
  }
  DeviceGuard g(device);
  void* p = nullptr;
  cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) {
    cudaGetLastError();
    *err = std::string("cudaIpcOpenMemHandle: ") + cudaGetErrorString(e);
    return nullptr;
  }
  g_mapped[key] = {static_cast<char*>(p), 1};
  return static_cast<char*>(p);
}

void unmap_window(char* p) {
  if (!p) return;
  std::lock_guard<std::mutex> lk(g_map_mu);
  for (auto it = g_mapped.begin(); it != g_mapped.end(); ++it)
    if (it->second.first == p) {
      if (--it->second.second == 0) {
        cudaIpcCloseMemHandle(p);
        g_mapped.erase(it);
      }
      return;
    }
}

}  // namespace

void FwdSignature::to_desc(ModelDesc* d) const {
  d->tmpl = tmpl == 0 ? Template::Affine : tmpl == 2 ? Template::Graph : Template::Mlp;
  d->in_dim = in_dim;
  d->out_dim = out_dim;
  d->input_dtype = input_dtype;
  d->input_name = input_name;
  d->output_name = output_name;
  d->input_shape = input_shape;
  d->output_shape = output_shape;
  d->inputs.clear();
  const int64_t S = input_names.empty() ? 0 : in_dim / (int64_t)input_names.size();
  for (size_t i = 0; i < input_names.size(); ++i)
    d->inputs.push_back({input_names[i], (InputRole)input_roles[i], (int64_t)i * S});
  // the ingress rank splits the packed response rows with the owner's layout rule (layout_outputs), never with its own manifest
  d->outputs.clear();
  d->head_n = head_n;
  d->head_k = head_k;
  for (size_t i = 0; i < output_names.size(); ++i) {
    ModelOutput o;
    o.name = output_names[i];
    o.kind = (OutputKind)output_kinds[i];
    d->outputs.push_back(o);
  }
  std::string err;
  if (!d->outputs.empty() && !layout_outputs(d, &err)) {  // unusable: no front-end can size a response for 0 words per row
    d->outputs.clear();
    d->head = HeadKind::None;
    d->out_dim = 0;
  }
}

FwdSignature FwdSignature::from_desc(const ModelDesc& d) {
  FwdSignature s;
  s.tmpl = d.tmpl == Template::Affine ? 0 : d.tmpl == Template::Graph ? 2 : 1;
  s.in_dim = d.in_dim;
  s.out_dim = d.out_dim;
  s.input_dtype = d.input_dtype;
  s.input_name = d.input_name;
  s.output_name = d.output_name;
  s.input_shape = d.input_shape;
  s.output_shape = d.output_shape;
  for (auto& mi : d.inputs) {
    s.input_names.push_back(mi.name);
    s.input_roles.push_back((int32_t)mi.role);
  }
  for (auto& mo : d.outputs) {
    s.output_names.push_back(mo.name);
    s.output_kinds.push_back((int32_t)mo.kind);
  }
  s.head_n = d.head_n;
  s.head_k = d.head_k;
  return s;
}

Forwarder::Forwarder(const FwdConfig& cfg, Node* node) : cfg_(cfg), node_(node) {}

bool Forwarder::init(std::string* err) {
  if (cfg_.rank < 0 || cfg_.rank >= (int)cfg_.endpoints.size()) {
    *err = "cluster.rank out of range of cluster.endpoints";
    return false;
  }
  if (cfg_.slots < 1 || cfg_.slot_bytes < 1024 || cfg_.slot_bytes % 512 != 0) {
    *err = "cluster.windowSlots >= 1 and cluster.slotBytes a multiple of 512 (>= 1024) required";
    return false;
  }
  DeviceGuard g(node_->device());
  cudaError_t e = cudaMalloc((void**)&window_, window_bytes());
  if (e == cudaSuccess) e = cudaMemset(window_, 0, window_bytes());
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&handle_, window_);
  for (auto& st : streams_)
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
  if (e != cudaSuccess) {
    cudaGetLastError();
    *err = std::string("forward window: ") + cudaGetErrorString(e);
    return false;
  }
  for (int i = cfg_.slots - 1; i >= 0; --i) free_slots_.push_back(i);

  sockaddr_un addr;
  socklen_t alen;
  if (!make_addr(cfg_.endpoints[cfg_.rank], &addr, &alen, &listen_path_)) {
    *err = "bad cluster endpoint '" + cfg_.endpoints[cfg_.rank] + "' (unix socket path, at most 107 bytes)";
    return false;
  }
  listen_fd_ = ::socket(AF_UNIX, SOCK_STREAM | SOCK_CLOEXEC, 0);
  if (listen_fd_ < 0) {
    *err = std::string("socket: ") + strerror(errno);
    return false;
  }
  if (listen_path_[0] != '@') ::unlink(listen_path_.c_str());
  if (::bind(listen_fd_, reinterpret_cast<sockaddr*>(&addr), alen) != 0 || ::listen(listen_fd_, 64) != 0) {
    *err = "bind/listen " + listen_path_ + ": " + strerror(errno);
    ::close(listen_fd_);
    listen_fd_ = -1;
    return false;
  }
  acceptor_ = std::thread([this] { accept_loop(); });
  for (int i = 0; i < cfg_.workers; ++i) workers_.emplace_back([this] { worker_loop(); });
  return true;
}

Forwarder::~Forwarder() {
  // let the node finish what other ranks already handed us (their buffers are our peers' memory), then tear down
  for (int i = 0; i < 500; ++i) {
    {
      std::lock_guard<std::mutex> lk(inc_mu_);
      if (incoming_.empty()) break;
    }
    std::this_thread::sleep_for(std::chrono::milliseconds(10));
  }
  stop_ = true;
  if (listen_fd_ >= 0) {
    ::shutdown(listen_fd_, SHUT_RDWR);
    ::close(listen_fd_);
  }
  if (acceptor_.joinable()) acceptor_.join();
  std::vector<std::shared_ptr<Conn>> all;
  {
    std::lock_guard<std::mutex> lk(conn_mu_);
    for (auto& kv : out_) all.push_back(kv.second);
    out_.clear();
  }
  {
    std::lock_guard<std::mutex> lk(in_mu_);
    for (auto& c : in_) all.push_back(c);
    in_.clear();
  }
  for (auto& c : all)
    if (c->fd >= 0) ::shutdown(c->fd, SHUT_RDWR);
  for (auto& c : all)
    if (c->reader.joinable()) c->reader.join();
  job_cv_.notify_all();
  for (auto& w : workers_)
    if (w.joinable()) w.join();
  for (auto& c : all) {
    if (c->fd >= 0) ::close(c->fd);
    unmap_window(c->peer_win);
  }
  if (!listen_path_.empty() && listen_path_[0] != '@') ::unlink(listen_path_.c_str());
  DeviceGuard g(node_->device());
  for (auto& st : streams_)
    if (st) cudaStreamDestroy(st);
  if (window_) cudaFree(window_);
}

bool Forwarder::send_msg(Conn* c, uint8_t type, const std::string& payload) {
  std::string frame;
  uint32_t len = (uint32_t)payload.size() + 1;
  frame.append(reinterpret_cast<const char*>(&len), 4);
  frame.push_back((char)type);
  frame.append(payload);
  std::lock_guard<std::mutex> lk(c->wmu);
  if (c->dead || !write_all(c->fd, frame.data(), frame.size())) {
    c->dead = true;
    return false;
  }
  return true;
}

// ------------------------------------------------------------------ connections ------
std::shared_ptr<Forwarder::Conn> Forwarder::get_conn(int peer, std::string* err) {
  if (peer < 0 || peer >= world() || peer == cfg_.rank) {
    *err = "forward: bad peer rank " + std::to_string(peer);
    return nullptr;
  }
  std::lock_guard<std::mutex> lk(conn_mu_);  // grpcConnMap's write lock: one dial per peer
  auto it = out_.find(peer);
  if (it != out_.end() && !it->second->dead) return it->second;
  if (it != out_.end()) {
    // the old connection died: its reader thread exits on its own; keep the object alive until then
    std::shared_ptr<Conn> old = it->second;
    out_.erase(it);
    if (old->reader.joinable()) old->reader.detach();
  }
  sockaddr_un addr;
  socklen_t alen;
  if (!make_addr(cfg_.endpoints[peer], &addr, &alen, nullptr)) {
    *err = "bad cluster endpoint '" + cfg_.endpoints[peer] + "'";
    return nullptr;
  }
  // the peer may still be starting (grpc.Dial WithBlock + proxy.grpcTimeout in the reference)
  const auto deadline = std::chrono::steady_clock::now() + std::chrono::duration<double>(cfg_.timeout_s);
  int fd = -1;
  for (;;) {
    fd = ::socket(AF_UNIX, SOCK_STREAM | SOCK_CLOEXEC, 0);
    if (fd < 0) {
      *err = std::string("socket: ") + strerror(errno);
      return nullptr;
    }
    if (::connect(fd, reinterpret_cast<sockaddr*>(&addr), alen) == 0) break;
    ::close(fd);
    fd = -1;
    if (stop_ || std::chrono::steady_clock::now() >= deadline) {
      *err = "forward: cannot reach rank " + std::to_string(peer) + " at " + cfg_.endpoints[peer] + ": " + strerror(errno);
      return nullptr;
    }
    std::this_thread::sleep_for(std::chrono::milliseconds(20));
  }
  auto c = std::make_shared<Conn>();
  c->fd = fd;
  c->peer = peer;
  Writer w;
  w.u32((uint32_t)cfg_.rank);
  w.u64(window_bytes());
  w.u64(cfg_.slot_bytes);
  w.raw(&handle_, sizeof handle_);
  uint8_t type = 0;
  std::string payload;
  set_rcv_timeout(fd, cfg_.timeout_s);
  if (!send_msg(c.get(), MSG_HELLO, w.b) || !read_msg(fd, &type, &payload) || type != MSG_HELLO_ACK) {
    *err = "forward: handshake with rank " + std::to_string(peer) + " failed";
    ::close(fd);
    return nullptr;
  }
  Reader r(payload);
  const int their_rank = (int)r.u32();
  c->peer_win_bytes = r.u64();
  c->peer_slot_bytes = r.u64();
  cudaIpcMemHandle_t h;
  r.take(&h, sizeof h);
  if (!r.ok || their_rank != peer) {
    *err = "forward: rank " + std::to_string(peer) + " answered a malformed handshake";
    ::close(fd);
    return nullptr;
  }
  c->peer_win = map_window(h, node_->device(), err);
  if (!c->peer_win) {
    ::close(fd);
    return nullptr;
  }
  set_rcv_timeout(fd, 0.0);   // the reader thread blocks until the peer speaks or the socket is shut down
  out_[peer] = c;
  c->reader = std::thread([this, c] { reader_loop(c, false); });
  return c;
}

char* Forwarder::peer_window(int peer, size_t* bytes, std::string* err) {
  auto c = get_conn(peer, err);
  if (!c) return nullptr;
  if (bytes) *bytes = c->peer_win_bytes;
  return c->peer_win;
}

void Forwarder::accept_loop() {
  while (!stop_) {
    pollfd pfd{listen_fd_, POLLIN, 0};
    int pr = ::poll(&pfd, 1, 200);
    if (pr <= 0) continue;
    int fd = ::accept4(listen_fd_, nullptr, nullptr, SOCK_CLOEXEC);
    if (fd < 0) {
      if (stop_) break;
      continue;
    }
    uint8_t type = 0;
    std::string payload;
    set_rcv_timeout(fd, 5.0);
    if (!read_msg(fd, &type, &payload) || type != MSG_HELLO) {
      ::close(fd);
      continue;
    }
    set_rcv_timeout(fd, 0.0);
    Reader r(payload);
    auto c = std::make_shared<Conn>();
    c->fd = fd;
    c->peer = (int)r.u32();
    c->peer_win_bytes = r.u64();
    c->peer_slot_bytes = r.u64();
    cudaIpcMemHandle_t h;
    r.take(&h, sizeof h);
    std::string err;
    if (r.ok) c->peer_win = map_window(h, node_->device(), &err);
    if (!r.ok || !c->peer_win) {
      ::close(fd);
      continue;
    }
    Writer w;
    w.u32((uint32_t)cfg_.rank);
    w.u64(window_bytes());
    w.u64(cfg_.slot_bytes);
    w.raw(&handle_, sizeof handle_);
    if (!send_msg(c.get(), MSG_HELLO_ACK, w.b)) {
      unmap_window(c->peer_win);
      ::close(fd);
      continue;
    }
    {
      std::lock_guard<std::mutex> lk(in_mu_);
      in_.push_back(c);
    }
    c->reader = std::thread([this, c] { reader_loop(c, true); });
  }
}

void Forwarder::fail_waiters(int peer, const std::string& why) {
  std::vector<std::shared_ptr<Waiter>> hit;
  {
    std::lock_guard<std::mutex> lk(wait_mu_);
    for (auto& kv : waiters_)
      if (kv.second.second == peer) hit.push_back(kv.second.first);
  }
  for (auto& w : hit) {
    std::lock_guard<std::mutex> lk(w->mu);
    if (!w->done) {
      w->done = true;
      w->rc = TFSC_E_INTERNAL;
      w->err = why;
      w->cv.notify_all();
    }
  }
}

void Forwarder::reader_loop(std::shared_ptr<Conn> c, bool incoming) {
  for (;;) {
    uint8_t type = 0;
    std::string payload;
    if (!read_msg(c->fd, &type, &payload)) break;
    if (incoming && type == MSG_FWD) {
      {
        std::lock_guard<std::mutex> lk(job_mu_);
        jobs_.push_back({c, std::move(payload)});
      }
      job_cv_.notify_one();
    } else if (!incoming && type == MSG_DONE) {
      Reader r(payload);
      const uint64_t id = r.u64();
      std::shared_ptr<Waiter> w;
      {
        std::lock_guard<std::mutex> lk(wait_mu_);
        auto it = waiters_.find(id);
        if (it != waiters_.end()) w = it->second.first;
      }
      if (!w) continue;
      std::lock_guard<std::mutex> lk(w->mu);
      w->rc = r.i32();
      w->outcome = r.i32();
      w->rows = r.i64();
      w->sig = read_sig(&r);
      w->err = r.str();
      if (!r.ok) {
        w->rc = TFSC_E_INTERNAL;
        w->err = "forward: malformed DONE message";
      }
      w->done = true;
      w->cv.notify_all();
    }
  }
  c->dead = true;
  if (!incoming) fail_waiters(c->peer, "forward: connection to rank " + std::to_string(c->peer) + " lost");
}

// ------------------------------------------------------------------ owner side ------
void Forwarder::worker_loop() {
  cudaSetDevice(node_->device());
  for (;;) {
    Job job;
    {
      std::unique_lock<std::mutex> lk(job_mu_);
      job_cv_.wait(lk, [&] { return stop_ || !jobs_.empty(); });
      if (jobs_.empty()) {
        if (stop_) return;
        continue;
      }
      job = std::move(jobs_.front());
      jobs_.erase(jobs_.begin());
    }
    handle_fwd(job.conn, job.payload);
  }
}

void Forwarder::send_done(Incoming* in, int rc, const std::string& err) {
  Writer w;
  w.u64(in->req_id);
  w.i32(rc);
  w.i32(in->outcome);
  w.i64(in->req.rows);
  write_sig(&w, in->sig);
  w.str(err);
  send_msg(in->conn.get(), MSG_DONE, w.b);
  if (rc == 0) {
    stats_.peer_bytes_read += (int64_t)in->in_bytes;
    stats_.peer_bytes_written += (int64_t)in->out_bytes;
  }
  std::lock_guard<std::mutex> lk(inc_mu_);
  incoming_.erase(in);  // destroys *in
}

void Forwarder::handle_fwd(const std::shared_ptr<Conn>& c, const std::string& payload) {
  Reader r(payload);
  auto owned = std::make_unique<Incoming>();
  Incoming* in = owned.get();
  in->conn = c;
  in->req_id = r.u64();
  const uint64_t x_off = r.u64(), y_off = r.u64();
  const int64_t n_elems = r.i64();
  const int dtype = r.i32();
  const int64_t deadline = r.i64();
  const std::string name = r.str();
  const int64_t version = r.i64();
  // the packed layout the ingress rank wrote: names and values per row in packed order, its batch size, and what its
  // manifest-free checks found (reported after residency, like every input error)
  InputLayout l;
  l.n_elems = n_elems;
  l.dtype = dtype;
  const uint32_t k = r.u32();
  if (k > 64) r.ok = false;
  for (uint32_t i = 0; r.ok && i < k; ++i) {
    l.names.push_back(r.str());
    l.row_elems.push_back(r.i64());
  }
  l.rows = r.i64();
  l.error = r.str();
  {
    std::lock_guard<std::mutex> lk(inc_mu_);
    incoming_[in] = std::move(owned);
  }
  stats_.in_requests++;
  if (!r.ok) return send_done(in, TFSC_E_INVALID, "forward: malformed FWD message");
  std::string err;
  // the owner node runs the cache tier exactly as for a local request: fetchModel (hit / reload / miss), then the batcher
  int rc = node_->prepare({name, version}, l, &in->req, &in->outcome, &err);
  if (rc < 0) return send_done(in, rc, err);
  const ModelDesc& d = in->req.dm->desc;
  in->sig = FwdSignature::from_desc(d);
  in->in_bytes = (size_t)in->req.rows * Node::row_in_bytes(d);
  in->out_bytes = (size_t)in->req.rows * Node::row_out_bytes(d);
  if (x_off % 16 || y_off % 16 || x_off + in->in_bytes > c->peer_win_bytes || y_off + in->out_bytes > c->peer_win_bytes ||
      in->out_bytes > c->peer_slot_bytes / 2) {
    node_->abandon(&in->req);
    return send_done(in, TFSC_E_EXHAUSTED, "forward: request / response does not fit the forward window slot (cluster.slotBytes)");
  }
  in->req.x = c->peer_win + x_off;  // the ingress rank's HBM: read over NVLink by the gather kernel
  in->req.y = c->peer_win + y_off;  // written over NVLink by the scatter kernel
  in->req.host_staged = false;
  // `deadline` travelled as a remaining budget (the two processes do not share a clock origin by contract)
  in->req.deadline_ns = deadline > 0 ? Node::now_ns() + deadline : 0;
  in->req.on_done = [this, in](PredictRequest* q) { send_done(in, q->rc, q->err); };
  node_->enqueue(&in->req);
}

// ------------------------------------------------------------------ ingress side ------
int Forwarder::acquire_slot(double timeout_s) {
  std::unique_lock<std::mutex> lk(slot_mu_);
  if (!slot_cv_.wait_for(lk, std::chrono::duration<double>(timeout_s), [&] { return !free_slots_.empty(); })) return -1;
  int s = free_slots_.back();
  free_slots_.pop_back();
  return s;
}

void Forwarder::release_slot(int s) {
  {
    std::lock_guard<std::mutex> lk(slot_mu_);
    free_slots_.push_back(s);
  }
  slot_cv_.notify_one();
}

int Forwarder::forward(int peer, const std::string& name, int64_t version, const std::vector<InTensor>& ts, const InputLayout& l,
                       const OutAllocFn& y_alloc, int* outcome, int64_t deadline_ns, std::string* err) {
  const int64_t n_elems = l.n_elems;
  const void* x = ts.empty() ? nullptr : ts[0].data;
  const auto t0 = std::chrono::steady_clock::now();
  stats_.out_requests++;
  auto failed = [&](int rc, const std::string& msg) {
    stats_.out_failures++;
    *err = msg;
    return rc;
  };
  std::shared_ptr<Conn> c = get_conn(peer, err);
  if (!c) {
    stats_.out_failures++;
    return TFSC_E_INTERNAL;
  }
  const size_t half = cfg_.slot_bytes / 2;
  const size_t in_bytes = (size_t)(n_elems > 0 ? n_elems : 0) * 4;
  if (!x || n_elems <= 0 || in_bytes > half)
    return failed(n_elems > 0 && x ? TFSC_E_EXHAUSTED : TFSC_E_INVALID,
                  "forward: request of " + std::to_string(in_bytes) + " bytes does not fit a forward window slot (cluster.slotBytes / 2 = " +
                      std::to_string(half) + ")");
  double budget = cfg_.timeout_s;
  if (deadline_ns > 0) {
    const double left = (double)(deadline_ns - Node::now_ns()) * 1e-9;
    if (left <= 0) return failed(TFSC_E_TIMEOUT, "deadline exceeded before the request was forwarded");
    if (left < budget) budget = left;
  }
  const int slot = acquire_slot(budget);
  if (slot < 0) return failed(TFSC_E_EXHAUSTED, "forward: no free window slot (cluster.windowSlots)");
  char* st = static_cast<char*>(node_->staging_alloc(half));
  if (!st) {
    release_slot(slot);
    return failed(TFSC_E_EXHAUSTED, "forward: cannot pin request staging");
  }
  DeviceGuard g(node_->device());
  cudaStream_t stream = streams_[rr_++ % 8];
  char* sx = window_ + (size_t)slot * cfg_.slot_bytes;
  char* sy = sx + half;
  // a layout that failed its manifest-free checks is not packed: the owner rejects it once the model is resident
  const size_t packed = l.error.empty() ? in_bytes : 0;
  if (packed) pack_rows(ts, l, l.rows, st);  // one tensor: the same bytes as a memcpy of it
  cudaError_t e = packed ? cudaMemcpyAsync(sx, st, packed, cudaMemcpyHostToDevice, stream) : cudaSuccess;
  if (e == cudaSuccess) e = cudaStreamSynchronize(stream);  // x sits in this rank's HBM before the owner is told about it
  if (e != cudaSuccess) {
    cudaGetLastError();
    node_->staging_free(st, half);
    release_slot(slot);
    return failed(TFSC_E_INTERNAL, std::string("forward: staging copy failed: ") + cudaGetErrorString(e));
  }
  const uint64_t id = next_id_++;
  auto w = std::make_shared<Waiter>();
  {
    std::lock_guard<std::mutex> lk(wait_mu_);
    waiters_[id] = {w, peer};
  }
  Writer m;
  m.u64(id);
  m.u64((uint64_t)(sx - window_));
  m.u64((uint64_t)(sy - window_));
  m.i64(n_elems);
  m.i32(l.dtype);
  m.i64(deadline_ns > 0 ? (int64_t)(budget * 1e9) : 0);
  m.str(name);
  m.i64(version);
  m.u32((uint32_t)l.names.size());
  for (size_t i = 0; i < l.names.size(); ++i) {
    m.str(l.names[i]);
    m.i64(l.row_elems[i]);
  }
  m.i64(l.rows);
  m.str(l.error);
  bool sent = send_msg(c.get(), MSG_FWD, m.b);
  bool got = false;
  if (sent) {
    std::unique_lock<std::mutex> lk(w->mu);
    got = w->cv.wait_for(lk, std::chrono::duration<double>(budget), [&] { return w->done; });
  }
  {
    std::lock_guard<std::mutex> lk(wait_mu_);
    waiters_.erase(id);
  }
  int rc;
  if (!sent) {
    rc = failed(TFSC_E_INTERNAL, "forward: connection to rank " + std::to_string(peer) + " lost");
    release_slot(slot);
  } else if (!got) {
    // the owner may still write into the slot: it is NOT returned to the free list (a leaked slot beats a corrupted one)
    rc = failed(TFSC_E_TIMEOUT, "forward: rank " + std::to_string(peer) + " did not answer within " + std::to_string(budget) + " s");
  } else {
    rc = w->rc;
    if (outcome) *outcome = w->outcome;
    if (rc < 0) {
      stats_.out_failures++;
      *err = w->err;
    } else {
      ModelDesc d;
      w->sig.to_desc(&d);
      const size_t out_bytes = (size_t)w->rows * Node::row_out_bytes(d);
      void* y = y_alloc(d, w->rows);
      if (!y) {
        rc = failed(TFSC_E_BUFFER, "output buffer too small");
      } else if (out_bytes > half) {
        rc = failed(TFSC_E_INTERNAL, "forward: response larger than the window slot");
      } else {
        e = cudaMemcpyAsync(st, sy, out_bytes, cudaMemcpyDeviceToHost, stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
        if (e != cudaSuccess) {
          cudaGetLastError();
          rc = failed(TFSC_E_INTERNAL, std::string("forward: result copy failed: ") + cudaGetErrorString(e));
        } else {
          memcpy(y, st, out_bytes);
        }
      }
    }
    release_slot(slot);
  }
  node_->staging_free(st, half);
  stats_.rtt_ns_sum += std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
  return rc;
}

}  // namespace tfsc
