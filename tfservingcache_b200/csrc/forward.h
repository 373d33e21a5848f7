// a6 / X7, the forward hop between PROCESSES (one rank per GPU, the torchrun layout): the reference forwards every
// request whose ring owner is another node over TCP, re-serialising the whole tensor at both tiers
// (pkg/taskhandler/taskhandler.go:95-147 restDirector / grpcDirector, conn pool grpcConnMap :28-31, dialled lazily).
// Here the tensor never leaves device memory:
//   * every rank owns a FORWARD WINDOW, a slab of its HBM split into slots [x | y], exported with cudaIpcGetMemHandle;
//   * the ingress rank puts the request rows into a slot of its own window (one H2D) and sends a ~100-byte FWD control
//     message to the owner over a unix socket (the pooled connection, dialled lazily like grpcConnMap);
//   * the owner maps the ingress window once (cudaIpcOpenMemHandle) and hands the batcher a request whose x / y ARE that
//     peer memory: the gather kernel pulls the rows over NVLink into the batch buffer next to local requests, the scatter
//     kernel pushes the result rows back over NVLink into the slot (csrc/nn_kernels.cu copy_segments_kernel); with
//     tfsc_predict_device the first / last layer kernels themselves read / write the peer window;
//   * a DONE message (status + the output signature) returns; the ingress rank reads y from its own HBM.
// No NCCL, no host bounce of the payload. Control messages are host traffic by design (the reference's are, too).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <condition_variable>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "node.h"

namespace tfsc {

struct FwdConfig {
  int rank = 0;
  std::vector<std::string> endpoints;   // endpoints[r] = unix socket path of rank r ("unix:" prefix optional)
  size_t slot_bytes = (size_t)1 << 20;  // per slot: x in the first half, y in the second
  int slots = 128;
  double timeout_s = 10.0;              // proxy.grpcTimeout analogue
  int workers = 8;                      // owner-side threads running fetchModel for incoming requests
};

struct FwdStats {
  std::atomic<int64_t> out_requests{0}, in_requests{0}, out_failures{0};
  std::atomic<int64_t> peer_bytes_read{0}, peer_bytes_written{0};  // owner side: bytes moved over NVLink by gather / scatter
  std::atomic<int64_t> rtt_ns_sum{0};
};

// what the ingress rank needs to know about the model to shape the response (it never loads the model itself)
struct FwdSignature {
  int tmpl = 1;
  int64_t in_dim = 0, out_dim = 0;
  int input_dtype = TFSC_DT_FLOAT;
  std::string input_name, output_name;
  std::vector<int64_t> input_shape, output_shape;
  std::vector<std::string> input_names;  // signature.inputs in packed order (empty: single-input model)
  std::vector<int32_t> input_roles;
  std::vector<std::string> output_names;  // signature.outputs in packed order (empty: single-output model)
  std::vector<int32_t> output_kinds;
  int32_t head_n = 0, head_k = 0;
  void to_desc(ModelDesc* d) const;
  static FwdSignature from_desc(const ModelDesc& d);
};

class Forwarder {
 public:
  Forwarder(const FwdConfig& cfg, Node* node);
  ~Forwarder();
  bool init(std::string* err);

  // ingress side: run `name:version` on rank `peer` with the host tensors ts (sorted and described by layout_inputs): they
  // are packed into this rank's window slot and the FWD message carries the layout, which the owner checks against its
  // manifest. y_alloc(sig, rows) supplies the host output buffer.
  using OutAllocFn = std::function<void*(const ModelDesc&, int64_t rows)>;
  int forward(int peer, const std::string& name, int64_t version, const std::vector<InTensor>& ts, const InputLayout& l,
              const OutAllocFn& y_alloc, int* outcome, int64_t deadline_ns, std::string* err);

  // device-resident use (bench `value`, tfsc_predict_device with peer pointers)
  char* window() const { return window_; }
  size_t window_bytes() const { return (size_t)cfg_.slots * cfg_.slot_bytes; }
  size_t slot_bytes() const { return cfg_.slot_bytes; }
  // device pointer of rank `peer`'s window in THIS process (connects and maps on first use)
  char* peer_window(int peer, size_t* bytes, std::string* err);
  const FwdStats& stats() const { return stats_; }
  int rank() const { return cfg_.rank; }
  int world() const { return (int)cfg_.endpoints.size(); }

 private:
  struct Conn {  // one socket: outgoing (we send FWD, read DONE) or incoming (we read FWD, send DONE)
    int fd = -1;
    int peer = -1;
    std::mutex wmu;  // writers
    std::thread reader;
    char* peer_win = nullptr;  // peer's window mapped here (incoming: the ingress window; outgoing: the owner's)
    size_t peer_win_bytes = 0, peer_slot_bytes = 0;
    std::atomic<bool> dead{false};
  };
  struct Waiter {  // an ingress-side caller parked until DONE arrives
    std::mutex mu;
    std::condition_variable cv;
    bool done = false;
    int rc = 0, outcome = 0;
    int64_t rows = 0;
    FwdSignature sig;
    std::string err;
  };
  struct Incoming {  // owner side: a forwarded request between FWD and DONE
    PredictRequest req;
    std::shared_ptr<Conn> conn;
    uint64_t req_id = 0;
    int outcome = 0;
    FwdSignature sig;
    size_t in_bytes = 0, out_bytes = 0;
  };
  struct Job {
    std::shared_ptr<Conn> conn;
    std::string payload;
  };

  std::shared_ptr<Conn> get_conn(int peer, std::string* err);  // grpcConnMap: lazily dialled, pooled
  void accept_loop();
  void reader_loop(std::shared_ptr<Conn> c, bool incoming);
  void worker_loop();
  void handle_fwd(const std::shared_ptr<Conn>& c, const std::string& payload);
  void send_done(Incoming* in, int rc, const std::string& err);
  bool send_msg(Conn* c, uint8_t type, const std::string& payload);
  int acquire_slot(double timeout_s);
  void release_slot(int s);
  void fail_waiters(int peer, const std::string& why);

  FwdConfig cfg_;
  Node* node_;
  char* window_ = nullptr;
  cudaIpcMemHandle_t handle_{};
  int listen_fd_ = -1;
  std::string listen_path_;
  std::thread acceptor_;
  std::atomic<bool> stop_{false};

  std::mutex conn_mu_;                            // guards out_; HELD ACROSS A DIAL (one dial per peer, like grpcConnMap's write lock)
  std::map<int, std::shared_ptr<Conn>> out_;      // by peer rank
  std::mutex in_mu_;                              // guards in_ only: the acceptor must never wait for a dial in progress --
  std::vector<std::shared_ptr<Conn>> in_;         // with >= 3 ranks dialling each other that closes a cycle (found at N = 8)

  std::mutex slot_mu_;
  std::condition_variable slot_cv_;
  std::vector<int> free_slots_;

  std::mutex wait_mu_;
  std::unordered_map<uint64_t, std::pair<std::shared_ptr<Waiter>, int>> waiters_;  // req_id -> (waiter, peer)
  std::atomic<uint64_t> next_id_{1};

  std::mutex job_mu_;
  std::condition_variable job_cv_;
  std::vector<Job> jobs_;
  std::vector<std::thread> workers_;

  std::mutex inc_mu_;
  std::unordered_map<Incoming*, std::unique_ptr<Incoming>> incoming_;

  cudaStream_t streams_[8] = {};
  std::atomic<unsigned> rr_{0};
  FwdStats stats_;
};

}  // namespace tfsc
