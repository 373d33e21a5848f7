/* tfsc_b200.h -- C ABI of libtfsc_b200.so, the H100-native replacement for the
 * route -> ensure-resident -> predict path of mKaloer/TFServingCache.
 *
 * This is the drop-in boundary (SURVEY.md section 8b): plain C, plain pointers and sizes, no
 * C++/torch types, callable from cgo, ctypes or JNI, from any thread, re-entrant.  Every entry
 * point cites the reference interface (file:line under the reference repo) it replaces.
 *
 * Conventions
 *   - return value: >= 0 success (meaning documented per call), < 0 one of TFSC_E_*.
 *   - tfsc_last_error() returns a thread-local message for the last failing call.
 *   - strings are NUL-terminated UTF-8; out buffers are caller-owned with an explicit capacity;
 *     a too-small buffer yields TFSC_E_BUFFER.
 *   - buffers returned through `void**` are library-owned and released with tfsc_free().
 *   - there is NO CPU fallback: every compute entry fails with TFSC_E_NO_DEVICE when no
 *     sm_90 (H100) device is usable.
 */
#ifndef TFSC_B200_H_
#define TFSC_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TFSC_ABI_VERSION 2

/* error codes; the gRPC status each one maps to is given in parentheses */
#define TFSC_OK 0
#define TFSC_E_INVALID (-3)       /* INVALID_ARGUMENT (3)  */
#define TFSC_E_TIMEOUT (-4)       /* DEADLINE_EXCEEDED (4): "Timeout: Model did not load in time" */
#define TFSC_E_NOT_FOUND (-5)     /* NOT_FOUND (5)         */
#define TFSC_E_EXHAUSTED (-8)     /* RESOURCE_EXHAUSTED (8)*/
#define TFSC_E_UNIMPLEMENTED (-12)/* UNIMPLEMENTED (12): MultiInference, tfservingproxy.go:215-217 */
#define TFSC_E_INTERNAL (-13)     /* INTERNAL (13)         */
#define TFSC_E_NO_DEVICE (-14)    /* UNAVAILABLE (14): CUDA device / extension missing */
#define TFSC_E_EMPTY_RING (-20)   /* consistent.ErrEmptyCircle, cluster.go:118-120 */
#define TFSC_E_BUFFER (-21)       /* caller buffer too small */

/* ModelVersionStatus_State, pkg/cachemanager/servingcontroller.go:29-54 */
#define TFSC_STATE_UNKNOWN 0
#define TFSC_STATE_START 10
#define TFSC_STATE_LOADING 20
#define TFSC_STATE_AVAILABLE 30
#define TFSC_STATE_UNLOADING 40
#define TFSC_STATE_END 50

/* fetchModel outcome, pkg/cachemanager/cachemanager.go:103-150 */
#define TFSC_FETCH_HIT 0     /* cached and resident: cache_hits_total++            */
#define TFSC_FETCH_RELOAD 1  /* in the host tier but not HBM-resident (:133-143)    */
#define TFSC_FETCH_MISS 2    /* not cached: provider load, cache_misses_total++     */

/* tensorflow.DataType subset, proto/tensorflow/core/framework/types.pb.go:30-55 */
#define TFSC_DT_FLOAT 1
#define TFSC_DT_INT32 3
#define TFSC_DT_INT64 9

int tfsc_abi_version(void);
const char* tfsc_last_error(void);
const char* tfsc_strerror(int code);
void tfsc_free(void* p);

/* ---------------------------------------------------------------- a3-a5: routing ring ------
 * Bit-exact restatement of stathat.com/c/consistent v1.0.0 as driven by
 * pkg/taskhandler/cluster.go:55 (New), :111 (Set), :117 (GetN). */
typedef struct tfsc_ring tfsc_ring;

uint32_t tfsc_crc32_ieee(const void* data, size_t len); /* Go crc32.ChecksumIEEE */
tfsc_ring* tfsc_ring_new(void);                         /* consistent.New(), cluster.go:55 */
void tfsc_ring_free(tfsc_ring* r);
/* consistent.Set(members): cluster.go:104-113 (clusterUpdated). member = "host:rest:grpc". */
int tfsc_ring_set(tfsc_ring* r, const char* const* members, int n_members);
int tfsc_ring_members(const tfsc_ring* r);              /* member count */
int tfsc_ring_points(const tfsc_ring* r);               /* ring points (<= 20 * members) */
/* consistent.GetN(key, n): cluster.go:116-130 (FindNodeForKey). Writes up to n member strings,
 * '\n'-separated, clockwise order, into buf. Returns the number of members written. */
int tfsc_ring_getn(const tfsc_ring* r, const char* key, int n, char* buf, size_t cap);
/* Replica choice among the GetN candidates: "random" = the reference (taskhandler.go:91), "first" = primary,
 * "hot-spread" = primary unless the key's recent request share exceeds hot_fraction / members (then random),
 * "balanced" = hot-spread + least-loaded-replica binding (tfsc_picker_pick_ids), "hash" = crc32(key) mod replicas
 * (stateless: independent processes agree on the replica of a key).
 * Deterministic for a given seed and call sequence. tfsc_picker_pick returns an index in [0, n_replicas). */
typedef struct tfsc_picker tfsc_picker;
tfsc_picker* tfsc_picker_new(const char* policy, uint64_t seed, double hot_fraction);
void tfsc_picker_free(tfsc_picker* p);
int tfsc_picker_pick(tfsc_picker* p, const char* key, int n_replicas, int members);
/* same with a stable integer id per candidate; policy "balanced" = hot-spread + sticky power-of-two-choices
 * (a cold key binds to the candidate that holds the fewest keys) */
int tfsc_picker_pick_ids(tfsc_picker* p, const char* key, const int* member_ids, int n_replicas, int members);
/* key = modelName + "##" + version (taskhandler.go:85). Returns strlen. */
int tfsc_model_key(const char* model_name, const char* version, char* buf, size_t cap);

/* ---------------------------------------------------------------- a9: LRU model cache ------
 * pkg/cachemanager/lrucache.go:20-105 (ModelCache interface :11-18). Not internally
 * synchronised, exactly like the reference (the cache manager holds the lock). */
typedef struct tfsc_lru tfsc_lru;

tfsc_lru* tfsc_lru_new(const char* base_dir, int64_t capacity_bytes); /* NewLRUCache :28 */
void tfsc_lru_free(tfsc_lru* c);
/* Put :54-65. Returns the number of entries evicted to make room. */
int tfsc_lru_put(tfsc_lru* c, const char* model_name, int64_t version, const char* path, int64_t size_on_disk);
/* Get :43-51 (touches recency). Returns 1 if present (fills size/path), 0 if not. */
int tfsc_lru_get(tfsc_lru* c, const char* model_name, int64_t version, int64_t* size_on_disk, char* path, size_t cap);
int tfsc_lru_ensure_free_bytes(tfsc_lru* c, int64_t bytes);           /* :68-87; returns #evicted */
int64_t tfsc_lru_current_size(const tfsc_lru* c);
int64_t tfsc_lru_capacity(const tfsc_lru* c);
int tfsc_lru_len(const tfsc_lru* c);
/* ListModels :89-97, MRU -> LRU, one "name\tversion\tsize\tpath\n" line per model. Returns count. */
int tfsc_lru_list(const tfsc_lru* c, char* buf, size_t cap);

/* ---------------------------------------------------------------- a1/a2/a7: request parsing -
 * tfServingRestURLMatch (tfservingproxy.go:24) + RestProxy.Serve status logic (:93-129).
 * Returns 200 (name+version filled, version verbatim incl. leading zeros), 404 or 400. */
int tfsc_rest_match_url(const char* url, char* model_name, size_t name_cap, char* version, size_t version_cap);
/* exact JSON error body json.NewEncoder would emit for 404 / 400 (tfservingproxy.go:99-124) */
const char* tfsc_rest_error_body(int http_status);
/* strconv.ParseInt(version, 10, 64), cachemanager.go:297. 0 or TFSC_E_INVALID. */
int tfsc_parse_version(const char* version, int64_t* out);
/* clientForSpec (tfservingproxy.go:246-250): scan a serialized ModelSpec-bearing request
 * (PredictRequest/ClassificationRequest/...: model_spec is field 1) and return name + version
 * string ("0" when absent). */
int tfsc_grpc_model_spec(const void* req, size_t len, char* model_name, size_t name_cap, char* version, size_t version_cap);

/* ---------------------------------------------------------------- a11: disk model provider --
 * diskmodelprovider.go:46-69 findSrcPathForModel (numeric version match), :71-83 ModelSize
 * (fixed: recursive byte size). */
int tfsc_disk_find_version_dir(const char* base_dir, const char* model_name, int64_t version, char* buf, size_t cap);
int64_t tfsc_disk_model_size(const char* base_dir, const char* model_name, int64_t version);
/* SURVEY 8f-1: TensorFlow SavedModel ingestion without TensorFlow. The disk provider imports a version directory that
 * holds `saved_model.pb` + `variables/variables.{index,data-*}` (and no tfsc_model.json) on the fly when the model is
 * fetched; this entry does the same conversion offline and writes tfsc_model.json + weights.bin into out_dir (may equal
 * version_dir). Recognised graphs: y = a*x + b (half_plus_two) and MatMul + BiasAdd (+ Relu) chains; anything else is
 * TFSC_E_INVALID with the offending node in tfsc_last_error(). Needs no GPU. */
int tfsc_savedmodel_convert(const char* version_dir, const char* out_dir);
uint32_t tfsc_crc32c(const void* data, size_t len);   /* CRC-32C (Castagnoli), the tensor-bundle / table checksum */
/* Checks a tfsc_model.json text with the rules the loader applies; needs no GPU. TFSC_E_INVALID with the loader's reason in
 * tfsc_last_error(), or writes {"in_dim", "out_dim", "head_n", "head_k", "outputs": [{"name", "kind", "offset", "width",
 * "dtype"}]} (the packed response row of signature.outputs, offsets and widths in 32-bit words) and returns its strlen. */
int tfsc_manifest_check(const char* manifest_json, char* buf, size_t cap);
/* The packed input layout of a tfsc_model.json as its owner has it and as an ingress rank of the forward hop rebuilds it from
 * the signature the owner sends: {"owner": L, "ingress": L}, L = {"in_dim", "out_dim", "inputs": [{"name", "role",
 * "offset", "width"}]} (role: 0 ids, 1 mask, 2 type_ids, 3 seed). Needs no GPU; TFSC_E_INVALID for a manifest the loader
 * refuses. */
int tfsc_signature_roundtrip(const char* manifest_json, char* buf, size_t cap);

/* ---------------------------------------------------------------- server (a6,a8,a10,X) ------
 * One server = the cache tier + proxy tier of cmd/taskhandler/main.go:45-113 for the GPUs of
 * this process: one "node" per GPU (ring member), each with its own LRU host tier, HBM arena,
 * residency table, copy stream and batcher. Configuration is a flat JSON object whose keys are
 * the reference's viper keys (SURVEY.md section 5), e.g.
 *   {"modelProvider.type":"diskProvider","modelProvider.diskProvider.baseDir":"/model_repo",
 *    "modelCache.size":68719476736,"serving.maxConcurrentModels":32,"proxy.replicasPerModel":2,
 *    "gpu.devices":[0,1],"gpu.arenaBytes":171798691840,"gpu.maxBatch":8,"gpu.members":["gpu0:0:0","gpu1:0:0"]}
 */
typedef struct tfsc_server tfsc_server;

typedef struct tfsc_tensor {
  const char* name;   /* signature key ("x", "y", "input_ids", ...); may be NULL for the only input/output, required when
                         a request passes several inputs */
  int32_t dtype;      /* TFSC_DT_* */
  int32_t rank;
  int64_t shape[8];
  void* data;         /* host pointer (tfsc_predict) or device pointer (tfsc_predict_device) */
  size_t nbytes;
} tfsc_tensor;

typedef struct tfsc_stats {
  /* names kept from cachemanager.go:24-43 / tfservingproxy.go:25-32 */
  int64_t cache_total, cache_hits_total, cache_misses_total;
  int64_t proxy_requests_rest, proxy_requests_grpc, proxy_failures_rest, proxy_failures_grpc;
  int64_t evictions_host, evictions_hbm;
  int64_t h2d_weight_bytes, h2d_input_bytes, d2h_output_bytes;
  int64_t kernel_launches, batches, batched_rows;
  int64_t arena_bytes_used, arena_bytes_capacity, resident_models, host_models;
  double cache_duration_seconds_sum, cache_fetch_duration_seconds_sum;
  /* forward hop (a6): requests sent to / received from other ranks, bytes the owner moved over NVLink */
  int64_t fwd_out_requests, fwd_in_requests, fwd_out_failures, fwd_peer_bytes_read, fwd_peer_bytes_written;
  double fwd_rtt_seconds_sum;
  /* HBM arena defragmentation: passes that moved resident blocks (device-to-device) and the bytes they moved */
  int64_t arena_compactions, arena_compacted_bytes;
} tfsc_stats;

tfsc_server* tfsc_server_create(const char* config_json); /* main.go:45-113 */
void tfsc_server_destroy(tfsc_server* s);
int tfsc_server_num_nodes(const tfsc_server* s);
/* DiscoveryService member update (cluster.go:25-30,104-113). Default members: "gpu<i>:0:0". */
int tfsc_server_set_members(tfsc_server* s, const char* const* members, int n);
/* nodeForKey (taskhandler.go:84-92): ring lookup + replica pick. Writes the ordered replica
 * set as local node indices (or -1 for non-local members) into nodes[0..cap) and returns the
 * picked index into that list via *picked. Return value = replica count. */
int tfsc_route(tfsc_server* s, const char* model_name, const char* version, int* nodes, int cap, int* picked);
/* fetchModel (cachemanager.go:91-152) on one node: ensure the model is HBM-resident.
 * Returns TFSC_FETCH_* or an error. Blocks only this caller (per-model load lock). */
int tfsc_model_ensure(tfsc_server* s, int node, const char* model_name, int64_t version);
/* Same decision and bookkeeping as tfsc_model_ensure, but returns as soon as the page-in is queued on the copy
 * stream (state LOADING); launches on the model wait for it on-device (event), the host never blocks. */
int tfsc_model_ensure_async(tfsc_server* s, int node, const char* model_name, int64_t version);
/* GetModelStatus (servingcontroller.go:114-138): TFSC_STATE_* or TFSC_E_NOT_FOUND. */
int tfsc_model_status(tfsc_server* s, int node, const char* model_name, int64_t version);
/* Resident set, MRU first: "name\tversion\tbytes\tstate\n" lines. Returns count. */
int tfsc_resident_list(tfsc_server* s, int node, char* buf, size_t cap);
/* LRU host tier listing (LocalCache.ListModels), same line format as tfsc_lru_list. */
int tfsc_host_list(tfsc_server* s, int node, char* buf, size_t cap);

/* proxyServiceServer.Predict (tfservingproxy.go:201-212) with the forward replaced by on-GPU
 * execution: route -> ensure-resident -> batch -> kernels. Host tensors in, host tensors out;
 * out[i].data/nbytes must be a caller buffer large enough for the result (shape is filled).
 * `version` is the verbatim string ("00000123" routes differently from "123": reference quirk).
 * Inputs: n_in >= 1 named tensors. A single-input model takes one tensor (its name may be NULL). A model whose manifest
 * declares signature.inputs (e.g. BERT: input_ids / input_mask / segment_ids) takes exactly those, each DT_INT32
 * [batch, seq] (or [seq]) with the same batch; a missing, extra or misnamed input, unequal batch sizes, a wrong per-row
 * size or a float tensor answer TFSC_E_INVALID naming the expected inputs (after the model is made resident, as every
 * input error; nothing is launched). The same holds for _deadline, _member and _submit.
 * Outputs: a single-output model fills out[0] (DT_FLOAT; out[0].name is not looked at) and ignores out[1..n_out). A model
 * whose manifest declares signature.outputs (logits, probabilities, classes, top_k_classes, top_k_probabilities, or the
 * question-answering start_logits, end_logits, span_starts, span_ends, span_scores, or the encoder sequence_output,
 * pooled_output, cls_embedding, mean_embedding, or the fill-mask masked_positions, masked_top_k_ids,
 * masked_top_k_probabilities, masked_top_k_logits) fills out[i] with the output named out[i].name, in the caller's order:
 * dtype (DT_INT64 for classes, DT_INT32 for top_k_classes, span_starts, span_ends, masked_positions and masked_top_k_ids,
 * DT_FLOAT otherwise), shape (batch dims, then [N], [S], [H] or [M], nothing, [k], [S, H] for sequence_output or [M, k]
 * for the fill-mask top-k outputs) and nbytes. A NULL, unknown or repeated
 * name is TFSC_E_INVALID and the message lists the outputs; a buffer too small for its output is TFSC_E_BUFFER. */
int tfsc_predict(tfsc_server* s, const char* model_name, const char* version,
                 const tfsc_tensor* in, int n_in, tfsc_tensor* out, int n_out);
/* tfsc_predict with a deadline (absolute, on the clock of tfsc_now_ns() = CLOCK_MONOTONIC; 0 = none): a request still
 * queued when its deadline passes is answered TFSC_E_TIMEOUT without being launched (grpc deadline / proxy.grpcTimeout). */
int tfsc_predict_deadline(tfsc_server* s, const char* model_name, const char* version,
                          const tfsc_tensor* in, int n_in, tfsc_tensor* out, int n_out, int64_t deadline_ns);
int64_t tfsc_now_ns(void);
/* The cache tier of one member, without the ring lookup (the reference's second tier: cachemanager.ServeRest / ServeGrpc on
 * cacheRestPort / cacheGrpcPort, cmd/taskhandler/main.go:60-84 -- a request that reaches a cache node is served there):
 * `member` indexes the current member list ("gpu.members" / tfsc_server_set_members order). A local member runs on its node;
 * a member of another rank takes the forward hop. For callers that route themselves (tfsc_route, or a front load balancer). */
int tfsc_predict_member(tfsc_server* s, int member, const char* model_name, const char* version,
                        const tfsc_tensor* in, int n_in, tfsc_tensor* out, int n_out, int64_t deadline_ns);
/* Asynchronous Predict: no OS thread is parked per in-flight request (a Go handler keeps a goroutine, not an M).
 *   submit: route -> ensure-resident (may block on a cold load of THIS model only) -> signature checks -> the input rows are
 *           copied to pinned staging, so `in` may be reused at once. out[0].data / nbytes is the caller's result buffer.
 *   wait  : timeout_ns < 0 blocks; >= 0 waits at most that long and answers TFSC_E_TIMEOUT while the request is still in
 *           flight (the ticket stays valid). On success out[0] holds dtype / shape / nbytes and the data.
 *   release: frees the ticket (waits for the request to retire first if it is still in flight). */
typedef struct tfsc_ticket tfsc_ticket;
int tfsc_predict_submit(tfsc_server* s, const char* model_name, const char* version, const tfsc_tensor* in, int n_in,
                        tfsc_tensor* out, int n_out, int64_t deadline_ns, tfsc_ticket** ticket);
int tfsc_predict_wait(tfsc_ticket* ticket, int64_t timeout_ns);
void tfsc_predict_release(tfsc_ticket* ticket);
/* Same, wire level: serialized tensorflow.serving.PredictRequest in, PredictResponse out
 * (library-owned; tfsc_free). This is what a cgo Predict handler calls. */
int tfsc_grpc_predict(tfsc_server* s, const void* req, size_t req_len, void** resp, size_t* resp_len);
/* proxyServiceServer.Classify / Regress (tfservingproxy.go:173-198) and SessionRun (:233-244), wire level like
 * tfsc_grpc_predict: serialized ClassificationRequest / RegressionRequest / SessionRunRequest in, the matching response out
 * (library-owned; tfsc_free). tf.Example inputs are mapped onto the model's input rows through the classify / regress
 * signatures the bundle declares ("extra_signatures" of the manifest; a SavedModel import carries over the signatures of
 * saved_model.pb, e.g. half_plus_two's regress_x_to_y / classify_x_to_y on feature "x"). A model without such a signature
 * answers INVALID_ARGUMENT with TF-Serving's message. MultiInference stays an error (tfservingproxy.go:215-217). */
int tfsc_grpc_classify(tfsc_server* s, const void* req, size_t req_len, void** resp, size_t* resp_len);
int tfsc_grpc_regress(tfsc_server* s, const void* req, size_t req_len, void** resp, size_t* resp_len);
int tfsc_grpc_session_run(tfsc_server* s, const void* req, size_t req_len, void** resp, size_t* resp_len);
/* RestProxy.Serve (tfservingproxy.go:93-129) with on-GPU execution: GET status / POST :predict.
 * Returns 0 and fills *http_status + body (library-owned; tfsc_free). */
int tfsc_rest_handle(tfsc_server* s, const char* method, const char* url, const void* body, size_t body_len,
                     int* http_status, void** resp, size_t* resp_len);

/* Device-resident predict on an explicit node/stream: x and y are DEVICE pointers (possibly
 * peer memory of another GPU: the forward hop a6 becomes NVLink loads/stores inside the first /
 * last kernel). rows = batch rows. stream = cudaStream_t or NULL for the node's compute stream.
 * The model must have been made resident (tfsc_model_ensure); it is pinned for the launch.
 * x holds `rows` packed rows of the model's in_dim values. A multi-input model's row is the concatenation of its inputs'
 * rows (seq int32 values each) in byte-wise sorted NAME order, e.g. input_ids | input_mask | segment_ids: the ids of row r
 * are x[r*3*seq .. r*3*seq + seq). The kernels read the ids, the attention mask and the segment ids from there.
 * y receives `rows` packed rows the same way. A multi-output model's row is the concatenation of its outputs' rows in
 * byte-wise sorted NAME order, in 32-bit words: logits / probabilities N floats, classes 2 words (the int64 index,
 * little-endian), top_k_classes k int32, top_k_probabilities k floats, start_logits / end_logits S floats, span_starts /
 * span_ends k int32, span_scores k floats, sequence_output S*H floats (token-major), pooled_output / cls_embedding /
 * mean_embedding H floats, masked_positions M int32, masked_top_k_ids M*k int32, masked_top_k_probabilities /
 * masked_top_k_logits M*k floats (slot-major); e.g. classes | logits | probabilities is 2 + 2N words per row, logits of row r at
 * y + r*(2+2N) + 2. A single-output model's row is its out_dim floats. */
int tfsc_predict_device(tfsc_server* s, int node, const char* model_name, int64_t version,
                        const void* x, int64_t rows, void* y, void* stream);
int tfsc_node_sync(tfsc_server* s, int node);
/* serving.maxConcurrentModels of one node at run time (takes effect at the next reload: cachemanager.go:167-170) */
int tfsc_node_set_max_resident(tfsc_server* s, int node, int max_concurrent_models);

/* ---------------------------------------------------------------- a6 / X7: forward hop between processes ------
 * One process per GPU (torchrun): config keys "cluster.rank", "cluster.endpoints" (one unix-socket path per entry of
 * "gpu.members", same order), "cluster.slotBytes", "cluster.windowSlots". A Predict whose ring owner is another rank is
 * forwarded there like restDirector / grpcDirector do (taskhandler.go:95-147), except that only a ~100-byte control message
 * crosses the socket: the request rows sit in this rank's FORWARD WINDOW (HBM exported with CUDA IPC), the owner's gather /
 * scatter kernels (or its first / last layer, with tfsc_predict_device) read x and write y there over NVLink.
 * tfsc_fwd_window: this rank's window (device pointer, bytes, slot size); returns the rank.
 * tfsc_fwd_peer_window: rank `peer_rank`'s window mapped into this process (dials the peer on first use). */
int tfsc_fwd_window(tfsc_server* s, void** dev_ptr, size_t* bytes, size_t* slot_bytes);
int tfsc_fwd_peer_window(tfsc_server* s, int peer_rank, void** dev_ptr, size_t* bytes);
/* synchronous copy between any two addresses of the unified address space (host, this GPU, a mapped peer window): how a
 * host program without its own CUDA binding fills / reads window slots for tfsc_predict_device */
int tfsc_device_memcpy(void* dst, const void* src, size_t nbytes);
int tfsc_get_stats(tfsc_server* s, int node, tfsc_stats* out); /* node = -1: sum over nodes */
/* number of kernels launched by this library since load (bench gpu_launches) */
int64_t tfsc_kernel_launches(void);

/* ---------------------------------------------------------------- raw kernels (X rows) ------
 * Direct launches on caller-provided device memory for parity tests and roofline timing.
 * y[rows,n] = act(x[rows,k] W[k,n] + b[n]); fp32; W row-major [k,n] (TF dense kernel layout). */
int tfsc_k_affine(const float* x, float* y, int64_t n, const float* a, const float* b, void* stream);      /* X1 */
int tfsc_k_dense(const float* x, const float* w, const float* b, float* y, int rows, int k, int n, int relu,
                 float* workspace, size_t workspace_bytes, void* stream);                                    /* X2 */
size_t tfsc_k_dense_workspace(int rows, int k, int n);
/* tfsc_k_dense with an explicit kernel choice: 0 auto (<= 8 rows: cluster-pair kernel with programmatic dependent launch,
 * csrc/dense_cluster.cu -- two CTAs split K and meet in distributed shared memory; more rows: tensor cores), 1 LDG-stream
 * SIMT kernel with split-K workspace (the round-1 default; still the fallback for shapes the cluster kernel does not take),
 * 2 / 4 bulk-copy (TMA) ring with 8 / 4 k-lanes, 3 tensor cores for every row count, 5 cluster-pair kernel for <= 8 rows and
 * the SIMT fallback otherwise. Same arguments, workspace and results (the fp32 summation order differs between variants; each
 * variant is bit-reproducible). */
int tfsc_k_dense_variant(int variant, const float* x, const float* w, const float* b, float* y, int rows, int k, int n,
                         int relu, float* workspace, size_t workspace_bytes, void* stream);
/* Grid of the <= 8-row cluster-pair kernel on the current device: the number of co-resident 2-CTA clusters (the grid never
 * exceeds it, so a pass runs in one wave) and the strip width in columns it uses for n output columns. */
int tfsc_k_dense_cluster_grid(int rows, int n, int* active_clusters, int* strip_cols);
/* X3: the wgmma (3xTF32) path alone, rows <= 64, n % 32 == 0, k % 4 == 0. tfsc_k_dense picks it
 * automatically for more than 8 rows; this entry exists for parity tests and roofline timing. */
int tfsc_k_dense_tc(const float* x, const float* w, const float* b, float* y, int rows, int k, int n, int relu,
                    float* workspace, size_t workspace_bytes, void* stream);

/* X6 (+ X7): batch gather / scatter as one kernel over a table of segments. src / dst may be pinned host memory, local HBM or
 * a peer's forward window (NVLink): this is the kernel the batcher uses to assemble a batch from its requests' rows and to
 * hand the result rows back (csrc/nn_kernels.cu copy_segments_kernel). */
typedef struct tfsc_copy_seg {
  const void* src;
  void* dst;
  uint64_t bytes;
} tfsc_copy_seg;
int tfsc_k_copy_segments(const tfsc_copy_seg* segs, int n, void* stream);

/* X4/X5 building blocks of the graph executor (conv nets), fp32, row-major / NHWC. act: 0 none, 1 relu, 2 gelu, 3 tanh,
 * 4 relu6 (min(max(x, 0), 6)), 5 silu (x / (1 + exp(-x))), 6 sigmoid (1 / (1 + exp(-x))), 7 gelu_tanh (0.5 x (1 + tanh(
 * sqrt(2 / pi) (x + 0.044715 x^3))), GPT-2's GELU); the same on tfsc_k_gemm_tc and tfsc_k_conv_tc.
 * C[M,N] = act(A[M,K] (row stride lda) * B[K,N] + bias[N] (+ R[M,N])); bias / R may be NULL. */
int tfsc_k_gemm(const float* a, const float* b, const float* bias, const float* r, float* c, int m, int n, int k, int lda,
                int act, void* stream);
/* the same GEMM on the tensor cores (wgmma, 3xTF32, fp32-accurate): m >= 64, n >= 64, n % 32 == 0, k >= 32, lda % 4 == 0 */
int tfsc_k_gemm_tc(const float* a, const float* b, const float* bias, const float* r, float* c, int m, int n, int k, int lda,
                   int act, void* stream);
/* X4: implicit-GEMM convolution on the tensor cores (wgmma, 3xTF32): y[B,OH,OW,cout] = act(conv2d(x[B,H,W,C] NHWC, w[KH,KW,C,cout] HWIO)
 * + bias (+ r)); the patch tiles are gathered from x by TMA im2col tensor maps, no patch matrix is materialised.
 * c % 32 == 0, cout >= 64 and % 32 == 0, batch*OH*OW >= 64. act: 0 none, 1 relu, 2 gelu, 3 tanh. */
int tfsc_k_conv_tc(const float* x, const float* w, const float* bias, const float* r, float* y, int batch, int h, int wd, int c,
                   int kh, int kw, int stride, int pad, int cout, int act, void* stream);
/* debugging aid kept for ABI compatibility: the clock-trace timeline belonged to the persistent GEMM kernel, which the
 * sm_90a build does not have; always returns TFSC_E_UNIMPLEMENTED and leaves out16 untouched */
int tfsc_debug_gemm_trace(long long* out16);
/* col[(b*OH+oh)*OW+ow][(kh*KW+kw)*C+c] patch matrix with row stride ldc >= KH*KW*C (zero padded) */
int tfsc_k_im2col(const float* x, float* col, int batch, int h, int w, int c, int kh, int kw, int stride, int pad, int ldc,
                  void* stream);
int tfsc_k_maxpool(const float* x, float* y, int batch, int h, int w, int c, int kh, int kw, int stride, int pad, void* stream);
int tfsc_k_avgpool(const float* x, float* y, int batch, int hw, int c, void* stream);
/* MobileNet / EfficientNet building blocks (fp32, device, NHWC). Depthwise convolution: y[b, oy, ox, ch] = act(sum_i sum_j
 * x[b, oy*stride - pad + i, ox*stride - pad + j, ch] * w[i, j, ch] + bias[ch]) with zero padding, OH = (h + 2 pad - kh) /
 * stride + 1 (OW likewise), w [kh, kw, c] (TF's [kh, kw, c, 1] depthwise layout), bias [c]. act: 0 none, 1 relu, 4 relu6,
 * 5 silu, 6 sigmoid. The taps are summed in the same order at every batch size and alignment, so a row's bits depend on
 * neither. TFSC_E_INVALID unless kh, kw in 1..7, stride in 1..2, pad <= kh / 2 and kw / 2, h * w * c < 2^31, and every
 * pointer is given. */
int tfsc_k_depthwise_conv(const float* x, const float* w, const float* bias, float* y, int batch, int h, int wd, int c, int kh, int kw,
                          int stride, int pad, int act, void* stream);
/* Squeeze-and-excitation gate: y[b, p, ch] = x[b, p, ch] * gate[b, ch] over hw positions p. TFSC_E_INVALID unless
 * hw * c < 2^31. */
int tfsc_k_channel_scale(const float* x, const float* gate, float* y, int batch, int hw, int c, void* stream);
/* Swin Transformer building blocks (fp32, device, NHWC). Shifted-window multi-head attention: qkv[batch, h, w, 3c] (q | k | v
 * of every token), ctx[batch, h, w, c], head width d = c / heads. The map is rolled by -shift on both axes and cut into
 * window x window windows of N = window^2 tokens; within a window, score(i, j) = q_i . k_j / sqrt(d) + bias[head, i, j]
 * (bias fp32 [heads, N, N], torchvision's relative_position_bias_table[relative_position_index]), plus -100 when shift > 0
 * and i, j lie in different regions of torchvision's shift mask; ctx_i = softmax_j(score) . v. A window's bits depend
 * neither on the batch nor on the alignment. TFSC_E_INVALID unless h and w are multiples of window, 1 <= window <= 16,
 * 0 <= shift < window, d <= 64, K and V of a window fit in 48 KB ((2d + 1) N floats plus 4 (N + d)), h * w * 3c < 2^31 and
 * every pointer is given. */
int tfsc_k_window_attention(const float* qkv, const float* bias, float* ctx, int batch, int h, int w, int c, int heads, int window,
                            int shift, void* stream);
/* Patch merging: y[b, oy, ox, q*c + ch] = x[b, 2 oy + (q & 1), 2 ox + (q >> 1), ch], [h, w, c] -> [h/2, w/2, 4c] (torchvision's
 * x0 | x1 | x2 | x3). TFSC_E_INVALID unless h and w are even, h * w * c < 2^31 and both pointers are given. */
int tfsc_k_patch_merge(const float* x, float* y, int batch, int h, int w, int c, void* stream);
/* X5 building blocks of the transformer graphs. Multi-head self-attention: qkv[batch, seq, 3*hidden] (q | k | v of every
 * token), ctx[batch, seq, hidden]; head width d = hidden / heads, scores scaled by 1/sqrt(d). ids[batch, seq] may be NULL;
 * a key whose id is 0 ([PAD]) gets the additive mask -10000 unless every key of its sequence is [PAD]. Every seq runs for
 * d % 4 == 0 and d <= 128 on 16-byte aligned qkv / ctx; other head widths while the row kernel's K / V fit in shared
 * memory. TFSC_E_INVALID for shapes no kernel can run. */
int tfsc_k_attention(const float* qkv, const int* ids, float* ctx, int batch, int seq, int hidden, int heads, void* stream);
/* The same with an explicit attention mask: key j of sequence b is masked iff mask[b*mask_stride + j] == 0 (the same
 * fully-masked rule). mask may be NULL; (ids, seq) gives tfsc_k_attention. TFSC_E_INVALID for mask_stride < seq. */
int tfsc_k_attention_mask(const float* qkv, const int* mask, int mask_stride, float* ctx, int batch, int seq, int hidden,
                          int heads, void* stream);
/* BERT embeddings: y[b*seq + s] = LayerNorm(word[id] + pos[s] + type[t]) * gamma + beta with id = ids[b*stride + s]
 * clamped to 0..vocab-1 and t = types[b*stride + s] clamped to 0..1 (types NULL: t = 0). word[vocab, hidden],
 * pos[>= seq, hidden], type[2, hidden]. TFSC_E_INVALID for stride < seq or hidden outside 1..12272. */
int tfsc_k_embed(const int* ids, const int* types, int stride, const float* word, const float* pos, const float* type,
                 const float* gamma, const float* beta, float* y, int batch, int seq, int hidden, int vocab, float eps,
                 void* stream);
/* y[t] = LayerNorm(x[t] (+ res[t])) * gamma + beta over rows of hidden floats (two-pass fp32 mean / variance); res may be
 * NULL; hidden in 1..12272. */
int tfsc_k_layernorm(const float* x, const float* res, const float* gamma, const float* beta, float* y, int tokens, int hidden,
                     float eps, void* stream);
/* Classification head of multi-output bundles, one launch for logits[rows, n] (fp32, device): probs[rows, n] = softmax
 * (max-subtracted, fp32), classes[rows] = argmax (ties: lowest index), topk_idx[rows, k] = the k largest logits' indices in
 * descending order (ties: lower index first, as tf.math.top_k), topk_prob[rows, k] = probs at those indices (the same bits).
 * Selection compares the fp32 logits exactly. Every output pointer may be NULL (not written). Logits must be finite.
 * TFSC_E_INVALID unless 1 <= n <= 32768 and 1 <= k <= min(n, 32). */
int tfsc_k_classify_head(const float* logits, int rows, int n, int k, float* probs, int64_t* classes, int32_t* topk_idx,
                         float* topk_prob, void* stream);
/* Span head of question-answering bundles, one launch for per-token logits[rows, S, 2] (start, end interleaved; fp32,
 * device): start_logits[rows, S], end_logits[rows, S], and the k best answer spans span_starts[rows, k] / span_ends[rows,
 * k] (int32) with span_scores[rows, k] = start[i] + end[j] (fp32). A candidate is a pair i <= j < i + max_answer_length
 * of eligible tokens; token p of row r is eligible when mask[q] != 0 (mask NULL: ids[q] != 0), types[q] == 1 and, with
 * sep_id >= 0, ids[q] != sep_id, q = r * stride + p (int32, device). Spans are ordered by score descending, then start,
 * then end ascending, compared exactly in fp32; a NaN score is never a candidate. Slots past the last candidate are
 * (-1, -1, -FLT_MAX). Every output pointer may be NULL (not written); without span pointers nothing but the logits is read.
 * TFSC_E_INVALID unless 1 <= S <= 4096, 1 <= max_answer_length <= S and 1 <= k <= 32, and for spans ids, types and
 * stride >= S. */
int tfsc_k_span_head(const float* logits, const int32_t* ids, const int32_t* mask, const int32_t* types, int stride, int rows, int S,
                     int max_answer_length, int k, int sep_id, float* start_logits, float* end_logits, int32_t* span_starts,
                     int32_t* span_ends, float* span_scores, void* stream);
/* Encoder head of embedding bundles, one launch for the last hidden states hidden[rows, S, H] and, for pooled_output, the
 * pooler output pooled[rows, H] (fp32, device): sequence_output[rows, S, H] and pooled_output[rows, H] (copies),
 * cls_embedding[rows, H] = hidden[r, 0] and mean_embedding[rows, H] = sum_p m[p] hidden[r, p] / max(sum_p m[p], 1e-9),
 * m[p] = mask[q] != 0 (mask NULL: ids[q] != 0), q = r * stride + p (int32, device). normalize_cls / normalize_mean != 0
 * divide that output by max(||x||_2, 1e-12). The hidden states are read once and every sum runs in an order fixed by S
 * and H, so a row's bits do not depend on the batch. Every output pointer may be NULL (not written). TFSC_E_INVALID unless
 * 1 <= S <= 8192 and 1 <= H <= 8192, hidden is given for sequence_output / cls_embedding / mean_embedding, pooled for
 * pooled_output, and ids with stride >= S for mean_embedding. */
int tfsc_k_encoder_head(const float* hidden, const float* pooled, const int32_t* ids, const int32_t* mask, int stride, int rows, int S,
                        int H, int normalize_cls, int normalize_mean, float* sequence_output, float* pooled_output,
                        float* cls_embedding, float* mean_embedding, void* stream);
/* Fill-mask gather of masked-language-model bundles, one launch for rows of hidden states hidden[rows, S, H] (fp32, device):
 * the candidates of row r are the tokens p with ids[q] == mask_token_id and, unless mask is NULL, mask[q] != 0,
 * q = r * stride + p (int32, device). The first `slots` = M of them in ascending p fill slots 0, 1, ...: positions[r * M + s]
 * = p and gathered[r, s, :] = hidden[r, p, :] (a bit-exact copy); empty slots hold -1 and zeros. Candidates past the
 * first M are not served. Every output pointer may be NULL (not written). TFSC_E_INVALID unless 1 <= M <= S <= 8192,
 * 1 <= H <= 8192, ids is given with stride >= S, and hidden is given for gathered. */
int tfsc_k_mask_gather(const float* hidden, const int32_t* ids, const int32_t* mask, int stride, int rows, int S, int H, int slots,
                       int mask_token_id, int32_t* positions, float* gathered, void* stream);
/* Fill-mask head, one launch for rows of M = `slots` slots: slot s of row r reads the first `vocab` logits of the row
 * logits + (r * M + s) * ld (fp32, device; ld >= vocab, the columns from vocab on are ignored) and the position
 * positions[r * M + s] (int32, device). A filled slot (position >= 0) writes its top k ids (descending logit, ties to the
 * lower id) to top_ids[r, s, :] (int32), their softmax probabilities over the vocab logits to top_probs[r, s, :] (the
 * same bits as tfsc_k_classify_head on those logits) and their logits to top_logits[r, s, :]; an empty slot writes -1, 0
 * and -FLT_MAX. Outputs are [rows, M, k]. Every output pointer may be NULL (not written). TFSC_E_INVALID unless
 * 1 <= M <= 8192, 1 <= vocab <= 32768 and 1 <= k <= min(vocab, 32), and positions, and logits for a top-k output, are
 * given. */
int tfsc_k_fill_mask_head(const float* logits, int64_t ld, const int32_t* positions, int rows, int slots, int vocab, int k,
                          int32_t* top_ids, float* top_probs, float* top_logits, void* stream);
/* GPT-2 building blocks (fp32, device). Causal multi-head self-attention: as tfsc_k_attention_mask, but query i of a sequence
 * sees keys j <= i only; a key it cannot see gets exactly zero weight. mask may be NULL (no key masked by it); a key whose
 * mask is 0 is masked by the same rule as tfsc_k_attention_mask. TFSC_E_INVALID unless d = hidden / heads has d % 4 == 0
 * and d <= 128, qkv and ctx are 16-byte aligned, and mask_stride >= seq for a mask. */
int tfsc_k_attention_causal(const float* qkv, const int* mask, int mask_stride, float* ctx, int batch, int seq, int hidden, int heads,
                            void* stream);
/* Embedding without LayerNorm: y[b*seq + s] = word[id] + pos[s] (one fp32 add) with id = ids[b*stride + s] clamped to
 * 0..vocab-1; word[vocab, hidden], pos[>= seq, hidden]. TFSC_E_INVALID for stride < seq or a null pointer. */
int tfsc_k_embed_positions(const int32_t* ids, int stride, const float* word, const float* pos, float* y, int batch, int seq,
                           int hidden, int vocab, void* stream);
/* Last attended token of rows of hidden states hidden[rows, S, H]: p = the highest position with mask[r * stride + p] != 0
 * (mask NULL: S - 1; no such position: -1). positions[r] = p (int32) and gathered[r, :] = hidden[r, p, :] (a bit-exact
 * copy; zeros for p = -1). Either output may be NULL. TFSC_E_INVALID for stride < S with a mask, or gathered without
 * hidden. */
int tfsc_k_last_token(const float* hidden, const int32_t* mask, int stride, int rows, int S, int H, int32_t* positions,
                      float* gathered, void* stream);
/* Next-token head: tfsc_k_fill_mask_head with one slot per row (row r reads logits + r * ld and positions[r]) and a vocabulary
 * of up to 57344. Outputs are [rows, k]; at vocab <= 32768 they carry the bits tfsc_k_fill_mask_head gives on the same logits.
 * TFSC_E_INVALID unless 1 <= vocab <= 57344 and 1 <= k <= min(vocab, 32), and positions, and logits for a top-k output, are
 * given. */
int tfsc_k_next_token_head(const float* logits, int64_t ld, const int32_t* positions, int rows, int vocab, int k, int32_t* top_ids,
                           float* top_probs, float* top_logits, void* stream);
/* Greedy generation. KV cache write: kc[r, s, :] = qkv[r, s, H:2H] and vc[r, s, :] = qkv[r, s, 2H:3H] for s < S, of a packed
 * qkv [rows, S, 3H] into caches [rows, T, H] (bit-exact copies). TFSC_E_INVALID for T < S or a NULL pointer. */
int tfsc_k_kv_cache_write(const float* qkv, float* kc, float* vc, int rows, int S, int T, int H, void* stream);
/* Decode attention of one query per row: qkv [rows, 3H] holds the q | k | v of the token at slot q_r = pos[r] + 1 + t
 * (pos[r] in -1..S-1). The query sees the cached keys j < q_r of kc / vc [rows, T, H] and its own key; a key j <= pos[r]
 * whose mask[r * mask_stride + j] is 0 gets the additive -10000 (mask may be NULL). Writes ctx [rows, H] and appends the
 * token's k and v at slot q_r. `work` holds work_bytes >= tfsc_k_decode_attention_work_bytes(rows, S + t + 1, H, heads)
 * bytes; it must be zero before the first launch and each launch leaves it so.
 * TFSC_E_INVALID unless 1 <= S + t + 1 <= min(T, 16384), the head width is d % 4 == 0, d <= 128, and mask_stride >= S with
 * a mask. */
int tfsc_k_decode_attention(const float* qkv, float* kc, float* vc, const int32_t* pos, int t, const int32_t* mask, int mask_stride,
                            int S, int T, float* ctx, int rows, int H, int heads, void* work, int64_t work_bytes, void* stream);
/* Bytes of the work buffer tfsc_k_decode_attention needs for rows over L = S + t + 1 keys. */
int64_t tfsc_k_decode_attention_work_bytes(int rows, int L, int H, int heads);
/* One greedy step: for row r, g = the argmax of logits[r * ld, +vocab) (ties to the lower id) and its log-probability
 * logit[g] - logsumexp. A row is live at t = 0 when pos[r] >= 0 and later while done[r] == 0; a live row writes
 * ids[r * ids_ld + t] = g, log_probs[r * lp_ld + t] and length[r * length_ld] = t + 1 and is done after g == eos (eos < 0:
 * none); any other row writes -1 and 0 (length 0 at t = 0). Unless last, y[r, :] = word[g] + pos_table[pos[r] + 1 + t]
 * (the bits of tfsc_k_embed_positions). Output pointers may be NULL. TFSC_E_INVALID unless 1 <= vocab <= 57344 and
 * ld >= vocab. */
int tfsc_k_generate_select(const float* logits, int64_t ld, int vocab, const int32_t* pos, int t, int last, int eos, int32_t* done,
                           int32_t* ids, int64_t ids_ld, float* log_probs, int64_t lp_ld, int32_t* length, int64_t length_ld,
                           const float* word, const float* pos_table, float* y, int rows, int H, void* stream);
/* One sampled step: tfsc_k_generate_select with g drawn instead of taken as the argmax. Of the tokens in rank order (logit
 * descending, ties to the lower id) it keeps the first top_k (0: all), weights them exp((z - max z) / temperature), keeps the
 * shortest prefix whose weight reaches top_p of theirs (1: all) and picks the first kept id, ascending, whose running weight
 * exceeds u * W (W the kept weight, u = the 53-bit uniform of Philox4x32-10 with key (seeds[r * seed_stride], 0) and
 * counter (t, 0, 0, 0)). top_k = 1 gives tfsc_k_generate_select's bits. The log-probability is logit[g] - logsumexp at
 * temperature 1, unfiltered, the bits tfsc_k_generate_select writes for the same g. TFSC_E_INVALID outside its limits and
 * unless temperature and its fp32 reciprocal are finite and > 0, 0 <= top_k <= vocab, 0 < top_p <= 1, seeds is given and seed_stride >= 1. */
int tfsc_k_generate_sample(const float* logits, int64_t ld, int vocab, const int32_t* pos, int t, int last, int eos, int32_t* done,
                           int32_t* ids, int64_t ids_ld, float* log_probs, int64_t lp_ld, int32_t* length, int64_t length_ld,
                           const float* word, const float* pos_table, float* y, int rows, int H, const int32_t* seeds,
                           int64_t seed_stride, float temperature, int top_k, float top_p, void* stream);
/* One step of a generate bundle with repetition control: tfsc_k_generate_select (seeds NULL) or tfsc_k_generate_sample (seeds
 * given, with temperature, top_k and top_p) with g chosen from the row's logits z after, in transformers' order: the
 * repetition penalty (z < 0 ? z * p : z / p in fp32, once per id of the row's history), the ban of every token that would
 * repeat an n-gram of the history (no_repeat_ngram_size = n, 0: off) and the ban of eos while t < min_new_tokens (0: off).
 * All banned: g = 0, no draw. The history is the row's attended prompt ids in position order, prompt_ids[r * stride + j] for
 * j <= pos[r] whose mask[r * stride + j] != 0 (mask NULL: all), each clamped to [0, vocab); the t = 0 step writes them to
 * hist[r * hist_ld ..] and their count to hist_len0[r], and every step appends g at hist[r * hist_ld + hist_len0[r] + t]
 * (pos[r] + N <= hist_ld). The log-probability is the raw row's, the bits tfsc_k_generate_select writes for the same g.
 * TFSC_E_INVALID outside tfsc_k_generate_select's limits, unless p's fp32 value is finite, > 0 and normal, n >= 0, m >= 0
 * with 0 <= eos < vocab when m > 0, prompt_ids, hist and hist_len0 are given, stride >= 1 and hist_ld > t, and with seeds
 * outside tfsc_k_generate_sample's. */
int tfsc_k_generate_process(const float* logits, int64_t ld, int vocab, const int32_t* pos, int t, int last, int eos, int32_t* done,
                            int32_t* ids, int64_t ids_ld, float* log_probs, int64_t lp_ld, int32_t* length, int64_t length_ld,
                            const float* word, const float* pos_table, float* y, int rows, int H, const int32_t* prompt_ids,
                            const int32_t* mask, int64_t stride, int32_t* hist, int64_t hist_ld, int32_t* hist_len0,
                            float repetition_penalty, int no_repeat_ngram_size, int min_new_tokens, const int32_t* seeds,
                            int64_t seed_stride, float temperature, int top_k, float top_p, void* stream);
/* Scoring. Token row i < n of logits[i * ld, +vocab) (ld >= vocab) is token g = first + i of a [rows, S] batch: row
 * r = g / S, position p = g % S. When p is attended (mask[r * stride + p] != 0; mask NULL: every position) and s = the
 * smallest attended position above p exists, it writes, with t = ids[r * stride + s] clamped to [0, vocab):
 * log_probs[r * S + s] = (z[t] - max z) - (float)log(sum_j exp(z[j] - max z)), fp32 exponentials summed in fp64 (the bits
 * tfsc_k_generate_select writes when t is the row's argmax), and ranks[r * S + s] = the number of j with z[j] > z[t] plus
 * the number of j < t with z[j] == z[t] (0: t is the next-token head's top-1). It writes nothing else; the padding columns
 * from vocab on are never read. TFSC_E_INVALID unless 1 <= S <= 16384, 1 <= vocab <= 57344, [first, first + n) lies within
 * rows * S, ld >= vocab and stride >= S. */
int tfsc_k_token_score(const float* logits, int64_t ld, int64_t first, int n, const int32_t* ids, const int32_t* mask, int64_t stride,
                       int rows, int S, int vocab, float* log_probs, int32_t* ranks, void* stream);
/* Score head: position s of row r is scored when it is attended (as above) and an attended position lies below it. Writes
 * token_log_probs[r * lp_ld + s] = log_probs[r * S + s] (0 unscored), token_ranks[r * ranks_ld + s] = ranks[r * S + s]
 * (-1 unscored), sum[r * sum_ld] = the scored log-probabilities summed in fp64 in an order fixed by S and rounded once
 * (0 for none) and count[r * count_ld] = the number of scored positions. log_probs and ranks are read at scored positions
 * only. Output pointers may be NULL. TFSC_E_INVALID unless 1 <= S <= 16384 and stride >= S. */
int tfsc_k_score_head(const float* log_probs, const int32_t* ranks, const int32_t* mask, int64_t stride, int rows, int S,
                      float* token_log_probs, int64_t lp_ld, int32_t* token_ranks, int64_t ranks_ld, float* sum, int64_t sum_ld,
                      int32_t* count, int64_t count_ld, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TFSC_B200_H_ */
