"""ctypes binding of libtfsc_b200.so (include/tfsc_b200.h).  There is no fallback: if the shared
library is missing the import fails loudly, and every compute entry point returns
TFSC_E_NO_DEVICE when no sm_90 GPU (H100) is present."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtfsc_b200.so")

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "or `make -C tfservingcache_b200/csrc` (nvcc, sm_90a). There is no CPU fallback.")

lib = C.CDLL(LIB_PATH)

TFSC_OK = 0
E_INVALID, E_TIMEOUT, E_NOT_FOUND, E_EXHAUSTED = -3, -4, -5, -8
E_UNIMPLEMENTED, E_INTERNAL, E_NO_DEVICE, E_EMPTY_RING, E_BUFFER = -12, -13, -14, -20, -21
STATE_UNKNOWN, STATE_START, STATE_LOADING, STATE_AVAILABLE, STATE_UNLOADING, STATE_END = 0, 10, 20, 30, 40, 50
FETCH_HIT, FETCH_RELOAD, FETCH_MISS = 0, 1, 2
DT_FLOAT, DT_INT32, DT_INT64 = 1, 3, 9


class TfscTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("dtype", C.c_int32), ("rank", C.c_int32),
                ("shape", C.c_int64 * 8), ("data", C.c_void_p), ("nbytes", C.c_size_t)]


class TfscStats(C.Structure):
    _fields_ = [(n, C.c_int64) for n in (
        "cache_total", "cache_hits_total", "cache_misses_total",
        "proxy_requests_rest", "proxy_requests_grpc", "proxy_failures_rest", "proxy_failures_grpc",
        "evictions_host", "evictions_hbm", "h2d_weight_bytes", "h2d_input_bytes", "d2h_output_bytes",
        "kernel_launches", "batches", "batched_rows",
        "arena_bytes_used", "arena_bytes_capacity", "resident_models", "host_models")] + [
        ("cache_duration_seconds_sum", C.c_double), ("cache_fetch_duration_seconds_sum", C.c_double)] + [
        (n, C.c_int64) for n in ("fwd_out_requests", "fwd_in_requests", "fwd_out_failures", "fwd_peer_bytes_read",
                                 "fwd_peer_bytes_written")] + [("fwd_rtt_seconds_sum", C.c_double)] + [
        ("arena_compactions", C.c_int64), ("arena_compacted_bytes", C.c_int64)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


def _sig(name, restype, *argtypes):
    fn = getattr(lib, name)
    fn.restype = restype
    fn.argtypes = list(argtypes)
    return fn


vp, cp, i64, sz = C.c_void_p, C.c_char_p, C.c_int64, C.c_size_t
_sig("tfsc_abi_version", C.c_int)
_sig("tfsc_last_error", cp)
_sig("tfsc_strerror", cp, C.c_int)
_sig("tfsc_free", None, vp)
_sig("tfsc_crc32_ieee", C.c_uint32, vp, sz)
_sig("tfsc_ring_new", vp)
_sig("tfsc_ring_free", None, vp)
_sig("tfsc_ring_set", C.c_int, vp, C.POINTER(cp), C.c_int)
_sig("tfsc_ring_members", C.c_int, vp)
_sig("tfsc_ring_points", C.c_int, vp)
_sig("tfsc_ring_getn", C.c_int, vp, cp, C.c_int, C.c_char_p, sz)
_sig("tfsc_model_key", C.c_int, cp, cp, C.c_char_p, sz)
_sig("tfsc_picker_new", vp, cp, C.c_uint64, C.c_double)
_sig("tfsc_picker_free", None, vp)
_sig("tfsc_picker_pick", C.c_int, vp, cp, C.c_int, C.c_int)
_sig("tfsc_picker_pick_ids", C.c_int, vp, cp, C.POINTER(C.c_int), C.c_int, C.c_int)
_sig("tfsc_lru_new", vp, cp, i64)
_sig("tfsc_lru_free", None, vp)
_sig("tfsc_lru_put", C.c_int, vp, cp, i64, cp, i64)
_sig("tfsc_lru_get", C.c_int, vp, cp, i64, C.POINTER(i64), C.c_char_p, sz)
_sig("tfsc_lru_ensure_free_bytes", C.c_int, vp, i64)
_sig("tfsc_lru_current_size", i64, vp)
_sig("tfsc_lru_capacity", i64, vp)
_sig("tfsc_lru_len", C.c_int, vp)
_sig("tfsc_lru_list", C.c_int, vp, C.c_char_p, sz)
_sig("tfsc_rest_match_url", C.c_int, cp, C.c_char_p, sz, C.c_char_p, sz)
_sig("tfsc_rest_error_body", cp, C.c_int)
_sig("tfsc_parse_version", C.c_int, cp, C.POINTER(i64))
_sig("tfsc_grpc_model_spec", C.c_int, vp, sz, C.c_char_p, sz, C.c_char_p, sz)
_sig("tfsc_disk_find_version_dir", C.c_int, cp, cp, i64, C.c_char_p, sz)
_sig("tfsc_disk_model_size", i64, cp, cp, i64)
_sig("tfsc_savedmodel_convert", C.c_int, cp, cp)
_sig("tfsc_crc32c", C.c_uint32, vp, sz)
_sig("tfsc_manifest_check", C.c_int, cp, C.c_char_p, sz)
_sig("tfsc_server_create", vp, cp)
_sig("tfsc_server_destroy", None, vp)
_sig("tfsc_server_num_nodes", C.c_int, vp)
_sig("tfsc_server_set_members", C.c_int, vp, C.POINTER(cp), C.c_int)
_sig("tfsc_route", C.c_int, vp, cp, cp, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int))
_sig("tfsc_model_ensure", C.c_int, vp, C.c_int, cp, i64)
_sig("tfsc_model_status", C.c_int, vp, C.c_int, cp, i64)
_sig("tfsc_model_ensure_async", C.c_int, vp, C.c_int, cp, i64)
_sig("tfsc_resident_list", C.c_int, vp, C.c_int, C.c_char_p, sz)
_sig("tfsc_host_list", C.c_int, vp, C.c_int, C.c_char_p, sz)
_sig("tfsc_predict", C.c_int, vp, cp, cp, C.POINTER(TfscTensor), C.c_int, C.POINTER(TfscTensor), C.c_int)
_sig("tfsc_predict_deadline", C.c_int, vp, cp, cp, C.POINTER(TfscTensor), C.c_int, C.POINTER(TfscTensor), C.c_int, i64)
_sig("tfsc_now_ns", i64)
_sig("tfsc_predict_member", C.c_int, vp, C.c_int, cp, cp, C.POINTER(TfscTensor), C.c_int, C.POINTER(TfscTensor), C.c_int, i64)
_sig("tfsc_predict_submit", C.c_int, vp, cp, cp, C.POINTER(TfscTensor), C.c_int, C.POINTER(TfscTensor), C.c_int, i64, C.POINTER(vp))
_sig("tfsc_predict_wait", C.c_int, vp, i64)
_sig("tfsc_predict_release", None, vp)
_sig("tfsc_fwd_window", C.c_int, vp, C.POINTER(vp), C.POINTER(sz), C.POINTER(sz))
_sig("tfsc_fwd_peer_window", C.c_int, vp, C.c_int, C.POINTER(vp), C.POINTER(sz))
_sig("tfsc_device_memcpy", C.c_int, vp, vp, sz)
_sig("tfsc_grpc_predict", C.c_int, vp, vp, sz, C.POINTER(vp), C.POINTER(sz))
for _n in ("tfsc_grpc_classify", "tfsc_grpc_regress", "tfsc_grpc_session_run"):
    _sig(_n, C.c_int, vp, vp, sz, C.POINTER(vp), C.POINTER(sz))
_sig("tfsc_rest_handle", C.c_int, vp, cp, cp, vp, sz, C.POINTER(C.c_int), C.POINTER(vp), C.POINTER(sz))
_sig("tfsc_predict_device", C.c_int, vp, C.c_int, cp, i64, vp, i64, vp, vp)
_sig("tfsc_node_sync", C.c_int, vp, C.c_int)
_sig("tfsc_node_set_max_resident", C.c_int, vp, C.c_int, C.c_int)


class TfscCopySeg(C.Structure):
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("bytes", C.c_uint64)]


_sig("tfsc_k_copy_segments", C.c_int, C.POINTER(TfscCopySeg), C.c_int, vp)
_sig("tfsc_get_stats", C.c_int, vp, C.c_int, C.POINTER(TfscStats))
_sig("tfsc_kernel_launches", i64)
_sig("tfsc_k_affine", C.c_int, vp, vp, i64, vp, vp, vp)
_sig("tfsc_k_dense", C.c_int, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, sz, vp)
_sig("tfsc_k_dense_workspace", sz, C.c_int, C.c_int, C.c_int)
_sig("tfsc_k_dense_variant", C.c_int, C.c_int, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, sz, vp)
_sig("tfsc_k_dense_cluster_grid", C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int))
_sig("tfsc_k_dense_tc", C.c_int, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, sz, vp)
_sig("tfsc_k_gemm", C.c_int, vp, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp)
_sig("tfsc_k_gemm_tc", C.c_int, vp, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp)
_sig("tfsc_k_conv_tc", C.c_int, vp, vp, vp, vp, vp, *([C.c_int] * 10), vp)
_sig("tfsc_k_im2col", C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp)
_sig("tfsc_k_maxpool", C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp)
_sig("tfsc_k_avgpool", C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, vp)
_sig("tfsc_k_depthwise_conv", C.c_int, vp, vp, vp, vp, *([C.c_int] * 9), vp)
_sig("tfsc_k_channel_scale", C.c_int, vp, vp, vp, C.c_int, C.c_int, C.c_int, vp)
_sig("tfsc_k_window_attention", C.c_int, vp, vp, vp, *([C.c_int] * 7), vp)
_sig("tfsc_k_patch_merge", C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp)
_sig("tfsc_k_attention", C.c_int, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp)
_sig("tfsc_k_attention_mask", C.c_int, vp, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp)
_sig("tfsc_k_embed", C.c_int, vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, vp)
_sig("tfsc_k_layernorm", C.c_int, vp, vp, vp, vp, vp, C.c_int, C.c_int, C.c_float, vp)
_sig("tfsc_k_classify_head", C.c_int, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp)
_sig("tfsc_k_span_head", C.c_int, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp)
_sig("tfsc_k_encoder_head", C.c_int, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp)
_sig("tfsc_k_mask_gather", C.c_int, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp)
_sig("tfsc_k_fill_mask_head", C.c_int, vp, C.c_int64, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp)


class TfscError(RuntimeError):
    def __init__(self, code: int, where: str = ""):
        self.code = code
        msg = lib.tfsc_last_error().decode(errors="replace")
        super().__init__(f"{where}: {lib.tfsc_strerror(code).decode()} ({code}): {msg}")


def check(rc: int, where: str = "") -> int:
    if rc < 0:
        raise TfscError(rc, where)
    return rc
