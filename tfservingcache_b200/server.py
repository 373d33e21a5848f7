"""Server: the cache tier + proxy tier (cmd/taskhandler/main.go:45-113) for this process's GPUs,
over the C ABI.  predict() = proxyServiceServer.Predict with the forward replaced by on-GPU
execution; grpc_predict()/rest_handle() are the wire-level entry points a front-end binds."""
from __future__ import annotations

import ctypes as C
import json

import numpy as np

from . import _lib
from ._lib import TfscStats, TfscTensor, check, lib


class Server:
    def __init__(self, config: dict):
        self._h = lib.tfsc_server_create(json.dumps(config).encode())
        if not self._h:
            code = _lib.E_NO_DEVICE if b"CUDA" in lib.tfsc_last_error() else _lib.E_INVALID
            raise _lib.TfscError(code, "server_create")
        self.config = config

    def close(self):
        if getattr(self, "_h", None):
            lib.tfsc_server_destroy(self._h)
            self._h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    @property
    def num_nodes(self) -> int:
        return lib.tfsc_server_num_nodes(self._h)

    def set_members(self, members: list[str]):
        arr = (C.c_char_p * len(members))(*[m.encode() for m in members])
        check(lib.tfsc_server_set_members(self._h, arr, len(members)), "set_members")

    def route(self, model_name: str, version: str):
        nodes = (C.c_int * 64)()
        picked = C.c_int()
        n = check(lib.tfsc_route(self._h, model_name.encode(), version.encode(), nodes, 64, C.byref(picked)), "route")
        return list(nodes[:n]), picked.value

    def ensure(self, node: int, model_name: str, version: int) -> int:
        return check(lib.tfsc_model_ensure(self._h, node, model_name.encode(), version), "model_ensure")

    def ensure_async(self, node: int, model_name: str, version: int) -> int:
        """fetchModel without waiting for the page-in (launches wait for it on-device)."""
        return check(lib.tfsc_model_ensure_async(self._h, node, model_name.encode(), version), "model_ensure_async")

    def status(self, node: int, model_name: str, version: int) -> int:
        return lib.tfsc_model_status(self._h, node, model_name.encode(), version)

    def _lines(self, fn, node):
        cap = 1 << 20
        buf = C.create_string_buffer(cap)
        check(fn(self._h, node, buf, cap), "list")
        return [l.split("\t") for l in buf.value.decode().splitlines()]

    def resident(self, node: int):
        return [(n, int(v), int(b), int(s)) for n, v, b, s in self._lines(lib.tfsc_resident_list, node)]

    def host_models(self, node: int):
        return [(n, int(v), int(b)) for n, v, b, _p in self._lines(lib.tfsc_host_list, node)]

    def predict(self, model_name: str, version: str, x, out_capacity_elems: int | None = None,
                input_name: str | None = None, outputs=None):
        """x: one array, or {name: array} for a model with several inputs (e.g. BERT's input_ids / input_mask /
        segment_ids, int32 [batch, seq] each). outputs: names of outputs of a multi-output model (signature.outputs,
        e.g. ("classes", "probabilities")): the result is then {name: ndarray} (classes int64, top-k classes int32);
        without it the result is the one ndarray of a single-output model."""
        _x, tin, tout, n_out, result = self._request(x, dict(out_capacity_elems=out_capacity_elems, input_name=input_name,
                                                             outputs=outputs))
        check(lib.tfsc_predict(self._h, model_name.encode(), version.encode(), tin, len(tin), tout, n_out), "predict")
        return result()

    @staticmethod
    def _request(x, kw):
        """(the input arrays kept alive, the input tensors, the output tensor(s), their count, result) of one Predict;
        result() reads what the call wrote: {name: ndarray} when kw["outputs"] names outputs, else one ndarray."""
        outputs = kw.get("outputs")
        if outputs is not None:
            outputs = list(outputs)
            arrays, tin, ys, touts = Server._tensors_multi(x, kw.get("out_capacity_elems"), kw.get("input_name"), outputs)
            return arrays, tin, touts, len(outputs), lambda: Server._results(ys, touts, outputs)
        arrays, tin, y, tout = Server._tensors(x, kw.get("out_capacity_elems"), kw.get("input_name"))
        return arrays, tin, C.byref(tout), 1, lambda: Server._result(y, tout)

    @staticmethod
    def _tensors_multi(x, out_capacity_elems, input_name, outputs):
        """_tensors with one named output tensor per entry of `outputs`, each with its own buffer"""
        arrays, tin, _y, _t = Server._tensors(x, 1, input_name)
        if out_capacity_elems is None:
            lead = arrays[0].shape[0] if arrays[0].ndim > 1 else 1
            out_capacity_elems = max(sum(a.size for a in arrays) * 4 + 65536, lead * 32768 * 2)
            if np.issubdtype(arrays[0].dtype, np.integer):
                # token-id requests: room for an encoder's [rows, S, H] sequence_output up to H = 1024
                out_capacity_elems = max(out_capacity_elems, arrays[0].size * 1024)
        ys, touts = [], (TfscTensor * len(outputs))()
        for t, name in zip(touts, outputs):
            y = np.empty(out_capacity_elems * 4, dtype=np.uint8)
            ys.append(y)
            t.name = name.encode()
            t.data = y.ctypes.data
            t.nbytes = y.nbytes
        return arrays, tin, ys, touts

    @staticmethod
    def _results(ys, touts, outputs) -> dict:
        np_dt = {_lib.DT_FLOAT: np.float32, _lib.DT_INT32: np.int32, _lib.DT_INT64: np.int64}
        res = {}
        for y, t, name in zip(ys, touts, outputs):
            shape = tuple(t.shape[i] for i in range(t.rank))
            res[name] = y[:t.nbytes].view(np_dt[t.dtype]).reshape(shape).copy()
        return res

    @staticmethod
    def _tensors(x, out_capacity_elems, input_name):
        """(the arrays kept alive, an array of input tensors, the output buffer, the output tensor). x is one array
        (named input_name, or unnamed) or a {name: array} dict."""
        items = list(x.items()) if isinstance(x, dict) else [(input_name, x)]
        arrays, tin = [], (TfscTensor * len(items))()
        for t, (name, a) in zip(tin, items):
            is_int = np.issubdtype(np.asarray(a).dtype, np.integer)   # token-id inputs (BERT bundles) travel as DT_INT32
            a = np.ascontiguousarray(a, dtype=np.int32 if is_int else np.float32)
            arrays.append(a)
            t.name = name.encode() if name else None
            t.dtype = _lib.DT_INT32 if is_int else _lib.DT_FLOAT
            t.rank = a.ndim
            for i, d in enumerate(a.shape):
                t.shape[i] = d
            t.data = a.ctypes.data
            t.nbytes = a.nbytes
        size = sum(a.size for a in arrays)
        cap = out_capacity_elems if out_capacity_elems is not None else max(size, 1) * 4 + 65536
        y = np.empty(cap, dtype=np.float32)
        tout = TfscTensor()
        tout.data = y.ctypes.data
        tout.nbytes = y.nbytes
        return arrays, tin, y, tout

    @staticmethod
    def _result(y, tout):
        shape = tuple(tout.shape[i] for i in range(tout.rank))
        n = int(np.prod(shape)) if shape else 1
        return y[:n].reshape(shape).copy()

    def predict_deadline(self, model_name: str, version: str, x: np.ndarray, deadline_ns: int, **kw) -> np.ndarray:
        """tfsc_predict_deadline: deadline is absolute on the clock of now_ns() (0 = none). outputs= as for predict()."""
        _x, tin, tout, n_out, result = self._request(x, kw)
        check(lib.tfsc_predict_deadline(self._h, model_name.encode(), version.encode(), tin, len(tin), tout, n_out,
                                        int(deadline_ns)), "predict")
        return result()

    def predict_member(self, member: int, model_name: str, version: str, x: np.ndarray, deadline_ns: int = 0, **kw) -> np.ndarray:
        """tfsc_predict_member: the cache tier of member `member` (index into gpu.members), no ring lookup. outputs= as for
        predict()."""
        _x, tin, tout, n_out, result = self._request(x, kw)
        check(lib.tfsc_predict_member(self._h, member, model_name.encode(), version.encode(), tin, len(tin), tout, n_out,
                                      int(deadline_ns)), "predict_member")
        return result()

    @staticmethod
    def now_ns() -> int:
        return lib.tfsc_now_ns()

    def predict_submit(self, model_name: str, version: str, x: np.ndarray, deadline_ns: int = 0, **kw) -> "Ticket":
        """Asynchronous Predict (tfsc_predict_submit): returns a Ticket; .wait() yields the result. outputs= as for
        predict()."""
        t = C.c_void_p()
        xk, tin, tout, n_out, result = self._request(x, kw)
        check(lib.tfsc_predict_submit(self._h, model_name.encode(), version.encode(), tin, len(tin), tout, n_out,
                                      int(deadline_ns), C.byref(t)), "predict_submit")
        return Ticket(t, result, keep=(xk, tout))

    def fwd_window(self):
        """(rank, device pointer, bytes, slot bytes) of this rank's forward window (needs cluster.endpoints)."""
        p, n, sb = C.c_void_p(), C.c_size_t(), C.c_size_t()
        rank = check(lib.tfsc_fwd_window(self._h, C.byref(p), C.byref(n), C.byref(sb)), "fwd_window")
        return rank, p.value, n.value, sb.value

    def fwd_peer_window(self, peer_rank: int):
        """(device pointer, bytes) of another rank's window mapped into this process (CUDA IPC)."""
        p, n = C.c_void_p(), C.c_size_t()
        check(lib.tfsc_fwd_peer_window(self._h, peer_rank, C.byref(p), C.byref(n)), "fwd_peer_window")
        return p.value, n.value

    def _wire_call(self, fn, request_bytes: bytes, where: str) -> bytes:
        resp = C.c_void_p()
        n = C.c_size_t()
        check(fn(self._h, request_bytes, len(request_bytes), C.byref(resp), C.byref(n)), where)
        try:
            return C.string_at(resp, n.value)
        finally:
            lib.tfsc_free(resp)

    def grpc_predict(self, request_bytes: bytes) -> bytes:
        return self._wire_call(lib.tfsc_grpc_predict, request_bytes, "grpc_predict")

    def grpc_classify(self, request_bytes: bytes) -> bytes:
        return self._wire_call(lib.tfsc_grpc_classify, request_bytes, "grpc_classify")

    def grpc_regress(self, request_bytes: bytes) -> bytes:
        return self._wire_call(lib.tfsc_grpc_regress, request_bytes, "grpc_regress")

    def grpc_session_run(self, request_bytes: bytes) -> bytes:
        return self._wire_call(lib.tfsc_grpc_session_run, request_bytes, "grpc_session_run")

    def rest_handle(self, method: str, url: str, body: bytes = b""):
        st = C.c_int()
        resp = C.c_void_p()
        n = C.c_size_t()
        check(lib.tfsc_rest_handle(self._h, method.encode(), url.encode(), body, len(body), C.byref(st), C.byref(resp),
                                   C.byref(n)), "rest_handle")
        try:
            return st.value, C.string_at(resp, n.value)
        finally:
            lib.tfsc_free(resp)

    def predict_device(self, node: int, model_name: str, version: int, x_ptr: int, rows: int, y_ptr: int, stream: int = 0):
        check(lib.tfsc_predict_device(self._h, node, model_name.encode(), version, x_ptr, rows, y_ptr, stream),
              "predict_device")

    def set_max_resident(self, node: int, n: int):
        check(lib.tfsc_node_set_max_resident(self._h, node, n), "set_max_resident")

    def sync(self, node: int = 0):
        check(lib.tfsc_node_sync(self._h, node), "node_sync")

    def stats(self, node: int = -1) -> dict:
        st = TfscStats()
        check(lib.tfsc_get_stats(self._h, node, C.byref(st)), "get_stats")
        return st.as_dict()


class Ticket:
    """An in-flight asynchronous Predict (tfsc_ticket). Keeps the output buffer alive until released."""

    def __init__(self, handle, result, keep=None):
        self._t, self._result, self._keep = handle, result, keep

    def wait(self, timeout_s: float | None = None):
        check(lib.tfsc_predict_wait(self._t, -1 if timeout_s is None else int(timeout_s * 1e9)), "predict_wait")
        return self._result()

    def release(self):
        if self._t:
            lib.tfsc_predict_release(self._t)
            self._t = None

    __del__ = release
