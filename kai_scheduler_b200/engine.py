"""ctypes binding of libkaigpu.so (the product).  No CPU fallback: a missing library or GPU raises."""
from __future__ import annotations

import ctypes as C
import os

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libkaigpu.so")
_LIB = None


class EngineError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"kai engine error {code}: {msg}")
        self.code = code


def lib() -> C.CDLL:
    """Load libkaigpu.so; fails loudly when the CUDA extension has not been built."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a).  There is no CPU fallback.")
        _LIB = C.CDLL(LIB_PATH)
        abi.bind_engine_api(_LIB, "kai_engine")
        _LIB.kai_last_error.argtypes = [C.c_void_p]
        _LIB.kai_last_error.restype = C.c_char_p
        _LIB.kai_abi_version.restype = C.c_int
        _LIB.kai_engine_export_peer_handle.argtypes = [C.c_void_p, C.POINTER(C.c_uint8)]
        _LIB.kai_engine_export_peer_handle.restype = C.c_int
        _LIB.kai_engine_wire_peers.argtypes = [C.c_void_p, C.POINTER(C.c_uint8)]
        _LIB.kai_engine_wire_peers.restype = C.c_int
        _LIB.kai_shard_range.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        _LIB.kai_shard_range.restype = C.c_int
    return _LIB


EXPORTED_SYMBOLS = [
    "kai_engine_create", "kai_engine_load_snapshot", "kai_engine_run", "kai_engine_fair_share",
    "kai_engine_stats", "kai_engine_export_peer_handle", "kai_engine_wire_peers", "kai_engine_destroy",
    "kai_last_error", "kai_abi_version", "kai_shard_range", "kai_engine_time_sweeps",
]


def shard_range(n_nodes: int, shard_count: int, shard_rank: int):
    """(first_rank, count): shard `shard_rank` owns the nodes of NAME RANK first_rank + k * shard_count, k < count."""
    b, c = C.c_int(), C.c_int()
    rc = lib().kai_shard_range(n_nodes, shard_count, shard_rank, C.byref(b), C.byref(c))
    if rc != 0:
        raise EngineError(rc, "kai_shard_range")
    return b.value, c.value


def shard_node_mask(node_name_rank, shard_count: int, shard_rank: int):
    """Boolean mask over node indices: the rows whose idle/releasing tables engine `shard_rank` returns."""
    import numpy as np
    return (np.asarray(node_name_rank) % shard_count) == shard_rank


class Engine:
    """One engine per GPU.  load() = OpenSession for the plugins on the path; run(action) = Action.Execute."""

    def __init__(self, cfg: abi.KaiConfig | None = None):
        self._lib = lib()
        self._cfg = cfg or abi.make_config()
        self._h = C.c_void_p()
        rc = self._lib.kai_engine_create(C.byref(self._cfg), C.byref(self._h))
        if rc != 0:
            raise EngineError(rc, "kai_engine_create failed (no CUDA device?)" if rc == abi.ERR_NO_DEVICE else "create")
        self._n_res = 4

    def _check(self, rc):
        if rc != 0:
            raise EngineError(rc, self._lib.kai_last_error(self._h).decode())

    def load(self, snap: abi.Snapshot):
        c = snap.to_c()
        self._n_res = snap.n_res
        self._check(self._lib.kai_engine_load_snapshot(self._h, C.byref(c)))

    def load_c(self, c_snap: abi.KaiSnapshot, n_res: int):
        """Load from an already marshalled kai_snapshot (host pointers) — the timed e2e path of bench.py."""
        self._n_res = n_res
        self._check(self._lib.kai_engine_load_snapshot(self._h, C.byref(c_snap)))

    def run(self, action, copy: bool = True):
        a = abi.ACTIONS[action] if isinstance(action, str) else action
        r = abi.KaiResult()
        self._check(self._lib.kai_engine_run(self._h, a, C.byref(r)))
        return abi.Result.from_c(r, self._n_res) if copy else r

    def fair_share(self) -> abi.Result:
        r = abi.KaiResult()
        self._check(self._lib.kai_engine_fair_share(self._h, C.byref(r)))
        return abi.Result.from_c(r, self._n_res)

    def stats(self) -> abi.KaiStats:
        s = abi.KaiStats()
        self._check(self._lib.kai_engine_stats(self._h, C.byref(s)))
        return s

    def time_sweeps(self, n_launches: int = 200):
        """(ms per sweep launch, ms per merge launch, node rows per launch): back-to-back launches, CUDA events."""
        ms, mms, rows = C.c_double(), C.c_double(), C.c_int64()
        fn = self._lib.kai_engine_time_sweeps
        fn.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int64)]
        fn.restype = C.c_int
        self._check(fn(self._h, n_launches, C.byref(ms), C.byref(mms), C.byref(rows)))
        return ms.value / n_launches, mms.value / n_launches, rows.value

    def export_peer_handle(self) -> bytes:
        buf = (C.c_uint8 * abi.PEER_HANDLE_BYTES)()
        self._check(self._lib.kai_engine_export_peer_handle(self._h, buf))
        return bytes(buf)

    def wire_peers(self, handles: list[bytes]):
        raw = b"".join(h.ljust(abi.PEER_HANDLE_BYTES, b"\0")[:abi.PEER_HANDLE_BYTES] for h in handles)
        buf = (C.c_uint8 * len(raw)).from_buffer_copy(raw)
        self._check(self._lib.kai_engine_wire_peers(self._h, buf))

    def close(self):
        if getattr(self, "_h", None):
            self._lib.kai_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
