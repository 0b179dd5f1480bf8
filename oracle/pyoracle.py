"""ctypes wrapper of oracle/libtgoracle.so — TEST INFRASTRUCTURE ONLY.

May be imported by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs; never by the distributed_crawler_b200 package.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from distributed_crawler_b200 import abi

_HERE = os.path.dirname(os.path.abspath(__file__))


class OrcResultC(C.Structure):  # oracle/tgoracle.h orc_result 
    _fields_ = [
        ("n", C.c_uint64), ("status", C.c_void_p), ("jsonl", C.c_void_p), ("jsonl_len", C.c_uint64),
        ("line_off", C.c_void_p), ("link_off", C.c_void_p), ("links", C.c_void_p),
        ("n_links", C.c_uint64), ("n_new", C.c_uint64), ("frontier_size", C.c_uint64)]



_LIB = None


def build(force: bool = False) -> str:
    so = os.path.join(_HERE, "libtgoracle.so")
    src = os.path.join(_HERE, "tgoracle.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return so


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        L.orc_create.argtypes = [C.POINTER(abi.ConfigC), C.POINTER(C.c_void_p)]
        L.orc_destroy.argtypes = [C.c_void_p]
        L.orc_set_clock.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_int32]
        L.orc_telegram_batch.argtypes = [C.c_void_p, C.POINTER(abi.TgBatchC), C.c_uint32, C.c_int,
                                         C.POINTER(OrcResultC)]
        L.orc_key_join.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p]
        L.orc_key_join.restype = None
        L.orc_generic_batch.argtypes = [C.c_void_p, C.POINTER(abi.GmBatchC), C.c_uint32, C.c_int,
                                        C.POINTER(OrcResultC)]
        L.orc_youtube_batch.argtypes = [C.c_void_p, C.POINTER(abi.YtBatchC), C.c_uint32, C.c_int,
                                        C.POINTER(OrcResultC)]
        L.orc_result_free.argtypes = [C.POINTER(OrcResultC)]
        L.orc_frontier_insert.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
        L.orc_frontier_size.restype = C.c_uint64
        L.orc_frontier_size.argtypes = [C.c_void_p]
        L.orc_frontier_export.restype = C.c_uint64
        L.orc_frontier_export.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        L.orc_frontier_clear.argtypes = [C.c_void_p]
        L.orc_set_add.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64]
        L.orc_set_clear.argtypes = [C.c_void_p, C.c_int]
        L.orc_set_clear.restype = None
        L.orc_set_now.argtypes = [C.c_void_p, C.c_int64]
        L.orc_set_now.restype = None
        L.orc_pending_edges.restype = C.c_uint64
        L.orc_pending_edges.argtypes = [C.c_void_p, C.POINTER(OrcResultC), C.c_void_p, C.c_uint32, C.c_int64, C.c_void_p, C.c_uint64]
        L.orc_utf16_offset_to_bytes.argtypes = [C.c_char_p, C.c_int64, C.c_int32, C.c_int32,
                                                C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.orc_filter_username.argtypes = [C.c_char_p, C.c_int64]
        L.orc_json_string.restype = C.c_uint64
        L.orc_json_string.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p]
        L.orc_json_time.argtypes = [C.c_int64, C.c_int32, C.c_int32, C.c_void_p]
        L.orc_parse_iso8601_duration.argtypes = [C.c_char_p, C.c_int64, C.POINTER(C.c_int64)]
        L.orc_json_float_of_int64.argtypes = [C.c_int64, C.c_void_p]
        _LIB = L
    return _LIB


class Result:
    """numpy copies of an orc_result / tgi_result (same field meaning)."""

    def __init__(self, n, status, jsonl, line_off, link_off, links, n_new, frontier_size):
        self.n, self.status, self.jsonl, self.line_off = n, status, jsonl, line_off
        self.link_off, self.links, self.n_new, self.frontier_size = link_off, links, n_new, frontier_size

    def line(self, i: int) -> bytes:
        return self.jsonl[int(self.line_off[i]):int(self.line_off[i + 1])].tobytes()

    def record_links(self, i: int) -> list[tuple[bytes, str]]:
        out = []
        for k in range(int(self.link_off[i]), int(self.link_off[i + 1])):
            l = self.links[k]
            out.append((l["name"][: int(l["len"])].tobytes(), abi.SRC_NAMES[int(l["src"])]))
        return out


def _copy(p, n, dt):
    if not n:
        return np.zeros(0, dt)
    return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), (n * np.dtype(dt).itemsize,)).view(dt).copy()


def result_from_c(r) -> Result:
    n = int(r.n)
    return Result(n, _copy(r.status, n, np.uint8), _copy(r.jsonl, int(r.jsonl_len), np.uint8),
                  _copy(r.line_off, n + 1, np.uint64), _copy(r.link_off, n + 1, np.uint32),
                  _copy(r.links, int(r.n_links), abi.LINK), int(r.n_new), int(r.frontier_size))


class OracleError(RuntimeError):
    """a call the library refuses with the same code (abi.E_ARG)"""

    def __init__(self, code: int, what: str):
        super().__init__(f"{what}: {code}")
        self.code = code


def _check(rc: int, what: str):
    if rc != 0:
        raise OracleError(rc, what)


class Oracle:
    def __init__(self, cfg: abi.ConfigC | None = None, **kw):
        self.cfg = cfg or abi.make_config(**kw)
        self.h = None
        h = C.c_void_p()
        _check(lib().orc_create(C.byref(self.cfg), C.byref(h)), "orc_create")
        self.h = h.value

    def close(self):
        if getattr(self, "h", None):
            lib().orc_destroy(self.h)
            self.h = None

    __del__ = close

    def set_clock(self, created_at_sec, created_at_nsec, capture_sec, capture_nsec):
        _check(lib().orc_set_clock(self.h, created_at_sec, created_at_nsec, capture_sec, capture_nsec), "orc_set_clock")

    def telegram(self, batch, run_flags=abi.RUN_JSONL | abi.RUN_LINKS, nthreads=1, copy=True):
        d = batch.descriptor()
        r = OrcResultC()
        _check(lib().orc_telegram_batch(self.h, C.byref(d), run_flags, nthreads, C.byref(r)), "orc_telegram_batch")
        out = result_from_c(r) if copy else (int(r.n), int(r.jsonl_len), int(r.n_links))
        self._last = (r, batch)  # the arrays stay valid until the next batch call (pending_edges reads them)
        return out

    # frontier -> validator hand-off (SURVEY 8f rank 3)
    def set_add(self, which, keys32, stamps=None):
        keys32 = np.ascontiguousarray(keys32, np.uint8).reshape(-1, 32)
        st = None if stamps is None else np.ascontiguousarray(stamps, np.int64)
        assert lib().orc_set_add(self.h, which, keys32.ctypes.data, None if st is None else st.ctypes.data, len(keys32)) == 0

    def set_now(self, now_sec):
        lib().orc_set_now(self.h, now_sec)

    def pending_edges(self, now_sec=0):
        r, batch = self._last
        cap = int(r.n_links)
        rows = np.zeros(cap, abi.EDGE)
        base = batch.recs.ctypes.data + batch.recs.dtype.fields["chan_idx"][1]
        m = lib().orc_pending_edges(self.h, C.byref(r), base, batch.recs.dtype.itemsize, now_sec, rows.ctypes.data, cap)
        return rows[: int(m)]

    def youtube(self, batch, run_flags=abi.RUN_JSONL | abi.RUN_LINKS, nthreads=1, copy=True):
        d = batch.descriptor()
        r = OrcResultC()
        _check(lib().orc_youtube_batch(self.h, C.byref(d), run_flags, nthreads, C.byref(r)), "orc_youtube_batch")
        out = result_from_c(r) if copy else (int(r.n), int(r.jsonl_len), int(r.n_links))
        lib().orc_result_free(C.byref(r))
        return out

    @staticmethod
    def key_join(a_keys, b_keys):
        a = np.ascontiguousarray(a_keys, dtype=np.int64).reshape(-1, 2)
        b = np.ascontiguousarray(b_keys, dtype=np.int64).reshape(-1, 2)
        out = np.full(len(b), -1, np.int64)
        lib().orc_key_join(a.ctypes.data, len(a), b.ctypes.data, len(b), out.ctypes.data)
        return out

    def generic(self, batch, run_flags=abi.RUN_JSONL, nthreads=1, copy=True):
        d = batch.descriptor()
        r = OrcResultC()
        _check(lib().orc_generic_batch(self.h, C.byref(d), run_flags, nthreads, C.byref(r)), "orc_generic_batch")
        out = result_from_c(r) if copy else (int(r.n), int(r.jsonl_len), int(r.n_links))
        lib().orc_result_free(C.byref(r))
        return out

    def frontier_insert(self, keys32: np.ndarray) -> np.ndarray:
        keys32 = np.ascontiguousarray(keys32, np.uint8).reshape(-1, 32)
        is_new = np.zeros(len(keys32), np.uint8)
        lib().orc_frontier_insert(self.h, keys32.ctypes.data, len(keys32), is_new.ctypes.data)
        return is_new

    def frontier_export(self) -> np.ndarray:
        n = int(lib().orc_frontier_size(self.h))
        out = np.zeros((n, 32), np.uint8)
        if n:
            lib().orc_frontier_export(self.h, out.ctypes.data, n)
        return out


# unit-level helpers -----------------------------------------------------------------------------
def utf16_offset_to_bytes(s: bytes, off: int, length: int) -> tuple[int, int]:
    a, b = C.c_int64(), C.c_int64()
    lib().orc_utf16_offset_to_bytes(s, len(s), off, length, C.byref(a), C.byref(b))
    return a.value, b.value


def filter_username(name: bytes) -> str:
    return abi.FU_REASONS[lib().orc_filter_username(name, len(name))]


def json_string(s: bytes) -> bytes:
    buf = C.create_string_buffer(len(s) * 6 + 2)
    n = lib().orc_json_string(s, len(s), buf)
    return buf.raw[:n]


def json_time(sec: int, nsec: int = 0, tz: int = 0) -> bytes:
    buf = C.create_string_buffer(64)
    n = lib().orc_json_time(sec, nsec, tz, buf)
    return buf.raw[:n]


def parse_iso8601_duration(s: bytes):
    v = C.c_int64()
    return v.value if lib().orc_parse_iso8601_duration(s, len(s), C.byref(v)) else None


def json_float_of_int64(v: int) -> bytes:
    buf = C.create_string_buffer(64)
    n = lib().orc_json_float_of_int64(v, buf)
    return buf.raw[:n]
