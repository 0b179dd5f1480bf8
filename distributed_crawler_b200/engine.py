"""Python binding of libtgingest.so (ctypes) — the host mirror of the reference's plug points.

`Engine.telegram(batch, ...)` is the batch form of `crawl.MessageProcessor.ProcessMessage`
(crawl/runner.go:1010-1038) + `StorePost` byte production; `Engine.frontier_*` is the set behind
`seenInBatch` / `urlCache` / `DiscoveredChannels`.  The extension is REQUIRED: there is no eager or
CPU fallback — if libtgingest.so is missing or no GPU is visible this module raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtgingest.so")
_LIB = None


class EngineError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libtgingest error {code}: {msg}")
        self.code = code


EXPORTED_SYMBOLS = [
    "tgi_create", "tgi_destroy", "tgi_last_error", "tgi_get_stats", "tgi_set_clock",
    "tgi_telegram_submit", "tgi_telegram_wait", "tgi_telegram_batch", "tgi_youtube_submit",
    "tgi_youtube_wait", "tgi_youtube_batch", "tgi_generic_batch", "tgi_key_join", "tgi_plan_chunks", "tgi_result_release", "tgi_telegram_upload",
    "tgi_telegram_run_resident", "tgi_youtube_upload", "tgi_youtube_run_resident",
    "tgi_result_read_jsonl", "tgi_result_read_rows", "tgi_frontier_insert", "tgi_frontier_size", "tgi_frontier_export",
    "tgi_frontier_clear", "tgi_frontier_export_dev", "tgi_frontier_insert_dev", "tgi_frontier_sync",
    "tgi_filter_usernames", "tgi_acquire_staging", "tgi_release_staging", "tgi_comm_unique_id", "tgi_comm_init",
    "tgi_comm_destroy", "tgi_frontier_merge", "tgi_frontier_global_export", "tgi_merge_get_stats",
    "tgi_set_add", "tgi_set_clear", "tgi_set_size", "tgi_set_now", "tgi_pending_edges", "tgi_plan_channel_appends",
    "tgi_set_growth", "tgi_set_info", "tgi_dapr_payloads", "tgi_plan_chunks_carry", "tgi_combine_open", "tgi_combine_add",
    "tgi_combine_flush", "tgi_channel_appends", "tgi_set_zone", "tgi_state_code", "tgi_state_set", "tgi_state_add_layer",
    "tgi_state_update_page", "tgi_state_update_messages", "tgi_state_read_page", "tgi_state_render", "tgi_state_layer_map",
    "tgi_state_add_pages", "tgi_state_export", "tgi_state_page_begin", "tgi_state_page_end",
    "tgi_state_page_close", "tgi_state_id_seed", "tgi_state_discover", "tgi_state_next_layer", "tgi_state_pages_begin",
    "tgi_state_pages_end", "tgi_state_pages_close", "tgi_state_pending_edges", "tgi_channel_batch",
    "tgi_state_read_pages", "tgi_state_read_layer", "tgi_state_layers", "tgi_state_edge_sql",
    "tgi_state_walkback", "tgi_state_validator_walkback", "tgi_state_rw_lookups", "tgi_state_rw_step", "tgi_set_export",
]


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; "
                               "g.build()'` (nvcc, sm_90a). There is no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        vp, u64, u32, i32 = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int
        L.tgi_create.argtypes = [C.POINTER(abi.ConfigC), C.POINTER(vp)]
        L.tgi_destroy.argtypes = [vp]
        L.tgi_destroy.restype = None
        L.tgi_last_error.restype = C.c_char_p
        L.tgi_last_error.argtypes = [vp]
        L.tgi_get_stats.argtypes = [vp, C.POINTER(abi.StatsC)]
        L.tgi_get_stats.restype = None
        L.tgi_set_clock.argtypes = [vp, C.c_int64, C.c_int32, C.c_int64, C.c_int32]
        L.tgi_telegram_submit.argtypes = [vp, i32, C.POINTER(abi.TgBatchC), u32]
        L.tgi_telegram_wait.argtypes = [vp, i32, C.POINTER(abi.ResultC)]
        L.tgi_telegram_batch.argtypes = [vp, C.POINTER(abi.TgBatchC), u32, C.POINTER(abi.ResultC)]
        L.tgi_youtube_submit.argtypes = [vp, i32, C.POINTER(abi.YtBatchC), u32]
        L.tgi_youtube_wait.argtypes = [vp, i32, C.POINTER(abi.ResultC)]
        L.tgi_youtube_batch.argtypes = [vp, C.POINTER(abi.YtBatchC), u32, C.POINTER(abi.ResultC)]
        L.tgi_result_release.argtypes = [vp, i32]
        L.tgi_result_release.restype = None
        L.tgi_telegram_upload.argtypes = [vp, i32, C.POINTER(abi.TgBatchC)]
        L.tgi_telegram_run_resident.argtypes = [vp, i32, u32, C.POINTER(abi.ResultC)]
        L.tgi_generic_batch.argtypes = [vp, C.POINTER(abi.GmBatchC), u32, C.POINTER(abi.ResultC)]
        L.tgi_channel_batch.argtypes = [vp, C.POINTER(abi.ChBatchC), u32, C.POINTER(abi.ResultC)]
        L.tgi_key_join.argtypes = [vp, vp, C.c_uint64, vp, C.c_uint64, vp]
        L.tgi_plan_chunks.argtypes = [vp, C.c_uint64, C.c_uint64, C.c_uint64, vp, C.c_uint64, C.POINTER(C.c_uint64), vp]
        L.tgi_youtube_upload.argtypes = [vp, i32, C.POINTER(abi.YtBatchC)]
        L.tgi_youtube_run_resident.argtypes = [vp, i32, u32, C.POINTER(abi.ResultC)]
        L.tgi_result_read_jsonl.argtypes = [vp, i32, u64, u64, vp]
        L.tgi_result_read_rows.argtypes = [vp, i32, i32, u64, u64, vp]
        L.tgi_frontier_insert.argtypes = [vp, vp, u64, vp]
        L.tgi_frontier_size.argtypes = [vp, C.POINTER(u64)]
        L.tgi_frontier_export.argtypes = [vp, vp, u64, C.POINTER(u64)]
        L.tgi_frontier_clear.argtypes = [vp]
        L.tgi_frontier_export_dev.argtypes = [vp, vp, u64, u64, C.POINTER(u64)]
        L.tgi_frontier_insert_dev.argtypes = [vp, vp, u64, vp]
        L.tgi_frontier_sync.argtypes = [vp]
        L.tgi_filter_usernames.argtypes = [vp, vp, vp, u64, vp]
        L.tgi_acquire_staging.argtypes = [vp, u64, C.POINTER(vp)]
        L.tgi_release_staging.argtypes = [vp, vp]
        L.tgi_comm_unique_id.argtypes = [vp]
        L.tgi_comm_init.argtypes = [vp, vp, i32, i32]
        L.tgi_comm_destroy.argtypes = [vp]
        L.tgi_frontier_merge.argtypes = [vp, C.POINTER(u64), C.POINTER(u64)]
        L.tgi_frontier_global_export.argtypes = [vp, vp, u64, C.POINTER(u64)]
        L.tgi_merge_get_stats.argtypes = [vp, C.POINTER(abi.MergeStatsC)]
        L.tgi_set_add.argtypes = [vp, i32, vp, vp, u64]
        L.tgi_set_clear.argtypes = [vp, i32]
        L.tgi_set_size.argtypes = [vp, i32, C.POINTER(u64)]
        L.tgi_set_now.argtypes = [vp, C.c_int64]
        L.tgi_pending_edges.argtypes = [vp, i32, C.c_int64, vp, u64, C.POINTER(u64)]
        L.tgi_plan_channel_appends.argtypes = [vp, vp, u32, u64, vp, u64, C.POINTER(u64)]
        L.tgi_set_growth.argtypes = [vp, u64]
        L.tgi_set_info.argtypes = [vp, i32, C.POINTER(abi.SetInfoC)]
        L.tgi_dapr_payloads.argtypes = [vp, i32, C.c_char_p, u32, C.POINTER(abi.DaprPayloadsC)]
        L.tgi_plan_chunks_carry.argtypes = [vp, u64, u64, u64, u64, vp, u64, C.POINTER(u64), vp, C.POINTER(u64)]
        L.tgi_combine_open.argtypes = [vp, u64, u64, C.c_char_p, u32]
        L.tgi_combine_add.argtypes = [vp, i32, C.c_int64, C.POINTER(abi.CombinedC)]
        L.tgi_combine_flush.argtypes = [vp, C.c_int64, C.POINTER(abi.CombinedC)]
        L.tgi_channel_appends.argtypes = [vp, i32, C.POINTER(abi.ChannelAppendsC)]
        L.tgi_set_zone.argtypes = [vp, vp, vp, u32]
        L.tgi_state_code.argtypes = [vp, C.c_char_p, u32, C.POINTER(C.c_uint16)]
        L.tgi_state_set.argtypes = [vp, vp, u32, vp, u64, vp, u64, vp, u64, vp]
        L.tgi_state_add_layer.argtypes = [vp, vp, u64, vp, u64, C.c_int64, vp]
        L.tgi_state_update_page.argtypes = [vp, vp, vp, u64, vp, C.POINTER(u32)]
        L.tgi_state_update_messages.argtypes = [vp, vp, u64, C.POINTER(u64)]
        L.tgi_state_read_page.argtypes = [vp, u32, vp, u64, C.POINTER(u64)]
        L.tgi_state_render.argtypes = [vp, vp, u64, vp, u64, C.POINTER(abi.StateJsonC)]
        L.tgi_state_layer_map.argtypes = [vp, C.POINTER(abi.StateJsonC)]
        L.tgi_state_add_pages.argtypes = [vp, C.c_int64, vp, u64, vp, u64, vp]
        L.tgi_state_export.argtypes = [vp, i32, u64, C.POINTER(abi.StateExportC)]
        L.tgi_state_page_begin.argtypes = [vp, u32, vp, vp, u64, vp, u64, u32, C.POINTER(abi.StateTurnC)]
        L.tgi_state_page_end.argtypes = [vp, u32, i32, vp, u64, C.POINTER(u64)]
        L.tgi_state_page_close.argtypes = [vp, u32, vp, vp, u64, u32, C.POINTER(abi.StateJsonC)]
        L.tgi_state_pages_begin.argtypes = [vp, vp, u32, vp, vp, u64, vp, u64, vp, u32, C.POINTER(abi.StatePagesC)]
        L.tgi_state_pages_end.argtypes = [vp, u32, i32, u64, vp, vp, C.POINTER(abi.StateEndC)]
        L.tgi_state_pages_close.argtypes = [vp, vp, u32, vp, vp, u64, u32, C.POINTER(abi.StatePagesC)]
        L.tgi_state_id_seed.argtypes = [vp, u64]
        L.tgi_state_discover.argtypes = [vp, i32, vp, u32, u32, C.c_int64, i32, C.c_int64, C.POINTER(abi.StateAddedC)]
        L.tgi_state_next_layer.argtypes = [vp, C.c_int64, u32, C.c_int64, i32, C.c_int64, C.POINTER(abi.StateAddedC)]
        L.tgi_state_pending_edges.argtypes = [vp, i32, vp, u32, C.c_int64, C.POINTER(abi.StateEdgesC)]
        L.tgi_state_read_pages.argtypes = [vp, vp, u64, u32, C.POINTER(abi.StateReadC)]
        L.tgi_state_read_layer.argtypes = [vp, C.c_int64, i32, u32, C.POINTER(abi.StateReadC)]
        L.tgi_state_layers.argtypes = [vp, C.POINTER(abi.StateLayersC)]
        L.tgi_state_edge_sql.argtypes = [vp, C.c_char_p, u32, C.c_int64, i32, u32, C.POINTER(abi.StateEdgeSqlC)]
        L.tgi_state_walkback.argtypes = [vp, C.c_char_p, u32, C.c_int64, i32, u32, C.POINTER(abi.StateWalkbackC)]
        L.tgi_state_validator_walkback.argtypes = [vp, C.POINTER(abi.ClaimedBatchesC), C.c_int64, C.c_char_p, u32,
                                                   C.c_int64, i32, u32, C.POINTER(abi.StateValidatorWalkbackC)]
        L.tgi_state_rw_lookups.argtypes = [vp, i32, vp, u32, C.c_int64, C.POINTER(abi.StateRwLookupsC)]
        L.tgi_state_rw_step.argtypes = [vp, vp, u64, C.c_int64, C.c_char_p, u32, C.c_int64, i32, u32,
                                        C.POINTER(abi.StateRwStepC)]
        L.tgi_set_export.argtypes = [vp, i32, vp, vp, u64, C.POINTER(u64)]
        _LIB = L
    return _LIB


def _view(p, n, dt):
    if not n or not p:
        return np.zeros(0, dt)
    return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), (n * np.dtype(dt).itemsize,)).view(dt)


def _copy(p, n, dt):
    return _view(p, n, dt).copy()


class Result:
    """Host copy of a tgi_result."""

    def __init__(self, r: abi.ResultC, copy: bool = True):
        n = int(r.n)
        self.n = n
        self.jsonl_len = int(r.jsonl_len)
        self.n_links = int(r.n_links)
        self.n_new = int(r.n_new)
        self.frontier_size = int(r.frontier_size)
        self.kernel_ms = float(r.kernel_ms)
        self.parse_ms = float(r.parse_ms)
        self.emit_ms = float(r.emit_ms)
        self.emit_main_ms = float(r.emit_main_ms)
        self.frontier_ms = float(r.frontier_ms)
        self.var_bytes = int(r.var_bytes)
        self.main_bytes_out = int(r.main_bytes_out)
        self.main_bytes_in = int(r.main_bytes_in)
        self.has_links = bool(r.link_off)
        self.has_jsonl = bool(r.line_off)
        self.jsonl_on_device = self.has_jsonl and not r.jsonl and self.jsonl_len > 0  # RUN_JSONL_DEVICE: not copied
        self.gpu_launches = int(r.gpu_launches)
        self.slot = int(r.slot)
        if copy:
            self.status = _copy(r.status, n, np.uint8)
            self.jsonl = _copy(r.jsonl, self.jsonl_len, np.uint8)
            self.line_off = _copy(r.line_off, n + 1, np.uint64) if r.line_off else np.zeros(n + 1, np.uint64)
            self.link_off = _copy(r.link_off, n + 1, np.uint32) if r.link_off else np.zeros(n + 1, np.uint32)
            self.links = _copy(r.links, self.n_links, abi.LINK)

    def d2h_bytes(self) -> int:
        """bytes the library copied device -> pinned host for this result"""
        b = self.n + 80  # status + scalars
        if self.has_jsonl:
            b += (0 if self.jsonl_on_device else self.jsonl_len) + 8 * (self.n + 1)
        if self.has_links:
            b += 4 * (self.n + 1) + 36 * self.n_links
        return b

    def line(self, i: int) -> bytes:
        return self.jsonl[int(self.line_off[i]):int(self.line_off[i + 1])].tobytes()

    def record_links(self, i: int):
        out = []
        for k in range(int(self.link_off[i]), int(self.link_off[i + 1])):
            l = self.links[k]
            out.append((l["name"][: int(l["len"])].tobytes(), abi.SRC_NAMES[int(l["src"])]))
        return out


class DaprPayloads:
    """Host copy of a tgi_dapr_payloads_t: record i's binding Data is data(i), its blob path path(i); both are empty
    for records without a post."""

    def __init__(self, r: abi.DaprPayloadsC):
        n = int(r.n)
        self.n = n
        self.data_len = int(r.data_len)
        self.path_len = int(r.path_len)
        self.kernel_ms = float(r.kernel_ms)
        self.gpu_launches = int(r.gpu_launches)
        self.data_off = _copy(r.data_off, n + 1, np.uint64)
        self.path_off = _copy(r.path_off, n + 1, np.uint64)
        self.data_blob = _copy(r.data, self.data_len, np.uint8)
        self.path_blob = _copy(r.path, self.path_len, np.uint8)

    def data(self, i: int) -> bytes:
        return self.data_blob[int(self.data_off[i]):int(self.data_off[i + 1])].tobytes()

    def path(self, i: int) -> bytes:
        return self.path_blob[int(self.path_off[i]):int(self.path_off[i + 1])].tobytes()


class ChannelAppends:
    """A tgi_channel_appends_t: the lines of one result grouped by channel.  groups is an abi.CHANNEL_GROUP array
    (copied); data and order are views of the library's pinned memory, valid until the release or the next call on the
    slot.  Group k's bytes are group(k)."""

    def __init__(self, r: abi.ChannelAppendsC):
        self.n_groups = int(r.n_groups)
        self.data_len = int(r.data_len)
        self.kernel_ms = float(r.kernel_ms)
        self.gpu_launches = int(r.gpu_launches)
        self.groups = _copy(r.groups, self.n_groups, abi.CHANNEL_GROUP)
        self.n_lines = int(self.groups["n_lines"].sum())
        self.data = _view(r.data, self.data_len, np.uint8)
        self.order = _view(r.order, self.n_lines, np.uint64)

    def __len__(self):
        return self.n_groups

    def group(self, k: int) -> memoryview:
        g = self.groups[k]
        return memoryview(self.data[int(g["byte_off"]):int(g["byte_off"]) + int(g["byte_len"])])


class CombinedBlobs:
    """Host copy of a tgi_combined_t: the combined-posts blobs one combine call closed.  Blob j's binding Data is
    blob(j), its path path(j); blobs[j] holds its n_lines, raw_bytes and unix_nano."""

    def __init__(self, r: abi.CombinedC):
        k = int(r.n_blobs)
        self.n_blobs = k
        self.blobs = [{f: getattr(r.blobs[j], f) for f, _ in abi.CombinedBlobC._fields_} for j in range(k)]
        data_len = max((b["data_off"] + b["data_len"] for b in self.blobs), default=0)
        path_len = max((b["path_off"] + b["path_len"] for b in self.blobs), default=0)
        self.data_blob = _copy(r.data, data_len, np.uint8)
        self.path_blob = _copy(r.path, path_len, np.uint8)
        self.dropped = _copy(r.dropped, int(r.n_dropped), np.uint64)
        self.open_lines = int(r.open_lines)
        self.open_bytes = int(r.open_bytes)
        self.kernel_ms = float(r.kernel_ms)
        self.gpu_launches = int(r.gpu_launches)

    def __len__(self):
        return self.n_blobs

    def blob(self, j: int) -> bytes:
        b = self.blobs[j]
        return self.data_blob[b["data_off"]:b["data_off"] + b["data_len"]].tobytes()

    def path(self, j: int) -> bytes:
        b = self.blobs[j]
        return self.path_blob[b["path_off"]:b["path_off"] + b["path_len"]].tobytes()


class Engine:
    def __init__(self, cfg: abi.ConfigC | None = None, set_growth: int = 0, **kw):
        """set_growth: let every resident set grow up to this many keys (see set_growth); 0 keeps them fixed"""
        self.cfg = cfg or abi.make_config(**kw)
        self.h = C.c_void_p()
        rc = lib().tgi_create(C.byref(self.cfg), C.byref(self.h))
        if rc != 0:
            msg = lib().tgi_last_error(None).decode()
            self.h = None
            raise EngineError(rc, msg)
        self._keep = {}
        if set_growth:
            self.set_growth(set_growth)

    def _check(self, rc: int):
        if rc != 0:
            raise EngineError(rc, lib().tgi_last_error(self.h).decode())

    def close(self):
        if getattr(self, "h", None):
            lib().tgi_destroy(self.h)
            self.h = None

    __del__ = close

    def set_clock(self, created_at_sec, created_at_nsec, capture_sec, capture_nsec):
        self._check(lib().tgi_set_clock(self.h, created_at_sec, created_at_nsec, capture_sec, capture_nsec))

    def set_zone(self, starts, offsets):
        """the local zone as transitions (tgi_set_zone): instant t takes offsets[i] of the last starts[i] <= t; an empty
        table goes back to the fixed tz_offset_sec"""
        s = np.ascontiguousarray(starts, np.int64)
        o = np.ascontiguousarray(offsets, np.int32)
        if len(s) != len(o):
            raise ValueError("starts and offsets differ in length")
        self._check(lib().tgi_set_zone(self.h, s.ctypes.data if len(s) else None, o.ctypes.data if len(o) else None, len(s)))

    # --- Telegram -------------------------------------------------------------------------------
    def telegram(self, batch, run_flags=abi.RUN_JSONL | abi.RUN_LINKS, copy=True) -> Result:
        d = batch.descriptor()
        r = abi.ResultC()
        self._check(lib().tgi_telegram_batch(self.h, C.byref(d), run_flags, C.byref(r)))
        out = Result(r, copy)
        lib().tgi_result_release(self.h, r.slot)
        return out

    def telegram_submit(self, slot, batch, run_flags):
        d = batch.descriptor()
        self._keep[slot] = (batch, d)  # inputs must outlive the call
        self._check(lib().tgi_telegram_submit(self.h, slot, C.byref(d), run_flags))

    def telegram_wait(self, slot, copy=False) -> Result:
        r = abi.ResultC()
        self._check(lib().tgi_telegram_wait(self.h, slot, C.byref(r)))
        return Result(r, copy)

    def release(self, slot):
        lib().tgi_result_release(self.h, slot)

    def telegram_upload(self, slot, batch):
        d = batch.descriptor()
        self._check(lib().tgi_telegram_upload(self.h, slot, C.byref(d)))

    def telegram_run_resident(self, slot, run_flags, copy=False) -> Result:
        r = abi.ResultC()
        self._check(lib().tgi_telegram_run_resident(self.h, slot, run_flags, C.byref(r)))
        out = Result(r, copy)
        lib().tgi_result_release(self.h, slot)
        return out

    def read_jsonl(self, slot, off, length) -> bytes:
        buf = np.zeros(max(length, 1), np.uint8)
        self._check(lib().tgi_result_read_jsonl(self.h, slot, off, length, buf.ctypes.data))
        return buf[:length].tobytes()

    def read_rows(self, slot, which, first, count) -> np.ndarray:
        """rows [first, first+count) of the slot's last status / link offsets / link rows, read from the device"""
        out = np.zeros(max(count, 1), {abi.ROWS_STATUS: np.uint8, abi.ROWS_LINK_OFF: np.uint32, abi.ROWS_LINKS: abi.LINK}[which])
        self._check(lib().tgi_result_read_rows(self.h, slot, which, first, count, out.ctypes.data))
        return out[:count]

    # --- YouTube --------------------------------------------------------------------------------
    def youtube(self, batch, run_flags=abi.RUN_JSONL | abi.RUN_LINKS, copy=True) -> Result:
        d = batch.descriptor()
        r = abi.ResultC()
        self._check(lib().tgi_youtube_batch(self.h, C.byref(d), run_flags, C.byref(r)))
        out = Result(r, copy)
        lib().tgi_result_release(self.h, r.slot)
        return out

    def youtube_submit(self, slot, batch, run_flags):
        d = batch.descriptor()
        self._keep[slot] = (batch, d)
        self._check(lib().tgi_youtube_submit(self.h, slot, C.byref(d), run_flags))

    def youtube_wait(self, slot, copy=False) -> Result:
        r = abi.ResultC()
        self._check(lib().tgi_youtube_wait(self.h, slot, C.byref(r)))
        return Result(r, copy)

    def youtube_upload(self, slot, batch):
        d = batch.descriptor()
        self._check(lib().tgi_youtube_upload(self.h, slot, C.byref(d)))

    def youtube_run_resident(self, slot, run_flags, copy=False) -> Result:
        r = abi.ResultC()
        self._check(lib().tgi_youtube_run_resident(self.h, slot, run_flags, C.byref(r)))
        out = Result(r, copy)
        lib().tgi_result_release(self.h, slot)
        return out

    # --- library-owned pinned input staging (tgi_acquire_staging) --------------------------------
    def stage(self, batch):
        """A copy of `batch` whose arrays live in ONE pinned block owned by the library: what a packer that builds
        its arrays in tgi_acquire_staging memory produces.  Release with unstage()."""
        fields = batch.FIELDS
        sizes = [(getattr(batch, k).nbytes + 16 + 63) & ~63 for k in fields]  # 16 readable pad bytes behind every array
        block = C.c_void_p()
        self._check(lib().tgi_acquire_staging(self.h, sum(sizes) + 64, C.byref(block)))
        whole = np.ctypeslib.as_array(C.cast(block, C.POINTER(C.c_uint8)), (sum(sizes) + 64,))
        whole[:] = 0
        arrays, o = {}, 0
        for k, sz in zip(fields, sizes):
            a = getattr(batch, k)
            v = whole[o:o + a.nbytes].view(a.dtype)
            if a.ndim > 1:
                v = v.reshape(a.shape)
            v[...] = a
            arrays[k] = v
            o += sz
        out = type(batch)(**arrays)
        out._staging_block = block
        return out

    def unstage(self, staged):
        blk = getattr(staged, "_staging_block", None)
        if blk is not None:
            for k in staged.FIELDS:
                setattr(staged, k, None)
            self._check(lib().tgi_release_staging(self.h, blk))
            staged._staging_block = None

    # --- multi-GPU dedup-set merge (tgi_comm_*, tgi_frontier_merge) ------------------------------
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = (C.c_uint8 * 128)()
        rc = lib().tgi_comm_unique_id(buf)
        if rc != 0:
            raise EngineError(rc, lib().tgi_last_error(None).decode())
        return bytes(buf)

    def comm_init(self, uid: bytes, rank: int, nranks: int):
        buf = (C.c_uint8 * 128).from_buffer_copy(uid)
        self._check(lib().tgi_comm_init(self.h, buf, rank, nranks))

    def frontier_merge(self) -> tuple[int, int]:
        g, o = C.c_uint64(), C.c_uint64()
        self._check(lib().tgi_frontier_merge(self.h, C.byref(g), C.byref(o)))
        return g.value, o.value

    def frontier_global_export(self) -> np.ndarray:
        n = C.c_uint64()
        self._check(lib().tgi_frontier_global_export(self.h, None, 0, C.byref(n)))
        out = np.zeros((n.value, 32), np.uint8)
        self._check(lib().tgi_frontier_global_export(self.h, out.ctypes.data, n.value, C.byref(n)))
        return out

    def merge_stats(self) -> dict:
        s = abi.MergeStatsC()
        self._check(lib().tgi_merge_get_stats(self.h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in s._fields_}

    # --- frontier -> validator hand-off (SURVEY 8f rank 3) -------------------------------------
    def set_add(self, which: int, keys32: np.ndarray, stamps: np.ndarray | None = None):
        keys32 = np.ascontiguousarray(keys32, np.uint8).reshape(-1, 32)
        st = None if stamps is None else np.ascontiguousarray(stamps, np.int64)
        self._check(lib().tgi_set_add(self.h, which, keys32.ctypes.data, None if st is None else st.ctypes.data, len(keys32)))

    def set_clear(self, which: int):
        self._check(lib().tgi_set_clear(self.h, which))

    def set_size(self, which: int) -> int:
        n = C.c_uint64()
        self._check(lib().tgi_set_size(self.h, which, C.byref(n)))
        return n.value

    def set_export(self, which: int) -> tuple:
        """a caller-filled set's keys in first-occurrence order, [n, 32] uint8, and for abi.SET_INVALID their stamps
        (else None)"""
        n = C.c_uint64()
        self._check(lib().tgi_set_export(self.h, which, None, None, 0, C.byref(n)))
        keys = np.zeros((n.value, 32), np.uint8)
        stamps = np.zeros(n.value, np.int64) if which == abi.SET_INVALID else None
        self._check(lib().tgi_set_export(self.h, which, keys.ctypes.data, None if stamps is None else stamps.ctypes.data,
                                         n.value, C.byref(n)))
        return keys, stamps

    def set_now(self, now_sec: int):
        self._check(lib().tgi_set_now(self.h, now_sec))

    def set_growth(self, max_keys: int):
        """let the dedup set, the exclusion sets and this rank's partition grow on demand up to max_keys keys each
        (frontier_capacity becomes their initial size); 0 = fixed capacity.  Not while a job is in flight."""
        self._check(lib().tgi_set_growth(self.h, max_keys))

    def set_info(self, which: int) -> dict:
        """count, capacity, table_slots and grows of one set (abi.SET_FRONTIER / SET_INVALID / SET_DISCOVERED / SET_OWNED)"""
        s = abi.SetInfoC()
        self._check(lib().tgi_set_info(self.h, which, C.byref(s)))
        return {k: getattr(s, k) for k, _ in s._fields_}

    def pending_edges(self, slot: int, now_sec: int = 0) -> np.ndarray:
        """the new edges of the slot's last batch as packed pending_edges rows (call before release)"""
        n = C.c_uint64()
        self._check(lib().tgi_pending_edges(self.h, slot, now_sec, None, 0, C.byref(n)))
        rows = np.zeros(n.value, abi.EDGE)
        if n.value:
            self._check(lib().tgi_pending_edges(self.h, slot, now_sec, rows.ctypes.data, n.value, C.byref(n)))
        return rows

    def dapr_payloads(self, slot: int, prefix: bytes) -> "DaprPayloads":
        """host copies of the StorePost binding payloads of the slot's last Telegram / YouTube result (call before
        release): the base64 of every line, and its blob path prefix | channelID | /posts/ | PostUID | .jsonl; for a
        channel_batch result the StoreChannelData payloads, path prefix | url | /channel_data.jsonl"""
        out = abi.DaprPayloadsC()
        self._check(lib().tgi_dapr_payloads(self.h, slot, prefix, len(prefix), C.byref(out)))
        return DaprPayloads(out)

    def channel_appends(self, slot: int) -> ChannelAppends:
        """the lines of the slot's last Telegram / YouTube result grouped by channelID on the device (call before
        release): one group per posts.jsonl file, each group's lines in record order, groups by first line"""
        out = abi.ChannelAppendsC()
        self._check(lib().tgi_channel_appends(self.h, slot, C.byref(out)))
        return ChannelAppends(out)

    # --- combine mode: combined-posts blobs (SURVEY §8f rank 1) -----------------------------------
    def combine_open(self, trigger: int, hard_cap: int, prefix: bytes):
        """(re)configure the combiner: processBatches' trigger / hard cap and the blob path prefix"""
        self._check(lib().tgi_combine_open(self.h, trigger, hard_cap, prefix, len(prefix)))

    def combine_add(self, slot: int, unix_nano: int) -> CombinedBlobs:
        """pass the lines of the slot's last Telegram / YouTube result to the combiner; the blobs this closes"""
        out = abi.CombinedC()
        self._check(lib().tgi_combine_add(self.h, slot, unix_nano, C.byref(out)))
        return CombinedBlobs(out)

    def combine_flush(self, unix_nano: int) -> CombinedBlobs:
        """close the open group (Chunker shutdown)"""
        out = abi.CombinedC()
        self._check(lib().tgi_combine_flush(self.h, unix_nano, C.byref(out)))
        return CombinedBlobs(out)

    # --- generic client.Message -> sparse Post (SURVEY a12) -------------------------------------
    def generic(self, batch, run_flags=abi.RUN_JSONL, copy=True) -> Result:
        d = batch.descriptor()
        r = abi.ResultC()
        self._check(lib().tgi_generic_batch(self.h, C.byref(d), run_flags, C.byref(r)))
        out = Result(r, copy)
        lib().tgi_result_release(self.h, r.slot)
        return out

    # --- random-walk channel records -> ChannelData lines (StoreChannelData) ----------------------
    def channel_batch(self, batch, run_flags=abi.RUN_JSONL, copy=True) -> Result:
        """the ChannelData line of every record (pack.pack_channels).  The slot's result stays readable after the
        release: Engine.dapr_payloads(result.slot, prefix) and combine_add(result.slot, ns) take it until the next job on
        that slot"""
        d = batch.descriptor()
        r = abi.ResultC()
        self._check(lib().tgi_channel_batch(self.h, C.byref(d), run_flags, C.byref(r)))
        out = Result(r, copy)
        lib().tgi_result_release(self.h, r.slot)
        return out

    # --- message-status join (SURVEY 8f rank 2) -------------------------------------------------
    def key_join(self, a_keys: np.ndarray, b_keys: np.ndarray) -> np.ndarray:
        """for every (chat_id, message_id) row of b: index of the first equal row of a, or -1"""
        a = np.ascontiguousarray(a_keys, dtype=np.int64).reshape(-1, 2)
        b = np.ascontiguousarray(b_keys, dtype=np.int64).reshape(-1, 2)
        out = np.full(len(b), -1, np.int64)
        self._check(lib().tgi_key_join(self.h, a.ctypes.data, len(a), b.ctypes.data, len(b), out.ctypes.data))
        return out

    # --- crawl progress state (tgi_state_*): pages as state_pack dicts, rows as the library returns them ----------------
    def state_code(self, s: bytes) -> int:
        """the string-table code of a message status / platform (registered on first use)"""
        codes = self.__dict__.setdefault("_st_codes", {c.encode(): i for i, c in enumerate(abi.STATE_CODES)})
        if s not in codes:
            v = C.c_uint16()
            self._check(lib().tgi_state_code(self.h, s, len(s), C.byref(v)))
            codes[s] = v.value
        return codes[s]

    def _st_rows(self):
        return self.__dict__.setdefault("_st_row_of", {})

    def _st_note_rows(self, pages, rows):
        ids = self.__dict__.setdefault("_st_ids", [])
        for p, r in zip(pages, rows):
            if r != abi.STATE_NO_PAGE:
                self._st_rows()[p.get("id", b"")] = int(r)
                ids.extend([b""] * (int(r) + 1 - len(ids)))
                ids[int(r)] = p.get("id", b"")

    def state_set_arrays(self, layers, recs, strs, msgs) -> np.ndarray:
        """tgi_state_set on packed arrays (abi.STATE_LAYER, STATE_PAGE, bytes, STATE_MSG): the rows of the pages"""
        layers = np.ascontiguousarray(layers, abi.STATE_LAYER)
        recs = np.ascontiguousarray(recs, abi.STATE_PAGE)
        strs = np.ascontiguousarray(strs, np.uint8)
        msgs = np.ascontiguousarray(msgs, abi.STATE_MSG)
        rows = np.zeros(max(len(recs), 1), np.uint32)
        self._check(lib().tgi_state_set(self.h, layers.ctypes.data, len(layers), recs.ctypes.data, len(recs), strs.ctypes.data,
                                        len(strs), msgs.ctypes.data, len(msgs), rows.ctypes.data))
        return rows[:len(recs)]

    def state_set(self, layers) -> list[int]:
        """SetState: layers = [(depth, [page, ...]), ...]; a message's pageId names a page of the call"""
        from .state_pack import pack_pages
        pages = [p for _, ps in layers for p in ps]
        index = {p.get("id", b""): i for i, p in enumerate(pages)}

        def msg_page(pid, i):
            if pid not in index:
                raise ValueError(f"pageId {pid!r} names no page of the state")
            return index[pid]
        recs, strs, msgs = pack_pages(pages, self.state_code, msg_page)
        lay = np.array([(d, len(ps)) for d, ps in layers], abi.STATE_LAYER)
        rows = self.state_set_arrays(lay, recs, strs, msgs)
        self.__dict__["_st_row_of"], self.__dict__["_st_ids"] = {}, []
        self._st_note_rows(pages, rows)
        return [int(r) for r in rows]

    def state_add_layer(self, pages, max_pages: int = 0) -> list[int]:
        """AddLayer (pages without messages, ids and timestamps filled): each page's row, or abi.STATE_NO_PAGE"""
        from .state_pack import pack_pages
        recs, strs, _ = pack_pages(pages, self.state_code, lambda pid, i: i)  # messages are refused by the library
        rows = np.zeros(max(len(pages), 1), np.uint32)
        self._check(lib().tgi_state_add_layer(self.h, recs.ctypes.data, len(recs), strs.ctypes.data, len(strs), max_pages,
                                              rows.ctypes.data))
        self._st_note_rows(pages, rows[:len(pages)])
        return [int(r) for r in rows[:len(pages)]]

    def state_update_page(self, page) -> int:
        """UpdatePage: the page's row"""
        from .state_pack import pack_pages
        own = page.get("id", b"")

        def msg_page(pid, i):
            if pid == own:
                return abi.STATE_NO_PAGE
            if pid not in self._st_rows():
                raise ValueError(f"pageId {pid!r} names no page of the state")
            return self._st_rows()[pid]
        recs, strs, msgs = pack_pages([page], self.state_code, msg_page)
        row = C.c_uint32()
        self._check(lib().tgi_state_update_page(self.h, recs.ctypes.data, strs.ctypes.data, len(strs),
                                                msgs.ctypes.data if len(msgs) else None, C.byref(row)))
        self._st_note_rows([page], [row.value])
        return row.value

    def state_update_messages(self, updates) -> int:
        """UpdateMessage once per (row, chat_id, message_id, status bytes), in order; returns the updates skipped for
        naming no page (row abi.STATE_NO_PAGE)"""
        u = np.zeros(max(len(updates), 1), abi.STATE_UPDATE)
        for j, (row, chat, msg, st) in enumerate(updates):
            u[j] = (chat, msg, row, self.state_code(st), 0)
        return self.state_update_arrays(u[:len(updates)])

    def state_update_arrays(self, u) -> int:
        u = np.ascontiguousarray(u, abi.STATE_UPDATE)
        skipped = C.c_uint64()
        self._check(lib().tgi_state_update_messages(self.h, u.ctypes.data, len(u), C.byref(skipped)))
        return skipped.value

    def state_read_page_arrays(self, row: int) -> np.ndarray:
        n = C.c_uint64()
        self._check(lib().tgi_state_read_page(self.h, row, None, 0, C.byref(n)))
        out = np.zeros(max(n.value, 1), abi.STATE_MSG)
        self._check(lib().tgi_state_read_page(self.h, row, out.ctypes.data, n.value, C.byref(n)))
        return out[:n.value]

    def state_read_page(self, row: int) -> list[dict]:
        """GetPage(id).Messages of a row"""
        names = {v: k for k, v in self.__dict__.get("_st_codes", {}).items()}
        names.update({i: c.encode() for i, c in enumerate(abi.STATE_CODES)})
        ids = self.__dict__.get("_st_ids", [])
        return [{"chatId": int(m["chat_id"]), "messageId": int(m["message_id"]), "status": names[int(m["status"])],
                 "pageId": ids[int(m["page_id"])], "platform": names[int(m["platform"])]}
                for m in self.state_read_page_arrays(row)]

    # --- layer reads: GetPage / GetLayerByDepth of many rows, GetMaxDepth, FindIncompleteCrawl's page test ---------------
    def _st_read_arrays(self, out: abi.StateReadC) -> dict:
        n = int(out.n_pages)
        self.state_read_ms = float(out.kernel_ms)
        self.state_read_launches = int(out.gpu_launches)
        res = {"rows": _view(out.rows, n, np.uint32).copy(), "pages": _view(out.pages, n, abi.STATE_PAGE).copy(),
               "strs": C.string_at(out.strs, out.strs_len) if out.strs_len else b"",
               "msgs": _view(out.msgs, int(out.n_msgs), abi.STATE_MSG).copy() if out.msgs else None,
               "msg_first": _view(out.msg_first, n, np.uint64).copy() if out.msg_first else None,
               "select": _view(out.select, n, np.uint8).copy() if out.select else None,
               "n_selected": int(out.n_selected)}
        return res

    def state_read_pages_arrays(self, rows, flags: int = abi.READ_MESSAGES) -> dict:
        """tgi_state_read_pages as arrays: {"rows", "pages" (abi.STATE_PAGE, n_msgs = the list's length), "strs", "msgs"
        (abi.STATE_MSG) and "msg_first" (None without abi.READ_MESSAGES), "select" (None), "n_selected"}"""
        rows = np.ascontiguousarray(rows, np.uint32)
        out = abi.StateReadC()
        self._check(lib().tgi_state_read_pages(self.h, rows.ctypes.data if len(rows) else None, len(rows), flags,
                                               C.byref(out)))
        return self._st_read_arrays(out)

    def state_read_layer_arrays(self, depth: int, select: int = abi.SELECT_NONE, flags: int = abi.READ_MESSAGES) -> dict:
        """tgi_state_read_layer as arrays, as state_read_pages_arrays returns them ("select": 1 per processed page)"""
        out = abi.StateReadC()
        self._check(lib().tgi_state_read_layer(self.h, depth, select, flags, C.byref(out)))
        return self._st_read_arrays(out)

    def _st_pages(self, a: dict) -> list[dict]:
        """the read's pages as state_pack dicts: every string, depth, timestamp (offset None for time.Local) and, when
        the lists were read, "messages" (pageIds by the rows this engine has seen)"""
        names = {v: k for k, v in self.__dict__.get("_st_codes", {}).items()}
        names.update({i: c.encode() for i, c in enumerate(abi.STATE_CODES)})
        ids = self.__dict__.get("_st_ids", [])
        strs, pages = a["strs"], []
        for k, r in enumerate(a["pages"]):
            o, p = int(r["str_off"]), {}
            for f, name in enumerate(abi.STATE_STRINGS):
                ln = int(r["str_len"][f])
                p[name] = strs[o:o + ln]
                o += ln
            off = int(r["ts_off"])
            p["depth"] = int(r["depth"])
            p["timestamp"] = (int(r["ts_sec"]), int(r["ts_nsec"]), None if off == abi.STATE_TS_LOCAL else off)
            if a["msgs"] is not None:
                f0 = int(a["msg_first"][k])
                p["messages"] = [{"chatId": int(m["chat_id"]), "messageId": int(m["message_id"]),
                                  "status": names[int(m["status"])], "pageId": ids[int(m["page_id"])],
                                  "platform": names[int(m["platform"])]}
                                 for m in a["msgs"][f0:f0 + int(r["n_msgs"])]]
            pages.append(p)
        return pages

    def state_read_pages(self, rows, messages: bool = True) -> list[dict]:
        """GetPage of every row, in order (a row listed twice comes back twice)"""
        return self._st_pages(self.state_read_pages_arrays(rows, abi.READ_MESSAGES if messages else 0))

    def state_read_layer(self, depth: int, select: int = abi.SELECT_NONE, messages: bool = True):
        """GetLayerByDepth(depth) -> (pages, selected): selected = one bool per page under the runner's selection
        (abi.SELECT_*), None with abi.SELECT_NONE; the pages' rows are left in self.state_read_rows"""
        a = self.state_read_layer_arrays(depth, select, abi.READ_MESSAGES if messages else 0)
        self.state_read_rows = [int(r) for r in a["rows"]]
        return self._st_pages(a), None if a["select"] is None else [bool(x) for x in a["select"]]

    def state_layers(self) -> dict:
        """{"layers": [(depth, listed pages)] in ascending depth, "max_depth": GetMaxDepth or None for "no layers found",
        "n_incomplete": listed pages whose status is not "fetched"}"""
        out = abi.StateLayersC()
        self._check(lib().tgi_state_layers(self.h, C.byref(out)))
        n = int(out.n_layers)
        depth = _view(out.depth, n, np.int64).tolist() if n else []
        count = _view(out.n_pages, n, np.uint64).tolist() if n else []
        return {"layers": [(int(d), int(c)) for d, c in zip(depth, count)],
                "max_depth": int(out.max_depth) if out.has_max_depth else None, "n_incomplete": int(out.n_incomplete)}

    def state_render(self, metadata: bytes, last_updated: bytes, copy: bool = True):
        """json.Marshal(GetState()) with the shim's marshalled metadata and lastUpdated spliced in (copy=False: a view of
        the library's pinned bytes, valid until the next state call); the device time of the call is left in
        self.state_render_ms"""
        out = abi.StateJsonC()
        self._check(lib().tgi_state_render(self.h, metadata, len(metadata), last_updated, len(last_updated), C.byref(out)))
        self.state_render_ms = float(out.kernel_ms)
        self.state_render_launches = int(out.gpu_launches)
        return C.string_at(out.data, out.len) if copy else _view(out.data, out.len, np.uint8)

    def state_layer_map(self) -> bytes:
        """json.Marshal(layerMap) of DaprStateManager.SaveState; the device time of the call is left in
        self.state_layer_map_ms"""
        out = abi.StateJsonC()
        self._check(lib().tgi_state_layer_map(self.h, C.byref(out)))
        self.state_layer_map_ms = float(out.kernel_ms)
        self.state_layer_map_launches = int(out.gpu_launches)
        return C.string_at(out.data, out.len)

    def state_add_pages(self, depth: int, pages) -> list[int]:
        """Dapr's AddLayer once the caller has dropped the pages its urlCache holds: every page stored and appended to
        the layer `depth` (pages[0]'s depth before the filtering); each page's row"""
        from .state_pack import pack_pages
        recs, strs, _ = pack_pages(pages, self.state_code, lambda pid, i: i)  # messages are refused by the library
        rows = np.zeros(max(len(pages), 1), np.uint32)
        self._check(lib().tgi_state_add_pages(self.h, depth, recs.ctypes.data, len(recs), strs.ctypes.data, len(strs),
                                              rows.ctypes.data))
        self._st_note_rows(pages, rows[:len(pages)])
        return [int(r) for r in rows[:len(pages)]]

    def state_export(self, mode: int = abi.STATE_EXPORT_DAPR, chunk_bytes: int = abi.STATE_EXPORT_CHUNK_DEFAULT):
        """the pages as JSONL chunks: [(data, raw JSONL length), ...], data base64 (abi.STATE_EXPORT_DAPR,
        ExportPagesToBinding's chunks) or the raw JSONL (abi.STATE_EXPORT_LOCAL, one chunk).  A Dapr export of a layer
        map without pages raises EngineError with code abi.E_NOPAGES.  The device time is left in
        self.state_export_ms"""
        out = abi.StateExportC()
        self._check(lib().tgi_state_export(self.h, mode, chunk_bytes, C.byref(out)))
        self.state_export_ms = float(out.kernel_ms)
        self.state_export_launches = int(out.gpu_launches)
        self.state_export_pages = int(out.n_pages)
        return [(C.string_at(out.data + out.off[k], out.len[k]) if out.len[k] else b"", int(out.raw_len[k]))
                for k in range(out.n_chunks)]

    def state_page_begin(self, row: int, fetched, page=None, page_json: bool = False):
        """addNewMessages + resampleMarker + UpdatePage for a fetched page: fetched = (chat_id, message_id) pairs in
        fetch order, page = a state_pack dict without messages that replaces the row's fields (None: keep them).
        Returns (turn, work, page_json): work[i] indexes fetched for owner message i's discMessage; page_json is
        json.Marshal(page) when asked for, else None.  The device time of the call is left in self.state_turn_ms"""
        f = np.ascontiguousarray(fetched, np.int64).reshape(-1, 2)
        recs = strs = None
        if page is not None:
            from .state_pack import pack_pages
            if page.get("messages"):
                raise ValueError("the page's message list comes from the fetch")
            recs, strs, _ = pack_pages([page], self.state_code, lambda pid, i: i)
        out = abi.StateTurnC()
        self._check(lib().tgi_state_page_begin(
            self.h, row, recs.ctypes.data if recs is not None else None, strs.ctypes.data if strs is not None else None,
            len(strs) if strs is not None else 0, f.ctypes.data if len(f) else None, len(f),
            abi.TURN_PAGE_JSON if page_json else 0, C.byref(out)))
        self.state_turn_ms = float(out.kernel_ms)
        self.state_turn_launches = int(out.gpu_launches)
        work = np.ctypeslib.as_array(out.work, (out.n_work,)).copy() if out.n_work else np.zeros(0, np.uint32)
        return int(out.turn), work, C.string_at(out.page_json, out.page_json_len) if out.page_json else None

    def state_page_end(self, turn: int, n_done: int, slot: int = -1, status=None) -> int:
        """the loop's first n_done UpdateMessage calls of a turn, with the statuses of the slot's last Telegram result
        (slot >= 0) or of `status` (abi.ST_* per owner message, slot < 0); returns the messages appended"""
        st = None if status is None else np.ascontiguousarray(status, np.uint8)
        appended = C.c_uint64()
        self._check(lib().tgi_state_page_end(self.h, turn, slot, st.ctypes.data if st is not None and len(st) else None,
                                             n_done, C.byref(appended)))
        return appended.value

    def state_page_close(self, row: int, page, page_json: bool = False):
        """UpdatePage(*owner) after a turn: page = a state_pack dict without messages whose fields replace the row's;
        the row's list becomes its owner view (the last begin's owner messages with the end's hits) while it holds one.
        Returns json.Marshal(page) when asked for, else None.  The device time is left in self.state_close_ms"""
        from .state_pack import pack_pages
        if page.get("messages"):
            raise ValueError("the page's message list is the owner view")
        recs, strs, _ = pack_pages([page], self.state_code, lambda pid, i: i)
        out = abi.StateJsonC()
        self._check(lib().tgi_state_page_close(self.h, row, recs.ctypes.data, strs.ctypes.data, len(strs),
                                               abi.TURN_PAGE_JSON if page_json else 0, C.byref(out)))
        self.state_close_ms = float(out.kernel_ms)
        self.state_close_launches = int(out.gpu_launches)
        return C.string_at(out.data, out.len) if page_json else None

    # --- multi-page turns: the bookkeeping of many channels' pages in one call per step -----------------------------
    def _st_lines(self, out: abi.StatePagesC) -> list[bytes]:
        n = int(out.n_pages)
        off = np.ctypeslib.as_array(out.json_off, (n + 1,)).tolist()
        lines = C.string_at(out.page_json, off[n]) if off[n] else b""
        return [lines[off[k]:off[k + 1] - 1] for k in range(n)]  # each value without its '\n'

    def state_pages_begin(self, rows, fetched, pages=None, page_json: bool = False):
        """state_page_begin of every row in order, in one call: fetched = one list of (chat_id, message_id) pairs per
        row, pages = None or one state_pack dict per row.  Returns (turn, work, work_off, page_json): work indexes the
        concatenated fetched keys, page k's owner messages are work[work_off[k]:work_off[k+1]]; page_json is the list of
        json.Marshal(page) when asked for, else None.  The device time is left in self.state_pages_ms"""
        rows = np.ascontiguousarray(rows, np.uint32)
        parts = [np.ascontiguousarray(f, np.int64).reshape(-1, 2) for f in fetched]
        foff = np.zeros(len(parts) + 1, np.uint64)
        foff[1:] = np.cumsum([len(f) for f in parts])
        f = np.ascontiguousarray(np.concatenate(parts) if parts else np.zeros((0, 2), np.int64))
        recs = strs = None
        if pages is not None:
            from .state_pack import pack_pages
            if any(p.get("messages") for p in pages):
                raise ValueError("the pages' message lists come from the fetch")
            recs, strs, _ = pack_pages(pages, self.state_code, lambda pid, i: i)
        out = abi.StatePagesC()
        self._check(lib().tgi_state_pages_begin(
            self.h, rows.ctypes.data, len(rows), recs.ctypes.data if recs is not None else None,
            strs.ctypes.data if strs is not None else None, len(strs) if strs is not None else 0,
            f.ctypes.data if len(f) else None, len(f), foff.ctypes.data, abi.TURN_PAGE_JSON if page_json else 0,
            C.byref(out)))
        self.state_pages_ms = float(out.kernel_ms)
        self.state_pages_launches = int(out.gpu_launches)
        n = int(out.n_work)
        work = np.ctypeslib.as_array(out.work, (n,)).copy() if n else np.zeros(0, np.uint32)
        work_off = np.ctypeslib.as_array(out.work_off, (len(rows) + 1,)).copy()
        return int(out.turn), work, work_off, self._st_lines(out) if page_json else None

    def state_pages_end(self, turn: int, n_done=None, slot: int = -1, first: int = 0, status=None) -> int:
        """state_page_end of every page of a turn: n_done = None (every record) or one count per page; the statuses are
        records [first, first + n_work) of the slot's last Telegram result (slot >= 0) or `status` (abi.ST_* per owner
        message of the turn, slot < 0); returns the messages appended.  The device time is left in self.state_pages_ms"""
        st = None if status is None else np.ascontiguousarray(status, np.uint8)
        nd = None if n_done is None else np.ascontiguousarray(n_done, np.uint64)
        out = abi.StateEndC()
        self._check(lib().tgi_state_pages_end(self.h, turn, slot, first, st.ctypes.data if st is not None and len(st) else None,
                                              nd.ctypes.data if nd is not None else None, C.byref(out)))
        self.state_pages_ms = float(out.kernel_ms)
        self.state_pages_launches = int(out.gpu_launches)
        return int(out.appended)

    def state_pages_close(self, rows, pages, page_json: bool = False):
        """state_page_close of every row in order with its page (state_pack dicts without messages), in one call;
        returns the list of json.Marshal(page) when asked for, else None.  The device time is left in
        self.state_pages_ms"""
        from .state_pack import pack_pages
        if any(p.get("messages") for p in pages):
            raise ValueError("the pages' message lists are the owner views")
        rows = np.ascontiguousarray(rows, np.uint32)
        recs, strs, _ = pack_pages(pages, self.state_code, lambda pid, i: i)
        out = abi.StatePagesC()
        self._check(lib().tgi_state_pages_close(self.h, rows.ctypes.data, len(rows), recs.ctypes.data, strs.ctypes.data,
                                                len(strs), abi.TURN_PAGE_JSON if page_json else 0, C.byref(out)))
        self.state_pages_ms = float(out.kernel_ms)
        self.state_pages_launches = int(out.gpu_launches)
        return self._st_lines(out) if page_json else None

    # --- snowball discovery: outlinks of processed pages as next-layer pages ---------------------------------------
    def state_id_seed(self, seed: int):
        """the key of the page-id generator (Philox4x32-10); no page is added before it is set"""
        self._check(lib().tgi_state_id_seed(self.h, seed))

    def _st_added(self, out: abi.StateAddedC, json: bool) -> dict:
        n = int(out.n_added)
        rows = np.ctypeslib.as_array(out.rows, (n,)).tolist() if n else []
        blob = C.string_at(out.ids, 36 * n) if n else b""
        ids = [blob[36 * k:36 * k + 36] for k in range(n)]
        self._st_note_rows([{"id": i} for i in ids], rows)
        self.state_discover_ms = float(out.kernel_ms)
        self.state_discover_launches = int(out.gpu_launches)
        res = {"n_candidates": int(out.n_candidates), "rows": rows, "ids": ids, "page_json": None}
        if json:
            off = np.ctypeslib.as_array(out.json_off, (n + 1,)).tolist()
            lines = C.string_at(out.page_json, off[n]) if off[n] else b""
            res["page_json"] = [lines[off[k]:off[k + 1] - 1] for k in range(n)]  # each value without its '\n'
        return res

    def state_discover(self, slot: int, spans, flags: int = abi.DISCOVER_NOW, now=(0, 0), max_pages: int = 0) -> dict:
        """the outlinks of the slot's last Telegram result as next-layer pages: spans = (row, first, n_records, n_done)
        per owner page; flags = abi.DISCOVER_*; now = (sec, nsec) of the added pages.  Returns {"n_candidates", "rows",
        "ids", "page_json"} (page_json: json.Marshal of every added page with abi.DISCOVER_PAGE_JSON, else None).  The
        device time is left in self.state_discover_ms"""
        sp = np.zeros(max(len(spans), 1), abi.STATE_SPAN)
        for k, (row, first, n_records, n_done) in enumerate(spans):
            sp[k] = (row, 0, first, n_records, n_done)
        out = abi.StateAddedC()
        self._check(lib().tgi_state_discover(self.h, slot, sp.ctypes.data, len(spans), flags, now[0], now[1], max_pages,
                                             C.byref(out)))
        return self._st_added(out, bool(flags & abi.DISCOVER_PAGE_JSON))

    def state_next_layer(self, layer_depth: int, flags: int = 0, now=(0, 0), max_pages: int = 0) -> dict:
        """the layer end over the pending list (first occurrence per URL, Depth = layer_depth + 1, then AddLayer under
        abi.DISCOVER_DAPR's rules or Base's); returns what state_discover returns"""
        out = abi.StateAddedC()
        self._check(lib().tgi_state_next_layer(self.h, layer_depth, flags, now[0], now[1], max_pages, C.byref(out)))
        return self._st_added(out, bool(flags & abi.DISCOVER_PAGE_JSON))

    # --- tandem hand-off: every page's pending-edge batch --------------------------------------------------------
    def state_pending_edges(self, slot: int, spans, now_sec: int = 0) -> dict:
        """the pending edges of the slot's last Telegram result, deduplicated per page: spans = (row, first, n_records,
        n_done) per owner page, now_sec = the clock of the invalid set's TTL.  Returns {"edges" (abi.STATE_EDGE rows),
        "batches" (abi.STATE_EDGE_BATCH rows), "span_batch" (per span, abi.STATE_NO_BATCH without edges),
        "n_candidates"}.  The device time is left in self.state_edges_ms"""
        sp = np.zeros(max(len(spans), 1), abi.STATE_SPAN)
        for k, (row, first, n_records, n_done) in enumerate(spans):
            sp[k] = (row, 0, first, n_records, n_done)
        out = abi.StateEdgesC()
        self._check(lib().tgi_state_pending_edges(self.h, slot, sp.ctypes.data, len(spans), now_sec, C.byref(out)))
        self.state_edges_ms = float(out.kernel_ms)
        self.state_edges_launches = int(out.gpu_launches)
        return {"edges": _view(out.edges, int(out.n_edges), abi.STATE_EDGE).copy(),
                "batches": _view(out.batches, int(out.n_batches), abi.STATE_EDGE_BATCH).copy(),
                "span_batch": _view(out.span_batch, len(spans), np.uint32).copy(),
                "n_candidates": int(out.n_candidates)}

    def state_edge_sql(self, crawl_id: bytes, now=(0, 0), rows_per_stmt: int = 1) -> list:
        """the Postgres binding calls that store the last state_pending_edges (nothing but it since among the state
        calls): every batch insert, every edge insert, every batch close, rows_per_stmt rows per statement.  Returns
        [(kind (abi.SQL_*), rows, sql, params)]; the device time and launches are left in self.state_sql_ms and
        self.state_sql_launches"""
        out = abi.StateEdgeSqlC()
        self._check(lib().tgi_state_edge_sql(self.h, crawl_id, len(crawl_id), now[0], now[1], rows_per_stmt, C.byref(out)))
        self.state_sql_ms = float(out.kernel_ms)
        self.state_sql_launches = int(out.gpu_launches)
        return self._st_stmts(out)

    def state_walkback(self, crawl_id: bytes, now=(0, 0), rows_per_stmt: int = 1) -> tuple:
        """the forced walkbacks of the last state_pending_edges (nothing but it, state_edge_sql and this since among the
        state calls): a channel picked from the discovered set for every span without edges, and the Postgres binding
        calls that store them, every page_buffer insert then every edge_records insert.  Returns (walkbacks, stmts):
        per edge-less span {"span", "status" (abi.WALK_*), "draws", "url", "page_id", "sequence_id"}, and
        [(kind (abi.SQL_*), rows, sql, params)]; the device time and launches are left in self.state_walk_ms and
        self.state_walk_launches"""
        out = abi.StateWalkbackC()
        self._check(lib().tgi_state_walkback(self.h, crawl_id, len(crawl_id), now[0], now[1], rows_per_stmt, C.byref(out)))
        self.state_walk_ms = float(out.kernel_ms)
        self.state_walk_launches = int(out.gpu_launches)
        wb = _view(out.walkbacks, int(out.n_walkbacks), abi.STATE_WALKBACK_SPAN)
        walkbacks = [{"span": int(w["span"]), "status": int(w["status"]), "draws": int(w["draws"]),
                      "url": bytes(w["url"][:int(w["url_len"])]), "page_id": bytes(w["page_id"]),
                      "sequence_id": bytes(w["sequence_id"])} for w in wb]
        return walkbacks, self._st_stmts(out)

    def state_validator_walkback(self, batches, walkback_rate: int, crawl_id: bytes, now=(0, 0),
                                 rows_per_stmt: int = 1) -> tuple:
        """processWalkbackBatch for claimed batches (a list of dicts for state_pack.pack_claimed_batches, or its packed
        tuple): each batch's decision and pick, and the Postgres binding calls of the OK ones, every page_buffer insert,
        every edge_records insert, every complete, every stats upsert, every delete.  Returns (results, stmts): per
        batch {"status" (abi.WALK_*), "walkback", "rnd", "draws", "n_valid", "forward_edge" (None for a walkback),
        "url", "page_id", "sequence_id"}, and [(kind (abi.SQL_*), rows, sql, params)]; the device time and launches are
        left in self.state_vw_ms and self.state_vw_launches"""
        from .state_pack import pack_claimed_batches
        recs, edge_off, edges, blob = batches if isinstance(batches, tuple) else pack_claimed_batches(batches)
        recs, edges = np.ascontiguousarray(recs, abi.CLAIMED_BATCH), np.ascontiguousarray(edges, abi.CLAIMED_EDGE)
        edge_off, blob = np.ascontiguousarray(edge_off, np.uint64), np.ascontiguousarray(blob, np.uint8)
        cin = abi.ClaimedBatchesC(len(recs), 0, recs.ctypes.data, edge_off.ctypes.data, edges.ctypes.data, len(edges),
                                  blob.ctypes.data, len(blob))
        out = abi.StateValidatorWalkbackC()
        self._check(lib().tgi_state_validator_walkback(self.h, C.byref(cin), walkback_rate, crawl_id, len(crawl_id),
                                                       now[0], now[1], rows_per_stmt, C.byref(out)))
        self.state_vw_ms = float(out.kernel_ms)
        self.state_vw_launches = int(out.gpu_launches)
        res = _view(out.batches, int(out.n_batches), abi.STATE_VALIDATOR_BATCH)
        results = [{"status": int(r["status"]), "walkback": bool(r["walkback"]), "rnd": int(r["rnd"]),
                    "draws": int(r["draws"]), "n_valid": int(r["n_valid"]),
                    "forward_edge": None if r["forward_edge"] == abi.VW_NO_EDGE else int(r["forward_edge"]),
                    "url": bytes(r["url"][:int(r["url_len"])]), "page_id": bytes(r["page_id"]),
                    "sequence_id": bytes(r["sequence_id"])} for r in res]
        return results, self._st_stmts(out)

    # --- standard random walk: SearchPublicChat lookups, then the step ------------------------------------------------
    def state_rw_lookups(self, slot: int, spans, now_sec: int = 0) -> dict:
        """the SearchPublicChat calls of the standard random walk over the slot's last Telegram result: spans = (row,
        first, n_records, n_done) per owner page, now_sec = the clock of the invalid set's TTL.  Returns {"lookups"
        (abi.RW_LOOKUP rows), "span_candidates", "n_candidates"}.  The device time is left in self.state_rw_lookups_ms"""
        sp = np.zeros(max(len(spans), 1), abi.STATE_SPAN)
        for k, (row, first, n_records, n_done) in enumerate(spans):
            sp[k] = (row, 0, first, n_records, n_done)
        out = abi.StateRwLookupsC()
        self._check(lib().tgi_state_rw_lookups(self.h, slot, sp.ctypes.data, len(spans), now_sec, C.byref(out)))
        self.state_rw_lookups_ms = float(out.kernel_ms)
        self.state_rw_lookups_launches = int(out.gpu_launches)
        return {"lookups": _view(out.lookups, int(out.n_lookups), abi.RW_LOOKUP).copy(),
                "span_candidates": _view(out.span_candidates, len(spans), np.uint64).copy(),
                "n_candidates": int(out.n_candidates)}

    def state_rw_step(self, outcomes, walkback_rate: int, crawl_id: bytes, now=(0, 0), rows_per_stmt: int = 1) -> tuple:
        """the step of the last state_rw_lookups: outcomes = one (code (abi.RW_*), chat_id) per lookup row, or an
        abi.RW_OUTCOME array.  Returns (spans, stats, stmts): per span {"status" (abi.WALK_* / RW_RETIRED /
        RW_DEFERRED), "walkback", "rnd", "draws", "n_new", "forward" (None for a walkback), "url", "page_id",
        "sequence_id"}, {"hits", "misses"} per abi.SRC_NAMES, and [(kind (abi.SQL_*), rows, sql, params)]; the device
        time and launches are left in self.state_rw_ms and self.state_rw_launches"""
        if not isinstance(outcomes, np.ndarray):
            oc = np.zeros(len(outcomes), abi.RW_OUTCOME)
            for q, (code, chat_id) in enumerate(outcomes):
                oc[q] = (chat_id, code, 0)
            outcomes = oc
        outcomes = np.ascontiguousarray(outcomes, abi.RW_OUTCOME)
        out = abi.StateRwStepC()
        self._check(lib().tgi_state_rw_step(self.h, outcomes.ctypes.data if len(outcomes) else None, len(outcomes),
                                            walkback_rate, crawl_id, len(crawl_id), now[0], now[1], rows_per_stmt,
                                            C.byref(out)))
        self.state_rw_ms = float(out.kernel_ms)
        self.state_rw_launches = int(out.gpu_launches)
        res = _view(out.spans, int(out.n_spans), abi.RW_SPAN)
        spans = [{"status": int(r["status"]), "walkback": bool(r["walkback"]), "rnd": int(r["rnd"]),
                  "draws": int(r["draws"]), "n_new": int(r["n_new"]),
                  "forward": None if r["forward"] == abi.RW_NO_FORWARD else int(r["forward"]),
                  "url": bytes(r["url"][:int(r["url_len"])]), "page_id": bytes(r["page_id"]),
                  "sequence_id": bytes(r["sequence_id"])} for r in res]
        stats = {"hits": list(out.hits), "misses": list(out.misses)}
        return spans, stats, self._st_stmts(out)

    @staticmethod
    def _st_stmts(out) -> list:
        """the statement table of a state_edge_sql, state_walkback or state_validator_walkback result:
        [(kind, rows, sql, params)]"""
        st = _view(out.stmts, int(out.n_stmts), abi.STATE_EDGE_STMT)
        data = C.string_at(out.data, int(out.data_len)) if out.data_len else b""
        return [(int(k), int(r), data[int(so):int(so + sl)], data[int(po):int(po + pl)])
                for k, r, so, sl, po, pl in st.tolist()]

    # --- frontier -------------------------------------------------------------------------------
    def frontier_insert(self, keys32: np.ndarray) -> np.ndarray:
        keys32 = np.ascontiguousarray(keys32, np.uint8).reshape(-1, 32)
        is_new = np.zeros(len(keys32), np.uint8)
        self._check(lib().tgi_frontier_insert(self.h, keys32.ctypes.data, len(keys32), is_new.ctypes.data))
        return is_new

    def frontier_size(self) -> int:
        n = C.c_uint64()
        self._check(lib().tgi_frontier_size(self.h, C.byref(n)))
        return n.value

    def frontier_export(self) -> np.ndarray:
        n = self.frontier_size()
        out = np.zeros((n, 32), np.uint8)
        m = C.c_uint64()
        self._check(lib().tgi_frontier_export(self.h, out.ctypes.data, n, C.byref(m)))
        return out

    def frontier_clear(self):
        self._check(lib().tgi_frontier_clear(self.h))

    def filter_usernames(self, names: list[bytes]) -> list[str]:
        off = np.zeros(len(names) + 1, np.uint32)
        off[1:] = np.cumsum([len(x) for x in names])
        blob = np.frombuffer(b"".join(names) + b"\0" * 16, np.uint8).copy()
        reason = np.zeros(len(names), np.uint8)
        self._check(lib().tgi_filter_usernames(self.h, blob.ctypes.data, off.ctypes.data, len(names),
                                               reason.ctypes.data))
        return [abi.FU_REASONS[int(x)] for x in reason]

    def stats(self) -> abi.StatsC:
        s = abi.StatsC()
        lib().tgi_get_stats(self.h, C.byref(s))
        return s


def names_to_keys32(names: list[bytes]) -> np.ndarray:
    k = np.zeros((len(names), 32), np.uint8)
    for i, nm in enumerate(names):
        k[i, : len(nm)] = np.frombuffer(nm[:32], np.uint8)
    return k
