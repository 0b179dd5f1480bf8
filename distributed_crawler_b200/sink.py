"""Sinks for the lines of an engine result.

Combined-blob sink (SURVEY §8f rank 1): groups the JSONL lines of one engine result into the blobs the reference's
chunk combiner would upload as combined_<ns>.jsonl (chunk/main.go:292-421), without one file per post.

The grouping rule is libtgingest's tgi_plan_chunks (a restatement of Chunker.processBatches); the bytes of a group are
a contiguous slice of the result's JSONL blob (minus lines dropped for exceeding the hard cap).

Local sink: append_posts (LocalStateManager.StorePost) over a result's host JSONL, one append per run of consecutive
lines of a channel; append_posts_grouped, fed by Engine.channel_appends, one append per channel file, also when the
lines stayed on the device or the channels interleave.  Dapr sink: store_posts_dapr (DaprStateManager.StorePost outside
combine mode), fed by Engine.dapr_payloads; in combine mode upload_combined_dapr (UploadCombinedFile), fed by
Engine.combine_add / combine_flush, which group and encode the lines on the device across results."""
from __future__ import annotations

import ctypes as C
import os
import time

import numpy as np

from . import engine

TRIGGER_DEFAULT = 170 * 1024 * 1024  # the deployment's trigger / hard cap (SURVEY §8f)
HARD_CAP_DEFAULT = 200 * 1024 * 1024


def plan_chunks(line_off: np.ndarray, trigger: int = TRIGGER_DEFAULT, hard_cap: int = HARD_CAP_DEFAULT):
    """-> (groups [(begin, end)], dropped uint8[n])"""
    line_off = np.ascontiguousarray(line_off, dtype=np.uint64)
    n = len(line_off) - 1
    cap = max(n, 1)
    groups = np.zeros(2 * cap, np.uint64)
    dropped = np.zeros(max(n, 1), np.uint8)
    ng = C.c_uint64()
    rc = engine.lib().tgi_plan_chunks(line_off.ctypes.data, n, trigger, hard_cap, groups.ctypes.data, cap, C.byref(ng), dropped.ctypes.data)
    if rc:
        raise RuntimeError(f"tgi_plan_chunks: {rc}")
    g = groups[: 2 * ng.value].reshape(-1, 2)
    return [(int(a), int(b)) for a, b in g], dropped[:n]


def plan_chunks_carry(line_off: np.ndarray, open_bytes: int, trigger: int = TRIGGER_DEFAULT, hard_cap: int = HARD_CAP_DEFAULT):
    """the streaming form (tgi_plan_chunks_carry): the lines of one result continue a group of open_bytes bytes
    -> (closed groups [(begin, end)], dropped uint8[n], open bytes after the result)"""
    line_off = np.ascontiguousarray(line_off, dtype=np.uint64)
    n = len(line_off) - 1
    cap = max(n + 1, 1)
    groups = np.zeros(2 * cap, np.uint64)
    dropped = np.zeros(max(n, 1), np.uint8)
    ng, ob = C.c_uint64(), C.c_uint64()
    rc = engine.lib().tgi_plan_chunks_carry(line_off.ctypes.data, n, trigger, hard_cap, open_bytes, groups.ctypes.data, cap,
                                            C.byref(ng), dropped.ctypes.data, C.byref(ob))
    if rc:
        raise RuntimeError(f"tgi_plan_chunks_carry: {rc}")
    g = groups[: 2 * ng.value].reshape(-1, 2)
    return [(int(a), int(b)) for a, b in g], dropped[:n], ob.value


def write_combined(jsonl: bytes | np.ndarray, line_off: np.ndarray, combine_dir: str, trigger: int = TRIGGER_DEFAULT,
                   hard_cap: int = HARD_CAP_DEFAULT, now_ns=time.time_ns) -> list[str]:
    """Writes one combined_<ns>.jsonl per group (chunk/main.go:378-380 naming); returns the paths."""
    buf = memoryview(jsonl)
    groups, dropped = plan_chunks(line_off, trigger, hard_cap)
    paths = []
    for a, b in groups:
        path = os.path.join(combine_dir, "combined_%d.jsonl" % now_ns())
        with open(path, "wb") as f:
            if not dropped[a:b].any():
                f.write(buf[int(line_off[a]): int(line_off[b])])
            else:
                for i in range(a, b):
                    if not dropped[i]:
                        f.write(buf[int(line_off[i]): int(line_off[i + 1])])
        paths.append(path)
    return paths


def plan_channel_appends(line_off: np.ndarray, recs: np.ndarray) -> np.ndarray:
    """runs of consecutive lines of one channel (tgi_plan_channel_appends) -> abi.APPEND_RUN[]"""
    from . import abi
    line_off = np.ascontiguousarray(line_off, dtype=np.uint64)
    n = len(line_off) - 1
    runs = np.zeros(max(n, 1), abi.APPEND_RUN)
    ng = C.c_uint64()
    base = recs.ctypes.data + recs.dtype.fields["chan_idx"][1] if n else None
    rc = engine.lib().tgi_plan_channel_appends(line_off.ctypes.data, base, recs.dtype.itemsize, n, runs.ctypes.data, len(runs), C.byref(ng))
    if rc:
        raise RuntimeError(f"tgi_plan_channel_appends: {rc}")
    return runs[: ng.value]


def append_posts(jsonl: bytes | np.ndarray, line_off: np.ndarray, recs: np.ndarray, channel_ids: list[str], base_path: str, crawl_id: str) -> int:
    """LocalStateManager.StorePost for a whole result (state/storageproviders.go:275-298): <base>/<crawl>/<channel>/posts/
    posts.jsonl gets the channel's lines, one append per run instead of one open / append / close per post.  Returns the
    number of appends."""
    buf = memoryview(jsonl)
    runs = plan_channel_appends(line_off, recs)
    for r in runs:
        d = os.path.join(base_path, crawl_id, channel_ids[int(r["chan_idx"])], "posts")
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "posts.jsonl"), "ab") as f:
            f.write(buf[int(r["byte_begin"]): int(r["byte_end"])])
    return len(runs)


def go_clean(p: bytes) -> bytes:
    """Go's filepath.Clean on a Unix path: repeated separators become one, "." elements go, ".." removes the element
    before it (a rooted path drops a leading ".."), no trailing separator; the empty result is "." ("/" if rooted).
    Unlike os.path.normpath, a leading "//" becomes "/"."""
    rooted = p.startswith(b"/")
    out: list[bytes] = []
    for e in p.split(b"/"):
        if e in (b"", b"."):
            continue
        if e == b"..":
            if out and out[-1] != b"..":
                out.pop()
            elif not rooted:
                out.append(e)
            continue
        out.append(e)
    s = b"/".join(out)
    return (b"/" + s) if rooted else (s or b".")


def go_join(*elems: bytes) -> bytes:
    """Go's filepath.Join: the non-empty elements joined with "/", then Clean; "" when every element is empty"""
    parts = [e for e in elems if e]
    return go_clean(b"/".join(parts)) if parts else b""


def append_posts_grouped(engine, slot: int, channel_ids, base_path, crawl_id) -> int:
    """LocalStateManager.StorePost for the slot's last Telegram / YouTube result (state/storageproviders.go:275-298),
    one append per channel file: filepath.Join(base, crawl, channelID, "posts")/posts.jsonl gets the channel's lines in
    record order, grouped on the device by Engine.channel_appends (call before release).  channel_ids[row] is the
    channelID of channel row `row` (str or bytes; the group's lowest row stands for every row with the same bytes).
    Returns the number of appends."""
    enc = lambda x: x if isinstance(x, bytes) else os.fsencode(x)
    ca = engine.channel_appends(slot)
    base, crawl = enc(base_path), enc(crawl_id)
    for k in range(ca.n_groups):
        d = go_join(base, crawl, enc(channel_ids[int(ca.groups[k]["chan_idx"])]), b"posts")
        os.makedirs(d, exist_ok=True)
        with open(go_join(d, b"posts.jsonl"), "ab") as f:
            f.write(ca.group(k))
    return ca.n_groups


def store_posts_dapr(invoke, payloads, binding: str, naming_key: str) -> int:
    """DaprStateManager.StorePost outside combine mode (state/daprstate.go:1141-1181) for a whole result: one
    invoke(binding, "create", data, metadata) per post, in record order, with data = the base64 of its line and metadata
    {naming_key: blob path, "operation": "append"}; the path is raw bytes, as a Go string holds it.  `payloads` is Engine.dapr_payloads(slot, prefix); naming_key is
    fetchFileNamingComponent's answer for the binding, resolved once per crawl.  Records without a post are skipped.
    Returns the number of requests."""
    k = 0
    for i in range(payloads.n):
        if payloads.data_off[i + 1] == payloads.data_off[i]:
            continue
        invoke(binding, "create", payloads.data(i), {naming_key: payloads.path(i), "operation": "append"})
        k += 1
    return k


def upload_combined_dapr(invoke, blobs, binding: str, naming_key: str) -> int:
    """DaprStateManager.UploadCombinedFile (state/daprstate.go:3734-3777) for every blob a combine call closed: one
    invoke(binding, "create", data, {naming_key: path, "operation": "append"}) per blob, in order, with data = the base64
    of the combined lines and path = <prefix>combined-posts/combined_<ns>.jsonl.  `blobs` is Engine.combine_add /
    combine_flush.  Returns the number of requests."""
    for j in range(blobs.n_blobs):
        invoke(binding, "create", blobs.blob(j), {naming_key: blobs.path(j), "operation": "append"})
    return blobs.n_blobs
