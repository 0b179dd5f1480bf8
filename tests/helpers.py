"""Builders that mirror the helpers of the reference's own tests
(telegramhelper/channel_links_test.go:34-60: msgText, msgPhoto, ...)."""
from __future__ import annotations

import contextlib
import os

import numpy as np

from distributed_crawler_b200 import abi
from distributed_crawler_b200.pack import Channel, Comment, FormattedText, Message, TextEntity, pack_telegram


def ft(text, entities=()):
    if text is None:
        return None
    return FormattedText(text, [TextEntity(o, l, t, u) for (o, l, t, u) in entities])


def msg(content_type="messageText", text=None, entities=(), **kw):
    return Message(content_type=content_type, text=ft(text, entities), **kw)


def vector_message(v):
    return msg(v["content_type"], v["text"], [tuple(e) for e in v["entities"]])


def names(result, i=0):
    return sorted(n.decode() for n, _ in result.record_links(i))


def assert_results_equal(ro, rg, flags, label=""):
    assert np.array_equal(ro.status, rg.status), f"{label}: status differs"
    if flags & abi.RUN_JSONL:
        if not np.array_equal(ro.line_off, rg.line_off) or not np.array_equal(ro.jsonl, rg.jsonl):
            for i in range(ro.n):
                a, c = ro.line(i), rg.line(i)
                if a != c:
                    j = next((k for k in range(min(len(a), len(c))) if a[k] != c[k]), min(len(a), len(c)))
                    raise AssertionError(f"{label}: line {i} differs at byte {j}: "
                                         f"oracle={a[max(0, j - 60):j + 60]!r} gpu={c[max(0, j - 60):j + 60]!r}")
            raise AssertionError(f"{label}: offsets differ")
    if flags & abi.RUN_LINKS:
        assert np.array_equal(ro.link_off, rg.link_off), f"{label}: link_off differs"
        assert np.array_equal(ro.links, rg.links), f"{label}: links differ"
    if flags & abi.RUN_FRONTIER:
        assert ro.n_new == rg.n_new, f"{label}: n_new {ro.n_new} != {rg.n_new}"
        assert ro.frontier_size == rg.frontier_size, f"{label}: frontier size"


ALL = abi.RUN_JSONL | abi.RUN_LINKS | abi.RUN_FRONTIER | abi.RUN_SKIP_SELF
TANDEM = abi.RUN_LINKS | abi.RUN_FRONTIER | abi.RUN_FILTER | abi.RUN_SKIP_SELF


@contextlib.contextmanager
def no_page():
    """The ordinary multi-launch pipeline also for page-sized batches (the library reads TGI_NO_PAGE per call)."""
    os.environ["TGI_NO_PAGE"] = "1"
    try:
        yield
    finally:
        del os.environ["TGI_NO_PAGE"]


# ---- the result sinks (Dapr payloads, combine mode, local appends) ----------------------------------------------------
PREFIX = b"/data/crawls/crawl-7/exec-2024-01-01/"
J = abi.RUN_JSONL
JL = ALL
DEV = abi.RUN_JSONL_DEVICE


def channel_ids(batch, yt: bool) -> list[bytes]:
    """channelID of every channel row: Telegram the row's name (tdutils.go:725), YouTube the row's id
    (youtube_crawler.go:396)"""
    out = []
    for ch in batch.chans:
        o = int(ch["str_off"])
        if yt:
            out.append(batch.chan_strs[o:o + int(ch["id_len"])].tobytes())
        else:
            o += int(ch["title_len"])
            out.append(batch.chan_strs[o:o + int(ch["name_len"])].tobytes())
    return out


def post_uid_tg(msg_id: int, channel_name: bytes) -> bytes:
    """tdutils.go:416,636,1008: fmt.Sprintf("%d-%s", message.Id/1048576, channelName); Go's / truncates toward zero"""
    q = -((-msg_id) // 1048576) if msg_id < 0 else msg_id // 1048576
    return b"%d-" % q + channel_name


def edge_batch():
    """escaped, non-UTF-8 and empty channel names, ids of both signs around multiples of 2^20, lines of 2-20 KB,
    skipped (min_post_date 1 600 000 000) and failed records"""
    names = [b'a"b', b"<tag>&x", "канал-é✓".encode(), b"bad\xff\xfeutf8\xc0", b"", b"plain_name"]
    chans = [Channel(title="T%d" % k, name=nm, username="u%d" % k) for k, nm in enumerate(names)]
    ids = [-(1 << 20) + 1, -1, -(1 << 20), -(1 << 20) - 1, -(5 << 20) - 3, 0, 1 << 20, (1 << 20) - 1, (1 << 62) + 12345,
           -(1 << 62), 7 << 20]
    ms = []
    for k in range(420):
        long_ = k % 37 == 5
        text = ("x" * (2000 + 97 * k) + " t.me/longchan") if long_ else ("m%d " % k) + "é" * (k % 23) + "y" * (k % 17)
        comments = [Comment(text="c" * (200 + k), handle="h%d" % j, view_count=j) for j in range(40)] if k % 53 == 7 else []
        ms.append(msg("messageText", text, id=ids[k % len(ids)], channel=k % len(chans), date=1_700_000_000 + k,
                      reactions=[("r%03d" % j, j) for j in range(k % 7 * 60)], comments=comments,
                      panics=k % 41 == 3))
    ms[10].date = 1_500_000_000  # before min_post_date: skipped (tdutils.go:419-421)
    ms[11].date = 1_400_000_000
    return pack_telegram(ms, chans)


def mem_available() -> int:
    """the host's MemAvailable in bytes, 0 if unknown"""
    try:
        with open("/proc/meminfo") as f:
            for line in f:
                if line.startswith("MemAvailable:"):
                    return int(line.split()[1]) * 1024
    except OSError:
        pass
    return 0


def on_slot(e, batch, flags, yt, slot, call):
    """one batch on `slot`: submit, wait, call(slot), release; returns the batch's result (copied) and what call
    returned, which must not point into the slot's buffers"""
    (e.youtube_submit if yt else e.telegram_submit)(slot, batch, flags)
    try:
        r = (e.youtube_wait if yt else e.telegram_wait)(slot, copy=True)
        return r, call(slot)
    finally:
        e.release(slot)
