"""Dapr storage-binding payloads (tgi_dapr_payloads, RUN_JSONL_DEVICE) against a restatement of
DaprStateManager.StorePost outside combine mode (state/daprstate.go:1141-1181): for every post, one InvokeBinding with
Operation "create", Data = base64.StdEncoding.EncodeToString(json.Marshal(post) + "\\n") (:1159) and Metadata
{<naming key>: <StorageRoot>/<CrawlID>/<CrawlExecutionID>/<channelID>/posts/<PostUID>.jsonl, "operation": "append"}
(:1150-1153, path format :2689-2698).  The lines are the oracle's; channelID and PostUID come from the packed batch."""
import base64
import ctypes as C
import os

import numpy as np
import pytest

from distributed_crawler_b200 import abi, sink
from distributed_crawler_b200.corpus import Corpus
from distributed_crawler_b200.engine import Engine, EngineError, _view, lib
from distributed_crawler_b200.pack import pack_telegram, pack_youtube
from helpers import J, JL, PREFIX, channel_ids, edge_batch, mem_available, on_slot, post_uid_tg
from oracle.pyoracle import Oracle
from yt_corpus import make_youtube

pytestmark = pytest.mark.gpu


def channel_and_uid(batch, yt: bool, i: int, ids):
    """channelID and PostUID of record i; ids = channel_ids(batch, yt)"""
    r = batch.recs[i]
    chan = ids[int(r["chan_idx"])]
    if yt:
        o = int(r["str_off"])
        return chan, batch.strs[o:o + int(r["id_len"])].tobytes()  # video.ID (youtube_crawler.go:701)
    return chan, post_uid_tg(int(r["id"]), chan)


def expected(batch, yt, ro, prefix, i, ids):
    """(Data, blob path) of record i, or (b"", b"") where the reference stores nothing"""
    if ro.status[i] != abi.ST_EMITTED:
        return b"", b""
    chan, uid = channel_and_uid(batch, yt, i, ids)
    return base64.b64encode(ro.line(i)), prefix + chan + b"/posts/" + uid + b".jsonl"


def check(batch, yt, ro, pay, prefix=PREFIX, label=""):
    assert pay.n == ro.n
    assert pay.data_off[0] == 0 and pay.path_off[0] == 0
    ids = channel_ids(batch, yt)
    for i in range(ro.n):
        d, p = expected(batch, yt, ro, prefix, i, ids)
        assert pay.data(i) == d, f"{label}: record {i}: data differs"
        assert pay.path(i) == p, f"{label}: record {i}: path {pay.path(i)!r} != {p!r}"
    assert pay.data_len == int(pay.data_off[-1]) and pay.path_len == int(pay.path_off[-1])


def run(e, batch, flags, yt=False, slot=0, prefix=PREFIX):
    """one batch on `slot`, its payloads, release"""
    return on_slot(e, batch, flags, yt, slot, lambda s: e.dapr_payloads(s, prefix))


def same_result(a, b):
    assert np.array_equal(a.status, b.status)
    assert np.array_equal(a.line_off, b.line_off)
    assert a.jsonl_len == b.jsonl_len
    assert np.array_equal(a.link_off, b.link_off) and np.array_equal(a.links, b.links)


def same_payloads(a, b):
    for k in ("data_off", "path_off", "data_blob", "path_blob"):
        assert np.array_equal(getattr(a, k), getattr(b, k)), k


@pytest.mark.parametrize("profile", [2, 3])
def test_telegram_bulk_with_and_without_jsonl_device(profile):
    c = Corpus(30000, profile=profile, first=4000)
    ro = Oracle().telegram(c.batch, J)
    e1, e2, e3 = Engine(), Engine(), Engine()
    r0, p0 = run(e1, c.batch, JL)
    r1, p1 = run(e2, c.batch, JL | abi.RUN_JSONL_DEVICE)
    r2, p2 = run(e3, c.batch, JL | abi.RUN_NO_D2H)
    assert r0.gpu_launches > 1 and r1.gpu_launches > 1
    same_result(r0, r1)
    assert r1.jsonl_on_device and r1.jsonl.size == 0 and not r0.jsonl_on_device
    assert np.array_equal(r0.jsonl, ro.jsonl)
    check(c.batch, False, ro, p0, label="copied")
    same_payloads(p0, p1)
    same_payloads(p0, p2)
    assert p1.gpu_launches >= 4 and p1.kernel_ms > 0
    for e in (e1, e2, e3):
        e.close()


@pytest.mark.parametrize("n", [100, 1000, 4000])
def test_telegram_pages(n):
    c = Corpus(n, profile=2, first=90 + n)
    ro = Oracle().telegram(c.batch, J)
    e = Engine()
    for flags in (JL, JL | abi.RUN_JSONL_DEVICE, J | abi.RUN_JSONL_DEVICE):
        r, pay = run(e, c.batch, flags)
        assert r.gpu_launches == 1, "a page-sized batch takes the one-launch path"
        assert (r.jsonl.size == 0) == bool(flags & abi.RUN_JSONL_DEVICE)
        check(c.batch, False, ro, pay, label=f"page {n} flags {flags:#x}")
    e.close()


def test_telegram_page_that_falls_back_to_bulk():
    c = Corpus(500, profile=2, first=31)
    ro = Oracle().telegram(c.batch, J)
    os.environ["TGI_PAGE_VAR_CAP"] = "65536"  # smaller than the page's JSONL: the bulk pipeline answers
    try:
        e = Engine()
        for flags in (JL, JL | abi.RUN_JSONL_DEVICE):
            r, pay = run(e, c.batch, flags)
            assert r.gpu_launches > 1
            check(c.batch, False, ro, pay, label="fallback")
        e.close()
    finally:
        del os.environ["TGI_PAGE_VAR_CAP"]


def test_youtube_bulk_and_pages():
    batch, _, _ = make_youtube(6000, seed=21)
    ro = Oracle().youtube(batch, J)
    assert (ro.status == abi.ST_NOLINE).any()  # the corpus holds unrepresentable dates: no binding call for them
    e = Engine()
    for flags in (J | abi.RUN_LINKS, J | abi.RUN_JSONL_DEVICE):
        r, pay = run(e, batch, flags, yt=True)
        assert r.gpu_launches > 1
        check(batch, True, ro, pay, label="youtube bulk")
    for k in range(0, 600, 50):  # Data API pages of 50 videos
        page = batch.slice(k, k + 50)
        rp = Oracle().youtube(page, J)
        for flags in (J | abi.RUN_LINKS | abi.RUN_FRONTIER, J | abi.RUN_JSONL_DEVICE):
            r, pay = run(e, page, flags, yt=True, slot=k // 50 % 3)
            assert r.gpu_launches == 1
            check(page, True, rp, pay, label=f"youtube page {k}")
    e.close()


@pytest.mark.parametrize("prefix", [b"", PREFIX, b"root/" + bytes(range(32, 127)) * 43 + b"/"])
def test_edge_corpus(prefix):
    batch = edge_batch()
    cfg = dict(min_post_date=1_600_000_000, crawl_label=b'c"l')
    ro = Oracle(**cfg).telegram(batch, J)
    st = set(int(x) for x in ro.status)
    assert {abi.ST_EMITTED, abi.ST_SKIPPED, abi.ST_FAILED} <= st
    lens = np.diff(ro.line_off)[ro.status == abi.ST_EMITTED]
    assert set(int(x) % 3 for x in lens) == {0, 1, 2}
    assert set(int(x) % 16 for x in ro.line_off[:-1][ro.status == abi.ST_EMITTED]) == set(range(16))
    assert lens.max() > 20000 and ((lens >= 2000) & (lens <= 20000)).sum() > 5
    e = Engine(**cfg)
    for flags in (JL, J | abi.RUN_JSONL_DEVICE):
        r, pay = run(e, batch, flags, prefix=prefix)
        check(batch, False, ro, pay, prefix, label=f"edge flags {flags:#x}")
        with pytest.MonkeyPatch.context() as mp:  # the same batch through the bulk pipeline
            mp.setenv("TGI_NO_PAGE", "1")
            r, pay = run(e, batch, flags, prefix=prefix)
            assert r.gpu_launches > 1
            check(batch, False, ro, pay, prefix, label=f"edge bulk flags {flags:#x}")
    e.close()


def test_noline_records_and_empty_batches():
    batch = edge_batch()
    cfg = dict(created_at_sec=400_000_000_000)  # year > 9999: json.Marshal fails for every post (TGI_ST_NOLINE)
    ro = Oracle(**cfg).telegram(batch, J)
    assert (ro.status == abi.ST_NOLINE).any()
    e = Engine(**cfg)
    r, pay = run(e, batch, J)
    check(batch, False, ro, pay, label="noline")
    e.close()
    e = Engine()
    for yt, empty in ((False, pack_telegram([])), (True, pack_youtube([]))):
        r, pay = run(e, empty, J | abi.RUN_JSONL_DEVICE, yt=yt)
        assert pay.n == 0 and list(pay.data_off) == [0] and list(pay.path_off) == [0] and pay.data_len == 0
    e.close()


def test_three_slots_in_flight():
    e = Engine()
    batches = [Corpus(20000, profile=2, first=1).batch, Corpus(3000, profile=3, first=50000).batch, edge_batch()]
    for s, b in enumerate(batches):
        e.telegram_submit(s, b, JL | abi.RUN_JSONL_DEVICE)
    pays = []
    for s in range(3):
        e.telegram_wait(s)
        pays.append(e.dapr_payloads(s, PREFIX))
    for s in range(3):
        e.release(s)
    for b, pay in zip(batches, pays):
        check(b, False, Oracle().telegram(b, J), pay, label="slots")
    e.close()


def _err(e, slot, prefix=PREFIX):
    out = abi.DaprPayloadsC()
    return lib().tgi_dapr_payloads(e.h, slot, prefix, 0 if prefix is None else len(prefix), C.byref(out))


def test_error_codes():
    from gm_corpus import make_generic
    e = Engine()
    c = Corpus(200, profile=2, first=3)
    assert _err(e, 0) == abi.E_STATE  # nothing has run on the slot
    e.telegram_submit(0, c.batch, abi.RUN_LINKS)
    e.telegram_wait(0)
    assert _err(e, 0) == abi.E_STATE  # no lines
    e.release(0)
    e.telegram_submit(1, c.batch, J)
    e.telegram_wait(1)
    assert _err(e, -1) == abi.E_ARG and _err(e, abi.SLOTS) == abi.E_ARG and _err(e, 1, None) == abi.E_ARG
    assert _err(e, 1) == abi.OK
    e.release(1)
    with pytest.raises(EngineError) as ei:
        e.telegram_submit(2, c.batch, abi.RUN_LINKS | abi.RUN_JSONL_DEVICE)
    assert ei.value.code == abi.E_ARG
    with pytest.raises(EngineError) as ei:
        e.telegram(c.batch, abi.RUN_JSONL_DEVICE)
    assert ei.value.code == abi.E_ARG
    g, _ = make_generic(50, seed=4)
    d = g.descriptor()
    r = abi.ResultC()
    assert lib().tgi_generic_batch(e.h, C.byref(d), J, C.byref(r)) == abi.OK
    assert _err(e, r.slot) == abi.E_STATE  # SavePost has no Dapr implementation
    lib().tgi_result_release(e.h, r.slot)
    e.close()


def store_post_restated(line: bytes, channel_id: bytes, post_uid: bytes, prefix: bytes, binding: str, naming_key: str):
    """DaprStateManager.StorePost, non-combine branch (daprstate.go:1141-1181) for one post whose json.Marshal succeeded:
    the storage path (:1150-1153 -> :2689-2698), the metadata and one InvokeBindingRequest (:1157-1166)"""
    storage_path = prefix + channel_id + b"/posts/" + post_uid + b".jsonl"
    metadata = {naming_key: storage_path, "operation": "append"}
    data = base64.b64encode(line)  # json.Marshal(post) + "\n", StdEncoding (:1159)
    return (binding, "create", data, metadata)


def test_store_posts_dapr_end_to_end():
    c = Corpus(5000, profile=2, first=777)
    ro = Oracle().telegram(c.batch, J)
    want = []
    ids = channel_ids(c.batch, False)
    for i in range(ro.n):
        if ro.status[i] == abi.ST_EMITTED:
            chan, uid = channel_and_uid(c.batch, False, i, ids)
            want.append(store_post_restated(ro.line(i), chan, uid, PREFIX, "telegramstorage", "blobName"))
    got = []
    e = Engine()
    _, pay = run(e, c.batch, J | abi.RUN_JSONL_DEVICE)
    assert sink.store_posts_dapr(lambda *req: got.append(req), pay, "telegramstorage", "blobName") == len(want)
    assert got == want
    e.close()


LARGE_N = 2_100_000  # config-2 messages: about 4.75 GB of JSONL
LARGE_HOST_BYTES = 24 << 30  # this test peaks at 17.6 GiB RSS (measured on an H100 host), plus room to spare


def test_batch_with_more_than_4gib_of_jsonl():
    """One batch whose JSONL passes 4 GiB, every payload compared.  The host holds the packed input, the library's pinned
    payloads (6.4 GB) and the oracle's lines (4.8 GB) once each: nothing is copied into Python objects but the small
    arrays the paths need, and the comparison reads both sides in place."""
    if mem_available() < LARGE_HOST_BYTES:
        pytest.skip(f"needs {LARGE_HOST_BYTES >> 30} GiB of available host memory")
    import resource
    from types import SimpleNamespace
    c = Corpus(LARGE_N, profile=2, first=10_000_000)
    b = c.batch
    small = SimpleNamespace(recs=b.recs.copy(), chans=b.chans.copy(), chan_strs=b.chan_strs.copy())
    e = Engine(max_records=LARGE_N)
    d = b.descriptor()
    r = abi.ResultC()
    assert lib().tgi_telegram_submit(e.h, 0, C.byref(d), J | abi.RUN_JSONL_DEVICE) == abi.OK
    assert lib().tgi_telegram_wait(e.h, 0, C.byref(r)) == abi.OK
    assert r.jsonl_len > (1 << 32) and not r.jsonl
    pay = abi.DaprPayloadsC()
    assert lib().tgi_dapr_payloads(e.h, 0, PREFIX, len(PREFIX), C.byref(pay)) == abi.OK
    assert pay.n == LARGE_N and pay.data_len > (1 << 32)
    o = Oracle()
    o.telegram(b, J, nthreads=os.cpu_count() or 1, copy=False)  # the oracle's arrays stay in C memory
    ro = o._last[0]
    del d, b
    c.close()
    n = LARGE_N
    o_status, o_off = _view(ro.status, n, np.uint8), _view(ro.line_off, n + 1, np.uint64)
    o_jsonl = _view(ro.jsonl, int(ro.jsonl_len), np.uint8)
    assert np.array_equal(o_off, _view(r.line_off, n + 1, np.uint64))
    assert np.array_equal(o_status, _view(r.status, n, np.uint8))
    do, po = _view(pay.data_off, n + 1, np.uint64), _view(pay.path_off, n + 1, np.uint64)
    data, path = _view(pay.data, int(pay.data_len), np.uint8), _view(pay.path, int(pay.path_len), np.uint8)
    assert do[0] == 0 and po[0] == 0 and do[n] == pay.data_len and po[n] == pay.path_len
    ids = channel_ids(small, False)
    for i in range(n):
        if o_status[i] != abi.ST_EMITTED:
            assert do[i + 1] == do[i] and po[i + 1] == po[i], i
            continue
        want = base64.b64encode(o_jsonl[int(o_off[i]):int(o_off[i + 1])].tobytes())
        assert data[int(do[i]):int(do[i + 1])].tobytes() == want, i
        chan, uid = channel_and_uid(small, False, i, ids)
        assert path[int(po[i]):int(po[i + 1])].tobytes() == PREFIX + chan + b"/posts/" + uid + b".jsonl", i
    print(f"peak RSS {resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20:.1f} GiB")
    lib().tgi_result_release(e.h, 0)
    o.close()
    e.close()
