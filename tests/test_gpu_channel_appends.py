"""Local sink on the device (tgi_channel_appends, sink.append_posts_grouped) against a restatement of
LocalStateManager.StorePost (state/storageproviders.go:39-53, 275-298): for every emitted record, in record order,
MkdirAll(filepath.Join(base, crawl, channelID, "posts")) and one O_APPEND write of its line to posts.jsonl there.
Every group's bytes, line count, first record and lowest channel row, and `order`, are compared with what that loop
appends per file; the directory tree append_posts_grouped writes is compared byte for byte with the loop's tree."""
import ctypes as C
import dataclasses
import os
import posixpath

import numpy as np
import pytest

from distributed_crawler_b200 import abi, sink
from distributed_crawler_b200.corpus import Corpus, YtCorpus
from distributed_crawler_b200.engine import Engine, EngineError, lib
from distributed_crawler_b200.pack import Channel, pack_telegram, pack_youtube
from helpers import DEV, J, JL, channel_ids, mem_available, msg, no_page, on_slot
from oracle.pyoracle import Oracle
from yt_corpus import make_youtube, make_youtube_config4

pytestmark = pytest.mark.gpu
CRAWL = b"crawl-7"


def filepath_join(*elems: bytes) -> bytes:
    """Go's filepath.Join on Unix: non-empty elements joined by "/", then Clean.  posixpath.normpath is Clean except
    that it keeps exactly two leading slashes, which Clean reduces to one."""
    parts = [e for e in elems if e]
    if not parts:
        return b""
    p = posixpath.normpath(b"/".join(parts))
    return p[1:] if p.startswith(b"//") and not p.startswith(b"///") else p


def store_post_loop(batch, yt, ro):
    """StorePost per emitted record, in record order: channelID -> (appended bytes, records), in first-append order"""
    ids = channel_ids(batch, yt)
    files = {}
    for i in range(ro.n):
        if ro.status[i] != abi.ST_EMITTED:
            continue  # skipped, failed and TGI_ST_NOLINE records never reach StorePost
        line = ro.line(i)
        cid = ids[int(batch.recs[i]["chan_idx"])]
        data, recs = files.setdefault(cid, (bytearray(), []))
        data += line
        recs.append(i)
    return files


def check(batch, yt, ro, ca, label=""):
    ids = channel_ids(batch, yt)
    lowest = {}
    for row, cid in enumerate(ids):
        lowest.setdefault(cid, row)
    want = store_post_loop(batch, yt, ro)
    assert ca.n_groups == len(want), f"{label}: {ca.n_groups} groups, want {len(want)}"
    order, off = [], 0
    for k, (cid, (data, recs)) in enumerate(want.items()):
        g = ca.groups[k]
        assert int(g["chan_idx"]) == lowest[cid], f"{label}: group {k}: row {int(g['chan_idx'])}, want {lowest[cid]}"
        assert int(g["n_lines"]) == len(recs) and int(g["first_record"]) == recs[0], f"{label}: group {k}"
        assert int(g["byte_off"]) == off and int(g["byte_len"]) == len(data), f"{label}: group {k}"
        assert bytes(ca.group(k)) == bytes(data), f"{label}: group {k} ({cid!r}): bytes differ"
        order += recs
        off += len(data)
    assert ca.data_len == off and ca.order.tolist() == order, label


class Snapshot:
    """the outputs of one channel_appends call, copied out of the library's pinned memory"""

    def __init__(self, ca):
        self.__dict__.update(ca.__dict__)
        self.data, self.order = ca.data.copy(), ca.order.copy()
        self.group = lambda k: type(ca).group(self, k)


def run(e, batch, flags, yt=False, slot=0):
    """one batch on `slot`, its channel appends, release"""
    return on_slot(e, batch, flags, yt, slot, lambda s: Snapshot(e.channel_appends(s)))[1]


def tree(root: bytes) -> dict:
    out = {}
    for d, _, files in os.walk(root):
        for f in files:
            p = os.path.join(d, f)
            with open(p, "rb") as fh:
                out[os.path.relpath(p, root)] = fh.read()
    return out


def check_tree(tmp_path, e, batch, yt, ro, flags, slot=0):
    """the files append_posts_grouped writes == the files one StorePost per post writes"""
    a, b = os.fsencode(tmp_path / "per_post"), os.fsencode(tmp_path / "grouped")
    ids = channel_ids(batch, yt)
    for i in range(ro.n):
        if ro.status[i] == abi.ST_EMITTED:
            d = filepath_join(a, CRAWL, ids[int(batch.recs[i]["chan_idx"])], b"posts")
            os.makedirs(d, exist_ok=True)
            with open(filepath_join(d, b"posts.jsonl"), "ab") as f:
                f.write(ro.line(i))
    names = [x.decode("utf-8", "surrogateescape") for x in ids]
    _, k = on_slot(e, batch, flags, yt, slot, lambda s: sink.append_posts_grouped(e, s, names, b, CRAWL))
    want = tree(a)
    assert k == len(want) and tree(b) == want


@pytest.mark.parametrize("profile", [1, 2, 3])
def test_telegram_profiles_bulk_and_page(profile):
    e = Engine()
    for n, first in ((100, 7), (1000, 300), (6000, 12_000)):
        c = Corpus(n, profile=profile, first=first)
        ro = Oracle().telegram(c.batch, J)
        for flags in (JL, J | DEV):
            ca = run(e, c.batch, flags)
            check(c.batch, False, ro, ca, f"page {n} profile {profile} flags {flags:#x}")
            assert ca.gpu_launches > 1 and ca.kernel_ms > 0
            with no_page():
                check(c.batch, False, ro, run(e, c.batch, flags), f"bulk {n} profile {profile} flags {flags:#x}")
    e.close()


def interleaved_batch(n=700):
    """channels interleaved record by record; rows 0/2 and 1/5 name the same channel, rows 3/6 have empty names;
    skipped (before min_post_date) and failed records in between"""
    names = [b"alpha", b"beta_2", b"alpha", b"", "канал_é".encode(), b"beta_2", b"", b"bad\xff\xfe_name"]
    chans = [Channel(title="T%d" % k, name=nm, username="u%d" % k) for k, nm in enumerate(names)]
    ms = []
    for k in range(n):
        text = ("m%d " % k) + "é" * (k % 23) + "y" * (k % 300)
        ms.append(msg("messageText", text, id=(k + 1) << 20, channel=(k * 5) % len(chans), date=1_700_000_000 + k,
                      panics=k % 41 == 3))
    for k in (10, 11, 12, 40):
        ms[k].date = 1_500_000_000  # skipped (tdutils.go:419-421)
    return pack_telegram(ms, chans)


def test_interleaved_duplicate_and_empty_names(tmp_path):
    batch = interleaved_batch()
    cfg = dict(min_post_date=1_600_000_000)
    ro = Oracle(**cfg).telegram(batch, J)
    assert {abi.ST_EMITTED, abi.ST_SKIPPED, abi.ST_FAILED} <= set(int(x) for x in ro.status)
    e = Engine(**cfg)
    for flags in (JL, J | DEV):
        ca = run(e, batch, flags)
        check(batch, False, ro, ca, f"page flags {flags:#x}")
        assert ca.n_groups == 5  # alpha, beta_2, "", канал_é, bad...
        with no_page():
            check(batch, False, ro, run(e, batch, flags), f"bulk flags {flags:#x}")
    check_tree(tmp_path / "page", e, batch, False, ro, J | DEV)
    with no_page():
        check_tree(tmp_path / "bulk", e, batch, False, ro, J | DEV, slot=2)
    runs = sink.plan_channel_appends(ro.line_off, batch.recs)
    assert len(runs) > 100 * ca.n_groups  # the host planner only merges consecutive lines
    e.close()


def test_youtube_bulk_pages_and_duplicate_ids(tmp_path):
    e = Engine()
    b4, _, _ = make_youtube_config4(3000, seed=3)
    ro = Oracle().youtube(b4, J)
    for flags in (J | abi.RUN_LINKS, J | DEV):
        check(b4, True, ro, run(e, b4, flags, yt=True), f"config-4 bulk flags {flags:#x}")
    batch, vids, chans = make_youtube(600, seed=21)
    chans = list(chans)
    chans[5] = dataclasses.replace(chans[5], id=chans[1].id)  # two rows, one channel
    chans[9] = dataclasses.replace(chans[9], id=chans[1].id)
    batch = pack_youtube(vids, chans)
    ro = Oracle().youtube(batch, J)
    assert (ro.status == abi.ST_NOLINE).any()
    ca = run(e, batch, J | DEV, yt=True)
    check(batch, True, ro, ca, "youtube duplicate ids")
    assert ca.n_groups == len(set(channel_ids(batch, True)) & {channel_ids(batch, True)[int(r["chan_idx"])] for r in batch.recs})
    for k in range(0, 600, 50):  # Data API pages of 50 videos
        page = batch.slice(k, k + 50)
        rp = Oracle().youtube(page, J)
        for flags in (J | abi.RUN_LINKS | abi.RUN_FRONTIER, J | DEV):
            check(page, True, rp, run(e, page, flags, yt=True, slot=k // 50 % 3), f"youtube page {k}")
    check_tree(tmp_path, e, batch, True, ro, J | DEV, slot=1)
    e.close()


def test_no_line_at_all_and_empty_batches():
    batch = interleaved_batch(200)
    cfg = dict(created_at_sec=400_000_000_000)  # year > 9999: json.Marshal fails for every post (TGI_ST_NOLINE)
    ro = Oracle(**cfg).telegram(batch, J)
    assert (ro.status == abi.ST_NOLINE).any() and not (ro.status == abi.ST_EMITTED).any()  # the rest failed
    e = Engine(**cfg)
    for flags in (J, J | DEV):
        ca = run(e, batch, flags)
        assert ca.n_groups == 0 and ca.data_len == 0 and ca.order.size == 0
    e.close()
    e = Engine()
    for yt, empty in ((False, pack_telegram([])), (True, pack_youtube([]))):
        ca = run(e, empty, J | DEV, yt=yt)
        assert ca.n_groups == 0 and ca.data_len == 0 and ca.order.size == 0
    e.close()


def test_one_channel():
    e = Engine()
    c = Corpus(100, profile=2, first=0)  # 100 records: one channel row
    ro = Oracle().telegram(c.batch, J)
    ca = run(e, c.batch, J | DEV)
    check(c.batch, False, ro, ca, "one channel page")
    assert ca.n_groups == 1
    batch = pack_telegram([msg("messageText", "post %d " % k + "z" * (k % 97), id=k << 20) for k in range(3000)])
    ro = Oracle().telegram(batch, J)
    with no_page():
        ca = run(e, batch, JL | DEV)
    check(batch, False, ro, ca, "one channel bulk")
    assert ca.n_groups == 1 and int(ca.groups[0]["n_lines"]) == 3000
    e.close()


def test_more_than_65536_channels():
    n = 140_000
    c = Corpus(n, profile=1, first=10_000_000 - n)  # 100 000 channel rows
    assert len(c.batch.chans) == 100_000
    c.batch.recs["chan_idx"] = (np.arange(n, dtype=np.uint64) * 7919) % 100_000  # every row, interleaved
    ro = Oracle().telegram(c.batch, J, nthreads=os.cpu_count() or 1)
    e = Engine(max_records=n)
    for flags in (J, J | DEV):
        ca = run(e, c.batch, flags)
        assert ca.n_groups > 1 << 16  # channels whose every record was skipped or failed have no group
        check(c.batch, False, ro, ca, f"100k channels flags {flags:#x}")
    e.close()


def test_no_d2h_and_jsonl_device_results():
    c = Corpus(20000, profile=2, first=4000)
    ro = Oracle().telegram(c.batch, J)
    e = Engine()
    base = run(e, c.batch, JL)
    check(c.batch, False, ro, base, "copied")
    for flags in (JL | DEV, JL | abi.RUN_NO_D2H, J | abi.RUN_NO_D2H | DEV):
        ca = run(e, c.batch, flags)
        assert np.array_equal(ca.groups, base.groups) and np.array_equal(ca.data, base.data)
        assert np.array_equal(ca.order, base.order), f"flags {flags:#x}"
    page = Corpus(300, profile=3, first=77)
    rp = Oracle().telegram(page.batch, J)
    for flags in (J | abi.RUN_NO_D2H, J | DEV):
        check(page.batch, False, rp, run(e, page.batch, flags), f"page flags {flags:#x}")
    e.close()


def test_pages_on_three_slots():
    e = Engine()
    batches = [Corpus(100, profile=2, first=500).batch, interleaved_batch(400), Corpus(1000, profile=3, first=9000).batch]
    for s, b in enumerate(batches):
        e.telegram_submit(s, b, JL | DEV)
    got = []
    for s in range(3):
        e.telegram_wait(s)
        got.append(Snapshot(e.channel_appends(s)))
    for s in range(3):
        e.release(s)
    for b, ca in zip(batches, got):
        check(b, False, Oracle().telegram(b, J), ca, "slots")
    e.close()


def _call(e, slot):
    out = abi.ChannelAppendsC()
    return lib().tgi_channel_appends(e.h, slot, C.byref(out)), out


def test_slot_rules():
    from gm_corpus import make_generic
    e = Engine()
    c = Corpus(2000, profile=2, first=3)
    ro = Oracle().telegram(c.batch, J)
    assert _call(e, 0)[0] == abi.E_STATE  # nothing has run on the slot
    assert _call(e, -1)[0] == abi.E_ARG and _call(e, abi.SLOTS)[0] == abi.E_ARG
    assert lib().tgi_channel_appends(e.h, 0, None) == abi.E_ARG
    e.telegram_submit(0, c.batch, abi.RUN_LINKS)
    e.telegram_wait(0)
    assert _call(e, 0)[0] == abi.E_STATE  # run without TGI_RUN_JSONL
    e.release(0)
    # the batch's tgi_result is the same before and after the call, and the call works after the release
    d = c.batch.descriptor()
    r = abi.ResultC()
    assert lib().tgi_telegram_submit(e.h, 1, C.byref(d), JL) == abi.OK
    assert lib().tgi_telegram_wait(e.h, 1, C.byref(r)) == abi.OK
    before = bytes(r)
    arrays = lambda: (np.ctypeslib.as_array(C.cast(r.status, C.POINTER(C.c_uint8)), (r.n,)).copy(),
                      np.ctypeslib.as_array(C.cast(r.line_off, C.POINTER(C.c_uint64)), (r.n + 1,)).copy(),
                      np.ctypeslib.as_array(C.cast(r.jsonl, C.POINTER(C.c_uint8)), (r.jsonl_len,)).copy())
    a0 = arrays()
    rc, out = _call(e, 1)
    assert rc == abi.OK and out.n_groups > 0
    assert bytes(r) == before and all(np.array_equal(x, y) for x, y in zip(a0, arrays()))
    lib().tgi_result_release(e.h, 1)
    check(c.batch, False, ro, Snapshot(e.channel_appends(1)), "after release")
    g, _ = make_generic(50, seed=4)
    gd = g.descriptor()
    rg = abi.ResultC()
    assert lib().tgi_generic_batch(e.h, C.byref(gd), J, C.byref(rg)) == abi.OK
    assert _call(e, rg.slot)[0] == abi.E_STATE  # generic posts go to SavePost
    lib().tgi_result_release(e.h, rg.slot)
    with pytest.raises(EngineError) as ei:
        e.channel_appends(rg.slot)
    assert ei.value.code == abi.E_STATE
    e.close()


LARGE_N = 2_000_000  # config-4 videos over 1 000 channels: a new channel almost every record
LARGE_HOST_BYTES = 24 << 30


def test_config4_batch_of_two_million_videos():
    if mem_available() < LARGE_HOST_BYTES:
        pytest.skip(f"needs {LARGE_HOST_BYTES >> 30} GiB of available host memory")
    yc = YtCorpus(LARGE_N)
    b = yc.batch
    e = Engine(max_records=LARGE_N)
    e.youtube_submit(0, b, J | DEV)
    r = e.youtube_wait(0)
    assert r.jsonl_on_device
    ca = e.channel_appends(0)
    o = Oracle()
    ro = o.youtube(b, J, nthreads=os.cpu_count() or 1)
    ids = channel_ids(b, True)
    emitted = np.flatnonzero((ro.status == abi.ST_EMITTED) & (np.diff(ro.line_off) > 0))
    key = np.array([ids.index(x) for x in ids], np.int64)[b.recs["chan_idx"][emitted].astype(np.int64)]
    _, first = np.unique(key, return_index=True)
    rank = np.empty(key.max() + 1, np.int64)
    rank[key[np.sort(first)]] = np.arange(len(first))
    want_order = emitted[np.argsort(rank[key], kind="stable")]
    assert ca.n_groups == len(set(ids[int(x)] for x in b.recs["chan_idx"][emitted]))
    assert np.array_equal(ca.order, want_order)
    jsonl, off = ro.jsonl, ro.line_off
    want = b"".join(jsonl[int(off[i]):int(off[i + 1])].tobytes() for i in want_order)
    assert ca.data_len == len(want) and ca.data.tobytes() == want
    starts = np.cumsum(np.r_[0, ca.groups["n_lines"][:-1]]).astype(np.int64)
    assert np.array_equal(ca.groups["first_record"], want_order[starts])
    runs = sink.plan_channel_appends(ro.line_off, b.recs)
    print(f"{ca.n_groups} groups, {len(runs)} host runs, {len(emitted)} lines, kernel {ca.kernel_ms:.2f} ms")
    assert len(runs) > 0.9 * len(emitted)  # about one run per record
    e.release(0)
    o.close()
    e.close()
    yc.close()
