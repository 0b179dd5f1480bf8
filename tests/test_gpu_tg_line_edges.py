"""The Telegram Post line at its edges (tests/tg_line_corpus.py:make_line_edges): int64 / int32 extremes and digit-count
boundaries of every number, ids around the truncating msgno division, channel strings of every length and kind whose
escaped segments end on 16k - 1 / 16k / 16k + 1, the record's other strings on both sides of the lane rule, reaction maps
on both sides of the simple-map rule, outlinks around LANE_LINKS_MAX, channel tables of 1 to 9 000 rows, records past the
grid passes, and a page whose channel strings outgrow its result block.  The GPU lines must equal, byte for byte, the CPU
oracle and the restatement of the Go rules (go_rules.telegram_post_line); on the bulk pipeline the lane emitter must
write exactly the bytes the lane rule gives it (lane_left_bytes).  The CPU tests pin the oracle on the same records with
the restatement and check that the generator reaches every cell."""
import contextlib
import functools
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

import go_rules
from distributed_crawler_b200 import abi
from distributed_crawler_b200.pack import Channel, FormattedText, Message, pack_telegram
from helpers import ALL, TANDEM, assert_results_equal, no_page
from oracle.pyoracle import Oracle
from test_zones import ZONES
from tg_line_corpus import (ID_EDGES, PAGE_MAX_IN_BYTES, PAGE_MAX_RECS, chan_segments, concat_batches, line_cells,
                            line_edge_cells, lane_left_bytes, make_line_edges, pages, with_table)
from zone_oracle import ZonedOracle

SEEDS = (1, 2)
NY = ZONES["America/New_York"]
LABEL = (b'lab"<el>\xff\\\n' + "é中😀".encode() + b"\xe2\x80\xa8") * 30  # 750 bytes that need escaping
CLOCKS = {  # the engine / oracle configuration of each run; "new-york" runs time.Local as New York's transitions
    "utc": {}, "tz-12600": dict(tz_offset_sec=-12600), "tz+19800": dict(tz_offset_sec=19800),
    "tz+86340": dict(tz_offset_sec=86340), "tz-86340": dict(tz_offset_sec=-86340), "new-york": dict(zone=NY),
    "label": dict(tz_offset_sec=19800, crawl_label=LABEL, created_at_nsec=120_000_000, capture_nsec=5_000)}
ST = {"emitted": abi.ST_EMITTED, "skipped": abi.ST_SKIPPED, "failed": abi.ST_FAILED}
J = abi.RUN_JSONL


def _cfg(clock):
    return {k: v for k, v in CLOCKS[clock].items() if k != "zone"}


def oracle_for(clock):
    c = CLOCKS[clock]
    return ZonedOracle(c["zone"]) if "zone" in c else Oracle(**c)


def engine_for(clock):
    from distributed_crawler_b200.engine import Engine
    e = Engine(**_cfg(clock))
    if "zone" in CLOCKS[clock]:
        e.set_zone(*CLOCKS[clock]["zone"])
    return e


@functools.lru_cache(maxsize=None)
def corpus(seed):
    msgs, chans = make_line_edges(seed)
    return msgs, chans, pack_telegram(msgs, chans)


def restate(msgs, chans, clock):
    """[(status, line or None, links)] of go_rules.telegram_post_line"""
    c = CLOCKS[clock]
    kw = dict(crawl_label=c.get("crawl_label", b""), created=(1_750_000_000, c.get("created_at_nsec", 0)),
              capture=(1_750_000_000, c.get("capture_nsec", 123_456_789)), tz=c.get("tz_offset_sec", 0), zone=c.get("zone"))
    return [go_rules.telegram_post_line(m, chans[m.channel], **kw) for m in msgs]


@functools.lru_cache(maxsize=None)
def restated(seed, clock):
    """(status, line_off, sha256 of the JSONL) of the restated lines of a seed's corpus"""
    msgs, chans, _ = corpus(seed)
    return summary(restate(msgs, chans, clock))


def summary(rows):
    status = np.array([ST[st] for st, _, _ in rows], np.uint8)
    off = np.zeros(len(rows) + 1, np.uint64)
    off[1:] = np.cumsum([len(x or b"") for _, x, _ in rows], dtype=np.uint64)
    h = hashlib.sha256()
    for _, x, _ in rows:
        h.update(x or b"")
    return status, off, h.hexdigest()


def assert_equals_restatement(jsonl, status, line_off, want, label):
    """the JSONL of a whole corpus (pages concatenated) against the restatement's digest"""
    st, off, digest = want
    assert np.array_equal(status, st), f"{label}: status differs from the restatement"
    assert np.array_equal(line_off, off), f"{label}: line lengths differ from the restatement"
    assert hashlib.sha256(jsonl).hexdigest() == digest, f"{label}: lines differ from the restatement"


def left_bytes(msgs, chans, r):
    """lane_left_bytes of every record, with the outlinks of result r"""
    return np.array([lane_left_bytes(m, chans[m.channel], [x for x, _ in r.record_links(i)]) for i, m in enumerate(msgs)],
                    np.int64)


@functools.lru_cache(maxsize=None)
def corpus_left_bytes(seed):
    msgs, chans, batch = corpus(seed)
    return left_bytes(msgs, chans, Oracle().telegram(batch, abi.RUN_LINKS))


def lane_bytes_expected(r, left):
    """what the lane emitter writes of a result: the emitted lines less what the lane rule leaves to the others"""
    emitted = r.status == abi.ST_EMITTED
    return int((np.diff(r.line_off.astype(np.int64))[emitted] - left[emitted]).sum())


def _up(v, a):
    return (v + a - 1) // a * a


def page_holds(batch, ro, flags):
    """Whether the page kernel's result block holds a page-sized batch, from the oracle's result ro: the channel job's
    segments must fit 8 x the channel strings + 1 KB per row + 1 KB (run_tg_page's blob_cap), and the links and lines
    6 x the input + 3 KB per record + 64 KB (page_prepare's var_cap).  Otherwise the page hands the batch to the bulk
    pipeline (tg_page.cuh, ERR_PAGE_OVERFLOW)."""
    if not flags & J:
        return True
    chan_total = 0
    for c in batch.chans:
        o, t, nm, u = int(c["str_off"]), int(c["title_len"]), int(c["name_len"]), int(c["user_len"])
        cs = batch.chan_strs[o:o + t + nm + u].tobytes()
        ch = Channel(cs[:t], cs[t:t + nm], cs[t + nm:], int(c["member_count"]), int(c["post_count"]), int(c["view_count"]))
        chan_total += sum(_up(v, 16) for v in chan_segments(ch).values())
    blob_cap = 8 * batch.chan_strs.size + 1024 * len(batch.chans) + 1024
    var_cap = _up(6 * batch.input_bytes() + 3072 * batch.n + 65536, 256)
    links = _up(len(ro.links) * 36, 256) if flags & abi.RUN_LINKS else 0
    return chan_total <= blob_cap and links + ro.jsonl.size <= var_cap


# ---- GPU -------------------------------------------------------------------------------------------------------------
def _run_pages(seed, clock, flags, bulk):
    """the corpus in pages through one engine and one oracle, the frontier compared after every page; the lines of all
    pages are compared with the restatement, on the bulk pipeline the lane emitter's byte count with the lane rule, and
    on the page leg each page takes the one-launch path exactly when its result block holds it (page_holds)"""
    msgs, chans, batch = corpus(seed)
    o, e = oracle_for(clock), engine_for(clock)
    label = f"seed {seed}, {clock}, flags {flags:#x}, {'bulk' if bulk else 'page'}"
    jsonl, status, lens, launches = [], [], [], []
    try:
        for a, b in pages(msgs, chans):
            part = batch.slice(a, b)
            ro, rg = o.telegram(part, flags), e.telegram(part, flags)
            assert_results_equal(ro, rg, flags, f"{label}, records [{a}, {b})")
            if flags & abi.RUN_FRONTIER:
                assert np.array_equal(o.frontier_export(), e.frontier_export()), f"{label}: frontier differs after [{a}, {b})"
            if flags & J:
                jsonl.append(rg.jsonl.tobytes())
                lens.append(np.diff(rg.line_off.astype(np.int64)))
                if bulk:
                    assert rg.main_bytes_out == lane_bytes_expected(ro, corpus_left_bytes(seed)[a:b]), \
                        f"{label}, records [{a}, {b}): the lane emitter wrote other bytes than the lane rule gives it"
            if not bulk:
                holds = page_holds(part, ro, flags)
                assert (rg.gpu_launches == 1) == holds, \
                    f"{label}, records [{a}, {b}): {rg.gpu_launches} launches, the block {'holds' if holds else 'cannot hold'} the page"
            status.append(rg.status)
            launches.append(rg.gpu_launches)
    finally:
        e.close()
    if flags & J:
        off = np.zeros(len(msgs) + 1, np.uint64)
        off[1:] = np.cumsum(np.concatenate(lens), dtype=np.uint64)
        assert_equals_restatement(b"".join(jsonl), np.concatenate(status), off, restated(seed, clock), label)
    if bulk:
        assert min(launches) > 1
    else:
        assert launches.count(1) >= 1, f"{label}: no page took the one-launch path"


@pytest.mark.gpu
@pytest.mark.parametrize("clock", sorted(CLOCKS))
@pytest.mark.parametrize("seed", SEEDS)
def test_edges_in_pages(seed, clock):
    """page kernel (pages of at most 8 192 records and 4 MB of input) and bulk pipeline, ALL, RUN_JSONL and TANDEM"""
    for flags in (ALL, J, TANDEM):
        _run_pages(seed, clock, flags, bulk=False)
        with no_page():
            _run_pages(seed, clock, flags, bulk=True)


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [1, 33, 300, 9000])
def test_channel_tables(rows):
    """the records over channel tables of 1 .. 9 000 rows (9 000: more rows than a page takes, and than records)"""
    msgs, chans = with_table(*corpus(1)[:2], rows)
    want = summary(restate(msgs, chans, "utc"))
    batch = pack_telegram(msgs, chans)
    # the page leg: up to 300 rows every page of the corpus is a one-launch page; 9 000 rows are more than a page takes
    o, e = Oracle(), engine_for("utc")
    jsonl, status, lens = [], [], []
    try:
        for a, b in (pages(msgs, chans) if rows <= PAGE_MAX_RECS else [(0, len(msgs))]):
            part = batch.slice(a, b)
            ro, rg = o.telegram(part, ALL), e.telegram(part, ALL)
            label = f"{rows} channel rows, page leg, records [{a}, {b})"
            assert_results_equal(ro, rg, ALL, label)
            assert np.array_equal(o.frontier_export(), e.frontier_export()), label
            if rows <= PAGE_MAX_RECS:
                assert page_holds(part, ro, ALL) and rg.gpu_launches == 1, f"{label}: {rg.gpu_launches} launches"
            else:
                assert rg.gpu_launches > 1, label
            jsonl.append(rg.jsonl.tobytes())
            status.append(rg.status)
            lens.append(np.diff(rg.line_off.astype(np.int64)))
    finally:
        e.close()
    off = np.zeros(len(msgs) + 1, np.uint64)
    off[1:] = np.cumsum(np.concatenate(lens), dtype=np.uint64)
    assert_equals_restatement(b"".join(jsonl), np.concatenate(status), off, want, f"{rows} channel rows, page leg")
    # the bulk leg: the whole batch at once
    o, e = Oracle(), engine_for("utc")
    try:
        with no_page():
            ro, rg = o.telegram(batch, ALL), e.telegram(batch, ALL)
    finally:
        e.close()
    label = f"{rows} channel rows, bulk"
    assert rg.gpu_launches > 1, label
    assert_results_equal(ro, rg, ALL, label)
    assert_equals_restatement(rg.jsonl.tobytes(), rg.status, rg.line_off, want, label)
    assert rg.main_bytes_out == lane_bytes_expected(ro, left_bytes(msgs, chans, ro)), label


def _filler(n, first):
    """n small records over channel 0: a short text, every third with a link"""
    return [Message(text=FormattedText(b"filler %d t.me/fill%05d" % (first + i, (first + i) % 9000) if i % 3 == 0 else
                                       b"f%d" % (first + i)), id=(first + i) << 20, channel=0) for i in range(n)]


def spread_edges(n, boundaries, edges, width):
    """(n records, indices of the edge records): filler, with `width` edge records (dealt from `edges` in turn) on each
    side of every boundary, at the start and at the end"""
    msgs, k = [None] * n, 0
    spots = [0, n - 2 * width] + [b - width for b in boundaries if width <= b <= n - width]
    for s in spots:
        for i in range(s, s + 2 * width):
            if msgs[i] is None:
                msgs[i] = edges[k % len(edges)]
                k += 1
    at = [i for i, m in enumerate(msgs) if m is not None]
    return [m if m is not None else _filler(1, i)[0] for i, m in enumerate(msgs)], at


def light_edges(seed):
    """the edge records whose channel strings are at most 4 097 bytes (lines of at most a few hundred KB)"""
    msgs, chans, _ = corpus(seed)
    keep = [m for m in msgs if max(len(go_rules._bs(x)) for x in (chans[m.channel].title, chans[m.channel].name,
                                                                   chans[m.channel].username)) <= 4097]
    return keep, chans


def check_grid_passes(n, lane_rows, parse_rows):
    """n records through the bulk pipeline at the grids in force, with the edge records around every multiple of the
    lane emitter's (lane_rows) and the parse / size / clean-up kernels' (parse_rows) records per pass"""
    edges, chans = light_edges(1)
    bounds = sorted({k * lane_rows for k in range(1, n // lane_rows + 1)} | {k * parse_rows for k in range(1, n // parse_rows + 1)})
    msgs, at = spread_edges(n, bounds, edges, 12)
    batch = pack_telegram(msgs, chans)
    from distributed_crawler_b200.engine import Engine
    e, o = Engine(), Oracle()
    try:
        rg = e.telegram(batch, ALL)
        ro = o.telegram(batch, ALL)
        assert rg.gpu_launches > 1
        assert_results_equal(ro, rg, ALL, f"{n} records")
        assert np.array_equal(o.frontier_export(), e.frontier_export())
        assert rg.main_bytes_out == lane_bytes_expected(ro, left_bytes(msgs, chans, ro)), "the lane emitter wrote other bytes than the lane rule"
        kw = dict(created=(1_750_000_000, 0), capture=(1_750_000_000, 123_456_789))
        for i in at:
            st, line, _ = go_rules.telegram_post_line(msgs[i], chans[msgs[i].channel], **kw)
            assert rg.status[i] == ST[st] and rg.line(i) == (line or b""), f"record {i} differs from the restatement"
    finally:
        e.close()
        o.close()


@pytest.mark.gpu
def test_edges_past_the_grid_passes_of_one_cta_per_sm():
    """TGI_LANE_MULT=1 TGI_GRID_MULT=1 (read once per process, hence a child process): about 120 000 records, so the lane
    emitter (SMs x 256 records per pass) and the other kernels (SMs x 8) go round many times, with edge records at the
    start, around every pass boundary and at the end"""
    code = (
        "import sys; sys.path.insert(0, 'tests')\n"
        "import torch\n"
        "import test_gpu_tg_line_edges as t\n"
        "sms = torch.cuda.get_device_properties(0).multi_processor_count\n"
        "t.check_grid_passes(120_000, sms * 256, sms * 8)\n"
        "print('ok')\n")
    env = dict(os.environ, TGI_LANE_MULT="1", TGI_GRID_MULT="1", TGI_NO_PAGE="1")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=1200)
    assert p.returncode == 0 and "ok" in p.stdout, (p.stdout[-2000:], p.stderr[-3000:])


@pytest.mark.gpu
def test_edges_past_the_lane_emitters_first_pass():
    """the default grids: more than SMs x 24 x 256 records (811 008 on 132 SMs), edge records at the head, around the
    lane emitter's first pass boundary and at the tail, Corpus records between them"""
    import torch
    from distributed_crawler_b200.corpus import Corpus
    from distributed_crawler_b200.engine import Engine
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    first_pass = sms * 24 * 256
    edges, chans = light_edges(2)
    head, mid, tail = edges[:600], edges[600:1200], edges[1200:1800]
    gap = first_pass - len(head) - len(mid) // 2
    filler = [Corpus(gap, profile=2, first=0), Corpus(40_000, profile=2, first=gap)]  # they own the batches' memory
    parts = [pack_telegram(head, chans), filler[0].batch, pack_telegram(mid, chans), filler[1].batch, pack_telegram(tail, chans)]
    batch = concat_batches(parts)
    assert batch.n > first_pass
    starts = np.cumsum([0] + [p.n for p in parts])
    e, o = Engine(), Oracle()
    try:
        rg, ro = e.telegram(batch, ALL), o.telegram(batch, ALL, nthreads=8)
        assert_results_equal(ro, rg, ALL, "past the first pass")
        assert np.array_equal(o.frontier_export(), e.frontier_export())
    finally:
        e.close()
        o.close()
    kw = dict(created=(1_750_000_000, 0), capture=(1_750_000_000, 123_456_789))
    for part, at in ((head, starts[0]), (mid, starts[2]), (tail, starts[4])):
        for j, m in enumerate(part):
            st, line, _ = go_rules.telegram_post_line(m, chans[m.channel], **kw)
            assert rg.status[at + j] == ST[st] and rg.line(int(at + j)) == (line or b""), f"record {at + j} differs"
    assert starts[2] < first_pass < starts[3]


def outgrowing_page():
    """100 messages with links in a channel whose title is 65 535 '<': 78 MB of lines from 70 KB of input"""
    chans = [Channel(b"<" * 65535, "bigtitle", "bigtitle_user", 1, 2, 3)]
    msgs = [Message(text=FormattedText(b"m%d t.me/grow%04d t.me/grow%04d" % (i, i, i // 2)), id=i << 20, channel=0)
            for i in range(100)]
    return msgs, chans


@pytest.mark.gpu
def test_page_whose_channel_strings_outgrow_its_block(monkeypatch):
    """the page kernel's result block (6 x input + 3 KB per record) cannot hold these lines: the page hands the batch to
    the bulk pipeline by itself (no TGI_PAGE_VAR_CAP), whose lines equal the oracle's, and the frontier takes the new
    names once"""
    from distributed_crawler_b200.engine import Engine
    monkeypatch.delenv("TGI_PAGE_VAR_CAP", raising=False)  # the block keeps its own size ...
    monkeypatch.delenv("TGI_NO_PAGE", raising=False)       # ... and the page kernel is tried first
    msgs, chans = outgrowing_page()
    batch = pack_telegram(msgs, chans)
    e, o = Engine(), Oracle()
    try:
        for k in range(2):  # the second time every name is known
            rg, ro = e.telegram(batch, ALL), o.telegram(batch, ALL)
            assert not page_holds(batch, ro, ALL) and rg.gpu_launches > 1, "the page kernel cannot have held these lines"
            assert rg.jsonl_len > 75_000_000
            assert_results_equal(ro, rg, ALL, f"outgrowing page, call {k}")
            assert np.array_equal(o.frontier_export(), e.frontier_export())
            assert rg.n_new == ro.n_new == (100 if k == 0 else 0)
    finally:
        e.close()
        o.close()
    want = summary(restate(msgs, chans, "utc"))
    assert_equals_restatement(rg.jsonl.tobytes(), rg.status, rg.line_off, want, "outgrowing page")


@pytest.mark.gpu
def test_resident_path():
    """telegram_upload + telegram_run_resident on one page of edge records, with and without the page kernel"""
    from distributed_crawler_b200.engine import Engine
    msgs, chans, batch = corpus(1)
    a, b = pages(msgs, chans)[0]
    part = batch.slice(a, b)
    for bulk in (False, True):
        e, o = Engine(), Oracle()
        try:
            with no_page() if bulk else contextlib.nullcontext():
                e.telegram_upload(0, part)
                rg = e.telegram_run_resident(0, ALL, copy=True)
            ro = o.telegram(part, ALL)
            assert (rg.gpu_launches == 1) != bulk
            assert_results_equal(ro, rg, ALL, f"resident, {'bulk' if bulk else 'page'}")
            assert np.array_equal(o.frontier_export(), e.frontier_export())
        finally:
            e.close()
            o.close()


# ---- CPU -------------------------------------------------------------------------------------------------------------
def test_msgno_truncates_an_int64():
    """message.Id / 1048576 is an int64 division: exact above 2^53 and truncated toward zero"""
    for mid, want in (((1 << 62) + (1 << 20) - 1, 4398046511104), ((1 << 63) - 1, 8796093022207),
                      ((1 << 53) + (1 << 20) - 1, 8589934592), (-(1 << 63), -8796093022208), (-(1 << 20) + 1, 0),
                      (-(1 << 20) - 1, -1)):
        m = Message(text=FormattedText(b"x"), id=mid)
        _, line, _ = go_rules.telegram_post_line(m, Channel("T", "nm", "usr"))
        assert line.startswith(b'{"post_link":"https://t.me/usr/%d","channel_id":"-1001234567890","post_uid":"%d-nm",' % (want, want))
        assert Oracle(capture_sec=1_750_000_001, capture_nsec=0).telegram(pack_telegram([m], [Channel("T", "nm", "usr")]), J).line(0) == line
    assert go_rules.go_div(-7, 2) == -3 and go_rules.go_div(7, -2) == -3 and go_rules.go_div(-(1 << 63), -1) == 1 << 63


@pytest.mark.parametrize("clock", sorted(CLOCKS))
def test_edges_oracle_vs_independent_restatement(clock):
    """every byte, status and outlink list of every edge record: the oracle against go_rules.telegram_post_line"""
    msgs, chans, batch = corpus(1)
    r = oracle_for(clock).telegram(batch, J | abi.RUN_LINKS)
    rows = restate(msgs, chans, clock)
    for i, (st, line, links) in enumerate(rows):
        assert r.status[i] == ST[st], (clock, i)
        assert r.line(i) == (line or b""), (clock, i, msgs[i].id, msgs[i].channel)
        assert [x for x, _ in r.record_links(i)] == [go_rules._bs(x) for x in links], (clock, i)
    assert restated(1, clock)[2] == summary(rows)[2]


def test_outgrowing_page_oracle_vs_restatement():
    msgs, chans = outgrowing_page()
    r = Oracle().telegram(pack_telegram(msgs, chans), J)
    assert summary(restate(msgs, chans, "utc"))[2] == hashlib.sha256(r.jsonl.tobytes()).hexdigest()
    assert r.jsonl.size > 75_000_000 > 6 * pack_telegram(msgs, chans).input_bytes() + 3072 * 100 + 65536


@pytest.mark.parametrize("seed", SEEDS)
def test_edges_reach_every_cell(seed):
    msgs, chans, batch = corpus(seed)
    cells = line_cells(msgs, chans)
    missing = sorted(line_edge_cells() - cells, key=str)
    assert not missing, missing[:40]
    for a, b in pages(msgs, chans):
        assert b - a <= PAGE_MAX_RECS and batch.slice(a, b).input_bytes() <= PAGE_MAX_IN_BYTES
    assert len(pages(msgs, chans)) >= 2
    assert set(ID_EDGES) <= {m.id for m in msgs}
