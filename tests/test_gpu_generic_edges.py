"""The generic client.Message -> sparse Post line at its edges (tests/gm_corpus.py:make_generic_edges): texts of every
length and kind at every strip boundary and start offset, 65 535-byte fields, int64 ends, reaction maps ordered by raw
bytes, the year bounds under every offset, nanoseconds, and the grid-stride loop of gm_size_kernel / gm_emit_kernel past
its first pass.  The GPU lines must equal, byte for byte, both the CPU oracle and the restatement of the Go rules
(go_rules.generic_post_line).  The CPU tests pin the oracle on the same records with the restatement, check that the
generator reaches every cell, and that the oracle refuses what the library refuses: a time whose nanoseconds are outside
[0, 1e9) and a zone offset of a day or more."""
import functools
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

import go_rules
from distributed_crawler_b200 import abi
from distributed_crawler_b200.pack import GenericMessage, pack_generic, pack_youtube
from gm_corpus import (NY_TRANSITIONS, generic_edge_cells, generic_edge_coverage, make_generic, make_generic_edges)
from helpers import assert_results_equal
from oracle.pyoracle import Oracle, OracleError
from test_zones import ZONES
from yt_corpus import make_youtube
from zone_oracle import ZonedOracle, go_json_time, go_offset

SEEDS = (1, 2, 3)
NY = ZONES["America/New_York"]
CLOCKS = {  # the engine / oracle configuration of each run; "zone" runs time.Local as New York's transitions
    "utc": {}, "tz-12600": dict(tz_offset_sec=-12600), "tz+19800": dict(tz_offset_sec=19800),
    "tz+86340": dict(tz_offset_sec=86340), "tz-86340": dict(tz_offset_sec=-86340), "new-york": dict(zone=NY),
    "trailing-zeros": dict(tz_offset_sec=19800, created_at_nsec=120_000_000, capture_nsec=5_000)}
BAD_NSEC = (-1, 10 ** 9, 2 ** 31 - 1)


def _cfg(clock):
    return {k: v for k, v in CLOCKS[clock].items() if k != "zone"}


def zone_derivable(msgs, zone):
    """ZonedOracle rewrites the lines of a UTC run: it cannot make a line for a record json.Marshal refuses in UTC but
    not in the zone (local 9999-12-31 from a UTC year 10000).  The zone runs leave those few records out."""
    return [m for m in msgs if go_json_time(m.ts_sec, m.ts_nsec, 0) or not go_json_time(m.ts_sec, m.ts_nsec, go_offset(zone, m.ts_sec))]


@functools.lru_cache(maxsize=None)
def edges(seed, clock):
    _, msgs = make_generic_edges(seed)
    if "zone" in CLOCKS[clock]:
        msgs = zone_derivable(msgs, CLOCKS[clock]["zone"])
    return pack_generic(msgs), msgs


def restated_lines(msgs, clock):
    c = CLOCKS[clock]
    kw = dict(created=(1_750_000_000, c.get("created_at_nsec", 0)), capture=(1_750_000_000, c.get("capture_nsec", 123_456_789)),
              tz=c.get("tz_offset_sec", 0), zone=c.get("zone"))
    return [go_rules.generic_post_line(m, **kw) for m in msgs]


def _summary(lines):
    """(status, line_off, sha256 of the JSONL) of restated lines (None = no line)"""
    status = np.array([abi.ST_NOLINE if x is None else abi.ST_EMITTED for x in lines], np.uint8)
    off = np.zeros(len(lines) + 1, np.uint64)
    off[1:] = np.cumsum([len(x or b"") for x in lines], dtype=np.uint64)
    h = hashlib.sha256()
    for x in lines:
        h.update(x or b"")
    return status, off, h.hexdigest()


@functools.lru_cache(maxsize=None)
def restated(seed, clock):
    return _summary(restated_lines(edges(seed, clock)[1], clock))


def oracle_for(clock):
    c = CLOCKS[clock]
    return ZonedOracle(c["zone"]) if "zone" in c else Oracle(**c)


def assert_equals_restatement(r, summary, label, msgs=None, clock=None):
    status, off, digest = summary
    ok = np.array_equal(r.status, status) and np.array_equal(r.line_off, off) and \
        hashlib.sha256(r.jsonl.tobytes()).hexdigest() == digest
    if not ok and msgs is not None:  # name the first record that differs
        for i, line in enumerate(restated_lines(msgs, clock)):
            assert r.line(i) == (line or b""), f"{label}: record {i} differs from the restatement"
    assert ok, f"{label}: differs from the restatement"


def mixed_with_filler(n, heavy, at):
    """n small records (make_generic) with the edge records `heavy` placed from index `at` on"""
    _, msgs = make_generic(n, seed=n % 97)
    msgs[at:at + len(heavy)] = heavy
    return msgs[:n]


def heavy_records(msgs):
    """the edge records that are not filler: long fields, big maps, edge times and nanoseconds"""
    def heavy(m):
        return (len(m.text) > 60 or len(m.id) > 20 or len(m.channel_id) > 20 or len(m.sender_name) > 20 or
                len(m.reactions) > 3 or not 1_600_000_000 <= m.ts_sec < 1_800_000_000)
    return [m for m in msgs if heavy(m)]


# ---- GPU -------------------------------------------------------------------------------------------------------------
def _engine_for(clock):
    from distributed_crawler_b200.engine import Engine
    e = Engine(**_cfg(clock))
    if "zone" in CLOCKS[clock]:
        e.set_zone(*CLOCKS[clock]["zone"])
    return e


@pytest.mark.gpu
@pytest.mark.parametrize("clock", sorted(CLOCKS))
@pytest.mark.parametrize("seed", SEEDS)
def test_edges_on_the_gpu(seed, clock):
    batch, msgs = edges(seed, clock)
    e = _engine_for(clock)
    try:
        rg = e.generic(batch)
    finally:
        e.close()
    assert rg.gpu_launches > 0
    assert_results_equal(oracle_for(clock).generic(batch), rg, abi.RUN_JSONL, f"seed {seed}, {clock}")
    assert_equals_restatement(rg, restated(seed, clock), f"seed {seed}, {clock}", msgs, clock)


@pytest.mark.gpu
def test_every_run_mode():
    """the status does not depend on the flags; TGI_RUN_FRONTIER is dropped (no links on this path), TGI_RUN_LINKS returns
    empty link arrays, TGI_RUN_JSONL_DEVICE keeps the lines on the device with the same offsets"""
    from distributed_crawler_b200.engine import Engine
    batch, msgs = edges(1, "utc")
    ro = Oracle().generic(batch)
    summary = restated(1, "utc")
    e = Engine()
    try:
        for flags in (abi.RUN_JSONL, abi.RUN_JSONL | abi.RUN_LINKS, abi.RUN_JSONL | abi.RUN_FRONTIER,
                      abi.RUN_JSONL | abi.RUN_LINKS | abi.RUN_FRONTIER | abi.RUN_FILTER | abi.RUN_SKIP_SELF | abi.RUN_SKIP_INVALID):
            rg = e.generic(batch, flags)
            assert_results_equal(ro, rg, abi.RUN_JSONL, f"flags {flags:#x}")
            assert_equals_restatement(rg, summary, f"flags {flags:#x}")
            assert rg.n_links == 0 and rg.n_new == 0 and rg.frontier_size == 0 and not rg.links.size
            if flags & abi.RUN_LINKS:
                assert rg.has_links and not rg.link_off.any()
        for flags in (0, abi.RUN_LINKS, abi.RUN_FRONTIER):
            rg = e.generic(batch, flags)
            assert np.array_equal(rg.status, ro.status) and rg.jsonl_len == 0 and not rg.has_jsonl, f"flags {flags:#x}"
            assert rg.n_links == 0 and not rg.link_off.any()
        rg = e.generic(batch, abi.RUN_JSONL | abi.RUN_JSONL_DEVICE)
        assert rg.jsonl_on_device and np.array_equal(rg.status, ro.status) and np.array_equal(rg.line_off, ro.line_off)
        rg = e.generic(batch, abi.RUN_JSONL | abi.RUN_NO_D2H, copy=False)
        assert rg.jsonl_len == int(ro.line_off[-1])
    finally:
        e.close()


@pytest.mark.gpu
def test_without_reaction_offsets():
    """react_off == NULL: every map is nil, whatever the reaction arrays hold"""
    from distributed_crawler_b200.engine import Engine
    _, msgs = edges(2, "utc")
    batch = pack_generic(msgs)
    assert batch.reacts.size > 5000
    batch.react_off = None
    bare = [GenericMessage(id=m.id, channel_id=m.channel_id, text=m.text, sender_name=m.sender_name, ts_sec=m.ts_sec,
                           ts_nsec=m.ts_nsec, views=m.views) for m in msgs]
    e = Engine()
    try:
        rg = e.generic(batch)
    finally:
        e.close()
    assert_results_equal(Oracle().generic(batch), rg, abi.RUN_JSONL, "react_off NULL")
    assert_equals_restatement(rg, _summary(restated_lines(bare, "utc")), "react_off NULL", bare, "utc")


@pytest.mark.gpu
def test_grid_stride_loop_past_its_first_pass():
    """SMs x 128 x 8 + 2 000 records: the grid is SMs x 128 CTAs of 8 warps, so records from SMs x 1024 on are a warp's
    second record.  The edge records sit on both sides of that boundary and at both ends of the batch."""
    import torch
    from distributed_crawler_b200.engine import Engine
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    per_pass = sms * 128 * 8
    heavy = heavy_records(edges(3, "utc")[1])
    msgs = mixed_with_filler(per_pass + 2000, heavy, per_pass - len(heavy) // 2)
    msgs[:40], msgs[-40:] = heavy[:40], heavy[-40:]
    batch = pack_generic(msgs)
    e = Engine(tz_offset_sec=-12600)
    try:
        rg = e.generic(batch)
    finally:
        e.close()
    ro = Oracle(tz_offset_sec=-12600).generic(batch)
    assert_results_equal(ro, rg, abi.RUN_JSONL, "two passes")
    lo, hi = per_pass - len(heavy) // 2 - 50, per_pass + len(heavy) // 2 + 50
    for i in list(range(60)) + list(range(lo, hi)) + list(range(len(msgs) - 60, len(msgs))):
        line = go_rules.generic_post_line(msgs[i], created=(1_750_000_000, 0), capture=(1_750_000_000, 123_456_789), tz=-12600)
        assert rg.line(i) == (line or b"") and rg.status[i] == (abi.ST_EMITTED if line else abi.ST_NOLINE), i


@pytest.mark.gpu
def test_edges_with_a_grid_of_one_cta_per_sm():
    """TGI_GRID_MULT=1 (read once per process, hence a child process): the edge batch takes many passes of the loop"""
    code = (
        "import sys; sys.path.insert(0, 'tests')\n"
        "from distributed_crawler_b200 import abi\n"
        "from distributed_crawler_b200.engine import Engine\n"
        "from oracle.pyoracle import Oracle\n"
        "from helpers import assert_results_equal\n"
        "import test_gpu_generic_edges as t\n"
        "for seed in (1, 2, 3):\n"
        "    for clock in ('utc', 'tz-86340'):\n"
        "        b, msgs = t.edges(seed, clock)\n"
        "        e = Engine(**t._cfg(clock))\n"
        "        r = e.generic(b)\n"
        "        e.close()\n"
        "        label = 'grid of one CTA per SM, seed %d, %s' % (seed, clock)\n"
        "        assert_results_equal(Oracle(**t._cfg(clock)).generic(b), r, abi.RUN_JSONL, label)\n"
        "        t.assert_equals_restatement(r, t.restated(seed, clock), label, msgs, clock)\n"
        "print('ok')\n")
    env = dict(os.environ, TGI_GRID_MULT="1")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and "ok" in p.stdout, p.stderr[-3000:]


def _good_generic():
    return pack_generic(make_generic(50, seed=21)[1])


def _bad_generic(where, nsec):
    _, msgs = make_generic(50, seed=21)
    i = {"first": 0, "middle": 25, "last": 49}[where]
    msgs[i].ts_nsec = nsec
    return pack_generic(msgs), i


def _bad_youtube(what, nsec):
    _, vids, chans = make_youtube(30, seed=5)
    if what == "video":
        vids[17].published_nsec = nsec
    else:
        chans[vids[3].channel].published_nsec = nsec
    return pack_youtube(vids, chans)


@pytest.mark.gpu
def test_rejected_calls_change_nothing():
    """every call with a time the library refuses is TGI_E_ARG, and the next call's output is what it would have been"""
    from distributed_crawler_b200.engine import Engine, EngineError
    good = _good_generic()
    yv, _, _ = make_youtube(30, seed=5)
    e = Engine()
    try:
        before, yt_before = e.generic(good), e.youtube(yv, abi.RUN_JSONL)
        assert_results_equal(Oracle().generic(good), before, abi.RUN_JSONL, "before")

        def rejected(call, *words):
            with pytest.raises(EngineError) as ei:
                call()
            assert ei.value.code == abi.E_ARG and all(w in str(ei.value) for w in words), str(ei.value)
            assert_results_equal(before, e.generic(good), abi.RUN_JSONL, "after a rejected call")
            assert_results_equal(yt_before, e.youtube(yv, abi.RUN_JSONL), abi.RUN_JSONL, "after a rejected call")

        for nsec in BAD_NSEC:
            for where in ("first", "middle", "last"):
                b, i = _bad_generic(where, nsec)
                rejected(lambda: e.generic(b), "ts_nsec %d" % nsec, "record %d" % i)
            for what in ("video", "channel"):
                b = _bad_youtube(what, nsec)
                rejected(lambda: e.youtube(b, abi.RUN_JSONL), "published_nsec %d" % nsec, what)
            rejected(lambda: e.set_clock(1_750_000_000, nsec, 1_750_000_000, 0), "created_at_nsec")
            rejected(lambda: e.set_clock(1_750_000_000, 0, 1_750_000_000, nsec), "capture_nsec")
    finally:
        e.close()
    for kw in [dict(created_at_nsec=n) for n in BAD_NSEC] + [dict(capture_nsec=n) for n in BAD_NSEC] + \
              [dict(tz_offset_sec=86400), dict(tz_offset_sec=-86400)]:
        with pytest.raises(EngineError) as ei:
            Engine(**kw)
        assert ei.value.code == abi.E_ARG, kw
    for off in (86399, -86399):  # the largest offsets still accepted
        e = Engine(tz_offset_sec=off)
        assert_results_equal(Oracle(tz_offset_sec=off).generic(good), e.generic(good), abi.RUN_JSONL, f"tz {off}")
        e.close()


# ---- CPU -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("clock", sorted(CLOCKS))
@pytest.mark.parametrize("seed", SEEDS)
def test_edges_oracle_vs_independent_restatement(seed, clock):
    batch, msgs = edges(seed, clock)
    r = oracle_for(clock).generic(batch)
    assert_equals_restatement(r, restated(seed, clock), f"oracle, seed {seed}, {clock}", msgs, clock)
    assert (r.status == abi.ST_NOLINE).sum() >= 4  # the int64 ends and the year bounds


def test_edges_oracle_vs_restatement_without_reaction_offsets():
    _, msgs = edges(1, "utc")
    batch = pack_generic(msgs)
    batch.react_off = None
    bare = [GenericMessage(id=m.id, channel_id=m.channel_id, text=m.text, sender_name=m.sender_name, ts_sec=m.ts_sec,
                           ts_nsec=m.ts_nsec, views=m.views) for m in msgs]
    r = Oracle().generic(batch)
    assert b'"reactions":{' not in r.jsonl.tobytes()
    assert_equals_restatement(r, _summary(restated_lines(bare, "utc")), "react_off NULL", bare, "utc")


@pytest.mark.parametrize("seed", SEEDS)
def test_edges_reach_every_cell(seed):
    _, msgs = make_generic_edges(seed)
    assert len(msgs) <= 8192  # one page of records
    cov = generic_edge_coverage(msgs)
    missing = [c for c in generic_edge_cells() if not cov[c]]
    assert not missing, missing
    assert set(NY_TRANSITIONS) <= set(NY[0])
    assert len(zone_derivable(msgs, NY)) >= len(msgs) - 8  # the zone runs leave out at most the instants past 9999 in UTC


def test_reaction_order_is_by_raw_bytes():
    """keys at and above 0x80 sort after 0x7f (unsigned bytes), prefixes first, and two invalid keys that escape alike
    are both written, in raw-byte order"""
    m = GenericMessage(id="1", channel_id="c", text="t", ts_sec=1_700_000_000,
                       reactions=[(b"\xff", 1), (b"\x80", 2), (b"\x7f", 3), (b"a\x00", 4), (b"a", 5), (b"", 6), (b"a", 7)])
    line = go_rules.generic_post_line(m, created=(1_750_000_000, 0), capture=(1_750_000_000, 0))
    want = b'"reactions":{"":6,"a":7,"a\\u0000":4,"\x7f":3,"\\ufffd":2,"\\ufffd":1}'
    assert want in line
    assert Oracle(capture_nsec=0).generic(pack_generic([m])).line(0) == line


def test_oracle_refuses_what_the_library_refuses():
    good = _good_generic()
    o = Oracle()
    want = o.generic(good)
    for nsec in BAD_NSEC:
        for where in ("first", "middle", "last"):
            with pytest.raises(OracleError) as ei:
                o.generic(_bad_generic(where, nsec)[0])
            assert ei.value.code == abi.E_ARG
        for what in ("video", "channel"):
            with pytest.raises(OracleError) as ei:
                o.youtube(_bad_youtube(what, nsec))
            assert ei.value.code == abi.E_ARG
        for clock in ((1_750_000_000, nsec, 1_750_000_000, 0), (1_750_000_000, 0, 1_750_000_000, nsec)):
            with pytest.raises(OracleError) as ei:
                o.set_clock(*clock)
            assert ei.value.code == abi.E_ARG
        assert_results_equal(want, o.generic(good), abi.RUN_JSONL, "the clock stays")
        for kw in (dict(created_at_nsec=nsec), dict(capture_nsec=nsec)):
            with pytest.raises(OracleError) as ei:
                Oracle(**kw)
            assert ei.value.code == abi.E_ARG
    for off in (86400, -86400, 2 ** 31 - 1, -(2 ** 31)):
        with pytest.raises(OracleError) as ei:
            Oracle(tz_offset_sec=off)
        assert ei.value.code == abi.E_ARG
    for ok in (dict(tz_offset_sec=86399), dict(tz_offset_sec=-86399), dict(created_at_nsec=999_999_999, capture_nsec=0)):
        Oracle(**ok).generic(good)
