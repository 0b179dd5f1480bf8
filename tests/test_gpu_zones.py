"""GPU tests: the local zone as a transition table (tgi_set_zone) on every path, byte for byte against the oracle."""
import base64
import re

import numpy as np
import pytest

from distributed_crawler_b200 import abi
from distributed_crawler_b200.corpus import Corpus
from distributed_crawler_b200.engine import Engine, EngineError, lib
from distributed_crawler_b200.pack import pack_generic
from gm_corpus import make_generic
from helpers import ALL, DEV, J, PREFIX, assert_results_equal
from oracle import pyoracle
from oracle.pyoracle import Oracle
from test_zones import ALL_ZONES, WINTER, ZONES
from yt_corpus import make_youtube
from zone_oracle import ZonedOracle

pytestmark = pytest.mark.gpu

SUMMER = 1719835200  # 2024-07-01T12:00:00Z
I32 = (-(1 << 31), (1 << 31) - 1)


def pinned_corpus(n, zone, first=0):
    """the seeded corpus (dates 2023-2025), every other record moved to a transition instant or the second before it"""
    c = Corpus(n, profile=2, nthreads=4, first=first)
    pins = [t for s in zone[0] for t in (s, s - 1) if I32[0] <= t <= I32[1]]
    dates = c.batch.recs["date"]
    for k in range(0, n, 2):
        dates[k] = pins[(k // 2) % len(pins)]
    return c


@pytest.mark.parametrize("name", sorted(ALL_ZONES))
def test_telegram_page_and_bulk(name):
    zone = ALL_ZONES[name]
    e = Engine()
    e.set_zone(*zone)
    for n, first in ((500, 0), (12000, 500)):
        c = pinned_corpus(n, zone, first)
        ro, rg = ZonedOracle(zone).telegram(c.batch, ALL), e.telegram(c.batch, ALL)
        assert_results_equal(ro, rg, ALL, f"{name} n={n}")
        assert (rg.gpu_launches == 1) == (n == 500)
        e.frontier_clear()
    e.close()


def test_generic_batch_and_the_year_range():
    _, msgs = make_generic(400, seed=11)
    zone = ZONES["Europe/Amsterdam"]
    pins = [t for s in zone[0] for t in (s, s - 1)]
    for k, m in enumerate(msgs[:200]):
        m.ts_sec = pins[k % len(pins)]
    msgs[200].ts_sec, msgs[200].ts_nsec = 253402297200, 5  # 9999-12-31T23:00:00Z: year 10000 at +01:00 and later
    g = pack_generic(msgs)
    e = Engine()
    rg0 = e.generic(g)
    assert rg0.status[200] == abi.ST_EMITTED
    e.set_zone(*zone)
    ro, rg = ZonedOracle(zone).generic(g), e.generic(g)
    assert_results_equal(ro, rg, J, "generic Amsterdam")
    assert rg.status[200] == abi.ST_NOLINE
    assert (rg.status == abi.ST_NOLINE).sum() == 1
    e.close()


@pytest.mark.parametrize("when,local", [(SUMMER, b"2024-07-01T08:00:00-04:00"), (WINTER, b"2024-01-01T07:00:00-05:00")])
def test_clocks_carry_the_offset_of_their_instant(when, local):
    zone = ZONES["America/New_York"]
    y, _, _ = make_youtube(60)
    g, _ = make_generic(60)
    c = Corpus(300, profile=2, nthreads=2)
    e, o = Engine(), ZonedOracle(zone)
    e.set_zone(*zone)
    e.set_clock(when, 0, when, 0)
    o.set_clock(when, 0, when, 0)
    for run, batch in (("youtube", y), ("generic", g), ("telegram", c.batch)):
        ro, rg = getattr(o, run)(batch, J), getattr(e, run)(batch, J)
        assert_results_equal(ro, rg, J, run)
        for i in range(rg.n):
            if rg.status[i] != abi.ST_EMITTED:
                continue
            line = rg.line(i)
            assert b'"capture_time":"' + local + b'"' in line, run
            if run == "telegram":  # created_at stays UTC (tdutils.go:611)
                assert b'"created_at":"' + time_utc(when) + b'"' in line
            else:
                assert b'"created_at":"' + local + b'"' in line, run
            if run == "youtube":  # the API's value keeps its zone
                assert re.search(rb'"published_at":"[^"]*Z"', line)
    e.close()


def time_utc(t):
    return pyoracle.json_time(t)[1:-1]


def test_resident_and_slot_paths():
    ny, lon = ZONES["America/New_York"], ZONES["Europe/London"]
    small = pinned_corpus(3000, ny)
    e = Engine()
    e.telegram_upload(0, small.batch)
    e.set_zone(*ny)
    assert_results_equal(ZonedOracle(ny).telegram(small.batch, J), e.telegram_run_resident(0, J, copy=True), J, "resident")
    big = Corpus(50000, profile=2, nthreads=8, first=7)
    e.telegram_submit(1, big.batch, J)
    s, o = np.array(lon[0], np.int64), np.array(lon[1], np.int32)
    rc = lib().tgi_set_zone(e.h, s.ctypes.data, o.ctypes.data, len(s))  # the job on slot 1 is in flight
    rg = e.telegram_wait(1, copy=True)
    e.release(1)
    assert rc == abi.E_STATE
    assert_results_equal(ZonedOracle(ny).telegram(big.batch, J), rg, J, "submit under New York")
    e.set_zone(*lon)
    e.telegram_submit(2, small.batch, J)
    rg = e.telegram_wait(2, copy=True)
    e.release(2)
    assert_results_equal(ZonedOracle(lon).telegram(small.batch, J), rg, J, "next batch under London")
    e.close()


@pytest.mark.parametrize("tz", [0, -30, 3600])
def test_clearing_restores_the_fixed_offset(tz):
    c = Corpus(400, profile=2, nthreads=2)
    g, _ = make_generic(100)
    plain, e = Engine(tz_offset_sec=tz), Engine(tz_offset_sec=tz)
    e.set_zone(*ZONES["Europe/London"])
    e.set_zone([], [])
    for run, batch in (("telegram", c.batch), ("generic", g)):
        a, b = getattr(plain, run)(batch, J), getattr(e, run)(batch, J)
        assert np.array_equal(a.status, b.status) and np.array_equal(a.line_off, b.line_off) and np.array_equal(a.jsonl, b.jsonl)
        assert_results_equal(getattr(Oracle(tz_offset_sec=tz), run)(batch, J), b, J, run)
    plain.close()
    e.close()


def test_rejected_arguments_keep_the_previous_table():
    ny = ZONES["America/New_York"]
    c = Corpus(400, profile=2, nthreads=2)
    e = Engine()
    e.set_zone(*ny)
    for starts, offsets in (([0, 0], [0, 0]), ([5, 1], [0, 0]), ([0], [86400]), ([0], [-86400]),
                            (list(range(abi.ZONE_MAX + 1)), [0] * (abi.ZONE_MAX + 1))):
        with pytest.raises(EngineError) as ei:
            e.set_zone(starts, offsets)
        assert ei.value.code == abi.E_ARG
    assert lib().tgi_set_zone(e.h, None, None, 3) == abi.E_ARG
    assert_results_equal(ZonedOracle(ny).telegram(c.batch, J), e.telegram(c.batch, J), J, "after rejections")
    e.close()


def test_sinks_carry_the_zoned_lines():
    lon = ZONES["Europe/London"]
    c = Corpus(10000, profile=2, nthreads=4, first=3)
    ro, utc = ZonedOracle(lon), Oracle()
    ro.set_clock(WINTER, 0, WINTER, 0)  # capture_time "Z": only published_at changes
    pyoracle.lib().orc_set_clock(utc.h, WINTER, 0, WINTER, 0)
    ro, utc = ro.telegram(c.batch, J), utc.telegram(c.batch, J)
    changed = np.diff(ro.line_off.astype(np.int64)) != np.diff(utc.line_off.astype(np.int64))
    assert changed.any() and not changed.all()
    e = Engine()
    e.set_zone(*lon)
    e.set_clock(WINTER, 0, WINTER, 0)
    e.telegram_submit(0, c.batch, J | DEV)
    e.telegram_wait(0)
    pay = e.dapr_payloads(0, PREFIX)
    app = e.channel_appends(0)
    groups = [(int(g["first_record"]), bytes(app.group(k))) for k, g in enumerate(app.groups)]
    order = app.order.copy()
    e.release(0)
    for i in range(ro.n):
        assert pay.data(i) == (base64.b64encode(ro.line(i)) if ro.status[i] == abi.ST_EMITTED else b""), i
    pos = 0
    for k, g in enumerate(app.groups):
        recs = order[pos:pos + int(g["n_lines"])]
        pos += int(g["n_lines"])
        assert groups[k][1] == b"".join(ro.line(int(r)) for r in recs)
    assert pos == int((ro.status == abi.ST_EMITTED).sum())
    e.close()
