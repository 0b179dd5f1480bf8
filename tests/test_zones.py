"""CPU tests: the local-zone rule (tgi_set_zone) as the zone tests expect it (tests/zone_oracle.py), over the committed
transition tables of tests/golden/zones.json and a synthetic zone with awkward offsets."""
import json
import os
import random

import numpy as np
import pytest

from distributed_crawler_b200 import abi
from distributed_crawler_b200.corpus import Corpus
from distributed_crawler_b200.pack import pack_generic
from gm_corpus import make_generic
from oracle import pyoracle
from oracle.pyoracle import Oracle
from yt_corpus import make_youtube
from zone_oracle import ZonedOracle, go_json_time, go_offset

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LO, HI = -(1 << 31), 1 << 32
WINTER = 1704110400  # 2024-01-01T12:00:00Z


def load_zones():
    with open(os.path.join(ROOT, "tests", "golden", "zones.json")) as f:
        return {n: (z["start"], z["offset"]) for n, z in json.load(f)["zones"].items()}


def synthetic_zone():
    """offsets of -30 s, -75 s, +59 s and +-23:59:59, entries at adjacent seconds, inside the corpus' 2023-2025 dates"""
    b = 1_700_000_000
    starts = [LO, b, b + 1, b + 2, b + 3, b + 4, b + 5, b + 9_000_000, b + 9_000_001, b + 30_000_000, b + 45_000_000]
    offsets = [-30, -75, 59, 86399, -86399, 0, -30, 1172, -75, 59, -86399]
    return starts, offsets


ZONES = load_zones()
ALL_ZONES = dict(ZONES, synthetic=synthetic_zone())


def instants(zone, rng, k=1500):
    starts = [s for s in zone[0] if LO < s < HI]
    ts = [rng.randrange(LO, HI) for _ in range(k)] + starts + [s - 1 for s in starts] + [LO, HI - 1]
    return [(t, rng.choice([0, 0, 1, 500_000_000, 999_999_999, rng.randrange(1, 10 ** 9)])) for t in ts]


@pytest.mark.parametrize("name", sorted(ALL_ZONES))
def test_zone_rule_agrees_with_the_oracle_at_each_offset(name):
    """the restatement's local fields equal the oracle's fixed-offset rendering at the offset the table gives; so does
    the suffix, except for the -1..-59 s offsets, where the fixed-offset rule keeps its own sign"""
    zone = ALL_ZONES[name]
    rng = random.Random(sum(map(ord, name)))
    for t, ns in instants(zone, rng):
        off = go_offset(zone, t)
        got, fixed = go_json_time(t, ns, off), pyoracle.json_time(t, ns, off)
        if -60 < off < 0:
            assert got[:-7] == fixed[:-7] and got[-7:] == b'+00:00"' and fixed[-7:] == b'-00:00"', (name, t, ns)
        else:
            assert got == fixed, (name, t, ns, off)


def test_offsets_and_year_range():
    assert go_offset(([10, 20], [1, 2]), 9) == 1 and go_offset(([10, 20], [1, 2]), 20) == 2
    assert go_json_time(0, 0, -30) == b'"1969-12-31T23:59:30+00:00"'
    assert go_json_time(0, 0, -75) == b'"1969-12-31T23:58:45-00:01"'
    assert go_json_time(0, 0, 1172) == b'"1970-01-01T00:19:32+00:19"'
    assert go_json_time(0, 0, 86399) == b'"1970-01-01T23:59:59+23:59"'
    assert pyoracle.json_time(0, 0, -30) == b'"1969-12-31T23:59:30-00:00"'  # the fixed offset's own rendering
    end = 253402300799  # 9999-12-31T23:59:59Z
    assert go_json_time(end, 0, 0) == b'"9999-12-31T23:59:59Z"' and go_json_time(end, 0, 1) == b""
    assert go_json_time(-62167219200, 0, 0) == b'"0000-01-01T00:00:00Z"' and go_json_time(-62167219200, 0, -60) == b""


@pytest.mark.parametrize("off", [0, 3600, -18000, 19800, 20700, -12600, 86340, -86340])
def test_one_entry_table_equals_fixed_offset(off):
    c = Corpus(300, profile=2, nthreads=2)
    g, _ = make_generic(200)
    y, _, _ = make_youtube(60)
    fixed, zoned = Oracle(tz_offset_sec=off), ZonedOracle(([0], [off]))
    for run, batch in (("telegram", c.batch), ("generic", g), ("youtube", y)):
        a, b = getattr(fixed, run)(batch, abi.RUN_JSONL), getattr(zoned, run)(batch, abi.RUN_JSONL)
        assert np.array_equal(a.status, b.status) and np.array_equal(a.line_off, b.line_off), run
        assert np.array_equal(a.jsonl, b.jsonl), run


def test_london_changes_line_lengths_with_the_season():
    c = Corpus(500, profile=2, nthreads=2)  # dates 2023-2025
    utc, lon = Oracle(), ZonedOracle(ZONES["Europe/London"])
    pyoracle.lib().orc_set_clock(utc.h, WINTER, 0, WINTER, 0)
    lon.set_clock(WINTER, 0, WINTER, 0)  # capture_time is "Z" in both
    a, b = utc.telegram(c.batch, abi.RUN_JSONL), lon.telegram(c.batch, abi.RUN_JSONL)
    d = np.diff(b.line_off.astype(np.int64)) - np.diff(a.line_off.astype(np.int64))
    assert set(d[a.status == abi.ST_EMITTED].tolist()) == {0, 5}  # "Z" in winter, "+01:00" in summer


def test_a_local_year_past_9999_drops_the_generic_line():
    _, msgs = make_generic(50, seed=3)
    msgs[7].ts_sec = 253402297200  # 9999-12-31T23:00:00Z
    g = pack_generic(msgs)
    a, b = Oracle().generic(g), ZonedOracle(ZONES["Europe/Amsterdam"]).generic(g)  # +01:00 or +02:00 there
    assert a.status[7] == abi.ST_EMITTED and b.status[7] == abi.ST_NOLINE and b.line(7) == b""
    assert (b.status == abi.ST_NOLINE).sum() == 1
