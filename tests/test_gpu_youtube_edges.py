"""The YouTube line at the edges of its GPU-only rules (tests/yt_corpus.py:make_youtube_edges): the three writers
yt_size_lane_kernel picks per record (lane copy, lane ASCII escaper with its pending long-string copies, warp writer),
the extractors' 16-byte lanes and 512-byte strips, float64 rendering of int64 view counts, sanitizeFilename, the time
bounds — CUDA through the C ABI vs the CPU oracle, byte equality, on the page kernel, the bulk pipeline and the
warp-per-record reference kernels.  The CPU tests pin the oracle on the same videos with the second restatement
(tests/go_rules.py) and check that the generator reaches every cell of the writer rule."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import go_rules
from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import Engine
from distributed_crawler_b200.pack import YouTubeChannel, YouTubeVideo, pack_youtube
from helpers import assert_results_equal, no_page
from oracle import pyoracle
from oracle.pyoracle import Oracle
from yt_corpus import (I64_MAX, I64_MIN, make_youtube_edges, make_youtube_edges_many, view_values, yt_edge_cells,
                       yt_edge_coverage, yt_writer_mode)

ALL = abi.RUN_JSONL | abi.RUN_LINKS | abi.RUN_FRONTIER
PAGE_MAX_RECS = 8192  # tgingest.cu: the largest batch the one-launch page kernel takes
SEEDS = (1, 2, 3)


def _against_oracle(batch, label, **cfg):
    o, e = Oracle(**cfg), Engine(**cfg)
    try:
        ro, rg = o.youtube(batch, ALL), e.youtube(batch, ALL)
        assert_results_equal(ro, rg, ALL, label)
        assert np.array_equal(o.frontier_export(), e.frontier_export()), f"{label}: frontier differs"
        return ro, rg
    finally:
        e.close()
        o.close()


# ---- GPU -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS)
def test_edges_page_kernel(seed):
    batch, _, _ = make_youtube_edges(seed)
    assert batch.n <= PAGE_MAX_RECS
    ro, rg = _against_oracle(batch, "page kernel")
    assert rg.gpu_launches == 1, "an edge batch is page-sized: it must take the one-launch path"
    assert (ro.status == abi.ST_NOLINE).sum() == 4  # the four unrepresentable dates


@pytest.mark.gpu
def test_edges_page_kernel_other_clock_and_label():
    batch, _, _ = make_youtube_edges(4)
    _, rg = _against_oracle(batch, "page kernel, tz / label", tz_offset_sec=-12600, crawl_label=b'yt"<lbl>\xff',
                            created_at_nsec=987_000_000, capture_nsec=1)
    assert rg.gpu_launches == 1


@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS)
def test_edges_bulk_pipeline(seed):
    """the lane writer (modes 1 and 2) and the warp writer (mode 0) of the bulk pipeline, side by side in every warp"""
    batch, vids, chans = make_youtube_edges(seed)
    with no_page():
        _, rg = _against_oracle(batch, "bulk pipeline")
    assert rg.gpu_launches > 1
    assert {yt_writer_mode(v, chans[v.channel]) for v in vids} == {None, 0, 1, 2}


@pytest.mark.gpu
def test_edges_warp_reference_kernels():
    """TGI_YT_WARP=1 (read once per process, hence a child process): the warp sizer and writer for every record"""
    code = (
        "import sys; sys.path.insert(0, 'tests')\n"
        "import numpy as np\n"
        "from distributed_crawler_b200 import abi\n"
        "from distributed_crawler_b200.engine import Engine\n"
        "from oracle.pyoracle import Oracle\n"
        "from helpers import assert_results_equal\n"
        "from yt_corpus import make_youtube_edges\n"
        "f = abi.RUN_JSONL | abi.RUN_LINKS | abi.RUN_FRONTIER\n"
        "for seed in (1, 2, 3):\n"
        "    b, _, _ = make_youtube_edges(seed)\n"
        "    o, e = Oracle(), Engine()\n"
        "    r = e.youtube(b, f)\n"
        "    assert r.gpu_launches > 1\n"
        "    assert_results_equal(o.youtube(b, f), r, f, 'warp kernels, seed %d' % seed)\n"
        "    assert np.array_equal(o.frontier_export(), e.frontier_export())\n"
        "    e.close()\n"
        "print('ok')\n")
    env = dict(os.environ, TGI_YT_WARP="1", TGI_NO_PAGE="1")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and "ok" in p.stdout, p.stderr[-3000:]


@pytest.mark.gpu
def test_edges_above_the_page_size():
    batch, _, _ = make_youtube_edges_many(PAGE_MAX_RECS + 1, seed=100)
    assert batch.n > PAGE_MAX_RECS
    _, rg = _against_oracle(batch, "bulk batch above the page size")
    assert rg.gpu_launches > 1


@pytest.mark.gpu
def test_page_whose_lines_outgrow_the_page_block():
    """A ~50 KB description of '<' is written three times at 6x (~900 KB of line), far above the page block's estimate
    (6 x input bytes + 3 KB per record + 64 KB, ~370 KB here): the page kernel must give the batch back to the bulk
    pipeline by itself, where the lane writer escapes the description through its pending long-string copies."""
    assert "TGI_PAGE_VAR_CAP" not in os.environ
    chans = [YouTubeChannel(id="UC" + "q" * 22, title="t", published_sec=1_600_000_000)]
    vids = [YouTubeVideo(id="big", title="t<" * 70, description="<" * 50_000, view_count=2 ** 62 + 512),
            YouTubeVideo(id="n1", title="plain", description="x" * 300),
            YouTubeVideo(id="n2", title=" ", description="<" * 129)]
    batch = pack_youtube(vids, chans)
    ro, rg = _against_oracle(batch, "page over its block")
    assert rg.gpu_launches > 1, "the page must fall back to the bulk pipeline"
    assert len(ro.line(0)) > 900_000
    assert [yt_writer_mode(v, chans[0]) for v in vids] == [2, 1, 0]


# ---- CPU -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", SEEDS)
def test_edges_reach_every_cell_of_the_writer_rule(seed):
    """all three writers in every raw-length class of the description and of the title, each combination of the two
    being longer than YT_LANE_LONG (128), raw <= 128 with escaped > 128, a raw 129-byte string with nothing to escape
    beside an escaped one, and both strings long and escaped in mode 2 (the pending slots run out)"""
    _, vids, chans = make_youtube_edges(seed)
    cov = yt_edge_coverage(vids, chans)
    missing = [c for c in yt_edge_cells() if not cov[c]]
    assert not missing, missing
    modes = [yt_writer_mode(v, chans[v.channel]) for v in vids]
    assert len({modes[k] for k in (0, 1, 2)}) == 3 and modes[31] != modes[32] and modes[63] != modes[64]


@pytest.mark.parametrize("seed,cfg", [(1, {}), (2, {}), (4, dict(tz_offset_sec=-12600, crawl_label=b'yt"<lbl>\xff',
                                                                    created_at_nsec=987_000_000, capture_nsec=1))])
def test_edges_oracle_vs_independent_restatement(seed, cfg):
    """every line, status and snowball id list of the edge videos: the oracle against tests/go_rules.py"""
    _, vids, chans = make_youtube_edges(seed)
    r = Oracle(**cfg).youtube(pack_youtube(vids, chans), abi.RUN_JSONL | abi.RUN_LINKS)
    kw = dict(crawl_label=cfg.get("crawl_label", b""), created=(1_750_000_000, cfg.get("created_at_nsec", 0)),
              capture=(1_750_000_000, cfg.get("capture_nsec", 123_456_789)), tz=cfg.get("tz_offset_sec", 0))
    for i, v in enumerate(vids):
        line, _, ids = go_rules.youtube_post_line(v, chans[v.channel], **kw)
        assert r.line(i) == (line or b""), i
        assert r.status[i] == (abi.ST_EMITTED if line else abi.ST_NOLINE), i
        assert [x for x, _ in r.record_links(i)] == [x[:32] for x in ids], i


def test_engagement_wraps_like_go():
    """engagement is an int64 sum in Go (youtube_crawler.go:561): it wraps"""
    ch = YouTubeChannel(cached=False)
    for like, comment, views, want in ((I64_MAX, 1, 0, I64_MIN), (I64_MIN, -1, 0, I64_MAX), (I64_MAX, I64_MAX, 100, -1),
                                       (I64_MIN, I64_MIN, -(2 ** 62), -(2 ** 62 // 100))):
        line, _, _ = go_rules.youtube_post_line(YouTubeVideo(like_count=like, comment_count=comment, view_count=views), ch)
        assert b',"engagement":%d,' % want in line


def _bound_ties(rng, n):
    """int64 values exactly halfway between two float64 neighbours, where a short decimal lies on the bound of the
    rounding interval: float64(v) rounds half to even, and the bound belongs to the interval only for an even mantissa"""
    out = []
    for _ in range(n):
        e = rng.randrange(54, 63)
        half = 1 << (e - 53)  # ulp / 2 of [2^e, 2^(e+1))
        k = rng.randrange(0, e - 52)  # a multiple of 10^k can sit on the half-ulp grid
        step = 10 ** k * 2 ** max(0, e - 53 - k)
        m = rng.randrange(2 ** e // step + 1, 2 ** (e + 1) // step)
        c = m * step
        if c % (2 * half) == half:  # exactly between two doubles
            out += [c, -c]
    return out


def test_float_of_int64_oracle_vs_independent_restatement():
    """strconv.FormatFloat(float64(v), 'f', -1, 64) of the oracle against Python's shortest repr (go_rules) on ~100 000
    view counts: the edge set, powers of two and their neighbours (the asymmetric interval), half-ulp values whose
    short candidates lie on the interval bound, and random values of every magnitude above 2^53.  An exact tie between
    two shortest candidates cannot occur here: a midpoint of two multiples of 10^k is an odd multiple of 5^k * 2^(k-1),
    which is a multiple of the ulp 2^(e-52) only when 10^k / 2 exceeds half an ulp, i.e. lies outside the interval.
    Nor does the narrower lower half-interval of a power of two decide any digit here: 2^53 ... 2^63 render the same
    with a symmetric interval.  What does decide digits is the half-ulp bound, included for an even mantissa only."""
    rng = random.Random(2053)
    vals = view_values(rng, n_random=25_000)
    vals += [s * (2 ** e + d) for e in range(53, 64) for d in range(-2100, 2101, 5) for s in (1, -1)]
    vals += _bound_ties(rng, 15_000)
    vals += [rng.randrange(2 ** rng.randrange(53, 63), 2 ** 63) * rng.choice((1, -1)) for _ in range(40_000)]
    vals = [min(max(v, I64_MIN), I64_MAX) for v in vals]
    assert len(vals) > 95_000
    for v in vals:
        assert pyoracle.json_float_of_int64(v) == go_rules._go_float_of_int(v), v
