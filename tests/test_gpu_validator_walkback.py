"""GPU tests: the validator walkback (tgi_state_validator_walkback) against tests/validator_walkback_rules.py — every
batch's outcome and every statement byte for byte at 1, 2, 7 and 8191 rows per statement, over random claimed sets
(empty, all-invalid, all-valid and mixed batches, the OTHER class, strings that need escaping, empty crawl_ids) at
rates -5, 0, 15, 100 and 250, with discovered sets that are empty, hold the source's name only, hold only excluded names,
are random or have grown; the counter across calls; refused calls that leave the next output unchanged; the end of a
live hand-off; a call past one grid pass and a batch of 10^4 edges; and the C layout."""
import ctypes as C
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest

import tandem_sql_rules as sr
import validator_walkback_rules as vr
from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import Engine, EngineError, names_to_keys32
from distributed_crawler_b200.state_pack import pack_claimed_batches
from test_gpu_state_discover import MIN_DATE
from test_gpu_state_tandem import NOW, RUN
from test_gpu_state_walkback import WalkSequence

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KS = (1, 2, 7, vr.MAX_ROWS)
RATES = (-5, 0, 15, 100, 250)
ODD = b'c<&>"\\ \xe2\x80\xa8 \xff\x00'  # escapes, U+2028, an invalid byte, NUL
CRAWL_IDS = [b"crawl-2025", ODD, b""]
CLOCKS = [(NOW, 0), (NOW, 120_000_000), (1710054000 - 1, 999_999_999)]
STATUSES = [b"valid", b"not_channel", b"invalid", b"duplicate", b"pending", b"Valid", b""]  # the last three are OTHER
TYPES = [b"mention", b"text_url", b"url", b"plaintext", b"", b"unknown", ODD]
NAMES = [b"chan%03d" % i for i in range(40)]


def refused(call, code):
    with pytest.raises(EngineError) as ei:
        call()
    assert ei.value.code == code


class Validator:
    """an engine with a seed, the discovered set's keys in insertion order and the count v of batches handled"""

    def __init__(self, seed):
        self.rnd = random.Random(seed)
        self.seed = 0x7A11D000 + seed
        self.e = Engine(min_post_date=MIN_DATE, frontier_capacity=1024, set_growth=1 << 20)
        self.e.state_id_seed(self.seed)
        self.disc, self.v = [], 0

    def add(self, names):
        self.e.set_add(abi.SET_DISCOVERED, names_to_keys32(names))
        self.disc += [n for n in dict.fromkeys(names) if n not in self.disc]

    def batch(self, kind=None, n_edges=None, source=None):
        r = self.rnd
        kind = kind or r.choice(["empty", "invalid", "valid", "mixed", "mixed"])
        m = 0 if kind == "empty" else n_edges if n_edges is not None else r.choice([1, 2, 3, 5, 9])
        edges = []
        for _ in range(m):
            st = (b"valid" if kind == "valid" else r.choice([b"invalid", b"not_channel", b"duplicate"]) if kind == "invalid"
                  else r.choice(STATUSES))
            dest = r.choice(NAMES + [ODD, b"x" * 40, b""])
            edges.append((dest, r.choice(TYPES), st))
        return {"batch_id": b"%08x-0000-4000-8000-%012x" % (r.getrandbits(32), r.getrandbits(48)),
                "crawl_id": r.choice(CRAWL_IDS), "source_channel": source or r.choice(NAMES + [ODD]),
                "source_page_id": r.choice([b"pid", ODD, b""]),
                "source_depth": r.choice([0, 1, 7, -3, (1 << 63) - 1, -(1 << 63)]),
                "sequence_id": r.choice([b"seq-1", ODD, b""]), "edges": edges}

    def check(self, batches, rate, crawl, now, k, packed=None):
        want = vr.run(batches, self.disc, rate, self.seed, self.v, crawl, sr.discovery_time(*now))
        got, stmts = self.e.state_validator_walkback(packed or batches, rate, crawl, now, k)
        assert got == [r for r, _ in want], (rate, k)
        assert stmts == vr.statements(want, k), (rate, crawl, now, k)
        assert (self.e.state_vw_launches == 0) == (not batches)
        self.v += len(batches)
        return want


@pytest.mark.parametrize("seed", range(3))
def test_random_claimed_sets_with_every_kind_of_discovered_set(seed):
    x = Validator(seed)
    r = x.rnd
    seen = {vr.WALK_OK: 0, vr.WALK_EXHAUSTED: 0, vr.WALK_EMPTY: 0, "forward": 0, "walkback": 0, "rows": 0}
    n_call = 0

    def run(n_calls, **kw):
        nonlocal n_call
        for _ in range(n_calls):
            batches = [x.batch(**kw) for _ in range(r.choice([0, 1, 4, 12]))]
            rate, k = RATES[n_call % len(RATES)], KS[n_call % len(KS)]
            want = x.check(batches, rate, CRAWL_IDS[n_call % 3], CLOCKS[n_call % 3], k)
            n_call += 1
            for res, calls in want:
                seen[res["status"]] += 1
                seen["walkback" if res["walkback"] else "forward"] += 1
                seen["rows"] += len(calls)

    run(6)  # a set never allocated: every walkback is TGI_WALK_EMPTY
    x.add([b"src"])  # the source's name only: its walkbacks are exhausted after 10 draws
    run(5, source=b"src")
    x.add([b"chan001", b"chan002"])  # now also names the batches' valid edges may exclude
    run(5, kind="valid", source=b"src")
    x.add(r.sample(NAMES, 20) + [ODD[:8]])  # random
    run(10)
    assert x.e.set_info(abi.SET_DISCOVERED)["grows"] == 0
    x.add([b"grown%05d" % i for i in range(3000)])  # through tgi_set_growth
    assert x.e.set_info(abi.SET_DISCOVERED)["grows"] > 0
    run(10)
    assert all(v > 0 for v in seen.values()), seen
    x.e.close()


def test_every_rate_and_k_on_one_claimed_set():
    x = Validator(7)
    x.add(NAMES[:10] + [b"src"])
    batches = [x.batch(kind=kd) for kd in ("empty", "invalid", "valid", "mixed") for _ in range(6)]
    batches += [x.batch(kind="valid", n_edges=3, source=b"src") for _ in range(3)]
    for rate in RATES:
        for k in KS:
            x.check(batches, rate, b"", CLOCKS[1], k)
    x.e.close()


def test_a_set_of_excluded_names_only():
    x = Validator(8)
    x.add([b"x1", b"x2"])
    b = {"batch_id": b"b", "source_channel": b"s", "edges": [(b"x1", b"url", b"valid"), (b"x2", b"", b"valid")]}
    want = x.check([b, dict(b, edges=b["edges"][:1])], 250, b"c", CLOCKS[0], 1)
    assert want[0][0]["status"] == vr.WALK_EXHAUSTED and want[0][1] == []
    assert want[1][0]["status"] == vr.WALK_OK and want[1][0]["url"] == b"x2"
    x.e.close()


def test_refused_calls_leave_the_next_output_unchanged():
    x = Validator(9)
    x.add(NAMES[:5])
    batches = [x.batch(kind="mixed") for _ in range(6)]
    recs, eoff, edges, blob = pack_claimed_batches(batches)
    e = x.e
    call = lambda p, k=7, now=(NOW, 5), rate=15: e.state_validator_walkback(p, rate, b"c", now, k)  # noqa: E731
    for k in (0, vr.MAX_ROWS + 1, 1 << 31):
        refused(lambda: call((recs, eoff, edges, blob), k), abi.E_ARG)
    for now in ((NOW, -1), (NOW, 1_000_000_000), (253402300800, 0), (-62167219201, 0)):
        refused(lambda: call((recs, eoff, edges, blob), 7, now), abi.E_ARG)
    bad = []
    o = eoff.copy(); o[0] = 1; bad.append((recs, o, edges, blob))  # noqa: E702
    o = eoff.copy(); o[-1] += 1; bad.append((recs, o, edges, blob))  # noqa: E702
    o = eoff.copy(); o[2], o[3] = o[3], o[2]; bad.append((recs, o, edges, blob))  # noqa: E702
    if o[2] == o[3]:
        bad.pop()
    rr = recs.copy(); rr[1]["str_len"][2] = len(blob) + 1; bad.append((rr, eoff, edges, blob))  # noqa: E702
    rr = recs.copy(); rr[0]["str_off"][0] = (1 << 64) - 1; rr[0]["str_len"][0] = 2; bad.append((rr, eoff, edges, blob))  # noqa: E702,E501
    ee = edges.copy(); ee[0]["cls"] = abi.EDGE_CLASS_OTHER + 1; bad.append((recs, eoff, ee, blob))  # noqa: E702
    ee = edges.copy(); ee[-1]["str_off"][1] = len(blob); ee[-1]["str_len"][1] = 1; bad.append((recs, eoff, ee, blob))  # noqa: E702,E501
    for p in bad:
        refused(lambda: call(p), abi.E_ARG)
    x.check(batches, 15, b"c", (NOW, 5), 7, packed=(recs, eoff, edges, blob))  # v as it was
    # a clock that json.Marshal refuses matters only when there is a row
    x.check([], 15, b"c", (253402300800, 0), 7)
    x.add([b"src"])
    excl = {"batch_id": b"b", "source_channel": b"src", "edges": [(n, b"url", b"valid") for n in NAMES[:5]]}
    refused(lambda: call([dict(excl, edges=excl["edges"][:4])], 7, (253402300800, 0), 250), abi.E_ARG)  # NAMES[4]: a row
    want = x.check([excl], 250, b"c", (253402300800, 0), 7)  # the source and every other key excluded: no row
    assert want[0][0]["status"] == vr.WALK_EXHAUSTED
    x.e.close()
    # no seed: a call with batches is refused, one without is not
    e2 = Engine(min_post_date=MIN_DATE)
    assert e2.state_validator_walkback([], 15, b"c", (NOW, 0), 1) == ([], [])
    refused(lambda: e2.state_validator_walkback(batches, 15, b"c", (NOW, 0), 1), abi.E_STATE)
    e2.state_id_seed(x.seed)
    got, _ = e2.state_validator_walkback(batches, 15, b"c", (NOW, 0), 1)
    assert got == [res for res, _ in vr.run(batches, [], 15, x.seed, 0, b"c", None)]
    e2.close()


def test_the_call_ends_a_live_handoff_and_leaves_the_forced_walkback_counter():
    sq = WalkSequence(21, n_owners=3)
    e = sq.e
    sq.add_discovered([b"k1", b"k2"])
    ids = list(sq.go.page_map)
    spans, status, links = sq.result(ids, RUN, 0, sizes=[0, 0, 0])
    got = e.state_pending_edges(0, spans, NOW)
    assert [int(s) for s in got["span_batch"]] == [abi.STATE_NO_BATCH] * 3
    b = {"batch_id": b"b", "source_channel": b"k1", "edges": [(b"k2", b"url", b"valid")]}
    res, stmts = e.state_validator_walkback([b], 100, b"c", (NOW, 0), 1)
    want = vr.run([b], sq.disc, 100, sq.x.seed, 0, b"c", sr.discovery_time(NOW, 0))
    assert res == [want[0][0]] and stmts == vr.statements(want, 1)
    assert res[0]["status"] == vr.WALK_EXHAUSTED  # k1 is the source, k2 excluded
    refused(lambda: e.state_edge_sql(b"c", (NOW, 0), 1), abi.E_STATE)
    refused(lambda: e.state_walkback(b"c", (NOW, 0), 1), abi.E_STATE)
    e.release(0)
    # the next hand-off's forced walkbacks start where the last hand-off left w
    spans, status, links = sq.result(ids, RUN, 1, sizes=[0, 0, 0])
    got = e.state_pending_edges(1, spans, NOW)
    assert sq.check_walkback(spans, [int(s) for s in got["span_batch"]])
    e.release(1)
    e.close()


def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_a_call_past_one_grid_pass_and_a_batch_of_ten_thousand_edges():
    x = Validator(30)
    x.add(NAMES[:30])
    n = max(300_000, sms() * 1024 + 2000)
    batches = [{"batch_id": b"b%07d" % i, "crawl_id": b"" if i % 7 == 0 else b"crawl",
                "source_channel": NAMES[i % 40], "source_page_id": b"p%d" % i, "source_depth": i,
                "sequence_id": b"s%d" % (i % 13),
                "edges": [(NAMES[(i + j) % 40], TYPES[(i + j) % 4], STATUSES[(i * 7 + j) % 5]) for j in range(i % 3)]}
               for i in range(n)]
    packed = pack_claimed_batches(batches)
    for k in (vr.MAX_ROWS, 1):
        x.check(batches, 40, b"cfg", (NOW, 0), k, packed=packed)
    big = [{"batch_id": b"big", "source_channel": b"chan000", "crawl_id": b"",
            "edges": [(b"d%05d" % j if j % 5 else NAMES[j % 40], TYPES[j % 7], STATUSES[j % 7]) for j in range(12_000)]},
           {"batch_id": b"big2", "source_channel": b"chan001",
            "edges": [(NAMES[j % 30], TYPES[j % 3], b"valid") for j in range(10_000)]}]
    for rate, k in ((0, vr.MAX_ROWS), (250, 7), (15, 1)):
        x.check(big, rate, b"cfg", (NOW, 0), k)
    x.e.close()


def test_layout_matches_the_header():
    src = r"""
#include <stddef.h>
#include <stdio.h>
#include "tgingest.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu\n", sizeof(tgi_claimed_batch), offsetof(tgi_claimed_batch, str_len),
         offsetof(tgi_claimed_batch, source_depth), sizeof(tgi_claimed_edge), offsetof(tgi_claimed_edge, cls));
  printf("%zu %zu %zu %zu %zu\n", sizeof(tgi_claimed_batches), offsetof(tgi_claimed_batches, edge_off),
         offsetof(tgi_claimed_batches, n_edges), offsetof(tgi_claimed_batches, strs),
         offsetof(tgi_claimed_batches, strs_len));
  printf("%zu %zu %zu %zu %zu\n", sizeof(tgi_state_validator_batch), offsetof(tgi_state_validator_batch, forward_edge),
         offsetof(tgi_state_validator_batch, url), offsetof(tgi_state_validator_batch, page_id),
         offsetof(tgi_state_validator_batch, sequence_id));
  printf("%zu %zu %zu\n", sizeof(tgi_state_validator_walkback_t), offsetof(tgi_state_validator_walkback_t, kernel_ms),
         offsetof(tgi_state_validator_walkback_t, gpu_launches));
  printf("%d %d %d %d %d %d %d %d %u\n", TGI_SQL_BATCH_COMPLETE, TGI_SQL_STATS_UPSERT, TGI_SQL_EDGES_DELETE,
         TGI_EDGE_CLASS_VALID, TGI_EDGE_CLASS_NOT_CHANNEL, TGI_EDGE_CLASS_INVALID, TGI_EDGE_CLASS_DUPLICATE,
         TGI_EDGE_CLASS_OTHER, TGI_VW_NO_EDGE);
  return 0;
}
"""
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "t.c"), os.path.join(d, "t")
        with open(c, "w") as f:
            f.write(src)
        subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        lines = [[int(v) for v in ln.split()] for ln in subprocess.check_output([exe], text=True).split("\n") if ln]
    b, e, o = abi.CLAIMED_BATCH, abi.CLAIMED_EDGE, abi.STATE_VALIDATOR_BATCH
    assert lines[0] == [b.itemsize, b.fields["str_len"][1], b.fields["source_depth"][1], e.itemsize, e.fields["cls"][1]]
    K = abi.ClaimedBatchesC
    assert lines[1] == [C.sizeof(K), K.edge_off.offset, K.n_edges.offset, K.strs.offset, K.strs_len.offset]
    assert lines[2] == [o.itemsize, o.fields["forward_edge"][1], o.fields["url"][1], o.fields["page_id"][1],
                        o.fields["sequence_id"][1]]
    W = abi.StateValidatorWalkbackC
    assert lines[3] == [C.sizeof(W), W.kernel_ms.offset, W.gpu_launches.offset]
    assert lines[4] == [abi.SQL_BATCH_COMPLETE, abi.SQL_STATS_UPSERT, abi.SQL_EDGES_DELETE, abi.EDGE_CLASS_VALID,
                        abi.EDGE_CLASS_NOT_CHANNEL, abi.EDGE_CLASS_INVALID, abi.EDGE_CLASS_DUPLICATE,
                        abi.EDGE_CLASS_OTHER, abi.VW_NO_EDGE]
    assert [vr.BATCH_COMPLETE, vr.STATS_UPSERT, vr.EDGES_DELETE] == lines[4][:3]
    assert np.dtype(o).itemsize == 136
