"""The streaming form of the chunk combiner's batching rule (tgi_plan_chunks_carry): chained over the results of a
stream, split anywhere, it must give Chunker.processBatches (chunk/main.go:292-345) over the whole stream, as the
reference's long-running chunker sees one file per post.  Also the C ABI mirror of the combiner's output structs."""
import ctypes as C
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest

from distributed_crawler_b200 import abi, sink
from test_sink import process_batches

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def chained(lens, cuts, trigger, hard_cap):
    """the stream's lines cut into results at `cuts`, planned result by result -> (batches of global line indices,
    dropped global indices, the open group's bytes before the final close)"""
    bounds = [0] + sorted(cuts) + [len(lens)]
    batches, dropped, cur, open_bytes = [], [], [], 0
    for lo, hi in zip(bounds, bounds[1:]):
        part = lens[lo:hi]
        off = np.concatenate([[0], np.cumsum(part, dtype=np.uint64)]).astype(np.uint64)
        groups, drop, open_out = sink.plan_chunks_carry(off, open_bytes, trigger, hard_cap)
        kept = [i for i in range(hi - lo) if 0 < part[i] <= hard_cap]
        assert [i for i in range(hi - lo) if drop[i]] == [i for i in range(hi - lo) if part[i] > hard_cap]
        dropped += [lo + i for i in range(hi - lo) if drop[i]]
        prev_end = 0
        for k, (a, b) in enumerate(groups):
            assert prev_end <= a <= b <= hi - lo
            if k == 0 and cur:
                assert a == 0, "the group carried in begins at 0"
            else:
                assert a == min(i for i in kept if i >= prev_end), "a new group begins at its first line"
            batch = cur + [lo + i for i in kept if a <= i < b]
            assert batch, "a closed group holds a line"
            batches.append(batch)
            cur, prev_end = [], b
        cur += [lo + i for i in kept if i >= prev_end]
        open_bytes = sum(lens[i] for i in cur)
        assert open_out == open_bytes
    tail = open_bytes
    if cur:
        batches.append(cur)
    return batches, dropped, tail


def reference(lens, trigger, hard_cap):
    files = [i for i, l in enumerate(lens) if l > 0]  # one file per post that produced a line
    return [[files[k] for k in b] for b in process_batches([lens[i] for i in files], trigger, hard_cap)]


def check(lens, cuts, trigger, hard_cap):
    got, dropped, _ = chained(lens, cuts, trigger, hard_cap)
    assert got == reference(lens, trigger, hard_cap), (lens, cuts, trigger, hard_cap)
    assert dropped == [i for i, l in enumerate(lens) if l > hard_cap]


def random_lens(rnd, n, top):
    return [rnd.choice([0, 0, rnd.randrange(1, top), rnd.randrange(1, top), rnd.randrange(1, 6 * top)]) for _ in range(n)]


def test_random_streams_split_randomly(engine_lib):
    rnd = random.Random(11)
    for _ in range(300):
        n = rnd.randrange(0, 150)
        trigger = rnd.randrange(1, 4000)
        hard_cap = rnd.choice([trigger + rnd.randrange(0, 1500), max(1, trigger - rnd.randrange(0, trigger))])
        lens = random_lens(rnd, n, 900)
        cuts = [rnd.randrange(0, n + 1) for _ in range(rnd.randrange(0, 12))] if n else []
        check(lens, cuts, trigger, hard_cap)


def test_edges(engine_lib):
    rnd = random.Random(5)
    for _ in range(100):
        n = rnd.randrange(1, 80)
        lens = random_lens(rnd, n, 300)
        cuts = [rnd.randrange(0, n + 1) for _ in range(rnd.randrange(0, 8))]
        check(lens, cuts, 1, 500)                       # trigger = 1: one line per group
        check(lens, cuts, 0, 500)                       # trigger = 0 as well
        check(lens, cuts, 5000, 400)                    # trigger > hard_cap: only the cap closes groups
        check(lens, cuts, 100, 0)                       # a cap below every line: everything is dropped
        check(lens, cuts, 100, min(l for l in lens if l) if any(lens) else 1)
        check([0] * n, cuts, 10, 20)                    # no lines at all
    check([], [], 10, 20)


def test_reference_vectors_split_everywhere(engine_lib, vectors):
    for v in vectors["chunk_batches"]:
        sizes, trig, cap = v["sizes"], v["trigger"], v["hard_cap"]
        want = process_batches(sizes, trig, cap)
        for cut in range(len(sizes) + 1):
            for second in (None, (cut + len(sizes)) // 2):
                cuts = [cut] + ([second] if second is not None else [])
                got, _, _ = chained(sizes, cuts, trig, cap)
                assert got == want, (v["name"], cuts)
        for k in range(1, len(sizes) + 1):  # one line per result
            got, _, _ = chained(sizes, list(range(k)), trig, cap)
            assert got == want, v["name"]


def test_carry_matches_plan_chunks_without_carry(engine_lib):
    rnd = random.Random(2)
    for _ in range(100):
        n = rnd.randrange(0, 100)
        lens = random_lens(rnd, n, 700)
        off = np.concatenate([[0], np.cumsum(lens, dtype=np.uint64)]).astype(np.uint64)
        trig, cap = rnd.randrange(1, 3000), rnd.randrange(1, 3000)
        full, drop_full = sink.plan_chunks(off, trig, cap)
        groups, drop, open_out = sink.plan_chunks_carry(off, 0, trig, cap)
        assert np.array_equal(drop, drop_full)
        assert full[: len(groups)] == groups
        assert len(full) == len(groups) + (1 if open_out else 0)


def test_carry_rejects_a_group_that_cannot_rest(engine_lib):
    off = np.array([0, 5], np.uint64)
    with pytest.raises(RuntimeError):
        sink.plan_chunks_carry(off, 101, 1000, 100)  # above hard_cap
    with pytest.raises(RuntimeError):
        sink.plan_chunks_carry(off, 50, 50, 100)     # has reached trigger
    groups, dropped, open_out = sink.plan_chunks_carry(off, 49, 50, 100)
    assert groups == [(0, 1)] and not dropped.any() and open_out == 0
    groups, _, open_out = sink.plan_chunks_carry(off, 96, 1000, 100)  # the carried group closes before line 0
    assert groups == [(0, 0)] and open_out == 5


def test_combined_structs_match_header():
    probe = r'''
#include <stdio.h>
#include <stddef.h>
#include "tgingest.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu\n", sizeof(tgi_combined_blob), sizeof(tgi_combined_t), offsetof(tgi_combined_blob, unix_nano),
         offsetof(tgi_combined_t, open_lines), offsetof(tgi_combined_t, gpu_launches));
  return 0;
}'''
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "p.c")
        with open(src, "w") as f:
            f.write(probe)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", os.path.join(d, "p")])
        got = list(map(int, subprocess.check_output([os.path.join(d, "p")]).decode().split()))
    assert got == [C.sizeof(abi.CombinedBlobC), C.sizeof(abi.CombinedC), abi.CombinedBlobC.unix_nano.offset,
                   abi.CombinedC.open_lines.offset, abi.CombinedC.gpu_launches.offset]
