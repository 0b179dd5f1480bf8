"""Cost of the validator edge pass (tgi_state_validator_lookups, tgi_state_validator_edges) for claims of N edges over
N / 4 names (popular names recur), a fifth of them in the invalid cache, every name answered by a scripted t.me:

  device      per repetition, one lookups call and one edge pass at 1 and at 8191 rows per statement through the C ABI,
              from the same starting sets: host clock of each call (checks, uploads, kernels, set inserts and read-back
              into pinned memory), device time, launches, lookup rows and statements.
  host        the same claim restated in Python (tests/validator_edge_rules.py's per-edge loop), once.  This only
              bounds the Go loop's cost from above; Go and the database and HTTP calls are not measured.

Prints the card and its power limit, and the median over the repetitions.

    python tools/prof_state_validator_edges.py [--reps 5] [--sizes 1000 100000]
"""
import argparse
import ctypes as C
import os
import random
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import validator_edge_rules as ve  # noqa: E402
from distributed_crawler_b200 import abi  # noqa: E402
from distributed_crawler_b200.engine import Engine, lib, names_to_keys32  # noqa: E402
from distributed_crawler_b200.state_pack import pack_claimed_edges  # noqa: E402
from prof_state import card  # noqa: E402

NOW = 1_760_000_000
ANSWERS = [(ve.VALID, 0), (ve.NOT_CHANNEL, 1), (ve.INVALID, 2), (ve.TRANSIENT, 0), (ve.BLOCKED, 0), (ve.OTHER, 0)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", type=int, nargs="+", default=[1_000, 100_000])
    a = ap.parse_args()
    print(f"card: {card()}")
    r = random.Random(7)
    for N in a.sizes:
        names = [b"name_%07d" % i for i in range(max(N // 4, 1))]
        invalid = {nm: NOW - 60 for nm in names[::5]}
        world = ve.World(invalid, (), names[1::7], names[2::11],
                         {nm: [r.choice(ANSWERS) for _ in range(3)] for nm in names})
        edges = [{"pending_id": j + 1, "destination": r.choice(names), "crawl_id": b"crawl-1", "source_type": b"mention"}
                 for j in range(N)]
        recs, blob = pack_claimed_edges(edges)
        claim = abi.PendingClaimC(recs.ctypes.data, len(recs), blob.ctypes.data, len(blob))
        w = world.copy()
        outcomes, attempts = ve.shim(w, edges, ve.lookups(w, edges, NOW))
        oc = np.array([(d, c, n, 0) for d, c, n in outcomes], abi.VALIDATOR_OUTCOME)
        at = np.array(attempts, abi.VALIDATOR_ATTEMPT)
        e = Engine(set_growth=1 << 24)
        res = {}
        for k in (1, ve.MAX_ROWS):
            lw, ew, ld, ed = [], [], [], []
            for rep in range(a.reps + 1):  # one warm-up
                for which in (abi.SET_INVALID, abi.SET_SEEDS):
                    e.set_clear(which)
                e.set_add(abi.SET_INVALID, names_to_keys32(list(invalid)), np.array(list(invalid.values()), np.int64))
                lk = abi.StateValidatorLookupsC()
                t0 = time.perf_counter()
                assert lib().tgi_state_validator_lookups(e.h, C.byref(claim), NOW, C.byref(lk)) == 0
                t1 = time.perf_counter()
                assert lk.n_lookups == len(oc)
                out = abi.StateValidatorEdgesC()
                t2 = time.perf_counter()
                assert lib().tgi_state_validator_edges(e.h, oc.ctypes.data, len(oc), at.ctypes.data, len(at), 0, NOW, k,
                                                       C.byref(out)) == 0
                t3 = time.perf_counter()
                if rep:
                    lw.append((t1 - t0) * 1e3)
                    ew.append((t3 - t2) * 1e3)
                    ld.append(lk.kernel_ms)
                    ed.append(out.kernel_ms)
                info = (int(lk.n_lookups), int(out.n_stmts), int(lk.gpu_launches), int(out.gpu_launches))
            res[k] = (statistics.median(lw), statistics.median(ld), statistics.median(ew), statistics.median(ed), info)
        t0 = time.perf_counter()
        ve.run_claim(world.copy(), edges, NOW, 0)
        host_ms = (time.perf_counter() - t0) * 1e3
        print(f"N = {N:>6} edges: " + " | ".join(
            f"k = {k}: lookups {v[0]:.3f} ms (device {v[1]:.3f} ms, {v[4][2]} launches, {v[4][0]} rows), pass "
            f"{v[2]:.3f} ms (device {v[3]:.3f} ms, {v[4][3]} launches, {v[4][1]} statements)" for k, v in res.items())
            + f" | Python restatement {host_ms:.1f} ms", flush=True)
        e.close()


if __name__ == "__main__":
    main()
