"""Cost of the standard random walk (tgi_state_rw_lookups, tgi_state_rw_step) for S pages of two records with six
t.me links each, over a discovered set of 10^5 channels, seeds and invalid names among the links, walkback rate 35:

  device      per repetition, one lookups call and one step at 1 and at 8191 rows per statement through the C ABI,
              every lookup answered NOT_FOUND or FOUND in turn, from the same starting sets: host clock of each call
              (checks, uploads, kernels, set inserts and read-back into pinned memory), device time, launches, lookups
              and statements.
  host        the same pages restated in Python (tests/random_walk_rules.py), once.  This only bounds the Go shim's
              cost from above; Go itself is not measured.

Prints the card and its power limit, and the median over the repetitions.

    python tools/prof_state_rw_step.py [--reps 5] [--sizes 1000 100000]
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

import random_walk_rules as rw  # noqa: E402
import tandem_sql_rules as sr  # noqa: E402
from distributed_crawler_b200 import abi  # noqa: E402
from distributed_crawler_b200.engine import Engine, lib, names_to_keys32  # noqa: E402
from distributed_crawler_b200.pack import pack_telegram  # noqa: E402
from helpers import msg  # noqa: E402
from prof_state import card  # noqa: E402
from test_gpu_state_discover import GOOD, MIN_DATE, oracle  # noqa: E402
from tg_link_corpus import CHANNELS  # noqa: E402

CRAWL = b"crawl-2025-10-17"
NOW = 1_760_000_000
N_DISC = 100_000
RATE = 35


def seed_sets(e, names, S):
    """the sets every repetition starts from: 10^5 discovered channels, a quarter of the pages' names as seeds and a
    quarter as invalid"""
    for which in (abi.SET_DISCOVERED, abi.SET_SEEDS, abi.SET_INVALID):
        e.set_clear(which)
    e.set_add(abi.SET_DISCOVERED, names_to_keys32([b"chan%07d" % i for i in range(N_DISC)]))
    e.set_add(abi.SET_SEEDS, names_to_keys32(names[: S // 4]))
    e.set_add(abi.SET_INVALID, names_to_keys32(names[S // 4: S // 2]), None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", type=int, nargs="+", default=[1_000, 100_000])
    a = ap.parse_args()
    print(f"card: {card()}")
    r = random.Random(5)
    for S in a.sizes:
        e = Engine(min_post_date=MIN_DATE, set_growth=1 << 24)
        e.state_id_seed(17)
        names = [b"name%07d" % i for i in range(4 * S)]
        owners = [{"id": b"%08d-0000-4000-8000-000000000000" % i, "url": b"owner%06d" % i, "depth": 1,
                   "status": b"fetched", "sequenceId": b"seq-%d" % i} for i in range(64)]
        e.state_set([(1, owners)])
        msgs = [msg("messageText", "p %d %s" % (p, " ".join("t.me/" + nm.decode() for nm in r.sample(names, 6))),
                    id=(p + 1) << 20, chat_id=-100777, channel=0, date=MIN_DATE + 5) for p in range(2 * S)]
        b = pack_telegram(msgs, CHANNELS)
        e.set_clock(*GOOD)
        e.telegram_submit(0, b, abi.RUN_LINKS)
        e.telegram_wait(0)
        rows = list(e._st_rows().values())
        sp = np.zeros(S, abi.STATE_SPAN)
        for p in range(S):
            sp[p] = (rows[p % len(rows)], 0, 2 * p, 2, 2)
        res = {}
        for k in (1, rw.MAX_ROWS):
            lw, sw, ld, sd = [], [], [], []
            for rep in range(a.reps + 1):  # one warm-up
                seed_sets(e, names, S)
                lk = abi.StateRwLookupsC()
                t0 = time.perf_counter()
                assert lib().tgi_state_rw_lookups(e.h, 0, sp.ctypes.data, S, NOW, C.byref(lk)) == 0
                t1 = time.perf_counter()
                oc = np.zeros(lk.n_lookups, abi.RW_OUTCOME)
                oc["code"] = np.where(np.arange(lk.n_lookups) % 2, rw.FOUND, rw.NOT_FOUND)
                oc["chat_id"] = np.arange(lk.n_lookups)
                out = abi.StateRwStepC()
                t2 = time.perf_counter()
                assert lib().tgi_state_rw_step(e.h, oc.ctypes.data, len(oc), RATE, CRAWL, len(CRAWL), NOW, 0, k,
                                               C.byref(out)) == 0
                t3 = time.perf_counter()
                if rep:
                    lw.append((t1 - t0) * 1e3)
                    sw.append((t3 - t2) * 1e3)
                    ld.append(lk.kernel_ms)
                    sd.append(out.kernel_ms)
                info = (int(lk.n_lookups), int(out.n_stmts), int(lk.gpu_launches), int(out.gpu_launches))
            res[k] = (statistics.median(lw), statistics.median(ld), statistics.median(sw), statistics.median(sd), info)
        e.release(0)
        # the restatement over the same pages and the same starting sets
        ro = oracle(GOOD).telegram(b, abi.RUN_LINKS)
        links = [[(nm, abi.SRC_NAMES.index(s)) for nm, s in ro.record_links(i)] for i in range(ro.n)]
        sm = rw.FakeState(invalid={nm: 0 for nm in names[S // 4: S // 2]}, discovered=[b"chan%07d" % i for i in range(N_DISC)],
                          seeds={nm: 1 for nm in names[: S // 4]})
        pages = [(owners[p % len(owners)], [0, 0], links[2 * p: 2 * p + 2], 2) for p in range(S)]
        n_look = [0]

        def search(name, record, src):
            n_look[0] += 1
            return (rw.FOUND if n_look[0] % 2 == 0 else rw.NOT_FOUND), n_look[0] - 1
        t0 = time.perf_counter()
        rw.run(sm, pages, search, NOW, RATE, 17, 0, CRAWL, sr.discovery_time(NOW, 0))
        host_ms = (time.perf_counter() - t0) * 1e3
        print(f"S = {S:>6} pages: " + " | ".join(
            f"k = {k}: lookups {v[0]:.3f} ms (device {v[1]:.3f} ms, {v[4][2]} launches, {v[4][0]} lookups), step "
            f"{v[2]:.3f} ms (device {v[3]:.3f} ms, {v[4][3]} launches, {v[4][1]} statements)" for k, v in res.items())
            + f" | Python restatement {host_ms:.1f} ms", flush=True)
        e.close()


if __name__ == "__main__":
    main()
