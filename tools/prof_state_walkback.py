"""Cost of the tandem forced walkback (tgi_state_walkback) after one tgi_state_pending_edges whose S spans all have no
edges, on a resident state of 10^3 pages and a discovered set of 10^5 channels:

  device      the first tgi_state_walkback call on a hand-off (the picks and the rows) at 1 row per statement, and a
              repeated call at 8191 rows per statement (the rows only), through the C ABI: host clock (the picks and
              params read back into pinned memory included), device time, launches, statements and bytes;
  host        the same branch restated in Python (tests/walkback_rules.py: the pick, then json.Marshal of the two
              rows' []any, one call per row) from the owners' strings and a Python copy of the discovered list, which
              the Go shim would have to keep.  This only bounds the Go shim's cost from above; Go itself is not
              measured.

Prints the card and its power limit, and the median over the repetitions (the host restatement runs once).

    python tools/prof_state_walkback.py [--reps 5]
"""
import argparse
import ctypes as C
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import tandem_sql_rules as sr  # noqa: E402
import walkback_rules as wr  # noqa: E402
from distributed_crawler_b200 import abi  # noqa: E402
from distributed_crawler_b200.engine import Engine, lib, names_to_keys32  # noqa: E402
from distributed_crawler_b200.pack import pack_telegram  # noqa: E402
from helpers import msg  # noqa: E402
from prof_state import card, state_arrays  # noqa: E402

CRAWL = b"crawl-2025-10-17"
NOW = 1_760_000_000
N_DISC = 100_000


def host_calls(e, spans, keys, seed, w0):
    """the reference's branch per span, restated in Python from the owners' strings"""
    rows = sorted({r for r, *_ in spans})
    own = dict(zip(rows, e.state_read_pages(rows, messages=False)))  # a state call: after the device renders
    t = sr.discovery_time(NOW, 0)
    t0 = time.perf_counter()
    n_calls = 0
    for j, (r, *_) in enumerate(spans):
        n_calls += len(wr.forced_walkback(own[r], keys, seed, w0 + j, CRAWL, t)[1])
    return (time.perf_counter() - t0) * 1e3, n_calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(f"card: {card()}")
    rng = np.random.default_rng(5)
    n_pages, seed = 1_000, 11
    e = Engine(set_growth=1 << 22)
    e.state_id_seed(seed)
    layers, recs, blob, msgs = state_arrays(n_pages, 1)
    e.state_set_arrays(layers, recs, blob, msgs)
    keys = [b"chan%07d" % i for i in range(N_DISC)]
    e.set_add(abi.SET_DISCOVERED, names_to_keys32(keys))
    e.telegram_submit(0, pack_telegram([msg("messageText", "t.me/chan0000001", id=1 << 20, chat_id=-1, date=NOW)]),
                      abi.RUN_LINKS | abi.RUN_NO_D2H)
    e.telegram_wait(0)
    w = 0
    for S in (1_000, 100_000):
        res = {k: [] for k in ("first", "first_ms", "again", "again_ms")}
        info = {}
        host_ms = n_calls = 0
        for rep in range(a.reps + 1):  # one warm-up
            spans = [(int(r), 0, 1, 0) for r in rng.integers(0, n_pages, S)]
            e.state_pending_edges(0, spans, NOW)
            for key, k in (("first", 1), ("again", wr.MAX_ROWS)):
                out = abi.StateWalkbackC()
                t0 = time.perf_counter()
                rc = lib().tgi_state_walkback(e.h, CRAWL, len(CRAWL), NOW, 0, k, C.byref(out))
                t1 = time.perf_counter()
                assert rc == 0
                if rep:
                    res[key].append((t1 - t0) * 1e3)
                    res[key + "_ms"].append(out.kernel_ms)
                info[key] = (int(out.n_stmts), int(out.data_len), int(out.gpu_launches))
            if rep == 1:
                host_ms, n_calls = host_calls(e, spans, keys, seed, w)
            w += S
        med = {k: statistics.median(v) for k, v in res.items()}
        print(f"S = {S:>6} edge-less spans: first call, k = 1: {med['first']:.3f} ms (device {med['first_ms']:.3f} ms, "
              f"{info['first'][2]} launches, {info['first'][0]} statements, {info['first'][1]} bytes) | repeated call, "
              f"k = {wr.MAX_ROWS}: {med['again']:.3f} ms (device {med['again_ms']:.3f} ms, {info['again'][0]} "
              f"statements) | Python restatement {host_ms:.1f} ms for {n_calls} calls", flush=True)
    e.release(0)
    e.close()


if __name__ == "__main__":
    main()
