"""Cost of the tandem hand-off's binding calls (tgi_state_edge_sql) after one tgi_state_pending_edges over a bulk
Telegram result of P pages x 100 messages, left on the device (TGI_RUN_NO_D2H), on a resident state of 10^3 pages, at
the corpus's link rate and at a link-heavy rate (12 t.me links per message from a pool of 5,000 names):

  device      one tgi_state_edge_sql call at 1 and at 8191 rows per statement through the C ABI: host clock (the
              params read back into pinned memory included), device time, launches, statements and bytes;
  host        the same calls restated in Python (tests/tandem_sql_rules.py: json.Marshal of every row's []any, one call
              per row) from the hand-off's rows and the owners' strings, which the Go shim would have to look up.  This
              only bounds the Go shim's cost from above; Go itself is not measured.

Prints the card and its power limit, and the median over the repetitions (the host restatement runs once).

    python tools/prof_state_edge_sql.py [--reps 5]
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
from distributed_crawler_b200.corpus import Corpus  # noqa: E402
from distributed_crawler_b200 import abi  # noqa: E402
from distributed_crawler_b200.engine import Engine, lib  # noqa: E402
from prof_state import card, state_arrays  # noqa: E402
from prof_state_pending_edges import NOW, PER_PAGE, RUN, link_batch  # noqa: E402

CRAWL = b"crawl-2025-10-17"


def host_calls(e, got, spans):
    """the reference's per-row calls, marshalled in Python from the hand-off and the owners' strings"""
    rows = sorted({spans[b["span"]][0] for b in got["batches"]})
    own = dict(zip(rows, e.state_read_pages(rows, messages=False)))  # a state call: after the device renders
    t0 = time.perf_counter()
    pages = []
    for b in got["batches"]:
        o = own[spans[b["span"]][0]]
        bt = {"batch_id": bytes(b["batch_id"]), "source_channel": o["url"], "source_page_id": o["id"],
              "source_depth": o.get("depth", 0), "sequence_id": o.get("sequenceId", b"")}
        es = got["edges"][b["first_edge"]:b["first_edge"] + b["n_edges"]]
        pages.append((bt, [{"destination": bytes(x["destination"][:x["dest_len"]]), "source_type": int(x["source_type"]),
                            "status": int(x["status"])} for x in es]))
    calls = sr.reference_calls(pages, CRAWL, sr.discovery_time(NOW, 0))
    return (time.perf_counter() - t0) * 1e3, len(calls)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(f"card: {card()}")
    rng = np.random.default_rng(3)
    n_pages = 1_000
    e = Engine(set_growth=1 << 22)
    e.state_id_seed(11)
    layers, recs, blob, msgs = state_arrays(n_pages, PER_PAGE)
    e.state_set_arrays(layers, recs, blob, msgs)
    for rate in ("corpus", "links"):
        for P in (1, 100, 1000):
            n = P * PER_PAGE
            b = Corpus(n, profile=2, nthreads=2, first=0).batch if rate == "corpus" else link_batch(n, rng)
            e.telegram_submit(0, b, RUN)
            e.telegram_wait(0)
            res = {k: [] for k in ("k1", "k1_ms", "kmax", "kmax_ms")}
            info = {}
            host_ms = n_calls = 0
            for rep in range(a.reps + 1):  # one warm-up
                rows = [int(x) for x in rng.choice(n_pages, P, replace=False)]
                spans = [(r, PER_PAGE * k, PER_PAGE, PER_PAGE) for k, r in enumerate(rows)]
                got = e.state_pending_edges(0, spans, NOW)
                for key, k in (("k1", 1), ("kmax", sr.MAX_ROWS)):
                    out = abi.StateEdgeSqlC()
                    t0 = time.perf_counter()
                    rc = lib().tgi_state_edge_sql(e.h, CRAWL, len(CRAWL), NOW, 0, k, C.byref(out))
                    t1 = time.perf_counter()
                    assert rc == 0
                    if rep:
                        res[key].append((t1 - t0) * 1e3)
                        res[key + "_ms"].append(out.kernel_ms)
                    info[key] = (int(out.n_stmts), int(out.data_len), int(out.gpu_launches))
                if rep == 1:
                    host_ms, n_calls = host_calls(e, got, spans)
                edges = len(got["edges"])
            e.release(0)
            med = {k: statistics.median(v) for k, v in res.items()}
            print(f"{rate:>6} rate, P = {P:>4}, {edges:>7} edges: k = 1 call {med['k1']:.3f} ms (device "
                  f"{med['k1_ms']:.3f} ms, {info['k1'][2]} launches, {info['k1'][0]} statements, {info['k1'][1]} bytes) | k = {sr.MAX_ROWS} call {med['kmax']:.3f} ms (device {med['kmax_ms']:.3f} ms, "
                  f"{info['kmax'][0]} statements) | Python restatement {host_ms:.1f} ms for {n_calls} calls", flush=True)
    e.close()


if __name__ == "__main__":
    main()
