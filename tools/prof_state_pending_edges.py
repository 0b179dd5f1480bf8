"""Cost of the tandem hand-off (tgi_state_pending_edges) for one bulk Telegram result of P pages x 100 messages, left on
the device (TGI_RUN_NO_D2H), on resident states of 10^3 and 10^5 pages, at the corpus's link rate and at a
link-heavy rate (12 t.me links per message from a pool of 5,000 names), with 1,000 invalid and 1,000 discovered names
in the exclusion sets:

  device      one tgi_state_pending_edges call over the P spans: host clock, device time, launches;
  host        the sequence it replaces: tgi_result_read_rows of the statuses, link offsets and link rows, then the
              per-page loop in Python (self compare with the owner URL, invalid TTL, FilterUsername, seenInBatch, one
              uuid4 per batch).  Like the discovery profile's, this bounds the Go shim's cost from above.

Prints the card and its power limit, and the median over the repetitions.

    python tools/prof_state_pending_edges.py [--reps 5]
"""
import argparse
import os
import statistics
import sys
import time
import uuid

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from distributed_crawler_b200 import abi  # noqa: E402
from distributed_crawler_b200.corpus import Corpus  # noqa: E402
from distributed_crawler_b200.engine import Engine, names_to_keys32  # noqa: E402
from distributed_crawler_b200.pack import pack_telegram  # noqa: E402
from helpers import msg  # noqa: E402
from prof_state import card, state_arrays  # noqa: E402

PER_PAGE = 100
RUN = abi.RUN_LINKS | abi.RUN_NO_D2H
NOW = 1_760_000_000
TTL = 30 * 24 * 3600


def link_batch(n, rng):
    pool = ["name%05d" % k for k in range(5_000)]
    ms = [msg("messageText", " ".join("t.me/" + pool[j] for j in rng.integers(0, len(pool), 12)), id=(k + 1) << 20,
              chat_id=-5, date=1_700_000_000) for k in range(n)]
    return pack_telegram(ms)


def host_loop(e, slot, n, spans, urls, invalid, discovered):
    """the read-back and the per-page loop of runner.go:1129, 1229-1306"""
    status = e.read_rows(slot, abi.ROWS_STATUS, 0, n)
    off = e.read_rows(slot, abi.ROWS_LINK_OFF, 0, n + 1)
    links = e.read_rows(slot, abi.ROWS_LINKS, 0, int(off[n]))
    names = [bytes(l["name"][:l["len"]]) for l in links]
    ok = (links["flags"] & abi.LF_FILTER_OK) != 0
    out = []
    for row, first, n_rec, n_done in spans:
        owner, seen, batch = urls[row], set(), None
        for i in range(first, first + n_done):
            if status[i] not in (abi.ST_EMITTED, abi.ST_NOLINE):
                continue
            for k in range(int(off[i]), int(off[i + 1])):
                o = names[k]
                if o == owner or (o in invalid and NOW - invalid[o] < TTL) or not ok[k] or o in seen:
                    continue
                seen.add(o)
                if batch is None:
                    batch = str(uuid.uuid4())
                out.append((batch, o, i, int(links[k]["src"]), o in discovered))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(f"card: {card()}")
    rng = np.random.default_rng(3)
    batches = {}
    for n_pages in (1_000, 100_000):
        e = Engine(set_growth=1 << 22)
        e.state_id_seed(11)
        layers, recs, blob, msgs = state_arrays(n_pages, PER_PAGE)
        e.state_set_arrays(layers, recs, blob, msgs)
        urls = [b"https://t.me/channel_%07d" % p for p in range(n_pages)]
        inv = [b"name%05d" % k for k in range(0, 5_000, 5)]
        disc = [b"name%05d" % k for k in range(1, 5_000, 5)]
        stamps = rng.choice([0, NOW - 40 * 86400, NOW - 86400], len(inv)).astype(np.int64)
        e.set_add(abi.SET_INVALID, names_to_keys32(inv), stamps)
        e.set_add(abi.SET_DISCOVERED, names_to_keys32(disc))
        invalid, discovered = dict(zip(inv, stamps.tolist())), set(disc)
        for rate in ("corpus", "links"):
            for P in (1, 100, 1000):
                n = P * PER_PAGE
                if (rate, n) not in batches:
                    batches[(rate, n)] = (Corpus(n, profile=2, nthreads=2, first=0).batch if rate == "corpus"
                                          else link_batch(n, rng))
                e.telegram_submit(0, batches[(rate, n)], RUN)
                e.telegram_wait(0)
                res = {k: [] for k in ("device", "device_ms", "host")}
                n_edges = n_batches = launches = 0
                for rep in range(a.reps + 1):  # one warm-up
                    rows = [int(x) for x in rng.choice(n_pages, P, replace=False)]
                    spans = [(r, PER_PAGE * k, PER_PAGE, PER_PAGE) for k, r in enumerate(rows)]
                    t0 = time.perf_counter()
                    got = e.state_pending_edges(0, spans, NOW)
                    t1 = time.perf_counter()
                    host_loop(e, 0, n, spans, urls, invalid, discovered)
                    t2 = time.perf_counter()
                    if rep:
                        res["device"].append((t1 - t0) * 1e3)
                        res["device_ms"].append(e.state_edges_ms)
                        res["host"].append((t2 - t1) * 1e3)
                    n_edges, n_batches, launches = len(got["edges"]), len(got["batches"]), e.state_edges_launches
                e.release(0)
                med = {k: statistics.median(v) for k, v in res.items()}
                print(f"{n_pages:>7} pages, {rate:>8} rate, P = {P:>4}: call {med['device']:.3f} ms (device "
                      f"{med['device_ms']:.3f} ms, {launches} launches, {n_edges} edges, {n_batches} batches) | host "
                      f"read-back + loop {med['host']:.3f} ms", flush=True)
        e.close()


if __name__ == "__main__":
    main()
