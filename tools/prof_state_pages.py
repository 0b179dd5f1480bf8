"""Cost of multi-page turns against the one-page calls, on resident states of 10^3 and 10^5 pages x 100 messages with P
pages of 100 fetched messages each (about half of them already in the page's list), host clock and device time per call:

  batched     tgi_state_pages_begin, tgi_state_pages_end with the statuses of a resident bulk Telegram result
              (TGI_RUN_JSONL_DEVICE, records [0, n_work)), tgi_state_pages_close;
  one-page    P tgi_state_page_begin, one read-back of the result's statuses, P tgi_state_page_end with host statuses,
              P tgi_state_page_close: the only path for a bulk result before the batched calls.

Prints the card and its power limit, and the median of each step over the repetitions.

    python tools/prof_state_pages.py [--reps 5]
"""
import argparse
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from distributed_crawler_b200 import abi  # noqa: E402
from distributed_crawler_b200.corpus import Corpus  # noqa: E402
from distributed_crawler_b200.engine import Engine  # noqa: E402
from prof_state import card, state_arrays  # noqa: E402

PER_PAGE = 100
RUN = abi.RUN_JSONL | abi.RUN_JSONL_DEVICE


def fetch(row, rep):
    f = np.zeros((PER_PAGE, 2), np.int64)
    f[:, 0] = -1001000000000 - row
    f[:, 1] = (np.arange(PER_PAGE, dtype=np.int64) + 50 + rep % 7) << 20
    return f


def page_of(recs, blob, row):
    o = int(recs[row]["str_off"])
    return {"id": bytes(blob[o:o + 36]), "url": bytes(blob[o + 36:o + 36 + int(recs[row]["str_len"][1])]),
            "status": b"fetched", "depth": 1, "timestamp": (1700000000, 0, 0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(f"card: {card()}")
    rng = np.random.default_rng(3)
    batches = {}
    for n_pages in (1_000, 100_000):
        e = Engine()
        layers, recs, blob, msgs = state_arrays(n_pages, PER_PAGE)
        e.state_set_arrays(layers, recs, blob, msgs)
        for P in (1, 10, 100, 1000):
            if P > n_pages:
                continue
            res = {k: [] for k in ("begin", "end", "close", "1-begin", "1-read", "1-end", "1-close")}
            dev = {k: [] for k in ("begin", "end", "close")}
            launches = {}
            for rep in range(a.reps + 1):  # one warm-up
                rows = [int(x) for x in rng.choice(n_pages, P, replace=False)]
                fetched = [fetch(r, rep) for r in rows]
                pages = [page_of(recs, blob, r) for r in rows]
                # batched
                t0 = time.perf_counter()
                h, work, off, _ = e.state_pages_begin(rows, fetched)
                t1 = time.perf_counter()
                dev_b, launches["begin"] = e.state_pages_ms, e.state_pages_launches
                n_work = len(work)
                if n_work not in batches:
                    batches[n_work] = Corpus(max(n_work, 1), profile=2, nthreads=2, first=0).batch
                e.telegram_submit(0, batches[n_work], RUN)
                e.telegram_wait(0)
                t2 = time.perf_counter()
                e.state_pages_end(h, None, slot=0, first=0)
                t3 = time.perf_counter()
                dev_e, launches["end"] = e.state_pages_ms, e.state_pages_launches
                e.state_pages_close(rows, pages)
                t4 = time.perf_counter()
                dev_c, launches["close"] = e.state_pages_ms, e.state_pages_launches
                e.release(0)
                # one page at a time, the same work
                rows = [int(x) for x in rng.choice(n_pages, P, replace=False)]
                fetched = [fetch(r, rep + 1) for r in rows]
                pages = [page_of(recs, blob, r) for r in rows]
                s0 = time.perf_counter()
                turns = [e.state_page_begin(r, f)[:2] for r, f in zip(rows, fetched)]
                s1 = time.perf_counter()
                n_work = sum(len(w) for _, w in turns)
                if n_work not in batches:
                    batches[n_work] = Corpus(max(n_work, 1), profile=2, nthreads=2, first=0).batch
                e.telegram_submit(0, batches[n_work], RUN)
                e.telegram_wait(0)
                s2 = time.perf_counter()
                status = e.read_rows(0, abi.ROWS_STATUS, 0, n_work)
                s3 = time.perf_counter()
                i = 0
                for t, w in turns:
                    e.state_page_end(t, len(w), status=status[i:i + len(w)])
                    i += len(w)
                s4 = time.perf_counter()
                for r, p in zip(rows, pages):
                    e.state_page_close(r, p)
                s5 = time.perf_counter()
                e.release(0)
                if rep:
                    for k, v in (("begin", t1 - t0), ("end", t3 - t2), ("close", t4 - t3), ("1-begin", s1 - s0),
                                 ("1-read", s3 - s2), ("1-end", s4 - s3), ("1-close", s5 - s4)):
                        res[k].append(v * 1e3)
                    dev["begin"].append(dev_b)
                    dev["end"].append(dev_e)
                    dev["close"].append(dev_c)
            med = {k: statistics.median(v) for k, v in res.items()}
            print(f"{n_pages:>7} pages x {PER_PAGE}, P = {P:>4}: batched begin {med['begin']:.3f} ms "
                  f"(device {statistics.median(dev['begin']):.3f}, {launches['begin']} launches), end {med['end']:.3f} ms "
                  f"(device {statistics.median(dev['end']):.3f}, {launches['end']} launches), "
                  f"close {med['close']:.3f} ms (device {statistics.median(dev['close']):.3f}, {launches['close']} launches), "
                  f"total {med['begin'] + med['end'] + med['close']:.3f} ms | one-page: begins {med['1-begin']:.3f} ms, "
                  f"read-back {med['1-read']:.3f} ms, ends {med['1-end']:.3f} ms, closes {med['1-close']:.3f} ms, total "
                  f"{med['1-begin'] + med['1-read'] + med['1-end'] + med['1-close']:.3f} ms", flush=True)
        e.close()


if __name__ == "__main__":
    main()
