"""Cost of the resident crawl state (tgi_state_*): state.json renders and one batched UpdateMessage call.

  render   100 k pages x 100 messages (10 M) and 1 page x 10^6 messages: the render's device time (kernel_ms: size pass
           and emit, not the read-back), the state.json bytes written over that time as a share of the H100's
           3.35 TB/s, and the whole tgi_state_render call on the host clock, read-back into pinned memory included;
  update   one tgi_state_update_messages call of 100 updates (the messages of one page, half of them new keys) on the
           100 k-page state, host clock.
Prints the card and its power limit, and the median and spread of each.

    python tools/prof_state.py [--reps 9]
"""
import argparse
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from distributed_crawler_b200 import abi  # noqa: E402
from distributed_crawler_b200.engine import Engine  # noqa: E402

PEAK = 3.35e12
META, LAST = b'{"crawlId":"c","executionId":"e","startTime":"2024-01-01T00:00:00Z","status":"running"}', b'"2024-01-02T03:04:05Z"'


def card():
    q = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"]
    return subprocess.check_output(q).decode().strip().splitlines()[0]


def state_arrays(n_pages, per_page):
    """n_pages pages (uuid-length ids, t.me URLs, time.Local timestamps) with per_page messages each"""
    ids = [b"%08x-0000-4000-8000-%012x" % (p, p) for p in range(n_pages)]
    urls = [b"https://t.me/channel_%07d" % p for p in range(n_pages)]
    recs = np.zeros(n_pages, abi.STATE_PAGE)
    recs["str_len"][:, 0] = [len(i) for i in ids]
    recs["str_len"][:, 1] = [len(u) for u in urls]
    recs["str_len"][:, 2] = 7
    recs["str_off"] = np.concatenate([[0], np.cumsum(recs["str_len"].sum(1).astype(np.uint64))[:-1]])
    blob = np.frombuffer(b"".join(i + u + b"fetched" for i, u in zip(ids, urls)) + b"\0" * 16, np.uint8)
    recs["depth"] = 1
    recs["ts_sec"] = 1700000000 + np.arange(n_pages)
    recs["ts_nsec"] = 123456789
    recs["ts_off"] = abi.STATE_TS_LOCAL
    recs["n_msgs"] = per_page
    msgs = np.zeros(n_pages * per_page, abi.STATE_MSG)
    msgs["chat_id"] = np.repeat(-1001000000000 - np.arange(n_pages, dtype=np.int64), per_page)
    msgs["message_id"] = np.tile(np.arange(per_page, dtype=np.int64) << 20, n_pages)
    msgs["page_id"] = np.repeat(np.arange(n_pages, dtype=np.uint32), per_page)
    msgs["status"] = 2
    return np.array([(1, n_pages)], abi.STATE_LAYER), recs, blob, msgs


def spread(xs):
    xs = sorted(xs)
    return f"median {statistics.median(xs):9.3f}  min {xs[0]:9.3f}  max {xs[-1]:9.3f}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    a = ap.parse_args()
    print(f"card: {card()}")
    e = Engine()
    for n_pages, per_page in ((100_000, 100), (1, 1_000_000)):
        e.state_set_arrays(*state_arrays(n_pages, per_page))
        ms, wall = [], []
        for rep in range(a.reps + 2):  # two warm-up renders
            t0 = time.perf_counter()
            out = e.state_render(META, LAST, copy=False)
            dt = (time.perf_counter() - t0) * 1e3
            if rep >= 2:
                ms.append(e.state_render_ms)
                wall.append(dt)
        body = len(out) - len(META) - len(LAST) - 40  # the bytes the device wrote (the frame is the host's)
        k = statistics.median(ms)
        print(f"render {n_pages} pages x {per_page} messages: {len(out)} B state.json, {e.state_render_launches} launches")
        print(f"  kernel ms {spread(ms)}  -> {body / (k * 1e-3) / 1e9:.1f} GB/s written = {body / (k * 1e-3) / PEAK:.1%} of 3.35 TB/s")
        print(f"  whole call incl. read-back, wall ms {spread(wall)}")
        if n_pages == 100_000:
            rng = np.random.default_rng(1)
            walls = []
            for rep in range(a.reps + 2):
                row = int(rng.integers(n_pages))
                u = np.zeros(100, abi.STATE_UPDATE)
                u["row"] = row
                u["chat_id"] = -1001000000000 - row
                u["message_id"] = (np.arange(100, dtype=np.int64) * 2 + 1000 * rep) << 20  # half inside the page's 100
                u["status"] = 2
                t0 = time.perf_counter()
                e.state_update_arrays(u)
                dt = (time.perf_counter() - t0) * 1e3
                if rep >= 2:
                    walls.append(dt)
            print(f"update_messages, 100 updates on the {n_pages}-page state: wall ms {spread(walls)}")
    e.close()


if __name__ == "__main__":
    main()
