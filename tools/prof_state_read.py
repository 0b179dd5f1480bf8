"""Cost of reading a layer's pages with their message lists, on a resident state of 10^5 pages x 100 messages whose
layer at depth 2 holds 10^4 of them:

  layer       one tgi_state_read_layer of the 10^4-page layer with TGI_READ_MESSAGES (and a selection);
  per page    the same pages' lists by 10^4 tgi_state_read_page calls, each a pass over every message row.

Host clock of the C calls, device time and launches.  tgi_state_read_page reports no device time: its gather is the n = 1
case of tgi_state_read_pages, whose kernel time and launches stand for each of the 10^4 calls.  Prints the card and its
power limit, checks that both ways return the same lists, and gives medians over the repetitions.

    python tools/prof_state_read.py [--reps 5]
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

from distributed_crawler_b200 import abi  # noqa: E402
from distributed_crawler_b200.engine import Engine, lib  # noqa: E402
from prof_state import card, state_arrays  # noqa: E402

N_PAGES, PER_PAGE, LAYER = 100_000, 100, 10_000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(f"card: {card()}")
    e = Engine()
    _, recs, blob, msgs = state_arrays(N_PAGES, PER_PAGE)
    recs["depth"][N_PAGES - LAYER:] = 2
    layers = np.array([(1, N_PAGES - LAYER), (2, LAYER)], abi.STATE_LAYER)
    e.state_set_arrays(layers, recs, blob, msgs)
    rows = list(range(N_PAGES - LAYER, N_PAGES))

    host, dev, launches = [], [], 0
    for rep in range(a.reps + 1):  # one warm-up
        out = abi.StateReadC()
        t0 = time.perf_counter()
        e._check(lib().tgi_state_read_layer(e.h, 2, abi.SELECT_STANDALONE_RESUME, abi.READ_MESSAGES, C.byref(out)))
        t1 = time.perf_counter()
        if rep:
            host.append((t1 - t0) * 1e3)
            dev.append(out.kernel_ms)
        launches = out.gpu_launches
    assert out.n_pages == LAYER and out.n_msgs == LAYER * PER_PAGE
    got = e.state_read_layer_arrays(2)
    print(f"read_layer of {LAYER} pages, {LAYER * PER_PAGE} messages: host {statistics.median(host):.3f} ms, "
          f"device {statistics.median(dev):.3f} ms, {launches} launches")

    one_dev, one_launches = [], 0
    for rep in range(a.reps + 1):
        e.state_read_pages_arrays([rows[rep]])
        if rep:
            one_dev.append(e.state_read_ms)
        one_launches = e.state_read_launches
    buf = np.zeros(PER_PAGE, abi.STATE_MSG)
    n = C.c_uint64()
    lists = []
    t0 = time.perf_counter()
    for r in rows:
        e._check(lib().tgi_state_read_page(e.h, r, buf.ctypes.data, PER_PAGE, C.byref(n)))
        lists.append(buf[:n.value].copy())
    t1 = time.perf_counter()
    assert all(np.array_equal(x, got["msgs"][int(f):int(f) + PER_PAGE]) for x, f in zip(lists, got["msg_first"]))
    d1 = statistics.median(one_dev)
    print(f"{LAYER} x read_page: host {(t1 - t0) * 1e3:.1f} ms ({(t1 - t0) * 1e3 / LAYER:.3f} ms per call), device "
          f"{d1:.3f} ms per call = {d1 * LAYER:.1f} ms, {one_launches} launches per call = {one_launches * LAYER}")
    print(f"same lists: yes; host ratio {(t1 - t0) * 1e3 / statistics.median(host):.0f}x")
    e.close()


if __name__ == "__main__":
    main()
