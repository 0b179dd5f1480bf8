"""Cost of one page close (UpdatePage(*owner) after a page turn of 100 fetched messages, none of them in the page's
list) on resident states of 10^3 and 10^5 pages x 100 messages, host clock per close:

  close       tgi_state_page_close after an untimed begin + end, without and with TGI_TURN_PAGE_JSON; its device time
              and launches;
  host seq    the sequence it replaces: tgi_state_read_page for the page's list, then tgi_state_update_page with the
              owner's part of it.

The close touches only the page's view, so its time should not grow with the state; read_page scans every message
row.  Prints the card, its power limit and max SM clock, and the median and spread of each.

    python tools/prof_state_close.py [--reps 50]
"""
import argparse
import ctypes as C
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from distributed_crawler_b200 import abi  # noqa: E402
from distributed_crawler_b200.engine import Engine, lib  # noqa: E402
from prof_state import card, spread, state_arrays  # noqa: E402

PER_PAGE = 100


def fetch(row, rep):
    """the page's fetch: message ids past the state's, so every key is new and the owner holds 100 messages"""
    f = np.zeros((PER_PAGE, 2), np.int64)
    f[:, 0] = -1001000000000 - row
    f[:, 1] = (np.arange(PER_PAGE, dtype=np.int64) + 1000 * (rep + 1)) << 20
    return f


def close(e, row, rec, blob, flags):
    out = abi.StateJsonC()
    e._check(lib().tgi_state_page_close(e.h, row, rec.ctypes.data, blob.ctypes.data, len(blob), flags, C.byref(out)))
    return out


def host_seq(e, row, rec, blob, k):
    """GetPage, then UpdatePage with the owner's k messages"""
    old = e.state_read_page_arrays(row)[:k].copy()
    old["page_id"] = abi.STATE_NO_PAGE
    r = rec.copy()
    r["n_msgs"] = len(old)
    out = C.c_uint32()
    e._check(lib().tgi_state_update_page(e.h, r.ctypes.data, blob.ctypes.data, len(blob),
                                         old.ctypes.data if len(old) else None, C.byref(out)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    print(f"card: {card()}")
    rng = np.random.default_rng(1)
    status = rng.choice(np.array([abi.ST_EMITTED, abi.ST_SKIPPED, abi.ST_FAILED], np.uint8), PER_PAGE)
    for n_pages in (1_000, 100_000):
        e = Engine()
        layers, recs, blob, msgs = state_arrays(n_pages, PER_PAGE)
        e.state_set_arrays(layers, recs, blob, msgs)
        for name in ("close", "close+json", "host seq"):
            walls, dev, launches = [], [], 0
            for rep in range(a.reps + 3):  # three warm-up closes
                row = int(rng.integers(n_pages))
                h, work, _ = e.state_page_begin(row, fetch(row, rep))
                e.state_page_end(h, len(work), status=status[:len(work)])
                rec = recs[row:row + 1].copy()
                rec["n_msgs"] = 0
                t0 = time.perf_counter()
                if name == "host seq":
                    host_seq(e, row, rec, blob, len(work))
                else:
                    out = close(e, row, rec, blob, abi.TURN_PAGE_JSON if name == "close+json" else 0)
                dt = (time.perf_counter() - t0) * 1e3
                if rep >= 3:
                    walls.append(dt)
                    if name != "host seq":
                        dev.append(float(out.kernel_ms))
                        launches = int(out.gpu_launches)
            line = f"{n_pages:>7} pages x {PER_PAGE}: {name:<10} wall ms per close {spread(walls)}"
            if dev:
                line += f"; device ms {spread(dev)}, {launches} launches"
            print(line)
        e.close()


if __name__ == "__main__":
    main()
