"""Cost of one page turn (processAllMessagesWithProcessor's bookkeeping for a fetched page of 100 messages, half of them
already in the page's list) on resident states of 10^3 and 10^5 pages x 100 messages, host clock per turn:

  turn        tgi_state_page_begin + tgi_state_page_end (statuses from the host), without and with TGI_TURN_PAGE_JSON;
  host shim   the sequence the shim ran before the turn entry points: tgi_state_read_page, the two tgi_key_join calls
              of addNewMessages and resampleMarker, tgi_state_update_page with the new list, and
              tgi_state_update_messages with the loop's (swapped) keys.

The turn touches only the page's messages, so its time should not grow with the state; read_page scans every message
row.  Prints the card and its power limit, and the median and spread of each.

    python tools/prof_state_turn.py [--reps 50]
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
    """the page's fetch: message ids 50..149 (+ a drift per rep), so about half are in its list"""
    f = np.zeros((PER_PAGE, 2), np.int64)
    f[:, 0] = -1001000000000 - row
    f[:, 1] = (np.arange(PER_PAGE, dtype=np.int64) + 50 + rep % 7) << 20
    return f


def shim_turn(e, row, rec, blob, fetched, status):
    """the host sequence: GetPage, addNewMessages / resampleMarker by key_join, UpdatePage, UpdateMessages"""
    old = e.state_read_page_arrays(row)
    ek = np.stack([old["chat_id"], old["message_id"]], 1)
    new = np.nonzero(e.key_join(ek, fetched) < 0)[0]
    keys = fetched[new]
    e.key_join(fetched, keys)  # resampleMarker: every new key is among the discovered, so all become "resample"
    msgs = np.zeros(len(keys), abi.STATE_MSG)
    msgs["chat_id"], msgs["message_id"] = keys[:, 0], keys[:, 1]
    msgs["page_id"], msgs["status"] = abi.STATE_NO_PAGE, 5
    r = rec.copy()
    r["n_msgs"] = len(keys)
    out = C.c_uint32()
    e._check(lib().tgi_state_update_page(e.h, r.ctypes.data, blob.ctypes.data, len(blob),
                                         msgs.ctypes.data if len(msgs) else None, C.byref(out)))
    u = np.zeros(len(keys), abi.STATE_UPDATE)
    u["chat_id"], u["message_id"], u["row"] = keys[:, 1], keys[:, 0], row
    u["status"] = np.where(status[:len(keys)] == abi.ST_FAILED, 3, 2)
    e.state_update_arrays(u)


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
        for name in ("turn", "turn+json", "host shim"):
            walls = []
            for rep in range(a.reps + 3):  # three warm-up turns
                row = int(rng.integers(n_pages))
                f = fetch(row, rep)
                t0 = time.perf_counter()
                if name == "host shim":
                    shim_turn(e, row, recs[row:row + 1], blob, f, status)
                else:
                    h, work, _ = e.state_page_begin(row, f, None, name == "turn+json")
                    e.state_page_end(h, len(work), status=status[:len(work)])
                dt = (time.perf_counter() - t0) * 1e3
                if rep >= 3:
                    walls.append(dt)
            print(f"{n_pages:>7} pages x {PER_PAGE}: {name:<10} wall ms per turn {spread(walls)}")
        e.close()


if __name__ == "__main__":
    main()
