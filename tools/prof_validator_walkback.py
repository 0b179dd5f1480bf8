"""Cost of the validator walkback (tgi_state_validator_walkback) for B claimed batches of about 8 edges each (a quarter
valid, four source types), at walkback rate 15 with a discovered set of 10^5 channels:

  device      one call at 1 and at 8191 rows per statement through the C ABI, the batches packed beforehand: host
              clock (upload, picks, rows and read-back into pinned memory), device time, launches, statements and bytes;
  host        the same batches restated in Python (tests/validator_walkback_rules.py: the decision, the pick, and
              json.Marshal of each call's []any, one call per row), once.  This only bounds the Go shim's cost from
              above; Go itself is not measured.

Prints the card and its power limit, and the median over the repetitions.

    python tools/prof_validator_walkback.py [--reps 5] [--sizes 1000 100000]
"""
import argparse
import ctypes as C
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import tandem_sql_rules as sr  # noqa: E402
import validator_walkback_rules as vr  # noqa: E402
from distributed_crawler_b200 import abi  # noqa: E402
from distributed_crawler_b200.engine import Engine, lib, names_to_keys32  # noqa: E402
from distributed_crawler_b200.state_pack import pack_claimed_batches  # noqa: E402
from prof_state import card  # noqa: E402

CRAWL = b"crawl-2025-10-17"
NOW = 1_760_000_000
N_DISC = 100_000
RATE = 15
TYPES = [b"mention", b"text_url", b"url", b"plaintext"]
STATUSES = [b"valid", b"not_channel", b"invalid", b"duplicate"]


def claimed(n):
    return [{"batch_id": b"%08d-0000-4000-8000-000000000000" % i, "crawl_id": CRAWL, "source_channel": b"src%07d" % i,
             "source_page_id": b"%08d-1111-4000-8000-000000000000" % i, "source_depth": i % 50,
             "sequence_id": b"%08d-2222-4000-8000-000000000000" % (i // 4),
             "edges": [(b"dest%07d_%d" % (i, j), TYPES[(i + j) % 4], STATUSES[(i * 3 + j) % 4])
                       for j in range(6 + i % 5)]} for i in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", type=int, nargs="+", default=[1_000, 100_000])
    a = ap.parse_args()
    print(f"card: {card()}")
    seed = 11
    e = Engine(set_growth=1 << 22)
    e.state_id_seed(seed)
    keys = [b"chan%07d" % i for i in range(N_DISC)]
    e.set_add(abi.SET_DISCOVERED, names_to_keys32(keys))
    for B in a.sizes:
        batches = claimed(B)
        recs, eoff, edges, blob = pack_claimed_batches(batches)
        cin = abi.ClaimedBatchesC(B, 0, recs.ctypes.data, eoff.ctypes.data, edges.ctypes.data, len(edges),
                                  blob.ctypes.data, len(blob))
        res, info = {}, {}
        for k in (1, vr.MAX_ROWS):
            wall, dev = [], []
            for rep in range(a.reps + 1):  # one warm-up
                out = abi.StateValidatorWalkbackC()
                t0 = time.perf_counter()
                rc = lib().tgi_state_validator_walkback(e.h, C.byref(cin), RATE, CRAWL, len(CRAWL), NOW, 0, k,
                                                        C.byref(out))
                t1 = time.perf_counter()
                assert rc == 0, rc
                if rep:
                    wall.append((t1 - t0) * 1e3)
                    dev.append(out.kernel_ms)
                info[k] = (int(out.n_stmts), int(out.data_len), int(out.gpu_launches))
            res[k] = (statistics.median(wall), statistics.median(dev))
        t = sr.discovery_time(NOW, 0)
        t0 = time.perf_counter()
        n_calls = sum(len(c) for _, c in vr.run(batches, keys, RATE, seed, 0, CRAWL, t))
        host_ms = (time.perf_counter() - t0) * 1e3
        print(f"B = {B:>6} batches ({len(edges)} edges): " + " | ".join(
            f"k = {k}: {res[k][0]:.3f} ms (device {res[k][1]:.3f} ms, {info[k][2]} launches, {info[k][0]} statements, "
            f"{info[k][1]} bytes)" for k in res) + f" | Python restatement {host_ms:.1f} ms for {n_calls} calls",
            flush=True)
    e.close()


if __name__ == "__main__":
    main()
