"""Cost of the local-zone lookup (tgi_set_zone) on the config-2 resident step.

One process, one resident Telegram corpus (profile 2, the bench's config 2 workload, JSONL + links + frontier + skip-self,
results left on the device), run alternately with no zone and with the America/New_York table of
tests/golden/zones.json.  Prints the card, its power limit, and the median and spread of each arm's kernel time.

    python tools/prof_zone.py [--n 2000000] [--reps 15]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from distributed_crawler_b200 import abi  # noqa: E402
from distributed_crawler_b200.corpus import Corpus  # noqa: E402
from distributed_crawler_b200.engine import Engine  # noqa: E402


def card():
    q = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"]
    return subprocess.check_output(q).decode().strip().splitlines()[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2_000_000)
    ap.add_argument("--reps", type=int, default=15)
    a = ap.parse_args()
    with open(os.path.join(ROOT, "tests", "golden", "zones.json")) as f:
        ny = json.load(f)["zones"]["America/New_York"]
    flags = abi.RUN_JSONL | abi.RUN_LINKS | abi.RUN_FRONTIER | abi.RUN_SKIP_SELF | abi.RUN_NO_D2H
    c = Corpus(a.n, profile=2)
    e = Engine()
    e.telegram_upload(0, c.batch)
    arms = {"no zone": ([], []), "America/New_York": (ny["start"], ny["offset"])}
    ms = {k: [] for k in arms}
    wall = {k: [] for k in arms}
    jsonl = {}
    for rep in range(a.reps + 2):  # the first two rounds warm up
        for name, (s, o) in arms.items():
            e.set_zone(s, o)
            e.frontier_clear()
            t0 = time.perf_counter()
            r = e.telegram_run_resident(0, flags)
            dt = (time.perf_counter() - t0) * 1e3
            jsonl[name] = r.jsonl_len
            if rep >= 2:
                ms[name].append(r.kernel_ms)
                wall[name].append(dt)
    print(f"card: {card()}")
    print(f"records: {a.n}, reps: {a.reps} per arm, alternated")
    for name in arms:
        k = sorted(ms[name])
        print(f"{name:18s} kernel ms median {statistics.median(k):8.3f}  min {k[0]:8.3f}  max {k[-1]:8.3f}  "
              f"wall ms median {statistics.median(wall[name]):8.3f}  jsonl {jsonl[name]} B")
    m0, m1 = statistics.median(ms["no zone"]), statistics.median(ms["America/New_York"])
    print(f"zone / no zone: {m1 / m0:.4f}")
    e.close()


if __name__ == "__main__":
    main()
