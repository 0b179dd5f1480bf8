"""Cost of growing a resident key set (tgi_set_growth).

1. One growth step of the dedup set at 4 M -> 8 M and 16 M -> 32 M keys: the set is filled to its capacity with
   tgi_frontier_insert, then one more key goes in.  That insert reads the exact count, allocates the bigger buffers,
   copies the pool, rebuilds the table (set_rehash_kernel) and frees the old buffers; a one-key insert into a set with
   room is subtracted.  Host clock around calls that end in a device synchronise.
2. A config-3-shaped step (profile-3 links, LINKS | FRONTIER | SKIP_SELF, the batch resident on the device): a fixed
   1 << 25 set against a set that starts at 1 << 10 and grows.  The first step of the growing set pays every growth
   step; frontier_clear keeps the grown capacity, so the steps after it run at the final size.

usage: python tools/prof_set_growth.py [--n RECORDS] [--steps K] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from distributed_crawler_b200 import abi  # noqa: E402
from distributed_crawler_b200.corpus import Corpus  # noqa: E402
from distributed_crawler_b200.engine import Engine  # noqa: E402


def keys(first, n):
    """n distinct 32-byte names: 'g' + 10 decimal digits of first .. first + n - 1"""
    ids = np.arange(first, first + n, dtype=np.int64)
    k = np.zeros((n, 32), np.uint8)
    k[:, 0] = ord("g")
    for d in range(10):
        k[:, 10 - d] = ord("0") + (ids // 10 ** d) % 10
    return k


def growth_step(cap, reps=3):
    out = []
    for _ in range(reps):
        e = Engine(frontier_capacity=cap, set_growth=1 << 30)
        e.frontier_insert(keys(0, cap))
        assert e.set_info(abi.SET_FRONTIER)["grows"] == 0
        t = time.perf_counter()
        e.frontier_insert(keys(cap, 1))
        t_grow = time.perf_counter() - t
        info = e.set_info(abi.SET_FRONTIER)
        assert info["grows"] == 1 and info["capacity"] == 2 * cap and info["count"] == cap + 1
        t = time.perf_counter()
        e.frontier_insert(keys(cap + 1, 1))
        t_plain = time.perf_counter() - t
        e.close()
        out.append((t_grow - t_plain) * 1e3)
    return {"keys": cap, "to": 2 * cap, "ms": out, "ms_min": min(out)}


def step_times(batch, flags, steps, **kw):
    e = Engine(**kw)
    e.telegram_upload(0, batch)

    def step():
        e.frontier_clear()
        t = time.perf_counter()
        r = e.telegram_run_resident(0, flags)  # returns after the device finished the batch
        return (time.perf_counter() - t) * 1e3, r

    first_ms, r = step()
    ms = [step()[0] for _ in range(steps)]
    info = e.set_info(abi.SET_FRONTIER)
    e.close()
    return {"first_step_ms": first_ms, "step_ms": ms, "step_ms_median": float(np.median(ms)), "frontier_size": r.frontier_size,
            "frontier_ms_last": r.frontier_ms, "set": info}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=20_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    res = {"gpu": gpu, "growth_step": [growth_step(1 << 22), growth_step(1 << 24)]}
    c = Corpus(a.n, profile=3, nthreads=min(os.cpu_count() or 1, 64))
    flags = abi.RUN_LINKS | abi.RUN_FRONTIER | abi.RUN_SKIP_SELF | abi.RUN_NO_D2H
    res["records"] = a.n
    res["fixed_1<<25"] = step_times(c.batch, flags, a.steps, frontier_capacity=1 << 25)
    res["grow_from_1<<10"] = step_times(c.batch, flags, a.steps, frontier_capacity=1 << 10, set_growth=1 << 28)
    assert res["fixed_1<<25"]["frontier_size"] == res["grow_from_1<<10"]["frontier_size"]
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
