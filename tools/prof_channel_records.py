"""Random-walk channel records (tgi_channel_batch): kernel_ms, launches and the host clock of one blocking call for 100,
10 000 and 1 000 000 records, with and without tgi_dapr_payloads on the result (the StoreChannelData payloads).  The
lines stay on the device (TGI_RUN_JSONL_DEVICE) when the payloads are made from them.  Prints the card and its power
limit.

    python tools/prof_channel_records.py [--sizes 100 10000 1000000] [--reps K]
"""
import argparse
import ctypes as C
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from distributed_crawler_b200 import abi  # noqa: E402
from distributed_crawler_b200.engine import Engine, EngineError, lib  # noqa: E402
from distributed_crawler_b200.pack import ChBatch, pack_channels  # noqa: E402
from test_channel_rules import make_channels  # noqa: E402

PREFIX = b"/data/crawls/crawl-7/exec-2024-01-01/"


def batch_of(n):
    """n records: 10 000 distinct ones (tests/test_channel_rules.make_channels) repeated, each repeat with its own strings"""
    import numpy as np
    base = pack_channels(make_channels(min(n, 10_000), seed=7))
    k = -(-n // base.n)
    recs = np.tile(base.recs, k)[:n]
    recs["str_off"] += np.repeat(np.arange(k, dtype=np.uint64) * np.uint64(base.strs.size), base.n)[:n]
    strs = np.zeros(base.strs.size * k + 16, np.uint8)
    strs[:base.strs.size * k] = np.tile(base.strs, k)
    return ChBatch(recs=recs, strs=strs[:base.strs.size * k])


def call(e, d, flags, payloads):
    """one tgi_channel_batch (and tgi_dapr_payloads) through the C ABI, outputs left in the library's buffers;
    -> (host ms, kernel ms, launches, line bytes)"""
    r = abi.ResultC()
    t = time.perf_counter()
    rc = lib().tgi_channel_batch(e.h, C.byref(d), flags, C.byref(r))
    if rc:
        raise EngineError(rc, lib().tgi_last_error(e.h).decode())
    ms, launches = r.kernel_ms, r.gpu_launches
    if payloads:
        p = abi.DaprPayloadsC()
        rc = lib().tgi_dapr_payloads(e.h, r.slot, PREFIX, len(PREFIX), C.byref(p))
        if rc:
            raise EngineError(rc, lib().tgi_last_error(e.h).decode())
        ms += p.kernel_ms
        launches += p.gpu_launches
    wall = (time.perf_counter() - t) * 1e3
    lib().tgi_result_release(e.h, r.slot)
    return wall, ms, launches, r.jsonl_len


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[100, 10_000, 1_000_000])
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    e = Engine(max_records=max(a.sizes))
    print("records | leg | host ms (median, min-max) | kernel_ms median | launches | line bytes")
    try:
        for n in a.sizes:
            b = batch_of(n)
            d = b.descriptor()
            for label, flags, payloads in (("lines to host", abi.RUN_JSONL, False),
                                           ("lines + dapr_payloads", abi.RUN_JSONL | abi.RUN_JSONL_DEVICE, True)):
                call(e, d, flags, payloads)  # warm-up: buffers grow on first use
                runs = [call(e, d, flags, payloads) for _ in range(a.reps)]
                walls, kms = [x[0] for x in runs], [x[1] for x in runs]
                print(f"{n} | {label} | {statistics.median(walls):.3f} ({min(walls):.3f}-{max(walls):.3f}) | "
                      f"{statistics.median(kms):.3f} | {runs[0][2]} | {runs[0][3]}")
    finally:
        e.close()


if __name__ == "__main__":
    main()
