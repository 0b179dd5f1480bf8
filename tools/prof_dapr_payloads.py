"""Dapr sink payloads (tgi_dapr_payloads): device time and bandwidth on a config-2-shaped batch, added cost per blocking
page call, and the Dapr-mode end-to-end leg with and without TGI_RUN_JSONL_DEVICE.  Prints the card and its power limit.

    python tools/prof_dapr_payloads.py [--sizes 10000000 8000000 ...] [--reps 10]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

from distributed_crawler_b200 import abi  # noqa: E402
from distributed_crawler_b200.corpus import Corpus  # noqa: E402
from distributed_crawler_b200.engine import Engine, EngineError, lib  # noqa: E402
from yt_corpus import make_youtube_config4  # noqa: E402

PREFIX = b"/data/crawls/crawl-7/exec-2024-01-01/"
HBM = 3.35e12  # H100 SXM data sheet
J = abi.RUN_JSONL


def payload_call(e, slot):
    """tgi_dapr_payloads through the C ABI: the payloads stay in the library's pinned buffers (Engine.dapr_payloads would
    copy them into numpy arrays, host work that is not the library's)"""
    p = abi.DaprPayloadsC()
    t = time.perf_counter()
    rc = lib().tgi_dapr_payloads(e.h, slot, PREFIX, len(PREFIX), C.byref(p))
    ms = (time.perf_counter() - t) * 1e3
    if rc:
        raise EngineError(rc, lib().tgi_last_error(e.h).decode())
    return p, ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[10_000_000, 8_000_000, 6_000_000, 4_000_000],
                    help="config-2-shaped batch sizes to try, largest first: the first that fits is measured")
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())

    # 1. device time of the payload kernels on a resident config-2-shaped batch: the largest of --sizes that fits
    with open("/proc/meminfo") as f:
        print("host:", " ".join(l.split(":")[0] + "=" + l.split()[1] + "kB" for l in f if l.startswith(("MemTotal", "MemAvailable"))))
    for n in a.sizes:
        c = Corpus(n, profile=2)
        e = Engine(max_records=n)
        try:
            e.telegram_submit(0, c.batch, J | abi.RUN_JSONL_DEVICE)
            r = e.telegram_wait(0)
            p, _ = payload_call(e, 0)
        except EngineError as err:
            print(f"config-2 shape, {n} messages: does not fit ({err})")
            e.close()
            c.close()
            continue
        ms = [p.kernel_ms]
        for _ in range(a.reps):
            p, _ = payload_call(e, 0)
            ms.append(p.kernel_ms)
        ms = sorted(ms[1:])
        algo = r.jsonl_len + p.data_len + p.path_len + 2 * 8 * (n + 1) + 2 * 4 * n  # lines + outputs + offsets + sizes
        med = ms[len(ms) // 2]
        print(f"config-2 shape: {n} messages, JSONL {r.jsonl_len / 1e9:.2f} GB, base64 {p.data_len / 1e9:.2f} GB, "
              f"paths {p.path_len / 1e6:.1f} MB, {p.gpu_launches} launches")
        print(f"  payload kernels (kernel_ms: sizes + scans, writer): min {ms[0]:.2f} ms, median {med:.2f} ms; "
              f"algorithmic {algo / 1e9:.2f} GB -> {algo / med / 1e6:.0f} GB/s = {100 * algo / (med * 1e-3) / HBM:.1f} % of 3.35 TB/s")
        # the writer alone, from a torch.profiler trace of one more call (CUDA activities only)
        try:
            import torch
            from torch.profiler import ProfilerActivity, profile
            torch.cuda.init()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                p, _ = payload_call(e, 0)
            for ev in prof.key_averages():
                if "dapr_" in ev.key:
                    t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                    print(f"  {ev.key[:60]}: {t / 1e3:.2f} ms ({ev.count} launch)")
                    if "dapr_write_kernel" in ev.key:
                        wb = r.jsonl_len + p.data_len + p.path_len + 2 * 8 * (n + 1)
                        print(f"  writer alone: {wb / 1e9:.2f} GB algorithmic -> {wb / (t * 1e3):.0f} GB/s = "
                              f"{100 * wb / (t * 1e-6) / HBM:.1f} % of 3.35 TB/s")
        except Exception as err:  # the profiler is a diagnostic: the numbers above stand without it
            print(f"  writer alone: not measured ({err})")
        e.release(0)
        e.close()
        c.close()
        break

    # 2. added cost per blocking call for pages
    e = Engine()
    for label, batch, yt in (("tg 100", Corpus(100, profile=2, first=7).batch, False),
                             ("tg 1000", Corpus(1000, profile=2, first=9).batch, False),
                             ("yt 50", make_youtube_config4(50, seed=5)[0], True)):
        base, withp = [], []
        for k in range(220):
            t = time.perf_counter()
            (e.youtube_submit if yt else e.telegram_submit)(0, batch, J | abi.RUN_LINKS)
            (e.youtube_wait if yt else e.telegram_wait)(0)
            t1 = time.perf_counter()
            if k % 2:
                payload_call(e, 0)
            t2 = time.perf_counter()
            e.release(0)
            if k >= 20:
                (withp if k % 2 else base).append(((t1 - t) * 1e3, (t2 - t1) * 1e3))
        b = np.median([x[0] for x in base])
        add = np.median([x[1] for x in withp])
        print(f"page {label}: batch call {b:.3f} ms, tgi_dapr_payloads adds {add:.3f} ms (median of 100)")
    e.close()

    # 3. Dapr-mode e2e leg: batch through host buffers + payloads, lines copied back or left on the device
    n = 2_000_000
    c = Corpus(n, profile=2, first=123)
    e = Engine(max_records=n)
    for _ in range(2):
        for flags in (J, J | abi.RUN_JSONL_DEVICE):
            walls = []
            for _ in range(3):
                t = time.perf_counter()
                e.telegram_submit(0, c.batch, flags)
                r = e.telegram_wait(0)
                p, _ = payload_call(e, 0)
                walls.append((time.perf_counter() - t) * 1e3)
                e.release(0)
            d2h = r.d2h_bytes() + p.data_len + p.path_len + 16 * (n + 1)
            print(f"e2e {n} messages, {'JSONL_DEVICE' if flags & abi.RUN_JSONL_DEVICE else 'JSONL copied'}: "
                  f"{d2h / 1e9:.2f} GB device->host, wall {min(walls):.1f} ms (min of 3)")
    e.close()


if __name__ == "__main__":
    main()
