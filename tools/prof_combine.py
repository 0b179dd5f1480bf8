"""Combine mode (tgi_combine_add / flush): the blob encoder's device time and bandwidth on a resident config-2-shaped
batch with the default trigger and cap (tgi_dapr_payloads timed on the same batch for comparison), the added host-clock
cost of a blocking 100-message page call that closes no blob, and the combine-mode e2e leg.  Prints the card and its
power limit.

    python tools/prof_combine.py [--sizes 10000000 8000000 ...] [--reps 3]
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

from distributed_crawler_b200 import abi, sink  # noqa: E402
from distributed_crawler_b200.corpus import Corpus  # noqa: E402
from distributed_crawler_b200.engine import Engine, EngineError, lib  # noqa: E402

PREFIX = b"/data/crawls/crawl-7/exec-2024-01-01/"
HBM = 3.35e12  # H100 SXM data sheet
J = abi.RUN_JSONL


def call(fn, *args):
    """a combine call through the C ABI: the blobs stay in the library's pinned buffers"""
    out = abi.CombinedC()
    t = time.perf_counter()
    rc = fn(*args, C.byref(out))
    ms = (time.perf_counter() - t) * 1e3
    if rc:
        raise EngineError(rc, lib().tgi_last_error(args[0]).decode())
    return out, ms


def encoded_bytes(out):
    """base64 bytes this call wrote: its closed blobs, minus what the open group held before, plus the open group"""
    return sum(out.blobs[j].data_len for j in range(out.n_blobs)) + out.open_bytes // 3 * 4


def kernel_times(fn):
    """device time per kernel name of one call of fn, from a torch.profiler trace (CUDA activities only)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    out = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        out[ev.key] = (t / 1e3, ev.count)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[10_000_000, 8_000_000, 6_000_000, 4_000_000],
                    help="config-2-shaped batch sizes to try, largest first: the first that fits is measured")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    trig, cap = sink.TRIGGER_DEFAULT, sink.HARD_CAP_DEFAULT

    # 1. the encoder on a resident config-2-shaped batch: every call starts from an empty open group
    for n in a.sizes:
        c = Corpus(n, profile=2)
        e = Engine(max_records=n)
        try:
            e.telegram_submit(0, c.batch, J | abi.RUN_JSONL_DEVICE)
            r = e.telegram_wait(0, copy=True)
            e.combine_open(trig, cap, PREFIX)
            out, wall = call(lib().tgi_combine_add, e.h, 0, 1)
        except EngineError as err:
            print(f"config-2 shape, {n} messages: does not fit ({err})")
            e.close()
            c.close()
            continue
        print(f"config-2 shape: {n} messages, JSONL {r.jsonl_len / 1e9:.2f} GB, {out.n_blobs} blobs closed, "
              f"{out.open_bytes / 1e6:.1f} MB left open, {out.gpu_launches} launches")
        ms, walls = [], []
        for _ in range(a.reps):  # the buffers stay: flush empties the open group
            call(lib().tgi_combine_flush, e.h, 1)
            out, wall = call(lib().tgi_combine_add, e.h, 0, 1)
            ms.append(out.kernel_ms)
            walls.append(wall)
        algo = r.jsonl_len + encoded_bytes(out)  # line bytes read + base64 bytes written
        med = sorted(ms)[len(ms) // 2]
        print(f"  kernel_ms (drops scan, posts per blob, encoder): median {med:.2f} ms of {a.reps}; algorithmic "
              f"{algo / 1e9:.2f} GB -> {algo / med / 1e6:.0f} GB/s = {100 * algo / (med * 1e-3) / HBM:.1f} % of 3.35 TB/s")
        print(f"  whole call (planning, encoder, {sum(out.blobs[j].data_len for j in range(out.n_blobs)) / 1e9:.2f} GB of "
              f"blobs to pinned memory): median {sorted(walls)[len(walls) // 2]:.1f} ms")
        # the host's share of planning: the boundaries by binary search; tgi_plan_chunks_carry adds a linear scan for
        # lines above the cap, which tgi_combine_add leaves to combine_drops_kernel
        pt = []
        for _ in range(3):
            t0 = time.perf_counter()
            groups, _, _ = sink.plan_chunks_carry(r.line_off, 0, trig, cap)
            pt.append((time.perf_counter() - t0) * 1e3)
        print(f"  host planning of {n} lines into {len(groups)} groups (tgi_plan_chunks_carry, with its linear scan for "
              f"dropped lines): min {min(pt):.2f} ms")
        try:
            call(lib().tgi_combine_flush, e.h, 1)
            kt = kernel_times(lambda: call(lib().tgi_combine_add, e.h, 0, 1))
            enc = sum(t for k, (t, _) in kt.items() if "combine_encode_kernel" in k)
            for k, (t, cnt) in kt.items():
                if "combine_" in k:
                    print(f"  {k[:60]}: {t:.2f} ms ({cnt} launches)")
            print(f"  encoder alone: {algo / 1e9:.2f} GB algorithmic -> {algo / (enc * 1e-3) / 1e9:.0f} GB/s = "
                  f"{100 * algo / (enc * 1e-3) / HBM:.1f} % of 3.35 TB/s")
        except Exception as err:  # the profiler is a diagnostic: the numbers above stand without it
            print(f"  encoder alone: not measured ({err})")
        # tgi_dapr_payloads on the same batch, after the combiner's buffers are gone (reconfiguring frees them)
        call(lib().tgi_combine_flush, e.h, 1)
        e.combine_open(trig, 1, PREFIX)
        dms = []
        for _ in range(a.reps + 1):
            p = abi.DaprPayloadsC()
            if lib().tgi_dapr_payloads(e.h, 0, PREFIX, len(PREFIX), C.byref(p)):
                print(f"  tgi_dapr_payloads: not measured ({lib().tgi_last_error(e.h).decode()})")
                break
            dms.append(p.kernel_ms)
        if len(dms) > 1:
            dmed = sorted(dms[1:])[len(dms[1:]) // 2]
            dalgo = r.jsonl_len + p.data_len + p.path_len + 2 * 8 * (n + 1) + 2 * 4 * n
            print(f"  tgi_dapr_payloads on the same batch: kernel_ms median {dmed:.2f} ms, {dalgo / 1e9:.2f} GB algorithmic "
                  f"-> {100 * dalgo / (dmed * 1e-3) / HBM:.1f} % of 3.35 TB/s")
        e.release(0)
        e.close()
        c.close()
        break

    # 2. added host-clock cost of a blocking 100-message page call that closes no blob
    e = Engine()
    e.combine_open(trig, cap, PREFIX)
    batch = Corpus(100, profile=2, first=7).batch
    base, withc = [], []
    for k in range(220):
        t = time.perf_counter()
        e.telegram_submit(0, batch, J | abi.RUN_LINKS | abi.RUN_JSONL_DEVICE)
        e.telegram_wait(0)
        t1 = time.perf_counter()
        if k % 2:
            out, _ = call(lib().tgi_combine_add, e.h, 0, 1)
            assert out.n_blobs == 0
        t2 = time.perf_counter()
        e.release(0)
        if k >= 20:
            (withc if k % 2 else base).append(((t1 - t) * 1e3, (t2 - t1) * 1e3))
    print(f"page tg 100: batch call {np.median([x[0] for x in base]):.3f} ms, tgi_combine_add adds "
          f"{np.median([x[1] for x in withc]):.3f} ms (median of 100, no blob closed)")
    e.close()

    # 3. combine-mode e2e leg: batch with the lines left on the device, then the blobs in pinned host memory
    n = 2_000_000
    c = Corpus(n, profile=2, first=123)
    e = Engine(max_records=n)
    e.combine_open(trig, cap, PREFIX)
    walls, nb = [], 0
    for _ in range(4):
        t = time.perf_counter()
        e.telegram_submit(0, c.batch, J | abi.RUN_JSONL_DEVICE)
        r = e.telegram_wait(0)
        out, _ = call(lib().tgi_combine_add, e.h, 0, 1)
        walls.append((time.perf_counter() - t) * 1e3)
        nb += out.n_blobs
        e.release(0)
    print(f"e2e {n} messages (JSONL {r.jsonl_len / 1e9:.2f} GB), lines on the device, {nb} blobs over 4 calls: "
          f"wall min {min(walls[1:]):.1f} ms, median {sorted(walls[1:])[1]:.1f} ms (of the last 3)")
    e.close()


if __name__ == "__main__":
    main()
