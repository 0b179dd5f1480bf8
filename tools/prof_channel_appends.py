"""Local sink on the device (tgi_channel_appends): device time, gather bandwidth, groups against the host planner's runs,
and the host wall time of writing the posts.jsonl files both ways into a tmpfs directory, for a config-2 batch (runs of
100 posts per channel) and a config-4 batch (channels interleaved record by record), lines left on the device.  Also the
added cost per blocking page call.  Prints the card and its power limit.

    python tools/prof_channel_appends.py [--n2 1000000] [--n4 500000] [--reps 10]
"""
import argparse
import ctypes as C
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

from distributed_crawler_b200 import abi, sink  # noqa: E402
from distributed_crawler_b200.corpus import Corpus, YtCorpus  # noqa: E402
from distributed_crawler_b200.engine import Engine, EngineError, lib  # noqa: E402
from helpers import channel_ids  # noqa: E402
from yt_corpus import make_youtube_config4  # noqa: E402

HBM = 3.35e12  # H100 SXM data sheet
J = abi.RUN_JSONL


def appends_call(e, slot):
    """tgi_channel_appends through the C ABI (the outputs stay in the library's pinned buffers)"""
    p = abi.ChannelAppendsC()
    t = time.perf_counter()
    rc = lib().tgi_channel_appends(e.h, slot, C.byref(p))
    ms = (time.perf_counter() - t) * 1e3
    if rc:
        raise EngineError(rc, lib().tgi_last_error(e.h).decode())
    return p, ms


def measure(label, batch, yt, n, reps, tmp):
    e = Engine(max_records=n)
    sub, wait = (e.youtube_submit, e.youtube_wait) if yt else (e.telegram_submit, e.telegram_wait)
    sub(0, batch, J | abi.RUN_JSONL_DEVICE)
    r = wait(0)
    p, _ = appends_call(e, 0)
    ms = sorted(appends_call(e, 0)[0].kernel_ms for _ in range(reps))
    med = ms[len(ms) // 2]
    print(f"{label}: {n} records, JSONL {r.jsonl_len / 1e9:.2f} GB, {p.n_groups} groups, {p.gpu_launches} launches")
    print(f"  kernel_ms (all kernels and scans, not the read-back): min {ms[0]:.2f} ms, median {med:.2f} ms")
    try:  # the gather alone, from a torch.profiler trace of one more call (CUDA activities only)
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            appends_call(e, 0)
        for ev in sorted(prof.key_averages(), key=lambda ev: -(getattr(ev, "device_time_total", 0) or 0)):
            if not any(s in ev.key for s in ("la_", "radix_", "scan_")):
                continue
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            line = f"  {ev.key[:48]:48s} {t / 1e3:8.3f} ms ({ev.count} launch)"
            if "la_gather_kernel" in ev.key:
                gb = 2 * r.jsonl_len  # every line byte read once and written once
                line += f"  gather {gb / (t * 1e3):.0f} GB/s = {100 * gb / (t * 1e-6) / HBM:.1f} % of 3.35 TB/s"
            print(line)
    except Exception as err:  # the profiler is a diagnostic: the numbers above stand without it
        print(f"  per-kernel times: not measured ({err})")
    e.release(0)
    # the same batch with its lines copied, for the host planner and the per-run appends
    sub(0, batch, J)
    rc = wait(0, copy=True)
    e.release(0)
    runs = sink.plan_channel_appends(rc.line_off, batch.recs)
    print(f"  groups {p.n_groups} vs tgi_plan_channel_appends runs {len(runs)}: {len(runs) / max(p.n_groups, 1):.1f}x fewer appends")
    ids = [x.decode("utf-8", "surrogateescape") for x in channel_ids(batch, yt)]
    walls = {}
    for way in ("runs", "grouped", "runs", "grouped"):
        d = tempfile.mkdtemp(dir=tmp)
        if way == "runs":
            t = time.perf_counter()
            k = sink.append_posts(rc.jsonl, rc.line_off, batch.recs, ids, d, "crawl")
        else:
            sub(0, batch, J | abi.RUN_JSONL_DEVICE)
            wait(0)
            t = time.perf_counter()
            k = sink.append_posts_grouped(e, 0, ids, d, "crawl")
            e.release(0)
        walls.setdefault(way, []).append((time.perf_counter() - t) * 1e3)
        shutil.rmtree(d)
    print(f"  files into {tmp}: per-run appends {min(walls['runs']):.1f} ms ({len(runs)} appends, host JSONL), "
          f"grouped {min(walls['grouped']):.1f} ms ({k} appends, tgi_channel_appends included); min of 2")
    e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n2", type=int, default=1_000_000)
    ap.add_argument("--n4", type=int, default=500_000)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    tmp = "/dev/shm" if os.path.isdir("/dev/shm") else tempfile.gettempdir()
    c = Corpus(a.n2, profile=2)
    measure("config 2", c.batch, False, a.n2, a.reps, tmp)
    c.close()
    y = YtCorpus(a.n4)
    measure("config 4", y.batch, True, a.n4, a.reps, tmp)
    y.close()

    # added cost per blocking page call
    e = Engine()
    for label, batch, yt in (("tg 100", Corpus(100, profile=2, first=7).batch, False),
                             ("tg 1000", Corpus(1000, profile=2, first=9).batch, False),
                             ("yt 50", make_youtube_config4(50, seed=5)[0], True)):
        base, add = [], []
        for k in range(220):
            t = time.perf_counter()
            (e.youtube_submit if yt else e.telegram_submit)(0, batch, J | abi.RUN_LINKS)
            (e.youtube_wait if yt else e.telegram_wait)(0)
            t1 = time.perf_counter()
            if k % 2:
                appends_call(e, 0)
            t2 = time.perf_counter()
            e.release(0)
            if k >= 20:
                (add if k % 2 else base).append((t2 - t1) * 1e3 if k % 2 else (t1 - t) * 1e3)
        print(f"page {label}: batch call {np.median(base):.3f} ms, tgi_channel_appends adds {np.median(add):.3f} ms (median of 100)")
    e.close()


if __name__ == "__main__":
    main()
