"""Per-kernel device times of one resident config-2 step (bench.py --config 2: 10 M Telegram messages, parse + links +
dedup + JSONL, batch resident in HBM, no read-back), from a torch.profiler trace with CUDA activities only.  The trace
goes to OUT/step_kernels.pt.trace.json, the table (kernel, launches, ms, share of the step's kernel time) to stdout and
OUT/step_kernels.md (OUT defaults to prof_step_kernels/ in the system's temporary directory).  Prints the card and its
power limit.

    python tools/prof_step_kernels.py [--n 10000000] [--warmup 3] [--out DIR]
"""
import argparse
import collections
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from distributed_crawler_b200 import abi  # noqa: E402
from distributed_crawler_b200.corpus import Corpus  # noqa: E402
from distributed_crawler_b200.engine import Engine  # noqa: E402

FLAGS = abi.RUN_JSONL | abi.RUN_LINKS | abi.RUN_FRONTIER | abi.RUN_SKIP_SELF  # bench.py config 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "prof_step_kernels"))
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()

    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    c = Corpus(args.n, seed=0x5EED0002, profile=2, nthreads=min(os.cpu_count() or 1, 64))  # bench.py's config-2 corpus
    e = Engine(frontier_capacity=1 << 23)
    e.telegram_upload(0, c.batch)

    def step():
        e.frontier_clear()
        return e.telegram_run_resident(0, FLAGS | abi.RUN_NO_D2H)

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        r = step()
        torch.cuda.synchronize()
    trace = os.path.join(args.out, "step_kernels.pt.trace.json")
    prof.export_chrome_trace(trace)

    agg = collections.defaultdict(lambda: [0, 0.0])
    for ev in json.load(open(trace))["traceEvents"]:
        if ev.get("cat") == "kernel":
            a = agg[ev["name"].split("(")[0].split("<")[0].replace("void ", "").replace("tgi::", "")]
            a[0] += 1
            a[1] += ev["dur"] / 1e3
    tot = sum(ms for _, ms in agg.values())
    lines = [f"card: {card}; {args.n} records, step kernel_ms {r.kernel_ms:.2f} (parse {r.parse_ms:.2f}, emit {r.emit_ms:.2f})",
             "", "| kernel | launches | ms | share |", "|---|---:|---:|---:|"]
    for k, (cnt, ms) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        lines.append(f"| `{k}` | {cnt} | {ms:.2f} | {ms / tot * 100:.1f} % |")
    lines.append(f"| all kernels | {sum(a for a, _ in agg.values())} | {tot:.2f} | |")
    text = "\n".join(lines)
    print(text)
    with open(os.path.join(args.out, "step_kernels.md"), "w") as f:
        f.write(text + "\n")
    e.close()


if __name__ == "__main__":
    main()
