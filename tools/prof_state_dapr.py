"""Cost of the resident crawl state's Dapr side: DaprStateManager.SaveState's json.Marshal(layerMap) and
ExportPagesToBinding.

  layer_map  10 k, 100 k and 1 M pages in one layer: tgi_state_layer_map's device time (kernel_ms) and the whole call on
             the host clock, read-back included; beside it a single-thread host rendering of the same bytes (Python's
             bytes join over the ids, which are plain ASCII and need no escaping), for comparison;
  export     100 k pages x 100 messages (10 M), TGI_STATE_EXPORT_DAPR at the reference's 100 MiB chunks: kernel_ms
             (JSONL passes and base64 encode, not the read-back), GB/s over JSONL + base64 bytes, and the whole call.
Prints the card and its power limit, and the median and spread of each.

    python tools/prof_state_dapr.py [--reps 9]
"""
import argparse
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from distributed_crawler_b200 import abi  # noqa: E402
from distributed_crawler_b200.engine import Engine  # noqa: E402
from prof_state import card, spread, state_arrays  # noqa: E402


def timed(reps, call):
    """(wall ms list, last result) over reps calls after two warm-up calls"""
    walls, out = [], None
    for rep in range(reps + 2):
        t0 = time.perf_counter()
        out = call()
        dt = (time.perf_counter() - t0) * 1e3
        if rep >= 2:
            walls.append(dt)
    return walls, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    a = ap.parse_args()
    print(f"card: {card()}")
    e = Engine()
    for n_pages in (10_000, 100_000, 1_000_000):
        e.state_set_arrays(*state_arrays(n_pages, 0))
        ms = []

        def lm():
            out = e.state_layer_map()
            ms.append(e.state_layer_map_ms)
            return out
        walls, out = timed(a.reps, lm)
        ids = [b"%08x-0000-4000-8000-%012x" % (p, p) for p in range(n_pages)]
        host, ref = timed(a.reps, lambda: b'{"1":[' + b",".join(b'"' + i + b'"' for i in ids) + b"]}")
        assert out == ref
        print(f"layer_map {n_pages} pages: {len(out)} B, {e.state_layer_map_launches} launches")
        print(f"  kernel ms {spread(ms[2:])}")
        print(f"  whole call incl. read-back, wall ms {spread(walls)}")
        print(f"  single-thread host join, wall ms {spread(host)}")
    e.state_set_arrays(*state_arrays(100_000, 100))
    ms = []

    def ex():
        out = e.state_export(abi.STATE_EXPORT_DAPR, abi.STATE_EXPORT_CHUNK_DEFAULT)
        ms.append(e.state_export_ms)
        return out
    walls, out = timed(a.reps, ex)
    raw, enc = sum(n for _, n in out), sum(len(d) for d, _ in out)
    k = statistics.median(ms[2:])
    print(f"export 100000 pages x 100 messages: {len(out)} chunks, {raw} B JSONL, {enc} B base64, "
          f"{e.state_export_launches} launches")
    print(f"  kernel ms {spread(ms[2:])}  -> {(raw + enc) / (k * 1e-3) / 1e9:.1f} GB/s (JSONL + base64 bytes)")
    print(f"  whole call incl. read-back, wall ms {spread(walls)}")
    e.close()


if __name__ == "__main__":
    main()
