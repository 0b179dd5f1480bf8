"""Cost of snowball discovery on the resident progress state, host clock per call:

  page        one 100-message page with ~28 outlinks: tgi_state_discover(TGI_DISCOVER_NOW) against the host sequence it
              replaces (read the status, link offsets and link rows back, build one page per non-self outlink with its
              own uuid4, dedup by URL, pack, tgi_state_add_layer), on states of 10^3 and 10^5 pages;
  layer end   the candidates of 10^4 pages (~28 each) with TGI_DISCOVER_DAPR | TGI_DISCOVER_PAGE_JSON against the host
              sequence: read the link rows back, dedup map, urlCache test, pack, tgi_state_add_pages and one JSON value
              per added page.  Both timers cover the same work: the library's includes the pending-mode
              tgi_state_discover that gathers the 10^4 spans, the host's the read-back of the link rows.

The host sequences run in Python here, where the shim runs them in Go: they bound the host side from above, not
exactly.  Prints the card and its power limit, medians and spreads, and the device time of the library calls.

    python tools/prof_state_discover.py [--reps 30]
"""
import argparse
import json
import os
import sys
import time
import uuid

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from distributed_crawler_b200 import abi  # noqa: E402
from distributed_crawler_b200.engine import Engine, lib, names_to_keys32  # noqa: E402
from distributed_crawler_b200.pack import pack_telegram  # noqa: E402
from distributed_crawler_b200.state_pack import pack_pages  # noqa: E402
from helpers import msg  # noqa: E402
from prof_state import card, spread, state_arrays  # noqa: E402

RUN = abi.RUN_JSONL | abi.RUN_LINKS
WARM = 10  # warm-up pages per series: the first calls of a fresh context grow its pinned and device scratch


def page_batch(tag, n_msgs, n_links, per_msg=1):
    """n_msgs messages; n_links of them carry per_msg t.me links to names fresh for `tag`"""
    ms = []
    for k in range(n_msgs):
        text = "post %d" % k
        if k < n_links:
            text += " " + " ".join("t.me/n%s_%d_%d" % (tag, k, q) for q in range(per_msg))
        ms.append(msg("messageText", text, id=(k + 1) << 20, chat_id=-5, date=1_700_000_000))
    return pack_telegram(ms)


def host_links(e, slot, n):
    """what the shim read back before: statuses, link offsets and 36-byte link rows"""
    st = e.read_rows(slot, abi.ROWS_STATUS, 0, n)
    off = e.read_rows(slot, abi.ROWS_LINK_OFF, 0, n + 1)
    rows = e.read_rows(slot, abi.ROWS_LINKS, 0, int(off[-1])) if off[-1] else np.zeros(0, abi.LINK)
    return st, off, rows


def host_candidates(e, slot, n, owners):
    """(name, owner id) per non-self outlink of the processed records, owners[i] = (id, url) of record i"""
    st, off, rows = host_links(e, slot, n)
    out = []
    for i in range(n):
        if st[i] not in (abi.ST_EMITTED, abi.ST_NOLINE):
            continue
        for k in range(int(off[i]), int(off[i + 1])):
            name = rows[k]["name"][: int(rows[k]["len"])].tobytes()
            if name != owners[i][1]:
                out.append((name, owners[i][0]))
    return out


def host_page(e, slot, n, owner, depth, now):
    seen, pages = set(), []
    for name, parent in host_candidates(e, slot, n, [owner] * n):
        if name in seen:
            continue
        seen.add(name)
        pages.append({"id": str(uuid.uuid4()).encode(), "url": name, "status": b"unfetched", "parentId": parent,
                      "depth": depth, "timestamp": (now[0], now[1], None)})
    if pages:
        e.state_add_layer(pages)


def host_layer_end(e, slot, n, owners, depth, url_cache, now):
    seen, pages = set(), []
    for name, parent in host_candidates(e, slot, n, owners):
        if name in seen or name in url_cache:
            continue
        seen.add(name)
        pages.append({"id": str(uuid.uuid4()).encode(), "url": name, "status": b"unfetched", "parentId": parent,
                      "depth": depth, "timestamp": (now[0], now[1], None)})
    if pages:
        recs, strs, _ = pack_pages(pages, e.state_code, lambda pid, i: i)
        rows = np.zeros(len(pages), np.uint32)
        e._check(lib().tgi_state_add_pages(e.h, depth, recs.ctypes.data, len(recs), strs.ctypes.data, len(strs),
                                           rows.ctypes.data))
    return [json.dumps({"id": p["id"].decode(), "url": p["url"].decode(), "depth": depth, "status": "unfetched",
                        "timestamp": "2023-11-14T22:13:20Z", "parentId": p["parentId"].decode()}).encode() for p in pages]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    print(f"card: {card()}")
    now = (1_700_000_000, 0)
    for n_pages in (1_000, 100_000):
        e = Engine()
        e.state_id_seed(12345)
        layers, recs, blob, msgs = state_arrays(n_pages, 10)
        e.state_set_arrays(layers, recs, blob, msgs)
        oid = bytes(blob[recs[0]["str_off"]: recs[0]["str_off"] + recs[0]["str_len"][0]])
        ourl = bytes(blob[recs[0]["str_off"] + recs[0]["str_len"][0]:][: recs[0]["str_len"][1]])
        for name in ("discover", "host"):
            walls, dev = [], []
            for rep in range(a.reps + WARM):
                b = page_batch("%s%d" % (name[0], rep), 100, 28)
                e.telegram_submit(0, b, RUN)
                e.telegram_wait(0)
                t0 = time.perf_counter()
                if name == "discover":
                    e.state_discover(0, [(0, 0, 100, 100)], abi.DISCOVER_NOW, now)
                else:
                    host_page(e, 0, 100, (oid, ourl), int(recs[0]["depth"]) + 1, now)
                dt = (time.perf_counter() - t0) * 1e3
                e.release(0)
                if rep >= WARM:
                    walls.append(dt)
                    if name == "discover":
                        dev.append(e.state_discover_ms)
            extra = f"; device ms {spread(dev)} ({e.state_discover_launches} launches)" if dev else ""
            print(f"page, {n_pages:>7} pages: {name:<9} wall ms per page {spread(walls)}{extra}")
        e.close()

    # the layer end of 10^4 pages' candidates, ~28 each, with Dapr's rules and the per-page JSON
    n_pages, per = 10_000, 28
    e = Engine(set_growth=1 << 24)
    e.state_id_seed(999)
    layers, recs, blob, msgs = state_arrays(n_pages, 1)
    cache = [b"n%d_%d_0" % (k, k) for k in range(0, 300_000, 7)]
    reps = max(3, a.reps // 6)
    for name in ("next_layer", "host"):
        walls, dev = [], []
        for rep in range(reps + 1):  # one warm-up layer
            e.state_set_arrays(layers, recs, blob, msgs)
            e.set_clear(abi.SET_URLS)
            e.set_add(abi.SET_URLS, names_to_keys32(cache))
            ms = [msg("messageText", " ".join("t.me/n%d_%d_%d" % ((k * per + q) % 150_000, k % 3, q % 2) for q in range(per)),
                      id=(k + 1) << 20, chat_id=-5, date=1_700_000_000) for k in range(n_pages)]
            e.telegram_submit(1, pack_telegram(ms), RUN)
            e.telegram_wait(1)
            spans = [(k, k, 1, 1) for k in range(n_pages)]
            if name == "next_layer":
                t0 = time.perf_counter()
                e.state_discover(1, spans, 0, now)
                gather_ms = e.state_discover_ms
                got = e.state_next_layer(1, abi.DISCOVER_DAPR | abi.DISCOVER_PAGE_JSON, now)
                dt = (time.perf_counter() - t0) * 1e3
                added = len(got["ids"])
            else:
                owners = []
                for k in range(n_pages):
                    o = int(recs[k]["str_off"])
                    owners.append((bytes(blob[o: o + recs[k]["str_len"][0]]),
                                   bytes(blob[o + recs[k]["str_len"][0]:][: recs[k]["str_len"][1]])))
                t0 = time.perf_counter()
                added = len(host_layer_end(e, 1, n_pages, owners, 2, set(cache), now))
                dt = (time.perf_counter() - t0) * 1e3
            e.release(1)
            if rep >= 1:
                walls.append(dt)
                if name == "next_layer":
                    dev.append(gather_ms + e.state_discover_ms)
        extra = f"; device ms {spread(dev)} ({e.state_discover_launches} launches)" if dev else ""
        print(f"layer end, {n_pages} pages x {per} candidates, {added} added: {name:<10} wall ms {spread(walls)}{extra}")
    # device time per kernel of one page discover and one layer end, in a run of its own under torch.profiler
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.zeros(1, device="cuda")
    e.state_set_arrays(layers, recs, blob, msgs)
    e.telegram_submit(0, page_batch("prof", 100, 28), RUN)
    e.telegram_wait(0)
    e.telegram_submit(1, pack_telegram(ms), RUN)
    e.telegram_wait(1)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.state_discover(0, [(0, 0, 100, 100)], abi.DISCOVER_NOW | abi.DISCOVER_DAPR | abi.DISCOVER_PAGE_JSON, now)
        e.state_discover(1, spans, 0, now)
        e.state_next_layer(1, abi.DISCOVER_DAPR | abi.DISCOVER_PAGE_JSON, now)
        torch.cuda.synchronize()
    for ev in sorted(prof.key_averages(), key=lambda x: -x.device_time_total):
        if ev.device_time_total > 0:
            print(f"  kernel {ev.key[:60]:<60} calls {ev.count:>3}  mean us {ev.device_time_total / ev.count:9.1f}")
    e.release(0)
    e.release(1)
    e.close()


if __name__ == "__main__":
    main()
