"""Every product path once on small inputs: run under `compute-sanitizer --tool memcheck` / `--tool racecheck`."""
import sys
import os; ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
from distributed_crawler_b200 import abi
from distributed_crawler_b200.corpus import Corpus
from distributed_crawler_b200.engine import Engine
from yt_corpus import make_youtube, make_youtube_config4
from gm_corpus import make_generic
e = Engine()
f = abi.RUN_JSONL | abi.RUN_LINKS | abi.RUN_FRONTIER | abi.RUN_SKIP_SELF
# page-sized batches take the one-launch page kernels; TGI_NO_PAGE=1 sends the same batches through the bulk pipeline
for no_page in (False, True):
    if no_page:
        os.environ["TGI_NO_PAGE"] = "1"
    for p in (1, 2, 3):
        c = Corpus(3000, profile=p, nthreads=4)
        r = e.telegram(c.batch, f)
        print("tg", p, r.jsonl_len, r.n_links, "launches", r.gpu_launches)
    for mk in (make_youtube, make_youtube_config4):
        b, _, _ = mk(600, seed=3)
        r = e.youtube(b, abi.RUN_JSONL | abi.RUN_LINKS | abi.RUN_FRONTIER)
        print("yt", r.jsonl_len, r.n_links, "launches", r.gpu_launches)
    os.environ.pop("TGI_NO_PAGE", None)
c = Corpus(20000, profile=2, nthreads=4)  # above the page limit: the bulk pipeline with its multi-launch scans
print("tg bulk", e.telegram(c.batch, f).gpu_launches)
g, _ = make_generic(500, seed=4)
print("gm", e.generic(g).jsonl_len)
print("join", e.key_join(np.arange(2000).reshape(-1, 2), np.arange(1000).reshape(-1, 2))[:4])
# round-2 paths: library-owned staging, exclusion sets + pending_edges rows, big maps / many links, single-rank merge
from distributed_crawler_b200.engine import names_to_keys32
from distributed_crawler_b200.pack import pack_telegram
from helpers import msg
c = Corpus(4000, profile=3, nthreads=4)
st = e.stage(c.batch)
print("staged", e.telegram(st, f).n_links)
e.unstage(st)
e.set_add(abi.SET_INVALID, names_to_keys32([b"name%05d" % i for i in range(500)]), np.full(500, 1_700_000_000, np.int64))
e.set_add(abi.SET_DISCOVERED, names_to_keys32([b"chan%05d" % i for i in range(500)]))
e.set_now(1_700_000_100)
T = abi.RUN_LINKS | abi.RUN_FRONTIER | abi.RUN_FILTER | abi.RUN_SKIP_SELF | abi.RUN_SKIP_INVALID
e.telegram_submit(1, c.batch, T)
r = e.telegram_wait(1)
print("edges", len(e.pending_edges(1, 1_700_000_100)), r.n_new)
e.release(1)
big = [msg("messageText", " ".join("t.me/chan_%05d" % i for i in range(3000)), reactions=[("k%02d" % (i % 47), i) for i in range(90)])]
print("big", e.telegram(pack_telegram(big), f).n_links)
e.comm_init(Engine.comm_unique_id(), 0, 1)
print("merge", e.frontier_merge(), len(e.frontier_global_export()))
# Dapr sink payloads after a bulk batch, a page and a YouTube page, with the lines left on the device
for b, yt in ((Corpus(20000, profile=2, nthreads=4).batch, False), (Corpus(300, profile=3, nthreads=4).batch, False),
              (make_youtube(50, seed=5)[0], True)):
    (e.youtube_submit if yt else e.telegram_submit)(0, b, abi.RUN_JSONL | abi.RUN_JSONL_DEVICE)
    (e.youtube_wait if yt else e.telegram_wait)(0)
    print("dapr", e.dapr_payloads(0, b"root/crawl/exec/").data_len)
    print("local appends", len(e.channel_appends(0)))
    e.release(0)
# combine mode: a page that stays in the open group, a bulk batch run without copies that closes blobs, the flush
e.combine_open(1_000_000, 1_500_000, b"root/crawl/exec/")
for b, flags in ((Corpus(100, profile=2, nthreads=4).batch, abi.RUN_JSONL), (Corpus(20000, profile=3, nthreads=4).batch,
                                                                             abi.RUN_JSONL | abi.RUN_NO_D2H)):
    e.telegram_submit(0, b, flags)
    e.telegram_wait(0)
    print("combine", e.combine_add(0, 1).n_blobs)
    e.release(0)
print("combine flush", e.combine_flush(2).n_blobs)
# tandem hand-off, its SQL and the forced walkbacks of its edge-less spans (one over the owner's URL only)
w = Engine(set_growth=1 << 20)
w.state_id_seed(7)
w.state_set([(0, [{"id": b"p%d" % k, "url": b"chan%05d" % k, "sequenceId": b"s"} for k in range(4)])])
w.set_add(abi.SET_DISCOVERED, names_to_keys32([b"chan00000"] + [b"disc%04d" % i for i in range(2000)]))
w.telegram_submit(0, pack_telegram([msg("messageText", "t.me/chan%05d t.me/other%d" % (k, k), id=(k + 1) << 20,
                                        chat_id=-1, date=1_700_000_000) for k in range(8)]), abi.RUN_LINKS)
w.telegram_wait(0)
print("handoff", w.state_pending_edges(0, [(0, 0, 2, 0), (1, 0, 4, 4), (2, 2, 2, 0), (3, 4, 4, 4)], 1_700_000_100)["span_batch"])
print("edge sql", len(w.state_edge_sql(b"c", (1_700_000_100, 0), 2)))
print("walkback", [r["status"] for r in w.state_walkback(b"c", (1_700_000_100, 0), 1)[0]],
      len(w.state_walkback(b"c", (1_700_000_100, 5), 7)[1]))
w.release(0)
w.close()
print("done")
