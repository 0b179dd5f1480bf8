"""GPU tests: the resident progress state at its edges (tests/state_edge_corpus.py), every byte against the
restatements: state.json, both exports, the layer map and the page reads of strings across the escapers' strips,
int64 ends, time bounds and offset signs, in a fixed offset and in New York's zone; row counts where the render's radix
pass count changes, with empty layers and message-less pages around the others, also under one CTA per SM; and the
4 GiB rule: a page, message, layer-map id or SQL row of 4 GiB or more is TGI_E_CAPACITY from every writer and leaves
the state as it was, while a state.json past 4 GiB renders exactly."""
import base64
import os
import subprocess
import sys

import numpy as np
import pytest

import close_rules as cr
import state_edge_corpus as ec
import tandem_sql_rules as sr
import walkback_rules as wr
from dapr_state_rules import export_dapr_chunks, export_local, marshal_layer_map
from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import Engine, EngineError
from helpers import mem_available
from state_rules import GoState, marshal_page
from test_gpu_state import LAST, META, big_state
from test_zones import ZONES

pytestmark = pytest.mark.gpu
NY = ZONES["America/New_York"]
WRAP = 716_000_000  # bytes of '<' whose escape (6 bytes each) passes 4 GiB in one string
HALF = 400_000_000  # two fields of this many '<' escape to 2.4 GB each: each under 4 GiB, the page over it


def check_state(e, go, zone=None, chunk_sizes=()):
    """render, both exports, the layer map and the page reads against the restatement"""
    want = go.marshal(META, LAST, zone)
    got = e.state_render(META, LAST)
    assert len(got) == len(want) and got == want
    assert e.state_layer_map() == marshal_layer_map(go.layer_map)
    (data, raw), = e.state_export(abi.STATE_EXPORT_LOCAL)
    assert data == export_local(go, zone) and raw == len(data)
    for cb in chunk_sizes:
        chunks = e.state_export(abi.STATE_EXPORT_DAPR, cb)
        want_chunks = export_dapr_chunks(go, cb, zone)
        assert [r for _, r in chunks] == [len(c) for c in want_chunks], cb
        assert [d for d, _ in chunks] == [base64.b64encode(c) for c in want_chunks], cb
    rows = e._st_rows()
    pids = list(go.page_map)
    for p in e.state_read_pages([rows[i] for i in pids]):
        w = go.page_map[p["id"]]
        assert all(p[f] == w.get(f, b"") for f in ec.FIELDS) and p["depth"] == w.get("depth", 0)
        assert p["timestamp"] == w["timestamp"]
        assert p["messages"] == [dict({"platform": b""}, **m) for m in w.get("messages") or []]


def run_edge_state():
    layers = ec.edge_state()
    go, e = GoState(), Engine()
    go.set_state(layers)
    e.state_set(layers)
    lines = [len(marshal_page(go.page_map[i])) + 1 for d in sorted(go.layer_map) for i in go.layer_map[d]]
    assert {n % 3 for n in lines} == {0, 1, 2}  # every base64 tail
    a, b = lines[0], lines[0] + lines[1]
    cuts = (0, 1, a - 1, a, a + 1, b - 1, b, b + 1, max(lines) - 1, 1 << 20, abi.STATE_EXPORT_CHUNK_DEFAULT)
    check_state(e, go, None, cuts)
    e.set_zone(*NY)
    check_state(e, go, NY, (0, a))
    check_page_json(e, go, NY)
    e.close()


def check_page_json(e, go, zone):
    """TGI_TURN_PAGE_JSON on the edge pages: a multi-page begin with empty fetches, then a close of the same rows with
    changed fields; every page's json.Marshal(page) against the restatement, and the state rendered after both"""
    pids = [p for p in go.page_map if p.startswith(b"id") or p.startswith(b"omit")]
    rows = [e._st_rows()[p] for p in pids]
    _, _, _, got = e.state_pages_begin(rows, [[] for _ in rows], page_json=True)
    views = [cr.page_begin(go, p, [])[0] for p in pids]
    assert got == [marshal_page(go.page_map[p], zone) for p in pids]
    pages = [{k: v for k, v in dict(go.page_map[p], status=b"fetched\xe2\x80\xa8<").items() if k != "messages"}
             for p in pids]
    got = e.state_pages_close(rows, pages, page_json=True)
    for pg, view in zip(pages, views):
        cr.page_close(go, pg, view)
    assert got == [marshal_page(go.page_map[p], zone) for p in pids]
    assert e.state_render(META, LAST) == go.marshal(META, LAST, zone)


def test_edge_strings_numbers_and_times():
    run_edge_state()


def test_edge_times_past_the_bounds_are_refused():
    go, e = GoState(), Engine()
    layers = [(0, [{"id": b"a", "url": b"u", "timestamp": (ec.YEAR9999_END, 999_999_999, 0)}])]
    go.set_state(layers)
    e.state_set(layers)
    for ts in ec.TIME_REFUSED:
        e.state_update_page({"id": b"b", "url": b"v", "depth": 0, "timestamp": ts})
        for call in (lambda: e.state_render(META, LAST), lambda: e.state_export(abi.STATE_EXPORT_LOCAL)):
            refused(call, abi.E_ARG)
    p = {"id": b"b", "url": b"v", "depth": 0, "timestamp": (ec.YEAR0, 0, 0)}
    e.state_update_page(p)
    go.update_page(p)
    assert e.state_render(META, LAST) == go.marshal(META, LAST)
    e.close()


def run_row_count(n):
    """n pages in two halves with empty layers first, between and last; every third page from the third on gets
    messages, appended by UpdateMessage in interleaved row order so that the grouping has to regroup them"""
    pages = [{"id": b"p%d" % k, "url": b"u%d" % k, "depth": 1, "status": b"fetched"} for k in range(n)]
    layers = [(0, []), (1, pages[:n // 2]), (2, []), (3, pages[n // 2:]), (4, [])]
    go, e = GoState(), Engine()
    go.set_state(layers)
    e.state_set(layers)
    rows = e._st_rows()
    ups = [(k, ec.INT_EDGES[(k + r) % len(ec.INT_EDGES)], r - k, b"fetched" if r else b"x<y")
           for r in range(2) for k in range(2, n - 2) if k % 3 == 2]
    for k, c, m, st in ups:
        assert go.update_message(b"p%d" % k, c, m, st)
    if ups:
        assert e.state_update_messages([(rows[b"p%d" % k], c, m, st) for k, c, m, st in ups]) == 0
    want = go.marshal(META, LAST)
    assert e.state_render(META, LAST) == want
    (data, _), = e.state_export(abi.STATE_EXPORT_LOCAL)
    assert data == export_local(go)
    e.close()


@pytest.mark.parametrize("n", ec.ROW_COUNTS)
def test_row_counts_around_the_radix_passes(n):
    run_row_count(n)


def test_edges_and_row_counts_under_one_cta_per_sm():
    """TGI_GRID_MULT=1: the warp-per-entry kernels past one pass with the edge corpus (3500 entries against 132 x 8
    warps) and the thread kernels with 65 537 rows' messages (87 000 against 132 x 256 threads)"""
    code = ("import sys; sys.path.insert(0, 'tests')\n"
            "import test_gpu_state_edges as t\n"
            "t.run_edge_state()\n"
            "t.run_row_count(65537)\n"
            "print('ok')\n")
    env = dict(os.environ, TGI_GRID_MULT="1")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=1200)
    assert p.returncode == 0 and "ok" in p.stdout, p.stderr[-3000:]


# ---- the tandem SQL and the walkback on edge owners -------------------------------------------------------------------
SQL_KS = (1, 7, sr.MAX_ROWS)
SQL_CLOCKS = [(ec.YEAR0, 0), (ec.YEAR9999_END, 999_999_999), (1_760_000_000, 1), (1_760_000_000, 100_000_000)]
SQL_REFUSED = [(ec.YEAR0 - 1, 0), (ec.YEAR9999_END + 1, 0)]


def edge_owners(urls):
    """owner pages whose id, URL and sequenceId carry escapes, runes, U+2028 and invalid bytes (thread escaper) and
    whose depths are the int64 ends; urls: the sequence's own channel names, which its pages link to"""
    short = [s for s, _, n in ec.short_strs() if 5 <= n <= 40]
    texts = [s for s in short if b"\xff" not in s]  # the sequence writes the URL into its messages' text
    depths = (ec.I64_MAX, ec.I64_MIN, ec.I64_MAX - 1, -1)
    return [{"id": b"o%d" % k + short[97 * k % len(short)], "url": urls[k] + texts[31 * k % len(texts)] if k % 2 else urls[k],
             "depth": depths[k % 4], "status": b"fetched", "sequenceId": short[53 * k % len(short)] if k % 3 else b""}
            for k in range(len(urls))]


def sql_crawl_ids():
    return [b""] + [s for s, _, n in ec.short_strs() if n in (1, 4, 5, 13, 40)][::5]


def test_edge_sql_on_edge_owners():
    from test_gpu_state_tandem import NOW, RUN, as_rows
    from test_gpu_state_tandem_sql import SqlSequence
    sq = SqlSequence(90, n_owners=4)
    e = sq.e
    urls = [sq.go.page_map[p]["url"] for p in sq.go.page_map]
    sq.state_set([(0, edge_owners(urls))])
    spans, status, links = sq.result(list(sq.go.page_map), RUN, 0, sizes=[6, 6, 6, 6])
    want = sq.expect(spans, status, links)
    assert as_rows(e.state_pending_edges(0, spans, NOW)) == want[:3]
    pages = sq.pages(spans, want)
    assert pages and {b["source_depth"] for b, _ in pages} & {ec.I64_MAX, ec.I64_MIN}
    for j, crawl in enumerate(sql_crawl_ids()):
        now = SQL_CLOCKS[j % len(SQL_CLOCKS)]
        for k in SQL_KS:
            assert e.state_edge_sql(crawl, now, k) == sr.statements(pages, crawl, sr.discovery_time(*now), k), (crawl, now, k)
    for now in SQL_REFUSED:
        refused(lambda: e.state_edge_sql(b"c", now, 1), abi.E_ARG)
    e.release(0)
    e.close()


def test_walkback_on_edge_owners():
    from test_gpu_state_tandem import NOW, RUN, as_rows
    from test_gpu_state_walkback import WalkSequence
    sq = WalkSequence(91, n_owners=4)
    e = sq.e
    urls = [sq.go.page_map[p]["url"] for p in sq.go.page_map]
    sq.state_set([(0, edge_owners(urls))])
    sq.add_discovered([b"walkchan%d" % k for k in range(5)])
    spans, status, links = sq.result(list(sq.go.page_map), RUN, 0, sizes=[3, 3, 3, 3])
    spans = [(row, first, n, 0) for row, first, n, _ in spans]  # nothing processed: every span walks back
    walks = sq.walks(spans, as_rows(e.state_pending_edges(0, spans, NOW))[2])
    assert len(walks) == 4 and {o["depth"] for o, _ in walks} >= {ec.I64_MAX, ec.I64_MIN}  # depth + 1 wraps at I64_MAX
    for now in SQL_REFUSED:
        refused(lambda: e.state_walkback(b"c", now, 1), abi.E_ARG)
    for j, crawl in enumerate(sql_crawl_ids()):
        now = SQL_CLOCKS[j % len(SQL_CLOCKS)]
        for k in SQL_KS:
            got, stmts = e.state_walkback(crawl, now, k)
            assert got == [r for _, r in walks]
            assert stmts == wr.statements(walks, crawl, sr.discovery_time(*now), k), (crawl, now, k)
    e.release(0)
    e.close()


# ---- the 4 GiB rule --------------------------------------------------------------------------------------------------
def need_memory(gib):
    if mem_available() < gib << 30:
        pytest.skip(f"needs {gib} GiB of available host memory")


def long_escapes():
    """a 716 MB string through the thread escaper takes ~130 s of one thread on an H100 (NVIDIA H100 80GB HBM3, 700 W
    power limit); the tests of the thread writers' 4 GiB rule run with TGI_TEST_LONG_ESCAPES=1"""
    if os.environ.get("TGI_TEST_LONG_ESCAPES") != "1":
        pytest.skip("a 716 MB single-thread escape per writer: set TGI_TEST_LONG_ESCAPES=1")


def refused(call, code=abi.E_CAPACITY):
    with pytest.raises(EngineError) as ei:
        call()
    assert ei.value.code == code


def small_state():
    pages = [{"id": b"a", "url": b"https://t.me/a", "depth": 0, "status": b"fetched", "timestamp": (1700000000, 5, 3600)},
             {"id": b"b", "url": b"https://t.me/b", "depth": 0, "status": b"deadend"}]
    go, e = GoState(), Engine()
    go.set_state([(0, pages)])
    e.state_set([(0, pages)])
    return go, e


def test_a_page_over_4gib_with_each_field_under_it():
    need_memory(12)
    go, e = small_state()
    big = {"id": b"<" * HALF, "url": b"<" * HALF, "depth": 0, "status": b"fetched"}
    row = e.state_update_page(big)
    for call in (lambda: e.state_render(META, LAST), lambda: e.state_export(abi.STATE_EXPORT_LOCAL),
                 lambda: e.state_export(abi.STATE_EXPORT_DAPR, 0)):
        refused(call)
    got = e.state_read_pages([row])[0]
    assert got["id"] == big["id"] and got["url"] == big["url"] and got["status"] == b"fetched"
    # the page JSON of a close fails after the update (Dapr's UpdatePage changes pageMap before json.Marshal)
    refused(lambda: e.state_page_close(row, dict(big, status=b"failed"), page_json=True))
    assert e.state_read_pages([row])[0]["status"] == b"failed"
    # under 4 GiB again (2.4 GB): the page renders exactly
    go.update_page(dict(big, id=b"@ID@", url=b"u", status=b"failed"))
    e.state_update_page(dict(big, url=b"u", status=b"failed"))
    want = go.marshal(META, LAST).replace(b'"@ID@"', b'"' + b"\\u003c" * HALF + b'"')
    got = e.state_render(META, LAST, copy=False)
    assert len(got) == len(want) and np.array_equal(got, np.frombuffer(want, np.uint8))
    e.close()


def test_one_field_past_4gib():
    need_memory(8)
    go, e = small_state()
    e.state_update_page({"id": b"c", "url": b"<" * WRAP, "depth": 0})  # warp_esc_len's 32-bit sum would wrap
    for call in (lambda: e.state_render(META, LAST), lambda: e.state_export(abi.STATE_EXPORT_LOCAL)):
        refused(call)
    e.state_update_page({"id": b"c", "url": b"u", "depth": 0})
    go.update_page({"id": b"c", "url": b"u", "depth": 0})
    assert e.state_render(META, LAST) == go.marshal(META, LAST)
    e.close()


def test_a_message_past_4gib():
    long_escapes()
    need_memory(8)
    go, e = small_state()
    h = {"id": b"<" * WRAP, "url": b"h", "depth": 7}  # no layer 7: in pageMap, listed nowhere
    e.state_update_page(h)
    msgs = [{"chatId": 1, "messageId": 2, "status": b"fetched", "pageId": h["id"]}]
    # on a page in no layer list the message is never written, so the render goes through (Go renders listed pages)
    e.state_update_page({"id": b"u", "url": b"v", "depth": 8, "messages": msgs})
    assert e.state_render(META, LAST) == go.marshal(META, LAST)
    # on a listed page its pageId wraps a 32-bit size: the entry is refused
    e.state_update_page({"id": b"a", "url": b"https://t.me/a", "depth": 0, "messages": msgs})
    refused(lambda: e.state_render(META, LAST))
    assert e.state_layer_map() == b'{"0":["a","b"]}'
    e.close()


def test_a_layer_map_id_past_4gib():
    long_escapes()
    need_memory(8)
    go, e = small_state()
    e.state_update_page({"id": b"<" * WRAP, "url": b"h", "depth": 0})  # listed in layer 0
    refused(lambda: e.state_layer_map())
    e.close()


def test_sql_rows_past_4gib():
    long_escapes()
    need_memory(8)
    from test_gpu_state_tandem import NOW, RUN, as_rows
    from test_gpu_state_tandem_sql import SqlSequence
    from test_gpu_state_walkback import WalkSequence
    huge = b"<" * WRAP
    sq = SqlSequence(70, n_owners=3)
    e = sq.e
    spans, status, links = sq.result(list(sq.go.page_map), RUN, 0, sizes=[5, 5, 5])
    want = sq.expect(spans, status, links)
    assert as_rows(e.state_pending_edges(0, spans, NOW)) == want[:3]
    pages = sq.pages(spans, want)
    assert pages
    refused(lambda: e.state_edge_sql(huge, (NOW, 5), 7))
    assert e.state_edge_sql(b"c", (NOW, 5), 7) == sr.statements(pages, b"c", sr.discovery_time(NOW, 5), 7)
    e.release(0)
    e.close()
    sq = WalkSequence(80, n_owners=3)
    e = sq.e
    sq.add_discovered([b"walkchan%d" % k for k in range(5)])
    spans, status, links = sq.result(list(sq.go.page_map), RUN, 0, sizes=[3, 3, 3])
    spans = [(row, first, n, 0) for row, first, n, _ in spans]  # nothing processed: every span walks back
    sb = as_rows(e.state_pending_edges(0, spans, NOW))[2]
    walks = sq.walks(spans, sb)
    assert walks
    refused(lambda: e.state_walkback(huge, (NOW, 0), 1))
    got, stmts = e.state_walkback(b"c", (NOW, 0), 1)  # the refused call kept no picks: the same ones again
    assert got == [r for _, r in walks]
    assert stmts == wr.statements(walks, b"c", sr.discovery_time(NOW, 0), 1)
    e.release(0)
    e.close()


def test_a_state_json_past_4gib_renders_exactly():
    need_memory(24)
    n_pages, per_page = 480, 100_000  # 48 M messages of ~93 bytes: 4.48 GB
    recs, strs, msgs, want = big_state(n_pages, per_page)
    assert len(want) > 1 << 32
    e = Engine()
    e.state_set_arrays(np.array([(1, n_pages)], abi.STATE_LAYER), recs, strs, msgs)
    got = e.state_render(META, LAST, copy=False)
    assert len(got) == len(want) and np.array_equal(got, np.frombuffer(want, np.uint8))
    e.close()
