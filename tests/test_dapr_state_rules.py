"""CPU tests of tests/dapr_state_rules.py: the cases of the reference's state/export_test.go
(TestExportPagesToBinding_*), Dapr's AddLayer rules, and hand-written json.Marshal(layerMap) answers."""
import base64

import pytest

from dapr_state_rules import NoPagesFound, dapr_add_layer, export_dapr, export_local, marshal_layer_map
from state_rules import GoState, MarshalError

ROOT, CFG, CRAWL, TS = "/test/root", "crawl-123", "crawl-123", "20250615-150640"


def state(layers):
    go = GoState()
    go.set_state([(d, [{"id": i, "url": b"https://t.me/" + i} for i in ids]) for d, ids in layers])
    return go


def decoded(calls):
    return [base64.b64decode(data) for _, data in calls]


def test_no_pages_is_an_error_and_makes_no_call():
    with pytest.raises(NoPagesFound):
        export_dapr(GoState(), ROOT, CFG, CRAWL, TS, 100 << 20)
    with pytest.raises(NoPagesFound):  # layers without pages
        export_dapr(state([(0, []), (3, [])]), ROOT, CFG, CRAWL, TS, 100 << 20)


def test_single_page_is_one_call_with_part0_and_the_crawl_id():
    calls = export_dapr(state([(0, [b"page-1"])]), ROOT, CFG, CRAWL, TS, 100 << 20)
    assert len(calls) == 1
    path, _ = calls[0]
    assert path == "/test/root/crawl-123/analysis/channels/channel-pages-crawl-123-20250615-150640-part0.jsonl"
    assert decoded(calls) == [b'{"id":"page-1","url":"https://t.me/page-1","depth":0,"status":"",'
                              b'"timestamp":"0001-01-01T00:00:00Z"}\n']


def test_five_pages_are_one_chunk():
    calls = export_dapr(state([(0, [b"x" + bytes([97 + i]) for i in range(5)])]), ROOT, CFG, CRAWL, TS, 100 << 20)
    assert len(calls) == 1 and decoded(calls)[0].count(b"\n") == 5


def test_chunk_bytes_1_gives_one_chunk_per_page():
    calls = export_dapr(state([(0, [b"a", b"b", b"c"])]), ROOT, CFG, CRAWL, TS, 1)
    assert [p.rsplit("-", 1)[1] for p, _ in calls] == ["part0.jsonl", "part1.jsonl", "part2.jsonl"]
    assert [c.count(b"\n") for c in decoded(calls)] == [1, 1, 1]
    assert len(export_dapr(state([(0, [b"a", b"b", b"c"])]), ROOT, CFG, CRAWL, TS, 0)) == 3  # Go's >= 0


def test_chunks_close_after_the_line_that_reaches_chunk_bytes():
    go = state([(0, [b"a", b"b", b"c", b"d"])])
    lines = export_local(go).splitlines(keepends=True)
    end2 = len(lines[0]) + len(lines[1])
    assert [len(c) for c in decoded(export_dapr(go, ROOT, CFG, CRAWL, TS, end2))] == [end2, end2]
    assert [len(c) for c in decoded(export_dapr(go, ROOT, CFG, CRAWL, TS, end2 + 1))] == [end2 + len(lines[2]), len(lines[3])]
    assert [len(c) for c in decoded(export_dapr(go, ROOT, CFG, CRAWL, TS, end2 - 1))] == [end2, end2]


def test_pages_across_layers_in_ascending_depth():
    calls = export_dapr(state([(1, [b"p3"]), (0, [b"p1", b"p2"])]), ROOT, CFG, CRAWL, TS, 100 << 20)
    assert len(calls) == 1
    assert [ln.split(b'"')[3] for ln in decoded(calls)[0].splitlines()] == [b"p1", b"p2", b"p3"]


def test_the_directory_takes_the_config_crawl_id_and_the_file_the_argument():
    path, _ = export_dapr(state([(0, [b"p1"])]), "/r", "cfg-crawl", "my-crawl-99", TS, 100 << 20)[0]
    assert path == "/r/cfg-crawl/analysis/channels/channel-pages-my-crawl-99-20250615-150640-part0.jsonl"


def test_a_page_json_cannot_marshal_fails_the_export():
    go = state([(0, [b"p1"])])
    go.page_map[b"p1"]["timestamp"] = (253402300800, 0, 0)
    with pytest.raises(MarshalError):
        export_dapr(go, ROOT, CFG, CRAWL, TS, 1)


def test_local_export_lists_every_page_once_in_row_order():
    go = state([(0, [b"b", b"a"]), (2, [b"a", b"c"])])  # a later layer lists "a" again: one page
    assert [ln.split(b'"')[3] for ln in export_local(go).splitlines()] == [b"b", b"a", b"c"]
    assert export_local(GoState()) == b""


def test_layer_map_keys_sort_as_strings():
    lm = {2: [b"a"], -1: [], 0: [b"b", b"b"], 100: [b"c"], 10: []}
    assert marshal_layer_map(lm) == b'{"-1":[],"0":["b","b"],"10":[],"100":["c"],"2":["a"]}'
    assert marshal_layer_map({}) == b"{}"
    assert marshal_layer_map({-12: [], -2: []}) == b'{"-12":[],"-2":[]}'


def test_layer_map_escapes_ids_html_safe():
    lm = {0: [b"<a>&", b"x\xe2\x80\xa8y", b"bad\xff", b'q"\\']}
    assert marshal_layer_map(lm) == (b'{"0":["\\u003ca\\u003e\\u0026","x\\u2028y","bad\\ufffd","q\\"\\\\"]}')


def test_dapr_add_layer_rules():
    go, cache = GoState(), {b"https://t.me/old": b"prev-crawl:x"}
    p = lambda i, url, depth=0: {"id": i, "url": url, "depth": depth}
    # pages[0] is filtered away but still gives the depth; duplicates within the call are kept; no MaxPages
    depth, added = dapr_add_layer(go, cache, [p(b"a", b"https://t.me/old", 5), p(b"b", b"u1", 1), p(b"c", b"u1", 2)])
    assert depth == 5 and [q["id"] for q in added] == [b"b", b"c"]
    assert go.layer_map == {5: [b"b", b"c"]} and cache[b"u1"] == b"c"
    # every page a duplicate: no layer is created
    assert dapr_add_layer(go, cache, [p(b"d", b"u1", 7)]) == (7, [])
    assert 7 not in go.layer_map
    # a reused id replaces the page and is listed again
    dapr_add_layer(go, cache, [p(b"b", b"u2", 5)])
    assert go.layer_map[5] == [b"b", b"c", b"b"] and go.page_map[b"b"]["url"] == b"u2"
    # random-walk skips the cache
    _, added = dapr_add_layer(go, cache, [p(b"e", b"u1", 0)], random_walk=True)
    assert [q["id"] for q in added] == [b"e"]
    assert marshal_layer_map(go.layer_map) == b'{"0":["e"],"5":["b","c","b"]}'
