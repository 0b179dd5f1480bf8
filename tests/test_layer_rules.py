"""CPU tests: the layer-read restatement (tests/layer_rules.py) on hand-made states whose answers are written out here —
Dapr's duplicate URLs, standalone resume against a new execution, empty and missing layers, negative depths, and a
layer that lists an id twice."""
import layer_rules as lr
from state_rules import GoState


def page(pid, url, status, depth=0):
    return {"id": pid, "url": url, "status": status, "depth": depth}


def test_dapr_records_a_url_before_its_status_test():
    layer = [page(b"a", b"u1", b"fetched"), page(b"b", b"u1", b"unfetched"), page(b"c", b"u2", b"error"),
             page(b"d", b"u2", b"unfetched"), page(b"e", b"u3", b"unfetched"), page(b"f", b"u3", b"unfetched"),
             page(b"g", b"U3", b"processing"), page(b"h", b"u4", b"failed")]
    # a fetched or errored first page hides every later page of its URL; URLs compare byte for byte
    assert lr.dapr_selection(layer) == [False, False, False, False, True, False, True, True]
    # the new-execution branch (not reachable from ProcessLayersIteratively) keeps fetched and errored first pages
    assert lr.dapr_selection(layer, resuming=False) == [True, False, True, False, True, False, True, True]


def test_standalone_resume_against_a_new_execution():
    layer = [page(b"a", b"u1", b"fetched"), page(b"b", b"u2", b"fetched"), page(b"c", b"u3", b"unfetched"),
             page(b"d", b"u4", b"fetched"), page(b"e", b"u3", b"error"), page(b"f", b"u5", b"Fetched")]
    assert lr.standalone_selection(layer, resuming=True) == [False, False, True, False, True, True]
    assert lr.standalone_selection(layer, resuming=False) == [True] * 6
    assert lr.standalone_selection([page(b"a", b"u", b"fetched")] * 3, resuming=True) == [False] * 3
    assert lr.standalone_selection([], resuming=True) == [] == lr.dapr_selection([])


def test_empty_missing_and_negative_layers():
    go = GoState()
    assert lr.get_layer_by_depth(go, 0) == [] and lr.get_max_depth(go) is None and lr.incomplete_pages(go) == 0
    go.set_state([(-3, [page(b"a", b"u1", b"unfetched", -3)]), (-1, [])])
    # GetMaxDepth starts at -1: layers at -1 and below leave it there, which is its "no layers found"
    assert lr.get_max_depth(go) is None
    assert [p["id"] for p in lr.get_layer_by_depth(go, -3)] == [b"a"]
    assert lr.get_layer_by_depth(go, -1) == [] and lr.get_layer_by_depth(go, 4) == []
    assert lr.incomplete_pages(go) == 1
    go.set_state([(-3, [page(b"a", b"u1", b"fetched", -3)]), (0, []), (2, [])])
    assert lr.get_max_depth(go) == 2 and lr.incomplete_pages(go) == 0
    go.set_state([(0, [page(b"a", b"u1", b"fetched")])])
    assert lr.get_max_depth(go) == 0


def test_a_layer_that_lists_an_id_twice():
    # SetState with a repeated id: pageMap keeps the later page, the layer lists the id twice
    go = GoState()
    go.set_state([(1, [page(b"a", b"u1", b"fetched", 1), page(b"b", b"u2", b"unfetched", 1),
                       page(b"a", b"u3", b"unfetched", 1)])])
    layer = lr.get_layer_by_depth(go, 1)
    assert [(p["id"], p["url"]) for p in layer] == [(b"a", b"u3"), (b"b", b"u2"), (b"a", b"u3")]
    assert lr.incomplete_pages(go) == 3
    assert lr.standalone_selection(layer, resuming=True) == [True, True, True]
    assert lr.dapr_selection(layer) == [True, True, False]
