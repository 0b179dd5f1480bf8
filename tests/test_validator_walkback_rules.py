"""CPU tests: tests/validator_walkback_rules.py, the restatement tgi_state_validator_walkback is checked against: the
reference's three processWalkbackBatch cases (crawl/validator_test.go:214-347), the walkback rate's edges, the
crawl_id fallback that the page and edge rows have and the stats rows do not, "unknown" for an empty source_type,
exhaustion by the exclude set alone, the five literals and the k-row grouping."""
import pytest

import tandem_sql_rules as sr
import validator_walkback_rules as vr
import walkback_rules as wr
from go_rules import _Raw

SEED = 0x5EED
T = _Raw(b'"2025-10-09T08:53:20.12Z"')


def batch(n=1, edges=(), **kw):
    b = {"batch_id": b"batch-%d" % n, "crawl_id": b"crawl-1", "source_channel": b"source_chan",
         "source_page_id": b"page-1", "source_depth": 0, "sequence_id": b"seq-1", "edges": list(edges)}
    b.update(kw)
    return b


def kinds(calls):
    return [k for k, _, _ in calls]


def test_forced_walkback_at_rate_50_with_a_one_key_set():
    b = batch(1, [(b"", b"mention", b"invalid"), (b"", b"url", b"not_channel")])
    res, calls = vr.process(b, [b"walkback_target"], 50, SEED, 0, b"cfg", T)
    assert res["status"] == vr.WALK_OK and res["walkback"] and res["rnd"] == -1 and res["draws"] == 1
    assert res["url"] == b"walkback_target" and res["forward_edge"] is None and res["n_valid"] == 0
    assert kinds(calls) == [vr.PAGE_BUFFER_INSERT, vr.EDGE_RECORD_INSERT, vr.BATCH_COMPLETE, vr.STATS_UPSERT,
                            vr.STATS_UPSERT, vr.EDGES_DELETE]
    page = sr.split_values(calls[0][2])
    assert page[2] == b"1" and page[3] == b'"walkback_target"' and page[5] == b'"%s"' % res["sequence_id"]
    edge = sr.split_values(calls[1][2])
    assert edge[2:4] == [b"true", b"false"] and edge[6] == b'"seq-1"'
    assert calls[3][2] == b'["crawl-1","mention",1,0,0,1,0]' and calls[4][2] == b'["crawl-1","url",1,0,1,0,0]'
    assert calls[2][2] == calls[5][2] == b'["batch-1"]'


def test_forward_at_rate_0_gives_one_primary_and_one_skipped_edge_and_no_draw_from_the_set():
    b = batch(2, [(b"chan_a", b"mention", b"valid"), (b"chan_b", b"url", b"valid"),
                  (b"bad_chan", b"plaintext", b"invalid")])
    res, calls = vr.process(b, [], 0, SEED, 3, b"cfg", T)  # an empty set: any draw from it would fail
    assert res["status"] == vr.WALK_OK and not res["walkback"] and 1 <= res["rnd"] <= 100 and res["draws"] == 0
    url = [b"chan_a", b"chan_b"][res["forward_edge"]]
    edges = [sr.split_values(p) for k, _, p in calls if k == vr.EDGE_RECORD_INSERT]
    assert [e[3] for e in edges] == [b"false", b"true"] and edges[0][2] == b"false"
    assert {edges[0][0], edges[1][0]} == {b'"chan_a"', b'"chan_b"'} and edges[0][0] == b'"%s"' % url
    page = sr.split_values(calls[0][2])
    assert page[3] == b'"%s"' % url and page[5] == b'"seq-1"'  # a forward page keeps the chain


def test_rate_100_gives_the_reference_call_order():
    b = batch(3, [(b"chan_a", b"mention", b"valid")])
    res, calls = vr.process(b, [b"walkback_url"], 100, SEED, 0, b"cfg", T)
    assert res["walkback"] and res["url"] == b"walkback_url" and 1 <= res["rnd"] <= 100
    # page, then SaveEdgeRecords (the primary and chan_a, which a walkback skips), complete, stats, delete
    assert kinds(calls) == [vr.PAGE_BUFFER_INSERT, vr.EDGE_RECORD_INSERT, vr.EDGE_RECORD_INSERT, vr.BATCH_COMPLETE,
                            vr.STATS_UPSERT, vr.EDGES_DELETE]
    assert sr.split_values(calls[2][2])[:4] == [b'"chan_a"', b'"source_chan"', b"false", b"true"]


@pytest.mark.parametrize("v", range(40))
def test_the_rate_bounds(v):
    b = batch(v, [(b"a", b"url", b"valid"), (b"b", b"url", b"duplicate")])
    keys = [b"k1", b"k2"]
    for rate in (-5, 0):
        assert not vr.process(b, keys, rate, SEED, v, b"", T)[0]["walkback"]
    for rate in (100, 250):
        assert vr.process(b, keys, rate, SEED, v, b"", T)[0]["walkback"]
    res = vr.process(b, keys, 15, SEED, v, b"", T)[0]
    assert res["walkback"] == (res["rnd"] <= 15)


def test_the_crawl_id_fallback_is_in_the_page_and_edge_rows_only():
    b = batch(4, [(b"a", b"url", b"valid"), (b"b", b"url", b"valid")], crawl_id=b"")
    _, calls = vr.process(b, [b"k"], 0, SEED, 0, b"configured", T)
    for k, _, p in calls:
        vals = sr.split_values(p)
        if k == vr.PAGE_BUFFER_INSERT:
            assert vals[4] == b'"configured"'
        elif k == vr.EDGE_RECORD_INSERT:
            assert vals[5] == b'"configured"'
        elif k == vr.STATS_UPSERT:
            assert vals[0] == b'""'


def test_an_empty_source_type_is_unknown_and_other_statuses_count_in_total_only():
    edges = [(b"a", b"", b"valid"), (b"b", b"unknown", b"pending"), (b"c", b"url", b"Valid"), (b"d", b"", b"duplicate")]
    assert vr.stats(edges) == [(b"unknown", [3, 1, 0, 0, 1]), (b"url", [1, 0, 0, 0, 0])]


def test_exhaustion_by_the_exclude_set_alone():
    b = batch(5, [(b"x1", b"url", b"valid"), (b"x2", b"url", b"valid")])
    res, calls = vr.process(b, [b"x1", b"x2"], 100, SEED, 0, b"", T)
    assert res["status"] == vr.WALK_EXHAUSTED and res["draws"] == 10 and res["url"] == b"" and calls == []
    res, calls = vr.process(b, [], 100, SEED, 0, b"", T)
    assert res["status"] == vr.WALK_EMPTY and res["draws"] == 0 and calls == []
    res, _ = vr.process(b, [b"x1", b"source_chan", b"X2", b"x2"], 100, SEED, 0, b"", T)
    assert res["status"] == vr.WALK_OK and res["url"] == b"X2"  # compares are byte for byte


def test_the_draw_stream_is_domain_5_and_the_ids_are_words_6_and_7():
    b = batch(6, [(b"a", b"url", b"valid")] * 3)
    res, _ = vr.process(b, [], 0, SEED, 9, b"", T)
    s = vr.words(SEED, 9)
    assert res["rnd"] == wr.lemire(100, s) + 1 and res["forward_edge"] == wr.lemire(3, s)
    assert (res["page_id"], res["sequence_id"]) == (wr.uuid(SEED, 9, 6), wr.uuid(SEED, 9, 7))


def test_texts_and_grouping():
    assert vr.sql_text(vr.BATCH_COMPLETE, 1) == vr.COMPLETE_SQL
    assert vr.sql_text(vr.BATCH_COMPLETE, 3) == \
        b"UPDATE pending_edge_batches SET status = 'completed', completed_at = NOW() WHERE batch_id IN ($1, $2, $3);"
    assert vr.sql_text(vr.EDGES_DELETE, 2) == b"DELETE FROM pending_edges WHERE batch_id IN ($1, $2);"
    assert vr.sql_text(vr.EDGE_RECORD_INSERT, 2).endswith(b"VALUES ($1, $2, $3, $4, $5, $6, $7), ($8, $9, $10, $11, "
                                                          b"$12, $13, $14);")
    with pytest.raises(AssertionError):
        vr.sql_text(vr.STATS_UPSERT, 2)
    bs = [batch(i, [(b"a%d" % i, b"url", b"valid"), (b"b", b"mention", b"valid")]) for i in range(5)]
    run = vr.run(bs, [b"k"], 50, SEED, 0, b"c", T)
    one = vr.statements(run, 1)
    assert [(k, s, p) for k, _, s, p in one] == sorted((c for _, cs in run for c in cs), key=lambda c: vr.KINDS.index(c[0]))
    for k in (2, 7, vr.MAX_ROWS):
        st = vr.statements(run, k)
        assert all(r == 1 for kind, r, _, _ in st if kind == vr.STATS_UPSERT)
        for kind in vr.KINDS:
            got = [v for kd, _, _, p in st if kd == kind for v in sr.split_values(p)]
            assert got == [v for kd, _, _, p in one if kd == kind for v in sr.split_values(p)]
