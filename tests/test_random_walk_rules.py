"""CPU tests: tests/random_walk_rules.py, the restatement of the standard random walk, pinned against the reference's
own tests of the branch (tests/golden/random_walk_vectors.json) and hand cases: self links, names repeated within and
across pages, seed hits, an expired invalid entry, the walkback's exclusion of the page's new channels, exhaustion, an
empty discovered set, and a retire in the middle of a page followed by deferred pages."""
import json
import os

import pytest

import random_walk_rules as rw
import walkback_rules as wr

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "random_walk_vectors.json")
OWNER = {"id": b"page-1", "url": b"source_channel", "depth": 0, "sequenceId": b"seq-1"}
NOW, SEED, TIME = 1_760_000_000, 0x5EED, "T"
CODE = {"found": rw.FOUND, "not_supergroup": rw.NOT_SUPERGROUP, "not_found": rw.NOT_FOUND, "retire": rw.RETIRE}
MENTION, URL = 0, 2


def one_page(sm, links, outcomes, rate=0, owner=OWNER, n_done=None, u=0):
    """one page of one record per link list; outcomes: name -> (code, chat id)"""
    status = [0] * len(links)
    calls = []

    def search(name, record, src):
        calls.append(name)
        return outcomes[name]
    out, stats, n = rw.run(sm, [(owner, status, links, len(links) if n_done is None else n_done)], search, NOW, rate,
                           SEED, u, b"crawl-1", TIME)
    return out[0], stats, calls


def kinds(calls):
    return [k for k, _, _ in calls]


@pytest.mark.parametrize("v", json.load(open(GOLDEN))["standard_walk"], ids=lambda v: v["name"])
def test_reference_tests(v):
    ex = v["expect"]
    name = v["outlink"].encode()
    sm = rw.FakeState(discovered=[d.encode() for d in v["discovered"]])
    (res, calls), _, searched = one_page(sm, [[(name, MENTION)]], {name: (CODE[v["outcome"][0]], v["outcome"][1])},
                                         v["walkback_rate"])
    assert searched == [name]
    upserts = [json.loads(p) for k, _, p in calls if k == rw.SEED_UPSERT]
    invalid = [json.loads(p) for k, _, p in calls if k == rw.INVALID_UPSERT]
    assert upserts == ex["upsert_seed"] and invalid == ex["mark_invalid"]
    assert [d for d in sm.discovered if d.decode() not in v["discovered"]] == [d.encode() for d in ex["added_discovered"]]
    if ex["error"]:
        assert res["status"] == rw.RETIRED and not calls
        return
    assert res["status"] == rw.WALK_OK and res["walkback"] == ex["walkback"]
    page = [json.loads(p) for k, _, p in calls if k == rw.PAGE_BUFFER_INSERT]
    edges = [json.loads(p) for k, _, p in calls if k == rw.EDGE_RECORD_INSERT]
    assert [p[3] for p in page] == [ex["page_url"]]
    assert edges[0][:4] == [ex["page_url"], "source_channel", ex["walkback"], False] and edges[0][6] == "seq-1"
    assert page[0][5] == ("seq-1" if not ex["walkback"] else wr.uuid(SEED, 0, 10).decode())
    assert kinds(calls)[-1 - len(edges):] == [rw.PAGE_BUFFER_INSERT] + [rw.EDGE_RECORD_INSERT] * len(edges)


def test_self_links_and_repeats_are_looked_up_once():
    sm = rw.FakeState(discovered=[b"old"])
    links = [[(b"source_channel", URL), (b"aaa", MENTION), (b"bbb", URL)], [(b"aaa", URL), (b"bbb", MENTION)]]
    (res, calls), stats, searched = one_page(sm, links, {b"aaa": (rw.FOUND, 1), b"bbb": (rw.NOT_FOUND, 0)}, rate=100)
    assert searched == [b"aaa", b"bbb"]
    assert stats == {b"mention": [1, 0], b"url": [0, 1]}
    assert sm.discovered == [b"old", b"aaa"] and sm.invalid == {b"bbb": NOW} and sm.seeds == {b"aaa": 1}
    assert res["n_new"] == 1 and res["walkback"]
    # a later page: every name is known now, nothing is looked up
    (res2, calls2), _, searched2 = one_page(sm, links, {}, u=1)
    assert searched2 == [] and res2["n_new"] == 0 and res2["walkback"]
    assert kinds(calls2) in ([], [rw.PAGE_BUFFER_INSERT, rw.EDGE_RECORD_INSERT])


def test_seed_hit_is_discovered_without_a_lookup_or_an_edge():
    sm = rw.FakeState(discovered=[b"old"], seeds={b"seedy": 7})
    (res, calls), _, searched = one_page(sm, [[(b"seedy", MENTION)], [(b"seedy", URL)]], {})
    assert searched == [] and sm.discovered == [b"old", b"seedy"] and res["n_new"] == 0
    edges = [json.loads(p) for k, _, p in calls if k == rw.EDGE_RECORD_INSERT]
    assert len(edges) == 1 and edges[0][2] is True  # the walkback edge only


def test_expired_invalid_entry_is_looked_up_and_stamped_again():
    sm = rw.FakeState(invalid={b"stale": NOW - 30 * 24 * 3600, b"live": NOW - 5, b"never": 0})
    _, _, searched = one_page(sm, [[(b"stale", URL), (b"live", URL), (b"never", URL)]], {b"stale": (rw.NOT_SUPERGROUP, 0)})
    assert searched == [b"stale"] and sm.invalid[b"stale"] == NOW


def test_walkback_excludes_the_pages_new_channels():
    sm = rw.FakeState(discovered=[b"x"])
    (res, calls), _, _ = one_page(sm, [[(b"n1", URL), (b"n2", URL)]], {b"n1": (rw.FOUND, 1), b"n2": (rw.FOUND, 2)},
                                  rate=100)
    assert res["walkback"] and res["status"] == rw.WALK_OK and res["url"] == b"x"
    edges = [json.loads(p) for k, _, p in calls if k == rw.EDGE_RECORD_INSERT]
    assert [e[0] for e in edges] == ["x", "n1", "n2"] and [e[3] for e in edges] == [False, True, True]


def test_forward_pick_leaves_the_followed_channel_out_of_the_skipped_edges():
    sm = rw.FakeState()
    (res, calls), _, _ = one_page(sm, [[(b"n%d" % i, URL)] for i in range(5)], {b"n%d" % i: (rw.FOUND, i) for i in range(5)},
                                  rate=-1)
    assert not res["walkback"] and res["forward"] is not None
    edges = [json.loads(p)[0].encode() for k, _, p in calls if k == rw.EDGE_RECORD_INSERT]
    assert edges[0] == res["url"] and sorted(edges[1:]) == sorted(set(b"n%d" % i for i in range(5)) - {res["url"]})


def test_exhausted_and_empty_keep_the_upserts():
    sm = rw.FakeState(discovered=[b"source_channel"])
    (res, calls), _, _ = one_page(sm, [[(b"gone", URL)]], {b"gone": (rw.NOT_FOUND, 0)})
    assert res["status"] == rw.WALK_EXHAUSTED and res["draws"] == wr.MAX_ATTEMPTS and kinds(calls) == [rw.INVALID_UPSERT]
    (res, calls), _, _ = one_page(rw.FakeState(), [[(b"gone", URL)]], {b"gone": (rw.NOT_FOUND, 0)})
    assert res["status"] == rw.WALK_EMPTY and res["draws"] == 0 and kinds(calls) == [rw.INVALID_UPSERT]


def test_retire_mid_page_keeps_earlier_effects_and_defers_later_pages():
    sm = rw.FakeState(discovered=[b"d"])
    owners = [dict(OWNER, id=b"p%d" % k) for k in range(3)]
    pages = [(owners[0], [0], [[(b"a", URL)]], 1), (owners[1], [0, 0], [[(b"b", URL)], [(b"c", URL), (b"e", URL)]], 2),
             (owners[2], [0], [[(b"f", URL)]], 1)]
    outcomes = {b"a": (rw.FOUND, 1), b"b": (rw.NOT_FOUND, 0), b"c": (rw.RETIRE, 0)}
    out, stats, n_dec = rw.run(sm, pages, lambda n, i, s: outcomes[n], NOW, 0, SEED, 0, b"c", TIME)
    assert [r["status"] for r, _ in out] == [rw.WALK_OK, rw.RETIRED, rw.DEFERRED] and n_dec == 1
    assert kinds(out[1][1]) == [rw.INVALID_UPSERT] and out[2][1] == []
    assert sm.discovered == [b"d", b"a"] and b"b" in sm.invalid and b"e" not in sm.invalid
    assert rw.lookups(rw.FakeState(discovered=[b"d"]), pages, NOW) == [(b"a", 0, 0, URL), (b"b", 1, 0, URL),
                                                                        (b"c", 1, 1, URL), (b"e", 1, 1, URL),
                                                                        (b"f", 2, 0, URL)]


def test_statement_grouping():
    sm = rw.FakeState()
    pages = [(dict(OWNER, id=b"p%d" % k), [0], [[(b"q%d" % k, URL), (b"r%d" % k, URL)]], 1) for k in range(3)]
    outcomes = {**{b"q%d" % k: (rw.FOUND, k) for k in range(3)}, **{b"r%d" % k: (rw.NOT_FOUND, 0) for k in range(3)}}
    out, _, _ = rw.run(sm, pages, lambda n, i, s: outcomes[n], NOW, 0, SEED, 0, b"c", TIME)
    one, many = rw.statements(out, 1), rw.statements(out, rw.MAX_ROWS)
    assert [s[0] for s in many] == list(rw.KINDS) and sum(s[1] for s in many) == len(one)
    assert many[1][2] == (b"INSERT INTO invalid_channels (channel_username, reason, invalidated_at) VALUES ($1, $2, NOW()), "
                          b"($3, $4, NOW()), ($5, $6, NOW()) ON CONFLICT (channel_username) DO UPDATE SET reason = "
                          b"EXCLUDED.reason, invalidated_at = NOW();")
    assert json.loads(many[0][3]) == [x for s in one if s[0] == rw.SEED_UPSERT for x in json.loads(s[3])]
