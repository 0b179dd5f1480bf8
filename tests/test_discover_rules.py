"""CPU tests: pin tests/discover_rules.py, the restatement of snowball discovery that tgi_state_discover /
tgi_state_next_layer are checked against, with the Philox known answers and hand-worked cases."""
import re

import discover_rules as dr
from state_rules import GoState

NOW = (1_700_000_000, 5)
E, S, F, N = dr.ST_EMITTED, dr.ST_SKIPPED, dr.ST_FAILED, dr.ST_NOLINE


def state(*pages, max_pages=0):
    go = GoState(max_pages)
    go.set_state([(0, [dict(p) for p in pages])])
    return go


def test_philox_known_answers():
    assert dr.philox4x32_10([0, 0, 0, 0], [0, 0]) == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    assert dr.philox4x32_10([dr.MASK] * 4, [dr.MASK] * 2) == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    assert dr.philox4x32_10([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], [0xA4093822, 0x299F31D0]) == \
        [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]


def test_page_ids_are_version_4_uuids():
    ids = [dr.page_id(seed, n) for seed in (0, 1, (1 << 64) - 1) for n in (0, 1, 2, 1 << 32, (1 << 64) - 1)]
    for u in ids:
        assert re.fullmatch(rb"[0-9a-f]{8}-[0-9a-f]{4}-4[0-9a-f]{3}-[89ab][0-9a-f]{3}-[0-9a-f]{12}", u), u
    assert len(set(ids)) == len(ids)
    # counter 0, key 0: the first known answer's bytes, little-endian, with the version and variant bits
    assert dr.page_id(0, 0) == b"d5e82766-8dc5-49e1-8cac-57bcd8db009b"


def test_outlinks_skip_the_owner_url_byte_for_byte_and_unprocessed_records():
    owner = {"id": b"o", "url": b"chan", "depth": 2}
    links = [[b"chan", b"a"], [b"b"], [b"c"], [b"d", b"chan"], [b"e"]]
    pages = dr.outlinks(owner, [E, S, F, N, E], links, 4)  # record 4 lies past n_done
    assert [p["url"] for p in pages] == [b"a", b"d"]
    assert all(p["parentId"] == b"o" and p["depth"] == 3 and p["status"] == b"unfetched" for p in pages)
    # the owner URL as the state holds it: a case-different URL is not the outlink
    assert [p["url"] for p in dr.outlinks({"id": b"o", "url": b"Chan"}, [E], [[b"chan"]], 1)] == [b"chan"]


def test_standalone_base_rules():
    go = state({"id": b"o", "url": b"chan", "depth": 0}, {"id": b"k", "url": b"known", "depth": 0})
    d = dr.Discovery(go, seed=7)
    added = d.standalone_page(b"o", [E, E], [[b"a", b"known", b"a"], [b"b", b"chan"]], 2, NOW)
    assert [p["url"] for p in added] == [b"a", b"b"]
    assert [p["id"] for p in added] == [dr.page_id(7, 0), dr.page_id(7, 1)]
    assert go.layer_map[1] == [p["id"] for p in added] and added[0]["timestamp"] == (NOW[0], NOW[1], None)
    # every candidate known: AddLayer still creates the layer of depth 1 (here it exists); from a depth-1 owner, depth 2
    assert d.standalone_page(added[0]["id"], [E], [[b"known"]], 1, NOW) == [] and go.layer_map[2] == []
    # no candidate at all: no call, no layer
    assert d.standalone_page(added[1]["id"], [E, F], [[b"b"], [b"x"]], 2, NOW) == [] and 3 not in go.layer_map
    assert d.n == 2


def test_max_pages_with_deadends():
    go = state({"id": b"o", "url": b"chan"}, {"id": b"x", "url": b"dead", "status": b"deadend"}, max_pages=2)
    d = dr.Discovery(go, seed=1)
    added = d.standalone_page(b"o", [E], [[b"a", b"b", b"c"]], 1, NOW, max_pages=2)
    assert [p["url"] for p in added] == [b"a"]  # the state is full: one replacement per deadend page
    assert d.standalone_page(b"o", [E], [[b"d"]], 1, NOW, max_pages=0)[0]["url"] == b"d"


def test_dapr_per_page_keeps_repeats_and_uses_the_url_cache():
    go = state({"id": b"o", "url": b"chan"})
    d = dr.Discovery(go, seed=3, url_cache={b"cached": b"id0"})
    added = d.standalone_page(b"o", [E, E], [[b"a", b"cached"], [b"a"]], 2, NOW, dapr=True)
    assert [p["url"] for p in added] == [b"a", b"a"] and d.url_cache[b"a"] == added[1]["id"]
    assert d.standalone_page(b"o", [E], [[b"a", b"cached"]], 1, NOW, dapr=True) == []
    assert sorted(go.layer_map) == [0, 1] and len(go.layer_map[1]) == 2


def test_layer_end_first_occurrence_wins_with_its_parent():
    go = state({"id": b"p", "url": b"P"}, {"id": b"q", "url": b"Q"})
    d = dr.Discovery(go, seed=9, url_cache={b"old": b"x"})
    disc = dr.outlinks(go.page_map[b"q"], [E], [[b"a", b"b"]], 1) + dr.outlinks(go.page_map[b"p"], [E], [[b"b", b"old"]], 1)
    added = d.layer_end(disc, 0, NOW)
    assert [(p["url"], p["parentId"], p["depth"]) for p in added] == [(b"a", b"q", 1), (b"b", b"q", 1)]
    assert d.layer_end([], 0, NOW) == [] and d.layer_end(disc, 0, NOW) == []
    assert sorted(go.layer_map) == [0, 1]  # Dapr: nothing added, no layer
    d.layer_end([c for c in disc if c["url"] != b"old"], 4, NOW, dapr=False)  # Base: every URL known, the layer is created
    assert go.layer_map[5] == []


def test_long_url_cache_entries_cannot_match_an_outlink():
    long = b"x" * 33
    assert dr.url_cache_keys([b"short", long, b"y" * 32]) == [b"short", b"y" * 32]
    for cache in ({long: b"1"}, {}):
        go = state({"id": b"o", "url": b"chan"})
        d = dr.Discovery(go, seed=2, url_cache=dict(cache))
        assert [p["url"] for p in d.standalone_page(b"o", [E], [[b"x" * 32]], 1, NOW, dapr=True)] == [b"x" * 32]
