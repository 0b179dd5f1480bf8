"""CPU tests: the restatement of the page close (tests/close_rules.py) on hand-built cases."""
import random

import close_rules as cr
import runner_rules as rr
from state_rules import GoState

F = 0  # any status but abi.ST_FAILED: "fetched"


def state(messages=()):
    go = GoState()
    go.set_state([(0, [{"id": b"p", "url": b"https://t.me/p", "depth": 0, "status": b"unfetched",
                        "messages": [dict(m, pageId=b"p") for m in messages]}])])
    return go


def fields(**kw):
    return dict({"id": b"p", "url": b"https://t.me/p", "depth": 0, "status": b"fetched"}, **kw)


def keys(go):
    return [(m["chatId"], m["messageId"], m["status"]) for m in go.page_map[b"p"].get("messages") or []]


def test_the_swapped_appends_are_dropped():
    go = state([{"chatId": -100, "messageId": 1 << 20, "status": b"fetched"}])
    fetched = [(-100, 1 << 20), (-100, 2 << 20), (-100, 3 << 20), (-100, 2 << 20)]
    owner, processed, _ = cr.page_begin(go, b"p", fetched)
    assert cr.page_end(go, b"p", owner, processed, [F, rr.ST_FAILED, F], 3) == 0
    assert len(go.page_map[b"p"]["messages"]) == 5  # the owner's three and two swapped keys (the third is the first's)
    cr.page_close(go, fields(), owner)
    assert keys(go) == [(-100, 2 << 20, b"resample"), (-100, 3 << 20, b"resample"), (-100, 2 << 20, b"resample")]
    assert go.page_map[b"p"]["status"] == b"fetched"


def test_hits_before_the_first_append_reach_the_owner():
    go = state()
    owner, processed, _ = cr.page_begin(go, b"p", [(5, 9), (9, 5), (7, 8)])
    # (9, 5) hits owner message 1, (5, 9) owner message 0, then (8, 7) appends
    assert cr.page_end(go, b"p", owner, processed, [rr.ST_FAILED, F, F], 3) == 2
    cr.page_close(go, fields(), owner)
    assert keys(go) == [(5, 9, b"fetched"), (9, 5, b"failed"), (7, 8, b"resample")]


def test_hits_after_the_first_append_do_not():
    go = state()
    owner, processed, _ = cr.page_begin(go, b"p", [(7, 8), (5, 9), (9, 5)])
    assert cr.page_end(go, b"p", owner, processed, [F, F, F], 3) == 0  # (8, 7) appends first
    assert keys(go)[:3] == [(7, 8, b"resample"), (5, 9, b"fetched"), (9, 5, b"fetched")]  # pageMap's own array
    cr.page_close(go, fields(), owner)
    assert keys(go) == [(7, 8, b"resample"), (5, 9, b"resample"), (9, 5, b"resample")]


def test_the_last_hit_wins_and_a_repeated_key_hits_its_first_message():
    go = state()
    owner, processed, _ = cr.page_begin(go, b"p", [(3, 3), (3, 3), (4, 6)])
    assert cr.page_end(go, b"p", owner, processed, [rr.ST_FAILED, F, F], 2) == 2
    cr.page_close(go, fields(), owner)
    assert keys(go) == [(3, 3, b"fetched"), (3, 3, b"resample"), (4, 6, b"resample")]


def test_a_close_without_a_view_changes_fields_only():
    msgs = [{"chatId": -1, "messageId": 4, "status": b"fetched"}, {"chatId": 4, "messageId": -1, "status": b"failed"}]
    go = state(msgs)
    before = keys(go)
    cr.page_close(go, fields(status=b"error", error=b"boom"), None)
    assert keys(go) == before
    assert go.page_map[b"p"]["status"] == b"error" and go.page_map[b"p"]["error"] == b"boom"


def test_a_second_close_is_idempotent():
    go = state()
    owner, processed, _ = cr.page_begin(go, b"p", [(-100, 1 << 20), (-100, 2 << 20)])
    cr.page_end(go, b"p", owner, processed, [F, F], 2)
    cr.page_close(go, fields(), owner)
    once = go.marshal(b"{}", b'""')
    cr.page_close(go, fields(), owner)
    assert go.marshal(b"{}", b'""') == once


def test_status_and_url_changes_move_what_add_layer_counts():
    go = GoState(max_pages=1)
    go.set_state([(0, [{"id": b"p", "url": b"https://t.me/p", "depth": 0, "status": b"unfetched"}])])
    owner, _, _ = cr.page_begin(go, b"p", [])
    new = {"id": b"n", "url": b"https://t.me/n", "depth": 1}
    assert go.add_layer([dict(new)]) == [False]  # the state is full and holds no deadend
    cr.page_close(go, fields(status=b"deadend", url=b"https://t.me/q"), owner)
    # the deadend buys one page past max_pages; the old URL no longer blocks, the new one does
    assert go.add_layer([{"id": b"x", "url": b"https://t.me/q", "depth": 1}, dict(new, url=b"https://t.me/p")]) == [False, True]
    go = GoState(max_pages=2)
    go.set_state([(0, [{"id": b"p", "url": b"https://t.me/p", "depth": 0, "status": b"deadend"},
                       {"id": b"o", "url": b"https://t.me/o", "depth": 0, "status": b"fetched"}])])
    cr.page_close(go, fields(), None)  # deadend -> fetched: no budget left
    assert go.add_layer([dict(new)]) == [False]


def test_telegram_keys_never_hit_the_owner():
    rnd = random.Random(5)
    for _ in range(300):
        go = state()
        fetched = [(-rnd.randrange(1, 4) * 1000000000000 - rnd.randrange(100), rnd.randrange(1, 60) << 20)
                   for _ in range(rnd.randrange(0, 40))]
        owner, processed, _ = cr.page_begin(go, b"p", fetched)
        statuses = [rnd.choice([F, rr.ST_FAILED]) for _ in processed]
        assert cr.page_end(go, b"p", owner, processed, statuses, rnd.randrange(len(processed) + 1)) == 0
        cr.page_close(go, fields(), owner)
        assert all(m["status"] == b"resample" for m in go.page_map[b"p"].get("messages") or [])
