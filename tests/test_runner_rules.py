"""CPU: tests/runner_rules.py, the restatement of processAllMessagesWithProcessor's bookkeeping, on hand-written cases
and against the same flow composed from state_join's functions over the oracle's join."""
import random

import numpy as np

import runner_rules as rr
from distributed_crawler_b200 import state_join
from oracle.pyoracle import Oracle
from state_rules import GoState

EMITTED, SKIPPED, FAILED, NOLINE = 0, 1, 2, 3


def state(msgs):
    go = GoState()
    go.set_state([(0, [{"id": b"p", "url": b"u", "messages": [
        {"chatId": c, "messageId": m, "status": s, "pageId": b"p"} for c, m, s in msgs]}])])
    return go


def listed(go):
    return [(m["chatId"], m["messageId"], m["status"]) for m in go.get_page(b"p").get("messages") or []]


def turn(go, fetched, statuses, n_done=None):
    processed, work = rr.page_begin(go, b"p", fetched)
    rr.page_end(go, b"p", processed, statuses, len(processed) if n_done is None else n_done)
    return work


def test_worked_example():
    go = state([(1, 10, b"fetched")])
    processed, work = rr.page_begin(go, b"p", [(1, 10), (1, 11), (1, 11), (2, 11)])
    assert listed(go) == [(1, 11, b"resample"), (1, 11, b"resample"), (2, 11, b"resample")]
    assert work == [1, 1, 1]
    rr.page_end(go, b"p", processed, [EMITTED, FAILED, SKIPPED], 3)
    assert listed(go) == [(1, 11, b"resample"), (1, 11, b"resample"), (2, 11, b"resample"), (11, 1, b"failed"),
                          (11, 2, b"fetched")]
    assert all(m["pageId"] == b"p" for m in go.get_page(b"p")["messages"])


def test_empty_fetch_empties_the_list():
    go = state([(1, 10, b"fetched"), (1, 11, b"unfetched")])
    assert turn(go, [], []) == []
    assert listed(go) == []


def test_all_known_fetch_drops_the_list():
    go = state([(1, 10, b"fetched"), (1, 11, b"failed")])
    assert turn(go, [(1, 11), (1, 10)], []) == []
    assert listed(go) == []


def test_duplicate_keys_are_kept_twice():
    go = state([])
    assert turn(go, [(5, 1), (5, 1), (5, 2)], [FAILED, EMITTED, NOLINE]) == [0, 0, 2]
    # (1, 5) is appended by the first update, and the second update of that swapped key hits it
    assert listed(go) == [(5, 1, b"resample"), (5, 1, b"resample"), (5, 2, b"resample"), (1, 5, b"fetched"),
                          (2, 5, b"fetched")]


def test_one_message_id_in_two_chats():
    go = state([])
    assert turn(go, [(7, 3), (8, 3)], [EMITTED, FAILED]) == [0, 0]
    assert listed(go) == [(7, 3, b"resample"), (8, 3, b"resample"), (3, 7, b"fetched"), (3, 8, b"failed")]


def test_swapped_keys_that_collide_with_real_keys():
    go = state([])
    # (4, 4) swaps to itself and hits its own message; (6, 9) swaps to (9, 6), which was fetched too
    assert turn(go, [(4, 4), (6, 9), (9, 6)], [FAILED, EMITTED, FAILED]) == [0, 1, 2]
    assert listed(go) == [(4, 4, b"failed"), (6, 9, b"failed"), (9, 6, b"fetched")]


def test_n_done_zero_and_partial():
    go = state([])
    assert turn(go, [(1, 1), (1, 2), (1, 3)], [FAILED] * 3, n_done=0) == [0, 1, 2]
    assert listed(go) == [(1, 1, b"resample"), (1, 2, b"resample"), (1, 3, b"resample")]
    go = state([])
    turn(go, [(1, 1), (1, 2), (1, 3)], [FAILED, EMITTED, EMITTED], n_done=2)
    assert listed(go) == [(1, 1, b"failed"), (1, 2, b"resample"), (1, 3, b"resample"), (2, 1, b"fetched")]


def composed(join, page_keys, fetched, statuses, n_done):
    """the same flow from state_join: the page's keys and statuses after the turn, and the work list"""
    fk = np.array(fetched, np.int64).reshape(-1, 2)
    keys = fk[state_join.add_new_messages(join, fk, np.array(page_keys, np.int64).reshape(-1, 2))]
    status = state_join.resample_marker(join, keys, ["unfetched"] * len(keys), fk)
    by_id = lambda k: np.stack([np.zeros(len(k), np.int64), k[:, 1]], 1)  # noqa: E731  the look-up ignores the chat
    work = state_join.find_fetched(join, by_id(fk), by_id(keys))
    upd = keys[:n_done, ::-1]
    keys, status = state_join.update_messages_batch(join, keys, status, upd,
                                                    ["failed" if s == FAILED else "fetched" for s in statuses[:n_done]])
    return [(int(c), int(m), s.encode()) for (c, m), s in zip(keys, status)], [int(w) for w in work]


def test_random_turns_match_the_state_join_composition():
    rnd = random.Random(5)
    for trial in range(300):
        pool = [(rnd.choice([1, 2, 3, 40]), rnd.randrange(1, 9)) for _ in range(12)]
        old = [(c, m, rnd.choice([b"fetched", b"failed", b"resample"])) for c, m in
               (rnd.choice(pool) for _ in range(rnd.randrange(0, 10)))]
        fetched = [rnd.choice(pool) for _ in range(rnd.randrange(0, 16))]
        go = state(old)
        processed, work = rr.page_begin(go, b"p", fetched)
        statuses = [rnd.choice([EMITTED, SKIPPED, FAILED, NOLINE]) for _ in processed]
        n_done = rnd.randrange(len(processed) + 1)
        rr.page_end(go, b"p", processed, statuses, n_done)
        want, want_work = composed(Oracle.key_join, [(c, m) for c, m, _ in old], fetched, statuses, n_done)
        assert (listed(go), work) == (want, want_work), trial
