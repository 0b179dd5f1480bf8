"""GPU tests: page turns (tgi_state_page_begin / tgi_state_page_end) against tests/runner_rules.py over the restatement
of BaseStateManager — state.json byte for byte after every begin and every end of seeded random sequences, the work
list and json.Marshal(page), statuses from a real Telegram batch, and rejected calls that leave the state as it was."""
import random

import numpy as np
import pytest

import runner_rules as rr
from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import Engine, EngineError
from distributed_crawler_b200.pack import Channel, pack_telegram
from helpers import J, msg
from oracle.pyoracle import Oracle
from state_rules import marshal_page
from test_gpu_state import LAST, META, Sequence
from yt_corpus import make_youtube

pytestmark = pytest.mark.gpu
ST = [abi.ST_EMITTED, abi.ST_SKIPPED, abi.ST_FAILED, abi.ST_NOLINE]


class TurnSequence(Sequence):
    """Sequence's operations mixed with turns; up to two turns (of different pages) are open at a time"""

    def __init__(self, seed):
        super().__init__(seed)
        self.open = {}  # handle -> (page id, processed owner messages)

    def fetch(self, pid):
        r = self.rnd
        known = [(m["chatId"], m["messageId"]) for m in self.go.page_map[pid].get("messages") or []]
        pool = [(r.choice([-1001, -1002, 5, 9]), r.choice([5, 9, r.randrange(1, 40) << 20])) for _ in range(10)]
        pool += [(k, k) for k in (5, 9)]  # chat == message id: a swapped key equal to a real one
        pool += r.sample(known, min(len(known), 4))
        return [r.choice(pool) for _ in range(r.choice([0, 1, 5, 30, 120]))]

    def begin(self):
        r = self.rnd
        busy = {pid for pid, _ in self.open.values()}
        ids = [i for i in self.ids() if i not in busy]
        if not ids:
            return
        pid = r.choice(ids)
        fetched = self.fetch(pid)
        page = None
        if r.random() < 0.4:  # new fields for the owner, possibly of a depth without a layer
            page = self.page(r.randrange(6), False, [])
            page["id"] = pid
        want_json = r.random() < 0.5
        processed, work = rr.page_begin(self.go, pid, fetched, page)
        h, got_work, pj = self.e.state_page_begin(self.e._st_rows()[pid], fetched, page, want_json)
        assert list(got_work) == work
        if want_json:
            assert pj == marshal_page(self.go.page_map[pid], self.zone)
            if r.random() < 0.3:
                lines = self.e.state_export(abi.STATE_EXPORT_LOCAL)[0][0].split(b"\n")
                assert lines[self.e._st_rows()[pid]] == pj
        else:
            assert pj is None
        self.open[h] = (pid, processed)

    def end(self):
        r = self.rnd
        h = r.choice(list(self.open))
        pid, processed = self.open.pop(h)
        statuses = [r.choice(ST) for _ in processed]
        n_done = len(processed) if r.random() < 0.6 else r.randrange(len(processed) + 1)
        rr.page_end(self.go, pid, processed, statuses, n_done)
        self.e.state_page_end(h, n_done, status=statuses)

    def step(self):
        before = self.go.page_map
        k = self.rnd.random()
        if k < 0.35:
            self.begin()
        elif k < 0.65 and self.open:
            self.end()
        else:
            super().step()  # set / add_layer / update_page / update_messages / zone, and the check
            if self.go.page_map is not before:  # SetState: the rows are renumbered and every open turn is dropped
                self.open.clear()
            return
        self.check()


@pytest.mark.parametrize("seed", range(5))
def test_random_turn_sequences_match_the_restatement(seed):
    sq = TurnSequence(seed)
    pages = [sq.page(0, True, []) for _ in range(3)]
    sq.go.set_state([(0, pages)])
    sq.e.state_set([(0, pages)])
    for _ in range(160):
        sq.step()
    sq.e.close()


def test_compaction_between_begin_and_end():
    sq = TurnSequence(42)
    pages = [{"id": b"a", "url": b"ua", "depth": 0}, {"id": b"b<&>\xe2\x80\xa8", "url": b"ub", "depth": 0}]
    sq.go.set_state([(0, pages)])
    sq.e.state_set([(0, pages)])
    a, b = b"a", pages[1]["id"]
    fetched = [(-1001, j << 20) for j in range(50)]
    processed, work = rr.page_begin(sq.go, a, fetched)
    h, got, _ = sq.e.state_page_begin(sq.e._st_rows()[a], fetched)
    assert list(got) == work
    sq.check()
    for k in range(12):  # every turn of b drops its list: the tombstones outnumber the live rows and compact
        f = [(7, (j + k) << 20) for j in range(300)]
        pr, _ = rr.page_begin(sq.go, b, f)
        hb, _, pj = sq.e.state_page_begin(sq.e._st_rows()[b], f, None, True)
        assert pj == marshal_page(sq.go.page_map[b])
        st = [ST[(j + k) % 4] for j in range(len(pr))]
        rr.page_end(sq.go, b, pr, st, len(pr))
        sq.e.state_page_end(hb, len(pr), status=st)
        sq.check()
    st = [ST[j % 4] for j in range(len(processed))]
    rr.page_end(sq.go, a, processed, st, len(processed))
    assert sq.e.state_page_end(h, len(processed), status=st) == len(processed)
    sq.check()
    sq.e.close()


def fetched_messages(rnd, n):
    """a page of fetched messages: repeated keys, one id in two chats, panicking records and records before
    min_post_date"""
    keys = [(-100123, rnd.randrange(1, 30) << 20) if rnd.random() < 0.8 else (-100999, rnd.randrange(1, 30) << 20)
            for _ in range(n)]
    return [msg("messageText", "m%d " % k + "é" * (k % 7), id=m, chat_id=c, date=1_700_000_000 + k if k % 9 else 1_500_000_000,
                panics=k % 11 == 4) for k, (c, m) in enumerate(keys)]


def test_statuses_from_a_telegram_batch():
    cfg = dict(min_post_date=1_600_000_000)
    e = Engine(**cfg)
    rnd = random.Random(8)
    sq = TurnSequence(3)
    sq.e.close()
    sq.e = e
    pages = [{"id": b"chan-%d" % k, "url": b"https://t.me/c%d" % k, "depth": 1, "status": b"fetched",
              "timestamp": (1700000000, 0, 3600)} for k in range(3)]
    sq.go.set_state([(1, pages)])
    e.state_set([(1, pages)])
    seen = set()
    for turn in range(8):
        pid = pages[turn % 3]["id"]
        ms = fetched_messages(rnd, rnd.choice([0, 40, 100]))
        fetched = [(m.chat_id, m.id) for m in ms]
        processed, work = rr.page_begin(sq.go, pid, fetched)
        h, got, pj = e.state_page_begin(e._st_rows()[pid], fetched, None, True)
        assert list(got) == work and pj == marshal_page(sq.go.page_map[pid])
        if not work:  # nothing to process
            e.state_page_end(h, 0, status=[])
            sq.check()
            continue
        batch = pack_telegram([ms[i] for i in work], [Channel(name=b"c%d" % (turn % 3))])
        status = Oracle(**cfg).telegram(batch, J).status
        seen |= set(int(s) for s in status)
        slot = turn % 3
        e.telegram_submit(slot, batch, J)
        e.telegram_wait(slot)
        n_done = len(work) if turn % 4 else len(work) // 2  # a random-walk retire stops the loop early
        rr.page_end(sq.go, pid, processed, list(status), n_done)
        e.state_page_end(h, n_done, slot=slot)
        e.release(slot)
        sq.check()
    assert {abi.ST_EMITTED, abi.ST_SKIPPED, abi.ST_FAILED} <= seen
    e.close()


def test_rejected_calls_leave_the_state_unchanged():
    e = Engine()
    pages = [{"id": b"p", "url": b"u", "depth": 0}, {"id": b"q", "url": b"v", "depth": 0}]
    e.state_set([(0, pages)])
    ms = [msg("messageText", "x", id=(k + 1) << 20, chat_id=-5) for k in range(4)]
    fetched = [(m.chat_id, m.id) for m in ms]
    h, work, _ = e.state_page_begin(0, fetched)
    before = e.state_render(META, LAST)

    def rejected(call, code=abi.E_ARG):
        with pytest.raises(EngineError) as ei:
            call()
        assert ei.value.code == code
        assert e.state_render(META, LAST) == before

    rejected(lambda: e.state_page_begin(7, fetched))                        # no such row
    rejected(lambda: e.state_page_begin(0, fetched, {"id": b"q", "url": b"u"}))  # the page's id is not the row's
    rejected(lambda: e.state_page_end(h + 100, 0, status=[]))               # unknown handle
    rejected(lambda: e.state_page_end(h, 5, status=[0] * 5))                # n_done > n_work
    # the slot's result: a different record count, a YouTube result, a released result
    e.telegram_submit(0, pack_telegram(ms[:3]), J)
    e.telegram_wait(0)
    rejected(lambda: e.state_page_end(h, 3, slot=0))
    e.release(0)
    yt, _, _ = make_youtube(4, seed=2)
    e.youtube_submit(1, yt, J)
    e.youtube_wait(1)
    rejected(lambda: e.state_page_end(h, 4, slot=1))
    e.release(1)
    e.telegram_submit(2, pack_telegram(ms), J)
    e.telegram_wait(2)
    e.release(2)
    rejected(lambda: e.state_page_end(h, 4, slot=2))
    # the handle is still open after the rejections; it is consumed once
    e.telegram_submit(2, pack_telegram(ms), J)
    e.telegram_wait(2)
    assert e.state_page_end(h, 4, slot=2) == 4
    e.release(2)
    before = e.state_render(META, LAST)
    rejected(lambda: e.state_page_end(h, 0, status=[]))
    # tgi_state_set drops every open turn
    h2, _, _ = e.state_page_begin(1, fetched)
    e.state_set([(0, pages)])
    before = e.state_render(META, LAST)
    rejected(lambda: e.state_page_end(h2, 0, status=[]))
    e.close()
