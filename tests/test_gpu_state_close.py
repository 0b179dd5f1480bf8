"""GPU tests: the page close (tgi_state_page_close) against tests/close_rules.py over the restatement of
BaseStateManager — state.json, the layer map, both exports and json.Marshal(page) byte for byte after every close of
seeded sequences of turns, discovery, closes and the other state calls on states of 10^3 and 10^5 pages; closes without
an end, after a compaction and fed by a resident Telegram result; a whole small crawl; rejected calls."""
import base64
import ctypes as C
import random

import pytest

import close_rules as cr
import discover_rules as dr
from dapr_state_rules import export_dapr_chunks, export_local, marshal_layer_map
from distributed_crawler_b200 import abi, engine as eng
from distributed_crawler_b200.engine import Engine, EngineError
from distributed_crawler_b200.pack import pack_telegram
from distributed_crawler_b200.state_pack import pack_pages
from state_rules import marshal_page
from test_gpu_state import LAST, META, Sequence
from test_gpu_state_dapr import check_dapr
from test_gpu_state_discover import GOOD, MIN_DATE, RUN, oracle, page_messages
from tg_link_corpus import CHANNELS

pytestmark = pytest.mark.gpu
ST = [abi.ST_EMITTED, abi.ST_SKIPPED, abi.ST_FAILED, abi.ST_NOLINE]


class CloseSequence(Sequence):
    """turns (begin, end from the host or from a slot's result, discovery), closes, UpdatePage, AddLayer and Dapr's
    AddLayer over the restatement; the owner view of each page is tracked beside it"""

    def __init__(self, seed, n_pages):
        super().__init__(seed)
        self.e.close()
        self.e = Engine(min_post_date=MIN_DATE)
        self.d = dr.Discovery(self.go, seed=0xC105E000 + seed)
        self.e.state_id_seed(self.d.seed)
        self.open = {}   # handle -> (page id, processed owner messages)
        self.views = {}  # page id -> (owner messages, the handle whose end reaches them)
        r = self.rnd
        pages = [{"id": b"p%d" % k, "url": b"https://t.me/c%d" % k, "depth": k % 3, "status": b"unfetched",
                  "timestamp": (1700000000 + k, 0, 0),
                  "messages": [{"chatId": -1001, "messageId": (j + 1) << 20, "status": b"fetched", "pageId": b"p%d" % k}
                               for j in range(r.choice([0, 1, 2]))]} for k in range(n_pages)]
        layers = [(d, [p for p in pages if p["depth"] == d]) for d in range(3)]
        self.go.set_state(layers)
        self.e.state_set(layers)

    def full_check(self):
        self.check()
        check_dapr(self.e, self.go, self.zone, self.rnd)

    def fetch(self, pid):
        r = self.rnd
        known = [(m["chatId"], m["messageId"]) for m in self.go.page_map[pid].get("messages") or []]
        pool = [(r.choice([-1001, -1002, 5, 9]), r.choice([5, 9, r.randrange(1, 40) << 20])) for _ in range(10)]
        pool += [(k, k) for k in (5, 9)]  # chat == message id: a swapped key equal to an owner key
        pool += r.sample(known, min(len(known), 4))
        return [r.choice(pool) for _ in range(r.choice([0, 1, 5, 30, 100]))]

    def pick(self):
        busy = {pid for pid, _ in self.open.values()}
        ids = [i for i in self.ids() if i not in busy]
        return self.rnd.choice(ids) if ids else None

    def begin(self, pid, fetched):
        owner, processed, work = cr.page_begin(self.go, pid, fetched)
        h, got, _ = self.e.state_page_begin(self.e._st_rows()[pid], fetched)
        assert list(got) == work
        self.open[h] = (pid, processed)
        self.views[pid] = (owner, h)
        return h, processed, work

    def end(self, h, statuses, n_done, slot=-1):
        pid, processed = self.open.pop(h)
        owner, vh = self.views.get(pid, (None, None))
        cr.page_end(self.go, pid, owner if vh == h else None, processed, statuses, n_done)
        if slot >= 0:
            self.e.state_page_end(h, n_done, slot=slot)
        else:
            self.e.state_page_end(h, n_done, status=statuses)

    def close(self, pid, want_json=None):
        r = self.rnd
        page = self.page(r.randrange(4), False, [])
        page["id"] = pid
        page["status"] = r.choice([b"fetched", b"error", b"deadend"])
        if page["status"] == b"error":
            page["error"] = self.s(b"boom")
        want_json = r.random() < 0.5 if want_json is None else want_json
        cr.page_close(self.go, page, self.views.get(pid, (None, None))[0])
        pj = self.e.state_page_close(self.e._st_rows()[pid], page, want_json)
        for h in [h for h, (p, _) in self.open.items() if p == pid]:  # the close ends the row's open turns
            del self.open[h]
            with pytest.raises(EngineError) as ei:
                self.e.state_page_end(h, 0, status=[])
            assert ei.value.code == abi.E_ARG
        if want_json:
            assert pj == marshal_page(self.go.page_map[pid], self.zone)
        else:
            assert pj is None
        self.full_check()

    def turn_with_batch(self, pid, slot, close=True):
        """the crawl's flow for one channel: begin, process the work list as a Telegram batch, end with the slot's
        statuses, snowball discovery from the slot's result, close"""
        r = self.rnd
        msgs = page_messages(r, self.go.page_map[pid]["url"], r.choice([0, 5, 40]))
        h, processed, work = self.begin(pid, [(m.chat_id, m.id) for m in msgs])
        if work:
            batch = pack_telegram([msgs[i] for i in work], CHANNELS)
            ro = oracle(GOOD).telegram(batch, RUN)
            status = [int(s) for s in ro.status]
            links = [[n for n, _ in ro.record_links(i)] for i in range(ro.n)]
            self.e.telegram_submit(slot, batch, RUN)
            self.e.telegram_wait(slot)
            n_done = len(work) if r.random() < 0.7 else r.randrange(len(work) + 1)
            self.end(h, status, n_done, slot)
            now = (1_700_000_100 + r.randrange(100), 0)
            want = self.d.standalone_page(pid, status, links, n_done, now)
            got = self.e.state_discover(slot, [(self.e._st_rows()[pid], 0, len(work), n_done)], abi.DISCOVER_NOW, now)
            self.e.release(slot)
            assert got["ids"] == [p["id"] for p in want]
        else:
            self.end(h, [], 0)
        if close:
            self.close(pid)

    def other(self):
        """UpdatePage, AddLayer or Dapr's AddLayer, possibly overwriting a page: its owner view ends"""
        r = self.rnd
        before = dict(self.go.page_map)
        k = r.random()
        if k < 0.4:
            p = self.page(r.randrange(4), True, self.ids())
            if r.random() < 0.6:
                p["id"] = r.choice(self.ids())
                for m in p["messages"]:
                    m["pageId"] = p["id"]
            self.go.update_page(p)
            self.e.state_update_page(p)
        elif k < 0.7:
            ps = [self.page(r.randrange(4), False, self.ids()) for _ in range(r.randrange(1, 5))]
            want = self.go.add_layer(ps)
            assert [x != abi.STATE_NO_PAGE for x in self.e.state_add_layer(ps)] == want
        else:
            ps = [self.page(r.randrange(4), False, self.ids()) for _ in range(r.randrange(1, 4))]
            for p in ps:
                self.go.page_map[p["id"]] = dict(p)
                self.go.layer_map.setdefault(ps[0]["depth"], []).append(p["id"])
            self.e.state_add_pages(ps[0]["depth"], ps)
        for pid in list(self.views):
            if self.go.page_map.get(pid) is not before.get(pid):
                del self.views[pid]

    def step(self, slot):
        r = self.rnd
        k = r.random()
        pid = self.pick()
        if k < 0.3 and pid is not None:
            h, processed, _ = self.begin(pid, self.fetch(pid))
            if r.random() < 0.6:
                statuses = [r.choice(ST) for _ in processed]
                self.end(h, statuses, len(processed) if r.random() < 0.6 else r.randrange(len(processed) + 1))
        elif k < 0.45 and self.open:
            h = r.choice(list(self.open))
            self.end(h, [r.choice(ST) for _ in self.open[h][1]], r.randrange(len(self.open[h][1]) + 1))
        elif k < 0.75:
            owned = [p for p in self.views if r.random() < 0.8] or self.ids()
            self.close(r.choice(owned))
        elif k < 0.85 and pid is not None:
            self.turn_with_batch(pid, slot, close=r.random() < 0.7)
        else:
            self.other()


@pytest.mark.parametrize("seed", range(3))
def test_random_sequences_on_a_thousand_pages(seed):
    sq = CloseSequence(seed, 1000)
    for i in range(120):
        sq.step(i % 3)
    sq.e.close()


def test_random_sequence_on_a_hundred_thousand_pages():
    sq = CloseSequence(11, 100_000)
    sq.full_check = sq.check  # the layer map and the exports of 10^5 pages are checked once, at the end
    closes = i = 0
    while closes < 8:
        k = sq.rnd.random()
        pid = sq.pick()
        if k < 0.4:
            h, processed, _ = sq.begin(pid, sq.fetch(pid))
            sq.end(h, [sq.rnd.choice(ST) for _ in processed], len(processed))
            sq.close(pid)
            closes += 1
        elif k < 0.6:
            sq.turn_with_batch(pid, i % 3)
            closes += 1
        else:
            sq.other()
        i += 1
    assert sq.e.state_layer_map() == marshal_layer_map(sq.go.layer_map)
    want = export_local(sq.go)
    assert sq.e.state_export(abi.STATE_EXPORT_LOCAL, 0) == [(want, len(want))]
    want = export_dapr_chunks(sq.go, abi.STATE_EXPORT_CHUNK_DEFAULT)
    assert [base64.b64decode(d) for d, _ in sq.e.state_export(abi.STATE_EXPORT_DAPR)] == want
    sq.e.close()


def test_close_without_end_after_compaction_and_twice():
    sq = CloseSequence(5, 4)
    a, b = b"p0", b"p1"
    fetched = [(-1001, j << 20) for j in range(1, 40)] + [(5, 9), (9, 5)]
    sq.begin(a, fetched)
    sq.close(a, True)  # no end: every owner message is still "resample"
    h, processed, _ = sq.begin(a, [(7, 7), (15, 19), (19, 15)] + [(-1001, j << 20) for j in range(100, 140)])
    for k in range(12):  # turns of b drop their lists: the tombstones outnumber the live rows and compact
        hb, pr, _ = sq.begin(b, [(7, (j + k) << 20) for j in range(300)])
        sq.end(hb, [ST[(j + k) % 4] for j in range(len(pr))], len(pr))
        sq.close(b, k % 2 == 0)
    sq.end(h, [abi.ST_FAILED] * len(processed), len(processed))  # (7, 7), (19, 15), (15, 19) hit before any append
    assert [m["status"] for m in sq.views[a][0][:3]] == [b"failed"] * 3
    sq.close(a, True)
    once = sq.e.state_render(META, LAST)
    page = {k: v for k, v in sq.go.page_map[a].items() if k != "messages"}
    sq.e.state_page_close(sq.e._st_rows()[a], page)  # the runner's UpdatePage(page) after the loop's: the same list
    assert sq.e.state_render(META, LAST) == once
    sq.e.close()


def test_a_small_crawl_equals_the_reference_state():
    sq = CloseSequence(21, 6)
    for layer in range(2):
        channels = [p for p in sq.ids() if sq.go.page_map[p].get("depth", 0) == layer][:6]
        for i, pid in enumerate(channels):
            sq.turn_with_batch(pid, i % 3)
    want = sq.go.marshal(META, LAST)
    assert sq.e.state_render(META, LAST) == want
    assert b'"status":"fetched"' in want and b'"messages":[' in want
    sq.e.close()


def test_rejected_calls_leave_the_state_unchanged():
    sq = CloseSequence(8, 3)
    e = sq.e
    h, processed, _ = sq.begin(b"p0", [(-5, (k + 1) << 20) for k in range(4)])
    before = e.state_render(META, LAST)
    page = {"id": b"p0", "url": b"u", "status": b"fetched"}

    def rejected(call):
        with pytest.raises(EngineError) as ei:
            call()
        assert ei.value.code == abi.E_ARG
        assert e.state_render(META, LAST) == before

    rejected(lambda: e.state_page_close(7, page))                       # no such row
    rejected(lambda: e.state_page_close(1, page))                       # the id is not the row's
    rejected(lambda: e.state_page_close(0, dict(page, timestamp=(0, 10**9, 0))))  # nsec out of range
    recs, strs, msgs = pack_pages([dict(page, messages=[{"chatId": 1, "messageId": 2, "status": b"fetched",
                                                         "pageId": b"p0"}])], e.state_code, lambda pid, i: 0)
    out = abi.StateJsonC()
    for rc in (eng.lib().tgi_state_page_close(e.h, 0, recs.ctypes.data, strs.ctypes.data, len(strs), 0, C.byref(out)),  # messages
               eng.lib().tgi_state_page_close(e.h, 0, recs.ctypes.data, strs.ctypes.data, len(strs), 8, C.byref(out)),  # flags
               eng.lib().tgi_state_page_close(e.h, 0, recs.ctypes.data, None, len(strs), 0, C.byref(out))):  # strings
        assert rc == abi.E_ARG
        assert e.state_render(META, LAST) == before
    # the turn is still open after the rejections; the close ends it
    sq.close(b"p0")
    with pytest.raises(EngineError) as ei:
        e.state_page_end(h, 0, status=[])
    assert ei.value.code == abi.E_ARG
    # a year json.Marshal refuses: TGI_E_ARG after the update, as Dapr's UpdatePage
    bad = dict(sq.go.page_map[b"p0"], timestamp=(400_000_000_000, 0, 0))
    bad.pop("messages", None)
    cr.page_close(sq.go, bad, sq.views[b"p0"][0])
    with pytest.raises(EngineError) as ei:
        e.state_page_close(0, bad, True)
    assert ei.value.code == abi.E_ARG
    assert e.state_read_page(0) == [dict({"platform": b""}, **m) for m in sq.go.page_map[b"p0"]["messages"]]
    e.close()
