"""GPU tests: multi-page turns (tgi_state_pages_begin / _end / _close) against the restatements applied page by page in
call order (tests/close_rules.py over state_rules.GoState), and against the one-page calls on a second context: state.json,
the layer map, both exports, every work list and page JSON; a bulk Telegram result whose turn sits inside it, read by the
end and by discovery from the spans of work_off; edge cases; rejected calls; launch counts that do not depend on P."""
import hashlib
import random

import numpy as np
import pytest

import close_rules as cr
import discover_rules as dr
from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import Engine, EngineError
from distributed_crawler_b200.pack import pack_telegram
from state_rules import marshal_page
from test_gpu_state import LAST, META
from test_gpu_state_close import ST, CloseSequence
from test_gpu_state_discover import GOOD, RUN, oracle, page_messages
from test_gpu_state import NY
from tg_link_corpus import CHANNELS
from yt_corpus import make_youtube

pytestmark = pytest.mark.gpu
PER_PAGE = 100


class PagesSequence(CloseSequence):
    """CloseSequence with multi-page begins, ends and closes mixed into its steps"""

    def pages_begin(self, pids, fetched, want_json):
        rows = [self.e._st_rows()[p] for p in pids]
        want = [cr.page_begin(self.go, p, f) for p, f in zip(pids, fetched)]
        h, work, off, pj = self.e.state_pages_begin(rows, fetched, None, want_json)
        base = np.concatenate([[0], np.cumsum([len(f) for f in fetched])])
        for k, (pid, (owner, processed, w)) in enumerate(zip(pids, want)):
            assert list(work[off[k]:off[k + 1]] - base[k]) == w
            self.views[pid] = (owner, h)
            if want_json:
                assert pj[k] == marshal_page(self.go.page_map[pid], self.zone)
        self.open[h] = (tuple(pids), [w[1] for w in want])
        self.check()
        return h, [w[1] for w in want]

    def pages_end(self, h, n_done):
        pids, processed = self.open.pop(h)
        status = []
        for pid, pr, nd in zip(pids, processed, n_done):
            st = [self.rnd.choice(ST) for _ in pr]
            owner, vh = self.views.get(pid, (None, None))
            cr.page_end(self.go, pid, owner if vh == h else None, pr, st, nd)
            status += st
        self.e.state_pages_end(h, n_done, status=status)
        self.check()

    def end(self, h, statuses, n_done, slot=-1):
        if isinstance(self.open[h][0], tuple):  # a multi-page handle: its pages' own counts
            return self.pages_end(h, [self.rnd.randrange(len(pr) + 1) for pr in self.open[h][1]])
        return super().end(h, statuses, n_done, slot)

    def pages_close(self, pids, want_json):
        pages = []
        for pid in pids:
            page = self.page(self.rnd.randrange(4), False, [])
            page["id"], page["status"] = pid, self.rnd.choice([b"fetched", b"deadend"])
            cr.page_close(self.go, page, self.views.get(pid, (None, None))[0])
            pages.append(page)
        pj = self.e.state_pages_close([self.e._st_rows()[p] for p in pids], pages, want_json)
        for h in [h for h, (p, _) in self.open.items() if set(p if isinstance(p, tuple) else (p,)) & set(pids)]:
            del self.open[h]  # a close of any of its rows ends the whole turn
            with pytest.raises(EngineError) as ei:
                self.e.state_pages_end(h, None, status=[])
            assert ei.value.code == abi.E_ARG
        if want_json:
            assert pj == [marshal_page(self.go.page_map[p], self.zone) for p in pids]
        self.full_check()

    def close(self, pid, want_json=None):
        multi = [h for h, (p, _) in self.open.items() if isinstance(p, tuple) and pid in p]
        for h in multi:
            del self.open[h]
        super().close(pid, want_json)
        for h in multi:  # the one-page close of any of its rows ends the whole turn
            with pytest.raises(EngineError):
                self.e.state_pages_end(h, None, status=[])

    def free(self):
        busy = set()
        for p, _ in self.open.values():
            busy |= set(p if isinstance(p, tuple) else (p,))
        return [i for i in self.ids() if i not in busy]

    def multi_step(self):
        r = self.rnd
        k = r.random()
        free = self.free()
        if k < 0.4 and len(free) >= 2:
            pids = r.sample(free, r.randrange(2, min(6, len(free)) + 1))
            h, processed = self.pages_begin(pids, [self.fetch(p) for p in pids], r.random() < 0.5)
            if r.random() < 0.6:
                self.pages_end(h, [r.choice([0, len(pr), r.randrange(len(pr) + 1)]) for pr in processed])
        elif k < 0.55 and any(isinstance(p, tuple) for p, _ in self.open.values()):
            h = r.choice([h for h, (p, _) in self.open.items() if isinstance(p, tuple)])
            self.pages_end(h, [r.randrange(len(pr) + 1) for pr in self.open[h][1]])
        elif k < 0.8:
            owned = [p for p in self.views if r.random() < 0.8] or self.ids()
            self.pages_close(r.sample(owned, min(len(owned), r.randrange(1, 5))), r.random() < 0.5)
        elif k < 0.85:  # time.Local changes: the page JSON and state.json render in the new zone
            self.zone = NY if self.zone is None else None
            self.e.set_zone(*(self.zone or ([], [])))
            self.check()
        else:
            self.step(0)


@pytest.mark.parametrize("seed", range(3))
def test_random_sequences_mix_multi_and_single_page_calls(seed):
    sq = PagesSequence(seed, 1000)
    for i in range(80):
        if sq.rnd.random() < 0.05:  # SetState drops every open turn and view
            layers = [(0, [dict(sq.go.page_map[p], messages=[]) for p in sq.ids()[:300]])]
            sq.go.set_state(layers)
            sq.e.state_set(layers)
            for h in list(sq.open):
                with pytest.raises(EngineError):
                    sq.e.state_pages_end(h, None, status=[])
            sq.open.clear()
            sq.views.clear()
            sq.check()
        sq.multi_step()
    sq.e.close()


def state_arrays(n_pages):
    ids = [b"%08x-0000-4000-8000-%012x" % (p, p) for p in range(n_pages)]
    urls = [b"https://t.me/channel_%07d" % p for p in range(n_pages)]
    recs = np.zeros(n_pages, abi.STATE_PAGE)
    recs["str_len"][:, 0] = [len(i) for i in ids]
    recs["str_len"][:, 1] = [len(u) for u in urls]
    recs["str_len"][:, 2] = 7
    recs["str_off"] = np.concatenate([[0], np.cumsum(recs["str_len"].sum(1).astype(np.uint64))[:-1]])
    blob = np.frombuffer(b"".join(i + u + b"fetched" for i, u in zip(ids, urls)) + b"\0" * 16, np.uint8)
    recs["depth"] = 1
    recs["ts_sec"] = 1700000000 + np.arange(n_pages)
    recs["ts_off"] = abi.STATE_TS_LOCAL
    recs["n_msgs"] = PER_PAGE
    msgs = np.zeros(n_pages * PER_PAGE, abi.STATE_MSG)
    msgs["chat_id"] = np.repeat(-1001000000000 - np.arange(n_pages, dtype=np.int64), PER_PAGE)
    msgs["message_id"] = np.tile(np.arange(PER_PAGE, dtype=np.int64) << 20, n_pages)
    msgs["page_id"] = np.repeat(np.arange(n_pages, dtype=np.uint32), PER_PAGE)
    msgs["status"] = 2
    return np.array([(0, 0), (1, n_pages)], abi.STATE_LAYER), recs, blob, msgs, ids


def fetch_for(rnd, row, ids_of_row):
    """100 fetched keys: message ids 50..149 of the page's chat (about half known), a repeated key, and keys whose
    message id another page also fetches"""
    chat = -1001000000000 - ids_of_row
    f = [(chat, (m + 50) << 20) for m in range(PER_PAGE - 4)]
    f += [f[3], f[10], (chat, 7), (7, chat)]
    rnd.shuffle(f)
    return f


@pytest.mark.parametrize("n_pages", [1000, 100_000])
@pytest.mark.parametrize("P", [1, 2, 64, 1000])
def test_batched_calls_equal_the_one_page_calls(n_pages, P):
    rnd = random.Random(P * 7 + n_pages)
    layers, recs, blob, msgs, ids = state_arrays(n_pages)
    a, b = Engine(), Engine()
    rows = a.state_set_arrays(layers, recs, blob, msgs)
    b.state_set_arrays(layers, recs, blob, msgs)
    page_of = {int(r): i for i, r in enumerate(rows)}  # page index (chat) of each row
    pick = rnd.sample(range(n_pages), P)
    fetched = [fetch_for(rnd, r, page_of[r]) for r in pick]
    h, work, off, pj = a.state_pages_begin(pick, fetched, None, True)
    assert a.state_pages_launches > 0
    base = np.concatenate([[0], np.cumsum([len(f) for f in fetched])])
    turns = []
    for k, r in enumerate(pick):
        t, w, j = b.state_page_begin(r, fetched[k], None, True)
        assert list(work[off[k]:off[k + 1]] - base[k]) == list(w)
        assert pj[k] == j
        turns.append((t, len(w)))
    status = rnd.choices(ST, k=len(work))
    n_done = [rnd.choice([0, n, rnd.randrange(n + 1)]) for _, n in turns]
    a.state_pages_end(h, n_done, status=status)
    for k, (t, n) in enumerate(turns):
        b.state_page_end(t, n_done[k], status=status[off[k]:off[k] + n_done[k]])
    pages = [{"id": ids[page_of[r]], "url": b"u%d" % r, "status": b"fetched", "depth": rnd.choice([0, 1])} for r in pick]
    got = a.state_pages_close(pick, pages, True)
    want = [b.state_page_close(r, p, True) for r, p in zip(pick, pages)]
    assert got == want
    for r in rnd.sample(pick, min(P, 20)):
        assert np.array_equal(a.state_read_page_arrays(r), b.state_read_page_arrays(r))
    assert a.state_layer_map() == b.state_layer_map()

    def digest(e):  # state.json and both exports (about 1 GB each on 10^5 pages): compared by hash
        h = [hashlib.sha256(e.state_render(META, LAST, copy=False)).digest()]
        for mode in (abi.STATE_EXPORT_LOCAL, abi.STATE_EXPORT_DAPR):
            h.append(hashlib.sha256(b"".join(d for d, _ in e.state_export(mode))).digest())
        return h
    assert digest(a) == digest(b)
    a.close()
    b.close()


@pytest.mark.parametrize("mode", [RUN | abi.RUN_JSONL_DEVICE, RUN | abi.RUN_NO_D2H])
def test_a_bulk_result_feeds_the_end_and_discovery(mode):
    sq = PagesSequence(31, 20)
    r = sq.rnd
    pids = sq.ids()[:6]
    msgs = [page_messages(r, sq.go.page_map[p]["url"], n) for p, n in zip(pids, [30, 0, 12, 40, 5, 25])]
    for k, m in enumerate(msgs[1:], 1):  # the same message ids in different pages
        for x in m[:3]:
            x.id = msgs[0][0].id
    fetched = [[(m.chat_id, m.id) for m in ms] for ms in msgs]
    h, processed = sq.pages_begin(pids, fetched, True)
    rows = [sq.e._st_rows()[p] for p in pids]
    lead = page_messages(r, b"other", 7)   # unrelated records before the turn, and after it
    tail = page_messages(r, b"other", 9)
    turn_msgs = []
    for k, pr in enumerate(processed):
        by_id = {}
        for i, (c, mid) in enumerate(fetched[k]):
            by_id.setdefault(mid, i)
        turn_msgs += [msgs[k][by_id[m["messageId"]]] for m in pr]
    want_work = turn_msgs  # fetched[work[i]] of the turn: each owner message's discMessage
    batch = pack_telegram(lead + want_work + tail, CHANNELS)
    ro = oracle(GOOD).telegram(batch, RUN)
    sq.e.telegram_submit(0, batch, mode)
    sq.e.telegram_wait(0)
    first, n_work = len(lead), len(want_work)
    status = [int(s) for s in sq.e.read_rows(0, abi.ROWS_STATUS, first, n_work)]
    assert status == [int(s) for s in ro.status[first:first + n_work]]
    n_done = [len(pr) if k % 2 == 0 else len(pr) // 2 for k, pr in enumerate(processed)]
    i = 0
    for k, pid in enumerate(pids):
        owner, vh = sq.views.get(pid, (None, None))
        cr.page_end(sq.go, pid, owner if vh == h else None, processed[k], status[i:i + len(processed[k])], n_done[k])
        i += len(processed[k])
    sq.open.pop(h)
    before = sq.e.state_render(META, LAST)
    with pytest.raises(EngineError):  # a result too short for the turn at this offset
        sq.e.state_pages_end(h, n_done, slot=0, first=first + len(tail) + 1)
    assert sq.e.state_render(META, LAST) == before
    sq.e.state_pages_end(h, n_done, slot=0, first=first)
    sq.check()
    # discovery over the spans of work_off
    woff = np.concatenate([[0], np.cumsum([len(pr) for pr in processed])])
    spans = [(rows[k], first + int(woff[k]), int(woff[k + 1] - woff[k]), n_done[k]) for k in range(len(pids))]
    now = (1_700_000_500, 0)
    links = [[n for n, _ in ro.record_links(first + j)] for j in range(n_work)]
    want = []
    for k, pid in enumerate(pids):
        want += sq.d.standalone_page(pid, status[woff[k]:woff[k + 1]], links[woff[k]:woff[k + 1]], n_done[k], now)
    got = sq.e.state_discover(0, spans, abi.DISCOVER_NOW, now)
    sq.e.release(0)
    assert got["ids"] == [p["id"] for p in want]
    sq.pages_close(pids, True)
    sq.e.close()


def test_edge_cases():
    sq = PagesSequence(41, 8)
    p = sq.ids()
    known = [(m["chatId"], m["messageId"]) for m in sq.go.page_map[p[2]].get("messages") or []]
    fetched = [[], known, [(5, 9), (5, 9), (9, 5)], [(-1001, 1 << 20)] * 3, [(5, 9), (-1001, 3 << 20)]]
    if not known:  # a page whose keys are all known: fetch its own list twice
        h, _ = sq.pages_begin([p[2]], [[(1, 2)]], False)
        sq.pages_end(h, [1])
        sq.pages_close([p[2]], False)
        fetched[1] = [(m["chatId"], m["messageId"]) for m in sq.go.page_map[p[2]]["messages"]]
    h, processed = sq.pages_begin(p[1:6], fetched, True)
    assert processed[0] == [] and processed[1] == []
    for k in range(12):  # turns of another page compact the message rows between begin and end
        hb, pr = sq.pages_begin([p[7]], [[(7, (j + k) << 20) for j in range(300)]], False)
        sq.pages_end(hb, [len(pr[0])])
        sq.pages_close([p[7]], False)
    sq.pages_end(h, [0, 0, len(processed[2]), min(1, len(processed[3])), 0])
    for k in range(12):
        hb, pr = sq.pages_begin([p[7]], [[(7, (j + k) << 21) for j in range(300)]], False)
        sq.pages_end(hb, [len(pr[0])])
        sq.pages_close([p[7]], k % 2 == 0)
    sq.pages_close(p[1:6], True)
    sq.e.close()


def test_rejected_calls_leave_everything_unchanged():
    sq = PagesSequence(51, 6)
    e = sq.e
    p = sq.ids()
    rows = [e._st_rows()[x] for x in p]
    h, processed = sq.pages_begin(p[:2], [[(-5, 1 << 20), (-5, 2 << 20)], [(-6, 1 << 20)]], False)
    # candidates on the pending next-layer list: a rejected call must leave them as they are
    owner = sq.go.page_map[p[4]]
    ms = page_messages(sq.rnd, owner["url"], 12)
    batch = pack_telegram(ms, CHANNELS)
    ro = oracle(GOOD).telegram(batch, RUN)
    e.telegram_submit(2, batch, RUN)
    e.telegram_wait(2)
    e.state_discover(2, [(rows[4], 0, len(ms), len(ms))], 0)
    e.release(2)
    pending = dr.outlinks(owner, [int(x) for x in ro.status], [[n for n, _ in ro.record_links(i)] for i in range(ro.n)],
                          len(ms))
    assert pending
    snap = lambda: (e.state_render(META, LAST), e.state_layer_map())  # noqa: E731
    before = snap()
    page = {"id": p[0], "url": b"u", "status": b"fetched"}

    def rejected(call, code=abi.E_ARG):
        with pytest.raises(EngineError) as ei:
            call()
        assert ei.value.code == code
        assert snap() == before

    f = [[(1, 2)], [(3, 4)]]
    rejected(lambda: e.state_pages_begin([rows[2], rows[2]], f))            # a row listed twice
    rejected(lambda: e.state_pages_begin([rows[2], 99], f))                 # an unknown row
    rejected(lambda: e.state_pages_begin([rows[2]], [[(1, 2)]], [dict(page)]))  # an id that is not the row's
    rejected(lambda: e.state_pages_close([rows[2], rows[2]], [page, page]))
    rejected(lambda: e.state_pages_close([rows[0]], [dict(page, id=p[3])]))
    rejected(lambda: e.state_pages_end(h, [3, 0], status=[0, 0, 0]))        # n_done past a page's work
    rejected(lambda: e.state_pages_end(h, None, slot=-1, status=None))      # no host statuses
    rejected(lambda: e.state_pages_end(h, None, slot=0))                    # no result in the slot
    rejected(lambda: e.state_pages_end(h + 1000, None, status=[0, 0, 0]))   # an unknown handle
    rejected(lambda: e.state_page_end(h, 0, status=[]))                     # a multi-page handle, one-page end
    # a non-monotone fetched_off, or one that does not end at n; pages carrying messages; unknown flags
    import ctypes as C
    from distributed_crawler_b200 import engine as eng
    from distributed_crawler_b200.state_pack import pack_pages
    r2 = np.array(rows[2:4], np.uint32)
    fk = np.array([[1, 2], [3, 4], [5, 6]], np.int64)
    out = abi.StatePagesC()
    for fo, fl in (([0, 2, 1], 0), ([0, 1, 2], 0), ([0, 1, 3], 8)):
        fo = np.array(fo, np.uint64)
        assert eng.lib().tgi_state_pages_begin(e.h, r2.ctypes.data, 2, None, None, 0, fk.ctypes.data, 3, fo.ctypes.data,
                                               fl, C.byref(out)) == abi.E_ARG
        assert snap() == before
    recs, strs, _ = pack_pages([dict(page, messages=[{"chatId": 1, "messageId": 2, "status": b"fetched",
                                                      "pageId": p[0]}])], e.state_code, lambda pid, i: 0)
    r0 = np.array(rows[:1], np.uint32)
    fo = np.array([0, 0], np.uint64)
    for rc in (eng.lib().tgi_state_pages_begin(e.h, r0.ctypes.data, 1, recs.ctypes.data, strs.ctypes.data, len(strs), None, 0,
                                               fo.ctypes.data, 0, C.byref(out)),
               eng.lib().tgi_state_pages_close(e.h, r0.ctypes.data, 1, recs.ctypes.data, strs.ctypes.data, len(strs), 0,
                                               C.byref(out))):
        assert rc == abi.E_ARG
        assert snap() == before
    # a released or too short result
    ms = page_messages(sq.rnd, b"x", 2)
    e.telegram_submit(1, pack_telegram(ms, CHANNELS), RUN | abi.RUN_JSONL_DEVICE)
    e.telegram_wait(1)
    rejected(lambda: e.state_pages_end(h, None, slot=1, first=0))           # 2 records, the turn has 3
    e.release(1)
    rejected(lambda: e.state_pages_end(h, None, slot=1, first=0))
    yt, _, _ = make_youtube(5, seed=3)  # a YouTube result
    e.youtube_submit(1, yt, abi.RUN_JSONL | abi.RUN_LINKS)
    e.youtube_wait(1)
    rejected(lambda: e.state_pages_end(h, None, slot=1, first=0))
    e.release(1)
    # the turn still ends; then it is consumed
    sq.pages_end(h, [len(x) for x in processed])
    before = snap()
    rejected(lambda: e.state_pages_end(h, None, status=[0, 0, 0]))
    # a turn whose row was closed
    h, processed = sq.pages_begin(p[:2], [[(-5, 1 << 20)], [(-6, 1 << 20)]], False)
    sq.pages_close([p[1]], False)
    # the pending list is the one discovery left: the layer end adds exactly its pages
    now = (1_700_000_900, 0)
    want = sq.d.layer_end(pending, 0, now, False)
    got = e.state_next_layer(0, 0, now)
    assert got["ids"] == [x["id"] for x in want]
    sq.check()
    e.close()


def test_launch_counts_do_not_depend_on_the_pages():
    layers, recs, blob, msgs, ids = state_arrays(3000)  # noqa: F841
    for flags in (False, True):
        counts = []
        for P in (2, 1000):
            e = Engine()
            rows = e.state_set_arrays(layers, recs, blob, msgs)
            page_of = {int(r): i for i, r in enumerate(rows)}
            pick = list(range(P))
            fetched = [fetch_for(random.Random(r), r, page_of[r]) for r in pick]
            h, work, off, _ = e.state_pages_begin(pick, fetched, None, flags)
            begin = e.state_pages_launches
            e.state_pages_end(h, None, status=[abi.ST_EMITTED] * len(work))
            end = e.state_pages_launches
            pages = [{"id": ids[page_of[r]], "url": b"u", "status": b"fetched", "depth": 0} for r in pick]
            e.state_pages_close(pick, pages, flags)
            close = e.state_pages_launches
            bare = list(range(P, 2 * P))  # rows no turn ran on: no owner view, their lists rendered as they are
            e.state_pages_close(bare, [{"id": ids[page_of[r]], "url": b"v", "status": b"fetched", "depth": 1} for r in bare],
                                flags)
            counts.append((begin, end, close, e.state_pages_launches))
            e.close()
        assert counts[0] == counts[1], counts
