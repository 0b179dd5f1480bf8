"""GPU tests: the resident crawl state (tgi_state_*) against the restatement of BaseStateManager and json.Marshal(State) in
tests/state_rules.py — state.json byte for byte and GetPage's messages after every step of seeded random operation
sequences, two large renders, and rejected calls that leave the state as it was."""
import random

import numpy as np
import pytest

from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import Engine, EngineError
from state_rules import GoState, marshal_time
from test_zones import ZONES

NY = ZONES["America/New_York"]
FALL_2023 = 1699164000  # America/New_York leaves DST: 2023-11-05T06:00:00Z
META, LAST = b'{"crawlId":"c","executionId":"e","startTime":"2024-01-01T00:00:00Z","status":"running"}', b'"2024-01-02T03:04:05.5Z"'
ODD = [b"", b"<b>&amp;", b"\xe2\x80\xa8x\xe2\x80\xa9", b"bad\xff\xfe", b'q"\\\n\t', "канал".encode()]
STATUSES = [b"unfetched", b"fetched", b"failed", b"deadend", b"error"]
MSG_STATUSES = [b"unfetched", b"fetched", b"failed", b"deleted", b"resample", b"custom<&>"]


class Sequence:
    def __init__(self, seed, max_pages=0):
        self.rnd = random.Random(seed)
        self.go = GoState(max_pages)
        self.e = Engine()
        self.max_pages = max_pages
        self.zone = None
        self.n = 0

    def s(self, stem):
        r = self.rnd
        return stem + (r.choice(ODD) if r.random() < 0.3 else b"")

    def ts(self):
        r = self.rnd
        k = r.random()
        if k < 0.4:
            return (FALL_2023 + r.randrange(-3, 3), r.choice([0, 1, 500000000, 123456789]), None)  # time.Local
        if k < 0.8:
            return (1700000000 + r.randrange(-10**6, 10**6), r.choice([0, 7]), r.choice([0, 3600, -18000, 19800, -14400]))
        return (-62135596800, 0, 0)  # the zero time

    def page(self, depth, with_msgs, ids):
        r = self.rnd
        self.n += 1
        pid = r.choice(ids) if ids and r.random() < 0.1 else self.s(b"id%d" % self.n)
        p = {"id": pid, "url": self.s(b"https://t.me/u%d" % r.randrange(60)), "depth": depth,
             "status": r.choice(STATUSES), "timestamp": self.ts()}
        for k in ("error", "platform", "parentId", "LastConnectionID", "sequenceId", "crawlId"):
            if r.random() < 0.3:
                p[k] = self.s(k.encode())
        if with_msgs:
            p["messages"] = [{"chatId": r.choice([-1001, -1002, 7]), "messageId": r.randrange(-2, 12) << 20,
                              "status": r.choice(MSG_STATUSES), "pageId": pid, "platform": r.choice([b"", b"", b"telegram"])}
                             for _ in range(r.choice([0, 1, 3, 12, 40]))]
        return p

    def ids(self):
        return list(self.go.page_map)

    def check(self):
        got = self.e.state_render(META, LAST)
        assert got == self.go.marshal(META, LAST, self.zone), self.diff(got)
        for pid in self.rnd.sample(self.ids(), min(3, len(self.ids()))):
            want = [dict({"platform": b""}, **m) for m in self.go.page_map[pid].get("messages") or []]
            assert self.e.state_read_page(self.e._st_rows()[pid]) == want

    def diff(self, got):
        want = self.go.marshal(META, LAST, self.zone)
        k = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
        return f"len {len(got)} vs {len(want)}; first difference at {k}: {got[k-80:k+80]!r} vs {want[k-80:k+80]!r}"

    def step(self):
        r = self.rnd
        op = r.random()
        if op < 0.08:
            layers = [(r.randrange(4), [self.page(r.randrange(3), True, []) for _ in range(r.randrange(0, 6))])
                      for _ in range(r.randrange(0, 4))]
            ids = [p["id"] for _, ps in layers for p in ps]
            for _, ps in layers:  # messages may name another page of the state
                for p in ps:
                    for m in p["messages"]:
                        if r.random() < 0.1:
                            m["pageId"] = r.choice(ids)
            self.go.set_state(layers)
            self.e.state_set(layers)
        elif op < 0.3:
            ps = [self.page(r.randrange(4), False, self.ids()) for _ in range(r.randrange(0, 8))]
            if ps:
                ps = [dict(p, depth=ps[0]["depth"]) if r.random() < 0.5 else p for p in ps]
            want = self.go.add_layer(ps)
            rows = self.e.state_add_layer(ps, self.max_pages)
            assert [x != abi.STATE_NO_PAGE for x in rows] == want
        elif op < 0.55:
            p = self.page(r.randrange(5), True, self.ids())
            if self.ids() and r.random() < 0.6:  # the usual case: replace a known page's message list
                p["id"] = r.choice(self.ids())
                for m in p["messages"]:
                    m["pageId"] = p["id"]
            self.go.update_page(p)
            self.e.state_update_page(p)
        elif op < 0.9:
            ups = []
            for _ in range(r.randrange(1, 60)):
                pid = r.choice(self.ids()) if self.ids() and r.random() < 0.9 else b"no such page"
                msgs = (self.go.page_map.get(pid) or {}).get("messages") or []
                if msgs and r.random() < 0.6:
                    m = r.choice(msgs)
                    key = (m["chatId"], m["messageId"])
                else:
                    key = (r.choice([-1001, 5]), r.randrange(20, 24) << 20)  # unknown keys, updated several times
                ups.append((pid, key, r.choice(MSG_STATUSES)))
            skipped = sum(not self.go.update_message(pid, c, m, st) for pid, (c, m), st in ups)
            rows = self.e._st_rows()
            assert self.e.state_update_messages([(rows[pid] if pid in self.go.page_map else abi.STATE_NO_PAGE, c, m, st)
                                                 for pid, (c, m), st in ups]) == skipped
        else:
            self.zone = NY if self.zone is None else None
            self.e.set_zone(*(self.zone or ([], [])))
        self.check()


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(6))
def test_random_sequences_match_the_restatement(seed):
    sq = Sequence(seed, max_pages=[0, 0, 0, 25, 40, 12][seed])
    for _ in range(120):
        sq.step()
    sq.e.close()


@pytest.mark.gpu
def test_tombstones_compaction_and_the_empty_state():
    sq = Sequence(99)
    assert sq.e.state_render(META, LAST) == b'{"layers":[],"metadata":%s,"lastUpdated":%s}' % (META, LAST)
    sq.go.set_state([(0, [{"id": b"a", "url": b"u"}])])
    sq.e.state_set([(0, [{"id": b"a", "url": b"u"}])])
    for k in range(30):  # every UpdatePage leaves the old list as tombstones; the table is rebuilt when they win
        p = {"id": b"a", "url": b"u", "depth": 0, "messages": [{"chatId": 1, "messageId": j % (5 + k), "status": b"fetched",
                                                               "pageId": b"a"} for j in range(200 + k)]}
        sq.go.update_page(p)
        sq.e.state_update_page(p)
        rows = sq.e._st_rows()
        ups = [(rows[b"a"], 1, j, b"failed") for j in range(0, 300, 7)] + [(rows[b"a"], 2, 5, b"deleted")] * 3
        for _, c, m, st in ups:
            sq.go.update_message(b"a", c, m, st)
        sq.e.state_update_messages(ups)
        sq.check()
    sq.e.close()


@pytest.mark.gpu
def test_rejected_calls_leave_the_state_unchanged():
    sq = Sequence(7)
    for _ in range(15):
        sq.step()
    e = sq.e
    before = e.state_render(META, LAST)
    nrows = len(e._st_ids)
    bad = [lambda: e.state_update_arrays(np.array([(1, 2, nrows + 3, 1, 0)], abi.STATE_UPDATE)),
           lambda: e.state_update_arrays(np.array([(1, 2, 0, 999, 0)], abi.STATE_UPDATE)),
           lambda: e.state_set_arrays(np.array([(0, 1)], abi.STATE_LAYER), np.zeros(1, abi.STATE_PAGE), np.zeros(16, np.uint8),
                                      np.array([(1, 2, 5, 1, 0)], abi.STATE_MSG)),  # a message of no page
           lambda: e.state_set_arrays(np.array([(0, 2)], abi.STATE_LAYER), np.zeros(1, abi.STATE_PAGE), np.zeros(16, np.uint8),
                                      np.zeros(0, abi.STATE_MSG)),  # the layers hold more pages than given
           lambda: e.state_add_layer([{"id": b"x", "url": b"new", "timestamp": (0, 10**9, 0)}]),  # nsec out of range
           lambda: e.state_add_layer([{"id": b"x", "url": b"new", "timestamp": (0, 0, 86400)}]),  # offset of a day
           lambda: e.state_add_layer([{"id": b"x", "url": b"new", "messages": [{"chatId": 1, "messageId": 1, "pageId": b"x"}]}]),
           lambda: e.state_read_page_arrays(nrows + 1)]
    for call in bad:
        with pytest.raises(EngineError) as ei:
            call()
        assert ei.value.code == abi.E_ARG
        assert e.state_render(META, LAST) == before
    # a timestamp json.Marshal cannot render: the render fails, the state is kept and renders again once fixed
    p = {"id": b"y10k", "url": b"y10k", "depth": 0, "timestamp": (253402300800, 0, 0)}
    e.state_update_page(p)
    with pytest.raises(EngineError) as ei:
        e.state_render(META, LAST)
    assert ei.value.code == abi.E_ARG
    p["timestamp"] = (253402300799, 0, 0)
    e.state_update_page(p)
    sq.go.update_page(p)
    sq.check()
    e.close()


def big_state(n_pages, per_page):
    """n_pages pages of depth 1 with per_page messages each, as packed arrays, and the expected state.json"""
    codes = [b"unfetched", b"fetched", b"failed", b"deleted", b"resample"]
    ids = [b"page-%07d" % p for p in range(n_pages)]
    urls = [b"https://t.me/c%07d" % p for p in range(n_pages)]
    recs = np.zeros(n_pages, abi.STATE_PAGE)
    lens = np.array([len(i) for i in ids], np.uint32)
    recs["str_len"][:, abi.STATE_STRINGS.index("id")] = lens
    recs["str_len"][:, abi.STATE_STRINGS.index("url")] = [len(u) for u in urls]
    recs["str_len"][:, abi.STATE_STRINGS.index("status")] = 7
    blob = b"".join(i + u + b"fetched" for i, u in zip(ids, urls))
    recs["str_off"] = np.concatenate([[0], np.cumsum(recs["str_len"].sum(1).astype(np.uint64))[:-1]])
    recs["depth"] = 1
    recs["ts_sec"] = 1700000000 + np.arange(n_pages)
    recs["ts_off"] = np.where(np.arange(n_pages) % 2 == 0, abi.STATE_TS_LOCAL, 3600)
    recs["n_msgs"] = per_page
    k = np.arange(per_page)
    msgs = np.zeros(n_pages * per_page, abi.STATE_MSG)
    msgs["chat_id"] = np.repeat(-1000000000000 - np.arange(n_pages, dtype=np.int64), per_page)
    msgs["message_id"] = np.tile(k.astype(np.int64) << 20, n_pages)
    msgs["page_id"] = np.repeat(np.arange(n_pages, dtype=np.uint32), per_page)
    msgs["status"] = np.tile(k % 5 + 1, n_pages)
    tmpl = b",".join(b'{"chatId":@C,"messageId":%d,"status":"%s","pageId":"@P"}' % (int(j) << 20, codes[j % 5]) for j in k)
    pages = []
    for p in range(n_pages):
        ts = marshal_time((1700000000 + p, 0, None if p % 2 == 0 else 3600), None, 0)
        pages.append(b'{"id":"%s","url":"%s","depth":1,"status":"fetched","timestamp":%s,"messages":[%s]}' % (
            ids[p], urls[p], ts, tmpl.replace(b"@C", b"%d" % (-1000000000000 - p)).replace(b"@P", ids[p])))
    want = b'{"layers":[{"depth":1,"pages":[' + b",".join(pages) + b']}],"metadata":%s,"lastUpdated":%s}' % (META, LAST)
    return recs, np.frombuffer(blob + b"\0" * 16, np.uint8), msgs, want


@pytest.mark.gpu
@pytest.mark.parametrize("n_pages,per_page", [(100_000, 100), (1, 1_000_000)])
def test_large_renders(n_pages, per_page):
    recs, strs, msgs, want = big_state(n_pages, per_page)
    e = Engine()
    rows = e.state_set_arrays(np.array([(1, n_pages)], abi.STATE_LAYER), recs, strs, msgs)
    assert list(rows[:3]) == [0, 1, 2][:n_pages]
    got = e.state_render(META, LAST)
    assert len(got) == len(want) and got == want
    r = int(rows[-1])
    m = e.state_read_page_arrays(r)
    assert np.array_equal(m, msgs[r * per_page:(r + 1) * per_page])
    e.close()
