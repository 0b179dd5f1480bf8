"""GPU tests: snowball discovery (tgi_state_discover / tgi_state_next_layer) against tests/discover_rules.py over the
restatements of BaseStateManager and DaprStateManager — state.json byte for byte, the layer map, the added rows, ids and
page JSONs and the urlCache after every call of seeded sequences on real Telegram batches, under every flag combination
and every result mode, and rejected calls that leave everything as it was."""
import functools
import random

import pytest

import discover_rules as dr
from dapr_state_rules import marshal_layer_map
from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import Engine, EngineError, names_to_keys32
from distributed_crawler_b200.corpus import Corpus
from distributed_crawler_b200.pack import pack_telegram
from helpers import msg
from oracle.pyoracle import Oracle
from state_rules import GoState, marshal_page
from test_gpu_state import LAST, META
from tg_link_corpus import CHANNELS, make_link_edges

pytestmark = pytest.mark.gpu
MIN_DATE = 1_600_000_000
RUN = abi.RUN_JSONL | abi.RUN_LINKS
RUN_MODES = [RUN, RUN | abi.RUN_JSONL_DEVICE, RUN | abi.RUN_NO_D2H,
             RUN | abi.RUN_FRONTIER | abi.RUN_SKIP_SELF | abi.RUN_FILTER | abi.RUN_SKIP_INVALID]
FLAGS = [f | j for f in (0, abi.DISCOVER_DAPR) for j in (0, abi.DISCOVER_PAGE_JSON)]
NAMES = [b"chan%03d" % k for k in range(40)]
GOOD = (1_750_000_000, 0, 1_750_000_000, 123_456_789)  # the configuration's clock (abi.make_config)
BAD = (400_000_000_000, 0, 400_000_000_000, 0)          # a year json.Marshal refuses: every line is TGI_ST_NOLINE


def oracle(clock):
    return Oracle(min_post_date=MIN_DATE, created_at_sec=clock[0], created_at_nsec=clock[1], capture_sec=clock[2],
                  capture_nsec=clock[3])


@functools.lru_cache(maxsize=None)
def edge_names():
    """the link corpus's messages (names of 31 / 32 / 33 bytes, mixed case, entity links) and its 32-byte outlinks"""
    _, msgs, _ = make_link_edges(7)
    ro = oracle(GOOD).telegram(pack_telegram(msgs, CHANNELS), RUN)
    return msgs, sorted({n for i in range(ro.n) for n, _ in ro.record_links(i) if len(n) == 32})


def page_messages(rnd, owner_url, n):
    """a page of messages with t.me links and mentions: repeats within and across messages, self links, links to the
    state's own pages, panicking records and records before min_post_date"""
    out = []
    for k in range(n):
        names = [rnd.choice(NAMES + [owner_url.lower()]) for _ in range(rnd.choice([0, 1, 3, 6]))]
        text = " ".join((b"t.me/" if rnd.random() < 0.6 else b"@").decode() + nm.decode() for nm in names)
        out.append(msg("messageText", "post %d %s" % (k, text), id=(k + 1) << 20, chat_id=-100777, channel=0,
                       date=MIN_DATE + 5 if rnd.random() < 0.85 else MIN_DATE - 5, panics=rnd.random() < 0.08))
    return out


class DiscoverSequence:
    def __init__(self, seed, n_owners=6, **cfg):
        self.rnd = random.Random(seed)
        self.e = Engine(min_post_date=MIN_DATE, **cfg)
        self.o = Oracle(min_post_date=MIN_DATE)
        self.go = GoState()
        self.d = dr.Discovery(self.go, seed=0x5EED0000 + seed)
        self.e.state_id_seed(self.d.seed)
        # owner URLs: channel names of the link pool (so outlinks meet them), one of them in another case, two 32-byte
        # outlinks of the link corpus (one as it is, one upper-cased), and a deadend page (AddLayer's MaxPages budget)
        long32 = edge_names()[1]
        urls = [NAMES[0], NAMES[1].upper(), long32[0], long32[1].upper(), NAMES[4], NAMES[5]]
        owners = [{"id": b"owner-%d" % k, "url": urls[k % len(urls)], "depth": 0,
                   "status": b"deadend" if k == 4 else b"fetched", "timestamp": (1_700_000_000, 0, 0)} for k in range(n_owners)]
        self.state_set([(0, owners)])
        self.corpus = Corpus(600, profile=2, nthreads=2, first=600 * seed)
        self.seen = {"noline": 0, "long": 0, "long_cached": 0}
        # urlCache from earlier crawls: one URL longer than a key, and a 32-byte outlink of the link corpus
        cache = [NAMES[30], NAMES[31], b"x" * 40, long32[2]]
        self.e.set_add(abi.SET_URLS, names_to_keys32(dr.url_cache_keys(cache)))
        self.d.url_cache.update({u: b"old" for u in cache})
        self.pending = []
        self.now = (1_700_000_100, 0)

    def state_set(self, layers):
        self.go.set_state(layers)
        self.e.state_set(layers)
        self.pending = []  # tgi_state_set drops the pending list

    def check(self):
        assert self.e.state_render(META, LAST) == self.go.marshal(META, LAST)
        assert self.e.state_layer_map() == marshal_layer_map(self.go.layer_map)
        assert self.e.set_size(abi.SET_URLS) == len(dr.url_cache_keys(self.d.url_cache))

    def batch(self, owners, run_flags, slot=0):
        """one result holding a page of every owner: its spans (row, first, n_records, n_done) and per-record links.
        The pages come from the seeded link pool, from the link corpus or from the seeded corpus; a third of the
        results run under a clock json.Marshal refuses, so their records are TGI_ST_NOLINE with their links."""
        r = self.rnd
        sizes = [r.choice([0, 1, 7, 20, 60]) for _ in owners]
        src = r.random()
        if src < 0.25:  # consecutive records of the seeded corpus
            a = r.randrange(self.corpus.batch.n - sum(sizes) + 1) if sum(sizes) < self.corpus.batch.n else 0
            b = self.corpus.batch.slice(a, a + sum(sizes))
        else:
            msgs = []
            for pid, n in zip(owners, sizes):
                if src < 0.6:
                    msgs += page_messages(r, self.go.page_map[pid]["url"], n)
                else:
                    pool = edge_names()[0]
                    a = r.randrange(len(pool) - n)
                    msgs += pool[a:a + n]
            b = pack_telegram(msgs, CHANNELS)
        spans, first = [], 0
        for pid, n in zip(owners, sizes):
            n_done = n if r.random() < 0.7 else r.randrange(n + 1)
            spans.append((self.e._st_rows()[pid], first, n, n_done))
            first += n
        clock = BAD if r.random() < 0.33 else GOOD
        ro = oracle(clock).telegram(b, RUN)
        self.e.set_clock(*clock)
        self.e.telegram_submit(slot, b, run_flags)
        self.e.telegram_wait(slot)
        self.e.set_clock(*GOOD)
        return spans, [int(s) for s in ro.status], [[n for n, _ in ro.record_links(i)] for i in range(ro.n)]

    def note(self, status, links, cands, dapr):
        """what the inputs held: processed NOLINE records with links, 32-byte candidates, 32-byte urlCache hits"""
        self.seen["noline"] += sum(1 for s, ls in zip(status, links) if s == abi.ST_NOLINE and ls)
        self.seen["long"] += sum(1 for c in cands if len(c["url"]) == 32)
        self.seen["long_cached"] += sum(1 for c in cands if len(c["url"]) == 32 and c["url"] in self.d.url_cache) if dapr else 0

    def expect_added(self, got, want, flags):
        assert got["ids"] == [p["id"] for p in want]
        if want:  # the local export walks pageMap in row order: line r is the page of row r
            lines = self.e.state_export(abi.STATE_EXPORT_LOCAL)[0][0].split(b"\n")
            assert [lines[r] for r in got["rows"]] == [marshal_page(p) for p in want]
        if flags & abi.DISCOVER_PAGE_JSON:
            assert got["page_json"] == [marshal_page(p) for p in want]
        else:
            assert got["page_json"] is None

    def discover(self, owners, flags, now_mode, run_flags, slot=0, max_pages=0):
        spans, status, links = self.batch(owners, run_flags, slot)
        dapr = bool(flags & abi.DISCOVER_DAPR)
        want, n_cand = [], 0
        for row, first, n_rec, n_done in spans:
            pid = next(p for p, x in self.e._st_rows().items() if x == row)
            cands = dr.outlinks(self.go.page_map[pid], status[first:first + n_rec], links[first:first + n_rec], n_done)
            self.note(status[first:first + n_done], links[first:first + n_done], cands, dapr)
            n_cand += len(cands)
            if now_mode:
                want += self.d.standalone_page(pid, status[first:first + n_rec], links[first:first + n_rec], n_done,
                                               self.now, dapr, max_pages)
            else:
                self.pending += cands
        got = self.e.state_discover(slot, spans, flags | (abi.DISCOVER_NOW if now_mode else 0), self.now, max_pages)
        self.e.release(slot)
        assert got["n_candidates"] == n_cand
        self.expect_added(got, want, flags)
        self.check()

    def next_layer(self, flags, depth, max_pages=0):
        want = self.d.layer_end(self.pending, depth, self.now, bool(flags & abi.DISCOVER_DAPR), max_pages)
        got = self.e.state_next_layer(depth, flags, self.now, max_pages)
        assert got["n_candidates"] == len(self.pending)
        self.pending = []
        self.expect_added(got, want, flags)
        self.check()


@pytest.mark.parametrize("seed", range(4))
def test_random_discovery_sequences_match_the_restatement(seed):
    sq = DiscoverSequence(seed)
    r = sq.rnd
    for step in range(40):
        sq.now = (sq.now[0] + 1, r.choice([0, 1, 999_999_999]))
        ids = list(sq.go.page_map)
        k = r.random()
        if k < 0.45:
            owners = r.sample(ids, min(len(ids), r.choice([1, 1, 3])))
            sq.discover(owners, r.choice(FLAGS), True, r.choice(RUN_MODES), slot=step % 3,
                        max_pages=r.choice([0, 0, len(ids), len(ids) + 3]))
        elif k < 0.75:
            owners = r.sample(ids, min(len(ids), r.choice([1, 4])))
            sq.discover(owners, r.choice(FLAGS), False, r.choice(RUN_MODES), slot=step % 3)
        elif k < 0.9:
            sq.next_layer(r.choice(FLAGS), r.randrange(3), max_pages=r.choice([0, 0, len(ids), len(ids) + 2]))
        elif k < 0.95:  # another state call in between: a page overwritten by UpdatePage
            p = dict(sq.go.page_map[r.choice(ids)])
            p["url"] = r.choice(NAMES)
            p.pop("messages", None)
            sq.go.update_page(p)
            sq.e.state_update_page(p)
            sq.check()
        else:  # SetState between discover and the layer end drops the pending list
            pages = [dict(sq.go.page_map[i]) for i in ids[:5]]
            for p in pages:
                p.pop("messages", None)
            sq.state_set([(0, pages)])
            sq.check()
    sq.next_layer(abi.DISCOVER_DAPR | abi.DISCOVER_PAGE_JSON, 7)
    assert sq.seen["noline"] > 0 and sq.seen["long"] > 0, sq.seen
    sq.e.close()


def test_noline_records_long_names_deadends_and_set_state():
    """the link corpus in one bulk result, six spans: NOLINE records with links, a 32-byte owner URL its own page links
    to (skipped), a 32-byte urlCache entry an outlink hits, MaxPages with a deadend page, and a tgi_state_set between
    discover and the layer end"""
    msgs, _ = edge_names()
    b = pack_telegram(msgs, CHANNELS)
    ro = oracle(BAD).telegram(b, RUN)
    status = [int(s) for s in ro.status]
    links = [[n for n, _ in ro.record_links(i)] for i in range(ro.n)]
    n, k6 = ro.n, ro.n // 6
    spans_rec = [(k * k6, k6 if k < 5 else n - 5 * k6) for k in range(6)]
    own = [sorted({nm for i in range(a, a + m) for nm in links[i] if len(nm) == 32 and status[i] != abi.ST_FAILED})
           for a, m in spans_rec]
    sq = DiscoverSequence(31, n_owners=6)
    e = sq.e
    urls = [own[0][0], own[1][0].upper(), b"chan004", b"chan005", b"chan006", b"chan007"]
    owners = [{"id": b"owner-%d" % k, "url": urls[k], "depth": 0, "status": b"deadend" if k == 4 else b"fetched",
               "timestamp": (1_700_000_000, 0, 0)} for k in range(6)]
    sq.state_set([(0, owners)])
    hit = next(nm for nm in own[3] if nm not in urls)
    e.set_add(abi.SET_URLS, names_to_keys32([hit]))
    sq.d.url_cache[hit] = b"old"
    rows = e._st_rows()
    spans = [(rows[b"owner-%d" % k], a, m, m) for k, (a, m) in enumerate(spans_rec)]
    assert sum(1 for s, ls in zip(status, links) if s == abi.ST_NOLINE and ls) > 100
    assert any(own[0][0] in links[i] for i in range(spans_rec[0][1]))  # the owner's own 32-byte URL among its outlinks

    def run(slot, clock, flags):
        e.set_clock(*clock)
        e.telegram_submit(slot, b, flags)
        e.telegram_wait(slot)
        e.set_clock(*GOOD)

    # Dapr rules, per page: the 32-byte urlCache hit is skipped, NOLINE records give their outlinks
    run(0, BAD, RUN | abi.RUN_NO_D2H)
    want = []
    for k, (a, m) in enumerate(spans_rec):
        want += sq.d.standalone_page(b"owner-%d" % k, status[a:a + m], links[a:a + m], m, sq.now, True)
    assert hit not in [p["url"] for p in want] and any(len(p["url"]) == 32 for p in want)
    got = e.state_discover(0, spans, abi.DISCOVER_NOW | abi.DISCOVER_DAPR | abi.DISCOVER_PAGE_JSON, sq.now)
    e.release(0)
    sq.expect_added(got, want, abi.DISCOVER_PAGE_JSON)
    sq.check()
    # Base rules, per page, with the state full: only as many pages as there are deadend pages go in
    run(1, GOOD, RUN | abi.RUN_JSONL_DEVICE)
    fresh = [(rows[b"owner-%d" % k], a, m, m) for k, (a, m) in enumerate(spans_rec)]
    full = len(sq.go.page_map)
    go_status = [int(s) for s in oracle(GOOD).telegram(b, RUN).status]
    want = []
    for k, (a, m) in enumerate(spans_rec):
        want += sq.d.standalone_page(b"owner-%d" % k, go_status[a:a + m], links[a:a + m], m, sq.now, False, full)
    got = e.state_discover(1, fresh, abi.DISCOVER_NOW, sq.now, full)
    e.release(1)
    assert want and len(sq.go.page_map) > full  # past MaxPages: the deadend page's replacement budget let pages in
    sq.expect_added(got, want, 0)
    sq.check()
    # pending, then SetState: the list is dropped and the layer end changes nothing
    run(2, BAD, RUN)
    assert e.state_discover(2, spans, 0, sq.now)["n_candidates"] > 0
    e.release(2)
    pages = [dict(p) for p in owners]
    sq.state_set([(0, pages)])
    got = e.state_next_layer(0, abi.DISCOVER_DAPR | abi.DISCOVER_PAGE_JSON, sq.now)
    assert got["n_candidates"] == 0 and got["ids"] == [] and got["page_json"] == []
    sq.check()
    e.close()


def test_empty_candidates_make_no_layer_and_a_known_only_list_does():
    sq = DiscoverSequence(11, n_owners=2)
    e, row = sq.e, sq.e._st_rows()[b"owner-0"]
    # a page whose only outlinks are self links, and one whose records all failed: no candidate, no layer
    for ms in ([msg("messageText", "t.me/chan000 @chan000", id=1 << 20, chat_id=-1, date=MIN_DATE + 1)],
               [msg("messageText", "t.me/chan005", id=1 << 20, chat_id=-1, date=MIN_DATE + 1, panics=True)]):
        e.telegram_submit(0, pack_telegram(ms), RUN)
        e.telegram_wait(0)
        got = e.state_discover(0, [(row, 0, 1, 1)], abi.DISCOVER_NOW, sq.now)
        e.release(0)
        assert got["n_candidates"] == 0 and got["ids"] == []
        sq.check()
    assert sorted(sq.go.layer_map) == [0]
    # an outlink naming a page already in the state: Base creates the layer of depth 1 with nothing in it, Dapr does not
    ms = [msg("messageText", "t.me/chan001", id=1 << 20, chat_id=-1, date=MIN_DATE + 1)]
    for flags in (abi.DISCOVER_NOW, abi.DISCOVER_NOW | abi.DISCOVER_DAPR):
        sq.go.update_page(dict(sq.go.page_map[b"owner-1"], url=b"chan001"))
        e.state_update_page(dict(sq.go.page_map[b"owner-1"]))
        sq.d.url_cache[b"chan001"] = b"owner-1"
        e.set_add(abi.SET_URLS, names_to_keys32([b"chan001"]))
        e.telegram_submit(0, pack_telegram(ms), RUN)
        e.telegram_wait(0)
        want = sq.d.standalone_page(b"owner-0", [0], [[b"chan001"]], 1, sq.now, bool(flags & abi.DISCOVER_DAPR))
        got = e.state_discover(0, [(row, 0, 1, 1)], flags, sq.now)
        e.release(0)
        assert got["n_candidates"] == 1 and got["ids"] == [] == want
        sq.check()
    assert sq.e.state_layer_map() == b'{"0":["owner-0","owner-1"],"1":[]}'
    e.close()


def test_large_pending_list_and_growing_url_cache():
    rnd = random.Random(5)
    n_pages, per = 10_000, 30
    e = Engine(min_post_date=MIN_DATE, frontier_capacity=1024, set_growth=1 << 22)
    go = GoState()
    d = dr.Discovery(go, seed=77)
    e.state_id_seed(77)
    owners = [{"id": b"o%d" % k, "url": b"owner%05d" % k, "depth": 3, "status": b"fetched"} for k in range(n_pages)]
    go.set_state([(3, owners)])
    e.state_set([(3, owners)])
    rows = e._st_rows()
    pool = [b"name%06d" % k for k in range(60_000)]
    ms = [msg("messageText", " ".join("t.me/" + rnd.choice(pool).decode() for _ in range(per)), id=(k + 1) << 20,
              chat_id=-5, date=MIN_DATE + 1) for k in range(n_pages)]
    b = pack_telegram(ms)
    ro = Oracle(min_post_date=MIN_DATE).telegram(b, RUN)
    pending = []
    for half in (0, 1):  # two bulk results, several spans each
        lo, hi = half * n_pages // 2, (half + 1) * n_pages // 2
        part = pack_telegram(ms[lo:hi])
        e.telegram_submit(half, part, RUN | abi.RUN_NO_D2H)
        e.telegram_wait(half)
        spans = [(rows[b"o%d" % k], k - lo, 1, 1) for k in range(lo, hi)]
        got = e.state_discover(half, spans, 0, (0, 0))
        e.release(half)
        before = len(pending)
        for k in range(lo, hi):
            pending += dr.outlinks(go.page_map[b"o%d" % k], [int(ro.status[k])], [[n for n, _ in ro.record_links(k)]], 1)
        assert got["n_candidates"] == len(pending) - before
    assert len(pending) >= n_pages * per * 0.9
    now = (1_700_000_000, 250)
    want = d.layer_end(pending, 3, now, dapr=True)
    got = e.state_next_layer(3, abi.DISCOVER_DAPR | abi.DISCOVER_PAGE_JSON, now)
    assert got["n_candidates"] == len(pending)
    assert got["ids"] == [p["id"] for p in want]
    assert got["page_json"] == [marshal_page(p) for p in want]
    assert e.state_render(META, LAST) == go.marshal(META, LAST)
    assert e.state_layer_map() == marshal_layer_map(go.layer_map)
    info = e.set_info(abi.SET_URLS)
    assert info["count"] == len(d.url_cache) and info["grows"] > 0
    e.close()


def test_rejected_calls_leave_everything_unchanged():
    sq = DiscoverSequence(21, n_owners=3)
    e = sq.e
    row = e._st_rows()[b"owner-0"]
    ms = [msg("messageText", "t.me/chan007 t.me/chan008", id=(k + 1) << 20, chat_id=-1, date=MIN_DATE + 1) for k in range(4)]
    # one candidate list pending, so a rejected call could disturb it
    e.telegram_submit(0, pack_telegram(ms), RUN)
    e.telegram_wait(0)
    e.state_discover(0, [(row, 0, 4, 4)], 0, sq.now)
    before = (e.state_render(META, LAST), e.state_layer_map(), e.set_size(abi.SET_URLS))

    def rejected(call, code):
        with pytest.raises(EngineError) as ei:
            call()
        assert ei.value.code == code
        assert (e.state_render(META, LAST), e.state_layer_map(), e.set_size(abi.SET_URLS)) == before

    now = abi.DISCOVER_NOW
    rejected(lambda: e.state_discover(0, [(99, 0, 4, 4)], now, sq.now), abi.E_ARG)            # no such row
    rejected(lambda: e.state_discover(0, [(row, 2, 3, 3)], now, sq.now), abi.E_ARG)           # outside the result
    rejected(lambda: e.state_discover(0, [(row, 0, 2, 3)], now, sq.now), abi.E_ARG)           # n_done > n_records
    rejected(lambda: e.state_discover(0, [(row, 0, 4, 4)], now, (0, 10**9)), abi.E_ARG)       # now_nsec
    rejected(lambda: e.state_discover(0, [(row, 0, 4, 4)], 64, sq.now), abi.E_ARG)            # unknown flag
    rejected(lambda: e.state_next_layer(0, abi.DISCOVER_PAGE_JSON, (-10**13, 0)), abi.E_ARG)  # a year json.Marshal refuses
    e.release(0)
    rejected(lambda: e.state_discover(0, [(row, 0, 4, 4)], now, sq.now), abi.E_STATE)         # a released result
    rejected(lambda: e.state_discover(2, [(row, 0, 4, 4)], now, sq.now), abi.E_STATE)         # no result
    e.telegram_submit(1, pack_telegram(ms), abi.RUN_JSONL)
    e.telegram_wait(1)
    rejected(lambda: e.state_discover(1, [(row, 0, 4, 4)], now, sq.now), abi.E_STATE)         # no TGI_RUN_LINKS
    e.release(1)
    from yt_corpus import make_youtube
    yt, _, _ = make_youtube(4, seed=2)
    e.youtube_submit(1, yt, RUN)
    e.youtube_wait(1)
    rejected(lambda: e.state_discover(1, [(row, 0, 4, 4)], now, sq.now), abi.E_STATE)         # a YouTube result
    e.release(1)
    # no seed: a call that would add a page is refused, one that adds nothing is not
    e2 = Engine(min_post_date=MIN_DATE)
    e2.state_set([(0, [{"id": b"p", "url": b"chan007"}])])
    e2.telegram_submit(0, pack_telegram(ms[:1]), RUN)
    e2.telegram_wait(0)
    e2.state_discover(0, [(0, 0, 1, 1)], 0, sq.now)  # pending only
    r0 = e2.state_render(META, LAST)
    with pytest.raises(EngineError) as ei:
        e2.state_discover(0, [(0, 0, 1, 1)], abi.DISCOVER_NOW, sq.now)
    assert ei.value.code == abi.E_STATE and e2.state_render(META, LAST) == r0
    with pytest.raises(EngineError) as ei:
        e2.state_next_layer(0, 0, sq.now)
    assert ei.value.code == abi.E_STATE and e2.state_render(META, LAST) == r0
    e2.state_id_seed(1)
    assert len(e2.state_next_layer(0, 0, sq.now)["ids"]) == 1  # the pending list survived the refusal
    e2.release(0)
    e2.close()
    # the pending list of the first engine survived every rejection
    want = sq.d.layer_end(dr.outlinks(sq.go.page_map[b"owner-0"], [0] * 4, [[b"chan007", b"chan008"]] * 4, 4), 0, sq.now)
    sq.expect_added(e.state_next_layer(0, abi.DISCOVER_DAPR | abi.DISCOVER_PAGE_JSON, sq.now), want, abi.DISCOVER_PAGE_JSON)
    sq.check()
    e.close()
