"""GPU tests: the tandem hand-off (tgi_state_pending_edges) against tests/tandem_rules.py — every page's edges, batch and
batch id, from bulk results of 1 to 1000 pages with other records around the spans and spans that overlap, under every
result mode, with the exclusion sets growing, interleaved with discovery, UpdatePage and SetState, and rejected calls
that leave the next call's ids and outputs as if they never happened."""
import random

import numpy as np
import pytest

import discover_rules as dr
import tandem_rules as tr
from discover_rules import ST_NOLINE, ST_EMITTED
from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import Engine, EngineError, names_to_keys32
from distributed_crawler_b200.pack import Channel, pack_telegram
from go_rules import filter_username
from helpers import msg
from state_rules import GoState
from test_gpu_state import LAST, META
from test_gpu_state_discover import BAD, GOOD, MIN_DATE, edge_names, oracle
from tg_link_corpus import CHANNELS

pytestmark = pytest.mark.gpu
NOW = 1_760_000_000
RUN = abi.RUN_LINKS
RUN_MODES = [RUN, RUN | abi.RUN_JSONL, RUN | abi.RUN_JSONL | abi.RUN_JSONL_DEVICE, RUN | abi.RUN_NO_D2H,
             RUN | abi.RUN_JSONL | abi.RUN_FRONTIER | abi.RUN_SKIP_SELF | abi.RUN_FILTER | abi.RUN_SKIP_INVALID]
NAMES = [b"chan%03d" % k for k in range(60)]
BAD_NAMES = [b"abcd", b"helper_bot", b"SomeBot", b"9starts"]  # FilterUsername refuses them
STAMPS = [0, NOW - tr.TTL - 1, NOW - tr.TTL, NOW - tr.TTL + 1, NOW - 5]


def page_messages(rnd, owner_url, n):
    """a page of messages: t.me links and mentions with repeats within and across messages and pages, self links in the
    owner's case and lower-cased, names FilterUsername refuses, panicking records and records before min_post_date"""
    out = []
    for k in range(n):
        pool = NAMES[:20] + BAD_NAMES + [owner_url, owner_url.lower()]
        names = [rnd.choice(pool) for _ in range(rnd.choice([0, 1, 3, 6]))]
        text = " ".join(("t.me/" if rnd.random() < 0.6 else "@") + nm.decode() for nm in names)
        out.append(msg("messageText", "post %d %s" % (k, text), id=(k + 1) << 20, chat_id=-100777, channel=0,
                       date=MIN_DATE + 5 if rnd.random() < 0.85 else MIN_DATE - 5, panics=rnd.random() < 0.08))
    return out


def as_rows(got):
    edges = [(bytes(e["destination"][:e["dest_len"]]), int(e["record"]), int(e["batch"]), int(e["source_type"]),
              int(e["status"])) for e in got["edges"]]
    batches = [(bytes(b["batch_id"]), int(b["span"]), int(b["first_edge"]), int(b["n_edges"])) for b in got["batches"]]
    return edges, batches, [int(x) for x in got["span_batch"]]


class TandemSequence:
    def __init__(self, seed, n_owners=8, growth=True):
        self.rnd = random.Random(seed)
        self.e = Engine(min_post_date=MIN_DATE, frontier_capacity=1024, set_growth=(1 << 20) if growth else 0)
        self.go = GoState()
        self.x = tr.Tandem(self.go, seed=0x7A4D0000 + seed)
        self.e.state_id_seed(self.x.seed)
        self.d = dr.Discovery(self.go, seed=self.x.seed)  # page ids: the same key, their own counter
        long32 = edge_names()[1]
        urls = [NAMES[0], NAMES[1].upper(), long32[0], long32[1].upper(), NAMES[4], b"Chan005"]
        owners = [{"id": b"owner-%d" % k, "url": urls[k % len(urls)], "depth": k % 3, "status": b"fetched",
                   "sequenceId": b"seq-%d" % k} for k in range(n_owners)]
        self.state_set([(0, owners)])

    def state_set(self, layers):
        self.go.set_state(layers)
        self.e.state_set(layers)

    def grow_sets(self, n):
        """n more names into the invalid set (stamps around the TTL) and the discovered set"""
        r = self.rnd
        inv = r.sample(NAMES + edge_names()[1][:40], n)
        st = [r.choice(STAMPS) for _ in inv]
        self.e.set_add(abi.SET_INVALID, names_to_keys32(inv), np.array(st, np.int64))
        for nm, t in zip(inv, st):
            self.x.invalid.setdefault(nm, t)  # re-adding a key keeps the first stamp
        disc = r.sample(NAMES + edge_names()[1][:40], n)
        self.e.set_add(abi.SET_DISCOVERED, names_to_keys32(disc))
        self.x.discovered.update(disc)

    def result(self, owners, run_flags, slot=0, sizes=None, overlap=False):
        """one bulk result: filler records, a page of every owner, filler records; returns the spans and the per-record
        statuses and (name, source) link rows"""
        r = self.rnd
        sizes = sizes or [r.choice([0, 1, 4, 9, 20]) for _ in owners]
        src = r.random()
        msgs = page_messages(r, b"filler", r.choice([0, 3]))
        first0 = len(msgs)
        for pid, n in zip(owners, sizes):
            if src < 0.7:
                msgs += page_messages(r, self.go.page_map[pid]["url"], n)
            else:
                pool = edge_names()[0]
                a = r.randrange(len(pool) - n)
                msgs += pool[a:a + n]
        msgs += page_messages(r, b"filler", r.choice([0, 2]))
        b = pack_telegram(msgs, CHANNELS)  # the link corpus's channel table: its messages name all three
        spans, first = [], first0
        rows = self.e._st_rows()
        for pid, n in zip(owners, sizes):
            n_done = n if r.random() < 0.7 else r.randrange(n + 1)
            spans.append((rows[pid], first, n, n_done))
            first += n
        if overlap and len(spans) > 1:  # a span over records another span holds too
            a = r.randrange(len(spans))
            spans.append((rows[owners[(a + 1) % len(owners)]],) + spans[a][1:])
        clock = BAD if r.random() < 0.3 else GOOD
        ro = oracle(clock).telegram(b, RUN)
        self.e.set_clock(*clock)
        self.e.telegram_submit(slot, b, run_flags)
        self.e.telegram_wait(slot)
        self.e.set_clock(*GOOD)
        status = [int(s) for s in ro.status]
        links = [[(n, abi.SRC_NAMES.index(s)) for n, s in ro.record_links(i)] for i in range(ro.n)]
        return spans, status, links

    def expect(self, spans, status, links):
        pid_of = {v: k for k, v in self.e._st_rows().items()}
        edges, batches, span_batch, n_cand = [], [], [], 0
        for k, (row, first, n, n_done) in enumerate(spans):
            owner = self.go.page_map[pid_of[row]]
            for i in range(first, first + n_done):
                if status[i] in (ST_EMITTED, ST_NOLINE):
                    n_cand += sum(1 for o, _ in links[i] if o != owner["url"] and filter_username(o) == ""
                                  and not tr.is_invalid_channel(self.x.invalid, o, NOW))
            batch, es = self.x.page(pid_of[row], status[first:first + n], links[first:first + n], n_done, NOW)
            if batch is None:
                assert not es
                span_batch.append(abi.STATE_NO_BATCH)
                continue
            span_batch.append(len(batches))
            batches.append((batch["batch_id"], k, len(edges), len(es)))
            edges += [(x["destination"], first + x["record"], len(batches) - 1, x["source_type"], x["status"]) for x in es]
        return edges, batches, span_batch, n_cand

    def call(self, spans, status, links, slot=0):
        before = (self.e.state_render(META, LAST), self.e.state_layer_map())
        want = self.expect(spans, status, links)
        got = self.e.state_pending_edges(slot, spans, NOW)
        assert as_rows(got) == want[:3]
        assert got["n_candidates"] == want[3]
        assert (self.e.state_render(META, LAST), self.e.state_layer_map()) == before  # the state is unchanged
        return want


@pytest.mark.parametrize("seed", range(3))
def test_random_sequences_match_the_restatement(seed):
    sq = TandemSequence(seed)
    sq.grow_sets(10)
    r = sq.rnd
    seen = {"edges": 0, "dup": 0, "no_batch": 0, "shared": 0}
    for step in range(30):
        ids = list(sq.go.page_map)
        k = r.random()
        if k < 0.15:
            sq.grow_sets(r.choice([3, 10]))
        elif k < 0.25:  # UpdatePage: a new URL, so the self compare changes
            p = dict(sq.go.page_map[r.choice(ids)])
            p["url"] = r.choice(NAMES[:20] + [NAMES[2].upper()])
            p.pop("messages", None)
            sq.go.update_page(p)
            sq.e.state_update_page(p)
        elif k < 0.3:  # SetState: the batch counter carries on
            pages = [dict(sq.go.page_map[i]) for i in ids]
            for p in pages:
                p.pop("messages", None)
            sq.state_set([(0, pages)])
        else:
            slot = step % 3
            owners = r.sample(ids, min(len(ids), r.choice([1, 2, 5])))
            spans, status, links = sq.result(owners, r.choice(RUN_MODES), slot, overlap=r.random() < 0.4)
            edges, batches, span_batch, _ = sq.call(spans, status, links, slot)
            seen["edges"] += len(edges)
            seen["dup"] += sum(1 for x in edges if x[4] == abi.EDGE_DUPLICATE)
            seen["no_batch"] += span_batch.count(abi.STATE_NO_BATCH)
            names = [set(x[0] for x in edges if x[2] == b) for b in range(len(batches))]
            seen["shared"] += sum(1 for a in range(len(names)) for b in range(a) if names[a] & names[b])
            if r.random() < 0.3:  # snowball discovery on the same result: new owner pages, page ids apart from batch ids
                pid_of = {v: k for k, v in sq.e._st_rows().items()}
                want = []
                for row, first, n, n_done in spans:
                    want += sq.d.standalone_page(pid_of[row], status[first:first + n],
                                                 [[nm for nm, _ in ls] for ls in links[first:first + n]], n_done, (NOW, 0))
                got = sq.e.state_discover(slot, spans, abi.DISCOVER_NOW, (NOW, 0))
                assert got["ids"] == [p["id"] for p in want]
            sq.e.release(slot)
    assert sq.e.state_render(META, LAST) == sq.go.marshal(META, LAST)
    assert all(v > 0 for v in seen.values()), seen
    sq.e.close()


@pytest.mark.parametrize("P", [1, 2, 64, 1000])
def test_bulk_results_of_many_pages(P):
    """P pages in one bulk result (the page kernel at P = 1, the bulk pipeline beyond), overlapping spans, two calls in
    a row: the batch counter continues; from P = 2 on the launches do not depend on P"""
    sq = TandemSequence(100 + P, n_owners=min(P, 50))
    sq.grow_sets(20)
    ids = list(sq.go.page_map)
    owners = [ids[k % len(ids)] for k in range(P)]
    launches = []
    for slot, mode in ((0, RUN | abi.RUN_NO_D2H), (1, RUN | abi.RUN_JSONL | abi.RUN_JSONL_DEVICE)):
        spans, status, links = sq.result(owners, mode, slot, sizes=[sq.rnd.choice([1, 3, 5]) for _ in owners],
                                         overlap=True)
        edges, batches, _, _ = sq.call(spans, status, links, slot)
        assert len(spans) == P + (P > 1) and (batches or P < 64)
        launches.append(sq.e.state_edges_launches)
        sq.e.release(slot)
    assert launches[0] == launches[1]
    sq.e.close()


def test_launches_do_not_depend_on_the_number_of_pages():
    sq = TandemSequence(7, n_owners=50)
    ids = list(sq.go.page_map)
    launches = []
    for P in (2, 64, 1000):
        owners = [ids[k % len(ids)] for k in range(P)]
        spans, status, links = sq.result(owners, RUN | abi.RUN_NO_D2H, 0, sizes=[3] * P)
        sq.call(spans, status, links, 0)
        launches.append(sq.e.state_edges_launches)
        sq.e.release(0)
    assert launches[0] == launches[1] == launches[2], launches
    sq.e.close()


def test_reference_tandem_vectors_on_the_gpu(vectors):
    for name, t in vectors["tandem"].items():
        e = Engine()
        e.state_id_seed(5)
        e.state_set([(0, [{"id": b"p", "url": t["owner_url"].encode()}])])
        if t.get("invalid"):
            e.set_add(abi.SET_INVALID, names_to_keys32([n.encode() for n in t["invalid"]]), np.zeros(len(t["invalid"]), np.int64))
        b = pack_telegram([msg("messageText", t["text"], [tuple(x) for x in t["entities"]])],
                          [Channel(name=t["owner_url"], username=t["owner_url"])])
        e.telegram_submit(0, b, RUN)
        e.telegram_wait(0)
        edges, batches, span_batch = as_rows(e.state_pending_edges(0, [(0, 0, 1, 1)], NOW))
        assert [x[0].decode() for x in edges] == t["expected_edges"], name
        assert span_batch == ([0] if t["expected_edges"] else [abi.STATE_NO_BATCH]), name
        if batches:
            assert batches[0][0] == tr.batch_id(5, 0)
        e.release(0)
        e.close()


def test_rejected_calls_change_nothing():
    sq = TandemSequence(41, n_owners=3)
    e, x = sq.e, sq.x
    row = e._st_rows()[b"owner-0"]
    ms = [msg("messageText", "t.me/chan007 t.me/chan008", id=(k + 1) << 20, chat_id=-1, date=MIN_DATE + 1) for k in range(4)]
    e.telegram_submit(0, pack_telegram(ms), RUN)
    e.telegram_wait(0)

    def rejected(call, code):
        with pytest.raises(EngineError) as ei:
            call()
        assert ei.value.code == code

    rejected(lambda: e.state_pending_edges(0, [(99, 0, 4, 4)], NOW), abi.E_ARG)   # no such row
    rejected(lambda: e.state_pending_edges(0, [(row, 2, 3, 3)], NOW), abi.E_ARG)  # outside the result
    rejected(lambda: e.state_pending_edges(0, [(row, 0, 2, 3)], NOW), abi.E_ARG)  # n_done > n_records
    rejected(lambda: e.state_pending_edges(2, [(row, 0, 4, 4)], NOW), abi.E_STATE)  # no result
    e.telegram_submit(1, pack_telegram(ms), abi.RUN_JSONL)
    e.telegram_wait(1)
    rejected(lambda: e.state_pending_edges(1, [(row, 0, 4, 4)], NOW), abi.E_STATE)  # no TGI_RUN_LINKS
    e.release(1)
    from yt_corpus import make_youtube
    yt, _, _ = make_youtube(4, seed=2)
    e.youtube_submit(1, yt, RUN)
    e.youtube_wait(1)
    rejected(lambda: e.state_pending_edges(1, [(row, 0, 4, 4)], NOW), abi.E_STATE)  # a YouTube result
    e.release(1)
    # the first accepted call gets the first batch id and the edges of a fresh call
    ro = oracle(GOOD).telegram(pack_telegram(ms), RUN)
    spans = [(row, 0, 4, 4), (row, 1, 3, 3)]
    got = sq.call(spans, [int(s) for s in ro.status],
                  [[(n, abi.SRC_NAMES.index(s)) for n, s in ro.record_links(i)] for i in range(ro.n)], 0)
    assert [b[0] for b in got[1]] == [tr.batch_id(x.seed, 0), tr.batch_id(x.seed, 1)] and len(got[0]) == 4
    e.release(0)
    rejected(lambda: e.state_pending_edges(0, spans, NOW), abi.E_STATE)  # a released result
    # no seed: a call that would make a batch is refused and leaves the counter; one that makes none is not
    e2 = Engine(min_post_date=MIN_DATE)
    e2.state_set([(0, [{"id": b"p", "url": b"chan007"}])])
    e2.telegram_submit(0, pack_telegram(ms[:1]), RUN)
    e2.telegram_wait(0)
    assert as_rows(e2.state_pending_edges(0, [(0, 0, 1, 0)], NOW))[2] == [abi.STATE_NO_BATCH]
    rejected(lambda: e2.state_pending_edges(0, [(0, 0, 1, 1)], NOW), abi.E_STATE)
    e2.state_id_seed(3)
    edges, batches, _ = as_rows(e2.state_pending_edges(0, [(0, 0, 1, 1)], NOW))
    assert [x[0] for x in edges] == [b"chan008"] and batches[0][0] == tr.batch_id(3, 0)
    e2.release(0)
    e2.close()
    e.close()
