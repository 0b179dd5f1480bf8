"""GPU tests: the tandem forced walkback (tgi_state_walkback) against tests/walkback_rules.py — every edge-less span's
pick, draws and ids, and every statement byte for byte at 1, 2, 7 and 8191 rows per statement, after the hand-offs of
the tandem test's sequences, with discovered sets of 0, 1, 2, random and grown sizes that hold the owners' URLs or not;
repeated calls on one hand-off; walkback and edge SQL in both orders with both pinned outputs intact; the end of the
hand-off; refused calls that leave the next output unchanged; and a hand-off past one grid pass."""
import ctypes as C

import numpy as np
import pytest

import tandem_sql_rules as sr
import walkback_rules as wr
from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import Engine, EngineError, lib, names_to_keys32
from distributed_crawler_b200.pack import pack_telegram
from helpers import msg
from test_gpu_state import LAST, META
from test_gpu_state_discover import MIN_DATE
from test_gpu_state_tandem import NAMES, NOW, RUN, RUN_MODES, TandemSequence, as_rows

pytestmark = pytest.mark.gpu
KS = (1, 2, 7, wr.MAX_ROWS)
CRAWL_IDS = [b"crawl-2025", b"c<&>\"\\ \xe2\x80\xa8 \xff", b""]
CLOCKS = [(NOW, 0), (NOW, 120_000_000), (1710054000 - 1, 999_999_999)]


class WalkSequence(TandemSequence):
    """the tandem sequence with the discovered set's keys kept in insertion order, as the resident set holds them, and
    the count w of edge-less spans handled"""

    def __init__(self, seed, **kw):
        super().__init__(seed, **kw)
        self.disc, self.w = [], 0
        add = self.e.set_add

        def set_add(which, keys32, stamps=None):
            add(which, keys32, stamps)
            if which == abi.SET_DISCOVERED:
                for k in np.asarray(keys32, np.uint8).reshape(-1, 32):
                    nm = bytes(k).rstrip(b"\0")
                    if nm not in self.disc:
                        self.disc.append(nm)
        self.e.set_add = set_add

    def add_discovered(self, names):
        self.e.set_add(abi.SET_DISCOVERED, names_to_keys32(names))
        self.x.discovered.update(names)

    def walks(self, spans, span_batch):
        """the restatement's (owner, result) of every edge-less span, at the current w"""
        pid_of = {v: k for k, v in self.e._st_rows().items()}
        out = []
        for j, (sp, b) in enumerate(zip(spans, span_batch)):
            if b != abi.STATE_NO_BATCH:
                continue
            owner = self.go.page_map[pid_of[sp[0]]]
            res, _ = wr.forced_walkback(owner, self.disc, self.x.seed, self.w + len(out), b"", None)
            out.append((owner, dict(res, span=j)))
        return out

    def check_walkback(self, spans, span_batch, n_call=0):
        """every k on the one hand-off: the same picks and ids each time, w advanced once"""
        walks = self.walks(spans, span_batch)
        first = None
        for j, k in enumerate(KS):
            crawl = CRAWL_IDS[(n_call + j) % len(CRAWL_IDS)]
            now = CLOCKS[(n_call + j) % len(CLOCKS)]
            got, stmts = self.e.state_walkback(crawl, now, k)
            assert got == [r for _, r in walks], k
            assert stmts == wr.statements(walks, crawl, sr.discovery_time(*now), k), (k, crawl, now)
            if first is None:
                first = got
                launches = self.e.state_walk_launches
                assert (launches == 0) == (not walks)
            else:
                assert got == first
        self.w += len(walks)
        return walks

    def step(self, owners, run_flags, slot, sizes=None, edge_sql_first=False, n_call=0):
        spans, status, links = self.result(owners, run_flags, slot, sizes=sizes)
        want = self.expect(spans, status, links)
        got = self.e.state_pending_edges(slot, spans, NOW)
        assert as_rows(got) == want[:3]
        if edge_sql_first:
            self.e.state_edge_sql(b"c", (NOW, 0), 7)
        walks = self.check_walkback(spans, want[2], n_call)
        if not edge_sql_first:
            self.e.state_edge_sql(b"c", (NOW, 0), 7)
            assert self.e.state_walkback(b"c", (NOW, 0), 3)[0] == [r for _, r in walks]
        assert as_rows(got) == want[:3]
        self.e.release(slot)
        return spans, want, walks


@pytest.mark.parametrize("seed", range(3))
def test_random_sequences_with_every_kind_of_discovered_set(seed):
    sq = WalkSequence(seed)
    r = sq.rnd
    ids = list(sq.go.page_map)
    owner_urls = [sq.go.page_map[i]["url"] for i in ids]
    seen = {wr.WALK_OK: 0, wr.WALK_EXHAUSTED: 0, wr.WALK_EMPTY: 0, "skips": 0, "rows": 0}
    n_call = 0

    def run(n_steps):
        nonlocal n_call
        for _ in range(n_steps):
            slot = n_call % 3
            owners = r.sample(ids, min(len(ids), r.choice([1, 2, 5, 8])))
            sizes = [r.choice([0, 0, 1, 4]) for _ in owners]
            _, _, walks = sq.step(owners, r.choice(RUN_MODES), slot, sizes=sizes, edge_sql_first=n_call % 2 == 1,
                                  n_call=n_call)
            n_call += 1
            for _, res in walks:
                seen[res["status"]] += 1
                seen["skips"] += res["draws"] > 1
                seen["rows"] += res["status"] == wr.WALK_OK

    run(3)  # a set never allocated: every edge-less span is TGI_WALK_EMPTY
    sq.add_discovered([owner_urls[0]])  # one key, some owner's URL: that owner's spans are exhausted after 10 draws
    run(4)
    sq.add_discovered([NAMES[30]])  # two keys
    run(3)
    sq.add_discovered(r.sample(NAMES[:30], 12) + owner_urls[:3])  # random, with owners' URLs inside
    run(4)
    assert sq.e.set_info(abi.SET_DISCOVERED)["grows"] == 0
    sq.add_discovered([b"grown%05d" % i for i in range(3000)] + [owner_urls[1].upper()])  # through tgi_set_growth
    assert sq.e.set_info(abi.SET_DISCOVERED)["grows"] > 0
    run(4)
    assert sq.e.set_size(abi.SET_DISCOVERED) == len(sq.disc)
    assert sq.e.state_render(META, LAST) == sq.go.marshal(META, LAST)
    assert all(v > 0 for v in seen.values()), seen
    sq.e.close()


def test_a_set_of_the_owner_url_only_and_case_sensitive_compares():
    sq = WalkSequence(10, n_owners=6)
    ids = list(sq.go.page_map)
    urls = [sq.go.page_map[i]["url"] for i in ids]
    sq.add_discovered([urls[1]])  # one key, owner 1's URL: exhausted after exactly 10 draws, the others take it
    _, _, walks = sq.step(ids, RUN, 0, sizes=[0] * len(ids))
    got = {o["url"]: (r["status"], r["draws"], r["url"]) for o, r in walks}
    assert got[urls[1]] == (wr.WALK_EXHAUSTED, 10, b"")
    assert got[urls[0]] == (wr.WALK_OK, 1, urls[1])
    sq.e.close()
    sq = WalkSequence(10, n_owners=6)
    assert urls[5] == b"Chan005"
    sq.add_discovered([b"chan005"])  # owner 5's URL in another case: not its URL
    _, _, walks = sq.step(ids, RUN, 0, sizes=[0] * len(ids))
    assert {o["url"]: (r["status"], r["draws"], r["url"]) for o, r in walks}[urls[5]] == (wr.WALK_OK, 1, b"chan005")
    sq.e.close()


def test_handoffs_without_edge_less_spans_launch_nothing():
    sq = WalkSequence(11, n_owners=4)
    sq.add_discovered([b"k1", b"k2"])
    e = sq.e
    ids = list(sq.go.page_map)
    for _ in range(10):
        spans, status, links = sq.result(ids, RUN, 0, sizes=[9] * len(ids))
        want = sq.expect(spans, status, links)
        assert as_rows(e.state_pending_edges(0, spans, NOW)) == want[:3]
        e.release(0)
        if abi.STATE_NO_BATCH not in want[2]:
            break
    else:
        pytest.fail("no hand-off with a batch for every span")
    assert e.state_walkback(b"c", (NOW, 0), 1) == ([], []) and e.state_walk_launches == 0
    # and a bad clock does not matter without rows
    assert e.state_walkback(b"c", (400_000_000_000, 0), 1) == ([], [])
    e.close()


def _raw_edge_sql(e, k):
    out = abi.StateEdgeSqlC()
    assert lib().tgi_state_edge_sql(e.h, b"c", 1, NOW, 0, k, C.byref(out)) == 0
    return out, C.string_at(out.stmts, 40 * out.n_stmts) + C.string_at(out.data, out.data_len)


def _raw_walkback(e, k):
    out = abi.StateWalkbackC()
    assert lib().tgi_state_walkback(e.h, b"c", 1, NOW, 0, k, C.byref(out)) == 0
    return out, (C.string_at(out.walkbacks, 120 * out.n_walkbacks) + C.string_at(out.stmts, 40 * out.n_stmts)
                 + C.string_at(out.data, out.data_len))


def _reread(out):
    if isinstance(out, abi.StateWalkbackC):
        return (C.string_at(out.walkbacks, 120 * out.n_walkbacks) + C.string_at(out.stmts, 40 * out.n_stmts)
                + C.string_at(out.data, out.data_len))
    return C.string_at(out.stmts, 40 * out.n_stmts) + C.string_at(out.data, out.data_len)


def test_walkback_and_edge_sql_in_both_orders_keep_both_outputs():
    sq = WalkSequence(12, n_owners=6)
    sq.add_discovered([b"k%d" % i for i in range(5)])
    ids = list(sq.go.page_map)
    for order in range(2):
        for _ in range(10):
            spans, status, links = sq.result(ids, RUN, 0, sizes=[0, 5, 0, 9, 1, 0])
            want = sq.expect(spans, status, links)
            sq.e.state_pending_edges(0, spans, NOW)
            if want[1] and abi.STATE_NO_BATCH in want[2]:
                break
            sq.e.release(0)
        else:
            pytest.fail("no step with both kinds of span")
        e = sq.e
        if order == 0:
            a, a_bytes = _raw_edge_sql(e, 2)
            b, b_bytes = _raw_walkback(e, 2)
            assert _reread(a) == a_bytes
            a2, a2_bytes = _raw_edge_sql(e, 2)
            assert _reread(b) == b_bytes and a2_bytes == a_bytes
        else:
            b, b_bytes = _raw_walkback(e, 1)
            a, a_bytes = _raw_edge_sql(e, 1)
            assert _reread(b) == b_bytes
            b2, b2_bytes = _raw_walkback(e, 1)
            assert _reread(a) == a_bytes and b2_bytes == b_bytes
        walks = sq.walks(spans, want[2])
        got, stmts = e.state_walkback(b"c", (NOW, 0), 1)
        assert got == [r for _, r in walks] and stmts == wr.statements(walks, b"c", sr.discovery_time(NOW, 0), 1)
        sq.w += len(walks)
        e.release(0)
    sq.e.close()


def test_any_other_state_call_ends_the_handoff():
    sq = WalkSequence(13, n_owners=3)
    e = sq.e
    sq.add_discovered([b"k1"])

    def refused(call, code):
        with pytest.raises(EngineError) as ei:
            call()
        assert ei.value.code == code

    refused(lambda: e.state_walkback(b"c", (NOW, 0), 1), abi.E_STATE)  # no hand-off yet
    ids = list(sq.go.page_map)
    for other in (lambda: e.state_layers(), lambda: e.state_render(META, LAST), lambda: e.state_layer_map(),
                  lambda: e.state_read_pages([0], messages=False)):
        spans, status, links = sq.result(ids, RUN, 0, sizes=[0, 0, 0])
        got = e.state_pending_edges(0, spans, NOW)
        walks = sq.check_walkback(spans, [int(x) for x in got["span_batch"]])
        assert len(walks) == 3
        other()
        refused(lambda: e.state_walkback(b"c", (NOW, 0), 1), abi.E_STATE)
        refused(lambda: e.state_edge_sql(b"c", (NOW, 0), 1), abi.E_STATE)
        e.release(0)
    e.close()


def test_refused_calls_leave_the_next_output_unchanged():
    sq = WalkSequence(14, n_owners=3)
    e = sq.e
    sq.add_discovered([b"k1", b"k2", b"k3"])

    def refused(call, code):
        with pytest.raises(EngineError) as ei:
            call()
        assert ei.value.code == code

    ids = list(sq.go.page_map)
    spans, status, links = sq.result(ids, RUN, 0, sizes=[0, 0, 0])
    got = e.state_pending_edges(0, spans, NOW)
    sb = [int(x) for x in got["span_batch"]]
    # refused first calls: nothing is picked and w stays
    for k in (0, wr.MAX_ROWS + 1, 1 << 31):
        refused(lambda: e.state_walkback(b"c", (NOW, 5), k), abi.E_ARG)
    for now in ((NOW, -1), (NOW, 1_000_000_000), (253402300800, 0), (-62167219201, 0)):
        refused(lambda: e.state_walkback(b"c", now, 7), abi.E_ARG)
    walks = sq.check_walkback(spans, sb)  # the picks of w as it was
    assert [r["status"] for _, r in walks] == [wr.WALK_OK] * 3
    good = e.state_walkback(b"c", (NOW, 5), 7)
    refused(lambda: e.state_walkback(b"c", (253402300800, 0), 7), abi.E_ARG)
    assert e.state_walkback(b"c", (NOW, 5), 7) == good
    e.release(0)
    # the next hand-off continues at w
    spans, status, links = sq.result(ids, RUN, 1, sizes=[0, 0, 0])
    sq.check_walkback(spans, [int(x) for x in e.state_pending_edges(1, spans, NOW)["span_batch"]])
    e.release(1)
    e.close()
    # no seed: a hand-off without batches is accepted, its walkbacks are not
    e2 = Engine(min_post_date=MIN_DATE)
    e2.state_set([(0, [{"id": b"p", "url": b"chan007"}])])
    e2.set_add(abi.SET_DISCOVERED, names_to_keys32([b"k1"]))
    e2.telegram_submit(0, pack_telegram([msg("messageText", "t.me/chan008", id=1 << 20, chat_id=-1,
                                             date=MIN_DATE + 1)]), RUN)
    e2.telegram_wait(0)
    assert as_rows(e2.state_pending_edges(0, [(0, 0, 1, 0)], NOW))[2] == [abi.STATE_NO_BATCH]
    refused(lambda: e2.state_walkback(b"c", (NOW, 0), 1), abi.E_STATE)
    e2.state_id_seed(3)  # a state call: the hand-off is over
    refused(lambda: e2.state_walkback(b"c", (NOW, 0), 1), abi.E_STATE)
    e2.state_pending_edges(0, [(0, 0, 1, 0)], NOW)
    got, stmts = e2.state_walkback(b"c", (NOW, 0), 1)
    res, calls = wr.forced_walkback({"id": b"p", "url": b"chan007"}, [b"k1"], 3, 0, b"c", sr.discovery_time(NOW, 0))
    assert got == [dict(res, span=0)] and [(k, s, p) for k, _, s, p in stmts] == calls
    e2.release(0)
    e2.close()


def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_a_handoff_past_one_grid_pass():
    """SMs x 1024 + 2000 edge-less spans: the pick and the SQL kernels take more than one pass of their grid-stride
    loops"""
    sq = WalkSequence(15, n_owners=40)
    sq.add_discovered([b"k%02d" % i for i in range(20)] + [sq.go.page_map[i]["url"] for i in list(sq.go.page_map)[:3]])
    e = sq.e
    rows = list(e._st_rows().values())
    e.telegram_submit(0, pack_telegram([msg("messageText", "t.me/chan008", id=1 << 20, chat_id=-1,
                                            date=MIN_DATE + 1)]), RUN)
    e.telegram_wait(0)
    n = sms() * 1024 + 2000
    spans = [(rows[j % len(rows)], 0, 1, 0) for j in range(n)]
    sb = [int(x) for x in e.state_pending_edges(0, spans, NOW)["span_batch"]]
    assert sb == [abi.STATE_NO_BATCH] * n
    walks = sq.walks(spans, sb)
    t = sr.discovery_time(NOW, 0)
    for k in (wr.MAX_ROWS, 1):
        got, stmts = e.state_walkback(b"crawl", (NOW, 0), k)
        assert got == [r for _, r in walks]
        assert stmts == wr.statements(walks, b"crawl", t, k), k
    assert sum(r["status"] == wr.WALK_OK for _, r in walks) > n - 10
    e.release(0)
    e.close()
