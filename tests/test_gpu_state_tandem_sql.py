"""GPU tests: the tandem hand-off's binding calls (tgi_state_edge_sql) against tests/tandem_sql_rules.py, byte for byte
at 1, 7 and 8191 rows per statement after every hand-off of the tandem test's sequences, in fixed offsets and local
zones; a hand-off past one grid pass of the SQL kernels, also in a child process under TGI_GRID_MULT=1; spans without
edges and steps without batches; and refused calls that leave the next output as it was."""
import os
import subprocess
import sys

import pytest

import tandem_sql_rules as sr
from discover_rules import ST_EMITTED
from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import Engine, EngineError
from distributed_crawler_b200.pack import pack_telegram
from helpers import msg
from test_gpu_state import LAST, META
from test_gpu_state_discover import GOOD, MIN_DATE, oracle
from test_gpu_state_tandem import NOW, RUN, RUN_MODES, TandemSequence, as_rows
from test_zones import ZONES

pytestmark = pytest.mark.gpu
NY = ZONES["America/New_York"]
KS = (1, 7, sr.MAX_ROWS)
CRAWL_IDS = [b"crawl-2025", b"c<&>\"\\ \xe2\x80\xa8 \xff", b""]
CLOCKS = [(NOW, 0), (NOW, 120_000_000), (1710054000 - 1, 999_999_999), (1730613600, 1)]  # around New York's transitions


class SqlSequence(TandemSequence):
    """the tandem sequence with every hand-off also rendered as binding calls, before any other state call"""

    def __init__(self, seed, zone=None, tz=0, **kw):
        super().__init__(seed, **kw)
        self.zone, self.tz, self.n_sql = zone, tz, 0
        if tz:  # the same state under a context whose time.Local is the fixed offset tz
            self.e.close()
            self.e = Engine(min_post_date=MIN_DATE, frontier_capacity=1024, set_growth=1 << 20, tz_offset_sec=tz)
            self.e.state_id_seed(self.x.seed)
            pages = [dict(p) for p in self.go.page_map.values()]
            for p in pages:
                p.pop("messages", None)
            self.e.state_set([(0, pages)])
        if zone is not None:
            self.e.set_zone(*zone)

    def pages(self, spans, want):
        """the restatement's (batch, edges) of every batch, the owner as the state holds it"""
        pid_of = {v: k for k, v in self.e._st_rows().items()}
        edges, batches = want[0], want[1]
        out = []
        for q, (bid, span, first, n) in enumerate(batches):
            o = self.go.page_map[pid_of[spans[span][0]]]
            b = {"batch_id": bid, "source_channel": o["url"], "source_page_id": o["id"], "source_depth": o.get("depth", 0),
                 "sequence_id": o.get("sequenceId", b"")}
            out.append((b, [{"destination": x[0], "source_type": x[3], "status": x[4]} for x in edges[first:first + n]]))
        return out

    def check_sql(self, spans, want):
        pages = self.pages(spans, want)
        for j, k in enumerate(KS):
            crawl = CRAWL_IDS[(self.n_sql + j) % len(CRAWL_IDS)]
            now = CLOCKS[(self.n_sql + j) % len(CLOCKS)]
            t = sr.discovery_time(*now, self.zone, self.tz)
            got = self.e.state_edge_sql(crawl, now, k)
            assert got == sr.statements(pages, crawl, t, k), (k, crawl, now)
            assert (self.e.state_sql_launches == 0) == (not pages)
        self.n_sql += 1
        return pages

    def call(self, spans, status, links, slot=0):
        before = (self.e.state_render(META, LAST), self.e.state_layer_map())
        want = self.expect(spans, status, links)
        got = self.e.state_pending_edges(slot, spans, NOW)
        assert as_rows(got) == want[:3]
        self.check_sql(spans, want)
        assert as_rows(got) == want[:3]  # the hand-off's own output outlives the renders
        assert (self.e.state_render(META, LAST), self.e.state_layer_map()) == before
        return want


@pytest.mark.parametrize("seed, zone, tz", [(0, None, 0), (1, NY, 0), (2, None, 5 * 3600 + 30 * 60 + 15),
                                            (3, None, -3600)])
def test_random_sequences_render_the_reference_calls(seed, zone, tz):
    sq = SqlSequence(seed, zone=zone, tz=tz)
    sq.grow_sets(10)
    r = sq.rnd
    seen = {"batches": 0, "empty": 0}
    for step in range(16):
        ids = list(sq.go.page_map)
        if r.random() < 0.15:
            sq.grow_sets(5)
            continue
        slot = step % 3
        owners = r.sample(ids, min(len(ids), r.choice([1, 2, 5])))
        spans, status, links = sq.result(owners, r.choice(RUN_MODES), slot, overlap=r.random() < 0.4)
        edges, batches, span_batch, _ = sq.call(spans, status, links, slot)
        seen["batches"] += len(batches)
        seen["empty"] += span_batch.count(abi.STATE_NO_BATCH)
        sq.e.release(slot)
    assert all(v > 0 for v in seen.values()), seen
    sq.e.close()


def big_handoff(sq, n_edges):
    """one bulk result whose hand-off holds at least n_edges edges: pages of 40-name messages, every name new to its page"""
    ids = list(sq.go.page_map)
    per_page = 600
    n_pages = (n_edges + per_page - 1) // per_page
    msgs, spans, rows = [], [], sq.e._st_rows()
    for p in range(n_pages):
        first = len(msgs)
        for m in range(per_page // 40):
            names = ["n%04dx%04d" % (p, 40 * m + j) for j in range(40)]
            msgs.append(msg("messageText", " ".join("t.me/" + x for x in names), id=(len(msgs) + 1) << 20,
                            chat_id=-100777, channel=0, date=MIN_DATE + 5))
        spans.append((rows[ids[p % len(ids)]], first, len(msgs) - first, len(msgs) - first))
    b = pack_telegram(msgs)
    ro = oracle(GOOD).telegram(b, RUN)
    sq.e.set_clock(*GOOD)
    sq.e.telegram_submit(0, b, RUN | abi.RUN_NO_D2H)
    sq.e.telegram_wait(0)
    status = [int(s) for s in ro.status]
    links = [[(n, abi.SRC_NAMES.index(s)) for n, s in ro.record_links(i)] for i in range(ro.n)]
    assert all(s == ST_EMITTED for s in status)
    return spans, status, links


def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_a_handoff_past_one_grid_pass():
    """SMs x 1024 + 2000 edges: the SQL kernels' rows take more than one pass of their grid-stride loops"""
    sq = SqlSequence(50, n_owners=40)
    spans, status, links = big_handoff(sq, sms() * 1024 + 2000)
    edges, batches, _, _ = sq.call(spans, status, links, 0)
    assert len(edges) >= sms() * 1024 + 2000 and sq.e.state_sql_launches >= 3
    sq.e.release(0)
    sq.e.close()


def test_a_big_handoff_with_a_grid_of_one_cta_per_sm():
    code = (
        "import sys; sys.path.insert(0, 'tests')\n"
        "import test_gpu_state_tandem_sql as t\n"
        "sq = t.SqlSequence(51, n_owners=40)\n"
        "spans, status, links = t.big_handoff(sq, 40_000)\n"
        "sq.call(spans, status, links, 0)\n"
        "sq.e.release(0)\n"
        "sq.e.close()\n"
        "print('ok')\n")
    env = dict(os.environ, TGI_GRID_MULT="1")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and "ok" in p.stdout, p.stderr[-3000:]


def test_spans_without_edges_and_steps_without_batches():
    sq = SqlSequence(60, n_owners=4)
    ids = list(sq.go.page_map)
    # spans that process nothing: no batch at all, 0 statements and no launch
    spans, status, links = sq.result(ids[:3], RUN, 0, sizes=[3, 0, 2])
    spans = [(row, first, n, 0) for row, first, n, _ in spans]
    want = sq.call(spans, status, links, 0)  # 0 statements and no launch at every k
    assert want[1] == []
    # a bad clock does not matter without edges (no time is marshalled)
    assert as_rows(sq.e.state_pending_edges(0, spans, NOW))[2] == [abi.STATE_NO_BATCH] * 3
    assert sq.e.state_edge_sql(b"c", (400_000_000_000, 0), 1) == [] and sq.e.state_sql_launches == 0
    sq.e.release(0)
    # some spans with a batch, some without
    for _ in range(6):
        spans, status, links = sq.result(ids, RUN, 0, sizes=[4, 0, 9, 1])
        want = sq.call(spans, status, links, 0)
        sq.e.release(0)
        if want[1] and abi.STATE_NO_BATCH in want[2]:
            break
    else:
        pytest.fail("no step with both kinds of span")
    sq.e.close()


def test_refused_calls_leave_the_next_output_unchanged():
    sq = SqlSequence(70, n_owners=3)
    e = sq.e

    def refused(call, code):
        with pytest.raises(EngineError) as ei:
            call()
        assert ei.value.code == code

    refused(lambda: e.state_edge_sql(b"c", (NOW, 0), 1), abi.E_STATE)  # no hand-off yet
    ids = list(sq.go.page_map)
    spans, status, links = sq.result(ids, RUN, 0, sizes=[5, 5, 5])
    want = sq.call(spans, status, links, 0)  # ends with a state_render: the hand-off is over
    refused(lambda: e.state_edge_sql(b"c", (NOW, 0), 1), abi.E_STATE)
    want = sq.expect(spans, status, links)
    assert as_rows(e.state_pending_edges(0, spans, NOW)) == want[:3]
    pages = sq.pages(spans, want)
    assert pages
    good = e.state_edge_sql(b"c", (NOW, 5), 7)
    assert good == sr.statements(pages, b"c", sr.discovery_time(NOW, 5), 7)
    for k in (0, sr.MAX_ROWS + 1, 1 << 31):
        refused(lambda: e.state_edge_sql(b"c", (NOW, 5), k), abi.E_ARG)
    for now in ((NOW, -1), (NOW, 1_000_000_000), (253402300800, 0), (-62167219201, 0)):
        refused(lambda: e.state_edge_sql(b"c", now, 7), abi.E_ARG)
    assert e.state_edge_sql(b"c", (NOW, 5), 7) == good
    e.state_layers()  # a state call between: the hand-off is over, the batch counter untouched
    refused(lambda: e.state_edge_sql(b"c", (NOW, 5), 7), abi.E_STATE)
    n0 = len(want[1])
    want = sq.expect(spans, status, links)
    assert as_rows(e.state_pending_edges(0, spans, NOW)) == want[:3]
    assert e.state_edge_sql(b"c", (NOW, 5), 7) == sr.statements(sq.pages(spans, want), b"c", sr.discovery_time(NOW, 5), 7)
    assert sq.x.n == 3 * n0 and want[1][0][0] != pages[0][0]["batch_id"]
    e.release(0)
    e.close()
