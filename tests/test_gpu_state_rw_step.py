"""GPU tests: the standard random walk (tgi_state_rw_lookups, tgi_state_rw_step) against tests/random_walk_rules.py —
the lookup rows, every span's step, the lookup stats, every statement byte for byte at 1 and 8191 rows per statement and
the three sets afterwards (sizes, first-occurrence exports, stamps), over bulk results under every result mode with
spans that share records, a link-heavy corpus, retires in the middle of a span, calls of 10^3 and 10^5 spans (the
second past one grid pass), refused calls that leave the sets and the next output unchanged, and the end of the lists."""
import numpy as np
import pytest

import random_walk_rules as rw
import tandem_sql_rules as sr
from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import EngineError, names_to_keys32
from test_gpu_state_tandem import NAMES, NOW, RUN, RUN_MODES, TandemSequence
from tg_link_corpus import CHANNELS

pytestmark = pytest.mark.gpu
KS = (1, rw.MAX_ROWS)
CRAWL = b"crawl-\xe2\x80\xa8<&>"
TIME = sr.discovery_time(NOW, 250_000_000)


def refused(call, code):
    with pytest.raises(EngineError) as ei:
        call()
    assert ei.value.code == code


class RwSequence(TandemSequence):
    """the tandem sequence's engine and results, with the three sets mirrored in a random_walk_rules.FakeState and the
    counter u of deciding spans"""

    def __init__(self, seed, **kw):
        super().__init__(seed, **kw)
        self.sm, self.u = rw.FakeState(), 0

    def seed_sets(self, names):
        r = self.rnd
        inv = r.sample(names, len(names) // 4)
        stamps = [r.choice([0, NOW - rw.wr.MAX_ROWS, NOW - 30 * 24 * 3600 - 1, NOW - 5]) for _ in inv]
        disc = r.sample(names, len(names) // 4)
        seeds = r.sample(names, len(names) // 5)
        self.e.set_add(abi.SET_INVALID, names_to_keys32(inv), np.array(stamps, np.int64))
        self.e.set_add(abi.SET_DISCOVERED, names_to_keys32(disc))
        self.e.set_add(abi.SET_SEEDS, names_to_keys32(seeds))
        for nm, t in zip(inv, stamps):
            self.sm.invalid.setdefault(nm, t)
        for nm in disc:
            self.sm.add_discovered_channel(nm)
        for nm in seeds:
            self.sm.seeds.setdefault(nm, 1)

    def pages(self, spans, status, links):
        pid_of = {v: k for k, v in self.e._st_rows().items()}
        return [(self.go.page_map[pid_of[row]], status[first:first + n], links[first:first + n], n_done)
                for row, first, n, n_done in spans]

    def sets(self):
        out = []
        for which in (abi.SET_INVALID, abi.SET_DISCOVERED, abi.SET_SEEDS):
            keys, stamps = self.e.set_export(which)
            names = [bytes(k).rstrip(b"\0") for k in keys]
            out.append(dict(zip(names, stamps.tolist())) if stamps is not None else names)
        return out

    def want_sets(self):
        return [self.sm.invalid, self.sm.discovered, list(self.sm.seeds)]

    def step(self, spans, status, links, k, rate, retire_at=None, slot=0):
        """one lookups call and one step against the restatement; returns the outcomes' codes"""
        r = self.rnd
        pages = self.pages(spans, status, links)
        got = self.e.state_rw_lookups(slot, spans, NOW)
        want = rw.lookups(self.sm, pages, NOW)
        assert [(bytes(x["name"][:x["name_len"]]), int(x["span"]), int(x["record"]), int(x["source_type"]))
                for x in got["lookups"]] == [(n, p, spans[p][1] + i, s) for n, p, i, s in want]
        assert got["n_candidates"] == sum(got["span_candidates"].tolist())
        outcome = {}
        for q, (name, _, _, _) in enumerate(want):
            code = rw.RETIRE if q == retire_at else r.choice([rw.FOUND, rw.FOUND, rw.NOT_SUPERGROUP, rw.NOT_FOUND])
            outcome[name] = (code, r.randrange(-(1 << 62), 1 << 62))
        spans_g, stats_g, stmts_g = self.e.state_rw_step([outcome[n] for n, _, _, _ in want], rate, CRAWL,
                                                         (NOW, 250_000_000), k)
        processed, stats, n_dec = rw.run(self.sm, pages, lambda n, i, s: outcome[n], NOW, rate, self.x.seed, self.u,
                                         CRAWL, TIME)
        self.u += n_dec
        for g, (w, _) in zip(spans_g, processed):
            assert g["status"] == w["status"]
            if w["status"] in (rw.RETIRED, rw.DEFERRED):
                continue
            assert {key: g[key] for key in w} == w
        assert len(spans_g) == len(processed)
        hits = {rw.SOURCE_TYPES[s]: [stats_g["hits"][s], stats_g["misses"][s]] for s in range(4)}
        assert {t: c for t, c in hits.items() if c != [0, 0]} == stats
        assert stmts_g == rw.statements(processed, k)
        assert self.sets() == self.want_sets()
        return [c for c, _ in outcome.values()]


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("mode", range(len(RUN_MODES)))
def test_bulk_results_match_the_restatement(mode, k):
    sq = RwSequence(10 + mode, n_owners=8)
    sq.seed_sets(NAMES[:20])
    r = sq.rnd
    seen = set()
    for step in range(6):
        owners = r.sample(list(sq.go.page_map), r.randint(1, 8))
        spans, status, links = sq.result(owners, RUN_MODES[mode], overlap=step % 2 == 1)
        rate = r.choice([-5, 0, 30, 100])
        codes = sq.step(spans, status, links, k, rate)
        seen.update(codes)
        sq.e.release(0)
    assert {rw.FOUND, rw.NOT_FOUND} <= seen


@pytest.mark.parametrize("k", KS)
def test_retire_in_the_middle_of_a_span(k):
    sq = RwSequence(40, n_owners=6)
    sq.seed_sets(NAMES[:12])
    r = sq.rnd
    done = 0
    for _ in range(12):
        owners = r.sample(list(sq.go.page_map), 6)
        spans, status, links = sq.result(owners, RUN, sizes=[9] * 6)
        n = len(sq.e.state_rw_lookups(0, spans, NOW)["lookups"])
        if n >= 3:
            sq.step(spans, status, links, k, 40, retire_at=n // 2)
            done += 1
        sq.e.release(0)
    assert done


def link_heavy(sq, n_spans, names, per_record, n_records=2):
    """a result of n_spans pages of n_records records, each with per_record distinct t.me links from `names`"""
    from helpers import msg
    from distributed_crawler_b200.pack import pack_telegram
    from test_gpu_state_discover import MIN_DATE, oracle, GOOD
    r = sq.rnd
    msgs = []
    for p in range(n_spans * n_records):
        text = " ".join("t.me/" + nm.decode() for nm in r.sample(names, per_record))
        msgs.append(msg("messageText", "p %d %s" % (p, text), id=(p + 1) << 20, chat_id=-100777, channel=0,
                        date=MIN_DATE + 5))
    b = pack_telegram(msgs, CHANNELS)
    ro = oracle(GOOD).telegram(b, RUN)
    sq.e.set_clock(*GOOD)
    sq.e.telegram_submit(0, b, RUN)
    sq.e.telegram_wait(0)
    status = [int(s) for s in ro.status]
    links = [[(nm, abi.SRC_NAMES.index(s)) for nm, s in ro.record_links(i)] for i in range(ro.n)]
    return status, links


@pytest.mark.parametrize("n_spans", [1000, 100_000])
def test_many_spans(n_spans):
    sq = RwSequence(50, n_owners=16)
    names = [b"name%05d" % i for i in range(3 * n_spans // 4 + 10)]
    sq.seed_sets(names[:200])
    status, links = link_heavy(sq, n_spans, names, 6)
    rows = list(sq.e._st_rows().values())
    spans = [(rows[p % len(rows)], 2 * p, 2, 2) for p in range(n_spans)]
    sq.step(spans, status, links, rw.MAX_ROWS, 35)
    sq.e.release(0)


def test_refused_calls_leave_everything_unchanged():
    sq = RwSequence(60, n_owners=6)
    sq.seed_sets(NAMES[:12])
    owners = list(sq.go.page_map)
    spans, status, links = sq.result(owners, RUN, sizes=[9] * 6)
    refused(lambda: sq.e.state_rw_step([], 10, CRAWL), -6)  # no lookups yet
    got = sq.e.state_rw_lookups(0, spans, NOW)
    n = len(got["lookups"])
    before = sq.sets()
    bad = [(rw.FOUND, 1)] * n
    refused(lambda: sq.e.state_rw_step(bad[:-1] if n else [(0, 0)], 10, CRAWL), -1)  # wrong count
    if n:
        refused(lambda: sq.e.state_rw_step([(7, 0)] + bad[1:], 10, CRAWL), -1)  # unknown code
    refused(lambda: sq.e.state_rw_step(bad, 10, CRAWL, rows_per_stmt=0), -1)
    refused(lambda: sq.e.state_rw_step(bad, 10, CRAWL, now=(NOW, 1_000_000_000)), -1)
    refused(lambda: sq.e.state_rw_step(bad, 10, CRAWL, now=(300_000_000_000, 0)), -1)  # year past 9999
    assert sq.sets() == before
    sq.step(spans, status, links, 1, 50)  # the lists are still live, and the counter where it was
    refused(lambda: sq.e.state_rw_step(bad, 10, CRAWL), -6)  # spent by the accepted step
    sq.e.state_rw_lookups(0, spans, NOW)
    refused(lambda: sq.e.state_edge_sql(CRAWL), -6)  # no tandem hand-off: the lookups ended it
    sq.e.state_pending_edges(0, spans, NOW)
    refused(lambda: sq.e.state_rw_step(bad, 10, CRAWL), -6)  # another state call ended the lists
    sq.e.release(0)
