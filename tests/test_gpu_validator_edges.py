"""GPU tests: the validator edge pass (tgi_state_validator_lookups, tgi_state_validator_edges) against
tests/validator_edge_rules.py — the lookup rows and their occurrence lists, every edge's status, reason, kind and count,
the counter out and its crossing, every statement byte for byte at 1, 3 and 8191 rows per statement, and the invalid and
seed sets afterwards — over claims of 10, 10^3 and 10^5 edges (the last past one grid pass), names of 1 and 32 bytes
and names that need JSON escapes, the TTL boundary, refused calls that leave the sets and the plan as they were, and the
plan's life across other state calls."""
import random

import numpy as np
import pytest

import validator_edge_rules as ve
from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import Engine, EngineError, names_to_keys32

pytestmark = pytest.mark.gpu
NOW = 1_760_000_000
KS = (1, 3, ve.MAX_ROWS)
ESCAPES = [b'q"uote', b"back\\slash", b"<tag>&amp", b"tab\tnl\n", b"\xe2\x80\xa8ls", b"caf\xc3\xa9", b"\x01ctl", b"x",
           b"y" * 32, b"z" * 31 + b"\xff"]


def refused(call, code):
    with pytest.raises(EngineError) as ei:
        call()
    assert ei.value.code == code


def names_for(r: random.Random, n: int) -> list:
    return ESCAPES + [b"ch_%d_%s" % (q, b"a" * r.randint(0, 20)) for q in range(n)]


def world_for(r: random.Random, names: list) -> ve.World:
    inv = {nm: r.choice([0, NOW - 5, NOW - ve.TTL, NOW - ve.TTL + 1, NOW - 2 * ve.TTL])
           for nm in r.sample(names, len(names) // 5)}
    answers = [(ve.VALID, 0), (ve.NOT_CHANNEL, 1), (ve.INVALID, 2), (ve.INVALID, 1), (ve.OTHER, 0), (ve.TRANSIENT, 0),
               (ve.BLOCKED, 0), (ve.BLOCKED, 0), (ve.BLOCKED, 0)]
    script = {nm: [r.choice(answers) for _ in range(r.randint(0, 5))] for nm in names}
    return ve.World(inv, r.sample(names, 4), r.sample(names, len(names) // 6), r.sample(names, len(names) // 6), script)


def claim_for(r: random.Random, names: list, n: int, pid0: int = 1) -> list:
    hot = r.sample(names, max(1, len(names) // 8))
    pids = r.sample(range(-(1 << 40), 1 << 40), n)
    return [{"pending_id": pids[j] if pid0 is None else pid0 + j,
             "destination": r.choice(hot if r.random() < 0.5 else names),
             "crawl_id": r.choice([b"crawl-1", b"crawl-\xe2\x80\xa8"]), "source_type": r.choice([b"mention", b""])}
            for j in range(n)]


def seed_engine(e: Engine, w: ve.World):
    if w.invalid:
        e.set_add(abi.SET_INVALID, names_to_keys32(list(w.invalid)), np.array(list(w.invalid.values()), np.int64))
    if w.seeds:
        e.set_add(abi.SET_SEEDS, names_to_keys32(w.seeds))


def engine_sets(e: Engine):
    keys, stamps = e.set_export(abi.SET_INVALID)
    inv = {bytes(k).rstrip(b"\0"): int(t) for k, t in zip(keys, stamps)}
    seeds = [bytes(k).rstrip(b"\0") for k in e.set_export(abi.SET_SEEDS)[0]]
    return inv, seeds


def check_lookups(got: dict, want: list):
    rows = [(bytes(x["name"][:x["name_len"]]), int(x["occ_off"]), int(x["m"])) for x in got["lookups"]]
    occ = got["occurrences"].tolist()
    assert [(nm, occ[o:o + m]) for nm, o, m in rows] == want
    assert sum(m for _, _, m in rows) == len(occ)


def one_pass(e: Engine, w: ve.World, edges: list, count: int, k: int, now: int = NOW):
    """one lookups call and one edge pass on the engine against the per-edge loop on a copy of the world; the world
    afterwards is the loop's"""
    got = e.state_validator_lookups(edges, now)
    rows = ve.lookups(w, edges, now)
    check_lookups(got, rows)
    assert got["n_cached"] == len(edges) - sum(len(o) for _, o in rows)
    return apply_pass(e, w, edges, count, k, now)


def apply_pass(e: Engine, w: ve.World, edges: list, count: int, k: int, now: int = NOW):
    """the edge pass of a plan made for `edges`, as one_pass checks it"""
    ref = w.copy()
    want_res, want_count, want_crossed, calls = ve.run_claim(ref, edges, now, count)
    outcomes, attempts = ve.shim(w, edges, ve.lookups(w, edges, now))
    res, counter, stmts = e.state_validator_edges(outcomes, attempts, count, now, k)
    assert [(x["status"], x["reason"], x["kind"], x["blocked_count"]) for x in res] == want_res
    assert counter == {"out": want_count, "crossed_at": want_crossed}
    assert stmts == ve.statements(calls, k)
    inv, seeds = engine_sets(e)
    assert inv == ref.invalid and seeds == ref.seeds
    w.__dict__.update(ref.__dict__)
    return want_count, want_crossed


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("n", (10, 1000, 100_000))
def test_claims_match_the_per_edge_loop(n, k):
    r = random.Random(n + k)
    names = names_for(r, max(8, n // 4))
    w = world_for(r, names)
    e = Engine()
    try:
        seed_engine(e, w)
        count = r.choice([0, 2, 4])
        for c in range(2 if n < 100_000 else 1):
            edges = claim_for(r, names, n, None)
            count, crossed = one_pass(e, w, edges, count, k, NOW + 7 * c)
            if crossed is not None:
                count = 0
    finally:
        e.close()


def test_crossing_mid_claim_and_across_claims():
    names = [b"b%d" % q for q in range(12)]
    w = ve.World(script={nm: [(ve.BLOCKED, 0)] * 2 for nm in names})
    e = Engine()
    try:
        count, crossed = one_pass(e, w, [{"pending_id": j, "destination": names[j]} for j in range(3)], 0, 1)
        assert (count, crossed) == (3, None)
        edges = [{"pending_id": 10 + j, "destination": names[3 + j]} for j in range(4)]
        assert one_pass(e, w, edges, count, 3) == (7, 1)
        # a transient and a definitive answer between blocked ones
        w.script.update({b"t": [(ve.TRANSIENT, 0)], b"v": [(ve.VALID, 0)]})
        edges = [{"pending_id": 20 + j, "destination": nm} for j, nm in enumerate([names[7], b"t", names[8], b"v", names[9]])]
        assert one_pass(e, w, edges, 4, ve.MAX_ROWS) == (1, 0)
    finally:
        e.close()


def test_ttl_boundary_and_name_lengths():
    e = Engine()
    try:
        w = ve.World({b"a": NOW - ve.TTL, b"b": NOW - ve.TTL + 1, b"c": 0, b"d" * 32: NOW - ve.TTL - 1},
                     script={b"a": [(ve.NOT_CHANNEL, 1)], b"d" * 32: [(ve.VALID, 0)], b"e": [(ve.INVALID, 2)]})
        seed_engine(e, w)
        edges = [{"pending_id": j, "destination": nm} for j, nm in enumerate([b"a", b"b", b"c", b"d" * 32, b"e", b"a"])]
        assert ve.lookups(w, edges, NOW) == [(b"a", [0, 5]), (b"d" * 32, [3]), (b"e", [4])]  # now - 30 d is expired
        one_pass(e, w, edges, 0, 1)
        assert w.invalid[b"a"] == NOW and w.seeds == [b"d" * 32]
    finally:
        e.close()


def test_refused_calls_leave_the_sets_and_the_plan():
    r = random.Random(5)
    names = names_for(r, 20)
    w = world_for(r, names)
    e = Engine()
    try:
        seed_engine(e, w)
        refused(lambda: e.state_validator_edges([], []), abi.E_STATE)  # no plan
        edges = claim_for(r, names, 40)
        got = e.state_validator_lookups(edges, NOW)
        before = engine_sets(e)
        bad_claims = [
            edges + [dict(edges[0])],                                                   # a pending_id twice
            edges + [{"pending_id": -1, "destination": b""}],                           # an empty name
            edges + [{"pending_id": -1, "destination": b"x" * 33}],                     # 33 bytes
        ]
        for bad in bad_claims:
            refused(lambda: e.state_validator_lookups(bad, NOW), abi.E_ARG)
        from distributed_crawler_b200.state_pack import pack_claimed_edges
        recs, blob = pack_claimed_edges(edges)
        recs[3]["str_off"][2], recs[3]["str_len"][2] = len(blob), 1  # a string past the blob
        refused(lambda: e.state_validator_lookups((recs, blob), NOW), abi.E_ARG)
        rows = [(bytes(x["name"][:x["name_len"]]), got["occurrences"][int(x["occ_off"]):int(x["occ_off"]) + int(x["m"])].tolist())
                for x in got["lookups"]]
        assert rows == ve.lookups(w, edges, NOW)
        multi = next(q for q, (_, o) in enumerate(rows) if len(o) > 1)
        single = next(q for q, (_, o) in enumerate(rows) if len(o) == 1)
        ok_o = [(0, 0, 1)] * len(rows)
        ok_a = [(ve.INVALID, 2)] * len(rows)

        def with_row(q, o, att):  # the rows' outcomes with row q's replaced
            oo, aa = list(ok_o), []
            oo[q] = o
            for p in range(len(rows)):
                aa += att if p == q else [ok_a[p]]
            return oo, aa

        bad_passes = [
            (ok_o[:-1], ok_a[:-1], 0, 1),                                             # n other than the lookups
            (ok_o, ok_a + [(ve.VALID, 0)], 0, 1),                                     # attempts' total
            (ok_o, ok_a, 0, 0), (ok_o, ok_a, 0, ve.MAX_ROWS + 1),                      # k
            (ok_o, ok_a, -1, 1),                                                      # a negative count
            (*with_row(multi, (1, 0, 1), [(ve.VALID, 0)]), 0, 1),                     # discovered with attempts
            (*with_row(multi, (0, 0, 0), []), 0, 1),                                  # no attempt
            (*with_row(single, (0, 0, 2), [(ve.TRANSIENT, 0)] * 2), 0, 1),            # more than m
            (*with_row(multi, (0, 0, 2), [(ve.VALID, 0), (ve.BLOCKED, 0)]), 0, 1),    # a final attempt before the last
            (*with_row(multi, (0, 0, 1), [(ve.TRANSIENT, 0)]), 0, 1),                 # not final, fewer than m
            (*with_row(multi, (0, 1, 1), [(ve.INVALID, 1)]), 0, 1),                   # claimed without VALID
            (*with_row(multi, (2, 0, 0), []), 0, 1),                                  # unknown codes
            (*with_row(multi, (0, 0, 1), [(6, 0)]), 0, 1),
            (*with_row(multi, (0, 0, 1), [(ve.INVALID, 3)]), 0, 1),
        ]
        for o, a, cnt, k in bad_passes:
            refused(lambda: e.state_validator_edges(o, a, cnt, NOW, k), abi.E_ARG)
        assert engine_sets(e) == before
        # the plan is still the first lookups': a valid pass applies it
        outcomes, attempts = ve.shim(w.copy(), edges, rows)
        e.state_validator_edges(outcomes, attempts, 0, NOW, 1)
        refused(lambda: e.state_validator_edges(outcomes, attempts, 0, NOW, 1), abi.E_STATE)  # an accepted pass ends it
    finally:
        e.close()


def test_plan_outlives_other_state_calls_and_a_second_lookups_replaces_it():
    r = random.Random(9)
    names = names_for(r, 30)
    w = world_for(r, names)
    e = Engine()
    try:
        seed_engine(e, w)
        e.state_id_seed(77)
        first = claim_for(r, names, 25)
        e.state_validator_lookups(first, NOW)
        batch = {"batch_id": b"b-1", "crawl_id": b"crawl-1", "source_channel": b"src", "source_page_id": b"p-1",
                 "sequence_id": b"seq-1", "source_depth": 2, "edges": [(b"dest", b"mention", b"valid")]}
        e.state_validator_walkback([batch], 100, b"crawl-1", (NOW, 0), 1)  # the walkback processor, beside the HTTP phase
        apply_pass(e, w, first, 0, 3)  # the plan outlived the walkback call
        e.state_validator_lookups(first, NOW)
        second = claim_for(r, names, 12, 500)
        one_pass(e, w, second, 0, 1)  # the second lookups replaced the first
    finally:
        e.close()


def test_empty_claim():
    e = Engine()
    try:
        got = e.state_validator_lookups([], NOW)
        assert len(got["lookups"]) == 0 and e.state_ve_lookups_launches == 0
        res, counter, stmts = e.state_validator_edges([], [], 3, NOW, 1)
        assert (res, counter, stmts, e.state_ve_launches) == ([], {"out": 3, "crossed_at": None}, [], 0)
    finally:
        e.close()
