"""CPU tests: tests/validator_edge_rules.py against the reference's own validator tests (tests/golden/
validator_edge_vectors.json), and the grouped loop (lookups, the shim, apply) against the per-edge loop on seeded worlds
with repeated names, unknown statuses, runs of transient and blocked attempts, lost claim races and threshold crossings
in the middle of a claim and across claims."""
import json
import os
import random

import pytest

import validator_edge_rules as ve

HERE = os.path.dirname(os.path.abspath(__file__))
KIND_OF = {"valid": ve.VALID, "not_channel": ve.NOT_CHANNEL, "invalid": ve.INVALID, "transient": ve.TRANSIENT,
           "blocked": ve.BLOCKED}
OUTCOME_KINDS = ("definitive", "transient", "blocked")
NOW = 1_760_000_000


@pytest.fixture(scope="module")
def vectors():
    with open(os.path.join(HERE, "golden", "validator_edge_vectors.json"), encoding="utf-8") as f:
        return json.load(f)


def world_of(w: dict) -> ve.World:
    script = {k.encode(): [(KIND_OF[s], ve.REASONS.index(r.encode())) for s, r in v] for k, v in w.get("script", {}).items()}
    return ve.World({k.encode(): 0 for k in w.get("invalid", ())}, (), [k.encode() for k in w.get("discovered", ())],
                    [k.encode() for k in w.get("raced", ())], script)


def edge_of(e) -> dict:
    return {"pending_id": e[0], "destination": e[1].encode(), "crawl_id": e[2].encode()}


def test_single_edge_vectors(vectors):
    for v in vectors["single_edge"]:
        w = world_of(v["world"])
        name = v["edge"][1].encode()
        st, rs, kd, calls = ve.validate_single_edge(w, edge_of(v["edge"]), NOW)
        ex = v["expect"]
        assert (ve.STATUSES[st], ve.REASONS[rs], OUTCOME_KINDS[kd]) == \
            (ex["status"].encode(), ex["reason"].encode(), ex["kind"]), v["name"]
        want = []
        for c in ex["calls"]:
            if c[0] == "UpsertSeedChannelChatID":
                want.append((ve.SEED_UPSERT, ve.marshal([c[1].encode(), c[2]])))
                assert name in w.seeds
            elif c[0] == "MarkChannelInvalid":
                want.append((ve.INVALID_UPSERT, ve.marshal([c[1].encode(), c[2].encode()])))
                assert w.invalid[name] == NOW
            else:  # ClaimDiscoveredChannel: a query, not an exec call; it leaves the name in discovered_channels
                assert name in w.db
        assert calls == want, v["name"]


def test_blocked_state_vectors(vectors):
    for v in vectors["blocked_state"]:
        w, count = world_of(v["world"]), 0
        for claim, ex in zip(v["claims"], v["expect"]):
            edges = [edge_of(e) for e in claim]
            results, count, crossed, calls = ve.run_claim(w, edges, NOW, count)
            updates = [[e["pending_id"], ve.STATUSES[r[0]].decode(), ve.REASONS[r[1]].decode()] for e, r in zip(edges, results)]
            assert updates == ex["updates"], v["name"]
            assert (crossed is not None) == ex["access_event"], v["name"]
            assert ((ve.ACCESS_EVENT, b'["ip_blocked"]') in calls) == ex["access_event"]
            if crossed is not None:  # blocked: the probe succeeds before the next claim (validator.go:113-125)
                count = 0


def test_literals_and_k_forms():
    assert ve.sql_text(ve.EDGE_UPDATE, 1) == ve.UPDATE_SQL
    assert ve.sql_text(ve.EDGE_UPDATE, 2) == (
        b"UPDATE pending_edges AS e SET validation_status = v.s, validation_reason = v.r, validated_at = NOW() FROM "
        b"(VALUES ($1, $2, $3::integer), ($4, $5, $6::integer)) AS v(s, r, id) WHERE e.pending_id = v.id;")
    assert ve.sql_text(ve.INVALID_UPSERT, 2).startswith(
        b"INSERT INTO invalid_channels (channel_username, reason, invalidated_at) VALUES ($1, $2, NOW()), ($3, $4, NOW()) ON")
    assert ve.marshal([b"pending", b"", 7]) == b'["pending","",7]'


def random_world(r: random.Random, names: list):
    inv = {nm: r.choice([0, NOW - 5, NOW - ve.TTL, NOW - ve.TTL + 1]) for nm in r.sample(names, len(names) // 5)}
    db = r.sample(names, len(names) // 6)
    raced = r.sample(names, len(names) // 6)
    answers = [(ve.VALID, 0), (ve.NOT_CHANNEL, 1), (ve.INVALID, 2), (ve.INVALID, 1), (ve.OTHER, 0), (ve.TRANSIENT, 0),
               (ve.BLOCKED, 0), (ve.BLOCKED, 0)]
    script = {nm: [r.choice(answers) for _ in range(r.randint(0, 6))] for nm in names}
    return ve.World(inv, r.sample(names, 3), db, raced, script)


def random_claim(r: random.Random, names: list, n: int, pid0: int):
    hot = r.sample(names, max(1, len(names) // 8))  # popular names recur
    return [{"pending_id": pid0 + j, "destination": r.choice(hot if r.random() < 0.5 else names),
             "crawl_id": r.choice([b"crawl-1", b"crawl-2"])} for j in range(n)]


def grouped(w: ve.World, edges: list, now: int, count: int):
    rows = ve.lookups(w, edges, now)
    outcomes, attempts = ve.shim(w, edges, rows)
    return ve.apply(w, edges, rows, outcomes, attempts, count, now)


@pytest.mark.parametrize("seed", range(12))
def test_grouped_loop_equals_the_per_edge_loop(seed):
    r = random.Random(seed)
    names = [b"ch%03d_%s" % (q, bytes([97 + q % 26])) for q in range(r.choice([4, 12, 60]))]
    a = random_world(r, names)
    b = a.copy()
    count_a = count_b = r.choice([0, 0, 3, 4])
    crossed_seen = 0
    for c in range(5):
        edges = random_claim(r, names, r.choice([1, 10, 10, 40]), 1000 * c)
        now = NOW + 60 * c
        ra, count_a, xa, calls_a = ve.run_claim(a, edges, now, count_a)
        rb, count_b, xb, calls_b = grouped(b, edges, now, count_b)
        assert rb == ra and count_b == count_a and xb == xa
        for k in (1, 3, ve.MAX_ROWS):
            assert ve.statements(calls_b, k) == ve.statements(calls_a, k)
        assert ve.statements(calls_a, 1) == sorted(ve.reference_statements(calls_a), key=lambda s: ve.KINDS.index(s[0]))
        assert (a.invalid, a.seeds, a.db) == (b.invalid, b.seeds, b.db)
        if xa is not None:  # the probe succeeds before the next claim
            count_a = count_b = 0
            crossed_seen += 1


def test_threshold_crossings_mid_claim_and_across_claims():
    names = [b"n%d" % q for q in range(12)]
    w = ve.World(script={nm: [(ve.BLOCKED, 0)] * 3 for nm in names})
    claim1 = [{"pending_id": j, "destination": names[j]} for j in range(3)]
    res, count, crossed, calls = grouped(w, claim1, NOW, 0)
    assert (count, crossed) == (3, None) and (ve.ACCESS_EVENT, b'["ip_blocked"]') not in calls
    claim2 = [{"pending_id": 10 + j, "destination": names[3 + j]} for j in range(6)]
    res, count, crossed, calls = grouped(w, claim2, NOW, count)  # 4, 5: crossed at the second edge, then 6, 7 ...
    assert crossed == 1 and count == 9 and [x[3] for x in res] == [4, 5, 6, 7, 8, 9]
    assert [c for c in calls if c[0] == ve.ACCESS_EVENT] == [(ve.ACCESS_EVENT, b'["ip_blocked"]')]
