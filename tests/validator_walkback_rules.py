"""A literal Python restatement of the validator pod's walkback processor (crawl/validator.go:360-489):
processWalkbackBatch's decision, pickWalkbackChannel with the batch's valid channels excluded (crawl/runner.go:120-139),
and the binding calls it makes, each sent by ExecuteDatabaseOperation (state/daprstate.go:3643-3678) as an `exec`
InvokeBinding: AddPageToPageBuffer (:3619-3641), SaveEdgeRecords of the primary and skipped edges (:3150-3204),
CompletePendingBatch and FlushBatchStats' upserts and delete (:4124-4174).  The expected output of
tgi_state_validator_walkback.

A batch is a dict with PendingEdgeBatch's strings ("batch_id", "crawl_id", "source_channel", "source_page_id",
"sequence_id", bytes), "source_depth" and "edges" = [(destination, source_type, validation_status)] as ClaimWalkbackBatch
returns them (:4016-4122).

Three things are fixed where Go is random.  The v-th batch draws rand.IntN(100), the forward index and the walkback's
Random() indices, in that order, with Lemire's multiply-and-reject from one stream of Philox4x32-10 blocks
(v_lo, v_hi, 5, j); uuid.New() becomes the page-id construction with counter word 2 = 6 (the page's ID) and 7 (a
walkback's new SequenceID); FlushBatchStats ranges over a map, whose order Go leaves random, and the library takes the
types' first-occurrence order.  time.Now() is read once per call."""
from __future__ import annotations

import tandem_sql_rules as sr
import walkback_rules as wr
from discover_rules import MASK, philox4x32_10

PAGE_BUFFER_INSERT, EDGE_RECORD_INSERT = wr.PAGE_BUFFER_INSERT, wr.EDGE_RECORD_INSERT
BATCH_COMPLETE, STATS_UPSERT, EDGES_DELETE = 5, 6, 7
KINDS = (PAGE_BUFFER_INSERT, EDGE_RECORD_INSERT, BATCH_COMPLETE, STATS_UPSERT, EDGES_DELETE)
WALK_OK, WALK_EXHAUSTED, WALK_EMPTY = wr.WALK_OK, wr.WALK_EXHAUSTED, wr.WALK_EMPTY
MAX_ROWS = wr.MAX_ROWS

# the three more literals, byte for byte (daprstate.go:4126, 4163, 4170)
COMPLETE_SQL = b"UPDATE pending_edge_batches SET status = 'completed', completed_at = NOW() WHERE batch_id = $1;"
UPSERT_SQL = (b"INSERT INTO source_type_stats (crawl_id, source_type, total, valid, not_channel, invalid, duplicate) "
              b"VALUES ($1, $2, $3, $4, $5, $6, $7) ON CONFLICT (crawl_id, source_type) DO UPDATE SET total = "
              b"source_type_stats.total + EXCLUDED.total, valid = source_type_stats.valid + EXCLUDED.valid, "
              b"not_channel = source_type_stats.not_channel + EXCLUDED.not_channel, invalid = "
              b"source_type_stats.invalid + EXCLUDED.invalid, duplicate = source_type_stats.duplicate + "
              b"EXCLUDED.duplicate;")
DELETE_SQL = b"DELETE FROM pending_edges WHERE batch_id = $1;"


# ---- the library's randomness ---------------------------------------------------------------------------------------
def words(seed: int, v: int):
    """the draw stream of the v-th claimed batch: block j = Philox (v_lo, v_hi, 5, j) gives x0 | x1 << 32, then
    x2 | x3 << 32"""
    j = 0
    while True:
        x = philox4x32_10([v & MASK, v >> 32, 5, j], [seed & MASK, seed >> 32])
        yield x[0] | x[1] << 32
        yield x[2] | x[3] << 32
        j += 1


# ---- the reference ----------------------------------------------------------------------------------------------------
def pick_walkback_channel(keys: list, source_url: bytes, exclude: set, draw):
    """pickWalkbackChannel(sm, sourceURL, exclude) (runner.go:120-139): (status, url, draws).  An empty set is Random()'s
    error, returned on the first attempt; a draw equal to sourceURL or in exclude (byte for byte) is retried, and the
    10th such draw is ErrWalkbackExhausted"""
    for attempt in range(wr.MAX_ATTEMPTS):
        if not keys:
            return WALK_EMPTY, b"", 0
        url = draw()
        if url == source_url or url in exclude:
            if attempt == wr.MAX_ATTEMPTS - 1:
                return WALK_EXHAUSTED, b"", attempt + 1
            continue
        return WALK_OK, url, attempt + 1
    return WALK_EXHAUSTED, b"", wr.MAX_ATTEMPTS


def stats(edges) -> list:
    """FlushBatchStats' aggregation (daprstate.go:4137-4160): [(source_type, [total, valid, not_channel, invalid,
    duplicate])] in the types' first-occurrence order, empty as "unknown"; any other status counts in total only"""
    agg = {}
    for _, st, status in edges:
        c = agg.setdefault(st or b"unknown", [0] * 5)
        c[0] += 1
        for f, name in enumerate((b"valid", b"not_channel", b"invalid", b"duplicate")):
            c[1 + f] += status == name
    return list(agg.items())


def process(batch: dict, keys: list, rate: int, seed: int, v: int, crawl_id: bytes, time):
    """processWalkbackBatch (validator.go:360-489) of the v-th claimed batch under the library's randomness: its result
    {"status", "walkback", "rnd", "draws", "n_valid", "forward_edge", "url", "page_id", "sequence_id"} and its calls in
    the reference's order, (kind, sql, params): none when the pick fails (the function returns its error first)"""
    edges = batch.get("edges", [])
    valid = [(q, d) for q, (d, _, status) in enumerate(edges) if status == b"valid"]
    stream = words(seed, v)
    walkback, rnd = not valid, -1
    if valid:
        rnd = wr.lemire(100, stream) + 1
        walkback = rate >= rnd
    res = {"status": WALK_OK, "walkback": walkback, "rnd": rnd, "draws": 0, "n_valid": len(valid),
           "forward_edge": None, "url": b"", "page_id": wr.uuid(seed, v, 6), "sequence_id": wr.uuid(seed, v, 7)}
    skipped = [d for _, d in valid]
    if walkback:
        status, url, draws = pick_walkback_channel(keys, batch.get("source_channel", b""), set(skipped),
                                                   lambda: keys[wr.lemire(len(keys), stream)])
        res.update(status=status, url=url, draws=draws)
        if status != WALK_OK:
            return res, []
        page_seq = res["sequence_id"]
    else:
        idx = wr.lemire(len(valid), stream)
        res["forward_edge"], url = valid[idx]
        del skipped[idx]
        page_seq = batch.get("sequence_id", b"")
    b = lambda name: batch.get(name, b"")  # noqa: E731
    crawl = b("crawl_id") or crawl_id
    page = [res["page_id"], b("source_page_id"), wr.go_int(batch.get("source_depth", 0) + 1), url, crawl, page_seq]
    recs = [[url, b("source_channel"), walkback, False, time, crawl, b("sequence_id")]]
    recs += [[ch, b("source_channel"), False, True, time, crawl, b("sequence_id")] for ch in skipped]
    calls = [(PAGE_BUFFER_INSERT, wr.PAGE_BUFFER_SQL, wr.marshal(page))]
    calls += [(EDGE_RECORD_INSERT, wr.EDGE_RECORD_SQL, wr.marshal(r)) for r in recs]
    calls.append((BATCH_COMPLETE, COMPLETE_SQL, wr.marshal([b("batch_id")])))
    calls += [(STATS_UPSERT, UPSERT_SQL, wr.marshal([b("crawl_id"), st] + c)) for st, c in stats(edges)]
    calls.append((EDGES_DELETE, DELETE_SQL, wr.marshal([b("batch_id")])))
    return res, calls


def run(batches, keys: list, rate: int, seed: int, v0: int, crawl_id: bytes, time):
    """every batch in input order, the i-th as the (v0 + i)-th: [(result, calls)]"""
    return [process(b, keys, rate, seed, v0 + i, crawl_id, time) for i, b in enumerate(batches)]


# ---- the library's grouping -------------------------------------------------------------------------------------------
def sql_text(kind: int, rows: int) -> bytes:
    """the text of a statement of `rows` rows: the literal for one row, else the VALUES tuple repeated with the
    placeholders numbered on, or WHERE batch_id IN (...); an upsert always has one row"""
    if kind in (PAGE_BUFFER_INSERT, EDGE_RECORD_INSERT):
        return wr.sql_text(kind, rows)
    lit = {BATCH_COMPLETE: COMPLETE_SQL, STATS_UPSERT: UPSERT_SQL, EDGES_DELETE: DELETE_SQL}[kind]
    if rows == 1:
        return lit
    assert kind != STATS_UPSERT
    return lit[:-len(b"= $1;")] + b"IN (" + b", ".join(b"$%d" % (p + 1) for p in range(rows)) + b");"


def statements(processed, k: int) -> list:
    """tgi_state_validator_walkback's statements, [(kind, rows, sql, params)], from run()'s output: each kind's one-row
    calls in batch order, kinds in KINDS order, cut into statements of k rows (the upserts of one row each), params
    the rows' values as one JSON array"""
    out = []
    for kind in KINDS:
        rows = [p for _, calls in processed for kd, _, p in calls if kd == kind]
        kk = 1 if kind == STATS_UPSERT else k
        for a in range(0, len(rows), kk):
            part = rows[a:a + kk]
            out.append((kind, len(part), sql_text(kind, len(part)), b"[" + b",".join(p[1:-1] for p in part) + b"]"))
    return out


def split_values(params: bytes) -> list:
    return sr.split_values(params)
