"""A literal Python restatement of the Postgres binding calls that store a tandem hand-off: CreatePendingBatch,
InsertPendingEdge and ClosePendingBatch (state/daprstate.go:3896-3941), each sent by ExecuteDatabaseOperation
(:3643-3678) as an `exec` InvokeBinding with metadata {"sql": the literal, "params": string(json.Marshal(params))}.
The rows are tandem_rules.Tandem.page's, the values those of crawl/runner.go:1276-1300.  The expected output of
tgi_state_edge_sql.

The reference makes one call per row, page by page (create, the edges, close).  The library returns the same calls
grouped by kind (every create, every edge, every close) and, with rows_per_stmt = k > 1, k rows per statement: the
VALUES tuple repeated with the placeholders numbered on, the close as WHERE batch_id IN (...), and params the k rows'
values as one array.  time.Now() is read once per call (the reference reads it per edge)."""
from __future__ import annotations

from go_rules import _go_time_checked, _marshal, _Raw
from zone_oracle import go_json_time, go_offset

BATCH_INSERT, EDGE_INSERT, BATCH_CLOSE = 0, 1, 2
MAX_ROWS = 8191  # 8 bind parameters per edge row, at most 65535 per Postgres statement
SOURCE_TYPES = [b"mention", b"text_url", b"url", b"plaintext"]  # TGI_SRC_* (tdutils.go:978-987)

# the three literals, byte for byte (daprstate.go:3897, 3915, 3935)
CREATE_SQL = (b"INSERT INTO pending_edge_batches (batch_id, crawl_id, source_channel, source_page_id, source_depth, "
              b"sequence_id, status) VALUES ($1, $2, $3, $4, $5, $6, $7);")
INSERT_SQL = (b"INSERT INTO pending_edges (batch_id, crawl_id, destination_channel, source_channel, sequence_id, "
              b"discovery_time, source_type, validation_status) VALUES ($1, $2, $3, $4, $5, $6, $7, $8);")
CLOSE_SQL = b"UPDATE pending_edge_batches SET status = 'closed', closed_at = NOW() WHERE batch_id = $1;"
PER_ROW = {BATCH_INSERT: 7, EDGE_INSERT: 8, BATCH_CLOSE: 1}


def discovery_time(sec: int, nsec: int, zone=None, tz: int = 0):
    """json.Marshal(time.Now()) in time.Local: the zone table (tgi_set_zone) or the fixed tz_offset_sec; None where
    json.Marshal fails (a local year outside [0, 9999])"""
    if zone is not None:
        t = go_json_time(sec, nsec, go_offset(zone, sec))
        return _Raw(t) if t else None
    return _go_time_checked(sec, nsec, tz)


def batch_values(batch: dict, crawl_id: bytes) -> list:
    """CreatePendingBatch's []any (daprstate.go:3898-3906) of runner.go:1276-1284's batch"""
    return [batch["batch_id"], crawl_id, batch["source_channel"], batch["source_page_id"], batch["source_depth"],
            batch["sequence_id"], "open"]


def edge_values(batch: dict, edge: dict, crawl_id: bytes, time) -> list:
    """InsertPendingEdge's []any (:3916-3925) of runner.go:1293-1302's edge: "pending" is the function's literal, so a
    duplicate edge writes it too"""
    return [batch["batch_id"], crawl_id, edge["destination"], batch["source_channel"], batch["sequence_id"], time,
            SOURCE_TYPES[edge["source_type"]], "pending"]


def close_values(batch: dict) -> list:
    """ClosePendingBatch's []any{batchID} (:3935-3936)"""
    return [batch["batch_id"]]


def marshal(values: list) -> bytes:
    """ExecuteDatabaseOperation's json.Marshal(params) of a []any (:3647)"""
    return _marshal(values)


def reference_calls(pages, crawl_id: bytes, time) -> list:
    """the reference's calls in its order, (kind, sql, params): per page with a batch, the create, every edge, the
    close (runner.go:1286, 1303, 1418).  pages = [(batch, edges)] of Tandem.page, batch not None"""
    out = []
    for batch, edges in pages:
        out.append((BATCH_INSERT, CREATE_SQL, marshal(batch_values(batch, crawl_id))))
        out += [(EDGE_INSERT, INSERT_SQL, marshal(edge_values(batch, e, crawl_id, time))) for e in edges]
        out.append((BATCH_CLOSE, CLOSE_SQL, marshal(close_values(batch))))
    return out


def sql_text(kind: int, rows: int) -> bytes:
    """the text of a statement of `rows` rows: the literal for one row, else the tuple repeated / the IN list"""
    if rows == 1:
        return (CREATE_SQL, INSERT_SQL, CLOSE_SQL)[kind]
    if kind == BATCH_CLOSE:
        return CLOSE_SQL[:-len(b"= $1;")] + b"IN (" + b", ".join(b"$%d" % (p + 1) for p in range(rows)) + b");"
    head = (CREATE_SQL, INSERT_SQL)[kind].split(b" VALUES ")[0] + b" VALUES "
    n = PER_ROW[kind]
    return head + b", ".join(b"(" + b", ".join(b"$%d" % (r * n + p + 1) for p in range(n)) + b")"
                             for r in range(rows)) + b";"


def statements(pages, crawl_id: bytes, time, k: int) -> list:
    """tgi_state_edge_sql's output, [(kind, rows, sql, params)]: every create, every edge, every close, each kind cut
    into statements of k rows (the last may hold fewer), params the rows' values as one JSON array"""
    rows = {BATCH_INSERT: [batch_values(b, crawl_id) for b, _ in pages],
            EDGE_INSERT: [edge_values(b, e, crawl_id, time) for b, es in pages for e in es],
            BATCH_CLOSE: [close_values(b) for b, _ in pages]}
    out = []
    for kind in (BATCH_INSERT, EDGE_INSERT, BATCH_CLOSE):
        r = rows[kind]
        for a in range(0, len(r), k):
            part = r[a:a + k]
            out.append((kind, len(part), sql_text(kind, len(part)), marshal([v for row in part for v in row])))
    return out


def split_values(params: bytes) -> list:
    """the top-level values of a JSON array, as bytes (a string's escapes kept as they are)"""
    assert params[:1] == b"[" and params[-1:] == b"]"
    out, depth, in_str, esc, start = [], 0, False, False, 1
    for i in range(1, len(params) - 1):
        c = params[i]
        if in_str:
            if esc:
                esc = False
            elif c == 0x5C:
                esc = True
            elif c == 0x22:
                in_str = False
        elif c == 0x22:
            in_str = True
        elif c in b"[{":
            depth += 1
        elif c in b"]}":
            depth -= 1
        elif c == 0x2C and depth == 0:
            out.append(params[start:i])
            start = i + 1
    if len(params) > 2:
        out.append(params[start:-1])
    return out
