"""A literal Python restatement of the forced walkback of a tandem step without edges (crawl/runner.go:1425-1455):
pickWalkbackChannel with exclude = nil (:115-139) over DiscoveredChannels.Random() (state/datamodels.go:152-162), the
page and edge it builds, and the two binding calls that store them, AddPageToPageBuffer (state/daprstate.go:3619-3641)
and SaveEdgeRecords of one record (:3150-3204), each sent by ExecuteDatabaseOperation (:3643-3678) as an `exec`
InvokeBinding with metadata {"sql": the literal, "params": string(json.Marshal(params))}.  The expected output of
tgi_state_walkback.

Two things are fixed where Go is random.  rand.Intn(len(keys)) becomes Lemire's multiply-and-reject over a stream of
64-bit words from Philox4x32-10 blocks (w_lo, w_hi, 2, j) under the page-id seed, w the number of edge-less spans
handled before; it is exactly uniform on [0, N) as rand.Intn is.  uuid.New() becomes page_id's construction with
counter word 2 = 3 (the page's ID) and 4 (its new SequenceID).  time.Now() is read once per call."""
from __future__ import annotations

from discover_rules import MASK, philox4x32_10
from go_rules import _marshal

PAGE_BUFFER_INSERT, EDGE_RECORD_INSERT = 3, 4
WALK_OK, WALK_EXHAUSTED, WALK_EMPTY = 0, 1, 2
MAX_ATTEMPTS = 10  # maxWalkbackAttempts (runner.go:118)
MAX_ROWS = 8191
U64 = (1 << 64) - 1

# the two literals, byte for byte (daprstate.go:3620, 3167)
PAGE_BUFFER_SQL = (b"INSERT INTO page_buffer (page_id, parent_id, depth, url, crawl_id, sequence_id) VALUES "
                   b"($1, $2, $3, $4, $5, $6);")
EDGE_RECORD_SQL = (b"INSERT INTO edge_records (destination_channel, source_channel, walkback, skipped, discovery_time, "
                   b"crawl_id, sequence_id) VALUES ($1, $2, $3, $4, $5, $6, $7);")
PER_ROW = {PAGE_BUFFER_INSERT: 6, EDGE_RECORD_INSERT: 7}


# ---- the library's randomness ---------------------------------------------------------------------------------------
def words(seed: int, w: int):
    """the draw stream of the w-th edge-less span: block j = Philox (w_lo, w_hi, 2, j) gives x0 | x1 << 32, then
    x2 | x3 << 32"""
    j = 0
    while True:
        x = philox4x32_10([w & MASK, w >> 32, 2, j], [seed & MASK, seed >> 32])
        yield x[0] | x[1] << 32
        yield x[2] | x[3] << 32
        j += 1


def lemire(n: int, stream, bits: int = 64) -> int:
    """an index in [0, n) from the 64-bit words of stream (Lemire, "Fast random integer generation in an interval",
    2019): m = x * n; while low64(m) < 2^64 mod n (tested only when low64(m) < n) take the next word; high64(m).
    bits < 64 is the same rule over narrower words, small enough to enumerate"""
    mask = (1 << bits) - 1
    x = next(stream)
    m = x * n
    if m & mask < n:
        t = ((1 << bits) - n) % n
        while m & mask < t:
            x = next(stream)
            m = x * n
    return m >> bits


def uuid(seed: int, n: int, domain: int) -> bytes:
    """id n of the seed in counter domain `domain` (word 2): discover_rules.page_id's construction"""
    w = philox4x32_10([n & MASK, n >> 32, domain, 0], [seed & MASK, seed >> 32])
    b = bytearray(b"".join(x.to_bytes(4, "little") for x in w))
    b[6] = b[6] & 0x0F | 0x40
    b[8] = b[8] & 0x3F | 0x80
    h = b.hex()
    return ("%s-%s-%s-%s-%s" % (h[:8], h[8:12], h[12:16], h[16:20], h[20:])).encode()


def library_draw(keys: list, seed: int, w: int):
    """GetRandomDiscoveredChannel as the library makes it for the w-th edge-less span: keys[index], index from the
    span's own stream"""
    stream = words(seed, w)
    return lambda: keys[lemire(len(keys), stream)]


# ---- the reference ----------------------------------------------------------------------------------------------------
def pick_walkback_channel(keys: list, source_url: bytes, draw):
    """pickWalkbackChannel(sm, sourceURL, nil) (runner.go:120-139): (status, url, draws).  An empty set is Random()'s
    error (datamodels.go:156-158), returned on the first attempt; a draw equal to sourceURL (byte for byte) is retried,
    and the 10th such draw is ErrWalkbackExhausted"""
    for attempt in range(MAX_ATTEMPTS):
        if not keys:
            return WALK_EMPTY, b"", 0
        url = draw()
        if url == source_url:
            if attempt == MAX_ATTEMPTS - 1:
                return WALK_EXHAUSTED, b"", attempt + 1
            continue
        return WALK_OK, url, attempt + 1
    return WALK_EXHAUSTED, b"", MAX_ATTEMPTS


def go_int(v: int) -> int:
    """Go's int (int64) arithmetic wraps"""
    return ((v + (1 << 63)) & U64) - (1 << 63)


def page_buffer_values(page_id: bytes, owner: dict, url: bytes, crawl_id: bytes, sequence_id: bytes) -> list:
    """AddPageToPageBuffer's []any (daprstate.go:3622-3633) of runner.go:1432-1439's page: the empty page.CrawlID falls
    back to the configured one"""
    return [page_id, owner["id"], go_int(owner.get("depth", 0) + 1), url, crawl_id, sequence_id]


def edge_record_values(owner: dict, url: bytes, crawl_id: bytes, time) -> list:
    """SaveEdgeRecords' []any (:3170-3184) of runner.go:1440-1447's edge: Walkback true, Skipped false, the empty
    record.CrawlID replaced by the configured one"""
    return [url, owner["url"], True, False, time, crawl_id, owner.get("sequenceId", b"")]


def marshal(values: list) -> bytes:
    """ExecuteDatabaseOperation's json.Marshal(params) of a []any (:3647)"""
    return _marshal(values)


def forced_walkback(owner: dict, keys: list, seed: int, w: int, crawl_id: bytes, time):
    """the branch for one page without edges (runner.go:1425-1455) under the library's randomness: the span's result
    {"status", "draws", "url", "page_id", "sequence_id"} and the reference's calls in its order, (kind, sql, params):
    none when the pick fails (the function returns its error)"""
    status, url, draws = pick_walkback_channel(keys, owner["url"], library_draw(keys, seed, w))
    res = {"status": status, "draws": draws, "url": url, "page_id": uuid(seed, w, 3), "sequence_id": uuid(seed, w, 4)}
    if status != WALK_OK:
        return res, []
    return res, [(PAGE_BUFFER_INSERT, PAGE_BUFFER_SQL,
                  marshal(page_buffer_values(res["page_id"], owner, url, crawl_id, res["sequence_id"]))),
                 (EDGE_RECORD_INSERT, EDGE_RECORD_SQL, marshal(edge_record_values(owner, url, crawl_id, time)))]


# ---- the library's grouping -------------------------------------------------------------------------------------------
def sql_text(kind: int, rows: int) -> bytes:
    """the text of a statement of `rows` rows: the literal for one row, else the VALUES tuple repeated with the
    placeholders numbered on"""
    lit = PAGE_BUFFER_SQL if kind == PAGE_BUFFER_INSERT else EDGE_RECORD_SQL
    if rows == 1:
        return lit
    n = PER_ROW[kind]
    head = lit.split(b" VALUES ")[0] + b" VALUES "
    return head + b", ".join(b"(" + b", ".join(b"$%d" % (r * n + p + 1) for p in range(n)) + b")"
                             for r in range(rows)) + b";"


def statements(walks, crawl_id: bytes, time, k: int) -> list:
    """tgi_state_walkback's statements, [(kind, rows, sql, params)]: walks = [(owner, result)] of the edge-less spans in
    span order; every page_buffer insert, then every edge_records insert of the WALK_OK ones, k rows per statement"""
    ok = [(o, r) for o, r in walks if r["status"] == WALK_OK]
    rows = {PAGE_BUFFER_INSERT: [page_buffer_values(r["page_id"], o, r["url"], crawl_id, r["sequence_id"]) for o, r in ok],
            EDGE_RECORD_INSERT: [edge_record_values(o, r["url"], crawl_id, time) for o, r in ok]}
    out = []
    for kind in (PAGE_BUFFER_INSERT, EDGE_RECORD_INSERT):
        r = rows[kind]
        for a in range(0, len(r), k):
            part = r[a:a + k]
            out.append((kind, len(part), sql_text(kind, len(part)), marshal([v for row in part for v in row])))
    return out
