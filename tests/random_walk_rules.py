"""A literal Python restatement of the standard random-walk branch of processAllMessagesWithProcessor (random-walk
without TandemCrawl: crawl/runner.go:1218-1227, 1245-1384, 1458-1540), one page after another over a fake state manager
with scripted SearchPublicChat outcomes: the lookups, their effects on the invalid, discovered and chatIDCache sets,
the walkback decision, the pick, and the binding calls, each sent by ExecuteDatabaseOperation
(state/daprstate.go:3643-3678) as an `exec` InvokeBinding: UpsertSeedChannelChatID (:3395-3402), MarkChannelInvalid
(:3569-3578), AddPageToPageBuffer (:3619-3641) and SaveEdgeRecords (:3150-3204).  The expected output of
tgi_state_rw_lookups and tgi_state_rw_step.

Four things are fixed where Go is random or concurrent.  Pages run one after another in span order (Go runs them on
goroutines; this is one valid serialisation).  The u-th deciding page draws rand.IntN(100), the forward index and the
walkback's Random() indices, in that order, with Lemire's rule from one stream of Philox4x32-10 blocks (u_lo, u_hi, 8, j);
uuid.New() becomes the page-id construction with counter word 2 = 9 (the page's ID) and 10 (a walkback's new
SequenceID).  newChannels is a map; the library takes its first-occurrence order.  time.Now() is read once per call."""
from __future__ import annotations

import walkback_rules as wr
from discover_rules import MASK, ST_EMITTED, ST_NOLINE, philox4x32_10
from tandem_rules import is_invalid_channel
from validator_walkback_rules import pick_walkback_channel

FOUND, NOT_SUPERGROUP, NOT_FOUND, RETIRE = 0, 1, 2, 3  # the SearchPublicChat outcomes a caller reports
WALK_OK, WALK_EXHAUSTED, WALK_EMPTY = wr.WALK_OK, wr.WALK_EXHAUSTED, wr.WALK_EMPTY
RETIRED, DEFERRED = 3, 4
PAGE_BUFFER_INSERT, EDGE_RECORD_INSERT = wr.PAGE_BUFFER_INSERT, wr.EDGE_RECORD_INSERT
SEED_UPSERT, INVALID_UPSERT = 8, 9
KINDS = (SEED_UPSERT, INVALID_UPSERT, PAGE_BUFFER_INSERT, EDGE_RECORD_INSERT)
MAX_ROWS = wr.MAX_ROWS
SOURCE_TYPES = (b"mention", b"text_url", b"url", b"plaintext")  # TGI_SRC_*

# the two more literals, byte for byte (daprstate.go:3400, 3576)
SEED_SQL = (b"INSERT INTO seed_channels (channel_username, chat_id) VALUES ($1, $2) ON CONFLICT (channel_username) DO "
            b"UPDATE SET chat_id = EXCLUDED.chat_id;")
INVALID_SQL = (b"INSERT INTO invalid_channels (channel_username, reason, invalidated_at) VALUES ($1, $2, NOW()) ON "
               b"CONFLICT (channel_username) DO UPDATE SET reason = EXCLUDED.reason, invalidated_at = NOW();")


class Retire(Exception):
    """SearchPublicChat's FLOOD_WAIT at or above floodWaitRetireThresholdSecs (runner.go:1333-1338)"""


class FakeState:
    """the state manager's side of the branch: invalidChannelCache (name -> stamp, 0 never expires),
    DiscoveredChannels (its keys in first-occurrence order) and chatIDCache (name -> chat id)"""

    def __init__(self, invalid=None, discovered=(), seeds=None):
        self.invalid = dict(invalid or {})
        self.discovered = list(dict.fromkeys(discovered))
        self._disc = set(self.discovered)
        self.seeds = dict(seeds or {})

    def copy(self):
        return FakeState(self.invalid, self.discovered, self.seeds)

    def is_invalid_channel(self, name, now_sec):  # daprstate.go:3556-3564
        return is_invalid_channel(self.invalid, name, now_sec)

    def is_discovered_channel(self, name):  # base.go:522-524
        return name in self._disc

    def add_discovered_channel(self, name):  # base.go:526-528
        if name not in self._disc:
            self._disc.add(name)
            self.discovered.append(name)

    def get_cached_chat_id(self, name):  # daprstate.go:3406-3411
        return self.seeds.get(name)

    def upsert_seed_channel_chat_id(self, name, chat_id):  # :3395-3402, its row aside
        self.seeds[name] = chat_id

    def mark_channel_invalid(self, name, now_sec):  # :3569-3578, its row aside
        self.invalid[name] = now_sec


def words(seed: int, u: int):
    """the draw stream of the u-th deciding page: block j = Philox (u_lo, u_hi, 8, j) gives x0 | x1 << 32, then
    x2 | x3 << 32"""
    j = 0
    while True:
        x = philox4x32_10([u & MASK, u >> 32, 8, j], [seed & MASK, seed >> 32])
        yield x[0] | x[1] << 32
        yield x[2] | x[3] << 32
        j += 1


def page(sm: FakeState, owner: dict, status, links, n_done: int, search, now_sec: int, rate: int, seed: int, u: int,
         crawl_id: bytes, time, stats: dict):
    """processAllMessagesWithProcessor's standard random-walk branch for one page under the library's randomness.
    status[i] and links[i] (the record's link rows as (name, TGI_SRC_* index), names unique) are the result of its
    i-th record; the loop processed the first n_done.  search(name, record, source) is SearchPublicChat's final
    outcome, (code, chat_id).  Returns (result, calls): result {"status", "walkback", "rnd", "draws", "n_new",
    "forward", "url", "page_id", "sequence_id"}, calls (kind, sql, params) in the reference's order.  A retiring
    outcome raises Retire carrying the calls made so far."""
    calls, new_channels = [], {}
    for i in range(n_done):
        if status[i] not in (ST_EMITTED, ST_NOLINE):  # a failed record returned an error, a date-skipped one Post{}
            continue
        src_map = {name: src for name, src in links[i]}  # :1218-1227
        for o, _ in links[i]:
            if o == owner["url"]:  # :1231
                continue
            if sm.is_invalid_channel(o, now_sec):  # :1247
                continue
            if sm.is_discovered_channel(o):  # :1310
                continue
            if sm.get_cached_chat_id(o) is not None:  # :1312-1316
                sm.add_discovered_channel(o)
                continue
            src = src_map.get(o)
            code, chat_id = search(o, i, src)  # :1323-1354
            if code == RETIRE:
                raise Retire(calls)
            st = SOURCE_TYPES[src] if src is not None else b"unknown"
            stats.setdefault(st, [0, 0])[code != FOUND] += 1  # lookupStats.record
            if code != FOUND:  # :1344-1371
                reason = b"not_found" if code == NOT_FOUND else b"not_supergroup"
                calls.append((INVALID_UPSERT, INVALID_SQL, wr.marshal([o, reason])))
                sm.mark_channel_invalid(o, now_sec)
                continue
            sm.add_discovered_channel(o)  # :1372-1382
            new_channels[o] = True
            calls.append((SEED_UPSERT, SEED_SQL, wr.marshal([o, chat_id])))
            sm.upsert_seed_channel_chat_id(o, chat_id)
    # :1458-1540
    stream = words(seed, u)
    nc = list(new_channels)
    walkback, rnd = not nc, -1
    if nc:
        rnd = wr.lemire(100, stream) + 1
    res = {"status": WALK_OK, "walkback": False, "rnd": rnd, "draws": 0, "n_new": len(nc), "forward": None,
           "url": b"", "page_id": wr.uuid(seed, u, 9), "sequence_id": wr.uuid(seed, u, 10)}
    if walkback or rate >= rnd:
        res["walkback"] = True
        keys = sm.discovered  # as it stands: this page's and earlier pages' insertions included
        status_, url, draws = pick_walkback_channel(keys, owner["url"], set(nc),
                                                    lambda: keys[wr.lemire(len(keys), stream)])
        res.update(status=status_, url=url, draws=draws)
        if status_ != WALK_OK:
            return res, calls  # :1485-1487: the error after the loop's effects
        page_seq = res["sequence_id"]
        skipped = nc
    else:
        idx = wr.lemire(len(nc), stream)
        url = nc[idx]
        res.update(url=url, forward=idx)
        skipped = nc[:idx] + nc[idx + 1:]
        page_seq = owner.get("sequenceId", b"")
    seq = owner.get("sequenceId", b"")
    calls.append((PAGE_BUFFER_INSERT, wr.PAGE_BUFFER_SQL,
                  wr.marshal([res["page_id"], owner["id"], wr.go_int(owner.get("depth", 0) + 1), url, crawl_id, page_seq])))
    calls.append((EDGE_RECORD_INSERT, wr.EDGE_RECORD_SQL,
                  wr.marshal([url, owner["url"], res["walkback"], False, time, crawl_id, seq])))
    calls += [(EDGE_RECORD_INSERT, wr.EDGE_RECORD_SQL, wr.marshal([ch, owner["url"], False, True, time, crawl_id, seq]))
              for ch in skipped]
    return res, calls


def run(sm: FakeState, pages, search, now_sec: int, rate: int, seed: int, u0: int, crawl_id: bytes, time):
    """every page in order, pages = [(owner, status, links, n_done)]: ([(result, calls)], stats, deciding pages).  The
    first retire ends its page (RETIRED, its calls so far stand) and every later page is DEFERRED, untouched"""
    out, stats, u = [], {}, u0
    for k, (owner, status, links, n_done) in enumerate(pages):
        try:
            res, calls = page(sm, owner, status, links, n_done, search, now_sec, rate, seed, u, crawl_id, time, stats)
        except Retire as e:
            out.append(({"status": RETIRED}, e.args[0]))
            out += [({"status": DEFERRED}, [])] * (len(pages) - k - 1)
            return out, stats, u - u0
        out.append((res, calls))
        u += 1
    return out, stats, u - u0


def lookups(sm: FakeState, pages, now_sec: int) -> list:
    """the SearchPublicChat calls of a run with no retire: (name, page, record, source) in call order.  A failed lookup
    changes nothing a later lookup of the call depends on but its own name, as a found one would"""
    calls, sm = [], sm.copy()
    for k, (owner, status, links, n_done) in enumerate(pages):
        def search(name, record, src, k=k):
            calls.append((name, k, record, src))
            return NOT_FOUND, 0
        page(sm, owner, status, links, n_done, search, now_sec, 0, 0, 0, b"", None, {})
    return calls


# ---- the library's grouping -------------------------------------------------------------------------------------------
def sql_text(kind: int, rows: int) -> bytes:
    """the text of a statement of `rows` rows: the literal for one row, else the VALUES tuple repeated with the
    placeholders numbered on (before the upserts' ON CONFLICT clause)"""
    if kind in (PAGE_BUFFER_INSERT, EDGE_RECORD_INSERT):
        return wr.sql_text(kind, rows)
    lit = SEED_SQL if kind == SEED_UPSERT else INVALID_SQL
    if rows == 1:
        return lit
    head, tail = lit.split(b" VALUES ")[0] + b" VALUES ", lit[lit.index(b" ON CONFLICT"):]
    extra = b", NOW()" if kind == INVALID_UPSERT else b""
    return head + b", ".join(b"($%d, $%d%s)" % (2 * r + 1, 2 * r + 2, extra) for r in range(rows)) + tail


def statements(processed, k: int) -> list:
    """tgi_state_rw_step's statements, [(kind, rows, sql, params)], from run()'s output: each kind's one-row calls in
    page order, kinds in KINDS order, cut into statements of k rows, params the rows' values as one JSON array"""
    out = []
    for kind in KINDS:
        rows = [p for _, calls in processed for kd, _, p in calls if kd == kind]
        for a in range(0, len(rows), k):
            part = rows[a:a + k]
            out.append((kind, len(part), sql_text(kind, len(part)), b"[" + b",".join(p[1:-1] for p in part) + b"]"))
    return out
