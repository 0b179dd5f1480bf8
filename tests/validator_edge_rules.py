"""A literal Python restatement of a validator pod's edge validator (runEdgeValidation + validateSingleEdge,
crawl/validator.go:94-309) over a fake world: one claim processed edge after edge, the blocked-state counter, and the
binding calls each DaprStateManager method sends through ExecuteDatabaseOperation (state/daprstate.go:3643-3678) as an
`exec` InvokeBinding: UpsertSeedChannelChatID (:3395-3402), MarkChannelInvalid (:3569-3578), InsertAccessEvent
(:4385-4391) and UpdatePendingEdge (:3999-4006).  The expected output of tgi_state_validator_lookups and
tgi_state_validator_edges.

Beside the per-edge loop it restates the shim's grouped loop: the claim's names in first-occurrence order, one
IsChannelDiscovered per name, then up to m HTTP attempts stopping at the first final one, and ClaimDiscoveredChannel
after a valid one.  The world makes both loops comparable: `validate` answers each name's calls in order from a script,
so the grouped loop asks a name the same questions in the same order as the per-edge loop."""
from __future__ import annotations

from tandem_rules import TTL, is_invalid_channel
from tandem_sql_rules import marshal

# ValidateChannelHTTP's outcomes as the shim reports them (attempt kinds) and the reasons it returns
VALID, NOT_CHANNEL, INVALID, OTHER, TRANSIENT, BLOCKED = 0, 1, 2, 3, 4, 5
FINAL = (VALID, NOT_CHANNEL, INVALID)
REASONS = (b"", b"not_supergroup", b"not_found", b"cached_invalid", b"unknown_status")  # TGI_VR_*
STATUSES = (b"pending", b"valid", b"duplicate", b"invalid", b"not_channel")               # TGI_VS_*
DEFINITIVE, TRANSIENT_KIND, BLOCKED_KIND = 0, 1, 2                                        # edgeOutcomeKind
BLOCKED_THRESHOLD = 5  # blockedThreshold (validator.go:35)
SEED_UPSERT, INVALID_UPSERT, ACCESS_EVENT, EDGE_UPDATE = 8, 9, 10, 11
KINDS = (SEED_UPSERT, INVALID_UPSERT, ACCESS_EVENT, EDGE_UPDATE)
MAX_ROWS = 8191

# the literals, byte for byte (daprstate.go:3400, 3576, 4386, 4001)
SEED_SQL = (b"INSERT INTO seed_channels (channel_username, chat_id) VALUES ($1, $2) ON CONFLICT (channel_username) DO "
            b"UPDATE SET chat_id = EXCLUDED.chat_id;")
INVALID_SQL = (b"INSERT INTO invalid_channels (channel_username, reason, invalidated_at) VALUES ($1, $2, NOW()) ON "
               b"CONFLICT (channel_username) DO UPDATE SET reason = EXCLUDED.reason, invalidated_at = NOW();")
ACCESS_SQL = b"INSERT INTO access_events (reason, occurred_at) VALUES ($1, NOW());"
UPDATE_SQL = (b"UPDATE pending_edges SET validation_status = $1, validation_reason = $2, validated_at = NOW() WHERE "
              b"pending_id = $3;")


class World:
    """what the edge validator reads and writes: invalidChannelCache (name -> stamp, 0 never expires), chatIDCache's
    names in first-occurrence order, the database's discovered_channels, the names another pod claims first (a lost
    ClaimDiscoveredChannel race) and the script of ValidateChannelHTTP: name -> [(kind, reason)], one per call; a name
    past its script answers TRANSIENT"""

    def __init__(self, invalid=None, seeds=(), db=(), raced=(), script=None):
        self.invalid = dict(invalid or {})
        self.seeds = list(dict.fromkeys(seeds))
        self.db = set(db)
        self.raced = set(raced)
        self.script = {k: list(v) for k, v in (script or {}).items()}
        self.calls = {}

    def copy(self):
        w = World(self.invalid, self.seeds, self.db, self.raced, self.script)
        w.calls = dict(self.calls)
        return w

    def is_channel_discovered(self, name):  # daprstate.go:4229-4236
        return name in self.db

    def validate(self, name):  # validateFn: the name's next scripted answer
        q = self.calls.get(name, 0)
        self.calls[name] = q + 1
        s = self.script.get(name, ())
        return s[q] if q < len(s) else (TRANSIENT, 0)

    def claim_discovered_channel(self, name):  # daprstate.go:4208-4227: false when the row exists
        if name in self.db or name in self.raced:
            self.db.add(name)
            return False
        self.db.add(name)
        return True

    def upsert_seed(self, name):  # UpsertSeedChannelChatID fills chatIDCache, its row aside
        if name not in self.seeds:
            self.seeds.append(name)

    def mark_invalid(self, name, now_sec):  # MarkChannelInvalid stamps invalidChannelCache, its row aside
        self.invalid[name] = now_sec


def validate_single_edge(w: World, edge: dict, now_sec: int):
    """validateSingleEdge (validator.go:194-309) -> (status, reason, kind, exec calls [(kind, params)])"""
    name = edge["destination"]
    if is_invalid_channel(w.invalid, name, now_sec):  # :206-213
        return 3, 3, DEFINITIVE, []
    if w.is_channel_discovered(name):  # :216-226
        return 2, 0, DEFINITIVE, []
    kind, reason = w.validate(name)  # :229-253 (the rate-limit wait's cancellation is a TRANSIENT answer)
    if kind == BLOCKED:
        return 0, 0, BLOCKED_KIND, []
    if kind == TRANSIENT:
        return 0, 0, TRANSIENT_KIND, []
    if kind == VALID:  # :260-280
        if not w.claim_discovered_channel(name):
            return 2, 0, DEFINITIVE, []
        w.upsert_seed(name)
        return 1, 0, DEFINITIVE, [(SEED_UPSERT, marshal([name, 0]))]
    if kind in (NOT_CHANNEL, INVALID):  # :282-300
        w.mark_invalid(name, now_sec)
        return (4 if kind == NOT_CHANNEL else 3), reason, DEFINITIVE, [(INVALID_UPSERT, marshal([name, REASONS[reason]]))]
    return 3, 4, DEFINITIVE, []  # :303-308


def run_claim(w: World, edges: list, now_sec: int, count: int = 0):
    """runEdgeValidation's loop over one claim (:144-182) from a state that is not active -> (results, count, crossed_at,
    calls): per edge (status, reason, kind, count after it), the counter after the claim, the edge that entered the
    blocked state (None), and every exec call in order [(kind, params)]"""
    active, crossed, results, calls = False, None, [], []
    for j, e in enumerate(edges):
        st, rs, kd, c = validate_single_edge(w, e, now_sec)
        calls += c
        if kd == BLOCKED_KIND:
            count += 1
            if not active and count >= BLOCKED_THRESHOLD:
                active, crossed = True, j
                calls.append((ACCESS_EVENT, marshal([b"ip_blocked"])))
        elif kd == TRANSIENT_KIND:
            count = max(count - 1, 0)
        else:
            count = 0
        results.append((st, rs, kd, count))
        calls.append((EDGE_UPDATE, marshal([STATUSES[st], REASONS[rs], e["pending_id"]])))
    return results, count, crossed, calls


# ---- the library's grouping -------------------------------------------------------------------------------------------
def lookups(w: World, edges: list, now_sec: int) -> list:
    """tgi_state_validator_lookups: [(name, [edge indices])] of the names the invalid cache does not decide, in
    first-occurrence order"""
    rows = {}
    for j, e in enumerate(edges):
        nm = e["destination"]
        if not is_invalid_channel(w.invalid, nm, now_sec):
            rows.setdefault(nm, []).append(j)
    return list(rows.items())


def shim(w: World, edges: list, rows: list):
    """the shim's loop per lookup row -> (outcomes [(discovered, claimed, n_attempts)], attempts [(kind, reason)])"""
    outcomes, attempts = [], []
    for name, occ in rows:
        if w.is_channel_discovered(name):
            outcomes.append((1, 0, 0))
            continue
        made, claimed = [], 0
        for j in occ:
            kind, reason = w.validate(name)
            made.append((kind, reason))
            if kind in FINAL:
                if kind == VALID:
                    claimed = int(w.claim_discovered_channel(name))
                break
        outcomes.append((0, claimed, len(made)))
        attempts += made
    return outcomes, attempts


def apply(w: World, edges: list, rows: list, outcomes: list, attempts: list, count: int, now_sec: int):
    """tgi_state_validator_edges: every edge's update from its row's outcome, the counter's replay, the sets' updates in
    edge order and the exec calls (seed upserts, invalid upserts, the access event, the updates, each in edge order) ->
    (results, count, crossed_at, calls)"""
    res = [(3, 3, DEFINITIVE)] * len(edges)  # invalid / cached_invalid unless a row decides otherwise
    seeds, invalid = [], []
    a = 0
    for (name, occ), (disc, claimed, na) in zip(rows, outcomes):
        att = attempts[a:a + na]
        a += na
        for r, j in enumerate(occ):
            if disc:
                res[j] = (2, 0, DEFINITIVE)
            elif r < na:
                kind, reason = att[r]
                res[j] = {VALID: (1 if claimed else 2, 0, DEFINITIVE), NOT_CHANNEL: (4, reason, DEFINITIVE),
                          INVALID: (3, reason, DEFINITIVE), OTHER: (3, 4, DEFINITIVE), TRANSIENT: (0, 0, TRANSIENT_KIND),
                          BLOCKED: (0, 0, BLOCKED_KIND)}[kind]
                if kind == VALID and claimed:
                    seeds.append((j, name))
                if kind in (NOT_CHANNEL, INVALID):
                    invalid.append((j, name, reason))
            else:
                res[j] = (2, 0, DEFINITIVE) if att[-1][0] == VALID else (3, 3, DEFINITIVE)
    results, crossed = [], None
    for j, (st, rs, kd) in enumerate(res):
        count = count + 1 if kd == BLOCKED_KIND else max(count - 1, 0) if kd == TRANSIENT_KIND else 0
        if kd == BLOCKED_KIND and crossed is None and count >= BLOCKED_THRESHOLD:
            crossed = j
        results.append((st, rs, kd, count))
    calls = []
    for j, name in sorted(seeds):
        w.upsert_seed(name)
        calls.append((SEED_UPSERT, marshal([name, 0])))
    for j, name, reason in sorted(invalid):
        w.mark_invalid(name, now_sec)
        calls.append((INVALID_UPSERT, marshal([name, REASONS[reason]])))
    if crossed is not None:
        calls.append((ACCESS_EVENT, marshal([b"ip_blocked"])))
    calls += [(EDGE_UPDATE, marshal([STATUSES[st], REASONS[rs], e["pending_id"]])) for (st, rs, _, _), e in
              zip(results, edges)]
    return results, count, crossed, calls


def sql_text(kind: int, rows: int) -> bytes:
    """the text of a statement of `rows` rows: the literal for one row, else the VALUES tuple repeated with the
    placeholders numbered on (before the upserts' ON CONFLICT clause), or the update's join on a VALUES list"""
    if rows == 1:
        return {SEED_UPSERT: SEED_SQL, INVALID_UPSERT: INVALID_SQL, ACCESS_EVENT: ACCESS_SQL, EDGE_UPDATE: UPDATE_SQL}[kind]
    if kind == EDGE_UPDATE:
        return (b"UPDATE pending_edges AS e SET validation_status = v.s, validation_reason = v.r, validated_at = NOW() "
                b"FROM (VALUES " + b", ".join(b"($%d, $%d, $%d::integer)" % (3 * r + 1, 3 * r + 2, 3 * r + 3)
                                              for r in range(rows)) + b") AS v(s, r, id) WHERE e.pending_id = v.id;")
    lit = SEED_SQL if kind == SEED_UPSERT else INVALID_SQL
    head, tail = lit.split(b" VALUES ")[0] + b" VALUES ", lit[lit.index(b" ON CONFLICT"):]
    extra = b", NOW()" if kind == INVALID_UPSERT else b""
    return head + b", ".join(b"($%d, $%d%s)" % (2 * r + 1, 2 * r + 2, extra) for r in range(rows)) + tail


def statements(calls: list, k: int) -> list:
    """tgi_state_validator_edges' statements, [(kind, rows, sql, params)], from the exec calls: each kind's calls in
    order, kinds in KINDS order, cut into statements of k rows (the access event always alone), params the rows' values
    as one JSON array"""
    out = []
    for kind in KINDS:
        rows = [p for kd, p in calls if kd == kind]
        kk = 1 if kind == ACCESS_EVENT else k
        for a in range(0, len(rows), kk):
            part = rows[a:a + kk]
            out.append((kind, len(part), sql_text(kind, len(part)), b"[" + b",".join(p[1:-1] for p in part) + b"]"))
    return out


def reference_statements(calls: list) -> list:
    """the reference's calls as they are sent, one row each, in execution order"""
    return [(kind, 1, sql_text(kind, 1), p) for kind, p in calls]


__all__ = ["World", "validate_single_edge", "run_claim", "lookups", "shim", "apply", "sql_text", "statements", "TTL"]
