"""Edge states for the resident progress state (tgi_state_*): pages, messages and layers, as state_pack dicts, that put
extreme values through every writer of state.cuh.

- Page strings go through the warp escaper (st_entry: warp_esc_len64 / esc_to_global, 128-byte strips): each of the
  nine fields at the lengths around one, two, four and 32 strips and at 64 KB and 100 KB, in every kind of STR_KINDS,
  with the feature placed where a strip ends.
- Short strings go through the thread escaper (st_thread_esc / thread_esc_len and its 4-byte ASCII step): message
  pageIds, registered status and platform codes, layer-map ids.  One escape, one non-ASCII rune, one U+2028 and one
  invalid byte at every offset of lengths 0-40 and at n-1 .. n-4, plus 4 KB and 64 KB.
- Numbers: chat and message ids at the int64 ends and +-1, around 2^32 and 10^18 and at every digit count; page and
  layer depths at the int64 ends (the layer map orders them as strings).
- Times: the year-0 and year-9999 bounds, fixed offsets of +-86399 s, +-1 .. +-59 s and with seconds, nsec trims.

state_cells() reads the (writer, field, length, kind) cells back from the state each writer is handed, and
expected_cells() lists the cells the corpus is meant to reach; tests/test_state_edge_rules.py checks they agree."""
from __future__ import annotations

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
FIELDS = ("id", "url", "status", "error", "platform", "parentId", "LastConnectionID", "sequenceId", "crawlId")
OMITEMPTY = ("error", "platform", "parentId", "LastConnectionID", "sequenceId", "crawlId")
STR_LENGTHS = (0, 1, 127, 128, 129, 255, 256, 257, 511, 512, 513, 4095, 4096, 4097, 65535, 100000)
STR_KINDS = ("clean", "lt", "ctrl", "rune2@125", "rune3@125", "rune4@125", "rune2@126", "rune3@126", "rune4@126",
             "rune2@127", "rune3@127", "rune4@127", "u2028@127", "u2029@126", "invalid@127", "invalid@128",
             "overlong_end", "surrogate_end", "truncated_end")
SHORT_FEATURES = {"esc": b"<", "rune": "é".encode(), "u2028": b"\xe2\x80\xa8", "invalid": b"\xff"}
SHORT_LENGTHS = tuple(range(41)) + (4096, 65536)

# numbers: the int64 ends and +-1, around 2^32 and 10^18 (render_u64 peels 9 digits past 2^32), every digit count
INT_EDGES = sorted({I64_MIN, I64_MIN + 1, I64_MIN + 2, -1, 0, 1, I64_MAX - 1, I64_MAX, (1 << 32) - 1, 1 << 32,
                    (1 << 32) + 1, -(1 << 32), 10 ** 18 - 1, 10 ** 18, 10 ** 18 + 1, -(10 ** 18)}
                   | {10 ** k - 1 for k in range(1, 19)} | {10 ** k for k in range(19)} | {-(10 ** k) for k in range(19)})
DEPTH_EDGES = (I64_MIN, I64_MIN + 1, -1, 0, 9, 10, I64_MAX - 1, I64_MAX)

# times: (sec, nsec, offset or None for time.Local); year 0 begins at -62167219200, year 9999 ends at 253402300799
YEAR0, YEAR9999_END = -62167219200, 253402300799
OFFSETS = (0, 86399, -86399, 1, -1, 59, -59, 60, -60, 19830, -19830, 3600, -18000)
NSECS = (0, 1, 10, 100_000_000, 999_999_999, 120_000_000)
TIME_EDGES = ([(YEAR0 - off, 0, off) for off in OFFSETS] + [(YEAR9999_END - off, 999_999_999, off) for off in OFFSETS]
              + [(1700000000, ns, off) for off in OFFSETS for ns in NSECS]
              + [(YEAR0 + 86400, 0, None), (YEAR9999_END - 86400, 999_999_999, None), (1699164000, 1, None)])
TIME_REFUSED = [(YEAR0 - 1, 0, 0), (YEAR9999_END + 1, 0, 0), (YEAR0 - 1 - 3600, 999_999_999, 3600),
                (YEAR9999_END + 1 + 18000, 0, -18000)]
ROW_COUNTS = (1, 2, 256, 257, 65536, 65537)  # the render's radix passes: 0, 1, 1, 2 (9 bits), 2, 3 (17 bits)


# what every generated string stands for: bytes -> {(length, kind)}; the cells are read back from the state a writer is
# handed, so a string counts only where a writer sees it
WARP_LABELS: dict[bytes, set] = {}
SHORT_LABELS: dict[bytes, set] = {}


def _fill(n: int, unit: bytes) -> bytes:
    return (unit * (n // len(unit) + 1))[:n]


def edge_str(kind: str, n: int, seed: int = 0) -> bytes:
    """n bytes of the kind; a feature that does not fit in n bytes is left out (the string stays n bytes)"""
    s = _edge_str(kind, n, seed)
    WARP_LABELS.setdefault(s, set()).add((n, kind))
    return s


def _edge_str(kind: str, n: int, seed: int) -> bytes:
    base = _fill(n, b"abcdefghijklmnopqrstuvwxyz0123456789-_./"[seed % 7:] + b"ABC")
    if kind == "clean":
        return base
    if kind == "lt":
        return b"<" * n
    if kind == "ctrl":
        return _fill(n, bytes([0, 1, 8, 9, 10, 12, 13, 31, 0x7F, ord('"'), ord("\\"), ord("&"), ord(">")]))
    if kind.endswith("_end"):
        tail = {"overlong_end": b"\xc0\xaf", "surrogate_end": b"\xed\xa0\x80", "truncated_end": b"\xe2\x82"}[kind]
        return base[:n - len(tail)] + tail if n >= len(tail) else base
    name, at = kind.split("@")
    at = int(at)
    feat = {"rune2": "é".encode(), "rune3": "€".encode(), "rune4": "😀".encode(), "u2028": b"\xe2\x80\xa8",
            "u2029": b"\xe2\x80\xa9", "invalid": b"\xff"}[name]
    # the feature repeats every 128 bytes: at byte `at` of every strip the string holds
    out = bytearray(base)
    for s in range(at, n - len(feat) + 1, 128):
        out[s:s + len(feat)] = feat
    return bytes(out)


def short_strs() -> list[tuple[bytes, str, int]]:
    """(string, feature, length): every feature at every offset of lengths 0-40 and at n-1 .. n-4 of the long ones"""
    out = []
    for n in SHORT_LENGTHS:
        for name, f in SHORT_FEATURES.items():
            if n < len(f):
                out.append((_fill(n, b"xyz0"), name, n))
                SHORT_LABELS.setdefault(out[-1][0], set()).add((n, name))
                continue
            offs = range(n - len(f) + 1) if n <= 40 else [n - len(f) - k for k in range(4)] + [0, 1, 2, 3]
            for k in offs:
                s = bytearray(_fill(n, b"xyz0"))
                s[k:k + len(f)] = f
                out.append((bytes(s), name, n))
                SHORT_LABELS.setdefault(out[-1][0], set()).add((n, name))
    return out


def edge_pages(tag: bytes = b"") -> list[dict]:
    """pages that put every (field, length, kind) of the warp escaper in front of st_entry.  Page (k, j) holds kind
    STR_KINDS[k] in every field, field f at length STR_LENGTHS[(j + f) % 16]; the id is made unique by a prefix (its
    label is the edge string's); two more pages hold the omitempty fields empty and at one byte"""
    pages = []
    for k, kind in enumerate(STR_KINDS):
        for j in range(len(STR_LENGTHS)):
            p = {}
            for f, name in enumerate(FIELDS):
                n = STR_LENGTHS[(j + f) % len(STR_LENGTHS)]
                s = edge_str(kind, n, k + f)
                if name == "id":
                    s = b"%sid%d.%d:" % (tag, k, j) + s
                    WARP_LABELS.setdefault(s, set()).add((n, kind))
                if s:
                    p[name] = s
            p["depth"] = DEPTH_EDGES[(k + j) % len(DEPTH_EDGES)]
            p["timestamp"] = TIME_EDGES[(k * len(STR_LENGTHS) + j) % len(TIME_EDGES)]
            pages.append(p)
    for j in (0, 1):  # the omitempty fields all empty, and all at one byte
        pages.append(dict({name: b"<" * j for name in OMITEMPTY if j}, id=b"%somit%d" % (tag, j), url=b"u", depth=j,
                          timestamp=(0, 0, 0)))
    return pages


def short_pages(tag: bytes = b"s") -> list[dict]:
    """pages whose ids are the short strings (a repeated string made unique by a prefix): layer-map ids, and the
    pageIds of edge_state's messages"""
    pages, seen = [], set()
    for q, (s, feat, n) in enumerate(short_strs()):
        pid = s if s not in seen else tag + b"%d:" % q + s
        seen.add(pid)
        if pid != s:
            SHORT_LABELS.setdefault(pid, set()).add((n, feat))
        pages.append({"id": pid, "url": b"u%d" % q, "depth": 1, "status": b"fetched", "timestamp": (1700000000 + q, 0, 0)})
    return pages


def custom_codes() -> list[bytes]:
    """registered status / platform codes with escapes, runes, U+2028 and invalid bytes (tgi_state_code)"""
    codes = [s for s, _, n in short_strs() if 0 < n <= 12][::3] + [b"fetched", b"<&>", b"\xe2\x80\xa9", b"\xff\xfe"]
    return list(dict.fromkeys(codes))


def message_edges(pids: list[bytes], codes: list[bytes], q0: int = 0) -> list[dict]:
    """one message per pageId of pids: chat and message ids cycle through INT_EDGES (both ends and every digit count),
    statuses through every code, platforms through every code and none"""
    out = []
    for i, pid in enumerate(pids):
        q = q0 + i
        out.append({"chatId": INT_EDGES[q % len(INT_EDGES)], "messageId": INT_EDGES[-1 - q % len(INT_EDGES)],
                    "status": codes[q % len(codes)], "pageId": pid,
                    "platform": codes[(q + len(codes) // 2) % len(codes)] if q % 3 else b""})
    return out


def edge_state() -> list:
    """the corpus as SetState layers: depths at the int64 ends, empty layers first, between and last; every short page
    id is the pageId of one message, the messages spread over four edge pages among message-less ones"""
    pages, short, codes = edge_pages(), short_pages(), custom_codes()
    pids = [p["id"] for p in short]
    for q, k in enumerate((7, 100, 150, 303)):
        part = pids[q::4]
        pages[k]["messages"] = message_edges(part, codes, q * len(part))
    return [(I64_MIN, []), (-1, pages[:150]), (0, []), (9, short), (10, pages[150:]), (I64_MAX, [])]


def state_cells(layers) -> set:
    """the cells a state reaches, read from what each writer is handed: every listed page's nine strings (st_entry),
    every listed id (the layer map), the pageId, status and platform of every message of a listed page (st_message)"""
    cells = set()
    listed = [p for _, ps in layers for p in ps]
    for p in listed:
        for f in FIELDS:
            s = p.get(f, b"")
            cells |= {("entry", f, n, kind) for n, kind in WARP_LABELS.get(s, ())}
            if f in OMITEMPTY and len(s) <= 1:
                cells.add(("entry", f, len(s), "omitempty"))
        cells |= {("layer_map", "id", n, feat) for n, feat in SHORT_LABELS.get(p.get("id", b""), ())}
        for m in p.get("messages") or []:
            cells |= {("message.pageId", "pageId", n, feat) for n, feat in SHORT_LABELS.get(m["pageId"], ())}
            cells.add(("code", "status", m["status"]))
            if m.get("platform"):
                cells.add(("code", "platform", m["platform"]))
    return cells


def expected_cells() -> set:
    want = {("entry", f, n, k) for f in FIELDS for n in STR_LENGTHS for k in STR_KINDS}
    want |= {("entry", f, n, "omitempty") for f in OMITEMPTY for n in (0, 1)}
    want |= {(w, fld, n, feat) for w, fld in (("message.pageId", "pageId"), ("layer_map", "id"))
             for n in SHORT_LENGTHS for feat in SHORT_FEATURES}
    want |= {("code", role, c) for role in ("status", "platform") for c in custom_codes()}
    return want
