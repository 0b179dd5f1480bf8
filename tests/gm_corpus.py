"""Seeded generic client.Message fixtures (SURVEY a12) for the oracle and GPU tests: make_generic (random messages) and
make_generic_edges (records built by rule at the edges of the GPU line, with the cells they must reach)."""
import collections
import random

import go_rules
from distributed_crawler_b200.pack import GenericMessage, pack_generic

_WORDS = ["hello", "мир", "世界", "t.me/somechan", "line\nbreak", "tab\there", 'quote"d', "back\\slash", "<b>&amp;</b>",
          "emoji😀", " sep", "ok", "https://example.org/a?b=c", "ctl\x01\x1f", "é", ""]
_KEYS = ["👍", "❤️", "🔥", "a", "zz", 'k"q', "long-reaction-key-number-one", "😀", "\x7f", "<"]


def make_generic(n: int, seed: int = 5):
    rnd = random.Random(seed)
    msgs = []
    for i in range(n):
        text = " ".join(rnd.choice(_WORDS) for _ in range(rnd.randrange(0, 40))).encode()
        if rnd.random() < 0.05:
            text += bytes(rnd.randrange(0x80, 0x100) for _ in range(rnd.randrange(1, 5)))  # invalid UTF-8
        k = rnd.randrange(0, 5) if rnd.random() < 0.7 else rnd.randrange(0, 12)
        reactions = [(rnd.choice(_KEYS), rnd.randrange(-3, 10 ** rnd.randrange(1, 12))) for _ in range(k)]  # duplicates happen
        msgs.append(GenericMessage(
            id=str(rnd.randrange(1, 1 << 50)), channel_id=rnd.choice(["chan_one", "Ünïcode", 'we"ird', ""]), text=text,
            sender_name=rnd.choice(["", "", "someone", "q\"x"]), ts_sec=rnd.randrange(1_600_000_000, 1_800_000_000),
            ts_nsec=0, views=rnd.choice([0, 1, 12345, rnd.randrange(0, 1 << 40), -7]), reactions=reactions))
    return pack_generic(msgs), msgs


# ---- make_generic_edges: records built by rule at the edges of the generic line -------------------------------------------
# The GPU escapes each text three times per line in 128-byte strips with a carry (esc_to_global), orders a reaction map by a
# warp-uniform selection over raw key bytes (gm_walk.cuh, key_cmp), renders int64s and times per record, and runs both gm
# kernels as grid-stride loops.  The cells below are where those go wrong; generic_edge_coverage measures them on the data.
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
INT_EDGES = [I64_MIN, I64_MIN + 1, -1, 0, I64_MAX] + [v for k in range(1, 19) for v in (10 ** k - 1, 10 ** k, 1 - 10 ** k, -10 ** k)]
TEXT_LENGTHS = (0, 1, 127, 128, 129, 255, 256, 257, 4096, 65536, 1 << 20)
STRIP = 128  # esc_to_global's strip
CROSS_KINDS = ("utf8-2@-1", "utf8-3@-1", "utf8-3@-2", "utf8-4@-1", "utf8-4@-2", "utf8-4@-3", "u2028", "u2029")
_RUNE = {2: "é".encode(), 3: "中".encode(), 4: "😀".encode()}
_ASCII_ESC = b'"\\<>&\n\t\x01\x1f'  # ASCII that encoding/json escapes
_CLEAN = (b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789 .,-_:/" * 4)[:256]  # bytes.translate table
_CUT = (b"\xe2\x80", b"\xf0\x9f\x98", b"\xc3", b"\xff", b"\xed\xa0")  # invalid UTF-8 that ends a text
TZS = (0, -12600, 19800, 86340, -86340)  # the fixed offsets the edge tests run under
Y0 = -62167219200          # 0000-01-01T00:00:00Z
Y9999 = 253402300799       # 9999-12-31T23:59:59Z
NY_OFFSETS = (-18000, -14400)
NY_TRANSITIONS = (1710054000, 1730613600, 1741503600, 1762063200)  # America/New_York 2024-2025, DST on / off


def _clean(rng, n: int) -> bytes:
    return rng.randbytes(n).translate(_CLEAN)


def edge_text(rng, n: int, kind: str) -> bytes:
    """n bytes of one kind: clean ASCII; an escape at the first / last byte; a 2-, 3- or 4-byte rune (or U+2028 / U+2029)
    starting k bytes before every 128-byte strip boundary; C0 and C1 controls and the bytes C0 / C1 around every boundary;
    invalid UTF-8 as the very last bytes"""
    out = bytearray(_clean(rng, n))
    if kind == "esc_first" and n:
        out[0] = rng.choice(_ASCII_ESC)
    elif kind == "esc_last" and n:
        out[-1] = rng.choice(_ASCII_ESC)
    elif kind.startswith("utf8-") or kind in ("u2028", "u2029"):
        if kind.startswith("utf8-"):
            seqs = [(_RUNE[int(kind[5])], int(kind[-1]))]
        else:  # E2 80 A8 / A9 from one and from two bytes before the boundary, in turn
            sep = ("\u2028" if kind == "u2028" else "\u2029").encode()
            seqs = [(sep, 2), (sep, 1)]
        for j, b in enumerate(range(STRIP, n, STRIP)):
            seq, k = seqs[j % len(seqs)]
            if b - k + len(seq) <= n:
                out[b - k:b - k + len(seq)] = seq
    elif kind == "c0c1":
        for b in range(STRIP, n, STRIP):
            piece = bytes([rng.randrange(0x20), 0x7f]) + "\u0085".encode() + bytes([0xC2, rng.randrange(0x80, 0xA0), 0xC0, 0xC1])
            p = min(b - 1, n - len(piece))  # straddles the boundary, also at the end of the text
            out[p:p + len(piece)] = piece
    elif kind == "invalid_end" and n:
        cut = _CUT[n % len(_CUT)][:n]
        out[n - len(cut):] = cut
    return bytes(out)


def _fits(kind: str, n: int) -> bool:
    """a rune of the kind can start k bytes before the first boundary and end inside the text"""
    w, k = (int(kind[5]), int(kind[-1])) if kind.startswith("utf8-") else (3, 2)
    return n > STRIP and STRIP - k + w <= n


def text_kinds(n: int) -> tuple:
    kinds = ("clean",) + (("esc_first", "esc_last", "invalid_end") if n else ())
    return kinds + tuple(k for k in CROSS_KINDS if _fits(k, n)) + (("c0c1",) if n > STRIP else ())


def _nsec(rng, digits: int) -> int:
    """nanoseconds with exactly `digits` fractional digits once trailing zeros are cut (0 for none)"""
    if not digits:
        return 0
    x = rng.randrange(10 ** (digits - 1), 10 ** digits)
    return (x if x % 10 else x + 1) * 10 ** (9 - digits)


def edge_times() -> list[int]:
    """the second of each year bound and the second past it at every offset the tests use (each moves the local year
    across the bound), the int64 ends and both sides of New York's transitions"""
    out = [I64_MIN, I64_MAX]
    for off in TZS + NY_OFFSETS:
        out += [Y0 - off, Y0 - off - 1, Y9999 - off, Y9999 - off + 1]
    for t in NY_TRANSITIONS:
        out += [t - 1, t, t + 1]
    return out


def _edge_reactions(rng) -> list[list]:
    big = edge_text(rng, 65535, "utf8-3@-2")
    maps = [[("👍", 3)], [("b", 1), ("a", 2)],
            [("k", 1), ("k", I64_MIN), ("k", 7), ("k", -5)],  # one key: the last entry wins
            [(b"ab", 1), (b"a\x00", 2), (b"a", 3), (b"abc", 4), (b"a\x00\x00", 5), (b"", 6)],  # prefix chains, the empty key
            [(b"\xff", 1), (b"\x7f", 2), (b"\x80", 3), (b"z", 4), ("é".encode(), 5), (b"\xe2\x80\xa8", 6)],  # 7f < 80 < ff
            [(b"", 9)],
            [('"', 1), ("\\", 2), ("<", 3), (">", 4), ("&", 5), ("\n", 6), ("\x00", 7), ("\u2028", 8), ('a"b', 9)],
            [(b"a\xff", 1), (b"a\xfe", 2), (b"a\xc0", 3)],  # invalid UTF-8 keys that all escape to "a\ufffd"
            [(big, 1), (big[:-1], 2), (big[:-1] + b"\xff", 3), (b"x", 4)],  # 65 535-byte keys, one a prefix of another
            [("v%02d" % j, v) for j, v in enumerate(INT_EDGES)]]  # every count edge
    keys = [("r%04d" % rng.randrange(900)).encode() for _ in range(1000)]
    maps.append([(k, rng.choice(INT_EDGES)) for k in keys])  # 1 000 entries, duplicates among them
    keys = [bytes(rng.choice((rng.randrange(256), rng.randrange(0x61, 0x64))) for _ in range(rng.randrange(0, 6))) for _ in range(4096)]
    maps.append([(k, rng.randrange(-10 ** 6, 10 ** 6)) for k in keys])  # 4 096 entries: short random keys, many duplicates
    for m in maps[3:]:  # in random order (maps[2] keeps its order: which entry is last is the point)
        rng.shuffle(m)
    return maps


def make_generic_edges(seed: int = 1, n: int = 4800):
    """(batch, messages): the edge records (texts of every length and kind at all 16 start offsets mod 16, 65 535-byte
    and empty ids / channels / senders, the reaction maps, the time edges) spread over n records of small filler"""
    rng = random.Random(0x6E0 + seed)
    edges = []  # (text, extra fields)
    for n_text in TEXT_LENGTHS:
        for kind in text_kinds(n_text):
            edges.append(dict(text=edge_text(rng, n_text, kind)))
    for what in ("id", "channel_id", "sender_name"):
        edges.append({what: edge_text(rng, 65535, rng.choice(("c0c1", "utf8-4@-3", "esc_last"))), "text": b"t"})
    edges.append(dict(id=edge_text(rng, 65535, "u2028"), channel_id=edge_text(rng, 65535, "c0c1"),
                      sender_name=edge_text(rng, 65535, "utf8-2@-1"), text=edge_text(rng, 300, "u2029")))
    edges.append(dict(id=b"", channel_id=b"", sender_name=b"", text=b""))
    edges += [dict(reactions=m, text=_clean(rng, rng.randrange(0, 40))) for m in _edge_reactions(rng)]
    edges += [dict(ts_sec=t, text=b"time") for t in edge_times()]
    edges += [dict(ts_nsec=ns, text=b"ns") for ns in [_nsec(rng, d) for d in range(10)] + [999_999_999, 1]]
    assert len(edges) < n
    slots = sorted(rng.sample(range(n), len(edges)))
    where = dict(zip(slots, edges))
    msgs, off, k_text = [], 0, 0
    for i in range(n):
        e = where.get(i, {})
        text = e.get("text", _clean(rng, rng.randrange(0, 60)))
        chan = e.get("channel_id", rng.choice((b"", b"chan", "канал".encode(), b'c"h')))
        mid = e.get("id")
        if mid is None:  # pad the id so that the text starts at the next offset mod 16 (the 16-byte loads of the escaper)
            want = k_text % 16 if len(text) > STRIP else rng.randrange(16)
            k_text += len(text) > STRIP
            base = str(rng.randrange(1, 10 ** 6)).encode()
            mid = base + b"0" * ((want - off - len(base) - len(chan)) % 16)
        sender = e.get("sender_name", rng.choice((b"", b"someone", b"q\"x")))
        m = GenericMessage(
            id=mid, channel_id=chan, text=text, sender_name=sender,
            ts_sec=e.get("ts_sec", rng.randrange(1_600_000_000, 1_800_000_000)),
            ts_nsec=e.get("ts_nsec", _nsec(rng, i % 10)), views=INT_EDGES[i % len(INT_EDGES)],
            reactions=e.get("reactions", [(rng.choice(_KEYS), rng.choice(INT_EDGES)) for _ in range(rng.choice((0, 0, 1, 2, 3)))]))
        off += len(m.id) + len(m.channel_id) + len(m.text) + len(m.sender_name)
        msgs.append(m)
    return pack_generic(msgs), msgs


# ---- coverage accounting -------------------------------------------------------------------------------------------------
def _b(s) -> bytes:
    return s.encode() if isinstance(s, str) else bytes(s)


def _esc_grows(b: bytes) -> bool:
    return len(go_rules.go_json_string(b)) - 2 != len(b)


def _text_cells(t: bytes) -> set:
    n, cells = len(t), set()
    if n not in TEXT_LENGTHS:
        return cells
    if t.isascii() and not _esc_grows(t):
        cells.add((n, "clean"))
    if n and t[0] < 0x80 and _esc_grows(t[:1]):
        cells.add((n, "esc_first"))
    if n and t[-1] < 0x80 and _esc_grows(t[-1:]):
        cells.add((n, "esc_last"))
    if n and t.decode("utf-8", "replace").endswith("\ufffd") and not t.endswith("\ufffd".encode()):
        cells.add((n, "invalid_end"))
    for b in range(STRIP, n, STRIP):
        for k in (1, 2, 3):  # a rune that starts k bytes before the boundary and crosses it
            if t[b - k] >= 0xC2:
                r, w = go_rules.go_decode_rune(t, b - k)
                if w > k and r != 0xFFFD:
                    cells.add((n, "u2028" if r == 0x2028 else "u2029" if r == 0x2029 else "utf8-%d@-%d" % (w, k)))
        near = t[max(b - 8, 0):b + 8]
        if b"\xc2\x85" in near and b"\xc0" in near and b"\xc1" in near and any(c < 0x20 for c in near):
            cells.add((n, "c0c1"))
    return cells


def generic_edge_coverage(msgs) -> collections.Counter:
    cov, off = collections.Counter(), 0
    for m in msgs:
        mid, chan, text, sender = _b(m.id), _b(m.channel_id), _b(m.text), _b(m.sender_name)
        for c in _text_cells(text):
            cov[("text",) + c] += 1
        if len(text) > STRIP:
            cov["text start mod 16", (off + len(mid) + len(chan)) % 16] += 1
        off += len(mid) + len(chan) + len(text) + len(sender)
        for what, s in (("id", mid), ("channel", chan), ("sender", sender)):
            if len(s) in (0, 65535):
                cov[what, len(s)] += 1
        cov["views", m.views] += 1
        keys = [_b(k) for k, _ in m.reactions]
        for _, v in m.reactions:
            cov["count", v] += 1
        if len(keys) in (0, 1, 2, 1000, 4096):
            cov["entries", len(keys)] += 1
        if len(keys) > 1 and len(set(keys)) == 1:
            cov["react", "one key"] += 1
        if {b"a", b"a\x00", b"ab"} <= set(keys):
            cov["react", "prefix chain"] += 1
        if {b"\x7f", b"\x80", b"\xff"} <= set(keys):
            cov["react", "7f < 80 < ff"] += 1
        if b"" in keys:
            cov["react", "empty key"] += 1
        if any(_esc_grows(k) and k.isascii() for k in keys):
            cov["react", "escaped key"] += 1
        if any(len(k) == 65535 for k in keys):
            cov["react", "65535-byte key"] += 1
        invalid = {}
        for k in set(keys):
            if k.decode("utf-8", "replace") != k.decode("utf-8", "ignore"):
                invalid.setdefault(go_rules.go_json_string(k), set()).add(k)
        if any(len(v) > 1 for v in invalid.values()):
            cov["react", "invalid keys that escape alike"] += 1
        ns = m.ts_nsec
        cov["nsec digits", len(("%09d" % ns).rstrip("0")) if ns else 0] += 1
        if ns == 999_999_999:
            cov["nsec", ns] += 1
        for tz in TZS:
            local = m.ts_sec + tz
            for name, t in (("year 0, first second", Y0), ("year -1, last second", Y0 - 1),
                            ("year 9999, last second", Y9999), ("year 10000, first second", Y9999 + 1)):
                if local == t:
                    cov[name, tz] += 1
        if m.ts_sec in (I64_MIN, I64_MAX):
            cov["ts_sec", m.ts_sec] += 1
        for t in NY_TRANSITIONS:
            if m.ts_sec - t in (-1, 0, 1):
                cov["New York transition", m.ts_sec - t] += 1
    return cov


def generic_edge_cells() -> list[tuple]:
    """the cells generic_edge_coverage must find non-empty"""
    cells = [("text", n, k) for n in TEXT_LENGTHS for k in text_kinds(n)]
    cells += [("text start mod 16", k) for k in range(16)]
    cells += [(what, n) for what in ("id", "channel", "sender") for n in (0, 65535)]
    cells += [("views", v) for v in INT_EDGES] + [("count", v) for v in INT_EDGES]
    cells += [("entries", k) for k in (0, 1, 2, 1000, 4096)]
    cells += [("react", c) for c in ("one key", "prefix chain", "7f < 80 < ff", "empty key", "escaped key", "65535-byte key",
                                     "invalid keys that escape alike")]
    cells += [("nsec digits", d) for d in range(10)] + [("nsec", 999_999_999)]
    cells += [(name, tz) for tz in TZS for name in ("year 0, first second", "year -1, last second", "year 9999, last second",
                                                    "year 10000, first second")]
    cells += [("ts_sec", I64_MIN), ("ts_sec", I64_MAX)] + [("New York transition", d) for d in (-1, 0, 1)]
    return cells
