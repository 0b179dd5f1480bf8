"""Telegram link extraction at the geometry of its GPU scanners (csrc/tg_links.cuh), messages built by rule rather than by
distribution: a `t.me/` at every lane offset of the 16-byte lanes and across the 512-byte strips of tme16 /
warp_scan_channel_links, names around warp_word_run's 32-byte cap, mention slices around warp_scan_username's 32-byte
steps, entity offsets around the 128-byte strips and 4-byte lanes of warp_utf16_to_bytes (fast and exact strips, the
carry across strips), around warp_map_entities' ASCII-prefix shortcut, records whose link bound is tight, dedup, flags and
the filter.  Records with and without entities share groups of 32 in every layout the ballot-driven kernels meet.

make_link_edges(seed) -> (page-sized TgBatch, messages, channels); link_cells(msgs) restates the scanners' geometry for
coverage accounting; mapping_cases(seed) lists the UTF-16 mapping records with the one-unit moves that change their
result."""
from __future__ import annotations

import bisect
import functools
import random

import go_rules
from distributed_crawler_b200.pack import Channel, FormattedText, Message, TextEntity, pack_telegram

PAGE_MAX_RECS = 8192  # tgingest.cu: the largest batch the one-launch page kernel takes
SEEDS = (1, 2, 3)
RESERVED = ("share", "proxy", "socks", "login", "addlist", "confirm", "joinchat", "addtheme", "addstickers", "setlanguage")
CARRIERS = ("messageText", "messagePhoto", "messageVideo", "messageDocument", "messageAnimation", "messageAudio",
            "messageVoiceNote")
CHANNELS = [Channel(title="self", name="selfchan1", username="selfchan1"),
            Channel(title="mixed", name="MixedCase_chan", username="MixedCase_chan"),
            Channel(title="", name="", username="")]
MIN_POST_DATE = 1_650_000_000  # the config variant's cut; records dated 1_600_000_000 lie before it
MAP_EDGES = (16, 128, 256, 512, 1024)
MAP_J = tuple(range(-3, 3))
MENTION_LENGTHS = (0, 1, 5, 6, 31, 32, 33)
URL_LENGTHS = MENTION_LENGTHS + (10,)  # 10 = "t.me/" and a 5-byte name: the shortest url slice that finds a link
MOVES = (("start", -1), ("start", 1), ("end", -1), ("end", 1))

_LOWER = b"abcdefghijklmnopqrstuvwxyz"
_FILL = b"abcdefghijklmnopqrsuvwxyz ,-"  # no 't', '.', '/': filler never forms a t.me/
_NONWORD = b" -!#%,;=+"
_RUNES = {1: [bytes([c]) for c in _NONWORD], 2: [s.encode() for s in "éдЯ"], 3: [s.encode() for s in "中€अ"],
          4: [s.encode() for s in "😀𝄞\U00010000"]}
_INVALID = [b"\x80", b"\xbf", b"\xff", b"\xe4\xb8", b"\xf0\x9f\x98", b"\xc0\x80", b"\xed\xa0\x80"]


# ---- UTF-16 under Go's decoding ---------------------------------------------------------------------------------------
def units(b: bytes) -> int:
    """UTF-16 length of b as utf16OffsetToBytes counts it: 2 per rune >= U+10000, 1 per other rune or invalid byte"""
    return _table(b)[1][-1] if b else 0


@functools.lru_cache(maxsize=4096)
def _table(b: bytes):
    """(rune start byte indexes, UTF-16 position at each of them, then the total)"""
    starts, pos, i, u = [], [], 0, 0
    while i < len(b):
        starts.append(i)
        pos.append(u)
        r, w = go_rules.go_decode_rune(b, i)
        u += 2 if r >= 0x10000 else 1
        i += w
    return starts, pos + [u]


def _table_ascii_tail(head: bytes, tail: bytes):
    """_table(head + tail) for an ASCII tail (it cannot change how head decodes)"""
    starts, pos = _table(head)
    u = pos[-1]
    return starts + list(range(len(head), len(head) + len(tail))), pos[:-1] + list(range(u, u + len(tail))) + [u + len(tail)]


def map16(table, n: int, off: int, length: int):
    """utf16OffsetToBytes (tdutils.go:55-78) by table lookup: the positions of the rune starts rise strictly, so the
    loop meets `off` and `stop` at most once each"""
    starts, pos = table
    stop = ((off + length + 2 ** 31) % 2 ** 32) - 2 ** 31
    pos = pos[:-1]

    def find(u):
        k = bisect.bisect_left(pos, u)
        return k if k < len(pos) and pos[k] == u else None

    io, isp = find(off), find(stop)
    if isp is not None:
        return (starts[io] if io is not None and io <= isp else -1), starts[isp]
    return (starts[io], n) if io is not None else (0, 0)


def expected(m: Message, min_post_date=None):
    """(status name, [(name, src)]) of one message by tests/go_rules.py"""
    if min_post_date is not None and m.date < min_post_date:
        return "skipped", []
    if m.panics:
        return "failed", []
    if m.content_type not in CARRIERS or m.text is None:
        return "emitted", []
    got = go_rules.extract_links(_b(m.text.text), [(e.offset, e.length, e.type, _b(e.url)) for e in m.text.entities])
    return ("failed", []) if got is None else ("emitted", got)


def _b(s) -> bytes:
    return s if isinstance(s, bytes) else str(s).encode()


# ---- builders ---------------------------------------------------------------------------------------------------------
def _fill(rng, n):
    return bytes(rng.choice(_FILL) for _ in range(max(n, 0)))


def _letters(rng, n):
    return bytes(rng.choice(_LOWER) for _ in range(n))


def _name(rng, n, first=None):
    """a word run of n bytes starting with a letter (or `first`)"""
    body = bytes(rng.choice(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789_") for _ in range(n - 1))
    return (first if first is not None else bytes([rng.choice(_LOWER)])) + body


def _msg(text, ents=(), **kw):
    kw.setdefault("channel", -1)  # -1: make_link_edges picks one
    return Message(content_type=kw.pop("ct", "messageText"), text=None if text is None else
                   FormattedText(text, [TextEntity(o, l, t, u) for (o, l, t, u) in ents]), **kw)


def _tme_plain(rng):
    """plaintext FindAllStringSubmatch: lane offsets, strip edges, text ends, name lengths, prefixes, chains, dense '/'"""
    F, out = (lambda n: _fill(rng, n)), []
    for base in (0, 1024):
        for k in range(16):  # the '/' of a t.me/ at lane offset k
            p = base + 48 + k
            out.append(F(p - 4) + b"t.me/" + _name(rng, 5 + k % 9) + b" " + F(20))
    for e in (512, 1024):
        for t in range(e - 5, e + 1):  # a t.me/ straddling the strip edge: its t at e-5 .. e
            out.append(F(t) + b"t.me/" + _name(rng, 8) + b" " + F(30))
            # chains: the next t.me/ begins with the t that ended the previous name, that t at e-5 .. e
            out.append(F(t - 10) + b"t.me/abcdet.me/" + _name(rng, 6) + b"t.me/" + _name(rng, 7) + b" " + F(9))
            out.append(F(t - 10) + b"t.me/abcdet.me/fghijt.me/klmno_t.me/" + _name(rng, 5))
        for ln in (4, 5, 31, 32, 33, 40):  # names crossing the strip edge
            out.append(F(e - ln // 2 - 5) + b"t.me/" + _name(rng, ln) + b" " + F(11))
            out.append(F(e - ln + 1 - 5) + b"t.me/" + _name(rng, ln) + b"." + F(3))
    out += [b"t.me/" + _name(rng, 9) + b" " + F(40), F(37) + b"t.me/", F(16) + b"t.me/", b"t.me/", b"t.me/abcde",
            F(29) + b"t.me/" + _name(rng, 12), F(30) + b"t.me/abc", F(27) + b"t.me/abcd", F(500) + b"t.me/" + _name(rng, 20),
            F(503) + b"t.me/abcd", b"t.me/1abcdef t.me/_abcdef t.me/9 t.me/a1234 t.me/Z____",
            b"https://t.me/httpsname x http://t.me/httpname T.ME/upper t.me//slashname tt.me/doublet t.mex/mexname "
            b".me/dotname t.me/ok_name1 https://T.me/mixed_case_a HTTPS://t.me/upper_scheme",
            b"t.me/joinchat t.me/realchan1 t.me/JoinChat/x t.me/after_reserved t.me/sharefoo t.me/Share t.me/ADDSTICKERS"]
    for k in range(6):  # dense: a '/' every 11th to 17th byte, some of them ending a t.me
        t = bytearray()
        while len(t) < 1100 + 97 * k:
            gap = rng.randrange(10, 17)
            t += (F(gap - 4) + b"t.me") if rng.random() < 0.3 else F(gap)
            t += b"/"
            if rng.random() < 0.5:
                t += _name(rng, rng.choice((3, 4, 5, 9)))
        out.append(bytes(t))
    return [_msg(t) for t in out]


def _entity_links(rng):
    """url / text_url (FindStringSubmatch: a reserved first match drops the entity) and mention slices"""
    F, out = (lambda n: _fill(rng, n)), []
    pair = b"t.me/joinchat t.me/realchannel"
    out.append(_msg(F(7) + pair + b" " + F(5), [(7, len(pair), "url", "")]))
    out.append(_msg(b"x" + pair, [(0, 1, "text_url", pair)]))
    for w in RESERVED:
        mixed = bytes(c - 32 if rng.random() < 0.5 else c for c in w.encode())
        s = b"t.me/" + mixed + b" t.me/validname"
        out.append(_msg(F(3) + s + b" " + F(4), [(3, len(s), "url", ""), (0, 1, "text_url", b"https://" + s)]))
        out.append(_msg(F(5) + b"t.me/" + mixed + b" t.me/after_" + w.encode() + b" t.me/" + mixed + b"x"))
        out.append(_msg(b"t.me/" + mixed + b"/x", [(0, 8 + len(w), "url", ""), (0, 2, "text_url", b"t.me/" + mixed + b"_ok")]))
    for st in range(32):  # url slices at every alignment relative to the text
        nm = _name(rng, 5 + st % 28)
        s = b"t.me/" + nm
        out.append(_msg(F(st) + s + b" " + F(9), [(st, len(s), "url", ""), (0, st, "text_url", F(st) + b"t.me/" + nm + b"x")]))
        out.append(_msg(F(st) + b"zt.me/" + nm + b" " + F(3), [(st + 1, len(s) - 1 - st % 3, "url", "")]))
    for L in (4, 5, 31, 32, 33, 63, 64, 65):  # mention slices
        for a in (0, 1, 13):
            nm = _name(rng, L)
            out.append(_msg(F(a) + b"@" + nm + b" " + F(6), [(a, L + 1, "mention", ""), (a + 1, L, "mention", "")]))
    for q in range(26, 35):  # the first valid start at slice byte q: the 4-byte look-ahead crosses the 32-byte step
        pre = (b"ab-cd-e1-_f2-" * 4)[:q - 1] + b"-"
        for tail in (5, 6, 9):
            s = pre + _letters(rng, tail)
            out.append(_msg(b"@" + s + b" " + F(8), [(1, len(s), "mention", "")]))
            out.append(_msg(b"@" + s + b" " + F(8), [(1, len(s) - 1, "mention", "")]))
    for s in (b"@leading_at", b"@@double_at", b"123digits_first", b"_underscore1", b"ab\xc3\xa9cdefgh", b"abcd\xe4\xb8\xadefghi",
              b"\xf0\x9f\x98\x80emoji_first", b"a\xffbcdefghij", b"@ab @abcd @abcde_ x", b"4567", b"abcd"):
        out.append(_msg(b"> " + s + b" <", [(2, units(s), "mention", "")]))
    return out


def _prefix(rng, target: int, invalid: bool) -> bytes:
    """a prefix of target bytes made of 1-4-byte runes whose last rune is multi-byte and ends at `target`; with
    `invalid`, strips of even index also hold invalid bytes (exact strips next to fast ones)"""
    w_last = 2 + target % 3
    out = bytearray()
    while len(out) < target - w_last:
        room = target - w_last - len(out)
        if invalid and (len(out) // 128) % 2 == 0 and rng.random() < 0.25:
            frag = rng.choice([f for f in _INVALID if len(f) <= room] or [b" "])
        else:
            frag = rng.choice(_RUNES[rng.choice([w for w in (1, 2, 3, 4) if w <= room])])
        out += frag
    return bytes(out) + rng.choice(_RUNES[w_last])


@functools.lru_cache(maxsize=None)
def mapping_cases(seed: int):
    """UTF-16 mapping: text = P + W, P's byte length at -5..+5 around 16 .. 1024 (its last rune straddling the walker's
    lanes and strips), entity offset units(P) + j, j = -3..+2.  The link text starts at the entity's start and ends at
    its end, so that a one-unit error in either changes the link: for j < 0 the first |j| bytes of the link end P.
    A mention's name is W's letters; a url holds t.me/ and a name shorter than 32 bytes.  The (edge, delta, P kind,
    entity kind, j, length) grid is split over the three seeds.  -> [(Message, kind, moves that change the result)]"""
    rng, out, k = random.Random(1000 + seed), [], 0
    for edge in MAP_EDGES:
        for delta in range(-5, 6):
            for invalid in (False, True):
                R = _prefix(rng, edge + delta, invalid)
                for kind, lengths in (("mention", MENTION_LENGTHS), ("url", URL_LENGTHS)):
                    for j in MAP_J:
                        for L in lengths:
                            k += 1
                            if k % 3 != seed % 3:
                                continue
                            out.append(_mapping_case(rng, R, kind, j, L))
    return out


def _mapping_case(rng, R, kind, j, L):
    if kind == "mention":
        link = _letters(rng, 48 + rng.randrange(0, 16))
    else:
        link = b"t.me/" + _letters(rng, max(L - 5, 5)) + _letters(rng, 20)
        link = (_letters(rng, j) if j > 0 else b"") + link
    cut = -j if j < 0 else 0
    P, W = R + link[:cut], link[cut:]
    if kind == "mention" and j > 0:
        W = link
    text = P + W
    table = _table_ascii_tail(R, link)
    off = units(R) if j < 0 else units(R) + j
    base = _links(text, table, off, L, kind)
    moves = []
    for what, d in MOVES:
        o2, l2 = (off + d, L - d) if what == "start" else (off, L + d)
        if _links(text, table, o2, l2, kind) != base:
            moves.append((what, d))
    return _msg(text, [(off, L, kind, "")], channel=rng.randrange(3)), kind, tuple(moves)


def _links(text, table, off, L, kind):
    return go_rules.extract_links(text, [(off, L, kind, b"")], utf16=lambda s, o, l: map16(table, len(s), o, l))


def moved(m: Message, what: str, d: int) -> Message:
    """m with its one entity's start (end fixed) or end moved by d units"""
    e = m.text.entities[0]
    o, l = (e.offset + d, e.length - d) if what == "start" else (e.offset, e.length + d)
    return Message(content_type=m.content_type, text=FormattedText(m.text.text, [TextEntity(o, l, e.type, e.url)]),
                   channel=m.channel)


def _mapping_extra(rng):
    """surrogate halves, zero / negative lengths, int32 wrap, and the ASCII-prefix shortcut's bound"""
    out = []
    emo = "😀".encode()
    for a in (0, 3, 127, 126, 511, 1023):
        t = _letters(rng, a) + emo + _letters(rng, 40)
        for kind in ("mention", "url"):
            out.append(_msg(t, [(a + 1, 6, kind, "")]))        # start inside the pair, stop reachable: FAILED
            out.append(_msg(t, [(a + 1, 0, kind, "")]))        # ... zero length: stop inside the pair too, never reached
            out.append(_msg(t, [(a + 1, 10 ** 6, kind, "")]))  # ... stop past the end: never reached
            out.append(_msg(t, [(a, 1, kind, "")]))            # stop inside the pair: the slice runs to the end
            out.append(_msg(t, [(a + 2, 0, kind, "")]))        # zero length on a rune start: (i, i), not FAILED
            out.append(_msg(t, [(a, 0, kind, "")]))
            out.append(_msg(t, [(a + 8, -3, kind, "")]))       # negative length
            out.append(_msg(t, [(a + 2, -1, kind, "")]))
            out.append(_msg(t, [(2 ** 31 - 3, 10, kind, "")]))  # offset + length wraps int32
            out.append(_msg(t, [(a + 2, 2 ** 31 - 1, kind, "")]))
            out.append(_msg(t, [(-1, a + 4, kind, "")]))
    for F in (15, 16, 17, 511, 512, 513, 1023, 1024, 1025):  # the first non-ASCII byte at F
        for x in (b"\xc3\xa9", b"\xe4\xb8\xad", emo, b"\xff"):
            for kind in ("mention", "url"):
                head = _fill(rng, F - 14) + (b"t.me/" if kind == "url" else b"@@@@@") + _letters(rng, 9)
                t = head + x + _letters(rng, 30)
                for d in (-1, 0, 1, 2):  # stop = ascii_prefix + d
                    for L in (6, 14):
                        out.append(_msg(t, [(F + d - L, L, kind, "")]))
                out.append(_msg(t, [(F - 14, 14, kind, ""), (F + 1, 5, kind, "")]))
    return out


def _bounds(rng):
    """records whose link upper bound (entities of the three kinds + t.me/ hits) is exactly their link count, entity
    counts 1-70, more than 32 links, OTHER entities interleaved"""
    out, serial = [], [0]

    def nm():
        serial[0] += 1
        return b"n%04d" % serial[0] + _letters(rng, rng.randrange(1, 10))

    for k in range(1, 71):
        t, ents = bytearray(), []
        for i in range(k):
            kind = ("mention", "url", "text_url", "bold")[i % 4] if k > 3 else ("mention", "url", "text_url")[i % 3]
            if kind == "mention":
                s = b"@" + nm()
                ents.append((len(t), len(s), kind, ""))
            elif kind == "url":  # the entity cuts the name, so the plaintext scan finds a longer, different one
                s = b"t.me/" + nm() + b"long"
                ents.append((len(t), len(s) - 2, kind, ""))
            elif kind == "text_url":
                s = b"~"
                ents.append((len(t), 1, kind, b"https://t.me/" + nm()))
            else:
                s = b"bold"
                ents.append((len(t), 4, kind, ""))
            t += s + b" "
        for tail in range(1, 16):  # the last t.me/ in the text's last partial lane
            if k % 15 == tail % 15:
                t += _fill(rng, tail) + b" t.me/" + nm()
                if len(t) % 16 == 0:
                    t += b"z"
        out.append(_msg(bytes(t), ents, channel=rng.randrange(3)))
    for n in range(54, 64):  # one t.me/ whose '/' lies in the text's last, partial lane; with and without entities
        t = _fill(rng, n - 11) + b" t.me/" + _letters(rng, 5)
        out.append(_msg(t))
        out.append(_msg(t, [(0, 1, "bold", "")]))
        out.append(_msg(b"@" + nm() + t, [(0, 10, "mention", "")]))
    for n in (1, 2, 3, 5, 13, 16, 17, 31, 32, 33):  # plaintext only, the last hit in a partial lane
        t = b" ".join(b"t.me/" + nm() for _ in range(n))
        out.append(_msg(t + b"x" * rng.randrange(0, 3)))
    for n in (33, 40, 66):  # more than 32 links, then repeats of earlier ones (the dedup loop passes 32)
        names = [nm() for _ in range(n)]
        t = b" ".join(b"t.me/" + x for x in names) + b" " + b" ".join(b"t.me/" + x.upper() for x in names[::-3])
        ents = [(0, 5 + len(names[0]), "url", ""), (0, 1, "bold", ""), (0, 1, "text_url", b"t.me/" + names[-1])]
        out.append(_msg(t, ents))
        out.append(_msg(t))
    return out


def _dedup_flags(rng):
    """first source wins over the same name in mixed case; a 32-byte name and its 31-byte prefix; filter reasons; the
    self flag (case-sensitive, as in Go) and an empty channel name"""
    out = []
    t = b"@SameName1 t.me/SAMENAME1 t.me/samename1"
    e_m, e_u, e_t = (0, 10, "mention", ""), (11, 14, "url", ""), (0, 1, "text_url", b"t.me/sAmEnAmE1")
    for ents in ([e_t, e_m, e_u], [e_m, e_t, e_u], [e_u, e_m, e_t], [e_m, e_u], []):
        out.append(_msg(t, ents))
    n32 = _name(rng, 32)
    out.append(_msg(b"t.me/" + n32 + b" t.me/" + n32[:31] + b" t.me/" + n32[:31].upper()))
    out.append(_msg(b"t.me/" + n32[:31] + b" t.me/" + n32 + b"zz"))
    out.append(_msg(b"t.me/ends_with_ t.me/some_bot t.me/somebot t.me/someBoT t.me/" + _name(rng, 29) + b"bot t.me/" +
                    _name(rng, 28) + b"_BOT t.me/robotx t.me/bot_x t.me/abcd_ t.me/bots1",
                    [(0, 1, "text_url", b"t.me/text_bot"), (0, 14, "url", "")]))
    for ch in range(3):
        out.append(_msg(b"t.me/selfchan1 t.me/SelfChan1 t.me/MixedCase_chan t.me/mixedcase_chan t.me/other_chan",
                        [(0, 1, "text_url", b"t.me/SELFCHAN1")], channel=ch))
    return out


def _shapes(rng):
    """one set of link texts as all seven carriers and a type without links, nil captions, records skipped by
    min_post_date or panicking while they hold links, outlink lists of 4 and 5 names of 32 bytes"""
    out = []
    texts = [(b"t.me/shape_one @shapetwo", [(15, 9, "mention", "")]), (b"see https://t.me/shape_three", []),
             (b"\xc3\xa9 @shape_four t.me/x", [(2, 11, "mention", ""), (0, 1, "text_url", b"t.me/shape_five")])]
    for t, ents in texts:
        for ct in CARRIERS + ("messageSticker", "messagePoll"):
            out.append(_msg(t, ents, ct=ct, alt="alt text", media="MEDIA1"))
        out.append(_msg(None, ct="messagePhoto", media="m"))
        out.append(_msg(t, ents, date=1_600_000_000))
        out.append(_msg(t, ents, panics=True))
    for k in (3, 4, 5, 6):
        names = [_name(rng, 32) for _ in range(k)]
        out.append(_msg(b" ".join(b"t.me/" + x for x in names), channel=rng.randrange(3)))
    return out


# ---- the batch --------------------------------------------------------------------------------------------------------
def _layout(rng, ent, plain):
    """records in groups of 32: every one with entities, none, only lane 0, only lane 31, alternate ones, mixed; the
    batch ends with a half-full group"""
    rng.shuffle(ent)
    rng.shuffle(plain)
    out, g = [], 0
    pats = ("all", "none", "lane0", "lane31", "alt")
    while ent or plain:
        pat = pats[(g // 3) % len(pats)] if g % 3 == 0 else "mixed"
        for lane in range(32):
            want = {"all": True, "none": False, "lane0": lane == 0, "lane31": lane == 31, "alt": lane % 2 == 0,
                    "mixed": rng.random() * (len(ent) + len(plain)) < len(ent)}[pat]
            pool = (ent if want else plain) or (plain if want else ent)
            if not pool:
                break
            out.append(pool.pop())
        g += 1
    while len(out) % 32 != 16:
        out.append(_msg(b"pad " + _letters(rng, 4), channel=0))
    return out


@functools.lru_cache(maxsize=None)
def make_link_edges(seed: int):
    rng = random.Random(seed)
    fams = _tme_plain(rng) + _entity_links(rng) + _mapping_extra(rng) + _bounds(rng) + _dedup_flags(rng) + _shapes(rng)
    fams += [m for m, _, _ in mapping_cases(seed)]
    for k, m in enumerate(fams):
        m.id = (k + 1) << 20
        if m.channel < 0:
            m.channel = rng.randrange(3)
        if k % 97 == 5:
            m.date = 1_600_000_000  # before MIN_POST_DATE
    ent = [m for m in fams if m.text is not None and m.text.entities]
    plain = [m for m in fams if m.text is None or not m.text.entities]
    msgs = _layout(rng, ent, plain)
    return pack_telegram(msgs, CHANNELS), msgs, CHANNELS


def link_bound(m: Message) -> int:
    """the parse's reservation for a record: entities of the three kinds + t.me/ occurrences (warp_link_upper_bound)"""
    if m.panics or m.content_type not in CARRIERS or m.text is None:
        return 0
    t = _b(m.text.text)
    return sum(e.type in ("mention", "url", "text_url") for e in m.text.entities) + t.count(b"t.me/")


# ---- coverage accounting ----------------------------------------------------------------------------------------------
def _exact_strips(b: bytes) -> set[int]:
    """128-byte strips of b that warp_load_strip hands to the exact per-byte path: an invalid byte, a lead >= 0xF4,
    C0 / C1, E2 80 (a U+2028/9 candidate), or a sequence carried in from an exact strip"""
    bad, i = set(), 0
    while i < len(b):
        c = b[i]
        r, w = go_rules.go_decode_rune(b, i)
        if c >= 0x80 and (w == 1 or c >= 0xF4 or c in (0xC0, 0xC1) or (c == 0xE2 and b[i + 1:i + 2] == b"\x80")):
            bad.add(i // 128)
        if i // 128 != (i + w - 1) // 128 and i // 128 in bad:
            bad.add((i + w - 1) // 128)
        i += w
    return bad


def _tme_cells(s: bytes, cells: set):
    p = s.find(b"t.me/")
    while p >= 0:
        cells.add(("lane", (p + 4) % 16))
        for e in range(512, len(s) + 1, 512):
            if e - 5 <= p <= e:
                cells.add(("edge", e % 1024 or 1024, p - e))
        run = 0
        while p + 5 + run < len(s) and s[p + 5 + run] in b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789_":
            run += 1
        if run and s[p + 5] in b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ":
            cells.add(("name", min(run, 34)))
            if (p + 5) // 512 != (p + 5 + run - 1) // 512:
                cells.add(("name_across_strip", min(run, 34)))
        p = s.find(b"t.me/", p + 1)


def link_cells(msgs) -> set:
    """the geometry the scanners meet, restated: for every t.me/ of a text, an url slice or a text_url its lane offset
    ('/' mod 16) and strip edge; every candidate name's length; for every mapped entity the branch warp_map_entities
    takes (ASCII shortcut, fast walker, exact strip) and, near the shortcut's bound, stop - ascii_prefix"""
    cells = set()
    for m in msgs:
        if m.text is None or m.content_type not in CARRIERS:
            continue
        t = _b(m.text.text)
        _tme_cells(t, cells)
        if not m.text.entities:
            continue
        table, exact = _table(t), None
        nonascii = next((i for i, c in enumerate(t) if c >= 0x80), len(t))
        for e in m.text.entities:
            if e.type == "text_url":
                _tme_cells(_b(e.url), cells)
                continue
            if e.type not in ("mention", "url"):
                continue
            stop = e.offset + e.length
            if nonascii < len(t) and -1 <= stop - nonascii <= 2:
                cells.add(("ascii_stop", stop - nonascii))
            if e.offset >= 0 and e.length >= 0 and stop <= nonascii:
                cells.add(("map", "ascii"))
            else:
                exact = _exact_strips(t) if exact is None else exact
                st, en = map16(table, len(t), e.offset, e.length)
                at = en if en > 0 and (st, en) != (0, 0) else max(st, 0)
                cells.add(("map", "exact" if min(at, max(len(t) - 1, 0)) // 128 in exact else "fast"))
            st, en = map16(table, len(t), e.offset, e.length)
            if e.type == "url" and 0 <= st < en <= len(t):
                _tme_cells(t[st:en], cells)
    return cells
