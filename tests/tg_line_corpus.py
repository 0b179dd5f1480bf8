"""Telegram Post line records built by rule at the edges of the GPU line (make_line_edges), the cells they must reach
(line_edge_cells, line_cells) and the bytes the lane emitter leaves to the other emit kernels (lane_left_bytes).

The lane emitter (tg_lane.cuh) renders five numbers into 16 / 32-byte blocks of its field row, copies the channel job's
four pre-rendered segments (tg_walk.cuh size_tg_chan / emit_tg_chan: escaped username | escaped name | "quoted title" |
channel_data tail, each 16-byte aligned and zero padded) in 16-byte blocks, copies the record's short clean strings,
renders "simple" reaction maps itself (<= 6 entries, clean keys of 1..8 bytes, duplicates last-wins by a big-endian
8-byte compare) and up to four outlinks.  Everything else goes to the esc / maps kernels.  The page kernel renders the
same line its own way, one warp per record.  The records below sit on the boundaries of each of those rules."""
import collections
import random
import re

import go_rules
from distributed_crawler_b200.pack import Channel, Comment, FormattedText, Message
from gm_corpus import I64_MAX, I64_MIN, INT_EDGES

I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
M20 = 1 << 20  # message.Id / 1048576: the message number of post_link and post_uid
# ids: the int64 ends, the truncation toward zero around +-2^20, and m * 2^20 + r for every msgno digit count (the
# largest msgno, I64_MAX / 2^20, has 13 digits: 10^13 * 2^20 is outside int64)
ID_EDGES = sorted({I64_MIN, I64_MIN + 1, -1, 0, 1, M20 - 1, M20, M20 + 1, -(M20 - 1), -M20, -(M20 + 1),
                   (1 << 53) + M20 - 1, (1 << 62) + M20 - 1, (1 << 63) - M20, I64_MAX} |
                  {s * (m * M20 + r) for k in range(1, 14) for m in (10 ** k - 1, 10 ** k) for r in (0, M20 - 1)
                   for s in (1, -1) if I64_MIN <= s * (m * M20 + r) <= I64_MAX})
I32_EDGES = [I32_MIN, I32_MIN + 1, -1, 0, I32_MAX] + [v for k in range(1, 10) for v in (10 ** k - 1, 10 ** k)]
DATES = (I32_MIN, I32_MAX, 0)
ALBUMS = (-1, I64_MIN)  # any non-zero album id gives "?single"
LANE_TEXT_MAX = 512     # tg_lane.cuh: longer or escaped strings go to the esc kernels
LANE_MAP_MAX = 6        # tg_walk.cuh: larger maps go to the maps kernel
LANE_LINKS_MAX = 4      # tg_lane.cuh: longer outlink lists go to the maps kernel
PAGE_MAX_RECS = 8192    # tgingest.cu: the largest batch the one-launch page kernel takes
PAGE_MAX_IN_BYTES = 4 << 20

# ---- channel strings --------------------------------------------------------------------------------------------------
CHAN_LENGTHS = (0, 1, 15, 16, 17, 31, 32, 33, 127, 128, 129, 255, 256, 257, 511, 512, 513, 4095, 4096, 4097, 65535)
CHAN_KINDS = ("clean", "utf8-2", "utf8-3", "utf8-4") + tuple("esc@%d" % k for k in range(16)) + ("lt", "invalid_end", "u2028")
CHAN_ROLES = ("title", "name", "username")
SEG_KINDS = ("clean", "utf8-2", "utf8-3", "utf8-4", "esc", "lt", "invalid_end", "u2028")  # kinds of the tuned segments
_RUNE = {2: "é".encode(), 3: "中".encode(), 4: "😀".encode()}
_CLEAN = (b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789 .,-_:/" * 4)[:256]
_ASCII_ESC = b'"\\<>&\n\t\x01\x1f'
_CUT = (b"\xe2\x80", b"\xf0\x9f\x98", b"\xc3", b"\xff", b"\xed\xa0")
_ASCII_GROWS = re.compile(rb'[\x00-\x1f"\\<>&]')  # ASCII that encoding/json escapes


def _clean(rng, n: int) -> bytes:
    return rng.randbytes(n).translate(_CLEAN)


def _last_block(n: int) -> int:
    """start of the last 16-byte block of an n-byte string"""
    return (n - 1) // 16 * 16


def chan_kind_fits(kind: str, n: int) -> bool:
    if kind == "clean":
        return True
    if kind.startswith("utf8-"):
        return n >= int(kind[-1])
    if kind.startswith("esc@"):
        return n and _last_block(n) + int(kind[4:]) < n
    return n >= (3 if kind == "u2028" else 1)


def chan_string(rng, n: int, kind: str) -> bytes:
    """n raw bytes of one kind: clean ASCII; whole 2/3/4-byte runes (ASCII in front where they do not fit); one ASCII
    escape at offset k of the last 16-byte block; all '<' (6x when escaped); invalid UTF-8 that ends the string; one
    U+2028"""
    if kind.startswith("utf8-"):
        r = _RUNE[int(kind[-1])]
        return _clean(rng, n % len(r)) + r * (n // len(r))
    out = bytearray(_clean(rng, n))
    if kind.startswith("esc@"):
        out[_last_block(n) + int(kind[4:])] = rng.choice(_ASCII_ESC)
    elif kind == "lt":
        out = bytearray(b"<" * n)
    elif kind == "invalid_end":
        cut = _CUT[n % len(_CUT)][:n]
        out[n - len(cut):] = cut
    elif kind == "u2028":
        p = rng.randrange(n - 2)
        out[p:p + 3] = "\u2028".encode()
    return bytes(out)


def esc_len(b: bytes) -> int:
    """encoding/json's escaped length of b, without the quotes"""
    return len(go_rules.go_json_string(b)) - 2


def _tuned(rng, kind: str, approx: int, extra: int, cls: int) -> bytes:
    """a string of the kind (SEG_KINDS) of about `approx` bytes whose escaped length + extra is 16k + cls (cls in -1, 0,
    1): clean ASCII in front pads it"""
    body = chan_string(rng, approx, "esc@3" if kind == "esc" else kind)
    pad = (cls - esc_len(body) - extra) % 16
    return _clean(rng, pad) + body


def cdata(ch: Channel) -> bytes:
    """the channel job's fourth segment: ,"channel_name": ... "published_at":"0001-01-01T00:00:00Z"}"""
    t, nm = go_rules.go_json_string(go_rules._bs(ch.title)), go_rules.go_json_string(go_rules._bs(ch.name))[1:-1]
    return (b',"channel_name":' + t + b',"channel_description":"","channel_profile_image":"","channel_engagement_data":'
            b'{"follower_count":%d,"following_count":0,"like_count":0,"post_count":%d,"views_count":%d,"comment_count":0,'
            b'"share_count":0},"channel_url_external":"https://t.me/c/%s","channel_url":"https://t.me/c/%s","country_code":"",'
            b'"published_at":"0001-01-01T00:00:00Z"}' % (ch.member_count, ch.post_count, ch.view_count, nm, nm))


def chan_segments(ch: Channel) -> dict:
    """the escaped length of each of the channel job's segments"""
    return {"username": esc_len(go_rules._bs(ch.username)), "name": esc_len(go_rules._bs(ch.name)),
            "title": esc_len(go_rules._bs(ch.title)) + 2, "cdata": len(cdata(ch))}


def _count_for_cdata(ch: Channel, cls: int, k: int) -> int:
    """a member count from the int64 edges that puts the cdata segment on 16k + cls"""
    for j in range(len(INT_EDGES)):
        v = INT_EDGES[(k + j) % len(INT_EDGES)]
        ch.member_count = v
        if (len(cdata(ch)) - cls) % 16 == 0:
            return v
    raise AssertionError("no member count fits")


def edge_channels(rng) -> list[Channel]:
    """row 0 an ordinary channel; then every (length, kind) of the three strings (kinds rotated over the roles); then
    strings tuned so that each segment's escaped length is 16k - 1, 16k and 16k + 1 for every kind, short and longer
    than the lane's 256-byte staging row"""
    chans = [Channel("Test Channel", "testchannel", "testchannel", 10, 20, 30)]
    k = 0
    for n in CHAN_LENGTHS:
        kinds = [x for x in CHAN_KINDS if chan_kind_fits(x, n)]
        for j in range(len(kinds)):
            s = [chan_string(rng, n, kinds[(j + r) % len(kinds)]) for r in range(3)]
            chans.append(Channel(s[0], s[1], s[2], INT_EDGES[k % len(INT_EDGES)], INT_EDGES[(k + 7) % len(INT_EDGES)],
                                 INT_EDGES[(k + 13) % len(INT_EDGES)]))
            k += 1
    for approx in (40, 300):
        for kind in SEG_KINDS:
            for cls in (-1, 0, 1):
                ch = Channel(_tuned(rng, kind, approx, 2, cls), _tuned(rng, kind, approx, 0, cls),
                             _tuned(rng, kind, approx // 4, 0, cls), 0, INT_EDGES[k % len(INT_EDGES)],
                             INT_EDGES[(k + 5) % len(INT_EDGES)])
                _count_for_cdata(ch, cls, k)
                chans.append(ch)
                k += 1
    return chans


# ---- the record's other strings -------------------------------------------------------------------------------------
REC_LENGTHS = {"handle": (0, 1, 15, 16, 17, 511, 512, 513, 4096, 65535),
               "media": (0, 1, 15, 16, 17, 511, 512, 513, 4096, 65535),
               "alt-desc": (0, 1, 15, 16, 17, 511, 512, 513, 4096, 65535, 65536, 100000),
               "alt-type": (1, 15, 16, 17, 511, 512, 513, 4096, 65535, 65536, 100000)}  # an empty alt is the type's name
REC_KINDS = ("clean", "multibyte", "nl", "lt", "quote", "invalid", "u2028")
ALT_DESC_TYPES = ("messageAnimatedEmoji", "messagePoll", "messageGiveaway", "messagePaidMedia", "messageDocument")
MEDIA_TYPES = ("messageVideo", "messageVideoNote", "messageDocument")
UNKNOWN_TYPES = ("messageLocation", "messageContact", "messageDice")


def rec_kind_fits(kind: str, n: int) -> bool:
    return kind == "clean" or n >= {"multibyte": 2, "u2028": 3}.get(kind, 1)


def rec_string(rng, n: int, kind: str) -> bytes:
    """n raw bytes: clean ASCII; clean 2/3/4-byte runes; one '\\n', '<' or '"'; invalid UTF-8; one U+2028"""
    if kind == "multibyte":
        out = bytearray()
        while len(out) < n:
            r = _RUNE[rng.choice((2, 3, 4))]
            out += r if len(out) + len(r) <= n else b"a" * (n - len(out))
        return bytes(out)
    out = bytearray(_clean(rng, n))
    p = rng.choice((0, n - 1, rng.randrange(n))) if n else 0
    if kind in ("nl", "lt", "quote"):
        out[p] = {"nl": 10, "lt": 60, "quote": 34}[kind]
    elif kind == "invalid":
        out[p] = rng.choice((0xFF, 0xC3, 0x80, 0xED))
    elif kind == "u2028":
        p = min(p, n - 3)
        out[p:p + 3] = "\u2028".encode()
    return bytes(out)


def _kind_of(s: bytes) -> str:
    """the REC_KINDS kind of a string of the corpus (rec_string's rules read back)"""
    if b"\xe2\x80\xa8" in s:
        return "u2028"
    if s.decode("utf-8", "replace") != s.decode("utf-8", "ignore"):
        return "invalid"
    for kind, c in (("nl", b"\n"), ("lt", b"<"), ("quote", b'"')):
        if c in s:
            return kind
    return "clean" if s.isascii() else "multibyte"


# ---- maps and lists ---------------------------------------------------------------------------------------------------
def _dup_maps() -> list:
    """6-entry lane maps where entry j repeats the key of entry i (i < j): the last entry must win"""
    keys = [b"k", b"ka", b"kz", b"kb\xc3\xa9", b"\x7fq", b"z"]
    out = []
    for j in range(1, 6):
        for i in range(j):
            ks = list(keys)
            ks[j] = ks[i]
            out.append(("dup %d %d" % (i, j), list(ks)))
    return out


def edge_maps() -> list:
    """(name, keys) of the reaction maps; counts are dealt from I32_EDGES"""
    maps = [("empty", [])]
    for n in range(1, 9):  # 1..8 distinct clean keys of 1..8 bytes
        maps.append(("entries %d" % n, [bytes([0x61 + j]) * (1 + (j + n) % 8) for j in range(n)]))
    maps += [("lens 1-6", [b"a", b"bb", b"ccc", b"dddd", b"eeeee", b"ffffff"]), ("lens 7-8", [b"ggggggg", b"hhhhhhhh"]),
             ("lens 9", [b"iiiiiiiii", b"a"]),
             ("high byte at 0", [b"\x7f", "é".encode(), b"z", "😀".encode(), "中".encode()]),
             ("high byte at 3", [b"abcz", "abcé".encode(), b"abc\x7f", b"abc"]),
             ("high byte at 6", ["abcdefé".encode(), b"abcdefzz", b"abcdef\x7fz", b"abcdefg"]),
             ("8-byte prefix, lane", [b"abcdefgh", b"abcdefgi", b"abcdefg"]),
             ("8-byte prefix, 9 bytes", [b"abcdefgh", b"abcdefghi", b"abcdefgh"]),
             ("empty key", [b"", b"a"]), ("escaped keys", [b'"', b"<", b"a\\", b"\n"]),
             ("escape alike", [b"\xff", b"\xfe", "\ufffd".encode()]),
             ("u2028 and its text", [b"\xe2\x80\xa8", b"\\u2028", b"u2028"])]
    maps += _dup_maps()
    return maps


def map_is_simple(keys) -> bool:
    """the lane emitter's rule (kernels.cuh tg_size_lane_kernel): <= 6 entries, every key 1..8 bytes and unescaped"""
    return len(keys) <= LANE_MAP_MAX and all(1 <= len(k) <= 8 and esc_len(k) == len(k) for k in keys)


def _link_name(rng, n: int) -> bytes:
    return bytes([rng.choice(b"abcdefghijklmnopqrstuvwxyz")]) + _clean(rng, n - 1).translate(
        (b"abcdefghijklmnopqrstuvwxyz0123456789_" * 7)[:256])


def outlink_text(rng, k: int) -> bytes:
    """a text with k distinct t.me/ names, 31 and 32 bytes long among them"""
    names = [_link_name(rng, (31, 32, 5, 12)[j % 4]) for j in range(k)]
    return b"see " + b" ".join(b"t.me/" + x for x in names) + b" end"


# ---- the corpus ---------------------------------------------------------------------------------------------------------
def _record_edges(rng) -> list[dict]:
    """one dict of Message fields per edge record (the numbers are dealt later)"""
    out = []
    for role, lens in REC_LENGTHS.items():
        j = 0
        for n in lens:
            for kind in REC_KINDS:
                if not rec_kind_fits(kind, n):
                    continue
                s = rec_string(rng, n, kind)
                if role == "handle":
                    out.append(dict(handle=s, text=FormattedText(b"h")))
                elif role == "media":
                    ct = MEDIA_TYPES[j % 3]
                    out.append(dict(content_type=ct, media=s, text=FormattedText(b"cap") if ct == "messageVideo" else None,
                                    alt=b"file.pdf" if ct == "messageDocument" else b""))
                elif role == "alt-desc":
                    out.append(dict(content_type=ALT_DESC_TYPES[j % 5], alt=s, text=None))
                else:
                    out.append(dict(content_type=UNKNOWN_TYPES[j % 3], alt=s, text=None))
                j += 1
    for name, keys in edge_maps():
        out.append(dict(reactions=keys, text=FormattedText(name)))
        out.append(dict(comments=[Comment(b"c", None), Comment(name, keys, handle=b"h"), Comment(b"", [])],
                        text=FormattedText(b"comments")))
    out += [dict(comments=None), dict(comments=[]), dict(comments=[Comment("only", [(b"x", 1)])])]
    for k in range(7):
        for _ in range(2):
            out.append(dict(text=FormattedText(outlink_text(rng, k))))
    return out


def make_line_edges(seed: int = 1):
    """(messages, channels): the edge records and the edge channels, deterministic per seed.  Records reference the
    channel rows in order (a page is a slice of consecutive rows); runs of one channel start at every lane of a warp, and
    some fill a whole warp.  Channels with a string longer than 4 097 bytes get runs of one or two records (their lines
    are up to 2.7 MB)"""
    rng = random.Random(0x7E1 + seed)
    chans = edge_channels(rng)
    edges = _record_edges(rng)
    lens = (1, 2, 3, 5, 7, 32, 1, 4, 33, 1, 6)
    chan_of = []
    for c, ch in enumerate(chans):
        big = max(len(go_rules._bs(x)) for x in (ch.title, ch.name, ch.username)) > 4097
        chan_of += [c] * (1 + c % 2 if big else lens[(c + seed) % len(lens)])
    n = len(chan_of)
    assert len(edges) < n // 2
    slots = set(rng.sample(range(n), len(edges)))
    edge_iter = iter(edges)
    maps = edge_maps()
    msgs, nc = [], 0
    for i in range(n):
        e = dict(next(edge_iter)) if i in slots else {}
        if not e:  # filler: a short text, sometimes a link, a small map
            keys = maps[i % len(maps)][1] if i % 5 == 0 else []
            e = dict(text=FormattedText(b"msg %d t.me/chan%04d" % (i, i % 300) if i % 3 == 0 else b"m%d" % i), reactions=keys)
        keys = e.pop("reactions", [])
        e["reactions"] = [(k, I32_EDGES[(i + j) % len(I32_EDGES)]) for j, k in enumerate(keys)]
        if e.get("comments"):  # every comment takes the next view / reply count edges
            cs = []
            for c in e["comments"]:
                cs.append(Comment(c.text, None if c.reactions is None else
                                  [(k, I32_EDGES[(i + j + 3) % len(I32_EDGES)]) for j, k in enumerate(c.reactions)],
                                  I32_EDGES[nc % len(I32_EDGES)], I32_EDGES[(nc + 7) % len(I32_EDGES)], c.handle))
                nc += 1
            e["comments"] = cs
        e.setdefault("text", FormattedText(b"m"))
        e.setdefault("comments", [])
        msgs.append(Message(id=ID_EDGES[i % len(ID_EDGES)], chat_id=INT_EDGES[i % len(INT_EDGES)],
                            date=DATES[i % 3] if i % 4 == 0 else 1_700_000_000 + i,
                            media_album_id=(0, ALBUMS[0], 0, ALBUMS[1])[i % 4],
                            view_count=I32_EDGES[i % len(I32_EDGES)], share_count=I32_EDGES[(i + 5) % len(I32_EDGES)],
                            channel=chan_of[i], **e))
    return msgs, chans


def pages(msgs, chans, max_recs: int = PAGE_MAX_RECS, max_bytes: int = PAGE_MAX_IN_BYTES - (256 << 10)):
    """[a, b) ranges of consecutive records whose slice of the packed batch fits one page: <= max_recs records and
    about <= max_bytes of input (records reference the channel rows in order)"""
    def rec_bytes(m):
        b = sum(len(go_rules._bs(x)) for x in (m.alt, m.media, m.handle)) + (len(go_rules._bs(m.text.text)) if m.text else 0)
        b += sum(len(go_rules._bs(k)) + 12 for k, _ in m.reactions)
        for c in m.comments or []:
            b += 32 + len(go_rules._bs(c.text)) + len(go_rules._bs(c.handle)) + sum(len(go_rules._bs(k)) + 12 for k, _ in c.reactions or [])
        return b + 80
    def chan_bytes(c):
        return 40 + sum(len(go_rules._bs(x)) for x in (c.title, c.name, c.username))
    out, a, size, last = [], 0, 0, None
    for i, m in enumerate(msgs):
        add = rec_bytes(m) + (chan_bytes(chans[m.channel]) if m.channel != last else 0)
        if i > a and (i - a >= max_recs or size + add > max_bytes):
            out.append((a, i))
            a, size = i, rec_bytes(m) + chan_bytes(chans[m.channel])
        else:
            size += add
        last = m.channel
    out.append((a, len(msgs)))
    return out


def with_table(msgs, chans, rows: int):
    """the records over a channel table of `rows` rows: the edge rows no longer than 513 bytes, repeated"""
    short = [c for c in chans if max(len(go_rules._bs(x)) for x in (c.title, c.name, c.username)) <= 513]
    table = [short[j % len(short)] for j in range(rows)]
    out = [Message(**{**m.__dict__, "channel": (i * rows) // len(msgs)}) for i, m in enumerate(msgs)]
    return out, table


# ---- what the lane emitter leaves to the other kernels ------------------------------------------------------------------
_LINK_CARRIERS = ("messageText", "messageVideo", "messagePhoto", "messageAnimation", "messageDocument", "messageAudio",
                  "messageVoiceNote")
_KNOWN = ("messageText", "messageVideo", "messagePhoto", "messageAnimation", "messageAnimatedEmoji", "messagePoll",
          "messageGiveaway", "messagePaidMedia", "messageSticker", "messageGiveawayWinners", "messageGiveawayCompleted",
          "messageVideoNote", "messageDocument", "messageAudio", "messageVoiceNote", "none")


def record_strings(m) -> dict:
    """the record's strings the line holds, by role: desc, media, handle, alt (alt only as the post_type of a type
    ParseMessage has no case for, as the packer stores it)"""
    ct, b = m.content_type, go_rules._bs
    out = {"handle": b(m.handle)}
    if ct in ("messageText", "messageVideo", "messagePhoto", "messageAnimation"):
        out["desc"] = b(m.text.text) if m.text is not None else b""
    elif ct in ALT_DESC_TYPES:
        out["desc"] = b(m.alt)
    if ct in ("messageVideoNote", "messageDocument") or (ct == "messageVideo" and m.video_shape == "ok"):
        out["media"] = b(m.media)
    if ct not in _KNOWN:
        out["alt"] = b(m.alt) or ct.encode()
    return out


def lane_left_bytes(m, ch, links=None) -> int:
    """The line bytes of one emitted record that the lane emitter leaves to the esc and maps kernels: the escaped length
    of each of desc / media / handle / alt that needs escaping or is longer than 512 bytes; the whole comment list when
    it is neither nil nor empty; the whole reaction map when it is not simple (map_is_simple); the outlink names when
    there are more than four.  This is the lane routing rule of tg_lane.cuh and the size pass, restated: a pull request
    that changes which kernel writes what changes it here, and only here.  links: the record's outlinks (go_rules)."""
    left = 0
    for s in record_strings(m).values():
        x = esc_len(s)
        if x != len(s) or len(s) > LANE_TEXT_MAX:
            left += x
    if m.comments:
        left += len(go_rules._marshal([[("text", go_rules._bs(c.text)),
                                        ("reactions", None if c.reactions is None else {go_rules._bs(k): v for k, v in c.reactions}),
                                        ("view_count", c.view_count), ("reply_count", c.reply_count),
                                        ("handle", go_rules._bs(c.handle))] for c in m.comments]))
    keys = [go_rules._bs(k) for k, _ in m.reactions]
    if keys and not map_is_simple(keys):
        left += len(go_rules._marshal({k: v for k, v in ((go_rules._bs(k), v) for k, v in m.reactions)}))
    if links is not None and len(links) > LANE_LINKS_MAX:
        left += len(go_rules._marshal([go_rules._bs(x) for x in links])) - 2  # the brackets are the lane's
    return left


# ---- coverage -------------------------------------------------------------------------------------------------------
def line_cells(msgs, chans) -> set:
    """the cells the records reach"""
    cells, maps = set(), edge_maps()
    for m in msgs:
        cells |= {("id", m.id), ("chat_id", m.chat_id), ("view_count", m.view_count), ("share_count", m.share_count),
                  ("date", m.date)}
        ch = chans[m.channel]
        if m.media_album_id in ALBUMS and go_rules._bs(ch.username):
            cells.add(("album", m.media_album_id))
        for _, v in m.reactions:
            cells.add(("reaction count", v))
        for c in m.comments or []:
            cells |= {("comment view_count", c.view_count), ("comment reply_count", c.reply_count)}
        for role, s in record_strings(m).items():
            role = {"desc": "alt-desc" if m.content_type in ALT_DESC_TYPES else "desc", "alt": "alt-type"}.get(role, role)
            if role == "alt-desc":
                cells.add(("alt-desc type", m.content_type))
            if role == "media":
                cells.add(("media type", m.content_type))
            if role in REC_LENGTHS and len(s) in REC_LENGTHS[role]:
                lane = esc_len(s) == len(s) and len(s) <= LANE_TEXT_MAX
                cells.add((role, len(s), _kind_of(s), "lane" if lane else "esc"))
        keys = [go_rules._bs(k) for k, _ in m.reactions]
        cells.add(("map entries", len(keys), "lane" if map_is_simple(keys) else "maps"))
        for k in keys:
            cells.add(("map key bytes", len(k)))
        cells |= {("map", name) for name, ks in maps if keys == ks}
        cells.add(("comments", "nil" if m.comments is None else "empty" if not m.comments else "filled"))
        for c in m.comments or []:
            ks = None if c.reactions is None else [go_rules._bs(k) for k, _ in c.reactions]
            cells.add(("comment map", "nil" if ks is None else "empty" if not ks else "lane" if map_is_simple(ks) else "maps"))
        if m.text is not None and m.content_type in _LINK_CARRIERS:
            got = go_rules.extract_links(go_rules._bs(m.text.text), [])
            if got is not None:
                cells.add(("outlinks", len(got)))
                cells |= {("outlink name bytes", len(x)) for x, _ in got if len(x) in (31, 32)}
    runs = collections.defaultdict(list)
    for i, m in enumerate(msgs):
        runs[m.channel].append(i)
    for c, rs in runs.items():
        cells.add(("channel run starts at lane", rs[0] % 32))
        if any(r % 32 == 0 and r + 31 in rs for r in rs):
            cells.add(("channel fills a warp",))
    for ch in chans:
        for role in CHAN_ROLES:
            s = go_rules._bs(getattr(ch, role))
            if len(s) in CHAN_LENGTHS:
                cells |= {("channel", role, len(s), k) for k in _chan_kinds(s)}
        seg = chan_segments(ch)
        for role in CHAN_ROLES:
            cls = (seg[role] + 1) % 16 - 1
            if cls in (-1, 0, 1):
                cells |= {("segment", role, cls, k) for k in _chan_kinds(go_rules._bs(getattr(ch, role)), tuned=True)}
        cls = (seg["cdata"] + 1) % 16 - 1
        if cls in (-1, 0, 1):
            cells.add(("segment", "cdata", cls))
        for v in (ch.member_count, ch.post_count, ch.view_count):
            cells.add(("channel count", v))
        for role in CHAN_ROLES:
            if not go_rules._bs(getattr(ch, role)):
                cells.add(("empty", role))
    return cells


def _chan_kinds(s: bytes, tuned: bool = False) -> set:
    """the kinds a channel string is (chan_string's rules read back): CHAN_KINDS, or SEG_KINDS with clean ASCII allowed
    in front when tuned"""
    n, out = len(s), set()
    if s.isascii() and esc_len(s) == n:
        out.add("clean")
    body = s.lstrip(_CLEAN) if tuned else s
    for w, r in _RUNE.items():
        rest = body if tuned else body[n % w:]
        if rest and rest == r * (len(rest) // w) and (tuned or body[:n % w].isascii()):
            out.add("utf8-%d" % w)
    grow = [x.start() for x in _ASCII_GROWS.finditer(s)] if s.isascii() else []
    if len(grow) == 1:
        if tuned:
            out.add("esc")
        elif grow[0] >= _last_block(n):
            out.add("esc@%d" % (grow[0] - _last_block(n)))
    if body and body == b"<" * len(body):
        out.add("lt")
    if n and s.decode("utf-8", "replace").endswith("\ufffd") and not s.endswith("\ufffd".encode()):
        out.add("invalid_end")
    if "\u2028".encode() in s:
        out.add("u2028")
    return out


def line_edge_cells() -> set:
    """the cells make_line_edges must reach"""
    cells = {("id", v) for v in ID_EDGES} | {("chat_id", v) for v in INT_EDGES} | {("date", v) for v in DATES}
    cells |= {(f, v) for f in ("view_count", "share_count", "reaction count", "comment view_count", "comment reply_count")
              for v in I32_EDGES}
    cells |= {("album", v) for v in ALBUMS} | {("channel count", v) for v in INT_EDGES}
    for role, lens in REC_LENGTHS.items():
        for n in lens:
            for kind in REC_KINDS:
                if rec_kind_fits(kind, n):
                    lane = kind in ("clean", "multibyte") and n <= LANE_TEXT_MAX
                    cells.add((role, n, kind, "lane" if lane else "esc"))
    cells |= {("alt-desc type", t) for t in ALT_DESC_TYPES} | {("media type", t) for t in MEDIA_TYPES}
    cells |= {("map entries", k, "lane" if k <= LANE_MAP_MAX else "maps") for k in range(9)} | {("map entries", 2, "maps")}
    cells |= {("map key bytes", k) for k in range(10)} | {("map", name) for name, _ in edge_maps()}
    cells |= {("comments", x) for x in ("nil", "empty", "filled")} | {("comment map", x) for x in ("nil", "empty", "lane", "maps")}
    cells |= {("outlinks", k) for k in range(7)} | {("outlink name bytes", k) for k in (31, 32)}
    cells |= {("channel run starts at lane", k) for k in range(32)} | {("channel fills a warp",)}
    for role in CHAN_ROLES:
        cells |= {("channel", role, n, k) for n in CHAN_LENGTHS for k in CHAN_KINDS if chan_kind_fits(k, n)}
        cells |= {("segment", role, cls, k) for cls in (-1, 0, 1) for k in SEG_KINDS} | {("empty", role)}
    cells |= {("segment", "cdata", cls) for cls in (-1, 0, 1)}
    return cells


def concat_batches(parts):
    """one packed batch holding the records of `parts` (pack.TgBatch) in order, each with its own channel rows.  The
    message reactions of all parts come first (a record's map is a range of one offset array); each part's reaction
    array follows once more for its comments' maps"""
    import numpy as np
    from distributed_crawler_b200.pack import TgBatch, _blob
    recs, ents, reacts, comments, chans = [], [], [], [], []
    ent_off, react_off, comment_off = [np.zeros(1, np.uint32)], [np.zeros(1, np.uint32)], [np.zeros(1, np.uint32)]
    strs, aux, cstrs = [], [], []
    o_str = o_aux = o_cstr = o_ent = o_react = o_comment = o_chan = 0
    o_creact = sum(int(b.react_off[-1]) for b in parts)
    creacts = []
    for b in parts:
        r = b.recs.copy()
        r["str_off"] += o_str
        r["chan_idx"] += o_chan
        e = b.ents.copy()
        e["url_off"] += o_aux
        x = b.reacts.copy()
        x["emoji_off"] += o_aux
        c = b.comments.copy()
        c["text_off"] += o_aux
        c["handle_off"] += o_aux
        c["react_start"] += o_creact
        creacts.append(x)
        o_creact += len(x)
        x = x[:int(b.react_off[-1])]
        ch = b.chans.copy()
        ch["str_off"] += o_cstr
        recs.append(r), ents.append(e), reacts.append(x), comments.append(c), chans.append(ch)
        ent_off.append(b.ent_off[1:] + o_ent), react_off.append(b.react_off[1:] + o_react)
        comment_off.append(b.comment_off[1:] + o_comment)
        strs.append(b.strs.tobytes()), aux.append(b.aux.tobytes()), cstrs.append(b.chan_strs.tobytes())
        o_str, o_aux, o_cstr = o_str + b.strs.size, o_aux + b.aux.size, o_cstr + b.chan_strs.size
        o_ent, o_react, o_comment, o_chan = o_ent + len(b.ents), o_react + len(x), o_comment + len(b.comments), o_chan + len(b.chans)
    cat = np.concatenate
    return TgBatch(recs=cat(recs), strs=_blob(b"".join(strs)), ent_off=cat(ent_off).astype(np.uint32), ents=cat(ents),
                   react_off=cat(react_off).astype(np.uint32), reacts=cat(reacts + creacts), comment_off=cat(comment_off).astype(np.uint32),
                   comments=cat(comments), aux=_blob(b"".join(aux)), chans=cat(chans), chan_strs=_blob(b"".join(cstrs)))
