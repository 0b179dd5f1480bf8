"""Independent pure-Python restatement of the Go standard-library rules the path depends on
(SURVEY.md Appendix A.6), written from the rules — NOT from oracle/tgoracle.c — so that the oracle is
cross-checked by a second implementation.  Pure-Python loops: small inputs only."""
from __future__ import annotations

import datetime as _dt
import functools
import re


def go_decode_rune(b: bytes, i: int):
    """unicode/utf8.DecodeRune: returns (rune, width); (0xFFFD, 1) for invalid."""
    n = len(b) - i
    b0 = b[i]
    if b0 < 0x80:
        return b0, 1
    # python's strict decoder rejects exactly what Go rejects (overlongs, surrogates, > U+10FFFF)
    for w in (2, 3, 4):
        if n >= w:
            try:
                s = b[i:i + w].decode("utf-8")
                if len(s) == 1:
                    return ord(s), w
            except UnicodeDecodeError:
                continue
    return 0xFFFD, 1


_PLAIN = re.compile(rb'[\x20\x21\x23-\x25\x27-\x3b\x3d\x3f-\x5b\x5d-\x7f]+')  # ASCII that encoding/json copies as is


def go_json_string(b: bytes) -> bytes:
    out = bytearray(b'"')
    i = 0
    while i < len(b):
        m = _PLAIN.match(b, i)
        if m:  # a run of bytes copied unchanged (long texts: one slice instead of a loop per byte)
            out += m.group()
            i = m.end()
            continue
        c = b[i]
        if c < 0x80:
            if c >= 0x20 and c not in b'"\\<>&':
                out.append(c)
            elif c in b'"\\':
                out += b"\\" + bytes([c])
            elif c == 8: out += b"\\b"
            elif c == 12: out += b"\\f"
            elif c == 10: out += b"\\n"
            elif c == 13: out += b"\\r"
            elif c == 9: out += b"\\t"
            else: out += b"\\u00%02x" % c
            i += 1
            continue
        r, w = go_decode_rune(b, i)
        if r == 0xFFFD and w == 1:
            out += b"\\ufffd"
        elif r in (0x2028, 0x2029):
            out += b"\\u%04x" % r
        else:
            out += b[i:i + w]
        i += w
    out += b'"'
    return bytes(out)


def go_time_json(sec: int, nsec: int = 0, tz: int = 0):
    t = _dt.datetime(1970, 1, 1) + _dt.timedelta(seconds=sec + tz)
    s = t.strftime("%Y-%m-%dT%H:%M:%S")
    if nsec:
        s += "." + ("%09d" % nsec).rstrip("0")
    if tz == 0:
        s += "Z"
    else:
        a = abs(tz)
        s += ("-" if tz < 0 else "+") + "%02d:%02d" % (a // 3600, a % 3600 // 60)
    return ('"' + s + '"').encode()


def utf16_offset_to_bytes(s: bytes, off: int, length: int):
    """telegramhelper/tdutils.go:55-78 restated literally."""
    i, u16, rune_start = 0, 0, -1
    stop = ((off + length + 2 ** 31) % 2 ** 32) - 2 ** 31
    while i < len(s):
        if u16 == off:
            rune_start = i
        if u16 == stop:
            return rune_start, i
        r, w = go_decode_rune(s, i)
        u16 += 2 if r >= 0x10000 else 1
        i += w
    if rune_start == -1:
        return 0, 0
    return rune_start, len(s)


_CHANNEL_RE = re.compile(rb"(https?://)?t\.me/([a-zA-Z][a-zA-Z0-9_]{4,31})")
_USER_RE = re.compile(rb"(?:@)?([a-zA-Z][a-zA-Z0-9_]{4,31})")
_RESERVED = {b"joinchat", b"addlist", b"addstickers", b"addtheme", b"setlanguage", b"share", b"c", b"s",
             b"iv", b"proxy", b"socks", b"login", b"confirm", b"bg"}


def extract_links(text: bytes | None, entities, aux_urls=None, utf16=None):
    """tdutils.go:897-949 with python's `re` standing in for Go's regexp (both leftmost, greedy; the
    patterns have no alternation whose priority could differ).  Returns [(name, src)] in first-
    insertion order, or None where Go would panic.  utf16(text, off, len) replaces utf16_offset_to_bytes
    (a table lookup for callers that map many entities over one text)."""
    utf16 = utf16 or utf16_offset_to_bytes
    out, seen = [], set()

    def add(name, src):
        name = name.lower()
        if name not in seen:
            seen.add(name)
            out.append((name, src))

    def chan(m, src):
        if m and m.group(2).lower() not in _RESERVED:
            add(m.group(2), src)

    if text is None:
        return out
    for off, ln, typ, url in entities:
        if typ == "text_url":
            chan(_CHANNEL_RE.search(url.encode() if isinstance(url, str) else url), "text_url")
        elif typ in ("mention", "url"):
            st, en = utf16(text, off, ln)
            if st < en and en <= len(text):
                if st < 0:
                    return None
                sl = text[st:en]
                if typ == "mention":
                    m = _USER_RE.search(sl)
                    if m:
                        add(m.group(1), "mention")
                else:
                    chan(_CHANNEL_RE.search(sl), "url")
    for m in _CHANNEL_RE.finditer(text):
        chan(m, "plaintext")
    return out


def filter_username(u: bytes) -> str:
    """username_filter.go:26-68."""
    if len(u) < 5: return "too_short"
    if len(u) > 32: return "too_long"
    if not (65 <= u[0] <= 90 or 97 <= u[0] <= 122): return "invalid_start_char"
    if u[-1:] == b"_": return "ends_with_underscore"
    if not re.fullmatch(rb"[A-Za-z0-9_]+", u): return "invalid_char"
    if u.lower().endswith(b"bot"): return "bot_suffix"
    return ""


_ISO = re.compile(rb"^P(?:(\d+)D)?(?:T(?:(\d+)H)?(?:(\d+)M)?(?:(\d+)S)?)?$")


def parse_iso8601_duration(s: bytes):
    m = _ISO.match(s)
    if not m or s.endswith(b"\n"):
        return None
    tot = 0
    for g, mul in zip(m.groups(), (86400, 3600, 60, 1)):
        if g:
            v = min(int(g), 2 ** 63 - 1)
            tot += v * mul
    tot &= 2 ** 64 - 1
    return tot - 2 ** 64 if tot >= 2 ** 63 else tot


# ---- the whole Telegram Post line, a second time ------------------------------------------------------------------------
# Written from model/data.go:9-139 (field order, pointer / slice / map types), telegramhelper/tdutils.go:380-732
# (ParseMessage), :953-1031 and encoding/json's rules (nil slice / pointer -> null, empty non-nil slice -> [], maps with
# sorted keys, structs in declaration order) — over the host-side Message model (distributed_crawler_b200/pack.py), NOT
# from oracle/tgoracle.c: tests/test_oracle_golden.py compares the two byte for byte on random messages.
def _bs(s) -> bytes:
    if s is None:
        return b""
    return bytes(s) if isinstance(s, (bytes, bytearray)) else str(s).encode("utf-8")


class _Raw(bytes):
    """already JSON"""


@functools.lru_cache(maxsize=None)
def _json_key(k: str) -> bytes:
    """a struct field's JSON key (a fixed set of names)"""
    return go_json_string(k.encode()) + b":"


def _marshal(v) -> bytes:
    if isinstance(v, _Raw):
        return bytes(v)
    if v is None:
        return b"null"
    if isinstance(v, bool):
        return b"true" if v else b"false"
    if isinstance(v, int):
        return str(v).encode()
    if isinstance(v, (bytes, bytearray, str)):
        return go_json_string(_bs(v))
    if isinstance(v, dict):  # map[string]int: keys sorted bytewise
        return b"{" + b",".join(go_json_string(k) + b":" + _marshal(v[k]) for k in sorted(v)) + b"}"
    if isinstance(v, list):
        if v and isinstance(v[0], tuple) and len(v[0]) == 2 and isinstance(v[0][0], str):  # struct: [(json key, value)]
            return b"{" + b",".join(_json_key(k) + _marshal(x) for k, x in v) + b"}"
        return b"[" + b",".join(_marshal(x) for x in v) + b"]"
    raise TypeError(type(v))


_LINK_CARRIERS = ("messageText", "messagePhoto", "messageVideo", "messageDocument", "messageAnimation", "messageAudio",
                  "messageVoiceNote")


def go_div(a: int, b: int) -> int:
    """Go's integer `/`: the quotient truncated toward zero (Python's // floors)"""
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


# the channel strings repeat in every line of the channel: escape each once (a 65 535-byte title of '<' costs a
# per-byte loop)
_chan_json = functools.lru_cache(maxsize=256)(go_json_string)


def _chan_str(prefix: bytes, s: bytes, suffix: bytes = b"") -> _Raw:
    """go_json_string(prefix + s + suffix) for ASCII prefix / suffix: an ASCII byte never joins a UTF-8 sequence, so the
    escaper treats the three parts alike apart"""
    return _Raw(go_json_string(prefix)[:-1] + _chan_json(s)[1:-1] + go_json_string(suffix)[1:])


def telegram_post_line(m, ch, *, crawl_label=b"", created=(1_750_000_000, 0), capture=(1_750_000_001, 0), tz=0,
                       min_post_date=None, zone=None):
    """-> ("skipped" | "failed" | "emitted", line or None, outlinks) for one pack.Message in channel `ch`.  zone =
    (starts, offsets): time.Local as a transition table (tests/zone_oracle.py's rule) instead of the fixed offset tz."""
    if min_post_date is not None and m.date < min_post_date:  # tdutils.go:419-421
        return "skipped", None, []
    if m.panics or (m.content_type == "messageVideo" and m.video_shape == "broken"):  # :395-405 recovered panic
        return "failed", None, []
    ct = m.content_type
    caption = _bs(m.text.text) if m.text is not None else None
    description, media = b"", b""
    if ct in ("messageText", "messageVideo", "messagePhoto", "messageAnimation"):  # :443-487: Text.Text / Caption.Text
        description = caption or b""
    elif ct in ("messageAnimatedEmoji", "messagePoll", "messageGiveaway", "messagePaidMedia", "messageDocument"):
        description = _bs(m.alt)  # emoji / question / prize type / paid-media caption / file name (:489-512, :561-563)
    if (ct == "messageVideo" and m.video_shape == "ok") or ct in ("messageVideoNote", "messageDocument"):
        media = _bs(m.media)      # Remote.Id of the video / video note / document (:188-199, :548-551, :573-576)
    # outlinks (:989-1001): only the seven carriers have a FormattedText; nil text -> []string{}
    links = []
    if ct in _LINK_CARRIERS and caption is not None:
        ents = [(e.offset, e.length, e.type, _bs(e.url)) for e in m.text.entities]
        got = extract_links(caption, ents)
        if got is None:
            return "failed", None, []  # slice bounds panic inside extractLinksFromFormattedText
        links = [n for n, _ in got]
    reactions = {}
    for emoji, cnt in m.reactions:  # :588-600: later entries of a key overwrite
        reactions[_bs(emoji)] = cnt
    if m.comments is None:
        comments = None
    else:
        comments = [[("text", _bs(c.text)),
                     ("reactions", None if c.reactions is None else {_bs(k): v for k, v in c.reactions}),
                     ("view_count", c.view_count), ("reply_count", c.reply_count), ("handle", _bs(c.handle))] for c in m.comments]
    ncomments = 0 if comments is None else len(comments)
    msgno = go_div(m.id, 1048576)  # message.Id/1048576 on an int64 (:1008): exact, truncated toward zero
    user, name, title = _bs(ch.username), _bs(ch.name), _bs(ch.title)
    link = b""
    if user:
        link = _chan_str(b"https://t.me/", user, b"/" + str(msgno).encode() + (b"?single" if m.media_album_id != 0 else b""))
    uid = _chan_str(str(msgno).encode() + b"-", name)
    churl = _chan_str(b"https://t.me/c/", name)
    title = _Raw(_chan_json(title))
    chat = str(m.chat_id).encode()
    known = ("messageText", "messageVideo", "messagePhoto", "messageAnimation", "messageAnimatedEmoji", "messagePoll",
             "messageGiveaway", "messagePaidMedia", "messageSticker", "messageGiveawayWinners", "messageGiveawayCompleted",
             "messageVideoNote", "messageDocument", "messageAudio", "messageVoiceNote")
    # MessageContentType() of a type ParseMessage has no case for travels in Message.alt (pack.py); nil content -> "unknown"
    post_type = ["unknown"] if ct == "none" else [ct] if ct in known else [_bs(m.alt) or _bs(ct)]
    if zone is None:
        local = lambda s, ns: _Raw(go_time_json(s, ns, tz))
    else:  # zone_oracle's rendering, which ZonedOracle uses as well: not a second check of the zone rule, which
        # tests/test_zones.py pins against the oracle's fixed-offset rendering at every offset of real zones
        from zone_oracle import go_json_time, go_offset
        local = lambda s, ns: _Raw(go_json_time(s, ns, go_offset(zone, s)))
    nil = None
    post = [
        ("post_link", link), ("channel_id", chat), ("post_uid", uid), ("url", link),
        ("published_at", local(m.date, 0)), ("created_at", _Raw(go_time_json(created[0], 0, 0))),  # time.Now().UTC().Truncate(time.Second)
        ("language_code", b""), ("engagement", m.view_count), ("view_count", m.view_count), ("like_count", 0),
        ("share_count", m.share_count), ("comment_count", ncomments), ("crawl_label", _bs(crawl_label)), ("list_ids", nil),
        ("channel_name", title), ("search_terms", nil), ("search_term_ids", nil), ("project_ids", nil), ("exercise_ids", nil),
        ("label_data", nil), ("labels_metadata", nil), ("project_labeled_post_ids", nil), ("labeler_ids", nil),
        ("all_labels", nil), ("label_ids", nil), ("is_ad", False), ("transcript_text", b""), ("image_text", b""),
        ("video_length", nil), ("is_verified", nil),
        ("channel_data", [("channel_id", chat), ("channel_name", title), ("channel_description", b""),
                          ("channel_profile_image", b""),
                          ("channel_engagement_data", [("follower_count", ch.member_count), ("following_count", 0),
                                                       ("like_count", 0), ("post_count", ch.post_count),
                                                       ("views_count", ch.view_count), ("comment_count", 0), ("share_count", 0)]),
                          ("channel_url_external", churl), ("channel_url", churl),
                          ("country_code", b""), ("published_at", _Raw(b'"0001-01-01T00:00:00Z"'))]),
        ("platform_name", b"Telegram"), ("shared_id", nil), ("quoted_id", nil), ("replied_id", nil), ("ai_label", nil),
        ("root_post_id", nil), ("engagement_steps_count", 0), ("ocr_data", nil),
        ("performance_scores", [("likes", nil), ("shares", nil), ("comments", nil), ("views", 0)]),
        ("has_embed_media", nil), ("description", description), ("repost_channel_data", nil), ("post_type", post_type),
        ("inner_link", _Raw(b"{}")), ("post_title", nil), ("media_data", [("document_name", b"")]), ("is_reply", nil),
        ("ad_fields", nil), ("likes_count", 0), ("shares_count", m.share_count), ("comments_count", ncomments),
        ("views_count", m.view_count), ("searchable_text", b""), ("all_text", b""), ("contrast_agent_project_ids", nil),
        ("agent_ids", nil), ("segment_ids", nil), ("thumb_url", b""),  # fetchAndUploadMedia returns "" under SkipMediaDownload (:233-239)
        ("media_url", media), ("comments", comments), ("reactions", reactions), ("outlinks", [_bs(x) for x in links]),
        ("capture_time", local(*capture)), ("handle", _bs(m.handle)),
    ]
    return "emitted", _marshal(post) + b"\n", links


# ---- the whole YouTube Post line, a second time ---------------------------------------------------------------------------
# From crawler/youtube/youtube_crawler.go:530-836 (convertVideoToPost), :461-527 (duration, extractURLs, sanitizeFilename),
# client/youtube_client.go:1856-1878 (snowball channel ids), time.Time.MarshalJSON and strconv's float formatting, over
# pack.YouTubeVideo / YouTubeChannel.  Where Go iterates a map (thumbnails -> ocr_data, unique URLs -> outlinks) the order is
# unspecified in Go; the engine's documented convention is used: thumbnail keys in the order youtube_client.go:1028-1044
# inserts them, URLs in first-occurrence order.
def _go_time_checked(sec: int, nsec: int, tz: int):
    """time.Time.MarshalJSON: error (None) when the year is outside [0, 9999]; proleptic Gregorian by day arithmetic"""
    local = sec + tz
    days, rem = divmod(local, 86400)
    z = days + 719468  # days since 0000-03-01 (civil-from-days)
    era = z // 146097
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    y = yoe + era * 400
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    d = doy - (153 * mp + 2) // 5 + 1
    mo = mp + 3 if mp < 10 else mp - 9
    if mo <= 2:
        y += 1
    if y < 0 or y > 9999:
        return None
    s = "%04d-%02d-%02dT%02d:%02d:%02d" % (y, mo, d, rem // 3600, rem % 3600 // 60, rem % 60)
    if nsec:
        s += "." + ("%09d" % nsec).rstrip("0")
    if tz == 0:
        s += "Z"
    else:
        a = abs(tz)
        s += ("-" if tz < 0 else "+") + "%02d:%02d" % (a // 3600, a % 3600 // 60)
    return _Raw(('"' + s + '"').encode())


def _go_float_of_int(v: int) -> bytes:
    """encoding/json of float64(v): shortest digits that round-trip, 'f' format below 1e21"""
    from decimal import Decimal
    f = float(v)
    if f == 0:
        return b"0"
    s = format(Decimal(repr(f)), "f")
    return (s[:-2] if s.endswith(".0") else s).encode()


_URL = re.compile(rb"https?://[^\t\n\f\r ]+")  # RE2's \S: everything but [\t\n\f\r ]
_UC = re.compile(rb"youtube\.com/channel/([a-zA-Z0-9_-]+)")
_HANDLE = re.compile(rb"youtube\.com/@([a-zA-Z0-9_.-]+)")


def _sanitize_filename(title: bytes) -> bytes:
    out, i = bytearray(), 0
    while i < len(title):
        r, w = go_decode_rune(title, i)
        c = title[i]
        out.append(c if w == 1 and r < 0x80 and (chr(c).isalnum() or c in b"_-.") else 0x5F)
        i += w
    return bytes(out[:50])


def youtube_post_line(v, ch, *, crawl_label=b"", created=(1_750_000_000, 0), capture=(1_750_000_000, 123_456_789), tz=0):
    """-> (line or None when a time is not representable, outlink URLs, snowball channel ids)"""
    vid, title, desc = _bs(v.id), _bs(v.title), _bs(v.description)
    chid = _bs(ch.id)
    vurl = b"https://www.youtube.com/watch?v=" + vid
    churl = (b"https://www.youtube.com/" if chid[:1] == b"@" else b"https://www.youtube.com/channel/") + chid
    # int(LikeCount + CommentCount + ViewCount/100): Go's integer division truncates toward zero (:561)
    engagement = v.like_count + v.comment_count + (abs(v.view_count) // 100) * (1 if v.view_count >= 0 else -1)
    engagement = (engagement + 2 ** 63) % 2 ** 64 - 2 ** 63  # an int64 sum in Go: wraps
    th = {k: _bs(x) for k, x in v.thumbnails.items()}
    thumb = b""
    for k in ("maxres", "high", "medium", "default"):
        if th.get(k):
            thumb = th[k]
            break
    vlen = None
    dur = _bs(v.duration)
    if dur and dur != b"P0D":
        vlen = parse_iso8601_duration(dur)
    urls, seen = [], set()
    for u in _URL.findall(desc):
        u = u.rstrip(b",.;:!?()'\"")
        if u not in seen:
            seen.add(u)
            urls.append(u)
    ids = [m for m in _UC.findall(desc)] + [b"@" + m for m in _HANDLE.findall(desc)]
    ocr = [[("ocr_text", b"YouTube thumbnail: " + k.encode() + b" quality"), ("thumb_url", th[k])]
           for k in ("default", "medium", "high", "standard", "maxres") if th.get(k)]
    pub = _go_time_checked(v.published_sec, v.published_nsec, 0)
    cre, cap = _go_time_checked(created[0], created[1], tz), _go_time_checked(capture[0], capture[1], tz)
    if ch.cached:
        chpub = _go_time_checked(ch.published_sec, ch.published_nsec, 0)
        cdata = [("channel_id", chid), ("channel_name", _bs(ch.title)), ("channel_description", _bs(ch.description)),
                 ("channel_profile_image", _bs(ch.thumb_default)),
                 ("channel_engagement_data", [("follower_count", ch.subscriber_count), ("following_count", 0), ("like_count", 0),
                                              ("post_count", ch.video_count), ("views_count", ch.view_count), ("comment_count", 0),
                                              ("share_count", 0)]),
                 ("channel_url_external", churl), ("channel_url", churl), ("country_code", _bs(ch.country)), ("published_at", chpub)]
        chname = _bs(ch.title)
    else:
        chpub = pub
        cdata = [("channel_id", chid), ("channel_name", chid), ("channel_description", b""), ("channel_profile_image", b""),
                 ("channel_engagement_data", [("follower_count", 0), ("following_count", 0), ("like_count", v.like_count),
                                              ("post_count", 0), ("views_count", v.view_count), ("comment_count", v.comment_count),
                                              ("share_count", 0)]),
                 ("channel_url_external", churl), ("channel_url", churl), ("country_code", b""), ("published_at", pub)]
        chname = chid
    if None in (pub, cre, cap, chpub):
        return None, urls, ids
    nil = None
    alltext = title + b" " + desc
    post = [
        ("post_link", vurl), ("channel_id", chid), ("post_uid", vid), ("url", vurl), ("published_at", pub), ("created_at", cre),
        ("language_code", _bs(v.language)), ("engagement", engagement), ("view_count", v.view_count), ("like_count", v.like_count),
        ("share_count", 0), ("comment_count", v.comment_count), ("crawl_label", _bs(crawl_label)), ("list_ids", nil),
        ("channel_name", chname), ("search_terms", nil), ("search_term_ids", nil), ("project_ids", nil), ("exercise_ids", nil),
        ("label_data", nil), ("labels_metadata", nil), ("project_labeled_post_ids", nil), ("labeler_ids", nil), ("all_labels", nil),
        ("label_ids", nil), ("is_ad", False), ("transcript_text", b""), ("image_text", b""), ("video_length", vlen),
        ("is_verified", nil), ("channel_data", cdata), ("platform_name", b"youtube"), ("shared_id", nil), ("quoted_id", nil),
        ("replied_id", nil), ("ai_label", nil), ("root_post_id", nil), ("engagement_steps_count", 0), ("ocr_data", ocr or None),
        ("performance_scores", [("likes", v.like_count), ("shares", nil), ("comments", v.comment_count),
                                ("views", _Raw(_go_float_of_int(v.view_count)))]),
        ("has_embed_media", True), ("description", desc), ("repost_channel_data", nil), ("post_type", [b"video"]),
        ("inner_link", _Raw(b"{}")), ("post_title", title),
        ("media_data", [("document_name", vid + b"-" + _sanitize_filename(title) + b".mp4")]), ("is_reply", nil), ("ad_fields", nil),
        ("likes_count", v.like_count), ("shares_count", 0), ("comments_count", v.comment_count), ("views_count", v.view_count),
        ("searchable_text", alltext), ("all_text", alltext), ("contrast_agent_project_ids", nil), ("agent_ids", nil),
        ("segment_ids", nil), ("thumb_url", thumb), ("media_url", vurl), ("comments", nil), ("reactions", {b"like": v.like_count}),
        ("outlinks", urls), ("capture_time", cap), ("handle", chid),
    ]
    return _marshal(post) + b"\n", urls, ids


# ---- the whole generic Post line, a second time ----------------------------------------------------------------------------
# From crawler/telegram/telegram_crawler.go:179-262 (convertMessageToPost over client.Message), model/data.go (field order and
# types: a nil map and nil slices marshal as null, zero structs with their zero fields, a zero time.Time as
# "0001-01-01T00:00:00Z") and time.Time.MarshalJSON: published_at = GetTimestamp(), created_at = capture_time = time.Now(),
# all three in time.Local.  zone = (starts, offsets) is time.Local as a transition table (tests/zone_oracle.py's rule);
# without one time.Local is the fixed offset tz.
def generic_post_line(m, *, created, capture, tz=0, zone=None):
    """-> the line of one pack.GenericMessage, or None when json.Marshal fails (a time outside year [0, 9999])"""
    if zone is None:
        when = lambda sec, nsec: _go_time_checked(sec, nsec, tz)
    else:
        from zone_oracle import go_json_time, go_offset
        when = lambda sec, nsec: _Raw(go_json_time(sec, nsec, go_offset(zone, sec))) or None
    pub, cre, cap = when(m.ts_sec, m.ts_nsec), when(*created), when(*capture)
    if None in (pub, cre, cap):
        return None
    reactions = {}
    for k, cnt in m.reactions:  # map assignment: a later entry of a key overwrites
        reactions[_bs(k)] = cnt
    chan, text = _bs(m.channel_id), _Raw(go_json_string(_bs(m.text)))  # the text is marshalled three times: escape it once
    nil = None
    post = [
        ("post_link", b""), ("channel_id", chan), ("post_uid", _bs(m.id)), ("url", b""), ("published_at", pub),
        ("created_at", cre), ("language_code", b""), ("engagement", 0), ("view_count", m.views), ("like_count", 0),
        ("share_count", 0), ("comment_count", 0), ("crawl_label", b""), ("list_ids", nil), ("channel_name", chan),
        ("search_terms", nil), ("search_term_ids", nil), ("project_ids", nil), ("exercise_ids", nil), ("label_data", nil),
        ("labels_metadata", nil), ("project_labeled_post_ids", nil), ("labeler_ids", nil), ("all_labels", nil),
        ("label_ids", nil), ("is_ad", False), ("transcript_text", b""), ("image_text", b""), ("video_length", nil),
        ("is_verified", nil),
        ("channel_data", [("channel_id", b""), ("channel_name", b""), ("channel_description", b""),
                          ("channel_profile_image", b""),
                          ("channel_engagement_data", [("follower_count", 0), ("following_count", 0), ("like_count", 0),
                                                       ("post_count", 0), ("views_count", 0), ("comment_count", 0),
                                                       ("share_count", 0)]),
                          ("channel_url_external", b""), ("channel_url", b""), ("country_code", b""),
                          ("published_at", _Raw(b'"0001-01-01T00:00:00Z"'))]),
        ("platform_name", b"telegram"), ("shared_id", nil), ("quoted_id", nil), ("replied_id", nil), ("ai_label", nil),
        ("root_post_id", nil), ("engagement_steps_count", 0), ("ocr_data", nil),
        ("performance_scores", [("likes", nil), ("shares", nil), ("comments", nil), ("views", 0)]),
        ("has_embed_media", nil), ("description", text), ("repost_channel_data", nil), ("post_type", nil),
        ("inner_link", _Raw(b"{}")), ("post_title", nil), ("media_data", [("document_name", b"")]), ("is_reply", nil),
        ("ad_fields", nil), ("likes_count", 0), ("shares_count", 0), ("comments_count", 0), ("views_count", m.views),
        ("searchable_text", text), ("all_text", text), ("contrast_agent_project_ids", nil), ("agent_ids", nil),
        ("segment_ids", nil), ("thumb_url", b""), ("media_url", b""), ("comments", nil),
        ("reactions", reactions or None),  # :250: the map only if it has entries, else nil
        ("outlinks", nil), ("capture_time", cap), ("handle", _bs(m.sender_name)),
    ]
    return _marshal(post) + b"\n"
