"""Small deterministic YouTube corpus for the config-4 parity tests (SURVEY.md §8d shape, Python
generated: sizes the oracle finishes in seconds), and make_youtube_edges: videos built by rule at the edges of the
GPU line's routing, escaping, extraction and rendering rules."""
import collections
import random

import go_rules
from distributed_crawler_b200.pack import YouTubeChannel, YouTubeVideo, pack_youtube

_B64 = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789-_"
_WORDS = ["video", "новости", "смотрите", "канал", "subscribe", "плейлист", "中文", "字幕", "😀", "live", "&", "<3", "\"quoted\"",
          "line\nbreak", "tab\there", "обзор", "2024", "часть", "#shorts", "مرحبا", " ", "a\\b"]


def make_youtube(n: int, seed: int = 7, n_chans: int = 37):
    rng = random.Random(seed)
    chans = []
    for c in range(n_chans):
        cid = ("@" + "".join(rng.choice("abcdefghij_.-") for _ in range(rng.randrange(3, 20)))) if c % 7 == 3 else \
              "UC" + "".join(rng.choice(_B64) for _ in range(22))
        chans.append(YouTubeChannel(
            id=cid, title=" ".join(rng.choice(_WORDS) for _ in range(rng.randrange(1, 5))),
            description=" ".join(rng.choice(_WORDS) for _ in range(rng.randrange(0, 30))),
            thumb_default="https://yt3.ggpht.com/" + "".join(rng.choice(_B64) for _ in range(30)) if c % 5 else "",
            country=rng.choice(["", "US", "RU", "DE"]), subscriber_count=rng.randrange(0, 10 ** 8),
            view_count=rng.randrange(0, 10 ** 11), video_count=rng.randrange(0, 10 ** 5),
            published_sec=rng.randrange(1_100_000_000, 1_700_000_000), published_nsec=rng.choice([0, 0, 123_000_000]),
            cached=(c % 6 != 5)))
    vids = []
    for i in range(n):
        words = []
        for _ in range(int(rng.lognormvariate(3.5, 1.0)) % 600):
            u = rng.random()
            if u < 0.05:
                tail = rng.choice(["", ".", ",", ")!", "?\"", "'", "/path?q=1&x=<y>", ":"])
                words.append(rng.choice(["http://", "https://"]) + rng.choice(["example.com/", "t.me/chan", "bit.ly/", "youtu.be/"]) +
                             "".join(rng.choice(_B64) for _ in range(rng.randrange(0, 9))) + tail)
            elif u < 0.065:
                words.append("https://www.youtube.com/channel/UC" + "".join(rng.choice(_B64) for _ in range(rng.choice([22, 22, 40]))))
            elif u < 0.08:
                words.append("youtube.com/@" + "".join(rng.choice("abcxyz019_.-") for _ in range(rng.choice([5, 12, 45]))) + rng.choice(["", "/videos", "!"]))
            elif u < 0.085:
                words.append(rng.choice(["http://", "https:// x", "https://", "http", "xhttps://a.b", "https://dup.example/1", "https://dup.example/1"]))
            else:
                words.append(rng.choice(_WORDS))
        desc = " ".join(words)
        if i % 97 == 0:
            desc = desc.encode()[: rng.randrange(0, 40)] + b"\xff\xe2\x80" + desc.encode()[:50]
        views = int(rng.lognormvariate(8, 3)) if i % 41 else rng.choice([0, 2 ** 53, 2 ** 53 + 1, 2 ** 62 + 12345, 9_223_372_036_854_775_807, 12345678901234567890 // 2])
        dur = rng.choice(["PT%dM%dS" % (rng.randrange(60), rng.randrange(60)), "PT%dH%dM%dS" % (rng.randrange(5), rng.randrange(60), rng.randrange(60)),
                          "P0D", "", "P1DT2H", "PT", "P", "PT15M", "PT1H2M3", "PT99999999999999999999S", "bogus", "PT5S "])
        keys = [k for k in ("default", "medium", "high", "standard", "maxres") if rng.random() < 0.8]
        thumbs = {k: ("https://i.ytimg.com/vi/%s/%s.jpg" % (i, k) if rng.random() < 0.95 else "") for k in keys}
        vids.append(YouTubeVideo(
            id="".join(rng.choice(_B64) for _ in range(11)), title=" ".join(rng.choice(_WORDS) for _ in range(rng.randrange(0, 12))),
            description=desc, published_sec=rng.randrange(1_100_000_000, 1_760_000_000) if i % 53 else rng.choice([-62135596800, 253402300800]),
            published_nsec=rng.choice([0, 0, 0, 500_000_000]), view_count=views, like_count=views // 30, comment_count=views // 300,
            duration=dur, thumbnails=thumbs, language=rng.choice(["", "en", "ru", "zh-Hans"]), channel=rng.randrange(n_chans)))
    return pack_youtube(vids, chans), vids, chans


_PLAIN = ["the", "video", "about", "channel", "new", "watch", "and", "more", "from", "this", "week", "episode", "review", "how", "to",
          "guide", "music", "official", "live", "part", "best", "of", "2024", "full", "with", "our", "your", "for", "you", "in"]


def make_youtube_config4(n: int, seed: int = 0x5EED0004, n_chans: int = 1000):
    """BASELINE config 4 shape (SURVEY.md §8d): title lognormal median 45 B, description lognormal median 400 B
    clipped at 5000 with URLs Poisson(1.5) of which 10 % are youtube.com/channel/UC… or youtube.com/@handle,
    views lognormal(8, 3), likes = views/30, comments = views/300, PT#H#M#S durations (1 % P0D, 0.5 % empty,
    0.5 % P1DT…), 3-5 thumbnails.  2 % of the descriptions carry characters that need escaping."""
    rng = random.Random(seed)
    chans = [YouTubeChannel(id="UC" + "".join(rng.choice(_B64) for _ in range(22)), title="Channel %d" % c,
                            description=" ".join(rng.choice(_PLAIN) for _ in range(20)),
                            thumb_default="https://yt3.ggpht.com/" + "".join(rng.choice(_B64) for _ in range(30)), country="US",
                            subscriber_count=rng.randrange(0, 10 ** 7), view_count=rng.randrange(0, 10 ** 10),
                            video_count=rng.randrange(0, 10 ** 4), published_sec=rng.randrange(1_100_000_000, 1_700_000_000),
                            cached=True) for c in range(n_chans)]

    def text(nbytes, urls):
        words, size = [], 0
        while size < nbytes:
            w = rng.choice(_PLAIN)
            words.append(w)
            size += len(w) + 1
        for _ in range(urls):
            u = rng.random()
            if u < 0.05:
                link = "https://www.youtube.com/channel/UC" + "".join(rng.choice(_B64) for _ in range(22))
            elif u < 0.10:
                link = "https://youtube.com/@" + "".join(rng.choice("abcdefghij_") for _ in range(rng.randrange(5, 15)))
            else:
                link = "https://example.com/" + "".join(rng.choice(_B64) for _ in range(rng.randrange(4, 20)))
            words.insert(rng.randrange(len(words) + 1), link)
        return " ".join(words)

    def poisson(lam):
        k, p, L = 0, 1.0, 2.718281828 ** -lam
        while True:
            p *= rng.random()
            if p <= L:
                return k
            k += 1

    vids = []
    for i in range(n):
        desc = text(min(int(rng.lognormvariate(5.99, 0.9)), 5000), poisson(1.5))
        if rng.random() < 0.02:
            desc = desc.replace(" ", "\n", 3) + ' "quoted" <tag> & more'
        views = int(rng.lognormvariate(8, 3))
        u = rng.random()
        dur = "P0D" if u < 0.01 else "" if u < 0.015 else "P1DT2H" if u < 0.02 else "PT%dH%dM%dS" % (rng.randrange(3), rng.randrange(60), rng.randrange(60))
        keys = ["default", "medium", "high", "standard", "maxres"][: rng.randrange(3, 6)]
        vids.append(YouTubeVideo(
            id="".join(rng.choice(_B64) for _ in range(11)), title=text(int(rng.lognormvariate(3.8, 0.5)), 0), description=desc,
            published_sec=rng.randrange(1_300_000_000, 1_760_000_000), view_count=views, like_count=views // 30, comment_count=views // 300,
            duration=dur, thumbnails={k: "https://i.ytimg.com/vi/%s/%s.jpg" % (i, k) for k in keys}, language="en",
            channel=rng.randrange(n_chans)))
    return pack_youtube(vids, chans), vids, chans


# ---- edges by rule ------------------------------------------------------------------------------------------------------
# The YouTube line has three writers, chosen per record by yt_size_lane_kernel (esc_len[3r+2]): 1 = nothing to escape (the
# lane writer copies), 2 = only the description / title need escaping and only ASCII bytes of them (the lane writer escapes:
# ld_copy_esc up to YT_LANE_LONG = 128 raw bytes, the warp's esc_ascii_to_global for longer strings, which the lane skips and
# hands over through YT_LANE_PENDING = 4 slots for the 6 writes of the two strings), 0 = anything else (the warp writer).
# make_youtube_edges puts strings on both sides of each of those rules and of the extractors' 16-byte lanes / 512-byte strips.
I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1
EDGE_LENGTHS = (0, 1, 15, 16, 17, 31, 32, 33, 127, 128, 129, 130, 255, 256, 257, 383, 384, 385, *range(508, 517),
                1023, 1024, 1025, 4999, 5000, 5001)
ASCII_SPECIALS = b'"\\<>&\b\f\n\r\t\x0b\x1f'
# invalid UTF-8, bytes >= 0xF4 and E2 80 xx send a string to the exact (per-byte) escaper; C2 80 is a plain valid rune
EXACT_TRIGGERS = ("\u2028".encode(), "\u2029".encode(), "\u2019".encode(), b"\xf4\x8f\xbf\xbf", b"\xc0\x80", b"\xed\xa0\x80",
                  b"\xff")
RUNES = ("\u00e9".encode(), "\u4e2d".encode(), "\U0001f600".encode(), b"\xc2\x80")
DURATIONS = (b"PT1H2M3S", b"P1DT2H", b"PT", b"P", b"P0D", b"PT15M", b"", b"PT1H2M3", b"P1D2H", b"PT1M1H",
             b"PT99999999999999999999S", b"XPT1S", b"PT1S ", b"P106751991167301D", b"PT1S\n", "P\u0661D".encode(),
             b"PT9223372036854775808S", b"PT007S", b"pt1s", b"P1DT", b"PT1H1H")
COUNTS = (0, 5, -1, I64_MAX, I64_MIN, I64_MAX - 7, I64_MIN + 3, 2 ** 62, -(2 ** 62))  # like + comment wraps both ways
_ALNUM = b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789"
_TEXT = (_ALNUM + b"  ") * 4  # 256 entries: bytes.translate maps random bytes onto clean text (no ':', '/' or '.')
_ID = bytes(_B64, "ascii") * 4


def view_values(rng: random.Random, n_random: int = 60) -> list[int]:
    """view counts where float64(v) formatting goes wrong: 10^k edges, 2^e + {0, ±1, ±511, ±512, ±513, ±1024, ±1025}
    (±ulp/2 is where float64(int64) rounds half to even), the int64 bounds, random values above 2^53"""
    vals = [0, 1, -1, 2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, -(2 ** 53) - 1, I64_MIN, I64_MIN + 1, I64_MAX, I64_MAX - 1]
    for k in range(19):
        vals += [10 ** k - 1, 10 ** k, -(10 ** k - 1), -(10 ** k)]
    for e in range(53, 63):
        for d in (0, 1, 511, 512, 513, 1024, 1025):
            vals += [2 ** e + d, 2 ** e - d, -(2 ** e + d), -(2 ** e - d)]
    vals += [rng.randrange(2 ** 53, 2 ** 63) * rng.choice((1, -1)) for _ in range(n_random)]
    return [min(max(v, I64_MIN), I64_MAX) for v in vals]


def _fill(rng, n: int, runes: bool = False) -> bytes:
    """n bytes of text that needs no escaping and holds no URL / channel-link syntax; `runes`: with valid 2-4 byte runes"""
    out = bytearray(rng.randbytes(n).translate(_TEXT))
    if runes:
        for _ in range(n // 24):
            r = rng.choice(RUNES)
            if n > len(r):
                p = rng.randrange(n - len(r) + 1)
                if all(c < 0x80 for c in out[max(p - 1, 0):p + len(r) + 1]):  # never cuts another rune
                    out[p:p + len(r)] = r
    return bytes(out)


def _specials(rng, s: bytes, k: int) -> bytes:
    """ASCII specials at the 16-byte block / 512-byte strip / partial-word edges of an ASCII string (k picks which)"""
    n = len(s)
    if not n:
        return s
    spots = [p for p in (0, 3, 4, 12, 15, 16, 48, 51, 52, 60, 63, 127, 128, 511, 512, n - 1) if p < n]
    out = bytearray(s)
    for j in range(1 + k % 3):
        out[spots[(k + 5 * j) % len(spots)]] = ASCII_SPECIALS[(k + j) % len(ASCII_SPECIALS)]
    if n % 4 and k % 2:
        out[n - 1] = ASCII_SPECIALS[k % len(ASCII_SPECIALS)]  # the last byte of a partial word
    return bytes(out)


def _exact(rng, s: bytes, k: int) -> bytes:
    """an exact-path trigger: anywhere, straddling byte 128 or 512, or a sequence cut by the end of the string"""
    n = len(s)
    if not n:
        return s
    trig = EXACT_TRIGGERS[k % len(EXACT_TRIGGERS)]
    where = (k // len(EXACT_TRIGGERS)) % 4
    if where == 3 or n < len(trig):
        cut = next(t for t in EXACT_TRIGGERS[k % 4:] + EXACT_TRIGGERS if len(t) > 1)  # a multi-byte trigger, truncated
        keep = min(len(cut) - 1, n, 1 + k % (len(cut) - 1))
        return s[:n - keep] + cut[:keep]
    if where in (1, 2) and n >= (128 if where == 1 else 512) + len(trig):
        edge = 128 if where == 1 else 512
        p = edge - 1 - (k % (len(trig) - 1) if len(trig) > 1 else 0)
    else:
        p = rng.randrange(n - len(trig) + 1)
    return s[:p] + trig + s[p + len(trig):]


def _make(rng, kind: str, n: int, k: int) -> bytes:
    if kind == "clean":
        return _fill(rng, n, runes=k % 2 == 0)
    base = _fill(rng, n)
    return _specials(rng, base, k) if kind == "ascii" else _exact(rng, base, k)


def _edge_channels(rng):
    cnt = lambda: rng.choice((0, 1, -1, I64_MAX, I64_MIN, 10 ** 18, 2 ** 53 + 1))
    pub = lambda: dict(published_sec=rng.randrange(1_100_000_000, 1_700_000_000), published_nsec=rng.choice((0, 1, 10, 120_000_000)))
    ch = lambda **kw: YouTubeChannel(**{**dict(id="UC" + "".join(rng.choice(_B64) for _ in range(22)), title="Channel t",
                                               description=_fill(rng, rng.randrange(0, 200), runes=True),
                                               thumb_default="https://yt3.ggpht.com/" + "".join(rng.choice(_B64) for _ in range(30)),
                                               country="US", subscriber_count=cnt(), view_count=cnt(), video_count=cnt(), **pub()), **kw})
    return [
        ch(),                                                   # 0 cached, clean
        ch(cached=False),                                       # 1 uncached, clean
        ch(id="@edge.handle-1"),                                # 2 cached handle
        ch(id="@h", cached=False),                              # 3 uncached handle
        ch(published_sec=-62167219200, published_nsec=0),       # 4 cached, 0000-01-01T00:00:00Z
        ch(published_sec=253402300799, published_nsec=999_999_999),  # 5 cached, the last representable instant
        # --- one dirty short field each (the warp writer) ---
        ch(title="line\nbreak"),                                # 6
        ch(description="para\u2028graph " + "x" * 40),          # 7
        ch(country='U"S'),                                      # 8
        ch(id="UC<x" + "a" * 20),                               # 9 cached
        ch(id="UC<y" + "b" * 20, cached=False),                 # 10 uncached
        ch(thumb_default="https://yt3.ggpht.com/a?b=1&c=2"),   # 11
        # --- no line: json.Marshal fails on the channel's published_at ---
        ch(published_sec=253402300800),                         # 12
        ch(published_sec=-62167219201),                         # 13
    ]


_CLEAN_CHANS = (0, 1, 2, 3, 4, 5)


def _url_descs(rng) -> list[bytes]:
    """extractURLs at its edges: the colon at every offset of a lane and around the strip edge, URLs across strips,
    TrimRight tails, duplicates, more than 32 URLs, no-match schemes"""
    f = lambda n: _fill(rng, n)
    out = []
    for scheme in (b"http", b"https"):
        for lane in (1, 6):
            for off in range(16):
                colon = 16 * lane + off
                out.append(f(colon - len(scheme)) + scheme + b"://u%d.example/%d " % (off, lane) + f(rng.randrange(0, 40)))
        for colon in (4, 5, 510, 511, 512, 513, 514):
            if colon >= len(scheme):
                out.append(f(colon - len(scheme)) + scheme + b"://s.example/" + f(3).replace(b" ", b"x") + b" " + f(20))
    out += [
        f(40) + b" https://a.example/" + b"x" * 600 + b"http://inner.example/" + b"y" * 30 + b" " + f(10),  # one URL over 2 strips
        f(500) + b" http://b.example/" + b"z" * 700 + b"https://inner.example " + f(30),
        b"http://a.example/c,.;:!?()'\" http://a.example/d) http://a.example/e' https://) http://,.; " + f(20),
        f(60) + b' see "http://q.example/r" and (https://q.example/s).',
        b"https://example.com/0123456789abcdef/A https://example.com/0123456789abcdef/B https://example.com/0123456789abcdef/A",
        b"http://a.b/c http://a.b/cd http://a.b/c http://a.b/cd.",
        b" ".join(b"http://u%02d.example/p" % j for j in range(40)),  # more than 32 unique URLs
        b"HTTP://upper.example Http://x.example hxxp://y.example http:/z http:// x https://\tx " + f(10),
        f(30) + b" trailing http://",
        f(30) + b" trailing https://x",
        f(31) + b" http://x",
        b"http://x",
    ]
    return out


def _channel_descs(rng) -> list[bytes]:
    """extractChannelIDsFromText at its edges: youtube.com/ at offset 0, on lane and strip edges and at the end; ids around
    the 32-byte key cut; overlapping matches; www. / m. prefixes; channel/ and @ matches interleaved"""
    f = lambda n: _fill(rng, n)
    uc = lambda n: b"UC" + bytes(rng.choice(_B64.encode()) for _ in range(n - 2))
    hd = lambda n: bytes(rng.choice(b"abcxyz019_.-") for _ in range(n))
    out = [b"youtube.com/channel/" + uc(24) + b" " + f(20), b"youtube.com/@" + hd(8) + b" " + f(10)]
    for slash in (16 + 0, 16 + 15, 32, 16 * 9 + 15, 511, 512, 513):
        out.append(f(slash - 11) + b"youtube.com/channel/" + uc(24) + b" " + f(20))
        out.append(f(slash - 11) + b"youtube.com/@" + hd(10) + b" " + f(20))
    for tail in (b"youtube.com/", b"youtube.com/channel/", b"youtube.com/@", b"youtube.com/@x", b"youtube.com/channel/U"):
        out.append(f(40) + b" " + tail)
    for n in (30, 31, 32, 33, 40):
        out.append(f(10) + b" https://www.youtube.com/channel/" + uc(n) + b" https://m.youtube.com/@" + hd(n) + b" " + f(10))
    out += [
        b"youtube.com/@a.youtube.com/@b " + f(10),
        b"x youtube.com/@a1 youtube.com/channel/UC1 youtube.com/@a2 https://youtube.com/channel/UC2/videos youtube.com/@a3!",
        f(490) + b" youtube.com/channel/" + uc(40) + b"youtube.com/@" + hd(33),
    ]
    return out


def make_youtube_edges(seed: int = 1):
    """videos and channels built by rule, not by distribution (see the block comment above): the routing grid (every
    length of EDGE_LENGTHS, exactly and 1-3 bytes over, for the description and for the title, clean / ASCII specials /
    exact triggers), both-long and raw <= 128 < escaped records, one dirty short field at a time, URL and channel-link
    edges, view counts around 2^53..2^63 and the int64 bounds, engagement that wraps, the year-0 / year-9999 bounds,
    odd durations and sanitizeFilename at 50 bytes.  Records of all three writers are interleaved, so that they share
    warps and 16-byte output blocks.  Returns (batch, videos, channels)."""
    rng = random.Random(seed)
    chans = _edge_channels(rng)
    views = view_values(rng)
    items = []  # (description, title, extra YouTubeVideo fields)

    k = 0
    for L in EDGE_LENGTHS:  # the routing grid
        for kind in ("clean", "ascii", "exact"):
            for slot in (0, 1):
                for n in (L, L + 1 + rng.randrange(3)):
                    k += 1
                    mine = _make(rng, kind, n, k)
                    other_kind = "clean" if kind == "clean" or n == 0 else rng.choice(("clean", kind))
                    if n == 0 and kind != "clean":
                        other_kind = kind
                    other = _make(rng, other_kind, rng.choice(EDGE_LENGTHS), k + 1)
                    items.append((mine, other, {}) if slot == 0 else (other, mine, {}))
    long_ = (129, 130, 255, 512, 513, 1024, 5001)
    for j, (a, b) in enumerate(zip(long_, long_[3:] + long_[:3])):  # both strings longer than YT_LANE_LONG
        for kinds in (("ascii", "ascii"), ("ascii", "clean"), ("clean", "ascii"), ("clean", "clean"), ("exact", "ascii")):
            items.append((_make(rng, kinds[0], a, j), _make(rng, kinds[1], b, j + 3), {}))
    for n, m, c in ((128, 1, b"<"), (128, 1, b"\n"), (100, 10, b"&"), (23, 22, b"<"), (127, 1, b'"'), (64, 40, b"\x1f")):
        s = bytearray(_fill(rng, n))  # raw <= 128, escaped > 128
        for p in rng.sample(range(n), m):
            s[p] = c[0]
        items.append((bytes(s), _fill(rng, 20), {}))
        items.append((_fill(rng, 20, runes=True), bytes(s), {}))
    items += [(_fill(rng, 129), b'ti"tle', {}), (b"d\tesc", _fill(rng, 129), {}),  # raw 129, nothing to escape, beside mode 2
              (_fill(rng, 129, runes=True), _specials(rng, _fill(rng, 300), 4), {})]
    items += [(b"", _fill(rng, 40) + b"\xff", {}), (_fill(rng, 40) + b"\xff", b"", {}), (b"", b'a"b', {}), (b'a"b', b"", {})]

    long_clean = lambda: _fill(rng, rng.randrange(600, 1100), runes=True)  # one dirty short field at a time
    for ch in (0, 1):
        items += [(long_clean(), b"title", dict(id=b'vi"d', channel=ch)), (long_clean(), b"title", dict(language=b"e<n", channel=ch)),
                  (long_clean(), b"title", dict(thumbnails={"default": "https://i.ytimg.com/vi/x/d.jpg?a=1&b=2", "high": "https://h"}, channel=ch)),
                  (long_clean() + b" https://out.example/p?a=1&b=2 " + _fill(rng, 20), b"t", dict(channel=ch)),
                  (long_clean() + b" http://out.example/\x0bq " + _fill(rng, 20), b"t", dict(channel=ch))]
    for ch in (6, 7, 8, 9, 10, 11, 2, 3):
        items.append((long_clean(), _fill(rng, rng.choice((5, 140))), dict(channel=ch)))

    items += [(d, _fill(rng, 30), {}) for d in _url_descs(rng)]
    items += [(d, _fill(rng, 30), {}) for d in _channel_descs(rng)]

    for sec, nsec in ((-62167219200, 0), (-62167219201, 0), (-62167219200, 1), (253402300799, 999_999_999), (253402300800, 0),
                      (253402300799, 10), (0, 120_000_000), (1_700_000_000, 1)):
        items.append((_fill(rng, 40), b"t", dict(published_sec=sec, published_nsec=nsec, channel=rng.choice((0, 1)))))
    for ch in (12, 13, 4, 5):
        items.append((_fill(rng, 40), b"t", dict(channel=ch)))

    for n in (49, 50, 51, 52):  # sanitizeFilename keeps 50 bytes
        for p, ins in ((None, b""), (47, RUNES[1]), (48, RUNES[0]), (49, RUNES[0]), (48, RUNES[2]), (49, b"\xff"), (50, b"\xe9"),
                       (48, b"\xf0\x9f\x98")):
            t = _fill(rng, n)
            if p is not None and p + len(ins) <= n:
                t = t[:p] + ins + t[p + len(ins):]
            items.append((_fill(rng, 60), t, {}))

    vids = []
    for i, (desc, title, kw) in enumerate(items):
        vid = kw.pop("id", None) or rng.randbytes(i % 16 + 1).translate(_ID)  # ids of 1-16 bytes: lines start at every offset
        keys = [key for key in ("default", "medium", "high", "standard", "maxres") if rng.random() < 0.6]
        v = YouTubeVideo(id=vid, title=title, description=desc, published_sec=rng.randrange(1_300_000_000, 1_760_000_000),
                         published_nsec=rng.choice((0, 0, 1, 10, 120_000_000, 999_999_999)), view_count=views[i % len(views)],
                         like_count=rng.choice(COUNTS), comment_count=rng.choice(COUNTS), duration=DURATIONS[i % len(DURATIONS)],
                         thumbnails={key: ("https://i.ytimg.com/vi/%s/%s.jpg" % (vid.decode("latin-1"), key) if rng.random() < 0.9 else "")
                                     for key in keys},
                         language=rng.choice(("", "en", "pt-BR", "zh-Hans")), channel=rng.choice(_CLEAN_CHANS))
        for key, val in kw.items():
            setattr(v, key, val)
        vids.append(v)
    vids = _interleave(rng, vids, chans)
    return pack_youtube(vids, chans), vids, chans


def _interleave(rng, vids, chans):
    """the three writers' records side by side: a random permutation of (0, 1, 2) per triple of records, so that every
    warp of 32 holds all three and records 31 / 32 and 63 / 64 (warp edges) belong to different writers"""
    by = {0: [], 1: [], 2: []}
    rest = []
    for v in vids:
        m = yt_writer_mode(v, chans[v.channel])
        (by[m] if m is not None else rest).append(v)
    for lst in by.values():
        rng.shuffle(lst)
    out = []
    while all(by.values()):
        for m in rng.sample((0, 1, 2), 3):
            out.append(by[m].pop())
    left = by[0] + by[1] + by[2] + rest
    rng.shuffle(left)
    return out + left


def make_youtube_edges_many(n_min: int, seed: int = 100):
    """make_youtube_edges over consecutive seeds until at least n_min videos (one channel list per seed, concatenated)"""
    vids, chans = [], []
    while len(vids) < n_min:
        _, v, c = make_youtube_edges(seed)
        for x in v:
            x.channel += len(chans)
        vids += v
        chans += c
        seed += 1
    return pack_youtube(vids, chans), vids, chans


# ---- the writer rule, restated for coverage accounting only -----------------------------------------------------------
def _esc_grows(b: bytes) -> bool:
    return len(go_rules.go_json_string(b)) - 2 != len(b)


def _needs_exact(b: bytes) -> bool:
    """warp_esc_len's exact flag: invalid UTF-8, a byte >= 0xF4, or E2 80 (a U+2028 / U+2029 candidate)"""
    try:
        b.decode("utf-8")
    except UnicodeDecodeError:
        return True
    return b"\xe2\x80" in b or any(c >= 0xF4 for c in b)


def yt_writer_mode(v, ch):
    """the writer of a video's line (esc_len[3r+2] of yt_size_lane_kernel): 1 nothing to escape, 2 only the description /
    title need escaping and only their ASCII bytes, 0 the warp writer; None when the record has no line"""
    b = go_rules._bs
    if go_rules._go_time_checked(v.published_sec, v.published_nsec, 0) is None or \
            (ch.cached and go_rules._go_time_checked(ch.published_sec, ch.published_nsec, 0) is None):
        return None
    desc, title = b(v.description), b(v.title)
    small = [b(v.id), b(ch.id), b(v.language)] + [b(x) for x in v.thumbnails.values()]
    if ch.cached:
        small += [b(ch.title), b(ch.description), b(ch.thumb_default), b(ch.country)]
    small += [u.rstrip(b",.;:!?()'\"") for u in go_rules._URL.findall(desc)]
    small_dirty = any(_esc_grows(s) for s in small)
    if not small_dirty and not _esc_grows(desc) and not _esc_grows(title):
        return 1
    return 0 if small_dirty or _needs_exact(desc) or _needs_exact(title) else 2


LEN_CLASSES = ((0, 0), (1, 16), (17, 127), (128, 128), (129, 129), (130, 512), (513, 4998), (4999, 1 << 30))


def yt_edge_coverage(vids, chans) -> collections.Counter:
    """(what, mode, ...) cells of the writer rule that the videos reach: the raw-length class of the description and of the
    title per writer, which of them are longer than YT_LANE_LONG, raw <= 128 with escaped > 128, raw 129 with nothing to
    escape beside an escaped string (the lane writer's pending plain copy)"""
    cls = lambda n: next(j for j, (a, b) in enumerate(LEN_CLASSES) if a <= n <= b)
    cov = collections.Counter()
    for v in vids:
        m = yt_writer_mode(v, chans[v.channel])
        if m is None:
            continue
        d, t = go_rules._bs(v.description), go_rules._bs(v.title)
        cov["desc", m, cls(len(d))] += 1
        cov["title", m, cls(len(t))] += 1
        cov["long", m, len(d) > 128, len(t) > 128] += 1
        for name, s in (("desc", d), ("title", t)):
            e = len(go_rules.go_json_string(s)) - 2
            if len(s) <= 128 < e:
                cov["raw<=128<escaped", m, name] += 1
            if len(s) == 129 and e == 129:
                cov["raw 129 clean", m, name] += 1
        if m == 2 and len(d) > 128 and len(t) > 128 and _esc_grows(d) and _esc_grows(t):
            cov["both long, both escaped", m] += 1
    return cov


def yt_edge_cells() -> list[tuple]:
    """the cells yt_edge_coverage must find non-empty"""
    cells = [(what, m, c) for what in ("desc", "title") for m in (0, 1, 2) for c in range(len(LEN_CLASSES))]
    cells += [("long", m, a, b) for m in (0, 1, 2) for a in (False, True) for b in (False, True)]
    cells += [("raw<=128<escaped", 2, name) for name in ("desc", "title")]
    cells += [("raw 129 clean", m, name) for m in (1, 2) for name in ("desc", "title")]
    cells += [("both long, both escaped", 2)]
    return cells
