"""tg_ent_map_kernel maps the UTF-16 entity offsets of 32 records per warp over one packed stream of 16-byte chunks (32
per pass), tg_parse_kernel counts and measures the texts of records with entities in its packed stream as well, and
tg_parse_ent_kernel only extracts their links, without the plaintext scan when the text holds no "t.me/".  Batches built
around that, byte for byte against the CPU oracle on the bulk pipeline (JSONL, links only, TANDEM): entity offsets and
ends on the chunk and pass seams of the stream, inside a surrogate pair (FAILED), negative, at the text's unit count,
past it, of length 0; several entities in one chunk and more than 32 in one record; texts without "t.me/"; records with
and without entities in one group; ASCII texts, whose entities tg_parse_kernel maps itself; texts that are not clean
(invalid UTF-8, E2 80 xx next to an entity), which take the warp-per-record mapping; and batches of n not a multiple of
32."""
import random

import pytest

from distributed_crawler_b200 import abi
from distributed_crawler_b200.pack import pack_telegram
from helpers import ALL, TANDEM, msg
from test_gpu_packed_scan import CHANNELS, MIN_POST_DATE, check, out_of_order

pytestmark = pytest.mark.gpu

PIECES = ["word ", "@mention_one ", "@Second_Name ", "t.me/chan_alpha ", "https://t.me/Chan_Beta/7 ", "t.me/selfchan1 ",
          "д", "中", "😀", "ok 😀😀 ", "x" * 20, "\n", '"q" ', "ab "]
PLAIN = [p for p in PIECES if "t.me" not in p]  # texts without "t.me/": tg_parse_ent_kernel skips the plaintext scan
ASCII = [p for p in PIECES if p.isascii()]  # ASCII texts: tg_parse_kernel maps their entities itself
CARRIERS = ["messageText", "messagePhoto", "messageVideo", "messageDocument"]
LENGTHS = [0, 1, 15, 16, 17, 31, 32, 33, 100, 300, 511, 512, 513, 1000, 1100]
KINDS = ["mention", "url", "mention", "url", "text_url", "bold"]
UNCLEAN = [b"\xff", b"\x80", b"\xc0\xaf", b"\xe2\x80\xa8", b"\xe2\x80\x8b", b"\xf4\x80\x80\x80", b"\xed\xa0\x80", b"\xe4\xb8"]
SEEDS = (1, 2, 3)


def text_of(rng, n, pieces):
    """whole pieces up to about n bytes (UTF-8)"""
    out = ""
    while len(out.encode()) < n:
        out += rng.choice(pieces)
    return out.encode()


def rune_starts(text):
    """(byte index, UTF-16 unit) of every rune start of a valid text, and its unit count"""
    out, b, u = [], 0, 0
    for ch in text.decode():
        out.append((b, u))
        b += len(ch.encode())
        u += 2 if ord(ch) >= 0x10000 else 1
    return out, u


def entities(rng, text, k):
    """k entities whose offsets and ends land on the stream's seams and its edge cases"""
    try:
        starts, total = rune_starts(text)
    except UnicodeDecodeError:  # not clean: offsets by bytes (the mapping walks the bytes Go's way)
        starts, total = [(i, i) for i in range(len(text))], len(text)
    seams = [u for b, u in starts if b % 16 in (0, 1, 15) or b % 512 in (0, 511)] or [0]
    pairs = [u + 1 for b, u in starts if text[b] >= 0xF0] or [0]  # the second unit of a surrogate pair
    out = []
    for _ in range(k):
        r = rng.random()
        off = (rng.choice(seams) if r < 0.45 else rng.choice(pairs) if r < 0.55 else rng.choice([-1, -7, total, total + 3])
               if r < 0.62 else rng.randrange(total + 1))
        r = rng.random()
        if r < 0.4:
            end = rng.choice(seams)
        elif r < 0.48:
            end = rng.choice(pairs)
        elif r < 0.58:
            end = total
        else:
            end = off + rng.choice([0, 0, 1, 5, 12, 40])
        ln = end - off if rng.random() < 0.9 else rng.choice([-1, -3, 1 << 30])
        out.append((off, ln, rng.choice(KINDS), "https://t.me/from_entity" if rng.random() < 0.5 else "https://x.org/a"))
    return out


def make_messages(seed, n):
    rng = random.Random(seed)
    ms = []
    for i in range(n):
        kw = dict(id=(i + 1) << 20, channel=i % len(CHANNELS))
        if rng.random() < 0.03:
            kw["date"] = 1_600_000_000  # before MIN_POST_DATE in the configured runs
        L = rng.choice(LENGTHS)
        text = text_of(rng, L, rng.choice([PLAIN, ASCII, PIECES, PIECES]))
        r = rng.random()
        if r < 0.15 and text:  # not clean: the warp-per-record mapping, bytes that are one rune each in Go
            p = rng.randrange(len(text) + 1)
            text = text[:p] + rng.choice(UNCLEAN) + text[p:]
        r = rng.random()
        if r < 0.3:
            ms.append(msg(rng.choice(CARRIERS), text, **kw))  # no entities, in the same groups
        elif r < 0.35:
            ms.append(msg("messageSticker", text, [(0, 3, "mention", "")], alt="🙂", **kw))  # no links carried
        elif r < 0.38:
            ms.append(msg("messagePhoto", b"", [(0, 0, "mention", ""), (0, 1, "url", "")], **kw))  # an empty text
        else:
            k = rng.choice([1, 1, 2, 3, 5, 8, 33, 40])
            ms.append(msg(rng.choice(CARRIERS), text, entities(rng, text, k), **kw))
    return ms


@pytest.mark.parametrize("flags", [ALL, TANDEM, abi.RUN_LINKS], ids=["all", "tandem", "links"])
@pytest.mark.parametrize("seed", SEEDS)
def test_packed_entities(seed, flags):
    n = 32 * 40 + 7 * seed  # not a multiple of 32
    batch = pack_telegram(make_messages(seed, n), CHANNELS)
    ro = check(batch, flags, f"seed {seed}")
    assert len(ro.links) > 100 and (ro.status == abi.ST_FAILED).sum() > 0
    check(out_of_order(batch, seed), flags, f"seed {seed}, strs out of record order")


def test_entities_on_every_unit():
    """one text with a rune of every length, an entity starting and one ending on each of its units, from one chunk
    into the next pass: every rune start of the stream is placed, and every unit inside a surrogate pair fails"""
    text = ("a" * 13 + "😀д中" + "b" * 470 + "中😀x" + "@mention_one t.me/chan_alpha " * 2).encode()
    _, total = rune_starts(text)
    ms = []
    for u in range(-1, total + 2):
        ms.append(msg("messageText", text, [(u, 5, "mention", ""), (0, u, "url", ""), (u, 0, "url", "")], id=(len(ms) + 1) << 20))
        ms.append(msg("messageText", text, [(u, total - u, "url", "")] * 3, id=(len(ms) + 1) << 20))
    batch = pack_telegram(ms, CHANNELS)
    for flags in (ALL, TANDEM):
        ro = check(batch, flags, "every unit")
        assert (ro.status == abi.ST_FAILED).sum() > 0 and (ro.status == abi.ST_EMITTED).sum() > 0


@pytest.mark.parametrize("n", [1, 5, 31, 33, 95])
def test_packed_entities_small_batches(n):
    """the last group short of 32 records, and min_post_date skipping records with entities"""
    batch = out_of_order(pack_telegram(make_messages(100 + n, n), CHANNELS), n)
    check(batch, ALL, f"n {n}", min_post_date=MIN_POST_DATE)
    check(batch, TANDEM, f"n {n}, tandem", min_post_date=MIN_POST_DATE)
