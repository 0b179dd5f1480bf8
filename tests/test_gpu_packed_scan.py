"""tg_parse_kernel scans the texts of a group of 32 records (the records without entities) as ONE packed stream of
16-byte chunks, 32 chunks (512 bytes) per pass, each lane on the chunk of whichever record holds it.  Batches built
around that stream's seams, byte for byte against the CPU oracle on the bulk pipeline: texts ending exactly on a chunk
or on a pass of the stream, a multi-byte sequence or a "t.me/" cut between two records' chunks (which must not join
up), texts stored out of record order in `strs` with such bytes in front of them, groups mixing records with and without
entities, records without text to scan, and batches of n not a multiple of 32.  The JSONL runs take the instance that
measures the texts as well and are also held against the size pass measuring every text itself (TGI_SIZE_TEXT_WARP=1);
TANDEM and RUN_LINKS alone take the link-only instance."""
import os
import random

import numpy as np
import pytest

from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import Engine
from distributed_crawler_b200.pack import Channel, TgBatch, pack_telegram
from helpers import ALL, TANDEM, assert_results_equal, msg, no_page
from oracle.pyoracle import Oracle

pytestmark = pytest.mark.gpu

CHANNELS = [Channel(title="self", name="selfchan1", username="selfchan1"), Channel(title="other", name="", username="")]
MIN_POST_DATE = 1_650_000_000
# (end of one record's text, start of the next one's): joined, they would be a valid sequence or a "t.me/" link
SEAMS = [(b"\xe4\xb8", b"\xad and more"), (b"\xf0\x9f", b"\x98\x80 x"), (b"\xd0", b"\xb4 y"), (b"go t.me", b"/seamchan_one z"),
         (b"see https://t.", b"me/seamchan_two"), (b"x t", b".me/seamchan_3"), ("ok д".encode(), b"/plain"),
         (b"a", b"a")]
PIECES = [b"word ", b"t.me/chan_alpha ", b"https://t.me/Chan_Beta/12 ", b"t.me/selfchan1 ", b"t.me/joinchat ", b"@mention_x ",
          "д".encode(), "中".encode(), "😀".encode(), b'"q" ', b"<b>&amp;", b"\n", b"\t", b"\\", b"t.me/ab ", b"x" * 40]
LENGTHS = [0, 1, 4, 15, 16, 17, 31, 32, 33, 100, 180, 315, 496, 511, 512, 513, 528, 1024, 1500, 2048]
CARRIERS = ["messageText", "messagePhoto", "messageVideo", "messageDocument"]
SEEDS = (1, 2, 3)


def body(rng, n, head=b"", tail=b""):
    """a text of exactly n bytes (n >= len(head) + len(tail)): head, whole pieces, 'a' padding, tail"""
    room = n - len(head) - len(tail)
    out = bytearray()
    while True:
        p = rng.choice(PIECES)
        if len(out) + len(p) > room:
            break
        out += p
    return head + bytes(out) + b"a" * (room - len(out)) + tail


def group_lengths(rng, k):
    """chunk counts that end records on the stream's seams: one pass, a pass split in two, one chunk each, ..."""
    pick = rng.randrange(5)
    if pick == 0:
        return [16 * rng.choice([1, 2, 12, 20, 31, 32, 33]) for _ in range(k)]  # texts ending on a chunk
    if pick == 1:
        a = rng.randrange(1, 32)
        return [16 * a, 16 * (32 - a)] * (k // 2) + [512] * (k % 2)  # pairs that fill a pass
    if pick == 2:
        return [16] * k  # one chunk each: one pass per group
    if pick == 3:
        return [rng.choice([511, 512, 513, 1023, 1024, 1025]) for _ in range(k)]
    return [rng.choice(LENGTHS) for _ in range(k)]


def make_messages(seed, n):
    rng = random.Random(seed)
    ms, lens = [], []
    while len(lens) < n:
        lens += group_lengths(rng, 32)
    carry = b""  # the start the previous text's seam asks for
    for i in range(n):
        seam = rng.choice(SEAMS)
        L = max(lens[i], len(carry) + len(seam[0]))
        text = body(rng, L, carry, seam[0])
        carry = seam[1]
        kw = dict(id=(i + 1) << 20, channel=i % len(CHANNELS))
        r = rng.random()
        if r < 0.03:
            kw["panics"] = True
        elif r < 0.06:
            kw["date"] = 1_600_000_000  # before MIN_POST_DATE in the configured runs
        r = rng.random()
        if r < 0.25:  # records with entities: tg_parse_ent_kernel, in the same groups
            ents = [(0, min(len(text), 5), "bold", ""), (0, 3, "url", ""), (1, 6, "mention", ""),
                    (0, 0, "text_url", "https://t.me/from_entity")]
            ms.append(msg(rng.choice(CARRIERS), text, ents[:rng.randrange(1, 5)], **kw))
        elif r < 0.32:
            ms.append(msg("messageSticker", text, alt="🙂", **kw))  # a text that carries no links
        elif r < 0.37:
            ms.append(msg("messagePhoto", None, **kw))  # no caption
        elif r < 0.42:
            ms.append(msg("messagePhoto", b"", **kw))  # an empty one
        else:
            ms.append(msg(rng.choice(CARRIERS), text, **kw))
    return ms


def out_of_order(batch, seed):
    """the same batch with every record's strings moved to a shuffled place in `strs`, each after bytes that would
    continue a sequence or a link if the scan read in front of the text"""
    rng = random.Random(seed)
    recs = batch.recs.copy()
    order = list(range(batch.n))
    rng.shuffle(order)
    strs = bytearray()
    for i in order:
        rc = batch.recs[i]
        a = int(rc["str_off"])
        m = int(rc["text_len"]) + int(rc["alt_len"]) + int(rc["media_len"]) + int(rc["handle_len"])
        strs += rng.choice([b"t.me", b"\xe4", b"\xf0\x9f\x98", b"", b"https://t.", b"\\"])
        recs[i]["str_off"] = len(strs)
        strs += batch.strs[a:a + m].tobytes()
    arrays = {k: getattr(batch, k) for k in TgBatch.FIELDS}
    arrays.update(recs=recs, strs=np.frombuffer(bytes(strs) + bytes(64), np.uint8).copy())
    return TgBatch(**arrays)


def check(batch, flags, label, **cfg):
    with no_page():
        o, e = Oracle(**cfg), Engine(**cfg)
        try:
            ro, rg = o.telegram(batch, flags), e.telegram(batch, flags)
            assert rg.gpu_launches > 1
            assert_results_equal(ro, rg, flags, label)
            if flags & abi.RUN_FRONTIER:
                assert np.array_equal(o.frontier_export(), e.frontier_export()), f"{label}: frontier differs"
        finally:
            e.close()
            o.close()
        if not flags & abi.RUN_JSONL:
            return ro
        os.environ["TGI_SIZE_TEXT_WARP"] = "1"
        try:
            e = Engine(**cfg)
            rw = e.telegram(batch, flags)
            e.close()
        finally:
            del os.environ["TGI_SIZE_TEXT_WARP"]
    assert np.array_equal(rw.jsonl, rg.jsonl), f"{label}: JSONL differs with TGI_SIZE_TEXT_WARP=1"
    assert (rw.main_bytes_out, rw.main_bytes_in) == (rg.main_bytes_out, rg.main_bytes_in), \
        f"{label}: the lane emitter copied other strings with TGI_SIZE_TEXT_WARP=1"
    return ro


@pytest.mark.parametrize("flags", [ALL, TANDEM, abi.RUN_LINKS], ids=["all", "tandem", "links"])
@pytest.mark.parametrize("seed", SEEDS)
def test_packed_scan_seams(seed, flags):
    n = 32 * 60 + 13 * seed  # not a multiple of 32
    batch = pack_telegram(make_messages(seed, n), CHANNELS)
    ro = check(batch, flags, f"seed {seed}")
    assert len(ro.links) > 100 and (ro.status == abi.ST_FAILED).sum() > 0
    check(out_of_order(batch, seed), flags, f"seed {seed}, strs out of record order")


@pytest.mark.parametrize("n", [1, 5, 31, 33, 95])
def test_packed_scan_small_batches(n):
    """the last group short of 32 records, and min_post_date skipping records that hold links"""
    batch = out_of_order(pack_telegram(make_messages(100 + n, n), CHANNELS), n)
    check(batch, ALL, f"n {n}", min_post_date=MIN_POST_DATE)
    check(batch, TANDEM, f"n {n}, tandem", min_post_date=MIN_POST_DATE)
