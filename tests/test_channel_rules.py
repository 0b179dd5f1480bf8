"""The random-walk StoreChannelData line (tgi_channel_batch) on the CPU: the C restatement (tests/channel_oracle.c)
against the independent Python restatement channel_rules.channel_data_line, byte for byte, on seeded batches and on an
edge corpus built here: chat ids at the int64 ends and every 10^k boundary, counts at the int32 ends, empty and 64 KiB
titles, every character class encoding/json escapes (and invalid or truncated UTF-8) at both ends of every string, and
URLs of 0 to 64 bytes.  The C restatement must refuse the malformed batches the library refuses, with its code.  tests/test_gpu_channel_records.py
runs the same corpus and the same refusals through the GPU."""
import random

import numpy as np
import pytest

import channel_rules
import go_rules
from distributed_crawler_b200 import abi
from distributed_crawler_b200.pack import ChannelRecord, pack_channels
from channel_oracle import ChannelOracle
from oracle.pyoracle import OracleError

SEEDS = (1, 2, 3)
I64_MIN, I64_MAX, I32_MIN, I32_MAX = -(2 ** 63), 2 ** 63 - 1, -(2 ** 31), 2 ** 31 - 1
STR_MAX = (1 << 24) - 1  # the library's limit per string

CHAT_IDS = sorted({I64_MIN, I64_MIN + 1, I64_MAX, I64_MAX - 1, 0, 1, -1} |
                  {s * (10 ** k + d) for k in range(1, 19) for d in (-1, 0) for s in (1, -1)})
COUNT_VALUES = (I32_MIN, I32_MIN + 1, -1, 0, 1, I32_MAX - 1, I32_MAX)
COUNT_FIELDS = ("member_count", "message_count", "total_views")
TITLE_LENS = (0, 1, 2, 15, 16, 17, 31, 32, 33, 127, 128, 129, 4096, 65535, 65536)
URL_LENS = tuple(range(65))
STRING_FIELDS = ("title", "image", "url")
# what encoding/json treats specially, and the rune widths it copies as they are; each piece is one class at an end
PIECES = {
    "lt": b"<", "gt": b">", "amp": b"&", "quote": b'"', "backslash": b"\\", "u2028": "\u2028".encode(),
    "u2029": "\u2029".encode(), "control": b"\x01", "nul": b"\x00", "newline": b"\n", "del": b"\x7f", "rune1": b"a",
    "rune2": "é".encode(), "rune3": "€".encode(), "rune4": "\U0001F600".encode(), "invalid": b"\xff",
    "continuation": b"\x80", "truncated": "€".encode()[:2], "truncated4": "\U0001F600".encode()[:3],
}
ENDS = ("start", "end")


def edge_cells():
    """every cell the edge corpus declares"""
    cells = {("chat_id", v) for v in CHAT_IDS}
    cells |= {("count", f, v) for f in COUNT_FIELDS for v in COUNT_VALUES}
    cells |= {("title_len", n) for n in TITLE_LENS}
    cells |= {("image", "empty"), ("image", "set")}
    cells |= {("url_len", n) for n in URL_LENS}
    cells |= {("end", f, k, at) for f in STRING_FIELDS for k in PIECES for at in ENDS}
    return cells


def _text(rng, n):
    """n bytes of mixed text: plain ASCII with escapes and runes of every width"""
    alphabet = [b"a", b"Z", b"0", b" ", b"_", b"<", b"&", b'"', b"\\", b"\x1f", "é".encode(), "€".encode(),
                "\U0001F600".encode(), "\u2028".encode()]
    out = bytearray()
    while len(out) < n:
        out += rng.choice(alphabet) if rng.random() < 0.3 else b"x"
    return bytes(out[:n])


def _url(rng, n):
    return bytes(rng.choice(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789_") for _ in range(n))


def _plain(rng):
    return ChannelRecord(chat_id=rng.randrange(-10 ** 13, 10 ** 13), title=_text(rng, rng.randrange(1, 40)),
                         image=_text(rng, rng.randrange(0, 60)) if rng.random() < 0.7 else b"",
                         url=_url(rng, rng.randrange(5, 33)), member_count=rng.randrange(0, 10 ** 7),
                         message_count=rng.randrange(0, 10 ** 5), total_views=rng.randrange(0, 10 ** 9))


def make_channels(n, seed):
    """n ordinary channel records"""
    rng = random.Random(seed)
    return [_plain(rng) for _ in range(n)]


def make_channel_edges(seed):
    """the edge records, in a seeded order, with a few ordinary ones among them"""
    rng = random.Random(1000 + seed)
    recs = []
    for v in CHAT_IDS:
        r = _plain(rng)
        r.chat_id = v
        recs.append(r)
    for f in COUNT_FIELDS:
        for v in COUNT_VALUES:
            r = _plain(rng)
            setattr(r, f, v)
            recs.append(r)
    for n in TITLE_LENS:
        r = _plain(rng)
        r.title = _text(rng, n)
        recs.append(r)
    for img in (b"", _text(rng, 300)):
        r = _plain(rng)
        r.image = img
        recs.append(r)
    for n in URL_LENS:
        r = _plain(rng)
        r.url = _url(rng, n)
        recs.append(r)
    for f in STRING_FIELDS:
        for k, piece in PIECES.items():
            for at in ENDS:
                r = _plain(rng)
                body = _url(rng, rng.randrange(1, 12))
                setattr(r, f, piece + body if at == "start" else body + piece)
                recs.append(r)
    recs += make_channels(40, seed)
    rng.shuffle(recs)
    return recs


def _end_class(b: bytes, at: str):
    """the class of the first / last character of b, as encoding/json sees it"""
    if not b:
        return None
    if at == "end":  # an incomplete sequence at the very end: a lead byte with fewer continuations than it needs
        for back in (1, 2, 3):
            if len(b) >= back and 0xC2 <= b[-back] <= 0xF4:
                need = 2 if b[-back] < 0xE0 else 3 if b[-back] < 0xF0 else 4
                if need > back and all(0x80 <= x < 0xC0 for x in b[len(b) - back + 1:]):
                    return "truncated" if need == 3 else "truncated4" if need == 4 else None
                break
        i = len(b) - 1
        while i > 0 and 0x80 <= b[i] < 0xC0 and len(b) - i < 4:
            i -= 1
        r, w = go_rules.go_decode_rune(b, i)
        if i + w != len(b):  # the last byte is a continuation byte that no lead claims
            return "continuation" if 0x80 <= b[-1] < 0xC0 else None
        first = b[i:]
    else:
        r, w = go_rules.go_decode_rune(b, 0)
        first = b[:w]
        if r == 0xFFFD and w == 1:
            if 0x80 <= b[0] < 0xC0:
                return "continuation"
            if b[0] >= 0xE0 and b[0] < 0xF0 and len(b) >= 2 and 0x80 <= b[1] < 0xC0 and (len(b) < 3 or not 0x80 <= b[2] < 0xC0):
                return "truncated"
            if b[0] >= 0xF0 and len(b) >= 3 and all(0x80 <= x < 0xC0 for x in b[1:3]) and (len(b) < 4 or not 0x80 <= b[3] < 0xC0):
                return "truncated4"
            return "invalid" if b[0] in (0xFF, 0xFE, 0xC0, 0xC1) or b[0] > 0xF4 else None
    for k, piece in PIECES.items():
        if first == piece and k not in ("truncated", "truncated4", "continuation"):
            return k
    if len(first) == 1 and first[0] < 0x20:
        return {0: "nul", 10: "newline", 1: "control"}.get(first[0], "control")
    return {1: "rune1", 2: "rune2", 3: "rune3", 4: "rune4"}[len(first)] if first.decode("utf-8", "ignore") else None


def edge_coverage(recs):
    """the cells the records reach, measured on the records themselves"""
    got = set()
    for r in recs:
        got.add(("chat_id", r.chat_id))
        for f in COUNT_FIELDS:
            got.add(("count", f, getattr(r, f)))
        got.add(("title_len", len(r.title)))
        got.add(("image", "set" if r.image else "empty"))
        got.add(("url_len", len(r.url)))
        for f in STRING_FIELDS:
            for at in ENDS:
                k = _end_class(bytes(getattr(r, f)), at)
                if k:
                    got.add(("end", f, k, at))
    return got


def restated(recs):
    """(status, line_off, jsonl) of the restatement"""
    lines = [channel_rules.channel_data_line(r) for r in recs]
    off = np.zeros(len(lines) + 1, np.uint64)
    off[1:] = np.cumsum([len(x) for x in lines], dtype=np.uint64)
    return np.full(len(lines), abi.ST_EMITTED, np.uint8), off, b"".join(lines)


def assert_equals_restatement(r, recs, label):
    status, off, jsonl = restated(recs)
    if r.jsonl.tobytes() != jsonl or not np.array_equal(r.line_off, off):
        for i, rec in enumerate(recs):
            assert r.line(i) == channel_rules.channel_data_line(rec), f"{label}: record {i} differs from the restatement"
    assert np.array_equal(r.status, status), f"{label}: status"
    assert np.array_equal(r.line_off, off) and r.jsonl.tobytes() == jsonl, f"{label}: differs from the restatement"


# ---- malformed batches: every string range is checked before anything reads it ---------------------------------------
def malformed(kind, at, n=50):
    """a batch of n records whose record `at` is broken in one way; -> (batch, at)"""
    recs = make_channels(n, seed=77)
    b = pack_channels(recs)
    r = b.recs[at]
    size = b.strs.size
    if kind == "past_end":  # the url runs one byte past strs
        r["url_len"] += size - int(r["str_off"] + r["title_len"] + r["image_len"] + r["url_len"]) + 1
    elif kind == "offset_past_end":
        r["str_off"] = size + 1
        r["title_len"] = r["image_len"] = r["url_len"] = 0
    elif kind == "wraps":  # str_off + lengths wraps around 2^64
        r["str_off"] = 2 ** 64 - 2
    elif kind == "title_past_end":
        r["title_len"] = size + 1
    elif kind == "too_long":  # a string of 16 MiB inside strs: refused by the length rule alone
        big = np.zeros(STR_MAX + 1 + 16, np.uint8)
        big[:size] = b.strs
        b.strs = big[:STR_MAX + 1]
        r["str_off"], r["title_len"], r["image_len"], r["url_len"] = 0, 0, STR_MAX + 1, 0
    else:
        raise ValueError(kind)
    return b, at


BAD_KINDS = ("past_end", "offset_past_end", "wraps", "title_past_end", "too_long")
BAD_AT = {"first": 0, "middle": 25, "last": 49}


# ---- tests -----------------------------------------------------------------------------------------------------------
def test_record_layout_matches_the_header():
    import re
    import os
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "tgingest.h")).read()
    body = re.search(r"typedef struct tgi_ch_rec \{.*?\} tgi_ch_rec;", hdr, re.S).group(0)
    names = re.findall(r"^\s*(?:u?int\d+_t)\s+(\w+);", body, re.M)
    assert names == list(abi.CH_REC.names) and abi.CH_REC.itemsize == 40
    assert [f for f, _ in abi.ChBatchC._fields_] == ["n", "recs", "strs", "strs_len"]


@pytest.mark.parametrize("seed", SEEDS)
def test_seeded_batches_oracle_vs_restatement(seed):
    recs = make_channels(500 + seed, seed)
    assert_equals_restatement(ChannelOracle().channel(pack_channels(recs)), recs, f"seed {seed}")


@pytest.mark.parametrize("seed", SEEDS)
def test_edges_oracle_vs_restatement(seed):
    recs = make_channel_edges(seed)
    for flags in (abi.RUN_JSONL, abi.RUN_JSONL | abi.RUN_JSONL_DEVICE):
        assert_equals_restatement(ChannelOracle().channel(pack_channels(recs), flags), recs, f"seed {seed}, flags {flags:#x}")


@pytest.mark.parametrize("seed", SEEDS)
def test_edges_reach_every_cell(seed):
    recs = make_channel_edges(seed)
    missing = sorted(edge_cells() - edge_coverage(recs), key=repr)
    assert not missing, missing


def test_restatement_spot_checks():
    """fixed lines, written out by hand from model/data.go and encoding/json"""
    r = ChannelRecord(chat_id=-1001234567890, title=b"A<b>&\xe2\x80\xa8\xff", image=b"", url=b"durov", member_count=I32_MAX,
                      message_count=I32_MIN, total_views=0)
    want = (b'{"channel_id":"-1001234567890","channel_name":"A\\u003cb\\u003e\\u0026\\u2028\\ufffd",'
            b'"channel_description":"","channel_profile_image":"","channel_engagement_data":{"follower_count":2147483647,'
            b'"following_count":0,"like_count":0,"post_count":-2147483648,"views_count":0,"comment_count":0,'
            b'"share_count":0},"channel_url_external":"https://t.me/durov","channel_url":"https://t.me/durov",'
            b'"country_code":"","published_at":"0001-01-01T00:00:00Z"}\n')
    assert channel_rules.channel_data_line(r) == want
    assert ChannelOracle().channel(pack_channels([r])).line(0) == want


def test_empty_batch_and_no_lines():
    o = ChannelOracle()
    r = o.channel(pack_channels([]))
    assert r.n == 0 and r.jsonl.size == 0 and list(r.line_off) == [0]
    recs = make_channels(10, 3)
    r = o.channel(pack_channels(recs), 0)  # without TGI_RUN_JSONL: the statuses, no lines
    assert (r.status == abi.ST_EMITTED).all() and r.jsonl.size == 0 and not r.line_off.any()


@pytest.mark.parametrize("kind", BAD_KINDS)
def test_oracle_refuses_malformed_ranges(kind):
    o = ChannelOracle()
    good = pack_channels(make_channels(50, seed=77))
    want = o.channel(good)
    for where, at in BAD_AT.items():
        b, _ = malformed(kind, at)
        with pytest.raises(OracleError) as ei:
            o.channel(b)
        assert ei.value.code == abi.E_ARG, (kind, where)
        r = o.channel(good)
        assert np.array_equal(r.jsonl, want.jsonl) and np.array_equal(r.line_off, want.line_off)


def test_oracle_refuses_other_run_flags():
    o = ChannelOracle()
    b = pack_channels(make_channels(5, 1))
    for flags in (abi.RUN_LINKS, abi.RUN_FRONTIER, abi.RUN_NO_D2H, abi.RUN_FILTER, abi.RUN_SKIP_SELF, abi.RUN_SKIP_INVALID,
                  abi.RUN_JSONL | abi.RUN_LINKS, 0x100):
        with pytest.raises(OracleError) as ei:
            o.channel(b, flags)
        assert ei.value.code == abi.E_ARG, hex(flags)


def test_longest_strings_accepted():
    """a string of 16 MiB - 1 bytes is inside the limit"""
    r = ChannelRecord(chat_id=5, title=b"<" * 1000, image=b"a" * STR_MAX, url=b"u")
    line = ChannelOracle().channel(pack_channels([r])).line(0)
    assert line == channel_rules.channel_data_line(r)
