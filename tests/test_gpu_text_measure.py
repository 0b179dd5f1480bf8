"""The parse kernels measure message texts for the size pass (tg_links.cuh warp_count_tme_esc): texts made by rule
around the 16-byte lanes and 512-byte strips of that scan, byte for byte against the oracle, and against the size pass
measuring every text itself (TGI_SIZE_TEXT_WARP=1).  Equal emitter byte counters on both paths mean the lane emitter
copied and left exactly the same strings, so no text changed its route to the escape kernels."""
import os

import numpy as np
import pytest

from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import Engine
from distributed_crawler_b200.pack import pack_telegram
from helpers import ALL, assert_results_equal, msg, no_page
from oracle.pyoracle import Oracle

pytestmark = pytest.mark.gpu

EDGES = (16, 32, 48, 128, 256, 496, 512, 1024, 1536, 2048)
ESCAPES = b'"\\\b\t\n\f\r\x00\x01\x1f<>&\x7f/'
SEQS = ["é".encode(), "д".encode(), "中".encode(), "😀".encode(), "अ".encode(), "퟿".encode(),
        "\U00010000".encode(), "\U000fffff".encode(), "\U0010ffff".encode(), "—".encode()]
BAD = [b"\xe2\x80\xa8", b"\xe2\x80\xa9", b"\xe2\x80\x99", b"\xf4\x90\x80\x80", b"\xf5\x80\x80\x80", b"\xc0\x80",
       b"\xc1\xbf", b"\xed\xa0\x80", b"\xe0\x80\x80", b"\xf0\x80\x80\x80", b"\x80", b"\xbf", b"\xff", b"\xf8\x88\x80\x80\x80",
       b"\xc3", b"\xe4\xb8", b"\xf0\x9f\x98", b"\xc3\x28", b"\xe4\x28\xad", b"\xf0\x9f\x28\x80"]


def lengths():
    out = set(range(0, 40))
    for m in range(16, 2101, 16):
        out |= {m - 1, m, m + 1}
    return sorted(x for x in out if x <= 2100)


def fill(n, unit=b"a"):
    """n bytes of whole `unit`s, 'a' in front where the units do not fit"""
    k = n // len(unit)
    return b"a" * (n - k * len(unit)) + unit * k


def texts_lengths():
    out = []
    for n in lengths():
        out += [fill(n), fill(n, "д".encode()), fill(n, "中".encode()), fill(n, "😀".encode()), fill(n, b"a<b>\n")]
        if n >= 2:
            out += [fill(n - 1) + b"\xd0", fill(n - 2, "д".encode()) + "中".encode()[:2]]  # a sequence cut by the end
    return out


def texts_escapes():
    out = []
    for c in ESCAPES:
        for p in list(range(0, 36)) + [127, 128, 129] + list(range(506, 530)):
            for bg in (b"a", "д".encode()):
                out.append(fill(p, bg) + bytes([c]) + fill(30 + p % 7))
        out.append(bytes([c]) * 600)
    return out


def texts_straddling(seqs):
    out = []
    for e in EDGES:
        for sq in seqs:
            for d in range(-len(sq), 2):
                for bg in (b"a", "д".encode()):
                    head = fill(e + d, bg)
                    out.append(head + sq + fill(40))
                    out.append(head + sq)  # the sequence ends the text
                    out.append(head + sq + fill(512 - (len(head) + len(sq)) % 512))  # ... or the text ends with its strip
    return out


def run(batch, label):
    with no_page():
        ro = Oracle().telegram(batch, ALL)
        e = Engine()
        rg = e.telegram(batch, ALL)
        e.close()
        assert rg.gpu_launches > 1
        assert_results_equal(ro, rg, ALL, label)
        os.environ["TGI_SIZE_TEXT_WARP"] = "1"
        try:
            e = Engine()
            rw = e.telegram(batch, ALL)
            e.close()
        finally:
            del os.environ["TGI_SIZE_TEXT_WARP"]
    assert np.array_equal(rw.status, rg.status), f"{label}: status differs with TGI_SIZE_TEXT_WARP=1"
    assert np.array_equal(rw.jsonl, rg.jsonl), f"{label}: JSONL differs with TGI_SIZE_TEXT_WARP=1"
    assert (rw.main_bytes_out, rw.main_bytes_in) == (rg.main_bytes_out, rg.main_bytes_in), \
        f"{label}: the lane emitter copied other strings with TGI_SIZE_TEXT_WARP=1"


def messages(texts):
    """every text as a plain message, as a photo caption, in a message with entities (the other parse kernel) and as the
    text of a document, whose description is its file name"""
    ms = []
    for i, t in enumerate(texts):
        k = i % 4
        if k == 0:
            ms.append(msg("messageText", t))
        elif k == 1:
            ms.append(msg("messagePhoto", t))
        elif k == 2:
            ms.append(msg("messageText", t + b" t.me/somechannel @othername", [(len(t) + 1, 16, "url", ""), (0, 3, "bold", "")]))
        else:
            ms.append(msg("messageDocument", t, alt="file<%d>.pdf" % i))
    return ms


@pytest.mark.parametrize("part", ["lengths", "escapes", "straddling", "bad"])
def test_text_measure(part):
    texts = {"lengths": texts_lengths, "escapes": texts_escapes, "straddling": lambda: texts_straddling(SEQS),
             "bad": lambda: texts_straddling(BAD)}[part]()
    for k in range(4):  # every text in every one of the four roles
        run(pack_telegram(messages(texts[k:] + texts[:k])), f"{part}/{k}")
