"""The parse kernels classify each lane's 16 text bytes before they measure them (tg_links.cuh warp_count_tme_esc):
ASCII, two-byte only (no byte >= 0xE0 in the lane or in the last three bytes in front of it), or anything else.
Texts whose class changes exactly at those boundaries — a lane's first byte, the 1-3 bytes in front of it, the last
lane of a 512-byte strip, the strip boundary, the end of the text — byte for byte against the oracle and against the
size pass measuring every text itself (TGI_SIZE_TEXT_WARP=1), with equal lane-emitter byte counters on both paths."""
import pytest

import test_gpu_text_measure as tm
from distributed_crawler_b200.pack import pack_telegram

pytestmark = pytest.mark.gpu

CYR = "д".encode()
EDGES = (16, 32, 496, 512, 1008, 1024)  # lane starts; 496 is a strip's last lane, 512 and 1024 strip starts
LONG = [b"\xe4\xb8\xad", "😀".encode(), b"\xe2\x84\xa2", b"\xe2\x80\x94", b"\xe2\x80\xa8", b"\xe2\x80\xa9", b"\xe2\x80\x99",
        b"\xf4\x90\x80\x80", b"\xf4\x8f\xbf\xbf", b"\xed\xa0\x80", b"\xed\x9f\xbf", b"\xe0\xa0\x80", b"\xe0\x80\x80",
        b"\xf0\x80\x80\x80", b"\xe4\xb8", b"\xf0\x9f\x98"]  # 3- and 4-byte sequences, clean, not clean and cut short


def texts_long_lead():
    """one 3- or 4-byte sequence in two-byte text, its lead on a lane's first byte, in the 1-4 bytes in front of it,
    in a strip's last lane or across a strip"""
    out = []
    for e in EDGES:
        for d in range(-4, 2):
            for sq in LONG:
                head = tm.fill(e + d, CYR)
                out += [head + sq + tm.fill(40, CYR), head + sq, head + sq + tm.fill(512 - (len(head) + len(sq)) % 512, CYR)]
    return out


def texts_overlong_two():
    """C0 80 / C1 BF inside Cyrillic text around the same boundaries"""
    out = []
    for e in EDGES:
        for d in range(-3, 3):
            for bad in (b"\xc0\x80", b"\xc1\xbf", b"\xc2\x80", b"\xdf\xbf"):
                out.append(tm.fill(e + d, CYR) + bad + tm.fill(24, CYR))
    return out


def texts_two_byte_lead_at_end():
    """a 2-byte lead as the last byte of a lane, a strip or the text: completed in the next lane, cut by ASCII, or cut
    by the end"""
    out = []
    for e in EDGES:
        for bg in (b"a", CYR):
            out += [tm.fill(e - 1, bg) + CYR + tm.fill(30, bg), tm.fill(e - 1, bg) + b"\xd0abc" + tm.fill(20, bg),
                    tm.fill(e - 1, bg) + b"\xd0", tm.fill(e - 1, bg) + b"\xd0\xd0\xb4" + tm.fill(20, bg)]
    return out


def texts_specials():
    """each special byte in each of the four words of an ASCII lane and of a two-byte lane, and lanes with several"""
    out = []
    for c in tm.ESCAPES:
        for base in (0, 16, 496, 512):
            for k in range(4):
                for j in (0, 1, 3):
                    for bg in (b"a", CYR):
                        p = base + 4 * k + j
                        out.append(tm.fill(p, bg) + bytes([c]) + tm.fill(30, bg))
    for p in range(0, 34):
        for bg in (b"a", CYR):
            out.append(tm.fill(p, bg) + b'\n"<' + tm.fill(5, bg) + b"\x00 &\\" + tm.fill(9, bg) + b"\t\r>" + tm.fill(20, bg))
    return out


@pytest.mark.parametrize("part", ["long_lead", "overlong_two", "lead_at_end", "specials"])
def test_text_classes(part):
    texts = {"long_lead": texts_long_lead, "overlong_two": texts_overlong_two, "lead_at_end": texts_two_byte_lead_at_end,
             "specials": texts_specials}[part]()
    for k in range(4):  # every text in every one of the four roles
        tm.run(pack_telegram(tm.messages(texts[k:] + texts[:k])), f"{part}/{k}")
