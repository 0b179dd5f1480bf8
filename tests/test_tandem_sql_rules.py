"""CPU tests: tests/tandem_sql_rules.py, the restatement tgi_state_edge_sql is checked against: the reference's literals,
encoding/json's string, integer and time rules on every value, the bulk texts, and the rule that cutting a bulk
statement's params into rows of 7 / 8 / 1 values gives the one-row calls; and the C layout of the output."""
import ctypes as C
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest

import tandem_sql_rules as sr
from distributed_crawler_b200 import abi
from test_zones import ZONES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NY = ZONES["America/New_York"]
NOW = 1_760_000_000


def batch(n=0, **kw):
    b = {"batch_id": b"%08d-0000-4000-8000-000000000000" % n, "source_channel": b"owner", "source_page_id": b"pid",
         "source_depth": 2, "sequence_id": b"seq"}
    b.update(kw)
    return b


def edge(name=b"chan01", src=0, status=0):
    return {"destination": name, "source_type": src, "status": status}


def test_one_row_texts_are_the_reference_literals():
    assert sr.sql_text(sr.BATCH_INSERT, 1) == (
        b"INSERT INTO pending_edge_batches (batch_id, crawl_id, source_channel, source_page_id, source_depth, "
        b"sequence_id, status) VALUES ($1, $2, $3, $4, $5, $6, $7);")
    assert sr.sql_text(sr.EDGE_INSERT, 1) == (
        b"INSERT INTO pending_edges (batch_id, crawl_id, destination_channel, source_channel, sequence_id, "
        b"discovery_time, source_type, validation_status) VALUES ($1, $2, $3, $4, $5, $6, $7, $8);")
    assert sr.sql_text(sr.BATCH_CLOSE, 1) == \
        b"UPDATE pending_edge_batches SET status = 'closed', closed_at = NOW() WHERE batch_id = $1;"


def test_bulk_texts_number_the_placeholders_on():
    assert sr.sql_text(sr.EDGE_INSERT, 2).endswith(
        b"VALUES ($1, $2, $3, $4, $5, $6, $7, $8), ($9, $10, $11, $12, $13, $14, $15, $16);")
    assert sr.sql_text(sr.BATCH_INSERT, 2).endswith(b"VALUES ($1, $2, $3, $4, $5, $6, $7), ($8, $9, $10, $11, $12, $13, $14);")
    assert sr.sql_text(sr.BATCH_CLOSE, 3) == \
        b"UPDATE pending_edge_batches SET status = 'closed', closed_at = NOW() WHERE batch_id IN ($1, $2, $3);"
    big = sr.sql_text(sr.EDGE_INSERT, sr.MAX_ROWS)
    assert big.endswith(b"$65527, $65528);") and big.count(b"$") == 8 * sr.MAX_ROWS <= 65535


def test_one_row_params_are_json_marshal_of_the_values():
    t = sr.discovery_time(NOW, 120_000_000)
    calls = sr.reference_calls([(batch(), [edge(b"chan01", 1), edge(b"chan02", 3, abi.EDGE_DUPLICATE)])], b"crawl-1", t)
    assert [c[0] for c in calls] == [sr.BATCH_INSERT, sr.EDGE_INSERT, sr.EDGE_INSERT, sr.BATCH_CLOSE]
    bid = b'"00000000-0000-4000-8000-000000000000"'
    assert calls[0][2] == b'[' + bid + b',"crawl-1","owner","pid",2,"seq","open"]'
    assert calls[1][2] == b'[' + bid + b',"crawl-1","chan01","owner","seq","2025-10-09T08:53:20.12Z","text_url","pending"]'
    assert calls[2][2].endswith(b'"plaintext","pending"]')  # a duplicate edge is still written "pending"
    assert calls[3][2] == b"[" + bid + b"]"


@pytest.mark.parametrize("raw, want", [
    (b'<a href="x">&amp;\\', rb'"\u003ca href=\"x\"\u003e\u0026amp;\\"'),
    ("\u2028 \u2029 \u00e9".encode(), b'"\\u2028 \\u2029 \xc3\xa9"'),
    (b"\xff bad \xc3\x28 \xe2\x82", rb'"\ufffd bad \ufffd( \ufffd\ufffd"'),
    (b"tab\tnl\n\x01\x7f", rb'"tab\tnl\n\u0001' + b'\x7f"'),
    (b"", b'""'),
])
def test_strings_take_encoding_json_html_safe_escaping(raw, want):
    for values in (sr.batch_values(batch(source_channel=raw, source_page_id=raw, sequence_id=raw), raw),
                   sr.edge_values(batch(source_channel=raw, sequence_id=raw), edge(), raw, sr.discovery_time(NOW, 0))):
        got = sr.split_values(sr.marshal(values))
        assert got[1] == want  # crawl_id
        assert got[2 if len(values) == 7 else 3] == want  # owner.URL
        assert got[5 if len(values) == 7 else 4] == want  # owner.SequenceID
    assert sr.split_values(sr.marshal(sr.batch_values(batch(source_page_id=raw), b"c")))[3] == want  # owner.ID


@pytest.mark.parametrize("sec, nsec, zone, tz, want", [
    (NOW, 0, None, 0, b'"2025-10-09T08:53:20Z"'),                       # zero nanoseconds: no fraction
    (NOW, 500_000_000, None, 0, b'"2025-10-09T08:53:20.5Z"'),          # trailing zeros trimmed
    (NOW, 1, None, 0, b'"2025-10-09T08:53:20.000000001Z"'),
    (NOW, 123_456_780, None, 3600, b'"2025-10-09T09:53:20.12345678+01:00"'),
    (NOW, 0, None, 5 * 3600 + 30 * 60 + 15, b'"2025-10-09T14:23:35+05:30"'),  # an offset with seconds: minutes shown
    (NOW, 0, ([0], [-30]), 0, b'"2025-10-09T08:52:50+00:00"'),       # Go's minutes-first sign in a zone
    (NOW, 0, ([0], [-(3 * 3600 + 45)]), 0, b'"2025-10-09T05:52:35-03:00"'),
    (1710054000 - 1, 0, NY, 0, b'"2024-03-10T01:59:59-05:00"'),        # New York springs forward
    (1710054000, 0, NY, 0, b'"2024-03-10T03:00:00-04:00"'),
    (1730613600 - 1, 0, NY, 0, b'"2024-11-03T01:59:59-04:00"'),        # and falls back
    (1730613600, 0, NY, 0, b'"2024-11-03T01:00:00-05:00"'),
    (253402300799, 999_999_999, None, 0, b'"9999-12-31T23:59:59.999999999Z"'),
    (253402300800, 0, None, 0, None),                                   # year 10000: json.Marshal fails
    (253402300799, 0, None, 1, None),                                   # ... in the local zone
    (-62167219200, 0, None, 0, b'"0000-01-01T00:00:00Z"'),
    (-62167219201, 0, None, 0, None),                                   # year -1
    (-62167219200, 0, None, -1, None),
])
def test_discovery_time_is_json_marshal_in_time_local(sec, nsec, zone, tz, want):
    got = sr.discovery_time(sec, nsec, zone, tz)
    assert (None if got is None else bytes(got)) == want
    if want is not None:
        assert sr.split_values(sr.marshal(sr.edge_values(batch(), edge(), b"c", got)))[5] == want


@pytest.mark.parametrize("depth", [0, -1, 7, -(1 << 63), (1 << 63) - 1])
def test_depth_is_a_decimal_int64(depth):
    assert sr.split_values(sr.marshal(sr.batch_values(batch(source_depth=depth), b"c")))[4] == b"%d" % depth


def random_pages(rnd, n_pages):
    pool = [b"chan%03d" % k for k in range(40)] + [b"x<y", "café".encode(), b"\xff"]
    pages = []
    for p in range(n_pages):
        b = batch(p, source_channel=rnd.choice(pool), source_page_id=b"p%d" % p, source_depth=rnd.randrange(-2, 5),
                  sequence_id=rnd.choice([b"", b"seq-\x80", b"seq"]))
        pages.append((b, [edge(rnd.choice(pool), rnd.randrange(4), rnd.randrange(2)) for _ in range(rnd.randrange(1, 9))]))
    return pages


@pytest.mark.parametrize("seed", range(4))
def test_bulk_statements_split_into_the_one_row_calls(seed):
    rnd = random.Random(seed)
    pages = random_pages(rnd, rnd.randrange(1, 12))
    t = sr.discovery_time(NOW, rnd.randrange(10**9), NY)
    ref = sr.reference_calls(pages, b"crawl<&>", t)
    one = sr.statements(pages, b"crawl<&>", t, 1)
    # k = 1: the reference's calls, grouped by kind in their order
    assert [(k, s, p) for k, _, s, p in one] == sorted(ref, key=lambda c: c[0])
    for k in (2, 3, 7, 8, 20, sr.MAX_ROWS):
        got = sr.statements(pages, b"crawl<&>", t, k)
        assert [x[0] for x in got] == sorted(x[0] for x in got)
        rows = []
        for kind, n, sql, params in got:
            assert 1 <= n <= k and sql == sr.sql_text(kind, n)
            v = sr.split_values(params)
            w = sr.PER_ROW[kind]
            assert len(v) == n * w
            rows += [(kind, b"[" + b",".join(v[a:a + w]) + b"]") for a in range(0, len(v), w)]
        assert rows == [(k1, p) for k1, _, _, p in one]
        for kind in (0, 1, 2):  # every statement of a kind is full but its last
            ns = [n for kk, n, _, _ in got if kk == kind]
            assert all(n == k for n in ns[:-1])


def test_output_layout_matches_the_header():
    src = r"""
#include <stddef.h>
#include <stdio.h>
#include "tgingest.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu\n", sizeof(tgi_state_edge_stmt), offsetof(tgi_state_edge_stmt, rows),
         offsetof(tgi_state_edge_stmt, sql_off), offsetof(tgi_state_edge_stmt, params_len), sizeof(tgi_state_edge_sql_t),
         offsetof(tgi_state_edge_sql_t, kernel_ms), offsetof(tgi_state_edge_sql_t, gpu_launches));
  printf("%d %d %d %u\n", TGI_SQL_BATCH_INSERT, TGI_SQL_EDGE_INSERT, TGI_SQL_BATCH_CLOSE, TGI_SQL_MAX_ROWS);
  return 0;
}
"""
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "t.c"), os.path.join(d, "t")
        with open(c, "w") as f:
            f.write(src)
        subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        lines = subprocess.check_output([exe], text=True).split("\n")
    s = abi.STATE_EDGE_STMT
    assert [int(x) for x in lines[0].split()] == [
        s.itemsize, s.fields["rows"][1], s.fields["sql_off"][1], s.fields["params_len"][1], C.sizeof(abi.StateEdgeSqlC),
        abi.StateEdgeSqlC.kernel_ms.offset, abi.StateEdgeSqlC.gpu_launches.offset]
    assert [int(x) for x in lines[1].split()] == [abi.SQL_BATCH_INSERT, abi.SQL_EDGE_INSERT, abi.SQL_BATCH_CLOSE,
                                                  abi.SQL_MAX_ROWS] == [sr.BATCH_INSERT, sr.EDGE_INSERT, sr.BATCH_CLOSE,
                                                                        sr.MAX_ROWS]
    assert np.dtype(s).itemsize == 40
