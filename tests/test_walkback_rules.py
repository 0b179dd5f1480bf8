"""CPU tests of tests/walkback_rules.py: the two literals and their multi-row forms, escaping in every string, Go's int
wrap of the depth, pickWalkbackChannel's skip, exhaustion and empty set, and the library's draw rule, Lemire's
multiply-and-reject, against exact enumeration and a chi-squared test."""
import itertools

import pytest
from scipy.stats import chisquare

import walkback_rules as wr
from discover_rules import page_id
from go_rules import _Raw
from tandem_sql_rules import discovery_time

T = discovery_time(1_760_000_000, 120_000_000)
OWNER = {"id": b"owner-1", "url": b"chan001", "depth": 2, "sequenceId": b"seq-1"}
PID, SID = b"p" * 36, b"s" * 36


def test_literals_at_one_row_and_their_multi_row_forms():
    assert wr.sql_text(wr.PAGE_BUFFER_INSERT, 1) == (
        b"INSERT INTO page_buffer (page_id, parent_id, depth, url, crawl_id, sequence_id) VALUES ($1, $2, $3, $4, $5, $6);")
    assert wr.sql_text(wr.EDGE_RECORD_INSERT, 1) == (
        b"INSERT INTO edge_records (destination_channel, source_channel, walkback, skipped, discovery_time, crawl_id, "
        b"sequence_id) VALUES ($1, $2, $3, $4, $5, $6, $7);")
    assert wr.sql_text(wr.PAGE_BUFFER_INSERT, 2) == (
        b"INSERT INTO page_buffer (page_id, parent_id, depth, url, crawl_id, sequence_id) VALUES "
        b"($1, $2, $3, $4, $5, $6), ($7, $8, $9, $10, $11, $12);")
    assert wr.sql_text(wr.EDGE_RECORD_INSERT, 3).endswith(
        b"VALUES ($1, $2, $3, $4, $5, $6, $7), ($8, $9, $10, $11, $12, $13, $14), ($15, $16, $17, $18, $19, $20, $21);")
    big = wr.sql_text(wr.EDGE_RECORD_INSERT, wr.MAX_ROWS)
    assert big.count(b"(") == wr.MAX_ROWS + 1 and big.endswith(b"$57337);")  # 7 x 8191 parameters, under 65535


def test_one_row_params_are_the_references_marshal():
    res, calls = wr.forced_walkback(OWNER, [b"chan001", b"chan002"], 5, 0, b"crawl-1", T)
    assert res["status"] == wr.WALK_OK and res["page_id"] == wr.uuid(5, 0, 3) and res["sequence_id"] == wr.uuid(5, 0, 4)
    url = res["url"]
    assert url == b"chan002"  # the owner's URL is skipped
    assert calls == [
        (wr.PAGE_BUFFER_INSERT, wr.PAGE_BUFFER_SQL,
         b'["%s","owner-1",3,"chan002","crawl-1","%s"]' % (res["page_id"], res["sequence_id"])),
        (wr.EDGE_RECORD_INSERT, wr.EDGE_RECORD_SQL,
         b'["chan002","chan001",true,false,%s,"crawl-1","seq-1"]' % bytes(T))]
    # the grouped form at k = 1 is the reference's calls, grouped by kind
    assert [(k, s, p) for k, _, s, p in wr.statements([(OWNER, res)], b"crawl-1", T, 1)] == calls


def test_multi_row_params_are_the_rows_values_as_one_array():
    owners = [dict(OWNER, id=b"o%d" % i, url=b"u%d" % i) for i in range(5)]
    walks = [(o, wr.forced_walkback(o, [b"k0", b"k1", b"k2"], 9, w, b"c", T)[0]) for w, o in enumerate(owners)]
    walks[2][1]["status"] = wr.WALK_EXHAUSTED  # a span without a row
    one = wr.statements(walks, b"c", T, 1)
    for k in (2, 3, 4, 8191):
        got = wr.statements(walks, b"c", T, k)
        assert [s[1] for s in got] == [min(k, 4 - a) for a in range(0, 4, k)] * 2
        for kind in (wr.PAGE_BUFFER_INSERT, wr.EDGE_RECORD_INSERT):
            rows = [p[1:-1] for kk, _, _, p in one if kk == kind]
            assert b"".join(b"[" + b",".join(rows[a:a + k]) + b"]" for a in range(0, 4, k)) == \
                b"".join(p for kk, _, _, p in got if kk == kind)
    assert [s[0] for s in one] == [wr.PAGE_BUFFER_INSERT] * 4 + [wr.EDGE_RECORD_INSERT] * 4


def test_escaping_in_the_owner_url_id_and_sequence_id_and_the_picked_url():
    owner = {"id": b"<id>&\xff", "url": b"a\"b\\c\xe2\x80\xa8", "depth": 0, "sequenceId": b"s\x01q\xe2\x80\xa9"}
    res, calls = wr.forced_walkback(owner, [b"x<y>"], 1, 3, b"c&\"", _Raw(b'"t"'))
    assert res["status"] == wr.WALK_OK and res["draws"] == 1
    assert calls[0][2] == b'["%s","\\u003cid\\u003e\\u0026\\ufffd",1,"x\\u003cy\\u003e","c\\u0026\\"","%s"]' % (
        res["page_id"], res["sequence_id"])
    assert calls[1][2] == (b'["x\\u003cy\\u003e","a\\"b\\\\c\\u2028",true,false,"t","c\\u0026\\"",'
                           b'"s\\u0001q\\u2029"]')


@pytest.mark.parametrize("depth, want", [(0, 1), (-1, 0), (2 ** 63 - 2, 2 ** 63 - 1), (2 ** 63 - 1, -2 ** 63),
                                         (-2 ** 63, -2 ** 63 + 1)])
def test_the_depth_wraps_as_go_int(depth, want):
    res, calls = wr.forced_walkback(dict(OWNER, depth=depth), [b"k"], 1, 0, b"c", T)
    assert calls[0][2].split(b",")[2] == str(want).encode()


def test_a_one_key_set_of_the_owner_url_is_exhausted_after_ten_draws():
    n = itertools.count()
    draw = lambda: (next(n), b"chan001")[1]  # noqa: E731
    assert wr.pick_walkback_channel([b"chan001"], b"chan001", draw) == (wr.WALK_EXHAUSTED, b"", 10)
    assert next(n) == 10
    res, calls = wr.forced_walkback(OWNER, [b"chan001"], 7, 11, b"c", T)
    assert (res["status"], res["draws"], res["url"], calls) == (wr.WALK_EXHAUSTED, 10, b"", [])


def test_an_empty_set_is_an_error_before_any_draw():
    res, calls = wr.forced_walkback(OWNER, [], 7, 0, b"c", T)
    assert (res["status"], res["draws"], calls) == (wr.WALK_EMPTY, 0, [])


def test_the_owner_comparison_is_case_sensitive_and_byte_for_byte():
    for key in (b"Chan001", b"chan001 ", b"chan0010", b"chan00"):
        res, _ = wr.forced_walkback(OWNER, [key], 3, 0, b"c", T)
        assert (res["status"], res["url"], res["draws"]) == (wr.WALK_OK, key, 1)


def test_skips_take_further_draws_from_the_same_stream():
    keys = [b"chan001", b"other"]
    for w in range(200):
        res, _ = wr.forced_walkback(OWNER, keys, 11, w, b"c", T)
        stream = wr.words(11, w)
        idx = [wr.lemire(2, stream) for _ in range(10)]
        first = next((j for j, i in enumerate(idx) if i == 1), None)
        if first is None:
            assert (res["status"], res["draws"]) == (wr.WALK_EXHAUSTED, 10)
        else:
            assert (res["status"], res["draws"], res["url"]) == (wr.WALK_OK, first + 1, b"other")


def test_ids_are_page_ids_of_their_own_counter_words():
    assert wr.uuid(42, 7, 0) == page_id(42, 7)
    ids = {wr.uuid(42, 7, d) for d in range(5)}
    assert len(ids) == 5 and all(i[14:15] == b"4" and i[19:20] in b"89ab" for i in ids)


def test_the_word_stream_is_philox_blocks_two_words_each():
    from discover_rules import philox4x32_10
    s = wr.words(0x1234_5678_9ABC_DEF0, (5 << 32) | 9)
    got = [next(s) for _ in range(6)]
    for j in range(3):
        x = philox4x32_10([9, 5, 2, j], [0x9ABC_DEF0, 0x1234_5678])
        assert got[2 * j:2 * j + 2] == [x[0] | x[1] << 32, x[2] | x[3] << 32]


@pytest.mark.parametrize("bits", [6, 8, 10])
def test_lemire_is_exactly_uniform_by_enumeration(bits):
    """every word of a narrow width: the accepted ones split evenly over [0, n), the rejected ones take the next word"""
    for n in range(1, 2 ** (bits - 2)):
        hist = [0] * n
        rejected = 0
        for x in range(2 ** bits):
            sentinel = object()
            stream = iter([x, sentinel])
            try:
                hist[wr.lemire(n, stream, bits)] += 1
            except TypeError:  # the sentinel was taken: x was rejected
                rejected += 1
        assert rejected == 2 ** bits % n, (bits, n)
        assert len(set(hist)) == 1, (bits, n, hist)


def _reject_bound_words(n):
    """the 64-bit words whose low64(x * n) is t - 1 (rejected) and t (accepted), t = 2^64 mod n, for odd n"""
    t = (1 << 64) % n
    inv = pow(n, -1, 1 << 64)
    return (t - 1) * inv % (1 << 64), t * inv % (1 << 64)


@pytest.mark.parametrize("n", [3, 5, 7, 1001, 2 ** 33 + 1, 2 ** 63 + 1, 2 ** 64 - 1])
def test_lemire_at_the_rejection_bound(n):
    bad, good = _reject_bound_words(n)
    assert bad * n % (1 << 64) == ((1 << 64) % n) - 1 and good * n % (1 << 64) == (1 << 64) % n
    assert wr.lemire(n, iter([bad, good])) == good * n >> 64  # the rejected word is passed over
    assert wr.lemire(n, iter([good, bad])) == good * n >> 64
    # a word whose low part is at least n never reads the bound
    x = (n + 5) * pow(n, -1, 1 << 64) % (1 << 64)
    assert wr.lemire(n, iter([x])) == x * n >> 64


def test_lemire_powers_of_two_never_reject():
    for b in (0, 1, 5, 63):
        n = 1 << b
        for x in (0, 1, (1 << 64) - 1, 0x8000_0000_0000_0000):
            assert wr.lemire(n, iter([x])) == x >> (64 - b)


@pytest.mark.parametrize("n", [2, 7, 10, 37])
def test_the_draws_are_uniform_over_many_seeds(n):
    counts = [0] * n
    for seed in range(40):
        for w in range(250):
            counts[wr.lemire(n, wr.words(seed * 0x9E3779B97F4A7C15 & wr.U64, w))] += 1
    assert chisquare(counts).pvalue > 1e-4, counts


def test_picks_are_uniform_over_the_other_keys():
    keys = [b"k%d" % i for i in range(6)]
    owner = dict(OWNER, url=b"k2")
    counts = {}
    for w in range(6000):
        res, _ = wr.forced_walkback(owner, keys, 99, w, b"c", T)
        counts[res["url"]] = counts.get(res["url"], 0) + 1
    assert b"k2" not in counts and len(counts) == 5
    assert chisquare(list(counts.values())).pvalue > 1e-4, counts
