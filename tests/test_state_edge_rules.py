"""CPU tests: the state edge corpus reaches every cell it is meant to, and the restatement the GPU edge tests compare
with is pinned by hand-written strings at the time bounds, the offset signs and the layer map's key order."""
import pytest

import state_edge_corpus as ec
import walkback_rules as wr
from dapr_state_rules import marshal_layer_map
from state_rules import MarshalError, marshal_message, marshal_time


def test_the_corpus_reaches_every_cell():
    got, want = ec.state_cells(ec.edge_state()), ec.expected_cells()
    assert sorted(want - got, key=repr) == [] and sorted(got - want, key=repr) == []


def test_the_cells_come_from_what_the_writers_see():
    """a message list or a layer dropped from the state loses its cells: the check reads the state, not the loops"""
    layers = ec.edge_state()
    full = ec.state_cells(layers)
    no_msgs = [(d, [dict(p, messages=[]) for p in ps]) for d, ps in layers]
    cut = ec.state_cells(no_msgs)
    assert not any(c[0] in ("message.pageId", "code") for c in cut) and cut < full
    assert not any(c[0] == "layer_map" for c in ec.state_cells([(d, ps) for d, ps in layers if d != 9]))


def test_edge_strings_have_their_length_and_feature():
    for kind in ec.STR_KINDS:
        for n in ec.STR_LENGTHS:
            assert len(ec.edge_str(kind, n)) == n, (kind, n)
    assert ec.edge_str("u2028@127", 300)[127:130] == b"\xe2\x80\xa8"  # split across byte 128
    assert ec.edge_str("u2028@127", 300)[255:258] == b"\xe2\x80\xa8"
    assert ec.edge_str("rune4@126", 256)[126:130] == "😀".encode()
    assert ec.edge_str("invalid@128", 129)[128] == 0xFF
    assert ec.edge_str("surrogate_end", 4097).endswith(b"\xed\xa0\x80")
    for s, feat, n in ec.short_strs():
        assert len(s) == n and (n < len(ec.SHORT_FEATURES[feat]) or ec.SHORT_FEATURES[feat] in s)


@pytest.mark.parametrize("ts,want", [
    ((ec.YEAR0, 0, 0), b'"0000-01-01T00:00:00Z"'),
    ((ec.YEAR9999_END, 999_999_999, 0), b'"9999-12-31T23:59:59.999999999Z"'),
    ((ec.YEAR0 - 3600, 0, 3600), b'"0000-01-01T00:00:00+01:00"'),
    ((ec.YEAR9999_END + 18000, 0, -18000), b'"9999-12-31T23:59:59-05:00"'),
    ((1700000000, 0, -59), b'"2023-11-14T22:12:21+00:00"'),  # Go's minutes-first sign: -59 s is +00:00
    ((1700000000, 0, -1), b'"2023-11-14T22:13:19+00:00"'),
    ((1700000000, 0, 59), b'"2023-11-14T22:14:19+00:00"'),
    ((1700000000, 0, -60), b'"2023-11-14T22:12:20-00:01"'),
    ((1700000000, 0, 19830), b'"2023-11-15T03:43:50+05:30"'),  # an offset with seconds: minutes truncated
    ((1700000000, 0, -19830), b'"2023-11-14T16:42:50-05:30"'),
    ((1700000000, 0, 86399), b'"2023-11-15T22:13:19+23:59"'),
    ((1700000000, 0, -86399), b'"2023-11-13T22:13:21-23:59"'),
    ((1700000000, 1, 0), b'"2023-11-14T22:13:20.000000001Z"'),
    ((1700000000, 10, 0), b'"2023-11-14T22:13:20.00000001Z"'),
    ((1700000000, 100_000_000, 0), b'"2023-11-14T22:13:20.1Z"'),
    ((1700000000, 999_999_999, 0), b'"2023-11-14T22:13:20.999999999Z"'),
])
def test_times_at_the_bounds_and_offset_signs(ts, want):
    assert marshal_time(ts) == want


@pytest.mark.parametrize("ts", ec.TIME_REFUSED)
def test_times_past_the_bounds_are_refused(ts):
    with pytest.raises(MarshalError):
        marshal_time(ts)


def test_every_corpus_time_renders():
    for ts in ec.TIME_EDGES:
        assert marshal_time(ts, None, 0)


def test_layer_map_keys_sort_as_strings():
    lm = {-1: [b"a"], ec.I64_MIN: [], 10: [b"<"], 9: [b"b", b"\xff"], ec.I64_MAX: [b"z"], 0: []}
    assert marshal_layer_map(lm) == (b'{"-1":["a"],"-9223372036854775808":[],"0":[],"10":["\\u003c"],'
                                     b'"9":["b","\\ufffd"],"9223372036854775807":["z"]}')


def test_int64_ends_in_messages_and_the_walkback_depth():
    m = {"chatId": ec.I64_MIN, "messageId": ec.I64_MAX, "status": b"a\xe2\x80\xa8", "pageId": b"<"}
    assert marshal_message(m) == (b'{"chatId":-9223372036854775808,"messageId":9223372036854775807,'
                                  b'"status":"a\\u2028","pageId":"\\u003c"}')
    assert wr.go_int(ec.I64_MAX + 1) == ec.I64_MIN  # owner.Depth + 1 wraps as Go's int
    assert wr.go_int(ec.I64_MIN - 1 + 1) == ec.I64_MIN
