"""CPU tests: the restatement of BaseStateManager and json.Marshal(State) in tests/state_rules.py, pinned by hand-written
known answers, and the batched UpdateMessage of state_join against the sequential calls."""
import json
import random

import numpy as np

from distributed_crawler_b200 import abi
from distributed_crawler_b200.state_join import update_messages_batch
from distributed_crawler_b200.state_pack import pack_pages
from oracle.pyoracle import Oracle
from state_rules import GoState, MarshalError, marshal_page

FULL = {"id": b"p1", "url": b"https://t.me/a", "depth": 1, "status": b"fetched", "error": b"e", "timestamp": (0, 0, 0),
        "platform": b"telegram", "parentId": b"p0", "LastConnectionID": b"c", "sequenceId": b"s", "crawlId": b"k",
        "messages": [{"chatId": -5, "messageId": -7, "status": b"fetched", "pageId": b"p1", "platform": b"tg"},
                     {"chatId": 3, "messageId": 4, "status": b"unfetched", "pageId": b"p1"}]}


def test_page_with_every_omitempty_field():
    assert marshal_page(FULL) == (
        b'{"id":"p1","url":"https://t.me/a","depth":1,"status":"fetched","error":"e","timestamp":"1970-01-01T00:00:00Z",'
        b'"platform":"telegram","parentId":"p0","messages":[{"chatId":-5,"messageId":-7,"status":"fetched","pageId":"p1",'
        b'"platform":"tg"},{"chatId":3,"messageId":4,"status":"unfetched","pageId":"p1"}],"LastConnectionID":"c",'
        b'"sequenceId":"s","crawlId":"k"}')


def test_page_without_omitempty_fields_and_the_zero_time():
    assert marshal_page({"id": b"x"}) == b'{"id":"x","url":"","depth":0,"status":"","timestamp":"0001-01-01T00:00:00Z"}'
    assert marshal_page({"id": b"x", "messages": []}) == marshal_page({"id": b"x"})  # empty messages are omitted


def test_timestamps_fixed_local_and_out_of_range():
    p = {"id": b"t", "timestamp": (1700000000, 5000, 3600)}
    assert b'"timestamp":"2023-11-14T23:13:20.000005+01:00"' in marshal_page(p)
    p["timestamp"] = (1700000000, 0, -30)  # Go takes the sign of the truncated minutes
    assert b'"timestamp":"2023-11-14T22:12:50+00:00"' in marshal_page(p)
    p["timestamp"] = (1700000000, 0, None)
    assert b'"timestamp":"2023-11-14T17:13:20-05:00"' in marshal_page(p, tz=-5 * 3600)
    ny = ([-(1 << 31), 1699164000], [-4 * 3600, -5 * 3600])  # EDT, then EST from 2023-11-05 06:00 UTC
    assert b'"2023-11-05T01:59:59-04:00"' in marshal_page({"id": b"t", "timestamp": (1699163999, 0, None)}, ny)
    assert b'"2023-11-05T01:00:00-05:00"' in marshal_page({"id": b"t", "timestamp": (1699164000, 0, None)}, ny)
    try:
        marshal_page({"id": b"t", "timestamp": (253402300800, 0, 0)})  # year 10000
        assert False
    except MarshalError:
        pass


def test_escaping_and_negative_ids():
    p = {"id": b"i", "url": b"<a>&\xe2\x80\xa8\xff\"", "messages": [{"chatId": -1001, "messageId": -(1 << 62), "status": b"x",
                                                                    "pageId": b"i"}]}
    out = marshal_page(p)
    assert b'"url":"\\u003ca\\u003e\\u0026\\u2028\\ufffd\\""' in out
    assert b'{"chatId":-1001,"messageId":-4611686018427387904,"status":"x","pageId":"i"}' in out


def test_empty_state_and_empty_layers():
    s = GoState()
    assert s.marshal(b"{}", b'"t"') == b'{"layers":[],"metadata":{},"lastUpdated":"t"}'
    s.set_state([(3, []), (1, [{"id": b"a", "url": b"u"}])])
    s.add_layer([{"id": b"b", "url": b"u", "depth": 2}])  # a duplicate URL: the layer is created empty
    out = s.marshal(b"{}", b'"t"')
    assert out.startswith(b'{"layers":[{"depth":1,"pages":[{"id":"a","url":"u",')
    assert out.endswith(b'{"depth":2,"pages":[]},{"depth":3,"pages":[]}],"metadata":{},"lastUpdated":"t"}')
    s.add_layer([])  # nothing: no layer either
    assert s.marshal(b"{}", b'"t"') == out
    json.loads(out)


def test_update_page_layer_quirk():
    s = GoState()
    s.set_state([(0, [{"id": b"a", "url": b"u"}])])
    s.update_page({"id": b"b", "url": b"v", "depth": 1})  # no layer 1: only in pageMap
    assert [p["id"] for p in json.loads(s.marshal(b"{}", b'"t"'))["layers"][0]["pages"]] == ["a"]
    assert s.get_page(b"b") is not None
    s.update_page({"id": b"b", "url": b"v", "depth": 0})  # layer 0 exists: appended once
    s.update_page({"id": b"b", "url": b"w", "depth": 0})
    assert [p["id"] for p in json.loads(s.marshal(b"{}", b'"t"'))["layers"][0]["pages"]] == ["a", "b"]
    assert not s.update_message(b"zz", 1, 2, b"fetched")  # unknown page: the reference's error


def test_max_pages_with_deadend_replacements():
    s = GoState(max_pages=3)
    s.set_state([(0, [{"id": b"a", "url": b"1", "status": b"deadend"}, {"id": b"b", "url": b"2", "status": b"deadend"},
                      {"id": b"c", "url": b"3"}])])
    added = s.add_layer([{"id": b"d", "url": b"1", "depth": 1}, {"id": b"e", "url": b"4", "depth": 1},
                         {"id": b"f", "url": b"4", "depth": 1}, {"id": b"g", "url": b"5", "depth": 1},
                         {"id": b"h", "url": b"6", "depth": 1}])
    assert added == [False, True, False, True, False]  # two replacements for two deadends, duplicates skipped first
    s2 = GoState(max_pages=10)
    s2.set_state([(0, [{"id": b"a", "url": b"1"}])])
    assert s2.add_layer([{"id": b"x%d" % i, "url": b"u%d" % i, "depth": 1} for i in range(12)]) == [True] * 12


def test_update_messages_batch_equals_sequential_update_message():
    rnd = random.Random(5)
    for trial in range(40):
        page = [(rnd.randrange(3), rnd.randrange(10)) for _ in range(rnd.randrange(0, 20))]
        status = [rnd.choice([b"unfetched", b"fetched"]) for _ in page]
        ups = [((rnd.randrange(3), rnd.randrange(14)), rnd.choice([b"fetched", b"failed", b"deleted"])) for _ in range(rnd.randrange(0, 30))]
        s = GoState()
        s.set_state([(0, [{"id": b"p", "messages": [{"chatId": c, "messageId": m, "status": st, "pageId": b"p"}
                                                     for (c, m), st in zip(page, status)]}])])
        for (c, m), st in ups:
            assert s.update_message(b"p", c, m, st)
        keys, got = update_messages_batch(Oracle.key_join, np.array(page, np.int64).reshape(-1, 2), status,
                                          np.array([k for k, _ in ups], np.int64).reshape(-1, 2), [st for _, st in ups])
        want = s.get_page(b"p")["messages"]
        assert [(int(a), int(b)) for a, b in keys] == [(m["chatId"], m["messageId"]) for m in want], trial
        assert got == [m["status"] for m in want], trial


def test_packer_layout():
    codes = {c.encode(): i for i, c in enumerate(abi.STATE_CODES)}
    recs, strs, msgs = pack_pages([FULL], lambda s: codes.setdefault(s, len(codes)), lambda pid, i: i)
    assert recs.itemsize == 72 and msgs.itemsize == 24
    assert bytes(strs[:recs[0]["str_len"].sum()]) == b"p1https://t.me/afetchedetelegramp0csk"
    assert list(msgs["status"]) == [codes[b"fetched"], codes[b"unfetched"]] and list(msgs["platform"]) == [6, 0]
    assert recs[0]["n_msgs"] == 2 and recs[0]["ts_off"] == 0
