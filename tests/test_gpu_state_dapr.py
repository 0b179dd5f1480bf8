"""GPU tests: the resident crawl state's Dapr side (tgi_state_layer_map, tgi_state_add_pages, tgi_state_export) against
the restatement in tests/dapr_state_rules.py — the layer map byte for byte, every export chunk raw and in base64, and
the local export, after every step of seeded random operation sequences; the empty state; rejected calls; a 10 k page
x 100 message export."""
import base64

import numpy as np
import pytest

from dapr_state_rules import NoPagesFound, dapr_add_layer, export_dapr, export_dapr_chunks, export_local, marshal_layer_map
from distributed_crawler_b200 import abi, sink
from distributed_crawler_b200.engine import Engine, EngineError
from test_gpu_state import LAST, META, Sequence, big_state

DEFAULT = abi.STATE_EXPORT_CHUNK_DEFAULT
DEPTHS = [-12, -1, 0, 1, 2, 10, 100]


class DaprSequence(Sequence):
    """Sequence's operations plus Dapr's AddLayer (with its urlCache) at negative and multi-digit depths; every check
    also compares the layer map and both exports"""

    def __init__(self, seed):
        super().__init__(seed)
        self.cache = {}  # urlCache: URL -> id, across calls

    def step(self):
        r = self.rnd
        if r.random() >= 0.3:
            return super().step()
        ps = [self.page(r.choice(DEPTHS), False, self.ids()) for _ in range(r.randrange(0, 8))]
        if len(ps) > 2 and r.random() < 0.5:
            ps[-1]["url"] = ps[0]["url"]  # a duplicate URL within the call is kept
        if ps and r.random() < 0.3:
            self.cache[ps[0].get("url")] = b"earlier-crawl"  # pages[0] filtered away, its depth still used
        depth, added = dapr_add_layer(self.go, self.cache, ps, random_walk=r.random() < 0.1)
        rows = self.e.state_add_pages(depth, added)
        assert rows == [self.e._st_rows()[p["id"]] for p in added]
        self.check()

    def check(self):
        super().check()
        check_dapr(self.e, self.go, self.zone, self.rnd)


def check_dapr(e, go, zone, rnd):
    assert e.state_layer_map() == marshal_layer_map(go.layer_map)
    want_local = export_local(go, zone)
    assert e.state_export(abi.STATE_EXPORT_LOCAL, 0) == [(want_local, len(want_local))]
    try:
        whole = export_dapr_chunks(go, 1 << 62, zone)[0]
    except NoPagesFound:
        with pytest.raises(EngineError) as ei:
            e.state_export(abi.STATE_EXPORT_DAPR, DEFAULT)
        assert ei.value.code == abi.E_NOPAGES
        return
    ends = np.cumsum([len(ln) for ln in whole.splitlines(keepends=True)])
    sizes = {0, 1, DEFAULT}
    for end in rnd.sample(list(ends), min(2, len(ends))):  # around cumulative line ends
        sizes |= {int(end) - 1, int(end), int(end) + 1}
    for cb in sorted(sizes):
        want = export_dapr_chunks(go, cb, zone)
        got = e.state_export(abi.STATE_EXPORT_DAPR, cb)
        assert [base64.b64decode(d) for d, _ in got] == want, cb
        assert [d for d, _ in got] == [base64.b64encode(w) for w in want], cb
        assert [n for _, n in got] == [len(w) for w in want]


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(6))
def test_random_sequences_match_the_restatement(seed):
    sq = DaprSequence(100 + seed)
    for _ in range(80):
        sq.step()
    sq.e.close()


@pytest.mark.gpu
def test_tombstones_compaction_and_reused_ids():
    sq = DaprSequence(5)
    sq.go.set_state([(0, [{"id": b"a", "url": b"u"}])])
    sq.e.state_set([(0, [{"id": b"a", "url": b"u"}])])
    for k in range(12):  # UpdatePage leaves tombstones; re-adding the id drops its messages again
        p = {"id": b"a", "url": b"u", "depth": 0, "messages": [{"chatId": 1, "messageId": j, "status": b"fetched",
                                                               "pageId": b"a"} for j in range(150 + k)]}
        sq.go.update_page(p)
        sq.e.state_update_page(p)
        q = {"id": b"a", "url": b"u%d" % k, "depth": -k}
        depth, added = dapr_add_layer(sq.go, sq.cache, [q])
        sq.e.state_add_pages(depth, added)
        sq.check()
    sq.e.close()


@pytest.mark.gpu
def test_the_empty_state_in_both_modes():
    e = Engine()
    assert e.state_layer_map() == b"{}"
    with pytest.raises(EngineError) as ei:
        e.state_export(abi.STATE_EXPORT_DAPR, DEFAULT)
    assert ei.value.code == abi.E_NOPAGES
    assert e.state_export(abi.STATE_EXPORT_LOCAL, DEFAULT) == [(b"", 0)]
    assert e.state_add_pages(3, []) == [] and e.state_layer_map() == b"{}"  # n == 0 creates no layer
    e.state_set([(0, []), (-5, [])])  # layers without pages
    assert e.state_layer_map() == b'{"-5":[],"0":[]}'
    with pytest.raises(EngineError) as ei:
        e.state_export(abi.STATE_EXPORT_DAPR, 0)
    assert ei.value.code == abi.E_NOPAGES
    e.close()


@pytest.mark.gpu
def test_rejected_calls_leave_the_state_unchanged():
    sq = DaprSequence(11)
    for _ in range(20):
        sq.step()
    e = sq.e
    depth, added = dapr_add_layer(sq.go, sq.cache, [{"id": b"seed", "url": b"seed-url", "depth": 0}])  # a page to export
    e.state_add_pages(depth, added)

    def snapshot():
        return (e.state_render(META, LAST), e.state_layer_map(), e.state_export(abi.STATE_EXPORT_LOCAL, 0),
                e.state_export(abi.STATE_EXPORT_DAPR, 1000))
    before = snapshot()
    for call in [lambda: e.state_add_pages(0, [{"id": b"x", "url": b"new", "timestamp": (0, 10**9, 0)}]),
                 lambda: e.state_add_pages(0, [{"id": b"x", "url": b"new", "timestamp": (0, 0, -86400)}]),
                 lambda: e.state_add_pages(0, [{"id": b"x", "url": b"new", "messages": [{"chatId": 1, "messageId": 1,
                                                                                          "pageId": b"x"}]}]),
                 lambda: e.state_export(2, 0)]:
        with pytest.raises(EngineError) as ei:
            call()
        assert ei.value.code == abi.E_ARG
        assert snapshot() == before
    # a timestamp json.Marshal cannot render: both exports fail and change nothing; the state exports again once fixed
    p = {"id": b"y10k", "url": b"y10k", "depth": 0, "timestamp": (253402300800, 0, 0)}
    e.state_update_page(p)
    lm = e.state_layer_map()
    for mode in (abi.STATE_EXPORT_DAPR, abi.STATE_EXPORT_LOCAL):
        with pytest.raises(EngineError) as ei:
            e.state_export(mode, 0)
        assert ei.value.code == abi.E_ARG
        assert e.state_layer_map() == lm
    p["timestamp"] = (253402300799, 0, 0)
    e.state_update_page(p)
    sq.go.update_page(p)
    sq.check()
    e.close()


@pytest.mark.gpu
def test_export_pages_dapr_paths():
    sq = DaprSequence(3)
    for _ in range(15):
        sq.step()
    if not any(sq.go.layer_map.values()):
        sq.go.set_state([(0, [{"id": b"p1", "url": b"u1"}])])
        sq.e.state_set([(0, [{"id": b"p1", "url": b"u1"}])])
    for cb in (0, 700, DEFAULT):
        got = sink.export_pages_dapr(sq.e, "/test/root", "cfg-crawl", "my-crawl-99", "20250615-150640", cb)
        assert got == export_dapr(sq.go, "/test/root", "cfg-crawl", "my-crawl-99", "20250615-150640", cb, sq.zone)
    sq.e.close()


@pytest.mark.gpu
def test_10k_pages_with_100_messages():
    n_pages, per_page = 10_000, 100
    recs, strs, msgs, want = big_state(n_pages, per_page)
    e = Engine()
    e.state_set_arrays(np.array([(1, n_pages)], abi.STATE_LAYER), recs, strs, msgs)
    head, tail = b'{"layers":[{"depth":1,"pages":[', b']}],"metadata":%s,"lastUpdated":%s}' % (META, LAST)
    [(local, n)] = e.state_export(abi.STATE_EXPORT_LOCAL, 0)
    # a page's JSON holds no raw newline: the lines joined by commas are the render's page list
    assert n == len(local) and local.count(b"\n") == n_pages
    assert head + local[:-1].replace(b"\n", b",") + tail == want
    lines = local.splitlines(keepends=True)
    ends = np.cumsum([len(ln) for ln in lines])
    for cb in (DEFAULT, 1 << 20, int(ends[4999]), int(ends[4999]) + 1):
        got = e.state_export(abi.STATE_EXPORT_DAPR, cb)
        exp, buf = [], b""
        for ln in lines:
            buf += ln
            if len(buf) >= cb:
                exp.append(buf)
                buf = b""
        exp += [buf] if buf else []
        assert [base64.b64decode(d) for d, _ in got] == exp
        assert [d for d, _ in got] == [base64.b64encode(x) for x in exp]
    assert e.state_layer_map() == b'{"1":[%s]}' % b",".join(b'"page-%07d"' % p for p in range(n_pages))
    e.close()


@pytest.mark.gpu
def test_cpp_host_demo_state_dapr():
    import os
    import subprocess
    from state_rules import GoState
    host = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "distributed_crawler_b200", "host")
    p = subprocess.run([os.path.join(host, "host_demo"), "--state-dapr"], capture_output=True, timeout=300)
    assert p.returncode == 0, p.stderr
    go = GoState()
    go.set_state([(0, [{"id": b"p1", "url": b"testchannel", "status": b"unfetched", "timestamp": (1750000000, 0, None),
                        "messages": [{"chatId": -1001234567890, "messageId": 5 << 20, "status": b"unfetched",
                                      "pageId": b"p1"}]}])])
    for pid, url in ((b"p2", b"url-2"), (b"p3", b"url-3")):  # StateAddPages(-1, ...) of two depth-0 pages
        go.page_map[pid] = {"id": pid, "url": url, "timestamp": (0, 0, 0)}  # the demo's zeroed ts_sec is 1970
        go.layer_map.setdefault(-1, []).append(pid)
    lines = p.stdout.split(b"\n")
    k = lines.index(marshal_layer_map(go.layer_map))
    assert lines[k + 1:-1] == [base64.b64encode(c) for c in export_dapr_chunks(go, 100, None, 3600)]
