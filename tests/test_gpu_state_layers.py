"""GPU tests: layer reads (tgi_state_read_layer / tgi_state_read_pages / tgi_state_layers) against tests/layer_rules.py
over the restatement the sequences keep in lockstep (state_rules, runner_rules, close_rules, discover_rules): after every
step of seeded sequences of SetState, AddLayer, Dapr's AddLayer, UpdatePage, UpdateMessage, one- and multi-page turns and
closes, and discovery in both modes with the layer end, every depth is read under every selection — fields, strings,
message lists and selection bytes — with random row lists (repeats included) and the layer summary.  Also: pages made
by discovery read back by row alone, a state with more message rows than one pass of the state kernels' grid, the
one-page read on the same path, launch counts that do not depend on n, and rejected calls."""
import os
import subprocess
import sys

import pytest

import layer_rules as lr
from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import Engine, EngineError
from distributed_crawler_b200.state_pack import ZERO_TIME
from state_rules import GoState
from test_gpu_state import LAST, META
from test_gpu_state_discover import FLAGS, RUN_MODES, DiscoverSequence
from test_gpu_state_pages import PagesSequence

pytestmark = pytest.mark.gpu
SELECTS = (abi.SELECT_NONE, abi.SELECT_STANDALONE, abi.SELECT_STANDALONE_RESUME, abi.SELECT_DAPR)


def full(p):
    """a restatement page in the form the engine reads it: every string, depth, timestamp and the message list"""
    q = {name: p.get(name, b"") for name in abi.STATE_STRINGS}
    q["depth"] = p.get("depth", 0)
    q["timestamp"] = tuple(p.get("timestamp", ZERO_TIME))
    q["messages"] = [dict({"platform": b""}, **m) for m in p.get("messages") or []]
    return q


def selection(layer, select):
    if select == abi.SELECT_NONE:
        return None
    if select == abi.SELECT_DAPR:
        return lr.dapr_selection(layer)
    return lr.standalone_selection(layer, select == abi.SELECT_STANDALONE_RESUME)


def check_layers(e, go, rnd):
    """every depth (and a missing one) under every selection, random row lists with repeats, the layer summary"""
    depths = sorted(go.layer_map)
    for depth in depths + [max(depths, default=0) + 1, min(depths, default=0) - 1]:
        want = lr.get_layer_by_depth(go, depth)
        select = rnd.choice(SELECTS)
        pages, sel = e.state_read_layer(depth, select)
        assert pages == [full(p) for p in want], depth
        assert e.state_read_rows == [e._st_rows()[p["id"]] for p in want]
        assert sel == selection(want, select)
        for other in SELECTS:  # the other selections, without the lists
            a = e.state_read_layer_arrays(depth, other, 0)
            s = selection(want, other)
            assert (a["select"] is None) == (s is None)
            if s is not None:
                assert [bool(x) for x in a["select"]] == s and a["n_selected"] == sum(s)
            assert a["msgs"] is None and a["msg_first"] is None and not a["pages"]["n_msgs"].any()
    rows = e._st_rows()
    ids = [i for i in go.page_map if i in rows]
    if ids:
        pick = [rnd.choice(ids) for _ in range(rnd.choice([1, 2, 9, 40]))]
        pick += rnd.sample(pick, rnd.randrange(len(pick) + 1))  # repeats
        rnd.shuffle(pick)
        assert e.state_read_pages([rows[p] for p in pick]) == [full(go.page_map[p]) for p in pick]
    assert e.state_layers() == {"layers": [(d, len(go.layer_map[d])) for d in depths],
                                "max_depth": lr.get_max_depth(go), "n_incomplete": lr.incomplete_pages(go)}


class LayersPagesSequence(PagesSequence):
    """PagesSequence (one- and multi-page turns and closes, UpdatePage, AddLayer, Dapr's AddLayer, discovery from a
    slot's result) with UpdateMessage calls and SetState with repeated ids mixed in, every layer read after each step"""

    def check(self):
        super().check()
        check_layers(self.e, self.go, self.rnd)

    def update_messages(self):
        r = self.rnd
        busy = set(self.views)
        for p, _ in self.open.values():
            busy |= set(p if isinstance(p, tuple) else (p,))
        free = [i for i in self.ids() if i not in busy]
        if not free:
            return
        ups = []
        for _ in range(r.randrange(1, 30)):
            pid = r.choice(free)
            msgs = self.go.page_map[pid].get("messages") or []
            key = (lambda m: (m["chatId"], m["messageId"]))(r.choice(msgs)) if msgs and r.random() < 0.6 else \
                (r.choice([-1001, 5]), r.randrange(20, 24) << 20)
            ups.append((pid, key, r.choice([b"fetched", b"failed", b"custom"])))
        for pid, (c, m), st in ups:
            self.go.update_message(pid, c, m, st)
        rows = self.e._st_rows()
        self.e.state_update_messages([(rows[pid], c, m, st) for pid, (c, m), st in ups])
        self.check()

    def set_with_repeats(self):
        """SetState whose layers list an id twice, and a negative depth: the open turns and views go"""
        keep = self.ids()[:60]
        pages = [dict(self.go.page_map[p], messages=[dict(m) if m["pageId"] in keep else dict(m, pageId=p)
                                                     for m in self.go.page_map[p].get("messages") or []])
                 for p in keep]
        for p in pages:
            p["status"] = self.rnd.choice([b"fetched", b"unfetched", b"error"])
        layers = [(0, pages[:30] + pages[:3]), (-2, pages[30:40]), (1, pages[40:] + [pages[45]])]
        self.go.set_state(layers)
        self.e.state_set(layers)
        self.open.clear()
        self.views.clear()
        self.check()


@pytest.mark.parametrize("seed", range(3))
def test_reads_after_every_turn_close_and_update(seed):
    sq = LayersPagesSequence(seed, 200)
    for i in range(60):
        k = sq.rnd.random()
        if k < 0.05:
            sq.set_with_repeats()
        elif k < 0.2:
            sq.update_messages()
        else:
            sq.multi_step()
    sq.e.close()


class LayersDiscoverSequence(DiscoverSequence):
    """DiscoverSequence with every layer read after each step, and the added pages read back by row alone"""

    def check(self):
        super().check()
        check_layers(self.e, self.go, self.rnd)

    def expect_added(self, got, want, flags):
        super().expect_added(got, want, flags)
        # the URLs the next layer must crawl, from the rows alone
        pages = self.e.state_read_pages(got["rows"])
        assert [p["url"] for p in pages] == [w["url"] for w in want]
        assert pages == [full(w) for w in want]


@pytest.mark.parametrize("seed", range(3))
def test_reads_after_discovery_and_the_layer_end(seed):
    sq = LayersDiscoverSequence(100 + seed)
    r = sq.rnd
    for step in range(30):
        sq.now = (sq.now[0] + 1, r.choice([0, 1, 999_999_999]))
        ids = list(sq.go.page_map)
        k = r.random()
        if k < 0.45:
            owners = r.sample(ids, min(len(ids), r.choice([1, 3])))
            sq.discover(owners, r.choice(FLAGS), True, r.choice(RUN_MODES), slot=step % 3)
        elif k < 0.75:
            owners = r.sample(ids, min(len(ids), r.choice([1, 4])))
            sq.discover(owners, r.choice(FLAGS), False, r.choice(RUN_MODES), slot=step % 3)
        else:
            sq.next_layer(r.choice(FLAGS), r.randrange(3))
    sq.e.close()


def big_state(n_msgs, n_pages=300):
    """layers of n_pages pages holding more than n_msgs messages, on every page but each ninth, some naming another page;
    the layer at depth 1 lists one page twice"""
    import random
    r = random.Random(5)
    per = n_msgs // (n_pages - n_pages // 9 - 1) + 2  # every ninth page has no messages
    pages = [{"id": b"big%d" % k, "url": b"https://t.me/b%d" % (k % 250), "depth": k % 4,
              "status": r.choice([b"fetched", b"unfetched", b"error"]), "timestamp": (1700000000 + k, k, None if k % 2 else 3600),
              "messages": [{"chatId": -1000 - k, "messageId": j << 20, "status": r.choice([b"fetched", b"resample"]),
                            "pageId": b"big%d" % ((k + (j % 7 == 0)) % n_pages), "platform": b"telegram" if j % 5 else b""}
                           for j in range(per if k % 9 else 0)]} for k in range(n_pages)]
    layers = [(d, [p for p in pages if p["depth"] == d] + ([pages[d]] if d == 1 else [])) for d in range(4)]
    return layers


def check_big(e, go, rnd):
    check_layers(e, go, rnd)
    rows = e._st_rows()
    for pid in rnd.sample(list(go.page_map), 4):  # the one-page read, the n = 1 case of the same path
        assert e.state_read_page(rows[pid]) == full(go.page_map[pid])["messages"]


def test_a_state_past_one_grid_pass():
    import random
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = sms * 16 * 256 + 2000  # st_grid: 16 CTAs of 256 threads per SM
    e, go, rnd = Engine(), GoState(), random.Random(1)
    layers = big_state(n)
    go.set_state(layers)
    e.state_set(layers)
    assert sum(len(p.get("messages") or []) for p in go.page_map.values()) > n
    # a dead generation: one page's list replaced, so tombstones sit among the rows (compaction keeps them below half)
    p = dict(go.page_map[b"big1"], messages=go.page_map[b"big1"]["messages"][:5])
    go.update_page(p)
    e.state_update_page(p)
    check_big(e, go, rnd)
    assert e.state_render(META, LAST) == go.marshal(META, LAST)
    e.close()


def test_reads_with_a_grid_of_one_cta_per_sm():
    """TGI_GRID_MULT=1 (read once per process, hence a child process) shrinks the record kernels' grids; the reads,
    whose kernels size their grids themselves (16 CTAs per SM), give the same lists under it"""
    code = (
        "import sys, random; sys.path.insert(0, 'tests')\n"
        "from distributed_crawler_b200.engine import Engine\n"
        "from state_rules import GoState\n"
        "import test_gpu_state_layers as t\n"
        "e, go = Engine(), GoState()\n"
        "layers = t.big_state(200_000)\n"
        "go.set_state(layers)\n"
        "e.state_set(layers)\n"
        "t.check_big(e, go, random.Random(2))\n"
        "e.close()\n"
        "print('ok')\n")
    env = dict(os.environ, TGI_GRID_MULT="1")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and "ok" in p.stdout, p.stderr[-3000:]


def test_launches_do_not_depend_on_n_and_the_one_page_read_uses_them():
    e, go = Engine(), GoState()
    layers = big_state(30_000, 400)
    go.set_state(layers)
    e.state_set(layers)
    rows = e._st_rows()
    ids = list(go.page_map)
    launches = set()
    for n in (1, 2, 17, 400, 1000):
        pick = [ids[(7 * k) % len(ids)] for k in range(n)]
        assert e.state_read_pages([rows[p] for p in pick]) == [full(go.page_map[p]) for p in pick]
        launches.add(e.state_read_launches)
    assert len(launches) == 1 and launches.pop() > 0
    e.state_read_pages([rows[ids[0]]], messages=False)
    assert e.state_read_launches == 0
    e.state_layers()
    e.close()


def test_rejected_calls_leave_the_state_unchanged():
    e, go = Engine(), GoState()
    layers = big_state(2000, 40)
    go.set_state(layers)
    e.state_set(layers)
    before = e.state_render(META, LAST)
    n_rows = len(go.page_map)

    def rejected(call):
        with pytest.raises(EngineError) as ei:
            call()
        assert ei.value.code == abi.E_ARG
        assert e.state_render(META, LAST) == before

    rejected(lambda: e.state_read_pages([0, n_rows]))
    rejected(lambda: e.state_read_pages([abi.STATE_NO_PAGE]))
    rejected(lambda: e.state_read_pages_arrays([0], flags=2))
    rejected(lambda: e.state_read_layer(0, select=4))
    rejected(lambda: e.state_read_layer(0, select=-1))
    rejected(lambda: e.state_read_layer_arrays(0, flags=abi.READ_MESSAGES | 8))
    # nothing to read is not an error: no rows, a missing layer, an empty state
    assert e.state_read_pages([]) == []
    assert e.state_read_layer(99, abi.SELECT_DAPR) == ([], [])
    e.state_set([])
    assert e.state_layers() == {"layers": [], "max_depth": None, "n_incomplete": 0}
    assert e.state_read_layer(0) == ([], None)
    e.close()
