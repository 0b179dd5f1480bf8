"""The library's open-addressed hash tables under crafted probe chains: keys that share one full hash (or one home
slot) at the table size the library picks, built by tests/hash_rules.py, with chains that wrap from the last slot to
slot 0.  Random keys leave every chain one or two slots long, so a probe that trusts a fingerprint, a lost first
occurrence or a lookup that stops at the wrong slot would pass every other test.

First, tests/hash_check.cu checks the restatements against the device functions value for value: without that a
"collision" here could quietly test nothing.  Then each case asserts that its keys collide under the restatement at
the table size the library uses, and that the library's answer equals a plain restatement of the API: an ordered set,
a dict, state_rules.GoState, or the local-sink loop of test_gpu_channel_appends."""
import functools
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import hash_rules as hr
from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import Engine, EngineError, names_to_keys32
from distributed_crawler_b200.pack import Channel, pack_telegram
from helpers import ALL, DEV, J, JL, TANDEM, assert_results_equal, channel_ids, msg, no_page
from oracle.pyoracle import Oracle
from state_rules import GoState
from test_gpu_channel_appends import check as sink_check, run as sink_run

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
WRAP = hr.wrap_target()
SIZES = (2, 33, 1000, 4096)
HC = np.dtype([("kind", "<u4"), ("len", "<u4"), ("a", "<u8"), ("b", "<u8"), ("c", "<u8"), ("d", "<u8"), ("key", "u1", 32)])


def _u64(v):
    return np.asarray(v, np.int64).view(np.uint64) if np.asarray(v).dtype.kind == "i" else np.asarray(v, np.uint64)


def test_device_hashes_equal_the_restatements():
    rng = np.random.default_rng(20)
    keys = np.concatenate([hr.keys_with_hash(300, WRAP), hr.keys_with_hash(200, WRAP, vary_first=True),
                           names_to_keys32(hr.usernames_colliding(20, 1 << 13, 1024, WRAP, rng)),
                           rng.integers(0, 256, (500, 32), dtype=np.uint8)])
    pairs = np.concatenate([hr.join_pairs(200, WRAP, rng), rng.integers(-(1 << 63), (1 << 63) - 1, (200, 2), dtype=np.int64)])
    st = np.array(hr.st_tuples(200, WRAP, rows=[0, 3, 1 << 31], gens=[0, 1, 7], rng=rng), dtype=object)
    names = hr.la_names_colliding(60, 128, 127, rng) + hr.la_prefix_chain(4, 64, hr.la_hash(b"") & 63, rng) + [b"x" * 32]
    recs, want = [], []

    def add(kind, want_v, a=0, b=0, c=0, d=0, key=None, ln=0):
        r = np.zeros(1, HC)
        r["kind"], r["len"], r["a"], r["b"], r["c"], r["d"] = kind, ln, a, b, c, d
        if key is not None:
            r["key"][0, :len(key)] = np.frombuffer(bytes(key), np.uint8)
        recs.append(r)
        want.append(int(want_v))

    h = hr.key_hash(keys)
    for i, k in enumerate(keys):
        add(0, h[i], key=k)
        add(1, hr.key_owner(h[i], 7), a=7, key=k)
        add(4, hr.st_first_hash(h[i], i, True), a=i, key=k)
    for c, m in pairs:
        add(2, hr.join_hash(c, m), a=_u64(c), b=_u64(m))
    for row, gen, c, m in st:
        add(3, hr.st_hash(row, gen, c, m), a=row, b=gen, c=_u64(c), d=_u64(m))
        add(6, hr.st_turn_slot(row, m, 256), a=row, b=_u64(m), c=256)
        add(7, hr.st_view_slot(row, c, m, 64), a=row, b=_u64(c), c=_u64(m), d=64)
    for nm in names:
        add(5, hr.la_hash(nm), key=nm, ln=len(nm))
    with tempfile.TemporaryDirectory() as d:
        exe, fin, fout = (os.path.join(d, x) for x in ("hash_check", "in.bin", "out.bin"))
        subprocess.check_call([NVCC, "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                               os.path.join(HERE, "hash_check.cu")])
        np.concatenate(recs).tofile(fin)
        r = subprocess.run([exe, fin, fout], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        got = np.fromfile(fout, np.uint64)
    kinds = np.concatenate(recs)["kind"]
    bad = np.nonzero(got != np.array(want, np.uint64))[0]
    assert len(got) == len(want) and not len(bad), f"{len(bad)} mismatches, kinds {sorted(set(kinds[bad].tolist()))}"


# ---- key sets ---------------------------------------------------------------------------------------------------------
class OrderedSet:
    def __init__(self):
        self.keys: dict[bytes, None] = {}

    def insert(self, keys):
        new = np.zeros(len(keys), np.uint8)
        for i, k in enumerate(keys):
            b = k.tobytes()
            if b not in self.keys:
                self.keys[b] = None
                new[i] = 1
        return new

    def export(self):
        return np.frombuffer(b"".join(self.keys), np.uint8).reshape(-1, 32)


def _calls(keys, rng):
    """the keys shuffled with repeats, in three calls: repeats inside a call and across calls"""
    n = len(keys)
    seq = np.concatenate([keys, keys[rng.integers(0, n, n // 2 + 1)]])[rng.permutation(n + n // 2 + 1)]
    a, b = len(seq) // 3, 2 * len(seq) // 3
    return [seq[:a], seq[a:b], np.concatenate([seq[b:], seq[:5]])]


def _chain(keys, tslots):
    """the chain's length at its home slot: every key's home slot is the same, and it is the last slot"""
    home = hr.set_home(hr.key_hash(keys), tslots)
    assert (home == np.uint64(tslots - 1)).all(), "the keys do not share the last home slot"
    return len(keys)


@pytest.mark.parametrize("n", SIZES)
def test_frontier_insert_one_full_hash_chain(n):
    rng = np.random.default_rng(n)
    cap = 8192
    tslots = hr.set_table_slots(cap)
    for keys in (hr.keys_with_hash(n, WRAP), hr.keys_with_hash(n, WRAP, prefix=b"same_prefix_"),
                 hr.keys_with_hash(min(n, 255), WRAP, vary_first=True)):
        assert _chain(keys, tslots) == len(keys) and len(set(hr.set_fp(hr.key_hash(keys)).tolist())) == 1
        e = Engine(frontier_capacity=cap)
        assert e.set_info(abi.SET_FRONTIER)["table_slots"] == tslots
        want = OrderedSet()
        for part in _calls(keys, rng):
            assert np.array_equal(e.frontier_insert(part), want.insert(part))
        assert np.array_equal(e.frontier_export(), want.export())
        print(f"frontier_insert: chain {len(keys)} at slot {tslots - 1} of {tslots}, wraps")
        e.close()


@pytest.mark.parametrize("n", SIZES)
def test_frontier_insert_dev_and_set_add_on_a_chain(n):
    import torch
    from distributed_crawler_b200.engine import lib
    rng = np.random.default_rng(100 + n)
    keys = hr.keys_with_hash(n, WRAP)
    dev, want = Engine(frontier_capacity=4096), OrderedSet()
    for part in _calls(keys, rng):
        d_keys = torch.from_numpy(part).cuda()
        d_new = torch.full((len(part),), 7, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        assert lib().tgi_frontier_insert_dev(dev.h, d_keys.data_ptr(), len(part), d_new.data_ptr()) == 0
        assert lib().tgi_frontier_sync(dev.h) == 0
        assert np.array_equal(d_new.cpu().numpy(), want.insert(part))
    assert np.array_equal(dev.frontier_export(), want.export())
    # the exclusion sets: a colliding key that is absent must not be taken for one that is present
    half = keys[: n // 2]
    for which in (abi.SET_INVALID, abi.SET_DISCOVERED):
        dev.set_add(which, np.concatenate([half, half[::-1]]))
        assert dev.set_size(which) == len(half)
        dev.set_add(which, keys[rng.permutation(n)])
        assert dev.set_size(which) == n
    tslots = dev.set_info(abi.SET_FRONTIER)["table_slots"]
    print(f"frontier_insert_dev, set_add: chain {_chain(keys, tslots)} at slot {tslots - 1} of {tslots}, wraps")
    dev.close()


def test_keys_differing_in_their_last_byte_probe_past_a_chain():
    rng = np.random.default_rng(3)
    cap = 1024
    tslots = hr.set_table_slots(cap)
    chain = hr.keys_with_hash(33, WRAP)
    tail = hr.keys_last_byte(tslots, tslots - 1, 34, rng)  # homes inside the chain's slots, across the wrap
    e, want = Engine(frontier_capacity=cap), OrderedSet()
    for part in (chain, tail[: len(tail) // 2], np.concatenate([tail, chain[:3]]), tail):
        assert np.array_equal(e.frontier_insert(part), want.insert(part))
    assert np.array_equal(e.frontier_export(), want.export())
    print(f"last byte: chain {_chain(chain, tslots)} at slot {tslots - 1} of {tslots} (wraps), {len(tail)} keys differing "
          f"in byte 31 at home slots {sorted(hr.set_home(hr.key_hash(tail), tslots).tolist())}")
    e.close()


def test_a_set_filled_to_capacity_with_one_chain():
    cap = 1024
    keys = hr.keys_with_hash(cap + 1, WRAP)
    e = Engine(frontier_capacity=cap)
    assert _chain(keys, e.set_info(abi.SET_FRONTIER)["table_slots"]) == cap + 1
    assert e.frontier_insert(keys[:cap]).all()
    assert e.frontier_size() == cap
    with pytest.raises(EngineError) as ei:
        e.frontier_insert(keys[cap:])
    assert ei.value.code == abi.E_CAPACITY
    assert e.frontier_size() == cap and np.array_equal(e.frontier_export(), keys[:cap])
    assert not e.frontier_insert(keys[:cap][::-1]).any()  # still all found, behind the full chain
    tslots = e.set_info(abi.SET_FRONTIER)["table_slots"]
    print(f"capacity: chain {cap} (+1 refused) at slot {tslots - 1} of {tslots}, wraps")
    e.close()


def test_growth_rehashes_a_long_chain():
    rng = np.random.default_rng(9)
    keys = hr.keys_with_hash(4096, WRAP)
    grow, fixed, want = Engine(frontier_capacity=64, set_growth=1 << 16), Engine(frontier_capacity=8192), OrderedSet()
    for part in _calls(keys, rng) + [keys[rng.permutation(4096)[:700]]]:
        new = want.insert(part)
        assert np.array_equal(grow.frontier_insert(part), new) and np.array_equal(fixed.frontier_insert(part), new)
    info = grow.set_info(abi.SET_FRONTIER)
    assert info["grows"] > 0 and info["table_slots"] == hr.set_table_slots(info["capacity"])
    _chain(keys, info["table_slots"])
    assert np.array_equal(grow.frontier_export(), want.export())
    assert np.array_equal(fixed.frontier_export(), want.export())
    print(f"growth: chain {len(keys)} rehashed {info['grows']} times, now at slot {info['table_slots'] - 1} of "
          f"{info['table_slots']}, wraps")
    grow.close()
    fixed.close()


# ---- the frontier batch table through Telegram batches ----------------------------------------------------------------
TG_CAP, TG_BSLOTS = 4096, 4096  # every batch below has <= 2 048 links: frontier_batch_slots(links) <= TG_BSLOTS
NOW, TTL = 1_760_000_000, 30 * 24 * 3600  # include/tgingest.h TGI_INVALID_TTL_SEC


@functools.lru_cache(maxsize=None)
def _tg_names():
    """usernames sharing the last home slot of the dedup set and the last slot of every batch table <= TG_BSLOTS"""
    return tuple(hr.usernames_colliding(40, hr.set_table_slots(TG_CAP), TG_BSLOTS, WRAP, np.random.default_rng(80)))


def _tg_batch(n, names, seed, carriers=400):
    """n records; `carriers` of them, spread over the batch, hold t.me/ links to the colliding names.  Record 0 names
    every name once, names[0] last (the thread of record 0 reaches its first occurrence last); names[0] is the first
    link of every other carrier"""
    rng = np.random.default_rng(seed)
    at = set(np.linspace(0, n - 1, carriers).astype(int).tolist())
    ms = []
    for k in range(n):
        if k == 0:
            chosen = [names[j] for j in rng.permutation(len(names) - 1) + 1] + [names[0]]
        elif k in at:
            chosen = [names[0]] + [names[j] for j in rng.integers(0, len(names), 3)]
        else:
            chosen = []
        text = "post %d " % k + " ".join("https://t.me/" + nm.decode() for nm in chosen)
        ms.append(msg("messageText", text, id=(k + 1) << 20, channel=k % 2, date=1_700_000_000 + k))
    return pack_telegram(ms, [Channel(title="a", name="ownchannel_a", username="ownchannel_a"),
                              Channel(title="b", name="ownchannel_b", username="ownchannel_b")])


def _tg_step(o, e, batch, flags, label, page):
    ro = o.telegram(batch, flags)
    e.telegram_submit(1, batch, flags)
    rg = e.telegram_wait(1, copy=True)
    assert_results_equal(ro, rg, flags, label)
    assert np.array_equal(o.frontier_export(), e.frontier_export()), f"{label}: frontier differs"
    if not flags & abi.RUN_SKIP_INVALID:
        assert (rg.gpu_launches == 1) == page, f"{label}: {rg.gpu_launches} launches"
    assert hr.frontier_batch_slots(len(ro.links)) <= TG_BSLOTS
    if flags & abi.RUN_SKIP_INVALID:
        assert np.array_equal(o.pending_edges(NOW), e.pending_edges(1, NOW)), f"{label}: pending edges differ"
    e.release(1)
    return ro


def _tg_sequence(page, big=False):
    """half the names into the dedup set, then batches naming all of them: the persistent set's chain, then the batch
    table's chain for the rest, for both run-flag sets"""
    names = list(_tg_names())
    n = 9000 if big else 300
    for flags in (ALL, TANDEM):
        o, e = Oracle(), Engine(frontier_capacity=TG_CAP)
        label = f"{'page' if page else 'bulk'} {n} records flags {flags:#x}"
        _tg_step(o, e, _tg_batch(n, names[::2], 1), flags, label + " (first)", page)
        ro = _tg_step(o, e, _tg_batch(n, names, 2), flags, label, page)
        if flags == ALL:  # no username filter: every name is a key
            assert e.frontier_size() == len(names) and (ro.links["flags"] & abi.LF_NEW != 0).sum() == len(names) // 2
        e.close()
        o.close()
    print(f"frontier batch table: {len(names)} names at home slot {hr.set_table_slots(TG_CAP) - 1} of "
          f"{hr.set_table_slots(TG_CAP)} and batch slot bmask of every table <= {TG_BSLOTS}, wraps")


def test_telegram_batches_on_one_chain_page_kernel():
    _tg_sequence(page=True)


def test_telegram_batches_on_one_chain_bulk_pipeline():
    with no_page():
        _tg_sequence(page=False)


def test_telegram_batches_on_one_chain_above_the_page_size():
    _tg_sequence(page=False, big=True)


def test_telegram_batches_on_one_chain_one_cta_per_sm():
    """TGI_GRID_MULT=1 (read once per process, hence a child process): the probe loop takes many records per thread"""
    code = ("import sys; sys.path.insert(0, 'tests')\n"
            "import test_gpu_hash_collisions as t\n"
            "t._tg_sequence(page=False, big=True)\n"
            "print('ok')\n")
    root = os.path.dirname(HERE)
    p = subprocess.run([sys.executable, "-c", code], cwd=root, env=dict(os.environ, TGI_GRID_MULT="1"),
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and "ok" in p.stdout, p.stderr[-3000:]


def test_invalid_stamps_around_the_ttl_on_one_chain():
    """invalid-set stamps 0 (never expires), TTL-1, TTL and TTL+1 seconds old on names of one chain, and discovered
    names in the same chain: TGI_RUN_SKIP_INVALID's LF_INVALID flags and the pending-edge statuses"""
    names = list(_tg_names())
    inv = names[:16]
    stamps = np.array([[0, NOW - (TTL - 1), NOW - TTL, NOW - (TTL + 1)][k % 4] for k in range(len(inv))], np.int64)
    disc = names[16:24] + names[:2]
    flags = TANDEM | abi.RUN_SKIP_INVALID
    for page, n in ((True, 300), (False, 9000)):
        o, e = Oracle(), Engine(frontier_capacity=TG_CAP)
        for x in (o, e):
            x.set_add(abi.SET_INVALID, names_to_keys32(inv), stamps)
            x.set_add(abi.SET_DISCOVERED, names_to_keys32(disc))
            x.set_now(NOW)
        ro = _tg_step(o, e, _tg_batch(n, names, 3), flags, f"invalid stamps, {n} records", page)
        flagged = {bytes(lk["name"][:lk["len"]]) for lk in ro.links if lk["flags"] & abi.LF_INVALID}
        assert flagged == {nm for nm, t in zip(inv, stamps) if t == 0 or NOW - t < TTL}
        e.close()
        o.close()


# ---- key join ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", (2, 33, 1000, 4096))
def test_key_join_on_one_full_hash_chain(n):
    rng = np.random.default_rng(40 + n)
    pairs = hr.join_pairs(n + n // 2 + 14, WRAP, rng)
    a_keys, absent = pairs[: n], pairs[n:]
    a = np.concatenate([a_keys, a_keys[rng.integers(0, n, n)]])[rng.permutation(2 * n)]  # repeats: lowest index wins
    assert (hr.join_hash(a[:, 0], a[:, 1]) & np.uint64(hr.join_slots(len(a)) - 1) == np.uint64(hr.join_slots(len(a)) - 1)).all()
    b = np.concatenate([a_keys, absent, a_keys[::-1]])[rng.permutation(2 * n + len(absent))]
    first = {}
    for i, (c, m) in enumerate(a.tolist()):
        first.setdefault((c, m), i)
    want = np.array([first.get((c, m), -1) for c, m in b.tolist()], np.int64)
    e = Engine()
    got = e.key_join(a, b)
    assert np.array_equal(got, want), f"{int((got != want).sum())} of {len(b)} differ"
    print(f"key_join: chain {len(a_keys)} distinct keys ({len(a)} rows) at slot {hr.join_slots(len(a)) - 1} of "
          f"{hr.join_slots(len(a))}, wraps")
    e.close()


# ---- progress state ---------------------------------------------------------------------------------------------------
META, LAST = b'{"crawlId":"c"}', b'"2024-01-02T03:04:05Z"'
TS = (1_700_000_000, 0, 0)


def _state_check(e, go, rows):
    """GetPage's messages of every row, and state.json, against GoState"""
    for pid, row in rows.items():
        want = [dict({"platform": b""}, **m) for m in go.page_map[pid].get("messages") or []]
        assert e.state_read_page(row) == want, pid
    assert e.state_render(META, LAST) == go.marshal(META, LAST), "state.json differs"


def _live(go):
    return sum(len(p.get("messages") or []) for p in go.page_map.values())


def test_update_messages_on_chains_across_rows_and_generations():
    rng = np.random.default_rng(50)
    pids = [b"p%d" % k for k in range(4)]
    pages = [{"id": p, "url": b"https://t.me/" + p, "depth": 0, "status": b"fetched", "timestamp": TS} for p in pids]
    # one full st_hash across rows (SetState's rows 0-3, generation 0): every page's messages in one chain
    tuples = hr.st_tuples(120, WRAP, rows=[0, 1, 2, 3], gens=[0], rng=rng)
    for row, _, c, m in tuples:
        pages[row].setdefault("messages", []).append({"chatId": c, "messageId": m, "status": b"unfetched", "pageId": pids[row]})
    go, e = GoState(), Engine()
    go.set_state([(0, pages)])
    rows = dict(zip(pids, e.state_set([(0, pages)])))
    assert list(rows.values()) == [0, 1, 2, 3]
    by_row = {v: k for k, v in rows.items()}
    tslots = hr.state_table_slots(hr.STATE_INITIAL_SLOTS, len(tuples))
    assert (hr.st_hash(*np.array(tuples, dtype=object).T.tolist()) & np.uint64(tslots - 1) == np.uint64(tslots - 1)).all()
    print(f"state: chain {len(tuples)} across 4 rows at slot {tslots - 1} of {tslots}, wraps")
    _state_check(e, go, rows)
    # keys of page p0 whose generation-1 and generation-2 forms share a home slot in every table of <= 2^12 slots:
    # after the next UpdatePage the old keys are tombstones in the chain the new generation probes
    row0 = rows[b"p0"]
    ms = hr.st_same_home_across_gens(8, row0, (1, 2), -77, 12, rng)
    print(f"state: {len(ms)} keys whose generation-1 tombstones share the home slot of their generation-2 form "
          f"in a table of {tslots}")
    page = dict(pages[0], messages=[{"chatId": -77, "messageId": m, "status": b"fetched", "pageId": b"p0"} for m in ms[:6]])
    go.update_page(page)
    e.state_update_page(page)  # generation 1
    page = dict(pages[0], messages=[{"chatId": -77, "messageId": m, "status": b"fetched", "pageId": b"p0"} for m in ms[4:]])
    go.update_page(page)
    e.state_update_page(page)  # generation 2: ms[:4] live only as generation-1 tombstones
    ups = [(b"p0", -77, m, b"deleted") for m in ms] + [(by_row[r], c, m, b"failed") for r, _, c, m in tuples[::3]]
    absent = hr.st_tuples(40, WRAP, rows=[rows[p] for p in pids], gens=[0], rng=np.random.default_rng(51))
    ups += [(by_row[r], c, m, b"resample") for r, _, c, m in absent[-20:]]
    ups += [ups[k] for k in rng.integers(0, len(ups), 30)]
    order = rng.permutation(len(ups))
    ups = [ups[k] for k in order]
    for pid, c, m, st in ups:
        assert go.update_message(pid, c, m, st)
    assert e.state_update_messages([(rows[pid], c, m, st) for pid, c, m, st in ups]) == 0
    _state_check(e, go, rows)


def test_update_batches_whose_keys_share_one_batch_slot():
    """distinct keys in one batch-table slot (bfirst / blast), repeated so the last writer and the first occurrence
    sit deep in the chain; enough rows to force the table's rebuild (2 * need > tslots); then a compaction (tombstones
    outnumber the live rows) and more batches over the same chains"""
    rng = np.random.default_rng(60)
    pids = [b"q%d" % k for k in range(3)]
    pages = [{"id": p, "url": b"u" + p, "depth": 0, "status": b"fetched", "timestamp": TS} for p in pids]
    go, e = GoState(), Engine()
    go.set_state([(0, pages)])
    rows = dict(zip(pids, e.state_set([(0, pages)])))
    by_row = {v: k for k, v in rows.items()}
    statuses = [b"fetched", b"failed", b"deleted", b"resample"]
    tslots = hr.STATE_INITIAL_SLOTS
    all_keys = []

    def batch_of(m_up):
        bslots = hr.state_batch_slots(m_up)
        keys = hr.st_batch_collisions(m_up // 3, bslots, bslots - 1, rows=list(rows.values()), chat=-9, rng=rng)
        all_keys.extend(keys)
        ups = [keys[k] for k in rng.integers(0, len(keys), m_up)]
        print(f"state: batch of {m_up} updates, {len(keys)} distinct keys at batch slot {bslots - 1} of {bslots}")
        return [(by_row[r], -9, m, statuses[k % 4]) for k, (r, m) in enumerate(ups)]

    def apply(batch):
        for pid, c, m, st in batch:
            go.update_message(pid, c, m, st)
        assert e.state_update_messages([(rows[p], c, m, st) for p, c, m, st in batch]) == 0
        _state_check(e, go, rows)

    for m_up in (60, 400, 3000):
        before = _live(go)
        apply(batch_of(m_up))
        tslots = hr.state_table_slots(tslots, _live(go))
        print(f"state: {before} -> {_live(go)} message rows, table of {tslots} slots")
    assert tslots > hr.STATE_INITIAL_SLOTS  # the table was rebuilt larger
    # compaction with the chains in place: two of the three lists replaced by five messages each, so the tombstones
    # outnumber the live rows (st_compact: n_dead > live)
    dead = 0
    for pid in pids[:2]:
        old = go.page_map[pid]["messages"]
        dead += len(old)
        page = dict(pages[pids.index(pid)], messages=old[:5])
        go.update_page(page)
        e.state_update_page(page)
    assert dead > _live(go), (dead, _live(go))
    print(f"state: {dead} tombstones against {_live(go)} live rows: compacted")
    _state_check(e, go, rows)
    # the same chains after the compaction: present, dropped and new keys of the chain in one batch
    again = [all_keys[k] for k in rng.integers(0, len(all_keys), 500)]
    apply([(by_row[r], -9, m, statuses[k % 4]) for k, (r, m) in enumerate(again)])
    apply(batch_of(800))


# ---- local sink ---------------------------------------------------------------------------------------------------------
def _sink_batch(names, n=600):
    chans = [Channel(title="T%d" % k, name=nm, username="u%d" % k) for k, nm in enumerate(names)]
    ms = [msg("messageText", "m%d " % k + "y" * (k % 50), id=(k + 1) << 20, channel=(k * 7) % len(chans),
              date=1_700_000_000 + k) for k in range(n)]
    return pack_telegram(ms, chans)


def test_local_sink_channel_ids_in_one_chain():
    rng = np.random.default_rng(70)
    rows = 60
    tslots = hr.sink_slots(rows)
    wrap = hr.la_names_colliding(20, tslots, tslots - 1, rng, lengths=(5, 9, 17))  # across the last slot
    empty_slot = hr.la_hash(b"") & (tslots - 1)
    chain = hr.la_prefix_chain(6, tslots, empty_slot, rng)  # "", then names that are prefixes of one another
    other = hr.la_names_colliding(10, tslots, empty_slot, rng, lengths=(2, 6, 12))
    distinct = wrap + chain + other
    names = list(distinct) + [distinct[k] for k in rng.integers(0, len(distinct), rows - len(distinct))]
    order = rng.permutation(rows)
    names = [names[k] for k in order]  # equal names on different rows: the lowest row must win
    batch = _sink_batch(names)
    ids = channel_ids(batch, False)
    assert ids == names and len(ids) == rows
    homes = [hr.la_hash(c) & (tslots - 1) for c in ids]
    assert sum(h == tslots - 1 for h in homes) >= 20 and sum(h == empty_slot for h in homes) >= 16
    ro = Oracle().telegram(batch, J)
    e = Engine()
    for flags in (JL, J | DEV):
        sink_check(batch, False, ro, sink_run(e, batch, flags), f"page flags {flags:#x}")
        with no_page():
            sink_check(batch, False, ro, sink_run(e, batch, flags), f"bulk flags {flags:#x}")
    print(f"local sink: {rows} rows, {len(distinct)} channelIDs in chains at slots {tslots - 1} (wraps) and "
          f"{empty_slot} of {tslots}")
    e.close()
