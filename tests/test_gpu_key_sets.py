"""The resident key sets through the C ABI: the exclusion sets before and at their first tgi_set_add, tgi_set_clear,
inserts past a fixed capacity, the device-pointer forms of the dedup set, and the single-rank partition across
tgi_frontier_clear and tgi_comm_destroy."""
import ctypes as C

import numpy as np
import pytest
import torch

from distributed_crawler_b200 import abi
from distributed_crawler_b200.corpus import Corpus
from distributed_crawler_b200.engine import Engine, EngineError, lib
from helpers import TANDEM, assert_results_equal
from oracle.pyoracle import Oracle

pytestmark = pytest.mark.gpu
EXCL = (abi.SET_INVALID, abi.SET_DISCOVERED)
EMPTY_INFO = dict(count=0, capacity=0, table_slots=0, grows=0)
NOW = 1_760_000_000


def _keys(ids):
    """distinct 32-byte keys "k" + 8 decimal digits, zero padded"""
    ids = np.asarray(ids)
    k = np.zeros((len(ids), 32), np.uint8)
    k[:, 0] = ord("k")
    for d in range(8):
        k[:, 8 - d] = ord("0") + (ids // 10 ** d) % 10
    return k


def _raises(code, fn, *args):
    with pytest.raises(EngineError) as ei:
        fn(*args)
    assert ei.value.code == code
    return ei.value


def test_exclusion_sets_before_their_first_add():
    c = Corpus(3000, profile=3, first=77)
    flags = TANDEM | abi.RUN_SKIP_INVALID
    e = Engine(frontier_capacity=1000)
    for which in EXCL:
        assert e.set_size(which) == 0
        assert e.set_info(which) == EMPTY_INFO
        e.set_clear(which)  # nothing to clear: still not allocated
        assert e.set_info(which) == EMPTY_INFO
    # the kernels see two empty sets: no link is skipped as invalid, every new edge is pending
    ro = Oracle().telegram(c.batch, flags)
    e.telegram_submit(1, c.batch, flags)
    rg = e.telegram_wait(1, copy=True)
    assert_results_equal(ro, rg, flags)
    assert (rg.links["flags"] & abi.LF_INVALID).sum() == 0
    rows = e.pending_edges(1, NOW)
    assert len(rows) == rg.n_new > 0 and (rows["status"] == abi.EDGE_PENDING).all()
    e.release(1)
    # an empty add allocates the set, growth off: the dedup set's capacity and table
    e.set_add(abi.SET_INVALID, np.zeros((0, 32), np.uint8))
    assert e.set_info(abi.SET_INVALID) == dict(count=0, capacity=1000, table_slots=2048, grows=0)
    assert e.set_info(abi.SET_DISCOVERED) == EMPTY_INFO
    e.close()


def test_first_add_sizes():
    none = np.zeros((0, 32), np.uint8)
    # growth on: min(frontier_capacity, 2^16) keys in a table of twice as many slots
    for fcap, cap in ((1000, 1000), (1 << 17, 1 << 16)):
        e = Engine(frontier_capacity=fcap, set_growth=1 << 20)
        e.set_add(abi.SET_DISCOVERED, none)
        assert e.set_info(abi.SET_DISCOVERED) == dict(count=0, capacity=cap, table_slots=2 * (1 << (cap - 1).bit_length()), grows=0)
        e.close()
    # growth on, the dedup set grows, growth off: the first add takes the dedup set's current size, not its initial one
    e = Engine(frontier_capacity=64, set_growth=1 << 20)
    e.frontier_insert(_keys(range(1000)))
    fr = e.set_info(abi.SET_FRONTIER)
    assert fr["capacity"] == 1024 and fr["grows"] > 0
    e.set_growth(0)
    for which in EXCL:
        e.set_add(which, none)
        assert e.set_info(which) == dict(count=0, capacity=fr["capacity"], table_slots=fr["table_slots"], grows=0)
    e.close()


def test_set_clear_empties_one_set():
    inv, disc, fr = _keys(range(1000)), _keys(range(5000, 5500)), _keys(range(9000, 9300))
    e = Engine(frontier_capacity=64, set_growth=1 << 20)
    e.set_add(abi.SET_INVALID, inv, np.full(len(inv), NOW, np.int64))
    e.set_add(abi.SET_DISCOVERED, disc)
    e.frontier_insert(fr)
    before = {w: e.set_info(w) for w in (abi.SET_FRONTIER,) + EXCL}
    assert before[abi.SET_INVALID]["grows"] > 0
    e.set_clear(abi.SET_INVALID)
    assert e.set_info(abi.SET_INVALID) == dict(before[abi.SET_INVALID], count=0)  # capacity and growth steps stay
    assert e.set_size(abi.SET_INVALID) == 0
    for w in (abi.SET_FRONTIER, abi.SET_DISCOVERED):
        assert e.set_info(w) == before[w]
    assert np.array_equal(e.frontier_export(), fr)
    # the cleared keys go in again
    e.set_add(abi.SET_INVALID, inv[:600])
    assert e.set_size(abi.SET_INVALID) == 600
    e.set_add(abi.SET_INVALID, inv)
    assert e.set_size(abi.SET_INVALID) == len(inv)
    e.set_clear(abi.SET_DISCOVERED)
    assert e.set_size(abi.SET_DISCOVERED) == 0 and e.set_size(abi.SET_INVALID) == len(inv)
    e.close()


def test_insert_past_a_fixed_capacity():
    a, b = _keys(range(60)), _keys(range(100, 160))
    e = Engine(frontier_capacity=100)
    assert e.frontier_insert(a).all()
    err = _raises(abi.E_CAPACITY, e.frontier_insert, b)
    assert "frontier capacity 100 exceeded" in str(err)
    assert e.frontier_size() == 60
    assert np.array_equal(e.frontier_export(), a)
    assert e.frontier_insert(np.concatenate([a[:10], b[:40]])).sum() == 40  # what fits still goes in
    for which in EXCL:
        e.set_add(which, a)
        err = _raises(abi.E_CAPACITY, e.set_add, which, b)
        assert "frontier capacity 100 exceeded" in str(err)
        assert e.set_size(which) == 60
        assert e.set_info(which) == dict(count=60, capacity=100, table_slots=256, grows=0)
    e.close()


def _export_dev(e, first, cap):
    out = torch.zeros((max(cap, 1), 32), dtype=torch.uint8, device="cuda")
    n = C.c_uint64()
    torch.cuda.synchronize()
    assert lib().tgi_frontier_export_dev(e.h, out.data_ptr(), cap, first, C.byref(n)) == 0
    return out[: n.value].cpu().numpy()


def test_device_pointer_forms_match_the_host_forms():
    rng = np.random.default_rng(11)
    rounds = [_keys(rng.integers(0, 3000, size)) for size in (2000, 2500, 1)]
    dev, host = Engine(frontier_capacity=1 << 14), Engine(frontier_capacity=1 << 14)
    for keys in rounds:
        d_keys = torch.from_numpy(keys).cuda()
        d_new = torch.full((len(keys),), 7, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        assert lib().tgi_frontier_insert_dev(dev.h, d_keys.data_ptr(), len(keys), d_new.data_ptr()) == 0
        assert lib().tgi_frontier_sync(dev.h) == 0
        assert np.array_equal(d_new.cpu().numpy(), host.frontier_insert(keys))
    want = host.frontier_export()
    total = len(want)
    assert dev.frontier_size() == total and np.array_equal(dev.frontier_export(), want)
    for first, cap in ((0, total), (0, 10_000), (17, 250), (total - 5, 100), (total, 10), (total + 3, 10), (3, 0)):
        assert np.array_equal(_export_dev(dev, first, cap), want[first:first + cap]), (first, cap)
    dev.close()
    host.close()


def test_single_rank_partition_clear_and_destroy():
    a, b = _keys(range(0, 4000, 2)), _keys(range(1000, 3000))
    e = Engine(frontier_capacity=1 << 13)
    e.comm_init(Engine.comm_unique_id(), 0, 1)
    e.frontier_insert(a)
    assert e.frontier_merge() == (len(a), len(a))
    owned = e.set_info(abi.SET_OWNED)
    assert owned["count"] == len(a)
    e.frontier_clear()  # the dedup set and the partition, capacities kept
    assert e.frontier_size() == 0
    assert e.set_info(abi.SET_OWNED) == dict(owned, count=0)
    assert e.set_info(abi.SET_FRONTIER)["capacity"] == 1 << 13
    assert e.frontier_insert(b).all()
    assert e.frontier_merge() == (len(b), len(b))
    assert np.array_equal(e.frontier_global_export(), b)
    assert lib().tgi_comm_destroy(e.h) == 0
    _raises(abi.E_STATE, e.set_info, abi.SET_OWNED)
    e.frontier_clear()  # no partition left to clear
    assert e.frontier_size() == 0
    e.close()
