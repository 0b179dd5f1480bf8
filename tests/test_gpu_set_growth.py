"""Resident key sets that grow on demand (tgi_set_growth): every result equals the oracle's, whose sets are unbounded, and
a set that was big enough from the start; growth past the limit fails like a fixed set and leaves the set untouched."""
import os
import socket

import numpy as np
import pytest
import torch

from distributed_crawler_b200 import abi
from distributed_crawler_b200.corpus import Corpus
from distributed_crawler_b200.engine import Engine, EngineError, names_to_keys32
from helpers import TANDEM, assert_results_equal
from oracle.pyoracle import Oracle

pytestmark = pytest.mark.gpu
N, PARTS = 300_000, 5
NOW = 1_760_000_000
DAY = 24 * 3600
CPUS = os.cpu_count() or 1


def _parts(c):
    step = N // PARTS
    return [c.batch.slice(k * step, (k + 1) * step) for k in range(PARTS)]


@pytest.fixture(scope="module")
def bulk():
    """the config-3 corpus in PARTS batches through the oracle: per-batch results and the frontier after each batch"""
    c = Corpus(N, profile=3, first=4242, nthreads=4)
    o = Oracle()
    res, exports = [], []
    for p in _parts(c):
        res.append(o.telegram(p, TANDEM, nthreads=CPUS))
        exports.append(o.frontier_export())
    o.close()
    return c, res, exports


def test_bulk_batches_grow_the_frontier(bulk):
    c, want, exports = bulk
    grow, fixed = Engine(frontier_capacity=64, set_growth=1 << 24), Engine(frontier_capacity=1 << 22)
    assert grow.set_info(abi.SET_FRONTIER) == dict(count=0, capacity=64, table_slots=128, grows=0)
    for k, p in enumerate(_parts(c)):
        rg, rf = grow.telegram(p, TANDEM), fixed.telegram(p, TANDEM)
        assert rg.gpu_launches > 1
        assert_results_equal(want[k], rg, TANDEM, f"batch {k} vs oracle")
        assert_results_equal(rf, rg, TANDEM, f"batch {k} vs fixed capacity")
        assert np.array_equal(grow.frontier_export(), exports[k]), f"batch {k}: export"
    info = grow.set_info(abi.SET_FRONTIER)
    assert info["grows"] > 0 and info["count"] == len(exports[-1]) <= info["capacity"] <= 1 << 24
    assert info["table_slots"] >= 2 * info["capacity"]
    assert fixed.set_info(abi.SET_FRONTIER)["grows"] == 0
    grow.frontier_clear()  # keeps the grown capacity
    assert grow.set_info(abi.SET_FRONTIER) == dict(info, count=0)
    grow.close()
    fixed.close()


def test_pages_on_three_slots_grow_through_the_fallback(bulk):
    """pages of 100 messages, three in flight at a time, from a set of 16 keys: a page whose new keys do not fit leaves
    the set alone and reruns through the bulk pipeline, which grows the set first"""
    c, want, _ = bulk
    first = want[0]  # the pages cover the first 30 000 records of the first bulk batch
    pages = [c.batch.slice(k * 100, (k + 1) * 100) for k in range(300)]
    e = Engine(frontier_capacity=16, set_growth=1 << 24)
    launches = []
    for g in range(0, len(pages), 3):
        for k in range(3):
            e.telegram_submit(k, pages[g + k], TANDEM)
        for k in range(3):
            r = e.telegram_wait(k, copy=True)
            a = (g + k) * 100
            lo, hi = int(first.link_off[a]), int(first.link_off[a + 100])
            assert np.array_equal(r.links, first.links[lo:hi]), f"page {g + k}: links"
            assert np.array_equal(r.link_off, first.link_off[a:a + 101] - lo), f"page {g + k}: link_off"
            assert np.array_equal(r.status, first.status[a:a + 100]), f"page {g + k}: status"
            assert r.n_new == int((r.links["flags"] & abi.LF_NEW != 0).sum())
            launches.append(r.gpu_launches)
            e.release(k)
    fl = first.links[: int(first.link_off[30_000])]
    new = fl[fl["flags"] & abi.LF_NEW != 0]
    assert np.array_equal(e.frontier_export(), new["name"]), "export order"
    assert launches[0] > 1, "the first page cannot fit 16 keys: it must take the fallback"
    assert launches.count(1) > len(launches) // 2, "most pages fit and stay on the one-launch path"
    assert e.set_info(abi.SET_FRONTIER)["grows"] >= 3
    e.close()


def _names(ids):
    k = np.zeros((len(ids), 32), np.uint8)
    k[:, 0] = ord("k")
    for d in range(8):
        k[:, 8 - d] = ord("0") + (ids // 10 ** d) % 10
    return k


def test_host_keys_grow_the_frontier():
    rng = np.random.default_rng(7)
    ids = rng.integers(0, 600_000, 1_000_000)
    _, first_at = np.unique(ids, return_index=True)
    want_new = np.zeros(len(ids), np.uint8)
    want_new[first_at] = 1
    e = Engine(frontier_capacity=16, set_growth=1 << 24)
    got = np.concatenate([e.frontier_insert(_names(ids[a:a + 250_000])) for a in range(0, len(ids), 250_000)])
    assert np.array_equal(got, want_new)
    assert np.array_equal(e.frontier_export(), _names(ids[np.sort(first_at)]))
    info = e.set_info(abi.SET_FRONTIER)
    assert info["count"] == len(first_at) and info["grows"] >= 2
    e.close()


def test_exclusion_sets_grow_and_keep_their_stamps():
    c = Corpus(200_000, profile=3, first=9)
    plain = Oracle().telegram(c.batch, abi.RUN_LINKS, nthreads=CPUS)
    names = sorted({bytes(l["name"][: l["len"]]) for l in plain.links})
    inv, disc = names[0::7], names[3::5]
    stamps = np.array([NOW - (i % 3) * 20 * DAY for i in range(len(inv))], np.int64)  # 0, 20 or 40 days old
    o, e = Oracle(), Engine(frontier_capacity=1024, set_growth=1 << 22)
    assert e.set_info(abi.SET_INVALID) == dict(count=0, capacity=0, table_slots=0, grows=0)
    for x in (o, e):
        for a in range(0, len(inv), 5000):  # several adds, the set grows between them
            x.set_add(abi.SET_INVALID, names_to_keys32(inv[a:a + 5000]), stamps[a:a + 5000])
        x.set_add(abi.SET_DISCOVERED, names_to_keys32(disc))
        x.set_now(NOW)
    for which, n in ((abi.SET_INVALID, len(inv)), (abi.SET_DISCOVERED, len(disc))):
        info = e.set_info(which)
        assert n > 1024 and info["count"] == e.set_size(which) == n and info["grows"] > 0, which
    flags = TANDEM | abi.RUN_SKIP_INVALID
    ro = o.telegram(c.batch, flags, nthreads=CPUS)
    e.telegram_submit(2, c.batch, flags)
    rg = e.telegram_wait(2, copy=True)
    assert_results_equal(ro, rg, flags)
    assert (rg.links["flags"] & abi.LF_INVALID).sum() > 0
    # at NOW the 40-day marks have expired (those channels are edges); 15 days earlier they had not: the stamps moved
    # with the set when it grew
    for now in (NOW, NOW - 15 * DAY):
        rows_o, rows_g = o.pending_edges(now), e.pending_edges(2, now)
        assert np.array_equal(rows_o, rows_g) and len(rows_g) == rg.n_new, now
        cached = int((rows_g["status"] == abi.EDGE_INVALID_CACHED).sum())
        assert (cached == 0) if now == NOW else (cached > 0)
    e.release(2)
    e.close()


def test_growth_limit(bulk):
    c, want, exports = bulk
    p0, p1 = _parts(c)[:2]
    n0, n1 = len(exports[0]), len(exports[1])
    e = Engine(frontier_capacity=64, set_growth=n1 - 1)
    assert_results_equal(want[0], e.telegram(p0, TANDEM), TANDEM, "batch 0")
    with pytest.raises(EngineError) as ei:
        e.telegram(p1, TANDEM)
    assert ei.value.code == abi.E_CAPACITY
    assert e.set_info(abi.SET_FRONTIER)["count"] == n0
    assert np.array_equal(e.frontier_export(), exports[0])
    e.set_growth(1 << 24)
    assert_results_equal(want[1], e.telegram(p1, TANDEM), TANDEM, "batch 1 after raising the limit")
    assert np.array_equal(e.frontier_export(), exports[1])
    e.close()
    # growth off: the fixed set fails exactly as before
    f = Engine(frontier_capacity=n1 - 1)
    f.telegram(p0, TANDEM)
    with pytest.raises(EngineError) as ei:
        f.telegram(p1, TANDEM)
    assert ei.value.code == abi.E_CAPACITY
    assert np.array_equal(f.frontier_export(), exports[0])
    assert f.set_info(abi.SET_FRONTIER) == dict(count=n0, capacity=n1 - 1, table_slots=1 << (2 * (n1 - 1) - 1).bit_length(), grows=0)
    f.close()


def test_set_info_arguments():
    e = Engine(frontier_capacity=1000)
    with pytest.raises(EngineError) as ei:
        e.set_info(abi.SET_OWNED)
    assert ei.value.code == abi.E_STATE
    with pytest.raises(EngineError) as ei:
        e.set_info(7)
    assert ei.value.code == abi.E_ARG
    with pytest.raises(EngineError) as ei:
        e.set_growth(1 << 40)
    assert ei.value.code == abi.E_ARG
    e.close()


def test_single_rank_partition_grows_in_the_merge(bulk):
    c, _, exports = bulk
    e = Engine(frontier_capacity=64, set_growth=1 << 24)
    e.comm_init(Engine.comm_unique_id(), 0, 1)
    assert e.set_info(abi.SET_OWNED)["capacity"] == 64
    for p in _parts(c)[:2]:
        e.telegram(p, TANDEM, copy=False)
        e.frontier_merge()
    assert np.array_equal(e.frontier_global_export(), exports[1])
    info = e.set_info(abi.SET_OWNED)
    assert info["count"] == len(exports[1]) and info["grows"] > 0
    e.close()


def _worker(rank, world, port, n_per, q):
    import torch.distributed as dist
    from distributed_crawler_b200.frontier_merge import make_merger
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)  # carries the NCCL id only
    torch.cuda.set_device(rank)
    e = Engine(device=rank, frontier_capacity=64, set_growth=1 << 24)
    m = make_merger(e, torch.device("cuda", rank))
    for rnd in range(2):
        e.telegram(Corpus(n_per, first=(rnd * world + rank) * n_per, profile=3, nthreads=4).batch, TANDEM, copy=False)
        m.merge()
    q.put((rank, m.global_export().tobytes(), e.set_info(abi.SET_OWNED)["grows"]))
    dist.barrier()
    e.close()
    dist.destroy_process_group()


def test_two_ranks_partitions_grow_in_the_merge():
    world, n_per = 2, 100_000
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, n_per, q)) for r in range(world)]
    for p in procs:
        p.start()
    out = sorted(q.get(timeout=600) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    o = Oracle()
    for rnd in range(2):
        o.telegram(Corpus(n_per * world, first=rnd * world * n_per, profile=3).batch, TANDEM, nthreads=CPUS, copy=False)
    want = o.frontier_export().tobytes()
    for rank, exp, grows in out:
        assert exp == want, f"rank {rank}: merged set differs from the single-process oracle set"
        assert grows > 0
