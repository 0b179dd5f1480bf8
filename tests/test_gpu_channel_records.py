"""Random-walk channel records on the GPU (tgi_channel_batch): the StoreChannelData lines of the edge corpus of
tests/test_channel_rules.py equal the C restatement (tests/channel_oracle.c) and the restatement channel_rules.channel_data_line byte for byte, with and
without TGI_RUN_JSONL_DEVICE, in batches of 0, 1, 100 and one grid pass + 2 000 records, and with a grid of one CTA per
SM.  The result feeds the Dapr sinks: tgi_dapr_payloads returns the base64 of each line and the path
<prefix><url>/channel_data.jsonl, tgi_combine_add puts the lines into the open group in call order beside Telegram
posts, as the chunker sees channel and post files in one watch directory.  tgi_channel_appends refuses the result (the
local manager stores no channel data), and refused calls leave the next call's output as it was."""
import base64
import os
import subprocess
import sys

import numpy as np
import pytest

import channel_rules
from distributed_crawler_b200 import abi
from distributed_crawler_b200.corpus import Corpus
from distributed_crawler_b200.pack import pack_channels
from helpers import DEV, J, PREFIX, on_slot
from channel_oracle import ChannelOracle
from oracle.pyoracle import Oracle
from test_channel_rules import BAD_AT, BAD_KINDS, SEEDS, assert_equals_restatement, make_channel_edges, make_channels, malformed
from test_gpu_combine import Chain, same

pytestmark = pytest.mark.gpu


@pytest.fixture()
def engine():
    from distributed_crawler_b200.engine import Engine
    e = Engine()
    yield e
    e.close()


def check(e, recs, flags, label):
    """one channel batch against the oracle and the restatement; the lines read back from the device under
    TGI_RUN_JSONL_DEVICE"""
    b = pack_channels(recs)
    r = e.channel_batch(b, flags)
    ro = ChannelOracle().channel(b, flags)
    assert r.n == len(recs) and np.array_equal(r.status, ro.status), label
    assert np.array_equal(r.line_off, ro.line_off), label
    if flags & DEV:
        assert r.jsonl_len == int(ro.line_off[-1]) and (r.jsonl_on_device or not r.jsonl_len), label
        r.jsonl = np.frombuffer(e.read_jsonl(r.slot, 0, r.jsonl_len), np.uint8) if r.jsonl_len else np.zeros(0, np.uint8)
    assert np.array_equal(r.jsonl, ro.jsonl), label
    assert_equals_restatement(r, recs, label)
    return r


@pytest.mark.parametrize("flags", [J, J | DEV])
@pytest.mark.parametrize("seed", SEEDS)
def test_edges_on_the_gpu(engine, seed, flags):
    r = check(engine, make_channel_edges(seed), flags, f"seed {seed}, flags {flags:#x}")
    assert r.gpu_launches >= 2


@pytest.mark.parametrize("flags", [J, J | DEV])
def test_batch_sizes(engine, flags):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    per_pass = sms * 1024  # SMs x 128 CTAs of 8 warps: from here on a warp's second record
    edges = make_channel_edges(2)
    for n in (0, 1, 100):
        check(engine, (edges * 2)[:n], flags, f"{n} records")
    recs = make_channels(per_pass + 2000, seed=9)
    at = per_pass - len(edges) // 2
    recs[at:at + len(edges)] = edges  # edge records on both sides of the pass boundary
    recs[:50], recs[-50:] = edges[:50], edges[-50:]
    check(engine, recs, flags, "one grid pass + 2 000")


def test_edges_with_a_grid_of_one_cta_per_sm():
    """TGI_GRID_MULT=1 (read once per process, hence a child process): the edge batch takes many passes of the loop"""
    code = (
        "import sys; sys.path.insert(0, 'tests')\n"
        "from distributed_crawler_b200 import abi\n"
        "from distributed_crawler_b200.engine import Engine\n"
        "import test_gpu_channel_records as t, test_channel_rules as cr\n"
        "e = Engine()\n"
        "for seed in cr.SEEDS:\n"
        "    for flags in (abi.RUN_JSONL, abi.RUN_JSONL | abi.RUN_JSONL_DEVICE):\n"
        "        t.check(e, cr.make_channel_edges(seed) * 20, flags, 'grid of one CTA per SM, seed %d' % seed)\n"
        "e.close()\n"
        "print('ok')\n")
    env = dict(os.environ, TGI_GRID_MULT="1")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and "ok" in p.stdout, p.stderr[-3000:]


@pytest.mark.parametrize("flags", [J, J | DEV])
def test_dapr_payloads(engine, flags):
    """StoreChannelData outside combine mode: Data = base64 of the line, path = <prefix><p.URL>/channel_data.jsonl"""
    for recs in (make_channel_edges(1), make_channels(70_000, seed=4)):
        b = pack_channels(recs)
        r = engine.channel_batch(b, flags)
        p = engine.dapr_payloads(r.slot, PREFIX)
        lines = [channel_rules.channel_data_line(c) for c in recs]
        assert p.n == len(recs)
        for i, (c, line) in enumerate(zip(recs, lines)):
            assert p.data(i) == base64.b64encode(line), i
            assert p.path(i) == PREFIX + bytes(c.url) + b"/channel_data.jsonl", i
        calls = []
        from distributed_crawler_b200 import sink
        assert sink.store_posts_dapr(lambda *a: calls.append(a), p, "storage", "key") == len(recs)
        assert calls[0] == ("storage", "create", base64.b64encode(lines[0]),
                            {"key": PREFIX + bytes(recs[0].url) + b"/channel_data.jsonl", "operation": "append"})
    r = engine.channel_batch(pack_channels([]), flags)
    p = engine.dapr_payloads(r.slot, PREFIX)
    assert p.n == 0 and p.data_len == 0 and p.path_len == 0


@pytest.mark.parametrize("trigger,hard_cap", [(3000, 5000), (60_000, 90_000), (1, 2500)])
def test_combine_with_telegram_posts(engine, trigger, hard_cap):
    """channel results and Telegram post results through one combiner, in call order: the chunker's blobs over the
    same files in arrival order"""
    e = engine
    e.combine_open(trigger, hard_cap, PREFIX)
    chain = Chain(trigger, hard_cap)
    edges = make_channel_edges(3)
    plan = [("tg", 100, J), ("ch", edges[:40], J), ("ch", edges[40:], J | DEV), ("tg", 2000, J | DEV),
            ("ch", make_channels(3000, 5), J), ("tg", 100, J), ("ch", edges[:1], J | DEV), ("ch", [], J)]
    first, ns = 11, 1_700_000_000_000_000_000
    for k, (kind, what, flags) in enumerate(plan):
        if kind == "tg":
            c = Corpus(what, profile=2, first=first)
            first += what
            ro = Oracle().telegram(c.batch, J)
            _, got = on_slot(e, c.batch, flags, False, k % 3, lambda s: e.combine_add(s, ns + k))
            lines = [ro.line(i) for i in range(ro.n)]
        else:
            r = e.channel_batch(pack_channels(what), flags)
            got = e.combine_add(r.slot, ns + k)
            lines = [channel_rules.channel_data_line(c) for c in what]
        same(got, chain.add(lines, ns + k), f"call {k} ({kind})")
        assert (got.open_lines, got.open_bytes) == (len(chain.files), chain.size)
    got = e.combine_flush(ns)
    same(got, (chain.flush(ns), []), "flush")
    chain.check_whole_stream()


def test_channel_appends_refuses_a_channel_result(engine):
    from distributed_crawler_b200.engine import EngineError
    r = engine.channel_batch(pack_channels(make_channels(10, 1)))
    with pytest.raises(EngineError) as ei:
        engine.channel_appends(r.slot)
    assert ei.value.code == abi.E_STATE and "channel data" in str(ei.value)
    engine.dapr_payloads(r.slot, PREFIX)  # the result itself stays readable


def test_rejected_calls_change_nothing(engine):
    """malformed string ranges (checked on the host for a small batch, on the device for one of 70 000 records) and run
    flags other than JSONL / JSONL_DEVICE are TGI_E_ARG, naming the record, and the next call's output is unchanged"""
    from distributed_crawler_b200.engine import EngineError
    e = engine
    good = pack_channels(make_channels(50, seed=77))
    before = e.channel_batch(good)
    assert_equals_restatement(before, make_channels(50, seed=77), "before")

    def rejected(batch, flags=J, *words):
        with pytest.raises(EngineError) as ei:
            e.channel_batch(batch, flags)
        assert ei.value.code == abi.E_ARG and all(w in str(ei.value) for w in words), str(ei.value)
        after = e.channel_batch(good)
        assert np.array_equal(after.jsonl, before.jsonl) and np.array_equal(after.line_off, before.line_off)
        p = e.dapr_payloads(after.slot, PREFIX)
        assert p.data(0) == base64.b64encode(before.line(0))

    for kind in BAD_KINDS:
        for at in BAD_AT.values():
            b, i = malformed(kind, at)
            rejected(b, J, "record %d" % i)
    for kind in ("past_end", "wraps", "too_long"):  # above the host's limit: the device check names the lowest bad record
        b, i = malformed(kind, 68_000, n=70_000)
        r = b.recs
        r[69_500] = r[68_000]
        rejected(b, J | DEV, "record 68000")
    for flags in (abi.RUN_LINKS, abi.RUN_FRONTIER, abi.RUN_NO_D2H, J | abi.RUN_LINKS, J | abi.RUN_SKIP_SELF, 0x100):
        rejected(good, flags, "run flags")
    rejected(good, DEV, "TGI_RUN_JSONL_DEVICE without TGI_RUN_JSONL")
