"""Combine mode on the device (tgi_combine_open / add / flush) against a restatement of the reference's chain:
StorePost writes one temp file per post in arrival order (state/daprstate.go:1117-1138), Chunker.processBatches groups
them (chunk/main.go:292-345), combineFiles concatenates each group (:386-421) and UploadCombinedFile sends its
base64.StdEncoding with the path <prefix>combined-posts/combined_<ns>.jsonl (daprstate.go:3734-3777, :2689-2698).
The lines are the oracle's."""
import base64
import ctypes as C
import os

import pytest

from distributed_crawler_b200 import abi, sink
from distributed_crawler_b200.corpus import Corpus
from distributed_crawler_b200.engine import Engine, EngineError, lib
from helpers import DEV, J, JL, PREFIX, edge_batch, on_slot
from oracle.pyoracle import Oracle
from test_sink import process_batches
from yt_corpus import make_youtube

pytestmark = pytest.mark.gpu


class Chain:
    """the reference's combine chain, one post (file) at a time in arrival order"""

    def __init__(self, trigger, hard_cap, prefix=PREFIX):
        self.trigger, self.hard_cap, self.prefix = trigger, hard_cap, prefix
        self.files, self.size, self.last_ns = [], 0, None
        self.streams = [[]]  # every post's line in arrival order, for processBatches; a flush ends a stream
        self.blob_lines = []  # the lines of every blob uploaded so far

    def _close(self, ns, out):
        if not self.files:
            return
        ns = ns if self.last_ns is None or ns > self.last_ns else self.last_ns + 1
        self.last_ns = ns
        data = b"".join(self.files)
        out.append(dict(data=base64.b64encode(data), path=self.prefix + b"combined-posts/combined_%d.jsonl" % ns,
                        n_lines=len(self.files), raw_bytes=len(data), unix_nano=ns))
        self.blob_lines.append(self.files)
        self.files, self.size = [], 0

    def add(self, lines, ns):
        out, dropped = [], []
        for i, line in enumerate(lines):
            if not line:  # no post: no file
                continue
            self.streams[-1].append(line)
            if len(line) > self.hard_cap:  # :316-322
                dropped.append(i)
                continue
            if self.size > 0 and self.size + len(line) > self.hard_cap:  # :324-327
                self._close(ns, out)
            self.files.append(line)
            self.size += len(line)
            if self.size >= self.trigger:  # :334-337
                self._close(ns, out)
        return out, dropped

    def flush(self, ns):
        out = []
        self._close(ns, out)
        self.streams.append([])
        return out

    def check_whole_stream(self):
        """the blobs so far are processBatches over each stream between flushes, the last one flushed"""
        want = []
        for s in self.streams:
            want += [[s[i] for i in b] for b in process_batches([len(x) for x in s], self.trigger, self.hard_cap)]
        assert self.blob_lines == want


def same(got, want, label=""):
    blobs, dropped = want
    assert got.n_blobs == len(blobs), f"{label}: {got.n_blobs} blobs, want {len(blobs)}"
    for j, w in enumerate(blobs):
        assert got.blob(j) == w["data"], f"{label}: blob {j} data differs"
        assert got.path(j) == w["path"], f"{label}: blob {j} path {got.path(j)!r}"
        for k in ("n_lines", "raw_bytes", "unix_nano"):
            assert got.blobs[j][k] == w[k], f"{label}: blob {j} {k}"
    assert list(got.dropped) == dropped, label


def lines_of(ro):
    return [ro.line(i) for i in range(ro.n)]


def open_state(chain):
    return len(chain.files), chain.size


def add(e, chain, batch, flags, slot, ns, yt=False, ro=None):
    """one batch on `slot`, tgi_combine_add, release; checks the closed blobs and the open group against the chain"""
    ro = ro or (Oracle().youtube(batch, J) if yt else Oracle().telegram(batch, J))
    r, got = on_slot(e, batch, flags, yt, slot, lambda s: e.combine_add(s, ns))
    same(got, chain.add(lines_of(ro), ns), f"slot {slot} flags {flags:#x} n {ro.n}")
    assert (got.open_lines, got.open_bytes) == open_state(chain)
    return r, got


def flush(e, chain, ns):
    got = e.combine_flush(ns)
    same(got, (chain.flush(ns), []), "flush")
    assert got.open_lines == 0 and got.open_bytes == 0
    return got


@pytest.mark.parametrize("trigger,hard_cap", [(3000, 5000), (200_000, 300_000), (9000, 4000), (1, 2500)])
def test_telegram_pages_and_bulk_on_three_slots(trigger, hard_cap):
    e = Engine()
    e.combine_open(trigger, hard_cap, PREFIX)
    ch = Chain(trigger, hard_cap)
    plan = [(100, JL), (1000, JL | DEV), (100, JL | abi.RUN_NO_D2H), (20000, JL | DEV), (100, J), (1000, JL),
            (20000, JL | abi.RUN_NO_D2H), (100, J | DEV), (5000, JL)]
    first, closed = 7, 0
    for k, (n, flags) in enumerate(plan):
        c = Corpus(n, profile=2, first=first)
        first += n
        r, got = add(e, ch, c.batch, flags, k % 3, 1_700_000_000_000_000_000 + k)
        if not flags & abi.RUN_NO_D2H and n != 5000:
            assert (r.gpu_launches == 1) == (n <= 1000), "pages take the one-launch path, 20 000 messages the bulk one"
        closed += got.n_blobs
    flush(e, ch, 1_700_000_000_000_000_000)
    ch.check_whole_stream()
    assert closed >= 2
    e.close()


def test_youtube_bulk_and_pages():
    batch, _, _ = make_youtube(3000, seed=21)
    e = Engine()
    e.combine_open(50_000, 80_000, PREFIX)
    ch = Chain(50_000, 80_000)
    add(e, ch, batch, J | abi.RUN_LINKS, 0, 5, yt=True)
    for k in range(0, 500, 50):
        add(e, ch, batch.slice(k, k + 50), J | DEV if k % 100 else J, k // 50 % 3, 6 + k, yt=True)
    flush(e, ch, 1)
    ch.check_whole_stream()
    e.close()


@pytest.mark.parametrize("trigger,hard_cap", [(10**9, 3000), (7000, 2500), (4001, 20000), (10**9, 10**9)])
def test_pending_phases_and_segment_boundaries(trigger, hard_cap):
    """the edge corpus (lines of every length residue mod 3 and every start alignment, 2-20 KB lines, records without a
    line) cut into results of every size from 1 to 23 records: the open group's pending bytes meet every segment
    boundary in every phase, and lines above the cap split runs"""
    batch = edge_batch()
    cfg = dict(min_post_date=1_600_000_000, crawl_label=b'c"l')
    e = Engine(**cfg)
    e.combine_open(trigger, hard_cap, PREFIX)
    ch = Chain(trigger, hard_cap)
    ro = Oracle(**cfg).telegram(batch, J)
    phases, k, a = set(), 0, 0
    while a < ro.n:
        b = min(ro.n, a + 1 + k % 23)
        part = batch.slice(a, b)
        rp = Oracle(**cfg).telegram(part, J)
        assert lines_of(rp) == [ro.line(i) for i in range(a, b)]
        phases.add(ch.size % 3)
        flags = (J, J | DEV, J | abi.RUN_NO_D2H)[k % 3]
        with pytest.MonkeyPatch.context() as mp:
            if k % 4 == 3:
                mp.setenv("TGI_NO_PAGE", "1")  # the same kind of result from the bulk pipeline
            add(e, ch, part, flags, k % 3, 42, ro=rp)
        a, k = b, k + 1
    flush(e, ch, 42)
    ch.check_whole_stream()
    assert phases == {0, 1, 2} or trigger < 10**9
    e.close()


def test_default_trigger_and_cap():
    """170 / 200 MiB: a profile-2 bulk batch that closes at least two blobs, then a stream of pages that closes one
    only after many calls"""
    o = Oracle()
    e = Engine(max_records=200_000)
    e.combine_open(sink.TRIGGER_DEFAULT, sink.HARD_CAP_DEFAULT, PREFIX)
    ch = Chain(sink.TRIGGER_DEFAULT, sink.HARD_CAP_DEFAULT)
    c = Corpus(200_000, profile=2, first=1)
    ro = o.telegram(c.batch, J, nthreads=os.cpu_count() or 1)
    assert int(ro.line_off[-1]) > 2 * sink.TRIGGER_DEFAULT
    _, got = add(e, ch, c.batch, J | DEV, 0, 10, ro=ro)
    assert got.n_blobs >= 2
    del ro, c
    flush(e, ch, 10)  # the page stream starts a group of its own
    calls, closed_at = 0, None
    while closed_at is None and calls < 200:
        p = Corpus(1000, profile=2, first=300_000 + 1000 * calls)
        _, got = add(e, ch, p.batch, JL, calls % 3, 11 + calls)
        calls += 1
        if got.n_blobs:
            closed_at = calls
    assert closed_at is not None and closed_at > 20
    flush(e, ch, 0)
    ch.check_whole_stream()
    e.close()


def test_flush_empty_and_nonempty():
    e = Engine()
    e.combine_open(10**6, 2 * 10**6, PREFIX)
    got = e.combine_flush(5)
    assert got.n_blobs == 0
    ch = Chain(10**6, 2 * 10**6)
    add(e, ch, Corpus(100, profile=2, first=3).batch, J, 1, 7)
    flush(e, ch, 8)
    assert e.combine_flush(9).n_blobs == 0
    e.close()


def test_slot_reused_right_after_add():
    """the open group holds none of the slot's bytes: another batch on the same slot right away changes nothing"""
    e = Engine()
    e.combine_open(10**6, 2 * 10**6, PREFIX)
    ch = Chain(10**6, 2 * 10**6)
    for k in range(4):
        add(e, ch, Corpus(1000, profile=2, first=1000 * k).batch, J | DEV, 0, 100 + k)
        e.telegram_submit(0, Corpus(4000, profile=3, first=90_000 + k).batch, JL | DEV)  # overwrites the slot's lines
        e.telegram_wait(0)
        e.release(0)
    flush(e, ch, 1)
    e.close()


def test_names_increase_within_one_call():
    e = Engine()
    e.combine_open(1, 10**6, b"")
    ch = Chain(1, 10**6, b"")
    _, got = add(e, ch, Corpus(300, profile=2, first=1).batch, J, 2, 1000)
    ns = [b["unix_nano"] for b in got.blobs]
    assert len(ns) > 100 and ns == list(range(1000, 1000 + len(ns)))
    _, got = add(e, ch, Corpus(10, profile=2, first=400).batch, J, 2, 5)  # an earlier clock: names still increase
    assert got.blobs[0]["unix_nano"] == ns[-1] + 1
    e.close()


def test_upload_combined_dapr():
    e = Engine()
    e.combine_open(40_000, 60_000, PREFIX)
    ch = Chain(40_000, 60_000)
    _, got = add(e, ch, Corpus(300, profile=2, first=9).batch, J, 0, 77)
    want = []
    for j, b in enumerate(ch.blob_lines):  # UploadCombinedFile: base64 of the whole file, one InvokeBinding
        want.append(("telegramstorage", "create", base64.b64encode(b"".join(b)),
                     {"blobName": PREFIX + b"combined-posts/combined_%d.jsonl" % (77 + j), "operation": "append"}))
    reqs = []
    assert sink.upload_combined_dapr(lambda *r: reqs.append(r), got, "telegramstorage", "blobName") == got.n_blobs > 0
    assert reqs == want
    e.close()


def _add(e, slot):
    out = abi.CombinedC()
    return lib().tgi_combine_add(e.h, slot, 1, C.byref(out))


def test_error_codes():
    from gm_corpus import make_generic
    e = Engine()
    c = Corpus(200, profile=2, first=3)
    e.telegram_submit(0, c.batch, J)
    e.telegram_wait(0)
    assert _add(e, 0) == abi.E_STATE  # no combiner is open
    out = abi.CombinedC()
    assert lib().tgi_combine_flush(e.h, 1, C.byref(out)) == abi.E_STATE
    e.combine_open(10**6, 2 * 10**6, PREFIX)
    assert _add(e, 1) == abi.E_STATE  # the slot holds no result
    assert _add(e, -1) == abi.E_ARG
    assert _add(e, 0) == abi.OK
    e.release(0)
    with pytest.raises(EngineError) as ei:  # reconfigure while the open group holds lines
        e.combine_open(10, 20, PREFIX)
    assert ei.value.code == abi.E_STATE
    e.telegram_submit(1, c.batch, abi.RUN_LINKS)
    e.telegram_wait(1)
    assert _add(e, 1) == abi.E_STATE  # no lines
    e.release(1)
    g, _ = make_generic(50, seed=4)
    d = g.descriptor()
    r = abi.ResultC()
    assert lib().tgi_generic_batch(e.h, C.byref(d), J, C.byref(r)) == abi.OK
    assert _add(e, r.slot) == abi.E_STATE  # SavePost has no Dapr implementation
    lib().tgi_result_release(e.h, r.slot)
    assert e.combine_flush(3).n_blobs == 1
    e.combine_open(10, 20, PREFIX)  # an empty open group may be reconfigured
    e.close()
