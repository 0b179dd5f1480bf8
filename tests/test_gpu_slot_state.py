"""A staging slot's resident batch and last result, as every reader and every resident run sees them: a slot's resident
batch is the batch of its last successful upload; its last result lives from a successful job until the next job is
claimed on the slot; calls that find neither get TGI_E_STATE."""
import ctypes as C

import numpy as np
import pytest

from distributed_crawler_b200 import abi
from distributed_crawler_b200.corpus import Corpus
from distributed_crawler_b200.engine import Engine, EngineError, lib
from helpers import ALL, assert_results_equal
from oracle.pyoracle import Oracle
from yt_corpus import make_youtube

pytestmark = pytest.mark.gpu

NOW = 1_760_000_000
PREFIX = b"root/crawl/exec/"
LF = abi.RUN_LINKS | abi.RUN_FRONTIER
READERS = ("read_rows", "read_jsonl", "pending_edges", "dapr_payloads")
NO_RESULT = dict.fromkeys(READERS, abi.E_STATE)


def reader_codes(e, slot):
    """the return codes of the four readers on `slot`, each asked for as little as it can be asked for"""
    buf = np.zeros(16, np.uint8)
    n = C.c_uint64()
    pay = abi.DaprPayloadsC()
    return {"read_rows": lib().tgi_result_read_rows(e.h, slot, abi.ROWS_STATUS, 0, 1, buf.ctypes.data),
            "read_jsonl": lib().tgi_result_read_jsonl(e.h, slot, 0, 0, buf.ctypes.data),
            "pending_edges": lib().tgi_pending_edges(e.h, slot, NOW, None, 0, C.byref(n)),
            "dapr_payloads": lib().tgi_dapr_payloads(e.h, slot, PREFIX, len(PREFIX), C.byref(pay))}


def run_resident_code(e, slot, flags=abi.RUN_LINKS):
    r = abi.ResultC()
    rc = lib().tgi_telegram_run_resident(e.h, slot, flags, C.byref(r))
    if rc == abi.OK:
        e.release(slot)
    return rc


def test_fresh_slots_hold_no_result():
    e = Engine()
    for slot in range(abi.SLOTS):
        assert reader_codes(e, slot) == NO_RESULT, slot
    e.close()


@pytest.mark.parametrize("n", [300, 12_000])  # the page kernel and the multi-kernel pipeline
def test_failed_job_leaves_no_result(n):
    c = Corpus(n, profile=2, first=41)
    e = Engine(max_out_bytes=10_000)  # below the batch's JSONL; a batch without TGI_RUN_JSONL is not limited
    e.telegram_submit(1, c.batch, LF)
    assert (e.telegram_wait(1).gpu_launches == 1) == (n == 300)
    e.release(1)
    # the same batch again, so that no buffer changes size: only the readers' answer tells the failure apart
    e.telegram_submit(1, c.batch, LF | abi.RUN_JSONL)
    with pytest.raises(EngineError) as ei:
        e.telegram_wait(1)
    assert ei.value.code == abi.E_CAPACITY
    assert reader_codes(e, 1) == NO_RESULT
    # the next successful batch on the slot is readable again
    e.frontier_clear()
    e.telegram_submit(1, c.batch, LF)
    rg = e.telegram_wait(1, copy=True)
    o = Oracle()
    ro = o.telegram(c.batch, LF)
    assert_results_equal(ro, rg, LF)
    assert np.array_equal(e.read_rows(1, abi.ROWS_STATUS, 0, n), ro.status)
    assert np.array_equal(e.read_rows(1, abi.ROWS_LINK_OFF, 0, n + 1), ro.link_off)
    assert np.array_equal(e.read_rows(1, abi.ROWS_LINKS, 0, len(ro.links)), ro.links)
    assert np.array_equal(e.pending_edges(1, NOW), o.pending_edges(NOW)) and ro.n_new > 0
    e.release(1)
    e.close()


def test_upload_only_job_leaves_no_result():
    c = Corpus(300, profile=3, first=8)
    e = Engine()
    e.telegram_submit(0, c.batch, ALL)
    e.telegram_wait(0)
    e.release(0)
    assert reader_codes(e, 0) == dict.fromkeys(READERS, abi.OK)
    e.telegram_upload(0, c.batch)  # the same batch: no buffer changes size
    assert reader_codes(e, 0) == NO_RESULT
    e.frontier_clear()
    rg = e.telegram_run_resident(0, ALL, copy=True)
    ro = Oracle().telegram(c.batch, ALL)
    assert_results_equal(ro, rg, ALL)
    assert e.read_jsonl(0, 0, rg.jsonl_len) == ro.jsonl.tobytes()
    e.close()


def test_resident_run_of_the_wrong_kind_is_refused():
    yb, _, _ = make_youtube(50, seed=3)
    e = Engine()
    e.youtube_upload(0, yb)
    assert run_resident_code(e, 0) == abi.E_STATE
    flags = abi.RUN_JSONL | abi.RUN_LINKS
    rg = e.youtube_run_resident(0, flags, copy=True)  # the YouTube batch is still resident
    assert_results_equal(Oracle().youtube(yb, flags), rg, flags)
    e.close()


def test_rejected_upload_drops_the_resident_batch():
    c = Corpus(200, profile=2, first=9)
    bad = c.batch.slice(0, c.batch.n)
    bad.recs["chan_idx"][0] = len(bad.chans)  # refused by the host range check, before any copy
    e = Engine()
    e.telegram_upload(1, c.batch)
    with pytest.raises(EngineError) as ei:
        e.telegram_upload(1, bad)
    assert ei.value.code == abi.E_ARG
    assert run_resident_code(e, 1) == abi.E_STATE
    e.telegram_upload(1, c.batch)
    rg = e.telegram_run_resident(1, ALL, copy=True)
    assert_results_equal(Oracle().telegram(c.batch, ALL), rg, ALL)
    e.close()
