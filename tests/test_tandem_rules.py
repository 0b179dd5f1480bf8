"""CPU tests: tests/tandem_rules.py, the restatement tgi_state_pending_edges is checked against, on the reference's tandem
vectors and the cases the per-page rules turn on; the C layout of its output; and agreement with the oracle's
tgi_pending_edges where the two rules coincide (one page, a fresh dedup set)."""
import ctypes as C
import os
import random
import subprocess
import tempfile

import numpy as np

import tandem_rules as tr
from discover_rules import ST_EMITTED, ST_FAILED, ST_NOLINE, ST_SKIPPED, page_id
from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import names_to_keys32
from distributed_crawler_b200.pack import Channel, pack_telegram
from go_rules import filter_username
from helpers import msg
from oracle.pyoracle import Oracle
from state_rules import GoState

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOW = 1_760_000_000
M, T, U, P = (abi.SRC_NAMES.index(s) for s in ("mention", "text_url", "url", "plaintext"))
TANDEM = abi.RUN_LINKS | abi.RUN_FRONTIER | abi.RUN_FILTER | abi.RUN_SKIP_SELF | abi.RUN_SKIP_INVALID


def tandem(*owners, seed=9):
    """a state of owner pages (url, depth, sequenceId) and a Tandem over it"""
    go = GoState()
    go.set_state([(0, [{"id": b"p%d" % k, "url": u, "depth": 2, "sequenceId": b"seq%d" % k} for k, u in enumerate(owners)])])
    return tr.Tandem(go, seed)


def names(edges):
    return [e["destination"] for e in edges]


def test_struct_layouts_match_the_header():
    probe = r'''
#include <stdio.h>
#include <stddef.h>
#include "tgingest.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(tgi_state_edge), offsetof(tgi_state_edge, record),
         offsetof(tgi_state_edge, batch), offsetof(tgi_state_edge, status), sizeof(tgi_state_edge_batch),
         offsetof(tgi_state_edge_batch, span), offsetof(tgi_state_edge_batch, n_edges), sizeof(tgi_state_edges_t),
         offsetof(tgi_state_edges_t, span_batch), offsetof(tgi_state_edges_t, gpu_launches));
  printf("%u\n", TGI_STATE_NO_BATCH);
  return 0;
}'''
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "p.c")
        open(src, "w").write(probe)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", os.path.join(d, "p")])
        got = list(map(int, subprocess.check_output([os.path.join(d, "p")]).decode().split()))
    E, B, O = abi.STATE_EDGE, abi.STATE_EDGE_BATCH, abi.StateEdgesC
    assert got == [48, E.fields["record"][1], E.fields["batch"][1], E.fields["status"][1], 48, B.fields["span"][1],
                   B.fields["n_edges"][1], 56, O.span_batch.offset, O.gpu_launches.offset, abi.STATE_NO_BATCH]
    assert (E.itemsize, B.itemsize, C.sizeof(O)) == (48, 48, 56)


def test_batch_ids_are_v4_uuids_apart_from_page_ids():
    ids = [tr.batch_id(s, n) for s in (0, 7, 2**64 - 1) for n in (0, 1, 2**32, 2**64 - 1)]
    assert len(set(ids)) == len(ids)
    for i in ids:
        assert len(i) == 36 and i[14:15] == b"4" and i[19:20] in b"89ab" and i.count(b"-") == 4
    assert all(tr.batch_id(7, n) != page_id(7, n) for n in range(100))
    assert tr.batch_id(7, 3) == tr.batch_id(7, 3)


def oracle_links(t):
    """a reference vector's message through the oracle's link extraction: [(name, source)] of its one record"""
    b = pack_telegram([msg("messageText", t["text"], [tuple(e) for e in t["entities"]])],
                      [Channel(name=t["owner_url"], username=t["owner_url"])])
    r = Oracle().telegram(b, abi.RUN_LINKS)
    return [(n, abi.SRC_NAMES.index(s)) for n, s in r.record_links(0)]


def test_reference_tandem_vectors(vectors):
    """crawl/runner_tandem_test.go: WithEdges (one batch, two edges), NoEdges (no batch: the walkback),
    InvalidChannelSkipped (IsInvalidChannel drops the only edge: no batch)"""
    for name, t in vectors["tandem"].items():
        x = tandem(t["owner_url"].encode())
        for inv in t.get("invalid", []):
            x.invalid[inv.encode()] = 0
        batch, edges = x.page(b"p0", [ST_EMITTED], [oracle_links(t)], 1, NOW)
        assert [e.decode() for e in names(edges)] == t["expected_edges"], name
        assert (batch is None) == (not t["expected_edges"]), name
        if batch:
            assert batch["source_channel"] == t["owner_url"].encode() and batch["status"] == "closed"
            assert batch["batch_id"] == tr.batch_id(9, 0) and x.n == 1


def test_two_pages_mentioning_one_channel_get_a_batch_each():
    x = tandem(b"owner_one", b"owner_two")
    b0, e0 = x.page(b"p0", [ST_EMITTED], [[(b"shared_chan", M)]], 1, NOW)
    b1, e1 = x.page(b"p1", [ST_EMITTED], [[(b"shared_chan", U)]], 1, NOW)
    assert names(e0) == names(e1) == [b"shared_chan"]
    assert (b0["batch_id"], b1["batch_id"]) == (tr.batch_id(9, 0), tr.batch_id(9, 1))
    assert (b0["source_page_id"], b1["source_page_id"], b1["source_depth"], b1["sequence_id"]) == (b"p0", b"p1", 2, b"seq1")
    assert e1[0]["source_type"] == U


def test_first_record_and_source_win_within_a_page():
    x = tandem(b"owner_one")
    _, edges = x.page(b"p0", [ST_EMITTED, ST_EMITTED], [[(b"other_chan", P), (b"dup_chan", T)],
                                                        [(b"dup_chan", M), (b"dup_chan", U), (b"third_chan", M)]], 2, NOW)
    assert [(e["destination"], e["record"], e["source_type"]) for e in edges] == [
        (b"other_chan", 0, P), (b"dup_chan", 0, T), (b"third_chan", 1, M)]


def test_self_compare_is_byte_for_byte():
    x = tandem(b"Owner_Chan")
    _, edges = x.page(b"p0", [ST_EMITTED], [[(b"owner_chan", M), (b"Owner_Chan", M)]], 1, NOW)
    assert names(edges) == [b"owner_chan"]  # the lower-cased link name is not the mixed-case URL


def test_invalid_ttl_boundaries():
    x = tandem(b"owner_one")
    stamps = {b"expired_one": NOW - tr.TTL - 1, b"expired_two": NOW - tr.TTL, b"live_chan": NOW - tr.TTL + 1,
              b"forever_chan": 0}
    x.invalid.update(stamps)
    _, edges = x.page(b"p0", [ST_EMITTED], [[(n, M) for n in stamps]], 1, NOW)
    assert names(edges) == [b"expired_one", b"expired_two"]


def test_every_filter_username_reason_drops_the_name():
    bad = {b"abcd": "too_short", b"a" * 33: "too_long", b"1chan_name": "invalid_start_char", b"chan_name_": "ends_with_underscore",
           b"chan-name": "invalid_char", b"helper_bot": "bot_suffix", b"helperBOT": "bot_suffix"}
    x = tandem(b"owner_one")
    for nm, why in bad.items():
        assert filter_username(nm) == why
    _, edges = x.page(b"p0", [ST_EMITTED], [[(n, M) for n in bad] + [(b"fine_name", M)]], 1, NOW)
    assert names(edges) == [b"fine_name"]


def test_statuses_and_n_done():
    x = tandem(b"owner_one")
    status = [ST_FAILED, ST_SKIPPED, ST_NOLINE, ST_EMITTED, ST_EMITTED]
    links = [[(b"failed_chan", M)], [(b"skipped_chan", M)], [(b"noline_chan", M)], [(b"emitted_chan", M)], [(b"late_chan", M)]]
    for n_done, want in ((0, []), (2, []), (3, [b"noline_chan"]), (4, [b"noline_chan", b"emitted_chan"]),
                         (5, [b"noline_chan", b"emitted_chan", b"late_chan"])):
        n0 = x.n
        batch, edges = x.page(b"p0", status, links, n_done, NOW)
        assert names(edges) == want and (batch is None) == (not want) and x.n == n0 + bool(want)
        assert [e["record"] for e in edges] == [2, 3, 4][:len(want)]


def test_discovered_names_are_duplicates():
    x = tandem(b"owner_one")
    x.discovered.add(b"known_chan")
    _, edges = x.page(b"p0", [ST_EMITTED], [[(b"known_chan", M), (b"new_chan", M)]], 1, NOW)
    assert [e["status"] for e in edges] == [tr.EDGE_DUPLICATE, tr.EDGE_PENDING]


def test_one_page_with_a_fresh_set_agrees_with_the_oracle():
    """tgi_pending_edges with a fresh dedup set and SKIP_SELF / FILTER / SKIP_INVALID on a one-channel batch keeps the
    same edges as the per-page rules: seenInBatch and the global set coincide"""
    rnd = random.Random(3)
    pool = [b"chan%03d" % k for k in range(30)] + [b"x_bot", b"abc", b"some_bot", b"trail_", b"owner_chan"]
    for trial in range(6):
        ms = []
        for k in range(40):
            nm = [rnd.choice(pool) for _ in range(rnd.choice([0, 1, 3, 5]))]
            text = " ".join(("t.me/" if rnd.random() < 0.5 else "@") + n.decode() for n in nm)
            ms.append(msg("messageText", "post %d %s" % (k, text), id=(k + 1) << 20, chat_id=-5, date=1_700_000_000,
                          panics=rnd.random() < 0.1))
        b = pack_telegram(ms, [Channel(name="owner_chan", username="owner_chan")])
        invalid = {n: NOW - rnd.choice([0, 20, 40]) * 24 * 3600 for n in rnd.sample(pool[:30], 6)}
        discovered = set(rnd.sample(pool[:30], 6))
        o = Oracle()
        o.set_add(abi.SET_INVALID, names_to_keys32(list(invalid)), np.array(list(invalid.values()), np.int64))
        o.set_add(abi.SET_DISCOVERED, names_to_keys32(sorted(discovered)))
        o.set_now(NOW)
        r = o.telegram(b, TANDEM)
        rows = o.pending_edges(NOW)
        want = [(bytes(e["destination"][:e["dest_len"]]), int(e["record"]), int(e["source_type"]), int(e["status"]))
                for e in rows]
        x = tandem(b"owner_chan")
        x.invalid, x.discovered = invalid, discovered
        links = [[(n, abi.SRC_NAMES.index(s)) for n, s in r.record_links(i)] for i in range(r.n)]
        batch, edges = x.page(b"p0", [int(s) for s in r.status], links, r.n, NOW)
        got = [(e["destination"], e["record"], e["source_type"], e["status"]) for e in edges]
        assert got == want and (batch is None) == (not want), trial
        assert want
