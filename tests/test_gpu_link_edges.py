"""Telegram link extraction at the edges of its GPU scanners (tests/tg_link_corpus.py:make_link_edges): t.me/ at every
lane offset and strip edge, names around the 32-byte cap, mention slices around the 32-byte steps, UTF-16 entity offsets
around the mapper's lanes, strips and ASCII shortcut, tight link bounds, dedup, flags and the filter — CUDA through the
C ABI vs the CPU oracle, byte equality of status, link_off, links (name, source, flags, filter reason), JSONL and the
frontier (content and order, batch after batch), on the page kernel, the bulk pipeline's JSONL instances and the
link-only instances that configs 3 and 5 run.  The CPU tests pin the oracle on the same messages with the second
restatement (tests/go_rules.py), check that the generator reaches every cell of the geometry, and that a one-unit
error in a mapped entity's start or end would change what the comparison sees."""
import random

import numpy as np
import pytest

import go_rules
from distributed_crawler_b200 import abi
from distributed_crawler_b200.engine import Engine
from distributed_crawler_b200.pack import FormattedText, Message, TextEntity, pack_telegram
from helpers import ALL, TANDEM, assert_results_equal, no_page
from oracle import pyoracle
from oracle.pyoracle import Oracle
from tg_link_corpus import (CARRIERS, CHANNELS, MIN_POST_DATE, MOVES, PAGE_MAX_RECS, SEEDS, expected,
                            link_bound, link_cells, make_link_edges, map16, mapping_cases, _table)

ST = {"emitted": abi.ST_EMITTED, "skipped": abi.ST_SKIPPED, "failed": abi.ST_FAILED}
CFG_VARIANT = dict(min_post_date=MIN_POST_DATE, tz_offset_sec=-12600, crawl_label=b'lab"<el>\xff\\')


def _seeds_in_sequence(flags, label, page, **cfg):
    """the edge batches of every seed through one engine and one oracle: the frontier's first-occurrence order is
    compared after every batch"""
    o, e = Oracle(**cfg), Engine(**cfg)
    try:
        for seed in SEEDS:
            batch, _, _ = make_link_edges(seed)
            ro, rg = o.telegram(batch, flags), e.telegram(batch, flags)
            assert_results_equal(ro, rg, flags, f"{label}, seed {seed}")
            if flags & abi.RUN_FRONTIER:
                assert np.array_equal(o.frontier_export(), e.frontier_export()), f"{label}, seed {seed}: frontier differs"
            assert (rg.gpu_launches == 1) == page, f"{label}: {rg.gpu_launches} launches"
            assert (ro.status == abi.ST_FAILED).sum() > 0 and len(ro.links) > 5000
    finally:
        e.close()
        o.close()


# ---- GPU -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("flags", [ALL, TANDEM], ids=["all", "tandem"])
def test_edges_page_kernel(flags):
    """parse_one_record<true|false, false> behind warp_map_entities, in one launch"""
    _seeds_in_sequence(flags, "page kernel", page=True)


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [ALL, TANDEM, abi.RUN_LINKS], ids=["all", "tandem", "links"])
def test_edges_bulk_pipeline(flags):
    """JSONL runs take the parse kernels' <true> instances (the link count measures the text as well), TANDEM and
    RUN_LINKS alone the <false> ones"""
    with no_page():
        _seeds_in_sequence(flags, "bulk pipeline", page=False)


@pytest.mark.gpu
@pytest.mark.parametrize("bulk", [False, True], ids=["page", "bulk"])
def test_edges_config_variant(bulk):
    """min_post_date skips records that hold links; another zone and a label that needs escaping"""
    if bulk:
        with no_page():
            _seeds_in_sequence(ALL, "bulk pipeline, config variant", page=False, **CFG_VARIANT)
    else:
        _seeds_in_sequence(ALL, "page kernel, config variant", page=True, **CFG_VARIANT)


@pytest.mark.gpu
def test_edges_above_the_page_size():
    msgs = [m for seed in SEEDS for m in make_link_edges(seed)[1]]
    batch = pack_telegram(msgs, CHANNELS)
    assert batch.n > PAGE_MAX_RECS
    for flags in (ALL, TANDEM):
        o, e = Oracle(), Engine()
        ro, rg = o.telegram(batch, flags), e.telegram(batch, flags)
        assert_results_equal(ro, rg, flags, "above the page size")
        assert np.array_equal(o.frontier_export(), e.frontier_export())
        assert rg.gpu_launches > 1
        e.close()
        o.close()


def _filter_names(rng):
    out = [b"", b"a", b"abcd", b"abcde", b"a" * 32, b"a" * 33, b"a" * 40, b"1abcde", b"_abcde", b"abcde_", b"abcdebot",
           b"abcdeBoT", b"abcde_bot", b"a" * 29 + b"bot", b"a" * 29 + b"BOT", b"a" * 30 + b"bot", b"abc\x80de", b"abc\x00de",
           b"abc/de", b"abc.de", b"abc~de", b"ab\xc3\xa9cd", b"\xc3\xa9abcd", b"abcd\xff", b"abcd\x00", b"bot", b"botbot",
           b"/abcde", b".abcde", b"~abcde", b"abcd/", b"abcd_\x80", b"_", b"Z____"]
    alpha = b"abcXYZ019_" * 4 + b"\x00\x80\xff\xc3/.~ @"
    for n in range(41):
        for k in range(4):
            body = bytes(rng.choice(alpha if k else b"abcXYZ019_") for _ in range(n))
            out.append(body)
            out.append(body[:max(n - 3, 0)] + b"bOt"[:n])
    return out


@pytest.mark.gpu
def test_filter_usernames_batches():
    """FilterUsername (tgi_filter_usernames: one warp per name, eight warps per block) against the oracle and the
    restatement, in batches of 1, 7, 8, 9 and 1000 names"""
    names = _filter_names(random.Random(7))
    want = [pyoracle.filter_username(x) for x in names]
    assert set(want) == set(abi.FU_REASONS) - {"looks_like_path"}  # every reason the rule can return
    e = Engine()
    try:
        for size in (1, 7, 8, 9, 1000):
            for a in range(0, len(names), size):
                assert e.filter_usernames(names[a:a + size]) == want[a:a + size], (size, a)
    finally:
        e.close()


# ---- CPU -------------------------------------------------------------------------------------------------------------
def _entity_map_cases(msgs):
    for m in msgs:
        if m.text is not None and m.content_type in CARRIERS:
            for e in m.text.entities:
                if e.type in ("mention", "url"):
                    yield bytes(m.text.text), e.offset, e.length


@pytest.mark.parametrize("seed", SEEDS)
def test_oracle_vs_independent_restatement(seed):
    """status and links (in order, with their source) of every edge record: the oracle against tests/go_rules.py;
    utf16OffsetToBytes of every mention / url entity: the oracle, go_rules and the corpus' table lookup"""
    batch, msgs, _ = make_link_edges(seed)
    cfgs = [({}, None)] + ([({"min_post_date": MIN_POST_DATE}, MIN_POST_DATE)] if seed == SEEDS[0] else [])
    for cfg, mpd in cfgs:
        r = Oracle(**cfg).telegram(batch, abi.RUN_LINKS)
        for i, m in enumerate(msgs):
            st, links = expected(m, mpd)
            assert r.status[i] == ST[st], (i, cfg)
            assert r.record_links(i) == links, (i, cfg)
    for t, off, ln in _entity_map_cases(msgs):
        want = go_rules.utf16_offset_to_bytes(t, off, ln)
        assert pyoracle.utf16_offset_to_bytes(t, off, ln) == want, (t[:40], off, ln)
        assert map16(_table(t), len(t), off, ln) == want, (t[:40], off, ln)


@pytest.mark.parametrize("seed", SEEDS)
def test_edges_reach_every_cell(seed):
    """lane offsets 0..15, the t of a t.me/ at bytes 507..512 and 1019..1024, names of 4 / 5 / 31 / 32 / 33 bytes (also
    across a strip edge), all three mapper branches and the ASCII shortcut's bound at -1..+2, the filter reasons links can
    reach, records whose link bound is tight, the group layouts of 32 records, and a page that fits the page arena"""
    batch, msgs, _ = make_link_edges(seed)
    cells = link_cells(msgs)
    want = {("lane", k) for k in range(16)} | {("edge", e, d) for e in (512, 1024) for d in range(-5, 1)}
    want |= {("name", n) for n in (4, 5, 31, 32, 33)} | {("name_across_strip", n) for n in (4, 5, 31, 32, 33)}
    want |= {("map", b) for b in ("ascii", "fast", "exact")} | {("ascii_stop", d) for d in (-1, 0, 1, 2)}
    assert not want - cells, sorted(want - cells)

    r = Oracle().telegram(batch, abi.RUN_LINKS)
    reasons = {abi.FU_REASONS[int(x)] for x in r.links["filter_reason"]}
    assert {"", "ends_with_underscore", "bot_suffix"} <= reasons
    assert r.links["flags"].max() & abi.LF_SELF and (r.links["src"] == 1).any()  # self links; text_url sources
    counts = np.diff(r.link_off.astype(np.int64))
    bounds = np.array([link_bound(m) for m in msgs])
    emitted = r.status == abi.ST_EMITTED
    assert (counts <= bounds).all()
    assert ((counts == bounds) & (bounds > 0) & emitted).sum() >= 150  # tight records
    assert ((counts == bounds) & (bounds > 32)).sum() >= 20
    assert bounds.sum() <= len(batch.ents) + 2 * batch.n + 1024, "the batch must fit the page kernel's link arena"
    assert batch.n <= PAGE_MAX_RECS and batch.input_bytes() <= 4 << 20

    has = np.diff(batch.ent_off.astype(np.int64)) > 0
    groups = [has[g:g + 32] for g in range(0, batch.n, 32)]
    kinds = {"all" if g.all() else "none" if not g.any() else "lane0" if g.sum() == 1 and g[0] else
             "lane31" if g.sum() == 1 and g[-1] else "alt" if len(g) == 32 and (g[::2].all() and not g[1::2].any()) else
             "mixed" for g in groups}
    assert kinds == {"all", "none", "lane0", "lane31", "alt", "mixed"}
    assert len(groups[-1]) == 16
    assert (r.status == abi.ST_FAILED).sum() > 50


def _with_entity(m, off, length):
    e = m.text.entities[0]
    return Message(content_type=m.content_type, text=FormattedText(m.text.text, [TextEntity(off, length, e.type, e.url)]),
                   channel=m.channel)


@pytest.mark.parametrize("seed", SEEDS)
def test_mapping_cases_see_one_unit_moves(seed):
    """Every UTF-16 mapping case declares which one-unit moves of its entity change the record's links or status (the
    start moved with the end fixed, the end moved); on the oracle each declared move changes them and no other does.
    Most cases of both kinds see a start move in one direction and an end move in one direction, so a GPU off-by-one
    in warp_utf16_to_bytes or the shortcut shows up in the comparison instead of vanishing in an unanchored regex."""
    cases = mapping_cases(seed)
    base = [_with_entity(m, m.text.entities[0].offset, m.text.entities[0].length) for m, _, _ in cases]
    mv = []
    for m in base:
        e = m.text.entities[0]
        for what, d in MOVES:
            mv.append(_with_entity(m, e.offset + d, e.length - d) if what == "start" else
                      _with_entity(m, e.offset, e.length + d))
    o = Oracle()
    rb, rm = o.telegram(pack_telegram(base, CHANNELS), abi.RUN_LINKS), o.telegram(pack_telegram(mv, CHANNELS), abi.RUN_LINKS)
    both = {"mention": 0, "url": 0}
    total = {"mention": 0, "url": 0}
    for i, (_, kind, declared) in enumerate(cases):
        seen = set()
        for k, move in enumerate(MOVES):
            j = 4 * i + k
            if (rm.status[j], rm.record_links(j)) != (rb.status[i], rb.record_links(i)):
                seen.add(move)
        assert seen == set(declared), (i, kind, seen, declared)
        total[kind] += 1
        both[kind] += any(w == "start" for w, _ in seen) and any(w == "end" for w, _ in seen)
    print(f"seed {seed}: cases that see a start move and an end move: mention {both['mention']} / {total['mention']}, "
          f"url {both['url']} / {total['url']}")
    for kind in both:
        assert both[kind] >= 0.6 * total[kind], (kind, both[kind], total[kind])


def test_filter_username_oracle_vs_restatement():
    for x in _filter_names(random.Random(7)):
        assert pyoracle.filter_username(x) == go_rules.filter_username(x), x
