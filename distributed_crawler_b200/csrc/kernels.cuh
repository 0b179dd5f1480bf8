// kernels.cuh — __global__ kernels of the ingest engine (sm_90a).  See DESIGN.md §4 for the data layout and the
// roofline bookkeeping.  All of it is integer/byte work:
//   tg_chan_size / tg_chan_emit            per-channel constant strings (once per batch, tiny)
//   tg_ent_map / tg_parse / tg_parse_ent   status + link extraction (split by code footprint): tg_parse scans 32
//                                          records' texts per warp as one packed stream, the other two take one warp
//                                          per record with entities
//   tg_size_lane                           JSONL line length, one LANE per record (+ the warp for the message text)
//   scan_*                                 exclusive scan u32 -> u64 offsets
//   tg_emit_lane                           the line, one LANE per record (tg_lane.cuh)
//   tg_emit_esc / tg_emit_maps             what the lane emitter leaves: strings that need escaping, comment lists ...
//   frontier_*                             exact open-addressed hash set over 32-byte keys
//   yt_* / gm_*                            YouTube (config 4) and generic-message (a12) lines
//   ch_*                                   random-walk channel records (StoreChannelData)
//   join_*                                 message-status join (SURVEY 8f)
// yt_size_kernel is the warp-per-record predecessor of the YouTube lane sizer, kept as an A/B reference (TGI_YT_WARP).
#pragma once
#include "scalars.cuh"
#include "tg_walk.cuh"
#include "tg_lane.cuh"
#include "yt_walk.cuh"
#include "gm_walk.cuh"
#include "ch_walk.cuh"
#include "yt_lane.cuh"

namespace tgi {

constexpr int WARPS_PER_CTA = 8;
constexpr int CTA_THREADS = WARPS_PER_CTA * 32;
// Resident CTAs per SM the compiler budgets registers for.  Swept on the config-2 step, device time of all kernels per
// 10 M messages on one H100 SXM at a 400 W power limit (tools/variants.sh, DESIGN.md §5): 4 (64 registers) 54.5 ms,
// 5: 52.9, 6 (40 registers): 52.9, 7: 57.0, 8: 57.0.  bench.py, config 2, 7 -> 6 (and LB_YT 6 -> 4), builds alternating:
// 56.2 -> 52.0 ms per step (DESIGN.md §5).
#ifndef LB_PARSE
#define LB_PARSE 6
#endif
#ifndef LB_SIZE
#define LB_SIZE 6
#endif
#ifndef LB_ESC
#define LB_ESC 6
#endif
#ifndef LB_MAPS
#define LB_MAPS 6
#endif
#ifndef LB_YT
#define LB_YT 4  // per 2 M config-4 records, same H100: 4: 31.6 ms, 5: 33.6, 6: 35.3, 7: 41.7, 8: 41.7 (tools/variants_yt.sh)
#endif

// ---- batch validation: every offset the kernels will follow stays inside its array ------------------------------
// A malformed batch that crossed the C ABI must come back as TGI_E_ARG, not as an illegal address (or as foreign
// bytes in the JSONL).  One thread per index of the longest array; big batches only (small ones are checked by the host).
struct TgBounds {
  uint64_t strs_len, n_ents, n_reacts, n_comments, aux_len, chan_strs_len;
};
__global__ void tg_validate_kernel(TgBatchDev b, TgBounds lim, uint64_t count, int* bad) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  int e = 0;
  if (i < b.n) {
    const tgi_tg_rec rc = b.recs[i];
    const uint64_t end = rc.str_off + (uint64_t)rc.text_len + rc.alt_len + rc.media_len + rc.handle_len;
    if (end > lim.strs_len || end < rc.str_off) e |= 1;
    if (rc.chan_idx >= b.n_chans || rc.content_type >= TGI_CT__COUNT) e |= 2;
    if (b.ent_off[i] > b.ent_off[i + 1] || b.ent_off[i + 1] > lim.n_ents) e |= 4;
    if (b.react_off[i] > b.react_off[i + 1] || b.react_off[i + 1] > lim.n_reacts) e |= 8;
    if (b.comment_off[i] > b.comment_off[i + 1] || b.comment_off[i + 1] > lim.n_comments) e |= 16;
  }
  if (i < lim.n_ents) {
    const tgi_entity en = b.ents[i];
    if (en.type == TGI_ENT_TEXT_URL && (uint64_t)en.url_off + en.url_len > lim.aux_len) e |= 32;
  }
  if (i < lim.n_reacts) {
    const tgi_reaction rc = b.reacts[i];
    if ((uint64_t)rc.emoji_off + rc.emoji_len > lim.aux_len) e |= 64;
  }
  if (i < lim.n_comments) {
    const tgi_comment cm = b.comments[i];
    if ((uint64_t)cm.text_off + cm.text_len > lim.aux_len || (uint64_t)cm.handle_off + cm.handle_len > lim.aux_len) e |= 128;
    if ((cm.flags & 1) && (uint64_t)cm.react_start + cm.react_count > lim.n_reacts) e |= 256;
  }
  if (i < b.n_chans) {
    const tgi_tg_chan ch = b.chans[i];
    if ((uint64_t)ch.str_off + ch.title_len + ch.name_len + ch.user_len > lim.chan_strs_len) e |= 512;
  }
  if (e) atomicOr(bad, e);
}

// ---- channel job -----------------------------------------------------------------------------------
// Every kernel of the Telegram pipeline is a *_body (grid-stride over blockIdx / gridDim) plus a one-line __global__
// wrapper: the page kernel (tg_page.cuh) runs the same bodies as phases of ONE cooperative launch.
DEVI void tg_chan_size_body(const TgBatchDev& b, ChanDerived* cd, uint32_t* len) {
  const int wid = threadIdx.x >> 5;
  for (uint32_t c = blockIdx.x * WARPS_PER_CTA + wid; c < b.n_chans; c += gridDim.x * WARPS_PER_CTA) {
    ChanDerived d = size_tg_chan(b, c);
    if (lane_id() == 0) {
      cd[c] = d;
      len[c] = pad16(d.user_len) + pad16(d.name_len) + pad16(d.title_len) + pad16(d.cdata_len);
    }
  }
}
__global__ void __launch_bounds__(CTA_THREADS) tg_chan_size_kernel(TgBatchDev b, ChanDerived* cd, uint32_t* len) { tg_chan_size_body(b, cd, len); }

DEVI void tg_chan_emit_body(const TgBatchDev& b, ChanDerived* cd, const uint64_t* off, uint8_t* blob, bool write_off = true) {
  __shared__ WarpScratch wss[WARPS_PER_CTA];
  const int wid = threadIdx.x >> 5;
  for (uint32_t c = blockIdx.x * WARPS_PER_CTA + wid; c < b.n_chans; c += gridDim.x * WARPS_PER_CTA) {
    if (write_off && lane_id() == 0) cd[c].off = off[c];
    emit_tg_chan(blob + off[c], &wss[wid], b, c);
    __syncwarp();
  }
}
__global__ void __launch_bounds__(CTA_THREADS) tg_chan_emit_kernel(TgBatchDev b, ChanDerived* cd, const uint64_t* off, uint8_t* blob) {
  tg_chan_emit_body(b, cd, off, blob);
}

// ---- parse: status + links + line length ---------------------------------------------------------
struct ParseOut {
  uint8_t* status;       // [n]
  uint32_t* linelen;     // [n] line length; until the size pass, the message text's escaped length if the parse measured it
  uint32_t* link_start;  // [n] arena index of the record's first link
  uint32_t* link_count;  // [n]
  uint32_t* xlen;        // [n][8] emitted lengths of the variable pieces (XL_*)
  unsigned long long* var_total;  // sum of the variable pieces' lengths (statistics)
  tgi_link* arena;
  uint32_t arena_cap;
  uint32_t* cursor;      // arena allocation cursor (keeps counting past arena_cap)
  int2* ent_range;       // [n_ents] byte range of every mention / url entity (tg_ent_map_kernel)
  int* err;
};

// link_count of a record with entities between tg_parse_kernel and tg_parse_ent_kernel: its reserved slots (< 2^20), with
// this bit if tg_parse_kernel mapped its entities (tg_ent_map_kernel skips it)
constexpr uint32_t LC_MAPPED = 1u << 31;

DEVI TgRecView load_rec_view(const TgBatchDev& b, uint64_t r) {
  TgRecView v;
  const tgi_tg_rec* rec = &b.recs[r];
  v.rec = rec;
  v.text = b.strs + rec->str_off;
  v.text_len = rec->text_len;
  v.alt = v.text + v.text_len;
  v.alt_len = rec->alt_len;
  v.media = v.alt + v.alt_len;
  v.media_len = rec->media_len;
  v.handle = v.media + v.media_len;
  v.handle_len = rec->handle_len;
  v.ct = rec->content_type;
  v.flags = rec->flags;
  v.e0 = b.ent_off[r];
  v.e1 = b.ent_off[r + 1];
  return v;
}

// One record (the page kernel).  ENTITIES == false: the record has no entities, so the whole UTF-16 offset machinery
// (warp_utf16_to_bytes, the exact UTF-8 path) is compiled out.
template <bool ENTITIES>
DEVI void parse_one_record(const TgBatchDev& b, const CfgDev& cfg, const ParseOut& o, uint64_t r, TgRecView v) {
  const int l = lane_id();
  uint32_t status = TGI_ST_EMITTED, nlinks = 0, lstart = 0;
  if ((cfg.flags & TGI_CFG_HAS_MIN_POST_DATE) && (int64_t)v.rec->date < cfg.min_post_date) {
    status = TGI_ST_SKIPPED;  // tdutils.go:419-421
  } else if (v.flags & TGI_RF_PANIC) {
    status = TGI_ST_FAILED;
  } else {
    if (!ENTITIES) v.e1 = v.e0;
    uint32_t ub = warp_link_upper_bound(v, b.ents);
    if (ub >= (1u << 20)) {  // seq packing of the frontier needs ordinal < 2^20 (SEQ_ORD_BITS)
      if (l == 0) atomicOr(o.err, ERR_TOO_MANY_LINKS);
      ub = 0;
    }
    if (ub) {
      if (l == 0) lstart = atomicAdd(o.cursor, ub);
      lstart = __shfl_sync(FULL, lstart, 0);
      if (lstart + ub > o.arena_cap || lstart + ub < lstart) {
        if (l == 0) atomicOr(o.err, ERR_ARENA_OVERFLOW);
      } else {
        const tgi_tg_chan* ch = &b.chans[v.rec->chan_idx];
        LinkSink ls;
        ls.out = o.arena + lstart;
        ls.cap = ub;
        ls.count = 0;
        ls.name_bytes = 0;
        ls.self = b.chan_strs + ch->str_off + ch->title_len;
        ls.self_len = ch->name_len;
        bool ok = warp_extract_links(v, b.ents, b.aux, o.ent_range, ls, true);
        nlinks = ls.count;
        if (!ok) {
          status = TGI_ST_FAILED;
          nlinks = 0;
        }
      }
    }
  }
  if (l == 0) {
    o.status[r] = (uint8_t)status;
    o.linelen[r] = 0u;  // the size pass measures the texts and overwrites the emitted ones
    o.link_start[r] = lstart;
    o.link_count[r] = nlinks;
  }
}

// The packed chunk stream of a group of 32 records (tg_parse_kernel, tg_ent_map_kernel): incl = the chunks of the lane's
// record and the records below it.  Returns the owner of chunk base + lane = the number of records whose chunks end at
// or before it (5 steps of a binary search on the scan, clamped to the pass so that it fits 32 bits).
DEVI int packed_chunk_owner(uint64_t incl, uint64_t base) {
  const uint32_t end = incl <= base ? 0u : (uint32_t)min(incl - base, (uint64_t)32);
  int ow = 0;
#pragma unroll
  for (int s = 16; s; s >>= 1)
    if (__shfl_sync(FULL, end, ow + s - 1) <= (uint32_t)lane_id()) ow += s;
  return ow;
}

// The parse step is split by instruction footprint (the SM's instruction caches hold only a few thousand instructions):
// tg_ent_map_kernel = UTF-16 entity offsets -> byte ranges, tg_parse_kernel = status, link bounds and text measurement
// of every record and the links of the records WITHOUT entities (small code), tg_parse_ent_kernel = links of the
// records with entities (lanes pick them out of groups of 32), tg_size_lane_kernel = line lengths.  Fusing them was tried twice
// (one parse kernel; parse + size in ONE pass over the text, fewer instructions in all): both fused kernels stalled on
// instruction fetch and were slower than the split ones.
//
// tg_parse_kernel takes the records 32 per warp, lane k owning record 32g + k, and scans their texts as ONE packed
// stream: text j's 16-byte chunks (cut from the text's start) follow text j - 1's in one chunk index space, and the
// warp walks that space 32 chunks per pass, each lane on the chunk of whichever record holds it.  A warp per record
// left most lanes idle (the median text fills about 20 of a strip's 32 lanes, a caption 7) and paid a full warp
// iteration for every record without text to scan.  Per chunk the lane counts "t.me/" (tme16) and measures the bytes
// (measure16); the totals go to the owning lane through shared-memory atomics on the (rare) nonzero values.  Only the
// records without entities and with a "t.me/" hit then take the warp-wide extraction, one after the other; a record
// with entities gets its arena slots (the bound) and leaves the extraction to tg_parse_ent_kernel, which keeps the
// entity code out of this kernel's instruction footprint.
template <bool MEASURE>
DEVI void tg_parse_body(const TgBatchDev& b, const CfgDev& cfg, uint32_t run_flags, const ParseOut& o) {
  // per record: "t.me/" hits, a byte >= 0x80, escape extras, not clean
  __shared__ uint32_t acc[WARPS_PER_CTA][MEASURE ? 4 : 2][32];
  const int wid = threadIdx.x >> 5, l = lane_id();
  const uint32_t SP = 0x20202020u;
  uint32_t* a_cnt = acc[wid][0];
  uint32_t* a_hi = acc[wid][1];
  uint32_t* a_extra = acc[wid][MEASURE ? 2 : 0];
  uint32_t* a_bad = acc[wid][MEASURE ? 3 : 0];
  const uint64_t ngroups = (b.n + 31) / 32, nwarps = (uint64_t)gridDim.x * WARPS_PER_CTA;
  for (uint64_t g = (uint64_t)blockIdx.x * WARPS_PER_CTA + wid; g < ngroups; g += nwarps) {
    const uint64_t r = g * 32 + l;
    uint32_t status = TGI_ST_EMITTED, len = 0, nents = 0;  // len: bytes of text to scan; nents: its link-kind entities
    bool ents = false;                                       // the record has entities (tg_parse_ent_kernel extracts)
    const uint8_t* text = b.strs;
    if (r < b.n) {
      const tgi_tg_rec* rec = &b.recs[r];
      const uint32_t fl = rec->flags, e0 = b.ent_off[r], e1 = b.ent_off[r + 1];
      ents = e1 != e0;
      if ((cfg.flags & TGI_CFG_HAS_MIN_POST_DATE) && (int64_t)rec->date < cfg.min_post_date) {
        status = TGI_ST_SKIPPED;  // tdutils.go:419-421
      } else if (fl & TGI_RF_PANIC) {
        status = TGI_ST_FAILED;
      } else if (ct_carries_links(rec->content_type) && (fl & TGI_RF_HAS_TEXT)) {
        text += rec->str_off;
        len = rec->text_len;
        for (uint32_t e = e0; e < e1; e++) nents += b.ents[e].type != TGI_ENT_OTHER;
      }
    }
    // the group's chunks: this record's are [incl - nch, incl) (64 bits: 32 texts of up to 4 GiB)
    const uint64_t nch = ((uint64_t)len + 15u) >> 4;
    uint64_t incl = nch;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint64_t t = __shfl_up_sync(FULL, incl, d);
      if (l >= d) incl += t;
    }
    const uint64_t total = __shfl_sync(FULL, incl, 31), first = incl - nch;
    a_cnt[l] = a_hi[l] = 0;
    if (MEASURE) a_extra[l] = a_bad[l] = 0;
    __syncwarp();
    uint32_t carry = SP;  // the last 4 bytes of lane 31's chunk in the previous pass
    for (uint64_t base = 0; base < total; base += 32) {
      const int ow = packed_chunk_owner(incl, base);
      const uint8_t* s = (const uint8_t*)__shfl_sync(FULL, (unsigned long long)text, ow);
      const uint64_t j = base + l - __shfl_sync(FULL, first, ow);  // chunk of that record
      const int64_t n = __shfl_sync(FULL, len, ow), p0 = (int64_t)(16 * j), rem = n - p0;
      const bool act = base + l < total;
      uint4 w = make_uint4(SP, SP, SP, SP);
      uint32_t cnt = 0, extra = 0, bad = 0;
      if (act) {
        w = ld16_unaligned(s + p0);
        cnt = __popc(tme16(s, p0, n, w));
        if (rem < 16) w = make_uint4(blank_from(w.x, rem), blank_from(w.y, rem - 4), blank_from(w.z, rem - 8), blank_from(w.w, rem - 12));
      }
      const uint32_t below = __shfl_up_sync(FULL, w.w, 1);
      const uint32_t pw = j == 0 ? SP : (l == 0 ? carry : below);  // a chunk in front of the text's first is not its
      carry = __shfl_sync(FULL, w.w, 31);
      if (MEASURE && act) {
        measure16(w, pw, bad, extra);
        // the text's last chunk: a sequence open at its end (one needs a high bit in the last three bytes)
        if (rem <= 16 && (w.w & 0x80808000u)) bad |= utf8_unclean4(w.w, SP);
      }
      if (cnt) atomicAdd(&a_cnt[ow], cnt);
      if ((w.x | w.y | w.z | w.w) & 0x80808080u) a_hi[ow] = 1u;
      if (MEASURE && extra) atomicAdd(&a_extra[ow], extra);
      if (MEASURE && bad) a_bad[ow] = 1u;
    }
    __syncwarp();
    uint32_t ub = a_cnt[l] + nents, text_esc = 0;  // the link bound: "t.me/" hits + entities of the three kinds
    if (MEASURE) text_esc = a_bad[l] ? 0u : len + a_extra[l];
    if (ub >= (1u << 20)) {  // seq packing of the frontier needs ordinal < 2^20 (SEQ_ORD_BITS)
      atomicOr(o.err, ERR_TOO_MANY_LINKS);
      ub = 0;
    }
    // one arena reservation for the group (links_compact puts the links in record order)
    const uint32_t ub_incl = warp_incl_scan(ub), ub_total = __shfl_sync(FULL, ub_incl, 31);
    uint32_t gstart = 0;
    if (ub_total) {
      if (l == 31) gstart = atomicAdd(o.cursor, ub_total);
      gstart = __shfl_sync(FULL, gstart, 31);
    }
    const uint32_t lstart = ub ? gstart + (ub_incl - ub) : 0u;
    const bool fits = (uint64_t)gstart + ub_incl <= o.arena_cap;
    if (ub && !fits) atomicOr(o.err, ERR_ARENA_OVERFLOW);
    uint32_t nlinks = 0;
    for (uint32_t todo = __ballot_sync(FULL, ub && fits && !ents); todo; todo &= todo - 1) {
      const int k = __ffs(todo) - 1;
      const tgi_tg_chan* ch = &b.chans[b.recs[g * 32 + k].chan_idx];
      LinkSink ls;
      ls.out = o.arena + __shfl_sync(FULL, lstart, k);
      ls.cap = __shfl_sync(FULL, ub, k);
      ls.count = 0;
      ls.name_bytes = 0;
      ls.self = b.chan_strs + ch->str_off + ch->title_len;
      ls.self_len = ch->name_len;
      // a record without entities: warp_extract_links is the plaintext scan alone
      warp_scan_channel_links(ls, (const uint8_t*)__shfl_sync(FULL, (unsigned long long)text, k), __shfl_sync(FULL, len, k),
                              TGI_SRC_PLAINTEXT, true);
      if (l == k) nlinks = ls.count;
    }
    // a record with entities keeps its reservation until tg_parse_ent_kernel.  An ASCII text has its entities mapped
    // here (a byte is a rune and a UTF-16 unit: utf16OffsetToBytes' loop meets unit i at byte i); tg_ent_map_kernel
    // maps the others
    const bool mapped = ents && ub && fits && a_hi[l] == 0;
    if (mapped) {
      for (uint32_t e = b.ent_off[r], e1 = b.ent_off[r + 1]; e < e1; e++) {
        const tgi_entity en = b.ents[e];
        if (en.type != TGI_ENT_MENTION && en.type != TGI_ENT_URL) continue;
        const int32_t off = en.offset, stop = (int32_t)((uint32_t)en.offset + (uint32_t)en.length), n = (int32_t)len;
        const bool s_in = off >= 0 && off < n;
        o.ent_range[e] = stop >= 0 && stop < n ? make_int2(s_in && off <= stop ? off : -1, stop)
                                               : (s_in ? make_int2(off, n) : make_int2(0, 0));
      }
    }
    if (r < b.n) {
      o.status[r] = (uint8_t)status;
      o.linelen[r] = MEASURE && status == TGI_ST_EMITTED ? text_esc : 0u;  // the size pass overwrites the emitted ones
      o.link_start[r] = lstart;
      o.link_count[r] = ents && fits && ub ? ub | (mapped ? LC_MAPPED : 0u) : nlinks;
    }
  }
}
template <bool MEASURE>
__global__ void __launch_bounds__(CTA_THREADS, LB_PARSE) tg_parse_kernel(TgBatchDev b, CfgDev cfg, uint32_t run_flags, ParseOut o) {
  tg_parse_body<MEASURE>(b, cfg, run_flags, o);
}
// utf16OffsetToBytes for every mention / url entity, 32 records per warp over one packed chunk stream as in
// tg_parse_kernel (a warp per record walked a non-ASCII text from its start once per entity).  A clean text (unclean16)
// decodes rune by rune the way Go's does, so a 16-byte chunk holds utf16_units16 units, and a scan over the pass (cut
// at the records' first chunks) plus the record's units of the earlier passes places every rune start.  The lane on a
// chunk looks for its record's entity offsets and ends in it and writes the byte index of the (one) rune start it finds
// to ent_range[e].x / .y; after the walk the owning lane applies the end of utf16OffsetToBytes to them.  A record whose
// text is not clean takes warp_map_entities, a warp each, which is exact on any bytes.
DEVI void tg_ent_map_body(const TgBatchDev& b, const ParseOut& o) {
  const int wid = threadIdx.x >> 5, l = lane_id();
  const uint32_t SP = 0x20202020u;
  const uint64_t ngroups = (b.n + 31) / 32, nwarps = (uint64_t)gridDim.x * WARPS_PER_CTA;
  for (uint64_t g = (uint64_t)blockIdx.x * WARPS_PER_CTA + wid; g < ngroups; g += nwarps) {
    const uint64_t r = g * 32 + l;
    uint32_t len = 0, e0 = 0, e1 = 0;  // [e0, e1): the entities to map (none: the record takes no part)
    uint32_t t_lo = 0x7FFFFFFFu, t_hi = 0;  // the unit positions looked for (int32 >= 0) lie in [t_lo, t_hi]
    bool any = false;
    const uint8_t* text = b.strs;
    if (r < b.n && o.status[r] == TGI_ST_EMITTED) {  // the records tg_parse_ent_kernel extracts, unless mapped
      e0 = b.ent_off[r];
      e1 = b.ent_off[r + 1];
      const tgi_tg_rec* rec = &b.recs[r];
      const uint32_t lc = o.link_count[r];
      if (e1 != e0 && lc != 0 && !(lc & LC_MAPPED) && ct_carries_links(rec->content_type) && (rec->flags & TGI_RF_HAS_TEXT)) {
        for (uint32_t e = e0; e < e1; e++) {
          const tgi_entity en = b.ents[e];
          if (en.type == TGI_ENT_MENTION || en.type == TGI_ENT_URL) {
            o.ent_range[e] = make_int2(-1, -1);  // no rune start found yet at the offset / at the end
            any = true;
            const int32_t stop = (int32_t)((uint32_t)en.offset + (uint32_t)en.length);
            if (en.offset >= 0) t_lo = min(t_lo, (uint32_t)en.offset), t_hi = max(t_hi, (uint32_t)en.offset);
            if (stop >= 0) t_lo = min(t_lo, (uint32_t)stop), t_hi = max(t_hi, (uint32_t)stop);
          }
        }
      }
      if (any) {
        text += rec->str_off;
        len = rec->text_len;
      } else {
        e1 = e0;
      }
    }
    // a rune of a clean text has at most 3 bytes per unit, so the one at unit t starts before byte 3t + 1: the walk
    // stops there (the chunks past it hold no position looked for, and Go's result does not depend on their bytes)
    const uint64_t nch = min(((uint64_t)len + 15u) >> 4, t_lo <= t_hi ? (3 * (uint64_t)t_hi + 16u) >> 4 : 0u);
    uint64_t incl = nch;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint64_t t = __shfl_up_sync(FULL, incl, d);
      if (l >= d) incl += t;
    }
    const uint64_t total = __shfl_sync(FULL, incl, 31), first = incl - nch;
    uint32_t units = 0;     // the record's units in the chunks of the passes so far
    bool unclean = false;   // the record's text is not clean
    uint32_t carry = SP;    // the last 4 bytes of lane 31's chunk in the previous pass
    __syncwarp();
    for (uint64_t base = 0; base < total; base += 32) {
      const int ow = packed_chunk_owner(incl, base);
      const uint8_t* s = (const uint8_t*)__shfl_sync(FULL, (unsigned long long)text, ow);
      const uint64_t j = base + l - __shfl_sync(FULL, first, ow);  // chunk of that record
      const int64_t n = __shfl_sync(FULL, len, ow), p0 = (int64_t)(16 * j), rem = n - p0;
      const bool act = base + l < total;
      uint4 w = make_uint4(SP, SP, SP, SP);
      uint32_t u = 0, bad = 0;
      if (act) {
        w = ld16_unaligned(s + p0);
        if (rem < 16) w = make_uint4(blank_from(w.x, rem), blank_from(w.y, rem - 4), blank_from(w.z, rem - 8), blank_from(w.w, rem - 12));
        u = utf16_units16(w, rem < 16 ? (uint32_t)rem : 16u);
      }
      const uint32_t below = __shfl_up_sync(FULL, w.w, 1);
      const uint32_t pw = j == 0 ? SP : (l == 0 ? carry : below);
      carry = __shfl_sync(FULL, w.w, 31);
      if (act) {
        unclean16(w, pw, bad);
        if (rem <= 16 && (w.w & 0x80808000u)) bad |= utf8_unclean4(w.w, SP);
      }
      // the segmented scan: this lane's record holds the pass's lanes [lo, hi)
      const uint32_t ui = warp_incl_scan(u), badm = __ballot_sync(FULL, bad != 0);
      const uint32_t hi = incl <= base ? 0u : (uint32_t)min(incl - base, (uint64_t)32);
      const uint32_t lo = first <= base ? 0u : (uint32_t)min(first - base, (uint64_t)32);
      const uint32_t top = __shfl_sync(FULL, ui, hi ? hi - 1 : 0), bot = __shfl_sync(FULL, ui, lo ? lo - 1 : 0);
      const uint32_t seg0 = lo ? bot : 0u;  // units of the pass in front of the record's chunks
      const uint32_t pos = __shfl_sync(FULL, units, ow) + ui - u - __shfl_sync(FULL, seg0, ow);  // units before the chunk
      const uint32_t me0 = __shfl_sync(FULL, e0, ow), me1 = __shfl_sync(FULL, e1, ow);
      const uint32_t mlo = __shfl_sync(FULL, t_lo, ow), mhi = __shfl_sync(FULL, t_hi, ow);
      if (hi > lo) {
        units += top - seg0;
        unclean = unclean || (badm & ((hi == 32 ? ~0u : (1u << hi) - 1u) & ~((1u << lo) - 1u)));
      }
      if (act && pos <= mhi && mlo < pos + u) {  // a position looked for can lie in this chunk
        for (uint32_t e = me0; e < me1; e++) {
          const tgi_entity en = b.ents[e];
          if (en.type != TGI_ENT_MENTION && en.type != TGI_ENT_URL) continue;
          // Go compares int32 unit positions: the end wraps as an int32 sum, a negative offset is never reached
          const uint32_t t0 = (uint32_t)en.offset - pos, t1 = (uint32_t)en.offset + (uint32_t)en.length - pos;
          if (t0 < u) {
            const int k = rune_at_unit16(w, t0);
            if (k >= 0) o.ent_range[e].x = (int)(p0 + k);
          }
          if (t1 < u) {
            const int k = rune_at_unit16(w, t1);
            if (k >= 0) o.ent_range[e].y = (int)(p0 + k);
          }
        }
      }
    }
    __syncwarp();
    if (!unclean) {  // the end of utf16OffsetToBytes
      for (uint32_t e = e0; e < e1; e++) {
        const uint32_t t = b.ents[e].type;
        if (t != TGI_ENT_MENTION && t != TGI_ENT_URL) continue;
        const int2 h = o.ent_range[e];
        int2 rg;
        if (h.y >= 0) rg = make_int2(h.x >= 0 && h.x <= h.y ? h.x : -1, h.y);  // a start past the end is never reached
        else rg = h.x >= 0 ? make_int2(h.x, (int)len) : make_int2(0, 0);
        o.ent_range[e] = rg;
      }
    }
    for (uint32_t todo = __ballot_sync(FULL, unclean && e1 != e0); todo; todo &= todo - 1)
      warp_map_entities(load_rec_view(b, g * 32 + (uint32_t)(__ffs(todo) - 1)), b.ents, o.ent_range);
  }
}
__global__ void __launch_bounds__(CTA_THREADS, LB_PARSE) tg_ent_map_kernel(TgBatchDev b, ParseOut o) { tg_ent_map_body(b, o); }
// The links of the records with entities that tg_parse_kernel left: their slots are reserved (link_count) and their
// entities mapped (ent_range), so the warp only extracts, record after record.  The plaintext scan is skipped when the
// reservation is the entities alone: the count found no "t.me/" in the text.
DEVI void tg_parse_ent_body(const TgBatchDev& b, const ParseOut& o) {
  const int wid = threadIdx.x >> 5, l = lane_id();
  const uint64_t ngroups = (b.n + 31) / 32, nwarps = (uint64_t)gridDim.x * WARPS_PER_CTA;
  for (uint64_t g = (uint64_t)blockIdx.x * WARPS_PER_CTA + wid; g < ngroups; g += nwarps) {
    const uint64_t rl = g * 32 + l;
    uint32_t todo = __ballot_sync(FULL, rl < b.n && b.ent_off[rl + 1] != b.ent_off[rl] && o.status[rl] == TGI_ST_EMITTED &&
                                            o.link_count[rl] != 0);
    while (todo) {
      const uint64_t r = g * 32 + (uint32_t)(__ffs(todo) - 1);
      todo &= todo - 1;
      const TgRecView v = load_rec_view(b, r);
      const tgi_tg_chan* ch = &b.chans[v.rec->chan_idx];
      LinkSink ls;
      ls.out = o.arena + o.link_start[r];
      ls.cap = o.link_count[r] & ~LC_MAPPED;
      ls.count = 0;
      ls.name_bytes = 0;
      ls.self = b.chan_strs + ch->str_off + ch->title_len;
      ls.self_len = ch->name_len;
      uint32_t c = 0;
      for (uint32_t e = v.e0 + l; e < v.e1; e += 32) c += b.ents[e].type != TGI_ENT_OTHER;
      const bool ok = warp_extract_links(v, b.ents, b.aux, o.ent_range, ls, ls.cap != warp_sum(c));
      if (l == 0) {
        if (!ok) {  // the reference panics: the same result as parse_one_record's
          o.status[r] = TGI_ST_FAILED;
          o.linelen[r] = 0;
        }
        o.link_count[r] = ok ? ls.count : 0u;
      }
    }
  }
}
__global__ void __launch_bounds__(CTA_THREADS, LB_PARSE) tg_parse_ent_kernel(TgBatchDev b, ParseOut o) { tg_parse_ent_body(b, o); }

// The same sizes, 32 records per warp: every lane sizes the small pieces of its own record (numbers,
// handle / media strings, comments, reactions, outlinks); the description, the one long string, is measured by the
// whole warp, record after record, unless it is a message text the parse already measured (linelen); the rare
// complicated pieces (a comment list, a reactions map that is not "simple") go through the warp-wide routines as well.
DEVI void tg_size_lane_body(const TgBatchDev& b, const CfgDev& cfg, const ParseOut& o) {
  const int wid = threadIdx.x >> 5, l = lane_id();
  const uint64_t ngroups = (b.n + 31) / 32, nwarps = (uint64_t)gridDim.x * WARPS_PER_CTA;
  uint64_t var_sum = 0;
  for (uint64_t g = (uint64_t)blockIdx.x * WARPS_PER_CTA + wid; g < ngroups; g += nwarps) {
    uint64_t r = g * 32 + l;
    bool active = r < b.n;
    if (!active) r = b.n - 1;
    active = active && o.status[r] == TGI_ST_EMITTED;
    if (!__any_sync(FULL, active)) continue;
    TgWalkArgs a;
    a.b = &b;
    a.cfg = &cfg;
    a.r = r;
    a.v = load_rec_view(b, r);
    a.links = o.arena + o.link_start[r];
    a.n_links = active ? o.link_count[r] : 0u;
    const tgi_tg_rec* rec = a.v.rec;
    const ChanDerived cd = b.chan_derived[rec->chan_idx];
    const TgDerived d = tg_derive(a, cd);
    uint32_t xl[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    uint32_t tot = 0;
    bool warp_comments = false, warp_map = false;
    const uint32_t r0 = b.react_off[r], nr = b.react_off[r + 1] - r0;
    // the parse's measurement (tg_parse_kernel), != 0 only for a text of >= 1 byte: then alt != text, and d.desc == text
    // says the description is the message text
    const uint32_t text_esc = active ? o.linelen[r] : 0u;
    const bool measured = text_esc != 0 && d.desc == a.v.text;
    if (active && !(cfg.flags & CFGDEV_CLOCK_INVALID)) {
      uint32_t L[8] = {ndigits_i64(rec->id / 1048576), ndigits_i64(rec->chat_id), ndigits_i64(rec->view_count),
                       ndigits_i64(rec->share_count), ndigits_i64(d.ncomments), zone_offset(cfg, rec->date) == 0 ? 22u : 27u, 0, 0};
      uint32_t chan[4] = {cd.user_len, cd.name_len, cd.title_len, cd.cdata_len};
      uint32_t cf[4] = {cfg.label_len, cfg.created_tg_len, cfg.created_yt_len, cfg.capture_len};
      tot = tg_size_fixed(L, chan, cf, d.has_user, d.album);
      tot += a.v.ct == TGI_CT_OTHER ? 0u : (uint32_t)kPostTypeLen[a.v.ct];
      if (measured) xl[XL_DESC] = text_esc;
      if (a.v.ct == TGI_CT_OTHER) xl[XL_ALT] = thread_esc_len(a.v.alt, a.v.alt_len);
      if (d.has_media) xl[XL_MEDIA] = thread_esc_len(a.v.media, a.v.media_len);
      xl[XL_HANDLE] = thread_esc_len(a.v.handle, a.v.handle_len);
      if (d.comments_nil) xl[XL_COMMENTS] = 4;
      else if (d.c1 == d.c0) xl[XL_COMMENTS] = 2;
      else warp_comments = true;
      if (nr == 0) {
        xl[XL_REACTIONS] = 2;
        xl[XL_FLAGS] = XLF_SIMPLE_MAP;
      } else if (nr <= LANE_MAP_MAX) {  // size_reaction_map, one lane: "key":n , ... ; simple = short clean keys
        uint32_t sz = 2u, live = 0;
        bool simple = true;
        for (uint32_t j = 0; j < nr; j++) {
          const tgi_reaction rc = b.reacts[r0 + j];
          const uint8_t* kp = b.aux + rc.emoji_off;
          const uint32_t el = thread_esc_len(kp, rc.emoji_len);
          simple = simple && el == rc.emoji_len && rc.emoji_len >= 1 && rc.emoji_len <= 8;
          bool last = true;  // a later entry with the same key overwrites this one (Go map assignment)
          for (uint32_t i = j + 1; i < nr; i++) {
            const tgi_reaction ri = b.reacts[r0 + i];
            if (key_cmp(b.aux + ri.emoji_off, ri.emoji_len, kp, rc.emoji_len) == 0) last = false;
          }
          if (last) {
            sz += 3u + el + ndigits_i64(rc.count);
            live++;
          }
        }
        if (simple) {
          xl[XL_REACTIONS] = sz + (live - 1u);
          xl[XL_FLAGS] = XLF_SIMPLE_MAP;
        } else {
          warp_map = true;
        }
      } else {
        warp_map = true;
      }
      if (a.n_links) {
        uint32_t s = a.n_links - 1u;
        for (uint32_t k = 0; k < a.n_links; k++) s += a.links[k].len + 2u;
        xl[XL_OUTLINKS] = s;
      }
    }
    // the other descriptions (and the texts the parse did not measure), one record at a time, all lanes
    const bool sized = active && !(cfg.flags & CFGDEV_CLOCK_INVALID);
    uint32_t todo = __ballot_sync(FULL, sized && d.desc_len != 0 && !measured);
    while (todo) {
      const int src = __ffs(todo) - 1;
      todo &= todo - 1;
      const uint8_t* p = (const uint8_t*)__shfl_sync(FULL, (unsigned long long)(uintptr_t)d.desc, src);
      const uint32_t n = __shfl_sync(FULL, d.desc_len, src);
      bool ex = false;
      const uint32_t e = warp_esc_len(p, n, &ex);
      if (l == src) {
        xl[XL_DESC] = e;
        if (ex) xl[XL_FLAGS] |= XLF_DESC_EXACT;
      }
    }
    todo = __ballot_sync(FULL, warp_comments);
    while (todo) {
      const int src = __ffs(todo) - 1;
      todo &= todo - 1;
      const uint32_t e = size_tg_comments(b, __shfl_sync(FULL, d.c0, src), __shfl_sync(FULL, d.c1, src));
      if (l == src) xl[XL_COMMENTS] = e;
    }
    todo = __ballot_sync(FULL, warp_map);
    while (todo) {
      const int src = __ffs(todo) - 1;
      todo &= todo - 1;
      const uint32_t q0 = __shfl_sync(FULL, r0, src), qn = __shfl_sync(FULL, nr, src);
      uint32_t simple = 0;
      const uint32_t e = size_reaction_map(b.reacts, q0, q0 + qn, b.aux, &simple);
      if (l == src) {
        xl[XL_REACTIONS] = e;
        xl[XL_FLAGS] = (xl[XL_FLAGS] & ~XLF_SIMPLE_MAP) | (simple ? XLF_SIMPLE_MAP : 0u);
      }
    }
    if (active) {
      uint32_t var = 0;
#pragma unroll
      for (int j = 0; j < XL_COUNT; j++) var += xl[j];
      const uint32_t llen = sized ? tot + var : 0u;
      *(uint4*)(o.xlen + r * 8) = make_uint4(xl[0], xl[1], xl[2], xl[3]);
      *(uint4*)(o.xlen + r * 8 + 4) = make_uint4(xl[4], xl[5], xl[6], xl[7]);
      if (llen == 0) o.status[r] = TGI_ST_NOLINE;
      o.linelen[r] = llen;
      if (llen) var_sum += var;
    }
  }
  for (int dd = 16; dd; dd >>= 1) var_sum += __shfl_down_sync(FULL, var_sum, dd);
  if (l == 0 && var_sum) atomicAdd(o.var_total, (unsigned long long)var_sum);
}
__global__ void __launch_bounds__(CTA_THREADS, LB_SIZE) tg_size_lane_kernel(TgBatchDev b, CfgDev cfg, ParseOut o) { tg_size_lane_body(b, cfg, o); }

// ---- emit --------------------------------------------------------------------------------------------------------
struct EmitIn {
  const uint8_t* status;
  const uint64_t* line_off;
  const uint32_t* link_start;
  const uint32_t* link_count;
  const uint32_t* xlen;  // [n][8] lengths of the variable pieces + flags
  uint32_t* xpos;        // [n][8] offsets of the variable pieces inside the line (written by the lane emitter)
  const tgi_link* arena;
  uint8_t* out;
  int* err;
  uint32_t lane_text_max;        // see emit_tg_escapes
  unsigned long long* counters;  // [0] JSONL bytes written by the main emit kernel, [1] source bytes it read from HBM
  // work lists written by the lane emitter: the records whose line it did not finish, by what is left
  uint32_t* list[3];             // WL_SPARSE, WL_DENSE, WL_MAPS: record indices
  uint32_t* list_count;          // [3]
};
enum { WL_SPARSE = 0, WL_DENSE = 1, WL_MAPS = 2 };
// warp-aggregated append of the lanes with `need` to a work list
DEVI void wl_append(uint32_t* list, uint32_t* count, bool need, uint32_t value) {
  const uint32_t m = __ballot_sync(FULL, need);
  if (!m) return;
  uint32_t base = 0;
  if (lane_id() == 0) base = atomicAdd(count, (uint32_t)__popc(m));
  base = __shfl_sync(FULL, base, 0);
  if (need) list[base + __popc(m & ((1u << lane_id()) - 1u))] = value;
}

// the same job, one LANE per record (tg_lane.cuh): 32 records per warp task
DEVI void tg_emit_lane_body(const TgBatchDev& b, const CfgDev& cfg, const EmitIn& in, LaneShared& sh) {
  static_assert(LANE_WARPS == WARPS_PER_CTA, "one field row block per warp");
  lane_shared_fill(sh);
  __syncthreads();
  const int wid = threadIdx.x >> 5, l = lane_id();
  const uint64_t ngroups = (b.n + 31) / 32, nwarps = (uint64_t)gridDim.x * WARPS_PER_CTA;
  LaneStream s;
  ls_init(s, smem_addr(sh.stage[wid][l]));
  uint64_t bytes_out = 0, bytes_in = 0;
  for (uint64_t g = (uint64_t)blockIdx.x * WARPS_PER_CTA + wid; g < ngroups; g += nwarps) {
    uint64_t r = g * 32 + l;
    bool active = r < b.n;
    if (!active) r = b.n - 1;
    active = active && in.status[r] == TGI_ST_EMITTED;
    if (!__any_sync(FULL, active)) continue;
    uint32_t left = 0;
    emit_tg_lane(sh, sh.rows[wid][l], s, b, cfg, r, active, in.out, in.line_off, in.xlen + r * 8, in.xpos + r * 8,
                 in.arena + in.link_start[r], active ? in.link_count[r] : 0u, in.err, bytes_out, bytes_in, left);
    // hand the unfinished lines to the clean-up kernels as lists (they used to re-derive this from every record)
    bool sparse = false;
    if (active && (left & 1u)) {
      const tgi_tg_rec* rec = &b.recs[r];
      const uint32_t ct = rec->content_type;
      const bool text_desc = ct == TGI_CT_TEXT || ct == TGI_CT_VIDEO || ct == TGI_CT_PHOTO || ct == TGI_CT_ANIMATION;
      const uint32_t dlen = text_desc ? ((rec->flags & TGI_RF_HAS_TEXT) ? rec->text_len : 0u) : rec->alt_len;
      sparse = esc_desc_is_sparse(in.xlen[r * 8 + XL_DESC], dlen, in.xlen[r * 8 + XL_FLAGS]);
    }
    wl_append(in.list[WL_SPARSE], in.list_count + WL_SPARSE, active && sparse, (uint32_t)r);
    wl_append(in.list[WL_DENSE], in.list_count + WL_DENSE, active && (((left & 1u) && !sparse) || (left & 0xEu)), (uint32_t)r);
    wl_append(in.list[WL_MAPS], in.list_count + WL_MAPS, active && (left & 16u), (uint32_t)r);
  }
  for (int dd = 16; dd; dd >>= 1) {
    bytes_out += __shfl_down_sync(FULL, bytes_out, dd);
    bytes_in += __shfl_down_sync(FULL, bytes_in, dd);
  }
  if (l == 0) {
    atomicAdd(in.counters, (unsigned long long)bytes_out);
    atomicAdd(in.counters + 1, (unsigned long long)bytes_in);
  }
}
// The lane emitter's residency is set by its shared memory (LaneShared: 2 CTAs per SM with LANE_STAGE 256, see
// tg_lane.cuh); 3 here is the register budget (80 registers).
#ifndef LB_LANE
#define LB_LANE 3
#endif
__global__ void __launch_bounds__(CTA_THREADS, LB_LANE) tg_emit_lane_kernel(TgBatchDev b, CfgDev cfg, EmitIn in) {
  extern __shared__ __align__(128) uint8_t lane_smem[];
  tg_emit_lane_body(b, cfg, in, *(LaneShared*)lane_smem);
}

// The esc and maps kernels take what the lane emitter left, from its work lists: one warp per listed record.
// Two instantiations of the escape kernel by instruction footprint: ESC_SPARSE writes the descriptions whose only specials
// are a few line breaks (segment copies), ESC_DENSE the rest (per-byte placement, exact UTF-8 path, long clean strings,
// the other three strings).
template <int MODE>
DEVI void tg_emit_esc_body(const TgBatchDev& b, const EmitIn& in) {
  const int wid = threadIdx.x >> 5;
  const uint32_t* list = in.list[MODE == ESC_SPARSE ? WL_SPARSE : WL_DENSE];
  const uint32_t cnt = in.list_count[MODE == ESC_SPARSE ? WL_SPARSE : WL_DENSE];
  const uint32_t nwarps = gridDim.x * WARPS_PER_CTA;
  for (uint32_t i = blockIdx.x * WARPS_PER_CTA + wid; i < cnt; i += nwarps) {
    const uint64_t rr = list[i];
    TgWalkArgs a;
    a.b = &b;
    a.cfg = nullptr;
    a.r = rr;
    a.v = load_rec_view(b, rr);
    emit_tg_escapes<MODE>(in.out + in.line_off[rr], a, in.xlen + rr * 8, in.xpos + rr * 8, in.lane_text_max);
  }
}
template <int MODE>
__global__ void __launch_bounds__(CTA_THREADS, LB_ESC) tg_emit_esc_kernel(TgBatchDev b, EmitIn in) { tg_emit_esc_body<MODE>(b, in); }

DEVI void tg_emit_maps_body(const TgBatchDev& b, const EmitIn& in) {
  __shared__ MapScratch mss[WARPS_PER_CTA];
  const int wid = threadIdx.x >> 5;
  const uint32_t cnt = in.list_count[WL_MAPS], nwarps = gridDim.x * WARPS_PER_CTA;
  for (uint32_t i = blockIdx.x * WARPS_PER_CTA + wid; i < cnt; i += nwarps) {
    const uint64_t r = in.list[WL_MAPS][i];
    uint8_t* line = in.out + in.line_off[r];
    const uint32_t* xp = in.xpos + r * 8;
    // the lane emitter wrote the simple cases itself (tg_lane.cuh): nil / empty comment lists, simple maps, short outlink lists
    const bool comments_nil = (b.recs[r].flags & TGI_RF_COMMENTS_NIL) != 0;
    const uint32_t c0 = b.comment_off[r], c1 = b.comment_off[r + 1];
    if (!comments_nil && c1 != c0) emit_tg_comments(line + xp[XL_COMMENTS], &mss[wid], b, c0, c1);
    const uint32_t r0 = b.react_off[r], r1 = b.react_off[r + 1];
    if (r1 != r0 && !(in.xlen[r * 8 + XL_FLAGS] & XLF_SIMPLE_MAP)) emit_reaction_map(line + xp[XL_REACTIONS], &mss[wid], b.reacts, r0, r1, b.aux);
    const uint32_t nl = in.link_count[r];
    if (nl > LANE_LINKS_MAX) emit_tg_outlinks(line + xp[XL_OUTLINKS], in.arena + in.link_start[r], nl);
    __syncwarp();
  }
}
__global__ void __launch_bounds__(CTA_THREADS, LB_MAPS) tg_emit_maps_kernel(TgBatchDev b, EmitIn in) { tg_emit_maps_body(b, in); }

// ---- YouTube (config 4) ------------------------------------------------------------------------------
struct YtOut {
  uint8_t* status;
  uint32_t* linelen;
  uint32_t* url_start;   // [n] first unique URL of the record in `urls`
  uint32_t* url_count;
  YtUrl* urls;
  uint32_t urls_cap;
  uint32_t* url_cursor;
  uint32_t* esc_len;     // [n][3] escaped length of the description / title, clean flag (size pass -> emit pass)
  uint32_t* link_start;  // [n] channel-id links (frontier candidates)
  uint32_t* link_count;
  tgi_link* arena;
  uint32_t arena_cap;
  uint32_t* cursor;
  int* err;
};

// unique outlink URLs (extractURLs) and snowball channel ids (extractChannelIDsFromText)
DEVI void yt_parse_body(const YtBatchDev& b, const CfgDev& cfg, uint32_t run_flags, const YtOut& o) {
  int wid = threadIdx.x >> 5, l = lane_id();
  uint64_t nwarps = (uint64_t)gridDim.x * WARPS_PER_CTA;
  for (uint64_t r = (uint64_t)blockIdx.x * WARPS_PER_CTA + wid; r < b.n; r += nwarps) {
    const tgi_yt_rec v = b.recs[r];
    const uint8_t* desc = b.strs + v.str_off + v.id_len + v.title_len;
    uint32_t us = 0, uc = 0, ls = 0, lc = 0;
    uint32_t ub = yt_count_http(desc, v.desc_len);
    if (ub) {
      if (l == 0) us = atomicAdd(o.url_cursor, ub);
      us = __shfl_sync(FULL, us, 0);
      if (us + ub > o.urls_cap || us + ub < us) {
        if (l == 0) atomicOr(o.err, ERR_ARENA_OVERFLOW);
      } else {
        uc = yt_extract_urls(desc, v.desc_len, o.urls + us, ub);
      }
    }
    if (run_flags & (TGI_RUN_LINKS | TGI_RUN_FRONTIER)) {
      uint32_t lb = yt_count_ytcom(desc, v.desc_len);
      if (lb >= (1u << 20)) {
        if (l == 0) atomicOr(o.err, ERR_TOO_MANY_LINKS);
        lb = 0;
      }
      if (lb) {
        if (l == 0) ls = atomicAdd(o.cursor, lb);
        ls = __shfl_sync(FULL, ls, 0);
        if (ls + lb > o.arena_cap || ls + lb < ls) {
          if (l == 0) atomicOr(o.err, ERR_ARENA_OVERFLOW);
        } else {
          lc = yt_channel_ids(desc, v.desc_len, o.arena + ls, lb);
        }
      }
    }
    if (l == 0) {
      // json.Marshal fails (no line, record still "fetched") when a time.Time is outside year
      // [0,9999]; decided here so that the status does not depend on TGI_RUN_JSONL
      uint8_t tmp[40];
      bool ok = !(cfg.flags & CFGDEV_CLOCK_INVALID) && cfg.created_yt_len != 0 &&
                render_time(tmp, v.published_sec, v.published_nsec, 0) != 0;
      if (ok) {
        const tgi_yt_chan& ch = b.chans[v.chan_idx];
        if (ch.cached) ok = render_time(tmp, ch.published_sec, ch.published_nsec, 0) != 0;
      }
      o.status[r] = ok ? TGI_ST_EMITTED : TGI_ST_NOLINE;
      o.linelen[r] = 0;
      o.url_start[r] = us;
      o.url_count[r] = uc;
      o.link_start[r] = ls;
      o.link_count[r] = lc;
    }
  }
}
__global__ void __launch_bounds__(CTA_THREADS, LB_YT) yt_parse_kernel(YtBatchDev b, CfgDev cfg, uint32_t run_flags, YtOut o) { yt_parse_body(b, cfg, run_flags, o); }

// one record by one warp (yt_size_kernel, yt_page_kernel)
DEVI void yt_size_record(const YtBatchDev& b, const CfgDev& cfg, const YtOut& o, uint64_t r, YtScratch* sc) {
  const int l = lane_id();
  {
    YtArgs a;
    a.b = &b;
    a.cfg = &cfg;
    a.r = r;
    a.urls = o.urls + o.url_start[r];
    a.n_urls = o.url_count[r];
    YtSizer z;
    z.sc = sc;
    {
      const tgi_yt_rec* rec = &b.recs[r];
      const uint8_t* title = b.strs + rec->str_off + rec->id_len;
      z.el[1] = warp_esc_len(title, rec->title_len);
      z.el[0] = warp_esc_len(title + rec->title_len, rec->desc_len);
    }
    bool ok = walk_yt_record(z, a);
    if (l == 0) {
      o.esc_len[3 * r] = z.el[0];
      o.esc_len[3 * r + 1] = z.el[1];
      o.esc_len[3 * r + 2] = z.dirty ? 0u : 1u;  // clean: the lane writer takes the record
      o.linelen[r] = ok ? (uint32_t)z.total : 0u;
      if (!ok) o.status[r] = TGI_ST_NOLINE;
    }
  }
}
__global__ void __launch_bounds__(CTA_THREADS, LB_YT) yt_size_kernel(YtBatchDev b, CfgDev cfg, YtOut o) {
  __shared__ YtScratch scs[WARPS_PER_CTA];
  int wid = threadIdx.x >> 5;
  uint64_t nwarps = (uint64_t)gridDim.x * WARPS_PER_CTA;
  for (uint64_t r = (uint64_t)blockIdx.x * WARPS_PER_CTA + wid; r < b.n; r += nwarps) {
    if (o.status[r] != TGI_ST_EMITTED) continue;  // linelen stays 0
    yt_size_record(b, cfg, o, r, &scs[wid]);
  }
}

// length pass, one lane per record (yt_lane.cuh); the description and the title are measured by the warp
__global__ void __launch_bounds__(CTA_THREADS, LB_YT) yt_size_lane_kernel(YtBatchDev b, CfgDev cfg, YtOut o) {
  const int wid = threadIdx.x >> 5, l = lane_id();
  const uint64_t ngroups = (b.n + 31) / 32, nwarps = (uint64_t)gridDim.x * WARPS_PER_CTA;
  for (uint64_t g = (uint64_t)blockIdx.x * WARPS_PER_CTA + wid; g < ngroups; g += nwarps) {
    uint64_t r = g * 32 + l;
    bool active = r < b.n;
    if (!active) r = b.n - 1;
    active = active && o.status[r] == TGI_ST_EMITTED;
    const tgi_yt_rec* rec = &b.recs[r];
    const uint8_t* title = b.strs + rec->str_off + rec->id_len;
    const uint32_t tn = rec->title_len, dn = rec->desc_len;
    uint32_t el0 = 0, el1 = 0;
    bool exact = false;  // the description / title holds invalid UTF-8 or U+2028/9: only the exact (warp) escaper may write it
    uint32_t todo = __ballot_sync(FULL, active);
    while (todo) {  // the two long strings of every record, all lanes
      const int src = __ffs(todo) - 1;
      todo &= todo - 1;
      const uint8_t* t = (const uint8_t*)__shfl_sync(FULL, (unsigned long long)(uintptr_t)title, src);
      const uint32_t a = __shfl_sync(FULL, tn, src), d = __shfl_sync(FULL, dn, src);
      bool x1 = false, x0 = false;
      const uint32_t e1 = warp_esc_len(t, a, &x1), e0 = warp_esc_len(t + a, d, &x0);
      if (l == src) {
        el0 = e0;
        el1 = e1;
        exact = x0 || x1;
      }
    }
    if (!active) continue;
    YtArgs a;
    a.b = &b;
    a.cfg = &cfg;
    a.r = r;
    a.urls = o.urls + o.url_start[r];
    a.n_urls = o.url_count[r];
    YtLaneSizer z;
    z.el[0] = el0;
    z.el[1] = el1;
    const bool ok = walk_yt_record(z, a);
    o.esc_len[3 * r] = el0;
    o.esc_len[3 * r + 1] = el1;
    // 1: clean, 2: the lane writer escapes the description / title itself, 0: left to the warp writer
    o.esc_len[3 * r + 2] = !z.dirty ? 1u : (!z.small_dirty && !exact) ? 2u : 0u;
    o.linelen[r] = ok ? (uint32_t)z.total : 0u;
    if (!ok) o.status[r] = TGI_ST_NOLINE;
  }
}

// warp writer: the records the lane writer does not take (a string needs escaping); lanes pick them out of
// groups of 32.  lane_mode == 0: every record (A/B reference, TGI_YT_WARP=1).
DEVI void yt_emit_record(const YtBatchDev& b, const CfgDev& cfg, const YtOut& o, const uint64_t* line_off, uint8_t* out, int* err,
                         uint64_t r, YtScratch* sc) {
  YtArgs a;
  a.b = &b;
  a.cfg = &cfg;
  a.r = r;
  a.urls = o.urls + o.url_start[r];
  a.n_urls = o.url_count[r];
  YtWriter w;
  w.sc = sc;
  w.el[0] = o.esc_len[3 * r];
  w.el[1] = o.esc_len[3 * r + 1];
  w.p = out + line_off[r];
  walk_yt_record(w, a);
  if (lane_id() == 0 && (uint64_t)(w.p - out) != line_off[r + 1]) atomicOr(err, ERR_LINE_MISMATCH);
  __syncwarp();
}
__global__ void __launch_bounds__(CTA_THREADS, LB_YT) yt_emit_kernel(YtBatchDev b, CfgDev cfg, YtOut o, const uint64_t* line_off, uint8_t* out, int* err,
                                                                 int lane_mode) {
  __shared__ YtScratch scs[WARPS_PER_CTA];
  int wid = threadIdx.x >> 5, l = lane_id();
  const uint64_t ngroups = (b.n + 31) / 32, nwarps = (uint64_t)gridDim.x * WARPS_PER_CTA;
  for (uint64_t g = (uint64_t)blockIdx.x * WARPS_PER_CTA + wid; g < ngroups; g += nwarps) {
    const uint64_t rl = g * 32 + l;
    uint32_t todo = __ballot_sync(FULL, rl < b.n && o.status[rl] == TGI_ST_EMITTED && !(lane_mode && o.esc_len[3 * rl + 2]));
    while (todo) {
      const uint64_t r = g * 32 + (uint32_t)(__ffs(todo) - 1);
      todo &= todo - 1;
      yt_emit_record(b, cfg, o, line_off, out, err, r, &scs[wid]);
    }
  }
}

// lane writer (yt_lane.cuh): one lane per clean record
__global__ void __launch_bounds__(CTA_THREADS, LB_YT) yt_emit_lane_kernel(YtBatchDev b, CfgDev cfg, YtOut o, const uint64_t* line_off, uint8_t* out, int* err) {
  const int wid = threadIdx.x >> 5, l = lane_id();
  const uint64_t ngroups = (b.n + 31) / 32, nwarps = (uint64_t)gridDim.x * WARPS_PER_CTA;
  for (uint64_t g = (uint64_t)blockIdx.x * WARPS_PER_CTA + wid; g < ngroups; g += nwarps) {
    const uint64_t r = g * 32 + l;
    const bool active = r < b.n && o.status[r] == TGI_ST_EMITTED && o.esc_len[3 * r + 2];
    YtLaneWriter w;
    if (active) {
      w.el[0] = o.esc_len[3 * r];
      w.el[1] = o.esc_len[3 * r + 1];
      YtArgs a;
      a.b = &b;
      a.cfg = &cfg;
      a.r = r;
      a.urls = o.urls + o.url_start[r];
      a.n_urls = o.url_count[r];
      w.begin((uint64_t)(uintptr_t)out + line_off[r]);
      walk_yt_record(w, a);
      w.end();
      if (w.s.pos != (uint64_t)(uintptr_t)out + line_off[r + 1]) atomicOr(err, ERR_LINE_MISMATCH);
    }
    __syncwarp();
    w.flush_pending(active);
  }
}

// ---- message-status join (SURVEY 8f rank 2): first index in A of every key of B ---------------------------------
DEVI uint64_t join_hash(long long chat, long long msg) {  // splitmix64 finaliser over both words
  uint64_t x = (uint64_t)chat * 0x9E3779B97F4A7C15ull ^ (uint64_t)msg;
  x ^= x >> 30; x *= 0xBF58476D1CE4E5B9ull;
  x ^= x >> 27; x *= 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
// table[slot] = 1 + smallest index of an A element with that slot's key, 0 = empty
__global__ void join_build_kernel(const longlong2* a, uint64_t na, uint32_t* table, uint64_t mask) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= na) return;
  const longlong2 k = a[i];
  for (uint64_t s = join_hash(k.x, k.y) & mask;; s = (s + 1) & mask) {
    uint32_t cur = atomicCAS(&table[s], 0u, (uint32_t)i + 1u);
    if (cur == 0) return;  // claimed
    const longlong2 o = a[cur - 1];  // the occupant's key never changes (only its index may get smaller)
    if (o.x == k.x && o.y == k.y) {
      atomicMin(&table[s], (uint32_t)i + 1u);
      return;
    }
  }
}
__global__ void join_probe_kernel(const longlong2* a, const uint32_t* table, uint64_t mask, const longlong2* b, uint64_t nb, long long* out) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nb) return;
  const longlong2 k = b[i];
  long long res = -1;
  for (uint64_t s = join_hash(k.x, k.y) & mask;; s = (s + 1) & mask) {
    const uint32_t cur = table[s];
    if (cur == 0) break;
    const longlong2 o = a[cur - 1];
    if (o.x == k.x && o.y == k.y) {
      res = (long long)cur - 1;
      break;
    }
  }
  out[i] = res;
}

// ---- generic client.Message -> sparse Post (a12) ---------------------------------------------------
__global__ void __launch_bounds__(CTA_THREADS, 4) gm_size_kernel(GmBatchDev b, CfgDev cfg, uint8_t* status, uint32_t* linelen) {
  __shared__ YtScratch scs[WARPS_PER_CTA];
  int wid = threadIdx.x >> 5, l = lane_id();
  uint64_t nwarps = (uint64_t)gridDim.x * WARPS_PER_CTA;
  for (uint64_t r = (uint64_t)blockIdx.x * WARPS_PER_CTA + wid; r < b.n; r += nwarps) {
    YtSizer z;
    z.sc = &scs[wid];
    bool ok = walk_gm_record(z, b, cfg, r);
    if (l == 0) {
      status[r] = ok ? TGI_ST_EMITTED : TGI_ST_NOLINE;
      linelen[r] = ok ? (uint32_t)z.total : 0u;
    }
  }
}
__global__ void __launch_bounds__(CTA_THREADS, 4) gm_emit_kernel(GmBatchDev b, CfgDev cfg, const uint8_t* status, const uint64_t* line_off,
                                                                 uint8_t* out, int* err) {
  __shared__ YtScratch scs[WARPS_PER_CTA];
  int wid = threadIdx.x >> 5, l = lane_id();
  uint64_t nwarps = (uint64_t)gridDim.x * WARPS_PER_CTA;
  for (uint64_t r = (uint64_t)blockIdx.x * WARPS_PER_CTA + wid; r < b.n; r += nwarps) {
    if (status[r] != TGI_ST_EMITTED) continue;
    YtWriter w;
    w.sc = &scs[wid];
    w.p = out + line_off[r];
    walk_gm_record(w, b, cfg, r);
    if (l == 0 && (uint64_t)(w.p - out) != line_off[r + 1]) atomicOr(err, ERR_LINE_MISMATCH);
  }
}

// ---- channel records -> ChannelData lines (StoreChannelData) -------------------------------------------
// big batches only (small ones are checked by the host): bad[0] gets the lowest record whose ranges leave strs
__global__ void ch_validate_kernel(ChBatchDev b, uint64_t strs_len, unsigned long long* bad) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < b.n; i += (uint64_t)gridDim.x * blockDim.x)
    if (!ch_rec_ok(b.recs[i], strs_len)) atomicMin(bad, (unsigned long long)i);
}
__global__ void __launch_bounds__(CTA_THREADS, 4) ch_size_kernel(ChBatchDev b, uint8_t* status, uint32_t* linelen) {
  __shared__ YtScratch scs[WARPS_PER_CTA];
  int wid = threadIdx.x >> 5, l = lane_id();
  uint64_t nwarps = (uint64_t)gridDim.x * WARPS_PER_CTA;
  for (uint64_t r = (uint64_t)blockIdx.x * WARPS_PER_CTA + wid; r < b.n; r += nwarps) {
    YtSizer z;
    z.sc = &scs[wid];
    walk_ch_record(z, b, r);
    if (l == 0) {
      status[r] = TGI_ST_EMITTED;  // json.Marshal of a ChannelData cannot fail
      linelen[r] = (uint32_t)z.total;
    }
  }
}
__global__ void __launch_bounds__(CTA_THREADS, 4) ch_emit_kernel(ChBatchDev b, const uint64_t* line_off, uint8_t* out, int* err) {
  __shared__ YtScratch scs[WARPS_PER_CTA];
  int wid = threadIdx.x >> 5, l = lane_id();
  uint64_t nwarps = (uint64_t)gridDim.x * WARPS_PER_CTA;
  for (uint64_t r = (uint64_t)blockIdx.x * WARPS_PER_CTA + wid; r < b.n; r += nwarps) {
    YtWriter w;
    w.sc = &scs[wid];
    w.p = out + line_off[r];
    walk_ch_record(w, b, r);
    if (l == 0 && (uint64_t)(w.p - out) != line_off[r + 1]) atomicOr(err, ERR_LINE_MISMATCH);
  }
}

// ---- exclusive scan u32 -> u64 (out has n+1 entries) ----------------------------------------------
constexpr int SCAN_THREADS = 256, SCAN_ITEMS = 8, SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

__device__ __forceinline__ uint64_t block_reduce_u64(uint64_t v, uint64_t* sm) {
  for (int d = 16; d; d >>= 1) v += __shfl_down_sync(FULL, v, d);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
  __syncthreads();
  uint64_t t = 0;
  if (threadIdx.x < 32) {
    t = threadIdx.x < (blockDim.x >> 5) ? sm[threadIdx.x] : 0;
    for (int d = 16; d; d >>= 1) t += __shfl_down_sync(FULL, t, d);
  }
  return t;  // valid in thread 0
}

__global__ void __launch_bounds__(SCAN_THREADS) scan_tile_sums_kernel(const uint32_t* in, uint64_t n, uint64_t* tile_sums) {
  __shared__ uint64_t sm[32];
  uint64_t base = (uint64_t)blockIdx.x * SCAN_TILE;
  uint64_t s = 0;
  for (int k = 0; k < SCAN_ITEMS; k++) {
    uint64_t i = base + (uint64_t)k * SCAN_THREADS + threadIdx.x;
    if (i < n) s += in[i];
  }
  uint64_t t = block_reduce_u64(s, sm);
  if (threadIdx.x == 0) tile_sums[blockIdx.x] = t;
}

// single block: exclusive scan of tile sums in place; total -> out_total
__global__ void __launch_bounds__(1024) scan_tiles_kernel(uint64_t* tile_sums, uint64_t ntiles, uint64_t* out_total) {
  __shared__ uint64_t sm[32];
  __shared__ uint64_t carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (uint64_t base = 0; base < ntiles; base += 1024) {
    uint64_t i = base + threadIdx.x;
    uint64_t v = i < ntiles ? tile_sums[i] : 0;
    uint64_t x = v;
    int l = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int d = 1; d < 32; d <<= 1) {
      uint64_t t = __shfl_up_sync(FULL, x, d);
      if (l >= d) x += t;
    }
    if (l == 31) sm[w] = x;
    __syncthreads();
    if (w == 0) {
      uint64_t y = sm[l];
      for (int d = 1; d < 32; d <<= 1) {
        uint64_t t = __shfl_up_sync(FULL, y, d);
        if (l >= d) y += t;
      }
      sm[l] = y;
    }
    __syncthreads();
    uint64_t carry = carry_s;
    uint64_t incl = x + (w ? sm[w - 1] : 0);
    if (i < ntiles) tile_sums[i] = carry + incl - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = carry + incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) *out_total = carry_s;
}

__global__ void __launch_bounds__(SCAN_THREADS) scan_apply_kernel(const uint32_t* in, uint64_t n, const uint64_t* tile_base,
                                                               const uint64_t* total, uint64_t* out) {
  __shared__ uint64_t sm[32];
  // blocked arrangement: thread t owns items [t*ITEMS, (t+1)*ITEMS) of the tile
  uint64_t base = (uint64_t)blockIdx.x * SCAN_TILE + (uint64_t)threadIdx.x * SCAN_ITEMS;
  uint32_t v[SCAN_ITEMS];
  uint64_t s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    v[k] = base + k < n ? in[base + k] : 0;
    s += v[k];
  }
  uint64_t x = s;
  int l = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int d = 1; d < 32; d <<= 1) {
    uint64_t t = __shfl_up_sync(FULL, x, d);
    if (l >= d) x += t;
  }
  if (l == 31) sm[w] = x;
  __syncthreads();
  if (w == 0) {
    uint64_t y = l < (SCAN_THREADS >> 5) ? sm[l] : 0;
    for (int d = 1; d < 32; d <<= 1) {
      uint64_t t = __shfl_up_sync(FULL, y, d);
      if (l >= d) y += t;
    }
    sm[l] = y;
  }
  __syncthreads();
  uint64_t excl = tile_base[blockIdx.x] + (w ? sm[w - 1] : 0) + x - s;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    if (base + k < n) out[base + k] = excl;
    excl += v[k];
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) out[n] = *total;
}

// the whole scan in ONE launch for page-sized batches (n <= SCAN_SMALL_MAX): one CTA, SCAN_SMALL_ITEMS per thread
constexpr int SCAN_SMALL_THREADS = 1024, SCAN_SMALL_ITEMS = 8, SCAN_SMALL_MAX = SCAN_SMALL_THREADS * SCAN_SMALL_ITEMS;
__global__ void __launch_bounds__(SCAN_SMALL_THREADS) scan_small_kernel(const uint32_t* in, uint64_t n, uint64_t* out, uint64_t* out_total) {
  __shared__ uint64_t sm[32];
  const uint64_t base = (uint64_t)threadIdx.x * SCAN_SMALL_ITEMS;
  uint32_t v[SCAN_SMALL_ITEMS];
  uint64_t s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_SMALL_ITEMS; k++) {
    v[k] = base + k < n ? in[base + k] : 0;
    s += v[k];
  }
  uint64_t x = s;
  const int l = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int d = 1; d < 32; d <<= 1) {
    const uint64_t t = __shfl_up_sync(FULL, x, d);
    if (l >= d) x += t;
  }
  if (l == 31) sm[w] = x;
  __syncthreads();
  if (w == 0) {
    uint64_t y = sm[l];
    for (int d = 1; d < 32; d <<= 1) {
      const uint64_t t = __shfl_up_sync(FULL, y, d);
      if (l >= d) y += t;
    }
    sm[l] = y;
  }
  __syncthreads();
  uint64_t excl = (w ? sm[w - 1] : 0) + x - s;
#pragma unroll
  for (int k = 0; k < SCAN_SMALL_ITEMS; k++) {
    if (base + k < n) out[base + k] = excl;
    excl += v[k];
  }
  if (threadIdx.x == SCAN_SMALL_THREADS - 1) {
    out[n] = sm[31];
    *out_total = sm[31];
  }
}

// ---- frontier: exact hash set of 32-byte keys ------------------------------------------------------
struct FrontierDev {
  uint8_t* pool;     // [cap][32] distinct keys in first-occurrence order
  uint64_t cap;
  uint64_t* table;   // persistent table: 0 = empty, else (pool_idx+1) | fp << 40
  uint64_t tmask;
  uint64_t* count;   // device scalar: number of keys in the pool
  uint64_t* payload; // optional [cap]: 64-bit payload of every key (the owned partition of the multi-GPU merge)
};
struct FrontierBatch {
  uint64_t* btable;  // per-batch table: 0 = empty, else ((rec << SEQ_ORD_BITS) | ordinal) + 1 (atomicMin'd)
  uint64_t bmask;
  uint32_t* lstate;  // per arena slot: LS_* or batch-table slot index
  uint32_t* rec_new; // [n] new keys first seen in this record
};
// sequence number of a link inside a batch: (record << 20) | ordinal.  Records < 2^40 (checked by the host), so a
// record may carry up to 2^20 link candidates (> 10 MB of text: beyond anything TDLib delivers; the host checks)
constexpr int SEQ_ORD_BITS = 20;
#define LS_INELIGIBLE 0xFFFFFFFFu
#define LS_KNOWN 0xFFFFFFFEu

struct Key32 {
  uint32_t w[8];
};
DEVI Key32 load_key(const uint8_t* p) {  // 4-byte aligned
  Key32 k;
  const uint32_t* q = (const uint32_t*)p;
#pragma unroll
  for (int i = 0; i < 8; i++) k.w[i] = q[i];
  return k;
}
DEVI void store_key(uint8_t* p, const Key32& k) {  // 4-byte aligned
  uint32_t* q = (uint32_t*)p;
#pragma unroll
  for (int i = 0; i < 8; i++) q[i] = k.w[i];
}
DEVI bool key_eq(const Key32& a, const Key32& b) {
  uint32_t d = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) d |= a.w[i] ^ b.w[i];
  return d == 0;
}
DEVI uint64_t key_hash(const Key32& k) {
  uint64_t h = 0x9E3779B97F4A7C15ull;
#pragma unroll
  for (int i = 0; i < 8; i += 2) {
    uint64_t x = (uint64_t)k.w[i] | ((uint64_t)k.w[i + 1] << 32);
    h = (h ^ x) * 0xFF51AFD7ED558CCDull;
    h ^= h >> 32;
  }
  h *= 0xC4CEB9FE1A85EC53ull;
  return h ^ (h >> 29);
}

// whether set f holds `key` (hash h), and if so its pool index pi.  Table entry: (pool index + 1) | fingerprint << 40,
// placed by set_place.
DEVI bool set_probe(const FrontierDev& f, const Key32& key, uint64_t h, uint64_t& pi) {
  const uint64_t fp = (h >> 40) | 1ull;  // 24-bit fingerprint, never 0
  for (uint64_t s = h & f.tmask;; s = (s + 1) & f.tmask) {
    const uint64_t e = f.table[s];
    if (e == 0) return false;
    if ((e >> 40) == fp) {
      pi = (e & 0xFFFFFFFFFFull) - 1;
      if (key_eq(key, load_key(f.pool + 32 * pi))) return true;
    }
  }
}
// pool index of `key` in exclusion set f, or -1: before its first tgi_set_add a set has no table and holds nothing
DEVI int64_t set_lookup(const FrontierDev& f, const Key32& key, uint64_t h) {
  uint64_t pi;
  return f.table && set_probe(f, key, h, pi) ? (int64_t)pi : -1;
}
// enters the key with hash h at pool index pi into f.table: the only writer of table entries, so the append and the
// rehash of a growing set produce the same table
DEVI void set_place(const FrontierDev& f, uint64_t pi, uint64_t h) {
  const uint64_t e = (pi + 1) | (((h >> 40) | 1ull) << 40);
  for (uint64_t s = h & f.tmask;; s = (s + 1) & f.tmask) {
    if (f.table[s] == 0 && atomicCAS((unsigned long long*)&f.table[s], 0ull, (unsigned long long)e) == 0) break;
  }
}
// the resident exclusion sets of the frontier -> validator hand-off (tgi_set_add): invalid channels expire after
// TGI_INVALID_TTL_SEC (state/daprstate.go:3556-3564: time.Since(t) < invalidChannelTTL), stamp 0 = never
struct ExclusionDev {
  FrontierDev invalid, discovered;
  long long now_sec;
};
DEVI bool set_invalid_hit(const ExclusionDev& x, const Key32& key, uint64_t h, long long now_sec) {
  const int64_t pi = set_lookup(x.invalid, key, h);
  if (pi < 0) return false;
  const long long t = (long long)x.invalid.payload[pi];
  return t == 0 || now_sec - t < (long long)TGI_INVALID_TTL_SEC;
}

DEVI bool link_eligible(const tgi_link& lk, uint32_t run_flags) {
  if ((run_flags & TGI_RUN_SKIP_SELF) && (lk.flags & TGI_LF_SELF)) return false;    // runner.go:1231
  if ((run_flags & TGI_RUN_FILTER) && !(lk.flags & TGI_LF_FILTER_OK)) return false; // runner.go:1261
  return true;
}

// phase 1: probe the persistent set; unseen keys race into the batch table, min sequence wins
DEVI void frontier_probe_body(uint64_t n, const uint32_t* link_start, const uint32_t* link_count, tgi_link* arena,
                              uint32_t run_flags, const FrontierDev& f, const FrontierBatch& fb, const ExclusionDev& x,
                              uint64_t t0, uint64_t nt) {  // thread t0 of nt: the whole grid, or one CTA (page kernel)
 for (uint64_t r = t0; r < n; r += nt) {
  uint32_t cnt = link_count[r];
  if (!cnt) continue;
  uint32_t ls = link_start ? link_start[r] : (uint32_t)r;
  for (uint32_t k = 0; k < cnt; k++) {
    uint32_t idx = ls + k;
    tgi_link& lk = arena[idx];
    if ((run_flags & TGI_RUN_SKIP_SELF) && (lk.flags & TGI_LF_SELF)) {  // runner.go:1231
      fb.lstate[idx] = LS_INELIGIBLE;
      continue;
    }
    Key32 key = load_key(lk.name);
    uint64_t h = key_hash(key);
    if ((run_flags & TGI_RUN_SKIP_INVALID) && set_invalid_hit(x, key, h, x.now_sec)) {  // runner.go:1247 (before the filter)
      lk.flags |= TGI_LF_INVALID;
      fb.lstate[idx] = LS_INELIGIBLE;
      continue;
    }
    if ((run_flags & TGI_RUN_FILTER) && !(lk.flags & TGI_LF_FILTER_OK)) {  // runner.go:1261
      fb.lstate[idx] = LS_INELIGIBLE;
      continue;
    }
    uint64_t pi;
    if (set_probe(f, key, h, pi)) {
      fb.lstate[idx] = LS_KNOWN;
      continue;
    }
    uint64_t v = (((uint64_t)r << SEQ_ORD_BITS) | k) + 1;
    for (uint64_t s = (h >> 7) & fb.bmask;; s = (s + 1) & fb.bmask) {
      uint64_t cur = fb.btable[s];
      if (cur == 0) {
        cur = atomicCAS((unsigned long long*)&fb.btable[s], 0ull, (unsigned long long)v);
        if (cur == 0) {
          fb.lstate[idx] = (uint32_t)s;
          break;
        }
      }
      uint64_t r2 = (cur - 1) >> SEQ_ORD_BITS, k2 = (cur - 1) & ((1u << SEQ_ORD_BITS) - 1u);
      uint32_t ls2 = link_start ? link_start[r2] : (uint32_t)r2;
      if (key_eq(key, load_key(arena[ls2 + k2].name))) {
        atomicMin((unsigned long long*)&fb.btable[s], (unsigned long long)v);
        fb.lstate[idx] = (uint32_t)s;
        break;
      }
    }
  }
 }
}
__global__ void frontier_probe_kernel(uint64_t n, const uint32_t* link_start, const uint32_t* link_count,
                                      tgi_link* arena, uint32_t run_flags, FrontierDev f, FrontierBatch fb, ExclusionDev x) {
  frontier_probe_body(n, link_start, link_count, arena, run_flags, f, fb, x, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, (uint64_t)gridDim.x * blockDim.x);
}

// phase 2: per record, how many of its links are the global first occurrence of a new key
DEVI void frontier_count_body(uint64_t n, const uint32_t* link_start, const uint32_t* link_count, const FrontierBatch& fb,
                              uint64_t t0, uint64_t nt) {
  for (uint64_t r = t0; r < n; r += nt) {
    uint32_t cnt = link_count[r], c = 0;
    uint32_t ls = link_start ? link_start[r] : (uint32_t)r;
    for (uint32_t k = 0; k < cnt; k++) {
      uint32_t st = fb.lstate[ls + k];
      if (st >= LS_KNOWN) continue;
      if (fb.btable[st] == (((uint64_t)r << SEQ_ORD_BITS) | k) + 1) c++;
    }
    fb.rec_new[r] = c;
  }
}
__global__ void frontier_count_kernel(uint64_t n, const uint32_t* link_start, const uint32_t* link_count,
                                      FrontierBatch fb) {
  frontier_count_body(n, link_start, link_count, fb, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, (uint64_t)gridDim.x * blockDim.x);
}

// phase 3: append the new keys to the pool in (record, ordinal) order and publish them
DEVI void frontier_append_body(uint64_t n, const uint32_t* link_start, const uint32_t* link_count, tgi_link* arena,
                               const FrontierDev& f, const FrontierBatch& fb, const uint64_t* new_off, int* err,
                               const uint64_t* payload_in, uint64_t t0, uint64_t nt) {
 for (uint64_t r = t0; r < n; r += nt) {
  if (!fb.rec_new[r]) continue;
  uint64_t base = *f.count, total = new_off[n];
  if (base + total > f.cap) {
    atomicOr(err, ERR_FRONTIER_FULL);
    return;
  }
  uint32_t cnt = link_count[r];
  uint32_t ls = link_start ? link_start[r] : (uint32_t)r;
  uint64_t pi = base + new_off[r];
  for (uint32_t k = 0; k < cnt; k++) {
    uint32_t st = fb.lstate[ls + k];
    if (st >= LS_KNOWN) continue;
    if (fb.btable[st] != (((uint64_t)r << SEQ_ORD_BITS) | k) + 1) continue;
    tgi_link& lk = arena[ls + k];
    Key32 key = load_key(lk.name);
    store_key(f.pool + 32 * pi, key);
    if (f.payload) f.payload[pi] = payload_in ? payload_in[r] : 0ull;  // keys mode: one key per "record"
    set_place(f, pi, key_hash(key));
    lk.flags |= TGI_LF_NEW;
    pi++;
  }
 }
}
__global__ void frontier_append_kernel(uint64_t n, const uint32_t* link_start, const uint32_t* link_count,
                                       tgi_link* arena, FrontierDev f, FrontierBatch fb,
                                       const uint64_t* new_off, int* err, const uint64_t* payload_in = nullptr) {
  frontier_append_body(n, link_start, link_count, arena, f, fb, new_off, err, payload_in, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, (uint64_t)gridDim.x * blockDim.x);
}
DEVI void frontier_commit_body(const FrontierDev& f, const uint64_t* new_off, uint64_t n, uint64_t* out_new, int* err) {
  uint64_t total = new_off[n];
  if (*f.count + total <= f.cap) {
    *f.count += total;
    *out_new = total;
  } else {
    *out_new = 0;
    atomicOr(err, ERR_FRONTIER_FULL);
  }
  out_new[1] = *f.count;
}
__global__ void frontier_commit_kernel(FrontierDev f, const uint64_t* new_off, uint64_t n, uint64_t* out_new, int* err) {
  frontier_commit_body(f, new_off, n, out_new, err);
}

// growth of a set (tgi_set_growth): index the first n keys of f.pool (already copied from the smaller set) in f.table,
// zeroed.  The entries are placed by set_place, as in frontier_append_body; the pool order is untouched, so the export
// order and the NEW flags of later batches are those of a set that was big enough from the start.
__global__ void set_rehash_kernel(FrontierDev f, uint64_t n) {
  const uint64_t pi = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pi >= n) return;
  set_place(f, pi, key_hash(load_key(f.pool + 32 * pi)));
}

// ---- multi-GPU merge (SURVEY 8e option A): bucket the new local keys by owner rank ----------------------------------
DEVI uint32_t key_owner(const Key32& k, uint32_t nranks) { return (uint32_t)((key_hash(k) >> 17) % nranks); }
__global__ void merge_count_kernel(const uint8_t* pool, uint64_t first, uint64_t m, uint32_t nranks, unsigned long long* cnt) {
  __shared__ unsigned int sc[64];
  if (threadIdx.x < 64) sc[threadIdx.x] = 0;
  __syncthreads();
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) atomicAdd(&sc[key_owner(load_key(pool + 32 * (first + i)), nranks)], 1u);
  __syncthreads();
  if (threadIdx.x < nranks && sc[threadIdx.x]) atomicAdd(&cnt[threadIdx.x], (unsigned long long)sc[threadIdx.x]);
}
// cursor[p] starts at the offset of bucket p in the send buffers; the order inside a bucket is irrelevant (the keys
// of one rank are distinct and every key carries its sequence number)
__global__ void merge_scatter_kernel(const uint8_t* pool, uint64_t first, uint64_t m, uint32_t nranks, unsigned long long* cursor,
                                     uint8_t* send_keys, uint64_t* send_pay, uint64_t pay_base) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const Key32 k = load_key(pool + 32 * (first + i));
  const unsigned long long pos = atomicAdd(&cursor[key_owner(k, nranks)], 1ull);
  store_key(send_keys + 32 * pos, k);
  send_pay[pos] = pay_base | (first + i);
}

// ---- frontier -> validator hand-off (SURVEY 8f rank 3): the new edges of a batch as packed pending_edges rows --------
// rec_new / new_off are what the frontier phase of the batch left behind: row index = new_off[r] + ordinal among the
// record's NEW links, i.e. (record, first-insertion) order — the order of the reference's INSERTs.
__global__ void edges_emit_kernel(uint64_t n, const uint32_t* link_start, const uint32_t* link_count, const tgi_link* arena,
                                  const uint32_t* chan_idx_of, uint32_t chan_stride, const uint64_t* new_off, ExclusionDev x,
                                  tgi_edge* rows, uint64_t cap) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const uint32_t cnt = link_count[r];
  if (!cnt) return;
  uint64_t row = new_off[r];
  const tgi_link* lk = arena + link_start[r];
  for (uint32_t k = 0; k < cnt; k++) {
    if (!(lk[k].flags & TGI_LF_NEW)) continue;
    if (row < cap) {
      const Key32 key = load_key(lk[k].name);
      const uint64_t h = key_hash(key);
      tgi_edge e;
      store_key(e.destination, key);
      e.record = r;
      e.chan_idx = chan_idx_of ? *(const uint32_t*)((const uint8_t*)chan_idx_of + (size_t)r * chan_stride) : 0u;
      e.dest_len = lk[k].len;
      e.source_type = lk[k].src;
      e.status = set_invalid_hit(x, key, h, x.now_sec) ? TGI_EDGE_INVALID_CACHED           // validator.go:205-212
                 : set_lookup(x.discovered, key, h) >= 0 ? TGI_EDGE_DUPLICATE : TGI_EDGE_PENDING;  // :214-226
      e.reserved = 0;
      rows[row] = e;
    }
    row++;
  }
}

// keys32 -> pseudo arena (one link per "record") for tgi_frontier_insert
__global__ void keys_to_links_kernel(const uint8_t* keys, uint64_t n, tgi_link* arena, uint32_t* link_count) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  tgi_link lk;
  int len = 0;
  for (int k = 0; k < 32; k++) {
    lk.name[k] = keys[32 * i + k];
    if (lk.name[k]) len = k + 1;
  }
  lk.len = (uint8_t)len;
  lk.src = 0;
  lk.flags = 0;
  lk.filter_reason = 0;
  arena[i] = lk;
  link_count[i] = 1;
}
__global__ void links_new_flags_kernel(const tgi_link* arena, uint64_t n, uint8_t* is_new) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) is_new[i] = (arena[i].flags & TGI_LF_NEW) ? 1 : 0;
}

// ---- compaction of the per-record links for the host result -----------------------------------------
DEVI void links_compact_body(uint64_t n, const uint32_t* link_start, const uint32_t* link_count, const uint64_t* link_off,
                             const tgi_link* arena, tgi_link* out, uint32_t* link_off32) {
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= n; r += (uint64_t)gridDim.x * blockDim.x) {
    link_off32[r] = (uint32_t)link_off[r];
    if (r == n) break;
    uint32_t cnt = link_count[r];
    const uint32_t* src = (const uint32_t*)(arena + link_start[r]);
    uint32_t* dst = (uint32_t*)(out + link_off[r]);
    for (uint32_t k = 0; k < cnt * 9; k++) dst[k] = src[k];
  }
}
__global__ void links_compact_kernel(uint64_t n, const uint32_t* link_start, const uint32_t* link_count,
                                     const uint64_t* link_off, const tgi_link* arena, tgi_link* out,
                                     uint32_t* link_off32) {
  links_compact_body(n, link_start, link_count, link_off, arena, out, link_off32);
}

// FilterUsername over a list of names (tgi_filter_usernames): one warp per name
__global__ void filter_usernames_kernel(const uint8_t* names, const uint32_t* off, uint64_t n, uint8_t* reason) {
  uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= n) return;
  int l = lane_id();
  uint32_t a = off[i], len = off[i + 1] - a;
  uint32_t c = ((uint32_t)l < len) ? ldb(names + a + l) : 0u;
  uint32_t res = warp_filter_username(c, len);  // names longer than a warp stop at too_long
  if (l == 0) reason[i] = (uint8_t)res;
}

}  // namespace tgi
