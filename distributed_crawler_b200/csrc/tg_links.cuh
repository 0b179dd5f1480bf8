// tg_links.cuh — warp-parallel link extraction for one Telegram record.
//
// Replaces telegramhelper/tdutils.go:897-949 extractLinksFromFormattedText (+ channelNameFromMatch
// :36-45, utf16OffsetToBytes :55-78, usernameRegex :82) and telegramhelper/username_filter.go:26-68.
// The two regexes are evaluated as hand-written scanners over 128-byte strips (4 bytes per lane):
//   channelLinkRegex (https?://)?t\.me/([a-zA-Z][a-zA-Z0-9_]{4,31})  -> find "t.me/" with a 40-bit
//     compare at every byte position, then validate the name; RE2 leftmost-first / non-overlapping
//     semantics are kept by processing candidates in position order with a `resume` cursor.
//   usernameRegex (?:@)?([a-zA-Z][a-zA-Z0-9_]{4,31}) -> first letter followed by >= 4 word chars.
#pragma once
#include "dev_common.cuh"

namespace tgi {

struct LinkSink {
  tgi_link* out;       // arena slots of this record (reserved: `cap` entries)
  uint32_t cap;
  uint32_t count;      // links written so far (warp-uniform)
  uint32_t name_bytes; // sum of their name lengths (the size pass turns it into the outlinks piece length)
  const uint8_t* self; // channel name of the record (for TGI_LF_SELF)
  uint32_t self_len;
};

// FilterUsername (username_filter.go:26-68) on a name held one byte per lane (c = 0 beyond len).
// Evaluation order of the reasons is the reference's.
DEVI uint32_t warp_filter_username(uint32_t c, uint32_t len) {
  int l = lane_id();
  if (len < 5) return TGI_FU_TOO_SHORT;
  if (len > 32) return TGI_FU_TOO_LONG;
  uint32_t first = __shfl_sync(FULL, c, 0);
  if (!is_letter(first)) return TGI_FU_INVALID_START_CHAR;
  uint32_t last = __shfl_sync(FULL, c, (int)len - 1);
  if (last == '_') return TGI_FU_ENDS_WITH_UNDERSCORE;
  bool bad = (uint32_t)l < len && !is_word(c);  // any byte >= 0x80 is (part of) a non-ASCII rune
  if (__any_sync(FULL, bad)) return TGI_FU_INVALID_CHAR;
  // looks_like_path is unreachable after the charset check ('/', '\\', '~', '.' are not word chars)
  uint32_t a = ascii_lower(__shfl_sync(FULL, c, (int)len - 3));
  uint32_t b = ascii_lower(__shfl_sync(FULL, c, (int)len - 2));
  uint32_t d = ascii_lower(last);
  if (a == 'b' && b == 'o' && d == 't') return TGI_FU_BOT_SUFFIX;
  return TGI_FU_VALID;
}

// telegramReservedPaths (tdutils.go:27-32); only the >= 5 char members can match a regex capture.
DEVI bool warp_is_reserved(uint32_t c, uint32_t len) {
  int l = lane_id();
  const char* w[10] = {"share", "proxy", "socks", "login", "addlist", "confirm", "joinchat",
                       "addtheme", "addstickers", "setlanguage"};
  const uint32_t wl[10] = {5, 5, 5, 5, 7, 7, 8, 8, 11, 11};
  bool res = false;
#pragma unroll
  for (int k = 0; k < 10; k++) {
    if (wl[k] == len) {
      bool eq = (uint32_t)l >= len || c == (uint32_t)w[k][l < 11 ? l : 0];
      if (__all_sync(FULL, eq)) res = true;
    }
  }
  return res;
}

// addIfNew (tdutils.go:902-906) on a candidate name at p[0..len): lower-case, optional reserved
// filter, dedup against the record's earlier links, append.  c-per-lane representation.
__device__ __noinline__ void warp_add_link(LinkSink& ls, const uint8_t* p, uint32_t len, uint32_t src, bool channel_rule) {
  int l = lane_id();
  uint32_t c = (uint32_t)l < len ? ascii_lower(ldb(p + l)) : 0u;
  if (channel_rule && warp_is_reserved(c, len)) return;
  for (uint32_t j = 0; j < ls.count; j++) {
    uint32_t o = ls.out[j].name[l];
    if (__all_sync(FULL, o == c)) return;  // zero padded on both sides => also compares lengths
  }
  if (ls.count >= ls.cap) return;  // cannot happen: cap is an upper bound computed by the count pass
  uint32_t reason = warp_filter_username(c, len);
  bool self = len == ls.self_len &&
              __all_sync(FULL, (uint32_t)l >= len || c == ldb(ls.self + (l < (int)len ? l : 0)));
  tgi_link* d = &ls.out[ls.count];
  d->name[l] = (uint8_t)c;
  if (l == 0) {
    d->len = (uint8_t)len;
    d->src = (uint8_t)src;
    d->flags = (uint8_t)((reason == TGI_FU_VALID ? TGI_LF_FILTER_OK : 0) | (self ? TGI_LF_SELF : 0));
    d->filter_reason = (uint8_t)reason;
  }
  __syncwarp();
  ls.count++;
  ls.name_bytes += len;
}

// greedy [a-zA-Z0-9_]{0,32} run length starting at p (bounded by end)
DEVI uint32_t warp_word_run(const uint8_t* p, const uint8_t* end) {
  int l = lane_id();
  bool ok = p + l < end && is_word(ldb(p + l));
  uint32_t m = __ballot_sync(FULL, !ok);
  return m ? (uint32_t)(__ffs(m) - 1) : 32u;
}

// A strip for the link scan = 512 bytes, 16 per lane (no UTF-8 bookkeeping is needed to find "t.me/").
// Returns the lane's 16-bit mask: bit k set if s[p0+k] is the '/' of a "t.me/" (p0 = base + 16*lane).
// '/' is rare in message text, so almost every strip ends after four SWAR compares per lane.
// tme16 computes it from the lane's bytes w = s[p0..p0+16), p0 < n.
DEVI uint32_t tme16(const uint8_t* s, int64_t p0, int64_t n, const uint4 w) {
  const uint8_t* q = s + p0;
  const uint32_t s0 = swar_eq(w.x, '/'), s1 = swar_eq(w.y, '/'), s2 = swar_eq(w.z, '/'), s3 = swar_eq(w.w, '/');
  if (!(s0 | s1 | s2 | s3)) return 0;
  uint32_t m = swar_movemask(s0) | (swar_movemask(s1) << 4) | (swar_movemask(s2) << 8) | (swar_movemask(s3) << 12);
  const int64_t rem = n - p0;
  if (rem < 16) m &= (1u << rem) - 1u;
  uint32_t out = 0;
  while (m) {
    const int k = __ffs(m) - 1;
    m &= m - 1;
    if (p0 + k >= 4 && ld_u32_unaligned(q + k - 4) == 0x656D2E74u) out |= 1u << k;  // "t.me"
  }
  return out;
}
DEVI uint32_t strip16_tme(const uint8_t* s, int64_t base, int64_t n) {
  const int64_t p0 = base + 16 * lane_id();
  if (p0 >= n) return 0;
  return tme16(s, p0, n, ld16_unaligned(s + p0));
}

// index of the first byte >= 0x80 of s[0..n), n if there is none.  In front of it UTF-16 offsets are byte offsets.
DEVI int64_t warp_first_non_ascii(const uint8_t* s, int64_t n) {
  for (int64_t base = 0; base < n; base += 512) {
    const int64_t p0 = base + 16 * lane_id();
    uint32_t m = 0;
    if (p0 < n) {
      const uint4 w = ld16_unaligned(s + p0);
      m = swar_movemask(w.x & 0x80808080u) | (swar_movemask(w.y & 0x80808080u) << 4) | (swar_movemask(w.z & 0x80808080u) << 8) |
          (swar_movemask(w.w & 0x80808080u) << 12);
      const int64_t rem = n - p0;
      if (rem < 16) m &= (1u << rem) - 1u;
    }
    const uint32_t lanes = __ballot_sync(FULL, m != 0);
    if (lanes) {
      const int src = __ffs(lanes) - 1;
      return base + 16 * src + (__ffs(__shfl_sync(FULL, m, src)) - 1);
    }
  }
  return n;
}

// number of "t.me/" occurrences in s[0..n): upper bound on plaintext matches
DEVI uint32_t warp_count_tme(const uint8_t* s, int64_t n) {
  uint32_t cnt = 0;
  for (int64_t base = 0; base < n; base += 512) cnt += __popc(strip16_tme(s, base, n));
  return warp_sum(cnt);
}

// The same count, and the text measured from the same 16 bytes per lane (JSONL runs): esc_len = its JSON-escaped length
// if it is clean (utf8_unclean4), 0 if not (or if n == 0).  The lane's 4 bytes in front come from the lane below, or
// for lane 0 from the previous strip's last lane.
DEVI uint32_t warp_count_tme_esc(const uint8_t* s, int64_t n, uint32_t& esc_len) {
  const int l = lane_id();
  const uint32_t SP = 0x20202020u;
  uint32_t cnt = 0, extra = 0, bad = 0, tail = SP;  // tail: the last 4 bytes of the previous strip
  for (int64_t base = 0; base < n; base += 512) {
    const int64_t p0 = base + 16 * l, rem = n - p0;
    uint4 w = make_uint4(SP, SP, SP, SP);
    if (rem > 0) {
      w = ld16_unaligned(s + p0);
      cnt += __popc(tme16(s, p0, n, w));
      if (rem < 16) w = make_uint4(blank_from(w.x, rem), blank_from(w.y, rem - 4), blank_from(w.z, rem - 8), blank_from(w.w, rem - 12));
    }
    const uint32_t below = __shfl_up_sync(FULL, w.w, 1);
    uint32_t pw = l == 0 ? tail : below;
    tail = __shfl_sync(FULL, w.w, 31);
    const bool ascii = ((w.x | w.y | w.z | w.w | pw) & 0x80808080u) == 0;
#pragma unroll 1
    for (int k = 0; k < 4; k++) {  // a word at a time: the parse kernels' code has to stay small (instruction cache)
      if (!ascii) bad |= utf8_unclean4(pw, w.x);
      extra += esc_extra4(w.x);
      pw = w.x;
      w = make_uint4(w.y, w.z, w.w, w.x);
    }
  }
  bad |= utf8_unclean4(tail, SP);  // a text that ends with its last strip: a sequence open at the end
  const uint32_t e = (uint32_t)n + warp_sum(extra);
  esc_len = __any_sync(FULL, bad != 0) ? 0u : e;
  return warp_sum(cnt);
}

// channelLinkRegex over s[0..n).  all == false: FindStringSubmatch (first match only, reserved names
// are dropped WITHOUT looking further).  all == true: FindAllStringSubmatch.
__device__ __noinline__ void warp_scan_channel_links(LinkSink& ls, const uint8_t* s, int64_t n, uint32_t src, bool all) {
  int64_t resume = 0;  // end of the previous match (non-overlapping search)
  for (int64_t base = 0; base < n; base += 512) {
    uint32_t m = strip16_tme(s, base, n);
    uint32_t lanes = __ballot_sync(FULL, m != 0);
    while (lanes) {
      int src_lane = __ffs(lanes) - 1;
      lanes &= lanes - 1;
      uint32_t mm = __shfl_sync(FULL, m, src_lane);
      while (mm) {
        int k = __ffs(mm) - 1;
        mm &= mm - 1;
        int64_t p = base + 16 * src_lane + k - 4;  // start of "t.me/"
        if (p < resume) continue;  // inside the previous match
        const uint8_t* q = s + p + 5;
        if (p + 5 >= n || !is_letter(ldb(q))) continue;
        uint32_t run = warp_word_run(q, s + n);
        if (run < 5) continue;
        warp_add_link(ls, q, run, src, true);
        if (!all) return;
        resume = p + 5 + run;
      }
    }
  }
}

// usernameRegex FindStringSubmatch over the mention slice s[0..n) (tdutils.go:920-929)
__device__ __noinline__ void warp_scan_username(LinkSink& ls, const uint8_t* s, int64_t n) {
  int l = lane_id();
  for (int64_t base = 0; base < n; base += 32) {
    int64_t q = base + l;
    bool cand = false;
    if (q < n && is_letter(ldb(s + q))) {
      cand = q + 5 <= n && is_word(ldb(s + q + 1)) && is_word(ldb(s + q + 2)) &&
             is_word(ldb(s + q + 3)) && is_word(ldb(s + q + 4));
    }
    uint32_t m = __ballot_sync(FULL, cand);
    if (m) {
      int64_t q0 = base + (__ffs(m) - 1);
      uint32_t run = warp_word_run(s + q0, s + n);
      warp_add_link(ls, s + q0, run, TGI_SRC_MENTION, false);
      return;
    }
  }
}

// utf16OffsetToBytes (tdutils.go:55-78).  Returns start/end exactly as Go does, including
// start == -1 with a valid end (the caller then marks the record FAILED: Go slices [-1:end] and
// panics) and the (0,0) / (start,len) fall-backs after the loop.
__device__ __noinline__ void warp_utf16_to_bytes(const uint8_t* s, int64_t n, int32_t off16, int32_t len16,
                              int64_t& start, int64_t& end) {
  int32_t stop = (int32_t)((uint32_t)off16 + (uint32_t)len16);
  int64_t rune_start = -1;
  uint32_t run = 0, carry = 0;  // u16pos at strip start (texts are < 2^31 units)
  int l = lane_id();
  for (int64_t base = 0; base < n; base += 128) {
    Strip st = warp_load_strip(s, base, n, carry);
    uint32_t e, u;
    strip_lane_totals(st, s, base, n, e, u);
    uint32_t incl = warp_incl_scan(u);
    {  // neither offset falls into this strip's units [run, run + total): nothing to look for (most strips of a long text)
      const uint32_t total = __shfl_sync(FULL, incl, 31);
      if ((uint32_t)off16 - run >= total && (uint32_t)stop - run >= total) {
        run += total;
        continue;
      }
    }
    uint32_t pos = run + incl - u;  // u16pos before this lane's first byte
    // visit the lane's rune starts in order
    int64_t hit_start = -1, hit_end = -1;
    for (uint32_t k = 0; k < st.nvalid; k++) {
      uint32_t units, is_start;
      if (st.exact) {
        ByteInfo bi = byte_info_exact(s, base + 4 * l + k, n);
        units = bi.u16;
        is_start = bi.start;
      } else {
        is_start = !((st.cont >> (8 * k + 7)) & 1u);
        units = is_start + ((st.l4 >> (8 * k + 7)) & 1u);  // 4-byte sequence = surrogate pair
      }
      if (is_start) {
        if ((int32_t)pos == off16 && hit_start < 0) hit_start = base + 4 * l + k;
        if ((int32_t)pos == stop && hit_end < 0) hit_end = base + 4 * l + k;
      }
      pos += units;
    }
    uint32_t ms = __ballot_sync(FULL, hit_start >= 0), me = __ballot_sync(FULL, hit_end >= 0);
    int64_t cs = -1, ce = -1;
    if (ms) cs = __shfl_sync(FULL, hit_start, __ffs(ms) - 1);
    if (me) ce = __shfl_sync(FULL, hit_end, __ffs(me) - 1);
    // Go checks "u16pos == off" before "u16pos == stop" at the same index, so a start found at
    // or before the end position counts; a start after the end position does not.
    if (ce >= 0) {
      if (cs >= 0 && cs <= ce) rune_start = cs;
      start = rune_start;
      end = ce;
      return;
    }
    if (cs >= 0) rune_start = cs;
    run += __shfl_sync(FULL, incl, 31);
  }
  if (rune_start == -1) {
    start = 0;
    end = 0;
  } else {
    start = rune_start;
    end = n;
  }
}

struct TgRecView {  // decoded view of one record, warp-uniform
  const tgi_tg_rec* rec;
  const uint8_t *text, *alt, *media, *handle;
  uint32_t text_len, alt_len, media_len, handle_len;
  uint32_t ct, flags;
  uint32_t e0, e1;
};

DEVI bool ct_carries_links(uint32_t ct) {  // extractFormattedTextFromMessage tdutils.go:953-972
  return ct == TGI_CT_TEXT || ct == TGI_CT_PHOTO || ct == TGI_CT_VIDEO || ct == TGI_CT_DOCUMENT ||
         ct == TGI_CT_ANIMATION || ct == TGI_CT_AUDIO || ct == TGI_CT_VOICE_NOTE;
}

// upper bound on the number of links of this record (entities of the three kinds + "t.me/" hits).  MEASURE: text_esc =
// the text's escaped length if the count found it clean, else 0 (warp_count_tme_esc); 0 for a record it does not scan.
template <bool MEASURE>
DEVI uint32_t warp_link_upper_bound(const TgRecView& v, const tgi_entity* ents, uint32_t& text_esc) {
  text_esc = 0;
  if (!ct_carries_links(v.ct) || !(v.flags & TGI_RF_HAS_TEXT)) return 0;
  uint32_t c = 0;
  for (uint32_t e = v.e0 + lane_id(); e < v.e1; e += 32) c += ents[e].type != TGI_ENT_OTHER;
  return warp_sum(c) + (MEASURE ? warp_count_tme_esc(v.text, v.text_len, text_esc) : warp_count_tme(v.text, v.text_len));
}

// utf16OffsetToBytes for every mention / url entity of the record -> ranges[e - v.e0... absolute e] = (start, end)
// (tg_ent_map_kernel; a kernel of its own so that the UTF-8 machinery and the link scan never share an
// instruction cache)
DEVI void warp_map_entities(const TgRecView& v, const tgi_entity* ents, int2* ranges) {
  if (!ct_carries_links(v.ct) || !(v.flags & TGI_RF_HAS_TEXT)) return;
  int64_t ascii_prefix = -1;  // computed when the first offset has to be mapped
  for (uint32_t e = v.e0; e < v.e1; e++) {
    const tgi_entity en = ents[e];
    if (en.type != TGI_ENT_MENTION && en.type != TGI_ENT_URL) continue;
    int64_t st, en_;
    if (ascii_prefix < 0) ascii_prefix = warp_first_non_ascii(v.text, v.text_len);
    const int64_t stop = (int64_t)en.offset + (int64_t)en.length;
    if (en.offset >= 0 && en.length >= 0 && stop <= ascii_prefix) {
      // every rune before `stop` is one byte and one UTF-16 unit: utf16OffsetToBytes returns (offset, stop)
      // (stop == len(text) comes out of its after-the-loop fallback with the same values)
      st = en.offset;
      en_ = stop;
    } else {
      warp_utf16_to_bytes(v.text, v.text_len, en.offset, en.length, st, en_);
    }
    if (lane_id() == 0) ranges[e] = make_int2((int)st, (int)en_);  // texts are < 2^31 bytes; st may be -1
  }
}

// returns false if the reference would panic (record FAILED).  ranges: warp_map_entities' output
DEVI bool warp_extract_links(const TgRecView& v, const tgi_entity* ents, const uint8_t* aux, const int2* ranges, LinkSink& ls) {
  if (!ct_carries_links(v.ct) || !(v.flags & TGI_RF_HAS_TEXT)) return true;
  for (uint32_t e = v.e0; e < v.e1; e++) {
    tgi_entity en = ents[e];
    if (en.type == TGI_ENT_TEXT_URL) {
      warp_scan_channel_links(ls, aux + en.url_off, en.url_len, TGI_SRC_TEXT_URL, false);
    } else if (en.type == TGI_ENT_MENTION || en.type == TGI_ENT_URL) {
      const int2 rg = ranges[e];
      const int64_t st = rg.x, en_ = rg.y;
      if (st < en_ && en_ <= (int64_t)v.text_len) {
        if (st < 0) return false;
        if (en.type == TGI_ENT_MENTION) warp_scan_username(ls, v.text + st, en_ - st);
        else warp_scan_channel_links(ls, v.text + st, en_ - st, TGI_SRC_URL, false);
      }
    }
  }
  warp_scan_channel_links(ls, v.text, v.text_len, TGI_SRC_PLAINTEXT, true);
  return true;
}

}  // namespace tgi
