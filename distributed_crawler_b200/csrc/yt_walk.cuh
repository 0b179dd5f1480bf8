// yt_walk.cuh — YouTube video -> model.Post line (config 4) and the YouTube snowball frontier links.
//
// Replaces crawler/youtube/youtube_crawler.go:530-836 convertVideoToPost (+ parseISO8601Duration
// :461-486, extractURLs :489-513, sanitizeFilename :516-527) followed by json.Marshal(post)+'\n',
// and client/youtube_client.go:1856-1878 extractChannelIDsFromText.
//
// One templated walk visits every byte range of the line in model.Post declaration order; it is
// instantiated with YtSizer (length pass) and YtWriter (emit pass), so the two passes cannot
// drift.  This path is a parity case (BASELINE config 4), not the bench line: it favours a small,
// obviously-correct formulation over the lane-parallel machinery of the Telegram path.
#pragma once
#include "dev_common.cuh"
#include "tg_links.cuh"

namespace tgi {

struct YtBatchDev {
  uint64_t n;
  const tgi_yt_rec* recs;
  const uint8_t* strs;
  uint32_t n_chans;
  const tgi_yt_chan* chans;
  const uint8_t* chan_strs;
};

struct YtUrl {  // one unique URL of a description (extractURLs), offsets into the description
  uint32_t off, len;
};

#define YLIT(w, str)                                                                           \
  do { /* 16-byte aligned and zero padded: the lane writer fetches literals in 16-byte blocks */  \
    static __device__ __align__(16) const char _lit[(sizeof(str) + 15) / 16 * 16] = str;          \
    (w).raw((const uint8_t*)_lit, sizeof(str) - 1);                                                \
  } while (0)

struct YtScratch {
  uint8_t num[64];  // >= 50 (sanitized file name), 40 (time), 20 (number)
};

// ---- writers ------------------------------------------------------------------------------------------
__device__ __noinline__ bool yt_parse_duration(const uint8_t* s, uint32_t n, int64_t& seconds);
__device__ __noinline__ int yt_render_float_of_int64(uint8_t* dst, int64_t v);
__device__ __noinline__ uint32_t yt_sanitize(const uint8_t* s, uint32_t n, uint8_t* dst);
// The walk is instantiated twice (sizer / writer) and every call below appears ~150 times in it: the
// byte movers are free __noinline__ functions so that the walk stays a few thousand instructions.
__device__ __noinline__ void yt_copy(uint8_t* p, const uint8_t* s, uint32_t n) {
  if (n >= 48) warp_copy_vec(p, s, n);
  else gcopy_g(p, s, n);
}
__device__ __noinline__ uint32_t yt_put_dec(uint8_t* p, uint8_t* scratch, int64_t v) {
  uint32_t n = 0;
  __syncwarp();
  if (lane_id() == 0) n = (uint32_t)render_i64(scratch, v);
  __syncwarp();
  n = __shfl_sync(FULL, n, 0);
  gcopy_s(p, smem_addr(scratch), n);
  __syncwarp();
  return n;
}
__device__ __noinline__ uint32_t yt_ndigits(int64_t v) { return ndigits_i64(v); }
// warp-mode helpers shared by the sizer and the warp writer: lane 0 renders into sc->num, everybody learns the length
DEVI uint32_t yt_warp_time(YtScratch* sc, int64_t sec, int32_t nsec) {
  uint32_t n = 0;
  __syncwarp();
  if (lane_id() == 0) n = (uint32_t)render_time(sc->num, sec, nsec, 0);
  __syncwarp();
  return __shfl_sync(FULL, n, 0);
}
struct YtSizer {
  static constexpr bool kLane = false;
  uint64_t total = 0;
  YtScratch* sc;
  uint32_t el[2];  // escaped lengths of the description / the title (each is written several times)
  bool dirty = false;  // some string needs escaping: the record is left to the warp writer
  DEVI uint32_t time_len(int64_t sec, int32_t nsec) { return yt_warp_time(sc, sec, nsec); }
  DEVI void time(int64_t sec, int32_t nsec) { total += yt_warp_time(sc, sec, nsec); }
  DEVI void fviews(int64_t v) {
    uint32_t n = 0;
    if (lane_id() == 0) n = (uint32_t)yt_render_float_of_int64(sc->num, v);
    total += __shfl_sync(FULL, n, 0);
    __syncwarp();
  }
  DEVI void sanitized(const uint8_t* t, uint32_t tn) {
    uint32_t n = 0;
    if (lane_id() == 0) n = yt_sanitize(t, tn, sc->num);
    total += __shfl_sync(FULL, n, 0);
    __syncwarp();
  }
  DEVI bool duration(const uint8_t* d, uint32_t dn, int64_t& vlen) {
    int ok = 0;
    if (lane_id() == 0) ok = yt_parse_duration(d, dn, vlen) ? 1 : 0;
    vlen = __shfl_sync(FULL, vlen, 0);
    return __shfl_sync(FULL, ok, 0) != 0;
  }
  DEVI void raw(const uint8_t*, uint32_t n) { total += n; }
  DEVI void esc(const uint8_t* s, uint32_t n) {
    const uint32_t e = warp_esc_len(s, n);
    dirty = dirty || e != n;
    total += e;
  }
  DEVI void esc_slot(int k, const uint8_t*, uint32_t n) {
    dirty = dirty || el[k] != n;
    total += el[k];
  }
  DEVI void ch(uint32_t) { total += 1; }
  DEVI void dec(int64_t v) { total += yt_ndigits(v); }
  DEVI void smem(uint32_t n) { total += n; }
};
struct YtWriter {
  static constexpr bool kLane = false;
  uint8_t* p;
  YtScratch* sc;
  uint32_t el[2];  // from the size pass
  DEVI uint32_t time_len(int64_t sec, int32_t nsec) { return yt_warp_time(sc, sec, nsec); }
  DEVI void time(int64_t sec, int32_t nsec) { smem(yt_warp_time(sc, sec, nsec)); }
  DEVI void fviews(int64_t v) {
    uint32_t n = 0;
    __syncwarp();
    if (lane_id() == 0) n = (uint32_t)yt_render_float_of_int64(sc->num, v);
    __syncwarp();
    smem(__shfl_sync(FULL, n, 0));
  }
  DEVI void sanitized(const uint8_t* t, uint32_t tn) {
    uint32_t n = 0;
    __syncwarp();
    if (lane_id() == 0) n = yt_sanitize(t, tn, sc->num);
    __syncwarp();
    smem(__shfl_sync(FULL, n, 0));
  }
  DEVI bool duration(const uint8_t* d, uint32_t dn, int64_t& vlen) {
    int ok = 0;
    if (lane_id() == 0) ok = yt_parse_duration(d, dn, vlen) ? 1 : 0;
    vlen = __shfl_sync(FULL, vlen, 0);
    return __shfl_sync(FULL, ok, 0) != 0;
  }
  DEVI void raw(const uint8_t* s, uint32_t n) {
    yt_copy(p, s, n);
    p += n;
  }
  DEVI void esc(const uint8_t* s, uint32_t n) { p += esc_to_global(p, s, n); }
  DEVI void esc_slot(int k, const uint8_t* s, uint32_t n) {  // nothing to escape: plain copy
    if (el[k] == n) {
      yt_copy(p, s, n);
      p += n;
    } else {
      p += esc_to_global(p, s, n);
    }
  }
  DEVI void ch(uint32_t c) {
    gput1(p, c);
    p += 1;
  }
  DEVI void dec(int64_t v) { p += yt_put_dec(p, sc->num, v); }
  DEVI void smem(uint32_t n) {  // n bytes already rendered in sc->num
    gcopy_s(p, smem_addr(sc->num), n);
    p += n;
    __syncwarp();
  }
};

// ---- helpers --------------------------------------------------------------------------------------------
DEVI bool yt_is_digit(uint32_t c) { return (c - '0') < 10u; }
DEVI bool yt_is_space(uint32_t c) { return c == '\t' || c == '\n' || c == '\f' || c == '\r' || c == ' '; }

// strconv.Atoi on digits: clamps to MaxInt64 (the error is ignored, youtube_crawler.go:473)
DEVI int64_t yt_atoi_clamp(const uint8_t* s, uint32_t n) {
  uint64_t v = 0;
  for (uint32_t i = 0; i < n; i++) {
    uint64_t d = ldb(s + i) - '0';
    if (v > 0x7FFFFFFFFFFFFFFFull / 10 || v * 10 > 0x7FFFFFFFFFFFFFFFull - d) return 0x7FFFFFFFFFFFFFFFll;
    v = v * 10 + d;
  }
  return (int64_t)v;
}
// parseISO8601Duration (:461-486): ^P(?:(\d+)D)?(?:T(?:(\d+)H)?(?:(\d+)M)?(?:(\d+)S)?)?$ ; single thread
__device__ __noinline__ bool yt_parse_duration(const uint8_t* s, uint32_t n, int64_t& seconds) {
  uint32_t i = 0;
  uint64_t total = 0;  // Go int arithmetic wraps
  if (i >= n || ldb(s + i) != 'P') return false;
  i++;
  uint32_t j = i;
  while (j < n && yt_is_digit(ldb(s + j))) j++;
  if (j > i && j < n && ldb(s + j) == 'D') {
    total += (uint64_t)yt_atoi_clamp(s + i, j - i) * 86400u;
    i = j + 1;
  }
  if (i < n && ldb(s + i) == 'T') {
    i++;
    const char unit[3] = {'H', 'M', 'S'};
    const uint64_t mul[3] = {3600, 60, 1};
#pragma unroll
    for (int u = 0; u < 3; u++) {
      j = i;
      while (j < n && yt_is_digit(ldb(s + j))) j++;
      if (j > i && j < n && ldb(s + j) == (uint32_t)unit[u]) {
        total += (uint64_t)yt_atoi_clamp(s + i, j - i) * mul[u];
        i = j + 1;
      }
    }
  }
  if (i != n) return false;
  seconds = (int64_t)total;
  return true;
}

// strconv.FormatFloat(float64(v), 'f', -1, 64): shortest decimal that round-trips, positional.
// Integers below 2^53 print exactly; above, the shortest digit string inside the rounding interval of
// the nearest double (closest to it), padded with zeros.  Single thread; returns the length.
__device__ __noinline__ int yt_render_float_of_int64(uint8_t* dst, int64_t v) {
  int o = 0;
  uint64_t a = v < 0 ? (uint64_t)0 - (uint64_t)v : (uint64_t)v;
  if (v < 0) dst[o++] = '-';
  if (a < (1ull << 53)) return o + render_u64(dst + o, a);
  double f = (double)a;  // round to nearest even, as Go's float64(int64)
  uint64_t F = (uint64_t)f;  // exact: f is an integer < 2^64
  int e = 63 - __clzll((long long)F);  // F in [2^e, 2^(e+1))
  uint64_t ulp = 1ull << (e - 52);
  uint64_t mant = F >> (e - 52);
  bool even = (mant & 1) == 0;
  uint64_t hi_half = ulp / 2, lo_half = (F == (1ull << e)) ? ulp / 4 : ulp / 2;
  // interval of integers that convert back to f: [F - lo_half, F + hi_half], bounds included iff even
  uint64_t lo = F - lo_half + (even ? 0 : 1), hi = F + hi_half - (even ? 0 : 1);
  uint64_t best = F, p = 1;
  for (int k = 1; k < 20; k++) {  // largest power of ten with a multiple inside the interval
    if (p > 0xFFFFFFFFFFFFFFFFull / 10) break;
    p *= 10;
    uint64_t q = F / p * p;  // multiple below (or equal)
    uint64_t cand = 0;
    bool ok = false;
    if (q >= lo && q <= hi) { cand = q; ok = true; }
    if (q + p >= q && q + p >= lo && q + p <= hi) {  // multiple above
      if (!ok || (q + p - F) < (F - q)) cand = q + p;
      else if (ok && (q + p - F) == (F - q)) cand = ((q / p) & 1) ? q + p : q;  // tie -> even digit
      ok = true;
    }
    if (!ok) break;
    best = cand;
  }
  return o + render_u64(dst + o, best);
}

// sanitizeFilename (:516-527): every rune outside [0-9A-Za-z_\-.] -> '_', truncated to 50 bytes.
// Single thread, output into dst (<= 50 bytes); returns the length.
__device__ __noinline__ uint32_t yt_sanitize(const uint8_t* s, uint32_t n, uint8_t* dst) {
  uint32_t o = 0;
  for (uint32_t i = 0; i < n && o < 50;) {
    uint32_t b = ldb(s + i);
    if (b < 0x80) {
      dst[o++] = (is_word(b) || b == '-' || b == '.') ? (uint8_t)b : (uint8_t)'_';
      i++;
    } else {
      int need = utf8_valid_lead(s, i, n);
      dst[o++] = '_';
      i += need ? (uint32_t)need : 1u;
    }
  }
  return o;
}

// extractURLs (:489-513): (https?://\S+) over the description, TrimRight(",.;:!?()'\""), unique in
// first-occurrence order.  Warp-cooperative candidate search; the unique list goes to `out` (cap
// entries, reserved from an upper bound = number of "http" occurrences).  Returns the count.
// 512-byte strips, 16 bytes per lane, with a ':' prefilter (':' is rare in running text): bit k of the lane's
// mask is set if s[p0+k] is the colon of "http://" / "https://" followed by a non-space (p0 = base + 16*lane)
DEVI uint32_t yt_strip16_scheme(const uint8_t* s, uint32_t base, uint32_t n) {
  const uint32_t p0 = base + 16u * (uint32_t)lane_id();
  if (p0 >= n) return 0;
  const uint4 w = ld16_unaligned(s + p0);
  const uint32_t c0 = swar_eq(w.x, ':'), c1 = swar_eq(w.y, ':'), c2 = swar_eq(w.z, ':'), c3 = swar_eq(w.w, ':');
  if (!(c0 | c1 | c2 | c3)) return 0;
  uint32_t m = swar_movemask(c0) | (swar_movemask(c1) << 4) | (swar_movemask(c2) << 8) | (swar_movemask(c3) << 12);
  if (n - p0 < 16) m &= (1u << (n - p0)) - 1u;
  uint32_t out = 0;
  while (m) {
    const uint32_t k = (uint32_t)__ffs(m) - 1u, c = p0 + k;
    m &= m - 1;
    if (c < 4 || c + 3 >= n) continue;
    if (ldb(s + c + 1) != '/' || ldb(s + c + 2) != '/' || yt_is_space(ldb(s + c + 3))) continue;
    const bool http = ld_u32_unaligned(s + c - 4) == 0x70747468u;                                   // "http"
    const bool https = c >= 5 && ldb(s + c - 1) == 's' && ld_u32_unaligned(s + c - 5) == 0x70747468u;  // "https"
    if (http || https) out |= 1u << k;
  }
  return out;
}
DEVI uint32_t yt_count_http(const uint8_t* s, uint32_t n) {  // number of places where a URL can start (upper bound on matches)
  uint32_t c = 0;
  for (uint32_t base = 0; base < n; base += 512) c += __popc(yt_strip16_scheme(s, base, n));
  return warp_sum(c);
}
DEVI uint32_t yt_extract_urls(const uint8_t* s, uint32_t n, YtUrl* out, uint32_t cap) {
  uint32_t m = 0, resume = 0;
  int l = lane_id();
  for (uint32_t base = 0; base < n; base += 512) {
    const uint32_t cm = yt_strip16_scheme(s, base, n);
    uint32_t lanes = __ballot_sync(FULL, cm != 0);
    while (lanes) {
      const int src_lane = __ffs(lanes) - 1;
      lanes &= lanes - 1;
      uint32_t mm = __shfl_sync(FULL, cm, src_lane);
     while (mm) {
      const uint32_t colon = base + 16u * (uint32_t)src_lane + (uint32_t)__ffs(mm) - 1u;
      mm &= mm - 1;
      const uint32_t p = colon - (ldb(s + colon - 1) == 's' ? 5u : 4u);  // start of the scheme
      if (p < resume) continue;  // inside the previous match
      // \S+ is greedy: up to the next RE2 whitespace
      uint32_t e = p;
      for (;;) {
        uint32_t q = e + l;
        uint32_t stop = __ballot_sync(FULL, q >= n || yt_is_space(ldb(s + (q < n ? q : 0))));
        if (stop) {
          e += __ffs(stop) - 1;
          break;
        }
        e += 32;
      }
      resume = e;
      uint32_t te = e;  // TrimRight
      for (;;) {
        if (te <= p) break;
        uint32_t c = ldb(s + te - 1);
        if (c == ',' || c == '.' || c == ';' || c == ':' || c == '!' || c == '?' || c == '(' || c == ')' || c == '\'' || c == '"') te--;
        else break;
      }
      uint32_t len = te - p;
      bool dup = false;
      for (uint32_t j = 0; j < m && !dup; j++) {
        if (out[j].len != len) continue;
        bool eq = true;
        for (uint32_t t = l; t < len; t += 32) eq &= ldb(s + out[j].off + t) == ldb(s + p + t);
        dup = __all_sync(FULL, eq);
      }
      if (!dup && m < cap) {
        if (l == 0) {
          out[m].off = p;
          out[m].len = len;
        }
        __syncwarp();
        m++;
      }
     }
    }
  }
  return m;
}

// extractChannelIDsFromText (youtube_client.go:1856-1878): all youtube\.com/channel/([\w-]+), then all
// youtube\.com/@([\w.-]+) ("@"+handle); no dedup here.  Keys are cut to 32 bytes (frontier key width).
DEVI bool yt_is_uc_char(uint32_t c) { return is_word(c) || c == '-'; }
DEVI bool yt_is_handle_char(uint32_t c) { return is_word(c) || c == '-' || c == '.'; }
// 512-byte strips with a '/' prefilter: bit k of the lane's mask is set if s[p0+k] is the slash of "youtube.com/"
DEVI uint32_t yt_strip16_ytcom(const uint8_t* s, uint32_t base, uint32_t n) {
  const uint32_t p0 = base + 16u * (uint32_t)lane_id();
  if (p0 >= n) return 0;
  const uint4 w = ld16_unaligned(s + p0);
  const uint32_t c0 = swar_eq(w.x, '/'), c1 = swar_eq(w.y, '/'), c2 = swar_eq(w.z, '/'), c3 = swar_eq(w.w, '/');
  if (!(c0 | c1 | c2 | c3)) return 0;
  uint32_t m = swar_movemask(c0) | (swar_movemask(c1) << 4) | (swar_movemask(c2) << 8) | (swar_movemask(c3) << 12);
  if (n - p0 < 16) m &= (1u << (n - p0)) - 1u;
  uint32_t out = 0;
  while (m) {
    const uint32_t k = (uint32_t)__ffs(m) - 1u, c = p0 + k;
    m &= m - 1;
    if (c >= 11 && ld_u32_unaligned(s + c - 11) == 0x74756F79u && ld_u32_unaligned(s + c - 7) == 0x2E656275u &&
        (ld_u32_unaligned(s + c - 3) & 0xFFFFFFu) == 0x6D6F63u)  // "yout" "ube." "com"
      out |= 1u << k;
  }
  return out;
}
DEVI uint32_t yt_count_ytcom(const uint8_t* s, uint32_t n) {  // upper bound on channel-id matches
  uint32_t c = 0;
  for (uint32_t base = 0; base < n; base += 512) c += __popc(yt_strip16_ytcom(s, base, n));
  return warp_sum(c);
}
DEVI uint32_t yt_channel_ids(const uint8_t* s, uint32_t n, tgi_link* out, uint32_t cap) {
  uint32_t m = 0;
  int l = lane_id();
  for (int pass = 0; pass < 2; pass++) {
    const uint32_t pl = pass ? 13u : 20u;  // "youtube.com/@" / "youtube.com/channel/"
    uint32_t resume = 0;
    for (uint32_t base = 0; base < n; base += 512) {
      const uint32_t cm = yt_strip16_ytcom(s, base, n);
      uint32_t lanes = __ballot_sync(FULL, cm != 0);
      while (lanes) {
        const int src_lane = __ffs(lanes) - 1;
        lanes &= lanes - 1;
        uint32_t mm = __shfl_sync(FULL, cm, src_lane);
       while (mm) {
        const uint32_t slash = base + 16u * (uint32_t)src_lane + (uint32_t)__ffs(mm) - 1u;
        mm &= mm - 1;
        const uint32_t p = slash - 11u;  // start of "youtube.com/"
        if (p + pl >= n) continue;
        if (pass) {
          if (ldb(s + slash + 1) != '@' || !yt_is_handle_char(ldb(s + p + pl))) continue;
        } else {
          if (ld_u32_unaligned(s + slash + 1) != 0x6E616863u || ld_u32_unaligned(s + slash + 5) != 0x2F6C656Eu ||  // "chan" "nel/"
              !yt_is_uc_char(ldb(s + p + pl)))
            continue;
        }
        if (p < resume) continue;
        uint32_t q = p + pl, e = q;
        for (;;) {
          uint32_t t = e + l;
          bool ok = t < n && (pass ? yt_is_handle_char(ldb(s + t)) : yt_is_uc_char(ldb(s + t)));
          uint32_t stop = __ballot_sync(FULL, !ok);
          if (stop) {
            e += __ffs(stop) - 1;
            break;
          }
          e += 32;
        }
        resume = e;
        if (m < cap) {
          uint32_t len = e - q;
          uint32_t c = 0;
          if (pass) c = l == 0 ? '@' : ((uint32_t)l <= len ? ldb(s + q + l - 1) : 0u);
          else c = (uint32_t)l < len ? ldb(s + q + l) : 0u;
          uint32_t klen = pass ? (len + 1 > 32 ? 32 : len + 1) : (len > 32 ? 32 : len);
          out[m].name[l] = (uint8_t)c;
          // informational only for YouTube ids (FilterUsername is the Telegram tandem validator)
          uint32_t reason = warp_filter_username(c, klen);
          if (l == 0) {
            out[m].len = (uint8_t)klen;
            out[m].src = (uint8_t)pass;
            out[m].flags = (uint8_t)(reason == TGI_FU_VALID ? TGI_LF_FILTER_OK : 0);
            out[m].filter_reason = (uint8_t)reason;
          }
          __syncwarp();
          m++;
        }
       }
      }
    }
  }
  return m;
}

// ---- the line ---------------------------------------------------------------------------------------------
struct YtArgs {
  const YtBatchDev* b;
  const CfgDev* cfg;
  uint64_t r;
  const YtUrl* urls;
  uint32_t n_urls;
};

__device__ __align__(16) const char kYtThumbKey[5][16] = {"default", "medium", "high", "standard", "maxres"};  // 16-byte rows: the lane writer fetches sources in aligned 16-byte blocks
__device__ const uint8_t kYtThumbKeyLen[5] = {7, 6, 4, 8, 6};

// returns false if a time field is not representable (Marshal error -> TGI_ST_NOLINE)
template <class W>
DEVI bool walk_yt_record(W& w, const YtArgs& a) {
  const YtBatchDev& b = *a.b;
  const CfgDev& cfg = *a.cfg;
  const tgi_yt_rec v = b.recs[a.r];
  const tgi_yt_chan ch = b.chans[v.chan_idx];
  const uint8_t* cs = b.chan_strs + ch.str_off;
  const uint8_t *chid = cs, *chtitle = chid + ch.id_len, *chdesc = chtitle + ch.title_len, *chthumb = chdesc + ch.desc_len,
                *chcountry = chthumb + ch.thumb_len;
  const uint8_t* p = b.strs + v.str_off;
  const uint8_t *id = p, *title = id + v.id_len, *desc = title + v.title_len, *dur = desc + v.desc_len, *lang = dur + v.duration_len;
  const uint8_t* th[5];
  uint32_t thn[5];
  {
    const uint8_t* q = lang + v.lang_len;
#pragma unroll
    for (int k = 0; k < 5; k++) {
      th[k] = q;
      thn[k] = v.thumb_len[k] == TGI_YT_THUMB_ABSENT ? 0u : v.thumb_len[k];
      q += thn[k];
    }
  }
  // times: published (UTC), channel published (UTC): rendered where needed; validity first
  const uint32_t pub_len = w.time_len(v.published_sec, v.published_nsec);
  uint32_t chpub_len = 1;
  if (ch.cached) chpub_len = w.time_len(ch.published_sec, ch.published_nsec);
  if (pub_len == 0 || chpub_len == 0 || (cfg.flags & CFGDEV_CLOCK_INVALID) || cfg.created_yt_len == 0) return false;

  const int64_t engagement = (int64_t)((uint64_t)v.like_count + (uint64_t)v.comment_count + (uint64_t)(v.view_count / 100));  // :561
  // :615-624 thumb priority maxres > high > medium > default
  const uint8_t* thumb = nullptr;
  uint32_t thumb_n = 0;
  {
    const int prio[4] = {4, 2, 1, 0};
#pragma unroll
    for (int k = 3; k >= 0; k--)
      if (thn[prio[k]]) { thumb = th[prio[k]]; thumb_n = thn[prio[k]]; }
  }
  // :631-643 duration
  int has_len = 0;
  int64_t vlen = 0;
  if (v.duration_len && !(v.duration_len == 3 && ldb(dur) == 'P' && ldb(dur + 1) == '0' && ldb(dur + 2) == 'D')) {
    has_len = w.duration(dur, v.duration_len, vlen) ? 1 : 0;
  }
  const uint8_t* cblob = cfg.blob;
  const uint8_t* created = cblob + cfg.off[2];
  const uint8_t* capture = cblob + cfg.off[3];
  const bool handle_url = ch.id_len > 0 && ldb(chid) == '@';

#define VURL()                                      \
  do {                                              \
    YLIT(w, "https://www.youtube.com/watch?v=");    \
    w.esc(id, v.id_len);                            \
  } while (0)
#define CHURL()                                                          \
  do {                                                                   \
    if (handle_url) YLIT(w, "https://www.youtube.com/");                 \
    else YLIT(w, "https://www.youtube.com/channel/");                    \
    w.esc(chid, ch.id_len);                                              \
  } while (0)
#define PUBTIME(sec, nsec) w.time((sec), (nsec))

  YLIT(w, "{\"post_link\":\""); VURL();
  YLIT(w, "\",\"channel_id\":\""); w.esc(chid, ch.id_len);
  YLIT(w, "\",\"post_uid\":\""); w.esc(id, v.id_len);
  YLIT(w, "\",\"url\":\""); VURL();
  YLIT(w, "\",\"published_at\":"); PUBTIME(v.published_sec, v.published_nsec);
  YLIT(w, ",\"created_at\":"); w.raw(created, cfg.created_yt_len);
  YLIT(w, ",\"language_code\":\""); w.esc(lang, v.lang_len);
  YLIT(w, "\",\"engagement\":"); w.dec(engagement);
  YLIT(w, ",\"view_count\":"); w.dec(v.view_count);
  YLIT(w, ",\"like_count\":"); w.dec(v.like_count);
  YLIT(w, ",\"share_count\":0,\"comment_count\":"); w.dec(v.comment_count);
  YLIT(w, ",\"crawl_label\":\""); w.raw(cblob, cfg.label_len);
  YLIT(w, "\",\"list_ids\":null,\"channel_name\":\"");
  if (ch.cached) w.esc(chtitle, ch.title_len); else w.esc(chid, ch.id_len);
  YLIT(w, "\",\"search_terms\":null,\"search_term_ids\":null,\"project_ids\":null,\"exercise_ids\":null,"
          "\"label_data\":null,\"labels_metadata\":null,\"project_labeled_post_ids\":null,"
          "\"labeler_ids\":null,\"all_labels\":null,\"label_ids\":null,\"is_ad\":false,"
          "\"transcript_text\":\"\",\"image_text\":\"\",\"video_length\":");
  if (has_len) w.dec(vlen); else YLIT(w, "null");
  YLIT(w, ",\"is_verified\":null,\"channel_data\":{\"channel_id\":\""); w.esc(chid, ch.id_len);
  if (ch.cached) {  // :784-805
    YLIT(w, "\",\"channel_name\":\""); w.esc(chtitle, ch.title_len);
    YLIT(w, "\",\"channel_description\":\""); w.esc(chdesc, ch.desc_len);
    YLIT(w, "\",\"channel_profile_image\":\""); w.esc(chthumb, ch.thumb_len);
    YLIT(w, "\",\"channel_engagement_data\":{\"follower_count\":"); w.dec(ch.subscriber_count);
    YLIT(w, ",\"following_count\":0,\"like_count\":0,\"post_count\":"); w.dec(ch.video_count);
    YLIT(w, ",\"views_count\":"); w.dec(ch.view_count);
    YLIT(w, ",\"comment_count\":0,\"share_count\":0},\"channel_url_external\":\""); CHURL();
    YLIT(w, "\",\"channel_url\":\""); CHURL();
    YLIT(w, "\",\"country_code\":\""); w.esc(chcountry, ch.country_len);
    YLIT(w, "\",\"published_at\":"); PUBTIME(ch.published_sec, ch.published_nsec);
  } else {  // :806-829
    YLIT(w, "\",\"channel_name\":\""); w.esc(chid, ch.id_len);
    YLIT(w, "\",\"channel_description\":\"\",\"channel_profile_image\":\"\",\"channel_engagement_data\":{"
            "\"follower_count\":0,\"following_count\":0,\"like_count\":");
    w.dec(v.like_count);
    YLIT(w, ",\"post_count\":0,\"views_count\":"); w.dec(v.view_count);
    YLIT(w, ",\"comment_count\":"); w.dec(v.comment_count);
    YLIT(w, ",\"share_count\":0},\"channel_url_external\":\""); CHURL();
    YLIT(w, "\",\"channel_url\":\""); CHURL();
    YLIT(w, "\",\"country_code\":\"\",\"published_at\":"); PUBTIME(v.published_sec, v.published_nsec);
  }
  YLIT(w, "},\"platform_name\":\"youtube\",\"shared_id\":null,\"quoted_id\":null,\"replied_id\":null,"
          "\"ai_label\":null,\"root_post_id\":null,\"engagement_steps_count\":0,\"ocr_data\":");
  {  // :668-677; canonical key order default,medium,high,standard,maxres; nil slice -> null
    bool any = false;
#pragma unroll
    for (int k = 0; k < 5; k++) {
      if (!thn[k]) continue;
      w.ch(any ? ',' : '[');
      any = true;
      YLIT(w, "{\"ocr_text\":\"YouTube thumbnail: ");
      w.raw((const uint8_t*)kYtThumbKey[k], kYtThumbKeyLen[k]);
      YLIT(w, " quality\",\"thumb_url\":\"");
      w.esc(th[k], thn[k]);
      YLIT(w, "\"}");
    }
    if (any) w.ch(']'); else YLIT(w, "null");
  }
  YLIT(w, ",\"performance_scores\":{\"likes\":"); w.dec(v.like_count);
  YLIT(w, ",\"shares\":null,\"comments\":"); w.dec(v.comment_count);
  YLIT(w, ",\"views\":");
  w.fviews(v.view_count);
  YLIT(w, "},\"has_embed_media\":true,\"description\":\""); w.esc_slot(0, desc, v.desc_len);
  YLIT(w, "\",\"repost_channel_data\":null,\"post_type\":[\"video\"],\"inner_link\":{},\"post_title\":\"");
  w.esc_slot(1, title, v.title_len);
  YLIT(w, "\",\"media_data\":{\"document_name\":\""); w.esc(id, v.id_len);
  w.ch('-');
  w.sanitized(title, v.title_len);
  YLIT(w, ".mp4\"},\"is_reply\":null,\"ad_fields\":null,\"likes_count\":"); w.dec(v.like_count);
  YLIT(w, ",\"shares_count\":0,\"comments_count\":"); w.dec(v.comment_count);
  YLIT(w, ",\"views_count\":"); w.dec(v.view_count);
  YLIT(w, ",\"searchable_text\":\""); w.esc_slot(1, title, v.title_len); w.ch(' '); w.esc_slot(0, desc, v.desc_len);
  YLIT(w, "\",\"all_text\":\""); w.esc_slot(1, title, v.title_len); w.ch(' '); w.esc_slot(0, desc, v.desc_len);
  YLIT(w, "\",\"contrast_agent_project_ids\":null,\"agent_ids\":null,\"segment_ids\":null,\"thumb_url\":\"");
  w.esc(thumb, thumb_n);
  YLIT(w, "\",\"media_url\":\""); VURL();
  YLIT(w, "\",\"comments\":null,\"reactions\":{\"like\":"); w.dec(v.like_count);
  YLIT(w, "},\"outlinks\":[");
  for (uint32_t k = 0; k < a.n_urls; k++) {
    w.ch(k ? ',' : '"');
    if (k) w.ch('"');
    w.esc(desc + a.urls[k].off, a.urls[k].len);
    w.ch('"');
  }
  YLIT(w, "],\"capture_time\":"); w.raw(capture, cfg.capture_len);
  YLIT(w, ",\"handle\":\""); w.esc(chid, ch.id_len);
  YLIT(w, "\"}\n");
#undef VURL
#undef CHURL
#undef PUBTIME
  return true;
}

}  // namespace tgi
