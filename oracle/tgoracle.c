/*
 * tgoracle.c — CPU restatement of the reference hot path.  TEST INFRASTRUCTURE ONLY (see tgoracle.h
 * for the parity-pinning statement).  Plain C11 + pthreads; nothing here is shipped in libtgingest.
 *
 * Each function cites the reference code (path:line relative to the reference tree) it follows.
 * The style is deliberately sequential and literal — it mirrors the Go control flow, it is not an
 * optimised implementation and shares no code with the CUDA kernels.
 */
#define _GNU_SOURCE
#include "tgoracle.h"

#include <pthread.h>
#include <sched.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------------------------- */
/* growable byte buffer                                                                          */
typedef struct {
  uint8_t* p;
  size_t len, cap;
} buf_t;

static void buf_reserve(buf_t* b, size_t extra) {
  if (b->len + extra <= b->cap) return;
  size_t nc = b->cap ? b->cap * 2 : 4096;
  while (nc < b->len + extra) nc *= 2;
  b->p = (uint8_t*)realloc(b->p, nc);
  if (!b->p) abort();
  b->cap = nc;
}
static void buf_put(buf_t* b, const void* s, size_t n) {
  buf_reserve(b, n);
  memcpy(b->p + b->len, s, n);
  b->len += n;
}
#define LIT(b, s) buf_put((b), (s), sizeof(s) - 1)

/* ------------------------------------------------------------------------------------------- */
/* Go unicode/utf8.DecodeRuneInString: returns width; *rune = 0xFFFD with width 1 when invalid    */
static int go_decode_rune(const uint8_t* s, int64_t n, uint32_t* rune) {
  if (n <= 0) {
    *rune = 0xFFFD;
    return 0;
  }
  uint8_t b0 = s[0];
  if (b0 < 0x80) {
    *rune = b0;
    return 1;
  }
  int need;
  uint8_t lo = 0x80, hi = 0xBF;
  if (b0 >= 0xC2 && b0 <= 0xDF) need = 2;
  else if (b0 == 0xE0) { need = 3; lo = 0xA0; }
  else if (b0 >= 0xE1 && b0 <= 0xEC) need = 3;
  else if (b0 == 0xED) { need = 3; hi = 0x9F; }
  else if (b0 >= 0xEE && b0 <= 0xEF) need = 3;
  else if (b0 == 0xF0) { need = 4; lo = 0x90; }
  else if (b0 >= 0xF1 && b0 <= 0xF3) need = 4;
  else if (b0 == 0xF4) { need = 4; hi = 0x8F; }
  else {
    *rune = 0xFFFD;
    return 1;
  }
  if (n < need) {
    *rune = 0xFFFD;
    return 1;
  }
  uint8_t b1 = s[1];
  if (b1 < lo || b1 > hi) {
    *rune = 0xFFFD;
    return 1;
  }
  if (need == 2) {
    *rune = ((uint32_t)(b0 & 0x1F) << 6) | (b1 & 0x3F);
    return 2;
  }
  uint8_t b2 = s[2];
  if (b2 < 0x80 || b2 > 0xBF) {
    *rune = 0xFFFD;
    return 1;
  }
  if (need == 3) {
    *rune = ((uint32_t)(b0 & 0x0F) << 12) | ((uint32_t)(b1 & 0x3F) << 6) | (b2 & 0x3F);
    return 3;
  }
  uint8_t b3 = s[3];
  if (b3 < 0x80 || b3 > 0xBF) {
    *rune = 0xFFFD;
    return 1;
  }
  *rune = ((uint32_t)(b0 & 0x07) << 18) | ((uint32_t)(b1 & 0x3F) << 12) |
          ((uint32_t)(b2 & 0x3F) << 6) | (b3 & 0x3F);
  return 4;
}

/* telegramhelper/tdutils.go:55-78 utf16OffsetToBytes.  start may come back as -1 (offset inside a
 * surrogate pair, never "reached") with end >= 0: the Go caller then slices [-1:end] and panics.  */
void orc_utf16_offset_to_bytes(const uint8_t* s, int64_t n, int32_t off16, int32_t len16,
                               int64_t* start, int64_t* end) {
  int64_t i = 0;
  int32_t u16pos = 0;
  int64_t rune_start = -1;
  int32_t stop = (int32_t)((uint32_t)off16 + (uint32_t)len16); /* Go int32 add wraps */
  while (i < n) {
    if (u16pos == off16) rune_start = i;
    if (u16pos == stop) {
      *start = rune_start;
      *end = i;
      return;
    }
    uint32_t r;
    int size = go_decode_rune(s + i, n - i, &r);
    u16pos += (r >= 0x10000) ? 2 : 1;
    i += size;
  }
  if (rune_start == -1) {
    *start = 0;
    *end = 0;
    return;
  }
  *start = rune_start;
  *end = n;
}

static int is_letter(uint8_t c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z'); }
static int is_word(uint8_t c) { return is_letter(c) || (c >= '0' && c <= '9') || c == '_'; }

/* telegramhelper/tdutils.go:23 channelLinkRegex = (https?://)?t\.me/([a-zA-Z][a-zA-Z0-9_]{4,31})
 * Go regexp (RE2): unanchored, leftmost-first, greedy.  The optional scheme group changes neither
 * the capture nor the match end, so "first match at or after `from`" is: the first position p >= from
 * with "t.me/" at p, a letter at p+5 and at least 4 more word chars; the name is greedy up to 32.   */
int orc_channel_link_first(const uint8_t* s, int64_t n, int64_t from, int64_t* name_start,
                           int64_t* name_end) {
  for (int64_t p = from; p + 5 < n; p++) {
    if (s[p] != 't' || s[p + 1] != '.' || s[p + 2] != 'm' || s[p + 3] != 'e' || s[p + 4] != '/')
      continue;
    int64_t q = p + 5;
    if (!is_letter(s[q])) continue;
    int64_t e = q + 1;
    while (e < n && e - q < 32 && is_word(s[e])) e++;
    if (e - q < 5) continue;
    *name_start = q;
    *name_end = e;
    return 1;
  }
  return 0;
}

/* telegramhelper/tdutils.go:82 usernameRegex = (?:@)?([a-zA-Z][a-zA-Z0-9_]{4,31}), FindStringSubmatch:
 * leftmost position where a letter is followed by >= 4 word chars (the optional '@' is immaterial). */
int orc_username_first(const uint8_t* s, int64_t n, int64_t* name_start, int64_t* name_end) {
  for (int64_t q = 0; q < n; q++) {
    if (!is_letter(s[q])) continue;
    int64_t e = q + 1;
    while (e < n && e - q < 32 && is_word(s[e])) e++;
    if (e - q < 5) continue;
    *name_start = q;
    *name_end = e;
    return 1;
  }
  return 0;
}

/* telegramhelper/tdutils.go:27-32 telegramReservedPaths */
int orc_is_reserved_path(const uint8_t* lower_name, int len) {
  static const char* reserved[] = {"joinchat", "addlist", "addstickers", "addtheme", "setlanguage",
                                   "share",    "c",       "s",           "iv",       "proxy",
                                   "socks",    "login",   "confirm",     "bg"};
  for (size_t i = 0; i < sizeof(reserved) / sizeof(reserved[0]); i++) {
    if ((int)strlen(reserved[i]) == len && memcmp(reserved[i], lower_name, (size_t)len) == 0) return 1;
  }
  return 0;
}

static uint8_t ascii_lower(uint8_t c) { return (c >= 'A' && c <= 'Z') ? (uint8_t)(c + 32) : c; }

/* telegramhelper/username_filter.go:26-68 FilterUsername; returns TGI_FU_* */
int orc_filter_username(const uint8_t* u, int64_t len) {
  if (len < 5) return TGI_FU_TOO_SHORT;
  if (len > 32) return TGI_FU_TOO_LONG;
  /* first := rune(username[0]); !unicode.IsLetter(first) || first > 127.  rune(byte) is Latin-1, so
   * bytes >= 0x80 may be "letters" but are rejected by first > 127 anyway. */
  if (!is_letter(u[0])) return TGI_FU_INVALID_START_CHAR;
  if (u[len - 1] == '_') return TGI_FU_ENDS_WITH_UNDERSCORE;
  for (int64_t i = 0; i < len;) { /* for _, ch := range username: any non-ASCII rune is invalid */
    uint32_t r;
    int w = go_decode_rune(u + i, len - i, &r);
    if (!(r < 0x80 && is_word((uint8_t)r))) return TGI_FU_INVALID_CHAR;
    i += w;
  }
  for (int64_t i = 0; i < len; i++)
    if (u[i] == '/' || u[i] == '\\' || u[i] == '~' || u[i] == '.') return TGI_FU_LOOKS_LIKE_PATH;
  if (len >= 3 && ascii_lower(u[len - 3]) == 'b' && ascii_lower(u[len - 2]) == 'o' &&
      ascii_lower(u[len - 1]) == 't')
    return TGI_FU_BOT_SUFFIX;
  return TGI_FU_VALID;
}

/* ------------------------------------------------------------------------------------------- */
/* per-message ordered set of links: sourceMap + addIfNew (tdutils.go:897-906), with the build's
 * canonical order = first insertion (Go's map order is random; SURVEY Appendix A.4).              */
typedef struct {
  tgi_link* v;
  int n, cap;
  int overflow;
  buf_t* store; /* batch driver: the set grows on demand (the reference has no cap); NULL = fixed caller array */
} linkset_t;

static void linkset_add(linkset_t* ls, const uint8_t* name, int len, int src) {
  uint8_t low[32];
  for (int i = 0; i < len; i++) low[i] = ascii_lower(name[i]); /* strings.ToLower on ASCII */
  for (int i = 0; i < ls->n; i++)
    if (ls->v[i].len == len && memcmp(ls->v[i].name, low, (size_t)len) == 0) return;
  if (ls->n >= ls->cap) {
    if (!ls->store) {
      ls->overflow = 1;
      return;
    }
    ls->store->len = sizeof(tgi_link) * (size_t)ls->cap;
    buf_reserve(ls->store, sizeof(tgi_link) * (size_t)ls->cap);
    ls->cap *= 2;
    ls->v = (tgi_link*)ls->store->p;
  }
  tgi_link* l = &ls->v[ls->n++];
  memset(l, 0, sizeof(*l));
  memcpy(l->name, low, (size_t)len);
  l->len = (uint8_t)len;
  l->src = (uint8_t)src;
}

/* channelNameFromMatch (tdutils.go:36-45): drop reserved paths, lower-case */
static void add_channel_match(linkset_t* ls, const uint8_t* s, int64_t ns, int64_t ne, int src) {
  uint8_t low[32];
  int len = (int)(ne - ns);
  for (int i = 0; i < len; i++) low[i] = ascii_lower(s[ns + i]);
  if (orc_is_reserved_path(low, len)) return;
  linkset_add(ls, low, len, src);
}

static int ct_carries_links(int ct) { /* extractFormattedTextFromMessage, tdutils.go:953-972 */
  return ct == TGI_CT_TEXT || ct == TGI_CT_PHOTO || ct == TGI_CT_VIDEO || ct == TGI_CT_DOCUMENT ||
         ct == TGI_CT_ANIMATION || ct == TGI_CT_AUDIO || ct == TGI_CT_VOICE_NOTE;
}

/* extractLinksFromFormattedText (tdutils.go:897-949). returns -1 if the Go code would panic.      */
static int extract_links(const tgi_tg_batch* b, uint64_t r, linkset_t* ls) {
  const tgi_tg_rec* rec = &b->recs[r];
  if (!ct_carries_links(rec->content_type) || !(rec->flags & TGI_RF_HAS_TEXT)) return 0;
  const uint8_t* text = b->strs + rec->str_off;
  int64_t tn = rec->text_len;
  uint32_t e0 = b->ent_off ? b->ent_off[r] : 0, e1 = b->ent_off ? b->ent_off[r + 1] : 0;
  for (uint32_t e = e0; e < e1; e++) {
    const tgi_entity* en = &b->ents[e];
    int64_t ns, ne;
    if (en->type == TGI_ENT_TEXT_URL) { /* :910-916 */
      const uint8_t* url = b->aux + en->url_off;
      if (orc_channel_link_first(url, en->url_len, 0, &ns, &ne))
        add_channel_match(ls, url, ns, ne, TGI_SRC_TEXT_URL);
    } else if (en->type == TGI_ENT_MENTION || en->type == TGI_ENT_URL) { /* :917-938 */
      int64_t st, en_;
      orc_utf16_offset_to_bytes(text, tn, en->offset, en->length, &st, &en_);
      if (st < en_ && en_ <= tn) {
        if (st < 0) return -1; /* ft.Text[-1:end] -> panic, recovered at :395-405 */
        if (en->type == TGI_ENT_MENTION) {
          if (orc_username_first(text + st, en_ - st, &ns, &ne))
            linkset_add(ls, text + st + ns, (int)(ne - ns), TGI_SRC_MENTION);
        } else {
          if (orc_channel_link_first(text + st, en_ - st, 0, &ns, &ne))
            add_channel_match(ls, text + st, ns, ne, TGI_SRC_URL);
        }
      }
    }
  }
  /* FindAllStringSubmatch over the whole text (:943-948): successive non-overlapping matches */
  int64_t from = 0, ns, ne;
  while (orc_channel_link_first(text, tn, from, &ns, &ne)) {
    add_channel_match(ls, text, ns, ne, TGI_SRC_PLAINTEXT);
    from = ne;
  }
  return 0;
}

int orc_extract_links(const tgi_tg_batch* b, uint64_t rec, tgi_link* out, int cap) {
  linkset_t ls = {out, 0, cap, 0, NULL};
  if (extract_links(b, rec, &ls) < 0) return -1;
  return ls.overflow ? -2 : ls.n;
}

/* ------------------------------------------------------------------------------------------- */
/* Go encoding/json string encoder (encode.go appendString, escapeHTML = true, go >= 1.22)         */
uint64_t orc_json_string(const uint8_t* s, uint64_t n, uint8_t* dst) {
  static const char hex[] = "0123456789abcdef";
  uint64_t o = 0;
#define PUT(c)                      \
  do {                              \
    if (dst) dst[o] = (uint8_t)(c); \
    o++;                            \
  } while (0)
  PUT('"');
  for (uint64_t i = 0; i < n;) {
    uint8_t b = s[i];
    if (b < 0x80) {
      if (b >= 0x20 && b != '"' && b != '\\' && b != '<' && b != '>' && b != '&') {
        PUT(b);
      } else {
        PUT('\\');
        switch (b) {
          case '\\': PUT('\\'); break;
          case '"': PUT('"'); break;
          case '\b': PUT('b'); break;
          case '\f': PUT('f'); break;
          case '\n': PUT('n'); break;
          case '\r': PUT('r'); break;
          case '\t': PUT('t'); break;
          default:
            PUT('u'); PUT('0'); PUT('0'); PUT(hex[b >> 4]); PUT(hex[b & 0xF]);
        }
      }
      i++;
      continue;
    }
    uint32_t r;
    int w = go_decode_rune(s + i, (int64_t)(n - i), &r);
    if (r == 0xFFFD && w == 1) {
      PUT('\\'); PUT('u'); PUT('f'); PUT('f'); PUT('f'); PUT('d');
      i += 1;
      continue;
    }
    if (r == 0x2028 || r == 0x2029) {
      PUT('\\'); PUT('u'); PUT('2'); PUT('0'); PUT('2'); PUT(hex[r & 0xF]);
      i += (uint64_t)w;
      continue;
    }
    for (int k = 0; k < w; k++) PUT(s[i + (uint64_t)k]);
    i += (uint64_t)w;
  }
  PUT('"');
#undef PUT
  return o;
}

static void put_jstr(buf_t* b, const uint8_t* s, uint64_t n) {
  buf_reserve(b, n * 6 + 2);
  b->len += orc_json_string(s, n, b->p + b->len);
}
static void put_int(buf_t* b, int64_t v) {
  char t[24];
  int k = snprintf(t, sizeof t, "%lld", (long long)v);
  buf_put(b, t, (size_t)k);
}

/* time.Time.MarshalJSON -> RFC3339Nano with quotes; local zone = fixed offset.  0 on year error */
int orc_json_time(int64_t sec, int32_t nsec, int32_t tz, uint8_t* dst) {
  int64_t t = sec + tz;
  int64_t days = t / 86400, rem = t % 86400;
  if (rem < 0) { rem += 86400; days -= 1; }
  /* civil from days (proleptic Gregorian) */
  int64_t z = days + 719468;
  int64_t era = (z >= 0 ? z : z - 146096) / 146097;
  int64_t doe = z - era * 146097;
  int64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  int64_t y = yoe + era * 400;
  int64_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
  int64_t mp = (5 * doy + 2) / 153;
  int64_t d = doy - (153 * mp + 2) / 5 + 1;
  int64_t m = mp < 10 ? mp + 3 : mp - 9;
  if (m <= 2) y += 1;
  if (y < 0 || y > 9999) return 0;
  int o = 0;
  o += sprintf((char*)dst + o, "\"%04d-%02d-%02dT%02d:%02d:%02d", (int)y, (int)m, (int)d,
               (int)(rem / 3600), (int)(rem % 3600 / 60), (int)(rem % 60));
  if (nsec != 0) {
    char f[16];
    sprintf(f, "%09d", nsec);
    int k = 9;
    while (k > 0 && f[k - 1] == '0') k--;
    dst[o++] = '.';
    memcpy(dst + o, f, (size_t)k);
    o += k;
  }
  if (tz == 0) {
    dst[o++] = 'Z';
  } else {
    int a = tz < 0 ? -tz : tz;
    /* Go prints zone as +hh:mm (seconds dropped; RFC3339 in MarshalJSON rejects non-minute
     * offsets only via the hour range check, so second-granular zones are not supported here) */
    o += sprintf((char*)dst + o, "%c%02d:%02d", tz < 0 ? '-' : '+', a / 3600, a % 3600 / 60);
  }
  dst[o++] = '"';
  return o;
}
static int put_time(buf_t* b, int64_t sec, int32_t nsec, int32_t tz) {
  buf_reserve(b, 48);
  int k = orc_json_time(sec, nsec, tz, b->p + b->len);
  b->len += (size_t)k;
  return k;
}

/* strconv.FormatFloat(float64(v), 'f', -1, 64): shortest decimal that round-trips, in plain
 * positional form (the values here are integers < 1e21 so encoding/json never switches to 'e'). */
int orc_json_float_of_int64(int64_t v, uint8_t* dst) {
  double f = (double)v;
  char t[64];
  for (int prec = 1; prec <= 17; prec++) {
    snprintf(t, sizeof t, "%.*e", prec - 1, f);
    if (strtod(t, NULL) == f) break;
  }
  /* t = d.ddddde+XX -> expand */
  char digits[32];
  int nd = 0, neg = 0;
  const char* p = t;
  if (*p == '-') { neg = 1; p++; }
  for (; *p && *p != 'e'; p++)
    if (*p >= '0' && *p <= '9') digits[nd++] = *p;
  int ex = atoi(p + 1);
  int o = 0;
  if (f == 0) {
    dst[o++] = '0';
    return o;
  }
  if (neg) dst[o++] = '-';
  /* integer values: exponent >= 0 always */
  for (int i = 0; i <= ex; i++) dst[o++] = (uint8_t)(i < nd ? digits[i] : '0');
  /* trailing non-zero fraction digits cannot occur for integral doubles with nd <= ex+1 */
  return o;
}

/* ------------------------------------------------------------------------------------------- */
/* frontier set: exact string set, first occurrence wins, insertion order kept.
 * The set is split into ORC_SHARDS independent shards by the top bits of the key hash so that the
 * batch driver can insert from many threads without a lock (one owner thread per shard).  Every key
 * carries the global sequence number of its first occurrence; the insertion order of the whole set
 * is the order of those numbers (orc_frontier_export sorts by them).  Sequentially (one thread, or
 * orc_frontier_insert) this is exactly the mutex-guarded Go map + append of the reference
 * (crawl/runner.go:1267-1272, state/daprstate.go:646-658).                                        */
#define ORC_SHARD_BITS 8
#define ORC_SHARDS (1 << ORC_SHARD_BITS)
typedef struct {
  uint8_t (*keys)[32];
  uint64_t* seq;   /* global first-occurrence sequence number of keys[i] */
  uint64_t n, cap;
  uint64_t* slots; /* index+1 into keys, 0 = empty */
  uint64_t nslots;
} fset_t;

static uint64_t key_hash(const uint8_t* k) {
  uint64_t h = 1469598103934665603ull;
  uint64_t w[4];
  memcpy(w, k, 32);
  for (int i = 0; i < 4; i++) {
    h = (h ^ w[i]) * 0xFF51AFD7ED558CCDull;
    h ^= h >> 32;
  }
  h *= 0xC4CEB9FE1A85EC53ull;
  return h ^ (h >> 29);
}
static void fset_grow(fset_t* f) {
  uint64_t ns = f->nslots ? f->nslots * 2 : 1 << 10;
  uint64_t* s = (uint64_t*)calloc(ns, sizeof(uint64_t));
  for (uint64_t i = 0; i < f->n; i++) {
    uint64_t h = key_hash(f->keys[i]) & (ns - 1);
    while (s[h]) h = (h + 1) & (ns - 1);
    s[h] = i + 1;
  }
  free(f->slots);
  f->slots = s;
  f->nslots = ns;
}
static int fset_insert_h(fset_t* f, const uint8_t* k, uint64_t hash, uint64_t seq) {
  if ((f->n + 1) * 2 > f->nslots) fset_grow(f);
  uint64_t h = hash & (f->nslots - 1);
  while (f->slots[h]) {
    if (memcmp(f->keys[f->slots[h] - 1], k, 32) == 0) return 0;
    h = (h + 1) & (f->nslots - 1);
  }
  if (f->n == f->cap) {
    f->cap = f->cap ? f->cap * 2 : 1 << 8;
    f->keys = realloc(f->keys, f->cap * 32);
    f->seq = realloc(f->seq, f->cap * 8);
  }
  memcpy(f->keys[f->n], k, 32);
  f->seq[f->n] = seq;
  f->slots[h] = ++f->n;
  return 1;
}
static inline unsigned key_shard(uint64_t hash) { return (unsigned)(hash >> (64 - ORC_SHARD_BITS)); }
static int64_t fset_find(const fset_t* f, const uint8_t* k) { /* index of k, or -1 */
  if (!f->nslots) return -1;
  uint64_t h = key_hash(k) & (f->nslots - 1);
  while (f->slots[h]) {
    if (memcmp(f->keys[f->slots[h] - 1], k, 32) == 0) return (int64_t)f->slots[h] - 1;
    h = (h + 1) & (f->nslots - 1);
  }
  return -1;
}
/* sm.IsInvalidChannel (state/daprstate.go:3556-3564): in the cache and time.Since(t) < invalidChannelTTL (30 days, :3489) */
static int is_invalid_channel(const fset_t* inv, const uint8_t* k, int64_t now_sec) {
  int64_t i = fset_find(inv, k);
  if (i < 0) return 0;
  int64_t t = (int64_t)inv->seq[i];
  return t == 0 || now_sec - t < (int64_t)TGI_INVALID_TTL_SEC;
}

/* per-thread scratch + result arrays are owned by the context and only grow: after one warm-up call
 * a batch of the same size touches no fresh pages (first-touch page faults would otherwise dominate
 * the timed CPU baseline). */
typedef struct work work_t;
struct work {
  const orc_ctx* c;
  const tgi_tg_batch* tg;
  const tgi_yt_batch* yt;
  const tgi_gm_batch* gm;
  uint64_t r0, r1;
  uint32_t run_flags;
  buf_t json;        /* lines of this range */
  buf_t links;       /* tgi_link[] */
  buf_t b_linelen, b_status, b_nlinks, b_tmp, scratch;
  uint64_t* linelen; /* [r1-r0] */
  uint8_t* status;   /* [r1-r0] */
  uint32_t* nlinks;  /* [r1-r0] */
  /* parallel driver */
  int tid, nthreads;
  struct batch_job* job;
  buf_t bucket[ORC_SHARDS]; /* indexes (into this thread's links) of the eligible links, per frontier shard */
  uint64_t json_base, link_base; /* prefix sums over the threads */
  uint64_t n_new;
};
struct orc_ctx {
  tgi_config cfg;
  char* label;
  fset_t fs[ORC_SHARDS];
  uint64_t seq; /* next global sequence number */
  fset_t xset[2]; /* frontier -> validator hand-off: invalid channels (seq[] = time marked), discovered channels */
  int64_t now_sec; /* clock of the invalid-channel TTL in the batch path; 0 = never expire */
  work_t* w;
  int nw;
  buf_t r_status, r_jsonl, r_line_off, r_link_off, r_links;
};

/* time.Time's nanoseconds, and time.FixedZone offsets under a day: what tgi_create / tgi_set_clock and the batch
 * uploads of the library accept (anything else is TGI_E_ARG there and here) */
static int nsec_ok(int32_t nsec) { return nsec >= 0 && nsec < 1000000000; }

int orc_create(const tgi_config* cfg, orc_ctx** out) {
  *out = NULL;
  if (!nsec_ok(cfg->created_at_nsec) || !nsec_ok(cfg->capture_nsec)) return TGI_E_ARG;
  if (cfg->tz_offset_sec <= -86400 || cfg->tz_offset_sec >= 86400) return TGI_E_ARG;
  orc_ctx* c = (orc_ctx*)calloc(1, sizeof(*c));
  c->cfg = *cfg;
  c->label = (char*)malloc(cfg->crawl_label_len + 1);
  if (cfg->crawl_label_len) memcpy(c->label, cfg->crawl_label, cfg->crawl_label_len);
  c->cfg.crawl_label = c->label;
  *out = c;
  return TGI_OK;
}
void orc_destroy(orc_ctx* c) {
  if (!c) return;
  for (int t = 0; t < c->nw; t++) {
    work_t* w = &c->w[t];
    free(w->json.p); free(w->links.p); free(w->b_linelen.p); free(w->b_status.p); free(w->b_nlinks.p);
    free(w->b_tmp.p); free(w->scratch.p);
    for (int i = 0; i < ORC_SHARDS; i++) free(w->bucket[i].p);
  }
  free(c->w);
  free(c->r_status.p); free(c->r_jsonl.p); free(c->r_line_off.p); free(c->r_link_off.p); free(c->r_links.p);
  free(c->label);
  for (int i = 0; i < ORC_SHARDS; i++) { free(c->fs[i].keys); free(c->fs[i].seq); free(c->fs[i].slots); }
  for (int i = 0; i < 2; i++) { free(c->xset[i].keys); free(c->xset[i].seq); free(c->xset[i].slots); }
  free(c);
}
int orc_set_clock(orc_ctx* c, int64_t cs, int32_t cn, int64_t ps, int32_t pn) {
  if (!nsec_ok(cn) || !nsec_ok(pn)) return TGI_E_ARG; /* the previous clock stays */
  c->cfg.created_at_sec = cs;
  c->cfg.created_at_nsec = cn;
  c->cfg.capture_sec = ps;
  c->cfg.capture_nsec = pn;
  return TGI_OK;
}
int orc_frontier_insert(orc_ctx* c, const uint8_t* keys32, uint64_t n, uint8_t* is_new) {
  for (uint64_t i = 0; i < n; i++) {
    const uint64_t h = key_hash(keys32 + 32 * i);
    int nw = fset_insert_h(&c->fs[key_shard(h)], keys32 + 32 * i, h, c->seq++);
    if (is_new) is_new[i] = (uint8_t)nw;
  }
  return 0;
}
uint64_t orc_frontier_size(orc_ctx* c) {
  uint64_t n = 0;
  for (int i = 0; i < ORC_SHARDS; i++) n += c->fs[i].n;
  return n;
}
typedef struct { uint64_t seq; const uint8_t* key; } seqkey_t;
static int seqkey_cmp(const void* a, const void* b) {
  const uint64_t x = ((const seqkey_t*)a)->seq, y = ((const seqkey_t*)b)->seq;
  return x < y ? -1 : (x > y ? 1 : 0);
}
/* keys in first-occurrence order */
uint64_t orc_frontier_export(orc_ctx* c, uint8_t* keys32, uint64_t cap) {
  const uint64_t tot = orc_frontier_size(c);
  seqkey_t* v = (seqkey_t*)malloc(sizeof(seqkey_t) * (tot ? tot : 1));
  uint64_t m = 0;
  for (int i = 0; i < ORC_SHARDS; i++)
    for (uint64_t k = 0; k < c->fs[i].n; k++) { v[m].seq = c->fs[i].seq[k]; v[m].key = c->fs[i].keys[k]; m++; }
  qsort(v, m, sizeof(seqkey_t), seqkey_cmp);
  const uint64_t n = tot < cap ? tot : cap;
  for (uint64_t k = 0; k < n; k++) memcpy(keys32 + 32 * k, v[k].key, 32);
  free(v);
  return n;
}
void orc_frontier_clear(orc_ctx* c) {
  for (int i = 0; i < ORC_SHARDS; i++) {
    c->fs[i].n = 0;
    if (c->fs[i].slots) memset(c->fs[i].slots, 0, c->fs[i].nslots * sizeof(uint64_t));
  }
}

/* ------------------------------------------------------------------------------------------- */
/* Telegram: ParseMessage (tdutils.go:380-732) + json.Marshal(post)+'\n' (storageproviders.go:276) */
static const char* const kPostType[TGI_CT__COUNT] = {
    "unknown",          "messageText",      "messageVideo",           "messagePhoto",
    "messageAnimation", "messageAnimatedEmoji", "messagePoll",        "messageGiveaway",
    "messagePaidMedia", "messageSticker",   "messageGiveawayWinners", "messageGiveawayCompleted",
    "messageVideoNote", "messageDocument",  "messageAudio",           "messageVoiceNote",
    NULL};

typedef struct {
  const uint8_t* p;
  uint64_t n;
  int32_t count;
} kv_t;
static int kv_cmp(const void* a, const void* b) { /* encoding/json sorts map keys bytewise */
  const kv_t *x = a, *y = b;
  uint64_t m = x->n < y->n ? x->n : y->n;
  int c = memcmp(x->p, y->p, m);
  if (c) return c;
  return x->n < y->n ? -1 : (x->n > y->n ? 1 : 0);
}
/* map[string]int from a reaction list (later duplicates overwrite: Go map assignment) */
static void put_reaction_map(buf_t* o, const tgi_tg_batch* b, uint32_t r0, uint32_t r1) {
  uint32_t cnt = r1 - r0;
  kv_t* kv = (kv_t*)malloc(sizeof(kv_t) * (cnt ? cnt : 1));
  uint32_t m = 0;
  for (uint32_t i = r0; i < r1; i++) {
    const tgi_reaction* rc = &b->reacts[i];
    const uint8_t* p = b->aux + rc->emoji_off;
    uint32_t j = 0;
    for (; j < m; j++)
      if (kv[j].n == rc->emoji_len && memcmp(kv[j].p, p, rc->emoji_len) == 0) break;
    if (j == m) m++;
    kv[j].p = p;
    kv[j].n = rc->emoji_len;
    kv[j].count = rc->count;
  }
  qsort(kv, m, sizeof(kv_t), kv_cmp);
  LIT(o, "{");
  for (uint32_t j = 0; j < m; j++) {
    if (j) LIT(o, ",");
    put_jstr(o, kv[j].p, kv[j].n);
    LIT(o, ":");
    put_int(o, kv[j].count);
  }
  LIT(o, "}");
  free(kv);
}

/* returns status; on TGI_ST_EMITTED appends one line to o and the links to ls */
static int tg_record(const orc_ctx* c, const tgi_tg_batch* b, uint64_t r, buf_t* o, linkset_t* ls, int want_json) {
  const tgi_config* cfg = &c->cfg;
  const tgi_tg_rec* rec = &b->recs[r];
  const tgi_tg_chan* ch = &b->chans[rec->chan_idx];
  const uint8_t* cs = b->chan_strs + ch->str_off;
  const uint8_t *title = cs, *cname = cs + ch->title_len, *user = cname + ch->name_len;
  const uint8_t* text = b->strs + rec->str_off;
  const uint8_t* alt = text + rec->text_len;
  const uint8_t* media = alt + rec->alt_len;
  const uint8_t* handle = media + rec->media_len;
  int ct = rec->content_type;

  /* tdutils.go:415-421 */
  int64_t msgno = rec->id / 1048576; /* Go integer division truncates toward zero, as C */
  if ((cfg->flags & TGI_CFG_HAS_MIN_POST_DATE) && (int64_t)rec->date < cfg->min_post_date)
    return TGI_ST_SKIPPED;
  if (rec->flags & TGI_RF_PANIC) return TGI_ST_FAILED;

  /* :443-587 description / media by content type */
  const uint8_t* desc = (const uint8_t*)"";
  uint64_t desc_len = 0;
  int has_text = (rec->flags & TGI_RF_HAS_TEXT) != 0;
  switch (ct) {
    case TGI_CT_TEXT: case TGI_CT_VIDEO: case TGI_CT_PHOTO: case TGI_CT_ANIMATION:
      if (has_text) { desc = text; desc_len = rec->text_len; }
      break;
    case TGI_CT_ANIMATED_EMOJI: case TGI_CT_POLL: case TGI_CT_GIVEAWAY: case TGI_CT_PAID_MEDIA:
    case TGI_CT_DOCUMENT:
      desc = alt; desc_len = rec->alt_len;
      break;
    default: break;
  }
  int has_media = (ct == TGI_CT_VIDEO || ct == TGI_CT_VIDEO_NOTE || ct == TGI_CT_DOCUMENT);

  /* :590 outlinks */
  if (extract_links(b, r, ls) < 0) return TGI_ST_FAILED;
  if (!want_json) return TGI_ST_EMITTED; /* link extraction + dedup only (BASELINE configs 3 / 5): no Post is built */

  size_t line_start = o->len;
  /* link, tdutils.go:1005-1031 */
  buf_t link = {0};
  if (ch->user_len) {
    LIT(&link, "https://t.me/");
    buf_put(&link, user, ch->user_len);
    LIT(&link, "/");
    put_int(&link, msgno);
    if (rec->media_album_id != 0) LIT(&link, "?single");
  }
  buf_t uid = {0};
  put_int(&uid, msgno);
  LIT(&uid, "-");
  buf_put(&uid, cname, ch->name_len);
  buf_t curl = {0};
  LIT(&curl, "https://t.me/c/");
  buf_put(&curl, cname, ch->name_len);
  char chatid[24];
  int chatid_n = snprintf(chatid, sizeof chatid, "%lld", (long long)rec->chat_id);
  uint32_t c0 = b->comment_off ? b->comment_off[r] : 0, c1 = b->comment_off ? b->comment_off[r + 1] : 0;
  int64_t ncomments = (rec->flags & TGI_RF_COMMENTS_NIL) ? 0 : (int64_t)(c1 - c0);

  int ok = 1;
  LIT(o, "{\"post_link\":"); put_jstr(o, link.p, link.len);
  LIT(o, ",\"channel_id\":"); put_jstr(o, (const uint8_t*)chatid, (uint64_t)chatid_n);
  LIT(o, ",\"post_uid\":"); put_jstr(o, uid.p, uid.len);
  LIT(o, ",\"url\":"); put_jstr(o, link.p, link.len);
  LIT(o, ",\"published_at\":"); ok &= put_time(o, rec->date, 0, cfg->tz_offset_sec) > 0;
  LIT(o, ",\"created_at\":"); ok &= put_time(o, cfg->created_at_sec, 0, 0) > 0;
  LIT(o, ",\"language_code\":\"\",\"engagement\":"); put_int(o, rec->view_count);
  LIT(o, ",\"view_count\":"); put_int(o, rec->view_count);
  LIT(o, ",\"like_count\":0,\"share_count\":"); put_int(o, rec->share_count);
  LIT(o, ",\"comment_count\":"); put_int(o, ncomments);
  LIT(o, ",\"crawl_label\":"); put_jstr(o, (const uint8_t*)cfg->crawl_label, cfg->crawl_label_len);
  LIT(o, ",\"list_ids\":null,\"channel_name\":"); put_jstr(o, title, ch->title_len);
  LIT(o, ",\"search_terms\":null,\"search_term_ids\":null,\"project_ids\":null,\"exercise_ids\":null,"
         "\"label_data\":null,\"labels_metadata\":null,\"project_labeled_post_ids\":null,"
         "\"labeler_ids\":null,\"all_labels\":null,\"label_ids\":null,\"is_ad\":false,"
         "\"transcript_text\":\"\",\"image_text\":\"\",\"video_length\":null,\"is_verified\":null,"
         "\"channel_data\":{\"channel_id\":");
  put_jstr(o, (const uint8_t*)chatid, (uint64_t)chatid_n);
  LIT(o, ",\"channel_name\":"); put_jstr(o, title, ch->title_len);
  LIT(o, ",\"channel_description\":\"\",\"channel_profile_image\":\"\",\"channel_engagement_data\":{"
         "\"follower_count\":");
  put_int(o, ch->member_count);
  LIT(o, ",\"following_count\":0,\"like_count\":0,\"post_count\":"); put_int(o, ch->post_count);
  LIT(o, ",\"views_count\":"); put_int(o, ch->view_count);
  LIT(o, ",\"comment_count\":0,\"share_count\":0},\"channel_url_external\":");
  put_jstr(o, curl.p, curl.len);
  LIT(o, ",\"channel_url\":"); put_jstr(o, curl.p, curl.len);
  LIT(o, ",\"country_code\":\"\",\"published_at\":\"0001-01-01T00:00:00Z\"},"
         "\"platform_name\":\"Telegram\",\"shared_id\":null,\"quoted_id\":null,\"replied_id\":null,"
         "\"ai_label\":null,\"root_post_id\":null,\"engagement_steps_count\":0,\"ocr_data\":null,"
         "\"performance_scores\":{\"likes\":null,\"shares\":null,\"comments\":null,\"views\":0},"
         "\"has_embed_media\":null,\"description\":");
  put_jstr(o, desc, desc_len);
  LIT(o, ",\"repost_channel_data\":null,\"post_type\":[");
  if (ct == TGI_CT_OTHER) put_jstr(o, alt, rec->alt_len);
  else put_jstr(o, (const uint8_t*)kPostType[ct], strlen(kPostType[ct]));
  LIT(o, "],\"inner_link\":{},\"post_title\":null,\"media_data\":{\"document_name\":\"\"},"
         "\"is_reply\":null,\"ad_fields\":null,\"likes_count\":0,\"shares_count\":");
  put_int(o, rec->share_count);
  LIT(o, ",\"comments_count\":"); put_int(o, ncomments);
  LIT(o, ",\"views_count\":"); put_int(o, rec->view_count);
  LIT(o, ",\"searchable_text\":\"\",\"all_text\":\"\",\"contrast_agent_project_ids\":null,"
         "\"agent_ids\":null,\"segment_ids\":null,\"thumb_url\":\"\",\"media_url\":");
  /* thumb_url is always "" under SkipMediaDownload (fetchAndUploadMedia returns "", :233-239) */
  if (has_media) put_jstr(o, media, rec->media_len); else LIT(o, "\"\"");
  LIT(o, ",\"comments\":");
  if (rec->flags & TGI_RF_COMMENTS_NIL) {
    LIT(o, "null");
  } else {
    LIT(o, "[");
    for (uint32_t k = c0; k < c1; k++) {
      const tgi_comment* cm = &b->comments[k];
      if (k > c0) LIT(o, ",");
      LIT(o, "{\"text\":"); put_jstr(o, b->aux + cm->text_off, cm->text_len);
      LIT(o, ",\"reactions\":");
      if (cm->flags & 1) put_reaction_map(o, b, cm->react_start, cm->react_start + cm->react_count);
      else LIT(o, "null");
      LIT(o, ",\"view_count\":"); put_int(o, cm->view_count);
      LIT(o, ",\"reply_count\":"); put_int(o, cm->reply_count);
      LIT(o, ",\"handle\":"); put_jstr(o, b->aux + cm->handle_off, cm->handle_len);
      LIT(o, "}");
    }
    LIT(o, "]");
  }
  LIT(o, ",\"reactions\":");
  {
    uint32_t r0 = b->react_off ? b->react_off[r] : 0, r1 = b->react_off ? b->react_off[r + 1] : 0;
    put_reaction_map(o, b, r0, r1);
  }
  LIT(o, ",\"outlinks\":[");
  for (int k = 0; k < ls->n; k++) {
    if (k) LIT(o, ",");
    put_jstr(o, ls->v[k].name, ls->v[k].len);
  }
  LIT(o, "],\"capture_time\":");
  ok &= put_time(o, cfg->capture_sec, cfg->capture_nsec, cfg->tz_offset_sec) > 0;
  LIT(o, ",\"handle\":"); put_jstr(o, handle, rec->handle_len);
  LIT(o, "}\n");
  free(link.p);
  free(uid.p);
  free(curl.p);
  if (!ok) { /* Marshal error: nothing is written (StorePost error is swallowed) */
    o->len = line_start;
    return TGI_ST_NOLINE;
  }
  return TGI_ST_EMITTED;
}

/* ------------------------------------------------------------------------------------------- */
/* YouTube helpers (crawler/youtube/youtube_crawler.go)                                          */
static int is_digit(uint8_t c) { return c >= '0' && c <= '9'; }

/* strconv.Atoi on a digit string: clamps to MaxInt64 on overflow (the error is ignored, :473) */
static int64_t atoi_clamp(const uint8_t* s, int64_t n) {
  uint64_t v = 0;
  for (int64_t i = 0; i < n; i++) {
    uint64_t d = (uint64_t)(s[i] - '0');
    if (v > (uint64_t)INT64_MAX / 10 || v * 10 > (uint64_t)INT64_MAX - d) return INT64_MAX;
    v = v * 10 + d;
  }
  return (int64_t)v;
}

/* :461-486 parseISO8601Duration: ^P(?:(\d+)D)?(?:T(?:(\d+)H)?(?:(\d+)M)?(?:(\d+)S)?)?$            */
int orc_parse_iso8601_duration(const uint8_t* s, int64_t n, int64_t* seconds) {
  int64_t i = 0;
  uint64_t total = 0; /* Go int arithmetic wraps */
  if (i >= n || s[i] != 'P') return 0;
  i++;
  int64_t j = i;
  while (j < n && is_digit(s[j])) j++;
  if (j > i && j < n && s[j] == 'D') {
    total += (uint64_t)atoi_clamp(s + i, j - i) * 86400u;
    i = j + 1;
  }
  if (i < n && s[i] == 'T') {
    i++;
    static const char unit[3] = {'H', 'M', 'S'};
    static const uint64_t mul[3] = {3600, 60, 1};
    for (int u = 0; u < 3; u++) {
      j = i;
      while (j < n && is_digit(s[j])) j++;
      if (j > i && j < n && s[j] == unit[u]) {
        total += (uint64_t)atoi_clamp(s + i, j - i) * mul[u];
        i = j + 1;
      }
    }
  }
  if (i != n) return 0;
  *seconds = (int64_t)total;
  return 1;
}

static int is_re2_space(uint8_t c) { return c == '\t' || c == '\n' || c == '\f' || c == '\r' || c == ' '; }

typedef struct { const uint8_t* p; uint64_t n; } span_t;

/* :489-513 extractURLs: (https?://\S+) FindAllString, TrimRight(",.;:!?()'\""), dedup; canonical
 * order = first occurrence (Go's map order is random).  Returns count, fills out[cap].          */
static int extract_urls(const uint8_t* s, uint64_t n, span_t* out, int cap) {
  int m = 0;
  uint64_t i = 0;
  while (i + 8 <= n) { /* "http://" + at least one \S */
    uint64_t k = 0;
    if (memcmp(s + i, "http://", 7) == 0) k = 7;
    else if (i + 8 <= n && memcmp(s + i, "https://", 8) == 0) k = 8;
    if (!k || i + k >= n || is_re2_space(s[i + k])) { i++; continue; }
    uint64_t e = i + k;
    while (e < n && !is_re2_space(s[e])) e++;
    uint64_t te = e;
    while (te > i && strchr(",.;:!?()'\"", s[te - 1]) && s[te - 1] != 0) te--;
    int dup = 0;
    for (int j = 0; j < m; j++)
      if (out[j].n == te - i && memcmp(out[j].p, s + i, te - i) == 0) { dup = 1; break; }
    if (!dup && m < cap) { out[m].p = s + i; out[m].n = te - i; m++; }
    i = e;
  }
  return m;
}

/* :516-527 sanitizeFilename: [^\w\-.] -> "_" per rune (invalid byte = U+FFFD = one rune), then
 * truncate to 50 bytes */
static void sanitize_filename(const uint8_t* s, uint64_t n, buf_t* o) {
  size_t start = o->len;
  for (uint64_t i = 0; i < n;) {
    uint32_t r;
    int w = go_decode_rune(s + i, (int64_t)(n - i), &r);
    uint8_t c = s[i];
    if (w == 1 && r < 0x80 && (is_word(c) || c == '-' || c == '.')) buf_put(o, &c, 1);
    else LIT(o, "_");
    i += (uint64_t)w;
  }
  if (o->len - start > 50) o->len = start + 50;
}

static int is_uc_char(uint8_t c) { return is_word(c) || c == '-'; }
static int is_handle_char(uint8_t c) { return is_word(c) || c == '-' || c == '.'; }

/* client/youtube_client.go:1856-1878 extractChannelIDsFromText: all youtube\.com/channel/([\w-]+)
 * matches, then all youtube\.com/@([\w.-]+) matches ("@"+h); no dedup here.                     */
static void yt_channel_ids(const uint8_t* s, uint64_t n, linkset_t* ls_nodedup) {
  static const char p1[] = "youtube.com/channel/";
  static const char p2[] = "youtube.com/@";
  for (int pass = 0; pass < 2; pass++) {
    const char* pat = pass ? p2 : p1;
    uint64_t pl = strlen(pat);
    uint64_t i = 0;
    while (i + pl < n) {
      if (memcmp(s + i, pat, pl) != 0) { i++; continue; }
      uint64_t q = i + pl, e = q;
      while (e < n && (pass ? is_handle_char(s[e]) : is_uc_char(s[e]))) e++;
      if (e == q) { i++; continue; }
      if (ls_nodedup->n < ls_nodedup->cap) {
        tgi_link* l = &ls_nodedup->v[ls_nodedup->n++];
        memset(l, 0, sizeof *l);
        /* keys longer than 32 bytes are truncated for the fixed-width frontier (documented limit:
         * real channel ids are 24 chars, handles <= 30) */
        uint64_t len = e - q, o = 0;
        if (pass) l->name[o++] = '@';
        for (uint64_t k = 0; k < len && o < 32; k++) l->name[o++] = s[q + k];
        l->len = (uint8_t)o;
        l->src = (uint8_t)pass;
      } else {
        ls_nodedup->overflow = 1;
      }
      i = e;
    }
  }
}

static const char* const kThumbKey[5] = {"default", "medium", "high", "standard", "maxres"};

static int yt_record(const orc_ctx* c, const tgi_yt_batch* b, uint64_t r, buf_t* o, linkset_t* ls) {
  const tgi_config* cfg = &c->cfg;
  const tgi_yt_rec* v = &b->recs[r];
  const tgi_yt_chan* ch = &b->chans[v->chan_idx];
  const uint8_t* cs = b->chan_strs + ch->str_off;
  const uint8_t *chid = cs, *chtitle = chid + ch->id_len, *chdesc = chtitle + ch->title_len,
                *chthumb = chdesc + ch->desc_len, *chcountry = chthumb + ch->thumb_len;
  const uint8_t* p = b->strs + v->str_off;
  const uint8_t *id = p, *title = id + v->id_len, *desc = title + v->title_len,
                *dur = desc + v->desc_len, *lang = dur + v->duration_len;
  const uint8_t* th[5];
  uint64_t thn[5];
  {
    const uint8_t* q = lang + v->lang_len;
    for (int k = 0; k < 5; k++) {
      th[k] = q;
      thn[k] = v->thumb_len[k] == TGI_YT_THUMB_ABSENT ? 0 : v->thumb_len[k];
      q += thn[k];
    }
  }
  /* :561 */
  int64_t engagement = (int64_t)((uint64_t)v->like_count + (uint64_t)v->comment_count +
                                 (uint64_t)(v->view_count / 100));
  /* :615-624 thumb priority maxres > high > medium > default */
  static const int prio[4] = {4, 2, 1, 0};
  const uint8_t* thumb = (const uint8_t*)"";
  uint64_t thumb_n = 0;
  for (int k = 0; k < 4; k++)
    if (thn[prio[k]]) { thumb = th[prio[k]]; thumb_n = thn[prio[k]]; break; }
  /* :631-643 duration */
  int has_len = 0;
  int64_t vlen = 0;
  if (v->duration_len && !(v->duration_len == 3 && memcmp(dur, "P0D", 3) == 0))
    has_len = orc_parse_iso8601_duration(dur, v->duration_len, &vlen);
  /* :664 */
  span_t urls[1024];
  int nurls = extract_urls(desc, v->desc_len, urls, 1024);
  /* snowball frontier candidates (youtube_client.go:1706) */
  yt_channel_ids(desc, v->desc_len, ls);

  size_t line_start = o->len;
  int ok = 1;
  buf_t vurl = {0};
  LIT(&vurl, "https://www.youtube.com/watch?v=");
  buf_put(&vurl, id, v->id_len);
  buf_t churl = {0};
  if (ch->id_len > 0 && chid[0] == '@') LIT(&churl, "https://www.youtube.com/");
  else LIT(&churl, "https://www.youtube.com/channel/");
  buf_put(&churl, chid, ch->id_len);
  const uint8_t* chname = ch->cached ? chtitle : chid;
  uint64_t chname_n = ch->cached ? ch->title_len : ch->id_len;
  buf_t alltext = {0};
  buf_put(&alltext, title, v->title_len);
  LIT(&alltext, " ");
  buf_put(&alltext, desc, v->desc_len);
  buf_t docname = {0};
  buf_put(&docname, id, v->id_len);
  LIT(&docname, "-");
  sanitize_filename(title, v->title_len, &docname);
  LIT(&docname, ".mp4");

  LIT(o, "{\"post_link\":"); put_jstr(o, vurl.p, vurl.len);
  LIT(o, ",\"channel_id\":"); put_jstr(o, chid, ch->id_len);
  LIT(o, ",\"post_uid\":"); put_jstr(o, id, v->id_len);
  LIT(o, ",\"url\":"); put_jstr(o, vurl.p, vurl.len);
  LIT(o, ",\"published_at\":"); ok &= put_time(o, v->published_sec, v->published_nsec, 0) > 0;
  LIT(o, ",\"created_at\":");
  ok &= put_time(o, cfg->created_at_sec, cfg->created_at_nsec, cfg->tz_offset_sec) > 0;
  LIT(o, ",\"language_code\":"); put_jstr(o, lang, v->lang_len);
  LIT(o, ",\"engagement\":"); put_int(o, engagement);
  LIT(o, ",\"view_count\":"); put_int(o, v->view_count);
  LIT(o, ",\"like_count\":"); put_int(o, v->like_count);
  LIT(o, ",\"share_count\":0,\"comment_count\":"); put_int(o, v->comment_count);
  LIT(o, ",\"crawl_label\":"); put_jstr(o, (const uint8_t*)cfg->crawl_label, cfg->crawl_label_len);
  LIT(o, ",\"list_ids\":null,\"channel_name\":"); put_jstr(o, chname, chname_n);
  LIT(o, ",\"search_terms\":null,\"search_term_ids\":null,\"project_ids\":null,\"exercise_ids\":null,"
         "\"label_data\":null,\"labels_metadata\":null,\"project_labeled_post_ids\":null,"
         "\"labeler_ids\":null,\"all_labels\":null,\"label_ids\":null,\"is_ad\":false,"
         "\"transcript_text\":\"\",\"image_text\":\"\",\"video_length\":");
  if (has_len) put_int(o, vlen); else LIT(o, "null");
  LIT(o, ",\"is_verified\":null,\"channel_data\":{\"channel_id\":"); put_jstr(o, chid, ch->id_len);
  if (ch->cached) { /* :784-805 */
    LIT(o, ",\"channel_name\":"); put_jstr(o, chtitle, ch->title_len);
    LIT(o, ",\"channel_description\":"); put_jstr(o, chdesc, ch->desc_len);
    LIT(o, ",\"channel_profile_image\":"); put_jstr(o, chthumb, ch->thumb_len);
    LIT(o, ",\"channel_engagement_data\":{\"follower_count\":"); put_int(o, ch->subscriber_count);
    LIT(o, ",\"following_count\":0,\"like_count\":0,\"post_count\":"); put_int(o, ch->video_count);
    LIT(o, ",\"views_count\":"); put_int(o, ch->view_count);
    LIT(o, ",\"comment_count\":0,\"share_count\":0},\"channel_url_external\":");
    put_jstr(o, churl.p, churl.len);
    LIT(o, ",\"channel_url\":"); put_jstr(o, churl.p, churl.len);
    LIT(o, ",\"country_code\":"); put_jstr(o, chcountry, ch->country_len);
    LIT(o, ",\"published_at\":"); ok &= put_time(o, ch->published_sec, ch->published_nsec, 0) > 0;
  } else { /* :806-829 */
    LIT(o, ",\"channel_name\":"); put_jstr(o, chid, ch->id_len);
    LIT(o, ",\"channel_description\":\"\",\"channel_profile_image\":\"\",\"channel_engagement_data\":{"
           "\"follower_count\":0,\"following_count\":0,\"like_count\":");
    put_int(o, v->like_count);
    LIT(o, ",\"post_count\":0,\"views_count\":"); put_int(o, v->view_count);
    LIT(o, ",\"comment_count\":"); put_int(o, v->comment_count);
    LIT(o, ",\"share_count\":0},\"channel_url_external\":"); put_jstr(o, churl.p, churl.len);
    LIT(o, ",\"channel_url\":"); put_jstr(o, churl.p, churl.len);
    LIT(o, ",\"country_code\":\"\",\"published_at\":");
    ok &= put_time(o, v->published_sec, v->published_nsec, 0) > 0;
  }
  LIT(o, "},\"platform_name\":\"youtube\",\"shared_id\":null,\"quoted_id\":null,\"replied_id\":null,"
         "\"ai_label\":null,\"root_post_id\":null,\"engagement_steps_count\":0,\"ocr_data\":");
  { /* :668-677; canonical key order default,medium,high,standard,maxres; nil slice -> null */
    int any = 0;
    for (int k = 0; k < 5; k++) {
      if (!thn[k]) continue;
      if (any) LIT(o, ","); else LIT(o, "[");
      any = 1;
      LIT(o, "{\"ocr_text\":\"YouTube thumbnail: ");
      buf_put(o, kThumbKey[k], strlen(kThumbKey[k]));
      LIT(o, " quality\",\"thumb_url\":");
      put_jstr(o, th[k], thn[k]);
      LIT(o, "}");
    }
    if (any) LIT(o, "]"); else LIT(o, "null");
  }
  LIT(o, ",\"performance_scores\":{\"likes\":"); put_int(o, v->like_count);
  LIT(o, ",\"shares\":null,\"comments\":"); put_int(o, v->comment_count);
  LIT(o, ",\"views\":");
  buf_reserve(o, 32);
  o->len += (size_t)orc_json_float_of_int64(v->view_count, o->p + o->len);
  LIT(o, "},\"has_embed_media\":true,\"description\":"); put_jstr(o, desc, v->desc_len);
  LIT(o, ",\"repost_channel_data\":null,\"post_type\":[\"video\"],\"inner_link\":{},\"post_title\":");
  put_jstr(o, title, v->title_len);
  LIT(o, ",\"media_data\":{\"document_name\":"); put_jstr(o, docname.p, docname.len);
  LIT(o, "},\"is_reply\":null,\"ad_fields\":null,\"likes_count\":"); put_int(o, v->like_count);
  LIT(o, ",\"shares_count\":0,\"comments_count\":"); put_int(o, v->comment_count);
  LIT(o, ",\"views_count\":"); put_int(o, v->view_count);
  LIT(o, ",\"searchable_text\":"); put_jstr(o, alltext.p, alltext.len);
  LIT(o, ",\"all_text\":"); put_jstr(o, alltext.p, alltext.len);
  LIT(o, ",\"contrast_agent_project_ids\":null,\"agent_ids\":null,\"segment_ids\":null,\"thumb_url\":");
  put_jstr(o, thumb, thumb_n);
  LIT(o, ",\"media_url\":"); put_jstr(o, vurl.p, vurl.len);
  LIT(o, ",\"comments\":null,\"reactions\":{\"like\":"); put_int(o, v->like_count);
  LIT(o, "},\"outlinks\":[");
  for (int k = 0; k < nurls; k++) {
    if (k) LIT(o, ",");
    put_jstr(o, urls[k].p, urls[k].n);
  }
  LIT(o, "],\"capture_time\":");
  ok &= put_time(o, cfg->capture_sec, cfg->capture_nsec, cfg->tz_offset_sec) > 0;
  LIT(o, ",\"handle\":"); put_jstr(o, chid, ch->id_len);
  LIT(o, "}\n");
  free(vurl.p); free(churl.p); free(alltext.p); free(docname.p);
  if (!ok) { o->len = line_start; return TGI_ST_NOLINE; }
  return TGI_ST_EMITTED;
}

/* ------------------------------------------------------------------------------------------- */
/* generic client.Message -> sparse Post (SURVEY a12)                                            */
/* TelegramCrawler.convertMessageToPost, crawler/telegram/telegram_crawler.go:179-262: the fields
 * it sets are listed at :183-246, the reactions map at :250-257 (only when non-empty); everything
 * else keeps Go's zero value, encoded per model/data.go:9-139 (nil slice / pointer / map -> null,
 * zero time -> "0001-01-01T00:00:00Z", nested structs with their zero fields).                  */
typedef struct {
  const uint8_t* p;
  uint64_t n;
  int64_t count;
} kv64_t;
static int kv64_cmp(const void* a, const void* b) {
  const kv64_t *x = a, *y = b;
  uint64_t m = x->n < y->n ? x->n : y->n;
  int c = memcmp(x->p, y->p, m);
  if (c) return c;
  return x->n < y->n ? -1 : (x->n > y->n ? 1 : 0);
}
static int gm_record(const orc_ctx* c, const tgi_gm_batch* b, uint64_t r, buf_t* o) {
  const tgi_config* cfg = &c->cfg;
  const tgi_gm_rec* rec = &b->recs[r];
  const uint8_t* id = b->strs + rec->str_off;
  const uint8_t* chan = id + rec->id_len;
  const uint8_t* text = chan + rec->channel_len;
  const uint8_t* sender = text + rec->text_len;
  size_t line_start = o->len;
  int ok = 1;
  LIT(o, "{\"post_link\":\"\",\"channel_id\":"); put_jstr(o, chan, rec->channel_len);          /* :184 */
  LIT(o, ",\"post_uid\":"); put_jstr(o, id, rec->id_len);                                        /* :185 */
  LIT(o, ",\"url\":\"\",\"published_at\":");
  ok &= put_time(o, rec->ts_sec, rec->ts_nsec, cfg->tz_offset_sec) > 0;                           /* :187 */
  LIT(o, ",\"created_at\":");
  ok &= put_time(o, cfg->created_at_sec, cfg->created_at_nsec, cfg->tz_offset_sec) > 0;           /* :188 time.Now() */
  LIT(o, ",\"language_code\":\"\",\"engagement\":0,\"view_count\":"); put_int(o, rec->views);      /* :191 */
  LIT(o, ",\"like_count\":0,\"share_count\":0,\"comment_count\":0,\"crawl_label\":\"\",\"list_ids\":null,"
         "\"channel_name\":");
  put_jstr(o, chan, rec->channel_len);                                                            /* :197 */
  LIT(o, ",\"search_terms\":null,\"search_term_ids\":null,\"project_ids\":null,\"exercise_ids\":null,"
         "\"label_data\":null,\"labels_metadata\":null,\"project_labeled_post_ids\":null,"
         "\"labeler_ids\":null,\"all_labels\":null,\"label_ids\":null,\"is_ad\":false,"
         "\"transcript_text\":\"\",\"image_text\":\"\",\"video_length\":null,\"is_verified\":null,"
         "\"channel_data\":{\"channel_id\":\"\",\"channel_name\":\"\",\"channel_description\":\"\","
         "\"channel_profile_image\":\"\",\"channel_engagement_data\":{\"follower_count\":0,"
         "\"following_count\":0,\"like_count\":0,\"post_count\":0,\"views_count\":0,\"comment_count\":0,"
         "\"share_count\":0},\"channel_url_external\":\"\",\"channel_url\":\"\",\"country_code\":\"\","
         "\"published_at\":\"0001-01-01T00:00:00Z\"},\"platform_name\":\"telegram\",\"shared_id\":null,"  /* :213 */
         "\"quoted_id\":null,\"replied_id\":null,\"ai_label\":null,\"root_post_id\":null,"
         "\"engagement_steps_count\":0,\"ocr_data\":null,\"performance_scores\":{\"likes\":null,"
         "\"shares\":null,\"comments\":null,\"views\":0},\"has_embed_media\":null,\"description\":");
  put_jstr(o, text, rec->text_len);                                                               /* :223 */
  LIT(o, ",\"repost_channel_data\":null,\"post_type\":null,\"inner_link\":{},\"post_title\":null,"
         "\"media_data\":{\"document_name\":\"\"},\"is_reply\":null,\"ad_fields\":null,\"likes_count\":0,"
         "\"shares_count\":0,\"comments_count\":0,\"views_count\":");
  put_int(o, rec->views);                                                                         /* :234 */
  LIT(o, ",\"searchable_text\":"); put_jstr(o, text, rec->text_len);                             /* :235 */
  LIT(o, ",\"all_text\":"); put_jstr(o, text, rec->text_len);                                    /* :236 */
  LIT(o, ",\"contrast_agent_project_ids\":null,\"agent_ids\":null,\"segment_ids\":null,\"thumb_url\":\"\","
         "\"media_url\":\"\",\"comments\":null,\"reactions\":");
  {
    uint32_t r0 = b->react_off ? b->react_off[r] : 0, r1 = b->react_off ? b->react_off[r + 1] : 0;
    if (r1 == r0) {                                                                               /* :250 */
      LIT(o, "null");
    } else {
      kv64_t* kv = (kv64_t*)malloc(sizeof(kv64_t) * (r1 - r0));
      uint32_t m = 0;
      for (uint32_t i = r0; i < r1; i++) {
        const tgi_gm_reaction* rc = &b->reacts[i];
        const uint8_t* p = b->aux + rc->key_off;
        uint32_t j = 0;
        for (; j < m; j++)
          if (kv[j].n == rc->key_len && memcmp(kv[j].p, p, rc->key_len) == 0) break;
        if (j == m) m++;
        kv[j].p = p;
        kv[j].n = rc->key_len;
        kv[j].count = rc->count;
      }
      qsort(kv, m, sizeof(kv64_t), kv64_cmp);
      LIT(o, "{");
      for (uint32_t j = 0; j < m; j++) {
        if (j) LIT(o, ",");
        put_jstr(o, kv[j].p, kv[j].n);
        LIT(o, ":");
        put_int(o, kv[j].count);
      }
      LIT(o, "}");
      free(kv);
    }
  }
  LIT(o, ",\"outlinks\":null,\"capture_time\":");
  ok &= put_time(o, cfg->capture_sec, cfg->capture_nsec, cfg->tz_offset_sec) > 0;                 /* :245 time.Now() */
  LIT(o, ",\"handle\":"); put_jstr(o, sender, rec->sender_len);                                  /* :246 */
  LIT(o, "}\n");
  if (!ok) { o->len = line_start; return TGI_ST_NOLINE; }
  return TGI_ST_EMITTED;
}

/* ------------------------------------------------------------------------------------------- */
/* batch drivers                                                                                 */

#define ORC_MAX_LINKS 4096

/* One batch = three phases on nthreads threads (the --concurrency analogue of the reference's worker
 * pool), separated by barriers; nthreads == 1 runs the same code sequentially:
 *   1. produce: every thread walks its contiguous record range (tg_record / yt_record / gm_record), appends the
 *      lines to its own buffer and buckets its frontier-eligible links by set shard;
 *   2. (thread 0) prefix sums over the threads' byte / link counts;
 *   3. place: every thread copies its lines and links to their final offsets (skipped for the lines with
 *      ORC_RUN_SLICES: the reference's workers append to per-channel files, there is no global concatenation on
 *      that path) and fills status / line_off / link_off of its range; then every thread inserts the links of the
 *      shards it owns, visiting the producing threads in order = global record order, so "first occurrence wins"
 *      and the NEW flags are the sequential ones.
 * No step is serial in the number of records.                                                                  */
struct batch_job {
  orc_ctx* c;
  orc_result* out;
  uint64_t n;
  uint32_t run_flags;
  pthread_barrier_t bar;
  int pin;
};

static void produce(work_t* w) {
  uint64_t m = w->r1 - w->r0;
  w->json.len = w->links.len = w->b_linelen.len = w->b_status.len = w->b_nlinks.len = w->b_tmp.len = 0;
  for (int i = 0; i < ORC_SHARDS; i++) w->bucket[i].len = 0;
  buf_reserve(&w->b_linelen, (m + 1) * 8); w->linelen = (uint64_t*)w->b_linelen.p;
  buf_reserve(&w->b_status, m + 1); w->status = w->b_status.p;
  buf_reserve(&w->b_nlinks, (m + 1) * 4); w->nlinks = (uint32_t*)w->b_nlinks.p;
  buf_reserve(&w->b_tmp, sizeof(tgi_link) * ORC_MAX_LINKS);
  const uint32_t rf = w->run_flags;
  for (uint64_t r = w->r0; r < w->r1; r++) {
    linkset_t ls = {(tgi_link*)w->b_tmp.p, 0, (int)(w->b_tmp.cap / sizeof(tgi_link)), 0, &w->b_tmp};
    buf_t* o = (rf & TGI_RUN_JSONL) ? &w->json : &w->scratch;
    w->scratch.len = 0;
    w->nlinks[r - w->r0] = 0;
    size_t before = o->len;
    int st = w->tg ? tg_record(w->c, w->tg, r, o, &ls, (rf & TGI_RUN_JSONL) != 0) : w->yt ? yt_record(w->c, w->yt, r, o, &ls) : gm_record(w->c, w->gm, r, o);
    w->status[r - w->r0] = (uint8_t)st;
    w->linelen[r - w->r0] = (rf & TGI_RUN_JSONL) ? o->len - before : 0;
    if (st == TGI_ST_EMITTED || st == TGI_ST_NOLINE) {
      const uint8_t* cname = NULL;
      uint32_t cname_n = 0;
      if (w->tg) {
        const tgi_tg_chan* ch = &w->tg->chans[w->tg->recs[r].chan_idx];
        cname = w->tg->chan_strs + ch->str_off + ch->title_len;
        cname_n = ch->name_len;
      }
      for (int k = 0; k < ls.n; k++) {
        tgi_link* l = &ls.v[k];
        l->filter_reason = (uint8_t)orc_filter_username(l->name, l->len);
        if (l->filter_reason == TGI_FU_VALID) l->flags |= TGI_LF_FILTER_OK;
        if (cname && l->len == cname_n && memcmp(l->name, cname, cname_n) == 0) l->flags |= TGI_LF_SELF;
        if (rf & TGI_RUN_FRONTIER) {
          if ((rf & TGI_RUN_SKIP_SELF) && (l->flags & TGI_LF_SELF)) continue;   /* runner.go:1231 */
          if ((rf & TGI_RUN_SKIP_INVALID) && is_invalid_channel(&w->c->xset[0], l->name, w->c->now_sec)) { /* runner.go:1247 */
            l->flags |= TGI_LF_INVALID;
            continue;
          }
          if ((rf & TGI_RUN_FILTER) && !(l->flags & TGI_LF_FILTER_OK)) continue; /* runner.go:1261 */
          const uint32_t idx = (uint32_t)(w->links.len / sizeof(tgi_link)) + (uint32_t)k;
          buf_put(&w->bucket[key_shard(key_hash(l->name))], &idx, 4);
        }
      }
      buf_put(&w->links, ls.v, sizeof(tgi_link) * (size_t)ls.n);
      w->nlinks[r - w->r0] = (uint32_t)ls.n;
    }
  }
}

static void place(work_t* w) {
  struct batch_job* j = w->job;
  orc_result* out = j->out;
  if (out->jsonl && w->json.len) memcpy(out->jsonl + w->json_base, w->json.p, w->json.len);
  if (w->links.len) memcpy(out->links + w->link_base, w->links.p, w->links.len);
  uint64_t a = w->json_base, bq = w->link_base;
  for (uint64_t r = w->r0; r < w->r1; r++) {
    out->status[r] = w->status[r - w->r0];
    out->line_off[r] = a;
    out->link_off[r] = (uint32_t)bq;
    a += w->linelen[r - w->r0];
    bq += w->nlinks[r - w->r0];
  }
}

static void insert_shards(work_t* w) {
  struct batch_job* j = w->job;
  orc_ctx* c = j->c;
  work_t* all = c->w;
  w->n_new = 0;
  for (int s = w->tid; s < ORC_SHARDS; s += w->nthreads) {
    fset_t* f = &c->fs[s];
    for (int t = 0; t < w->nthreads; t++) {
      const uint32_t* idx = (const uint32_t*)all[t].bucket[s].p;
      const uint64_t cnt = all[t].bucket[s].len / 4;
      tgi_link* links = j->out->links + all[t].link_base;
      for (uint64_t k = 0; k < cnt; k++) {
        tgi_link* l = &links[idx[k]];
        if (fset_insert_h(f, l->name, key_hash(l->name), c->seq + all[t].link_base + idx[k])) {
          l->flags |= TGI_LF_NEW;
          w->n_new++;
        }
      }
    }
  }
}

static void* worker(void* arg) {
  work_t* w = (work_t*)arg;
  struct batch_job* j = w->job;
  if (j->pin) { /* one thread per core, so that a thread's buffers stay on its NUMA node */
    cpu_set_t set;
    CPU_ZERO(&set);
    CPU_SET(w->tid, &set);
    pthread_setaffinity_np(pthread_self(), sizeof set, &set);
  }
  produce(w);
  if (w->nthreads > 1) pthread_barrier_wait(&j->bar);
  if (w->tid == 0) {
    orc_ctx* c = j->c;
    orc_result* out = j->out;
    uint64_t jl = 0, nl = 0;
    for (int t = 0; t < w->nthreads; t++) {
      c->w[t].json_base = jl;
      c->w[t].link_base = nl;
      jl += c->w[t].json.len;
      nl += c->w[t].links.len / sizeof(tgi_link);
    }
    const uint64_t n = j->n;
    c->r_status.len = c->r_jsonl.len = c->r_line_off.len = c->r_link_off.len = c->r_links.len = 0;
    buf_reserve(&c->r_status, n + 1); out->status = c->r_status.p;
    buf_reserve(&c->r_line_off, 8 * (n + 1)); out->line_off = (uint64_t*)c->r_line_off.p;
    buf_reserve(&c->r_link_off, 4 * (n + 1)); out->link_off = (uint32_t*)c->r_link_off.p;
    if (!(j->run_flags & ORC_RUN_SLICES)) { buf_reserve(&c->r_jsonl, jl + 1); out->jsonl = c->r_jsonl.p; }
    buf_reserve(&c->r_links, sizeof(tgi_link) * (nl + 1)); out->links = (tgi_link*)c->r_links.p;
    out->line_off[n] = jl;
    out->link_off[n] = (uint32_t)nl;
    out->jsonl_len = jl;
    out->n_links = nl;
  }
  if (w->nthreads > 1) pthread_barrier_wait(&j->bar);
  place(w);
  if (w->nthreads > 1) pthread_barrier_wait(&j->bar);
  if (j->run_flags & TGI_RUN_FRONTIER) insert_shards(w);
  return NULL;
}

static int run_batch(orc_ctx* c, const tgi_tg_batch* tg, const tgi_yt_batch* yt, const tgi_gm_batch* gm, uint32_t run_flags,
                     int nthreads, orc_result* out) {
  uint64_t n = tg ? tg->n : yt ? yt->n : gm->n;
  if (nthreads < 1) nthreads = 1;
  if ((uint64_t)nthreads > n) nthreads = n ? (int)n : 1;
  if (c->nw < nthreads) {
    c->w = (work_t*)realloc(c->w, sizeof(work_t) * (size_t)nthreads);
    memset(c->w + c->nw, 0, sizeof(work_t) * (size_t)(nthreads - c->nw));
    c->nw = nthreads;
  }
  work_t* w = c->w;
  memset(out, 0, sizeof *out);
  out->n = n;
  struct batch_job job;
  job.c = c; job.out = out; job.n = n; job.run_flags = run_flags;
  job.pin = (run_flags & ORC_RUN_PIN) != 0;
  if (nthreads > 1) pthread_barrier_init(&job.bar, NULL, (unsigned)nthreads);
  pthread_t* th = (pthread_t*)calloc((size_t)nthreads, sizeof(pthread_t));
  for (int t = 0; t < nthreads; t++) {
    w[t].c = c; w[t].tg = tg; w[t].yt = yt; w[t].gm = gm; w[t].run_flags = run_flags;
    w[t].tid = t; w[t].nthreads = nthreads; w[t].job = &job;
    w[t].r0 = n * (uint64_t)t / (uint64_t)nthreads;
    w[t].r1 = n * (uint64_t)(t + 1) / (uint64_t)nthreads;
    if (nthreads > 1) pthread_create(&th[t], NULL, worker, &w[t]);
    else worker(&w[t]);
  }
  if (nthreads > 1) {
    for (int t = 0; t < nthreads; t++) pthread_join(th[t], NULL);
    pthread_barrier_destroy(&job.bar);
  }
  if (run_flags & TGI_RUN_FRONTIER) {
    for (int t = 0; t < nthreads; t++) out->n_new += w[t].n_new;
    c->seq += out->n_links;
  }
  out->frontier_size = orc_frontier_size(c);
  free(th);
  return 0;
}

int orc_telegram_batch(orc_ctx* c, const tgi_tg_batch* in, uint32_t run_flags, int nthreads,
                       orc_result* out) {
  return run_batch(c, in, NULL, NULL, run_flags, nthreads, out);
}
int orc_youtube_batch(orc_ctx* c, const tgi_yt_batch* in, uint32_t run_flags, int nthreads,
                      orc_result* out) {
  for (uint64_t i = 0; i < in->n; i++)
    if (!nsec_ok(in->recs[i].published_nsec)) return TGI_E_ARG;
  for (uint32_t i = 0; i < in->n_chans; i++)
    if (!nsec_ok(in->chans[i].published_nsec)) return TGI_E_ARG;
  return run_batch(c, NULL, in, NULL, run_flags, nthreads, out);
}
/* crawl/runner.go:1580-1584,1667-1671 build map["%d_%d"]bool and :1171-1176 scans linearly; both are "is / where is
 * this (ChatID, MessageID) in that list".  Sequential restatement: sort the indices of a by (key, index), binary search. */
static const int64_t* g_join_keys;
static int join_cmp(const void* x, const void* y) {
  uint64_t i = *(const uint64_t*)x, j = *(const uint64_t*)y;
  const int64_t *p = g_join_keys + 2 * i, *q = g_join_keys + 2 * j;
  if (p[0] != q[0]) return p[0] < q[0] ? -1 : 1;
  if (p[1] != q[1]) return p[1] < q[1] ? -1 : 1;
  return i < j ? -1 : (i > j ? 1 : 0);
}
void orc_key_join(const int64_t* a, uint64_t na, const int64_t* b, uint64_t nb, int64_t* out) {
  uint64_t* idx = (uint64_t*)malloc(sizeof(uint64_t) * (na ? na : 1));
  for (uint64_t i = 0; i < na; i++) idx[i] = i;
  g_join_keys = a;
  qsort(idx, na, sizeof(uint64_t), join_cmp);
  for (uint64_t k = 0; k < nb; k++) {
    const int64_t c = b[2 * k], m = b[2 * k + 1];
    uint64_t lo = 0, hi = na;  /* first position whose key >= (c, m) */
    while (lo < hi) {
      uint64_t mid = (lo + hi) / 2;
      const int64_t* p = a + 2 * idx[mid];
      if (p[0] < c || (p[0] == c && p[1] < m)) lo = mid + 1; else hi = mid;
    }
    out[k] = (lo < na && a[2 * idx[lo]] == c && a[2 * idx[lo] + 1] == m) ? (int64_t)idx[lo] : -1;
  }
  free(idx);
}

int orc_generic_batch(orc_ctx* c, const tgi_gm_batch* in, uint32_t run_flags, int nthreads, orc_result* out) {
  for (uint64_t i = 0; i < in->n; i++)
    if (!nsec_ok(in->recs[i].ts_nsec)) return TGI_E_ARG;
  return run_batch(c, NULL, NULL, in, run_flags, nthreads, out);
}
void orc_result_free(orc_result* r) { /* arrays are context-owned; valid until the next batch call */
  memset(r, 0, sizeof *r);
}

/* ---- frontier -> validator hand-off (SURVEY 8f rank 3) ------------------------------------------------------------- */
int orc_set_add(orc_ctx* c, int which, const uint8_t* keys32, const int64_t* stamp_sec, uint64_t n) {
  if (which != TGI_SET_INVALID && which != TGI_SET_DISCOVERED) return -1;
  fset_t* f = &c->xset[which == TGI_SET_INVALID ? 0 : 1];
  for (uint64_t i = 0; i < n; i++)
    fset_insert_h(f, keys32 + 32 * i, key_hash(keys32 + 32 * i), (which == TGI_SET_INVALID && stamp_sec) ? (uint64_t)stamp_sec[i] : 0);
  return 0;
}
void orc_set_clear(orc_ctx* c, int which) {
  fset_t* f = &c->xset[which == TGI_SET_INVALID ? 0 : 1];
  f->n = 0;
  if (f->slots) memset(f->slots, 0, f->nslots * sizeof(uint64_t));
}
void orc_set_now(orc_ctx* c, int64_t now_sec) { c->now_sec = now_sec; }
/* The rows the reference would INSERT for the last batch (crawl/runner.go:1264-1306: one edge per outlink that survived
 * self / invalid / FilterUsername / seenInBatch, in message order), each with the verdict of the validator's two cache
 * look-ups (crawl/validator.go:205-226).  `r` = the result of that batch, `chan_idx_of` / stride as in the engine. */
uint64_t orc_pending_edges(orc_ctx* c, const orc_result* r, const void* chan_idx_of, uint32_t stride, int64_t now_sec,
                           tgi_edge* rows, uint64_t cap) {
  uint64_t m = 0;
  for (uint64_t rec = 0; rec < r->n; rec++) {
    for (uint32_t k = r->link_off[rec]; k < r->link_off[rec + 1]; k++) {
      const tgi_link* l = &r->links[k];
      if (!(l->flags & TGI_LF_NEW)) continue;
      if (m < cap) {
        tgi_edge* e = &rows[m];
        memset(e, 0, sizeof *e);
        memcpy(e->destination, l->name, 32);
        e->record = rec;
        e->chan_idx = chan_idx_of ? *(const uint32_t*)((const uint8_t*)chan_idx_of + (size_t)rec * stride) : 0;
        e->dest_len = l->len;
        e->source_type = l->src;
        e->status = is_invalid_channel(&c->xset[0], l->name, now_sec) ? TGI_EDGE_INVALID_CACHED
                    : fset_find(&c->xset[1], l->name) >= 0 ? TGI_EDGE_DUPLICATE : TGI_EDGE_PENDING;
      }
      m++;
    }
  }
  return m;
}
