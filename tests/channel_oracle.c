/*
 * channel_oracle.c — CPU restatement of the random-walk StoreChannelData line (tgi_channel_batch).  TEST
 * INFRASTRUCTURE ONLY: tests/channel_oracle.py compiles it into a temporary directory and links it against the CPU
 * oracle (oracle/libtgoracle.so), whose orc_json_string is the encoding/json string rule every oracle line uses.
 *
 * RunForChannel builds a model.ChannelData for the page (crawl/runner.go:587-607) and, in random-walk mode, passes it to
 * sm.StoreChannelData(p.URL, channelData) (:620-626); DaprStateManager.StoreChannelData marshals it and appends '\n'
 * (state/daprstate.go:3089-3094).  Fields in declaration order (model/data.go:89-111, EngagementData :102-111); the
 * unset ones keep their zero values, PublishedAt the zero time.Time.  json.Marshal cannot fail on this struct.
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "tgingest.h"
#include "tgoracle.h"

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
  if (n) memcpy(b->p + b->len, s, n);
  b->len += n;
}
#define LIT(b, s) buf_put((b), (s), sizeof(s) - 1)
static void put_jstr(buf_t* b, const uint8_t* s, uint64_t n) { /* a Go string through encoding/json, quotes included */
  buf_reserve(b, n * 6 + 2);
  b->len += orc_json_string(s, n, b->p + b->len);
}
static void put_int(buf_t* b, int64_t v) { /* strconv.FormatInt(v, 10), and an int field's JSON */
  char t[24];
  int k = snprintf(t, sizeof t, "%lld", (long long)v);
  buf_put(b, t, (size_t)k);
}

/* the result arrays of the last call (an orc_result points into them) */
typedef struct {
  buf_t status, jsonl, line_off, link_off, url, scratch;
} chorc_ctx;

chorc_ctx* chorc_create(void) { return (chorc_ctx*)calloc(1, sizeof(chorc_ctx)); }
void chorc_destroy(chorc_ctx* c) {
  if (!c) return;
  free(c->status.p); free(c->jsonl.p); free(c->line_off.p); free(c->link_off.p); free(c->url.p); free(c->scratch.p);
  free(c);
}

#define CH_STR_MAX ((1u << 24) - 1) /* the library's limit per string (tgi_channel_batch) */
static int ch_rec_ok(const tgi_ch_rec* r, uint64_t strs_len) {
  if (r->title_len > CH_STR_MAX || r->image_len > CH_STR_MAX || r->url_len > CH_STR_MAX) return 0;
  const uint64_t end = r->str_off + (uint64_t)r->title_len + r->image_len + r->url_len;
  return end <= strs_len && end >= r->str_off;
}

static void ch_record(chorc_ctx* c, const tgi_ch_batch* b, uint64_t i, buf_t* o) {
  const tgi_ch_rec* r = &b->recs[i];
  const uint8_t* title = b->strs + r->str_off;
  const uint8_t* image = title + r->title_len;
  const uint8_t* url = image + r->image_len;
  LIT(o, "{\"channel_id\":\"");
  put_int(o, r->chat_id);                                              /* runner.go:593 strconv.FormatInt(chat.Id, 10) */
  LIT(o, "\",\"channel_name\":"); put_jstr(o, title, r->title_len);    /* :594 chat.Title */
  LIT(o, ",\"channel_description\":\"\",\"channel_profile_image\":");
  put_jstr(o, image, r->image_len);                                    /* :596, :588-591 chat.Photo.Extra or "" */
  LIT(o, ",\"channel_engagement_data\":{\"follower_count\":");
  put_int(o, r->member_count);                                         /* :598 int(memberCount) */
  LIT(o, ",\"following_count\":0,\"like_count\":0,\"post_count\":");
  put_int(o, r->message_count);                                        /* :601 int(messageCount) */
  LIT(o, ",\"views_count\":");
  put_int(o, r->total_views);                                          /* :602 int(totalViews) */
  LIT(o, ",\"comment_count\":0,\"share_count\":0},\"channel_url_external\":");
  c->url.len = 0;                                                      /* :606-607 fmt.Sprintf("https://t.me/%s", p.URL) */
  LIT(&c->url, "https://t.me/");
  buf_put(&c->url, url, r->url_len);
  put_jstr(o, c->url.p, c->url.len);
  LIT(o, ",\"channel_url\":");
  put_jstr(o, c->url.p, c->url.len);
  LIT(o, ",\"country_code\":\"\",\"published_at\":\"0001-01-01T00:00:00Z\"}\n");
}

/* the line of every record; TGI_E_ARG, nothing run, for run flags other than TGI_RUN_JSONL / TGI_RUN_JSONL_DEVICE and for
 * a record whose strings leave strs or reach 16 MiB, as tgi_channel_batch refuses them */
int chorc_channel_batch(chorc_ctx* c, const tgi_ch_batch* in, uint32_t run_flags, orc_result* out) {
  if (run_flags & ~(uint32_t)(TGI_RUN_JSONL | TGI_RUN_JSONL_DEVICE)) return TGI_E_ARG;
  if (in->n && !in->recs) return TGI_E_ARG;
  if (in->strs_len && !in->strs) return TGI_E_ARG;
  for (uint64_t i = 0; i < in->n; i++)
    if (!ch_rec_ok(&in->recs[i], in->strs_len)) return TGI_E_ARG;
  const uint64_t n = in->n;
  c->status.len = c->jsonl.len = c->line_off.len = c->link_off.len = 0;
  buf_reserve(&c->status, n + 1);
  buf_reserve(&c->line_off, (n + 1) * 8);
  buf_reserve(&c->link_off, (n + 1) * 4);
  buf_reserve(&c->jsonl, 1);
  uint64_t* line_off = (uint64_t*)c->line_off.p;
  buf_t* o = (run_flags & TGI_RUN_JSONL) ? &c->jsonl : &c->scratch;
  line_off[0] = 0;
  for (uint64_t i = 0; i < n; i++) {
    c->scratch.len = 0;
    ch_record(c, in, i, o);
    c->status.p[i] = TGI_ST_EMITTED;
    line_off[i + 1] = c->jsonl.len;
  }
  memset(c->link_off.p, 0, (n + 1) * 4);
  memset(out, 0, sizeof *out);
  out->n = n;
  out->status = c->status.p;
  out->jsonl = c->jsonl.p;
  out->jsonl_len = c->jsonl.len;
  out->line_off = line_off;
  out->link_off = (uint32_t*)c->link_off.p;
  return TGI_OK;
}
