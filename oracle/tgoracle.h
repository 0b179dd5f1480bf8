/*
 * tgoracle.h — CPU restatement of the reference hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this library.  It is never linked into libtgingest and the product has no CPU fallback.
 *
 * Parity pinning (SURVEY.md §8c):
 *   - link extraction, UTF-16 offsets, reserved paths, FilterUsername: PINNED by the reference's
 *     own known-answer tests (telegramhelper/channel_links_test.go, username_filter_test.go,
 *     crawl/runner_tandem_test.go), transcribed in tests/golden/reference_vectors.json.
 *   - JSON bytes (encoding/json, time formatting, ParseMessage / convertVideoToPost field map):
 *     PARITY UNPINNED — the reference holds no test or fixture for them (its ParseMessage tests
 *     are t.Skip'ped, crawl/message_processing_test.go:22,254) and Go is not installed here, so the
 *     restatement follows the Go 1.25 standard-library rules from source reading only.
 *
 * Works on the packed batch structs of include/tgingest.h so the oracle and the CUDA engine are fed
 * bit-identical inputs.
 */
#ifndef TGORACLE_H
#define TGORACLE_H

#include "../include/tgingest.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct orc_ctx orc_ctx; /* holds config + the frontier set */

typedef struct orc_result { /* arrays are owned by the orc_ctx, valid until its next batch call */
  uint64_t n;
  uint8_t* status;
  uint8_t* jsonl;
  uint64_t jsonl_len;
  uint64_t* line_off;
  uint32_t* link_off;
  tgi_link* links;
  uint64_t n_links;
  uint64_t n_new;
  uint64_t frontier_size;
} orc_result;

/* TGI_E_ARG (and *out = NULL) for a configuration tgi_create refuses: a clock nsec outside [0, 1e9), |tz_offset_sec| >=
 * 86400.  TGI_E_ARG from orc_set_clock (the previous clock stays) and from the batch calls (nothing is run) for an nsec
 * outside [0, 1e9), as the library's tgi_set_clock and batch uploads.                                                  */
int orc_create(const tgi_config* cfg, orc_ctx** out);
void orc_destroy(orc_ctx* c);
int orc_set_clock(orc_ctx* c, int64_t created_at_sec, int32_t created_at_nsec, int64_t capture_sec,
                  int32_t capture_nsec);

/* oracle-only run flags (beside TGI_RUN_*): how the timed CPU arm is run */
#define ORC_RUN_SLICES 0x10000u /* leave the lines in the worker threads' own buffers (result.jsonl == NULL, jsonl_len and
                                   line_off are still the global ones): the reference's workers append to per-channel files,
                                   nothing on that path concatenates the output of different workers                      */
#define ORC_RUN_PIN 0x20000u    /* pin worker t to core t (NUMA-local buffers)                                          */

/* nthreads <= 1: sequential like the reference loop (crawl/runner.go:1161). nthreads > 1: records
 * are split into contiguous ranges (the --concurrency analogue); output is identical.            */
int orc_telegram_batch(orc_ctx* c, const tgi_tg_batch* in, uint32_t run_flags, int nthreads,
                       orc_result* out);
/* SURVEY 8f rank 2: first index in a of every key of b, -1 if absent (keys = {chat_id, message_id}) */
void orc_key_join(const int64_t* a_keys, uint64_t na, const int64_t* b_keys, uint64_t nb, int64_t* b_index);
int orc_generic_batch(orc_ctx* c, const tgi_gm_batch* in, uint32_t run_flags, int nthreads, orc_result* out);
int orc_youtube_batch(orc_ctx* c, const tgi_yt_batch* in, uint32_t run_flags, int nthreads,
                      orc_result* out);
void orc_result_free(orc_result* r);

int orc_frontier_insert(orc_ctx* c, const uint8_t* keys32, uint64_t n, uint8_t* is_new);
uint64_t orc_frontier_size(orc_ctx* c);
uint64_t orc_frontier_export(orc_ctx* c, uint8_t* keys32, uint64_t cap);
void orc_frontier_clear(orc_ctx* c);

/* SURVEY 8f rank 3: resident exclusion sets + the pending_edges rows of the last batch (see tgi_pending_edges) */
int orc_set_add(orc_ctx* c, int which, const uint8_t* keys32, const int64_t* stamp_sec, uint64_t n);
void orc_set_clear(orc_ctx* c, int which);
void orc_set_now(orc_ctx* c, int64_t now_sec);
uint64_t orc_pending_edges(orc_ctx* c, const orc_result* r, const void* chan_idx_of, uint32_t stride, int64_t now_sec,
                           tgi_edge* rows, uint64_t cap);

/* unit-level entry points (each cites the reference function it restates in tgoracle.c) */
void orc_utf16_offset_to_bytes(const uint8_t* s, int64_t n, int32_t off16, int32_t len16,
                               int64_t* start, int64_t* end);
/* first match of channelLinkRegex; returns 1 and [name_start,name_end) or 0 */
int orc_channel_link_first(const uint8_t* s, int64_t n, int64_t from, int64_t* name_start,
                           int64_t* name_end);
int orc_username_first(const uint8_t* s, int64_t n, int64_t* name_start, int64_t* name_end);
int orc_is_reserved_path(const uint8_t* lower_name, int len);
int orc_filter_username(const uint8_t* name, int64_t len);
/* appends the Go-encoding/json string form of s (with the quotes) to dst; returns bytes written;
 * dst == NULL only counts */
uint64_t orc_json_string(const uint8_t* s, uint64_t n, uint8_t* dst);
/* RFC3339Nano as time.Time.MarshalJSON (with quotes). returns length, 0 if year out of [0,9999] */
int orc_json_time(int64_t sec, int32_t nsec, int32_t tz_offset_sec, uint8_t* dst);
/* parseISO8601Duration: returns 1 + *seconds on match, 0 otherwise */
int orc_parse_iso8601_duration(const uint8_t* s, int64_t n, int64_t* seconds);
/* strconv.FormatFloat(float64(v), 'f', -1, 64) as encoding/json prints PerformanceScores.Views */
int orc_json_float_of_int64(int64_t v, uint8_t* dst);
/* extract links of one record into out[cap]; returns count, or -1 if Go would panic */
int orc_extract_links(const tgi_tg_batch* b, uint64_t rec, tgi_link* out, int cap);

#ifdef __cplusplus
}
#endif
#endif
