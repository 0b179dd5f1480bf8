/*
 * tgingest.h — C ABI of libtgingest, the H100-native (sm_90a) message-ingest engine.
 *
 * This is the drop-in boundary for ONE hot path of researchaccelerator-hub/distributed-crawler:
 * parse -> link-extract -> filter/dedup -> JSONL-serialize.  Every entry point below names the
 * reference interface (file:line, relative to the reference tree) it replaces.  The reference is
 * Go; a Go maintainer binds these through cgo (see INTEGRATION.md for the stub).  All types are
 * plain C: fixed-width integers, flat buffers, no pointers inside array elements, so the cgo
 * pointer-passing rules hold (the batch descriptor itself is built in C memory by the shim).
 *
 * The same packed-batch structs are consumed by the CPU oracle (oracle/tgoracle.c), which is test
 * infrastructure only and is never linked into libtgingest.
 *
 * Conventions
 *   - every function returns 0 on success, <0 (TGI_E_*) on a batch-level error; the message is
 *     available from tgi_last_error().  Per-record outcomes are in tgi_result.status[] and mirror
 *     crawl/runner.go:1199-1214 (fetched / failed) and tdutils.go:419-421 (date-skipped).
 *   - inputs are caller-owned and only read during the call; outputs live in library-owned pinned
 *     host memory and stay valid until tgi_result_release() / the next call on the same slot.
 *   - device memory never crosses this ABI except through the explicitly named *_dev entry points
 *     used by the multi-GPU frontier merge.
 */
#ifndef TGINGEST_H
#define TGINGEST_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TGI_ABI_VERSION 2

/* ---- error codes ---------------------------------------------------------------------------- */
#define TGI_OK 0
#define TGI_E_ARG (-1)      /* bad argument / malformed batch                                     */
#define TGI_E_CUDA (-2)     /* CUDA runtime error (message in tgi_last_error)                     */
#define TGI_E_NOMEM (-3)    /* host or device allocation failed                                   */
#define TGI_E_CAPACITY (-4) /* a capacity from tgi_config (or the tgi_set_growth limit) exceeded  */
#define TGI_E_NODEVICE (-5) /* no CUDA device: there is NO CPU fallback in the product            */
#define TGI_E_STATE (-6)    /* call sequence error (slot busy, result not released, ...)          */

/* ---- per-record status (tgi_result.status) -------------------------------------------------- */
#define TGI_ST_EMITTED 0 /* one JSONL line written; message marked "fetched"                      */
#define TGI_ST_SKIPPED 1 /* published before MinPostDate: no line, still "fetched" (tdutils.go:419) */
#define TGI_ST_FAILED 2  /* Go would have panicked+recovered: no line, marked "failed"            */
#define TGI_ST_NOLINE 3  /* json.Marshal error (time year outside [0,9999]): StorePost error is
                            logged and swallowed (tdutils.go:724-729): no line, still "fetched"   */

/* ---- Telegram content types (go-tdlib v0.7.4 client.MessageContent variants) ----------------
 * Order of the enum is ABI.  The type string emitted in "post_type" is MessageContentType()
 * (tdutils.go:606-609).  TGI_CT_OTHER carries its type string in the record's `alt` slot.       */
enum {
  TGI_CT_NONE = 0,             /* message.Content == nil  -> post_type ["unknown"]                */
  TGI_CT_TEXT = 1,             /* messageText            description=text, links from text        */
  TGI_CT_VIDEO = 2,            /* messageVideo           description=caption, media_url=alt/media */
  TGI_CT_PHOTO = 3,            /* messagePhoto           description=caption                       */
  TGI_CT_ANIMATION = 4,        /* messageAnimation       description=caption                       */
  TGI_CT_ANIMATED_EMOJI = 5,   /* messageAnimatedEmoji   description=alt (emoji), no links         */
  TGI_CT_POLL = 6,             /* messagePoll            description=alt (question), no links      */
  TGI_CT_GIVEAWAY = 7,         /* messageGiveaway        description=alt (prize type), no links    */
  TGI_CT_PAID_MEDIA = 8,       /* messagePaidMedia       description=alt (caption), no links       */
  TGI_CT_STICKER = 9,          /* messageSticker         description=""                            */
  TGI_CT_GIVEAWAY_WINNERS = 10,
  TGI_CT_GIVEAWAY_COMPLETED = 11,
  TGI_CT_VIDEO_NOTE = 12,      /* messageVideoNote       media_url=media                           */
  TGI_CT_DOCUMENT = 13,        /* messageDocument        description=alt (file name), links from caption */
  TGI_CT_AUDIO = 14,           /* messageAudio           description="", links from caption        */
  TGI_CT_VOICE_NOTE = 15,      /* messageVoiceNote       description="", links from caption        */
  TGI_CT_OTHER = 16,           /* any other variant: post_type [alt], description=""              */
  TGI_CT__COUNT = 17
};

/* tgi_tg_rec.flags */
#define TGI_RF_HAS_TEXT 0x01     /* the FormattedText (Text / Caption) pointer is non-nil         */
#define TGI_RF_COMMENTS_NIL 0x02 /* comments slice is nil (JSON null) rather than empty ([])      */
#define TGI_RF_PANIC 0x04        /* walking this message nil-derefs in the reference (e.g. a video
                                    with a thumbnail but no caption, tdutils.go:186-194): the panic
                                    is recovered (:395-405) and the message is marked "failed"     */

/* entity types that matter (tdutils.go:909-939); everything else is TGI_ENT_OTHER */
enum { TGI_ENT_OTHER = 0, TGI_ENT_TEXT_URL = 1, TGI_ENT_MENTION = 2, TGI_ENT_URL = 3 };

/* link source types (tdutils.go:93-97); the numeric order is first-wins irrelevant, pure labels  */
enum { TGI_SRC_MENTION = 0, TGI_SRC_TEXT_URL = 1, TGI_SRC_URL = 2, TGI_SRC_PLAINTEXT = 3 };

/* FilterUsername reasons (username_filter.go:26-68), evaluation order preserved */
enum {
  TGI_FU_VALID = 0,
  TGI_FU_TOO_SHORT = 1,
  TGI_FU_TOO_LONG = 2,
  TGI_FU_INVALID_START_CHAR = 3,
  TGI_FU_ENDS_WITH_UNDERSCORE = 4,
  TGI_FU_INVALID_CHAR = 5,
  TGI_FU_LOOKS_LIKE_PATH = 6,
  TGI_FU_BOT_SUFFIX = 7
};

/* ---- packed Telegram batch (SURVEY Appendix B) ----------------------------------------------
 * One record = one already-fetched client.Message with the RPC results pre-resolved
 * (share count: telegramutils.go:250, poster handle: :748, comments: :311).                     */
typedef struct tgi_tg_rec { /* 64 bytes, 16-byte aligned */
  int64_t id;              /* message.Id (TDLib internal id; public id = id / 1048576)            */
  int64_t chat_id;         /* message.ChatId                                                      */
  int64_t media_album_id;  /* != 0 -> "?single" suffix (tdutils.go:1023)                          */
  uint64_t str_off;        /* offset in `strs` of this record's strings: text|alt|media|handle    */
  int32_t date;            /* message.Date (unix seconds)                                         */
  int32_t view_count;      /* InteractionInfo.ViewCount, 0 when InteractionInfo == nil            */
  int32_t share_count;     /* pre-resolved ForwardCount (GetMessageShareCount)                    */
  uint32_t chan_idx;       /* row of the channel table                                            */
  uint32_t text_len;       /* bytes of FormattedText.Text (the link carrier)                      */
  uint32_t alt_len;        /* bytes of the alternate string (see content type table)              */
  uint16_t media_len;      /* bytes of the remote file id that becomes media_url                  */
  uint16_t handle_len;     /* bytes of the pre-resolved poster (GetPoster)                        */
  uint8_t content_type;    /* TGI_CT_*                                                            */
  uint8_t flags;           /* TGI_RF_*                                                            */
  uint16_t reserved;
} tgi_tg_rec;

typedef struct tgi_entity { /* 16 bytes: one client.TextEntity */
  int32_t offset;   /* UTF-16 code units                                                          */
  int32_t length;   /* UTF-16 code units                                                          */
  uint32_t url_off; /* TGI_ENT_TEXT_URL: offset of Url in `aux`                                   */
  uint16_t url_len;
  uint8_t type;     /* TGI_ENT_*                                                                  */
  uint8_t reserved;
} tgi_entity;

typedef struct tgi_reaction { /* 12 bytes: ReactionTypeEmoji + TotalCount (tdutils.go:591-603) */
  uint32_t emoji_off; /* offset in `aux`                                                          */
  uint16_t emoji_len;
  uint16_t reserved;
  int32_t count;
} tgi_reaction;

typedef struct tgi_comment { /* 32 bytes: one model.Comment (telegramutils.go:589-635) */
  uint32_t text_off; /* offset in `aux`                                                           */
  uint32_t text_len;
  uint32_t handle_off;
  uint16_t handle_len;
  uint8_t flags; /* bit0: Reactions map non-nil                                                   */
  uint8_t reserved;
  int32_t view_count;
  int32_t reply_count;
  uint32_t react_start; /* range in `reacts`                                                      */
  uint32_t react_count;
} tgi_comment;

typedef struct tgi_tg_chan { /* 40 bytes: per-channel constants of ParseMessage */
  uint32_t str_off;   /* offset in chan_strs: title|name|username                                 */
  uint16_t title_len; /* chat.Title                                                               */
  uint16_t name_len;  /* channelName argument (= page URL)                                        */
  uint16_t user_len;  /* supergroup.Usernames.ActiveUsernames[0], 0 = none -> link ""             */
  uint16_t reserved;
  uint32_t reserved2;
  int64_t member_count; /* supergroupInfo.MemberCount (0 if nil)                                  */
  int64_t post_count;   /* postcount argument                                                     */
  int64_t view_count;   /* viewcount argument                                                     */
} tgi_tg_chan;

typedef struct tgi_tg_batch {
  uint64_t n;                 /* records                                                          */
  const tgi_tg_rec* recs;     /* [n]                                                              */
  const uint8_t* strs;        /* per-record strings                                               */
  uint64_t strs_len;
  const uint32_t* ent_off;    /* [n+1] ranges into ents                                           */
  const tgi_entity* ents;
  const uint32_t* react_off;  /* [n+1] ranges into reacts (message reactions)                     */
  const tgi_reaction* reacts; /* message reactions first, then comment reactions                  */
  uint64_t n_reacts;
  const uint32_t* comment_off; /* [n+1] ranges into comments                                      */
  const tgi_comment* comments;
  uint64_t n_comments;
  const uint8_t* aux;         /* entity URLs, emoji, comment strings                              */
  uint64_t aux_len;
  uint32_t n_chans;
  uint32_t reserved;
  const tgi_tg_chan* chans;   /* [n_chans]                                                        */
  const uint8_t* chan_strs;
  uint64_t chan_strs_len;
} tgi_tg_batch;

/* ---- packed YouTube batch (model/youtube/types.go:10-36) ------------------------------------ */
#define TGI_YT_THUMB_ABSENT 0xFFFFu
typedef struct tgi_yt_rec { /* 80 bytes, 16-byte aligned */
  uint64_t str_off;     /* in `strs`: id|title|description|duration|language|thumb[0..4]          */
  int64_t published_sec; /* video.PublishedAt as unix seconds (zone given by tz of the value: UTC) */
  int64_t view_count;
  int64_t like_count;
  int64_t comment_count;
  uint32_t desc_len;
  uint32_t chan_idx;     /* row of the channel table = GetChannelInfo(video.ChannelID)            */
  uint16_t id_len;
  uint16_t title_len;
  uint16_t duration_len;
  uint16_t lang_len;
  uint16_t thumb_len[5]; /* default, medium, high, standard, maxres; TGI_YT_THUMB_ABSENT = no key */
  uint16_t reserved;
  int32_t published_nsec;
  uint64_t reserved2;
} tgi_yt_rec;

typedef struct tgi_yt_chan { /* 64 bytes; cached == 0 -> fallback branch youtube_crawler.go:808 */
  uint32_t str_off;     /* in chan_strs: id|title|description|thumb_default|country               */
  uint16_t id_len;
  uint16_t title_len;
  uint32_t desc_len;
  uint16_t thumb_len;
  uint16_t country_len;
  int64_t subscriber_count;
  int64_t view_count;
  int64_t video_count;
  int64_t published_sec;
  int32_t published_nsec;
  uint8_t cached;
  uint8_t reserved[11];
} tgi_yt_chan;

typedef struct tgi_yt_batch {
  uint64_t n;
  const tgi_yt_rec* recs;
  const uint8_t* strs;
  uint64_t strs_len;
  uint32_t n_chans;
  uint32_t reserved;
  const tgi_yt_chan* chans;
  const uint8_t* chan_strs;
  uint64_t chan_strs_len;
} tgi_yt_batch;

/* ---- generic client.Message (SURVEY §8 a12) -------------------------------------------------------
 * The secondary Telegram path: client.Message (client/interfaces.go:56-100) as
 * TelegramClient.getMessagesWithClient fills it (client/clients.go:296-339), converted by
 * TelegramCrawler.convertMessageToPost (crawler/telegram/telegram_crawler.go:179-262) into a SPARSE
 * model.Post: channel_id / channel_name = GetChannelID(), post_uid = GetID(), published_at =
 * GetTimestamp(), created_at = capture_time = time.Now(), view_count = views_count = GetViews(),
 * platform_name "telegram", description = searchable_text = all_text = GetText(), handle =
 * GetSenderName(), reactions = the map if it is non-empty else nil; every other key keeps its zero
 * value.  No link extraction on this path.                                                          */
typedef struct tgi_gm_reaction { /* 16 bytes: one entry of map[string]int64 */
  uint32_t key_off; /* offset in `aux`                                                               */
  uint16_t key_len;
  uint16_t reserved;
  int64_t count;
} tgi_gm_reaction;

typedef struct tgi_gm_rec { /* 48 bytes */
  uint64_t str_off;   /* in `strs`: id | channel_id | text | sender_name                            */
  int64_t ts_sec;     /* GetTimestamp(): time.Unix(sec, nsec) shown in the context's zone           */
  int64_t views;      /* GetViews()                                                                  */
  int32_t ts_nsec;
  uint32_t text_len;
  uint16_t id_len;
  uint16_t channel_len;
  uint16_t sender_len;
  uint16_t reserved;
  uint32_t reserved2;
  uint32_t reserved3;
} tgi_gm_rec;

typedef struct tgi_gm_batch {
  uint64_t n;
  const tgi_gm_rec* recs;
  const uint8_t* strs;
  uint64_t strs_len;
  const uint32_t* react_off; /* [n+1] ranges into reacts; entries of one record = its map, later
                                duplicates of a key overwrite earlier ones                          */
  const tgi_gm_reaction* reacts;
  uint64_t n_reacts;
  const uint8_t* aux;        /* reaction keys                                                      */
  uint64_t aux_len;
} tgi_gm_batch;

/* ---- configuration -------------------------------------------------------------------------- */
#define TGI_CFG_HAS_MIN_POST_DATE 0x01 /* !cfg.MinPostDate.IsZero()                               */
#define TGI_CFG_SKIP_MEDIA 0x02        /* cfg.SkipMediaDownload; REQUIRED (media download is RPC) */

typedef struct tgi_config {
  uint32_t abi_version;    /* TGI_ABI_VERSION                                                     */
  int32_t device;          /* CUDA ordinal                                                        */
  uint32_t flags;          /* TGI_CFG_*                                                           */
  int32_t tz_offset_sec;   /* fixed offset of the process-local zone (time.Unix -> Local)         */
  int64_t min_post_date;   /* unix seconds                                                        */
  int64_t created_at_sec;  /* injected time.Now(): Telegram uses .UTC().Truncate(time.Second)
                              (tdutils.go:611); YouTube keeps zone + nanoseconds (youtube_crawler.go:704) */
  int64_t capture_sec;     /* injected time.Now() (tdutils.go:715, youtube_crawler.go:769)        */
  int32_t capture_nsec;
  int32_t created_at_nsec;
  uint32_t crawl_label_len;
  uint32_t reserved;
  const char* crawl_label; /* Post.CrawlLabel as the sink would see it (daprstate.go:1113-1115)   */
  uint64_t frontier_capacity; /* max distinct names in the frontier set (0 = default 1<<22); with
                                 tgi_set_growth the initial size of the resident sets           */
  uint64_t max_records;    /* per-call record capacity (0 = default 1<<20)                        */
  uint64_t max_in_bytes;   /* per-call input byte capacity, all arrays (0 = grow on demand)       */
  uint64_t max_out_bytes;  /* per-call JSONL capacity (0 = grow on demand)                        */
} tgi_config;

/* ---- run options ---------------------------------------------------------------------------- */
#define TGI_RUN_JSONL 0x01      /* size -> scan -> emit; jsonl/line_off filled                    */
#define TGI_RUN_LINKS 0x02      /* return per-record outlinks (links/link_off)                    */
#define TGI_RUN_FRONTIER 0x04   /* insert outlinks into the global frontier set; link.flags NEW   */
#define TGI_RUN_FILTER 0x08     /* tandem mode: FilterUsername gate before the set (runner.go:1261) */
#define TGI_RUN_SKIP_SELF 0x10  /* drop o == owner.URL (runner.go:1231)                           */
#define TGI_RUN_NO_D2H 0x20     /* bench only: leave results on the device (kernel-only timing)   */
#define TGI_RUN_SKIP_INVALID 0x40 /* tandem mode: drop outlinks found in the resident invalid-channel set before they
                                   reach the dedup set (crawl/runner.go:1247 sm.IsInvalidChannel); link.flags INVALID */
#define TGI_RUN_JSONL_DEVICE 0x80 /* with TGI_RUN_JSONL: lines are emitted but stay on the device; tgi_result.jsonl is
                                     NULL, jsonl_len and line_off are filled (for tgi_dapr_payloads / tgi_result_read_jsonl) */

#define TGI_LF_FILTER_OK 0x01 /* FilterUsername(name).Valid                                       */
#define TGI_LF_NEW 0x02       /* first occurrence in the global frontier set                      */
#define TGI_LF_SELF 0x04      /* equals the record's channel name                                 */
#define TGI_LF_INVALID 0x08   /* found in the resident invalid-channel set (TGI_RUN_SKIP_INVALID)  */

typedef struct tgi_link { /* 36 bytes */
  uint8_t name[32]; /* lower-cased, zero padded                                                   */
  uint8_t len;
  uint8_t src;   /* TGI_SRC_*                                                                     */
  uint8_t flags; /* TGI_LF_*                                                                      */
  uint8_t filter_reason; /* TGI_FU_*                                                              */
} tgi_link;

typedef struct tgi_result {
  uint64_t n;
  const uint8_t* status;    /* [n] TGI_ST_*                                                       */
  const uint8_t* jsonl;     /* concatenated lines, each ends with '\n'                            */
  uint64_t jsonl_len;
  const uint64_t* line_off; /* [n+1]; skipped/failed records have empty ranges                    */
  const uint32_t* link_off; /* [n+1]                                                              */
  const tgi_link* links;    /* per-record outlinks in first-insertion order                       */
  uint64_t n_links;
  uint64_t n_new;           /* names this call added to the frontier                              */
  uint64_t frontier_size;   /* distinct names after this call                                     */
  float kernel_ms;          /* device time of the kernels of this call (CUDA events)              */
  uint32_t gpu_launches;    /* kernels launched by this call                                      */
  float parse_ms;           /* device time of the parse pass (link extraction + size kernels)     */
  float emit_ms;            /* device time of the JSONL emit pass (three kernels)                 */
  int32_t slot;             /* staging slot that owns the buffers: pass to tgi_result_release     */
  float emit_main_ms;       /* device time of the main emit kernel (tg_emit_tile_kernel / yt_emit_lane_kernel) */
  uint64_t var_bytes;       /* JSONL bytes of the variable pieces (strings, comments, maps, outlinks) */
  uint64_t main_bytes_out;  /* JSONL bytes written by the main emit kernel                         */
  uint64_t main_bytes_in;   /* bytes it read from HBM-resident sources to produce them (strings, channel blob) */
  float frontier_ms;        /* device time of the frontier (dedup set) kernels of this call       */
  uint32_t reserved;
} tgi_result;

typedef struct tgi_stats {
  uint64_t records, bytes_in, bytes_out, links, frontier_size, launches;
  double kernel_ms_total;
} tgi_stats;

typedef struct tgi_ctx tgi_ctx;

/* lifecycle.  Replaces nothing in the reference; owned by the Go shim's init (see INTEGRATION.md). */
int tgi_create(const tgi_config* cfg, tgi_ctx** out);
void tgi_destroy(tgi_ctx* ctx);
const char* tgi_last_error(tgi_ctx* ctx); /* ctx may be NULL: last create error                   */
void tgi_get_stats(tgi_ctx* ctx, tgi_stats* out);
/* injected clock can change per channel batch (tdutils.go:611,715 call time.Now per message).    */
/* must not be called while a job is in flight on any slot (returns TGI_E_STATE)                  */
int tgi_set_clock(tgi_ctx* ctx, int64_t created_at_sec, int32_t created_at_nsec, int64_t capture_sec,
                  int32_t capture_nsec);

/* The local zone with its transitions — time.Local of a natively built crawler is the host's zone (e.g.
 * America/New_York, with DST), which tz_offset_sec can only model as one fixed offset.  The table is n entries;
 * start_sec is strictly increasing, and instant t is shown at offset_sec[i] of the last entry with start_sec[i] <= t
 * (entry 0 before start_sec[0]).  While a table is set it replaces tz_offset_sec everywhere time.Local is used:
 * Telegram published_at (time.Unix(message.Date, 0), tdutils.go:417) and generic published_at (GetTimestamp()) per
 * record; YouTube and generic created_at and every capture_time, rendered at tgi_create / tgi_set_clock /
 * tgi_set_zone.  Telegram created_at stays UTC (tdutils.go:611) and YouTube published_at keeps the zone of the API
 * value (UTC).
 *   Format   Go's appendFormatRFC3339 / appendStrictRFC3339: the local fields come from t + offset, seconds of the offset
 *            included; 'Z' only when the offset is exactly 0; otherwise minutes = offset / 60 truncated toward zero and
 *            the sign is that of the minutes (-30 s is "+00:00", -75 s is "-00:01", +00:19:32 is "+00:19").  A local year
 *            outside [0, 9999] is TGI_ST_NOLINE, with the offset in effect at that record.  Zones whose offset is 0 for
 *            part of the year (Europe/London) change the line length with it: line_off and the sinks follow.
 *   Clearing n == 0 removes the table: tz_offset_sec applies again, byte for byte as without a table.
 *   Errors   TGI_E_STATE while a job is in flight on any slot (as tgi_set_clock).  TGI_E_ARG: a NULL array with n > 0,
 *            starts that are not strictly increasing, |offset| >= 86400, or n > TGI_ZONE_MAX.  A rejected call leaves
 *            the previous table in effect.
 *   Go shim  LocalZoneTable() (INTEGRATION.md) walks time.Local with Time.ZoneBounds() from time.Unix(math.MinInt32, 0)
 *            (Telegram's Date is an int32) to a horizon, one entry per zone period, and calls tgi_set_zone once after
 *            tgi_create.  Beyond the horizon the last entry applies, so int64 generic timestamps past it are exact only
 *            up to the horizon.  Every tzdata zone has a few hundred transitions over that range.                  */
#define TGI_ZONE_MAX 4096
int tgi_set_zone(tgi_ctx* ctx, const int64_t* start_sec, const int32_t* offset_sec, uint32_t n);

/* Telegram: replaces the loop body crawl/runner.go:1161-1244 -> processMessage (:1720) ->
 * telegramhelper.ParseMessage (tdutils.go:380-732) -> extractChannelLinksFromMessage (:989) ->
 * json.Marshal+'\n' (state/storageproviders.go:276-282, state/daprstate.go:1118-1120) for a whole
 * slice of messages in one call.  `slot` selects one of TGI_SLOTS independent staging slots so
 * calls from different goroutines / pipelined calls overlap (H2D, kernels and D2H on the slot's
 * stream).  Inputs must stay valid until the matching wait returns.  tgi_telegram_batch = claim a
 * free slot + submit + wait; its result is released with tgi_result_release(ctx, out->slot).
 *
 * Batch size.  A batch of at most 8192 records and 4 MB — the reference calls ParseMessage with one
 * page of 100 messages (crawl/runner.go:1110) — runs as ONE cooperative kernel launch with one copy
 * in and one copy out (tgi_result.gpu_launches == 1; 0.14 ms per 100 messages on an H100); bigger
 * batches take the multi-kernel pipeline (~27 launches; through host buffers PCIe-bound, 20.5 M
 * messages/s on an H100).  The bytes
 * are the same either way.  tgi_youtube_batch: the same split (a Data-API page is 50 videos).
 *
 * Order.  Batches with TGI_RUN_FRONTIER enter the dedup set in the order in which they were
 * SUBMITTED (tgi_*_submit / the blocking calls), whichever slot or thread carries them: TGI_LF_NEW,
 * n_new and the export order are those of one thread processing the batches one after the other.
 *
 * Diagnostics (environment, read per call or at first use; none changes results): TGI_NO_PAGE=1 the
 * multi-kernel pipeline for every size; TGI_PAGE_TRACE=1 phase clock of the page kernels on
 * stderr; TGI_TRACE_SLOTS=1 host-side timeline of the slots' synchronisation points;
 * TGI_GRID_MULT / TGI_LANE_MULT grid sizes in CTAs per SM (defaults 128 / 24); TGI_SIZE_TEXT_WARP=1
 * the multi-kernel pipeline's parse leaves the message texts unmeasured and the size pass measures
 * every one of them (the path before the parse measured them).                                    */
#define TGI_SLOTS 3
int tgi_telegram_submit(tgi_ctx* ctx, int slot, const tgi_tg_batch* in, uint32_t run_flags);
int tgi_telegram_wait(tgi_ctx* ctx, int slot, tgi_result* out);
int tgi_telegram_batch(tgi_ctx* ctx, const tgi_tg_batch* in, uint32_t run_flags, tgi_result* out);

/* YouTube: replaces the worker body crawler/youtube/youtube_crawler.go:380-418 ->
 * convertVideoToPost (:530-836) + json.Marshal+'\n'; links = extractChannelIDsFromText
 * (client/youtube_client.go:1856-1878) for the snowball frontier (:1706-1721).  A link row holds the
 * first 32 bytes of an id (tgi_link.name): real channel ids are 24 characters and handles at most 30,
 * so only malformed ids are cut; the JSONL line itself is never shortened.                       */
int tgi_youtube_submit(tgi_ctx* ctx, int slot, const tgi_yt_batch* in, uint32_t run_flags);
int tgi_youtube_wait(tgi_ctx* ctx, int slot, tgi_result* out);
int tgi_youtube_batch(tgi_ctx* ctx, const tgi_yt_batch* in, uint32_t run_flags, tgi_result* out);

/* SURVEY §8f rank 1 — the chunk combiner's batching rule (chunk/main.go:292-345, processBatches) applied to the lines
 * of one result, instead of one temp file per post (state/daprstate.go:1117-1138) + fsnotify + io.Copy concat
 * (chunk/main.go:378-421): consecutive lines are grouped into the blobs that become combined_<ns>.jsonl.
 *   - a line longer than hard_cap is dropped (:316-322);
 *   - a group is closed BEFORE a line that would push it over hard_cap (:324-327);
 *   - a group is closed AFTER the line that makes it reach trigger (:334-337);
 *   - what is left forms the last group (:339-343).
 * Records without a line (line length 0) are not files and are ignored.  Group g = lines [groups[2g], groups[2g+1])
 * minus the dropped / empty ones; groups are disjoint and increasing.  dropped (optional, n bytes) is set to 1 for
 * dropped lines.  Pure host arithmetic over line_off (as returned in tgi_result); returns TGI_E_CAPACITY if more than
 * max_groups groups are needed.                                                                        */
int tgi_plan_chunks(const uint64_t* line_off, uint64_t n, uint64_t trigger, uint64_t hard_cap, uint64_t* groups,
                    uint64_t max_groups, uint64_t* n_groups, uint8_t* dropped);
/* The same rule as a stream: the lines of one result continue a group that already holds open_bytes_in bytes of earlier
 * results (0: none), and the group left open at the end is NOT closed: its bytes go to *open_bytes_out.  groups gets
 * the groups this call closes; the first one has begin 0 when it is the group carried in (it may then hold no line of
 * this result: the carried group closes before line `end` that would push it over hard_cap).  The open group's lines
 * of this result are the kept ones behind the last closed group.  Chaining the calls over the results of a stream, then
 * closing what is left, gives the groups of tgi_plan_chunks over the whole stream; tgi_plan_chunks is the case
 * open_bytes_in = 0 plus that last close.  TGI_E_ARG: open_bytes_in above hard_cap, or above 0 and not below
 * trigger (no group rests there).  Each boundary is a binary search over line_off; only the scan for dropped lines is linear. */
int tgi_plan_chunks_carry(const uint64_t* line_off, uint64_t n, uint64_t trigger, uint64_t hard_cap, uint64_t open_bytes_in,
                          uint64_t* groups, uint64_t max_groups, uint64_t* n_groups, uint8_t* dropped,
                          uint64_t* open_bytes_out);

/* Combine mode on the device — with --combine-files (dapr/standalone.go:256-264) DaprStateManager.StorePost writes one
 * temp file per post into a watch directory (state/daprstate.go:1117-1138); Chunker.processBatches (chunk/main.go:
 * 292-345) groups those files, combineFiles concatenates each group into combined_<unixnano>.jsonl (:386-421) and
 * UploadCombinedFile (daprstate.go:3734-3777) sends ONE InvokeBinding per file, with Data = its base64 and the path
 * <prefix>combined-posts/combined_<ns>.jsonl.  The combiner is context state that takes the lines of each result in
 * call order and returns, for every blob a call closes, that Data and that path.  The lines never leave the device.
 *   Rule     processBatches over the stream of every line passed so far.  Records without a line (length 0: skipped,
 *            failed, TGI_ST_NOLINE) are not files and are ignored.  A line longer than hard_cap is dropped and its
 *            record index reported in `dropped` (:316-322).  A group closes BEFORE a line that would push it over
 *            hard_cap (:324-327) and AFTER the line that makes it reach trigger (:334-337).  tgi_combine_flush closes the
 *            open group if it holds a line (:339-343, Chunker shutdown).  Any trigger / hard_cap is accepted, trigger >
 *            hard_cap included.
 *   Data     base64.StdEncoding of the blob's concatenated lines: '=' padding, no line breaks, 4*ceil(raw_bytes/3)
 *            bytes, data[data_off, data_off + data_len).
 *   Path     path_prefix verbatim, then "combined-posts/combined_<ns>.jsonl" (generateCrawlExecutableStoragePath,
 *            daprstate.go:2689-2698, :3743-3746): path[path_off, path_off + path_len).  <ns> = max(unix_nano, previous
 *            <ns> + 1) for every blob, so names are unique and increase when one call closes several blobs.
 *   Inputs   tgi_combine_add takes the slot's last result (Telegram or YouTube, bulk or page) like tgi_dapr_payloads,
 *            also after TGI_RUN_JSONL_DEVICE and TGI_RUN_NO_D2H.  TGI_E_STATE: no combiner is open, the slot holds no
 *            result, the result ran without TGI_RUN_JSONL, or it is a tgi_generic_batch one (SavePost has no Dapr
 *            implementation).  The open group never points into the slot: once tgi_combine_add returns, the slot may
 *            be released and reused.
 *   Open     tgi_combine_open allocates the open blob's encoded buffer (4*ceil(hard_cap/3) bytes on the device).  On an
 *            open combiner it reconfigures it, and returns TGI_E_STATE while the open group holds lines.  prefix is
 *            copied.  tgi_destroy frees everything.
 *   Order    Calls are serialised by a combiner lock and apply in call order, whatever their slots.  A call whose lines
 *            all fit in the open group (open_bytes + jsonl_len below trigger and at most hard_cap) and whose line
 *            offsets are on the host (not TGI_RUN_NO_D2H) only enqueues on the slot's stream and records an event that
 *            the next call waits on: it does not synchronise, and reports kernel_ms = 0.  Other calls synchronise once
 *            to plan, and once when their blobs are in host memory.
 * Outputs live in library-owned pinned memory and stay valid until the next combine call.                             */
typedef struct tgi_combined_blob {
  uint64_t data_off, data_len;  /* base64 of the blob in tgi_combined_t.data                                */
  uint64_t path_off, path_len;  /* its blob path in tgi_combined_t.path                                     */
  uint64_t n_lines, raw_bytes;  /* posts in it and their bytes (Chunker.postsUploaded / totalUploadSize)    */
  int64_t unix_nano;            /* the <ns> of combined_<ns>.jsonl                                          */
} tgi_combined_blob;
typedef struct tgi_combined_t {
  uint64_t n_blobs;  const tgi_combined_blob* blobs;  /* blobs CLOSED by this call, in order                  */
  const uint8_t* data;  const uint8_t* path;          /* library-owned pinned memory                          */
  uint64_t n_dropped;  const uint64_t* dropped;       /* record indices of this result's lines > hard_cap     */
  uint64_t open_lines, open_bytes;                    /* the group still open after the call                  */
  float kernel_ms;                                    /* device time of this call's launches (0: not waited)  */
  uint32_t gpu_launches;
} tgi_combined_t;
int tgi_combine_open(tgi_ctx* ctx, uint64_t trigger, uint64_t hard_cap, const char* path_prefix, uint32_t prefix_len);
int tgi_combine_add(tgi_ctx* ctx, int slot, int64_t unix_nano, tgi_combined_t* out);  /* the slot's last result        */
int tgi_combine_flush(tgi_ctx* ctx, int64_t unix_nano, tgi_combined_t* out);           /* Chunker shutdown: :339-343     */

/* SURVEY 8f rank 1, local sink — LocalStateManager.StorePost opens, appends to and closes <crawl>/<channel>/posts/posts.jsonl
 * once per POST (state/storageproviders.go:39-53,275-298).  The lines of consecutive records of one channel are contiguous
 * in the result blob, so a run of them is ONE append of jsonl[byte_begin, byte_end): same file contents, one open / write
 * / close per run instead of per post.  chan_idx / chan_stride: the channel row of every record (e.g. &recs[0].chan_idx,
 * sizeof(tgi_tg_rec)); records without a line neither start nor break a run.  Pure host arithmetic.                   */
typedef struct tgi_append_run {
  uint32_t chan_idx;   /* channel row: the caller maps it to the channelID argument of StorePost                         */
  uint32_t n_lines;    /* posts in this run                                                                             */
  uint64_t first, end; /* records [first, end)                                                                          */
  uint64_t byte_begin, byte_end; /* their lines in tgi_result.jsonl                                                     */
} tgi_append_run;
int tgi_plan_channel_appends(const uint64_t* line_off, const void* chan_idx, uint32_t chan_stride, uint64_t n,
                             tgi_append_run* runs, uint64_t max_runs, uint64_t* n_runs);

/* Local sink on the device — the same posts.jsonl files as one LocalStateManager.StorePost per post, written with ONE
 * append per channel file per result, also when the result's lines stay on the device and when one channel's lines are
 * interleaved with other channels' (a YouTube batch, several channels' pages in one bulk call).  tgi_channel_appends
 * groups the lines of the slot's last result by channel on the device and returns every group's bytes, contiguous.
 *   Input    the slot's last Telegram or YouTube result, bulk or page, like tgi_dapr_payloads: also after
 *            TGI_RUN_JSONL_DEVICE (this call is then the only time the lines cross PCIe) and TGI_RUN_NO_D2H.
 *   Lines    only records with status TGI_ST_EMITTED and a non-empty line take part.  Skipped, failed and
 *            TGI_ST_NOLINE records never reach StorePost: they neither start nor break a group.
 *   Channel  channelID as tgi_dapr_payloads reads it: Telegram = the channel row's name (tdutils.go:725), YouTube = the
 *            channel row's id (youtube_crawler.go:396).  Rows whose channelID bytes are equal are ONE channel (one file,
 *            so one group); chan_idx is the lowest such row.  IDs that differ as bytes but that filepath.Clean maps to
 *            one path (e.g. "a" and "a/") are distinct groups: real usernames are [A-Za-z0-9_] and channel ids
 *            [A-Za-z0-9_-], so this cannot happen with real data.
 *   Order    inside a group, lines in record order: what the per-post appends leave in the file.  Groups are ordered by
 *            their first line.  order[] lists the record index of every grouped line, group after group.
 *   Errors   TGI_E_STATE: the slot holds no result (see tgi_result_read_jsonl), the result ran without TGI_RUN_JSONL,
 *            or it is a tgi_generic_batch one (its posts go to SavePost).  TGI_E_ARG: bad slot or NULL out.
 *            TGI_E_NOMEM: allocation failed (the batch result stays valid).  TGI_E_CAPACITY: 2^32 - 16 records or more.
 * The call synchronises once.  Outputs live in library-owned pinned memory and stay valid until the release or the
 * next call on that slot.  The batch's tgi_result is not changed.                                                     */
typedef struct tgi_channel_group {
  uint32_t chan_idx;      /* first channel row (lowest index) carrying this channelID                              */
  uint32_t reserved;
  uint64_t n_lines;       /* posts of this channel in the result                                                   */
  uint64_t first_record;  /* record index of its first line                                                        */
  uint64_t byte_off, byte_len; /* its lines, in record order, in tgi_channel_appends_t.data                        */
} tgi_channel_group;
typedef struct tgi_channel_appends_t {
  uint64_t n_groups;  const tgi_channel_group* groups; /* ordered by first_record                                  */
  const uint8_t* data; uint64_t data_len;              /* all emitted lines, grouped (pinned)                     */
  const uint64_t* order;                               /* [n_lines total] record index of each grouped line        */
  float kernel_ms;      /* device time of this call's kernels and scans (not the read-back)                        */
  uint32_t gpu_launches;
} tgi_channel_appends_t;
int tgi_channel_appends(tgi_ctx* ctx, int slot, tgi_channel_appends_t* out);

/* Dapr sink — DaprStateManager.StorePost outside combine mode (state/daprstate.go:1141-1181) sends, per post, ONE
 * InvokeBinding with Operation "create", Data = base64.StdEncoding.EncodeToString(json.Marshal(post) + "\n") (:1159)
 * and Metadata {<file naming key>: <blob path>, "operation": "append"} (:1150-1153, path format :2689-2698).
 * tgi_dapr_payloads computes both byte strings on the device for every record of the slot's last Telegram or YouTube
 * result, from the lines that are still resident (run the batch with TGI_RUN_JSONL_DEVICE to leave them there).
 *   path_prefix  StorageRoot + "/" + CrawlID + "/" + CrawlExecutionID + "/", taken verbatim (prefix_len bytes).
 *   data         record i's line, '\n' included, in Go's StdEncoding: A-Z a-z 0-9 + /, '=' padding, no line breaks,
 *                4*ceil(len/3) bytes; data[data_off[i], data_off[i+1]).
 *   path         prefix | channelID | "/posts/" | PostUID | ".jsonl", raw bytes (not JSON-escaped);
 *                path[path_off[i], path_off[i+1]).  Telegram: channelID = the channel row's name (the channelName
 *                argument, tdutils.go:725), PostUID = FormatInt(id / 1048576) + "-" + channelName (tdutils.go:416,636,
 *                1008; truncating division).  YouTube: channelID = the channel row's id (video.ChannelID,
 *                youtube_crawler.go:396), PostUID = the record's id (video.ID, :701).
 * Only records with status TGI_ST_EMITTED get a payload; the others get empty ranges: a date-skipped message never
 * reaches StorePost (tdutils.go:419-421), a failed one panicked before it, and a TGI_ST_NOLINE one failed json.Marshal
 * before any binding call (daprstate.go:1141-1144).
 * Call between tgi_*_wait / tgi_*_batch and tgi_result_release (like tgi_pending_edges); works after TGI_RUN_NO_D2H and
 * TGI_RUN_JSONL_DEVICE.  Outputs live in library-owned pinned memory and stay valid until the release or the next call
 * on that slot.  TGI_E_STATE: the slot holds no result (see tgi_result_read_jsonl), the last result is a
 * tgi_generic_batch one (its posts go to SavePost, crawler/common/runner.go:55, which has no Dapr implementation) or
 * ran without TGI_RUN_JSONL; TGI_E_ARG: bad slot or NULL prefix / out; TGI_E_NOMEM: allocation failed (the batch
 * result stays valid).                                                                                                */
typedef struct tgi_dapr_payloads_t {
  uint64_t n;
  const uint8_t* data;  uint64_t data_len;  const uint64_t* data_off;  /* [n+1] base64 of record i's line          */
  const uint8_t* path;  uint64_t path_len;  const uint64_t* path_off;  /* [n+1] blob path of record i               */
  float kernel_ms;      /* device time of this call's kernels (sizes + scans, writer; not the read-back between) */
  uint32_t gpu_launches;
} tgi_dapr_payloads_t;
int tgi_dapr_payloads(tgi_ctx* ctx, int slot, const char* path_prefix, uint32_t prefix_len, tgi_dapr_payloads_t* out);

/* SURVEY §8f rank 2 — the message-status join.  The reference looks messages up by (ChatID, MessageID) with
 * string-keyed maps or linear scans: resampleMarker (crawl/runner.go:1572-1635), addNewMessages (:1650-1697), the
 * per-message search for the fetched *client.Message (:1171-1176), BaseStateManager.UpdateMessage's scan
 * (state/base.go:191-210).  All of them are one primitive: for every key of list B, the index of the FIRST element of
 * list A with the same key, or -1.  Keys are pairs of int64 {chat_id, message_id}; a and b are host arrays of
 * 2*na / 2*nb int64; b_index gets nb entries.  Exact (an open-addressed hash table over A on the device).        */
int tgi_key_join(tgi_ctx* ctx, const int64_t* a_keys, uint64_t na, const int64_t* b_keys, uint64_t nb, int64_t* b_index);

/* Generic client.Message -> sparse Post line: replaces the loop body
 * crawler/telegram/telegram_crawler.go:148-156 (convertMessageToPost :179-262) + json.Marshal+'\n'.
 * Blocking; picks a free slot.  status[] is TGI_ST_EMITTED or TGI_ST_NOLINE; no links.             */
int tgi_generic_batch(tgi_ctx* ctx, const tgi_gm_batch* in, uint32_t run_flags, tgi_result* out);

void tgi_result_release(tgi_ctx* ctx, int slot);

/* Device-resident variant used for kernel-only measurement and by pipelines that already hold the
 * packed batch in HBM: upload once, run many times.  Same kernels as tgi_telegram_batch.
 * A slot's resident batch is the batch of its last successful upload (tgi_*_upload, tgi_*_submit or tgi_*_batch of
 * Telegram or YouTube); tgi_telegram_run_resident / tgi_youtube_run_resident return TGI_E_STATE unless it is of their
 * kind.  The upload call returns once the copy has landed.                                                           */
int tgi_telegram_upload(tgi_ctx* ctx, int slot, const tgi_tg_batch* in);
int tgi_telegram_run_resident(tgi_ctx* ctx, int slot, uint32_t run_flags, tgi_result* out);
int tgi_youtube_upload(tgi_ctx* ctx, int slot, const tgi_yt_batch* in);
int tgi_youtube_run_resident(tgi_ctx* ctx, int slot, uint32_t run_flags, tgi_result* out);
/* The readers (tgi_result_read_jsonl, tgi_result_read_rows, tgi_pending_edges, tgi_dapr_payloads) read a slot's last
 * result, which lives from a successful job until the next job is claimed on the slot: after tgi_result_release too,
 * but not after a failed or upload-only job.  A reader that finds no result, or a job in flight on the slot, returns
 * TGI_E_STATE.
 * tgi_result_read_jsonl: copy [off, off+len) of the slot's device JSONL to dst (host); for spot checks of huge runs */
int tgi_result_read_jsonl(tgi_ctx* ctx, int slot, uint64_t off, uint64_t len, uint8_t* dst);
/* copy rows [first, first+count) of the slot's last per-record status (uint8), link offsets (uint32, n+1) or link rows
 * (tgi_link) to dst (host): what a TGI_RUN_NO_D2H run left on the device; TGI_E_ARG for rows the result does not have */
enum { TGI_ROWS_STATUS = 0, TGI_ROWS_LINK_OFF = 1, TGI_ROWS_LINKS = 2 };
int tgi_result_read_rows(tgi_ctx* ctx, int slot, int which, uint64_t first, uint64_t count, void* dst);

/* Frontier set: replaces seenInBatch (crawl/runner.go:1267-1272), newLayerUniqueURLs
 * (dapr/standalone.go:650-658), urlCache (state/daprstate.go:646-658), existingURLs
 * (state/base.go:255-281), DiscoveredChannels (state/datamodels.go:136-146) and YouTube
 * processedChannels (client/youtube_client.go:1709-1714): exact string-set membership, first
 * occurrence wins, insertion order preserved.  Keys are 32-byte zero-padded names.               */
int tgi_frontier_insert(tgi_ctx* ctx, const uint8_t* keys32, uint64_t n, uint8_t* is_new);
int tgi_frontier_size(tgi_ctx* ctx, uint64_t* n);
int tgi_frontier_export(tgi_ctx* ctx, uint8_t* keys32, uint64_t cap, uint64_t* n);
int tgi_frontier_clear(tgi_ctx* ctx);
/* device-pointer forms for the multi-GPU set merge (NCCL exchange is done by the caller, who owns
 * the communicator; see distributed_crawler_b200/frontier_merge.py)                             */
int tgi_frontier_export_dev(tgi_ctx* ctx, void* d_keys32, uint64_t cap, uint64_t first, uint64_t* n);
int tgi_frontier_insert_dev(tgi_ctx* ctx, const void* d_keys32, uint64_t n, void* d_is_new);
int tgi_frontier_sync(tgi_ctx* ctx);

/* Library-owned pinned host memory for the packed input arrays (SURVEY 8b "Ownership").  The packer (the Go shim's
 * Batch, host/tgingest.hpp, pack.py) builds its arrays directly in blocks obtained here, so the host -> device copies
 * of tgi_*_submit run at link speed from page-locked memory; with pageable (Go heap / malloc) buffers the copy engine
 * reaches about half of that.  Blocks are 4096-byte aligned, recycled through a per-context pool, and stay valid
 * until tgi_release_staging / tgi_destroy.  Replaces nothing in the reference (its messages live on the Go heap).   */
int tgi_acquire_staging(tgi_ctx* ctx, uint64_t bytes, void** out);
int tgi_release_staging(tgi_ctx* ctx, void* block);

/* Multi-GPU dedup-set merge (SURVEY 8e option A).  One process per GPU; the record path shards on record index with
 * no collective, only the set is global: it replaces the shared urlCache / seenInBatch state that the reference's
 * workers reach through the Dapr state store (state/daprstate.go:646-658, crawl/runner.go:1267-1272).
 *   tgi_comm_unique_id   rank 0 creates the 128-byte NCCL id; the host distributes it to the other ranks by its own
 *                        means (the Go shim: a Dapr pub/sub message or a file; the Python mirror: torch.distributed).
 *   tgi_comm_init        every rank: create the communicator (ncclCommInitRank) on the context's device.
 *   tgi_frontier_merge   collective.  Keys added to the local set since the last merge are bucketed on the device by
 *                        owner = hash(key) % nranks, exchanged with grouped ncclSend / ncclRecv (counts first, one
 *                        ncclAllGather), and inserted by the owner into its partition of the global set; a key keeps
 *                        the sequence number (merge round, source rank, position in the source's set) of its first
 *                        occurrence, so the union of the partitions ordered by that number is exactly the set a
 *                        single process would have built over the ranks' shards in rank order.  *global_size = number
 *                        of distinct keys over all ranks; *owned (optional) = keys in this rank's partition.
 *   tgi_frontier_global_export   collective.  All partitions, ordered as above, on every rank (hand-off / tests).
 * libnccl.so.2 is loaded with dlopen at tgi_comm_init (a process that already carries NCCL, e.g. through PyTorch,
 * shares that copy); single-GPU users never need it.                                                                */
#define TGI_COMM_ID_BYTES 128
int tgi_comm_unique_id(uint8_t id[TGI_COMM_ID_BYTES]);
int tgi_comm_init(tgi_ctx* ctx, const uint8_t id[TGI_COMM_ID_BYTES], int rank, int nranks);
int tgi_comm_destroy(tgi_ctx* ctx);
int tgi_frontier_merge(tgi_ctx* ctx, uint64_t* global_size, uint64_t* owned);
int tgi_frontier_global_export(tgi_ctx* ctx, uint8_t* keys32, uint64_t cap, uint64_t* n);
typedef struct tgi_merge_stats {
  uint64_t merges, keys_sent, keys_received, keys_owned, bytes_sent;
  double bucket_ms, exchange_ms, insert_ms; /* device time between the phases' events, summed over the merges: includes
                                               waiting for the slowest rank and, in the first merge, NCCL's connection set-up */
  double last_bucket_ms, last_exchange_ms, last_insert_ms; /* the same for the most recent merge only */
} tgi_merge_stats;
int tgi_merge_get_stats(tgi_ctx* ctx, tgi_merge_stats* out);

/* SURVEY 8f rank 3 — frontier -> validator hand-off.  The reference walks the outlinks of every message, asks
 * sm.IsInvalidChannel (state/daprstate.go:3556-3564: an in-memory cache with a 30-day TTL), FilterUsername, seenInBatch,
 * and writes ONE pending_edges row per surviving edge with its own INSERT (crawl/runner.go:1247-1306,
 * state/daprstate.go:3914-3931, sql/validator-schema.sql:54-76); the validator then asks IsInvalidChannel and
 * IsChannelDiscovered per edge before any HTTP request (crawl/validator.go:205-226).  Here the two exclusion sets are
 * resident on the GPU next to the dedup set, the batch call drops invalid channels on the way into the dedup set
 * (TGI_RUN_SKIP_INVALID), and tgi_pending_edges returns every new edge of the slot's last batch as ONE packed row buffer,
 * already classified the way the validator's two look-ups would classify it.
 *   tgi_set_add       add keys (32-byte zero-padded names) to a resident set; stamp_sec[i] = when the channel was marked
 *                     invalid (unix seconds; NULL = now is irrelevant: never expires); re-adding a key keeps the first stamp
 *   tgi_pending_edges rows in (record, first-insertion) order = the order the reference inserts them; status:
 *                     TGI_EDGE_PENDING (needs the HTTP check), TGI_EDGE_DUPLICATE (already discovered: validator.go:214-226),
 *                     TGI_EDGE_INVALID_CACHED (validator.go:205-212; only if the batch ran without TGI_RUN_SKIP_INVALID or
 *                     the channel was marked invalid in between).  Call between tgi_*_wait / tgi_*_batch and
 *                     tgi_result_release.  0 rows for an empty batch; TGI_E_STATE for a slot that holds no result
 *                     (see tgi_result_read_jsonl) or a non-empty one that ran without TGI_RUN_FRONTIER.  The per-batch
 *                     constants of a row (batch_id, crawl_id, sequence_id, discovery_time) stay with the caller;
 *                     source_channel = the name of channel row `chan_idx`.                                             */
#define TGI_SET_INVALID 1     /* invalid_channels (state/daprstate.go:3489-3564)                  */
#define TGI_SET_DISCOVERED 2  /* discovered_channels (state/base.go:522-528)                      */
#define TGI_INVALID_TTL_SEC (30 * 24 * 3600)
#define TGI_EDGE_PENDING 0
#define TGI_EDGE_DUPLICATE 1
#define TGI_EDGE_INVALID_CACHED 2
typedef struct tgi_edge { /* 48 bytes */
  uint8_t destination[32]; /* destination_channel, lower-cased, zero padded                       */
  uint64_t record;         /* source record of the batch                                          */
  uint32_t chan_idx;       /* its channel row: source_channel                                     */
  uint8_t dest_len;
  uint8_t source_type;     /* TGI_SRC_*: 'mention' | 'text_url' | 'url' | 'plaintext'             */
  uint8_t status;          /* TGI_EDGE_*                                                          */
  uint8_t reserved;
} tgi_edge;
int tgi_set_add(tgi_ctx* ctx, int which, const uint8_t* keys32, const int64_t* stamp_sec, uint64_t n);
int tgi_set_clear(tgi_ctx* ctx, int which);
int tgi_set_size(tgi_ctx* ctx, int which, uint64_t* n);
/* the clock tgi_*_batch uses for the invalid-channel TTL (TGI_RUN_SKIP_INVALID); default: never expire */
int tgi_set_now(tgi_ctx* ctx, int64_t now_sec);
int tgi_pending_edges(tgi_ctx* ctx, int slot, int64_t now_sec, tgi_edge* rows, uint64_t cap, uint64_t* n);

/* Resident key sets that grow on demand, as the reference's maps do (seenInBatch, urlCache, existingURLs,
 * DiscoveredChannels, invalidChannelCache grow without limit).
 *   tgi_set_growth   every resident set (the dedup set, the two exclusion sets, this rank's partition of the global set)
 *                    may grow up to max_keys keys (< 2^40); 0 = fixed capacity, the default.  tgi_config.frontier_capacity
 *                    is then the initial capacity of the dedup set and the partition; the exclusion sets start at
 *                    min(frontier_capacity, 1<<16) keys.  A batch or insert that brings more keys than fit moves the set
 *                    into buffers for next_pow2(count + incoming) keys first: the keys keep their first-occurrence order,
 *                    so every result and the export equal those of a set that was big enough from the start.  Device
 *                    memory peaks at old + new buffers during the move.  Past max_keys the call fails with
 *                    TGI_E_CAPACITY and leaves the set untouched.  Must not be called while a job is in flight on any
 *                    slot (returns TGI_E_STATE).
 *   tgi_set_info     count, capacity, table slots and number of growth steps of one set (all 0 for an exclusion set
 *                    before its first tgi_set_add); TGI_SET_OWNED before tgi_comm_init returns TGI_E_STATE.          */
#define TGI_SET_FRONTIER 0    /* the dedup set (tgi_frontier_*, TGI_RUN_FRONTIER)                  */
#define TGI_SET_OWNED 3       /* this rank's partition of the global set (tgi_frontier_merge)      */
typedef struct tgi_set_info_t {
  uint64_t count;       /* keys in the set                                                        */
  uint64_t capacity;    /* keys it holds before it grows (or fails with TGI_E_CAPACITY)           */
  uint64_t table_slots; /* slots of its open-addressed hash table                                 */
  uint64_t grows;       /* growth steps since it was created or last allocated                    */
} tgi_set_info_t;
int tgi_set_growth(tgi_ctx* ctx, uint64_t max_keys);
int tgi_set_info(tgi_ctx* ctx, int which, tgi_set_info_t* out);

/* Crawl progress state on the device — BaseStateManager's pageMap / layerMap (state/base.go) with state.Page and
 * state.Message (state/datamodels.go:41-71), so LocalStateManager can write state.json ONCE per page (or per channel)
 * instead of after every UpdateMessage / UpdatePage / AddLayer (state/storageproviders.go:246-272, 431-464).  The state
 * has its own lock; every call applies atomically in call order and a rejected call leaves the state unchanged.
 *   Rows     one page row per page id (pageMap).  The calls that create rows return them; a row stays valid until the
 *            next tgi_state_set.  TGI_STATE_NO_PAGE names no page.
 *   Pages    tgi_state_page: the nine strings (TGI_PS_*, in that order, back to back at strs[str_off]), depth, and the
 *            timestamp: ts_sec / ts_nsec (0 <= nsec < 1e9) with ts_off = seconds east of UTC (|ts_off| < 86400; a
 *            page reloaded from state.json keeps the offset it was written with; the zero time is -62135596800, 0, 0)
 *            or TGI_STATE_TS_LOCAL (time.Now(): rendered in the context's local zone, tgi_set_zone / tz_offset_sec,
 *            at render time).
 *   Codes    message status and platform are indices into a string table: 0 "", 1 "unfetched", 2 "fetched",
 *            3 "failed", 4 "deleted", 5 "resample"; tgi_state_code registers others (or returns the existing code).
 *   Messages tgi_state_msg.page_id is the row whose id is the message's pageId (normally its own page's).
 *            tgi_state_set: an index into that call's pages; tgi_state_update_page: a row, or TGI_STATE_NO_PAGE for
 *            the page being written.  A pageId that names no page of the state cannot be expressed.
 *   Set      tgi_state_set = SetState (base.go:375-398) / Initialize (:54-93): replaces everything.  layers[k] takes
 *            the next layers[k].n_pages pages; pages[i] owns the next pages[i].n_msgs messages.  A later layer of the
 *            same depth replaces the earlier list; a later page with the same id replaces the earlier one (pageMap),
 *            messages included.  rows (optional, n_pages) gets each page's row.  The resume path: the shim parses
 *            state.json itself and hands it over.
 *   AddLayer tgi_state_add_layer = AddLayer (base.go:219-322) for pages without messages: skips URLs already in the
 *            state or earlier in the call; max_pages > 0 caps the state at max_pages pages, past which only as many
 *            pages as there were "deadend" pages at the call's start are added; every page goes to the layer of
 *            pages[0].depth (created even if nothing is added).  The caller fills empty ids and zero timestamps
 *            beforehand (uuid.New(), time.Now()).  rows (optional) gets each page's row or TGI_STATE_NO_PAGE (skipped).
 *   Update   tgi_state_update_page = UpdatePage (base.go:123-149): replaces the page with that id (a new row if none)
 *            and its whole message list; the row is appended to the layer of its depth only if that layer exists and
 *            does not hold it.
 *   Messages tgi_state_update_messages = UpdateMessage (base.go:182-215) once per update, in order: the first message
 *            of the row with that (chat_id, message_id) takes the status, an unknown key is appended as {chat, msg,
 *            status, pageId = the page} and later updates of it hit the appended message.  An update whose row is
 *            TGI_STATE_NO_PAGE is skipped and counted in *skipped (the reference returns an error its caller ignores).
 *   Read     tgi_state_read_page = GetPage(id).Messages: *n = the row's message count; the messages are written
 *            when cap >= *n.
 *   Render   tgi_state_render = json.Marshal(GetState()) (base.go:345-372), byte for byte: {"layers":[...],
 *            "metadata":<metadata>,"lastUpdated":<last_updated>} where the two spliced values are the shim's own
 *            json.Marshal of CrawlMetadata and of the time.  Layers in ascending depth (Go iterates layerMap in
 *            random order: every order is a valid json.Marshal output, this one is fixed); omitempty strings and
 *            empty message lists are left out; strings use encoding/json's HTML-safe escaping.  A timestamp whose
 *            year leaves [0, 9999] is TGI_E_ARG (json.Marshal's error).  The bytes live in library-owned pinned
 *            memory until the next state call.
 *   Errors   TGI_E_ARG: malformed input (string ranges, layer / message counts, an unknown code, a row that is
 *            neither a row nor TGI_STATE_NO_PAGE, nsec / offset out of range, messages in tgi_state_add_layer);
 *            TGI_E_NOMEM.  More than 2^32 - 2 message rows is TGI_E_CAPACITY.                                     */
#define TGI_STATE_NO_PAGE 0xFFFFFFFFu
#define TGI_STATE_TS_LOCAL 0x7FFFFFFF
enum { TGI_PS_ID, TGI_PS_URL, TGI_PS_STATUS, TGI_PS_ERROR, TGI_PS_PLATFORM, TGI_PS_PARENT, TGI_PS_CONN, TGI_PS_SEQ,
       TGI_PS_CRAWL, TGI_PS_COUNT };
typedef struct tgi_state_page { /* 72 bytes: one state.Page without its messages */
  uint64_t str_off;                  /* id | url | status | error | platform | parentId | LastConnectionID |
                                        sequenceId | crawlId, back to back                                     */
  uint32_t str_len[TGI_PS_COUNT];
  int32_t ts_off;                    /* seconds east of UTC, or TGI_STATE_TS_LOCAL                             */
  int64_t depth;
  int64_t ts_sec;
  int32_t ts_nsec;
  uint32_t n_msgs;                   /* tgi_state_set / tgi_state_update_page: its messages                    */
} tgi_state_page;
typedef struct tgi_state_msg { /* 24 bytes: one state.Message */
  int64_t chat_id, message_id;
  uint32_t page_id;                  /* see Messages above                                                     */
  uint16_t status, platform;         /* codes                                                                  */
} tgi_state_msg;
typedef struct tgi_state_update { /* 24 bytes: the arguments of one UpdateMessage */
  int64_t chat_id, message_id;
  uint32_t row;                      /* the page (TGI_STATE_NO_PAGE: not found)                                */
  uint16_t status, reserved;
} tgi_state_update;
typedef struct tgi_state_layer { int64_t depth; uint64_t n_pages; } tgi_state_layer;
typedef struct tgi_state_json_t {
  const uint8_t* data;  uint64_t len;  /* state.json, pinned                                                    */
  float kernel_ms;                     /* device time of the render's kernels and scans (not the read-back)     */
  uint32_t gpu_launches;
} tgi_state_json_t;
int tgi_state_code(tgi_ctx* ctx, const char* s, uint32_t len, uint16_t* code);
int tgi_state_set(tgi_ctx* ctx, const tgi_state_layer* layers, uint32_t n_layers, const tgi_state_page* pages,
                  uint64_t n_pages, const uint8_t* strs, uint64_t strs_len, const tgi_state_msg* msgs, uint64_t n_msgs,
                  uint32_t* rows);
int tgi_state_add_layer(tgi_ctx* ctx, const tgi_state_page* pages, uint64_t n, const uint8_t* strs, uint64_t strs_len,
                        int64_t max_pages, uint32_t* rows);
int tgi_state_update_page(tgi_ctx* ctx, const tgi_state_page* page, const uint8_t* strs, uint64_t strs_len,
                          const tgi_state_msg* msgs, uint32_t* row);
int tgi_state_update_messages(tgi_ctx* ctx, const tgi_state_update* ups, uint64_t n, uint64_t* skipped);
int tgi_state_read_page(tgi_ctx* ctx, uint32_t row, tgi_state_msg* out, uint64_t cap, uint64_t* n);
int tgi_state_render(tgi_ctx* ctx, const uint8_t* metadata, uint64_t metadata_len, const uint8_t* last_updated,
                     uint64_t last_updated_len, tgi_state_json_t* out);

/* pure helpers exposed for host code and tests (each runs the device code path on tiny inputs) */
int tgi_filter_usernames(tgi_ctx* ctx, const uint8_t* names, const uint32_t* off, uint64_t n,
                         uint8_t* reason);

#ifdef __cplusplus
}
#endif
#endif /* TGINGEST_H */
