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
  int32_t published_nsec; /* 0 <= nsec < 1e9, as Time.Nanosecond(); anything else: the batch is TGI_E_ARG   */
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
  int32_t published_nsec; /* 0 <= nsec < 1e9, as Time.Nanosecond(); anything else: the batch is TGI_E_ARG   */
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
  int32_t ts_nsec;    /* 0 <= ts_nsec < 1e9, as Time.Nanosecond(); anything else: the batch is TGI_E_ARG */
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

/* ---- channel records: the random-walk StoreChannelData line ----------------------------------------
 * A random-walk crawl stores no posts (DaprStateManager.StorePost returns early, state/daprstate.go:1109-1111); its
 * one stored line per channel page is the model.ChannelData that RunForChannel builds (crawl/runner.go:592-610) and
 * passes to sm.StoreChannelData(p.URL, channelData) (:620-626) before the activity check, marshalled with json.Marshal
 * + '\n' (daprstate.go:3088-3148).  One record per channel page, filled by the shim from TDLib's chat and the counts
 * of getChannelInfo (runner.go:975-983).                                                                            */
typedef struct tgi_ch_rec { /* 40 bytes */
  int64_t chat_id;        /* chat.Id: channel_id = strconv.FormatInt(chat_id, 10)                              */
  uint64_t str_off;       /* in `strs`: title | image | url                                                     */
  int32_t member_count;   /* int32(memberCount) (runner.go:982): follower_count                                 */
  int32_t message_count;  /* int32(messageCount) (:981): post_count                                              */
  int32_t total_views;    /* int32(totalViews) (:980): views_count                                               */
  uint32_t title_len;     /* chat.Title: channel_name                                                           */
  uint32_t image_len;     /* chat.Photo.Extra, 0 when chat.Photo == nil: channel_profile_image                  */
  uint32_t url_len;       /* p.URL: channel_url_external = channel_url = "https://t.me/" + p.URL                */
} tgi_ch_rec;

typedef struct tgi_ch_batch {
  uint64_t n;
  const tgi_ch_rec* recs;
  const uint8_t* strs;
  uint64_t strs_len;
} tgi_ch_batch;

/* ---- configuration -------------------------------------------------------------------------- */
#define TGI_CFG_HAS_MIN_POST_DATE 0x01 /* !cfg.MinPostDate.IsZero()                               */
#define TGI_CFG_SKIP_MEDIA 0x02        /* cfg.SkipMediaDownload; REQUIRED (media download is RPC) */

typedef struct tgi_config {
  uint32_t abi_version;    /* TGI_ABI_VERSION                                                     */
  int32_t device;          /* CUDA ordinal                                                        */
  uint32_t flags;          /* TGI_CFG_*                                                           */
  int32_t tz_offset_sec;   /* fixed offset of the process-local zone (time.Unix -> Local); |offset| < 86400 */
  int64_t min_post_date;   /* unix seconds                                                        */
  int64_t created_at_sec;  /* injected time.Now(): Telegram uses .UTC().Truncate(time.Second)
                              (tdutils.go:611); YouTube keeps zone + nanoseconds (youtube_crawler.go:704) */
  int64_t capture_sec;     /* injected time.Now() (tdutils.go:715, youtube_crawler.go:769)        */
  int32_t capture_nsec;    /* 0 <= nsec < 1e9 (both), as Time.Nanosecond()                       */
  int32_t created_at_nsec; /* tgi_create refuses anything else, and |tz_offset_sec| >= 86400, with TGI_E_ARG */
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
/* must not be called while a job is in flight on any slot (returns TGI_E_STATE).  0 <= nsec < 1e9  */
/* for both, else TGI_E_ARG; a rejected call leaves the previous clock in effect.                  */
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
 *   Inputs   tgi_combine_add takes the slot's last result (Telegram or YouTube, bulk or page, or tgi_channel_batch: its
 *            channel_<id>_<ns>.jsonl files land in the same watch directory) like tgi_dapr_payloads,
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
 *            or it is a tgi_generic_batch one (its posts go to SavePost) or a tgi_channel_batch one (the local manager
 *            stores no channel data).  TGI_E_ARG: bad slot or NULL out.
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
 *                youtube_crawler.go:396), PostUID = the record's id (video.ID, :701).  A tgi_channel_batch result
 *                (StoreChannelData, daprstate.go:3114-3117): prefix | url | "/channel_data.jsonl".
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

/* Channel records -> model.ChannelData lines: replaces the random-walk branch of RunForChannel (crawl/runner.go:592-626)
 * up to json.Marshal+'\n' in StoreChannelData (state/daprstate.go:3089-3094), for the channel pages of a whole step.
 * Blocking; picks a free slot, like tgi_generic_batch.
 *   Line     {"channel_id":"<chat_id>","channel_name":<title>,"channel_description":"","channel_profile_image":<image>,
 *            "channel_engagement_data":{"follower_count":<member_count>,"following_count":0,"like_count":0,
 *            "post_count":<message_count>,"views_count":<total_views>,"comment_count":0,"share_count":0},
 *            "channel_url_external":"https://t.me/<url>","channel_url":"https://t.me/<url>","country_code":"",
 *            "published_at":"0001-01-01T00:00:00Z"} and '\n' (model/data.go:89-111).  Strings in encoding/json's
 *            HTML-safe escaping, invalid UTF-8 as �.  json.Marshal cannot fail here: every status is
 *            TGI_ST_EMITTED.  No links.
 *   Flags    TGI_RUN_JSONL and TGI_RUN_JSONL_DEVICE only; any other flag is TGI_E_ARG.
 *   Sinks    the result feeds tgi_dapr_payloads (Data = base64 of each line, path = path_prefix | url |
 *            "/channel_data.jsonl", generateCrawlExecutableStoragePath daprstate.go:2689-2698 with channelID = p.URL) and
 *            tgi_combine_add (the channel_<id>_<ns>.jsonl files enter the chunker's watch directory beside the post files,
 *            daprstate.go:3096-3111).  tgi_channel_appends refuses it with TGI_E_STATE: the local manager stores no
 *            channel data (state/base.go:530-532).
 *   Errors   TGI_E_ARG, naming the first bad record: a range title | image | url outside strs, or a string of 16 MiB or
 *            more.  Small batches are checked on the host, big ones on the device, before any kernel reads a string. */
int tgi_channel_batch(tgi_ctx* ctx, const tgi_ch_batch* in, uint32_t run_flags, tgi_result* out);

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
 *            when cap >= *n, gathered as tgi_state_read_pages gathers them (its n = 1 case).
 *   Render   tgi_state_render = json.Marshal(GetState()) (base.go:345-372), byte for byte: {"layers":[...],
 *            "metadata":<metadata>,"lastUpdated":<last_updated>} where the two spliced values are the shim's own
 *            json.Marshal of CrawlMetadata and of the time.  Layers in ascending depth (Go iterates layerMap in
 *            random order: every order is a valid json.Marshal output, this one is fixed); omitempty strings and
 *            empty message lists are left out; strings use encoding/json's HTML-safe escaping.  A timestamp whose
 *            year leaves [0, 9999] is TGI_E_ARG (json.Marshal's error).  The bytes live in library-owned pinned
 *            memory until the next state call.
 *   Errors   TGI_E_ARG: malformed input (string ranges, layer / message counts, an unknown code, a row that is
 *            neither a row nor TGI_STATE_NO_PAGE, nsec / offset out of range, messages in tgi_state_add_layer);
 *            TGI_E_NOMEM.  More than 2^32 - 2 message rows is TGI_E_CAPACITY.  Every writer of this state (render,
 *            exports, page and discovery JSON, layer map, edge SQL, walkback) refuses a page, message, layer-map id or
 *            SQL row that renders to 4 GiB or more with TGI_E_CAPACITY before writing it; the whole output may pass
 *            4 GiB.  Calls whose page JSON fails after their update (Dapr's UpdatePage) fail so for this too.       */
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

/* The same state for DaprStateManager (state/daprstate.go), whose SaveState marshals the whole layer map after every
 * channel and whose ExportPagesToBinding marshals every page at the end of a crawl.
 *   LayerMap tgi_state_layer_map = json.Marshal(layerMap), a map[int][]string (daprstate.go:947), byte for byte: the
 *            keys are the decimal depths sorted as strings (-1, 0, 10, 2), as encoding/json sorts integer map keys; an
 *            empty layer is [] and an empty map {}; ids use the HTML-safe escaper and a row listed twice is listed
 *            twice.  Pinned bytes in out, like tgi_state_render's.
 *   AddPages tgi_state_add_pages = the in-memory part of Dapr's AddLayer (daprstate.go:625-780) once the caller has
 *            dropped the pages whose URL is in its urlCache (or dropped none, in random-walk mode): every page is
 *            stored as pageMap[id] = page (an existing id keeps its row and loses its messages) and its row appended to
 *            the layer `depth`, created if missing; depth is pages[0].Depth BEFORE that filtering.  No URL dedup, no
 *            max_pages; n = 0 changes nothing (Dapr creates no layer when every page was a duplicate).  rows
 *            (optional, n) gets each page's row.  Pages carrying messages are TGI_E_ARG.
 *   Export   tgi_state_export renders every page as one JSONL line, json.Marshal(page) + '\n':
 *            TGI_STATE_EXPORT_DAPR = DaprStateManager.ExportPagesToBinding (daprstate.go:2911-3012): the pages of the
 *              layer map in its order (layers in ascending depth, as tgi_state_render), cut into chunks: a chunk
 *              closes right after the line that brings it to chunk_bytes or more (0: one page per chunk), the last
 *              chunk is the rest.  Each chunk is base64.StdEncoding-encoded on the device; chunk k is len[k] bytes at
 *              data + off[k] (off[k] % 16 == 0) and encodes raw_len[k] JSONL bytes.  A layer map without pages is
 *              TGI_E_NOPAGES (the reference's "no pages found to export").  The shim names chunk k
 *              <StorageRoot>/<config CrawlID>/analysis/channels/channel-pages-<crawlID>-<ts>-part<k>.jsonl.
 *            TGI_STATE_EXPORT_LOCAL = LocalStateManager.ExportPagesToBinding (storageproviders.go:550-587): every page
 *              of pageMap once, in row order (Go's map order is random), raw JSONL in one chunk (empty without pages).
 *            Timestamps, omitempty fields and message lists are those of tgi_state_render; a timestamp whose year
 *            leaves [0, 9999] is TGI_E_ARG (where Go logs the marshal error and skips the page).  The output lives in
 *            library-owned pinned memory until the next state call. */
#define TGI_E_NOPAGES (-7)  /* tgi_state_export: the layer map holds no page                                */
#define TGI_STATE_EXPORT_DAPR 0
#define TGI_STATE_EXPORT_LOCAL 1
typedef struct tgi_state_export_t {
  const uint8_t* data;       /* the chunks: base64 (Dapr) or raw JSONL (local), pinned                         */
  const uint64_t* off;       /* [n_chunks] chunk k starts at data + off[k]                                     */
  const uint64_t* len;       /* [n_chunks] its bytes in data                                                   */
  const uint64_t* raw_len;   /* [n_chunks] its JSONL bytes before encoding                                     */
  uint64_t n_chunks;
  uint64_t n_pages;          /* lines exported                                                                 */
  float kernel_ms;           /* device time of the kernels and scans (not the read-back)                      */
  uint32_t gpu_launches;
} tgi_state_export_t;
int tgi_state_layer_map(tgi_ctx* ctx, tgi_state_json_t* out);
int tgi_state_add_pages(tgi_ctx* ctx, int64_t depth, const tgi_state_page* pages, uint64_t n, const uint8_t* strs,
                        uint64_t strs_len, uint32_t* rows);
int tgi_state_export(tgi_ctx* ctx, int mode, uint64_t chunk_bytes, tgi_state_export_t* out);

/* Page turns — the bookkeeping processAllMessagesWithProcessor runs once per fetched page (crawl/runner.go:1132-1147,
 * 1161-1211), in two calls that touch only that page's messages (no call reads every message row of the state).  The
 * caller's `owner` is the state's own page (row), with no other update of it between its GetPage and the turn.
 *   Begin    tgi_state_page_begin = addNewMessages + resampleMarker + UpdatePage(*owner).  fetched holds the page's
 *            fetched messages, chat_id and message_id, in fetch order (n = 0 empties the list, as the reference does).
 *            The page's list becomes the fetched keys that were NOT in its list before, in fetch order, a key fetched
 *            twice kept twice; the earlier messages are dropped.  Every new message is {chat, msg, "resample", pageId =
 *            the page, no platform}: all came from the fetch, so resampleMarker marks each one.  page (optional) replaces
 *            the row's fields as tgi_state_update_page does; its id must be the row's and it carries no messages (NULL:
 *            the fields as stored).  Either way the row joins the layer of its depth if that layer exists and does not
 *            hold it (UpdatePage's rule).
 *            out->work[i] (n_work entries, pinned) is the index into fetched of owner message i's discMessage: the FIRST
 *            fetched message with the same message id, the chat id ignored (:1171-1176).  It always exists, so the
 *            loop's "deleted" branch (:1185) cannot be reached from this flow.  The caller packs its batch as
 *            fetched[work[i]] in that order and processes it.
 *            TGI_TURN_PAGE_JSON: out->page_json = json.Marshal(page) after UpdatePage, the value DaprStateManager's
 *            UpdatePage saves (daprstate.go:1370-1407); the same bytes as the page's tgi_state_export line without its
 *            '\n'.  A timestamp whose year leaves [0, 9999] is then TGI_E_ARG AFTER the update (Dapr changes pageMap
 *            before its marshal fails) and no turn opens.  work and page_json live until the next state call.
 *   End      tgi_state_page_end = the loop's first n_done UpdateMessage calls, in order, against the state as it is at
 *            the call: exactly tgi_state_update_messages with owner message i's key SWAPPED, (message_id, chat_id) as
 *            the reference passes them, and status "failed" for TGI_ST_FAILED, "fetched" for TGI_ST_EMITTED,
 *            TGI_ST_SKIPPED and TGI_ST_NOLINE.  The swapped key usually misses and appends {msg, chat, s, pageId = the
 *            page}; later updates of the same swapped key hit that message.  n_done < n_work: the loop stopped early
 *            (the random-walk FLOOD_WAIT retire, :1333-1338).  The statuses are the resident status array of the slot's
 *            last result, not read back (slot >= 0), or status[n_done] from the host (slot < 0).  *appended (optional)
 *            gets the messages appended.  A handle is consumed once; tgi_state_set drops every open turn.
 *   Errors   TGI_E_ARG, the state unchanged: no such row, a page whose id is not the row's; an unknown or consumed
 *            handle, a slot result that is not Telegram, has been released or holds another record count than n_work,
 *            n_done > n_work.  TGI_E_STATE: a job in flight on the slot.                                              */
#define TGI_TURN_PAGE_JSON 1u
typedef struct tgi_state_turn_t {
  uint32_t turn;              /* handle for tgi_state_page_end (never 0)                                        */
  uint32_t row;
  uint64_t n_work;            /* len(owner.Messages) after addNewMessages: the records the loop processes        */
  const uint32_t* work;       /* [n_work] index into fetched of each owner message's discMessage (pinned)        */
  const uint8_t* page_json;   /* json.Marshal(page) with TGI_TURN_PAGE_JSON, else NULL (pinned)                  */
  uint64_t page_json_len;
  float kernel_ms;            /* device time of the call's kernels and scans (not the copies between them)       */
  uint32_t gpu_launches;
} tgi_state_turn_t;
int tgi_state_page_begin(tgi_ctx* ctx, uint32_t row, const tgi_state_page* page, const uint8_t* strs, uint64_t strs_len,
                         const int64_t* fetched, uint64_t n, uint32_t flags, tgi_state_turn_t* out);
int tgi_state_page_end(tgi_ctx* ctx, uint32_t turn, int slot, const uint8_t* status, uint64_t n_done, uint64_t* appended);

/* Page close — UpdatePage(*owner) at the end of the loop (crawl/runner.go:1543-1544, owner.Status = "fetched") and the
 * Dapr runner's UpdatePage(page) after it (dapr/standalone.go:589-609, "fetched", or "error" with Error set).
 *   Fields   page (required, no messages, its id the row's) replaces the row's fields exactly as
 *            tgi_state_update_page does, the timestamp included; the row joins the layer of its depth if that layer
 *            exists and does not hold it.
 *   Owner    tgi_state_page_begin leaves the row an owner view: the turn's n_work owner messages in fetch order with
 *            their keys, "resample", pageId = the page, no platform.  The view lives until the row's next begin, a
 *            tgi_state_update_page of the row, a tgi_state_add_layer / tgi_state_add_pages / discovery that overwrites
 *            the row, or tgi_state_set.  With a view the close makes the row's list exactly the view: the swapped-key
 *            messages the end appended, and anything else appended since the begin, are dropped (Go's owner slice
 *            still has its begin-time length).  Without one the list stays as it is and only the fields change.  A
 *            second close of the same view gives the same list.  The close ends every open turn of the row: a later
 *            tgi_state_page_end of it is TGI_E_ARG.
 *   Hits     parity unpinned: Go's owner shares its backing array with pageMap's page until an append reallocates
 *            it, which depends on cap(owner.Messages) (growslice and malloc size classes).  The library counts the
 *            array as full: an UpdateMessage of tgi_state_page_end that hits an owner message BEFORE the end's first
 *            append gives that status to the first owner message with the key (the last such hit wins); later hits
 *            do not reach the owner.  With Telegram's keys this never happens: the swapped key has a positive chat id
 *            and a channel's chat ids are negative.
 *   JSON     TGI_TURN_PAGE_JSON: out->data / len = json.Marshal(page) after the close (Dapr's UpdatePage value), as
 *            tgi_state_page_begin renders it; a timestamp whose year leaves [0, 9999] is then TGI_E_ARG AFTER the
 *            update.  out may be NULL without the flag; else it gets kernel_ms / gpu_launches and the bytes live until
 *            the next state call.
 *   Errors   TGI_E_ARG, the state unchanged: no such row, an id that is not the row's, messages in page, unknown
 *            flags, strings outside strs.                                                                            */
int tgi_state_page_close(tgi_ctx* ctx, uint32_t row, const tgi_state_page* page, const uint8_t* strs, uint64_t strs_len,
                         uint32_t flags, tgi_state_json_t* out);

/* Multi-page turns — the bookkeeping of P pages (crawl/runner.go:1132-1211, 1543-1544, dapr/standalone.go:589-609) in
 * one call per step, so that the pages of a worker's channels share one bulk batch: begin them all, pack every work list
 * into one batch and run it (TGI_RUN_JSONL_DEVICE keeps the statuses on the device), end them all from that result,
 * close them all.  For the same flags a call's synchronises, and its launches from P = 2 on, do not depend on P (a
 * one-page call keeps the one-launch scans); the one-page calls above are its P = 1 case.  The launches still follow the
 * data in two places: an end launches nothing without a processed record and its view passes only for pages whose row
 * still holds the turn's view, and a TGI_TURN_PAGE_JSON close of any row without an owner view adds one scan of the
 * message rows and the render's radix passes, whose number is set by the state's row count.
 *   Begin    tgi_state_pages_begin = tgi_state_page_begin of rows[0], rows[1], ... in that order, each with its own
 *            fetched keys fetched[fetched_off[k] .. fetched_off[k+1]) (fetched_off[0] = 0, ascending, fetched_off[P] = n)
 *            and pages[k] (pages NULL: every row keeps its fields).  One handle covers the P pages.  Page k's owner
 *            messages are work[work_off[k] .. work_off[k+1]) of out->work[n_work]; work[i] indexes the call's whole
 *            fetched array, so the caller packs fetched[work[i]] for i = 0 .. n_work-1 as one batch.  Each page's
 *            equal message ids are matched within the page only.  TGI_TURN_PAGE_JSON: page_json holds
 *            json.Marshal(page) + '\n' of every page in call order, page k's line being [json_off[k], json_off[k+1]),
 *            as tgi_state_discover returns its pages.
 *   End      tgi_state_pages_end = tgi_state_page_end of every page in page order, page k with its first n_done[k]
 *            records (n_done NULL: all of them).  The turn's n_work records are [first, first + n_work) of the slot's
 *            last Telegram result, which may hold other records before and after them (slot >= 0), or status[n_work]
 *            from the host (slot < 0; records past a page's n_done are not read).  The owner views' hits follow the
 *            close's rules, page by page.  tgi_state_pages_end takes a one-page handle; tgi_state_page_end of a handle
 *            that covers more than one page is TGI_E_ARG.  out (optional) gets the messages appended, the device time
 *            and the launches; with out the call waits for its kernels.
 *   Close    tgi_state_pages_close = tgi_state_page_close of rows[0], rows[1], ... with pages[k] (required), in that
 *            order.  TGI_TURN_PAGE_JSON: out->page_json / json_off as the begin's.  Closing any row of an open turn
 *            ends that whole turn: a later end of it is TGI_E_ARG.  out may be NULL without the flag.
 *   Errors   every check runs before anything changes, so a rejected call leaves the state, the open turns and the
 *            views unchanged.  TGI_E_ARG: no pages, a row unknown or listed twice, a page whose id is not its row's,
 *            that carries messages or whose strings lie outside strs, a fetched_off that decreases or does not run
 *            from 0 to n, unknown flags; an unknown or consumed handle, a slot result that is released, not Telegram
 *            or shorter than first + n_work, n_done[k] greater than page k's work, no host statuses with slot < 0.
 *            TGI_E_STATE: a job in flight on the slot.  As with the one-page calls, a timestamp whose year leaves
 *            [0, 9999] fails a TGI_TURN_PAGE_JSON call after the update (the begin then opens no turn).
 *            tgi_state_set drops every open turn.  All of out lives until the next state call.                         */
typedef struct tgi_state_pages_t {
  uint32_t turn;              /* handle for tgi_state_pages_end (never 0); 0 from a close                         */
  uint32_t n_pages;
  uint64_t n_work;            /* owner messages of all pages: the records the loops process                       */
  const uint32_t* work;       /* [n_work] index into fetched of each owner message's discMessage (pinned)         */
  const uint64_t* work_off;   /* [n_pages+1] page k's owner messages are [work_off[k], work_off[k+1])             */
  const uint8_t* page_json;   /* with TGI_TURN_PAGE_JSON: the pages' lines, else NULL (pinned)                     */
  const uint64_t* json_off;   /* [n_pages+1] page k's line is [json_off[k], json_off[k+1]), its '\n' last          */
  float kernel_ms;            /* device time of the call's kernels and scans (not the copies between them)        */
  uint32_t gpu_launches;
} tgi_state_pages_t;
int tgi_state_pages_begin(tgi_ctx* ctx, const uint32_t* rows, uint32_t n_pages, const tgi_state_page* pages,
                          const uint8_t* strs, uint64_t strs_len, const int64_t* fetched, uint64_t n,
                          const uint64_t* fetched_off, uint32_t flags, tgi_state_pages_t* out);
typedef struct tgi_state_end_t {
  uint64_t appended;          /* messages the ends appended                                                       */
  float kernel_ms;            /* device time of the call's kernels and scans (not the copies between them)        */
  uint32_t gpu_launches;
} tgi_state_end_t;
int tgi_state_pages_end(tgi_ctx* ctx, uint32_t turn, int slot, uint64_t first, const uint8_t* status,
                        const uint64_t* n_done, tgi_state_end_t* out);
int tgi_state_pages_close(tgi_ctx* ctx, const uint32_t* rows, uint32_t n_pages, const tgi_state_page* pages,
                          const uint8_t* strs, uint64_t strs_len, uint32_t flags, tgi_state_pages_t* out);

/* Snowball discovery — the outlinks of processed pages become the next layer's pages (crawl/runner.go:1199-1244 outside
 * random-walk, then standalone/runner.go:835-850 or dapr/standalone.go:612-616, 645-688), read straight from a slot's
 * resident Telegram result: nothing is read back before the dedup, so it works after TGI_RUN_JSONL_DEVICE and
 * TGI_RUN_NO_D2H, and only the deduplicated survivors (name, parent) cross to the host.
 *   Candidates  span k names one owner page (row) and its records [first, first+n_records) of the result, of which the
 *            loop processed the first n_done.  Every link row of a processed record whose status is TGI_ST_EMITTED or
 *            TGI_ST_NOLINE is a candidate (a failed record returned an error and a date-skipped one an empty Post: no
 *            outlinks), unless its name is byte-equal to the owner row's URL as the state holds it (`o == owner.URL`,
 *            case-sensitive: not TGI_LF_SELF, which compares with the record's channel name).  Candidate order is
 *            (span, record, link row); Go ranges over a per-message map, so every order inside a message is a valid
 *            output and this one is fixed.  TGI_RUN_FILTER / SKIP_SELF / SKIP_INVALID only gate the dedup-set insert;
 *            the link rows stay whole.  Each candidate becomes {URL: name, Status: "unfetched", ParentID: owner.ID,
 *            Depth: owner.Depth + 1} with the owner as it is at the call.
 *   Discover tgi_state_discover.  TGI_DISCOVER_NOW: each span with at least one candidate is one AddLayer, in span
 *            order, under BaseStateManager's rules (base.go:219-322, as tgi_state_add_layer: first occurrence per URL
 *            within the span, URLs already in the state skipped, max_pages with the deadend budget, the layer of
 *            owner.Depth + 1 created even if every page is skipped) or with TGI_DISCOVER_DAPR DaprStateManager's
 *            (daprstate.go:625-780: a URL in the urlCache set TGI_SET_URLS is skipped, NO dedup within the call, so a
 *            page that mentions a channel twice adds it twice; no max_pages; no layer when nothing is added; the added
 *            URLs then enter TGI_SET_URLS).  A span without candidates makes no call and creates no layer.  Without
 *            TGI_DISCOVER_NOW the candidates (name, owner row) are appended to the state's pending next-layer list on
 *            the device and the state is otherwise unchanged.
 *   Layer end tgi_state_next_layer = the layer end of dapr/standalone.go:647-688 over the pending list: the first
 *            occurrence of every URL, its ParentID included, with Depth = layer_depth + 1, then AddLayer under the
 *            chosen rules, then the list is emptied.  An empty list changes nothing.  tgi_state_set drops the list.
 *   Pages    every added page gets an id and the timestamp (now_sec, now_nsec) in time.Local (TGI_STATE_TS_LOCAL): one
 *            clock reading per call, where Go reads it per page.  out->rows / ids list the added pages in the order
 *            AddLayer appended them.  TGI_DISCOVER_PAGE_JSON: page_json holds json.Marshal(page) + '\n' of every added
 *            page (its tgi_state_export line), page k's value being [json_off[k], json_off[k+1] - 1): the values of
 *            Dapr's per-page SaveState("<execID>/page/<id>").  All of out lives until the next state call.
 *   Ids      uuid.New() is random; the library makes its own version-4 ids.  The n-th page added under the context (n
 *            counts added pages only, and tgi_state_set does not reset it) takes the id from Philox4x32-10 with counter
 *            (n_lo, n_hi, 0, 0) and key (seed_lo, seed_hi): the four words little-endian as 16 bytes, then
 *            b[6] = b[6]&0x0f|0x40 and b[8] = b[8]&0x3f|0x80, as lowercase 8-4-4-4-12 hex.  Philox is a bijection of the
 *            counter and only the 6 version / variant bits are overwritten, so two ids of one seed collide as often as
 *            two random v4 uuids.  tgi_state_id_seed sets the key (the shim seeds it once from crypto/rand); without it a
 *            call that would add a page returns TGI_E_STATE: a built-in seed would repeat ids across processes.
 *   urlCache TGI_SET_URLS is Dapr's urlCache on the device: the shim seeds it with tgi_set_add from initializeURLCache
 *            / loadURLsForCrawl, skipping URLs longer than 32 bytes (a key holds 32; an outlink name is 5-32 bytes and
 *            can never equal them); Dapr-rule AddLayers grow it, as tgi_set_growth lets every set grow.
 *   Cost     the call sizes its scratch (flags, scans, the batch table) by the result's link rows times the largest
 *            number of spans that share a record, without reading anything back: pass all the spans of one result in
 *            one call (a page-sized result: its one span), not one call per page of a bulk result.
 *   Errors   a rejected call (TGI_E_ARG, TGI_E_STATE, and TGI_E_CAPACITY when TGI_SET_URLS cannot take the added URLs:
 *            the set's insert is all or nothing) leaves the state, the pending list and TGI_SET_URLS unchanged; after
 *            TGI_E_CUDA or TGI_E_NOMEM the added URLs may be in TGI_SET_URLS without their pages.  TGI_E_ARG: an unknown row, a span outside
 *            the result, n_done > n_records, now_nsec outside [0, 1e9), unknown flags, and with
 *            TGI_DISCOVER_PAGE_JSON a clock whose year leaves [0, 9999].  TGI_E_STATE: no, a released or a non-Telegram
 *            result, a result run without TGI_RUN_LINKS, a job in flight on the slot, no seed.  Lock order: the slot,
 *            then the state (as tgi_state_page_end).                                                                */
#define TGI_SET_URLS 4              /* Dapr's urlCache (daprstate.go:646-658): seeded with tgi_set_add            */
/* TGI_SET_SEEDS 5, Dapr's chatIDCache, is with tgi_state_rw_lookups below */
#define TGI_DISCOVER_NOW 1u         /* AddLayer per span now (standalone/runner.go:835-850); else append to pending */
#define TGI_DISCOVER_DAPR 2u        /* DaprStateManager.AddLayer's rules instead of BaseStateManager's            */
#define TGI_DISCOVER_PAGE_JSON 4u   /* json.Marshal of every added page (Dapr's per-page SaveState value)         */
typedef struct tgi_state_span {     /* 32 bytes: one owner page's records in the slot's result                    */
  uint32_t row;                     /* the owner page: its URL, id and depth at the call                          */
  uint32_t reserved;
  uint64_t first, n_records, n_done;
} tgi_state_span;
typedef struct tgi_state_added_t {
  uint64_t n_candidates;            /* outlinks considered after the self test                                   */
  uint64_t n_added;
  const uint32_t* rows;             /* [n_added] the new rows, in the order AddLayer appended them (pinned)      */
  const uint8_t* ids;               /* [n_added][36] their uuid strings (pinned)                                 */
  const uint8_t* page_json;         /* with TGI_DISCOVER_PAGE_JSON: the added pages' lines, else NULL (pinned)   */
  const uint64_t* json_off;         /* [n_added+1] line k is [json_off[k], json_off[k+1]), its '\n' last         */
  float kernel_ms;                  /* device time of the call's kernels and scans (not the copies between them) */
  uint32_t gpu_launches;
} tgi_state_added_t;
int tgi_state_id_seed(tgi_ctx* ctx, uint64_t seed);
int tgi_state_discover(tgi_ctx* ctx, int slot, const tgi_state_span* spans, uint32_t n_spans, uint32_t flags,
                       int64_t now_sec, int32_t now_nsec, int64_t max_pages, tgi_state_added_t* out);
int tgi_state_next_layer(tgi_ctx* ctx, int64_t layer_depth, uint32_t flags, int64_t now_sec, int32_t now_nsec,
                         int64_t max_pages, tgi_state_added_t* out);

/* Tandem hand-off — the random-walk tandem branch of processAllMessagesWithProcessor (crawl/runner.go:1129, 1229-1306,
 * 1414-1455): every page's pending-edge batch for the validator, read straight from a slot's resident Telegram result,
 * with seenInBatch per page.  tgi_pending_edges stays the single-batch form, deduplicated by the global set.
 *   Spans    as tgi_state_discover's: the owner row, its records [first, first + n_records) of the slot's last result,
 *            the first n_done of them processed.  Spans may share records.
 *   Candidates  every link row of a processed record whose status is TGI_ST_EMITTED or TGI_ST_NOLINE, except names
 *            byte-equal to the owner row's URL at the call (`o == owner.URL`), names FilterUsername refuses
 *            (tgi_link.flags without TGI_LF_FILTER_OK) and names in TGI_SET_INVALID still live at now_sec (the TTL
 *            predicate of TGI_RUN_SKIP_INVALID; an empty or unallocated set drops nothing).  The run flags FILTER /
 *            SKIP_SELF / SKIP_INVALID / FRONTIER play no part; the result needs TGI_RUN_LINKS only.
 *   Edges    per span, the first occurrence of every candidate name in (record, link row) order (seenInBatch), with the
 *            record and source_type of that occurrence; status TGI_EDGE_DUPLICATE for a name in TGI_SET_DISCOVERED,
 *            else TGI_EDGE_PENDING (the validator's cache look-ups; invalid names were dropped).  Edge order is (span,
 *            record, link row): Go ranges over a per-message map, so every order inside a message is valid.
 *   Batches  one per span with at least one edge, in span order: PendingEdgeBatch{SourceChannel: owner.URL,
 *            SourcePageID: owner.ID, SourceDepth: owner.Depth, SequenceID: owner.SequenceID} of row spans[span].row.
 *            A span without edges has span_batch = TGI_STATE_NO_BATCH: the crawler's forced walkback.  The n-th batch
 *            made under the context takes the id of tgi_state_discover's page ids with counter (n_lo, n_hi, 1, 0): word
 *            2 = 1 keeps batch ids apart from page ids under one seed.  n counts batches only, and tgi_state_set does
 *            not reset it.  Without tgi_state_id_seed a call that would make a batch is TGI_E_STATE.
 *   Cost     scratch is sized as tgi_state_discover's, without a read-back: pass all spans of one result in one call.
 *            One synchronise for the totals, one for the read-back; from n_spans = 2 on the launches do not depend on
 *            n_spans.
 *   Errors   every check runs before anything changes; a rejected call leaves the state, the sets and the batch counter
 *            as they were, and a successful one changes only the batch counter.  TGI_E_ARG: an unknown row, a span
 *            outside the result, n_done > n_records.  TGI_E_STATE: no, a released or a non-Telegram result, a result
 *            run without TGI_RUN_LINKS, a job in flight on the slot, no seed while a batch is due.  Lock order: the
 *            slot, then the state.  All of out lives until the next state call; the device-side edges, batches and
 *            spans live as long, for tgi_state_edge_sql.                                                               */
#define TGI_STATE_NO_BATCH 0xFFFFFFFFu
typedef struct tgi_state_edge {        /* 48 bytes: one pending_edges row                                              */
  uint8_t destination[32];             /* destination_channel, lower-cased, zero padded                               */
  uint64_t record;                     /* the result record of its first occurrence in the page                       */
  uint32_t batch;                      /* index into batches                                                          */
  uint8_t dest_len;
  uint8_t source_type;                 /* TGI_SRC_*                                                                   */
  uint8_t status;                      /* TGI_EDGE_PENDING | TGI_EDGE_DUPLICATE                                       */
  uint8_t reserved;
} tgi_state_edge;
typedef struct tgi_state_edge_batch {  /* 48 bytes: one pending_edge_batches row                                      */
  uint8_t batch_id[36];                /* version-4 uuid string                                                       */
  uint32_t span;                       /* owner = spans[span].row: source_channel / _page_id / _depth, sequence_id   */
  uint32_t first_edge, n_edges;        /* its edges are edges[first_edge .. first_edge + n_edges)                     */
} tgi_state_edge_batch;
typedef struct tgi_state_edges_t {
  uint64_t n_candidates;               /* candidates before seenInBatch                                               */
  uint64_t n_edges;
  uint32_t n_batches;
  uint32_t reserved;
  const tgi_state_edge* edges;         /* [n_edges] (pinned)                                                          */
  const tgi_state_edge_batch* batches; /* [n_batches] (pinned)                                                        */
  const uint32_t* span_batch;          /* [n_spans] batch index of every span, or TGI_STATE_NO_BATCH (pinned)         */
  float kernel_ms;                     /* device time of the call's kernels and scans (not the copies between them)   */
  uint32_t gpu_launches;
} tgi_state_edges_t;
int tgi_state_pending_edges(tgi_ctx* ctx, int slot, const tgi_state_span* spans, uint32_t n_spans, int64_t now_sec,
                            tgi_state_edges_t* out);

/* Tandem hand-off SQL — the Postgres binding calls that store a hand-off: CreatePendingBatch, InsertPendingEdge and
 * ClosePendingBatch (state/daprstate.go:3896-3941), each sent by ExecuteDatabaseOperation (:3643-3678) as an `exec`
 * InvokeBinding with metadata {"sql": the text, "params": json.Marshal of its []any}.  The call renders them from the
 * device-side edges, batches and spans of the context's last successful tgi_state_pending_edges; nothing is uploaded
 * again but crawl_id and the clock.
 *   Input    the last tgi_state_pending_edges.  Any other state call since (tgi_state_*, accepted or refused) ends it;
 *            tgi_state_edge_sql and tgi_state_walkback do not, so one hand-off may be rendered many times, and the
 *            hand-off's own output and tgi_state_walkback's stay valid.  No hand-off to render is TGI_E_STATE.
 *   Order    every batch insert, then every edge insert, then every batch close: a batch row exists before its edges
 *            (pending_edges.batch_id REFERENCES pending_edge_batches) and is closed only after all of them are written
 *            (crawl/runner.go:1414-1421).  Within a kind the hand-off's order: batches in span order, edges in (span,
 *            record, link row) order, so the SERIAL pending_id comes out as with the reference's per-edge inserts.
 *   Rows     rows_per_stmt = k rows per statement for each kind, the last statement of a kind holding the rest.
 *            1 <= k <= 8191 (8 * 8191 bind parameters fit Postgres's 65535).  A statement's text depends only on its
 *            kind and row count: one row is the reference's literal, byte for byte; more rows repeat the VALUES tuple
 *            joined by ", " with the placeholders numbered on ("($1, ..., $8), ($9, ..., $16)"), and a close of more
 *            rows is "WHERE batch_id IN ($1, $2, ...)".  Statements of one (kind, rows) share one copy of the text in
 *            data.  params is one JSON array of the rows' values in order: cut into runs of 7 / 8 / 1 values it gives
 *            json.Marshal of each row's []any, exactly what k = 1 sends.
 *   Values   batch insert [batch_id, crawl_id, owner.URL, owner.ID, owner.Depth, owner.SequenceID, "open"]; edge insert
 *            [batch_id, crawl_id, destination, owner.URL, owner.SequenceID, discovery_time, source_type, "pending"]
 *            (crawl/runner.go:1276-1300; "pending" is InsertPendingEdge's literal, so a TGI_EDGE_DUPLICATE edge writes
 *            it too); batch close [batch_id].  The owner is the batch's span row as the device state holds it; strings
 *            take encoding/json's HTML-safe escaping, six characters \ufffd per invalid UTF-8 byte; Depth is a decimal int64;
 *            source_type is "mention" | "text_url" | "url" | "plaintext" (TGI_SRC_*).
 *   Clock    discovery_time = json.Marshal(time.Time) of (now_sec, now_nsec) in time.Local (tgi_set_zone, else
 *            tz_offset_sec), RFC3339Nano with trailing zeros trimmed.  The reference reads time.Now() per edge; the
 *            library reads the clock once per call, as discovery does, so every edge of a call has the same time.
 *   Cost     a thread per row sizes it, a scan places it, a thread per row writes it and each statement's entry; two
 *            launches and a scan, two synchronises.  A hand-off without batches gives 0 statements and launches nothing.
 *   Errors   every check runs before anything is written: a refused call leaves the state, the batch counter and the
 *            hand-off as they were.  TGI_E_ARG: k outside [1, 8191], now_nsec outside [0, 1e9), crawl_id NULL with a
 *            length, and when the hand-off has edges a clock whose local year leaves [0, 9999] (json.Marshal fails).
 *            TGI_E_STATE: no hand-off to render.  All of out lives in pinned memory until the next state call.        */
#define TGI_SQL_BATCH_INSERT 0     /* CreatePendingBatch                                                              */
#define TGI_SQL_EDGE_INSERT 1      /* InsertPendingEdge                                                               */
#define TGI_SQL_BATCH_CLOSE 2      /* ClosePendingBatch                                                               */
#define TGI_SQL_MAX_ROWS 8191u     /* 8 bind parameters per edge row, at most 65535 per statement                    */
typedef struct tgi_state_edge_stmt {   /* 40 bytes: one exec InvokeBinding                                            */
  uint32_t kind;                       /* TGI_SQL_*                                                                   */
  uint32_t rows;
  uint64_t sql_off, sql_len;           /* metadata "sql": data[sql_off .. sql_off + sql_len)                          */
  uint64_t params_off, params_len;     /* metadata "params": data[params_off .. params_off + params_len)             */
} tgi_state_edge_stmt;
typedef struct tgi_state_edge_sql_t {
  uint64_t n_stmts;
  const tgi_state_edge_stmt* stmts;    /* [n_stmts] in execution order (pinned)                                       */
  const uint8_t* data;                 /* the texts, then the params (pinned)                                         */
  uint64_t data_len;
  float kernel_ms;                     /* device time of the call's kernels and scan (not the copies)                 */
  uint32_t gpu_launches;
} tgi_state_edge_sql_t;
int tgi_state_edge_sql(tgi_ctx* ctx, const char* crawl_id, uint32_t crawl_id_len, int64_t now_sec, int32_t now_nsec,
                       uint32_t rows_per_stmt, tgi_state_edge_sql_t* out);

/* Tandem forced walkback — the branch of a tandem step for a page without edges (crawl/runner.go:1425-1455): pick a
 * walkback channel (pickWalkbackChannel, :115-139, exclude = nil), start a new chain at it with AddPageToPageBuffer
 * (state/daprstate.go:3619-3641) and store the step with SaveEdgeRecords of one EdgeRecord{Walkback: true}
 * (:3150-3204), each sent by ExecuteDatabaseOperation as an `exec` InvokeBinding.  The pick draws from the resident
 * TGI_SET_DISCOVERED, so a shim keeps no copy of the discovered channels.
 *   Input    the last tgi_state_pending_edges, as for tgi_state_edge_sql: every span with TGI_STATE_NO_BATCH, in span
 *            order.  tgi_state_walkback and tgi_state_edge_sql both leave the hand-off in place and have their own
 *            outputs, so either may come first and either may be called again; any other state call ends it.  No
 *            hand-off is TGI_E_STATE.
 *   Pick     the set's N keys in first-occurrence order (DiscoveredChannels.keys); key i is pool entry i without its
 *            zero padding.  Up to 10 draws: a draw equal to the owner row's URL (byte for byte, case-sensitive, as
 *            url == sourceURL) is skipped; TGI_WALK_EXHAUSTED after 10 such draws, TGI_WALK_EMPTY when N = 0 (also a
 *            set never allocated), else TGI_WALK_OK with the first usable key.  N is the set as it is at the call.
 *   Random   the w-th edge-less span the context has handled (w is not reset by tgi_state_set) draws from the 64-bit
 *            words of Philox4x32-10 blocks (w_lo, w_hi, 2, j), j = 0, 1, ... under the page-id seed: x0 | x1 << 32,
 *            then x2 | x3 << 32.  A draw is Lemire's multiply-and-reject over those words (m = x * N; when low64(m) <
 *            (2^64 - N) mod N take the next word; the index is high64(m)), exactly uniform on [0, N) as rand.Intn.
 *            The page ID and its new SequenceID are ids of the page-id construction with counter (w, 3) and (w, 4).
 *            Without tgi_state_id_seed a hand-off with an edge-less span is TGI_E_STATE.
 *   Once     the first accepted call on a hand-off makes its picks and ids and advances w; later calls on the same
 *            hand-off return the same picks and ids (with any clock or rows_per_stmt), so a retried render cannot
 *            start a second walkback page for a span.
 *   Rows     each TGI_WALK_OK span gives a page_buffer row [ID, owner.ID, owner.Depth + 1, url, crawl_id, SequenceID]
 *            and an edge_records row [url, owner.URL, true, false, discovery_time, crawl_id, owner.SequenceID]; the
 *            records' empty CrawlID falls back to the configured one, so crawl_id is the call's.  Depth + 1 is a
 *            decimal int64 and wraps as Go's int.  Strings, the clock and the year check are tgi_state_edge_sql's.
 *   Order    every page_buffer insert (TGI_SQL_PAGE_BUFFER_INSERT), then every edge_records insert
 *            (TGI_SQL_EDGE_RECORD_INSERT), rows_per_stmt = k rows per statement by tgi_state_edge_sql's rule: k = 1
 *            gives the reference's literals and json.Marshal of each []any byte for byte.
 *   Cost     a thread per edge-less span picks, a scan ranks the usable ones, a thread per row sizes it, a scan, a
 *            thread per row writes it and the statement table.  A hand-off without edge-less spans launches nothing.
 *   Errors   every check runs before anything changes: a refused call leaves the state, w and the hand-off as they
 *            were.  TGI_E_ARG: k outside [1, 8191], now_nsec outside [0, 1e9), crawl_id NULL with a length, and when
 *            there is a row a clock whose local year leaves [0, 9999].  TGI_E_STATE: no hand-off, no seed.  All of out
 *            lives in pinned memory until the next state call.                                                      */
#define TGI_SQL_PAGE_BUFFER_INSERT 3  /* AddPageToPageBuffer                                                          */
#define TGI_SQL_EDGE_RECORD_INSERT 4  /* SaveEdgeRecords, one record                                                  */
#define TGI_WALK_OK 0                 /* a walkback channel was picked                                                */
#define TGI_WALK_EXHAUSTED 1          /* 10 draws, all the owner's URL (ErrWalkbackExhausted)                         */
#define TGI_WALK_EMPTY 2              /* no discovered channel to pull from                                           */
#define TGI_WALK_MAX_DRAWS 10         /* maxWalkbackAttempts                                                          */
typedef struct tgi_state_walkback_span { /* 120 bytes: one edge-less span                                             */
  uint32_t span;                       /* its index in the hand-off's spans                                           */
  uint32_t status;                     /* TGI_WALK_*                                                                  */
  uint32_t draws;                      /* draws made, 0 for TGI_WALK_EMPTY                                            */
  uint32_t url_len;
  uint8_t url[32];                     /* the walkback channel (TGI_WALK_OK), zero padded                            */
  uint8_t page_id[36];                 /* the new page's ID                                                           */
  uint8_t sequence_id[36];             /* its SequenceID: the new chain                                               */
} tgi_state_walkback_span;
typedef struct tgi_state_walkback_t {
  uint32_t n_walkbacks;                /* the hand-off's edge-less spans                                              */
  uint32_t reserved;
  const tgi_state_walkback_span* walkbacks; /* [n_walkbacks] in span order (pinned)                                   */
  uint64_t n_stmts;
  const tgi_state_edge_stmt* stmts;    /* [n_stmts] in execution order (pinned)                                       */
  const uint8_t* data;                 /* the texts, then the params (pinned)                                         */
  uint64_t data_len;
  float kernel_ms;                     /* device time of the call's kernels and scans (not the copies)               */
  uint32_t gpu_launches;
} tgi_state_walkback_t;
int tgi_state_walkback(tgi_ctx* ctx, const char* crawl_id, uint32_t crawl_id_len, int64_t now_sec, int32_t now_nsec,
                       uint32_t rows_per_stmt, tgi_state_walkback_t* out);

/* Validator walkback — the validator pod's walkback processor (crawl/validator.go:314-489) for n claimed batches in one
 * call: processWalkbackBatch's decision, its forward or walkback pick (pickWalkbackChannel, crawl/runner.go:115-139,
 * with the batch's valid channels excluded), AddPageToPageBuffer (state/daprstate.go:3619-3641), SaveEdgeRecords of
 * the primary and skipped edges (:3150-3204), CompletePendingBatch and FlushBatchStats (:4124-4206), each sent by
 * ExecuteDatabaseOperation as an `exec` InvokeBinding.  The walkback pick draws from the resident TGI_SET_DISCOVERED.
 *   Input    what ClaimWalkbackBatch (:4016-4122) returns, per batch: tgi_claimed_batch (its five strings as (offset,
 *            length) pairs into strs, source_depth) and its edges edges[edge_off[i] .. edge_off[i+1]) in the order the
 *            database returned them, each with its destination, its source_type and its validation_status mapped to a
 *            TGI_EDGE_CLASS_* by exact match ("valid", "not_channel", "invalid", "duplicate", anything else OTHER).
 *            Nothing is read from a crawler hand-off.  It is a state call, so it ends a live tgi_state_pending_edges
 *            hand-off (a following tgi_state_edge_sql or tgi_state_walkback is TGI_E_STATE).
 *   Decide   per batch, in input order: validFirstClaimed = the destinations of its VALID edges, in edge order.  None:
 *            walk back, rnd = -1.  Else rnd = IntN(100) + 1 and the batch walks back iff walkback_rate >= rnd.
 *   Pick     walkback: pickWalkbackChannel(source_channel, exclude = validFirstClaimed) over the set's N keys in
 *            first-occurrence order, as tgi_state_walkback's pick: up to 10 draws, a draw equal (byte for byte) to the
 *            source channel or to any excluded name is retried; TGI_WALK_OK, TGI_WALK_EXHAUSTED after 10 such draws,
 *            TGI_WALK_EMPTY when N = 0.  The page's SequenceID is a new id, the primary edge's the batch's.  Forward:
 *            idx = IntN(n_valid); the page URL is that destination, which leaves the skipped list (order kept); the page
 *            and the primary edge take the batch's SequenceID.  A batch whose pick fails writes nothing (the reference
 *            returns the error before its first write) and keeps its result, so the shim can log it and leave the batch
 *            claimed.
 *   Random   the v-th batch the context handles (v is not reset by tgi_state_set, and tgi_state_walkback's counter is
 *            separate) draws from the 64-bit words of Philox4x32-10 blocks (v_lo, v_hi, 5, j) under the page-id seed:
 *            x0 | x1 << 32, then x2 | x3 << 32.  rnd, the forward index and the walkback draws are Lemire's
 *            multiply-and-reject over that one stream, in that order.  The page ID and the new SequenceID are ids of the
 *            page-id construction with counter (v, 6) and (v, 7).  v advances by n on an accepted call only.  Without
 *            tgi_state_id_seed a call with batches is TGI_E_STATE.
 *   Rows     per TGI_WALK_OK batch: page_buffer [ID, source_page_id, source_depth + 1, url, crawl_id, page SequenceID];
 *            edge_records primary [url, source_channel, walkback, false, discovery_time, crawl_id, batch SequenceID],
 *            then one skipped row [ch, source_channel, false, true, discovery_time, crawl_id, batch SequenceID] per
 *            remaining valid channel; complete [batch_id]; one stats upsert [batch crawl_id, st, total, valid,
 *            not_channel, invalid, duplicate] per distinct source_type of all its edges (empty is "unknown"), in
 *            first-occurrence order; delete [batch_id].  crawl_id of the page and edge rows is the batch's, or the call's
 *            when the batch's is empty; the stats rows take the batch's as it is (FlushBatchStats has no fallback).
 *            source_depth + 1 wraps as Go's int.  OTHER counts in total only.  Strings, the clock and the year check
 *            are tgi_state_edge_sql's; the clock is read once per call.
 *   Order    every page_buffer insert (TGI_SQL_PAGE_BUFFER_INSERT), every edge_records insert (per batch: primary, then
 *            skipped), every complete (TGI_SQL_BATCH_COMPLETE), every upsert (TGI_SQL_STATS_UPSERT), every delete
 *            (TGI_SQL_EDGES_DELETE), each kind in batch order: a batch's page, edges, complete, stats and delete keep the
 *            reference's order.  rows_per_stmt = k rows per statement by tgi_state_edge_sql's rule for every kind but
 *            the upserts; complete and delete of more rows are "WHERE batch_id IN ($1, ...)".  A stats upsert is always
 *            one row per statement: rows of two batches of one crawl share the key (crawl_id, source_type), and Postgres
 *            refuses an ON CONFLICT DO UPDATE that touches one row twice.  k = 1 gives the reference's calls.
 *   Cost     a thread per batch decides, picks, lists its valid edges and its distinct source types (a compare against
 *            each type found so far, so m edges of d types cost m * d compares) and counts its rows; three scans place
 *            them; a thread per row sizes it, a scan, a thread per row writes it and the statement table.  A stats row
 *            counts its type over the batch's edges.  Three synchronises.  n = 0 launches nothing.
 *   Errors   every check runs before anything changes: a refused call makes nothing and leaves v as it was.  TGI_E_ARG:
 *            k outside [1, 8191], now_nsec outside [0, 1e9), crawl_id NULL with a length, a NULL array with a count,
 *            edge_off[0] != 0, edge_off decreasing or edge_off[n] != n_edges, a batch of 2^32 - 1 edges or more, a
 *            string outside strs, a class code past OTHER, and when there is a row a clock whose local year leaves
 *            [0, 9999].  TGI_E_STATE: no seed.  TGI_E_CAPACITY: a row of 4 GiB or more.  All of out lives in pinned
 *            memory until the next state call.                                                                       */
#define TGI_SQL_BATCH_COMPLETE 5      /* CompletePendingBatch                                                         */
#define TGI_SQL_STATS_UPSERT 6        /* FlushBatchStats: one source_type's upsert                                    */
#define TGI_SQL_EDGES_DELETE 7        /* FlushBatchStats: the batch's pending_edges                                   */
#define TGI_EDGE_CLASS_VALID 0        /* validation_status "valid"                                                    */
#define TGI_EDGE_CLASS_NOT_CHANNEL 1  /* "not_channel"                                                                */
#define TGI_EDGE_CLASS_INVALID 2      /* "invalid"                                                                    */
#define TGI_EDGE_CLASS_DUPLICATE 3    /* "duplicate"                                                                  */
#define TGI_EDGE_CLASS_OTHER 4        /* anything else: counted in total only                                         */
#define TGI_CB_BATCH_ID 0             /* tgi_claimed_batch strings                                                    */
#define TGI_CB_CRAWL_ID 1
#define TGI_CB_SOURCE_CHANNEL 2
#define TGI_CB_SOURCE_PAGE_ID 3
#define TGI_CB_SEQUENCE_ID 4
#define TGI_CE_DESTINATION 0          /* tgi_claimed_edge strings                                                     */
#define TGI_CE_SOURCE_TYPE 1
#define TGI_VW_NO_EDGE 0xFFFFFFFFu    /* tgi_state_validator_batch.forward_edge of a walkback                         */
typedef struct tgi_claimed_batch {    /* 72 bytes: one PendingEdgeBatch                                               */
  uint64_t str_off[5];                /* TGI_CB_*: strs[str_off[f] .. + str_len[f])                                   */
  uint32_t str_len[5];
  uint32_t reserved;
  int64_t source_depth;
} tgi_claimed_batch;
typedef struct tgi_claimed_edge {     /* 32 bytes: one PendingEdge                                                    */
  uint64_t str_off[2];                /* TGI_CE_*                                                                     */
  uint32_t str_len[2];
  uint32_t cls;                       /* TGI_EDGE_CLASS_*                                                             */
  uint32_t reserved;
} tgi_claimed_edge;
typedef struct tgi_claimed_batches {
  uint32_t n_batches;
  uint32_t reserved;
  const tgi_claimed_batch* batches;   /* [n_batches]                                                                  */
  const uint64_t* edge_off;           /* [n_batches+1]: batch i's edges are edges[edge_off[i] .. edge_off[i+1])       */
  const tgi_claimed_edge* edges;      /* [n_edges]                                                                    */
  uint64_t n_edges;
  const uint8_t* strs;                /* every string of the batches and edges                                        */
  uint64_t strs_len;
} tgi_claimed_batches;
typedef struct tgi_state_validator_batch { /* 136 bytes: one batch's outcome                                          */
  uint32_t status;                    /* TGI_WALK_* (a forward batch is TGI_WALK_OK)                                  */
  uint32_t walkback;                  /* 1: walked back                                                               */
  int32_t rnd;                        /* IntN(100) + 1, or -1 without a valid edge                                    */
  uint32_t draws;                     /* walkback draws made                                                          */
  uint32_t n_valid;                   /* len(validFirstClaimed)                                                       */
  uint32_t forward_edge;              /* the followed edge's index within the batch, or TGI_VW_NO_EDGE                */
  uint32_t url_len;
  uint32_t reserved;
  uint8_t url[32];                    /* the walkback channel (TGI_WALK_OK walkback), zero padded                     */
  uint8_t page_id[36];                /* the new page's ID                                                            */
  uint8_t sequence_id[36];            /* the new chain's SequenceID, which the page takes when it walks back          */
} tgi_state_validator_batch;
typedef struct tgi_state_validator_walkback_t {
  uint32_t n_batches;
  uint32_t reserved;
  const tgi_state_validator_batch* batches; /* [n_batches] in input order (pinned)                                    */
  uint64_t n_stmts;
  const tgi_state_edge_stmt* stmts;   /* [n_stmts] in execution order (pinned)                                        */
  const uint8_t* data;                /* the texts, then the params (pinned)                                          */
  uint64_t data_len;
  float kernel_ms;                    /* device time of the call's kernels and scans (not the copies)                */
  uint32_t gpu_launches;
} tgi_state_validator_walkback_t;
int tgi_state_validator_walkback(tgi_ctx* ctx, const tgi_claimed_batches* in, int64_t walkback_rate, const char* crawl_id,
                                 uint32_t crawl_id_len, int64_t now_sec, int32_t now_nsec, uint32_t rows_per_stmt,
                                 tgi_state_validator_walkback_t* out);

/* Standard random walk — the random-walk branch of processAllMessagesWithProcessor without TandemCrawl
 * (crawl/runner.go:1218-1227, 1245-1384, 1458-1540) for many pages in two calls: tgi_state_rw_lookups lists the
 * SearchPublicChat calls the pages make; the caller makes them; tgi_state_rw_step applies their outcomes to the three
 * resident sets, makes every page's walkback decision and pick, and renders the binding calls.  Only the RPC stays with
 * the caller.
 *   Spans    as tgi_state_pending_edges's: the owner row, its records of the slot's last result (run with
 *            TGI_RUN_LINKS), the first n_done processed.  Spans may share records.  They are replayed as if they ran one
 *            after another in span order (Go runs pages on concurrent goroutines: this is one valid serialisation).
 *   Candidates  every link row of a processed record with status TGI_ST_EMITTED or TGI_ST_NOLINE, except names
 *            byte-equal to the owner row's URL (`o == owner.URL`), in (span, record, link row) order.  No FilterUsername.
 *   Classes  a name's candidates depend only on its own history.  Its first candidate of the call is skipped when the
 *            name is in TGI_SET_INVALID live at now_sec (IsInvalidChannel) or in TGI_SET_DISCOVERED
 *            (IsDiscoveredChannel); else it is a seed hit when TGI_SET_SEEDS holds it (GetCachedChatID: Dapr's
 *            chatIDCache, seeded by the shim from LoadSeedChannels), which only adds it to the discovered set; else it
 *            is a lookup.  Every later candidate of the name is skipped: after a seed hit or a found lookup the name is
 *            discovered, after a failed one it is invalid, and a retiring one ends the replay.
 *   Lookups  tgi_state_rw_lookups: one row per lookup in candidate order, with the name, its span, its record and its
 *            source_type (msgSourceMap's value: the link row's source), and every span's candidate count.  It changes
 *            nothing, not even a counter.  Its lists stay on the device for tgi_state_rw_step; any other state call
 *            ends them, and so does an accepted tgi_state_rw_step.  The classes use the sets as they are at this call.
 *   Outcomes one per lookup row: TGI_RW_FOUND (a chatTypeSupergroup, with its chat id), TGI_RW_NOT_SUPERGROUP,
 *            TGI_RW_NOT_FOUND (any non-flood search error), TGI_RW_RETIRE (a FLOOD_WAIT at or above the retire
 *            threshold).  The caller sleeps and retries short FLOOD_WAITs itself and reports the final outcome.
 *   Replay   tgi_state_rw_step, in span order: a seed hit does AddDiscoveredChannel; FOUND does AddDiscoveredChannel,
 *            adds the name to the span's newChannels, emits a seed_channels upsert [name, chat_id] and inserts the name
 *            into TGI_SET_SEEDS (UpsertSeedChannelChatID fills chatIDCache too); NOT_FOUND / NOT_SUPERGROUP emit an
 *            invalid_channels upsert [name, "not_found" | "not_supergroup"] and stamp the name into TGI_SET_INVALID at
 *            now_sec (MarkChannelInvalid: a stamp that expired is replaced).  The first RETIRE ends its span: the
 *            effects of the span's earlier candidates stand, the span is TGI_RW_RETIRED and writes no page or edge rows.
 *            Every later span is TGI_RW_DEFERRED: no change and no rows, for the caller to submit again; the outcomes
 *            of its lookups are not used.  The sets' inserts keep candidate order, so TGI_SET_DISCOVERED's
 *            first-occurrence order is the replay's.
 *   Decide   per span that is neither (runner.go:1458-1504): newChannels in first-occurrence order, n_new of them.  With
 *            n_new = 0 it walks back and rnd = -1; else rnd = IntN(100) + 1 and it walks back iff walkback_rate >= rnd.
 *            Walkback: pickWalkbackChannel(owner.URL, exclude = newChannels) over the first N_s keys of
 *            TGI_SET_DISCOVERED, N_s = the set as the replay leaves it after this span's candidates (earlier spans'
 *            inserts and its own included), with tgi_state_walkback's rule (10 draws; TGI_WALK_EXHAUSTED,
 *            TGI_WALK_EMPTY); the page takes a new SequenceID.  Forward: idx = IntN(n_new), the page URL is
 *            newChannels[idx], which leaves the list (order kept); the page takes owner.SequenceID.
 *   Random   the u-th deciding span under the context (u is not reset by tgi_state_set, and no other call shares its
 *            counter) draws rnd, the forward index and the walkback draws, in that order, by Lemire's rule from the
 *            64-bit words of Philox4x32-10 blocks (u_lo, u_hi, 8, j) under the page-id seed.  The page ID and the new
 *            SequenceID are ids of the page-id construction with counter (u, 9) and (u, 10).  u advances by the
 *            deciding spans of an accepted call.  Without tgi_state_id_seed a call with a deciding span is TGI_E_STATE.
 *   Rows     per span: its upserts in candidate order; then, when its pick is TGI_WALK_OK, page_buffer [ID, owner.ID,
 *            owner.Depth + 1, url, crawl_id, SequenceID] and edge_records: the primary [url, owner.URL, walkback, false,
 *            discovery_time, crawl_id, owner.SequenceID], then [ch, owner.URL, false, true, discovery_time, crawl_id,
 *            owner.SequenceID] per remaining new channel in order.  A span whose pick fails keeps its upserts and set
 *            changes and writes no page or edge rows (Go returns the error after those effects).  The page and its edges
 *            leave CrawlID empty, so crawl_id is the call's.  Strings, Depth + 1, the clock and the year check are
 *            tgi_state_walkback's.
 *   Order    every seed_channels upsert (TGI_SQL_SEED_UPSERT), every invalid_channels upsert (TGI_SQL_INVALID_UPSERT),
 *            every page_buffer insert, every edge_records insert, each kind in candidate / span order, rows_per_stmt =
 *            k rows per statement by tgi_state_edge_sql's rule for every kind (the upserts' names are distinct within a
 *            call, so no ON CONFLICT touches a row twice): "VALUES ($1, $2), ($3, $4) ON CONFLICT ...", an invalid
 *            tuple "($1, $2, NOW())".  k = 1 gives the reference's calls byte for byte.
 *   Stats    per TGI_SRC_* the hits (FOUND) and misses (NOT_FOUND, NOT_SUPERGROUP) of the applied lookups:
 *            lookupStats' counts, for the shim's log lines.
 *   Cost     lookups: the discovery gather, one first-occurrence table over the call, a thread per candidate classifies
 *            it, a scan, a thread per lookup writes its row; one synchronise for the totals, one for the read-back.
 *            step: a thread per lookup and candidate flags the effects, three scans, one compaction (one synchronise);
 *            the three ordered set inserts; a thread per span decides and picks, two scans (one synchronise); then the
 *            rows as tgi_state_edge_sql renders them.
 *   Errors   every check runs before anything changes: a refused call leaves the sets, u and the lists as they were.
 *            lookups: TGI_E_ARG for an unknown row, a span outside the result, n_done > n_records; TGI_E_STATE for no,
 *            a released or a non-Telegram result, a result run without TGI_RUN_LINKS, a job in flight on the slot.
 *            step: TGI_E_ARG for k outside [1, 8191], now_nsec outside [0, 1e9), crawl_id NULL with a length,
 *            outcomes NULL with lookups, n_outcomes other than the lookups' count, an unknown outcome code, and when a
 *            span decides a clock whose local year leaves [0, 9999]; TGI_E_STATE for no lists or no seed.  After
 *            TGI_E_CAPACITY (a set past its capacity or growth limit: each set's insert is all or nothing) or
 *            TGI_E_CUDA the sets inserted before may hold their keys.  Lock order: the slot, then the state, then the
 *            sets.  All of out lives in pinned memory until the next state call.                                      */
#define TGI_SET_SEEDS 5                /* Dapr's chatIDCache (daprstate.go:3375-3411): seeded with tgi_set_add      */
#define TGI_RW_FOUND 0                 /* SearchPublicChat found a chatTypeSupergroup                                 */
#define TGI_RW_NOT_SUPERGROUP 1        /* found, another chat type                                                    */
#define TGI_RW_NOT_FOUND 2             /* any non-flood search error                                                  */
#define TGI_RW_RETIRE 3                /* FLOOD_WAIT at or above floodWaitRetireThresholdSecs                         */
#define TGI_RW_RETIRED 3               /* tgi_rw_span.status past TGI_WALK_*: the span met the retiring lookup        */
#define TGI_RW_DEFERRED 4              /* a span after it: submit it again                                           */
#define TGI_RW_NO_FORWARD 0xFFFFFFFFu  /* tgi_rw_span.forward of a walkback                                           */
#define TGI_SQL_SEED_UPSERT 8          /* UpsertSeedChannelChatID                                                    */
#define TGI_SQL_INVALID_UPSERT 9       /* MarkChannelInvalid                                                          */
typedef struct tgi_rw_lookup {         /* 48 bytes: one SearchPublicChat call                                         */
  uint8_t name[32];                    /* the username, zero padded                                                   */
  uint64_t record;                     /* the result record of the candidate                                          */
  uint32_t span;
  uint8_t name_len;
  uint8_t source_type;                 /* TGI_SRC_*                                                                   */
  uint16_t reserved;
} tgi_rw_lookup;
typedef struct tgi_rw_outcome {        /* 16 bytes                                                                    */
  int64_t chat_id;                     /* TGI_RW_FOUND: chat.Id                                                       */
  uint32_t code;                       /* TGI_RW_*                                                                    */
  uint32_t reserved;
} tgi_rw_outcome;
typedef struct tgi_state_rw_lookups_t {
  uint64_t n_candidates;
  uint64_t n_lookups;
  const tgi_rw_lookup* lookups;        /* [n_lookups] in candidate order (pinned)                                     */
  const uint64_t* span_candidates;     /* [n_spans] (pinned)                                                          */
  float kernel_ms;                     /* device time of the call's kernels and scans (not the copies)               */
  uint32_t gpu_launches;
} tgi_state_rw_lookups_t;
typedef struct tgi_rw_span {           /* 136 bytes: one page's step                                                  */
  uint32_t status;                     /* TGI_WALK_* (a forward pick is TGI_WALK_OK), TGI_RW_RETIRED, TGI_RW_DEFERRED */
  uint32_t walkback;                   /* 1: walked back                                                              */
  int32_t rnd;                         /* IntN(100) + 1, or -1 without new channels                                   */
  uint32_t draws;                      /* walkback draws made                                                         */
  uint32_t n_new;                      /* len(newChannels)                                                            */
  uint32_t forward;                    /* the followed channel's index in newChannels, or TGI_RW_NO_FORWARD           */
  uint32_t url_len;
  uint32_t reserved;
  uint8_t url[32];                     /* the next page's URL (TGI_WALK_OK), zero padded                              */
  uint8_t page_id[36];                 /* the next page's ID                                                          */
  uint8_t sequence_id[36];             /* the new chain's SequenceID, which the page takes when it walks back         */
} tgi_rw_span;
typedef struct tgi_state_rw_step_t {
  uint32_t n_spans;
  uint32_t reserved;
  const tgi_rw_span* spans;            /* [n_spans] (pinned)                                                          */
  uint64_t hits[4], misses[4];         /* per TGI_SRC_*                                                               */
  uint64_t n_stmts;
  const tgi_state_edge_stmt* stmts;    /* [n_stmts] in execution order (pinned)                                       */
  const uint8_t* data;                 /* the texts, then the params (pinned)                                         */
  uint64_t data_len;
  float kernel_ms;                     /* device time of the call's kernels and scans (not the copies)               */
  uint32_t gpu_launches;
} tgi_state_rw_step_t;
int tgi_state_rw_lookups(tgi_ctx* ctx, int slot, const tgi_state_span* spans, uint32_t n_spans, int64_t now_sec,
                         tgi_state_rw_lookups_t* out);
int tgi_state_rw_step(tgi_ctx* ctx, const tgi_rw_outcome* outcomes, uint64_t n_outcomes, int64_t walkback_rate,
                      const char* crawl_id, uint32_t crawl_id_len, int64_t now_sec, int32_t now_nsec,
                      uint32_t rows_per_stmt, tgi_state_rw_step_t* out);
/* tgi_set_export: the first min(count, cap) keys of a caller-filled set (TGI_SET_INVALID, _DISCOVERED, _URLS, _SEEDS)
 * in first-occurrence order, and with stamps_sec (TGI_SET_INVALID only) their stamps; *n = the set's count. */
int tgi_set_export(tgi_ctx* ctx, int which, uint8_t* keys32, int64_t* stamps_sec, uint64_t cap, uint64_t* n);

/* Layer reads — the reads that begin every depth of both runners (standalone/runner.go:594-700,
 * dapr/standalone.go:948-1021 and 454-498) and FindIncompleteCrawl's page test, by row, so a shim that runs discovery on
 * the device never holds a copy of the page table: layer read, tgi_state_pages_begin of the selected rows, one bulk
 * batch, tgi_state_pages_end, tgi_state_discover, tgi_state_pages_close, tgi_state_next_layer, next layer read.
 *   Pages    tgi_state_read_pages = GetPage(id) (base.go:110-120) of rows[0 .. n) in one call.  out->pages[k] is row
 *            out->rows[k] = rows[k]'s record as stored, its strings at out->strs + pages[k].str_off (a TGI_STATE_TS_LOCAL timestamp
 *            stays TGI_STATE_TS_LOCAL).  TGI_READ_MESSAGES: page k's list is msgs[msg_first[k] .. msg_first[k] +
 *            pages[k].n_msgs), the row's live messages in list order, page_id as tgi_state_read_page gives it; a row
 *            requested twice is returned twice and its list may be stored once, so msg_first need not increase.
 *            Without the flag n_msgs is 0, msgs and msg_first are NULL and nothing is launched.
 *   Layer    tgi_state_read_layer = GetLayerByDepth(depth) (base.go:325-342): the rows of the layer in list order, as
 *            tgi_state_read_pages returns them, out->rows naming them; a row the layer lists twice is returned twice.  A depth without a
 *            layer gives 0 pages, as Base returns [].  DaprStateManager's override (daprstate.go:3014-3074) differs only
 *            when a listed id is missing from pageMap, which a row of the device state never is.  select fills
 *            out->select[k] (1: the runner processes page k) and out->n_selected:
 *            TGI_SELECT_NONE   nothing (select NULL).
 *            TGI_SELECT_STANDALONE  a new execution: every page (standalone/runner.go:636-694).
 *            TGI_SELECT_STANDALONE_RESUME  the same execution resumed: every page whose status is not "fetched" (the
 *                              startIndex scan and the in-loop skip together).
 *            TGI_SELECT_DAPR   processLayerInParallel (dapr/standalone.go:454-498, which always resumes: :420): the first
 *                              page of every URL, byte for byte, and only if its status is neither "fetched" nor
 *                              "error".  The URL is recorded before the status test, so a fetched first page hides a
 *                              later unfetched page with the same URL.
 *            The selected rows go to tgi_state_pages_begin as they are.
 *   Layers   tgi_state_layers: every layer's depth and listed pages in ascending depth; GetMaxDepth (base.go:446-462):
 *            max_depth = the largest depth above -1, has_max_depth = 0 when there is none (its "no layers found": a
 *            state whose layers all lie at depth -1 or below has none); n_incomplete = the listed pages whose status is
 *            not "fetched", a row listed twice counted twice (FindIncompleteCrawl's in-memory test, base.go:482-502, is
 *            n_incomplete > 0).  Host mirror only: nothing is launched.
 *   Cost     with TGI_READ_MESSAGES, one pass over the message rows per call whatever n: flags of the live messages of
 *            the distinct rows, a scan, the render's stable radix passes (their number set by the state's row count),
 *            the rows' counts and their scan, one gather.  The launches do not depend on n; two synchronises (the
 *            lists' lengths, then the lists).  tgi_state_read_page is its n = 1 case.
 *   Errors   TGI_E_ARG, the state unchanged: an unknown row, unknown flags or selection, rows NULL with n > 0.  The
 *            state lock only (no slot is read).  All of out lives in pinned memory until the next state call.       */
#define TGI_READ_MESSAGES 1u
#define TGI_SELECT_NONE 0
#define TGI_SELECT_STANDALONE 1
#define TGI_SELECT_STANDALONE_RESUME 2
#define TGI_SELECT_DAPR 3
typedef struct tgi_state_read_t {
  uint64_t n_pages;
  const uint32_t* rows;          /* [n_pages] each page's row (pinned)                                               */
  const tgi_state_page* pages;   /* [n_pages] the rows' records; str_off into strs, n_msgs = the list's length (pinned) */
  const uint8_t* strs;           /* the pages' strings (pinned)                                                     */
  uint64_t strs_len;
  const tgi_state_msg* msgs;     /* [n_msgs] with TGI_READ_MESSAGES: the distinct rows' lists (pinned), else NULL   */
  const uint64_t* msg_first;     /* [n_pages] page k's list starts at msgs[msg_first[k]] (pinned), else NULL        */
  uint64_t n_msgs;
  const uint8_t* select;         /* [n_pages] tgi_state_read_layer with a selection: 1 = processed (pinned), else NULL */
  uint64_t n_selected;
  float kernel_ms;               /* device time of the call's kernels and scans (not the copies)                   */
  uint32_t gpu_launches;
} tgi_state_read_t;
typedef struct tgi_state_layers_t {
  uint64_t n_layers;
  const int64_t* depth;          /* [n_layers] ascending (pinned)                                                   */
  const uint64_t* n_pages;       /* [n_layers] the ids each layer lists (pinned)                                     */
  int64_t max_depth;             /* GetMaxDepth: the largest depth above -1, else -1                                 */
  uint32_t has_max_depth;        /* 0: GetMaxDepth's "no layers found"                                               */
  uint32_t reserved;
  uint64_t n_incomplete;         /* listed pages whose status is not "fetched"                                       */
} tgi_state_layers_t;
int tgi_state_read_pages(tgi_ctx* ctx, const uint32_t* rows, uint64_t n, uint32_t flags, tgi_state_read_t* out);
int tgi_state_read_layer(tgi_ctx* ctx, int64_t depth, int select, uint32_t flags, tgi_state_read_t* out);
int tgi_state_layers(tgi_ctx* ctx, tgi_state_layers_t* out);

/* pure helpers exposed for host code and tests (each runs the device code path on tiny inputs) */
int tgi_filter_usernames(tgi_ctx* ctx, const uint8_t* names, const uint32_t* off, uint64_t n,
                         uint8_t* reason);

#ifdef __cplusplus
}
#endif
#endif /* TGINGEST_H */
