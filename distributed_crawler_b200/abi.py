"""ctypes / numpy mirror of include/tgingest.h (the C ABI of libtgingest).

Field order and widths are ABI; tests/test_abi.py checks every sizeof against the header by
compiling a probe with gcc.  No torch types appear here: buffers are numpy arrays (host) whose
pointers are handed to C.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

ABI_VERSION = 2

# error codes
OK, E_ARG, E_CUDA, E_NOMEM, E_CAPACITY, E_NODEVICE, E_STATE = 0, -1, -2, -3, -4, -5, -6
# per-record status
ST_EMITTED, ST_SKIPPED, ST_FAILED, ST_NOLINE = 0, 1, 2, 3

# content types (order is ABI)
CT_NAMES = [
    "none", "messageText", "messageVideo", "messagePhoto", "messageAnimation",
    "messageAnimatedEmoji", "messagePoll", "messageGiveaway", "messagePaidMedia", "messageSticker",
    "messageGiveawayWinners", "messageGiveawayCompleted", "messageVideoNote", "messageDocument",
    "messageAudio", "messageVoiceNote", "other",
]
CT = {n: i for i, n in enumerate(CT_NAMES)}
CT_LINK_CARRIERS = {CT[k] for k in ("messageText", "messagePhoto", "messageVideo", "messageDocument",
                                    "messageAnimation", "messageAudio", "messageVoiceNote")}

RF_HAS_TEXT, RF_COMMENTS_NIL, RF_PANIC = 1, 2, 4
ENT_OTHER, ENT_TEXT_URL, ENT_MENTION, ENT_URL = 0, 1, 2, 3
SRC_NAMES = ["mention", "text_url", "url", "plaintext"]
FU_REASONS = ["", "too_short", "too_long", "invalid_start_char", "ends_with_underscore",
              "invalid_char", "looks_like_path", "bot_suffix"]

CFG_HAS_MIN_POST_DATE, CFG_SKIP_MEDIA = 1, 2
RUN_JSONL, RUN_LINKS, RUN_FRONTIER, RUN_FILTER, RUN_SKIP_SELF, RUN_NO_D2H = 1, 2, 4, 8, 16, 32
LF_FILTER_OK, LF_NEW, LF_SELF = 1, 2, 4
SLOTS = 3
ZONE_MAX = 4096  # entries of a tgi_set_zone table
YT_THUMB_ABSENT = 0xFFFF
YT_THUMB_KEYS = ["default", "medium", "high", "standard", "maxres"]

# ---- numpy record dtypes (array element layouts) ---------------------------------------------
TG_REC = np.dtype([
    ("id", "<i8"), ("chat_id", "<i8"), ("media_album_id", "<i8"), ("str_off", "<u8"),
    ("date", "<i4"), ("view_count", "<i4"), ("share_count", "<i4"), ("chan_idx", "<u4"),
    ("text_len", "<u4"), ("alt_len", "<u4"), ("media_len", "<u2"), ("handle_len", "<u2"),
    ("content_type", "u1"), ("flags", "u1"), ("reserved", "<u2")])
ENTITY = np.dtype([("offset", "<i4"), ("length", "<i4"), ("url_off", "<u4"), ("url_len", "<u2"),
                   ("type", "u1"), ("reserved", "u1")])
REACTION = np.dtype([("emoji_off", "<u4"), ("emoji_len", "<u2"), ("reserved", "<u2"),
                     ("count", "<i4")])
COMMENT = np.dtype([("text_off", "<u4"), ("text_len", "<u4"), ("handle_off", "<u4"),
                    ("handle_len", "<u2"), ("flags", "u1"), ("reserved", "u1"),
                    ("view_count", "<i4"), ("reply_count", "<i4"), ("react_start", "<u4"),
                    ("react_count", "<u4")])
TG_CHAN = np.dtype([("str_off", "<u4"), ("title_len", "<u2"), ("name_len", "<u2"),
                    ("user_len", "<u2"), ("reserved", "<u2"), ("reserved2", "<u4"),
                    ("member_count", "<i8"), ("post_count", "<i8"), ("view_count", "<i8")])
YT_REC = np.dtype([
    ("str_off", "<u8"), ("published_sec", "<i8"), ("view_count", "<i8"), ("like_count", "<i8"),
    ("comment_count", "<i8"), ("desc_len", "<u4"), ("chan_idx", "<u4"), ("id_len", "<u2"),
    ("title_len", "<u2"), ("duration_len", "<u2"), ("lang_len", "<u2"), ("thumb_len", "<u2", (5,)),
    ("reserved", "<u2"), ("published_nsec", "<i4"), ("reserved2", "<u8")])
YT_CHAN = np.dtype([
    ("str_off", "<u4"), ("id_len", "<u2"), ("title_len", "<u2"), ("desc_len", "<u4"),
    ("thumb_len", "<u2"), ("country_len", "<u2"), ("subscriber_count", "<i8"), ("view_count", "<i8"),
    ("video_count", "<i8"), ("published_sec", "<i8"), ("published_nsec", "<i4"), ("cached", "u1"),
    ("reserved", "u1", (11,))])
LINK = np.dtype([("name", "u1", (32,)), ("len", "u1"), ("src", "u1"), ("flags", "u1"),
                 ("filter_reason", "u1")])
EDGE = np.dtype([("destination", "u1", (32,)), ("record", "<u8"), ("chan_idx", "<u4"), ("dest_len", "u1"), ("source_type", "u1"),
                 ("status", "u1"), ("reserved", "u1")])  # tgi_edge
assert EDGE.itemsize == 48
APPEND_RUN = np.dtype([("chan_idx", "<u4"), ("n_lines", "<u4"), ("first", "<u8"), ("end", "<u8"), ("byte_begin", "<u8"),
                       ("byte_end", "<u8")])  # tgi_append_run
assert APPEND_RUN.itemsize == 40
SET_FRONTIER, SET_INVALID, SET_DISCOVERED, SET_OWNED = 0, 1, 2, 3  # tgi_set_info / tgi_set_add
SET_URLS = 4  # Dapr's urlCache (tgi_state_discover): seeded with tgi_set_add
EDGE_PENDING, EDGE_DUPLICATE, EDGE_INVALID_CACHED = 0, 1, 2
ROWS_STATUS, ROWS_LINK_OFF, ROWS_LINKS = 0, 1, 2  # tgi_result_read_rows
RUN_SKIP_INVALID = 0x40
RUN_JSONL_DEVICE = 0x80  # with RUN_JSONL: the lines stay on the device (tgi_result.jsonl is NULL)
LF_INVALID = 0x08

assert TG_REC.itemsize == 64 and ENTITY.itemsize == 16 and REACTION.itemsize == 12
assert COMMENT.itemsize == 32 and TG_CHAN.itemsize == 40 and YT_REC.itemsize == 80
GM_REC = np.dtype([  # tgi_gm_rec: one client.Message (SURVEY a12)
    ("str_off", "<u8"), ("ts_sec", "<i8"), ("views", "<i8"), ("ts_nsec", "<i4"), ("text_len", "<u4"),
    ("id_len", "<u2"), ("channel_len", "<u2"), ("sender_len", "<u2"), ("reserved", "<u2"), ("reserved2", "<u4"), ("reserved3", "<u4")])
GM_REACTION = np.dtype([("key_off", "<u4"), ("key_len", "<u2"), ("reserved", "<u2"), ("count", "<i8")])
assert YT_CHAN.itemsize == 64 and LINK.itemsize == 36 and GM_REC.itemsize == 48 and GM_REACTION.itemsize == 16
CH_REC = np.dtype([  # tgi_ch_rec: one channel page's StoreChannelData record
    ("chat_id", "<i8"), ("str_off", "<u8"), ("member_count", "<i4"), ("message_count", "<i4"), ("total_views", "<i4"),
    ("title_len", "<u4"), ("image_len", "<u4"), ("url_len", "<u4")])
assert CH_REC.itemsize == 40


# ---- ctypes structs ---------------------------------------------------------------------------
class TgBatchC(C.Structure):
    _fields_ = [
        ("n", C.c_uint64), ("recs", C.c_void_p), ("strs", C.c_void_p), ("strs_len", C.c_uint64),
        ("ent_off", C.c_void_p), ("ents", C.c_void_p), ("react_off", C.c_void_p),
        ("reacts", C.c_void_p), ("n_reacts", C.c_uint64), ("comment_off", C.c_void_p),
        ("comments", C.c_void_p), ("n_comments", C.c_uint64), ("aux", C.c_void_p),
        ("aux_len", C.c_uint64), ("n_chans", C.c_uint32), ("reserved", C.c_uint32),
        ("chans", C.c_void_p), ("chan_strs", C.c_void_p), ("chan_strs_len", C.c_uint64)]


class YtBatchC(C.Structure):
    _fields_ = [
        ("n", C.c_uint64), ("recs", C.c_void_p), ("strs", C.c_void_p), ("strs_len", C.c_uint64),
        ("n_chans", C.c_uint32), ("reserved", C.c_uint32), ("chans", C.c_void_p),
        ("chan_strs", C.c_void_p), ("chan_strs_len", C.c_uint64)]


class GmBatchC(C.Structure):
    _fields_ = [
        ("n", C.c_uint64), ("recs", C.c_void_p), ("strs", C.c_void_p), ("strs_len", C.c_uint64),
        ("react_off", C.c_void_p), ("reacts", C.c_void_p), ("n_reacts", C.c_uint64), ("aux", C.c_void_p),
        ("aux_len", C.c_uint64)]


class ChBatchC(C.Structure):
    _fields_ = [("n", C.c_uint64), ("recs", C.c_void_p), ("strs", C.c_void_p), ("strs_len", C.c_uint64)]


class ConfigC(C.Structure):
    _fields_ = [
        ("abi_version", C.c_uint32), ("device", C.c_int32), ("flags", C.c_uint32),
        ("tz_offset_sec", C.c_int32), ("min_post_date", C.c_int64), ("created_at_sec", C.c_int64),
        ("capture_sec", C.c_int64), ("capture_nsec", C.c_int32), ("created_at_nsec", C.c_int32),
        ("crawl_label_len", C.c_uint32), ("reserved", C.c_uint32), ("crawl_label", C.c_char_p),
        ("frontier_capacity", C.c_uint64), ("max_records", C.c_uint64), ("max_in_bytes", C.c_uint64),
        ("max_out_bytes", C.c_uint64)]


class ResultC(C.Structure):
    _fields_ = [
        ("n", C.c_uint64), ("status", C.c_void_p), ("jsonl", C.c_void_p), ("jsonl_len", C.c_uint64),
        ("line_off", C.c_void_p), ("link_off", C.c_void_p), ("links", C.c_void_p),
        ("n_links", C.c_uint64), ("n_new", C.c_uint64), ("frontier_size", C.c_uint64),
        ("kernel_ms", C.c_float), ("gpu_launches", C.c_uint32), ("parse_ms", C.c_float),
        ("emit_ms", C.c_float), ("slot", C.c_int32), ("emit_main_ms", C.c_float), ("var_bytes", C.c_uint64),
        ("main_bytes_out", C.c_uint64), ("main_bytes_in", C.c_uint64), ("frontier_ms", C.c_float), ("reserved", C.c_uint32)]


class MergeStatsC(C.Structure):
    _fields_ = [("merges", C.c_uint64), ("keys_sent", C.c_uint64), ("keys_received", C.c_uint64), ("keys_owned", C.c_uint64),
                ("bytes_sent", C.c_uint64), ("bucket_ms", C.c_double), ("exchange_ms", C.c_double), ("insert_ms", C.c_double),
                ("last_bucket_ms", C.c_double), ("last_exchange_ms", C.c_double), ("last_insert_ms", C.c_double)]


class SetInfoC(C.Structure):  # tgi_set_info_t
    _fields_ = [("count", C.c_uint64), ("capacity", C.c_uint64), ("table_slots", C.c_uint64), ("grows", C.c_uint64)]


class DaprPayloadsC(C.Structure):  # tgi_dapr_payloads_t
    _fields_ = [("n", C.c_uint64), ("data", C.c_void_p), ("data_len", C.c_uint64), ("data_off", C.c_void_p),
                ("path", C.c_void_p), ("path_len", C.c_uint64), ("path_off", C.c_void_p), ("kernel_ms", C.c_float),
                ("gpu_launches", C.c_uint32)]


class CombinedBlobC(C.Structure):  # tgi_combined_blob
    _fields_ = [("data_off", C.c_uint64), ("data_len", C.c_uint64), ("path_off", C.c_uint64), ("path_len", C.c_uint64),
                ("n_lines", C.c_uint64), ("raw_bytes", C.c_uint64), ("unix_nano", C.c_int64)]


class CombinedC(C.Structure):  # tgi_combined_t
    _fields_ = [("n_blobs", C.c_uint64), ("blobs", C.POINTER(CombinedBlobC)), ("data", C.c_void_p), ("path", C.c_void_p),
                ("n_dropped", C.c_uint64), ("dropped", C.c_void_p), ("open_lines", C.c_uint64), ("open_bytes", C.c_uint64),
                ("kernel_ms", C.c_float), ("gpu_launches", C.c_uint32)]


CHANNEL_GROUP = np.dtype([("chan_idx", "<u4"), ("reserved", "<u4"), ("n_lines", "<u8"), ("first_record", "<u8"),
                          ("byte_off", "<u8"), ("byte_len", "<u8")])  # tgi_channel_group
assert CHANNEL_GROUP.itemsize == 40


class ChannelAppendsC(C.Structure):  # tgi_channel_appends_t
    _fields_ = [("n_groups", C.c_uint64), ("groups", C.c_void_p), ("data", C.c_void_p), ("data_len", C.c_uint64),
                ("order", C.c_void_p), ("kernel_ms", C.c_float), ("gpu_launches", C.c_uint32)]


# crawl progress state (tgi_state_*)
STATE_NO_PAGE = 0xFFFFFFFF
STATE_TS_LOCAL = 0x7FFFFFFF  # tgi_state_page.ts_off of a time.Now() page: rendered in the context's local zone
STATE_STRINGS = ("id", "url", "status", "error", "platform", "parentId", "LastConnectionID", "sequenceId", "crawlId")
STATE_CODES = ("", "unfetched", "fetched", "failed", "deleted", "resample")  # preset status / platform codes
STATE_PAGE = np.dtype([("str_off", "<u8"), ("str_len", "<u4", (9,)), ("ts_off", "<i4"), ("depth", "<i8"),
                       ("ts_sec", "<i8"), ("ts_nsec", "<i4"), ("n_msgs", "<u4")])
STATE_MSG = np.dtype([("chat_id", "<i8"), ("message_id", "<i8"), ("page_id", "<u4"), ("status", "<u2"), ("platform", "<u2")])
STATE_UPDATE = np.dtype([("chat_id", "<i8"), ("message_id", "<i8"), ("row", "<u4"), ("status", "<u2"), ("reserved", "<u2")])
STATE_LAYER = np.dtype([("depth", "<i8"), ("n_pages", "<u8")])
assert (STATE_PAGE.itemsize, STATE_MSG.itemsize, STATE_UPDATE.itemsize, STATE_LAYER.itemsize) == (72, 24, 24, 16)


class StateJsonC(C.Structure):  # tgi_state_json_t
    _fields_ = [("data", C.c_void_p), ("len", C.c_uint64), ("kernel_ms", C.c_float), ("gpu_launches", C.c_uint32)]


E_NOPAGES = -7  # tgi_state_export: the layer map holds no page ("no pages found to export")
TURN_PAGE_JSON = 1  # tgi_state_page_begin / _close: also json.Marshal(page), the value Dapr's UpdatePage saves


class StateTurnC(C.Structure):  # tgi_state_turn_t
    _fields_ = [("turn", C.c_uint32), ("row", C.c_uint32), ("n_work", C.c_uint64), ("work", C.POINTER(C.c_uint32)),
                ("page_json", C.c_void_p), ("page_json_len", C.c_uint64), ("kernel_ms", C.c_float),
                ("gpu_launches", C.c_uint32)]


class StatePagesC(C.Structure):  # tgi_state_pages_t
    _fields_ = [("turn", C.c_uint32), ("n_pages", C.c_uint32), ("n_work", C.c_uint64), ("work", C.POINTER(C.c_uint32)),
                ("work_off", C.POINTER(C.c_uint64)), ("page_json", C.c_void_p), ("json_off", C.POINTER(C.c_uint64)),
                ("kernel_ms", C.c_float), ("gpu_launches", C.c_uint32)]


class StateEndC(C.Structure):  # tgi_state_end_t
    _fields_ = [("appended", C.c_uint64), ("kernel_ms", C.c_float), ("gpu_launches", C.c_uint32)]


DISCOVER_NOW = 1       # tgi_state_discover: AddLayer per span now (else the candidates go to the pending list)
DISCOVER_DAPR = 2       # DaprStateManager.AddLayer's rules instead of BaseStateManager's
DISCOVER_PAGE_JSON = 4  # json.Marshal of every added page (Dapr's per-page SaveState value)
STATE_SPAN = np.dtype([("row", "<u4"), ("reserved", "<u4"), ("first", "<u8"), ("n_records", "<u8"), ("n_done", "<u8")])


class StateAddedC(C.Structure):  # tgi_state_added_t
    _fields_ = [("n_candidates", C.c_uint64), ("n_added", C.c_uint64), ("rows", C.POINTER(C.c_uint32)),
                ("ids", C.c_void_p), ("page_json", C.c_void_p), ("json_off", C.POINTER(C.c_uint64)),
                ("kernel_ms", C.c_float), ("gpu_launches", C.c_uint32)]


STATE_NO_BATCH = 0xFFFFFFFF  # tgi_state_pending_edges: a span without edges (the crawler's forced walkback)
STATE_EDGE = np.dtype([("destination", "u1", (32,)), ("record", "<u8"), ("batch", "<u4"), ("dest_len", "u1"),
                       ("source_type", "u1"), ("status", "u1"), ("reserved", "u1")])  # tgi_state_edge
STATE_EDGE_BATCH = np.dtype([("batch_id", "S36"), ("span", "<u4"), ("first_edge", "<u4"),
                             ("n_edges", "<u4")])  # tgi_state_edge_batch
assert STATE_EDGE.itemsize == 48 and STATE_EDGE_BATCH.itemsize == 48


class StateEdgesC(C.Structure):  # tgi_state_edges_t
    _fields_ = [("n_candidates", C.c_uint64), ("n_edges", C.c_uint64), ("n_batches", C.c_uint32), ("reserved", C.c_uint32),
                ("edges", C.c_void_p), ("batches", C.c_void_p), ("span_batch", C.c_void_p), ("kernel_ms", C.c_float),
                ("gpu_launches", C.c_uint32)]


# tgi_state_edge_sql: the statement kinds (CreatePendingBatch, InsertPendingEdge, ClosePendingBatch) and the largest
# rows_per_stmt (8 bind parameters per edge row, at most 65535 per Postgres statement)
SQL_BATCH_INSERT, SQL_EDGE_INSERT, SQL_BATCH_CLOSE = 0, 1, 2
SQL_MAX_ROWS = 8191
STATE_EDGE_STMT = np.dtype([("kind", "<u4"), ("rows", "<u4"), ("sql_off", "<u8"), ("sql_len", "<u8"),
                            ("params_off", "<u8"), ("params_len", "<u8")])  # tgi_state_edge_stmt
assert STATE_EDGE_STMT.itemsize == 40


class StateEdgeSqlC(C.Structure):  # tgi_state_edge_sql_t
    _fields_ = [("n_stmts", C.c_uint64), ("stmts", C.c_void_p), ("data", C.c_void_p), ("data_len", C.c_uint64),
                ("kernel_ms", C.c_float), ("gpu_launches", C.c_uint32)]


# tgi_state_walkback: its statement kinds (AddPageToPageBuffer, SaveEdgeRecords of one record), each edge-less span's
# outcome (a channel picked; 10 draws of the owner's URL; no discovered channel) and pickWalkbackChannel's draws
SQL_PAGE_BUFFER_INSERT, SQL_EDGE_RECORD_INSERT = 3, 4
WALK_OK, WALK_EXHAUSTED, WALK_EMPTY = 0, 1, 2
WALK_MAX_DRAWS = 10
STATE_WALKBACK_SPAN = np.dtype([("span", "<u4"), ("status", "<u4"), ("draws", "<u4"), ("url_len", "<u4"),
                                ("url", "u1", 32), ("page_id", "S36"), ("sequence_id", "S36")])  # tgi_state_walkback_span
assert STATE_WALKBACK_SPAN.itemsize == 120


class StateWalkbackC(C.Structure):  # tgi_state_walkback_t
    _fields_ = [("n_walkbacks", C.c_uint32), ("reserved", C.c_uint32), ("walkbacks", C.c_void_p),
                ("n_stmts", C.c_uint64), ("stmts", C.c_void_p), ("data", C.c_void_p), ("data_len", C.c_uint64),
                ("kernel_ms", C.c_float), ("gpu_launches", C.c_uint32)]


# tgi_state_validator_walkback: its three more statement kinds (CompletePendingBatch, FlushBatchStats' upsert and
# delete), the validation classes of a claimed edge, the input rows (ClaimWalkbackBatch's batch and edges, strings as
# (offset, length) into one blob) and each batch's outcome
SQL_BATCH_COMPLETE, SQL_STATS_UPSERT, SQL_EDGES_DELETE = 5, 6, 7
EDGE_CLASS_VALID, EDGE_CLASS_NOT_CHANNEL, EDGE_CLASS_INVALID, EDGE_CLASS_DUPLICATE, EDGE_CLASS_OTHER = 0, 1, 2, 3, 4
EDGE_CLASS_OF = {b"valid": EDGE_CLASS_VALID, b"not_channel": EDGE_CLASS_NOT_CHANNEL, b"invalid": EDGE_CLASS_INVALID,
                 b"duplicate": EDGE_CLASS_DUPLICATE}  # validation_status by exact match; anything else is OTHER
CLAIMED_BATCH_STRINGS = ("batch_id", "crawl_id", "source_channel", "source_page_id", "sequence_id")  # TGI_CB_*
VW_NO_EDGE = 0xFFFFFFFF
CLAIMED_BATCH = np.dtype([("str_off", "<u8", 5), ("str_len", "<u4", 5), ("reserved", "<u4"),
                          ("source_depth", "<i8")])  # tgi_claimed_batch
CLAIMED_EDGE = np.dtype([("str_off", "<u8", 2), ("str_len", "<u4", 2), ("cls", "<u4"),
                         ("reserved", "<u4")])  # tgi_claimed_edge
STATE_VALIDATOR_BATCH = np.dtype([("status", "<u4"), ("walkback", "<u4"), ("rnd", "<i4"), ("draws", "<u4"),
                                  ("n_valid", "<u4"), ("forward_edge", "<u4"), ("url_len", "<u4"), ("reserved", "<u4"),
                                  ("url", "u1", 32), ("page_id", "S36"),
                                  ("sequence_id", "S36")])  # tgi_state_validator_batch
assert (CLAIMED_BATCH.itemsize, CLAIMED_EDGE.itemsize, STATE_VALIDATOR_BATCH.itemsize) == (72, 32, 136)


class ClaimedBatchesC(C.Structure):  # tgi_claimed_batches
    _fields_ = [("n_batches", C.c_uint32), ("reserved", C.c_uint32), ("batches", C.c_void_p), ("edge_off", C.c_void_p),
                ("edges", C.c_void_p), ("n_edges", C.c_uint64), ("strs", C.c_void_p), ("strs_len", C.c_uint64)]


class StateValidatorWalkbackC(C.Structure):  # tgi_state_validator_walkback_t
    _fields_ = [("n_batches", C.c_uint32), ("reserved", C.c_uint32), ("batches", C.c_void_p),
                ("n_stmts", C.c_uint64), ("stmts", C.c_void_p), ("data", C.c_void_p), ("data_len", C.c_uint64),
                ("kernel_ms", C.c_float), ("gpu_launches", C.c_uint32)]


# tgi_state_rw_lookups / tgi_state_rw_step: the standard random walk.  Dapr's chatIDCache set, the SearchPublicChat
# outcome codes, the span statuses past WALK_*, the two upsert kinds, a lookup row, an outcome and a span's step
SET_SEEDS = 5
RW_FOUND, RW_NOT_SUPERGROUP, RW_NOT_FOUND, RW_RETIRE = 0, 1, 2, 3
RW_RETIRED, RW_DEFERRED = 3, 4
RW_NO_FORWARD = 0xFFFFFFFF
SQL_SEED_UPSERT, SQL_INVALID_UPSERT = 8, 9
RW_LOOKUP = np.dtype([("name", "u1", 32), ("record", "<u8"), ("span", "<u4"), ("name_len", "u1"), ("source_type", "u1"),
                      ("reserved", "<u2")])  # tgi_rw_lookup
RW_OUTCOME = np.dtype([("chat_id", "<i8"), ("code", "<u4"), ("reserved", "<u4")])  # tgi_rw_outcome
RW_SPAN = np.dtype([("status", "<u4"), ("walkback", "<u4"), ("rnd", "<i4"), ("draws", "<u4"), ("n_new", "<u4"),
                    ("forward", "<u4"), ("url_len", "<u4"), ("reserved", "<u4"), ("url", "u1", 32), ("page_id", "S36"),
                    ("sequence_id", "S36")])  # tgi_rw_span
assert (RW_LOOKUP.itemsize, RW_OUTCOME.itemsize, RW_SPAN.itemsize) == (48, 16, 136)


class StateRwLookupsC(C.Structure):  # tgi_state_rw_lookups_t
    _fields_ = [("n_candidates", C.c_uint64), ("n_lookups", C.c_uint64), ("lookups", C.c_void_p),
                ("span_candidates", C.c_void_p), ("kernel_ms", C.c_float), ("gpu_launches", C.c_uint32)]


class StateRwStepC(C.Structure):  # tgi_state_rw_step_t
    _fields_ = [("n_spans", C.c_uint32), ("reserved", C.c_uint32), ("spans", C.c_void_p), ("hits", C.c_uint64 * 4),
                ("misses", C.c_uint64 * 4), ("n_stmts", C.c_uint64), ("stmts", C.c_void_p), ("data", C.c_void_p),
                ("data_len", C.c_uint64), ("kernel_ms", C.c_float), ("gpu_launches", C.c_uint32)]


# tgi_state_validator_lookups / tgi_state_validator_edges: the validator's edge pass.  A claimed PendingEdge (strings as
# (offset, length) into one blob), a lookup row, a row's outcome and attempts, an edge's result, and their codes
VE_STRINGS = ("destination", "crawl_id", "source_type")  # TGI_VE_*
VA_VALID, VA_NOT_CHANNEL, VA_INVALID, VA_OTHER, VA_TRANSIENT, VA_BLOCKED = 0, 1, 2, 3, 4, 5
VR_NONE, VR_NOT_SUPERGROUP, VR_NOT_FOUND, VR_CACHED_INVALID, VR_UNKNOWN_STATUS = 0, 1, 2, 3, 4
VS_PENDING, VS_VALID, VS_DUPLICATE, VS_INVALID, VS_NOT_CHANNEL = 0, 1, 2, 3, 4
VK_DEFINITIVE, VK_TRANSIENT, VK_BLOCKED = 0, 1, 2
VR_NAMES = (b"", b"not_supergroup", b"not_found", b"cached_invalid", b"unknown_status")
VS_NAMES = (b"pending", b"valid", b"duplicate", b"invalid", b"not_channel")
VE_BLOCKED_THRESHOLD = 5
VE_NOT_CROSSED = 0xFFFFFFFFFFFFFFFF
SQL_ACCESS_EVENT, SQL_EDGE_UPDATE = 10, 11
PENDING_CLAIM_EDGE = np.dtype([("pending_id", "<i8"), ("str_off", "<u8", 3), ("str_len", "<u4", 3),
                               ("reserved", "<u4")])  # tgi_pending_claim_edge
VALIDATOR_LOOKUP = np.dtype([("name", "u1", 32), ("occ_off", "<u8"), ("m", "<u4"), ("name_len", "u1"),
                             ("reserved", "u1", 3)])  # tgi_validator_lookup
VALIDATOR_OUTCOME = np.dtype([("discovered", "<u4"), ("claimed", "<u4"), ("n_attempts", "<u4"),
                              ("reserved", "<u4")])  # tgi_validator_outcome
VALIDATOR_ATTEMPT = np.dtype([("kind", "<u4"), ("reason", "<u4")])  # tgi_validator_attempt
VALIDATOR_EDGE_RESULT = np.dtype([("blocked_count", "<i8"), ("status", "u1"), ("reason", "u1"), ("kind", "u1"),
                                  ("reserved", "u1", 5)])  # tgi_validator_edge_result
assert (PENDING_CLAIM_EDGE.itemsize, VALIDATOR_LOOKUP.itemsize, VALIDATOR_OUTCOME.itemsize, VALIDATOR_ATTEMPT.itemsize,
        VALIDATOR_EDGE_RESULT.itemsize) == (48, 48, 16, 8, 16)


class PendingClaimC(C.Structure):  # tgi_pending_claim
    _fields_ = [("edges", C.c_void_p), ("n_edges", C.c_uint64), ("strs", C.c_void_p), ("strs_len", C.c_uint64)]


class StateValidatorLookupsC(C.Structure):  # tgi_state_validator_lookups_t
    _fields_ = [("n_edges", C.c_uint64), ("n_cached", C.c_uint64), ("n_lookups", C.c_uint64), ("lookups", C.c_void_p),
                ("occurrences", C.c_void_p), ("kernel_ms", C.c_float), ("gpu_launches", C.c_uint32)]


class StateValidatorEdgesC(C.Structure):  # tgi_state_validator_edges_t
    _fields_ = [("n_edges", C.c_uint64), ("edges", C.c_void_p), ("blocked_count_out", C.c_int64),
                ("crossed_at", C.c_uint64), ("n_stmts", C.c_uint64), ("stmts", C.c_void_p), ("data", C.c_void_p),
                ("data_len", C.c_uint64), ("kernel_ms", C.c_float), ("gpu_launches", C.c_uint32)]


READ_MESSAGES = 1  # tgi_state_read_pages / _read_layer: also each page's message list, gathered on the device
# tgi_state_read_layer's page selection: none, standalone (new execution / resumed), Dapr's processLayerInParallel
SELECT_NONE, SELECT_STANDALONE, SELECT_STANDALONE_RESUME, SELECT_DAPR = 0, 1, 2, 3


class StateReadC(C.Structure):  # tgi_state_read_t
    _fields_ = [("n_pages", C.c_uint64), ("rows", C.c_void_p), ("pages", C.c_void_p), ("strs", C.c_void_p), ("strs_len", C.c_uint64),
                ("msgs", C.c_void_p), ("msg_first", C.c_void_p), ("n_msgs", C.c_uint64), ("select", C.c_void_p),
                ("n_selected", C.c_uint64), ("kernel_ms", C.c_float), ("gpu_launches", C.c_uint32)]


class StateLayersC(C.Structure):  # tgi_state_layers_t
    _fields_ = [("n_layers", C.c_uint64), ("depth", C.c_void_p), ("n_pages", C.c_void_p), ("max_depth", C.c_int64),
                ("has_max_depth", C.c_uint32), ("reserved", C.c_uint32), ("n_incomplete", C.c_uint64)]


STATE_EXPORT_DAPR, STATE_EXPORT_LOCAL = 0, 1
STATE_EXPORT_CHUNK_DEFAULT = 100 * 1024 * 1024  # exportChunkSizeBytes (state/daprstate.go:2909)


class StateExportC(C.Structure):  # tgi_state_export_t
    _fields_ = [("data", C.c_void_p), ("off", C.POINTER(C.c_uint64)), ("len", C.POINTER(C.c_uint64)),
                ("raw_len", C.POINTER(C.c_uint64)), ("n_chunks", C.c_uint64), ("n_pages", C.c_uint64),
                ("kernel_ms", C.c_float), ("gpu_launches", C.c_uint32)]


class StatsC(C.Structure):
    _fields_ = [("records", C.c_uint64), ("bytes_in", C.c_uint64), ("bytes_out", C.c_uint64),
                ("links", C.c_uint64), ("frontier_size", C.c_uint64), ("launches", C.c_uint64),
                ("kernel_ms_total", C.c_double)]


def ptr(a: np.ndarray | None) -> int | None:
    """address of a C-contiguous numpy array (None -> NULL)."""
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data


def make_config(*, device: int = 0, min_post_date: int | None = None, tz_offset_sec: int = 0,
                created_at_sec: int = 1_750_000_000, created_at_nsec: int = 0,
                capture_sec: int = 1_750_000_000, capture_nsec: int = 123_456_789,
                crawl_label: bytes = b"", frontier_capacity: int = 0, max_records: int = 0,
                max_in_bytes: int = 0, max_out_bytes: int = 0) -> ConfigC:
    c = ConfigC()
    c.abi_version = ABI_VERSION
    c.device = device
    c.flags = CFG_SKIP_MEDIA | (CFG_HAS_MIN_POST_DATE if min_post_date is not None else 0)
    c.tz_offset_sec = tz_offset_sec
    c.min_post_date = min_post_date or 0
    c.created_at_sec = created_at_sec
    c.created_at_nsec = created_at_nsec
    c.capture_sec = capture_sec
    c.capture_nsec = capture_nsec
    c._label_keepalive = crawl_label  # keep the bytes object alive with the struct
    c.crawl_label = crawl_label
    c.crawl_label_len = len(crawl_label)
    c.frontier_capacity = frontier_capacity
    c.max_records = max_records
    c.max_in_bytes = max_in_bytes
    c.max_out_bytes = max_out_bytes
    return c
