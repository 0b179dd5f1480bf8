// tgingest.cu — host side of libtgingest: the C ABI of include/tgingest.h on top of the sm_90a
// kernels in kernels.cuh.  One context = one GPU.  Three staging slots, each with its own stream
// and worker thread, so H2D of one batch, kernels of another and D2H of a third overlap.
// There is no CPU fallback: without a CUDA device tgi_create fails with TGI_E_NODEVICE.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>  // types only: the library itself is loaded with dlopen at tgi_comm_init

#include <algorithm>
#include <charconv>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <numeric>
#include <map>
#include <memory>
#include <string>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "kernels.cuh"
#include "dapr.cuh"
#include "combine.cuh"
#include "local_appends.cuh"
#include "state.cuh"
#include "tg_page.cuh"
#include "yt_page.cuh"

using namespace tgi;

namespace {

constexpr size_t PAD = 64;  // zero bytes behind every device blob (kernels over-read <= 31 bytes)

struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }  // error paths of the one-shot entry points must not leak device memory
  cudaError_t ensure(size_t bytes) {
    bytes += PAD;
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    size_t want = bytes + bytes / 8;
    cudaError_t e = cudaMalloc(&p, want);
    cap = e == cudaSuccess ? want : 0;
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  void swap(DevBuf& o) {
    std::swap(p, o.p);
    std::swap(cap, o.cap);
  }
  template <class T>
  T* as() const { return (T*)p; }
};
struct HostBuf {  // pinned
  void* p = nullptr;
  size_t cap = 0;
  unsigned flags = cudaHostAllocDefault;
  HostBuf() = default;
  HostBuf(const HostBuf&) = delete;
  HostBuf& operator=(const HostBuf&) = delete;
  ~HostBuf() { release(); }
  cudaError_t ensure(size_t bytes) {
    if (bytes <= cap && p) return cudaSuccess;
    if (p) cudaFreeHost(p);
    p = nullptr;
    size_t want = bytes + bytes / 8 + 64;
    cudaError_t e = cudaHostAlloc(&p, want, flags);
    cap = e == cudaSuccess ? want : 0;
    return e;
  }
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
  }
  template <class T>
  T* as() const { return (T*)p; }
};

enum RecKind { REC_NONE, REC_TG, REC_YT, REC_GM, REC_CH };

// One job on a staging slot: upload a batch (which becomes the slot's resident batch), run the resident batch, or both.
enum JobStages : uint32_t { JOB_UPLOAD = 1, JOB_RUN = 2 };
struct Job {
  RecKind kind;
  uint32_t stages;    // JOB_UPLOAD | JOB_RUN
  const void* batch;  // JOB_UPLOAD: the tgi_tg_batch / tgi_yt_batch / tgi_gm_batch / tgi_ch_batch of `kind`
  uint32_t flags;     // JOB_RUN: TGI_RUN_*
};

struct ResultArrays {  // where a batch's result arrays are, on the host or on the device
  const uint8_t* status;
  const uint64_t* line_off;
  const uint8_t* jsonl;
  const uint32_t* link_off;
  const tgi_link* links;
};
// What the readers (tgi_result_read_*, tgi_pending_edges, tgi_dapr_payloads) read: the result of the slot's last job,
// from its success until the next job is claimed on the slot.  kind == REC_NONE: the slot holds no result.
struct LastResult {
  RecKind kind = REC_NONE;
  uint64_t n = 0;
  uint32_t flags = 0;  // the run flags that shaped it
  uint64_t n_new = 0, n_links = 0, jsonl_len = 0;
  ResultArrays dev{};  // its arrays on the device; line_off / link_off / links are null when the run did not make them
  const uint64_t* host_line_off = nullptr;  // its line offsets in pinned host memory (null: TGI_RUN_NO_D2H or no lines)
};

// one batch's frontier phases: the batch hash table, per-link state, per-record NEW counts and their offsets
struct FrontierScratch {
  DevBuf btable, lstate, rec_new, new_off;
};

struct InsertScratch {
  DevBuf arena, cnt, tiles, sc;
  FrontierScratch fs;
};

// one device-resident key set: its buffers, the kernels' view of them, and what the host knows of its fill
struct KeySet {
  DevBuf pool, table, count, payload;
  FrontierDev dev{};   // dev.table == nullptr: not allocated (an exclusion set before its first tgi_set_add)
  uint64_t bound = 0;  // upper bound of the set's count: the keys it held when last read plus every key enqueued since
  uint64_t grows = 0;  // rehashes into bigger buffers (set_grow)
};

// the NCCL entry points the merge uses, resolved at run time
struct NcclApi {
  void* h = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};

// tgi_dapr_payloads: its device scratch and outputs, and the pinned host copies it returns
struct DaprBufs {
  DevBuf prefix, lens, off, data, path, sc;
  HostBuf h_off, h_data, h_path, h_sc;
};

// tgi_channel_appends: the channelID table and row map, the per-record / per-line / per-run arrays (u32s, u64s), the
// radix counts and their scan, its outputs and the pinned host copies it returns
struct LocalBufs {
  DevBuf table, rows, u32s, u64s, counts, roff, groups, order, data, sc;
  HostBuf h_groups, h_order, h_data, h_sc;
};

// tgi_combine_*: the combiner's settings, its open group (encoded on the device, 0-2 bytes pending) and its scratch
struct Combiner {
  std::mutex mu;
  bool open = false;
  uint64_t trigger = 0, hard_cap = 0;
  std::string prefix;
  uint64_t open_lines = 0, open_bytes = 0;  // the open group: its posts and raw bytes; enc holds open_bytes / 3 words
  DevBuf enc;        // the open blob's base64, 4*ceil(hard_cap/3) bytes
  DevBuf pend;       // two 32-byte halves: the pending bytes (open_bytes % 3) in half `cur`, the next call's in the other
  int cur = 0;
  int64_t last_ns = 0;
  bool any_ns = false;
  cudaStream_t stream = nullptr;  // tgi_combine_flush's work (the adds run on their slot's stream)
  cudaEvent_t ev = nullptr, t0 = nullptr, t1 = nullptr;  // ev: the last call's work; t0 / t1: its device time
  bool ev_valid = false;
  DevBuf out, tables, drops, counts;  // closed blobs past the first, task / segment tables, dropped lines, posts per group
  HostBuf h_blobs, h_data, h_path, h_tables, h_drops, h_counts, h_line_off;
};

// tgi_state_*: the crawl progress state (state.cuh).  The host keeps the layers, the page rows (a mirror of the device
// rows and their strings), the id and URL maps of AddLayer / UpdatePage and the string table; the messages and the
// lookup table live on the device only.
struct CrawlState {
  std::mutex mu;
  cudaStream_t stream = nullptr;
  cudaEvent_t t0 = nullptr, t1 = nullptr, t2 = nullptr, t3 = nullptr;  // the render's size pass and emit
  cudaEvent_t t4 = nullptr, t5 = nullptr;                              // the export's base64 encode
  std::vector<tgi_state_page> rows;  // str_off into blob
  std::string blob;
  std::vector<uint32_t> gen;         // mirror of row_gen
  std::unordered_map<std::string, uint32_t> by_id;   // pageMap: id -> row
  std::unordered_map<std::string, uint64_t> urls;    // URL -> pages of pageMap with it (AddLayer's existingURLs)
  uint64_t deadends = 0;                             // pages with status "deadend"
  std::map<int64_t, std::vector<uint32_t>> layers;   // layerMap, ascending depth
  std::vector<std::string> codes;
  std::unordered_map<std::string, uint16_t> code_of;
  bool codes_dirty = true;
  uint64_t rows_synced = 0, blob_synced = 0;         // rows / blob bytes already on the device
  uint64_t n_msgs = 0, n_dead = 0;                   // message rows on the device, and how many are tombstones
  uint64_t tslots = 0;
  DevBuf pages, dblob, row_gen, row_cnt, msgs, table, code_blob, code_off;
  DevBuf upd, bfirst, blast, slot_of, flag, pos, tiles, sc, spare;  // scratch
  DevBuf entries, keys, vals, row_base, msize, moff, e32, e64, counts, roff, out;
  DevBuf lm_keys, cb_tasks, cb_segs, b64;  // the layer map's openings; the export's encode tasks and output
  HostBuf h_out, h_sc, h_read, h_chunks;
  // page turns (tgi_state_pages_begin / _end / _close): each open turn's rows and owner keys, by handle, and each row's
  // owner view (tgi_state_pages_close): the last begin's owner keys of the row and their statuses, a slice of the
  // buffer of that begin's call.  A buffer neither a turn nor a view holds is kept for the next begins.
  struct Turn {
    std::vector<uint32_t> rows;    // [P] the pages
    std::vector<uint64_t> off;     // [P+1] page k's owner messages are [off[k], off[k+1])
    std::shared_ptr<DevBuf> keys;  // [n_work][2] chat_id, message_id, then the views' uint16 statuses [n_work]
    uint64_t n_work() const { return off.back(); }
  };
  struct View {
    uint64_t off = 0, k = 0, total = 0;  // owner messages [off, off + k) of a buffer that holds `total`
    std::shared_ptr<DevBuf> keys;        // as Turn::keys
    const long long* key_ptr() const { return keys->as<long long>() + 2 * off; }
    uint16_t* status_ptr() const { return (uint16_t*)(keys->as<uint8_t>() + 16 * total) + off; }
  };
  std::map<uint32_t, Turn> turns;
  std::unordered_map<uint32_t, View> views;  // by row
  std::vector<std::shared_ptr<DevBuf>> turn_pool;
  uint32_t next_turn = 1;
  cudaEvent_t ev_slot = nullptr;  // tgi_state_pages_end: the slot's work the state stream waits for
  cudaEvent_t ev_seg = nullptr;   // the last upload from h_seg: a call that rewrites h_seg waits for it first
  DevBuf turn_in;                 // the fetched keys of tgi_state_pages_begin
  DevBuf seg, pg;                 // the pages' arrays of a turn call (rows, offsets, row puts, views); each key's page
  HostBuf h_work, h_woff, h_seg, h_old;
  std::vector<uint8_t> row_mark;  // st_join_layers' marks, a byte per row, all 0 between calls
  // snowball discovery (tgi_state_discover / _next_layer): the pending next-layer list (StCand, grown on demand), the
  // id generator's key and next counter, and the scratch of the candidates and survivors
  DevBuf pend, cand, surv, spans, cnt, soff, coff, lnk, spn, uuids, url_keys;
  uint64_t n_pend = 0;
  uint64_t id_seed = 0, id_next = 0;
  bool seeded = false;
  HostBuf h_surv, h_coff, h_ids, h_rows, h_json_off;
  // tandem hand-off (tgi_state_pending_edges): the batch-id counter (ids under id_seed) and the call's outputs
  uint64_t batch_next = 0;
  DevBuf clink, edges, ebatches, span_batch;
  HostBuf h_edges, h_ebatches, h_span_batch;
  // tandem hand-off SQL (tgi_state_edge_sql): whether the last state call was an accepted hand-off, whose edges,
  // batches and spans above then still hold it; the rows' sizes and offsets, and the pinned output
  bool handoff_live = false;
  uint64_t handoff_ne = 0, handoff_nb = 0;
  DevBuf sql_in, sql_size, sql_off, sql_out, sql_stmts;
  HostBuf h_sql, h_sql_stmts;
  // tandem forced walkback (tgi_state_walkback): the hand-off's edge-less spans as (span, row) pairs, whether its picks
  // are made (then wb / wb_rank hold them and n_ok counts the usable ones), the counter of edge-less spans handled, the
  // picks on the device and the pinned outputs
  std::vector<uint32_t> wb_spans;
  bool wb_picked = false;
  uint64_t wb_n_ok = 0, walk_next = 0;
  DevBuf wb_in, wb, wb_ok, wb_rank;
  HostBuf h_wb, h_wb_sql, h_wb_stmts;
  // validator walkback (tgi_state_validator_walkback): the counter of claimed batches handled, the uploaded batches,
  // the per-batch outcomes, lists, counts and their scans, and the pinned outputs
  uint64_t vw_next = 0;
  DevBuf vw_b, vw_eoff, vw_e, vw_s, vw_out, vw_list, vw_cnt, vw_rank;
  HostBuf h_vw, h_vw_sql, h_vw_stmts;
  // standard random walk (tgi_state_rw_lookups / _step): whether the lookups' lists are live (cand, coff and spans
  // above then hold them, with each candidate's class and lookup index and the lookup rows), their sizes, the counter of
  // deciding spans, the step's scratch and the pinned outputs
  bool rw_live = false;
  uint32_t rw_n_spans = 0;
  uint64_t rw_n_cand = 0, rw_n_lk = 0, rw_next = 0;
  DevBuf rw_cls, rw_lpos, rw_lk, rw_oc, rw_flag, rw_pos, rw_list, rw_keys, rw_new, rw_nflag, rw_npos, rw_n0, rw_out,
      rw_cnt, rw_rank;
  HostBuf h_rw_lk, h_rw_cand, h_rw_out, h_rw_sql, h_rw_stmts;
  // validator edge pass (tgi_state_validator_lookups / _edges): whether a plan is live (only the next lookups or an
  // accepted pass ends it, so its buffers are its own), its claim, lookup rows and each edge's row and occurrence on the
  // device, the lookup rows on the host, the pass's scratch and the pinned outputs
  bool ve_live = false;
  uint64_t ve_n = 0, ve_nl = 0;
  DevBuf ve_e, ve_s, ve_cand, ve_bfirst, ve_slot, ve_flag, ve_lpos, ve_keys, ve_vals, ve_loff, ve_elk, ve_rank, ve_lk;
  DevBuf ve_oc, ve_aoff, ve_at, ve_res, ve_pos, ve_list, ve_names;
  HostBuf h_ve_lk, h_ve_occ, h_ve_aoff, h_ve_res, h_ve_sql, h_ve_stmts;
  // page reads (tgi_state_read_pages / _read_layer, tgi_state_layers): the read set with its counts and offsets on the
  // device and its staging, and the pinned outputs
  DevBuf rset;
  HostBuf h_rset, h_rrows, h_rpages, h_rstrs, h_rmsgs, h_rfirst, h_rsel, h_rdepth, h_rcount;
};

struct Slot {
  int idx = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev_k0 = nullptr, ev_k1 = nullptr, ev_p0 = nullptr, ev_p1 = nullptr, ev_e0 = nullptr, ev_e1 = nullptr, ev_f1 = nullptr, ev_fr0 = nullptr, ev_fr1 = nullptr;
  // device inputs
  DevBuf d_recs, d_strs, d_ent_off, d_ents, d_react_off, d_reacts, d_comment_off, d_comments, d_aux,
      d_chans, d_chan_strs;
  // device intermediates / outputs
  DevBuf d_chan_derived, d_chan_len, d_chan_off, d_chan_blob, d_status, d_linelen, d_line_off,
      d_link_start, d_link_count, d_xlen, d_xpos, d_lists, d_arena, d_link_off, d_links_out, d_link_off32, d_tiles, d_scalars, d_jsonl, d_url_start, d_url_count, d_urls, d_ent_range;
  // pinned host outputs
  HostBuf h_status, h_line_off, h_jsonl, h_link_off, h_links, h_scalars;
  FrontierScratch fs;
  // page-sized Telegram batches (tg_page.cuh): the input arrays in ONE block / copy, the result arrays in one block / copy
  DevBuf d_page_in, d_page_out;
  HostBuf h_page_in, h_page_out;
  uint32_t page_bpr = 3072;              // running estimate of result bytes per record (sizes the speculative read)
  // batch descriptors, filled by the uploads (`resident` says which one still describes the batch on the device)
  TgBatchDev tg{};
  YtBatchDev yt{};
  GmBatchDev gm{};
  ChBatchDev ch{};
  uint64_t yt_desc_bytes = 0;
  uint64_t n_ents = 0, n_reacts = 0, n_comments = 0, in_bytes = 0, chan_strs_len = 0;
  RecKind resident = REC_NONE;  // REC_TG / REC_YT: tg / yt describes the batch of the last successful upload
  LastResult last;
  DaprBufs dapr;
  LocalBufs local;
  // job hand-off (under mu)
  std::mutex mu;
  std::condition_variable cv;
  enum { IDLE, QUEUED, QUIT } worker_state = IDLE;  // what the worker thread has to do: nothing, `job`, exit
  Job job{};
  bool busy = false, done = false, claimed = false;
  uint64_t ticket = 0;
  bool has_ticket = false;
  int rc = 0;
  tgi_result res{};
  std::thread worker;
};

}  // namespace

struct tgi_ctx {
  tgi_config cfg{};
  std::string label;
  int device = 0;
  int sms = 132;
  std::string err;
  std::mutex err_mu;
  Slot slots[TGI_SLOTS];
  HostBuf h_zero;  // PAD pinned zero bytes (h2d)
  // config blob on device
  DevBuf d_cfg;
  CfgDev cfgdev{};
  std::mutex cfg_mu;
  std::vector<ZoneEnt> zone;  // tgi_set_zone (empty: tz_offset_sec) and its device copy
  DevBuf d_zone;
  // the resident key sets, indexed by TGI_SET_*: the dedup set (every key this GPU has seen), the exclusion sets of the
  // frontier -> validator hand-off (tgi_set_add), this rank's partition of the multi-GPU set (tgi_comm_init) and Dapr's
  // urlCache (tgi_state_discover), Dapr's chatIDCache (tgi_state_rw_step)
  KeySet sets[6];
  int64_t now_sec = 0;     // tgi_set_now: the clock the TTL of the invalid set is checked against
  uint64_t fr_cap0 = 0;    // tgi_config.frontier_capacity: the size the dedup set started at
  uint64_t grow_max = 0;   // tgi_set_growth: sets grow up to this many keys (0: fixed size)
  std::mutex fr_mu;
  cudaEvent_t fr_event = nullptr;
  bool fr_event_valid = false;
  // frontier turns: batches with TGI_RUN_FRONTIER take a ticket when they are submitted and enter their frontier phase in
  // ticket order, so NEW flags / n_new / the export order are those of one thread processing the batches in submission order
  std::mutex tk_mu;
  std::condition_variable tk_cv;
  uint64_t tk_next = 0, tk_serving = 0;
  InsertScratch ins;  // scratch of tgi_frontier_insert* / tgi_set_add / the merge (under fr_mu)
  Combiner cb;        // tgi_combine_*
  CrawlState state;   // tgi_state_*
  // multi-GPU merge: communicator (this rank's partition is sets[TGI_SET_OWNED])
  NcclApi* nccl = nullptr;
  ncclComm_t comm = nullptr;
  int rank = 0, nranks = 1;
  uint64_t merged_upto = 0, merge_round = 0;
  DevBuf m_cnt, m_all, m_cursor, m_send_keys, m_send_pay, m_recv_keys, m_recv_pay, m_gsize;
  HostBuf m_host;
  cudaEvent_t m_ev[4] = {nullptr, nullptr, nullptr, nullptr};
  tgi_merge_stats mstats{};
  // pinned input staging blocks handed to the packer
  std::mutex stg_mu;
  std::map<void*, size_t> stg_live;
  std::multimap<size_t, void*> stg_free;
  // stats
  std::mutex st_mu;
  tgi_stats stats{};
  // slot allocation for the blocking entry points
  std::mutex alloc_mu;
  std::condition_variable alloc_cv;
};

namespace {

std::string g_create_err;

void set_err(tgi_ctx* c, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (c) {
    std::lock_guard<std::mutex> g(c->err_mu);
    c->err = buf;
  } else {
    g_create_err = buf;
  }
}

// TGI_TRACE_SLOTS=1: host time (ms since the first stamp) at the synchronisation points of a bulk batch, one line each,
// to stderr — the only timeline tool this image has (no nsys): which slot's copies / kernels overlap with which
void trace_slot(const Slot& s, const char* what) {
  static const bool on = getenv("TGI_TRACE_SLOTS") != nullptr;
  if (!on) return;
  static const auto t0 = std::chrono::steady_clock::now();
  const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  fprintf(stderr, "slot %d %9.3f ms  %s\n", s.idx, ms, what);
}

#define CK(call)                                                                        \
  do {                                                                                  \
    cudaError_t _e = (call);                                                            \
    if (_e != cudaSuccess) {                                                            \
      set_err(c, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return _e == cudaErrorMemoryAllocation ? TGI_E_NOMEM : TGI_E_CUDA;                \
    }                                                                                   \
  } while (0)

// the nanoseconds of a time.Time: every entry point that takes a (sec, nsec) time refuses anything else (TGI_E_ARG)
bool nsec_ok(int32_t nsec) { return nsec >= 0 && nsec < 1000000000; }

// ---- host-side rendering of the injected clock (same rules as render_time on the device) --------
int host_render_time(char* dst, int64_t sec, int32_t nsec, int32_t tz) {
  int64_t t = sec + tz;
  int64_t days = t / 86400, rem = t % 86400;
  if (rem < 0) { rem += 86400; days -= 1; }
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
  int o = snprintf(dst, 40, "\"%04d-%02d-%02dT%02d:%02d:%02d", (int)y, (int)m, (int)d, (int)(rem / 3600),
                   (int)(rem % 3600 / 60), (int)(rem % 60));
  if (nsec) {
    char f[16];
    snprintf(f, sizeof f, "%09d", nsec);
    int k = 9;
    while (k > 0 && f[k - 1] == '0') k--;
    dst[o++] = '.';
    memcpy(dst + o, f, k);
    o += k;
  }
  if (tz == 0) dst[o++] = 'Z';
  else {
    int a = tz < 0 ? -tz : tz;
    o += snprintf(dst + o, 8, "%c%02d:%02d", tz < 0 ? '-' : '+', a / 3600, a % 3600 / 60);
  }
  dst[o++] = '"';
  return o;
}
// the same in the zone table z (render_zone_time on the device); an empty table is the fixed offset tz
int host_render_zone_time(char* dst, int64_t sec, int32_t nsec, const std::vector<ZoneEnt>& z, int32_t tz) {
  if (z.empty()) return host_render_time(dst, sec, nsec, tz);
  const auto it = std::upper_bound(z.begin(), z.end(), sec, [](int64_t t, const ZoneEnt& e) { return t < e.start; });
  const int32_t off = (it == z.begin() ? z.front() : it[-1]).off;
  const int o = host_render_time(dst, sec, nsec, off);
  if (o && off < 0 && off > -60) dst[o - 7] = '+';
  return o;
}

// Builds the per-context constant blob (escaped label + clock strings) and uploads it.  The label
// is JSON-escaped ON THE DEVICE by the same Emitter code that escapes everything else.
__global__ void cfg_label_size_kernel(const uint8_t* s, uint32_t n, uint32_t* out) {
  uint32_t e = warp_esc_len(s, n);
  if (lane_id() == 0) *out = e;
}
__global__ void cfg_label_emit_kernel(const uint8_t* s, uint32_t n, uint8_t* out) { esc_to_global(out, s, n); }

int build_cfg_blob(tgi_ctx* c) {
  const tgi_config& cfg = c->cfg;
  char t_tg[48], t_yt[48], t_cap[48];
  int n_tg = host_render_time(t_tg, cfg.created_at_sec, 0, 0);
  int n_yt = host_render_zone_time(t_yt, cfg.created_at_sec, cfg.created_at_nsec, c->zone, cfg.tz_offset_sec);
  int n_cap = host_render_zone_time(t_cap, cfg.capture_sec, cfg.capture_nsec, c->zone, cfg.tz_offset_sec);
  cudaStream_t s = c->slots[0].stream;
  uint32_t n = (uint32_t)c->label.size();
  DevBuf raw, len;
  CK(raw.ensure(n));
  CK(len.ensure(4));
  CK(cudaMemsetAsync(raw.p, 0, n + PAD, s));
  if (n) CK(cudaMemcpyAsync(raw.p, c->label.data(), n, cudaMemcpyHostToDevice, s));
  cfg_label_size_kernel<<<1, 32, 0, s>>>(raw.as<uint8_t>(), n, len.as<uint32_t>());
  uint32_t esc = 0;
  CK(cudaMemcpyAsync(&esc, len.p, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  auto pad16 = [](size_t x) { return (x + 15) & ~(size_t)15; };
  const size_t o_tg = pad16(esc), o_yt = o_tg + pad16(n_tg), o_cap = o_yt + pad16(n_yt);
  size_t total = o_cap + pad16(n_cap);
  CK(c->d_cfg.ensure(total + 16));
  CK(cudaMemsetAsync(c->d_cfg.p, 0, total + 16 + PAD, s));
  cfg_label_emit_kernel<<<1, 32, 0, s>>>(raw.as<uint8_t>(), n, c->d_cfg.as<uint8_t>());
  uint8_t* b = c->d_cfg.as<uint8_t>();
  if (n_tg) CK(cudaMemcpyAsync(b + o_tg, t_tg, n_tg, cudaMemcpyHostToDevice, s));
  if (n_yt) CK(cudaMemcpyAsync(b + o_yt, t_yt, n_yt, cudaMemcpyHostToDevice, s));
  if (n_cap) CK(cudaMemcpyAsync(b + o_cap, t_cap, n_cap, cudaMemcpyHostToDevice, s));
  CK(cudaStreamSynchronize(s));
  raw.release();
  len.release();
  CfgDev d{};
  d.blob = b;
  d.off[0] = 0;
  d.off[1] = (uint32_t)o_tg;
  d.off[2] = (uint32_t)o_yt;
  d.off[3] = (uint32_t)o_cap;
  d.label_len = esc;
  d.created_tg_len = (uint32_t)n_tg;
  d.created_yt_len = (uint32_t)n_yt;
  d.capture_len = (uint32_t)n_cap;
  d.flags = cfg.flags | ((n_tg == 0 || n_cap == 0) ? CFGDEV_CLOCK_INVALID : 0);
  d.tz = cfg.tz_offset_sec;
  d.min_post_date = cfg.min_post_date;
  d.zone = c->zone.empty() ? nullptr : c->d_zone.as<ZoneEnt>();
  d.zone_n = (uint32_t)c->zone.size();
  c->cfgdev = d;
  return TGI_OK;
}

uint64_t next_pow2(uint64_t v) {
  uint64_t p = 1;
  while (p < v) p <<= 1;
  return p;
}

// exclusive scan u32[n] -> u64[n+1]; total also lands in *d_total.  A page-sized n takes one launch instead of three
// unless `tiled` asks for the three-launch scan (over `tiles`) at every size.
int launch_scan(tgi_ctx* c, cudaStream_t st, DevBuf& tiles, const uint32_t* in, uint64_t n, uint64_t* out, uint64_t* d_total,
                uint32_t& launches, bool tiled = false) {
  if (!tiled && n <= (uint64_t)SCAN_SMALL_MAX) {
    scan_small_kernel<<<1, SCAN_SMALL_THREADS, 0, st>>>(in, n, out, d_total);
    launches += 1;
    CK(cudaGetLastError());
    return TGI_OK;
  }
  uint64_t ntiles = (n + SCAN_TILE - 1) / SCAN_TILE;
  if (ntiles == 0) ntiles = 1;
  CK(tiles.ensure(ntiles * 8));
  scan_tile_sums_kernel<<<(unsigned)ntiles, SCAN_THREADS, 0, st>>>(in, n, tiles.as<uint64_t>());
  scan_tiles_kernel<<<1, 1024, 0, st>>>(tiles.as<uint64_t>(), ntiles, d_total);
  scan_apply_kernel<<<(unsigned)ntiles, SCAN_THREADS, 0, st>>>(in, n, tiles.as<uint64_t>(), d_total, out);
  launches += 3;
  CK(cudaGetLastError());
  return TGI_OK;
}
int launch_scan(tgi_ctx* c, Slot& s, const uint32_t* in, uint64_t n, uint64_t* out, uint64_t* d_total, uint32_t& launches) {
  return launch_scan(c, s.stream, s.d_tiles, in, n, out, d_total, launches);
}

// The passes of a radix sort of keys up to kmax: over the bits of kmax, 8 bits or fewer each.  The sorted pairs end in
// side `out` of the ping-pong, so a caller that needs them in a given place puts that place there before the sort.
struct RadixPlan {
  uint32_t passes, width;
  int out;
  explicit RadixPlan(uint64_t kmax) {
    uint32_t bits = 0;
    while (bits < 32 && kmax >> bits) bits++;
    passes = (bits + 7) / 8;
    width = passes ? (bits + passes - 1) / passes : 0;
    out = passes & 1;
  }
};

// The stable LSD radix sort (radix.cuh) of the *d_n pairs (keys[0], vals[0]) by key, by plan's passes, the pairs
// ping-ponging between sides 0 and 1; n_max >= *d_n sizes the tiles, counts and roff hold the digit counts and their
// scan, whose total goes to *d_total.  tiled: the scans take their multi-launch form.  Nothing is waited for.
int radix_sort(tgi_ctx* c, cudaStream_t st, DevBuf& tiles, uint32_t* const keys[2], uint32_t* const vals[2], const uint64_t* d_n,
               uint64_t n_max, const RadixPlan& plan, DevBuf& counts, DevBuf& roff, uint64_t* d_total, bool tiled,
               uint32_t& launches) {
  const uint32_t radix = 1u << plan.width;
  const uint64_t ntiles = std::max<uint64_t>((n_max + RS_TILE - 1) / RS_TILE, 1);
  CK(counts.ensure(radix * ntiles * 4));
  CK(roff.ensure((radix * ntiles + 1) * 8));
  int rc;
  for (uint32_t p = 0, cur = 0; p < plan.passes; p++, cur ^= 1) {
    const uint32_t shift = p * plan.width;
    radix_hist_kernel<<<(unsigned)ntiles, RS_WARPS * 32, 0, st>>>(keys[cur], d_n, shift, radix, (uint32_t)ntiles,
                                                                   counts.as<uint32_t>());
    launches++;
    if ((rc = launch_scan(c, st, tiles, counts.as<uint32_t>(), radix * ntiles, roff.as<uint64_t>(), d_total, launches, tiled)))
      return rc;
    radix_scatter_kernel<<<(unsigned)ntiles, RS_WARPS * 32, 0, st>>>(keys[cur], vals[cur], keys[cur ^ 1], vals[cur ^ 1], d_n,
                                                                      shift, radix, (uint32_t)ntiles, roff.as<uint64_t>());
    launches++;
  }
  return TGI_OK;
}

// Sizes the frontier scratch for a batch of n records and `links` links (the hash table holds at least twice as many
// slots, the per-link state covers `lstate_rows`) and returns the kernels' view of it.  The table is not zeroed.
int frontier_scratch(tgi_ctx* c, FrontierScratch& z, uint64_t n, uint64_t links, uint64_t lstate_rows, FrontierBatch& fb) {
  const uint64_t bslots = next_pow2(std::max<uint64_t>(2 * links, 1024));
  CK(z.btable.ensure(bslots * 8));
  CK(z.lstate.ensure((size_t)lstate_rows * 4));
  CK(z.rec_new.ensure(n * 4));
  CK(z.new_off.ensure((n + 1) * 8));
  fb.btable = z.btable.as<uint64_t>();
  fb.bmask = bslots - 1;
  fb.lstate = z.lstate.as<uint32_t>();
  fb.rec_new = z.rec_new.as<uint32_t>();
  return TGI_OK;
}

// The set `which` (TGI_SET_*) names, or nullptr.  With exclusion_only, only the sets the caller fills are named (the
// tgi_set_add / _clear / _size / _export family: the exclusion sets, the urlCache and the chatIDCache).
KeySet* key_set(tgi_ctx* c, int which, bool exclusion_only) {
  if (which == TGI_SET_INVALID || which == TGI_SET_DISCOVERED || which == TGI_SET_URLS || which == TGI_SET_SEEDS)
    return &c->sets[which];
  if (!exclusion_only && (which == TGI_SET_FRONTIER || which == TGI_SET_OWNED)) return &c->sets[which];
  return nullptr;
}
// the kernels' view of the exclusion sets, with the invalid set's TTL checked against now_sec
ExclusionDev exclusion(const tgi_ctx* c, int64_t now_sec) {
  return ExclusionDev{c->sets[TGI_SET_INVALID].dev, c->sets[TGI_SET_DISCOVERED].dev, (long long)now_sec};
}

// An empty device key set of `cap` keys in a table of `tslots` slots (with a u64 payload per key if asked), zeroed on
// slot 0's stream; the caller synchronises.
int set_alloc(tgi_ctx* c, KeySet& k, uint64_t cap, uint64_t tslots, bool payload) {
  cudaStream_t st = c->slots[0].stream;
  CK(k.pool.ensure(cap * 32));
  CK(k.table.ensure(tslots * 8));
  CK(k.count.ensure(16));
  if (payload) CK(k.payload.ensure(cap * 8));
  CK(cudaMemsetAsync(k.table.p, 0, tslots * 8, st));
  CK(cudaMemsetAsync(k.count.p, 0, 16, st));
  FrontierDev& f = k.dev;
  f.pool = k.pool.as<uint8_t>();
  f.cap = cap;
  f.table = k.table.as<uint64_t>();
  f.tmask = tslots - 1;
  f.count = k.count.as<uint64_t>();
  f.payload = payload ? k.payload.as<uint64_t>() : nullptr;
  k.bound = 0;
  k.grows = 0;
  return TGI_OK;
}

// The number of keys in set k (0 while it is not allocated), under fr_mu.  Reads and clears of a set go through slot 0's
// stream (the library's streams are non-blocking: work on the legacy default stream would not be ordered with them) and
// are synchronised before the entry point returns.
int set_count(tgi_ctx* c, const KeySet& k, uint64_t* n) {
  *n = 0;
  if (!k.dev.table) return TGI_OK;
  cudaStream_t st = c->slots[0].stream;
  if (c->fr_event_valid) CK(cudaStreamWaitEvent(st, c->fr_event, 0));
  CK(cudaMemcpyAsync(n, k.dev.count, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return TGI_OK;
}
// empties allocated set k but keeps its capacity and growth steps; the caller orders it behind fr_event and synchronises
int set_clear(tgi_ctx* c, KeySet& k) {
  cudaStream_t st = c->slots[0].stream;
  CK(cudaMemsetAsync(k.dev.table, 0, (k.dev.tmask + 1) * 8, st));
  CK(cudaMemsetAsync(k.dev.count, 0, 8, st));
  k.bound = 0;
  return TGI_OK;
}

// Makes room for up to `need` more keys in set k before a caller inserts them on stream st, when growth is on
// (tgi_set_growth).  Runs under fr_mu, inside the caller's frontier turn.  The host bound decides without a device round
// trip; only when it says the set might overflow is the exact count read, and only when that overflows too does the set
// move into buffers for next_pow2(count + need) keys (at most grow_max): the pool and payload are copied, the bigger
// table is rebuilt by set_rehash_kernel.  Past grow_max the insert still fails with TGI_E_CAPACITY and leaves the set as
// it was.
//
// Freeing the old buffers: kernels take FrontierDev / ExclusionDev by value, so a kernel enqueued earlier may still read
// them.  Every such reader runs under fr_mu and either synchronises its stream before it lets go of the lock (inserts,
// exports, the merge, tgi_pending_edges) or records fr_event behind its kernels (the batches' frontier phases, the page
// kernels).  This function enqueues its work behind fr_event and synchronises st before it frees anything, so every
// earlier reader has finished by then, and later ones see only the new buffers.
int set_grow(tgi_ctx* c, KeySet& k, uint64_t need, cudaStream_t st) {
  const FrontierDev& f = k.dev;
  if (c->grow_max && f.cap < c->grow_max && k.bound + need > f.cap) {
    if (c->fr_event_valid) CK(cudaStreamWaitEvent(st, c->fr_event, 0));
    uint64_t count = 0;
    CK(cudaMemcpyAsync(&count, f.count, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    k.bound = count;
    if (count + need > f.cap) {
      const uint64_t cap = std::min(next_pow2(count + need), c->grow_max), tslots = next_pow2(2 * cap);
      KeySet nb;
      CK(nb.pool.ensure(cap * 32));
      CK(nb.table.ensure(tslots * 8));
      if (f.payload) CK(nb.payload.ensure(cap * 8));
      CK(cudaMemsetAsync(nb.table.p, 0, tslots * 8, st));
      FrontierDev g = f;
      g.pool = nb.pool.as<uint8_t>();
      g.cap = cap;
      g.table = nb.table.as<uint64_t>();
      g.tmask = tslots - 1;
      g.payload = f.payload ? nb.payload.as<uint64_t>() : nullptr;
      if (count) {
        CK(cudaMemcpyAsync(g.pool, f.pool, count * 32, cudaMemcpyDeviceToDevice, st));
        if (f.payload) CK(cudaMemcpyAsync(g.payload, f.payload, count * 8, cudaMemcpyDeviceToDevice, st));
        set_rehash_kernel<<<(unsigned)((count + 255) / 256), 256, 0, st>>>(g, count);
        CK(cudaGetLastError());
      }
      CK(cudaStreamSynchronize(st));
      k.pool.swap(nb.pool);  // nb now holds the old buffers and frees them on return
      k.table.swap(nb.table);
      k.payload.swap(nb.payload);
      k.dev = g;
      k.grows++;
    }
  }
  k.bound += need;
  return TGI_OK;
}

// Enqueues the frontier phases that insert the keys of n records' links into set k on stream st, behind every earlier
// user of the sets (fr_event): make room for `links` more keys (set_grow), size the scratch (a batch table for `links`
// keys, per-link state for `lstate_rows` arena rows), zero the batch table, probe, count, scan, append, commit, and
// record fr_event.  link_start == nullptr: record r is the one link arena[r], and payload[r] (if given) is its key's
// payload.  out_new[0..1] receive the NEW count and the set's size; a full set is left untouched and sets
// ERR_FRONTIER_FULL in *err.  The caller reads both after it synchronises st.  `tiled` asks launch_scan for the
// three-launch scan at every size.  ev0 / ev1 (if given) time the phases.  Runs under fr_mu.
int set_insert(tgi_ctx* c, KeySet& k, cudaStream_t st, uint64_t n, const uint32_t* link_start, const uint32_t* link_count,
               tgi_link* arena, uint64_t links, uint64_t lstate_rows, uint32_t run_flags, const ExclusionDev& x,
               FrontierScratch& z, DevBuf& tiles, bool tiled, uint64_t* out_new, int* err, const uint64_t* payload,
               uint32_t& launches, cudaEvent_t ev0 = nullptr, cudaEvent_t ev1 = nullptr) {
  if (c->fr_event_valid) CK(cudaStreamWaitEvent(st, c->fr_event, 0));
  int rc = set_grow(c, k, links, st);  // at most one new key per link
  if (rc) return rc;
  FrontierBatch fb;
  rc = frontier_scratch(c, z, n, links, lstate_rows, fb);
  if (rc) return rc;
  if (ev0) CK(cudaEventRecord(ev0, st));
  CK(cudaMemsetAsync(fb.btable, 0, (fb.bmask + 1) * 8, st));
  const unsigned g = (unsigned)((n + 255) / 256);
  frontier_probe_kernel<<<g, 256, 0, st>>>(n, link_start, link_count, arena, run_flags, k.dev, fb, x);
  frontier_count_kernel<<<g, 256, 0, st>>>(n, link_start, link_count, fb);
  launches += 2;
  rc = launch_scan(c, st, tiles, fb.rec_new, n, z.new_off.as<uint64_t>(), out_new, launches, tiled);
  if (rc) return rc;
  frontier_append_kernel<<<g, 256, 0, st>>>(n, link_start, link_count, arena, k.dev, fb, z.new_off.as<uint64_t>(), err, payload);
  frontier_commit_kernel<<<1, 1, 0, st>>>(k.dev, z.new_off.as<uint64_t>(), n, out_new, err);
  launches += 2;
  CK(cudaGetLastError());
  if (ev1) CK(cudaEventRecord(ev1, st));
  CK(cudaEventRecord(c->fr_event, st));
  c->fr_event_valid = true;
  return TGI_OK;
}

CfgDev cfg_snapshot(tgi_ctx* c) {
  std::lock_guard<std::mutex> g(c->cfg_mu);
  return c->cfgdev;
}

int h2d(tgi_ctx* c, Slot& s, DevBuf& d, const void* src, size_t bytes) {
  cudaStream_t st = s.stream;
  CK(d.ensure(bytes));
  if (bytes) CK(cudaMemcpyAsync(d.p, src, bytes, cudaMemcpyHostToDevice, st));
  // the pad behind the array: a COPY of zeros, not a memset — a memset is a kernel and would queue behind whatever the
  // other slots' (persistent, SM-filling) kernels are doing, which chains every one of the eleven uploads to them
  CK(cudaMemcpyAsync((uint8_t*)d.p + bytes, c->h_zero.p, PAD, cudaMemcpyHostToDevice, st));
  s.in_bytes += bytes;
  return TGI_OK;
}

// Small read-backs (the scalars block between the size and the emit pass, the validation flag) do NOT go through the copy
// engine: a device->host cudaMemcpyAsync queues behind the other slots' bulk result copies (1.1 GB each at 500 K messages)
// and the slot's host thread then waits for two other slots' result copies to get 96 bytes (TGI_TRACE_SLOTS shows it).  A
// one-warp kernel stores them into mapped pinned memory instead; the host sees them after the stream synchronises.
__global__ void publish_kernel(const uint64_t* src, uint64_t* dst_mapped, int n) {
  if ((int)threadIdx.x < n) dst_mapped[threadIdx.x] = src[threadIdx.x];
  __threadfence_system();
}
int publish(tgi_ctx* c, const void* d_src, HostBuf& h, int n_words, cudaStream_t st) {
  void* dp = nullptr;
  CK(cudaHostGetDevicePointer(&dp, h.p, 0));
  publish_kernel<<<1, 32, 0, st>>>((const uint64_t*)d_src, (uint64_t*)dp, n_words);
  CK(cudaGetLastError());
  return TGI_OK;
}

constexpr uint64_t HOST_VALIDATE_MAX = 1u << 16;  // batches up to this many elements are range-checked on the host

// the checks of tg_validate_kernel, on the host (small batches: no extra launch / sync in a page-sized call)
int host_validate_tg(const tgi_tg_batch* in) {
  const uint64_t n = in->n, n_ents = n ? in->ent_off[n] : 0;
  int e = 0;
  for (uint64_t i = 0; i < n; i++) {
    const tgi_tg_rec& rc = in->recs[i];
    const uint64_t end = rc.str_off + (uint64_t)rc.text_len + rc.alt_len + rc.media_len + rc.handle_len;
    if (end > in->strs_len || end < rc.str_off) e |= 1;
    if (rc.chan_idx >= in->n_chans || rc.content_type >= TGI_CT__COUNT) e |= 2;
    if (in->ent_off[i] > in->ent_off[i + 1]) e |= 4;
    if (in->react_off[i] > in->react_off[i + 1] || in->react_off[i + 1] > in->n_reacts) e |= 8;
    if (in->comment_off[i] > in->comment_off[i + 1] || in->comment_off[i + 1] > in->n_comments) e |= 16;
  }
  if (e) return e;  // the entity count itself comes from ent_off: do not follow it if the offsets are broken
  for (uint64_t i = 0; i < n_ents; i++)
    if (in->ents[i].type == TGI_ENT_TEXT_URL && (uint64_t)in->ents[i].url_off + in->ents[i].url_len > in->aux_len) e |= 32;
  for (uint64_t i = 0; i < in->n_reacts; i++)
    if ((uint64_t)in->reacts[i].emoji_off + in->reacts[i].emoji_len > in->aux_len) e |= 64;
  for (uint64_t i = 0; i < in->n_comments; i++) {
    const tgi_comment& cm = in->comments[i];
    if ((uint64_t)cm.text_off + cm.text_len > in->aux_len || (uint64_t)cm.handle_off + cm.handle_len > in->aux_len) e |= 128;
    if ((cm.flags & 1) && (uint64_t)cm.react_start + cm.react_count > in->n_reacts) e |= 256;
  }
  for (uint32_t i = 0; i < in->n_chans; i++) {
    const tgi_tg_chan& ch = in->chans[i];
    if ((uint64_t)ch.str_off + ch.title_len + ch.name_len + ch.user_len > in->chan_strs_len) e |= 512;
  }
  return e;
}

int validate_tg(tgi_ctx* c, const tgi_tg_batch* in) {
  if (!in) { set_err(c, "null batch"); return TGI_E_ARG; }
  if (in->n && (!in->recs || !in->ent_off || !in->react_off || !in->comment_off || !in->chans)) {
    set_err(c, "telegram batch: recs/ent_off/react_off/comment_off/chans must be non-null");
    return TGI_E_ARG;
  }
  if (in->n >= (1ull << 32)) { set_err(c, "telegram batch: too many records (the work lists hold 32-bit record indices)"); return TGI_E_ARG; }
  if (!(c->cfg.flags & TGI_CFG_SKIP_MEDIA)) {
    set_err(c, "TGI_CFG_SKIP_MEDIA is required: media download is an RPC outside this path");
    return TGI_E_ARG;
  }
  const uint64_t n_ents = in->n ? in->ent_off[in->n] : 0;
  if ((n_ents && !in->ents) || (in->n_reacts && !in->reacts) || (in->n_comments && !in->comments) ||
      (in->strs_len && !in->strs) || (in->aux_len && !in->aux) || (in->chan_strs_len && !in->chan_strs)) {
    set_err(c, "telegram batch: a non-empty array has a null pointer");
    return TGI_E_ARG;
  }
  if (in->n + n_ents + in->n_reacts + in->n_comments + in->n_chans <= HOST_VALIDATE_MAX) {
    const int e = host_validate_tg(in);
    if (e) { set_err(c, "telegram batch: offsets outside their arrays (mask 0x%x)", e); return TGI_E_ARG; }
  }
  return TGI_OK;
}

// CTAs per SM in the grids of the grid-stride kernels.  Records differ in cost (text length, entities, comments), so a
// grid of exactly the resident CTAs leaves SMs idle behind the slowest stride; many more CTAs than fit let the hardware
// scheduler balance: on an H100, 48 and 256 per SM were within 1 % of 128 (TGI_GRID_MULT, DESIGN.md §5)
unsigned grid_mult() {
  static const unsigned v = [] {
    const char* e = getenv("TGI_GRID_MULT");
    return e && atoi(e) > 0 ? (unsigned)atoi(e) : 128u;
  }();
  return v;
}

// ---- page-sized batches: one block in, one launch, one block out (tg_page.cuh, yt_page.cuh) ---------------------------
constexpr uint64_t PAGE_MAX_RECS = 8192;          // the in-kernel scans are single-CTA
constexpr uint64_t PAGE_MAX_IN_BYTES = 4u << 20;
bool page_enabled() {
  return getenv("TGI_NO_PAGE") == nullptr;  // A/B switch (read per call): the ordinary pipeline for every size
}
bool size_text_in_parse() {
  return getenv("TGI_SIZE_TEXT_WARP") == nullptr;  // A/B switch (read per call): the size pass measures every text itself
}
// the size rule of the page kernels, for packing the input and for running it
bool page_fits(uint64_t n, uint64_t n_chans, uint64_t in_bytes) {
  return page_enabled() && n && n <= PAGE_MAX_RECS && n_chans <= PAGE_MAX_RECS && in_bytes <= PAGE_MAX_IN_BYTES;
}
bool page_run_ok(const Slot& s, uint64_t n, uint64_t n_chans, uint32_t flags) {
  if (!page_fits(n, n_chans, s.in_bytes)) return false;
  if (flags & TGI_RUN_NO_D2H) return false;  // a device-resident result keeps the ordinary buffers
  return (flags & (TGI_RUN_JSONL | TGI_RUN_LINKS | TGI_RUN_FRONTIER)) != 0;
}

// A batch's input arrays on their way to the device, each followed by PAD readable zero bytes.
struct InArrays {
  static constexpr int MAX = 11;
  int k = 0;
  const void* src[MAX];
  size_t bytes[MAX];
  DevBuf* buf[MAX];  // the array's own buffer (ordinary upload)
  uint8_t* dev[MAX];  // where it landed
  void add(DevBuf& b, const void* p, size_t n) {
    buf[k] = &b;
    src[k] = p;
    bytes[k] = n;
    k++;
  }
  static size_t packed_size(size_t b) { return (b + PAD + 15) & ~(size_t)15; }
  size_t packed_total() const {
    size_t o = 0;
    for (int i = 0; i < k; i++) o += packed_size(bytes[i]);
    return o;
  }
};
// `packed`: all arrays in one pinned block and ONE copy (a page-sized batch: eleven copies + eleven pad copies are a
// third of what a 100-message call costs otherwise; the pack is a host memcpy of tens of KB).  Otherwise one copy per array.
int upload_arrays(tgi_ctx* c, Slot& s, InArrays& a, bool packed) {
  if (!packed) {
    for (int i = 0; i < a.k; i++) {
      const int rc = h2d(c, s, *a.buf[i], a.src[i], a.bytes[i]);
      if (rc) return rc;
      a.dev[i] = a.buf[i]->as<uint8_t>();
    }
    return TGI_OK;
  }
  const size_t total = a.packed_total();
  CK(s.h_page_in.ensure(total));
  CK(s.d_page_in.ensure(total));
  uint8_t* h = s.h_page_in.as<uint8_t>();
  size_t o = 0;
  for (int i = 0; i < a.k; i++) {
    if (a.bytes[i]) memcpy(h + o, a.src[i], a.bytes[i]);
    memset(h + o + a.bytes[i], 0, InArrays::packed_size(a.bytes[i]) - a.bytes[i]);
    a.dev[i] = s.d_page_in.as<uint8_t>() + o;
    s.in_bytes += a.bytes[i];
    o += InArrays::packed_size(a.bytes[i]);
  }
  CK(cudaMemcpyAsync(s.d_page_in.p, h, total, cudaMemcpyHostToDevice, s.stream));
  return TGI_OK;
}

int upload_tg(tgi_ctx* c, Slot& s, const tgi_tg_batch* in) {
  int rc = validate_tg(c, in);
  if (rc) return rc;
  trace_slot(s, "upload: enqueue");
  uint64_t n = in->n;
  s.in_bytes = 0;
  uint64_t n_ents = n ? in->ent_off[n] : 0;
  InArrays a;
  a.add(s.d_recs, in->recs, n * sizeof(tgi_tg_rec));
  a.add(s.d_strs, in->strs, in->strs_len);
  a.add(s.d_ent_off, in->ent_off, (n + 1) * 4);
  a.add(s.d_ents, in->ents, n_ents * sizeof(tgi_entity));
  a.add(s.d_react_off, in->react_off, (n + 1) * 4);
  a.add(s.d_reacts, in->reacts, in->n_reacts * sizeof(tgi_reaction));
  a.add(s.d_comment_off, in->comment_off, (n + 1) * 4);
  a.add(s.d_comments, in->comments, in->n_comments * sizeof(tgi_comment));
  a.add(s.d_aux, in->aux, in->aux_len);
  a.add(s.d_chans, in->chans, in->n_chans * sizeof(tgi_tg_chan));
  a.add(s.d_chan_strs, in->chan_strs, in->chan_strs_len);
  // small batches were range-checked on the host by validate_tg; the others are checked on the device below
  const bool host_checked = n + n_ents + in->n_reacts + in->n_comments + in->n_chans <= HOST_VALIDATE_MAX;
  rc = upload_arrays(c, s, a, host_checked && page_fits(n, in->n_chans, a.packed_total()));
  if (rc) return rc;
  TgBatchDev& b = s.tg;
  b.n = n;
  b.recs = (const tgi_tg_rec*)a.dev[0];
  b.strs = a.dev[1];
  b.ent_off = (const uint32_t*)a.dev[2];
  b.ents = (const tgi_entity*)a.dev[3];
  b.react_off = (const uint32_t*)a.dev[4];
  b.reacts = (const tgi_reaction*)a.dev[5];
  b.comment_off = (const uint32_t*)a.dev[6];
  b.comments = (const tgi_comment*)a.dev[7];
  b.aux = a.dev[8];
  b.n_chans = in->n_chans;
  b.chans = (const tgi_tg_chan*)a.dev[9];
  b.chan_strs = a.dev[10];
  s.n_ents = n_ents;
  s.n_reacts = in->n_reacts;
  s.n_comments = in->n_comments;
  s.chan_strs_len = in->chan_strs_len;
  if (!host_checked) {
    CK(s.d_scalars.ensure(SC_COUNT * 8));
    int* bad = (int*)s.d_scalars.p;
    CK(cudaMemsetAsync(bad, 0, 4, s.stream));
    TgBounds lim{in->strs_len, n_ents, in->n_reacts, in->n_comments, in->aux_len, in->chan_strs_len};
    const uint64_t count = std::max<uint64_t>({n, n_ents, in->n_reacts, in->n_comments, (uint64_t)in->n_chans});
    tg_validate_kernel<<<(unsigned)((count + 255) / 256), 256, 0, s.stream>>>(b, lim, count, bad);
    CK(s.h_scalars.ensure(SC_COUNT * 8));
    {
      const int prc = publish(c, bad, s.h_scalars, 1, s.stream);
      if (prc) return prc;
    }
    CK(cudaStreamSynchronize(s.stream));
    const int hbad = *s.h_scalars.as<int>();
    trace_slot(s, "upload: landed + validated");
    if (hbad) { set_err(c, "telegram batch: offsets outside their arrays (mask 0x%x)", hbad); return TGI_E_ARG; }
  }
  return TGI_OK;
}

// ---- frontier turns ---------------------------------------------------------------------------------------------------
void turn_begin(tgi_ctx* c, Slot& s) {
  if (!s.has_ticket) return;
  std::unique_lock<std::mutex> lk(c->tk_mu);
  c->tk_cv.wait(lk, [&] { return c->tk_serving == s.ticket; });
}
void turn_end(tgi_ctx* c, Slot& s) {
  if (!s.has_ticket) return;
  {
    std::lock_guard<std::mutex> g(c->tk_mu);
    c->tk_serving++;
    s.has_ticket = false;
  }
  c->tk_cv.notify_all();
}
// a job that ended without a frontier phase (error, empty batch) still has to let the next ticket through
void turn_pass(tgi_ctx* c, Slot& s) {
  if (!s.has_ticket) return;
  turn_begin(c, s);
  turn_end(c, s);
}

// ---- results ----------------------------------------------------------------------------------------------------------
uint32_t sc_cursor(const uint64_t* hsc) { return ((const uint32_t*)(hsc + SC_CURSOR))[0]; }
int sc_err(const uint64_t* hsc) { return ((const int*)(hsc + SC_CURSOR))[1]; }

// the device errors that fail a batch once it has run to the end
int check_dev_err(tgi_ctx* c, int err) {
  if (err & ERR_FRONTIER_FULL) { set_err(c, "frontier capacity %llu exceeded", (unsigned long long)c->sets[TGI_SET_FRONTIER].dev.cap); return TGI_E_CAPACITY; }
  if (err & ERR_LINE_MISMATCH) { set_err(c, "internal: sized and emitted line lengths disagree"); return TGI_E_STATE; }
  return TGI_OK;
}
int check_max_out(tgi_ctx* c, uint64_t line_total) {
  if (c->cfg.max_out_bytes && line_total > c->cfg.max_out_bytes) {
    set_err(c, "JSONL output %llu bytes exceeds max_out_bytes", (unsigned long long)line_total);
    return TGI_E_CAPACITY;
  }
  return TGI_OK;
}

// Fills *out, the slot's last result (the readers') and the context stats from a batch that has run to the end; hsc is
// its scalars block on the host.  `host` is nullptr when the result stays on the device.
void fill_result(tgi_ctx* c, Slot& s, RecKind kind, uint64_t n, uint32_t flags, const uint64_t* hsc, uint64_t line_total,
                 uint32_t launches, const ResultArrays* host, const ResultArrays& dev, tgi_result* out) {
  const bool want_json = flags & TGI_RUN_JSONL, want_links = flags & TGI_RUN_LINKS, want_fr = flags & TGI_RUN_FRONTIER;
  memset(out, 0, sizeof *out);
  out->n = n;
  float ms = 0;
  cudaEventElapsedTime(&ms, s.ev_k0, s.ev_k1);
  out->kernel_ms = ms;
  out->gpu_launches = launches;
  out->slot = s.idx;
  if (n && want_json) {
    out->var_bytes = hsc[SC_LONG];
    out->main_bytes_out = hsc[SC_LANE_OUT];
    out->main_bytes_in = hsc[SC_LANE_IN];
  }
  out->jsonl_len = want_json ? line_total : 0;
  out->n_links = want_links ? hsc[SC_LINK_TOTAL] : 0;
  out->n_new = want_fr ? hsc[SC_NEW] : 0;
  out->frontier_size = want_fr ? hsc[SC_FSIZE] : 0;
  if (host) {
    out->status = host->status;
    if (want_json) {
      out->jsonl = (flags & TGI_RUN_JSONL_DEVICE) ? nullptr : host->jsonl;
      out->line_off = host->line_off;
    }
    if (want_links) {
      out->link_off = host->link_off;
      out->links = host->links;
    }
  }
  s.last = LastResult{kind, n, flags, out->n_new, out->n_links, out->jsonl_len,
                      {dev.status, want_json ? dev.line_off : nullptr, dev.jsonl, want_links ? dev.link_off : nullptr,
                       want_links ? dev.links : nullptr},
                      host && want_json ? host->line_off : nullptr};
  std::lock_guard<std::mutex> g(c->st_mu);
  c->stats.records += n;
  c->stats.bytes_in += s.in_bytes;
  c->stats.bytes_out += out->jsonl_len;
  c->stats.links += out->n_links;
  c->stats.launches += launches;
  c->stats.kernel_ms_total += ms;
  if (want_fr) c->stats.frontier_size = out->frontier_size;
}

// ---- bulk batches -----------------------------------------------------------------------------------------------------
// the scalars block (device + mapped pinned mirror) and the per-record arrays every bulk pipeline writes; starts the
// batch's kernel clock and zeroes the scalars
int bulk_prologue(tgi_ctx* c, Slot& s, uint64_t n) {
  CK(s.d_scalars.ensure(SC_COUNT * 8));
  CK(s.h_scalars.ensure(SC_COUNT * 8));
  CK(s.d_status.ensure(n));
  CK(s.d_linelen.ensure(n * 4));
  CK(s.d_line_off.ensure((n + 1) * 8));
  CK(s.d_link_start.ensure(n * 4));
  CK(s.d_link_count.ensure(n * 4));
  CK(cudaEventRecord(s.ev_k0, s.stream));
  CK(cudaMemsetAsync(s.d_scalars.p, 0, SC_COUNT * 8, s.stream));
  return TGI_OK;
}

struct Totals {
  uint64_t line_total;
  uint32_t cursor;  // the link arena's fill
  int err;
};
// Between the size and the emit pass: scan the line lengths, publish the scalars block, wait for it and decode it.  An
// arena overflow comes back in t.err for the caller to handle; the other device errors and max_out_bytes fail the batch.
int bulk_totals(tgi_ctx* c, Slot& s, uint64_t n, bool want_json, uint32_t& launches, Totals& t) {
  uint64_t* dsc = s.d_scalars.as<uint64_t>();
  const uint64_t* hsc = s.h_scalars.as<uint64_t>();
  if (want_json) {
    const int rc = launch_scan(c, s, s.d_linelen.as<uint32_t>(), n, s.d_line_off.as<uint64_t>(), dsc + SC_LINE_TOTAL, launches);
    if (rc) return rc;
  }
  CK(cudaGetLastError());
  const int rc = publish(c, dsc, s.h_scalars, SC_COUNT, s.stream);
  if (rc) return rc;
  launches++;
  trace_slot(s, "parse + size: enqueued");
  CK(cudaStreamSynchronize(s.stream));
  trace_slot(s, "parse + size: done");
  t.line_total = hsc[SC_LINE_TOTAL];
  t.cursor = sc_cursor(hsc);
  t.err = sc_err(hsc);
  if (t.err & ERR_ARENA_OVERFLOW) return TGI_OK;
  if (t.err & ERR_TOO_MANY_LINKS) { set_err(c, "a record has 2^20 or more link candidates"); return TGI_E_ARG; }
  return want_json ? check_max_out(c, t.line_total) : TGI_OK;
}

// shared tail of the bulk pipelines: frontier phases, link compaction, D2H, result
int finish_batch(tgi_ctx* c, Slot& s, RecKind kind, uint64_t n, uint32_t flags, uint64_t line_total, uint32_t arena_used,
                 uint64_t arena_cap, uint32_t launches, tgi_result* out) {
  cudaStream_t st = s.stream;
  const bool want_json = flags & TGI_RUN_JSONL, want_links = flags & TGI_RUN_LINKS, want_fr = flags & TGI_RUN_FRONTIER;
  uint64_t* dsc = s.d_scalars.as<uint64_t>();
  uint64_t* hsc = s.h_scalars.as<uint64_t>();

  if (want_fr && n) {
    // frontier phases of different slots are serialised in submission order (tickets)
    turn_begin(c, s);
    std::unique_lock<std::mutex> fg(c->fr_mu);
    const int rc = set_insert(c, c->sets[TGI_SET_FRONTIER], st, n, s.d_link_start.as<uint32_t>(), s.d_link_count.as<uint32_t>(),
                              s.d_arena.as<tgi_link>(), arena_used, arena_cap, flags, exclusion(c, c->now_sec), s.fs, s.d_tiles,
                              false, dsc + SC_NEW, (int*)(dsc + SC_CURSOR) + 1, nullptr, launches, s.ev_fr0, s.ev_fr1);
    if (rc) return rc;
    fg.unlock();
    turn_end(c, s);
  }
  if (want_links) {
    CK(s.d_link_off.ensure((n + 1) * 8));
    CK(s.d_link_off32.ensure((n + 1) * 4));
    int rc = launch_scan(c, s, s.d_link_count.as<uint32_t>(), n, s.d_link_off.as<uint64_t>(), dsc + SC_LINK_TOTAL, launches);
    if (rc) return rc;
    CK(s.d_links_out.ensure((size_t)arena_used * sizeof(tgi_link) + 64));
    unsigned g = (unsigned)((n + 1 + 255) / 256);
    links_compact_kernel<<<g, 256, 0, st>>>(n, s.d_link_start.as<uint32_t>(), s.d_link_count.as<uint32_t>(),
                                            s.d_link_off.as<uint64_t>(), s.d_arena.as<tgi_link>(),
                                            s.d_links_out.as<tgi_link>(), s.d_link_off32.as<uint32_t>());
    launches++;
    CK(cudaGetLastError());
  }
  CK(cudaEventRecord(s.ev_k1, st));
  CK(cudaMemcpyAsync(hsc, dsc, SC_COUNT * 8, cudaMemcpyDeviceToHost, st));

  const bool d2h = !(flags & TGI_RUN_NO_D2H);
  if (d2h) {
    CK(s.h_status.ensure(n + 1));
    CK(cudaMemcpyAsync(s.h_status.p, s.d_status.p, n, cudaMemcpyDeviceToHost, st));
    if (want_json) {
      CK(s.h_line_off.ensure((n + 1) * 8));
      if (!(flags & TGI_RUN_JSONL_DEVICE)) CK(s.h_jsonl.ensure(line_total + 1));  // the lines may stay on the device
      CK(cudaMemcpyAsync(s.h_line_off.p, s.d_line_off.p, (n + 1) * 8, cudaMemcpyDeviceToHost, st));
      if (line_total && !(flags & TGI_RUN_JSONL_DEVICE)) CK(cudaMemcpyAsync(s.h_jsonl.p, s.d_jsonl.p, line_total, cudaMemcpyDeviceToHost, st));
    }
    if (want_links) {
      // the exact link count is one more host round trip away (behind the other slots' bulk copies on the copy engine);
      // the arena's fill is an upper bound the host already has: copy that many rows, the tail past n_links is unused
      CK(s.h_link_off.ensure((n + 1) * 4));
      CK(s.h_links.ensure((size_t)arena_used * sizeof(tgi_link) + 64));
      CK(cudaMemcpyAsync(s.h_link_off.p, s.d_link_off32.p, (n + 1) * 4, cudaMemcpyDeviceToHost, st));
      if (arena_used) CK(cudaMemcpyAsync(s.h_links.p, s.d_links_out.p, (size_t)arena_used * sizeof(tgi_link), cudaMemcpyDeviceToHost, st));
    }
  }
  trace_slot(s, "emit + frontier + result copy: enqueued");
  CK(cudaStreamSynchronize(st));
  trace_slot(s, "result landed");
  const int rc = check_dev_err(c, sc_err(hsc));
  if (rc) return rc;
  if (want_links && hsc[SC_LINK_TOTAL] > arena_used) { set_err(c, "internal: more links than arena rows"); return TGI_E_STATE; }
  const ResultArrays dev{s.d_status.as<uint8_t>(), s.d_line_off.as<uint64_t>(), s.d_jsonl.as<uint8_t>(), s.d_link_off32.as<uint32_t>(),
                         s.d_links_out.as<tgi_link>()};
  const ResultArrays host{s.h_status.as<uint8_t>(), s.h_line_off.as<uint64_t>(), s.h_jsonl.as<uint8_t>(), s.h_link_off.as<uint32_t>(),
                          s.h_links.as<tgi_link>()};
  fill_result(c, s, kind, n, flags, hsc, line_total, launches, d2h ? &host : nullptr, dev, out);
  if (n) cudaEventElapsedTime(&out->parse_ms, s.ev_p0, s.ev_p1);
  if (n && want_json) {
    cudaEventElapsedTime(&out->emit_ms, s.ev_e0, s.ev_e1);
    cudaEventElapsedTime(&out->emit_main_ms, s.ev_e0, s.ev_f1);
  }
  if (want_fr && n) cudaEventElapsedTime(&out->frontier_ms, s.ev_fr0, s.ev_fr1);
  return TGI_OK;
}

// the outputs of the Telegram parse / size passes, for a link arena of arena_cap rows
ParseOut tg_parse_out(Slot& s, uint8_t* status, uint64_t* dsc, uint64_t arena_cap) {
  ParseOut po;
  po.status = status;
  po.linelen = s.d_linelen.as<uint32_t>();
  po.link_start = s.d_link_start.as<uint32_t>();
  po.link_count = s.d_link_count.as<uint32_t>();
  po.xlen = s.d_xlen.as<uint32_t>();
  po.var_total = (unsigned long long*)(dsc + SC_LONG);
  po.arena = s.d_arena.as<tgi_link>();
  po.arena_cap = (uint32_t)arena_cap;
  po.cursor = (uint32_t*)(dsc + SC_CURSOR);
  po.err = (int*)(dsc + SC_CURSOR) + 1;
  po.ent_range = s.d_ent_range.as<int2>();
  return po;
}
// what the Telegram emit passes read and write besides the batch (ei.out: the caller's)
EmitIn tg_emit_in(Slot& s, const ParseOut& po, const uint64_t* line_off, uint64_t* dsc, uint64_t n) {
  EmitIn ei;
  ei.status = po.status;
  ei.line_off = line_off;
  ei.link_start = po.link_start;
  ei.link_count = po.link_count;
  ei.xlen = po.xlen;
  ei.xpos = s.d_xpos.as<uint32_t>();
  ei.arena = po.arena;
  ei.out = nullptr;
  ei.err = po.err;
  ei.lane_text_max = LANE_TEXT_MAX;
  ei.counters = (unsigned long long*)(dsc + SC_LANE_OUT);
  for (int k = 0; k < 3; k++) ei.list[k] = s.d_lists.as<uint32_t>() + (size_t)k * n;  // record indices: n < 2^32 checked at upload
  ei.list_count = (uint32_t*)(dsc + SC_LISTS);
  return ei;
}
// The outputs of the YouTube parse / size passes.  Upper bounds on the capacities: every URL needs "http://x"
// (8 bytes), every channel link "youtube.com/" (12 bytes).
uint64_t yt_arena_cap(const Slot& s) { return s.yt_desc_bytes / 12 + 1024; }
int yt_parse_out(tgi_ctx* c, Slot& s, uint64_t n, uint8_t* status, uint64_t* dsc, YtOut& yo) {
  const uint64_t urls_cap = s.yt_desc_bytes / 4 + 1024, arena_cap = yt_arena_cap(s);
  CK(s.d_linelen.ensure(n * 4));
  CK(s.d_link_start.ensure(n * 4));
  CK(s.d_link_count.ensure(n * 4));
  CK(s.d_url_start.ensure(n * 4));
  CK(s.d_url_count.ensure(n * 4));
  CK(s.d_urls.ensure(urls_cap * sizeof(YtUrl)));
  CK(s.d_arena.ensure(arena_cap * sizeof(tgi_link)));
  CK(s.d_xlen.ensure(n * 12));
  yo.status = status;
  yo.linelen = s.d_linelen.as<uint32_t>();
  yo.esc_len = s.d_xlen.as<uint32_t>();
  yo.url_start = s.d_url_start.as<uint32_t>();
  yo.url_count = s.d_url_count.as<uint32_t>();
  yo.urls = s.d_urls.as<YtUrl>();
  yo.urls_cap = (uint32_t)std::min<uint64_t>(urls_cap, 0xFFFFFFFFu);
  yo.url_cursor = (uint32_t*)(dsc + SC_URL_CURSOR);
  yo.link_start = s.d_link_start.as<uint32_t>();
  yo.link_count = s.d_link_count.as<uint32_t>();
  yo.arena = s.d_arena.as<tgi_link>();
  yo.arena_cap = (uint32_t)std::min<uint64_t>(arena_cap, 0xFFFFFFFFu);
  yo.cursor = (uint32_t*)(dsc + SC_CURSOR);
  yo.err = (int*)(dsc + SC_CURSOR) + 1;
  return TGI_OK;
}

// ---- page batches: one cooperative launch and one result copy -----------------------------------------------------------
// PAGE_FALLBACK: the batch did not fit the estimate-sized result block or the link arena (nothing was committed): the
// caller goes on with the bulk pipeline on the same resident input.
constexpr int PAGE_FALLBACK = -1000;
int page_occupancy(const void* kernel) {  // resident CTAs per SM of a page kernel; 0: no page launches
  int o = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, kernel, CTA_THREADS, 0) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return o;
}
struct PageOut {  // the result block: scalars | status | line_off | link_off | links, JSONL
  uint64_t o_status, o_line_off, o_link_off, o_var, var_cap;
  uint64_t links_max;  // the link arena's capacity: an upper bound of the keys the page adds to the frontier
};
// Lays out and sizes the result block and the frontier scratch, and fills the kernel's result arguments but for the
// frontier and the exclusion sets, which page_launch_and_read reads under the frontier lock.
int page_prepare(tgi_ctx* c, Slot& s, uint64_t n, uint64_t arena_cap, uint32_t flags, PageOut& L, PageResult& r) {
  auto up = [](uint64_t v, uint64_t a) { return (v + a - 1) / a * a; };
  L.o_status = 256;
  L.o_line_off = L.o_status + up(n + 1, 16);
  L.o_link_off = L.o_line_off + (n + 1) * 8;
  L.o_var = up(L.o_link_off + (n + 1) * 4, 256);
  L.var_cap = up(6 * s.in_bytes + 3072 * n + 65536, 256);
  L.links_max = arena_cap;
  if (const char* v = getenv("TGI_PAGE_VAR_CAP")) L.var_cap = up(strtoull(v, nullptr, 10), 256);  // tests: force the fallback
  CK(s.d_page_out.ensure(L.o_var + L.var_cap));
  CK(s.h_page_out.ensure(L.o_var + L.var_cap));
  CK(s.d_link_off.ensure((n + 1) * 8));
  if (flags & TGI_RUN_FRONTIER) {
    const int rc = frontier_scratch(c, s.fs, n, arena_cap, arena_cap, r.fb);
    if (rc) return rc;
    r.bslots = r.fb.bmask + 1;
  }
  uint8_t* d = s.d_page_out.as<uint8_t>();
  r.scalars = (uint64_t*)d;
  r.line_off = (uint64_t*)(d + L.o_line_off);
  r.link_off = s.d_link_off.as<uint64_t>();
  r.link_off32 = (uint32_t*)(d + L.o_link_off);
  r.var = d + L.o_var;
  r.var_cap = L.var_cap;
  r.max_out = c->cfg.max_out_bytes;
  r.new_off = s.fs.new_off.as<uint64_t>();
  return TGI_OK;
}
// launch (in the batch's frontier turn), ONE read of the result block, the result.  PAGE_FALLBACK: nothing was committed.
int page_launch_and_read(tgi_ctx* c, Slot& s, RecKind kind, uint32_t flags, uint64_t n, const void* kernel, void** kargs, int occ,
                         const PageOut& L, PageResult& r, const char* name, tgi_result* out) {
  cudaStream_t st = s.stream;
  const bool want_json = flags & TGI_RUN_JSONL, want_links = flags & TGI_RUN_LINKS, want_fr = flags & TGI_RUN_FRONTIER;
  auto up = [](uint64_t v, uint64_t a) { return (v + a - 1) / a * a; };
  uint8_t* d = s.d_page_out.as<uint8_t>();
  uint8_t* h = s.h_page_out.as<uint8_t>();
  const unsigned grid = (unsigned)std::min<uint64_t>((uint64_t)c->sms * occ, std::max<uint64_t>(1, (n + WARPS_PER_CTA - 1) / WARPS_PER_CTA));
  {
    // the launch holds frontier phases: serialised with the other slots' in submission order, like finish_batch
    std::unique_lock<std::mutex> fg(c->fr_mu, std::defer_lock);
    if (want_fr) {
      turn_begin(c, s);
      fg.lock();
      if (c->fr_event_valid) CK(cudaStreamWaitEvent(st, c->fr_event, 0));
      KeySet& fr = c->sets[TGI_SET_FRONTIER];
      r.fr = fr.dev;
      r.excl = exclusion(c, c->now_sec);
      fr.bound += L.links_max;
    }
    CK(cudaEventRecord(s.ev_k0, st));
    if (cudaLaunchCooperativeKernel(kernel, dim3(grid), dim3(CTA_THREADS), kargs, 0, st) != cudaSuccess) {
      cudaGetLastError();  // e.g. the device is shared and cannot hold the grid: the bulk pipeline needs no co-residency
      return PAGE_FALLBACK;
    }
    CK(cudaEventRecord(s.ev_k1, st));
    if (want_fr) {
      CK(cudaEventRecord(c->fr_event, st));
      c->fr_event_valid = true;
    }
  }
  // ONE read of the result block, sized by what the previous pages needed; a second one only for the rest of a bigger page
  const uint64_t spec = std::min<uint64_t>(L.var_cap, up((uint64_t)s.page_bpr * n * 5 / 4 + 4096, 256));
  CK(cudaMemcpyAsync(h, d, L.o_var + spec, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const uint64_t* hsc = (const uint64_t*)h;
  const int dev_err = sc_err(hsc);
  if (dev_err & (ERR_ARENA_OVERFLOW | ERR_TOO_MANY_LINKS | ERR_PAGE_OVERFLOW)) return PAGE_FALLBACK;  // keeps its turn
  // a full frontier left the set untouched: with growth on, the bulk pipeline grows it and runs the page again
  if ((dev_err & ERR_FRONTIER_FULL) && c->grow_max) return PAGE_FALLBACK;
  turn_end(c, s);
  int rc = check_dev_err(c, dev_err);
  if (rc) return rc;
  const uint64_t line_total = want_json ? hsc[SC_LINE_TOTAL] : 0, n_links_total = want_links ? hsc[SC_LINK_TOTAL] : 0;
  const uint64_t links_bytes = want_links ? up(n_links_total * sizeof(tgi_link), 256) : 0;
  rc = check_max_out(c, line_total);
  if (rc) return rc;
  const uint64_t need = links_bytes + ((flags & TGI_RUN_JSONL_DEVICE) ? 0 : line_total);  // the lines may stay behind
  if (need > spec) {
    CK(cudaMemcpyAsync(h + L.o_var + spec, d + L.o_var + spec, need - spec, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  if (getenv("TGI_PAGE_TRACE")) {
    const uint64_t* t = hsc + PAGE_TRACE_AT;
    fprintf(stderr, "%s n=%llu grid=%u phases us:", name, (unsigned long long)n, grid);
    for (int k = 0; k < PAGE_PHASES; k++) fprintf(stderr, " P%d %.1f", k, (double)(t[k + 1] - t[k]) * 1e-3);
    fprintf(stderr, "  total %.1f |", (double)(t[PAGE_PHASES] - t[0]) * 1e-3);
    static const char* const what[3] = {"parse", "size", "emit"};
    for (int k = 0; k < 3; k++)  // SM cycles (1.965 GHz)
      fprintf(stderr, " slowest %s: rec %u %.1f us", what[k], (unsigned)t[PAGE_PHASES + 1 + k], (double)(t[PAGE_PHASES + 1 + k] >> 32) / 1965.0);
    fprintf(stderr, "\n");
  }
  // the estimate learns from whole results only: a result whose lines stayed behind would under-size the next read
  if (!(flags & TGI_RUN_JSONL_DEVICE))
    s.page_bpr = (uint32_t)std::min<uint64_t>(1u << 20, (3ull * s.page_bpr + need / n + 1) / 4 + (need > spec ? need / n / 4 : 0));
  const ResultArrays dev{d + L.o_status, (const uint64_t*)(d + L.o_line_off), d + L.o_var + links_bytes, (const uint32_t*)(d + L.o_link_off),
                         (const tgi_link*)(d + L.o_var)};
  const ResultArrays host{h + L.o_status, (const uint64_t*)(h + L.o_line_off), h + L.o_var + links_bytes, (const uint32_t*)(h + L.o_link_off),
                          (const tgi_link*)(h + L.o_var)};
  fill_result(c, s, kind, n, flags, hsc, line_total, 1, &host, dev, out);
  return TGI_OK;
}

int run_tg_page(tgi_ctx* c, Slot& s, uint32_t flags, tgi_result* out) {
  TgBatchDev& b = s.tg;
  const uint64_t n = b.n;
  static const int occ = page_occupancy((const void*)tg_page_kernel);
  if (occ <= 0) return PAGE_FALLBACK;
  PageArgs pa{};
  pa.cfg = cfg_snapshot(c);
  pa.run_flags = flags;
  const uint64_t arena_cap = s.n_ents + 2 * n + 1024;
  const uint64_t blob_cap = 8 * s.chan_strs_len + 1024ull * b.n_chans + 1024;
  // scratch (the buffers of the ordinary pipeline, so that tgi_pending_edges finds the same arrays afterwards)
  CK(s.d_linelen.ensure(n * 4));
  CK(s.d_link_start.ensure(n * 4));
  CK(s.d_link_count.ensure(n * 4));
  CK(s.d_xlen.ensure(n * 32));
  CK(s.d_xpos.ensure(n * 32));
  CK(s.d_lists.ensure(3 * n * 4));
  CK(s.d_arena.ensure(arena_cap * sizeof(tgi_link)));
  CK(s.d_ent_range.ensure((size_t)s.n_ents * sizeof(int2)));
  CK(s.d_chan_derived.ensure((size_t)b.n_chans * sizeof(ChanDerived)));
  CK(s.d_chan_len.ensure((size_t)b.n_chans * 4));
  CK(s.d_chan_off.ensure(((size_t)b.n_chans + 1) * 8));
  CK(s.d_chan_blob.ensure(blob_cap));
  PageOut L;
  const int rc = page_prepare(c, s, n, arena_cap, flags, L, pa.res);
  if (rc) return rc;
  b.chan_derived = s.d_chan_derived.as<ChanDerived>();
  b.chan_blob = s.d_chan_blob.as<uint8_t>();
  pa.b = b;
  pa.po = tg_parse_out(s, s.d_page_out.as<uint8_t>() + L.o_status, pa.res.scalars, arena_cap);
  pa.ei = tg_emit_in(s, pa.po, pa.res.line_off, pa.res.scalars, n);
  pa.chan_derived = s.d_chan_derived.as<ChanDerived>();
  pa.chan_len = s.d_chan_len.as<uint32_t>();
  pa.chan_off = s.d_chan_off.as<uint64_t>();
  pa.chan_blob = s.d_chan_blob.as<uint8_t>();
  pa.chan_blob_cap = blob_cap;
  void* kargs[] = {&pa};
  return page_launch_and_read(c, s, REC_TG, flags, n, (const void*)tg_page_kernel, kargs, occ, L, pa.res, "tg_page", out);
}

int run_tg(tgi_ctx* c, Slot& s, uint32_t flags, tgi_result* out) {
  TgBatchDev& b = s.tg;
  uint64_t n = b.n;
  cudaStream_t st = s.stream;
  uint32_t launches = 0;
  const bool want_json = flags & TGI_RUN_JSONL;
  if (page_run_ok(s, n, b.n_chans, flags)) {
    const int rc = run_tg_page(c, s, flags, out);
    if (rc != PAGE_FALLBACK) return rc;
  }
  const CfgDev cfg = cfg_snapshot(c);
  CK(s.d_xlen.ensure(n * 32));
  CK(s.d_ent_range.ensure((size_t)s.n_ents * sizeof(int2)));
  uint64_t arena_cap = s.n_ents + n / 2 + 1024;
  if (s.d_arena.cap / sizeof(tgi_link) > arena_cap + 8) arena_cap = (s.d_arena.cap - PAD) / sizeof(tgi_link);
  int rc = bulk_prologue(c, s, n);
  if (rc) return rc;
  uint64_t* dsc = s.d_scalars.as<uint64_t>();
  const uint64_t* hsc = s.h_scalars.as<uint64_t>();

  Totals t{};
  ParseOut po{};
  for (int attempt = 0; attempt < 3; attempt++) {
    if (attempt) CK(cudaMemsetAsync(dsc, 0, SC_COUNT * 8, st));  // the rerun starts from zeroed scalars
    CK(s.d_arena.ensure(arena_cap * sizeof(tgi_link)));
    if (want_json) {
      CK(s.d_chan_derived.ensure((size_t)b.n_chans * sizeof(ChanDerived)));
      CK(s.d_chan_len.ensure((size_t)b.n_chans * 4));
      CK(s.d_chan_off.ensure(((size_t)b.n_chans + 1) * 8));
      b.chan_derived = s.d_chan_derived.as<ChanDerived>();
      unsigned g = (b.n_chans + WARPS_PER_CTA - 1) / WARPS_PER_CTA;
      if (g) {
        tg_chan_size_kernel<<<g, CTA_THREADS, 0, st>>>(b, s.d_chan_derived.as<ChanDerived>(), s.d_chan_len.as<uint32_t>());
        launches++;
      }
      rc = launch_scan(c, s, s.d_chan_len.as<uint32_t>(), b.n_chans, s.d_chan_off.as<uint64_t>(), dsc + SC_CHAN_TOTAL, launches);
      if (rc) return rc;
    }
    po = tg_parse_out(s, s.d_status.as<uint8_t>(), dsc, arena_cap);
    if (n) {
      CK(cudaEventRecord(s.ev_p0, st));
      const uint64_t groups = (n + 31) / 32;
      unsigned ge = (unsigned)std::min<uint64_t>((groups + WARPS_PER_CTA - 1) / WARPS_PER_CTA, (uint64_t)c->sms * grid_mult());
      // JSONL: the link count measures the message texts as well (the size pass then skips the clean ones); runs without
      // JSONL take the instances without that code
      const bool measure = want_json && size_text_in_parse();
      // status, link bounds, the entity offsets of ASCII texts and the links of the records without entities; then the
      // entity offsets of the other texts; then the links of the records with entities (three kernels by instruction
      // footprint)
      if (measure) tg_parse_kernel<true><<<ge, CTA_THREADS, 0, st>>>(b, cfg, flags, po);
      else tg_parse_kernel<false><<<ge, CTA_THREADS, 0, st>>>(b, cfg, flags, po);
      launches++;
      if (s.n_ents) {
        tg_ent_map_kernel<<<ge, CTA_THREADS, 0, st>>>(b, po);
        tg_parse_ent_kernel<<<ge, CTA_THREADS, 0, st>>>(b, po);
        launches += 2;
      }
      if (want_json) {
        tg_size_lane_kernel<<<ge, CTA_THREADS, 0, st>>>(b, cfg, po);
        launches++;
      }
      CK(cudaEventRecord(s.ev_p1, st));
    }
    rc = bulk_totals(c, s, n, want_json, launches, t);
    if (rc) return rc;
    if (!(t.err & ERR_ARENA_OVERFLOW)) break;
    arena_cap = (uint64_t)t.cursor + 1024;  // exact demand is known now: rerun the parse
  }
  if (t.err & ERR_ARENA_OVERFLOW) { set_err(c, "link arena overflow persisted"); return TGI_E_CAPACITY; }
  const uint64_t chan_total = hsc[SC_CHAN_TOTAL];

  if (want_json) {
    CK(s.d_chan_blob.ensure(chan_total));
    CK(s.d_jsonl.ensure(t.line_total));
    if (chan_total) CK(cudaMemsetAsync(s.d_chan_blob.p, 0, chan_total, st));  // segment padding must read as zero
    b.chan_blob = s.d_chan_blob.as<uint8_t>();
    unsigned g = (b.n_chans + WARPS_PER_CTA - 1) / WARPS_PER_CTA;
    if (g) {
      tg_chan_emit_kernel<<<g, CTA_THREADS, 0, st>>>(b, s.d_chan_derived.as<ChanDerived>(), s.d_chan_off.as<uint64_t>(), s.d_chan_blob.as<uint8_t>());
      launches++;
    }
    if (n) {
      static const bool attr_set = [] {
        return cudaFuncSetAttribute(tg_emit_lane_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(LaneShared)) == cudaSuccess;
      }();
      if (!attr_set) { set_err(c, "cannot reserve %zu bytes of shared memory for the lane emitter", sizeof(LaneShared)); return TGI_E_CUDA; }
      const uint64_t groups = (n + 31) / 32;
      const uint64_t ctas = (groups + WARPS_PER_CTA - 1) / WARPS_PER_CTA;
      CK(cudaEventRecord(s.ev_e0, st));
      CK(s.d_xpos.ensure(n * 32));
      CK(s.d_lists.ensure(3 * n * 4));  // work lists of the clean-up kernels
      EmitIn ei = tg_emit_in(s, po, s.d_line_off.as<uint64_t>(), dsc, n);
      ei.out = s.d_jsonl.as<uint8_t>();
      // one LANE per record (tg_lane.cuh): 2 resident CTAs per SM by shared memory, persistent over the record groups
      static const unsigned lane_mult = [] { const char* e = getenv("TGI_LANE_MULT"); return e && atoi(e) > 0 ? (unsigned)atoi(e) : 24u; }();  // H100: 12, 24 and 48 within 0.3 ms of each other
      unsigned gl = (unsigned)std::min<uint64_t>(ctas, (uint64_t)c->sms * lane_mult);
      tg_emit_lane_kernel<<<gl, CTA_THREADS, sizeof(LaneShared), st>>>(b, cfg, ei);
      launches++;
      CK(cudaEventRecord(s.ev_f1, st));
      unsigned gg = (unsigned)std::min<uint64_t>(ctas, (uint64_t)c->sms * grid_mult());
      tg_emit_esc_kernel<ESC_SPARSE><<<gg, CTA_THREADS, 0, st>>>(b, ei);  // descriptions with a few line breaks
      tg_emit_esc_kernel<ESC_DENSE><<<gg, CTA_THREADS, 0, st>>>(b, ei);   // the other strings that need escaping or are long
      tg_emit_maps_kernel<<<gg, CTA_THREADS, 0, st>>>(b, ei);  // comment lists, non-trivial maps, long outlink lists
      launches += 3;
      CK(cudaEventRecord(s.ev_e1, st));
    }
    CK(cudaGetLastError());
  }
  return finish_batch(c, s, REC_TG, n, flags, t.line_total, t.cursor, arena_cap, launches, out);
}

int upload_yt(tgi_ctx* c, Slot& s, const tgi_yt_batch* in) {
  if (!in) { set_err(c, "null batch"); return TGI_E_ARG; }
  if (in->n && (!in->recs || !in->chans)) { set_err(c, "youtube batch: recs/chans must be non-null"); return TGI_E_ARG; }
  if (in->n >= (1ull << 40)) { set_err(c, "youtube batch: too many records"); return TGI_E_ARG; }
  {  // every offset the kernels will follow stays inside its array (O(n) on the host: 80-byte records, no side arrays), and
     // every time is a time.Time's (0 <= nsec < 1e9)
    int e = 0;
    uint64_t bad_rec = 0;
    uint32_t bad_chan = 0;
    for (uint64_t i = 0; i < in->n; i++) {
      const tgi_yt_rec& r = in->recs[i];
      uint64_t end = r.str_off + (uint64_t)r.id_len + r.title_len + r.desc_len + r.duration_len + r.lang_len;
      for (int k = 0; k < 5; k++) end += r.thumb_len[k] == TGI_YT_THUMB_ABSENT ? 0u : r.thumb_len[k];
      if (end > in->strs_len || end < r.str_off) e |= 1;
      if (r.chan_idx >= in->n_chans) e |= 2;
      if (!nsec_ok(r.published_nsec)) {
        if (!(e & 4)) bad_rec = i;
        e |= 4;
      }
    }
    for (uint32_t i = 0; i < in->n_chans; i++) {
      const tgi_yt_chan& ch = in->chans[i];
      if ((uint64_t)ch.str_off + ch.id_len + ch.title_len + ch.desc_len + ch.thumb_len + ch.country_len > in->chan_strs_len) e |= 512;
      if (!nsec_ok(ch.published_nsec)) {
        if (!(e & 1024)) bad_chan = i;
        e |= 1024;
      }
    }
    if (e & ~(4 | 1024)) { set_err(c, "youtube batch: offsets outside their arrays (mask 0x%x)", e); return TGI_E_ARG; }
    if (e & 4) { set_err(c, "youtube batch: published_nsec %d of video %llu is outside [0, 1e9)", in->recs[bad_rec].published_nsec, (unsigned long long)bad_rec); return TGI_E_ARG; }
    if (e) { set_err(c, "youtube batch: published_nsec %d of channel %u is outside [0, 1e9)", in->chans[bad_chan].published_nsec, bad_chan); return TGI_E_ARG; }
  }
  s.in_bytes = 0;
  InArrays a;
  a.add(s.d_recs, in->recs, in->n * sizeof(tgi_yt_rec));
  a.add(s.d_strs, in->strs, in->strs_len);
  a.add(s.d_chans, in->chans, in->n_chans * sizeof(tgi_yt_chan));
  a.add(s.d_chan_strs, in->chan_strs, in->chan_strs_len);
  const int rc = upload_arrays(c, s, a, page_fits(in->n, in->n_chans, a.packed_total()));
  if (rc) return rc;
  YtBatchDev& b = s.yt;
  b.recs = (const tgi_yt_rec*)a.dev[0];
  b.strs = a.dev[1];
  b.chans = (const tgi_yt_chan*)a.dev[2];
  b.chan_strs = a.dev[3];
  b.n = in->n;
  b.n_chans = in->n_chans;
  s.yt_desc_bytes = in->strs_len;
  return TGI_OK;
}

// a page of the Data API (50 videos) in one cooperative launch (yt_page.cuh); PAGE_FALLBACK as in run_tg_page
int run_yt_page(tgi_ctx* c, Slot& s, uint32_t flags, tgi_result* out) {
  const uint64_t n = s.yt.n;
  static const int occ = page_occupancy((const void*)yt_page_kernel);
  if (occ <= 0) return PAGE_FALLBACK;
  YtPageArgs pa{};
  pa.cfg = cfg_snapshot(c);
  pa.run_flags = flags;
  pa.b = s.yt;
  PageOut L;
  int rc = page_prepare(c, s, n, yt_arena_cap(s), flags, L, pa.res);
  if (rc) return rc;
  rc = yt_parse_out(c, s, n, s.d_page_out.as<uint8_t>() + L.o_status, pa.res.scalars, pa.yo);
  if (rc) return rc;
  void* kargs[] = {&pa};
  return page_launch_and_read(c, s, REC_YT, flags, n, (const void*)yt_page_kernel, kargs, occ, L, pa.res, "yt_page", out);
}

int run_yt(tgi_ctx* c, Slot& s, uint32_t flags, tgi_result* out) {
  YtBatchDev& b = s.yt;
  uint64_t n = b.n;
  cudaStream_t st = s.stream;
  uint32_t launches = 0;
  const bool want_json = flags & TGI_RUN_JSONL;
  if (page_run_ok(s, n, b.n_chans, flags)) {
    const int rc = run_yt_page(c, s, flags, out);
    if (rc != PAGE_FALLBACK) return rc;
  }
  const CfgDev cfg = cfg_snapshot(c);
  int rc = bulk_prologue(c, s, n);
  if (rc) return rc;
  uint64_t* dsc = s.d_scalars.as<uint64_t>();
  YtOut yo;
  rc = yt_parse_out(c, s, n, s.d_status.as<uint8_t>(), dsc, yo);
  if (rc) return rc;
  unsigned g = (unsigned)std::min<uint64_t>((n + WARPS_PER_CTA - 1) / WARPS_PER_CTA, (uint64_t)c->sms * grid_mult());
  static const bool yt_warp = getenv("TGI_YT_WARP") != nullptr;  // A/B switch: the warp sizer and writer for every record
  if (n) {
    CK(cudaEventRecord(s.ev_p0, st));
    yt_parse_kernel<<<g, CTA_THREADS, 0, st>>>(b, cfg, flags, yo);
    launches++;
    if (want_json) {
      if (yt_warp) {
        yt_size_kernel<<<g, CTA_THREADS, 0, st>>>(b, cfg, yo);
      } else {
        const uint64_t groups = (n + 31) / 32;
        unsigned gs = (unsigned)std::min<uint64_t>((groups + WARPS_PER_CTA - 1) / WARPS_PER_CTA, (uint64_t)c->sms * grid_mult());
        yt_size_lane_kernel<<<gs, CTA_THREADS, 0, st>>>(b, cfg, yo);
      }
      launches++;
    }
    CK(cudaEventRecord(s.ev_p1, st));
  }
  Totals t{};
  rc = bulk_totals(c, s, n, want_json, launches, t);
  if (rc) return rc;
  if (t.err & ERR_ARENA_OVERFLOW) { set_err(c, "youtube url/link arena overflow (cannot happen: capacities are upper bounds)"); return TGI_E_CAPACITY; }
  if (want_json) {
    CK(s.d_jsonl.ensure(t.line_total));
    if (n) {
      CK(cudaEventRecord(s.ev_e0, st));
      const uint64_t groups = (n + 31) / 32;
      unsigned gg = (unsigned)std::min<uint64_t>((groups + WARPS_PER_CTA - 1) / WARPS_PER_CTA, (uint64_t)c->sms * grid_mult());
      if (!yt_warp) {
        yt_emit_lane_kernel<<<gg, CTA_THREADS, 0, st>>>(b, cfg, yo, s.d_line_off.as<uint64_t>(), s.d_jsonl.as<uint8_t>(), yo.err);
        launches++;
      }
      yt_emit_kernel<<<gg, CTA_THREADS, 0, st>>>(b, cfg, yo, s.d_line_off.as<uint64_t>(), s.d_jsonl.as<uint8_t>(), yo.err, yt_warp ? 0 : 1);
      CK(cudaEventRecord(s.ev_f1, st));
      CK(cudaEventRecord(s.ev_e1, st));
      launches++;
    }
    CK(cudaGetLastError());
  }
  return finish_batch(c, s, REC_YT, n, flags, t.line_total, t.cursor, yt_arena_cap(s), launches, out);
}

// generic client.Message batch (a12): upload, then size, scan, emit; no links
int upload_gm(tgi_ctx* c, Slot& s, const tgi_gm_batch* in) {
  if (!in) { set_err(c, "null batch"); return TGI_E_ARG; }
  if (in->n && !in->recs) { set_err(c, "generic batch: recs must be non-null"); return TGI_E_ARG; }
  if (in->n >= (1ull << 40)) { set_err(c, "generic batch: too many records"); return TGI_E_ARG; }
  {  // offsets inside their arrays, and GetTimestamp() a time.Time (0 <= nsec < 1e9)
    int e = 0;
    uint64_t bad = 0;
    for (uint64_t i = 0; i < in->n; i++) {
      const tgi_gm_rec& r = in->recs[i];
      const uint64_t end = r.str_off + (uint64_t)r.id_len + r.channel_len + r.text_len + r.sender_len;
      if (end > in->strs_len || end < r.str_off) e |= 1;
      if (in->react_off && (in->react_off[i] > in->react_off[i + 1] || in->react_off[i + 1] > in->n_reacts)) e |= 8;
      if (!nsec_ok(r.ts_nsec)) {
        if (!(e & 16)) bad = i;
        e |= 16;
      }
    }
    for (uint64_t i = 0; i < in->n_reacts; i++)
      if ((uint64_t)in->reacts[i].key_off + in->reacts[i].key_len > in->aux_len) e |= 64;
    if (e & ~16) { set_err(c, "generic batch: offsets outside their arrays (mask 0x%x)", e); return TGI_E_ARG; }
    if (e) { set_err(c, "generic batch: ts_nsec %d of record %llu is outside [0, 1e9)", in->recs[bad].ts_nsec, (unsigned long long)bad); return TGI_E_ARG; }
  }
  const uint64_t n = in->n;
  s.in_bytes = 0;
  InArrays a;
  a.add(s.d_recs, in->recs, n * sizeof(tgi_gm_rec));
  a.add(s.d_strs, in->strs, in->strs_len);
  a.add(s.d_react_off, in->react_off, in->react_off ? (n + 1) * 4 : 0);
  a.add(s.d_reacts, in->reacts, in->n_reacts * sizeof(tgi_gm_reaction));
  a.add(s.d_aux, in->aux, in->aux_len);
  const int rc = upload_arrays(c, s, a, false);
  if (rc) return rc;
  GmBatchDev& b = s.gm;
  b.n = n;
  b.recs = (const tgi_gm_rec*)a.dev[0];
  b.strs = a.dev[1];
  b.react_off = in->react_off ? (const uint32_t*)a.dev[2] : nullptr;
  b.reacts = (const tgi_gm_reaction*)a.dev[3];
  b.aux = a.dev[4];
  return TGI_OK;
}

int run_gm(tgi_ctx* c, Slot& s, uint32_t flags, tgi_result* out) {
  const GmBatchDev& b = s.gm;
  const uint64_t n = b.n;
  cudaStream_t st = s.stream;
  uint32_t launches = 0;
  const bool want_json = flags & TGI_RUN_JSONL;
  const CfgDev cfg = cfg_snapshot(c);
  CK(s.d_arena.ensure(1024 * sizeof(tgi_link)));
  int rc = bulk_prologue(c, s, n);
  if (rc) return rc;
  if (n) {
    CK(cudaMemsetAsync(s.d_link_start.p, 0, n * 4, st));
    CK(cudaMemsetAsync(s.d_link_count.p, 0, n * 4, st));
  }
  int* derr = (int*)(s.d_scalars.as<uint64_t>() + SC_CURSOR) + 1;
  unsigned g = (unsigned)std::min<uint64_t>((n + WARPS_PER_CTA - 1) / WARPS_PER_CTA, (uint64_t)c->sms * grid_mult());
  CK(cudaEventRecord(s.ev_p0, st));
  if (n) {  // the status does not depend on TGI_RUN_JSONL: the size pass always runs
    gm_size_kernel<<<g, CTA_THREADS, 0, st>>>(b, cfg, s.d_status.as<uint8_t>(), s.d_linelen.as<uint32_t>());
    launches++;
  }
  CK(cudaEventRecord(s.ev_p1, st));
  Totals t{};
  if (want_json) {
    rc = bulk_totals(c, s, n, want_json, launches, t);
    if (rc) return rc;
    CK(s.d_jsonl.ensure(t.line_total));
    CK(cudaEventRecord(s.ev_e0, st));
    if (n) {
      gm_emit_kernel<<<g, CTA_THREADS, 0, st>>>(b, cfg, s.d_status.as<uint8_t>(), s.d_line_off.as<uint64_t>(), s.d_jsonl.as<uint8_t>(), derr);
      launches++;
    }
    CK(cudaEventRecord(s.ev_f1, st));
    CK(cudaEventRecord(s.ev_e1, st));
    CK(cudaGetLastError());
  }
  return finish_batch(c, s, REC_GM, n, flags, t.line_total, 0, 1024, launches, out);
}

// channel records (StoreChannelData): upload, range check (host for small batches, device above), size, scan, emit
int upload_ch(tgi_ctx* c, Slot& s, const tgi_ch_batch* in) {
  if (!in) { set_err(c, "null batch"); return TGI_E_ARG; }
  if (in->n && !in->recs) { set_err(c, "channel batch: recs must be non-null"); return TGI_E_ARG; }
  if (in->strs_len && !in->strs) { set_err(c, "channel batch: a non-empty strs has a null pointer"); return TGI_E_ARG; }
  if (in->n >= (1ull << 40)) { set_err(c, "channel batch: too many records"); return TGI_E_ARG; }
  const uint64_t n = in->n;
  const bool host_checked = n <= HOST_VALIDATE_MAX;
  if (host_checked) {
    for (uint64_t i = 0; i < n; i++)
      if (!ch_rec_ok(in->recs[i], in->strs_len)) {
        set_err(c, "channel batch: record %llu: title | image | url outside strs, or a string of 16 MiB or more", (unsigned long long)i);
        return TGI_E_ARG;
      }
  }
  s.in_bytes = 0;
  InArrays a;
  a.add(s.d_recs, in->recs, n * sizeof(tgi_ch_rec));
  a.add(s.d_strs, in->strs, in->strs_len);
  const int rc = upload_arrays(c, s, a, false);
  if (rc) return rc;
  ChBatchDev& b = s.ch;
  b.n = n;
  b.recs = (const tgi_ch_rec*)a.dev[0];
  b.strs = a.dev[1];
  if (!host_checked) {
    CK(s.d_scalars.ensure(SC_COUNT * 8));
    CK(s.h_scalars.ensure(SC_COUNT * 8));
    unsigned long long* bad = (unsigned long long*)s.d_scalars.p;
    CK(cudaMemsetAsync(bad, 0xFF, 8, s.stream));
    const unsigned vg = (unsigned)std::min<uint64_t>((n + 255) / 256, (uint64_t)c->sms * 16);
    ch_validate_kernel<<<vg, 256, 0, s.stream>>>(b, in->strs_len, bad);
    CK(cudaGetLastError());
    const int prc = publish(c, bad, s.h_scalars, 1, s.stream);
    if (prc) return prc;
    CK(cudaStreamSynchronize(s.stream));
    const unsigned long long hbad = *s.h_scalars.as<unsigned long long>();
    if (hbad != ~0ull) {
      set_err(c, "channel batch: record %llu: title | image | url outside strs, or a string of 16 MiB or more", hbad);
      return TGI_E_ARG;
    }
  }
  return TGI_OK;
}

int run_ch(tgi_ctx* c, Slot& s, uint32_t flags, tgi_result* out) {
  const ChBatchDev& b = s.ch;
  const uint64_t n = b.n;
  cudaStream_t st = s.stream;
  uint32_t launches = 0;
  const bool want_json = flags & TGI_RUN_JSONL;
  CK(s.d_arena.ensure(1024 * sizeof(tgi_link)));
  int rc = bulk_prologue(c, s, n);
  if (rc) return rc;
  if (n) {
    CK(cudaMemsetAsync(s.d_link_start.p, 0, n * 4, st));
    CK(cudaMemsetAsync(s.d_link_count.p, 0, n * 4, st));
  }
  int* derr = (int*)(s.d_scalars.as<uint64_t>() + SC_CURSOR) + 1;
  unsigned g = (unsigned)std::min<uint64_t>((n + WARPS_PER_CTA - 1) / WARPS_PER_CTA, (uint64_t)c->sms * grid_mult());
  CK(cudaEventRecord(s.ev_p0, st));
  if (n) {  // the status does not depend on TGI_RUN_JSONL: the size pass always runs
    ch_size_kernel<<<g, CTA_THREADS, 0, st>>>(b, s.d_status.as<uint8_t>(), s.d_linelen.as<uint32_t>());
    launches++;
  }
  CK(cudaEventRecord(s.ev_p1, st));
  Totals t{};
  if (want_json) {
    rc = bulk_totals(c, s, n, want_json, launches, t);
    if (rc) return rc;
    CK(s.d_jsonl.ensure(t.line_total));
    CK(cudaEventRecord(s.ev_e0, st));
    if (n) {
      ch_emit_kernel<<<g, CTA_THREADS, 0, st>>>(b, s.d_line_off.as<uint64_t>(), s.d_jsonl.as<uint8_t>(), derr);
      launches++;
    }
    CK(cudaEventRecord(s.ev_f1, st));
    CK(cudaEventRecord(s.ev_e1, st));
    CK(cudaGetLastError());
  }
  return finish_batch(c, s, REC_CH, n, flags, t.line_total, 0, 1024, launches, out);
}

// ---- jobs -------------------------------------------------------------------------------------------------------------
// Upload if the job uploads (an upload-only job waits for the copy to land), run if it runs.
int run_job(tgi_ctx* c, Slot& s) {
  const Job& j = s.job;
  if (j.stages & JOB_UPLOAD) {
    const int rc = j.kind == REC_TG   ? upload_tg(c, s, (const tgi_tg_batch*)j.batch)
                   : j.kind == REC_YT ? upload_yt(c, s, (const tgi_yt_batch*)j.batch)
                   : j.kind == REC_GM ? upload_gm(c, s, (const tgi_gm_batch*)j.batch)
                                      : upload_ch(c, s, (const tgi_ch_batch*)j.batch);
    if (rc != TGI_OK) return rc;
    if (!(j.stages & JOB_RUN)) {
      const cudaError_t e = cudaStreamSynchronize(s.stream);
      if (e != cudaSuccess) { set_err(c, "upload sync: %s", cudaGetErrorString(e)); return TGI_E_CUDA; }
    }
    if (j.kind == REC_TG || j.kind == REC_YT) s.resident = j.kind;  // generic and channel batches are not run resident
  }
  if (!(j.stages & JOB_RUN)) return TGI_OK;
  return j.kind == REC_TG   ? run_tg(c, s, j.flags, &s.res)
         : j.kind == REC_YT ? run_yt(c, s, j.flags, &s.res)
         : j.kind == REC_GM ? run_gm(c, s, j.flags, &s.res)
                            : run_ch(c, s, j.flags, &s.res);
}

// runs the slot's claimed job to its end, on the worker thread or the caller's
int do_job(tgi_ctx* c, Slot& s) {
  const int rc = run_job(c, s);
  turn_pass(c, s);
  std::lock_guard<std::mutex> lk(s.mu);
  s.rc = rc;
  s.done = true;
  return rc;
}

void worker_main(tgi_ctx* c, Slot* s) {
  cudaSetDevice(c->device);
  for (;;) {
    {
      std::unique_lock<std::mutex> lk(s->mu);
      s->cv.wait(lk, [&] { return s->worker_state != Slot::IDLE; });
      if (s->worker_state == Slot::QUIT) return;
      s->worker_state = Slot::IDLE;
    }
    do_job(c, *s);
    s->cv.notify_all();
  }
}

bool run_flags_ok(tgi_ctx* c, uint32_t flags) {
  if ((flags & TGI_RUN_JSONL_DEVICE) && !(flags & TGI_RUN_JSONL)) {
    set_err(c, "TGI_RUN_JSONL_DEVICE without TGI_RUN_JSONL");
    return false;
  }
  return true;
}

// Claims slot s for job j, all under s.mu: the run flags, the busy check, the resident check, the job, its frontier
// ticket (frontier phases enter the dedup set in claim order), and the end of the slot's last result.  A job that
// uploads also ends the slot's resident batch: only a successful upload sets it again (run_job).
int claim_job(tgi_ctx* c, Slot& s, const Job& j) {
  if (!run_flags_ok(c, j.flags)) return TGI_E_ARG;
  std::lock_guard<std::mutex> lk(s.mu);
  if (s.busy) { set_err(c, "slot %d is busy (wait/release it first)", s.idx); return TGI_E_STATE; }
  if (!(j.stages & JOB_UPLOAD) && s.resident != j.kind) { set_err(c, "slot %d holds no resident batch of this kind", s.idx); return TGI_E_STATE; }
  s.busy = true;
  s.done = false;
  s.job = j;
  s.last = LastResult{};
  if (j.stages & JOB_UPLOAD) s.resident = REC_NONE;
  if ((j.stages & JOB_RUN) && (j.flags & TGI_RUN_FRONTIER)) {
    std::lock_guard<std::mutex> g(c->tk_mu);
    s.ticket = c->tk_next++;
    s.has_ticket = true;
  }
  return TGI_OK;
}

// tgi_*_submit: the slot's worker thread runs the job, tgi_*_wait collects it
int submit(tgi_ctx* c, int slot, const Job& j) {
  if (!c) return TGI_E_ARG;
  if (slot < 0 || slot >= TGI_SLOTS) { set_err(c, "bad slot %d", slot); return TGI_E_ARG; }
  Slot& s = c->slots[slot];
  const int rc = claim_job(c, s, j);
  if (rc != TGI_OK) return rc;
  {
    std::lock_guard<std::mutex> lk(s.mu);
    s.worker_state = Slot::QUEUED;
  }
  s.cv.notify_all();
  return TGI_OK;
}

int wait_job(tgi_ctx* c, int slot, tgi_result* out) {
  if (!c || slot < 0 || slot >= TGI_SLOTS) return TGI_E_ARG;
  Slot& s = c->slots[slot];
  std::unique_lock<std::mutex> lk(s.mu);
  if (!s.busy) { set_err(c, "slot %d has no submitted job", slot); return TGI_E_STATE; }
  s.cv.wait(lk, [&] { return s.done; });
  if (out) *out = s.res;
  int rc = s.rc;
  if (rc != TGI_OK) s.busy = false;  // nothing to release after a failed job (blocking callers still call
                                     // tgi_result_release, which also clears `claimed` and wakes the waiters)
  return rc;
}

// tgi_*_upload and tgi_*_run_resident: submit and wait.  The slot stays claimed only by a job that leaves a result.
int submit_wait(tgi_ctx* c, int slot, const Job& j, tgi_result* out) {
  int rc = submit(c, slot, j);
  if (rc != TGI_OK) return rc;
  rc = wait_job(c, slot, out);
  if (rc != TGI_OK || !(j.stages & JOB_RUN)) tgi_result_release(c, slot);
  return rc;
}

int claim_slot(tgi_ctx* c) {
  std::unique_lock<std::mutex> lk(c->alloc_mu);
  for (;;) {
    for (int i = 0; i < TGI_SLOTS; i++) {
      Slot& s = c->slots[i];
      std::lock_guard<std::mutex> g(s.mu);
      if (!s.busy && !s.claimed) { s.claimed = true; return i; }
    }
    c->alloc_cv.wait(lk);
  }
}

// Blocking calls run the job on the CALLER's thread in a free slot (claimed exclusively): two condition-variable
// hand-offs per call are most of what a page-sized batch costs besides the launches themselves.  The result stays
// valid until tgi_result_release(ctx, out->slot); a failed call releases the slot itself.
int run_blocking(tgi_ctx* c, const Job& j, tgi_result* out) {
  if (!c) return TGI_E_ARG;
  const int slot = claim_slot(c);
  Slot& s = c->slots[slot];
  int rc = claim_job(c, s, j);
  if (rc == TGI_OK) {
    cudaSetDevice(c->device);
    rc = do_job(c, s);
  }
  if (rc != TGI_OK) tgi_result_release(c, slot);
  else if (out) *out = s.res;
  return rc;
}

// a job is in flight on slot s: claimed and not finished (the caller holds s.mu)
bool in_flight(const Slot& s) { return s.busy && !s.done; }

// the first slot with a job in flight, or -1
int slot_in_flight(tgi_ctx* c) {
  for (int i = 0; i < TGI_SLOTS; i++) {
    std::lock_guard<std::mutex> lk(c->slots[i].mu);
    if (in_flight(c->slots[i])) return i;
  }
  return -1;
}

// The readers' view of slot `slot`: its last result.  TGI_E_ARG for a bad slot; TGI_E_STATE while a job is in flight on
// it or when it holds no result (nothing has run there, or its last job failed or only uploaded).
int slot_result(tgi_ctx* c, int slot, const char* who, LastResult* r) {
  if (slot < 0 || slot >= TGI_SLOTS) { set_err(c, "%s: bad slot %d", who, slot); return TGI_E_ARG; }
  Slot& s = c->slots[slot];
  std::lock_guard<std::mutex> lk(s.mu);
  if (in_flight(s)) { set_err(c, "%s: slot %d is in flight", who, slot); return TGI_E_STATE; }
  if (s.last.kind == REC_NONE) { set_err(c, "%s: slot %d holds no result", who, slot); return TGI_E_STATE; }
  *r = s.last;
  return TGI_OK;
}

// The sinks' view of slot `slot`: its last result, which must be a Telegram, YouTube or (Dapr sinks only, `dapr`)
// channel-record one with lines; with src, also the device arrays the sink kernels read (sink_src.cuh).  Selects the
// context's device.
int sink_source(tgi_ctx* c, int slot, const char* who, LastResult& r, SinkSrc* src, bool dapr) {
  const int rc = slot_result(c, slot, who, &r);
  if (rc != TGI_OK) return rc;
  if (r.kind == REC_GM) { set_err(c, "%s: generic posts go to SavePost, not to the StorePost sinks", who); return TGI_E_STATE; }
  // StoreChannelData: Dapr appends or combine files (daprstate.go:3088-3148); BaseStateManager's is a no-op (base.go:530)
  if (r.kind == REC_CH && !dapr) { set_err(c, "%s: the local manager stores no channel data", who); return TGI_E_STATE; }
  if (!r.dev.line_off) { set_err(c, "%s: the slot's last result has no lines (run it with TGI_RUN_JSONL)", who); return TGI_E_STATE; }
  cudaSetDevice(c->device);
  if (!src) return TGI_OK;
  const Slot& s = c->slots[slot];
  *src = SinkSrc{};
  src->n = r.n;
  src->status = r.dev.status;
  src->line_off = r.dev.line_off;
  src->jsonl = r.dev.jsonl;
  src->yt = r.kind == REC_YT;
  src->ch = r.kind == REC_CH;
  // the resident batch descriptor, not the upload buffers: a page-sized batch lives in the slot's one-block upload
  if (src->ch) {
    src->ch_recs = s.ch.recs, src->strs = s.ch.strs;
  } else if (src->yt) {
    src->yt_recs = s.yt.recs, src->yt_chans = s.yt.chans, src->strs = s.yt.strs, src->chan_strs = s.yt.chan_strs;
    src->n_chans = s.yt.n_chans;
  } else {
    src->tg_recs = s.tg.recs, src->tg_chans = s.tg.chans, src->strs = s.tg.strs, src->chan_strs = s.tg.chan_strs;
    src->n_chans = s.tg.n_chans;
  }
  return TGI_OK;
}

// the grid of a grid-stride sink launch: one CTA per per_cta items, at most per_sm CTAs per SM
unsigned sink_grid(const tgi_ctx* c, uint64_t items, uint64_t per_cta, uint64_t per_sm) {
  return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((items + per_cta - 1) / per_cta, (uint64_t)c->sms * per_sm));
}

// Chunker.processBatches (chunk/main.go:292-345) over lines [0, n) of one result, continuing a group that holds open_in
// bytes of earlier results; drops are the sorted indices of the lines longer than hard_cap.  Every group the rule closes
// goes to emit(begin, end) (false: stop with TGI_E_CAPACITY): lines [begin, end) minus the empty and dropped ones, begin
// 0 for the group carried in.  The group left open holds *open_out bytes; its first line of this result is *open_begin.
// K(i), the kept bytes before line i, is line_off[i] minus the dropped bytes before i: monotone, so every boundary is a
// binary search and the walk costs O(groups * log n * log drops), not O(n).
template <class Emit>
int plan_groups(const uint64_t* line_off, uint64_t n, uint64_t trigger, uint64_t hard_cap, uint64_t open_in,
                const std::vector<uint64_t>& drops, Emit emit, uint64_t* open_out, uint64_t* open_begin) {
  std::vector<uint64_t> dbytes(drops.size() + 1, 0);
  for (size_t k = 0; k < drops.size(); k++) dbytes[k + 1] = dbytes[k] + (line_off[drops[k] + 1] - line_off[drops[k]]);
  auto K = [&](uint64_t i) {
    const size_t k = std::lower_bound(drops.begin(), drops.end(), i) - drops.begin();
    return line_off[i] - line_off[0] - dbytes[k];
  };
  // the first m in (p, n] with K(m) - base > thr, or n + 1
  auto first_over = [&](uint64_t p, uint64_t base, uint64_t thr) {
    if (K(n) - base <= thr) return n + 1;
    uint64_t lo = p + 1, hi = n;
    while (lo < hi) {
      const uint64_t mid = lo + (hi - lo) / 2;
      if (K(mid) - base > thr) hi = mid;
      else lo = mid + 1;
    }
    return lo;
  };
  uint64_t p = 0, size = open_in, begin = 0;
  while (p < n) {
    const uint64_t base = K(p);
    // line mc - 1 would push the group over hard_cap (:324-327); line mt - 1 makes it reach trigger (:334-337)
    const uint64_t mc = first_over(p, base, hard_cap - size);
    const uint64_t mt = first_over(p, base, (trigger > size ? trigger - size : 1) - 1);
    if (!size && K(n) > base) begin = first_over(p, base, 0) - 1;  // the group's first line
    if (mc > n && mt > n) {  // every line left joins the open group
      size += K(n) - base;
      break;
    }
    if (mc <= mt) {  // close before line mc - 1, which starts the next group
      if (!emit(begin, mc - 1)) return TGI_E_CAPACITY;
      p = mc - 1;
    } else {         // close after line mt - 1
      if (!emit(begin, mt)) return TGI_E_CAPACITY;
      p = mt;
    }
    size = 0;
  }
  *open_out = size;
  *open_begin = size ? begin : n;
  return TGI_OK;
}

// tgi_plan_chunks(_carry): the dropped lines by a scan, then plan_groups; `close` closes the group left open (:339-343)
int plan_host(const uint64_t* line_off, uint64_t n, uint64_t trigger, uint64_t hard_cap, uint64_t open_in, uint64_t* groups,
              uint64_t max_groups, uint64_t* n_groups, uint8_t* dropped, uint64_t* open_out, bool close) {
  std::vector<uint64_t> drops;
  for (uint64_t i = 0; i < n; i++) {
    const bool d = line_off[i + 1] - line_off[i] > hard_cap;
    if (dropped) dropped[i] = d;
    if (d) drops.push_back(i);
  }
  uint64_t g = 0, open_begin = 0;
  auto emit = [&](uint64_t a, uint64_t b) {
    if (g >= max_groups) return false;
    groups[2 * g] = a;
    groups[2 * g + 1] = b;
    g++;
    return true;
  };
  const int rc = plan_groups(line_off, n, trigger, hard_cap, open_in, drops, emit, open_out, &open_begin);
  if (rc) return rc;
  if (close && *open_out) {
    if (!emit(open_begin, n)) return TGI_E_CAPACITY;
    *open_out = 0;
  }
  *n_groups = g;
  return TGI_OK;
}

}  // namespace

extern "C" {

int tgi_create(const tgi_config* cfg, tgi_ctx** out) {
  tgi_ctx* c = nullptr;
  if (!cfg || !out) { set_err(nullptr, "null argument"); return TGI_E_ARG; }
  if (cfg->abi_version != TGI_ABI_VERSION) { set_err(nullptr, "ABI version mismatch: library %d, caller %u", TGI_ABI_VERSION, cfg->abi_version); return TGI_E_ARG; }
  if (!nsec_ok(cfg->created_at_nsec) || !nsec_ok(cfg->capture_nsec)) {
    set_err(nullptr, "created_at_nsec %d / capture_nsec %d: outside [0, 1e9)", cfg->created_at_nsec, cfg->capture_nsec);
    return TGI_E_ARG;
  }
  if (cfg->tz_offset_sec <= -86400 || cfg->tz_offset_sec >= 86400) { set_err(nullptr, "tz_offset_sec %d is a day or more", cfg->tz_offset_sec); return TGI_E_ARG; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    set_err(nullptr, "no CUDA device visible: libtgingest has no CPU fallback");
    return TGI_E_NODEVICE;
  }
  if (cfg->device < 0 || cfg->device >= ndev) { set_err(nullptr, "device %d out of range (%d visible)", cfg->device, ndev); return TGI_E_ARG; }
  tgi_ctx* ctx = new tgi_ctx();
  ctx->cfg = *cfg;
  ctx->label.assign(cfg->crawl_label ? cfg->crawl_label : "", cfg->crawl_label ? cfg->crawl_label_len : 0);
  ctx->cfg.crawl_label = nullptr;
  ctx->device = cfg->device;
  c = ctx;
  auto fail = [&](int rc) {
    g_create_err = ctx->err;
    tgi_destroy(ctx);
    return rc;
  };
  if (cudaSetDevice(ctx->device) != cudaSuccess) { set_err(c, "cudaSetDevice failed"); return fail(TGI_E_CUDA); }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, ctx->device) == cudaSuccess) ctx->sms = prop.multiProcessorCount;
  if (ctx->h_zero.ensure(PAD) != cudaSuccess) { set_err(c, "pinned allocation failed"); return fail(TGI_E_CUDA); }
  memset(ctx->h_zero.p, 0, PAD);
  for (int i = 0; i < TGI_SLOTS; i++) {
    Slot& s = ctx->slots[i];
    s.idx = i;
    s.h_scalars.flags = cudaHostAllocMapped;  // publish() stores into it from the device
    if (cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreate(&s.ev_k0) != cudaSuccess || cudaEventCreate(&s.ev_k1) != cudaSuccess ||
        cudaEventCreate(&s.ev_p0) != cudaSuccess || cudaEventCreate(&s.ev_p1) != cudaSuccess ||
        cudaEventCreate(&s.ev_e0) != cudaSuccess || cudaEventCreate(&s.ev_e1) != cudaSuccess || cudaEventCreate(&s.ev_f1) != cudaSuccess ||
        cudaEventCreate(&s.ev_fr0) != cudaSuccess || cudaEventCreate(&s.ev_fr1) != cudaSuccess) {
      set_err(c, "stream/event creation failed: %s", cudaGetErrorString(cudaGetLastError()));
      return fail(TGI_E_CUDA);
    }
  }
  if (cudaEventCreateWithFlags(&ctx->fr_event, cudaEventDisableTiming) != cudaSuccess) { set_err(c, "event creation failed"); return fail(TGI_E_CUDA); }
  // frontier
  uint64_t fcap = cfg->frontier_capacity ? cfg->frontier_capacity : (1ull << 22);
  uint64_t tslots = next_pow2(2 * fcap);
  ctx->fr_cap0 = fcap;
  if (set_alloc(ctx, ctx->sets[TGI_SET_FRONTIER], fcap, tslots, false) != TGI_OK) {
    set_err(c, "frontier allocation failed (%llu keys)", (unsigned long long)fcap);
    return fail(TGI_E_NOMEM);
  }
  cudaStreamSynchronize(ctx->slots[0].stream);
  int rc = build_cfg_blob(ctx);
  if (rc) return fail(rc);
  for (int i = 0; i < TGI_SLOTS; i++) ctx->slots[i].worker = std::thread(worker_main, ctx, &ctx->slots[i]);
  *out = ctx;
  return TGI_OK;
}

void tgi_destroy(tgi_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  tgi_comm_destroy(c);  // while the stream its collectives ran on still exists
  for (int i = 0; i < TGI_SLOTS; i++) {
    Slot& s = c->slots[i];
    if (s.worker.joinable()) {
      {
        std::unique_lock<std::mutex> lk(s.mu);
        s.cv.wait(lk, [&] { return s.worker_state == Slot::IDLE; });
        s.worker_state = Slot::QUIT;
      }
      s.cv.notify_all();
      s.worker.join();
    }
    if (s.stream) cudaStreamSynchronize(s.stream);
    for (cudaEvent_t e : {s.ev_k0, s.ev_k1, s.ev_p0, s.ev_p1, s.ev_e0, s.ev_e1, s.ev_f1, s.ev_fr0, s.ev_fr1}) if (e) cudaEventDestroy(e);
    if (s.stream) cudaStreamDestroy(s.stream);
  }
  for (auto& f : c->stg_free) cudaFreeHost(f.second);
  for (auto& f : c->stg_live) cudaFreeHost(f.first);
  if (c->fr_event) cudaEventDestroy(c->fr_event);
  if (c->cb.stream) {
    cudaStreamSynchronize(c->cb.stream);
    cudaStreamDestroy(c->cb.stream);
  }
  for (cudaEvent_t e : {c->cb.ev, c->cb.t0, c->cb.t1}) if (e) cudaEventDestroy(e);
  if (c->state.stream) {
    cudaStreamSynchronize(c->state.stream);
    cudaStreamDestroy(c->state.stream);
  }
  for (cudaEvent_t e : {c->state.t0, c->state.t1, c->state.t2, c->state.t3, c->state.t4, c->state.t5, c->state.ev_slot}) if (e) cudaEventDestroy(e);
  delete c;  // the device and pinned buffers free themselves
}

const char* tgi_last_error(tgi_ctx* c) {
  if (!c) return g_create_err.c_str();
  std::lock_guard<std::mutex> g(c->err_mu);
  return c->err.c_str();
}

void tgi_get_stats(tgi_ctx* c, tgi_stats* out) {
  if (!c || !out) return;
  std::lock_guard<std::mutex> g(c->st_mu);
  *out = c->stats;
}

int tgi_set_clock(tgi_ctx* c, int64_t created_at_sec, int32_t created_at_nsec, int64_t capture_sec, int32_t capture_nsec) {
  if (!c) return TGI_E_ARG;
  if (!nsec_ok(created_at_nsec) || !nsec_ok(capture_nsec)) {  // the previous clock stays in effect
    set_err(c, "tgi_set_clock: created_at_nsec %d / capture_nsec %d: outside [0, 1e9)", created_at_nsec, capture_nsec);
    return TGI_E_ARG;
  }
  cudaSetDevice(c->device);
  if (const int i = slot_in_flight(c); i >= 0) { set_err(c, "tgi_set_clock while slot %d is in flight", i); return TGI_E_STATE; }
  std::lock_guard<std::mutex> g(c->cfg_mu);
  c->cfg.created_at_sec = created_at_sec;
  c->cfg.created_at_nsec = created_at_nsec;
  c->cfg.capture_sec = capture_sec;
  c->cfg.capture_nsec = capture_nsec;
  return build_cfg_blob(c);
}

int tgi_set_zone(tgi_ctx* c, const int64_t* start_sec, const int32_t* offset_sec, uint32_t n) {
  if (!c) return TGI_E_ARG;
  if (n > TGI_ZONE_MAX) { set_err(c, "tgi_set_zone: %u entries (at most %d)", n, TGI_ZONE_MAX); return TGI_E_ARG; }
  if (n && (!start_sec || !offset_sec)) { set_err(c, "tgi_set_zone: NULL table"); return TGI_E_ARG; }
  std::vector<ZoneEnt> z(n);
  for (uint32_t i = 0; i < n; i++) {
    if (offset_sec[i] <= -86400 || offset_sec[i] >= 86400) { set_err(c, "tgi_set_zone: offset %d of entry %u is a day or more", offset_sec[i], i); return TGI_E_ARG; }
    if (i && start_sec[i] <= start_sec[i - 1]) { set_err(c, "tgi_set_zone: start of entry %u is not after entry %u", i, i - 1); return TGI_E_ARG; }
    z[i] = ZoneEnt{start_sec[i], offset_sec[i], 0};
  }
  cudaSetDevice(c->device);
  if (const int i = slot_in_flight(c); i >= 0) { set_err(c, "tgi_set_zone while slot %d is in flight", i); return TGI_E_STATE; }
  DevBuf d;
  if (n) {
    CK(d.ensure(n * sizeof(ZoneEnt)));
    CK(cudaMemcpy(d.p, z.data(), n * sizeof(ZoneEnt), cudaMemcpyHostToDevice));
  }
  std::lock_guard<std::mutex> g(c->cfg_mu);
  c->zone.swap(z);
  c->d_zone.swap(d);
  const int rc = build_cfg_blob(c);
  if (rc) {  // the previous table stays in effect
    c->zone.swap(z);
    c->d_zone.swap(d);
    build_cfg_blob(c);
  }
  return rc;
}

int tgi_telegram_submit(tgi_ctx* c, int slot, const tgi_tg_batch* in, uint32_t run_flags) {
  return submit(c, slot, {REC_TG, JOB_UPLOAD | JOB_RUN, in, run_flags});
}
int tgi_telegram_wait(tgi_ctx* c, int slot, tgi_result* out) { return wait_job(c, slot, out); }

void tgi_result_release(tgi_ctx* c, int slot) {
  if (!c || slot < 0 || slot >= TGI_SLOTS) return;
  Slot& s = c->slots[slot];
  {
    // alloc_mu is held across the state change: a claim_slot() that has scanned the slots and not yet started to
    // wait would otherwise miss this notification
    std::lock_guard<std::mutex> ag(c->alloc_mu);
    std::lock_guard<std::mutex> lk(s.mu);
    s.busy = false;
    s.claimed = false;
  }
  c->alloc_cv.notify_all();
}

int tgi_telegram_batch(tgi_ctx* c, const tgi_tg_batch* in, uint32_t run_flags, tgi_result* out) {
  return run_blocking(c, {REC_TG, JOB_UPLOAD | JOB_RUN, in, run_flags}, out);
}

int tgi_telegram_upload(tgi_ctx* c, int slot, const tgi_tg_batch* in) {
  return submit_wait(c, slot, {REC_TG, JOB_UPLOAD, in, 0}, nullptr);
}
int tgi_telegram_run_resident(tgi_ctx* c, int slot, uint32_t run_flags, tgi_result* out) {
  return submit_wait(c, slot, {REC_TG, JOB_RUN, nullptr, run_flags}, out);
}

int tgi_result_read_jsonl(tgi_ctx* c, int slot, uint64_t off, uint64_t len, uint8_t* dst) {
  if (!c || !dst) return TGI_E_ARG;
  LastResult r;
  const int rc = slot_result(c, slot, "read_jsonl", &r);
  if (rc != TGI_OK) return rc;
  cudaSetDevice(c->device);
  if (off + len > r.jsonl_len) { set_err(c, "read_jsonl out of range"); return TGI_E_ARG; }
  CK(cudaMemcpy(dst, r.dev.jsonl + off, len, cudaMemcpyDeviceToHost));
  return TGI_OK;
}

int tgi_result_read_rows(tgi_ctx* c, int slot, int which, uint64_t first, uint64_t count, void* dst) {
  if (!c || !dst) return TGI_E_ARG;
  LastResult r;
  const int rc = slot_result(c, slot, "read_rows", &r);
  if (rc != TGI_OK) return rc;
  cudaSetDevice(c->device);
  const void* base = nullptr;
  uint64_t rows = 0, size = 0;
  if (which == TGI_ROWS_STATUS) base = r.dev.status, rows = r.n, size = 1;
  if (which == TGI_ROWS_LINK_OFF) base = r.dev.link_off, rows = r.n + 1, size = 4;
  if (which == TGI_ROWS_LINKS) base = r.dev.links, rows = r.n_links, size = sizeof(tgi_link);
  if (!base || first > rows || count > rows - first) { set_err(c, "read_rows: no such rows in the slot's last result"); return TGI_E_ARG; }
  CK(cudaMemcpy(dst, (const uint8_t*)base + first * size, count * size, cudaMemcpyDeviceToHost));
  return TGI_OK;
}

int tgi_youtube_submit(tgi_ctx* c, int slot, const tgi_yt_batch* in, uint32_t run_flags) {
  return submit(c, slot, {REC_YT, JOB_UPLOAD | JOB_RUN, in, run_flags});
}
int tgi_youtube_wait(tgi_ctx* c, int slot, tgi_result* out) { return wait_job(c, slot, out); }
int tgi_youtube_batch(tgi_ctx* c, const tgi_yt_batch* in, uint32_t run_flags, tgi_result* out) {
  return run_blocking(c, {REC_YT, JOB_UPLOAD | JOB_RUN, in, run_flags}, out);
}
int tgi_key_join(tgi_ctx* c, const int64_t* a_keys, uint64_t na, const int64_t* b_keys, uint64_t nb, int64_t* b_index) {
  if (!c || (na && !a_keys) || (nb && (!b_keys || !b_index))) return TGI_E_ARG;
  if (na >= 0xFFFFFFFFull) { set_err(c, "key join: list A has too many elements"); return TGI_E_ARG; }
  cudaSetDevice(c->device);
  if (!nb) return TGI_OK;
  const uint64_t slots = next_pow2(std::max<uint64_t>(2 * na, 1024));
  DevBuf da, db, dt, dout;
  CK(da.ensure(na * 16 + 16));
  CK(db.ensure(nb * 16));
  CK(dt.ensure(slots * 4));
  CK(dout.ensure(nb * 8));
  CK(cudaMemset(dt.p, 0, slots * 4));
  if (na) CK(cudaMemcpy(da.p, a_keys, na * 16, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(db.p, b_keys, nb * 16, cudaMemcpyHostToDevice));
  if (na) join_build_kernel<<<(unsigned)((na + 255) / 256), 256>>>((const longlong2*)da.p, na, dt.as<uint32_t>(), slots - 1);
  join_probe_kernel<<<(unsigned)((nb + 255) / 256), 256>>>((const longlong2*)da.p, dt.as<uint32_t>(), slots - 1, (const longlong2*)db.p, nb,
                                                       (long long*)dout.p);
  CK(cudaGetLastError());
  CK(cudaMemcpy(b_index, dout.p, nb * 8, cudaMemcpyDeviceToHost));
  da.release();
  db.release();
  dt.release();
  dout.release();
  return TGI_OK;
}

int tgi_plan_chunks(const uint64_t* line_off, uint64_t n, uint64_t trigger, uint64_t hard_cap, uint64_t* groups,
                    uint64_t max_groups, uint64_t* n_groups, uint8_t* dropped) {
  if (!line_off || !groups || !n_groups) return TGI_E_ARG;
  uint64_t open_out = 0;
  return plan_host(line_off, n, trigger, hard_cap, 0, groups, max_groups, n_groups, dropped, &open_out, true);
}

int tgi_plan_chunks_carry(const uint64_t* line_off, uint64_t n, uint64_t trigger, uint64_t hard_cap, uint64_t open_bytes_in,
                          uint64_t* groups, uint64_t max_groups, uint64_t* n_groups, uint8_t* dropped,
                          uint64_t* open_bytes_out) {
  if (!line_off || !n_groups || !open_bytes_out || (max_groups && !groups)) return TGI_E_ARG;
  if (open_bytes_in > hard_cap || (open_bytes_in && open_bytes_in >= trigger)) return TGI_E_ARG;  // no group rests there
  return plan_host(line_off, n, trigger, hard_cap, open_bytes_in, groups, max_groups, n_groups, dropped, open_bytes_out, false);
}

int tgi_plan_channel_appends(const uint64_t* line_off, const void* chan_idx, uint32_t chan_stride, uint64_t n, tgi_append_run* runs,
                             uint64_t max_runs, uint64_t* n_runs) {
  if (!line_off || !n_runs || (n && !chan_idx) || (max_runs && !runs)) return TGI_E_ARG;
  uint64_t g = 0;
  bool open = false;
  tgi_append_run cur{};
  for (uint64_t i = 0; i < n; i++) {
    if (line_off[i + 1] == line_off[i]) continue;  // no post was stored for this record
    const uint32_t ch = *(const uint32_t*)((const uint8_t*)chan_idx + (size_t)i * chan_stride);
    if (open && ch == cur.chan_idx) {  // lines without a post in between are empty ranges: the bytes stay contiguous
      cur.end = i + 1;
      cur.byte_end = line_off[i + 1];
      cur.n_lines++;
      continue;
    }
    if (open) {
      if (g >= max_runs) return TGI_E_CAPACITY;
      runs[g++] = cur;
    }
    cur.chan_idx = ch;
    cur.n_lines = 1;
    cur.first = i;
    cur.end = i + 1;
    cur.byte_begin = line_off[i];
    cur.byte_end = line_off[i + 1];
    open = true;
  }
  if (open) {
    if (g >= max_runs) return TGI_E_CAPACITY;
    runs[g++] = cur;
  }
  *n_runs = g;
  return TGI_OK;
}

int tgi_generic_batch(tgi_ctx* c, const tgi_gm_batch* in, uint32_t run_flags, tgi_result* out) {
  // generic messages have no links: no frontier phase, no frontier turn
  return run_blocking(c, {REC_GM, JOB_UPLOAD | JOB_RUN, in, run_flags & ~(uint32_t)TGI_RUN_FRONTIER}, out);
}
int tgi_channel_batch(tgi_ctx* c, const tgi_ch_batch* in, uint32_t run_flags, tgi_result* out) {
  if (!c) return TGI_E_ARG;
  if (run_flags & ~(uint32_t)(TGI_RUN_JSONL | TGI_RUN_JSONL_DEVICE)) {
    set_err(c, "channel batch: run flags 0x%x (only TGI_RUN_JSONL and TGI_RUN_JSONL_DEVICE)", run_flags);
    return TGI_E_ARG;
  }
  return run_blocking(c, {REC_CH, JOB_UPLOAD | JOB_RUN, in, run_flags}, out);
}
int tgi_youtube_upload(tgi_ctx* c, int slot, const tgi_yt_batch* in) {
  return submit_wait(c, slot, {REC_YT, JOB_UPLOAD, in, 0}, nullptr);
}
int tgi_youtube_run_resident(tgi_ctx* c, int slot, uint32_t run_flags, tgi_result* out) {
  return submit_wait(c, slot, {REC_YT, JOB_RUN, nullptr, run_flags}, out);
}

// ---- frontier host API ------------------------------------------------------------------------------
// Enqueues the insert of n (> 0) device-resident 32-byte keys, each with its payload if d_payload is given, into set k
// (the dedup set, an exclusion set, or this rank's partition of the global set), and their NEW flags into d_is_new if
// given.  Runs on slot 0's stream under the frontier lock (taken by the caller); the scratch lives in the context.
static int frontier_insert_enqueue(tgi_ctx* c, KeySet& k, const void* d_keys, const uint64_t* d_payload, uint64_t n, void* d_is_new) {
  cudaStream_t st = c->slots[0].stream;
  InsertScratch& z = c->ins;
  CK(z.arena.ensure(n * sizeof(tgi_link)));
  CK(z.cnt.ensure(n * 4));
  CK(z.sc.ensure(64));
  CK(cudaMemsetAsync(z.sc.p, 0, 64, st));
  const unsigned g = (unsigned)((n + 255) / 256);
  keys_to_links_kernel<<<g, 256, 0, st>>>((const uint8_t*)d_keys, n, z.arena.as<tgi_link>(), z.cnt.as<uint32_t>());
  uint32_t launches = 0;  // not reported by the insert API
  const int rc = set_insert(c, k, st, n, nullptr, z.cnt.as<uint32_t>(), z.arena.as<tgi_link>(), n, n, 0, ExclusionDev{}, z.fs,
                            z.tiles, true, z.sc.as<uint64_t>(), (int*)(z.sc.as<uint64_t>() + 4), d_payload, launches);
  if (rc) return rc;
  if (d_is_new) links_new_flags_kernel<<<g, 256, 0, st>>>(z.arena.as<tgi_link>(), n, (uint8_t*)d_is_new);
  CK(cudaGetLastError());
  return TGI_OK;
}
static int frontier_insert_check(tgi_ctx* c, const KeySet& k) {  // after a stream synchronize
  int herr = 0;
  CK(cudaMemcpy(&herr, (int*)(c->ins.sc.as<uint64_t>() + 4), 4, cudaMemcpyDeviceToHost));
  if (herr & ERR_FRONTIER_FULL) { set_err(c, "frontier capacity %llu exceeded", (unsigned long long)k.dev.cap); return TGI_E_CAPACITY; }
  return TGI_OK;
}
static int frontier_insert_impl(tgi_ctx* c, const void* d_keys, uint64_t n, void* d_is_new) {
  std::unique_lock<std::mutex> fg(c->fr_mu);
  KeySet& fr = c->sets[TGI_SET_FRONTIER];
  const int rc = frontier_insert_enqueue(c, fr, d_keys, nullptr, n, d_is_new);
  if (rc) return rc;
  CK(cudaStreamSynchronize(c->slots[0].stream));
  return frontier_insert_check(c, fr);
}

int tgi_frontier_insert(tgi_ctx* c, const uint8_t* keys32, uint64_t n, uint8_t* is_new) {
  if (!c || (n && !keys32)) return TGI_E_ARG;
  if (n >= (1ull << 32)) { set_err(c, "too many keys in one call"); return TGI_E_ARG; }
  cudaSetDevice(c->device);
  if (!n) return TGI_OK;
  cudaStream_t st = c->slots[0].stream;
  DevBuf dk, dn;
  CK(dk.ensure(n * 32));
  CK(dn.ensure(n));
  CK(cudaMemcpyAsync(dk.p, keys32, n * 32, cudaMemcpyHostToDevice, st));
  int rc = frontier_insert_impl(c, dk.p, n, dn.p);
  if (rc == TGI_OK && is_new) {
    CK(cudaMemcpyAsync(is_new, dn.p, n, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  return rc;
}
int tgi_frontier_insert_dev(tgi_ctx* c, const void* d_keys32, uint64_t n, void* d_is_new) {
  if (!c || (n && !d_keys32)) return TGI_E_ARG;
  cudaSetDevice(c->device);
  if (!n) return TGI_OK;
  return frontier_insert_impl(c, d_keys32, n, d_is_new);
}
int tgi_frontier_sync(tgi_ctx* c) {
  if (!c) return TGI_E_ARG;
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> g(c->fr_mu);
  if (c->fr_event_valid) CK(cudaEventSynchronize(c->fr_event));
  return TGI_OK;
}
int tgi_frontier_size(tgi_ctx* c, uint64_t* n) {
  if (!c || !n) return TGI_E_ARG;
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> g(c->fr_mu);
  return set_count(c, c->sets[TGI_SET_FRONTIER], n);
}
int tgi_frontier_export(tgi_ctx* c, uint8_t* keys32, uint64_t cap, uint64_t* n) {
  if (!c || !n) return TGI_E_ARG;
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> g(c->fr_mu);
  const KeySet& fr = c->sets[TGI_SET_FRONTIER];
  uint64_t sz = 0;
  int rc = set_count(c, fr, &sz);
  if (rc) return rc;
  uint64_t m = sz < cap ? sz : cap;
  if (m && keys32) {
    CK(cudaMemcpyAsync(keys32, fr.dev.pool, m * 32, cudaMemcpyDeviceToHost, c->slots[0].stream));
    CK(cudaStreamSynchronize(c->slots[0].stream));
  }
  *n = sz;
  return TGI_OK;
}
int tgi_frontier_export_dev(tgi_ctx* c, void* d_keys32, uint64_t cap, uint64_t first, uint64_t* n) {
  if (!c || !n) return TGI_E_ARG;
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> g(c->fr_mu);
  const KeySet& fr = c->sets[TGI_SET_FRONTIER];
  uint64_t sz = 0;
  int rc = set_count(c, fr, &sz);
  if (rc) return rc;
  uint64_t avail = first < sz ? sz - first : 0;
  uint64_t m = avail < cap ? avail : cap;
  if (m && d_keys32) {
    CK(cudaMemcpyAsync(d_keys32, fr.dev.pool + 32 * first, m * 32, cudaMemcpyDeviceToDevice, c->slots[0].stream));
    CK(cudaStreamSynchronize(c->slots[0].stream));  // the caller's stream may read the keys as soon as this returns
  }
  *n = m;
  return TGI_OK;
}
int tgi_frontier_clear(tgi_ctx* c) {
  if (!c) return TGI_E_ARG;
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> g(c->fr_mu);
  cudaStream_t st = c->slots[0].stream;
  if (c->fr_event_valid) CK(cudaStreamWaitEvent(st, c->fr_event, 0));
  KeySet& owned = c->sets[TGI_SET_OWNED];
  int rc = set_clear(c, c->sets[TGI_SET_FRONTIER]);
  if (rc == TGI_OK && owned.dev.table) rc = set_clear(c, owned);
  if (rc) return rc;
  c->merged_upto = 0;
  CK(cudaEventRecord(c->fr_event, st));
  c->fr_event_valid = true;
  CK(cudaStreamSynchronize(st));
  return TGI_OK;
}

// ---- frontier -> validator hand-off (SURVEY 8f rank 3) ------------------------------------------------------------
}  // extern "C"
namespace {
// a caller-filled set on first use (under fr_mu): the dedup set's capacity, or at most 2^16 keys when the sets grow on
// their own
int set_first_use(tgi_ctx* c, KeySet& k, bool stamps) {
  if (k.dev.table) return TGI_OK;
  const FrontierDev& fr = c->sets[TGI_SET_FRONTIER].dev;
  const uint64_t cap = std::min<uint64_t>(c->fr_cap0, 1u << 16);
  return c->grow_max ? set_alloc(c, k, cap, next_pow2(2 * cap), stamps) : set_alloc(c, k, fr.cap, fr.tmask + 1, stamps);
}
}  // namespace
extern "C" {
int tgi_set_add(tgi_ctx* c, int which, const uint8_t* keys32, const int64_t* stamp_sec, uint64_t n) {
  if (!c || (n && !keys32)) return TGI_E_ARG;
  KeySet* k = key_set(c, which, true);
  if (!k) { set_err(c, "tgi_set_add: unknown set %d", which); return TGI_E_ARG; }
  if (n >= (1ull << 32)) { set_err(c, "too many keys in one call"); return TGI_E_ARG; }
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> g(c->fr_mu);
  cudaStream_t st = c->slots[0].stream;
  const bool stamps = which == TGI_SET_INVALID;
  if (const int rc = set_first_use(c, *k, stamps)) return rc;
  if (!n) return TGI_OK;
  DevBuf dk, dp;
  CK(dk.ensure(n * 32));
  CK(cudaMemcpyAsync(dk.p, keys32, n * 32, cudaMemcpyHostToDevice, st));
  const uint64_t* pay = nullptr;
  if (stamps && stamp_sec) {
    CK(dp.ensure(n * 8));
    CK(cudaMemcpyAsync(dp.p, stamp_sec, n * 8, cudaMemcpyHostToDevice, st));
    pay = dp.as<uint64_t>();
  }
  const int rc = frontier_insert_enqueue(c, *k, dk.p, pay, n, nullptr);
  if (rc) return rc;
  CK(cudaStreamSynchronize(st));
  return frontier_insert_check(c, *k);
}
int tgi_set_clear(tgi_ctx* c, int which) {
  if (!c) return TGI_E_ARG;
  KeySet* k = key_set(c, which, true);
  if (!k) return TGI_E_ARG;
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> g(c->fr_mu);
  if (!k->dev.table) return TGI_OK;
  cudaStream_t st = c->slots[0].stream;
  if (c->fr_event_valid) CK(cudaStreamWaitEvent(st, c->fr_event, 0));
  const int rc = set_clear(c, *k);
  if (rc) return rc;
  CK(cudaStreamSynchronize(st));
  return TGI_OK;
}
int tgi_set_size(tgi_ctx* c, int which, uint64_t* n) {
  if (!c || !n) return TGI_E_ARG;
  KeySet* k = key_set(c, which, true);
  if (!k) return TGI_E_ARG;
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> g(c->fr_mu);
  return set_count(c, *k, n);
}
int tgi_set_export(tgi_ctx* c, int which, uint8_t* keys32, int64_t* stamps_sec, uint64_t cap, uint64_t* n) {
  if (!c || !n) return TGI_E_ARG;
  KeySet* k = key_set(c, which, true);
  if (!k) { set_err(c, "tgi_set_export: unknown set %d", which); return TGI_E_ARG; }
  if (stamps_sec && which != TGI_SET_INVALID) { set_err(c, "tgi_set_export: only TGI_SET_INVALID has stamps"); return TGI_E_ARG; }
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> g(c->fr_mu);
  uint64_t sz = 0;
  if (const int rc = set_count(c, *k, &sz)) return rc;
  const uint64_t m = std::min(sz, cap);
  cudaStream_t st = c->slots[0].stream;
  if (m && keys32) CK(cudaMemcpyAsync(keys32, k->dev.pool, m * 32, cudaMemcpyDeviceToHost, st));
  if (m && stamps_sec) CK(cudaMemcpyAsync(stamps_sec, k->dev.payload, m * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  *n = sz;
  return TGI_OK;
}
int tgi_set_now(tgi_ctx* c, int64_t now_sec) {
  if (!c) return TGI_E_ARG;
  std::lock_guard<std::mutex> g(c->fr_mu);
  c->now_sec = now_sec;
  return TGI_OK;
}
int tgi_set_growth(tgi_ctx* c, uint64_t max_keys) {
  if (!c) return TGI_E_ARG;
  if (max_keys >= (1ull << 40)) { set_err(c, "tgi_set_growth: a set holds fewer than 2^40 keys"); return TGI_E_ARG; }
  if (const int i = slot_in_flight(c); i >= 0) { set_err(c, "tgi_set_growth while slot %d is in flight", i); return TGI_E_STATE; }
  std::lock_guard<std::mutex> g(c->fr_mu);
  c->grow_max = max_keys;
  return TGI_OK;
}
int tgi_set_info(tgi_ctx* c, int which, tgi_set_info_t* out) {
  if (!c || !out) return TGI_E_ARG;
  const KeySet* k = key_set(c, which, false);
  if (!k) { set_err(c, "tgi_set_info: unknown set %d", which); return TGI_E_ARG; }
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> g(c->fr_mu);
  if (which == TGI_SET_OWNED && !c->comm) { set_err(c, "tgi_set_info: TGI_SET_OWNED needs tgi_comm_init first"); return TGI_E_STATE; }
  memset(out, 0, sizeof *out);
  if (!k->dev.table) return TGI_OK;  // an exclusion set before its first tgi_set_add
  const int rc = set_count(c, *k, &out->count);
  if (rc) return rc;
  out->capacity = k->dev.cap;
  out->table_slots = k->dev.tmask + 1;
  out->grows = k->grows;
  return TGI_OK;
}
int tgi_pending_edges(tgi_ctx* c, int slot, int64_t now_sec, tgi_edge* rows, uint64_t cap, uint64_t* n) {
  if (!c || !n || (cap && !rows)) return TGI_E_ARG;
  *n = 0;
  LastResult r;
  const int rc = slot_result(c, slot, "tgi_pending_edges", &r);
  if (rc != TGI_OK) return rc;
  if (r.n && !(r.flags & TGI_RUN_FRONTIER)) { set_err(c, "tgi_pending_edges: the slot's last batch ran without TGI_RUN_FRONTIER"); return TGI_E_STATE; }
  *n = r.n_new;
  const uint64_t m = r.n_new < cap ? r.n_new : cap;
  if (!m) return TGI_OK;
  cudaSetDevice(c->device);
  Slot& s = c->slots[slot];
  std::lock_guard<std::mutex> g(c->fr_mu);
  cudaStream_t st = s.stream;
  if (c->fr_event_valid) CK(cudaStreamWaitEvent(st, c->fr_event, 0));
  DevBuf drows;
  CK(drows.ensure(m * sizeof(tgi_edge)));
  const ExclusionDev x = exclusion(c, now_sec);
  // the resident batch descriptor, not the upload buffers: a page-sized batch lives in the slot's one-block upload
  const uint32_t* chan = r.kind == REC_YT ? &s.yt.recs->chan_idx : &s.tg.recs->chan_idx;
  const uint32_t stride = r.kind == REC_YT ? (uint32_t)sizeof(tgi_yt_rec) : (uint32_t)sizeof(tgi_tg_rec);
  edges_emit_kernel<<<(unsigned)((r.n + 255) / 256), 256, 0, st>>>(r.n, s.d_link_start.as<uint32_t>(), s.d_link_count.as<uint32_t>(),
                                                                  s.d_arena.as<tgi_link>(), chan, stride, s.fs.new_off.as<uint64_t>(), x,
                                                                  drows.as<tgi_edge>(), m);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(rows, drows.p, m * sizeof(tgi_edge), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return TGI_OK;
}

// Dapr sink payloads (dapr.cuh): size, two scans, one synchronise for the totals, write, the four copies, one synchronise.
int tgi_dapr_payloads(tgi_ctx* c, int slot, const char* path_prefix, uint32_t prefix_len, tgi_dapr_payloads_t* out) {
  if (!c || !out || !path_prefix) return TGI_E_ARG;
  LastResult r;
  SinkSrc src;
  int rc = sink_source(c, slot, "tgi_dapr_payloads", r, &src, true);
  if (rc != TGI_OK) return rc;
  Slot& s = c->slots[slot];
  DaprBufs& z = s.dapr;
  cudaStream_t st = s.stream;
  const uint64_t n = r.n;
  memset(out, 0, sizeof *out);
  out->n = n;
  CK(z.h_off.ensure(2 * (n + 1) * 8));
  uint64_t* h_off = z.h_off.as<uint64_t>();
  out->data_off = h_off;
  out->path_off = h_off + n + 1;
  if (!n) {
    h_off[0] = h_off[1] = 0;
    return TGI_OK;
  }
  CK(z.prefix.ensure(prefix_len));
  if (prefix_len) CK(cudaMemcpyAsync(z.prefix.p, path_prefix, prefix_len, cudaMemcpyHostToDevice, st));
  CK(z.lens.ensure(2 * n * 4));
  CK(z.off.ensure(2 * (n + 1) * 8));
  CK(z.sc.ensure(4 * 8));
  CK(z.h_sc.ensure(4 * 8));
  uint64_t* dsc = z.sc.as<uint64_t>();  // data total | path total | error word
  DaprOut o{};
  o.data_len = z.lens.as<uint32_t>();
  o.path_len = o.data_len + n;
  o.data_off = z.off.as<uint64_t>();
  o.path_off = o.data_off + n + 1;
  o.err = (int*)(dsc + 2);
  o.prefix = z.prefix.as<uint8_t>();
  o.prefix_len = prefix_len;
  uint32_t launches = 0;
  // device time = [ev_p0, ev_p1] (size kernel, scans) + [ev_e0, ev_e1] (writer): the totals' read-back and the host's
  // allocations between them are left out.  The batch's own times were read into its result already.
  CK(cudaMemsetAsync(dsc, 0, 4 * 8, st));
  CK(cudaEventRecord(s.ev_p0, st));
  dapr_size_kernel<<<sink_grid(c, n, 256, 16), 256, 0, st>>>(src, o);
  launches++;
  rc = launch_scan(c, s, o.data_len, n, (uint64_t*)o.data_off, dsc, launches);
  if (rc) return rc;
  rc = launch_scan(c, s, o.path_len, n, (uint64_t*)o.path_off, dsc + 1, launches);
  if (rc) return rc;
  CK(cudaEventRecord(s.ev_p1, st));
  CK(cudaMemcpyAsync(z.h_sc.p, dsc, 4 * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const uint64_t* hsc = z.h_sc.as<uint64_t>();
  if (hsc[2]) { set_err(c, "tgi_dapr_payloads: a payload or path of 4 GiB or more"); return TGI_E_CAPACITY; }
  const uint64_t data_total = hsc[0], path_total = hsc[1];
  CK(z.data.ensure(data_total));
  CK(z.path.ensure(path_total));
  CK(z.h_data.ensure(data_total + 1));
  CK(z.h_path.ensure(path_total + 1));
  o.data = z.data.as<uint8_t>();
  o.path = z.path.as<uint8_t>();
  CK(cudaEventRecord(s.ev_e0, st));
  dapr_write_kernel<<<sink_grid(c, n, WARPS_PER_CTA, 32), CTA_THREADS, 0, st>>>(src, o);  // 5 resident CTAs per SM
  launches++;
  CK(cudaGetLastError());
  CK(cudaEventRecord(s.ev_e1, st));
  CK(cudaMemcpyAsync(h_off, o.data_off, 2 * (n + 1) * 8, cudaMemcpyDeviceToHost, st));
  if (data_total) CK(cudaMemcpyAsync(z.h_data.p, o.data, data_total, cudaMemcpyDeviceToHost, st));
  if (path_total) CK(cudaMemcpyAsync(z.h_path.p, o.path, path_total, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  out->data = z.h_data.as<uint8_t>();
  out->data_len = data_total;
  out->path = z.h_path.as<uint8_t>();
  out->path_len = path_total;
  float size_ms = 0, write_ms = 0;
  cudaEventElapsedTime(&size_ms, s.ev_p0, s.ev_p1);
  cudaEventElapsedTime(&write_ms, s.ev_e0, s.ev_e1);
  out->kernel_ms = size_ms + write_ms;
  out->gpu_launches = launches;
  return TGI_OK;
}

// Local sink appends (local_appends.cuh): every kernel and scan is sized by upper bounds the host knows (records,
// channel rows, the result's JSONL bytes) and reads the exact counts from the device, so the whole pipeline and the
// read-back are enqueued at once and the call synchronises once.
int tgi_channel_appends(tgi_ctx* c, int slot, tgi_channel_appends_t* out) {
  if (!c || !out) return TGI_E_ARG;
  LastResult r;
  SinkSrc src;
  int rc = sink_source(c, slot, "tgi_channel_appends", r, &src, false);
  if (rc != TGI_OK) return rc;
  memset(out, 0, sizeof *out);
  const uint64_t n = r.n, total = r.jsonl_len;  // every byte of the JSONL belongs to a line that takes part
  if (!n || !total) return TGI_OK;
  if (n > 0xFFFFFFF0ull) { set_err(c, "tgi_channel_appends: %llu records (at most 2^32 - 16)", (unsigned long long)n); return TGI_E_CAPACITY; }
  Slot& s = c->slots[slot];
  LocalBufs& z = s.local;
  cudaStream_t st = s.stream;
  const uint64_t nc = src.n_chans, n2 = n + 2;
  const uint64_t gmax = std::min<uint64_t>(n, nc);  // groups: at most one per record and one per row
  const uint64_t tslots = next_pow2(std::max<uint64_t>(2 * nc, 64));
  CK(z.table.ensure(tslots * 4));
  CK(z.rows.ensure(2 * nc * 4));
  CK(z.u32s.ensure(11 * n2 * 4));
  CK(z.u64s.ensure(7 * n2 * 8));
  CK(z.groups.ensure(gmax * sizeof(tgi_channel_group)));
  CK(z.order.ensure(n * 8));
  CK(z.data.ensure(total));
  CK(z.sc.ensure(LA_SC_COUNT * 8));
  CK(z.h_groups.ensure(gmax * sizeof(tgi_channel_group)));
  CK(z.h_order.ensure(n * 8));
  CK(z.h_data.ensure(total + 1));
  CK(z.h_sc.ensure(LA_SC_COUNT * 8));
  LaWork w{};
  w.sc = z.sc.as<uint64_t>();
  w.table = z.table.as<uint32_t>();
  w.tmask = tslots - 1;
  w.canon = z.rows.as<uint32_t>();
  w.first_line = w.canon + nc;
  uint32_t* u = z.u32s.as<uint32_t>();
  uint32_t** u32_arrays[] = {&w.flag, &w.gflag, &w.lrec, &w.lkey, &w.run_start, &w.keys[0], &w.keys[1], &w.vals[0],
                             &w.vals[1], &w.cnt, &w.inv};
  for (size_t k = 0; k < sizeof u32_arrays / sizeof *u32_arrays; k++) *u32_arrays[k] = u + k * n2;
  uint64_t* v = z.u64s.as<uint64_t>();
  uint64_t** u64_arrays[] = {&w.pos, &w.rpos, &w.gpos, &w.lpos, &w.goff, &w.rsrc, &w.rdst};
  for (size_t k = 0; k < sizeof u64_arrays / sizeof *u64_arrays; k++) *u64_arrays[k] = v + k * n2;
  w.groups = z.groups.as<tgi_channel_group>();
  w.order = z.order.as<uint64_t>();
  w.data = z.data.as<uint8_t>();
  uint32_t launches = 0;
  auto grid = [&](uint64_t items) { return sink_grid(c, items, LA_THREADS, 16); };
  CK(cudaMemsetAsync(w.table, 0xFF, tslots * 4, st));
  CK(cudaMemsetAsync(w.first_line, 0xFF, nc * 4, st));
  CK(cudaMemsetAsync(w.sc, 0, LA_SC_COUNT * 8, st));
  CK(cudaEventRecord(s.ev_p0, st));
  la_canon_insert_kernel<<<grid(nc), LA_THREADS, 0, st>>>(src, w);
  la_canon_flag_kernel<<<grid(std::max(n, nc)), LA_THREADS, 0, st>>>(src, w);
  launches += 2;
  if ((rc = launch_scan(c, s, w.flag, n, w.pos, w.sc + LA_SC_LINES, launches))) return rc;
  la_compact_kernel<<<grid(n), LA_THREADS, 0, st>>>(src, w);
  la_flags_kernel<<<grid(n), LA_THREADS, 0, st>>>(n, w);
  launches += 2;
  if ((rc = launch_scan(c, s, w.flag, n, w.rpos, w.sc + LA_SC_RUNS, launches))) return rc;
  if ((rc = launch_scan(c, s, w.gflag, n, w.gpos, w.sc + LA_SC_GROUPS, launches))) return rc;
  la_runs_kernel<<<grid(n), LA_THREADS, 0, st>>>(n, w);
  launches++;
  const RadixPlan plan(gmax - 1);  // by group id
  if ((rc = radix_sort(c, st, s.d_tiles, w.keys, w.vals, w.sc + LA_SC_RUNS, n, plan, z.counts, z.roff, w.sc + LA_SC_RADIX, false,
                       launches)))
    return rc;
  const uint32_t* sorted = w.vals[plan.out];
  la_sorted_counts_kernel<<<grid(n), LA_THREADS, 0, st>>>(n, sorted, w);
  launches++;
  if ((rc = launch_scan(c, s, w.cnt, n, w.lpos, w.sc + LA_SC_SORTED_LINES, launches))) return rc;
  la_inverse_kernel<<<grid(n), LA_THREADS, 0, st>>>(sorted, w);
  la_order_kernel<<<grid(n), LA_THREADS, 0, st>>>(src, w);
  launches += 2;
  if ((rc = launch_scan(c, s, w.cnt, n, w.goff, w.sc + LA_SC_BYTES, launches))) return rc;
  la_tables_kernel<<<grid(n), LA_THREADS, 0, st>>>(src, w.keys[plan.out], sorted, w);
  la_gather_kernel<<<sink_grid(c, (total + 15) / 16, LA_GATHER_ITEMS * LA_THREADS, 8), LA_THREADS, 0, st>>>(src, w, total);
  launches += 2;
  CK(cudaGetLastError());
  CK(cudaEventRecord(s.ev_p1, st));
  // the read-back: the scalars, the group table and `order` at their upper bounds, the grouped bytes exactly
  CK(cudaMemcpyAsync(z.h_sc.p, w.sc, LA_SC_COUNT * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(z.h_groups.p, w.groups, gmax * sizeof(tgi_channel_group), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(z.h_order.p, w.order, n * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(z.h_data.p, w.data, total, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const uint64_t* hsc = z.h_sc.as<uint64_t>();
  const uint64_t lines = hsc[LA_SC_LINES], n_groups = hsc[LA_SC_GROUPS];
  if (hsc[LA_SC_BYTES] != total || hsc[LA_SC_SORTED_LINES] != lines || n_groups > gmax) {
    set_err(c, "tgi_channel_appends: %llu grouped bytes of %llu, %llu grouped lines of %llu", (unsigned long long)hsc[LA_SC_BYTES],
            (unsigned long long)total, (unsigned long long)hsc[LA_SC_SORTED_LINES], (unsigned long long)lines);
    return TGI_E_CUDA;
  }
  // the device left every group's first grouped line in n_lines and its first byte in byte_off: the next group's start
  // (or the end) turns them into counts
  tgi_channel_group* g = z.h_groups.as<tgi_channel_group>();
  for (uint64_t k = 0; k < n_groups; k++) {
    g[k].n_lines = (k + 1 < n_groups ? g[k + 1].n_lines : lines) - g[k].n_lines;
    g[k].byte_len = (k + 1 < n_groups ? g[k + 1].byte_off : total) - g[k].byte_off;
  }
  out->n_groups = n_groups;
  out->groups = g;
  out->data = z.h_data.as<uint8_t>();
  out->data_len = total;
  out->order = z.h_order.as<uint64_t>();
  cudaEventElapsedTime(&out->kernel_ms, s.ev_p0, s.ev_p1);
  out->gpu_launches = launches;
  return TGI_OK;
}

}  // extern "C"

// ---- combine mode (combine.cuh) ---------------------------------------------------------------------------------------
namespace {

// one launch of combine_encode_kernel being built: its tasks and their segments
struct CbPlan {
  std::vector<CbTask> t;
  std::vector<CbSeg> s;
  uint64_t units = 0;
  void add(uint8_t* dst, bool last, const std::vector<CbSeg>& segs) {
    CbTask k{dst, 0, units, (uint32_t)s.size(), (uint32_t)segs.size(), last ? 1u : 0u};
    for (const CbSeg& g : segs) k.bytes += g.len;
    if (!k.bytes) return;
    s.insert(s.end(), segs.begin(), segs.end());
    units += cb_units(k);
    t.push_back(k);
  }
};

// the kept lines of [a, b) as segments of the result's JSONL behind stream position pos (a dropped line splits a run)
void cb_runs(const uint64_t* off, const uint8_t* jsonl, uint64_t a, uint64_t b, const std::vector<uint64_t>& drops,
             std::vector<CbSeg>& segs, uint64_t& pos) {
  size_t k = std::lower_bound(drops.begin(), drops.end(), a) - drops.begin();
  while (a < b) {
    const bool d = k < drops.size() && drops[k] < b;
    const uint64_t e = d ? drops[k] : b;
    if (off[e] > off[a]) {
      segs.push_back({pos, off[e] - off[a], jsonl + off[a]});
      pos += off[e] - off[a];
    }
    a = d ? e + 1 : b;
    k++;
  }
}

// P's tasks: inline in the launch parameters, or in the device tables dt / ds
int cb_launch(tgi_ctx* c, cudaStream_t st, const CbPlan& P, const CbTask* dt, const CbSeg* ds, uint8_t* pend_out,
              uint32_t& launches) {
  if (!P.units) return TGI_OK;
  CbLaunch L{};
  L.n_tasks = (uint32_t)P.t.size();
  L.units = P.units;
  L.pend_out = pend_out;
  if (P.t.size() <= (size_t)CB_INLINE && P.s.size() <= (size_t)CB_INLINE) {
    std::copy(P.t.begin(), P.t.end(), L.t);
    std::copy(P.s.begin(), P.s.end(), L.s);
  } else {
    L.tasks = dt;
    L.segs = ds;
  }
  combine_encode_kernel<<<sink_grid(c, P.units, 256, 16), 256, 0, st>>>(L);
  launches++;
  CK(cudaGetLastError());
  return TGI_OK;
}

std::string cb_path(const Combiner& z, int64_t ns) {
  return z.prefix + "combined-posts/combined_" + std::to_string(ns) + ".jsonl";
}

// the next blob name: max(unix_nano, previous + 1)
int64_t cb_next_ns(Combiner& z, int64_t unix_nano) {
  const int64_t ns = z.any_ns && unix_nano <= z.last_ns ? z.last_ns + 1 : unix_nano;
  z.last_ns = ns;
  z.any_ns = true;
  return ns;
}

// the paths of out's blobs, once their data is in place
int cb_finish(tgi_ctx* c, Combiner& z, int64_t unix_nano, tgi_combined_blob* blobs, uint64_t k, tgi_combined_t* out) {
  std::string paths;
  for (uint64_t j = 0; j < k; j++) {
    const std::string p = cb_path(z, cb_next_ns(z, unix_nano));
    blobs[j].unix_nano = z.last_ns;
    blobs[j].path_off = paths.size();
    blobs[j].path_len = p.size();
    paths += p;
  }
  CK(z.h_path.ensure(paths.size() + 1));
  memcpy(z.h_path.p, paths.data(), paths.size());
  out->n_blobs = k;
  out->blobs = blobs;
  out->data = z.h_data.as<uint8_t>();
  out->path = z.h_path.as<uint8_t>();
  return TGI_OK;
}

}  // namespace

extern "C" {

int tgi_combine_open(tgi_ctx* c, uint64_t trigger, uint64_t hard_cap, const char* path_prefix, uint32_t prefix_len) {
  if (!c || (prefix_len && !path_prefix)) return TGI_E_ARG;
  Combiner& z = c->cb;
  std::lock_guard<std::mutex> g(z.mu);
  if (z.open && z.open_bytes) { set_err(c, "tgi_combine_open: the open group holds lines (tgi_combine_flush first)"); return TGI_E_STATE; }
  if (hard_cap >= (1ull << 62)) { set_err(c, "tgi_combine_open: hard_cap %llu cannot be allocated", (unsigned long long)hard_cap); return TGI_E_NOMEM; }
  cudaSetDevice(c->device);
  if (!z.ev) {
    CK(cudaStreamCreateWithFlags(&z.stream, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&z.ev, cudaEventDisableTiming));
    CK(cudaEventCreate(&z.t0));
    CK(cudaEventCreate(&z.t1));
  }
  if (z.ev_valid) CK(cudaEventSynchronize(z.ev));
  z.open = false;
  for (DevBuf* d : {&z.out, &z.tables, &z.drops, &z.counts}) d->release();  // a new stream starts with no scratch
  for (HostBuf* h : {&z.h_blobs, &z.h_data, &z.h_path, &z.h_tables, &z.h_drops, &z.h_counts, &z.h_line_off}) h->release();
  z.enc.release();  // exactly the largest blob: 4*ceil(hard_cap/3), plus the pad every device blob carries
  const size_t enc = (hard_cap + 2) / 3 * 4 + PAD;
  CK(cudaMalloc(&z.enc.p, enc));
  z.enc.cap = enc;
  CK(z.pend.ensure(64));
  z.trigger = trigger;
  z.hard_cap = hard_cap;
  z.prefix.assign(path_prefix ? path_prefix : "", prefix_len);
  z.open_lines = z.open_bytes = 0;
  z.cur = 0;
  z.open = true;
  return TGI_OK;
}

// The fast path (the lines fit in the open group) enqueues one launch.  Otherwise: the dropped lines and, for a
// TGI_RUN_NO_D2H result, the line offsets are read back; the host plans the groups; launch 1 encodes the blobs that
// close (the first one behind the open group's encoded bytes) and the open group if none closes, the closed blobs are
// copied to pinned memory, launch 2 encodes the new open group from the start of the (now copied) open buffer.
int tgi_combine_add(tgi_ctx* c, int slot, int64_t unix_nano, tgi_combined_t* out) {
  if (!c || !out) return TGI_E_ARG;
  LastResult r;
  int rc = sink_source(c, slot, "tgi_combine_add", r, nullptr, true);
  if (rc != TGI_OK) return rc;
  Combiner& z = c->cb;
  std::lock_guard<std::mutex> g(z.mu);
  if (!z.open) { set_err(c, "tgi_combine_add: no combiner is open (tgi_combine_open)"); return TGI_E_STATE; }
  memset(out, 0, sizeof *out);
  cudaStream_t st = c->slots[slot].stream;
  const uint64_t n = r.n, L = r.jsonl_len;
  uint8_t* pend_in = z.pend.as<uint8_t>() + 32 * z.cur;
  uint8_t* pend_out = z.pend.as<uint8_t>() + 32 * (1 - z.cur);
  uint8_t* enc = z.enc.as<uint8_t>();
  const uint64_t p0 = z.open_bytes % 3;
  const CbSeg pend{0, p0, pend_in};  // the open blob's pending bytes: its continuation's input starts with them
  uint32_t launches = 0;
  if (z.ev_valid) CK(cudaStreamWaitEvent(st, z.ev, 0));
  if (r.host_line_off && z.open_bytes + L < z.trigger && z.open_bytes + L <= z.hard_cap) {
    if (L) {
      const uint64_t* off = r.host_line_off;
      uint64_t lines = 0;
      for (uint64_t i = 0; i < n; i++) lines += off[i + 1] != off[i];
      std::vector<CbSeg> segs;
      if (p0) segs.push_back(pend);
      segs.push_back({p0, L, r.dev.jsonl + off[0]});
      CbPlan P;
      P.add(enc + z.open_bytes / 3 * 4, false, segs);
      rc = cb_launch(c, st, P, nullptr, nullptr, pend_out, launches);
      if (rc) return rc;
      CK(cudaEventRecord(z.ev, st));
      z.ev_valid = true;
      z.open_bytes += L;
      z.open_lines += lines;
      z.cur ^= 1;
    }
    out->open_lines = z.open_lines;
    out->open_bytes = z.open_bytes;
    out->gpu_launches = launches;
    return TGI_OK;
  }
  // 1. the dropped lines (at most L / (hard_cap + 1) of them) and the line offsets on the host
  const uint64_t max_drops = std::min<uint64_t>(n, L / (z.hard_cap + 1));
  CK(z.drops.ensure(8 * (1 + max_drops)));
  CK(z.h_drops.ensure(8 * (1 + max_drops)));
  uint64_t* d_drops = z.drops.as<uint64_t>();
  CK(cudaEventRecord(z.t0, st));
  CK(cudaMemsetAsync(d_drops, 0, 8, st));
  if (n && max_drops) {
    combine_drops_kernel<<<sink_grid(c, n, 256, 16), 256, 0, st>>>(r.dev.line_off, n, z.hard_cap, d_drops + 1, max_drops, (unsigned long long*)d_drops);
    launches++;
    CK(cudaGetLastError());
  }
  CK(cudaEventRecord(z.t1, st));
  CK(cudaMemcpyAsync(z.h_drops.p, d_drops, 8 * (1 + max_drops), cudaMemcpyDeviceToHost, st));
  const uint64_t* off = r.host_line_off;
  if (!off) {
    CK(z.h_line_off.ensure((n + 1) * 8));
    CK(cudaMemcpyAsync(z.h_line_off.p, r.dev.line_off, (n + 1) * 8, cudaMemcpyDeviceToHost, st));
    off = z.h_line_off.as<uint64_t>();
  }
  CK(cudaStreamSynchronize(st));
  float ms0 = 0;
  cudaEventElapsedTime(&ms0, z.t0, z.t1);
  uint64_t* hd = z.h_drops.as<uint64_t>();
  const uint64_t nd = std::min(hd[0], max_drops);
  std::vector<uint64_t> drops(hd + 1, hd + 1 + nd);
  std::sort(drops.begin(), drops.end());
  // 2. the groups (the rule of tgi_plan_chunks)
  std::vector<uint64_t> ends;
  uint64_t open_out = 0, open_begin = 0;
  rc = plan_groups(off, n, z.trigger, z.hard_cap, z.open_bytes, drops,
                   [&](uint64_t, uint64_t e) { ends.push_back(e); return true; }, &open_out, &open_begin);
  if (rc) return rc;
  const uint64_t k = ends.size();
  // 3. the tasks: closed group 0 continues the open blob in enc, closed groups 1.. go to `out` at 16-byte aligned
  // offsets, the group left open (index k) continues enc (nothing closed: launch 1) or restarts it (launch 2)
  std::vector<std::vector<CbSeg>> gsegs(k + 1);
  std::vector<uint64_t> raw(k + 1), dev_off(k + 1, 0);
  uint64_t out_bytes = 0;
  for (uint64_t j = 0; j <= k; j++) {
    if (!j && p0) gsegs[j].push_back(pend);
    uint64_t pos = j ? 0 : p0;
    cb_runs(off, r.dev.jsonl, j ? ends[j - 1] : 0, j < k ? ends[j] : n, drops, gsegs[j], pos);
    raw[j] = pos + (j ? 0 : z.open_bytes - p0);
    if (j && j < k) {
      dev_off[j] = out_bytes;
      out_bytes += ((raw[j] + 2) / 3 * 4 + 15) & ~15ull;
    }
  }
  CK(z.out.ensure(out_bytes));
  uint8_t* cont = enc + z.open_bytes / 3 * 4;  // where the open blob continues
  CbPlan P1, P2;
  for (uint64_t j = 0; j < k; j++) P1.add(j ? z.out.as<uint8_t>() + dev_off[j] : cont, true, gsegs[j]);
  if (k) P2.add(enc, false, gsegs[k]);
  else P1.add(cont, false, gsegs[0]);
  // tables: ends | P1 tasks | P1 segs | P2 tasks | P2 segs, one copy
  const size_t tb = 8 * k, t1b = sizeof(CbTask) * P1.t.size(), s1b = sizeof(CbSeg) * P1.s.size(),
               t2b = sizeof(CbTask) * P2.t.size(), s2b = sizeof(CbSeg) * P2.s.size(), all = tb + t1b + s1b + t2b + s2b;
  CK(z.tables.ensure(all));
  CK(z.h_tables.ensure(all));
  uint8_t* ht = z.h_tables.as<uint8_t>();
  memcpy(ht, ends.data(), tb);
  memcpy(ht + tb, P1.t.data(), t1b);
  memcpy(ht + tb + t1b, P1.s.data(), s1b);
  memcpy(ht + tb + t1b + s1b, P2.t.data(), t2b);
  memcpy(ht + tb + t1b + s1b + t2b, P2.s.data(), s2b);
  uint8_t* dtb = z.tables.as<uint8_t>();
  if (all) CK(cudaMemcpyAsync(dtb, ht, all, cudaMemcpyHostToDevice, st));
  CK(z.counts.ensure(8 * (k + 1)));
  CK(z.h_counts.ensure(8 * (k + 1)));
  uint64_t data_bytes = 0;
  for (uint64_t j = 0; j < k; j++) data_bytes += (raw[j] + 2) / 3 * 4;
  CK(z.h_data.ensure(data_bytes + 1));
  CK(z.h_blobs.ensure(sizeof(tgi_combined_blob) * (k + 1)));
  // 4. posts per group, launch 1, the copies of the closed blobs, launch 2
  CK(cudaEventRecord(z.t0, st));
  CK(cudaMemsetAsync(z.counts.p, 0, 8 * (k + 1), st));
  if (n) {
    combine_count_kernel<<<sink_grid(c, n, 256, 16), 256, 0, st>>>(r.dev.line_off, n, z.hard_cap, (const uint64_t*)dtb,
                                                                   (uint32_t)k, z.counts.as<unsigned long long>());
    launches++;
    CK(cudaGetLastError());
  }
  rc = cb_launch(c, st, P1, (const CbTask*)(dtb + tb), (const CbSeg*)(dtb + tb + t1b), pend_out, launches);
  if (rc) return rc;
  CK(cudaEventRecord(z.t1, st));
  tgi_combined_blob* blobs = z.h_blobs.as<tgi_combined_blob>();
  uint64_t hoff = 0;
  for (uint64_t j = 0; j < k; j++) {
    const uint64_t len = (raw[j] + 2) / 3 * 4;
    const uint8_t* src = j ? z.out.as<uint8_t>() + dev_off[j] : enc;
    if (len) CK(cudaMemcpyAsync(z.h_data.as<uint8_t>() + hoff, src, len, cudaMemcpyDeviceToHost, st));
    blobs[j] = tgi_combined_blob{hoff, len, 0, 0, 0, raw[j], 0};
    hoff += len;
  }
  rc = cb_launch(c, st, P2, (const CbTask*)(dtb + tb + t1b + s1b), (const CbSeg*)(dtb + tb + t1b + s1b + t2b), pend_out, launches);
  if (rc) return rc;
  CK(cudaMemcpyAsync(z.h_counts.p, z.counts.p, 8 * (k + 1), cudaMemcpyDeviceToHost, st));
  CK(cudaEventRecord(z.ev, st));
  z.ev_valid = true;
  CK(cudaStreamSynchronize(st));
  float ms1 = 0;
  cudaEventElapsedTime(&ms1, z.t0, z.t1);
  const uint64_t* cnt = z.h_counts.as<uint64_t>();
  for (uint64_t j = 0; j < k; j++) blobs[j].n_lines = cnt[j] + (j ? 0 : z.open_lines);
  z.open_lines = cnt[k] + (k ? 0 : z.open_lines);
  z.open_bytes = open_out;
  z.cur ^= 1;
  rc = cb_finish(c, z, unix_nano, blobs, k, out);
  if (rc) return rc;
  out->n_dropped = nd;
  memcpy(hd + 1, drops.data(), 8 * nd);
  out->dropped = hd + 1;
  out->open_lines = z.open_lines;
  out->open_bytes = z.open_bytes;
  out->kernel_ms = ms0 + ms1;
  out->gpu_launches = launches;
  return TGI_OK;
}

int tgi_combine_flush(tgi_ctx* c, int64_t unix_nano, tgi_combined_t* out) {
  if (!c || !out) return TGI_E_ARG;
  Combiner& z = c->cb;
  std::lock_guard<std::mutex> g(z.mu);
  if (!z.open) { set_err(c, "tgi_combine_flush: no combiner is open (tgi_combine_open)"); return TGI_E_STATE; }
  cudaSetDevice(c->device);
  memset(out, 0, sizeof *out);
  if (!z.open_bytes) return TGI_OK;
  cudaStream_t st = z.stream;
  const uint64_t p0 = z.open_bytes % 3, len = (z.open_bytes + 2) / 3 * 4;
  uint32_t launches = 0;
  if (z.ev_valid) CK(cudaStreamWaitEvent(st, z.ev, 0));
  CbPlan P;
  P.add(z.enc.as<uint8_t>() + z.open_bytes / 3 * 4, true, {{0, p0, z.pend.as<uint8_t>() + 32 * z.cur}});
  CK(cudaEventRecord(z.t0, st));
  int rc = cb_launch(c, st, P, nullptr, nullptr, nullptr, launches);
  if (rc) return rc;
  CK(cudaEventRecord(z.t1, st));
  CK(z.h_data.ensure(len + 1));
  CK(z.h_blobs.ensure(sizeof(tgi_combined_blob)));
  CK(cudaMemcpyAsync(z.h_data.p, z.enc.p, len, cudaMemcpyDeviceToHost, st));
  CK(cudaEventRecord(z.ev, st));
  z.ev_valid = true;
  CK(cudaStreamSynchronize(st));
  tgi_combined_blob* blobs = z.h_blobs.as<tgi_combined_blob>();
  blobs[0] = tgi_combined_blob{0, len, 0, 0, z.open_lines, z.open_bytes, 0};
  z.open_lines = z.open_bytes = 0;
  rc = cb_finish(c, z, unix_nano, blobs, 1, out);
  if (rc) return rc;
  cudaEventElapsedTime(&out->kernel_ms, z.t0, z.t1);
  out->gpu_launches = launches;
  return TGI_OK;
}


// ---- pinned input staging ---------------------------------------------------------------------------------
int tgi_acquire_staging(tgi_ctx* c, uint64_t bytes, void** out) {
  if (!c || !out) return TGI_E_ARG;
  cudaSetDevice(c->device);
  if (bytes == 0) bytes = 1;
  std::lock_guard<std::mutex> g(c->stg_mu);
  auto it = c->stg_free.lower_bound(bytes);
  if (it != c->stg_free.end() && it->first <= bytes + bytes / 2 + 4096) {  // recycle a block that is not much larger
    *out = it->second;
    c->stg_live[it->second] = it->first;
    c->stg_free.erase(it);
    return TGI_OK;
  }
  const size_t want = (bytes + 4095 + 64) & ~(size_t)4095;
  void* p = nullptr;
  cudaError_t e = cudaHostAlloc(&p, want, cudaHostAllocDefault);
  if (e != cudaSuccess) {
    set_err(c, "cudaHostAlloc(%zu) failed: %s", want, cudaGetErrorString(e));
    return TGI_E_NOMEM;
  }
  c->stg_live[p] = want;
  *out = p;
  return TGI_OK;
}
int tgi_release_staging(tgi_ctx* c, void* block) {
  if (!c || !block) return TGI_E_ARG;
  std::lock_guard<std::mutex> g(c->stg_mu);
  auto it = c->stg_live.find(block);
  if (it == c->stg_live.end()) { set_err(c, "tgi_release_staging: not a live staging block"); return TGI_E_ARG; }
  size_t held = 0;
  for (auto& f : c->stg_free) held += f.first;
  if (held + it->second > (4ull << 30)) cudaFreeHost(block);  // keep at most 4 GiB of idle pinned memory around
  else c->stg_free.emplace(it->second, block);
  c->stg_live.erase(it);
  return TGI_OK;
}

// ---- multi-GPU merge (SURVEY 8e option A) ---------------------------------------------------------------------
#define NK(call)                                                                                  \
  do {                                                                                            \
    ncclResult_t _r = (call);                                                                     \
    if (_r != ncclSuccess) {                                                                      \
      set_err(c, "%s failed: %s", #call, c->nccl && c->nccl->GetErrorString ? c->nccl->GetErrorString(_r) : "?"); \
      return TGI_E_CUDA;                                                                          \
    }                                                                                             \
  } while (0)

static NcclApi* load_nccl(std::string& why) {
  static std::mutex mu;
  static NcclApi api;
  std::lock_guard<std::mutex> g(mu);
  if (api.h) return &api;
  void* h = nullptr;
  for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
    h = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
    if (h) break;
  }
  if (!h) { why = std::string("cannot load libnccl.so.2: ") + (dlerror() ? dlerror() : "?"); return nullptr; }
#define SYM(field, name)                                        \
  api.field = (decltype(api.field))dlsym(h, name);              \
  if (!api.field) { why = std::string("libnccl lacks ") + name; return nullptr; }
  SYM(GetUniqueId, "ncclGetUniqueId") SYM(CommInitRank, "ncclCommInitRank") SYM(CommDestroy, "ncclCommDestroy")
  SYM(AllGather, "ncclAllGather") SYM(AllReduce, "ncclAllReduce") SYM(Broadcast, "ncclBroadcast") SYM(Send, "ncclSend")
  SYM(Recv, "ncclRecv") SYM(GroupStart, "ncclGroupStart") SYM(GroupEnd, "ncclGroupEnd") SYM(GetErrorString, "ncclGetErrorString")
#undef SYM
  api.h = h;
  return &api;
}

int tgi_comm_unique_id(uint8_t id[TGI_COMM_ID_BYTES]) {
  if (!id) return TGI_E_ARG;
  std::string why;
  NcclApi* a = load_nccl(why);
  if (!a) { set_err(nullptr, "%s", why.c_str()); return TGI_E_STATE; }
  ncclUniqueId u;
  static_assert(sizeof(u) == TGI_COMM_ID_BYTES, "ncclUniqueId is 128 bytes");
  if (a->GetUniqueId(&u) != ncclSuccess) { set_err(nullptr, "ncclGetUniqueId failed"); return TGI_E_CUDA; }
  memcpy(id, &u, sizeof u);
  return TGI_OK;
}

int tgi_comm_init(tgi_ctx* c, const uint8_t id[TGI_COMM_ID_BYTES], int rank, int nranks) {
  if (!c || !id || nranks < 1 || nranks > 64 || rank < 0 || rank >= nranks) return TGI_E_ARG;
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> g(c->fr_mu);
  if (c->comm) { set_err(c, "communicator already initialised"); return TGI_E_STATE; }
  std::string why;
  c->nccl = load_nccl(why);
  if (!c->nccl) { set_err(c, "%s", why.c_str()); return TGI_E_STATE; }
  ncclUniqueId u;
  memcpy(&u, id, sizeof u);
  NK(c->nccl->CommInitRank(&c->comm, nranks, u, rank));
  c->rank = rank;
  c->nranks = nranks;
  // this rank's partition of the global set: sized like the local set (a skewed hash cannot overflow it before the
  // local sets do)
  const FrontierDev& fr = c->sets[TGI_SET_FRONTIER].dev;
  const int rc = set_alloc(c, c->sets[TGI_SET_OWNED], fr.cap, fr.tmask + 1, true);
  if (rc) return rc;
  cudaStream_t st = c->slots[0].stream;
  CK(c->m_cnt.ensure(64 * 8));
  CK(c->m_all.ensure(64 * 64 * 8));
  CK(c->m_cursor.ensure(64 * 8));
  CK(c->m_gsize.ensure(16));
  CK(c->m_host.ensure(64 * 64 * 8 + 64));
  for (auto& e : c->m_ev) CK(cudaEventCreate(&e));
  CK(cudaStreamSynchronize(st));
  c->merged_upto = 0;
  c->merge_round = 0;
  return TGI_OK;
}

int tgi_comm_destroy(tgi_ctx* c) {
  if (!c) return TGI_E_ARG;
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> g(c->fr_mu);
  if (c->comm) {
    cudaStreamSynchronize(c->slots[0].stream);
    c->nccl->CommDestroy(c->comm);
    c->comm = nullptr;
  }
  for (auto& e : c->m_ev) if (e) { cudaEventDestroy(e); e = nullptr; }
  c->sets[TGI_SET_OWNED].dev = FrontierDev{};
  return TGI_OK;
}

int tgi_frontier_merge(tgi_ctx* c, uint64_t* global_size, uint64_t* owned) {
  if (!c) return TGI_E_ARG;
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> g(c->fr_mu);
  if (!c->comm) { set_err(c, "tgi_frontier_merge needs tgi_comm_init first"); return TGI_E_STATE; }
  NcclApi& N = *c->nccl;
  const int G = c->nranks, me = c->rank;
  cudaStream_t st = c->slots[0].stream;
  uint64_t* hb = c->m_host.as<uint64_t>();
  const uint8_t* pool = c->sets[TGI_SET_FRONTIER].dev.pool;
  KeySet& part = c->sets[TGI_SET_OWNED];  // this rank's partition
  uint64_t sz = 0;
  int rc = set_count(c, c->sets[TGI_SET_FRONTIER], &sz);
  if (rc) return rc;
  const uint64_t first = c->merged_upto, m = sz > first ? sz - first : 0;
  // 1. how many of my new keys go to each owner; every rank learns every count
  CK(cudaEventRecord(c->m_ev[0], st));
  CK(cudaMemsetAsync(c->m_cnt.p, 0, 64 * 8, st));
  if (m) merge_count_kernel<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(pool, first, m, (uint32_t)G, c->m_cnt.as<unsigned long long>());
  CK(cudaGetLastError());
  NK(N.AllGather(c->m_cnt.p, c->m_all.p, (size_t)G, ncclUint64, c->comm, st));
  CK(cudaMemcpyAsync(hb, c->m_all.p, (size_t)G * G * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  std::vector<uint64_t> send_off(G + 1, 0), recv_off(G + 1, 0);
  for (int p = 0; p < G; p++) {
    send_off[p + 1] = send_off[p] + hb[(size_t)me * G + p];
    recv_off[p + 1] = recv_off[p] + hb[(size_t)p * G + me];
  }
  const uint64_t R = recv_off[G];
  if (send_off[G] != m) { set_err(c, "merge: bucket counts do not add up"); return TGI_E_STATE; }
  // 2. bucket my new keys by owner
  CK(c->m_send_keys.ensure(m * 32));
  CK(c->m_send_pay.ensure(m * 8));
  CK(c->m_recv_keys.ensure(R * 32));
  CK(c->m_recv_pay.ensure(R * 8));
  uint64_t* hcur = hb + (size_t)G * G;
  for (int p = 0; p < G; p++) hcur[p] = send_off[p];
  CK(cudaMemcpyAsync(c->m_cursor.p, hcur, (size_t)G * 8, cudaMemcpyHostToDevice, st));
  const uint64_t pay_base = (c->merge_round << 52) | ((uint64_t)me << 44);
  if (m) merge_scatter_kernel<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(pool, first, m, (uint32_t)G, c->m_cursor.as<unsigned long long>(),
                                                                      c->m_send_keys.as<uint8_t>(), c->m_send_pay.as<uint64_t>(), pay_base);
  CK(cudaGetLastError());
  CK(cudaEventRecord(c->m_ev[1], st));
  // 3. exchange: grouped send / recv, the receive buffer laid out by source rank
  NK(N.GroupStart());
  for (int p = 0; p < G; p++) {
    const uint64_t sc = send_off[p + 1] - send_off[p], rc2 = recv_off[p + 1] - recv_off[p];
    if (p == me) continue;
    if (sc) {
      NK(N.Send(c->m_send_keys.as<uint8_t>() + 32 * send_off[p], sc * 32, ncclUint8, p, c->comm, st));
      NK(N.Send(c->m_send_pay.as<uint64_t>() + send_off[p], sc, ncclUint64, p, c->comm, st));
    }
    if (rc2) {
      NK(N.Recv(c->m_recv_keys.as<uint8_t>() + 32 * recv_off[p], rc2 * 32, ncclUint8, p, c->comm, st));
      NK(N.Recv(c->m_recv_pay.as<uint64_t>() + recv_off[p], rc2, ncclUint64, p, c->comm, st));
    }
  }
  NK(N.GroupEnd());
  {
    const uint64_t sc = send_off[me + 1] - send_off[me];
    if (sc) {
      CK(cudaMemcpyAsync(c->m_recv_keys.as<uint8_t>() + 32 * recv_off[me], c->m_send_keys.as<uint8_t>() + 32 * send_off[me], sc * 32, cudaMemcpyDeviceToDevice, st));
      CK(cudaMemcpyAsync(c->m_recv_pay.as<uint64_t>() + recv_off[me], c->m_send_pay.as<uint64_t>() + send_off[me], sc * 8, cudaMemcpyDeviceToDevice, st));
    }
  }
  CK(cudaEventRecord(c->m_ev[2], st));
  // 4. the owner inserts what it received (source-rank-major: the lowest rank's copy of a key wins)
  if (R) {
    rc = frontier_insert_enqueue(c, part, c->m_recv_keys.p, c->m_recv_pay.as<uint64_t>(), R, nullptr);
    if (rc) return rc;
  }
  // 5. global size = sum of the partitions
  NK(N.AllReduce(part.dev.count, c->m_gsize.p, 1, ncclUint64, ncclSum, c->comm, st));
  CK(cudaEventRecord(c->m_ev[3], st));
  CK(cudaMemcpyAsync(hb, c->m_gsize.p, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(hb + 1, part.dev.count, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (R) {
    rc = frontier_insert_check(c, part);
    if (rc) return rc;
  }
  if (global_size) *global_size = hb[0];
  if (owned) *owned = hb[1];
  float t0 = 0, t1 = 0, t2 = 0;
  cudaEventElapsedTime(&t0, c->m_ev[0], c->m_ev[1]);
  cudaEventElapsedTime(&t1, c->m_ev[1], c->m_ev[2]);
  cudaEventElapsedTime(&t2, c->m_ev[2], c->m_ev[3]);
  c->mstats.merges++;
  c->mstats.keys_sent += m - (send_off[me + 1] - send_off[me]);
  c->mstats.keys_received += R - (recv_off[me + 1] - recv_off[me]);
  c->mstats.keys_owned = hb[1];
  c->mstats.bytes_sent += (m - (send_off[me + 1] - send_off[me])) * 40;
  c->mstats.bucket_ms += t0;
  c->mstats.exchange_ms += t1;
  c->mstats.insert_ms += t2;
  c->mstats.last_bucket_ms = t0;
  c->mstats.last_exchange_ms = t1;
  c->mstats.last_insert_ms = t2;
  c->merged_upto = sz;
  c->merge_round++;
  return TGI_OK;
}

int tgi_merge_get_stats(tgi_ctx* c, tgi_merge_stats* out) {
  if (!c || !out) return TGI_E_ARG;
  std::lock_guard<std::mutex> g(c->fr_mu);
  *out = c->mstats;
  return TGI_OK;
}

int tgi_frontier_global_export(tgi_ctx* c, uint8_t* keys32, uint64_t cap, uint64_t* n) {
  if (!c || !n) return TGI_E_ARG;
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> g(c->fr_mu);
  if (!c->comm) { set_err(c, "tgi_frontier_global_export needs tgi_comm_init first"); return TGI_E_STATE; }
  NcclApi& N = *c->nccl;
  const int G = c->nranks;
  cudaStream_t st = c->slots[0].stream;
  uint64_t* hb = c->m_host.as<uint64_t>();
  const FrontierDev& owned = c->sets[TGI_SET_OWNED].dev;
  if (c->fr_event_valid) CK(cudaStreamWaitEvent(st, c->fr_event, 0));
  NK(N.AllGather(owned.count, c->m_all.p, 1, ncclUint64, c->comm, st));
  CK(cudaMemcpyAsync(hb, c->m_all.p, (size_t)G * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  std::vector<uint64_t> off(G + 1, 0);
  for (int p = 0; p < G; p++) off[p + 1] = off[p] + hb[p];
  const uint64_t T = off[G];
  DevBuf dk, dp;
  CK(dk.ensure(T * 32));
  CK(dp.ensure(T * 8));
  for (int p = 0; p < G; p++) {
    const uint64_t cnt = off[p + 1] - off[p];
    if (!cnt) continue;
    NK(N.Broadcast(owned.pool, dk.as<uint8_t>() + 32 * off[p], cnt * 32, ncclUint8, p, c->comm, st));
    NK(N.Broadcast(owned.payload, dp.as<uint64_t>() + off[p], cnt, ncclUint64, p, c->comm, st));
  }
  std::vector<uint8_t> hk(T * 32);
  std::vector<uint64_t> hp(T);
  if (T) {
    CK(cudaMemcpyAsync(hk.data(), dk.p, T * 32, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(hp.data(), dp.p, T * 8, cudaMemcpyDeviceToHost, st));
  }
  CK(cudaStreamSynchronize(st));
  std::vector<uint64_t> idx(T);
  for (uint64_t i = 0; i < T; i++) idx[i] = i;
  std::sort(idx.begin(), idx.end(), [&](uint64_t a, uint64_t b) { return hp[a] < hp[b]; });
  const uint64_t m = T < cap ? T : cap;
  if (keys32)
    for (uint64_t i = 0; i < m; i++) memcpy(keys32 + 32 * i, hk.data() + 32 * idx[i], 32);
  *n = T;
  return TGI_OK;
}

int tgi_filter_usernames(tgi_ctx* c, const uint8_t* names, const uint32_t* off, uint64_t n, uint8_t* reason) {
  if (!c || !off || !reason) return TGI_E_ARG;
  cudaSetDevice(c->device);
  if (!n) return TGI_OK;
  DevBuf dn, doff, dr;
  uint32_t total = off[n];
  CK(dn.ensure(total));
  CK(doff.ensure((n + 1) * 4));
  CK(dr.ensure(n));
  CK(cudaMemset(dn.p, 0, total + PAD));
  if (total) CK(cudaMemcpy(dn.p, names, total, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(doff.p, off, (n + 1) * 4, cudaMemcpyHostToDevice));
  unsigned g = (unsigned)((n * 32 + 255) / 256);
  filter_usernames_kernel<<<g, 256>>>(dn.as<uint8_t>(), doff.as<uint32_t>(), n, dr.as<uint8_t>());
  CK(cudaGetLastError());
  CK(cudaMemcpy(reason, dr.p, n, cudaMemcpyDeviceToHost));
  dn.release();
  doff.release();
  dr.release();
  return TGI_OK;
}

}  // extern "C"

// ---- crawl progress state (state.cuh) ---------------------------------------------------------------------------------
namespace {

const char* const kPresetCodes[] = {"", "unfetched", "fetched", "failed", "deleted", "resample"};

std::string st_field(const CrawlState& S, const tgi_state_page& p, int f) {
  uint64_t o = p.str_off;
  for (int k = 0; k < f; k++) o += p.str_len[k];
  return S.blob.substr(o, p.str_len[f]);
}
std::string in_field(const tgi_state_page& p, const uint8_t* strs, int f) {
  uint64_t o = p.str_off;
  for (int k = 0; k < f; k++) o += p.str_len[k];
  return std::string((const char*)strs + o, p.str_len[f]);
}
uint64_t page_str_bytes(const tgi_state_page& p) {
  uint64_t t = 0;
  for (int k = 0; k < TGI_PS_COUNT; k++) t += p.str_len[k];
  return t;
}
bool page_ok(tgi_ctx* c, const tgi_state_page& p, const uint8_t* strs, uint64_t strs_len, const char* who) {
  const uint64_t t = page_str_bytes(p);
  if ((t && !strs) || p.str_off > strs_len || t > strs_len - p.str_off) { set_err(c, "%s: page strings outside strs", who); return false; }
  if (p.ts_nsec < 0 || p.ts_nsec >= 1000000000) { set_err(c, "%s: ts_nsec %d out of range", who, p.ts_nsec); return false; }
  if (p.ts_off != TGI_STATE_TS_LOCAL && (p.ts_off <= -86400 || p.ts_off >= 86400)) { set_err(c, "%s: ts_off %d is a day or more", who, p.ts_off); return false; }
  return true;
}

// the state's stream, events, preset codes and minimal buffers, on first use (under S.mu).  Every state call but
// tgi_state_edge_sql, tgi_state_walkback and tgi_state_rw_step passes here, so this is also where the hand-off and the
// lookups' lists end.
int st_init(tgi_ctx* c, CrawlState& S) {
  cudaSetDevice(c->device);
  S.handoff_live = false;
  S.rw_live = false;
  if (S.stream) return TGI_OK;
  CK(cudaStreamCreateWithFlags(&S.stream, cudaStreamNonBlocking));
  CK(cudaEventCreate(&S.t0));
  CK(cudaEventCreate(&S.t1));
  CK(cudaEventCreate(&S.t2));
  CK(cudaEventCreate(&S.t3));
  CK(cudaEventCreate(&S.t4));
  CK(cudaEventCreate(&S.t5));
  CK(cudaEventCreateWithFlags(&S.ev_slot, cudaEventDisableTiming));
  CK(cudaEventCreateWithFlags(&S.ev_seg, cudaEventDisableTiming));
  for (const char* s : kPresetCodes) {
    S.code_of[s] = (uint16_t)S.codes.size();
    S.codes.push_back(s);
  }
  for (DevBuf* b : {&S.pages, &S.dblob, &S.row_gen, &S.row_cnt, &S.msgs}) CK(b->ensure(64));
  S.tslots = 1024;
  CK(S.table.ensure(S.tslots * 4));
  CK(cudaMemsetAsync(S.table.p, 0xFF, S.tslots * 4, S.stream));
  return TGI_OK;
}

// b holds `used` bytes that must survive; make room for `need`
int st_grow(tgi_ctx* c, CrawlState& S, DevBuf& b, size_t used, size_t need) {
  if (need + PAD <= b.cap) return TGI_OK;
  DevBuf n;
  CK(n.ensure(std::max(need, 2 * used)));
  if (used) CK(cudaMemcpyAsync(n.p, b.p, used, cudaMemcpyDeviceToDevice, S.stream));
  CK(cudaStreamSynchronize(S.stream));
  b.swap(n);
  return TGI_OK;
}

StDev st_dev(const CrawlState& S) {
  StDev d{};
  d.pages = S.pages.as<tgi_state_page>();
  d.blob = S.dblob.as<uint8_t>();
  d.row_gen = S.row_gen.as<uint32_t>();
  d.row_cnt = S.row_cnt.as<uint32_t>();
  d.msgs = S.msgs.as<StMsg>();
  d.table = S.table.as<uint32_t>();
  d.tmask = S.tslots - 1;
  d.codes = StCodes{S.code_blob.as<uint8_t>(), S.code_off.as<uint32_t>()};
  return d;
}
unsigned st_grid(const tgi_ctx* c, uint64_t n) { return sink_grid(c, n, ST_THREADS, 16); }

// writes row r (a new row when r == rows.size()) from page p, its strings appended to the blob; keeps the id / URL maps
// and the deadend count
void st_put_row(CrawlState& S, uint32_t r, const tgi_state_page& p, const uint8_t* strs) {
  if (r < S.rows.size()) {
    const std::string url = st_field(S, S.rows[r], TGI_PS_URL);
    if (--S.urls[url] == 0) S.urls.erase(url);
    if (st_field(S, S.rows[r], TGI_PS_STATUS) == "deadend") S.deadends--;
  }
  tgi_state_page q = p;
  q.str_off = S.blob.size();
  q.n_msgs = 0;
  S.blob.append((const char*)strs + p.str_off, page_str_bytes(p));
  S.urls[in_field(p, strs, TGI_PS_URL)]++;
  if (in_field(p, strs, TGI_PS_STATUS) == "deadend") S.deadends++;
  if (r == S.rows.size()) {
    S.rows.push_back(q);
    S.gen.push_back(0);
    S.by_id[in_field(p, strs, TGI_PS_ID)] = r;
  } else {
    S.rows[r] = q;
  }
}

// the rows and strings the device does not have yet, and the rewritten rows in `dirty` (their gen too; their message
// count is set to 0, as for new rows)
int st_sync_rows(tgi_ctx* c, CrawlState& S, const std::vector<uint32_t>& dirty) {
  cudaStream_t st = S.stream;
  const uint64_t nr = S.rows.size(), r0 = S.rows_synced;
  int rc;
  if ((rc = st_grow(c, S, S.dblob, S.blob_synced, S.blob.size()))) return rc;
  if (S.blob.size() > S.blob_synced)
    CK(cudaMemcpyAsync(S.dblob.as<uint8_t>() + S.blob_synced, S.blob.data() + S.blob_synced, S.blob.size() - S.blob_synced,
                       cudaMemcpyHostToDevice, st));
  S.blob_synced = S.blob.size();
  if ((rc = st_grow(c, S, S.pages, r0 * sizeof(tgi_state_page), nr * sizeof(tgi_state_page)))) return rc;
  if ((rc = st_grow(c, S, S.row_gen, r0 * 4, nr * 4))) return rc;
  if ((rc = st_grow(c, S, S.row_cnt, r0 * 4, (nr + 1) * 4))) return rc;
  if (nr > r0) {
    CK(cudaMemcpyAsync(S.pages.as<tgi_state_page>() + r0, S.rows.data() + r0, (nr - r0) * sizeof(tgi_state_page), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(S.row_gen.as<uint32_t>() + r0, S.gen.data() + r0, (nr - r0) * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(S.row_cnt.as<uint32_t>() + r0, 0, (nr - r0) * 4, st));
  }
  for (uint32_t r : dirty) {
    if (r >= r0) continue;
    CK(cudaMemcpyAsync(S.pages.as<tgi_state_page>() + r, &S.rows[r], sizeof(tgi_state_page), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(S.row_gen.as<uint32_t>() + r, &S.gen[r], 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(S.row_cnt.as<uint32_t>() + r, 0, 4, st));
  }
  S.rows_synced = nr;
  CK(cudaStreamSynchronize(st));  // the host rows may move once this returns
  return TGI_OK;
}

int st_row_count(tgi_ctx* c, CrawlState& S, uint32_t r, uint32_t* n) {
  CK(cudaMemcpyAsync(n, S.row_cnt.as<uint32_t>() + r, 4, cudaMemcpyDeviceToHost, S.stream));
  CK(cudaStreamSynchronize(S.stream));
  return TGI_OK;
}

// the lookup table at `slots` slots, rebuilt from the live messages
int st_rebuild_table(tgi_ctx* c, CrawlState& S, uint64_t slots) {
  if (slots != S.tslots) {
    CK(cudaStreamSynchronize(S.stream));
    CK(S.table.ensure(slots * 4));
    S.tslots = slots;
  }
  CK(cudaMemsetAsync(S.table.p, 0xFF, slots * 4, S.stream));
  if (S.n_msgs) st_table_insert_kernel<<<st_grid(c, S.n_msgs), ST_THREADS, 0, S.stream>>>(st_dev(S), 0, S.n_msgs);
  CK(cudaGetLastError());
  return TGI_OK;
}

// room for `extra` more message rows, in the buffer and at a table load of at most one half
int st_reserve(tgi_ctx* c, CrawlState& S, uint64_t extra) {
  const uint64_t need = S.n_msgs + extra;
  if (need >= 0xFFFFFFFEull) { set_err(c, "state: %llu message rows (at most 2^32 - 2)", (unsigned long long)need); return TGI_E_CAPACITY; }
  int rc;
  if ((rc = st_grow(c, S, S.msgs, S.n_msgs * sizeof(StMsg), need * sizeof(StMsg)))) return rc;
  if (2 * need > S.tslots) return st_rebuild_table(c, S, next_pow2(std::max<uint64_t>(4 * need, 1024)));
  return TGI_OK;
}

// the live messages moved to the front in storage order once the tombstones outnumber them, and the table rebuilt
int st_compact(tgi_ctx* c, CrawlState& S) {
  const uint64_t n = S.n_msgs, live = n - S.n_dead;
  if (S.n_dead <= live) return TGI_OK;
  cudaStream_t st = S.stream;
  CK(S.flag.ensure(n * 4));
  CK(S.pos.ensure((n + 1) * 8));
  CK(S.sc.ensure(ST_SC_COUNT * 8));
  CK(S.spare.ensure(std::max<uint64_t>(live, 1) * sizeof(StMsg)));
  const StDev d = st_dev(S);
  st_live_flag_kernel<<<st_grid(c, n), ST_THREADS, 0, st>>>(d, n, ST_NONE, S.flag.as<uint32_t>());
  uint32_t launches = 0;
  int rc;
  if ((rc = launch_scan(c, st, S.tiles, S.flag.as<uint32_t>(), n, S.pos.as<uint64_t>(), S.sc.as<uint64_t>(), launches))) return rc;
  st_compact_kernel<<<st_grid(c, n), ST_THREADS, 0, st>>>(d, n, S.flag.as<uint32_t>(), S.pos.as<uint64_t>(), S.spare.as<StMsg>());
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(st));
  S.msgs.swap(S.spare);
  S.n_msgs = live;
  S.n_dead = 0;
  return st_rebuild_table(c, S, S.tslots);
}

// message rows of the host form, uploaded behind the existing ones and entered in the table
int st_append_msgs(tgi_ctx* c, CrawlState& S, const std::vector<StMsg>& m) {
  if (m.empty()) return TGI_OK;
  int rc;
  if ((rc = st_reserve(c, S, m.size()))) return rc;
  CK(cudaMemcpyAsync(S.msgs.as<StMsg>() + S.n_msgs, m.data(), m.size() * sizeof(StMsg), cudaMemcpyHostToDevice, S.stream));
  st_table_insert_kernel<<<st_grid(c, m.size()), ST_THREADS, 0, S.stream>>>(st_dev(S), S.n_msgs, S.n_msgs + m.size());
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(S.stream));
  S.n_msgs += m.size();
  return TGI_OK;
}

int st_upload_codes(tgi_ctx* c, CrawlState& S) {
  if (!S.codes_dirty) return TGI_OK;
  std::string blob;
  std::vector<uint32_t> off(1, 0);
  for (const std::string& s : S.codes) {
    blob += s;
    off.push_back((uint32_t)blob.size());
  }
  CK(S.code_blob.ensure(blob.size()));
  CK(S.code_off.ensure(off.size() * 4));
  CK(cudaMemsetAsync(S.code_blob.p, 0, blob.size() + PAD, S.stream));
  if (!blob.empty()) CK(cudaMemcpyAsync(S.code_blob.p, blob.data(), blob.size(), cudaMemcpyHostToDevice, S.stream));
  CK(cudaMemcpyAsync(S.code_off.p, off.data(), off.size() * 4, cudaMemcpyHostToDevice, S.stream));
  CK(cudaStreamSynchronize(S.stream));
  S.codes_dirty = false;
  return TGI_OK;
}

// a key buffer of a turn or a view lets go; the last holder returns it to the pool
void st_release(CrawlState& S, std::shared_ptr<DevBuf>& b) {
  if (b && b.use_count() == 1) S.turn_pool.push_back(std::move(b));
  b.reset();
}

void st_drop_view(CrawlState& S, uint32_t r) {
  const auto it = S.views.find(r);
  if (it == S.views.end()) return;
  st_release(S, it->second.keys);
  S.views.erase(it);
}

// the row's message generation moves on: its messages become tombstones, and a page that replaces the row (UpdatePage,
// an overwriting AddLayer) ends its owner view
int st_drop_messages(tgi_ctx* c, CrawlState& S, uint32_t r) {
  uint32_t cnt = 0;
  int rc;
  if ((rc = st_row_count(c, S, r, &cnt))) return rc;
  S.n_dead += cnt;
  S.gen[r]++;
  st_drop_view(S, r);
  return TGI_OK;
}

// r over the state's render buffers for ne entries: the zone, S.sc, row_base, msize and moff as the caller sized them,
// and the per-entry arrays in S.entries, S.e32 and S.e64, sized here
int st_render_bind(tgi_ctx* c, CrawlState& S, uint64_t ne, StRender& r) {
  CK(S.entries.ensure(ne * sizeof(StEntry)));
  CK(S.e32.ensure(4 * ne * 4));
  CK(S.e64.ensure(2 * (ne + 1) * 8));
  r.entries = S.entries.as<StEntry>();
  r.n_entries = ne;
  r.zone = c->cfgdev.zone;
  r.zone_n = c->cfgdev.zone_n;
  r.tz = c->cfgdev.tz;
  r.sc = S.sc.as<uint64_t>();
  r.row_base = S.row_base.as<uint64_t>();
  r.msize = S.msize.as<uint32_t>();
  r.moff = S.moff.as<uint64_t>();
  r.esize_lo = S.e32.as<uint32_t>();
  r.ebytes = r.esize_lo + ne;
  r.ecnt = r.ebytes + ne;
  r.esz = r.ecnt + ne;
  r.eoff = S.e64.as<uint64_t>();
  r.eslot = r.eoff + ne + 1;
  return TGI_OK;
}

// json.Marshal(page) of the P rows by the export's line passes: their cnt messages are sorted[0, cnt) (message indices
// grouped by row, each row's in list order; srows[] holds the row of each), and the caller has set row_base[row] for
// every listed row (its first grouped message; with cnt = 0, 0 for every row, as st_entry_size reads moff[row_base[row]]).
// The size pass is enqueued into r (no synchronise); once the host has S.sc in hs, st_page_json_emit writes the lines
// and brings them back.  tiled: the scans take their multi-launch form whatever their length, so the launch count does
// not depend on P.
int st_page_json_size(tgi_ctx* c, CrawlState& S, const uint32_t* rows, uint32_t P, const uint32_t* sorted, const uint32_t* srows,
                      uint64_t cnt, bool tiled, StRender& r, uint32_t& launches) {
  cudaStream_t st = S.stream;
  int rc;
  CK(S.msize.ensure(cnt * 4));
  CK(S.moff.ensure((cnt + 1) * 8));
  if ((rc = st_render_bind(c, S, P, r))) return rc;
  const StDev d = st_dev(S);
  std::vector<StEntry> E(P);
  for (uint32_t k = 0; k < P; k++) E[k] = StEntry{(long long)S.rows[rows[k]].depth, rows[k], 0};
  CK(cudaMemcpyAsync(S.entries.p, E.data(), P * sizeof(StEntry), cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(r.moff, 0, 8, st));
  CK(cudaMemsetAsync(S.sc.p, 0, ST_SC_COUNT * 8, st));
  if (cnt) {
    st_msg_size_kernel<<<st_grid(c, cnt), ST_THREADS, 0, st>>>(d, r, sorted, srows, cnt);
    launches++;
    if ((rc = launch_scan(c, st, S.tiles, r.msize, cnt, r.moff, r.sc + ST_SC_MBYTES, launches, tiled))) return rc;
  }
  st_line_size_kernel<<<sink_grid(c, P, ST_WARPS, 16), ST_WARPS * 32, 0, st>>>(d, r);
  launches++;
  if ((rc = launch_scan(c, st, S.tiles, r.esz, P, r.eoff, r.sc + ST_SC_BYTES, launches, tiled))) return rc;
  // the message slots: read only by st_msg_emit_kernel, which runs only when there are messages
  if (cnt && (rc = launch_scan(c, st, S.tiles, r.ecnt, P, r.eslot, r.sc + ST_SC_SLOTS, launches, tiled))) return rc;
  CK(cudaGetLastError());
  return TGI_OK;
}

// the pages' lines after their size pass (hs = the size pass's S.sc): *data holds json.Marshal(page) + '\n' of each,
// page k's line being [(*json_off)[k], (*json_off)[k+1]).  Dapr's UpdatePage has changed pageMap before json.Marshal
// fails (daprstate.go:1378-1387): a timestamp that does not render, or a page of 4 GiB or more, fails the call after the
// update.
int st_page_json_emit(tgi_ctx* c, CrawlState& S, StRender& r, const uint32_t* sorted, uint64_t cnt, const uint64_t* hs,
                      const char* who, const uint8_t** data, const uint64_t** json_off, float* ms, uint32_t& launches) {
  cudaStream_t st = S.stream;
  int rc;
  if (hs[ST_SC_ERR]) {
    rc = st_compact(c, S);
    if (!rc) set_err(c, "%s: the page's timestamp year is outside [0, 9999] (json.Marshal fails)", who);
    return rc ? rc : TGI_E_ARG;
  }
  if (hs[ST_SC_BIG]) {
    rc = st_compact(c, S);
    if (!rc) set_err(c, "%s: the page renders to 4 GiB or more", who);
    return rc ? rc : TGI_E_CAPACITY;
  }
  const uint64_t body = hs[ST_SC_BYTES], ne = r.n_entries;
  CK(S.out.ensure(body));
  CK(S.h_out.ensure(body));
  CK(S.h_json_off.ensure((ne + 1) * 8));
  r.out = S.out.as<uint8_t>();
  const StDev d = st_dev(S);
  CK(cudaEventRecord(S.t4, st));
  st_line_emit_kernel<<<sink_grid(c, ne, ST_WARPS, 16), ST_WARPS * 32, 0, st>>>(d, r);
  if (cnt) st_msg_emit_kernel<<<st_grid(c, cnt), ST_THREADS, 0, st>>>(d, r, sorted);
  launches += 1 + (cnt != 0);
  CK(cudaGetLastError());
  CK(cudaEventRecord(S.t5, st));
  CK(cudaMemcpyAsync(S.h_out.p, S.out.p, body, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(S.h_json_off.p, r.eoff, (ne + 1) * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  cudaEventElapsedTime(ms, S.t4, S.t5);
  *data = S.h_out.as<uint8_t>();
  *json_off = S.h_json_off.as<uint64_t>();
  return TGI_OK;
}

// The live messages of every row (set == nullptr) or of the rows set[0, ns) (ascending), grouped by row in storage order:
// their message indices in S.vals[at, at + live) and their rows in S.keys[at, at + live), live (<= bound) in ST_SC_LIVE.
// S.keys and S.vals are sized for at + 2 * bound here; a caller with pairs below `at` sizes them first, since a buffer
// that grows does not keep its contents.  tiled: the scans take their multi-launch form.  Nothing is waited for.
int st_group_rows(tgi_ctx* c, CrawlState& S, const uint32_t* set, uint32_t ns, uint64_t bound, uint64_t at, bool tiled,
                  uint32_t& launches) {
  const uint64_t nm = S.n_msgs, nr = S.rows.size();
  cudaStream_t st = S.stream;
  int rc;
  CK(S.flag.ensure(nm * 4));
  CK(S.pos.ensure((nm + 1) * 8));
  CK(S.keys.ensure((at + 2 * bound) * 4));
  CK(S.vals.ensure((at + 2 * bound) * 4));
  const RadixPlan plan(std::max<uint64_t>(nr, 1) - 1);  // by row
  uint32_t* flag = S.flag.as<uint32_t>();
  uint64_t* pos = S.pos.as<uint64_t>();
  StGroup g{flag, pos};
  g.keys[plan.out] = S.keys.as<uint32_t>() + at;
  g.keys[plan.out ^ 1] = S.keys.as<uint32_t>() + at + bound;
  g.vals[plan.out] = S.vals.as<uint32_t>() + at;
  g.vals[plan.out ^ 1] = S.vals.as<uint32_t>() + at + bound;
  const StDev d = st_dev(S);
  uint64_t* live = S.sc.as<uint64_t>() + ST_SC_LIVE;
  if (set) st_rows_flag_kernel<<<st_grid(c, nm), ST_THREADS, 0, st>>>(d, nm, set, ns, flag);
  else st_live_flag_kernel<<<st_grid(c, nm), ST_THREADS, 0, st>>>(d, nm, ST_NONE, flag);
  launches++;
  if ((rc = launch_scan(c, st, S.tiles, flag, nm, pos, live, launches, tiled))) return rc;
  st_render_pairs_kernel<<<st_grid(c, nm), ST_THREADS, 0, st>>>(d, nm, g);
  launches++;
  return radix_sort(c, st, S.tiles, g.keys, g.vals, live, bound, plan, S.counts, S.roff, S.sc.as<uint64_t>() + ST_SC_RADIX, tiled,
                    launches);
}

// the entries' bytes in S.out by the render's two passes, their offsets in S.e64 ([ne+1]); *body = their length,
// *size_ms = the size pass.  The emit is enqueued behind S.t2 and ends at S.t3, not waited for.
int st_emit_entries(tgi_ctx* c, CrawlState& S, const std::vector<StEntry>& E, bool lines, const char* who, uint64_t* body,
                    float* size_ms, uint32_t& launches) {
  const uint64_t ne = E.size(), nr = S.rows.size(), nm = S.n_msgs, live = nm - S.n_dead;
  cudaStream_t st = S.stream;
  int rc;
  CK(S.sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_sc.ensure(ST_SC_COUNT * 8));
  CK(S.row_base.ensure((nr + 1) * 8));
  CK(S.msize.ensure(live * 4));
  CK(S.moff.ensure((live + 1) * 8));
  StRender r{};
  if ((rc = st_render_bind(c, S, ne, r))) return rc;
  const StDev d = st_dev(S);
  CK(cudaMemcpyAsync(S.entries.p, E.data(), ne * sizeof(StEntry), cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(S.sc.p, 0, ST_SC_COUNT * 8, st));
  CK(cudaEventRecord(S.t0, st));
  if ((rc = st_group_rows(c, S, nullptr, 0, live, 0, false, launches))) return rc;
  const uint32_t* sorted = S.vals.as<uint32_t>();
  if ((rc = launch_scan(c, st, S.tiles, d.row_cnt, nr, r.row_base, r.sc + ST_SC_ROWS, launches))) return rc;
  st_msg_size_kernel<<<st_grid(c, live), ST_THREADS, 0, st>>>(d, r, sorted, S.keys.as<uint32_t>(), live);
  launches++;
  if ((rc = launch_scan(c, st, S.tiles, r.msize, live, r.moff, r.sc + ST_SC_MBYTES, launches))) return rc;
  (lines ? st_line_size_kernel : st_entry_size_kernel)<<<sink_grid(c, ne, ST_WARPS, 16), ST_WARPS * 32, 0, st>>>(d, r);
  launches++;
  if ((rc = launch_scan(c, st, S.tiles, r.esz, ne, r.eoff, r.sc + ST_SC_BYTES, launches))) return rc;
  if ((rc = launch_scan(c, st, S.tiles, r.ecnt, ne, r.eslot, r.sc + ST_SC_SLOTS, launches))) return rc;
  CK(cudaGetLastError());
  CK(cudaEventRecord(S.t1, st));
  CK(cudaMemcpyAsync(S.h_sc.p, S.sc.p, ST_SC_COUNT * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const uint64_t* h = S.h_sc.as<uint64_t>();
  if (h[ST_SC_LIVE] != live) { set_err(c, "%s: %llu live messages, expected %llu", who, (unsigned long long)h[ST_SC_LIVE], (unsigned long long)live); return TGI_E_CUDA; }
  if (h[ST_SC_ERR]) { set_err(c, "%s: a page timestamp's year is outside [0, 9999] (json.Marshal fails)", who); return TGI_E_ARG; }
  if (h[ST_SC_BIG]) { set_err(c, "%s: a page renders to 4 GiB or more", who); return TGI_E_CAPACITY; }
  *body = h[ST_SC_BYTES];
  const uint64_t slots = h[ST_SC_SLOTS];
  cudaEventElapsedTime(size_ms, S.t0, S.t1);
  CK(S.out.ensure(*body));
  r.out = S.out.as<uint8_t>();
  CK(cudaEventRecord(S.t2, st));
  (lines ? st_line_emit_kernel : st_entry_emit_kernel)<<<sink_grid(c, ne, ST_WARPS, 16), ST_WARPS * 32, 0, st>>>(d, r);
  if (slots) st_msg_emit_kernel<<<st_grid(c, slots), ST_THREADS, 0, st>>>(d, r, sorted);
  launches += 1 + (slots != 0);
  CK(cudaGetLastError());
  CK(cudaEventRecord(S.t3, st));
  return TGI_OK;
}

// The two passes of a writer with a thread per piece (a layer-map id, a SQL row) and block ST_THREADS: size writes the n
// pieces' sizes to sz, which the scan turns into off and their total in ST_SC_BYTES, read back with one synchronise.  A
// piece of 4 GiB or more refuses the call (noun names it) before anything is written; else *body is the output's
// length, and st_rows_emit sizes out for it, points *dst at it and enqueues emit.  Once the emit has finished,
// st_rows_ms is the device time of both passes.
template <class A>
int st_rows_size(tgi_ctx* c, CrawlState& S, void (*size)(StDev, A), const A& a, unsigned grid, const uint32_t* sz, uint64_t n,
                 uint64_t* off, const char* who, const char* noun, uint64_t* body, uint32_t& launches) {
  cudaStream_t st = S.stream;
  int rc;
  CK(cudaMemsetAsync(S.sc.p, 0, ST_SC_COUNT * 8, st));
  CK(cudaEventRecord(S.t0, st));
  size<<<grid, ST_THREADS, 0, st>>>(st_dev(S), a);
  launches++;
  if ((rc = launch_scan(c, st, S.tiles, sz, n, off, S.sc.as<uint64_t>() + ST_SC_BYTES, launches))) return rc;
  CK(cudaGetLastError());
  CK(cudaEventRecord(S.t1, st));
  CK(cudaMemcpyAsync(S.h_sc.p, S.sc.p, ST_SC_COUNT * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const uint64_t* hs = S.h_sc.as<uint64_t>();
  if (hs[ST_SC_BIG]) { set_err(c, "%s: %s renders to 4 GiB or more", who, noun); return TGI_E_CAPACITY; }
  *body = hs[ST_SC_BYTES];
  return TGI_OK;
}
template <class A>
int st_rows_emit(tgi_ctx* c, CrawlState& S, void (*emit)(StDev, A), A& a, uint8_t** dst, DevBuf& out, uint64_t body,
                 unsigned grid, uint32_t& launches) {
  cudaStream_t st = S.stream;
  CK(out.ensure(body));
  *dst = out.as<uint8_t>();
  CK(cudaEventRecord(S.t2, st));
  emit<<<grid, ST_THREADS, 0, st>>>(st_dev(S), a);
  launches++;
  CK(cudaGetLastError());
  CK(cudaEventRecord(S.t3, st));
  return TGI_OK;
}
float st_rows_ms(const CrawlState& S) {
  float size_ms = 0, emit_ms = 0;
  cudaEventElapsedTime(&size_ms, S.t0, S.t1);
  cudaEventElapsedTime(&emit_ms, S.t2, S.t3);
  return size_ms + emit_ms;
}

// the m UpdateMessage calls in S.upd, in order (rows valid, st_reserve(m) done): the batch table, one probe per distinct
// key, the new keys appended in first-occurrence order and entered in the table.  launches counts the kernels; tiled:
// the scan takes its multi-launch form whatever m; ms (optional) gets the kernels' device time.
int st_apply_updates(tgi_ctx* c, CrawlState& S, uint64_t m, uint32_t& launches, bool tiled = false, float* ms = nullptr) {
  cudaStream_t st = S.stream;
  int rc;
  const uint64_t bslots = next_pow2(std::max<uint64_t>(2 * m, 64));
  CK(S.bfirst.ensure(bslots * 4));
  CK(S.blast.ensure(bslots * 4));
  CK(S.slot_of.ensure(m * 4));
  CK(S.flag.ensure(m * 4));
  CK(S.pos.ensure((m + 1) * 8));
  CK(S.sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_sc.ensure(ST_SC_COUNT * 8));
  CK(cudaMemsetAsync(S.bfirst.p, 0xFF, bslots * 4, st));
  CK(cudaMemsetAsync(S.blast.p, 0, bslots * 4, st));
  StUpd w{};
  w.u = S.upd.as<tgi_state_update>();
  w.n = m;
  w.bfirst = S.bfirst.as<uint32_t>();
  w.blast = S.blast.as<uint32_t>();
  w.bmask = bslots - 1;
  w.slot_of = S.slot_of.as<uint32_t>();
  w.flag = S.flag.as<uint32_t>();
  w.pos = S.pos.as<uint64_t>();
  w.n_msgs = S.n_msgs;
  const StDev d = st_dev(S);
  if (ms) CK(cudaEventRecord(S.t4, st));
  st_upd_build_kernel<<<st_grid(c, m), ST_THREADS, 0, st>>>(w);
  st_upd_resolve_kernel<<<st_grid(c, m), ST_THREADS, 0, st>>>(d, w);
  launches += 2;
  if ((rc = launch_scan(c, st, S.tiles, w.flag, m, w.pos, S.sc.as<uint64_t>(), launches, tiled))) return rc;
  st_upd_append_kernel<<<st_grid(c, m), ST_THREADS, 0, st>>>(d, w);
  launches++;
  CK(cudaGetLastError());
  if (ms) CK(cudaEventRecord(S.t5, st));
  CK(cudaMemcpyAsync(S.h_sc.p, S.sc.p, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  float t = 0;
  if (ms) {
    cudaEventElapsedTime(&t, S.t4, S.t5);
    *ms += t;
    CK(cudaEventRecord(S.t4, st));
  }
  const uint64_t added = *S.h_sc.as<uint64_t>();
  if (added) st_table_insert_kernel<<<st_grid(c, added), ST_THREADS, 0, st>>>(d, S.n_msgs, S.n_msgs + added);
  launches += added != 0;
  CK(cudaGetLastError());
  if (ms) CK(cudaEventRecord(S.t5, st));
  CK(cudaStreamSynchronize(st));
  if (ms) {
    cudaEventElapsedTime(&t, S.t4, S.t5);
    *ms += t;
  }
  S.n_msgs += added;
  return TGI_OK;
}

std::string_view st_view(const CrawlState& S, const tgi_state_page& p, int f) {
  uint64_t o = p.str_off;
  for (int k = 0; k < f; k++) o += p.str_len[k];
  return std::string_view(S.blob.data() + o, p.str_len[f]);
}

// GetPage of n known rows into the pinned read buffers: the records and strings from the host mirror, and with `lists`
// the rows' message lists from the device.  st_group_rows groups the live messages of the distinct rows by row (storage
// order inside a row) and one gather writes them out;
// the rows' counts, scanned, place each row's list.  The launches follow the state's row count, not n; two
// synchronises: the lists' lengths, then the lists.
int st_read_rows(tgi_ctx* c, CrawlState& S, const uint32_t* rows, uint64_t n, bool lists, const char* who, tgi_state_read_t* out) {
  uint64_t sl = 0;
  for (uint64_t k = 0; k < n; k++) sl += page_str_bytes(S.rows[rows[k]]);
  CK(S.h_rrows.ensure(std::max<uint64_t>(n, 1) * 4));
  CK(S.h_rpages.ensure(std::max<uint64_t>(n, 1) * sizeof(tgi_state_page)));
  if (n) memcpy(S.h_rrows.p, rows, n * 4);
  CK(S.h_rstrs.ensure(std::max<uint64_t>(sl, 1)));
  tgi_state_page* pg = S.h_rpages.as<tgi_state_page>();
  uint8_t* hs = S.h_rstrs.as<uint8_t>();
  for (uint64_t k = 0, o = 0; k < n; k++) {
    pg[k] = S.rows[rows[k]];
    const uint64_t b = page_str_bytes(pg[k]);
    if (b) memcpy(hs + o, S.blob.data() + pg[k].str_off, b);
    pg[k].str_off = o;
    pg[k].n_msgs = 0;
    o += b;
  }
  out->n_pages = n;
  out->rows = S.h_rrows.as<uint32_t>();
  out->pages = pg;
  out->strs = hs;
  out->strs_len = sl;
  if (!lists) return TGI_OK;
  CK(S.h_rfirst.ensure(std::max<uint64_t>(n, 1) * 8));
  CK(S.h_rmsgs.ensure(sizeof(tgi_state_msg)));
  uint64_t* first = S.h_rfirst.as<uint64_t>();
  out->msg_first = first;
  out->msgs = S.h_rmsgs.as<tgi_state_msg>();
  std::vector<uint32_t> set(rows, rows + n);  // the distinct rows, ascending
  std::sort(set.begin(), set.end());
  set.erase(std::unique(set.begin(), set.end()), set.end());
  const uint32_t ns = (uint32_t)set.size();
  const uint64_t live = S.n_msgs - S.n_dead;
  if (!n || !live) {
    for (uint64_t k = 0; k < n; k++) first[k] = 0;
    return TGI_OK;
  }
  cudaStream_t st = S.stream;
  int rc;
  // S.rset: the set [ns] | its counts [ns] | their scan [ns+1]; h_rset stages the set and takes the scan back
  const size_t o_cnt = 4ull * ns, o_off = 8ull * ns, rbytes = o_off + 8ull * (ns + 1);
  CK(S.rset.ensure(rbytes));
  CK(S.h_rset.ensure(rbytes));
  CK(S.sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_sc.ensure(ST_SC_COUNT * 8));
  CK(S.spare.ensure(live * sizeof(tgi_state_msg)));
  uint8_t* dr = S.rset.as<uint8_t>();
  const uint32_t* d_set = (const uint32_t*)dr;
  uint32_t* d_cnt = (uint32_t*)(dr + o_cnt);
  uint64_t* d_off = (uint64_t*)(dr + o_off);
  uint64_t* sc = S.sc.as<uint64_t>();
  memcpy(S.h_rset.p, set.data(), 4ull * ns);
  CK(cudaMemcpyAsync(dr, S.h_rset.p, 4ull * ns, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(S.sc.p, 0, ST_SC_COUNT * 8, st));
  const StDev d = st_dev(S);
  uint32_t launches = 0;
  CK(cudaEventRecord(S.t0, st));
  if ((rc = st_group_rows(c, S, d_set, ns, live, 0, false, launches))) return rc;
  st_set_counts_kernel<<<st_grid(c, ns), ST_THREADS, 0, st>>>(d.row_cnt, d_set, ns, d_cnt);
  launches++;
  if ((rc = launch_scan(c, st, S.tiles, d_cnt, ns, d_off, sc + ST_SC_ROWS, launches, true))) return rc;
  st_gather_kernel<<<st_grid(c, live), ST_THREADS, 0, st>>>(d, S.vals.as<uint32_t>(), sc + ST_SC_LIVE, S.spare.as<tgi_state_msg>());
  launches++;
  CK(cudaGetLastError());
  CK(cudaEventRecord(S.t1, st));
  CK(cudaMemcpyAsync(S.h_sc.p, S.sc.p, ST_SC_COUNT * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(S.h_rset.as<uint8_t>() + o_off, d_off, 8ull * (ns + 1), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const uint64_t* off = (const uint64_t*)(S.h_rset.as<uint8_t>() + o_off);
  const uint64_t total = S.h_sc.as<uint64_t>()[ST_SC_LIVE];
  if (total != off[ns]) {
    set_err(c, "%s: %llu live messages flagged, the rows count %llu", who, (unsigned long long)total, (unsigned long long)off[ns]);
    return TGI_E_CUDA;
  }
  CK(S.h_rmsgs.ensure(std::max<uint64_t>(total, 1) * sizeof(tgi_state_msg)));
  if (total) CK(cudaMemcpyAsync(S.h_rmsgs.p, S.spare.p, total * sizeof(tgi_state_msg), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  cudaEventElapsedTime(&out->kernel_ms, S.t0, S.t1);
  for (uint64_t k = 0; k < n; k++) {
    const uint64_t j = std::lower_bound(set.begin(), set.end(), rows[k]) - set.begin();
    first[k] = off[j];
    pg[k].n_msgs = (uint32_t)(off[j + 1] - off[j]);
  }
  out->msgs = S.h_rmsgs.as<tgi_state_msg>();
  out->n_msgs = total;
  out->gpu_launches = launches;
  return TGI_OK;
}

}  // namespace

extern "C" {

int tgi_state_code(tgi_ctx* c, const char* s, uint32_t len, uint16_t* code) {
  if (!c || (len && !s) || !code) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  const std::string k(s ? s : "", len);
  const auto it = S.code_of.find(k);
  if (it != S.code_of.end()) {
    *code = it->second;
    return TGI_OK;
  }
  if (S.codes.size() >= 0xFFFF) { set_err(c, "tgi_state_code: 65535 codes registered"); return TGI_E_CAPACITY; }
  *code = (uint16_t)S.codes.size();
  S.code_of[k] = *code;
  S.codes.push_back(k);
  S.codes_dirty = true;
  return TGI_OK;
}

int tgi_state_set(tgi_ctx* c, const tgi_state_layer* layers, uint32_t n_layers, const tgi_state_page* pages, uint64_t n_pages,
                  const uint8_t* strs, uint64_t strs_len, const tgi_state_msg* msgs, uint64_t n_msgs, uint32_t* rows) {
  if (!c || (n_layers && !layers) || (n_pages && !pages) || (n_msgs && !msgs)) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  uint64_t in_layers = 0, owned = 0;
  for (uint32_t k = 0; k < n_layers; k++) in_layers += layers[k].n_pages;
  if (in_layers != n_pages) { set_err(c, "tgi_state_set: the layers hold %llu pages, not %llu", (unsigned long long)in_layers, (unsigned long long)n_pages); return TGI_E_ARG; }
  for (uint64_t i = 0; i < n_pages; i++) {
    if (!page_ok(c, pages[i], strs, strs_len, "tgi_state_set")) return TGI_E_ARG;
    owned += pages[i].n_msgs;
  }
  if (owned != n_msgs) { set_err(c, "tgi_state_set: the pages own %llu messages, not %llu", (unsigned long long)owned, (unsigned long long)n_msgs); return TGI_E_ARG; }
  if (n_msgs >= 0xFFFFFFFEull) { set_err(c, "tgi_state_set: %llu messages (at most 2^32 - 2)", (unsigned long long)n_msgs); return TGI_E_CAPACITY; }
  for (uint64_t j = 0; j < n_msgs; j++)
    if (msgs[j].page_id >= n_pages || msgs[j].status >= S.codes.size() || msgs[j].platform >= S.codes.size()) {
      set_err(c, "tgi_state_set: message %llu names an unknown page or code", (unsigned long long)j);
      return TGI_E_ARG;
    }
  // SetState: new maps, layer by layer; a later page with the same id replaces the row (and its messages).  The rows
  // are renumbered, so the open turns and the owner views go.
  for (auto& [h, T] : S.turns) st_release(S, T.keys);
  for (auto& [r, V] : S.views) st_release(S, V.keys);
  S.turns.clear();
  S.views.clear();
  S.n_pend = 0;  // the pending next-layer list names rows
  S.rows.clear();
  S.blob.clear();
  S.gen.clear();
  S.by_id.clear();
  S.urls.clear();
  S.layers.clear();
  S.deadends = 0;
  S.rows_synced = S.blob_synced = 0;
  S.n_msgs = S.n_dead = 0;
  std::vector<uint32_t> row_of(n_pages);
  std::vector<uint64_t> winner;  // the page whose messages a row keeps
  uint64_t i = 0;
  for (uint32_t k = 0; k < n_layers; k++) {
    std::vector<uint32_t>& L = S.layers[layers[k].depth];
    L.clear();
    for (uint64_t q = 0; q < layers[k].n_pages; q++, i++) {
      const auto it = S.by_id.find(in_field(pages[i], strs, TGI_PS_ID));
      const uint32_t r = it == S.by_id.end() ? (uint32_t)S.rows.size() : it->second;
      st_put_row(S, r, pages[i], strs);
      if (r == winner.size()) winner.push_back(i);
      else winner[r] = i;
      row_of[i] = r;
      L.push_back(r);
    }
  }
  std::vector<StMsg> m;
  std::vector<uint32_t> cnt(S.rows.size(), 0);
  uint64_t j = 0;
  for (i = 0; i < n_pages; i++) {
    const uint32_t r = row_of[i];
    for (uint32_t q = 0; q < pages[i].n_msgs; q++, j++) {
      if (winner[r] != i) continue;
      const tgi_state_msg& x = msgs[j];
      m.push_back(StMsg{(long long)x.chat_id, (long long)x.message_id, r, 0, row_of[x.page_id], x.status, x.platform});
      cnt[r]++;
    }
  }
  rc = st_sync_rows(c, S, std::vector<uint32_t>());
  if (rc) return rc;
  if (!cnt.empty()) CK(cudaMemcpyAsync(S.row_cnt.p, cnt.data(), cnt.size() * 4, cudaMemcpyHostToDevice, S.stream));
  if ((rc = st_rebuild_table(c, S, next_pow2(std::max<uint64_t>(4 * m.size(), 1024))))) return rc;
  if ((rc = st_append_msgs(c, S, m))) return rc;
  if (rows) memcpy(rows, row_of.data(), n_pages * 4);
  return TGI_OK;
}

int tgi_state_add_layer(tgi_ctx* c, const tgi_state_page* pages, uint64_t n, const uint8_t* strs, uint64_t strs_len,
                        int64_t max_pages, uint32_t* rows) {
  if (!c || (n && !pages)) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  if (!n) return TGI_OK;  // base.go:220-222: no layer is created
  for (uint64_t i = 0; i < n; i++) {
    if (!page_ok(c, pages[i], strs, strs_len, "tgi_state_add_layer")) return TGI_E_ARG;
    if (pages[i].n_msgs) { set_err(c, "tgi_state_add_layer: page %llu carries messages", (unsigned long long)i); return TGI_E_ARG; }
  }
  const bool reached = max_pages > 0 && (int64_t)S.rows.size() >= max_pages;
  int64_t replacements = (int64_t)S.deadends;
  std::vector<uint32_t>& L = S.layers[pages[0].depth];
  std::vector<uint32_t> dirty;
  std::unordered_map<std::string, int> gone;  // URLs of overwritten pages: still in existingURLs for this call
  for (uint64_t i = 0; i < n; i++) {
    if (rows) rows[i] = TGI_STATE_NO_PAGE;
    const std::string url = in_field(pages[i], strs, TGI_PS_URL);
    if (S.urls.count(url) || gone.count(url)) continue;
    if (reached) {
      if (replacements <= 0) continue;
      replacements--;
    }
    const auto it = S.by_id.find(in_field(pages[i], strs, TGI_PS_ID));
    uint32_t r = (uint32_t)S.rows.size();
    if (it != S.by_id.end()) {  // pageMap[id] = page: the old page and its messages go
      r = it->second;
      gone[st_field(S, S.rows[r], TGI_PS_URL)] = 1;
      if (std::find(dirty.begin(), dirty.end(), r) == dirty.end()) {  // the device count is read once per call
        if (r < S.rows_synced && (rc = st_drop_messages(c, S, r))) return rc;
        dirty.push_back(r);
      }
    }
    st_put_row(S, r, pages[i], strs);
    L.push_back(r);
    if (rows) rows[i] = r;
  }
  if ((rc = st_sync_rows(c, S, dirty))) return rc;
  return st_compact(c, S);
}

int tgi_state_update_page(tgi_ctx* c, const tgi_state_page* page, const uint8_t* strs, uint64_t strs_len,
                          const tgi_state_msg* msgs, uint32_t* row) {
  if (!c || !page || (page->n_msgs && !msgs)) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  if (!page_ok(c, *page, strs, strs_len, "tgi_state_update_page")) return TGI_E_ARG;
  for (uint32_t j = 0; j < page->n_msgs; j++)
    if ((msgs[j].page_id != TGI_STATE_NO_PAGE && msgs[j].page_id >= S.rows.size()) || msgs[j].status >= S.codes.size() ||
        msgs[j].platform >= S.codes.size()) {
      set_err(c, "tgi_state_update_page: message %u names an unknown row or code", j);
      return TGI_E_ARG;
    }
  if (S.n_msgs + page->n_msgs >= 0xFFFFFFFEull) { set_err(c, "tgi_state_update_page: more than 2^32 - 2 message rows"); return TGI_E_CAPACITY; }
  const auto it = S.by_id.find(in_field(*page, strs, TGI_PS_ID));
  uint32_t r = (uint32_t)S.rows.size();
  std::vector<uint32_t> dirty;
  if (it != S.by_id.end()) {
    r = it->second;
    if ((rc = st_drop_messages(c, S, r))) return rc;
    dirty.push_back(r);
  }
  st_put_row(S, r, *page, strs);
  // base.go:131-146: appended only to a layer of its depth that exists and does not hold it yet
  const auto lit = S.layers.find(page->depth);
  if (lit != S.layers.end() && std::find(lit->second.begin(), lit->second.end(), r) == lit->second.end()) lit->second.push_back(r);
  if ((rc = st_sync_rows(c, S, dirty))) return rc;
  std::vector<StMsg> m(page->n_msgs);
  for (uint32_t j = 0; j < page->n_msgs; j++)
    m[j] = StMsg{(long long)msgs[j].chat_id, (long long)msgs[j].message_id, r, S.gen[r],
                 msgs[j].page_id == TGI_STATE_NO_PAGE ? r : msgs[j].page_id, msgs[j].status, msgs[j].platform};
  const uint32_t cnt = page->n_msgs;
  CK(cudaMemcpyAsync(S.row_cnt.as<uint32_t>() + r, &cnt, 4, cudaMemcpyHostToDevice, S.stream));
  if ((rc = st_append_msgs(c, S, m))) return rc;
  CK(cudaStreamSynchronize(S.stream));
  if (row) *row = r;
  return st_compact(c, S);
}

int tgi_state_update_messages(tgi_ctx* c, const tgi_state_update* ups, uint64_t n, uint64_t* skipped) {
  if (!c || (n && !ups)) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  std::vector<tgi_state_update> u;
  u.reserve(n);
  uint64_t skip = 0;
  for (uint64_t j = 0; j < n; j++) {
    if (ups[j].row == TGI_STATE_NO_PAGE) {
      skip++;
      continue;
    }
    if (ups[j].row >= S.rows.size() || ups[j].status >= S.codes.size()) {
      set_err(c, "tgi_state_update_messages: update %llu names an unknown row or code", (unsigned long long)j);
      return TGI_E_ARG;
    }
    u.push_back(ups[j]);
  }
  if (skipped) *skipped = skip;
  const uint64_t m = u.size();
  if (!m) return TGI_OK;
  if ((rc = st_reserve(c, S, m))) return rc;
  CK(S.upd.ensure(m * sizeof(tgi_state_update)));
  CK(cudaMemcpyAsync(S.upd.p, u.data(), m * sizeof(tgi_state_update), cudaMemcpyHostToDevice, S.stream));
  uint32_t launches = 0;
  return st_apply_updates(c, S, m, launches);
}

int tgi_state_read_page(tgi_ctx* c, uint32_t row, tgi_state_msg* out, uint64_t cap, uint64_t* n) {
  if (!c || !n) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  if (row >= S.rows.size()) { set_err(c, "tgi_state_read_page: no row %u", row); return TGI_E_ARG; }
  uint32_t cnt = 0;
  if ((rc = st_row_count(c, S, row, &cnt))) return rc;
  *n = cnt;
  if (!out || cap < cnt || !cnt) return TGI_OK;
  tgi_state_read_t r{};
  if ((rc = st_read_rows(c, S, &row, 1, true, "tgi_state_read_page", &r))) return rc;
  memcpy(out, r.msgs + r.msg_first[0], r.pages[0].n_msgs * sizeof(tgi_state_msg));
  return TGI_OK;
}

int tgi_state_read_pages(tgi_ctx* c, const uint32_t* rows, uint64_t n, uint32_t flags, tgi_state_read_t* out) {
  if (!c || !out || (n && !rows)) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  memset(out, 0, sizeof *out);
  if (flags & ~TGI_READ_MESSAGES) { set_err(c, "tgi_state_read_pages: unknown flags 0x%x", flags); return TGI_E_ARG; }
  for (uint64_t k = 0; k < n; k++)
    if (rows[k] >= S.rows.size()) { set_err(c, "tgi_state_read_pages: no row %u (rows[%llu])", rows[k], (unsigned long long)k); return TGI_E_ARG; }
  return st_read_rows(c, S, rows, n, flags & TGI_READ_MESSAGES, "tgi_state_read_pages", out);
}

int tgi_state_read_layer(tgi_ctx* c, int64_t depth, int select, uint32_t flags, tgi_state_read_t* out) {
  if (!c || !out) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  memset(out, 0, sizeof *out);
  if (flags & ~TGI_READ_MESSAGES) { set_err(c, "tgi_state_read_layer: unknown flags 0x%x", flags); return TGI_E_ARG; }
  if (select < TGI_SELECT_NONE || select > TGI_SELECT_DAPR) { set_err(c, "tgi_state_read_layer: unknown selection %d", select); return TGI_E_ARG; }
  const auto it = S.layers.find(depth);  // base.go:329-332: no layer, no pages
  const uint32_t* rows = it == S.layers.end() ? nullptr : it->second.data();
  const uint64_t n = it == S.layers.end() ? 0 : it->second.size();
  if ((rc = st_read_rows(c, S, rows, n, flags & TGI_READ_MESSAGES, "tgi_state_read_layer", out))) return rc;
  if (select == TGI_SELECT_NONE) return TGI_OK;
  CK(S.h_rsel.ensure(std::max<uint64_t>(n, 1)));
  uint8_t* sel = S.h_rsel.as<uint8_t>();
  std::unordered_set<std::string_view> seen;  // processLayerInParallel's uniquePages
  uint64_t picked = 0;
  for (uint64_t k = 0; k < n; k++) {
    const tgi_state_page& p = S.rows[rows[k]];
    const std::string_view status = st_view(S, p, TGI_PS_STATUS);
    bool on = true;  // TGI_SELECT_STANDALONE: a new execution processes every page (standalone/runner.go:636-694)
    if (select == TGI_SELECT_STANDALONE_RESUME) {
      on = status != "fetched";  // the startIndex scan and the in-loop skip (:636-671, 672-694)
    } else if (select == TGI_SELECT_DAPR) {
      // dapr/standalone.go:459-463 records the URL before the status test at :477-497 (resuming: :420)
      on = seen.insert(st_view(S, p, TGI_PS_URL)).second && status != "fetched" && status != "error";
    }
    sel[k] = on;
    picked += on;
  }
  out->select = sel;
  out->n_selected = picked;
  return TGI_OK;
}

int tgi_state_layers(tgi_ctx* c, tgi_state_layers_t* out) {
  if (!c || !out) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  memset(out, 0, sizeof *out);
  const uint64_t nl = S.layers.size();
  CK(S.h_rdepth.ensure(std::max<uint64_t>(nl, 1) * 8));
  CK(S.h_rcount.ensure(std::max<uint64_t>(nl, 1) * 8));
  int64_t* depth = S.h_rdepth.as<int64_t>();
  uint64_t* count = S.h_rcount.as<uint64_t>();
  int64_t max_depth = -1;  // base.go:450-455: only a depth above -1 counts
  uint64_t k = 0, incomplete = 0;
  for (const auto& [dp, L] : S.layers) {
    depth[k] = dp;
    count[k++] = L.size();
    max_depth = std::max<int64_t>(max_depth, dp);
    for (uint32_t r : L) incomplete += st_view(S, S.rows[r], TGI_PS_STATUS) != "fetched";  // base.go:485-495
  }
  out->n_layers = nl;
  out->depth = depth;
  out->n_pages = count;
  out->max_depth = max_depth;
  out->has_max_depth = max_depth != -1;
  out->n_incomplete = incomplete;
  return TGI_OK;
}

// json.Marshal(GetState()): the layers' bytes on the device (two passes), the frame and the spliced values on the host
int tgi_state_render(tgi_ctx* c, const uint8_t* metadata, uint64_t metadata_len, const uint8_t* last_updated,
                     uint64_t last_updated_len, tgi_state_json_t* out) {
  if (!c || !out || (metadata_len && !metadata) || (last_updated_len && !last_updated)) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  if ((rc = st_upload_codes(c, S))) return rc;
  memset(out, 0, sizeof *out);
  std::vector<StEntry> E;
  for (const auto& [depth, L] : S.layers) {
    const uint32_t fl = E.empty() ? (uint32_t)ST_E_FIRST_LAYER : 0u;
    if (L.empty()) E.push_back(StEntry{(long long)depth, ST_NONE, ST_E_FIRST | ST_E_LAST | fl});
    for (size_t k = 0; k < L.size(); k++)
      E.push_back(StEntry{(long long)depth, L[k], (k == 0 ? ST_E_FIRST | fl : 0u) | (k + 1 == L.size() ? (uint32_t)ST_E_LAST : 0u)});
  }
  static const char kHead[] = "{\"layers\":[", kMeta[] = "],\"metadata\":", kLast[] = ",\"lastUpdated\":";
  cudaStream_t st = S.stream;
  uint32_t launches = 0;
  uint64_t body = 0;
  // the zone table must not change under the kernels that read it (tgi_set_zone swaps it under cfg_mu)
  std::lock_guard<std::mutex> zg(c->cfg_mu);
  if (!E.empty()) {
    float size_ms = 0, emit_ms = 0;
    if ((rc = st_emit_entries(c, S, E, false, "tgi_state_render", &body, &size_ms, launches))) return rc;
    CK(S.h_out.ensure(sizeof kHead + body + sizeof kMeta + metadata_len + sizeof kLast + last_updated_len + 2));
    CK(cudaMemcpyAsync(S.h_out.as<uint8_t>() + sizeof kHead - 1, S.out.p, body, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    cudaEventElapsedTime(&emit_ms, S.t2, S.t3);
    out->kernel_ms = size_ms + emit_ms;
  } else {
    CK(S.h_out.ensure(sizeof kHead + sizeof kMeta + metadata_len + sizeof kLast + last_updated_len + 2));
  }
  uint8_t* o = S.h_out.as<uint8_t>();
  uint64_t k = 0;
  memcpy(o, kHead, sizeof kHead - 1);
  k = sizeof kHead - 1 + body;
  memcpy(o + k, kMeta, sizeof kMeta - 1);
  k += sizeof kMeta - 1;
  if (metadata_len) memcpy(o + k, metadata, metadata_len);
  k += metadata_len;
  memcpy(o + k, kLast, sizeof kLast - 1);
  k += sizeof kLast - 1;
  if (last_updated_len) memcpy(o + k, last_updated, last_updated_len);
  k += last_updated_len;
  o[k++] = '}';
  out->data = o;
  out->len = k;
  out->gpu_launches = launches;
  return TGI_OK;
}

// Dapr's AddLayer after the caller's urlCache test (daprstate.go:625-780): pageMap[id] = page, the row appended to the
// layer `depth`; the URL map and the deadend count stay right for later tgi_state_add_layer calls
int tgi_state_add_pages(tgi_ctx* c, int64_t depth, const tgi_state_page* pages, uint64_t n, const uint8_t* strs,
                        uint64_t strs_len, uint32_t* rows) {
  if (!c || (n && !pages)) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  if (!n) return TGI_OK;  // daprstate.go:658-662: every page was a duplicate, no layer is created
  for (uint64_t i = 0; i < n; i++) {
    if (!page_ok(c, pages[i], strs, strs_len, "tgi_state_add_pages")) return TGI_E_ARG;
    if (pages[i].n_msgs) { set_err(c, "tgi_state_add_pages: page %llu carries messages", (unsigned long long)i); return TGI_E_ARG; }
  }
  std::vector<uint32_t>& L = S.layers[depth];
  std::vector<uint32_t> dirty;
  for (uint64_t i = 0; i < n; i++) {
    const auto it = S.by_id.find(in_field(pages[i], strs, TGI_PS_ID));
    uint32_t r = (uint32_t)S.rows.size();
    if (it != S.by_id.end()) {  // the old page and its messages go
      r = it->second;
      if (std::find(dirty.begin(), dirty.end(), r) == dirty.end()) {
        if (r < S.rows_synced && (rc = st_drop_messages(c, S, r))) return rc;
        dirty.push_back(r);
      }
    }
    st_put_row(S, r, pages[i], strs);
    L.push_back(r);
    if (rows) rows[i] = r;
  }
  if ((rc = st_sync_rows(c, S, dirty))) return rc;
  return st_compact(c, S);
}

// json.Marshal(map[int][]string): the keys' order and the layers' openings on the host, every id sized and written by
// one thread on the device
int tgi_state_layer_map(tgi_ctx* c, tgi_state_json_t* out) {
  if (!c || !out) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  memset(out, 0, sizeof *out);
  std::vector<std::pair<std::string, const std::vector<uint32_t>*>> K;
  for (const auto& [depth, L] : S.layers) K.emplace_back(std::to_string(depth), &L);
  std::sort(K.begin(), K.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
  std::string keys;
  std::vector<StLmEntry> E;
  for (const auto& [key, L] : K) {
    const uint32_t pre = (uint32_t)keys.size();
    keys += (pre ? ",\"" : "\"") + key + "\":[";
    const uint32_t pl = (uint32_t)keys.size() - pre;
    if (L->empty()) E.push_back(StLmEntry{ST_NONE, pre, pl, 1});
    for (size_t k = 0; k < L->size(); k++) E.push_back(StLmEntry{(*L)[k], pre, k ? 0u : pl, k + 1 == L->size() ? 1u : 0u});
  }
  const uint64_t ne = E.size();
  cudaStream_t st = S.stream;
  uint32_t launches = 0;
  uint64_t body = 0;
  if (ne) {
    CK(S.entries.ensure(ne * sizeof(StLmEntry)));
    CK(S.lm_keys.ensure(keys.size()));
    CK(S.e32.ensure(ne * 4));
    CK(S.e64.ensure((ne + 1) * 8));
    CK(S.sc.ensure(ST_SC_COUNT * 8));
    CK(S.h_sc.ensure(ST_SC_COUNT * 8));
    StLm L{};
    L.entries = S.entries.as<StLmEntry>();
    L.n = ne;
    L.keys = S.lm_keys.as<uint8_t>();
    L.size = S.e32.as<uint32_t>();
    L.off = S.e64.as<uint64_t>();
    L.sc = S.sc.as<uint64_t>();
    CK(cudaMemcpyAsync(S.entries.p, E.data(), ne * sizeof(StLmEntry), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(S.lm_keys.p, keys.data(), keys.size(), cudaMemcpyHostToDevice, st));
    const unsigned grid = st_grid(c, ne);
    if ((rc = st_rows_size(c, S, st_lm_size_kernel, L, grid, L.size, ne, L.off, "tgi_state_layer_map", "an id", &body, launches)))
      return rc;
    CK(S.h_out.ensure(body + 2));
    if ((rc = st_rows_emit(c, S, st_lm_emit_kernel, L, &L.out, S.out, body, grid, launches))) return rc;
    CK(cudaMemcpyAsync(S.h_out.as<uint8_t>() + 1, S.out.p, body, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    out->kernel_ms = st_rows_ms(S);
  } else {
    CK(S.h_out.ensure(2));
  }
  uint8_t* o = S.h_out.as<uint8_t>();
  o[0] = '{';
  o[body + 1] = '}';
  out->data = o;
  out->len = body + 2;
  out->gpu_launches = launches;
  return TGI_OK;
}

// the pages as JSONL lines by the render's passes (st_entry in line mode); Dapr mode cuts them into chunks at the
// line ends on the host and base64-encodes every chunk with the combiner's encoder, each into its own 16-byte aligned
// range of the output
int tgi_state_export(tgi_ctx* c, int mode, uint64_t chunk_bytes, tgi_state_export_t* out) {
  if (!c || !out || (mode != TGI_STATE_EXPORT_DAPR && mode != TGI_STATE_EXPORT_LOCAL)) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  if ((rc = st_upload_codes(c, S))) return rc;
  memset(out, 0, sizeof *out);
  std::vector<StEntry> E;
  if (mode == TGI_STATE_EXPORT_DAPR) {
    for (const auto& [depth, L] : S.layers)
      for (uint32_t r : L) E.push_back(StEntry{(long long)depth, r, 0});
    if (E.empty()) { set_err(c, "tgi_state_export: no pages found to export"); return TGI_E_NOPAGES; }
  } else {
    for (uint32_t r = 0; r < (uint32_t)S.rows.size(); r++) E.push_back(StEntry{S.rows[r].depth, r, 0});
  }
  const uint64_t ne = E.size();
  cudaStream_t st = S.stream;
  uint32_t launches = 0;
  uint64_t body = 0;
  float size_ms = 0, emit_ms = 0, enc_ms = 0;
  std::lock_guard<std::mutex> zg(c->cfg_mu);  // the zone table, as in tgi_state_render
  if (ne && (rc = st_emit_entries(c, S, E, true, "tgi_state_export", &body, &size_ms, launches))) return rc;
  // chunk k's raw bytes are [start[k], start[k+1]) of S.out
  std::vector<uint64_t> start(1, 0);
  if (mode == TGI_STATE_EXPORT_DAPR) {
    std::vector<uint64_t> eoff(ne + 1);
    CK(cudaMemcpyAsync(eoff.data(), S.e64.p, (ne + 1) * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (uint64_t s = 0; s < body;) {  // the first line end at or past s + chunk_bytes (every line is longer than 0)
      const uint64_t want = chunk_bytes > body - s ? body + 1 : std::max<uint64_t>(s + chunk_bytes, s + 1);
      const auto it = std::lower_bound(eoff.begin() + 1, eoff.end(), want);
      s = it == eoff.end() ? body : *it;
      start.push_back(s);
    }
  } else {
    start.push_back(body);
  }
  const uint64_t nc = start.size() - 1;
  CK(S.h_chunks.ensure(3 * nc * 8 + 8));
  uint64_t* off = S.h_chunks.as<uint64_t>();
  uint64_t *len = off + nc, *raw = len + nc, total = 0;
  const bool enc = mode == TGI_STATE_EXPORT_DAPR;
  for (uint64_t k = 0; k < nc; k++) {
    raw[k] = start[k + 1] - start[k];
    len[k] = enc ? (raw[k] + 2) / 3 * 4 : raw[k];
    off[k] = total;
    total = enc ? (total + len[k] + 15) & ~15ull : total + len[k];
  }
  CK(S.h_out.ensure(total));
  if (enc) {
    CK(S.b64.ensure(total));
    CbPlan P;
    for (uint64_t k = 0; k < nc; k++)
      P.add(S.b64.as<uint8_t>() + off[k], true, {CbSeg{0, raw[k], S.out.as<uint8_t>() + start[k]}});
    const bool tables = P.t.size() > (size_t)CB_INLINE || P.s.size() > (size_t)CB_INLINE;
    if (tables) {
      CK(S.cb_tasks.ensure(P.t.size() * sizeof(CbTask)));
      CK(S.cb_segs.ensure(P.s.size() * sizeof(CbSeg)));
      CK(cudaMemcpyAsync(S.cb_tasks.p, P.t.data(), P.t.size() * sizeof(CbTask), cudaMemcpyHostToDevice, st));
      CK(cudaMemcpyAsync(S.cb_segs.p, P.s.data(), P.s.size() * sizeof(CbSeg), cudaMemcpyHostToDevice, st));
    }
    CK(cudaEventRecord(S.t4, st));
    if ((rc = cb_launch(c, st, P, S.cb_tasks.as<CbTask>(), S.cb_segs.as<CbSeg>(), nullptr, launches))) return rc;
    CK(cudaEventRecord(S.t5, st));
    if (total) CK(cudaMemcpyAsync(S.h_out.p, S.b64.p, total, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));  // also keeps P's inline tasks alive until the launch has read them
    cudaEventElapsedTime(&enc_ms, S.t4, S.t5);
  } else if (total) {
    CK(cudaMemcpyAsync(S.h_out.p, S.out.p, total, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  if (ne) cudaEventElapsedTime(&emit_ms, S.t2, S.t3);
  out->data = S.h_out.as<uint8_t>();
  out->off = off;
  out->len = len;
  out->raw_len = raw;
  out->n_chunks = nc;
  out->n_pages = ne;
  out->kernel_ms = size_ms + emit_ms + enc_ms;
  out->gpu_launches = launches;
  return TGI_OK;
}

}  // extern "C"

// ---- page turns over P pages (state.cuh): tgi_state_pages_begin / _end / _close, and the one-page calls as P = 1 ------
namespace {

// the rows of a turn call: at least one, each known, none listed twice
int st_check_rows(tgi_ctx* c, const CrawlState& S, const uint32_t* rows, uint32_t P, const char* who) {
  if (!P) { set_err(c, "%s: no pages", who); return TGI_E_ARG; }
  std::unordered_set<uint32_t> seen;
  for (uint32_t k = 0; k < P; k++) {
    if (rows[k] >= S.rows.size()) { set_err(c, "%s: no row %u", who, rows[k]); return TGI_E_ARG; }
    if (!seen.insert(rows[k]).second) { set_err(c, "%s: row %u is listed twice", who, rows[k]); return TGI_E_ARG; }
  }
  return TGI_OK;
}

// a page whose fields replace row r's: strings inside strs, no messages (`list` says where the list comes from), the
// row's id
bool st_check_page(tgi_ctx* c, const CrawlState& S, uint32_t r, const tgi_state_page& p, const uint8_t* strs,
                   uint64_t strs_len, const char* who, const char* list) {
  if (!page_ok(c, p, strs, strs_len, who)) return false;
  if (p.n_msgs) { set_err(c, "%s: the page carries messages (%s)", who, list); return false; }
  if (in_field(p, strs, TGI_PS_ID) != st_field(S, S.rows[r], TGI_PS_ID)) { set_err(c, "%s: the page's id is not row %u's", who, r); return false; }
  return true;
}

// UpdatePage's layer rule for every row of the call (base.go:131-146): the row joins the layer of its depth if that
// layer exists and does not hold it.  The rows of one depth are marked in a byte per row and the layer is read once,
// so a call costs one pass over each layer it touches, whatever P, and allocates nothing once the marks have grown.
void st_join_layers(CrawlState& S, const uint32_t* rows, uint32_t P) {
  if (P == 1) {  // one row: the search stops where it finds the row
    const auto lit = S.layers.find(S.rows[rows[0]].depth);
    if (lit != S.layers.end() && std::find(lit->second.begin(), lit->second.end(), rows[0]) == lit->second.end())
      lit->second.push_back(rows[0]);
    return;
  }
  std::vector<uint8_t>& mark = S.row_mark;  // all 0 between calls
  if (mark.size() < S.rows.size()) mark.resize(S.rows.size(), 0);
  std::vector<std::pair<int64_t, uint32_t>> by_depth(P);
  for (uint32_t k = 0; k < P; k++) by_depth[k] = {S.rows[rows[k]].depth, k};
  std::sort(by_depth.begin(), by_depth.end());
  for (size_t i = 0; i < by_depth.size();) {
    size_t j = i;
    while (j < by_depth.size() && by_depth[j].first == by_depth[i].first) j++;
    const auto lit = S.layers.find(by_depth[i].first);
    if (lit != S.layers.end()) {
      std::vector<uint32_t>& L = lit->second;
      for (size_t q = i; q < j; q++) mark[rows[by_depth[q].second]] = 1;
      for (uint32_t r : L) mark[r] = 0;  // held already
      for (size_t q = i; q < j; q++) {   // in call order, as P UpdatePage calls append them
        const uint32_t r = rows[by_depth[q].second];
        if (mark[r]) L.push_back(r);
        mark[r] = 0;
      }
    }
    i = j;
  }
}

std::shared_ptr<DevBuf> st_take_keys(CrawlState& S) {
  if (S.turn_pool.empty()) return std::make_shared<DevBuf>();
  std::shared_ptr<DevBuf> b = std::move(S.turn_pool.back());
  S.turn_pool.pop_back();
  return b;
}

size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

// the pinned staging of a turn call's page arrays, `bytes` of it.  Its uploads are asynchronous and a call may return
// before they have run (a close without TGI_TURN_PAGE_JSON and without out), so the buffer is reused, or regrown, only
// once the last upload from it has finished; st_seg_upload records that upload.
int st_seg_host(tgi_ctx* c, CrawlState& S, size_t bytes, uint8_t** h) {
  CK(cudaEventSynchronize(S.ev_seg));
  CK(S.h_seg.ensure(bytes));
  *h = S.h_seg.as<uint8_t>();
  return TGI_OK;
}
int st_seg_upload(tgi_ctx* c, CrawlState& S, size_t off, size_t bytes) {
  CK(cudaMemcpyAsync(S.seg.as<uint8_t>() + off, S.h_seg.as<uint8_t>() + off, bytes, cudaMemcpyHostToDevice, S.stream));
  CK(cudaEventRecord(S.ev_seg, S.stream));
  return TGI_OK;
}

// addNewMessages + resampleMarker + UpdatePage for P pages (crawl/runner.go:1132-1147), touching only the pages' own
// messages: a thread per fetched key probes its page's list in the resident table, one scan lays the new lists out in
// (page, fetch) order, and each page's segment is appended as its row's next generation.  Three synchronises whatever
// P: the new lists' lengths (and the old ones', for the tombstone count), the row strings' upload, and the work list;
// with TGI_TURN_PAGE_JSON the pages' sizes come back with the work list and one more synchronise brings their lines.
int st_pages_begin(tgi_ctx* c, CrawlState& S, const uint32_t* rows, uint32_t P, const tgi_state_page* pages, const uint8_t* strs,
                   uint64_t strs_len, const int64_t* fetched, uint64_t n, const uint64_t* foff, uint32_t flags, const char* who,
                   tgi_state_pages_t* out) {
  int rc;
  if ((rc = st_init(c, S))) return rc;
  memset(out, 0, sizeof *out);
  if (flags & ~TGI_TURN_PAGE_JSON) { set_err(c, "%s: unknown flags 0x%x", who, flags); return TGI_E_ARG; }
  if ((rc = st_check_rows(c, S, rows, P, who))) return rc;
  if (foff[0] != 0 || foff[P] != n) { set_err(c, "%s: fetched_off runs from %llu to %llu, not 0 to n = %llu", who, (unsigned long long)foff[0], (unsigned long long)foff[P], (unsigned long long)n); return TGI_E_ARG; }
  for (uint32_t k = 0; k < P; k++)
    if (foff[k + 1] < foff[k]) { set_err(c, "%s: fetched_off decreases at page %u", who, k); return TGI_E_ARG; }
  if (pages)
    for (uint32_t k = 0; k < P; k++)
      if (!st_check_page(c, S, rows[k], pages[k], strs, strs_len, who, "its list comes from the fetch")) return TGI_E_ARG;
  if ((rc = st_upload_codes(c, S))) return rc;
  if ((rc = st_reserve(c, S, n))) return rc;
  cudaStream_t st = S.stream;
  const bool json = flags & TGI_TURN_PAGE_JSON, tiled = P > 1;
  std::shared_ptr<DevBuf> keys = st_take_keys(S);
  const uint64_t bslots = next_pow2(std::max<uint64_t>(2 * n, 64));
  // S.seg: foff [P+1] | woff [P+1] | prow [P] | old [P] | row puts [P]
  const size_t o_woff = (P + 1) * 8ull, o_prow = 2 * o_woff, o_old = o_prow + 4ull * P, o_put = align16(o_old + 4ull * P);
  const size_t seg_bytes = o_put + P * sizeof(StRowPut);
  CK(keys->ensure(n * 18));
  CK(S.turn_in.ensure(n * 16));
  CK(S.seg.ensure(seg_bytes));
  uint8_t* hseg;
  if ((rc = st_seg_host(c, S, seg_bytes, &hseg))) return rc;
  CK(S.pg.ensure(n * 4));
  CK(S.bfirst.ensure(bslots * 4));
  CK(S.flag.ensure(n * 4));
  CK(S.pos.ensure((n + 1) * 8));
  CK(S.slot_of.ensure(n * 4));
  CK(S.vals.ensure(n * 4));
  CK(S.keys.ensure(n * 4));
  CK(S.row_base.ensure((S.rows.size() + 1) * 8));
  CK(S.sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_work.ensure(n * 4));
  CK(S.h_woff.ensure((P + 1) * 8));
  CK(S.h_old.ensure(P * 4));
  uint8_t* dseg = S.seg.as<uint8_t>();
  memcpy(hseg, foff, (P + 1) * 8);
  memcpy(hseg + o_prow, rows, P * 4);
  StTurn t{};
  t.fetched = S.turn_in.as<long long>();
  t.n = n;
  t.foff = (const uint64_t*)dseg;
  t.prow = (const uint32_t*)(dseg + o_prow);
  t.P = P;
  t.pg = S.pg.as<uint32_t>();
  t.bfirst = S.bfirst.as<uint32_t>();
  t.bmask = bslots - 1;
  t.flag = S.flag.as<uint32_t>();
  t.pos = S.pos.as<uint64_t>();
  t.woff = (uint64_t*)(dseg + o_woff);
  t.n_msgs = S.n_msgs;
  t.keys = keys->as<long long>();
  t.work = S.slot_of.as<uint32_t>();
  t.sorted = S.vals.as<uint32_t>();
  t.rows = S.keys.as<uint32_t>();
  uint32_t* d_old = (uint32_t*)(dseg + o_old);
  uint32_t launches = 0;
  // 1. which fetched keys their pages' lists lack, every page's segment of the new lists, and the old lists' lengths
  CK(cudaEventRecord(S.t0, st));
  if ((rc = st_seg_upload(c, S, 0, o_old))) return rc;
  if (n) {
    CK(cudaMemcpyAsync(S.turn_in.p, fetched, n * 16, cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(S.bfirst.p, 0xFF, bslots * 4, st));
    st_turn_probe_kernel<<<st_grid(c, n), ST_THREADS, 0, st>>>(st_dev(S), t);
    launches++;
    if ((rc = launch_scan(c, st, S.tiles, t.flag, n, t.pos, S.sc.as<uint64_t>(), launches, tiled))) return rc;
  }
  st_turn_meta_kernel<<<st_grid(c, P + 1), ST_THREADS, 0, st>>>(S.row_cnt.as<uint32_t>(), t.prow, P, t.foff, n ? t.pos : nullptr,
                                                                 t.woff, d_old);
  launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(S.h_woff.p, t.woff, (P + 1) * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(S.h_old.p, d_old, P * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaEventRecord(S.t1, st));
  CK(cudaStreamSynchronize(st));
  const uint64_t* wo = S.h_woff.as<uint64_t>();
  const uint32_t* old = S.h_old.as<uint32_t>();
  const uint64_t n_new = wo[P];
  // 2. UpdatePage(*owner) of every page: the old lists become tombstones; each row takes its page's fields and joins the
  // layer of its depth if that layer exists and does not hold it (base.go:131-146).  Each new list is its row's owner
  // view, a slice of this call's key buffer, its statuses "resample" (0) until the end's hits.
  for (uint32_t k = 0; k < P; k++) {
    S.n_dead += old[k];
    S.gen[rows[k]]++;
    if (pages) st_put_row(S, rows[k], pages[k], strs);
  }
  st_join_layers(S, rows, P);
  rc = st_sync_rows(c, S, std::vector<uint32_t>());  // the new strings
  if (rc) return rc;
  StRowPut* put = (StRowPut*)(hseg + o_put);
  for (uint32_t k = 0; k < P; k++) {
    const uint32_t r = rows[k];
    put[k] = StRowPut{S.rows[r], r, S.gen[r], (uint32_t)(wo[k + 1] - wo[k]), 1u, json ? wo[k] : ST_NO_BASE};
    st_drop_view(S, r);
    S.views[r] = CrawlState::View{wo[k], wo[k + 1] - wo[k], n_new, keys};
  }
  if ((rc = st_seg_upload(c, S, o_put, P * sizeof(StRowPut)))) return rc;
  if (n_new) CK(cudaMemsetAsync(keys->as<uint8_t>() + 16 * n_new, 0, 2 * n_new, st));
  const StDev d = st_dev(S);
  CK(cudaEventRecord(S.t2, st));
  st_rows_put_kernel<<<st_grid(c, P), ST_THREADS, 0, st>>>(S.pages.as<tgi_state_page>(), d.row_gen, d.row_cnt,
                                                           (const StRowPut*)(dseg + o_put), P, S.row_base.as<uint64_t>());
  launches++;
  if (n_new) {
    st_turn_append_kernel<<<st_grid(c, n), ST_THREADS, 0, st>>>(d, t);
    st_table_insert_kernel<<<st_grid(c, n_new), ST_THREADS, 0, st>>>(d, S.n_msgs, S.n_msgs + n_new);
    launches += 2;
  }
  S.n_msgs += n_new;
  // 3. json.Marshal(page) of every page by the export's line passes over the rows, their new lists being the fresh
  // segments in the call's order
  StRender r{};
  uint64_t* hs = S.h_sc.as<uint64_t>();
  std::unique_lock<std::mutex> zg(c->cfg_mu, std::defer_lock);  // the zone table, as in tgi_state_render
  if (json) {
    zg.lock();
    if ((rc = st_page_json_size(c, S, rows, P, t.sorted, t.rows, n_new, tiled, r, launches))) return rc;
    CK(cudaMemcpyAsync(hs, S.sc.p, ST_SC_COUNT * 8, cudaMemcpyDeviceToHost, st));
  }
  CK(cudaGetLastError());
  CK(cudaEventRecord(S.t3, st));
  if (n_new) CK(cudaMemcpyAsync(S.h_work.p, t.work, n_new * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  float ms0 = 0, ms1 = 0, ms2 = 0;
  cudaEventElapsedTime(&ms0, S.t0, S.t1);
  cudaEventElapsedTime(&ms1, S.t2, S.t3);
  // a page that does not marshal: the new lists and their views stay, no turn opens, as the reference returns before
  // its loop
  if (json && (rc = st_page_json_emit(c, S, r, t.sorted, n_new, hs, who, &out->page_json, &out->json_off, &ms2, launches)))
    return rc;
  if ((rc = st_compact(c, S))) return rc;
  const uint32_t h = S.next_turn++;
  if (!S.next_turn) S.next_turn = 1;
  CrawlState::Turn& T = S.turns[h];
  T.rows.assign(rows, rows + P);
  T.off.assign(wo, wo + P + 1);
  T.keys = std::move(keys);
  out->turn = h;
  out->n_pages = P;
  out->n_work = n_new;
  out->work = S.h_work.as<uint32_t>();
  out->work_off = wo;
  out->kernel_ms = ms0 + ms1 + ms2;
  out->gpu_launches = launches;
  return TGI_OK;
}

// the loop's first n_done[k] UpdateMessage calls of every page k of a turn (crawl/runner.go:1161-1211), in page order,
// as one tgi_state_update_messages batch built on the device from the turn's keys and the statuses; then the owner
// views' hits, a segment per page.  one: tgi_state_page_end (a one-page turn, a result of exactly its records).  Lock
// order: the slot, then the state; no other entry point holds both.  The slot's lock is held until the kernels that
// read its status array have finished.
int st_pages_end(tgi_ctx* c, uint32_t turn, int slot, uint64_t first, const uint8_t* status, const uint64_t* n_done, bool one,
                 uint64_t* appended, tgi_state_end_t* out) {
  const char* const who = one ? "tgi_state_page_end" : "tgi_state_pages_end";
  if (slot >= TGI_SLOTS) { set_err(c, "%s: bad slot %d", who, slot); return TGI_E_ARG; }
  Slot* s = slot >= 0 ? &c->slots[slot] : nullptr;
  std::unique_lock<std::mutex> sl;
  if (s) {
    sl = std::unique_lock<std::mutex>(s->mu);
    if (in_flight(*s)) { set_err(c, "%s: slot %d is in flight", who, slot); return TGI_E_STATE; }
    if (!s->busy || s->last.kind == REC_NONE) { set_err(c, "%s: slot %d holds no result (released or none)", who, slot); return TGI_E_ARG; }
    if (s->last.kind != REC_TG || !s->last.dev.status) { set_err(c, "%s: slot %d's result is not a Telegram one", who, slot); return TGI_E_ARG; }
  }
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  const auto it = S.turns.find(turn);
  if (it == S.turns.end()) { set_err(c, "%s: no open turn %u", who, turn); return TGI_E_ARG; }
  CrawlState::Turn& T = it->second;
  const uint32_t P = (uint32_t)T.rows.size();
  const uint64_t N = T.n_work();
  if (one && P != 1) { set_err(c, "%s: turn %u covers %u pages (tgi_state_pages_end)", who, turn, P); return TGI_E_ARG; }
  if (s && one && s->last.n != N) {
    set_err(c, "%s: the slot's result holds %llu records, the turn %llu", who, (unsigned long long)s->last.n, (unsigned long long)N);
    return TGI_E_ARG;
  }
  if (s && (first > s->last.n || N > s->last.n - first)) {
    set_err(c, "%s: records [%llu, %llu + %llu) lie outside the result's %llu", who, (unsigned long long)first, (unsigned long long)first,
            (unsigned long long)N, (unsigned long long)s->last.n);
    return TGI_E_ARG;
  }
  std::vector<uint64_t> uoff(P + 1, 0);
  uint64_t reach = 0;  // statuses read: [0, reach) of the turn's records
  for (uint32_t k = 0; k < P; k++) {
    const uint64_t cnt = T.off[k + 1] - T.off[k], nd = n_done ? n_done[k] : cnt;
    if (nd > cnt) { set_err(c, "%s: page %u: n_done %llu > n_work %llu", who, k, (unsigned long long)nd, (unsigned long long)cnt); return TGI_E_ARG; }
    uoff[k + 1] = uoff[k] + nd;
    if (nd) reach = T.off[k] + nd;
  }
  const uint64_t m = uoff[P];
  if (!s && m && !status) { set_err(c, "%s: no statuses (slot < 0 takes them from the host)", who); return TGI_E_ARG; }
  const uint64_t before = S.n_msgs;
  uint32_t launches = 0;
  float ms = 0;
  if (m) {
    if ((rc = st_reserve(c, S, m))) return rc;
    cudaStream_t st = S.stream;
    // S.seg: woff [P+1] | uoff [P+1] | prow [P] | live [P] | app [P]
    const size_t o_uoff = (P + 1) * 8ull, o_prow = 2 * o_uoff, o_live = o_prow + 4ull * P, o_app = o_live + 4ull * P;
    const size_t seg_bytes = o_app + 4ull * P;
    CK(S.seg.ensure(seg_bytes));
    uint8_t* hseg;
    if ((rc = st_seg_host(c, S, seg_bytes, &hseg))) return rc;
    CK(S.upd.ensure(m * sizeof(tgi_state_update)));
    uint8_t* dseg = S.seg.as<uint8_t>();
    memcpy(hseg, T.off.data(), (P + 1) * 8);
    memcpy(hseg + o_uoff, uoff.data(), (P + 1) * 8);
    memcpy(hseg + o_prow, T.rows.data(), P * 4);
    uint32_t* live = (uint32_t*)(hseg + o_live);
    bool any = false;
    for (uint32_t k = 0; k < P; k++) {  // the pages whose row still holds this turn's keys as its owner view
      const auto vit = S.views.find(T.rows[k]);
      live[k] = vit != S.views.end() && vit->second.keys == T.keys && vit->second.off == T.off[k] && T.off[k + 1] > T.off[k];
      any = any || live[k];
    }
    if ((rc = st_seg_upload(c, S, 0, o_app))) return rc;
    StEnd e{};
    e.keys = T.keys->as<long long>();
    e.woff = (const uint64_t*)dseg;
    e.uoff = (const uint64_t*)(dseg + o_uoff);
    e.prow = (const uint32_t*)(dseg + o_prow);
    e.live = (const uint32_t*)(dseg + o_live);
    e.P = P;
    if (s) {
      CK(cudaEventRecord(S.ev_slot, s->stream));
      CK(cudaStreamWaitEvent(st, S.ev_slot, 0));
      e.status = s->last.dev.status + first;
    } else {
      CK(S.turn_in.ensure(reach));
      CK(cudaMemcpyAsync(S.turn_in.p, status, reach, cudaMemcpyHostToDevice, st));
      e.status = S.turn_in.as<uint8_t>();
    }
    // the device time is taken only when out asks for it: the one-page end pays no event
    if (out) CK(cudaEventRecord(S.t0, st));
    st_turn_updates_kernel<<<st_grid(c, m), ST_THREADS, 0, st>>>(e, m, S.upd.as<tgi_state_update>());
    launches++;
    CK(cudaGetLastError());
    if (out) CK(cudaEventRecord(S.t1, st));
    if ((rc = st_apply_updates(c, S, m, launches, P > 1, out ? &ms : nullptr))) return rc;  // synchronises
    float t = 0;
    if (out) {
      cudaEventElapsedTime(&t, S.t0, S.t1);
      ms += t;
    }
    // the owner's side of the updates, on the pages whose views are still this turn's keys
    if (any) {
      const uint64_t vslots = next_pow2(std::max<uint64_t>(2 * N, 64));
      CK(S.bfirst.ensure(vslots * 4));
      CK(S.blast.ensure(N * 4));
      StView v{};
      v.e = e;
      v.status = (uint16_t*)(T.keys->as<uint8_t>() + 16 * N);
      v.k = N;
      v.vfirst = S.bfirst.as<uint32_t>();
      v.vmask = vslots - 1;
      v.last = S.blast.as<uint32_t>();
      v.app = (uint32_t*)(dseg + o_app);
      CK(cudaMemsetAsync(v.vfirst, 0xFF, vslots * 4, st));
      CK(cudaMemsetAsync(v.last, 0, N * 4, st));
      CK(cudaMemsetAsync(v.app, 0xFF, P * 4, st));
      const tgi_state_update* u = S.upd.as<tgi_state_update>();
      if (out) CK(cudaEventRecord(S.t2, st));
      st_view_build_kernel<<<st_grid(c, std::max(N, m)), ST_THREADS, 0, st>>>(v, S.flag.as<uint32_t>(), m);
      st_view_hit_kernel<<<st_grid(c, m), ST_THREADS, 0, st>>>(v, u, m);
      st_view_status_kernel<<<st_grid(c, N), ST_THREADS, 0, st>>>(v, u);
      launches += 3;
      CK(cudaGetLastError());
      if (out) {
        CK(cudaEventRecord(S.t3, st));
        CK(cudaEventSynchronize(S.t3));
        cudaEventElapsedTime(&t, S.t2, S.t3);
        ms += t;
      }
    }
  }
  if (appended) *appended = S.n_msgs - before;
  if (out) {
    out->appended = S.n_msgs - before;
    out->kernel_ms = ms;
    out->gpu_launches = launches;
  }
  st_release(S, T.keys);
  S.turns.erase(it);
  return TGI_OK;
}

// UpdatePage(*owner) for P pages whose lists came from page turns (crawl/runner.go:1543-1544, dapr/standalone.go:589-609):
// each page's fields replace its row's; a row with an owner view makes the view its list, appended as its next
// generation.  All rows' fields go up in one upload and one kernel, every view is appended by one kernel.  The row
// strings' upload synchronises, as every row rewrite does; beyond it the call waits only for the pages' read-back
// (TGI_TURN_PAGE_JSON) or, given out, for its kernels' time.
int st_pages_close(tgi_ctx* c, CrawlState& S, const uint32_t* rows, uint32_t P, const tgi_state_page* pages, const uint8_t* strs,
                   uint64_t strs_len, uint32_t flags, const char* who, tgi_state_pages_t* out) {
  int rc;
  if ((rc = st_init(c, S))) return rc;
  if (out) memset(out, 0, sizeof *out);
  if (flags & ~TGI_TURN_PAGE_JSON) { set_err(c, "%s: unknown flags 0x%x", who, flags); return TGI_E_ARG; }
  if ((rc = st_check_rows(c, S, rows, P, who))) return rc;
  for (uint32_t k = 0; k < P; k++)
    if (!st_check_page(c, S, rows[k], pages[k], strs, strs_len, who, "its list is the owner view")) return TGI_E_ARG;
  const bool json = flags & TGI_TURN_PAGE_JSON, tiled = P > 1;
  if (json && (rc = st_upload_codes(c, S))) return rc;
  std::vector<const CrawlState::View*> view(P, nullptr);
  std::vector<uint32_t> bare;  // the rows without a view, ascending
  uint64_t K = 0;
  uint32_t Q = 0;
  for (uint32_t k = 0; k < P; k++) {
    const auto vit = S.views.find(rows[k]);
    if (vit == S.views.end()) {
      bare.push_back(rows[k]);
      continue;
    }
    view[k] = &vit->second;
    K += vit->second.k;
    Q++;
  }
  std::sort(bare.begin(), bare.end());
  if (K && (rc = st_reserve(c, S, K))) return rc;
  cudaStream_t st = S.stream;
  // S.seg: prow [P] | old [P] | bare rows [P] | row puts [P] | views [Q]
  const size_t o_old = 4ull * P, o_bare = 8ull * P, o_put = align16(12ull * P), o_view = o_put + P * sizeof(StRowPut);
  const size_t seg_bytes = o_view + Q * sizeof(StViewSeg);
  CK(S.seg.ensure(seg_bytes));
  uint8_t* hseg;
  if ((rc = st_seg_host(c, S, seg_bytes, &hseg))) return rc;
  CK(S.h_old.ensure(P * 4));
  CK(S.sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_sc.ensure(ST_SC_COUNT * 8));
  CK(S.row_base.ensure((S.rows.size() + 1) * 8));
  // no UpdateMessage of the loop follows: every open turn that lists one of the rows ends here
  {
    const std::unordered_set<uint32_t> closing(rows, rows + P);
    for (auto it = S.turns.begin(); it != S.turns.end();) {
      if (std::none_of(it->second.rows.begin(), it->second.rows.end(), [&](uint32_t r) { return closing.count(r) > 0; })) {
        ++it;
        continue;
      }
      st_release(S, it->second.keys);
      it = S.turns.erase(it);
    }
  }
  uint8_t* dseg = S.seg.as<uint8_t>();
  const uint32_t* d_rows = (const uint32_t*)dseg;
  uint32_t* d_old = (uint32_t*)(dseg + o_old);
  memcpy(hseg, rows, P * 4);
  memcpy(hseg + o_bare, bare.data(), bare.size() * 4);
  uint32_t launches = 0;
  // the old lists' lengths, brought back by the row strings' synchronise
  if ((rc = st_seg_upload(c, S, 0, o_put))) return rc;
  st_turn_meta_kernel<<<st_grid(c, P + 1), ST_THREADS, 0, st>>>(S.row_cnt.as<uint32_t>(), d_rows, P, nullptr, nullptr, nullptr, d_old);
  launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(S.h_old.p, d_old, P * 4, cudaMemcpyDeviceToHost, st));
  for (uint32_t k = 0; k < P; k++) {
    st_put_row(S, rows[k], pages[k], strs);
    if (view[k]) S.gen[rows[k]]++;
  }
  st_join_layers(S, rows, P);
  rc = st_sync_rows(c, S, std::vector<uint32_t>());  // the new strings
  if (rc) return rc;
  const uint32_t* old = S.h_old.as<uint32_t>();
  uint64_t M = 0;  // messages of the rows without a view
  StRowPut* put = (StRowPut*)(hseg + o_put);
  StViewSeg* vs = (StViewSeg*)(hseg + o_view);
  for (uint32_t k = 0, q = 0, voff = 0; k < P; k++) {
    const uint32_t r = rows[k];
    if (!view[k]) M += old[k];
    else S.n_dead += old[k];
    put[k] = StRowPut{S.rows[r], r, S.gen[r], view[k] ? (uint32_t)view[k]->k : 0u, view[k] ? 1u : 0u,
                      json ? (view[k] ? voff : 0) : ST_NO_BASE};
    if (view[k]) {
      vs[q++] = StViewSeg{view[k]->key_ptr(), view[k]->status_ptr(), voff, r, 0};
      voff += (uint32_t)view[k]->k;
    }
  }
  // the grouped order: the views' K messages, then (TGI_TURN_PAGE_JSON) the M of the rows without a view and the radix
  // passes' other buffer
  const uint64_t grouped = K + (json ? 2 * M : 0);
  CK(S.vals.ensure(grouped * 4));
  CK(S.keys.ensure(grouped * 4));
  if ((rc = st_seg_upload(c, S, o_put, seg_bytes - o_put))) return rc;
  const uint64_t n0 = S.n_msgs;
  const StDev d = st_dev(S);
  CK(cudaEventRecord(S.t2, st));
  st_rows_put_kernel<<<st_grid(c, P), ST_THREADS, 0, st>>>(S.pages.as<tgi_state_page>(), d.row_gen, d.row_cnt,
                                                           (const StRowPut*)(dseg + o_put), P, S.row_base.as<uint64_t>());
  launches++;
  if (K) {
    st_view_append_kernel<<<st_grid(c, K), ST_THREADS, 0, st>>>(d, (const StViewSeg*)(dseg + o_view), Q, K, n0, S.vals.as<uint32_t>(),
                                                                S.keys.as<uint32_t>());
    st_table_insert_kernel<<<st_grid(c, K), ST_THREADS, 0, st>>>(d, n0, n0 + K);
    launches += 2;
  }
  S.n_msgs += K;
  CK(cudaGetLastError());
  float ms1 = 0, ms2 = 0;
  StRender r{};
  uint64_t* hs = S.h_sc.as<uint64_t>();
  std::unique_lock<std::mutex> zg(c->cfg_mu, std::defer_lock);  // the zone table, as in tgi_state_render
  if (json) {
    // the rows without a view render their lists as they are: their live messages, found by a scan of the message rows
    // and grouped by row like the render's, follow the views' K messages
    if (M) {
      if ((rc = st_group_rows(c, S, (const uint32_t*)(dseg + o_bare), (uint32_t)bare.size(), M, K, tiled, launches))) return rc;
      st_row_starts_kernel<<<st_grid(c, M), ST_THREADS, 0, st>>>(S.keys.as<uint32_t>() + K, S.sc.as<uint64_t>() + ST_SC_LIVE, K,
                                                                 S.row_base.as<uint64_t>());
      launches++;
      CK(cudaGetLastError());
    }
    zg.lock();
    if ((rc = st_page_json_size(c, S, rows, P, S.vals.as<uint32_t>(), S.keys.as<uint32_t>(), K + M, tiled, r, launches))) return rc;
    CK(cudaMemcpyAsync(hs, S.sc.p, ST_SC_COUNT * 8, cudaMemcpyDeviceToHost, st));
  }
  CK(cudaGetLastError());
  CK(cudaEventRecord(S.t3, st));
  if (json) {
    CK(cudaStreamSynchronize(st));
    cudaEventElapsedTime(&ms1, S.t2, S.t3);
    if ((rc = st_page_json_emit(c, S, r, S.vals.as<uint32_t>(), K + M, hs, who, &out->page_json, &out->json_off, &ms2, launches)))
      return rc;
  }
  if ((rc = st_compact(c, S))) return rc;
  if (out) {
    if (!json) {
      CK(cudaEventSynchronize(S.t3));
      cudaEventElapsedTime(&ms1, S.t2, S.t3);
    }
    out->n_pages = P;
    out->kernel_ms = ms1 + ms2;
    out->gpu_launches = launches;
  }
  return TGI_OK;
}

}  // namespace

extern "C" {

int tgi_state_pages_begin(tgi_ctx* c, const uint32_t* rows, uint32_t n_pages, const tgi_state_page* pages, const uint8_t* strs,
                          uint64_t strs_len, const int64_t* fetched, uint64_t n, const uint64_t* fetched_off, uint32_t flags,
                          tgi_state_pages_t* out) {
  if (!c || !out || (n_pages && !rows) || !fetched_off || (n && !fetched)) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  return st_pages_begin(c, S, rows, n_pages, pages, strs, strs_len, fetched, n, fetched_off, flags, "tgi_state_pages_begin", out);
}

int tgi_state_pages_end(tgi_ctx* c, uint32_t turn, int slot, uint64_t first, const uint8_t* status, const uint64_t* n_done,
                        tgi_state_end_t* out) {
  if (!c) return TGI_E_ARG;
  if (out) memset(out, 0, sizeof *out);
  return st_pages_end(c, turn, slot, first, status, n_done, false, nullptr, out);
}

int tgi_state_pages_close(tgi_ctx* c, const uint32_t* rows, uint32_t n_pages, const tgi_state_page* pages, const uint8_t* strs,
                          uint64_t strs_len, uint32_t flags, tgi_state_pages_t* out) {
  if (!c || (n_pages && (!rows || !pages)) || (!out && (flags & TGI_TURN_PAGE_JSON))) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  return st_pages_close(c, S, rows, n_pages, pages, strs, strs_len, flags, "tgi_state_pages_close", out);
}

// the one-page calls: P = 1 of the calls above
int tgi_state_page_begin(tgi_ctx* c, uint32_t row, const tgi_state_page* page, const uint8_t* strs, uint64_t strs_len,
                         const int64_t* fetched, uint64_t n, uint32_t flags, tgi_state_turn_t* out) {
  if (!c || !out || (n && !fetched)) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  memset(out, 0, sizeof *out);
  const uint64_t foff[2] = {0, n};
  tgi_state_pages_t o;
  const int rc = st_pages_begin(c, S, &row, 1, page, strs, strs_len, fetched, n, foff, flags, "tgi_state_page_begin", &o);
  if (rc) return rc;
  out->turn = o.turn;
  out->row = row;
  out->n_work = o.n_work;
  out->work = o.work;
  out->page_json = o.page_json;
  out->page_json_len = o.page_json ? o.json_off[1] - 1 : 0;  // the line without its '\n'
  out->kernel_ms = o.kernel_ms;
  out->gpu_launches = o.gpu_launches;
  return TGI_OK;
}

int tgi_state_page_end(tgi_ctx* c, uint32_t turn, int slot, const uint8_t* status, uint64_t n_done, uint64_t* appended) {
  if (!c || (slot < 0 && n_done && !status)) return TGI_E_ARG;
  return st_pages_end(c, turn, slot, 0, status, &n_done, true, appended, nullptr);
}

int tgi_state_page_close(tgi_ctx* c, uint32_t row, const tgi_state_page* page, const uint8_t* strs, uint64_t strs_len,
                         uint32_t flags, tgi_state_json_t* out) {
  if (!c || !page || (!out && (flags & TGI_TURN_PAGE_JSON))) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  if (out) memset(out, 0, sizeof *out);
  tgi_state_pages_t o;
  const int rc = st_pages_close(c, S, &row, 1, page, strs, strs_len, flags, "tgi_state_page_close", out ? &o : nullptr);
  if (rc || !out) return rc;
  out->data = o.page_json;
  out->len = o.page_json ? o.json_off[1] - 1 : 0;
  out->kernel_ms = o.kernel_ms;
  out->gpu_launches = o.gpu_launches;
  return TGI_OK;
}

}  // extern "C"

// ---- snowball discovery (state.cuh) -----------------------------------------------------------------------------------
namespace {

// one AddLayer of a discovery call: its depth, whether the call has a page at all (Base rules create the layer then),
// and its survivors [s0, s1) of S.h_surv
struct DiscGroup {
  int64_t depth;
  bool any;
  uint64_t s0, s1;
};

// the checks both discovery calls share; with TGI_DISCOVER_PAGE_JSON the clock must render (json.Marshal's year rule)
int disc_args(tgi_ctx* c, uint32_t flags, uint32_t allowed, int64_t now_sec, int32_t now_nsec, const char* who) {
  if (flags & ~allowed) { set_err(c, "%s: unknown flags 0x%x", who, flags); return TGI_E_ARG; }
  if (now_nsec < 0 || now_nsec >= 1000000000) { set_err(c, "%s: now_nsec %d out of range", who, now_nsec); return TGI_E_ARG; }
  if (flags & TGI_DISCOVER_PAGE_JSON) {
    char b[48];
    std::lock_guard<std::mutex> zg(c->cfg_mu);
    if (!host_render_zone_time(b, now_sec, now_nsec, c->zone, c->cfgdev.tz)) {
      set_err(c, "%s: the clock's year is outside [0, 9999] (json.Marshal fails)", who);
      return TGI_E_ARG;
    }
  }
  return TGI_OK;
}

// the page-JSON outputs of a call that adds nothing: json_off = {0}
int disc_json_empty(tgi_ctx* c, CrawlState& S, tgi_state_added_t* out) {
  CK(S.h_json_off.ensure(8));
  CK(S.h_out.ensure(1));
  S.h_json_off.as<uint64_t>()[0] = 0;
  out->json_off = S.h_json_off.as<uint64_t>();
  out->page_json = S.h_out.as<uint8_t>();
  return TGI_OK;
}

// What the span calls (tgi_state_discover, tgi_state_pending_edges) need of slot s, under its lock: a finished
// Telegram result with its link rows
int disc_slot(tgi_ctx* c, const Slot& s, int slot, const char* who) {
  if (in_flight(s)) { set_err(c, "%s: slot %d is in flight", who, slot); return TGI_E_STATE; }
  if (!s.busy || s.last.kind == REC_NONE) { set_err(c, "%s: slot %d holds no result (released or none)", who, slot); return TGI_E_STATE; }
  if (s.last.kind != REC_TG) { set_err(c, "%s: slot %d's result is not a Telegram one", who, slot); return TGI_E_STATE; }
  if (!s.last.dev.link_off || !s.last.dev.links) { set_err(c, "%s: slot %d's result has no links (run it with TGI_RUN_LINKS)", who, slot); return TGI_E_STATE; }
  return TGI_OK;
}

// The spans' checks against slot s's result, and the gather's bound: the result's link rows times the largest number
// of spans that share a processed record (no read-back)
int disc_bound(tgi_ctx* c, const CrawlState& S, const Slot& s, const tgi_state_span* spans, uint32_t n_spans,
               const char* who, uint64_t* bound) {
  const uint64_t n = s.last.n;
  std::vector<std::pair<uint64_t, int>> ev;  // the processed records' intervals
  for (uint32_t k = 0; k < n_spans; k++) {
    const tgi_state_span& sp = spans[k];
    if (sp.row >= S.rows.size()) { set_err(c, "%s: span %u: no row %u", who, k, sp.row); return TGI_E_ARG; }
    if (sp.first > n || sp.n_records > n - sp.first) { set_err(c, "%s: span %u lies outside the result's %llu records", who, k, (unsigned long long)n); return TGI_E_ARG; }
    if (sp.n_done > sp.n_records) { set_err(c, "%s: span %u: n_done %llu > n_records %llu", who, k, (unsigned long long)sp.n_done, (unsigned long long)sp.n_records); return TGI_E_ARG; }
    if (sp.n_done) {
      ev.emplace_back(sp.first, 1);
      ev.emplace_back(sp.first + sp.n_done, -1);
    }
  }
  std::sort(ev.begin(), ev.end(), [](const auto& a, const auto& b) { return a.first != b.first ? a.first < b.first : a.second < b.second; });
  int64_t cover = 0, most = 0;
  for (const auto& e : ev) most = std::max(most, cover += e.second);
  *bound = (uint64_t)most * s.last.n_links;  // link rows over the spans' processed records, at most
  return TGI_OK;
}

// The discovery gather on the state stream, behind the slot's work: the spans' candidates (status, n_done, owner URL)
// into out in (span, record, link row) order, every span's first candidate in gd.coff (the count at [n_spans]).  The
// device time runs from S.t0; no synchronise.
int disc_gather(tgi_ctx* c, CrawlState& S, Slot& s, const tgi_state_span* spans, uint32_t n_spans, uint64_t bound,
                StCand* out, bool tiled, StDisc& gd, uint32_t& launches) {
  cudaStream_t st = S.stream;
  CK(S.spans.ensure(n_spans * sizeof(tgi_state_span)));
  CK(S.cnt.ensure(n_spans * 4));
  CK(S.soff.ensure((n_spans + 1) * 8));
  CK(S.coff.ensure((n_spans + 1) * 8));
  CK(S.lnk.ensure(bound * 4));
  CK(S.spn.ensure(bound * 4));
  CK(S.flag.ensure(bound * 4));
  CK(S.pos.ensure((bound + 1) * 8));
  CK(S.sc.ensure(ST_SC_COUNT * 8));
  gd = StDisc{};
  gd.spans = S.spans.as<tgi_state_span>();
  gd.n_spans = n_spans;
  gd.status = s.last.dev.status;
  gd.link_off = s.last.dev.link_off;
  gd.links = s.last.dev.links;
  gd.soff = S.soff.as<uint64_t>();
  gd.bound = bound;
  gd.flag = S.flag.as<uint32_t>();
  gd.lnk = S.lnk.as<uint32_t>();
  gd.spn = S.spn.as<uint32_t>();
  gd.pos = S.pos.as<uint64_t>();
  gd.out = out;
  gd.coff = S.coff.as<uint64_t>();
  int rc;
  CK(cudaMemcpyAsync(S.spans.p, spans, n_spans * sizeof(tgi_state_span), cudaMemcpyHostToDevice, st));
  CK(cudaEventRecord(S.ev_slot, s.stream));  // the result is complete on the slot's stream
  CK(cudaStreamWaitEvent(st, S.ev_slot, 0));
  CK(cudaEventRecord(S.t0, st));
  st_disc_count_kernel<<<st_grid(c, n_spans), ST_THREADS, 0, st>>>(gd, S.cnt.as<uint32_t>());
  launches++;
  if ((rc = launch_scan(c, st, S.tiles, S.cnt.as<uint32_t>(), n_spans, S.soff.as<uint64_t>(), S.sc.as<uint64_t>() + 1, launches, tiled))) return rc;
  st_disc_flag_kernel<<<st_grid(c, bound), ST_THREADS, 0, st>>>(st_dev(S), gd);
  launches++;
  if ((rc = launch_scan(c, st, S.tiles, gd.flag, bound, gd.pos, S.sc.as<uint64_t>() + 2, launches, tiled))) return rc;
  st_disc_emit_kernel<<<st_grid(c, bound), ST_THREADS, 0, st>>>(gd);
  launches++;
  CK(cudaGetLastError());
  return TGI_OK;
}

// First occurrences (per span, or over the list) and, with url_test, Dapr's urlCache test over the candidates at d_cands
// (count d_n on the device, at most bound), compacted into S.surv; the survivors come back to S.h_surv with one id each
// from counter id_next on (S.h_ids).  Two synchronises: the survivors' count, then their rows and ids.  The urlCache is
// read under fr_mu, behind its last change.
int st_survivors(tgi_ctx* c, CrawlState& S, const StCand* d_cands, const uint64_t* d_n, uint64_t bound, bool per_span,
                 bool dedup, bool url_test, uint64_t* n_surv, float* ms, uint32_t& launches) {
  cudaStream_t st = S.stream;
  std::unique_lock<std::mutex> fg(c->fr_mu, std::defer_lock);
  FrontierDev urls{};
  if (url_test) {
    fg.lock();
    if (c->fr_event_valid) CK(cudaStreamWaitEvent(st, c->fr_event, 0));
    urls = c->sets[TGI_SET_URLS].dev;
  }
  const uint64_t bslots = next_pow2(std::max<uint64_t>(2 * bound, 64));
  CK(S.bfirst.ensure(bslots * 4));
  CK(S.slot_of.ensure(bound * 4));
  CK(S.flag.ensure(bound * 4));
  CK(S.pos.ensure((bound + 1) * 8));
  CK(S.surv.ensure(bound * sizeof(StCand)));
  CK(S.sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_sc.ensure(ST_SC_COUNT * 8));
  StFirst w{};
  w.c = d_cands;
  w.n = d_n;
  w.bound = bound;
  w.per_span = per_span;
  w.dedup = dedup;
  w.urls = urls;
  w.bfirst = S.bfirst.as<uint32_t>();
  w.bmask = bslots - 1;
  w.slot_of = S.slot_of.as<uint32_t>();
  w.flag = S.flag.as<uint32_t>();
  w.pos = S.pos.as<uint64_t>();
  w.out = S.surv.as<StCand>();
  int rc;
  CK(cudaEventRecord(S.t2, st));
  if (dedup) {
    CK(cudaMemsetAsync(w.bfirst, 0xFF, bslots * 4, st));
    st_first_kernel<<<st_grid(c, bound), ST_THREADS, 0, st>>>(w);
    launches++;
  }
  st_keep_kernel<<<st_grid(c, bound), ST_THREADS, 0, st>>>(w);
  launches++;
  if ((rc = launch_scan(c, st, S.tiles, w.flag, bound, w.pos, S.sc.as<uint64_t>(), launches))) return rc;
  st_survivors_kernel<<<st_grid(c, bound), ST_THREADS, 0, st>>>(w);
  launches++;
  CK(cudaGetLastError());
  CK(cudaEventRecord(S.t3, st));
  CK(cudaMemcpyAsync(S.h_sc.p, S.sc.p, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const uint64_t m = *S.h_sc.as<uint64_t>();
  float t = 0;
  cudaEventElapsedTime(&t, S.t2, S.t3);
  *ms += t;
  CK(S.h_surv.ensure(m * sizeof(StCand)));
  CK(S.h_ids.ensure(m * 36));
  if (m) {
    CK(S.uuids.ensure(m * 36));
    CK(cudaMemcpyAsync(S.h_surv.p, S.surv.p, m * sizeof(StCand), cudaMemcpyDeviceToHost, st));
    CK(cudaEventRecord(S.t2, st));
    st_uuid_kernel<<<st_grid(c, m), ST_THREADS, 0, st>>>(S.id_seed, S.id_next, m, S.uuids.as<uint8_t>());
    launches++;
    CK(cudaGetLastError());
    CK(cudaEventRecord(S.t3, st));
    CK(cudaMemcpyAsync(S.h_ids.p, S.uuids.p, m * 36, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    cudaEventElapsedTime(&t, S.t2, S.t3);
    *ms += t;
  }
  *n_surv = m;
  return TGI_OK;
}

// AddLayer of every group in order under Base's or Dapr's rules, on the survivors in S.h_surv and their ids in S.h_ids.
// The host mirror's URL map decides which pages go in (pageMap changes under UpdatePage / AddLayer overwrites, which a
// key set cannot follow); nothing changes before every check has passed.
int st_discover_apply(tgi_ctx* c, CrawlState& S, const std::vector<DiscGroup>& G, bool dapr, bool json, int64_t now_sec,
                      int32_t now_nsec, int64_t max_pages, const char* who, tgi_state_added_t* out, float* ms,
                      uint32_t& launches) {
  const StCand* sv = S.h_surv.as<StCand>();
  auto url_of = [&](const StCand& k) { return std::string((const char*)k.name, k.len); };
  // 1. the pages each AddLayer adds, in append order
  std::vector<uint64_t> pick;
  std::vector<size_t> gend;
  std::unordered_set<std::string> seen;  // URLs added earlier in the call: in pageMap (Base) or in the urlCache (Dapr)
  uint64_t rows = S.rows.size();
  for (const DiscGroup& g : G) {
    const bool reached = max_pages > 0 && (int64_t)rows >= max_pages;
    int64_t replacements = (int64_t)S.deadends;
    std::vector<std::string> added;
    for (uint64_t j = g.s0; j < g.s1; j++) {
      std::string u = url_of(sv[j]);
      if (seen.count(u)) continue;
      if (!dapr) {
        if (S.urls.count(u)) continue;
        if (reached) {
          if (replacements <= 0) continue;
          replacements--;
        }
        seen.insert(std::move(u));
      } else {
        added.push_back(std::move(u));  // Dapr's urlCache takes the URLs after its loop: a repeat within the page stays
      }
      pick.push_back(j);
      rows++;
    }
    for (std::string& u : added) seen.insert(std::move(u));
    gend.push_back(pick.size());
  }
  const uint64_t n_add = pick.size();
  if (n_add && !S.seeded) { set_err(c, "%s: no id seed (tgi_state_id_seed)", who); return TGI_E_STATE; }
  int rc;
  // 2. Dapr: the added URLs enter the urlCache first.  The insert is all or nothing (a full set is left untouched,
  // frontier_append_body), so a set that cannot take them leaves the state as it was
  if (dapr && n_add) {
    std::vector<uint8_t> keys(n_add * 32);
    for (uint64_t k = 0; k < n_add; k++) memcpy(keys.data() + 32 * k, sv[pick[k]].name, 32);
    std::lock_guard<std::mutex> fg(c->fr_mu);
    KeySet& U = c->sets[TGI_SET_URLS];
    if ((rc = set_first_use(c, U, false))) return rc;
    cudaStream_t st0 = c->slots[0].stream;
    CK(S.url_keys.ensure(n_add * 32));
    CK(cudaMemcpyAsync(S.url_keys.p, keys.data(), n_add * 32, cudaMemcpyHostToDevice, st0));
    if ((rc = frontier_insert_enqueue(c, U, S.url_keys.p, nullptr, n_add, nullptr))) return rc;
    CK(cudaStreamSynchronize(st0));
    if ((rc = frontier_insert_check(c, U))) return rc;
  }
  // 3. the pages {id, URL, "unfetched", ParentID = the owner's id, depth, the clock in time.Local} on their layers
  CK(S.h_rows.ensure(n_add * 4 + 4));
  uint32_t* hr = S.h_rows.as<uint32_t>();
  const uint8_t* ids = S.h_ids.as<uint8_t>();
  std::vector<uint32_t> dirty;
  std::string strs;
  size_t k = 0;
  for (size_t gi = 0; gi < G.size(); gi++) {
    const size_t k1 = gend[gi];
    if (dapr ? k1 == k : !G[gi].any) continue;  // Dapr creates no layer when nothing is added
    std::vector<uint32_t>& L = S.layers[G[gi].depth];
    for (; k < k1; k++) {
      const StCand& cd = sv[pick[k]];
      const std::string parent = st_field(S, S.rows[cd.parent], TGI_PS_ID);
      strs.assign((const char*)ids + 36 * k, 36);
      strs.append((const char*)cd.name, cd.len);
      strs += "unfetched";
      strs += parent;
      tgi_state_page p{};
      p.str_len[TGI_PS_ID] = 36;
      p.str_len[TGI_PS_URL] = cd.len;
      p.str_len[TGI_PS_STATUS] = 9;
      p.str_len[TGI_PS_PARENT] = (uint32_t)parent.size();
      p.ts_off = TGI_STATE_TS_LOCAL;
      p.depth = G[gi].depth;
      p.ts_sec = now_sec;
      p.ts_nsec = now_nsec;
      const auto it = S.by_id.find(strs.substr(0, 36));
      uint32_t r = (uint32_t)S.rows.size();
      if (it != S.by_id.end()) {  // pageMap[id] = page: the old page and its messages go, as in AddLayer
        r = it->second;
        if (std::find(dirty.begin(), dirty.end(), r) == dirty.end()) {
          if (r < S.rows_synced && (rc = st_drop_messages(c, S, r))) return rc;
          dirty.push_back(r);
        }
      }
      st_put_row(S, r, p, (const uint8_t*)strs.data());
      L.push_back(r);
      hr[k] = r;
    }
  }
  if ((rc = st_sync_rows(c, S, dirty))) return rc;
  if ((rc = st_compact(c, S))) return rc;
  S.id_next += n_add;
  out->n_added = n_add;
  out->rows = hr;
  out->ids = ids;
  if (!json) return TGI_OK;
  // 4. json.Marshal of every added page by the page turns' line passes over the added rows, which hold no messages
  if (!n_add) return disc_json_empty(c, S, out);
  if ((rc = st_upload_codes(c, S))) return rc;
  std::lock_guard<std::mutex> zg(c->cfg_mu);  // the zone table, as in tgi_state_render
  cudaStream_t st = S.stream;
  const uint64_t nr = S.rows.size();
  CK(S.row_base.ensure((nr + 1) * 8));
  CK(cudaMemsetAsync(S.row_base.p, 0, (nr + 1) * 8, st));
  StRender r{};
  uint64_t* hs = S.h_sc.as<uint64_t>();
  CK(cudaEventRecord(S.t4, st));
  if ((rc = st_page_json_size(c, S, hr, (uint32_t)n_add, nullptr, nullptr, 0, false, r, launches))) return rc;
  CK(cudaEventRecord(S.t5, st));
  CK(cudaMemcpyAsync(hs, S.sc.p, ST_SC_COUNT * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  float size_ms = 0, emit_ms = 0;
  cudaEventElapsedTime(&size_ms, S.t4, S.t5);
  if ((rc = st_page_json_emit(c, S, r, nullptr, 0, hs, who, &out->page_json, &out->json_off, &emit_ms, launches))) return rc;
  *ms += size_ms + emit_ms;
  return TGI_OK;
}

// The SQL text of a statement of `rows` rows (TGI_SQL_*): for one row the literal of CreatePendingBatch,
// InsertPendingEdge, ClosePendingBatch, AddPageToPageBuffer, SaveEdgeRecords, CompletePendingBatch or FlushBatchStats'
// upsert and delete, UpsertSeedChannelChatID, MarkChannelInvalid, InsertAccessEvent or UpdatePendingEdge
// (state/daprstate.go:3897, 3915, 3935, 3620, 3167, 4126, 4163, 4170, 3400, 3576, 4386, 4001); for more the VALUES tuple
// repeated with the placeholders numbered on (before the ON CONFLICT clause of the upserts), WHERE batch_id IN (...), or
// the update's join on a VALUES list.  The stats upsert and the access event always have one row.
void edge_sql_text(uint32_t kind, uint32_t rows, std::string& s) {
  if (kind == TGI_SQL_EDGE_UPDATE) {  // UpdatePendingEdge (daprstate.go:4001); more rows join a VALUES list on the id
    if (rows == 1) {
      s = "UPDATE pending_edges SET validation_status = $1, validation_reason = $2, validated_at = NOW() WHERE pending_id = $3;";
      return;
    }
    s = "UPDATE pending_edges AS e SET validation_status = v.s, validation_reason = v.r, validated_at = NOW() FROM (VALUES ";
    for (uint32_t r = 0; r < rows; r++) {
      s += r ? ", ($" : "($";
      s += std::to_string(3 * r + 1) + ", $" + std::to_string(3 * r + 2) + ", $" + std::to_string(3 * r + 3) + "::integer)";
    }
    s += ") AS v(s, r, id) WHERE e.pending_id = v.id;";
    return;
  }
  static const char* const head[11] = {
      "INSERT INTO pending_edge_batches (batch_id, crawl_id, source_channel, source_page_id, source_depth, sequence_id, "
      "status) VALUES ",
      "INSERT INTO pending_edges (batch_id, crawl_id, destination_channel, source_channel, sequence_id, discovery_time, "
      "source_type, validation_status) VALUES ",
      "UPDATE pending_edge_batches SET status = 'closed', closed_at = NOW() WHERE batch_id ",
      "INSERT INTO page_buffer (page_id, parent_id, depth, url, crawl_id, sequence_id) VALUES ",
      "INSERT INTO edge_records (destination_channel, source_channel, walkback, skipped, discovery_time, crawl_id, "
      "sequence_id) VALUES ",
      "UPDATE pending_edge_batches SET status = 'completed', completed_at = NOW() WHERE batch_id ",
      "INSERT INTO source_type_stats (crawl_id, source_type, total, valid, not_channel, invalid, duplicate) VALUES ($1, "
      "$2, $3, $4, $5, $6, $7) ON CONFLICT (crawl_id, source_type) DO UPDATE SET total = source_type_stats.total + "
      "EXCLUDED.total, valid = source_type_stats.valid + EXCLUDED.valid, not_channel = source_type_stats.not_channel + "
      "EXCLUDED.not_channel, invalid = source_type_stats.invalid + EXCLUDED.invalid, duplicate = "
      "source_type_stats.duplicate + EXCLUDED.duplicate;",
      "DELETE FROM pending_edges WHERE batch_id ",
      "INSERT INTO seed_channels (channel_username, chat_id) VALUES ",
      "INSERT INTO invalid_channels (channel_username, reason, invalidated_at) VALUES ",
      "INSERT INTO access_events (reason, occurred_at) VALUES "};
  static const uint32_t per_row[11] = {7, 8, 1, 6, 7, 1, 7, 1, 2, 2, 1};
  const uint32_t per = per_row[kind];
  s = head[kind];
  if (kind == TGI_SQL_STATS_UPSERT) return;
  s.reserve(s.size() + (size_t)rows * (per * 8 + 4) + 8);
  char num[16] = {'$'};
  auto param = [&](uint32_t p) { s.append(num, (size_t)(std::to_chars(num + 1, num + sizeof num, p).ptr - num)); };
  if (kind == TGI_SQL_BATCH_CLOSE || kind == TGI_SQL_BATCH_COMPLETE || kind == TGI_SQL_EDGES_DELETE) {
    if (rows == 1) {
      s += "= $1;";
      return;
    }
    s += "IN (";
    for (uint32_t r = 0; r < rows; r++) {
      if (r) s += ", ";
      param(r + 1);
    }
    s += ");";
    return;
  }
  for (uint32_t r = 0; r < rows; r++) {
    s += r ? ", (" : "(";
    for (uint32_t k = 0; k < per; k++) {
      if (k) s += ", ";
      param(r * per + k + 1);
    }
    s += kind == TGI_SQL_INVALID_UPSERT || kind == TGI_SQL_ACCESS_EVENT ? ", NOW())" : ")";
  }
  if (kind == TGI_SQL_SEED_UPSERT) s += " ON CONFLICT (channel_username) DO UPDATE SET chat_id = EXCLUDED.chat_id";
  if (kind == TGI_SQL_INVALID_UPSERT)
    s += " ON CONFLICT (channel_username) DO UPDATE SET reason = EXCLUDED.reason, invalidated_at = NOW()";
  s += ";";
}

// An accepted hand-off's edge-less spans (tgi_state_walkback's input) from its span_batch, read back already; its
// walkbacks are not picked yet
void handoff_walkbacks(CrawlState& S, const tgi_state_span* spans, uint32_t n_spans) {
  const uint32_t* sb = S.h_span_batch.as<uint32_t>();
  S.wb_spans.clear();
  for (uint32_t k = 0; k < n_spans; k++)
    if (sb[k] == TGI_STATE_NO_BATCH) {
      S.wb_spans.push_back(k);
      S.wb_spans.push_back(spans[k].row);
    }
  S.wb_picked = false;
  S.wb_n_ok = 0;
}

// the checks the SQL calls make, in order: rows_per_stmt, now_nsec, crawl_id, and for the hand-off's two a live hand-off
int sql_args(tgi_ctx* c, const CrawlState& S, uint32_t k, int32_t now_nsec, const char* crawl_id, uint32_t crawl_id_len,
             const char* who, bool handoff = true) {
  if (k < 1 || k > TGI_SQL_MAX_ROWS) { set_err(c, "%s: rows_per_stmt %u outside [1, %u]", who, k, TGI_SQL_MAX_ROWS); return TGI_E_ARG; }
  if (now_nsec < 0 || now_nsec >= 1000000000) { set_err(c, "%s: now_nsec %d out of range", who, now_nsec); return TGI_E_ARG; }
  if (crawl_id_len && !crawl_id) { set_err(c, "%s: crawl_id is NULL", who); return TGI_E_ARG; }
  if (handoff && !S.handoff_live) { set_err(c, "%s: no tandem hand-off (tgi_state_pending_edges, then no other state call)", who); return TGI_E_STATE; }
  return TGI_OK;
}

// discovery_time: the clock in time.Local, rendered with its quotes into tb[0, *tl); a year outside [0, 9999] refuses
int sql_clock(tgi_ctx* c, int64_t now_sec, int32_t now_nsec, const char* who, char (&tb)[48], uint32_t* tl) {
  std::lock_guard<std::mutex> zg(c->cfg_mu);
  *tl = (uint32_t)host_render_zone_time(tb, now_sec, now_nsec, c->zone, c->cfgdev.tz);
  if (!*tl) { set_err(c, "%s: the clock's local year is outside [0, 9999] (json.Marshal fails)", who); return TGI_E_ARG; }
  return TGI_OK;
}

// The statements of q.p (kind, k and rows of its kinds set) over `threads` row threads: their texts on the host (one per kind and
// row count, a kind's last statement maybe shorter), crawl_id and the clock tb[0, tl) uploaded, the params by the
// two-pass writer (accepted() once the size pass has passed), and the texts, params and statement table read back into
// h and hst.  Adds its device time and launches to out's.
template <class Q, class Out, class F>
int sql_render(tgi_ctx* c, CrawlState& S, Q& q, void (*size)(StDev, Q), void (*emit)(StDev, Q), uint64_t threads,
               const char* crawl_id, uint32_t crawl_id_len, const char* tb, uint32_t tl, const char* who, F&& accepted,
               HostBuf& h, HostBuf& hst, Out* out) {
  StSqlPlan& p = q.p;
  uint64_t n_rows = 0;
  std::string texts, t;
  for (uint32_t i = 0; i < ST_SQL_KINDS; i++) {
    const uint32_t k = p.k[i] ? p.k[i] : 1;  // a kind past the call's has no rows
    p.m[i] = (p.rows[i] + k - 1) / k;
    p.n_stmts += p.m[i];
    n_rows += p.rows[i];
    const uint32_t rows[2] = {p.rows[i] >= k ? k : 0u, (uint32_t)(p.rows[i] % k)};
    for (int j = 0; j < 2; j++) {
      if (!rows[j]) continue;
      edge_sql_text(p.kind[i], rows[j], t);
      p.sql_off[2 * i + j] = texts.size();
      p.sql_len[2 * i + j] = t.size();
      texts += t;
    }
  }
  cudaStream_t st = S.stream;
  const size_t t_at = (crawl_id_len + 15) & ~(size_t)15;
  CK(S.sql_in.ensure(t_at + 48));
  CK(S.sql_size.ensure(n_rows * 4));
  CK(S.sql_off.ensure((n_rows + 1) * 8));
  CK(S.sql_stmts.ensure(p.n_stmts * sizeof(tgi_state_edge_stmt)));
  CK(S.sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_sc.ensure(ST_SC_COUNT * 8));
  std::vector<uint8_t> in(t_at + tl);
  if (crawl_id_len) memcpy(in.data(), crawl_id, crawl_id_len);
  if (tl) memcpy(in.data() + t_at, tb, tl);
  if (!in.empty()) CK(cudaMemcpyAsync(S.sql_in.p, in.data(), in.size(), cudaMemcpyHostToDevice, st));
  p.crawl = S.sql_in.as<uint8_t>();
  p.crawl_len = crawl_id_len;
  p.time = p.crawl + t_at;
  p.time_len = tl;
  p.size = S.sql_size.as<uint32_t>();
  p.off = S.sql_off.as<uint64_t>();
  p.sc = S.sc.as<uint64_t>();
  p.stmts = S.sql_stmts.as<tgi_state_edge_stmt>();
  p.base = texts.size();
  const unsigned grid = sink_grid(c, std::max(threads, p.n_stmts), ST_THREADS, 4);  // one pass: SMs x 1024 rows
  uint32_t launches = 0;
  uint64_t body = 0;
  int rc;
  if ((rc = st_rows_size(c, S, size, q, grid, p.size, n_rows, p.off, who, "a row", &body, launches))) return rc;
  accepted();
  CK(h.ensure(texts.size() + body));
  CK(hst.ensure(p.n_stmts * sizeof(tgi_state_edge_stmt)));
  if ((rc = st_rows_emit(c, S, emit, q, &p.out, S.sql_out, body, grid, launches))) return rc;
  uint8_t* o = h.as<uint8_t>();
  CK(cudaMemcpyAsync(o + texts.size(), S.sql_out.p, body, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(hst.p, S.sql_stmts.p, p.n_stmts * sizeof(tgi_state_edge_stmt), cudaMemcpyDeviceToHost, st));
  memcpy(o, texts.data(), texts.size());  // beside the copies: another part of the buffer
  CK(cudaStreamSynchronize(st));
  out->n_stmts = p.n_stmts;
  out->stmts = hst.as<tgi_state_edge_stmt>();
  out->data = o;
  out->data_len = texts.size() + body;
  out->kernel_ms += st_rows_ms(S);
  out->gpu_launches += launches;
  return TGI_OK;
}

// The claimed batches' checks (TGI_E_ARG): every array, offset, length and class code, before anything is uploaded
int vw_input(tgi_ctx* c, const tgi_claimed_batches* in, const char* who) {
  const uint64_t n = in->n_batches, ne = in->n_edges, sl = in->strs_len;
  if (n && (!in->batches || !in->edge_off)) { set_err(c, "%s: batches or edge_off is NULL", who); return TGI_E_ARG; }
  if (ne && !in->edges) { set_err(c, "%s: edges is NULL", who); return TGI_E_ARG; }
  if (sl && !in->strs) { set_err(c, "%s: strs is NULL", who); return TGI_E_ARG; }
  if (!n) return TGI_OK;
  if (in->edge_off[0] != 0 || in->edge_off[n] != ne) {
    set_err(c, "%s: edge_off[0] must be 0 and edge_off[n] n_edges (%llu)", who, (unsigned long long)ne);
    return TGI_E_ARG;
  }
  auto out_of = [&](uint64_t off, uint32_t len) { return off > sl || len > sl - off; };
  for (uint64_t i = 0; i < n; i++) {
    const uint64_t a = in->edge_off[i], b = in->edge_off[i + 1];
    if (b < a) { set_err(c, "%s: edge_off decreases at batch %llu", who, (unsigned long long)i); return TGI_E_ARG; }
    if (b - a >= TGI_VW_NO_EDGE) { set_err(c, "%s: batch %llu has 2^32 - 1 edges or more", who, (unsigned long long)i); return TGI_E_ARG; }
    const tgi_claimed_batch& B = in->batches[i];
    for (int f = 0; f < 5; f++)
      if (out_of(B.str_off[f], B.str_len[f])) { set_err(c, "%s: batch %llu string %d outside strs", who, (unsigned long long)i, f); return TGI_E_ARG; }
  }
  for (uint64_t j = 0; j < ne; j++) {
    const tgi_claimed_edge& E = in->edges[j];
    if (E.cls > TGI_EDGE_CLASS_OTHER) { set_err(c, "%s: edge %llu has class %u", who, (unsigned long long)j, E.cls); return TGI_E_ARG; }
    for (int f = 0; f < 2; f++)
      if (out_of(E.str_off[f], E.str_len[f])) { set_err(c, "%s: edge %llu string %d outside strs", who, (unsigned long long)j, f); return TGI_E_ARG; }
  }
  return TGI_OK;
}

// A claim's checks (TGI_E_ARG): its arrays, strings, destinations and pending_ids, before anything is uploaded
int ve_input(tgi_ctx* c, const tgi_pending_claim* in, const char* who) {
  const uint64_t n = in->n_edges, sl = in->strs_len;
  if (n && !in->edges) { set_err(c, "%s: edges is NULL", who); return TGI_E_ARG; }
  if (sl && !in->strs) { set_err(c, "%s: strs is NULL", who); return TGI_E_ARG; }
  if (n >= ST_NONE) { set_err(c, "%s: a claim of 2^32 - 1 edges or more", who); return TGI_E_ARG; }
  std::vector<int64_t> ids(n);
  for (uint64_t j = 0; j < n; j++) {
    const tgi_pending_claim_edge& E = in->edges[j];
    for (int f = 0; f < 3; f++)
      if (E.str_off[f] > sl || E.str_len[f] > sl - E.str_off[f]) {
        set_err(c, "%s: edge %llu string %d outside strs", who, (unsigned long long)j, f);
        return TGI_E_ARG;
      }
    const uint32_t dl = E.str_len[TGI_VE_DESTINATION];
    if (dl < 1 || dl > 32) { set_err(c, "%s: edge %llu has a destination of %u bytes (1 to 32)", who, (unsigned long long)j, dl); return TGI_E_ARG; }
    ids[j] = E.pending_id;
  }
  std::sort(ids.begin(), ids.end());
  const auto d = std::adjacent_find(ids.begin(), ids.end());
  if (d != ids.end()) { set_err(c, "%s: pending_id %lld twice in the claim", who, (long long)*d); return TGI_E_ARG; }
  return TGI_OK;
}

// The outcomes' checks (TGI_E_ARG) against the plan's lookup rows L; aoff[l] = row l's first attempt
int ve_outcomes(tgi_ctx* c, const tgi_validator_lookup* L, const tgi_validator_outcome* oc, uint64_t n,
                const tgi_validator_attempt* at, uint64_t n_at, uint64_t* aoff, const char* who) {
  uint64_t a = 0;
  auto bad = [&](uint64_t l, const char* what) {
    set_err(c, "%s: lookup %llu: %s", who, (unsigned long long)l, what);
    return TGI_E_ARG;
  };
  auto final_kind = [](uint32_t k) { return k == TGI_VA_VALID || k == TGI_VA_NOT_CHANNEL || k == TGI_VA_INVALID; };
  for (uint64_t l = 0; l < n; l++) {
    const tgi_validator_outcome& o = oc[l];
    const uint32_t na = o.n_attempts;
    if (o.discovered > 1 || o.claimed > 1) return bad(l, "discovered or claimed past 1");
    if (na > n_at - a) return bad(l, "more attempts than n_attempts holds");
    aoff[l] = a;
    if (o.discovered && na) return bad(l, "discovered with attempts");
    if (!o.discovered && (!na || na > L[l].m)) return bad(l, "no attempt, or more attempts than occurrences");
    for (uint32_t q = 0; q < na; q++) {
      const tgi_validator_attempt& t = at[a + q];
      if (t.kind > TGI_VA_BLOCKED || t.reason > TGI_VR_NOT_FOUND) return bad(l, "an unknown attempt kind or reason");
      if (final_kind(t.kind) && q + 1 < na) return bad(l, "a final attempt before the last one");
    }
    const bool last_final = na && final_kind(at[a + na - 1].kind);
    if (na && !last_final && na < L[l].m) return bad(l, "a last attempt that is not final while fewer than m were made");
    if (o.claimed && !(na && at[a + na - 1].kind == TGI_VA_VALID)) return bad(l, "claimed without a final VALID");
    a += na;
  }
  if (a != n_at) { set_err(c, "%s: the rows make %llu attempts, n_attempts is %llu", who, (unsigned long long)a, (unsigned long long)n_at); return TGI_E_ARG; }
  return TGI_OK;
}

}  // namespace

extern "C" {

int tgi_state_id_seed(tgi_ctx* c, uint64_t seed) {
  if (!c) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  S.id_seed = seed;
  S.seeded = true;
  return TGI_OK;
}

// The candidates of the spans gathered from the slot's resident result (a thread per processed link row, a scan, the
// compaction), then either appended to the pending list or deduplicated per span, tested against the urlCache and read
// back as survivors for the AddLayers.  Lock order: the slot, then the state (as tgi_state_page_end); the slot's lock is
// held until the kernels that read its result have finished.
int tgi_state_discover(tgi_ctx* c, int slot, const tgi_state_span* spans, uint32_t n_spans, uint32_t flags, int64_t now_sec,
                       int32_t now_nsec, int64_t max_pages, tgi_state_added_t* out) {
  static const char* const who = "tgi_state_discover";
  if (!c || !out || (n_spans && !spans)) return TGI_E_ARG;
  if (slot < 0 || slot >= TGI_SLOTS) { set_err(c, "%s: bad slot %d", who, slot); return TGI_E_ARG; }
  Slot& s = c->slots[slot];
  std::lock_guard<std::mutex> sl(s.mu);
  int rc;
  if ((rc = disc_slot(c, s, slot, who))) return rc;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  if ((rc = st_init(c, S))) return rc;
  memset(out, 0, sizeof *out);
  if ((rc = disc_args(c, flags, TGI_DISCOVER_NOW | TGI_DISCOVER_DAPR | TGI_DISCOVER_PAGE_JSON, now_sec, now_nsec, who))) return rc;
  if ((flags & TGI_DISCOVER_PAGE_JSON) && (rc = disc_json_empty(c, S, out))) return rc;
  uint64_t bound = 0;
  if ((rc = disc_bound(c, S, s, spans, n_spans, who, &bound))) return rc;
  const bool now = flags & TGI_DISCOVER_NOW, dapr = flags & TGI_DISCOVER_DAPR, json = flags & TGI_DISCOVER_PAGE_JSON;
  if (!bound) return TGI_OK;  // no candidate: no AddLayer call, nothing pending
  if (!now && (rc = st_grow(c, S, S.pend, S.n_pend * sizeof(StCand), (S.n_pend + bound) * sizeof(StCand)))) return rc;
  cudaStream_t st = S.stream;
  if (now) CK(S.cand.ensure(bound * sizeof(StCand)));
  CK(S.h_coff.ensure((n_spans + 1) * 8));
  StDisc gd;
  uint32_t launches = 0;
  float ms = 0;
  if ((rc = disc_gather(c, S, s, spans, n_spans, bound, now ? S.cand.as<StCand>() : S.pend.as<StCand>() + S.n_pend, false,
                        gd, launches))) return rc;
  CK(cudaEventRecord(S.t1, st));
  CK(cudaMemcpyAsync(S.h_coff.p, gd.coff, (n_spans + 1) * 8, cudaMemcpyDeviceToHost, st));
  const uint64_t* coff = S.h_coff.as<uint64_t>();
  if (!now) {
    CK(cudaStreamSynchronize(st));
    cudaEventElapsedTime(&ms, S.t0, S.t1);
    S.n_pend += coff[n_spans];
    out->n_candidates = coff[n_spans];
    out->kernel_ms = ms;
    out->gpu_launches = launches;
    return TGI_OK;
  }
  // per span: first occurrences under Base's rules (none under Dapr's) and Dapr's urlCache test
  uint64_t n_surv = 0;
  if ((rc = st_survivors(c, S, S.cand.as<StCand>(), gd.coff + n_spans, bound, true, !dapr, dapr, &n_surv, &ms, launches))) return rc;
  float gather_ms = 0;
  cudaEventElapsedTime(&gather_ms, S.t0, S.t1);
  ms += gather_ms;
  const StCand* sv = S.h_surv.as<StCand>();
  std::vector<DiscGroup> G(n_spans);
  uint64_t j = 0;
  for (uint32_t k = 0; k < n_spans; k++) {
    G[k].depth = S.rows[spans[k].row].depth + 1;
    G[k].any = coff[k + 1] > coff[k];
    G[k].s0 = j;
    while (j < n_surv && sv[j].span == k) j++;
    G[k].s1 = j;
  }
  out->n_candidates = coff[n_spans];
  if ((rc = st_discover_apply(c, S, G, dapr, json, now_sec, now_nsec, max_pages, who, out, &ms, launches))) {
    out->n_candidates = 0;
    return rc;
  }
  out->kernel_ms = ms;
  out->gpu_launches = launches;
  return TGI_OK;
}

// The layer end of dapr/standalone.go:647-688 over the pending list: first occurrences over the whole list, Dapr's
// urlCache test, the survivors read back for one AddLayer at layer_depth + 1; the list is emptied once it applied.
int tgi_state_next_layer(tgi_ctx* c, int64_t layer_depth, uint32_t flags, int64_t now_sec, int32_t now_nsec,
                         int64_t max_pages, tgi_state_added_t* out) {
  static const char* const who = "tgi_state_next_layer";
  if (!c || !out) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  memset(out, 0, sizeof *out);
  if ((rc = disc_args(c, flags, TGI_DISCOVER_DAPR | TGI_DISCOVER_PAGE_JSON, now_sec, now_nsec, who))) return rc;
  if ((flags & TGI_DISCOVER_PAGE_JSON) && (rc = disc_json_empty(c, S, out))) return rc;
  if (!S.n_pend) return TGI_OK;
  const bool dapr = flags & TGI_DISCOVER_DAPR, json = flags & TGI_DISCOVER_PAGE_JSON;
  const uint64_t m = S.n_pend;
  cudaStream_t st = S.stream;
  CK(S.h_coff.ensure(8));
  CK(S.coff.ensure(8));
  *S.h_coff.as<uint64_t>() = m;
  CK(cudaMemcpyAsync(S.coff.p, S.h_coff.p, 8, cudaMemcpyHostToDevice, st));
  uint32_t launches = 0;
  float ms = 0;
  uint64_t n_surv = 0;
  if ((rc = st_survivors(c, S, S.pend.as<StCand>(), S.coff.as<uint64_t>(), m, false, true, dapr, &n_surv, &ms, launches))) return rc;
  const std::vector<DiscGroup> G(1, DiscGroup{layer_depth + 1, true, 0, n_surv});
  if ((rc = st_discover_apply(c, S, G, dapr, json, now_sec, now_nsec, max_pages, who, out, &ms, launches))) return rc;
  S.n_pend = 0;
  out->n_candidates = m;
  out->kernel_ms = ms;
  out->gpu_launches = launches;
  return TGI_OK;
}

// The discovery gather, st_first_kernel per span (seenInBatch), the name tests and the keep scan, the per-span batch
// scan and one kernel for the edges and batches; one synchronise for the totals, one for the read-back.  Lock order: the
// slot, then the state, then the sets.
int tgi_state_pending_edges(tgi_ctx* c, int slot, const tgi_state_span* spans, uint32_t n_spans, int64_t now_sec,
                            tgi_state_edges_t* out) {
  static const char* const who = "tgi_state_pending_edges";
  if (!c || !out || (n_spans && !spans)) return TGI_E_ARG;
  if (slot < 0 || slot >= TGI_SLOTS) { set_err(c, "%s: bad slot %d", who, slot); return TGI_E_ARG; }
  Slot& s = c->slots[slot];
  std::lock_guard<std::mutex> sl(s.mu);
  int rc;
  if ((rc = disc_slot(c, s, slot, who))) return rc;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  if ((rc = st_init(c, S))) return rc;
  memset(out, 0, sizeof *out);
  uint64_t bound = 0;
  if ((rc = disc_bound(c, S, s, spans, n_spans, who, &bound))) return rc;
  CK(S.h_span_batch.ensure(std::max<uint64_t>(n_spans, 1) * 4));
  out->span_batch = S.h_span_batch.as<uint32_t>();
  if (!bound) {  // no processed link row: no edge, no batch
    std::fill_n(S.h_span_batch.as<uint32_t>(), n_spans, TGI_STATE_NO_BATCH);
    S.handoff_live = true;
    S.handoff_ne = S.handoff_nb = 0;
    handoff_walkbacks(S, spans, n_spans);
    return TGI_OK;
  }
  cudaStream_t st = S.stream;
  const bool tiled = n_spans > 1;  // launches that do not depend on the number of pages
  const uint64_t bslots = next_pow2(std::max<uint64_t>(2 * bound, 64));
  CK(S.cand.ensure(bound * sizeof(StCand)));
  CK(S.bfirst.ensure(bslots * 4));
  CK(S.slot_of.ensure(bound * 4));
  CK(S.clink.ensure(bound * 4));
  CK(S.edges.ensure(bound * sizeof(tgi_state_edge)));
  CK(S.ebatches.ensure(n_spans * sizeof(tgi_state_edge_batch)));
  CK(S.span_batch.ensure(n_spans * 4));
  CK(S.h_sc.ensure(ST_SC_COUNT * 8));
  StDisc gd;
  uint32_t launches = 0;
  if ((rc = disc_gather(c, S, s, spans, n_spans, bound, S.cand.as<StCand>(), tiled, gd, launches))) return rc;
  st_edge_link_kernel<<<st_grid(c, bound), ST_THREADS, 0, st>>>(gd, S.clink.as<uint32_t>());
  launches++;
  // seenInBatch: the first occurrence of every name within its span
  StFirst w{};
  w.c = S.cand.as<StCand>();
  w.n = gd.coff + n_spans;
  w.bound = bound;
  w.per_span = true;
  w.dedup = true;
  w.bfirst = S.bfirst.as<uint32_t>();
  w.bmask = bslots - 1;
  w.slot_of = S.slot_of.as<uint32_t>();
  CK(cudaMemsetAsync(w.bfirst, 0xFF, bslots * 4, st));
  st_first_kernel<<<st_grid(c, bound), ST_THREADS, 0, st>>>(w);
  launches++;
  // the gather is done with its flags, offsets and counts: the edges' keep flags and scans reuse them
  uint64_t* dsc = S.sc.as<uint64_t>();  // [3] candidates, [4] edges, [5] batches
  StEdges e{};
  e.c = S.cand.as<StCand>();
  e.link = S.clink.as<uint32_t>();
  e.coff = gd.coff;
  e.bound = bound;
  e.bfirst = w.bfirst;
  e.slot_of = w.slot_of;
  e.spans = gd.spans;
  e.n_spans = n_spans;
  e.link_off = gd.link_off;
  e.links = gd.links;
  e.n_cand = (unsigned long long*)(dsc + 3);
  e.flag = gd.flag;
  e.pos = gd.pos;
  e.has = S.cnt.as<uint32_t>();
  e.bpos = S.soff.as<uint64_t>();
  e.seed = S.id_seed;
  e.batch0 = S.batch_next;
  e.edges = S.edges.as<tgi_state_edge>();
  e.batches = S.ebatches.as<tgi_state_edge_batch>();
  e.span_batch = S.span_batch.as<uint32_t>();
  CK(cudaMemsetAsync(dsc + 3, 0, 8, st));
  {
    std::lock_guard<std::mutex> fg(c->fr_mu);  // the exclusion sets: probed by the kernels below, not changed
    if (c->fr_event_valid) CK(cudaStreamWaitEvent(st, c->fr_event, 0));
    e.x = exclusion(c, now_sec);
    st_edge_keep_kernel<<<st_grid(c, bound), ST_THREADS, 0, st>>>(e);
    launches++;
    if ((rc = launch_scan(c, st, S.tiles, e.flag, bound, e.pos, dsc + 4, launches, tiled))) return rc;
    st_edge_spans_kernel<<<st_grid(c, n_spans), ST_THREADS, 0, st>>>(e);
    launches++;
    if ((rc = launch_scan(c, st, S.tiles, e.has, n_spans, e.bpos, dsc + 5, launches, tiled))) return rc;
    st_edge_emit_kernel<<<st_grid(c, std::max<uint64_t>(bound, n_spans)), ST_THREADS, 0, st>>>(e);
    launches++;
    CK(cudaGetLastError());
    CK(cudaEventRecord(S.t1, st));
    CK(cudaMemcpyAsync(S.h_sc.p, S.sc.p, ST_SC_COUNT * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  const uint64_t* hs = S.h_sc.as<uint64_t>();
  const uint64_t n_edges = hs[4], n_batches = hs[5];
  if (n_batches && !S.seeded) { set_err(c, "%s: no id seed (tgi_state_id_seed)", who); return TGI_E_STATE; }
  float ms = 0;
  cudaEventElapsedTime(&ms, S.t0, S.t1);
  CK(S.h_edges.ensure(std::max<uint64_t>(n_edges, 1) * sizeof(tgi_state_edge)));
  CK(S.h_ebatches.ensure(std::max<uint64_t>(n_batches, 1) * sizeof(tgi_state_edge_batch)));
  if (n_edges) CK(cudaMemcpyAsync(S.h_edges.p, S.edges.p, n_edges * sizeof(tgi_state_edge), cudaMemcpyDeviceToHost, st));
  if (n_batches) CK(cudaMemcpyAsync(S.h_ebatches.p, S.ebatches.p, n_batches * sizeof(tgi_state_edge_batch), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(S.h_span_batch.p, S.span_batch.p, n_spans * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  S.batch_next += n_batches;
  S.handoff_live = true;  // S.edges, S.ebatches and S.spans hold it until the next state call
  S.handoff_ne = n_edges;
  S.handoff_nb = n_batches;
  handoff_walkbacks(S, spans, n_spans);
  out->n_candidates = hs[3];
  out->n_edges = n_edges;
  out->n_batches = (uint32_t)n_batches;
  out->edges = S.h_edges.as<tgi_state_edge>();
  out->batches = S.h_ebatches.as<tgi_state_edge_batch>();
  out->kernel_ms = ms;
  out->gpu_launches = launches;
  return TGI_OK;
}

// The binding calls of the last hand-off: the texts on the host (one per kind and row count), the params on the device
// (a thread per row sizes it, a scan, a thread per row writes it and the emit also fills the statement table); one
// synchronise for the params' length, one for the read-back
int tgi_state_edge_sql(tgi_ctx* c, const char* crawl_id, uint32_t crawl_id_len, int64_t now_sec, int32_t now_nsec,
                       uint32_t rows_per_stmt, tgi_state_edge_sql_t* out) {
  static const char* const who = "tgi_state_edge_sql";
  if (!c || !out) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  cudaSetDevice(c->device);  // not st_init: that would end the hand-off
  S.rw_live = false;
  int rc;
  if ((rc = sql_args(c, S, rows_per_stmt, now_nsec, crawl_id, crawl_id_len, who))) return rc;
  const uint64_t nb = S.handoff_nb, ne = S.handoff_ne;
  char tb[48];
  uint32_t tl = 0;
  if (ne && (rc = sql_clock(c, now_sec, now_nsec, who, tb, &tl))) return rc;
  memset(out, 0, sizeof *out);
  if (!nb) return TGI_OK;
  StSql q{};
  std::iota(q.p.kind, q.p.kind + ST_SQL_KINDS, (uint32_t)TGI_SQL_BATCH_INSERT);
  std::fill_n(q.p.k, 3, rows_per_stmt);
  q.p.rows[0] = q.p.rows[2] = nb;
  q.p.rows[1] = ne;
  q.edges = S.edges.as<tgi_state_edge>();
  q.batches = S.ebatches.as<tgi_state_edge_batch>();
  q.spans = S.spans.as<tgi_state_span>();
  return sql_render(c, S, q, st_sql_size_kernel, st_sql_emit_kernel, 2 * nb + ne, crawl_id, crawl_id_len, tb, tl, who, [] {},
                    S.h_sql, S.h_sql_stmts, out);
}

// The forced walkbacks of the last hand-off.  The first call on a hand-off picks (a thread per edge-less span, a scan
// that ranks the usable ones, one synchronise for the picks and their count); every call renders the rows as
// tgi_state_edge_sql does (a thread per row sizes it, a scan, a thread per row writes it and the statement table; one
// synchronise for the params' length, one for the read-back)
int tgi_state_walkback(tgi_ctx* c, const char* crawl_id, uint32_t crawl_id_len, int64_t now_sec, int32_t now_nsec,
                       uint32_t rows_per_stmt, tgi_state_walkback_t* out) {
  static const char* const who = "tgi_state_walkback";
  if (!c || !out) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  cudaSetDevice(c->device);  // not st_init: that would end the hand-off
  S.rw_live = false;
  int rc;
  if ((rc = sql_args(c, S, rows_per_stmt, now_nsec, crawl_id, crawl_id_len, who))) return rc;
  const uint64_t n = S.wb_spans.size() / 2;
  if (!n) {  // every span has a batch: nothing to pick, no launch
    memset(out, 0, sizeof *out);
    return TGI_OK;
  }
  if (!S.seeded) { set_err(c, "%s: no id seed (tgi_state_id_seed)", who); return TGI_E_STATE; }
  cudaStream_t st = S.stream;
  uint32_t launches = 0;
  float ms = 0;
  uint64_t n_ok = S.wb_n_ok;
  if (!S.wb_picked) {  // the hand-off's picks: made here, kept only once the call is accepted
    CK(S.wb_in.ensure(n * 8));
    CK(S.wb.ensure(n * sizeof(tgi_state_walkback_span)));
    CK(S.wb_ok.ensure(n * 4));
    CK(S.wb_rank.ensure((n + 1) * 8));
    CK(S.sc.ensure(ST_SC_COUNT * 8));
    CK(S.h_sc.ensure(ST_SC_COUNT * 8));
    CK(S.h_wb.ensure(n * sizeof(tgi_state_walkback_span)));
    CK(cudaMemcpyAsync(S.wb_in.p, S.wb_spans.data(), n * 8, cudaMemcpyHostToDevice, st));
    StWalk w{};
    w.spans = S.wb_in.as<uint32_t>();
    w.n = n;
    w.seed = S.id_seed;
    w.w0 = S.walk_next;
    w.out = S.wb.as<tgi_state_walkback_span>();
    w.ok = S.wb_ok.as<uint32_t>();
    {
      std::lock_guard<std::mutex> fg(c->fr_mu);  // the discovered set: read by the pick, not changed
      if (c->fr_event_valid) CK(cudaStreamWaitEvent(st, c->fr_event, 0));
      w.disc = c->sets[TGI_SET_DISCOVERED].dev;
      CK(cudaEventRecord(S.t0, st));
      st_walk_pick_kernel<<<sink_grid(c, n, ST_THREADS, 4), ST_THREADS, 0, st>>>(st_dev(S), w);
      launches++;
      if ((rc = launch_scan(c, st, S.tiles, w.ok, n, S.wb_rank.as<uint64_t>(), S.sc.as<uint64_t>() + ST_SC_ROWS, launches))) return rc;
      CK(cudaGetLastError());
      CK(cudaEventRecord(S.t1, st));
      CK(cudaMemcpyAsync(S.h_sc.p, S.sc.p, ST_SC_COUNT * 8, cudaMemcpyDeviceToHost, st));
      CK(cudaMemcpyAsync(S.h_wb.p, w.out, n * sizeof(tgi_state_walkback_span), cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
    }
    cudaEventElapsedTime(&ms, S.t0, S.t1);
    n_ok = S.h_sc.as<uint64_t>()[ST_SC_ROWS];
  }
  char tb[48];
  uint32_t tl = 0;
  if (n_ok && (rc = sql_clock(c, now_sec, now_nsec, who, tb, &tl))) return rc;
  auto accept = [&]() {  // the picks are kept once the call is accepted: a refused first call picks the same again
    if (S.wb_picked) return;
    S.wb_picked = true;
    S.wb_n_ok = n_ok;
    S.walk_next += n;
  };
  memset(out, 0, sizeof *out);
  out->n_walkbacks = (uint32_t)n;
  out->walkbacks = S.h_wb.as<tgi_state_walkback_span>();
  out->kernel_ms = ms;
  out->gpu_launches = launches;
  if (!n_ok) {
    accept();
    return TGI_OK;
  }
  StWalkSql q{};
  std::iota(q.p.kind, q.p.kind + ST_SQL_KINDS, (uint32_t)TGI_SQL_PAGE_BUFFER_INSERT);
  std::fill_n(q.p.k, 2, rows_per_stmt);
  q.p.rows[0] = q.p.rows[1] = n_ok;
  q.spans = S.wb_in.as<uint32_t>();
  q.wb = S.wb.as<tgi_state_walkback_span>();
  q.rank = S.wb_rank.as<uint64_t>();
  q.n = n;
  return sql_render(c, S, q, st_walk_size_kernel, st_walk_emit_kernel, 2 * n, crawl_id, crawl_id_len, tb, tl, who, accept,
                    S.h_wb_sql, S.h_wb_stmts, out);
}

// processWalkbackBatch for every claimed batch: the upload, a thread per batch decides and picks, three scans place its
// rows (one synchronise for the outcomes and totals), then the rows as tgi_state_edge_sql renders them (a thread per row
// sizes it, a scan, a thread per row writes it and the statement table; one synchronise for the params' length, one
// for the read-back)
int tgi_state_validator_walkback(tgi_ctx* c, const tgi_claimed_batches* in, int64_t walkback_rate, const char* crawl_id,
                                 uint32_t crawl_id_len, int64_t now_sec, int32_t now_nsec, uint32_t rows_per_stmt,
                                 tgi_state_validator_walkback_t* out) {
  static const char* const who = "tgi_state_validator_walkback";
  if (!c || !out || !in) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;  // a state call: a live hand-off ends here
  if ((rc = sql_args(c, S, rows_per_stmt, now_nsec, crawl_id, crawl_id_len, who, false))) return rc;
  if ((rc = vw_input(c, in, who))) return rc;
  const uint64_t n = in->n_batches, ne = in->n_edges;
  if (!n) {
    memset(out, 0, sizeof *out);
    return TGI_OK;
  }
  if (!S.seeded) { set_err(c, "%s: no id seed (tgi_state_id_seed)", who); return TGI_E_STATE; }
  cudaStream_t st = S.stream;
  CK(S.vw_b.ensure(n * sizeof(tgi_claimed_batch)));
  CK(S.vw_eoff.ensure((n + 1) * 8));
  CK(S.vw_e.ensure(ne * sizeof(tgi_claimed_edge)));
  CK(S.vw_s.ensure(in->strs_len));
  CK(S.vw_out.ensure(n * sizeof(tgi_state_validator_batch)));
  CK(S.vw_list.ensure(2 * ne * 4));
  CK(S.vw_cnt.ensure(3 * n * 4));
  CK(S.vw_rank.ensure(3 * (n + 1) * 8));
  CK(S.sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_vw.ensure(n * sizeof(tgi_state_validator_batch)));
  CK(cudaMemcpyAsync(S.vw_b.p, in->batches, n * sizeof(tgi_claimed_batch), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(S.vw_eoff.p, in->edge_off, (n + 1) * 8, cudaMemcpyHostToDevice, st));
  if (ne) CK(cudaMemcpyAsync(S.vw_e.p, in->edges, ne * sizeof(tgi_claimed_edge), cudaMemcpyHostToDevice, st));
  if (in->strs_len) CK(cudaMemcpyAsync(S.vw_s.p, in->strs, in->strs_len, cudaMemcpyHostToDevice, st));
  StVw v{};
  v.b = S.vw_b.as<tgi_claimed_batch>();
  v.eoff = S.vw_eoff.as<uint64_t>();
  v.e = S.vw_e.as<tgi_claimed_edge>();
  v.s = S.vw_s.as<uint8_t>();
  v.n = n;
  v.rate = walkback_rate;
  v.seed = S.id_seed;
  v.v0 = S.vw_next;
  v.out = S.vw_out.as<tgi_state_validator_batch>();
  v.vlist = S.vw_list.as<uint32_t>();
  v.tlist = v.vlist + ne;
  v.cnt = S.vw_cnt.as<uint32_t>();
  uint64_t* rank = S.vw_rank.as<uint64_t>();
  uint64_t* dsc = S.sc.as<uint64_t>();  // [ST_SC_ROWS] OK batches, [ST_SC_BYTES] edge rows, [ST_SC_SLOTS] stats rows
  static const int tot[3] = {ST_SC_ROWS, ST_SC_BYTES, ST_SC_SLOTS};
  uint32_t launches = 0;
  {
    std::lock_guard<std::mutex> fg(c->fr_mu);  // the discovered set: read by the pick, not changed
    if (c->fr_event_valid) CK(cudaStreamWaitEvent(st, c->fr_event, 0));
    v.disc = c->sets[TGI_SET_DISCOVERED].dev;
    CK(cudaEventRecord(S.t0, st));
    st_vw_pick_kernel<<<sink_grid(c, n, ST_THREADS, 4), ST_THREADS, 0, st>>>(v);
    launches++;
    for (int k = 0; k < 3; k++)
      if ((rc = launch_scan(c, st, S.tiles, v.cnt + k * n, n, rank + k * (n + 1), dsc + tot[k], launches))) return rc;
    CK(cudaGetLastError());
    CK(cudaEventRecord(S.t1, st));
    CK(cudaMemcpyAsync(S.h_sc.p, S.sc.p, ST_SC_COUNT * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(S.h_vw.p, v.out, n * sizeof(tgi_state_validator_batch), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  float ms = 0;
  cudaEventElapsedTime(&ms, S.t0, S.t1);
  const uint64_t* hs = S.h_sc.as<uint64_t>();
  const uint64_t n_ok = hs[ST_SC_ROWS], n_edge_rows = hs[ST_SC_BYTES], n_stats = hs[ST_SC_SLOTS];
  char tb[48];
  uint32_t tl = 0;
  if (n_ok && (rc = sql_clock(c, now_sec, now_nsec, who, tb, &tl))) return rc;
  auto accept = [&]() { S.vw_next += n; };  // a refused call leaves v where it was
  memset(out, 0, sizeof *out);
  out->n_batches = (uint32_t)n;
  out->batches = S.h_vw.as<tgi_state_validator_batch>();
  out->kernel_ms = ms;
  out->gpu_launches = launches;
  if (!n_ok) {
    accept();
    return TGI_OK;
  }
  StVwSql q{};
  std::iota(q.p.kind, q.p.kind + ST_SQL_KINDS, (uint32_t)TGI_SQL_PAGE_BUFFER_INSERT);
  const uint64_t rows[5] = {n_ok, n_edge_rows, n_ok, n_stats, n_ok};
  for (int k = 0; k < 5; k++) {
    q.p.rows[k] = rows[k];
    q.p.k[k] = k == TGI_SQL_STATS_UPSERT - TGI_SQL_PAGE_BUFFER_INSERT ? 1u : rows_per_stmt;  // upserts: one row each
  }
  q.v = v;
  q.rank = rank;
  return sql_render(c, S, q, st_vw_size_kernel, st_vw_emit_kernel, 3 * n_ok + n_edge_rows + n_stats, crawl_id,
                    crawl_id_len, tb, tl, who, accept, S.h_vw_sql, S.h_vw_stmts, out);
}

// The standard random walk's lookups: the discovery gather, st_first_kernel over the call, the classes under the
// three sets, a scan and the lookup rows; one synchronise for the totals, one for the read-back.  Lock order: the
// slot, then the state, then the sets.
int tgi_state_rw_lookups(tgi_ctx* c, int slot, const tgi_state_span* spans, uint32_t n_spans, int64_t now_sec,
                         tgi_state_rw_lookups_t* out) {
  static const char* const who = "tgi_state_rw_lookups";
  if (!c || !out || (n_spans && !spans)) return TGI_E_ARG;
  if (slot < 0 || slot >= TGI_SLOTS) { set_err(c, "%s: bad slot %d", who, slot); return TGI_E_ARG; }
  Slot& s = c->slots[slot];
  std::lock_guard<std::mutex> sl(s.mu);
  int rc;
  if ((rc = disc_slot(c, s, slot, who))) return rc;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  if ((rc = st_init(c, S))) return rc;
  memset(out, 0, sizeof *out);
  uint64_t bound = 0;
  if ((rc = disc_bound(c, S, s, spans, n_spans, who, &bound))) return rc;
  CK(S.h_rw_cand.ensure(std::max<uint64_t>(n_spans, 1) * 8));
  out->span_candidates = S.h_rw_cand.as<uint64_t>();
  S.rw_n_spans = n_spans;
  S.rw_n_cand = S.rw_n_lk = 0;
  if (!n_spans) {
    S.rw_live = true;
    return TGI_OK;
  }
  bound = std::max<uint64_t>(bound, 1);  // the step reads the spans and their (empty) offsets from the gather
  cudaStream_t st = S.stream;
  const bool tiled = n_spans > 1;  // launches that do not depend on the number of pages
  const uint64_t bslots = next_pow2(std::max<uint64_t>(2 * bound, 64));
  CK(S.cand.ensure(bound * sizeof(StCand)));
  CK(S.bfirst.ensure(bslots * 4));
  CK(S.slot_of.ensure(bound * 4));
  CK(S.clink.ensure(bound * 4));
  CK(S.rw_cls.ensure(bound * 4));
  CK(S.rw_lpos.ensure((bound + 1) * 8));
  CK(S.rw_lk.ensure(bound * sizeof(tgi_rw_lookup)));
  CK(S.h_sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_coff.ensure((n_spans + 1) * 8));
  StDisc gd;
  uint32_t launches = 0;
  if ((rc = disc_gather(c, S, s, spans, n_spans, bound, S.cand.as<StCand>(), tiled, gd, launches))) return rc;
  st_edge_link_kernel<<<st_grid(c, bound), ST_THREADS, 0, st>>>(gd, S.clink.as<uint32_t>());
  launches++;
  // the first candidate of every name over the whole call
  StFirst w{};
  w.c = S.cand.as<StCand>();
  w.n = gd.coff + n_spans;
  w.bound = bound;
  w.dedup = true;
  w.bfirst = S.bfirst.as<uint32_t>();
  w.bmask = bslots - 1;
  w.slot_of = S.slot_of.as<uint32_t>();
  CK(cudaMemsetAsync(w.bfirst, 0xFF, bslots * 4, st));
  st_first_kernel<<<st_grid(c, bound), ST_THREADS, 0, st>>>(w);
  launches++;
  StRw r{};  // the gather is done with its flags: the lookups' flags reuse them
  r.c = w.c;
  r.link = S.clink.as<uint32_t>();
  r.coff = gd.coff;
  r.bound = bound;
  r.bfirst = w.bfirst;
  r.slot_of = w.slot_of;
  r.spans = gd.spans;
  r.n_spans = n_spans;
  r.link_off = gd.link_off;
  r.links = gd.links;
  r.cls = S.rw_cls.as<uint32_t>();
  r.flag = gd.flag;
  r.pos = S.rw_lpos.as<uint64_t>();
  r.out = S.rw_lk.as<tgi_rw_lookup>();
  uint64_t* dsc = S.sc.as<uint64_t>();  // [3] lookups
  {
    std::lock_guard<std::mutex> fg(c->fr_mu);  // the three sets: probed by the kernels below, not changed
    if (c->fr_event_valid) CK(cudaStreamWaitEvent(st, c->fr_event, 0));
    r.x = exclusion(c, now_sec);
    r.seeds = c->sets[TGI_SET_SEEDS].dev;
    st_rw_class_kernel<<<st_grid(c, bound), ST_THREADS, 0, st>>>(r);
    launches++;
    if ((rc = launch_scan(c, st, S.tiles, r.flag, bound, r.pos, dsc + 3, launches, tiled))) return rc;
    st_rw_lookup_kernel<<<st_grid(c, bound), ST_THREADS, 0, st>>>(r);
    launches++;
    CK(cudaGetLastError());
    CK(cudaEventRecord(S.t1, st));
    CK(cudaMemcpyAsync(S.h_sc.p, S.sc.p, ST_SC_COUNT * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(S.h_coff.p, gd.coff, (n_spans + 1) * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  const uint64_t nl = S.h_sc.as<uint64_t>()[3];
  const uint64_t* coff = S.h_coff.as<uint64_t>();
  float ms = 0;
  cudaEventElapsedTime(&ms, S.t0, S.t1);
  CK(S.h_rw_lk.ensure(std::max<uint64_t>(nl, 1) * sizeof(tgi_rw_lookup)));
  if (nl) {
    CK(cudaMemcpyAsync(S.h_rw_lk.p, r.out, nl * sizeof(tgi_rw_lookup), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  for (uint32_t k = 0; k < n_spans; k++) S.h_rw_cand.as<uint64_t>()[k] = coff[k + 1] - coff[k];
  S.rw_live = true;  // cand, coff, spans, rw_cls, rw_lpos and rw_lk hold the lists until the next state call
  S.rw_n_cand = coff[n_spans];
  S.rw_n_lk = nl;
  out->n_candidates = coff[n_spans];
  out->n_lookups = nl;
  out->lookups = S.h_rw_lk.as<tgi_rw_lookup>();
  out->kernel_ms = ms;
  out->gpu_launches = launches;
  return TGI_OK;
}

// The standard random walk's step over the last lookups' lists: the outcomes' checks and the retire point on the host;
// a thread per lookup and candidate flags the effects, three scans, one compaction (one synchronise); the three ordered
// set inserts on the sets' stream; a thread per span decides and picks over the discovered set as the replay leaves it,
// two scans place its rows (one synchronise); then the rows as tgi_state_edge_sql renders them.
int tgi_state_rw_step(tgi_ctx* c, const tgi_rw_outcome* outcomes, uint64_t n_outcomes, int64_t walkback_rate,
                      const char* crawl_id, uint32_t crawl_id_len, int64_t now_sec, int32_t now_nsec,
                      uint32_t rows_per_stmt, tgi_state_rw_step_t* out) {
  static const char* const who = "tgi_state_rw_step";
  if (!c || !out) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  cudaSetDevice(c->device);  // not st_init: that would end the lists this call reads
  S.handoff_live = false;    // a state call: a live tandem hand-off ends here
  int rc;
  if ((rc = sql_args(c, S, rows_per_stmt, now_nsec, crawl_id, crawl_id_len, who, false))) return rc;
  if (!S.rw_live) { set_err(c, "%s: no lookups (tgi_state_rw_lookups, then no other state call)", who); return TGI_E_STATE; }
  const uint64_t n = S.rw_n_lk, nc = S.rw_n_cand;
  const uint32_t n_spans = S.rw_n_spans;
  if (n_outcomes != n) { set_err(c, "%s: %llu outcomes for %llu lookups", who, (unsigned long long)n_outcomes, (unsigned long long)n); return TGI_E_ARG; }
  if (n && !outcomes) { set_err(c, "%s: outcomes is NULL", who); return TGI_E_ARG; }
  uint64_t nl = n;  // the lookups that apply: those before the first retire
  for (uint64_t q = 0; q < n; q++) {
    if (outcomes[q].code > TGI_RW_RETIRE) { set_err(c, "%s: outcome %llu has code %u", who, (unsigned long long)q, outcomes[q].code); return TGI_E_ARG; }
    if (outcomes[q].code == TGI_RW_RETIRE && nl == n) nl = q;
  }
  const tgi_rw_lookup* L = S.h_rw_lk.as<tgi_rw_lookup>();
  const uint32_t n_dec = nl < n ? L[nl].span : n_spans;  // the deciding spans; span n_dec retired
  if (n_dec && !S.seeded) { set_err(c, "%s: no id seed (tgi_state_id_seed)", who); return TGI_E_STATE; }
  char tb[48];
  uint32_t tl = 0;
  if (n_dec && (rc = sql_clock(c, now_sec, now_nsec, who, tb, &tl))) return rc;
  memset(out, 0, sizeof *out);
  for (uint64_t q = 0; q < nl; q++) {  // lookupStats.record
    const uint32_t src = L[q].source_type & 3;
    if (outcomes[q].code == TGI_RW_FOUND) out->hits[src]++;
    else out->misses[src]++;
  }
  out->n_spans = n_spans;
  if (!n_spans) {
    S.rw_live = false;
    return TGI_OK;
  }
  cudaStream_t st = S.stream;
  CK(S.rw_oc.ensure(std::max<uint64_t>(n, 1) * sizeof(tgi_rw_outcome)));
  CK(S.rw_flag.ensure((2 * nl + nc + 1) * 4));
  CK(S.rw_pos.ensure((2 * (nl + 1) + nc + 1) * 8));
  CK(S.rw_list.ensure((2 * nl + 1) * 4));
  CK(S.rw_keys.ensure((2 * nl + nc + 1) * 32));
  CK(S.rw_new.ensure(nc + 1));
  CK(S.rw_nflag.ensure((nc + 1) * 4));
  CK(S.rw_npos.ensure((nc + 1) * 8));
  CK(S.rw_n0.ensure(8));
  CK(S.rw_out.ensure(n_spans * sizeof(tgi_rw_span)));
  CK(S.rw_cnt.ensure(2 * n_spans * 4));
  CK(S.rw_rank.ensure(2 * (n_spans + 1) * 8));
  CK(S.sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_rw_out.ensure(n_spans * sizeof(tgi_rw_span)));
  if (n) CK(cudaMemcpyAsync(S.rw_oc.p, outcomes, n * sizeof(tgi_rw_outcome), cudaMemcpyHostToDevice, st));
  StRwStep w{};
  w.c = S.cand.as<StCand>();
  w.cls = S.rw_cls.as<uint32_t>();
  w.lpos = S.rw_lpos.as<uint64_t>();
  w.coff = S.coff.as<uint64_t>();
  w.spans = S.spans.as<tgi_state_span>();
  w.n_spans = n_spans;
  w.n_dec = n_dec;
  w.lk = S.rw_lk.as<tgi_rw_lookup>();
  w.oc = S.rw_oc.as<tgi_rw_outcome>();
  w.nl = nl;
  w.cut = nc;  // a candidate applies when the lookups up to it are before the retire: lpos[j + 1] <= nl
  w.flag = S.rw_flag.as<uint32_t>();
  w.pos = S.rw_pos.as<uint64_t>();
  w.pos_i = w.pos + nl + 1;
  w.pos_d = w.pos_i + nl + 1;
  w.flist = S.rw_list.as<uint32_t>();
  w.ilist = w.flist + nl;
  w.fkeys = S.rw_keys.as<uint8_t>();
  w.ikeys = w.fkeys + 32 * nl;
  w.dkeys = w.ikeys + 32 * nl;
  w.dnew = S.rw_nflag.as<uint32_t>();
  w.npos = S.rw_npos.as<uint64_t>();
  w.n0 = S.rw_n0.as<uint64_t>();
  w.rate = walkback_rate;
  w.seed = S.id_seed;
  w.u0 = S.rw_next;
  w.out = S.rw_out.as<tgi_rw_span>();
  w.cnt = S.rw_cnt.as<uint32_t>();
  uint64_t* dsc = S.sc.as<uint64_t>();  // [3] seed upserts, [4] invalid upserts, [5] discovered inserts, [6] pages, [7] edges
  const uint64_t* hs = S.h_sc.as<uint64_t>();
  uint32_t launches = 0;
  const bool tiled = true;  // launches that do not depend on the sizes
  CK(cudaEventRecord(S.t0, st));
  st_rw_flags_kernel<<<st_grid(c, std::max(nl, nc)), ST_THREADS, 0, st>>>(w);
  launches++;
  if ((rc = launch_scan(c, st, S.tiles, w.flag, nl, w.pos, dsc + 3, launches, tiled))) return rc;
  if ((rc = launch_scan(c, st, S.tiles, w.flag + nl, nl, w.pos_i, dsc + 4, launches, tiled))) return rc;
  if ((rc = launch_scan(c, st, S.tiles, w.flag + 2 * nl, nc, w.pos_d, dsc + 5, launches, tiled))) return rc;
  st_rw_compact_kernel<<<st_grid(c, std::max(nl, nc)), ST_THREADS, 0, st>>>(w);
  launches++;
  CK(cudaGetLastError());
  CK(cudaEventRecord(S.t1, st));
  CK(cudaMemcpyAsync(S.h_sc.p, S.sc.p, ST_SC_COUNT * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  float ms = 0, t = 0;
  cudaEventElapsedTime(&ms, S.t0, S.t1);
  const uint64_t n_found = hs[3], n_fail = hs[4], n_ins = hs[5];
  {
    std::lock_guard<std::mutex> fg(c->fr_mu);
    cudaStream_t st0 = c->slots[0].stream;
    KeySet& SD = c->sets[TGI_SET_DISCOVERED];
    KeySet& SI = c->sets[TGI_SET_INVALID];
    KeySet& SS = c->sets[TGI_SET_SEEDS];
    // AddDiscoveredChannel of the seed hits and found names in candidate order, after the set's count is kept as N0
    if (n_ins && (rc = set_first_use(c, SD, false))) return rc;
    if (SD.dev.table) CK(cudaMemcpyAsync(S.rw_n0.p, SD.dev.count, 8, cudaMemcpyDeviceToDevice, st0));
    else CK(cudaMemsetAsync(S.rw_n0.p, 0, 8, st0));
    if (n_ins) {
      if ((rc = frontier_insert_enqueue(c, SD, w.dkeys, nullptr, n_ins, S.rw_new.p))) return rc;
      CK(cudaStreamSynchronize(st0));
      if ((rc = frontier_insert_check(c, SD))) return rc;
    }
    // MarkChannelInvalid: the failed names in, then every one of them stamped with the call's clock
    if (n_fail) {
      if ((rc = set_first_use(c, SI, true))) return rc;
      if ((rc = frontier_insert_enqueue(c, SI, w.ikeys, nullptr, n_fail, nullptr))) return rc;
      CK(cudaStreamSynchronize(st0));
      if ((rc = frontier_insert_check(c, SI))) return rc;
      st_rw_stamp_kernel<<<st_grid(c, n_fail), ST_THREADS, 0, st0>>>(SI.dev, w.ikeys, n_fail, (long long)now_sec);
      launches++;
    }
    // UpsertSeedChannelChatID fills chatIDCache
    if (n_found) {
      if ((rc = set_first_use(c, SS, false))) return rc;
      if ((rc = frontier_insert_enqueue(c, SS, w.fkeys, nullptr, n_found, nullptr))) return rc;
      CK(cudaStreamSynchronize(st0));
      if ((rc = frontier_insert_check(c, SS))) return rc;
    }
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st0));
    w.disc = SD.dev;
    CK(cudaEventRecord(S.t2, st));
    st_rw_new_kernel<<<st_grid(c, n_ins), ST_THREADS, 0, st>>>(S.rw_new.as<uint8_t>(), n_ins, S.rw_nflag.as<uint32_t>());
    launches++;
    if ((rc = launch_scan(c, st, S.tiles, w.dnew, n_ins, S.rw_npos.as<uint64_t>(), dsc + 5, launches, tiled))) return rc;
    st_rw_span_kernel<<<sink_grid(c, n_spans, ST_THREADS, 4), ST_THREADS, 0, st>>>(st_dev(S), w);
    launches++;
    uint64_t* rank = S.rw_rank.as<uint64_t>();
    for (int k = 0; k < 2; k++)
      if ((rc = launch_scan(c, st, S.tiles, w.cnt + k * n_spans, n_spans, rank + k * (n_spans + 1), dsc + 6 + k, launches, tiled)))
        return rc;
    CK(cudaGetLastError());
    CK(cudaEventRecord(S.t3, st));
    CK(cudaMemcpyAsync(S.h_sc.p, S.sc.p, ST_SC_COUNT * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(S.h_rw_out.p, w.out, n_spans * sizeof(tgi_rw_span), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  cudaEventElapsedTime(&t, S.t2, S.t3);
  ms += t;
  const uint64_t n_pages = hs[6], n_edges = hs[7];
  auto accept = [&]() {  // the lists are spent once the call is accepted
    S.rw_next += n_dec;
    S.rw_live = false;
  };
  out->spans = S.h_rw_out.as<tgi_rw_span>();
  out->kernel_ms = ms;
  out->gpu_launches = launches;
  if (!(n_found + n_fail + n_pages)) {
    accept();
    return TGI_OK;
  }
  StRwSql q{};
  q.p.kind[0] = TGI_SQL_SEED_UPSERT;
  q.p.kind[1] = TGI_SQL_INVALID_UPSERT;
  q.p.kind[2] = TGI_SQL_PAGE_BUFFER_INSERT;
  q.p.kind[3] = TGI_SQL_EDGE_RECORD_INSERT;
  const uint64_t rows[4] = {n_found, n_fail, n_pages, n_edges};
  for (int k = 0; k < 4; k++) {
    q.p.rows[k] = rows[k];
    q.p.k[k] = rows_per_stmt;
  }
  q.w = w;
  q.rank = S.rw_rank.as<uint64_t>();
  return sql_render(c, S, q, st_rw_size_kernel, st_rw_emit_kernel, n_found + n_fail + n_pages + n_edges, crawl_id,
                    crawl_id_len, tb, tl, who, accept, S.h_rw_sql, S.h_rw_stmts, out);
}

// The validator edge pass's lookups: the upload, a thread per edge builds its key, st_first_kernel over the claim, a
// thread per edge classifies it against the invalid set, a scan, the stable radix sort by first occurrence, a thread
// per sorted edge places the rows and occurrences; one synchronise for the totals, one for the read-back.  Lock order:
// the state, then the sets.
int tgi_state_validator_lookups(tgi_ctx* c, const tgi_pending_claim* claim, int64_t now_sec,
                                tgi_state_validator_lookups_t* out) {
  static const char* const who = "tgi_state_validator_lookups";
  if (!c || !out || !claim) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  if ((rc = ve_input(c, claim, who))) return rc;
  const uint64_t n = claim->n_edges;
  memset(out, 0, sizeof *out);
  S.ve_live = false;  // the plan before is gone from here
  S.ve_n = n;
  S.ve_nl = 0;
  if (!n) {
    S.ve_live = true;
    return TGI_OK;
  }
  cudaStream_t st = S.stream;
  const uint64_t bslots = next_pow2(std::max<uint64_t>(2 * n, 64));
  CK(S.ve_e.ensure(n * sizeof(tgi_pending_claim_edge)));
  CK(S.ve_s.ensure(std::max<uint64_t>(claim->strs_len, 1)));
  CK(S.ve_cand.ensure(n * sizeof(StCand)));
  CK(S.ve_bfirst.ensure(bslots * 4));
  CK(S.ve_slot.ensure(n * 4));
  CK(S.ve_flag.ensure(2 * n * 4));
  CK(S.ve_lpos.ensure((n + 1) * 8));
  CK(S.ve_keys.ensure(2 * n * 4));
  CK(S.ve_vals.ensure(2 * n * 4));
  CK(S.ve_loff.ensure((n + 1) * 8));
  CK(S.ve_elk.ensure(n * 4));
  CK(S.ve_rank.ensure(n * 4));
  CK(S.ve_lk.ensure(n * sizeof(tgi_validator_lookup)));
  CK(S.sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_sc.ensure(ST_SC_COUNT * 8));
  CK(cudaMemcpyAsync(S.ve_e.p, claim->edges, n * sizeof(tgi_pending_claim_edge), cudaMemcpyHostToDevice, st));
  if (claim->strs_len) CK(cudaMemcpyAsync(S.ve_s.p, claim->strs, claim->strs_len, cudaMemcpyHostToDevice, st));
  uint64_t* dsc = S.sc.as<uint64_t>();  // [3] lookup rows, [4] their edges, [5] the sort's digit total, [6] n
  StVe v{};
  v.e = S.ve_e.as<tgi_pending_claim_edge>();
  v.s = S.ve_s.as<uint8_t>();
  v.n = n;
  v.d_n = dsc + 6;
  v.c = S.ve_cand.as<StCand>();
  v.flag = S.ve_flag.as<uint32_t>();
  v.lpos = S.ve_lpos.as<uint64_t>();
  v.nl = dsc + 3;
  v.n_occ = dsc + 4;
  v.loff = S.ve_loff.as<uint64_t>();
  v.elk = S.ve_elk.as<uint32_t>();
  v.rank = S.ve_rank.as<uint32_t>();
  v.out = S.ve_lk.as<tgi_validator_lookup>();
  const RadixPlan plan(n);  // by first occurrence; n for the names the invalid set decides
  uint32_t* keys[2] = {S.ve_keys.as<uint32_t>(), S.ve_keys.as<uint32_t>() + n};
  uint32_t* vals[2] = {S.ve_vals.as<uint32_t>(), S.ve_vals.as<uint32_t>() + n};
  v.keys = keys[0];
  v.vals = vals[0];
  v.skeys = keys[plan.out];
  v.svals = vals[plan.out];
  uint32_t launches = 0;
  CK(cudaEventRecord(S.t0, st));
  st_ve_key_kernel<<<st_grid(c, n), ST_THREADS, 0, st>>>(v);
  launches++;
  StFirst w{};  // the first occurrence of every name over the claim
  w.c = v.c;
  w.n = v.d_n;
  w.bound = n;
  w.dedup = true;
  w.bfirst = S.ve_bfirst.as<uint32_t>();
  w.bmask = bslots - 1;
  w.slot_of = S.ve_slot.as<uint32_t>();
  CK(cudaMemsetAsync(w.bfirst, 0xFF, bslots * 4, st));
  st_first_kernel<<<st_grid(c, n), ST_THREADS, 0, st>>>(w);
  launches++;
  v.bfirst = w.bfirst;
  v.slot_of = w.slot_of;
  {
    std::lock_guard<std::mutex> fg(c->fr_mu);  // the invalid set: probed, not changed
    if (c->fr_event_valid) CK(cudaStreamWaitEvent(st, c->fr_event, 0));
    v.x = exclusion(c, now_sec);
    st_ve_class_kernel<<<st_grid(c, n), ST_THREADS, 0, st>>>(v);
    launches++;
    CK(cudaGetLastError());
  }
  if ((rc = launch_scan(c, st, S.tiles, v.flag, n, v.lpos, dsc + 3, launches, true))) return rc;
  if ((rc = radix_sort(c, st, S.tiles, keys, vals, v.d_n, n, plan, S.counts, S.roff, dsc + 5, true, launches))) return rc;
  CK(cudaMemsetAsync(v.loff, 0, 8, st));  // no row: loff[0] = 0 ends them
  CK(cudaMemsetAsync(v.n_occ, 0, 8, st));
  st_ve_group_kernel<<<st_grid(c, n), ST_THREADS, 0, st>>>(v);
  st_ve_rows_kernel<<<st_grid(c, n), ST_THREADS, 0, st>>>(v);
  launches += 2;
  CK(cudaGetLastError());
  CK(cudaEventRecord(S.t1, st));
  CK(cudaMemcpyAsync(S.h_sc.p, S.sc.p, ST_SC_COUNT * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const uint64_t nl = S.h_sc.as<uint64_t>()[3], n_occ = S.h_sc.as<uint64_t>()[4];
  float ms = 0;
  cudaEventElapsedTime(&ms, S.t0, S.t1);
  CK(S.h_ve_lk.ensure(std::max<uint64_t>(nl, 1) * sizeof(tgi_validator_lookup)));
  CK(S.h_ve_occ.ensure(std::max<uint64_t>(n_occ, 1) * 4));
  if (nl) CK(cudaMemcpyAsync(S.h_ve_lk.p, v.out, nl * sizeof(tgi_validator_lookup), cudaMemcpyDeviceToHost, st));
  if (n_occ) CK(cudaMemcpyAsync(S.h_ve_occ.p, v.svals, n_occ * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  S.ve_live = true;  // ve_e, ve_s, ve_elk, ve_rank and h_ve_lk hold the plan
  S.ve_nl = nl;
  out->n_edges = n;
  out->n_cached = n - n_occ;
  out->n_lookups = nl;
  out->lookups = S.h_ve_lk.as<tgi_validator_lookup>();
  out->occurrences = S.h_ve_occ.as<uint32_t>();
  out->kernel_ms = ms;
  out->gpu_launches = launches;
  return TGI_OK;
}

// The validator edge pass over the plan: the outcomes' checks on the host; a thread per edge derives its update, one
// block scans the counter, two scans and a compaction place the upsert rows (one synchronise); the two ordered set
// inserts on the sets' stream; then the rows as tgi_state_edge_sql renders them.
int tgi_state_validator_edges(tgi_ctx* c, const tgi_validator_outcome* outcomes, uint64_t n_outcomes,
                              const tgi_validator_attempt* attempts, uint64_t n_attempts, int64_t blocked_count_in,
                              int64_t now_sec, uint32_t rows_per_stmt, tgi_state_validator_edges_t* out) {
  static const char* const who = "tgi_state_validator_edges";
  if (!c || !out) return TGI_E_ARG;
  CrawlState& S = c->state;
  std::lock_guard<std::mutex> g(S.mu);
  int rc;
  if ((rc = st_init(c, S))) return rc;
  if ((rc = sql_args(c, S, rows_per_stmt, 0, nullptr, 0, who, false))) return rc;
  if (!S.ve_live) { set_err(c, "%s: no plan (tgi_state_validator_lookups)", who); return TGI_E_STATE; }
  if (blocked_count_in < 0 || blocked_count_in > (1ll << 62)) { set_err(c, "%s: blocked_count_in %lld outside [0, 2^62]", who, (long long)blocked_count_in); return TGI_E_ARG; }
  const uint64_t n = S.ve_n, nl = S.ve_nl;
  if (n_outcomes != nl) { set_err(c, "%s: %llu outcomes for %llu lookups", who, (unsigned long long)n_outcomes, (unsigned long long)nl); return TGI_E_ARG; }
  if ((nl && !outcomes) || (n_attempts && !attempts)) { set_err(c, "%s: outcomes or attempts is NULL", who); return TGI_E_ARG; }
  CK(S.h_ve_aoff.ensure(std::max<uint64_t>(nl, 1) * 8));
  if ((rc = ve_outcomes(c, S.h_ve_lk.as<tgi_validator_lookup>(), outcomes, nl, attempts, n_attempts, S.h_ve_aoff.as<uint64_t>(), who)))
    return rc;
  memset(out, 0, sizeof *out);
  out->blocked_count_out = blocked_count_in;
  out->crossed_at = TGI_VE_NOT_CROSSED;
  if (!n) {
    S.ve_live = false;
    return TGI_OK;
  }
  cudaStream_t st = S.stream;
  CK(S.ve_oc.ensure(std::max<uint64_t>(nl, 1) * sizeof(tgi_validator_outcome)));
  CK(S.ve_aoff.ensure(std::max<uint64_t>(nl, 1) * 8));
  CK(S.ve_at.ensure(std::max<uint64_t>(n_attempts, 1) * sizeof(tgi_validator_attempt)));
  CK(S.ve_res.ensure(n * sizeof(tgi_validator_edge_result)));
  CK(S.ve_flag.ensure(2 * n * 4));
  CK(S.ve_pos.ensure(2 * (n + 1) * 8));
  CK(S.ve_list.ensure(2 * n * 4));
  CK(S.ve_names.ensure(2 * n * 32));
  CK(S.sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_ve_res.ensure(n * sizeof(tgi_validator_edge_result)));
  if (nl) {
    CK(cudaMemcpyAsync(S.ve_oc.p, outcomes, nl * sizeof(tgi_validator_outcome), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(S.ve_aoff.p, S.h_ve_aoff.p, nl * 8, cudaMemcpyHostToDevice, st));
  }
  if (n_attempts) CK(cudaMemcpyAsync(S.ve_at.p, attempts, n_attempts * sizeof(tgi_validator_attempt), cudaMemcpyHostToDevice, st));
  uint64_t* dsc = S.sc.as<uint64_t>();  // [0] the count after the claim, [1] the crossing, [3] seed rows, [4] invalid rows
  StVeApply a{};
  a.e = S.ve_e.as<tgi_pending_claim_edge>();
  a.s = S.ve_s.as<uint8_t>();
  a.n = n;
  a.elk = S.ve_elk.as<uint32_t>();
  a.rank = S.ve_rank.as<uint32_t>();
  a.oc = S.ve_oc.as<tgi_validator_outcome>();
  a.aoff = S.ve_aoff.as<uint64_t>();
  a.at = S.ve_at.as<tgi_validator_attempt>();
  a.count_in = blocked_count_in;
  a.res = S.ve_res.as<tgi_validator_edge_result>();
  a.flag = S.ve_flag.as<uint32_t>();
  a.pos = S.ve_pos.as<uint64_t>();
  a.pos_i = a.pos + n + 1;
  a.list = S.ve_list.as<uint32_t>();
  a.keys = S.ve_names.as<uint8_t>();
  a.sc = dsc;
  uint32_t launches = 0;
  CK(cudaEventRecord(S.t0, st));
  st_ve_edge_kernel<<<st_grid(c, n), ST_THREADS, 0, st>>>(a);
  st_ve_counter_kernel<<<1, ST_VE_THREADS, 0, st>>>(a);
  launches += 2;
  if ((rc = launch_scan(c, st, S.tiles, a.flag, n, a.pos, dsc + 3, launches, true))) return rc;
  if ((rc = launch_scan(c, st, S.tiles, a.flag + n, n, a.pos_i, dsc + 4, launches, true))) return rc;
  st_ve_compact_kernel<<<st_grid(c, n), ST_THREADS, 0, st>>>(a);
  launches++;
  CK(cudaGetLastError());
  CK(cudaEventRecord(S.t1, st));
  CK(cudaMemcpyAsync(S.h_sc.p, S.sc.p, ST_SC_COUNT * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(S.h_ve_res.p, a.res, n * sizeof(tgi_validator_edge_result), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  float ms = 0;
  cudaEventElapsedTime(&ms, S.t0, S.t1);
  const uint64_t* hs = S.h_sc.as<uint64_t>();
  const uint64_t n_seed = hs[3], n_inv = hs[4], crossed = hs[1];
  const int64_t count_out = (int64_t)hs[0];
  {
    std::lock_guard<std::mutex> fg(c->fr_mu);
    cudaStream_t st0 = c->slots[0].stream;
    KeySet& SI = c->sets[TGI_SET_INVALID];
    KeySet& SS = c->sets[TGI_SET_SEEDS];
    if (n_seed) {  // UpsertSeedChannelChatID fills chatIDCache
      if ((rc = set_first_use(c, SS, false))) return rc;
      if ((rc = frontier_insert_enqueue(c, SS, a.keys, nullptr, n_seed, nullptr))) return rc;
      CK(cudaStreamSynchronize(st0));
      if ((rc = frontier_insert_check(c, SS))) return rc;
    }
    if (n_inv) {  // MarkChannelInvalid: the names in, then every one of them stamped with the call's clock
      const uint8_t* ikeys = a.keys + 32 * n;
      if ((rc = set_first_use(c, SI, true))) return rc;
      if ((rc = frontier_insert_enqueue(c, SI, ikeys, nullptr, n_inv, nullptr))) return rc;
      CK(cudaStreamSynchronize(st0));
      if ((rc = frontier_insert_check(c, SI))) return rc;
      st_rw_stamp_kernel<<<st_grid(c, n_inv), ST_THREADS, 0, st0>>>(SI.dev, ikeys, n_inv, (long long)now_sec);
      launches++;
      CK(cudaGetLastError());
      CK(cudaStreamSynchronize(st0));
    }
  }
  out->n_edges = n;
  out->edges = S.h_ve_res.as<tgi_validator_edge_result>();
  out->blocked_count_out = count_out;
  out->crossed_at = crossed;
  out->kernel_ms = ms;
  out->gpu_launches = launches;
  StVeSql q{};
  q.p.kind[0] = TGI_SQL_SEED_UPSERT;
  q.p.kind[1] = TGI_SQL_INVALID_UPSERT;
  q.p.kind[2] = TGI_SQL_ACCESS_EVENT;
  q.p.kind[3] = TGI_SQL_EDGE_UPDATE;
  const uint64_t rows[4] = {n_seed, n_inv, crossed != TGI_VE_NOT_CROSSED ? 1u : 0u, n};
  for (int k = 0; k < 4; k++) {
    q.p.rows[k] = rows[k];
    q.p.k[k] = k == 2 ? 1u : rows_per_stmt;
  }
  q.a = a;
  auto accept = [&]() { S.ve_live = false; };
  return sql_render(c, S, q, st_ve_size_kernel, st_ve_emit_kernel, n_seed + n_inv + rows[2] + n, nullptr, 0, nullptr, 0,
                    who, accept, S.h_ve_sql, S.h_ve_stmts, out);
}

}  // extern "C"
