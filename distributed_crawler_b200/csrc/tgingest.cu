// tgingest.cu — host side of libtgingest: the C ABI of include/tgingest.h on top of the sm_90a
// kernels in kernels.cuh.  One context = one GPU.  Three staging slots, each with its own stream
// and worker thread, so H2D of one batch, kernels of another and D2H of a third overlap.
// There is no CPU fallback: without a CUDA device tgi_create fails with TGI_E_NODEVICE.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>  // types only: the library itself is loaded with dlopen at tgi_comm_init

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <map>
#include <string>
#include <thread>
#include <unordered_map>
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

enum RecKind { REC_NONE, REC_TG, REC_YT, REC_GM };

// One job on a staging slot: upload a batch (which becomes the slot's resident batch), run the resident batch, or both.
enum JobStages : uint32_t { JOB_UPLOAD = 1, JOB_RUN = 2 };
struct Job {
  RecKind kind;
  uint32_t stages;    // JOB_UPLOAD | JOB_RUN
  const void* batch;  // JOB_UPLOAD: the tgi_tg_batch / tgi_yt_batch / tgi_gm_batch of `kind`
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
  HostBuf h_out, h_sc, h_read;
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
  // frontier -> validator hand-off (tgi_set_add) and this rank's partition of the multi-GPU set (tgi_comm_init)
  KeySet sets[4];
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

// The set `which` (TGI_SET_*) names, or nullptr.  With exclusion_only, only the exclusion sets are named (the
// tgi_set_add / _clear / _size family).
KeySet* key_set(tgi_ctx* c, int which, bool exclusion_only) {
  if (which == TGI_SET_INVALID || which == TGI_SET_DISCOVERED) return &c->sets[which];
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
      uint64_t want = (n + WARPS_PER_CTA - 1) / WARPS_PER_CTA;
      unsigned g = (unsigned)std::min<uint64_t>(want, (uint64_t)c->sms * grid_mult());
      CK(cudaEventRecord(s.ev_p0, st));
      const uint64_t groups = (n + 31) / 32;
      unsigned ge = (unsigned)std::min<uint64_t>((groups + WARPS_PER_CTA - 1) / WARPS_PER_CTA, (uint64_t)c->sms * grid_mult());
      // JSONL: the link count measures the message texts as well (the size pass then skips the clean ones); runs without
      // JSONL take the instances without that code
      const bool measure = want_json && size_text_in_parse();
      if (s.n_ents) {  // records with entities first: status + links (two kernels by instruction footprint)
        tg_ent_map_kernel<<<ge, CTA_THREADS, 0, st>>>(b, po);
        if (measure) tg_parse_ent_kernel<true><<<ge, CTA_THREADS, 0, st>>>(b, cfg, flags, po);
        else tg_parse_ent_kernel<false><<<ge, CTA_THREADS, 0, st>>>(b, cfg, flags, po);
        launches += 2;
      }
      if (measure) tg_parse_kernel<true><<<g, CTA_THREADS, 0, st>>>(b, cfg, flags, po);  // records without entities
      else tg_parse_kernel<false><<<g, CTA_THREADS, 0, st>>>(b, cfg, flags, po);
      launches++;
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
  {  // every offset the kernels will follow stays inside its array (O(n) on the host: 80-byte records, no side arrays)
    int e = 0;
    for (uint64_t i = 0; i < in->n; i++) {
      const tgi_yt_rec& r = in->recs[i];
      uint64_t end = r.str_off + (uint64_t)r.id_len + r.title_len + r.desc_len + r.duration_len + r.lang_len;
      for (int k = 0; k < 5; k++) end += r.thumb_len[k] == TGI_YT_THUMB_ABSENT ? 0u : r.thumb_len[k];
      if (end > in->strs_len || end < r.str_off) e |= 1;
      if (r.chan_idx >= in->n_chans) e |= 2;
    }
    for (uint32_t i = 0; i < in->n_chans; i++) {
      const tgi_yt_chan& ch = in->chans[i];
      if ((uint64_t)ch.str_off + ch.id_len + ch.title_len + ch.desc_len + ch.thumb_len + ch.country_len > in->chan_strs_len) e |= 512;
    }
    if (e) { set_err(c, "youtube batch: offsets outside their arrays (mask 0x%x)", e); return TGI_E_ARG; }
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
  {
    int e = 0;
    for (uint64_t i = 0; i < in->n; i++) {
      const tgi_gm_rec& r = in->recs[i];
      const uint64_t end = r.str_off + (uint64_t)r.id_len + r.channel_len + r.text_len + r.sender_len;
      if (end > in->strs_len || end < r.str_off) e |= 1;
      if (in->react_off && (in->react_off[i] > in->react_off[i + 1] || in->react_off[i + 1] > in->n_reacts)) e |= 8;
    }
    for (uint64_t i = 0; i < in->n_reacts; i++)
      if ((uint64_t)in->reacts[i].key_off + in->reacts[i].key_len > in->aux_len) e |= 64;
    if (e) { set_err(c, "generic batch: offsets outside their arrays (mask 0x%x)", e); return TGI_E_ARG; }
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

// ---- jobs -------------------------------------------------------------------------------------------------------------
// Upload if the job uploads (an upload-only job waits for the copy to land), run if it runs.
int run_job(tgi_ctx* c, Slot& s) {
  const Job& j = s.job;
  if (j.stages & JOB_UPLOAD) {
    const int rc = j.kind == REC_TG   ? upload_tg(c, s, (const tgi_tg_batch*)j.batch)
                   : j.kind == REC_YT ? upload_yt(c, s, (const tgi_yt_batch*)j.batch)
                                      : upload_gm(c, s, (const tgi_gm_batch*)j.batch);
    if (rc != TGI_OK) return rc;
    if (!(j.stages & JOB_RUN)) {
      const cudaError_t e = cudaStreamSynchronize(s.stream);
      if (e != cudaSuccess) { set_err(c, "upload sync: %s", cudaGetErrorString(e)); return TGI_E_CUDA; }
    }
    if (j.kind != REC_GM) s.resident = j.kind;  // generic batches are not run resident
  }
  if (!(j.stages & JOB_RUN)) return TGI_OK;
  return j.kind == REC_TG   ? run_tg(c, s, j.flags, &s.res)
         : j.kind == REC_YT ? run_yt(c, s, j.flags, &s.res)
                            : run_gm(c, s, j.flags, &s.res);
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

// The sinks' view of slot `slot`: its last result, which must be a Telegram or YouTube one with lines; with src, also
// the device arrays the sink kernels read (sink_src.cuh).  Selects the context's device.
int sink_source(tgi_ctx* c, int slot, const char* who, LastResult& r, SinkSrc* src) {
  const int rc = slot_result(c, slot, who, &r);
  if (rc != TGI_OK) return rc;
  if (r.kind == REC_GM) { set_err(c, "%s: generic posts go to SavePost, not to the StorePost sinks", who); return TGI_E_STATE; }
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
  // the resident batch descriptor, not the upload buffers: a page-sized batch lives in the slot's one-block upload
  if (src->yt) {
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
  for (cudaEvent_t e : {c->state.t0, c->state.t1, c->state.t2, c->state.t3}) if (e) cudaEventDestroy(e);
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
int tgi_set_add(tgi_ctx* c, int which, const uint8_t* keys32, const int64_t* stamp_sec, uint64_t n) {
  if (!c || (n && !keys32)) return TGI_E_ARG;
  KeySet* k = key_set(c, which, true);
  if (!k) { set_err(c, "tgi_set_add: unknown set %d", which); return TGI_E_ARG; }
  if (n >= (1ull << 32)) { set_err(c, "too many keys in one call"); return TGI_E_ARG; }
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> g(c->fr_mu);
  cudaStream_t st = c->slots[0].stream;
  const bool stamps = which == TGI_SET_INVALID;
  if (!k->dev.table) {  // first use: same capacity as the dedup set, or at most 2^16 keys when the sets grow on their own
    const FrontierDev& fr = c->sets[TGI_SET_FRONTIER].dev;
    const uint64_t cap = std::min<uint64_t>(c->fr_cap0, 1u << 16);
    const int rc = c->grow_max ? set_alloc(c, *k, cap, next_pow2(2 * cap), stamps)
                               : set_alloc(c, *k, fr.cap, fr.tmask + 1, stamps);
    if (rc) return rc;
  }
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
  int rc = sink_source(c, slot, "tgi_dapr_payloads", r, &src);
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
  int rc = sink_source(c, slot, "tgi_channel_appends", r, &src);
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
  // radix passes over the bits of the largest group id, 8 bits or fewer each
  uint32_t bits = 0;
  while (bits < 32 && (gmax - 1) >> bits) bits++;
  const uint32_t passes = (bits + 7) / 8, width = passes ? (bits + passes - 1) / passes : 0, radix = 1u << width;
  const uint64_t ntiles = (n + RS_TILE - 1) / RS_TILE;
  CK(z.table.ensure(tslots * 4));
  CK(z.rows.ensure(2 * nc * 4));
  CK(z.u32s.ensure(11 * n2 * 4));
  CK(z.u64s.ensure(7 * n2 * 8));
  CK(z.counts.ensure(radix * ntiles * 4));
  CK(z.roff.ensure((radix * ntiles + 1) * 8));
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
  int cur = 0;  // the ping-pong side that holds the sorted pairs
  for (uint32_t p = 0; p < passes; p++, cur ^= 1) {
    const uint32_t shift = p * width;
    la_radix_hist_kernel<<<(unsigned)ntiles, RS_WARPS * 32, 0, st>>>(w.keys[cur], w.sc + LA_SC_RUNS, shift, radix,
                                                                     (uint32_t)ntiles, z.counts.as<uint32_t>());
    launches++;
    if ((rc = launch_scan(c, s, z.counts.as<uint32_t>(), radix * ntiles, z.roff.as<uint64_t>(), w.sc + LA_SC_RADIX, launches))) return rc;
    la_radix_scatter_kernel<<<(unsigned)ntiles, RS_WARPS * 32, 0, st>>>(w.keys[cur], w.vals[cur], w.keys[cur ^ 1],
                                                                        w.vals[cur ^ 1], w.sc + LA_SC_RUNS, shift, radix,
                                                                        (uint32_t)ntiles, z.roff.as<uint64_t>());
    launches++;
  }
  const uint32_t* sorted = w.vals[cur];
  la_sorted_counts_kernel<<<grid(n), LA_THREADS, 0, st>>>(n, sorted, w);
  launches++;
  if ((rc = launch_scan(c, s, w.cnt, n, w.lpos, w.sc + LA_SC_SORTED_LINES, launches))) return rc;
  la_inverse_kernel<<<grid(n), LA_THREADS, 0, st>>>(sorted, w);
  la_order_kernel<<<grid(n), LA_THREADS, 0, st>>>(src, w);
  launches += 2;
  if ((rc = launch_scan(c, s, w.cnt, n, w.goff, w.sc + LA_SC_BYTES, launches))) return rc;
  la_tables_kernel<<<grid(n), LA_THREADS, 0, st>>>(src, w.keys[cur], sorted, w);
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
  int rc = sink_source(c, slot, "tgi_combine_add", r, nullptr);
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

// the state's stream, events, preset codes and minimal buffers, on first use (under S.mu)
int st_init(tgi_ctx* c, CrawlState& S) {
  cudaSetDevice(c->device);
  if (S.stream) return TGI_OK;
  CK(cudaStreamCreateWithFlags(&S.stream, cudaStreamNonBlocking));
  CK(cudaEventCreate(&S.t0));
  CK(cudaEventCreate(&S.t1));
  CK(cudaEventCreate(&S.t2));
  CK(cudaEventCreate(&S.t3));
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

// the row's message generation moves on: its messages become tombstones
int st_drop_messages(tgi_ctx* c, CrawlState& S, uint32_t r) {
  uint32_t cnt = 0;
  int rc;
  if ((rc = st_row_count(c, S, r, &cnt))) return rc;
  S.n_dead += cnt;
  S.gen[r]++;
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
  // SetState: new maps, layer by layer; a later page with the same id replaces the row (and its messages)
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
  cudaStream_t st = S.stream;
  const uint64_t bslots = next_pow2(std::max<uint64_t>(2 * m, 64));
  CK(S.upd.ensure(m * sizeof(tgi_state_update)));
  CK(S.bfirst.ensure(bslots * 4));
  CK(S.blast.ensure(bslots * 4));
  CK(S.slot_of.ensure(m * 4));
  CK(S.flag.ensure(m * 4));
  CK(S.pos.ensure((m + 1) * 8));
  CK(S.sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_sc.ensure(ST_SC_COUNT * 8));
  CK(cudaMemcpyAsync(S.upd.p, u.data(), m * sizeof(tgi_state_update), cudaMemcpyHostToDevice, st));
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
  uint32_t launches = 0;
  st_upd_build_kernel<<<st_grid(c, m), ST_THREADS, 0, st>>>(w);
  st_upd_resolve_kernel<<<st_grid(c, m), ST_THREADS, 0, st>>>(d, w);
  if ((rc = launch_scan(c, st, S.tiles, w.flag, m, w.pos, S.sc.as<uint64_t>(), launches))) return rc;
  st_upd_append_kernel<<<st_grid(c, m), ST_THREADS, 0, st>>>(d, w);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(S.h_sc.p, S.sc.p, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const uint64_t added = *S.h_sc.as<uint64_t>();
  if (added) st_table_insert_kernel<<<st_grid(c, added), ST_THREADS, 0, st>>>(d, S.n_msgs, S.n_msgs + added);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(st));
  S.n_msgs += added;
  return TGI_OK;
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
  cudaStream_t st = S.stream;
  const uint64_t nm = S.n_msgs;
  CK(S.flag.ensure(nm * 4));
  CK(S.pos.ensure((nm + 1) * 8));
  CK(S.sc.ensure(ST_SC_COUNT * 8));
  CK(S.spare.ensure(cnt * sizeof(tgi_state_msg)));
  const StDev d = st_dev(S);
  uint32_t launches = 0;
  st_live_flag_kernel<<<st_grid(c, nm), ST_THREADS, 0, st>>>(d, nm, row, S.flag.as<uint32_t>());
  if ((rc = launch_scan(c, st, S.tiles, S.flag.as<uint32_t>(), nm, S.pos.as<uint64_t>(), S.sc.as<uint64_t>(), launches))) return rc;
  st_read_kernel<<<st_grid(c, nm), ST_THREADS, 0, st>>>(d, nm, S.flag.as<uint32_t>(), S.pos.as<uint64_t>(), S.spare.as<tgi_state_msg>());
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, S.spare.p, cnt * sizeof(tgi_state_msg), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
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
  const uint64_t ne = E.size(), nr = S.rows.size(), nm = S.n_msgs, live = nm - S.n_dead;
  cudaStream_t st = S.stream;
  uint32_t launches = 0;
  uint64_t body = 0;
  CK(S.sc.ensure(ST_SC_COUNT * 8));
  CK(S.h_sc.ensure(ST_SC_COUNT * 8));
  // the zone table must not change under the kernels that read it (tgi_set_zone swaps it under cfg_mu)
  std::lock_guard<std::mutex> zg(c->cfg_mu);
  if (ne) {
    CK(S.flag.ensure(nm * 4));
    CK(S.pos.ensure((nm + 1) * 8));
    CK(S.keys.ensure(2 * live * 4));
    CK(S.vals.ensure(2 * live * 4));
    CK(S.row_base.ensure((nr + 1) * 8));
    CK(S.msize.ensure(live * 4));
    CK(S.moff.ensure((live + 1) * 8));
    CK(S.entries.ensure(ne * sizeof(StEntry)));
    CK(S.e32.ensure(4 * ne * 4));
    CK(S.e64.ensure(2 * (ne + 1) * 8));
    StRender r{};
    r.entries = S.entries.as<StEntry>();
    r.n_entries = ne;
    r.zone = c->cfgdev.zone;
    r.zone_n = c->cfgdev.zone_n;
    r.tz = c->cfgdev.tz;
    r.sc = S.sc.as<uint64_t>();
    r.flag = S.flag.as<uint32_t>();
    r.pos = S.pos.as<uint64_t>();
    r.keys[0] = S.keys.as<uint32_t>();
    r.keys[1] = r.keys[0] + live;
    r.vals[0] = S.vals.as<uint32_t>();
    r.vals[1] = r.vals[0] + live;
    r.row_base = S.row_base.as<uint64_t>();
    r.msize = S.msize.as<uint32_t>();
    r.moff = S.moff.as<uint64_t>();
    r.esize_lo = S.e32.as<uint32_t>();
    r.ebytes = r.esize_lo + ne;
    r.ecnt = r.ebytes + ne;
    r.esz = r.ecnt + ne;
    r.eoff = S.e64.as<uint64_t>();
    r.eslot = r.eoff + ne + 1;
    // radix passes over the bits of the largest row
    uint32_t bits = 0;
    while (bits < 32 && nr > 1 && (nr - 1) >> bits) bits++;
    const uint32_t passes = (bits + 7) / 8, width = passes ? (bits + passes - 1) / passes : 0, radix = 1u << width;
    const uint64_t ntiles = std::max<uint64_t>((live + RS_TILE - 1) / RS_TILE, 1);
    CK(S.counts.ensure(radix * ntiles * 4));
    CK(S.roff.ensure((radix * ntiles + 1) * 8));
    const StDev d = st_dev(S);
    CK(cudaMemcpyAsync(S.entries.p, E.data(), ne * sizeof(StEntry), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(S.sc.p, 0, ST_SC_COUNT * 8, st));
    CK(cudaEventRecord(S.t0, st));
    st_render_flag_kernel<<<st_grid(c, nm), ST_THREADS, 0, st>>>(d, nm, r);
    launches++;
    if ((rc = launch_scan(c, st, S.tiles, r.flag, nm, r.pos, r.sc + ST_SC_LIVE, launches))) return rc;
    st_render_pairs_kernel<<<st_grid(c, nm), ST_THREADS, 0, st>>>(d, nm, r);
    launches++;
    int cur = 0;
    for (uint32_t p = 0; p < passes; p++, cur ^= 1) {
      const uint32_t shift = p * width;
      la_radix_hist_kernel<<<(unsigned)ntiles, RS_WARPS * 32, 0, st>>>(r.keys[cur], r.sc + ST_SC_LIVE, shift, radix, (uint32_t)ntiles,
                                                                     S.counts.as<uint32_t>());
      launches++;
      if ((rc = launch_scan(c, st, S.tiles, S.counts.as<uint32_t>(), radix * ntiles, S.roff.as<uint64_t>(), r.sc + ST_SC_RADIX, launches))) return rc;
      la_radix_scatter_kernel<<<(unsigned)ntiles, RS_WARPS * 32, 0, st>>>(r.keys[cur], r.vals[cur], r.keys[cur ^ 1], r.vals[cur ^ 1],
                                                                        r.sc + ST_SC_LIVE, shift, radix, (uint32_t)ntiles,
                                                                        S.roff.as<uint64_t>());
      launches++;
    }
    if ((rc = launch_scan(c, st, S.tiles, d.row_cnt, nr, r.row_base, r.sc + ST_SC_ROWS, launches))) return rc;
    st_msg_size_kernel<<<st_grid(c, live), ST_THREADS, 0, st>>>(d, r, r.vals[cur], r.keys[cur], live);
    launches++;
    if ((rc = launch_scan(c, st, S.tiles, r.msize, live, r.moff, r.sc + ST_SC_MBYTES, launches))) return rc;
    st_entry_size_kernel<<<sink_grid(c, ne, ST_WARPS, 16), ST_WARPS * 32, 0, st>>>(d, r);
    launches++;
    if ((rc = launch_scan(c, st, S.tiles, r.esz, ne, r.eoff, r.sc + ST_SC_BYTES, launches))) return rc;
    if ((rc = launch_scan(c, st, S.tiles, r.ecnt, ne, r.eslot, r.sc + ST_SC_SLOTS, launches))) return rc;
    CK(cudaGetLastError());
    CK(cudaEventRecord(S.t1, st));
    CK(cudaMemcpyAsync(S.h_sc.p, S.sc.p, ST_SC_COUNT * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    const uint64_t* h = S.h_sc.as<uint64_t>();
    if (h[ST_SC_LIVE] != live) { set_err(c, "tgi_state_render: %llu live messages, expected %llu", (unsigned long long)h[ST_SC_LIVE], (unsigned long long)live); return TGI_E_CUDA; }
    if (h[ST_SC_ERR]) { set_err(c, "tgi_state_render: a page timestamp's year is outside [0, 9999] (json.Marshal fails)"); return TGI_E_ARG; }
    if (h[ST_SC_BIG]) { set_err(c, "tgi_state_render: a page renders to 4 GiB or more"); return TGI_E_CAPACITY; }
    body = h[ST_SC_BYTES];
    const uint64_t slots = h[ST_SC_SLOTS];
    float size_ms = 0, emit_ms = 0;
    cudaEventElapsedTime(&size_ms, S.t0, S.t1);
    CK(S.out.ensure(body));
    CK(S.h_out.ensure(sizeof kHead + body + sizeof kMeta + metadata_len + sizeof kLast + last_updated_len + 2));
    r.out = S.out.as<uint8_t>();
    CK(cudaEventRecord(S.t2, st));
    st_entry_emit_kernel<<<sink_grid(c, ne, ST_WARPS, 16), ST_WARPS * 32, 0, st>>>(d, r);
    if (slots) st_msg_emit_kernel<<<st_grid(c, slots), ST_THREADS, 0, st>>>(d, r, r.vals[cur]);
    launches += 1 + (slots != 0);
    CK(cudaGetLastError());
    CK(cudaEventRecord(S.t3, st));
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

}  // extern "C"
