// dapr.cuh — DaprStateManager.StorePost payloads (state/daprstate.go:1141-1181, non-combine branch) for every line of a
// batch result that is still resident on the device (sm_90a).
//
// For every record with status TGI_ST_EMITTED the reference sends
//   Data     = base64.StdEncoding.EncodeToString(json.Marshal(post) + "\n")          (daprstate.go:1159)
//   Metadata = the blob path <prefix><channelID>/posts/<PostUID>.jsonl                (:1150-1153, format :2689-2698)
// Two kernels: dapr_size_kernel measures both per record (the host scans them into u64 offsets with launch_scan),
// dapr_write_kernel encodes each line once, a warp per record, and writes its path.
#pragma once
#include "sink_src.cuh"

namespace tgi {

constexpr int DAPR_CHUNK = 768;             // line bytes a warp encodes per step: 256 base64 words, 8 per lane
constexpr int DAPR_VECS = DAPR_CHUNK / 16 + 1;  // aligned 16-byte loads that cover a chunk at any start alignment
constexpr int DAPR_ERR_TOO_LONG = 1;        // a payload or a path of 2^32 bytes or more
// the path's literals, little-endian in immediates (no device globals: the other kernels' SASS stays as it was)
constexpr uint64_t DAPR_POSTS = 0x2f7374736f702full;  // "/posts/"
constexpr uint64_t DAPR_JSONL = 0x6c6e6f736a2eull;    // ".jsonl"

struct DaprOut {
  uint32_t* data_len;  // [n] sizes (dapr_size_kernel)
  uint32_t* path_len;
  const uint64_t* data_off;  // [n+1] their exclusive scans
  const uint64_t* path_off;
  uint8_t* data;
  uint8_t* path;
  int* err;
  const uint8_t* prefix;  // StorageRoot/CrawlID/CrawlExecutionID/, verbatim
  uint32_t prefix_len;
};

struct DaprPath {
  const uint8_t* chan;  // channelID
  uint32_t chan_len;
  const uint8_t* uid;   // PostUID, or (Telegram) its tail after the number and the '-'
  uint32_t uid_len;
  int64_t num;          // Telegram: id / 1048576, Go's truncating division (tdutils.go:1008)
  uint32_t num_len;     // digits of num, 0 for YouTube
};

// PostUID: Telegram id/2^20 "-" channel name (tdutils.go:1008), YouTube the video id (youtube_crawler.go:701)
DEVI DaprPath dapr_path(const SinkSrc& s, uint64_t i) {
  DaprPath p;
  if (s.yt) {
    const tgi_yt_rec& r = s.yt_recs[i];
    p.chan = sink_chan_id(s, r.chan_idx, p.chan_len);
    p.uid = s.strs + r.str_off;
    p.uid_len = r.id_len;
    p.num = 0;
    p.num_len = 0;
  } else {
    const tgi_tg_rec& r = s.tg_recs[i];
    p.chan = sink_chan_id(s, r.chan_idx, p.chan_len);
    p.uid = p.chan;
    p.uid_len = p.chan_len;
    p.num = r.id / 1048576;
    p.num_len = ndigits_i64(p.num) + 1;  // the number and its '-'
  }
  return p;
}
DEVI uint64_t dapr_path_len(const DaprOut& o, const DaprPath& p) {
  return (uint64_t)o.prefix_len + p.chan_len + 7 + p.num_len + p.uid_len + 6;  // "/posts/" ... ".jsonl"
}

// one thread per record: base64 length 4*ceil(len/3) of its line and the length of its path; 0 for records without a
// post (skipped, failed, TGI_ST_NOLINE: the reference calls no binding for them)
__global__ void dapr_size_kernel(SinkSrc s, DaprOut o) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < s.n; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t d = 0, p = 0;
    if (s.status[i] == TGI_ST_EMITTED) {
      d = (s.line_off[i + 1] - s.line_off[i] + 2) / 3 * 4;
      p = dapr_path_len(o, dapr_path(s, i));
    }
    if ((d | p) >> 32) {
      atomicOr(o.err, DAPR_ERR_TOO_LONG);
      d = p = 0;
    }
    o.data_len[i] = (uint32_t)d;
    o.path_len[i] = (uint32_t)p;
  }
}

struct DaprShared {
  uint4 line[WARPS_PER_CTA][DAPR_VECS];  // one chunk of a line per warp, from aligned 16-byte loads
  uint8_t num[WARPS_PER_CTA][24];        // the Telegram PostUID's number
};

// A warp per record, grid-stride.  The line is read once, in chunks of DAPR_CHUNK bytes: the warp stages the aligned
// 16-byte words that cover the chunk in shared memory (lines start at any byte; the loads stay within 15 bytes of the
// line's end, inside the PAD bytes every device blob carries), then lane l encodes output words l, l+32, ...: 3 line
// bytes -> one 4-byte word, stored at a 4-byte aligned address (payload lengths are multiples of 4), coalesced.
__global__ void __launch_bounds__(CTA_THREADS, 5) dapr_write_kernel(SinkSrc s, DaprOut o) {
  __shared__ DaprShared sh;
  const int l = lane_id(), w = threadIdx.x >> 5;
  const uint8_t* sm = (const uint8_t*)sh.line[w];
  const uint64_t warps = (uint64_t)gridDim.x * WARPS_PER_CTA;
  for (uint64_t i = blockIdx.x * (uint64_t)WARPS_PER_CTA + w; i < s.n; i += warps) {
    if (s.status[i] != TGI_ST_EMITTED) continue;  // warp-uniform
    const uint64_t lo = s.line_off[i], len = s.line_off[i + 1] - lo;
    uint32_t* out = (uint32_t*)(o.data + o.data_off[i]);
    for (uint64_t c0 = 0; c0 < len; c0 += DAPR_CHUNK) {
      const uint32_t m = len - c0 < (uint64_t)DAPR_CHUNK ? (uint32_t)(len - c0) : (uint32_t)DAPR_CHUNK;
      const uintptr_t a = (uintptr_t)(s.jsonl + lo + c0);
      const uint32_t shift = (uint32_t)(a & 15);
      const uint4* src = (const uint4*)(a - shift);
      const uint32_t nvec = (shift + m + 15) >> 4;
      uint4 v0, v1;
      if (l < nvec) v0 = __ldg(src + l);
      if (l + 32 < nvec) v1 = __ldg(src + l + 32);
      if (l < nvec) sh.line[w][l] = v0;
      if (l + 32 < nvec) sh.line[w][l + 32] = v1;
      __syncwarp();
      const uint32_t words = (m + 2) / 3;
      uint32_t* dst = out + c0 / 3;
#pragma unroll
      for (int k = 0; k < DAPR_CHUNK / 96; k++) {
        const uint32_t q = l + 32 * k;
        if (q < words) {
          // written out rather than through b64_word: with its byte count m - 3q the compiler cannot rule out the
          // wrap-around, and this loop grows by 16 instructions
          const uint32_t b = 3 * q;
          const uint32_t x = ((uint32_t)sm[shift + b] << 16) | (b + 1 < m ? (uint32_t)sm[shift + b + 1] << 8 : 0u) |
                             (b + 2 < m ? (uint32_t)sm[shift + b + 2] : 0u);
          const uint32_t c2 = b + 1 < m ? b64_char((x >> 6) & 63) : '=';
          const uint32_t c3 = b + 2 < m ? b64_char(x & 63) : '=';
          dst[q] = b64_char(x >> 18) | (b64_char((x >> 12) & 63) << 8) | (c2 << 16) | (c3 << 24);
        }
      }
      __syncwarp();
    }
    // the path: prefix | channelID | "/posts/" | [number "-"] PostUID | ".jsonl", one byte per lane and step
    const DaprPath p = dapr_path(s, i);
    if (p.num_len && l == 0) {
      const int k = render_i64(sh.num[w], p.num);
      sh.num[w][k] = '-';
    }
    __syncwarp();
    uint8_t* dp = o.path + o.path_off[i];
    const uint64_t e0 = o.prefix_len, e1 = e0 + p.chan_len, e2 = e1 + 7, e3 = e2 + p.num_len, e4 = e3 + p.uid_len,
                   e5 = e4 + 6;
    for (uint64_t j = l; j < e5; j += 32) {
      uint32_t c;
      if (j < e0) c = ldb(o.prefix + j);
      else if (j < e1) c = ldb(p.chan + (j - e0));
      else if (j < e2) c = (uint32_t)(DAPR_POSTS >> (8 * (j - e1))) & 0xFF;
      else if (j < e3) c = sh.num[w][j - e2];
      else if (j < e4) c = ldb(p.uid + (j - e3));
      else c = (uint32_t)(DAPR_JSONL >> (8 * (j - e4))) & 0xFF;
      dp[j] = (uint8_t)c;
    }
    __syncwarp();
  }
}

}  // namespace tgi
