// combine.cuh — the chunk combiner's combined-posts blobs (chunk/main.go:292-421 + DaprStateManager.UploadCombinedFile,
// state/daprstate.go:3734-3777) for lines that are still resident on the device (sm_90a).
//
// A blob's binding Data is base64.StdEncoding of its lines, concatenated.  Base64 is a streaming code, so the open blob
// is kept ENCODED: every call encodes its new line bytes once, behind what the open blob already holds, and only the
// 0-2 bytes that do not fill a 3-byte group wait in a small pending buffer.  One launch encodes a list of tasks; a task
// is one output stream (a blob, or the open blob's continuation) whose input is a short list of byte segments: the
// pending bytes, then runs of kept lines in the result's JSONL (a dropped line splits a run).
//
// Work is mapped from the output side: a thread owns one 16-byte aligned output vector (4 base64 words, 12 input bytes),
// reads its 12 bytes with two aligned 16-byte loads and a funnel shift, and stores one uint4.  The 0-3 words in front of
// a task's first aligned vector belong to its unit 0, which also writes the pending tail of a task that stays open.  Only
// a window that straddles two segments is assembled byte by byte.
#pragma once
#include "sink_src.cuh"

namespace tgi {

struct CbSeg {
  uint64_t pos;        // the segment's first byte in its task's input stream
  uint64_t len;
  const uint8_t* src;  // device bytes; at least 16 readable bytes behind src + len (PAD)
};
struct CbTask {
  uint8_t* dst;        // where its first base64 word goes (4-byte aligned)
  uint64_t bytes;      // input bytes
  uint64_t unit0;      // its first unit in the launch
  uint32_t seg0, nseg; // its segments
  uint32_t last;       // 1: the blob ends here ('=' padding); 0: bytes % 3 wait in CbLaunch::pend_out
};
constexpr int CB_INLINE = 4;  // tasks / segments that travel in the launch parameters (the page call's one task)
struct CbLaunch {
  const CbTask* tasks;  // device tables, or nullptr: t / s below
  const CbSeg* segs;
  uint32_t n_tasks;
  uint64_t units;
  uint8_t* pend_out;
  CbTask t[CB_INLINE];
  CbSeg s[CB_INLINE];
};

__host__ __device__ inline uint64_t cb_words(const CbTask& t) { return t.last ? (t.bytes + 2) / 3 : t.bytes / 3; }
// words before the task's first 16-byte aligned output vector
__host__ __device__ inline uint64_t cb_head(const CbTask& t) {
  const uint64_t h = ((16 - ((uintptr_t)t.dst & 15)) & 15) >> 2, w = cb_words(t);
  return h < w ? h : w;
}
// threads of a task: unit 0 (the head words, the pending tail), then one per 4 words
__host__ __device__ inline uint64_t cb_units(const CbTask& t) { return 1 + (cb_words(t) - cb_head(t) + 3) / 4; }

// byte k of task input at position q (byte by byte across segments; segment j covers q)
DEVI uint32_t cb_byte(const CbSeg* sg, uint32_t& j, uint32_t nseg, uint64_t q) {
  while (j + 1 < nseg && q >= sg[j + 1].pos) j++;
  return ldb(sg[j].src + (q - sg[j].pos));
}

__global__ void __launch_bounds__(256) combine_encode_kernel(const __grid_constant__ CbLaunch L) {
  const CbTask* tasks = L.tasks ? L.tasks : L.t;
  const CbSeg* segs = L.segs ? L.segs : L.s;
  // a thread's units increase, and tasks and segments are long: the current task and segment stay in registers, and
  // the binary searches run only when a unit leaves them
  CbTask t{};
  uint64_t t_end = 0;  // one past the cached task's last unit (0: none cached)
  CbSeg sc{0, 0, nullptr};
  uint32_t jc = 0;     // the cached segment's index in its task
  for (uint64_t u = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; u < L.units; u += (uint64_t)gridDim.x * blockDim.x) {
    if (u >= t_end || u < t.unit0) {
      uint32_t lo = 0, hi = L.n_tasks - 1;  // the last task with unit0 <= u
      while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (tasks[mid].unit0 <= u) lo = mid;
        else hi = mid - 1;
      }
      t = tasks[lo];
      t_end = t.unit0 + cb_units(t);
      sc.len = 0;
    }
    const CbSeg* sg = segs + t.seg0;
    const uint64_t k = u - t.unit0, words = cb_words(t), head = cb_head(t);
    const uint64_t w0 = k == 0 ? 0 : head + 4 * (k - 1);
    const uint64_t w1 = k == 0 ? head : (w0 + 4 < words ? w0 + 4 : words);
    if (k == 0 && !t.last) {  // the pending tail: bytes % 3 of a task that stays open
      const uint64_t q0 = t.bytes / 3 * 3;
      uint32_t j = 0;
      for (uint64_t q = q0; q < t.bytes; q++) L.pend_out[q - q0] = (uint8_t)cb_byte(sg, j, t.nseg, q);
    }
    if (w0 >= w1) continue;
    const uint64_t q = 3 * w0;
    const uint32_t m = (uint32_t)((3 * w1 < t.bytes ? 3 * w1 : t.bytes) - q);  // input bytes of this unit, <= 12
    if (q < sc.pos || q >= sc.pos + sc.len) {  // the segment that holds q
      uint32_t a = 0, b = t.nseg - 1;
      while (a < b) {
        const uint32_t mid = (a + b + 1) >> 1;
        if (sg[mid].pos <= q) a = mid;
        else b = mid - 1;
      }
      jc = a;
      sc = sg[a];
    }
    uint32_t j = jc;
    uint32_t r0 = 0, r1 = 0, r2 = 0;  // the unit's input bytes, little-endian
    if (q + m <= sc.pos + sc.len) {  // inside one segment: two aligned 16-byte loads and a funnel shift
      // written out rather than through ld16_unaligned, whose fourth word this unit does not need: that version ran
      // 0.8 % slower (H100 80GB HBM3, 400 W)
      const uintptr_t a = (uintptr_t)(sc.src + (q - sc.pos));
      const uint4* p = (const uint4*)(a & ~(uintptr_t)15);
      const uint4 v0 = __ldg(p), v1 = __ldg(p + 1);
      const uint32_t sh = (uint32_t)(a & 15), kw = sh >> 2, bs = 8 * (sh & 3);
      const uint32_t x0 = kw == 0 ? v0.x : kw == 1 ? v0.y : kw == 2 ? v0.z : v0.w;
      const uint32_t x1 = kw == 0 ? v0.y : kw == 1 ? v0.z : kw == 2 ? v0.w : v1.x;
      const uint32_t x2 = kw == 0 ? v0.z : kw == 1 ? v0.w : kw == 2 ? v1.x : v1.y;
      const uint32_t x3 = kw == 0 ? v0.w : kw == 1 ? v1.x : kw == 2 ? v1.y : v1.z;
      r0 = __funnelshift_r(x0, x1, bs);
      r1 = __funnelshift_r(x1, x2, bs);
      r2 = __funnelshift_r(x2, x3, bs);
    } else {  // the window straddles segments
      uint64_t lo64 = 0;
      uint32_t hi32 = 0;
      for (uint32_t i = 0; i < m; i++) {
        const uint32_t c = cb_byte(sg, j, t.nseg, q + i);
        if (i < 8) lo64 |= (uint64_t)c << (8 * i);
        else hi32 |= c << (8 * (i - 8));
      }
      r0 = (uint32_t)lo64;
      r1 = (uint32_t)(lo64 >> 32);
      r2 = hi32;
    }
    // word i takes bytes 3i..3i+2 of r0|r1|r2
    const uint32_t o0 = b64_word(r0 & 0xFF, (r0 >> 8) & 0xFF, (r0 >> 16) & 0xFF, m);
    const uint32_t o1 = b64_word(r0 >> 24, r1 & 0xFF, (r1 >> 8) & 0xFF, m > 3 ? m - 3 : 0);
    const uint32_t o2 = b64_word((r1 >> 16) & 0xFF, r1 >> 24, r2 & 0xFF, m > 6 ? m - 6 : 0);
    const uint32_t o3 = b64_word((r2 >> 8) & 0xFF, (r2 >> 16) & 0xFF, r2 >> 24, m > 9 ? m - 9 : 0);
    uint32_t* out = (uint32_t*)(t.dst + 4 * w0);
    const uint32_t nw = (uint32_t)(w1 - w0);
    if (k != 0 && nw == 4) {
      *(uint4*)out = make_uint4(o0, o1, o2, o3);
    } else {
      out[0] = o0;
      if (nw > 1) out[1] = o1;
      if (nw > 2) out[2] = o2;
      if (nw > 3) out[3] = o3;
    }
  }
}

// the lines longer than hard_cap (chunk/main.go:316-322), unordered; there are at most jsonl_len / (hard_cap + 1)
__global__ void combine_drops_kernel(const uint64_t* line_off, uint64_t n, uint64_t hard_cap, uint64_t* list, uint64_t cap,
                                     unsigned long long* count) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    if (line_off[i + 1] - line_off[i] > hard_cap) {
      const unsigned long long k = atomicAdd(count, 1ull);
      if (k < cap) list[k] = i;
    }
  }
}

// posts per group: a kept line i (0 < length <= hard_cap) belongs to the first group g with i < ends[g], or to the open
// group (index n_groups) behind the last end.  One atomic per warp and group.
__global__ void combine_count_kernel(const uint64_t* line_off, uint64_t n, uint64_t hard_cap, const uint64_t* ends,
                                     uint32_t n_groups, unsigned long long* counts) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t base = blockIdx.x * (uint64_t)blockDim.x; base < n; base += stride) {  // warp-uniform trip count
    const uint64_t i = base + threadIdx.x;
    uint32_t g = 0;
    bool kept = false;
    if (i < n) {
      const uint64_t len = line_off[i + 1] - line_off[i];
      kept = len > 0 && len <= hard_cap;
      uint32_t a = 0, b = n_groups;  // the first g with i < ends[g]; n_groups if none
      while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        if (i < ends[mid]) b = mid;
        else a = mid + 1;
      }
      g = a;
    }
    const uint32_t kept_mask = __ballot_sync(FULL, kept), peers = __match_any_sync(FULL, g);
    if (lane_id() == __ffs(peers) - 1) {
      const uint32_t c = __popc(peers & kept_mask);
      if (c) atomicAdd(counts + g, (unsigned long long)c);
    }
  }
}

}  // namespace tgi
