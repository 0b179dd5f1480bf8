// local_appends.cuh — LocalStateManager.StorePost (state/storageproviders.go:39-53, 275-298) for a whole batch result
// whose lines are still resident on the device (sm_90a): the lines grouped by channel, so that the host appends ONE
// byte range per posts.jsonl file instead of opening, appending to and closing the file once per post.
//
// The grouping key is the channelID byte string (Telegram: the channel row's name; YouTube: the row's id), so two rows
// that name one channel are one group.  Inside a group lines stay in record order; groups are ordered by their first
// line.  Pipeline (every step one launch or one launch_scan, no host round trip in between):
//   1. canonical row: a hash table over the channelID bytes maps every row to the lowest row with the same bytes;
//   2. lines: the emitted, non-empty records, compacted in record order (flag + scan); each canonical channel keeps the
//      index of its first line (atomicMin);
//   3. runs: maximal spans of consecutive lines of one canonical channel (flag + scan); groups: the lines that are
//      their channel's first line (flag + scan), so a group's id is the rank of its first line;
//   4. a stable LSD radix sort of the runs by group id, 8 bits or fewer per pass, with a block-local stable scatter;
//   5. an exclusive scan of the run line counts in sorted order places every line in `order`, a scan of the line
//      lengths in that order gives every run its destination byte, and the gather copies the bytes, mapped from the
//      output side: a thread per 16-byte output vector.
// Sizes the host does not know yet (lines, runs, groups) stay on the device: kernels are launched for their upper
// bounds (records, channel rows) and read the exact counts from the scalars block.
#pragma once
#include "sink_src.cuh"

namespace tgi {

constexpr uint32_t LA_NONE = 0xFFFFFFFFu;
constexpr int LA_THREADS = 256;
// radix sort: a tile of RS_TILE runs per CTA; warp w owns RS_ROUNDS * 32 consecutive runs of it
constexpr int RS_WARPS = 8, RS_ROUNDS = 8, RS_TILE = RS_WARPS * RS_ROUNDS * 32, RS_RADIX = 256;
// gather: a CTA copies LA_GATHER_ITEMS * LA_THREADS consecutive output vectors per step (64 KiB)
constexpr int LA_GATHER_ITEMS = 16;
// the scalars block: counts the scans leave on the device
enum { LA_SC_LINES, LA_SC_RUNS, LA_SC_GROUPS, LA_SC_SORTED_LINES, LA_SC_BYTES, LA_SC_RADIX, LA_SC_COUNT };

struct LaWork {
  uint64_t* sc;           // LA_SC_*
  uint32_t* table;        // channelID hash table: a row of each distinct channelID, the lowest once inserted
  uint64_t tmask;
  uint32_t* canon;        // [n_chans] lowest row with the same channelID
  uint32_t* first_line;   // [n_chans] (canonical rows) the channel's first line, LA_NONE: none
  uint32_t* flag;         // [n] line flags, then run flags
  uint32_t* gflag;        // [n] group flags
  uint64_t* pos;          // [n+1] scans of flag (lines), flag (runs), gflag (groups)
  uint64_t* rpos;
  uint64_t* gpos;
  uint32_t* lrec;         // [lines] record of every line
  uint32_t* lkey;         // [lines] canonical row of every line
  uint32_t* run_start;    // [runs+1] first line of every run
  uint32_t* keys[2];      // radix ping-pong: group id, run index
  uint32_t* vals[2];
  uint32_t* cnt;          // [n] lines of every run, sorted order; then line lengths, grouped order
  uint64_t* lpos;         // [n+1] scans of cnt: first grouped line of every sorted run, then byte offsets of lines
  uint64_t* goff;
  uint32_t* inv;          // [runs] first grouped line of every run, by run index
  uint64_t* rsrc;         // [runs] sorted runs: source byte in jsonl
  uint64_t* rdst;         // [runs+1] sorted runs: destination byte in data
  tgi_channel_group* groups;  // [groups]
  uint64_t* order;        // [lines] record index of every grouped line
  uint8_t* data;          // grouped line bytes
};

DEVI uint64_t la_hash(const uint8_t* p, uint32_t len) {  // FNV-1a over every byte, then a final mix
  uint64_t h = 0xcbf29ce484222325ull ^ len;
  for (uint32_t k = 0; k < len; k++) h = (h ^ ldb(p + k)) * 0x100000001b3ull;
  return h ^ (h >> 31);
}

DEVI bool la_same_id(const SinkSrc& s, uint32_t a, const uint8_t* p, uint32_t len) {
  uint32_t la;
  const uint8_t* q = sink_chan_id(s, a, la);
  if (la != len) return false;
  for (uint32_t k = 0; k < len; k++)
    if (ldb(q + k) != ldb(p + k)) return false;
  return true;
}

// 1a. every row into the table (emptied to LA_NONE): a slot, once claimed, only ever holds rows of one channelID, and
// atomicMin leaves the lowest of them
__global__ void la_canon_insert_kernel(SinkSrc s, LaWork w) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < s.n_chans; i += gridDim.x * blockDim.x) {
    uint32_t len;
    const uint8_t* p = sink_chan_id(s, i, len);
    for (uint64_t slot = la_hash(p, len) & w.tmask;; slot = (slot + 1) & w.tmask) {
      const uint32_t prev = atomicCAS(w.table + slot, LA_NONE, i);
      if (prev == LA_NONE) break;
      if (la_same_id(s, prev, p, len)) {
        atomicMin(w.table + slot, i);
        break;
      }
    }
  }
}

// 1b. every row's canonical row; 2a. the line flag of every record (emitted with a non-empty line)
__global__ void la_canon_flag_kernel(SinkSrc s, LaWork w) {
  const uint64_t end = s.n > s.n_chans ? s.n : s.n_chans;
  for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < end; t += (uint64_t)gridDim.x * blockDim.x) {
    if (t < s.n_chans) {
      uint32_t len;
      const uint8_t* p = sink_chan_id(s, (uint32_t)t, len);
      uint64_t slot = la_hash(p, len) & w.tmask;
      while (!la_same_id(s, w.table[slot], p, len)) slot = (slot + 1) & w.tmask;
      w.canon[t] = w.table[slot];
    }
    if (t < s.n) w.flag[t] = s.status[t] == TGI_ST_EMITTED && s.line_off[t + 1] > s.line_off[t];
  }
}

// 2b. compaction: line j = pos[i] of record i; its canonical channel keeps its first line
__global__ void la_compact_kernel(SinkSrc s, LaWork w) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < s.n; i += (uint64_t)gridDim.x * blockDim.x) {
    if (!w.flag[i]) continue;
    const uint32_t j = (uint32_t)w.pos[i];
    const uint32_t key = w.canon[sink_rec_chan(s, i)];
    w.lrec[j] = (uint32_t)i;
    w.lkey[j] = key;
    atomicMin(w.first_line + key, j);
  }
}

// 3a. run flags (a line whose channel differs from the line before) and group flags (its channel's first line); zero
// past the last line, where the scans still read
__global__ void la_flags_kernel(uint64_t n, LaWork w) {
  const uint64_t m = w.sc[LA_SC_LINES];
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t rf = 0, gf = 0;
    if (j < m) {
      const uint32_t k = w.lkey[j];
      rf = j == 0 || w.lkey[j - 1] != k;
      gf = w.first_line[k] == j;
    }
    w.flag[j] = rf;
    w.gflag[j] = gf;
  }
}

// 3b. the run table: first line and group id of every run; the radix sort's input pairs (group id, run index)
__global__ void la_runs_kernel(uint64_t n, LaWork w) {
  const uint64_t m = w.sc[LA_SC_LINES];
  if (blockIdx.x == 0 && threadIdx.x == 0) w.run_start[w.sc[LA_SC_RUNS]] = (uint32_t)m;
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < m; j += (uint64_t)gridDim.x * blockDim.x) {
    if (!w.flag[j]) continue;
    const uint32_t r = (uint32_t)w.rpos[j];
    w.run_start[r] = (uint32_t)j;
    w.keys[0][r] = (uint32_t)w.gpos[w.first_line[w.lkey[j]]];
    w.vals[0][r] = r;
  }
}

// 4a. digit counts of one tile of runs, digit-major: counts[d * ntiles + tile]
__global__ void __launch_bounds__(RS_WARPS * 32) la_radix_hist_kernel(const uint32_t* keys, const uint64_t* count,
                                                                      uint32_t shift, uint32_t radix, uint32_t ntiles,
                                                                      uint32_t* counts) {
  __shared__ uint32_t h[RS_RADIX];
  for (uint32_t d = threadIdx.x; d < radix; d += blockDim.x) h[d] = 0;
  __syncthreads();
  const uint64_t n = *count, base = (uint64_t)blockIdx.x * RS_TILE;
  for (uint32_t t = threadIdx.x; t < RS_TILE; t += blockDim.x)
    if (base + t < n) atomicAdd(h + ((keys[base + t] >> shift) & (radix - 1)), 1u);
  __syncthreads();
  for (uint32_t d = threadIdx.x; d < radix; d += blockDim.x) counts[(uint64_t)d * ntiles + blockIdx.x] = h[d];
}

// 4b. stable scatter of one tile: off[d * ntiles + tile] (the scan of the counts) is where the tile's runs with digit d
// start.  Warp w walks its runs in order, 32 at a time: __match_any_sync finds the lanes with the same digit, and a
// run's rank is the number of such lanes below it plus the runs of that digit the warp already placed.  The first walk
// counts per warp and digit, the prefix over the warps turns the counts into starts, the second walk places.
__global__ void __launch_bounds__(RS_WARPS * 32) la_radix_scatter_kernel(const uint32_t* kin, const uint32_t* vin,
                                                                         uint32_t* kout, uint32_t* vout,
                                                                         const uint64_t* count, uint32_t shift,
                                                                         uint32_t radix, uint32_t ntiles,
                                                                         const uint64_t* off) {
  __shared__ uint32_t wh[RS_WARPS][RS_RADIX];
  const int l = lane_id(), w = threadIdx.x >> 5;
  for (uint32_t d = threadIdx.x; d < RS_WARPS * RS_RADIX; d += blockDim.x) (&wh[0][0])[d] = 0;
  __syncthreads();
  const uint64_t n = *count, base = (uint64_t)blockIdx.x * RS_TILE + (uint64_t)w * (RS_ROUNDS * 32);
  uint32_t kk[RS_ROUNDS], vv[RS_ROUNDS];
#pragma unroll
  for (int k = 0; k < RS_ROUNDS; k++) {
    const uint64_t i = base + k * 32 + l;
    const bool ok = i < n;
    kk[k] = ok ? kin[i] : 0;
    vv[k] = ok ? vin[i] : 0;
    const uint32_t d = ok ? (kk[k] >> shift) & (radix - 1) : LA_NONE;
    const uint32_t peers = __match_any_sync(FULL, d);
    if (ok && l == __ffs(peers) - 1) wh[w][d] += __popc(peers);
    __syncwarp();
  }
  __syncthreads();
  for (uint32_t d = threadIdx.x; d < radix; d += blockDim.x) {
    uint32_t run = (uint32_t)off[(uint64_t)d * ntiles + blockIdx.x];
    for (int x = 0; x < RS_WARPS; x++) {
      const uint32_t c = wh[x][d];
      wh[x][d] = run;
      run += c;
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < RS_ROUNDS; k++) {
    const bool ok = base + k * 32 + l < n;
    const uint32_t d = ok ? (kk[k] >> shift) & (radix - 1) : LA_NONE;
    const uint32_t peers = __match_any_sync(FULL, d);
    if (ok) {
      const uint32_t dst = wh[w][d] + __popc(peers & ((1u << l) - 1));
      kout[dst] = kk[k];
      vout[dst] = vv[k];
    }
    __syncwarp();
    if (ok && l == __ffs(peers) - 1) wh[w][d] += __popc(peers);
    __syncwarp();
  }
}

// 5a. lines of every run in sorted order (zero past the last run, where the scan still reads)
__global__ void la_sorted_counts_kernel(uint64_t n, const uint32_t* sorted, LaWork w) {
  const uint64_t runs = w.sc[LA_SC_RUNS];
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < n; k += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t c = 0;
    if (k < runs) {
      const uint32_t r = sorted[k];
      c = w.run_start[r + 1] - w.run_start[r];
    }
    w.cnt[k] = c;
  }
}

// 5b. the first grouped line of every run, by run index
__global__ void la_inverse_kernel(const uint32_t* sorted, LaWork w) {
  const uint64_t runs = w.sc[LA_SC_RUNS];
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < runs; k += (uint64_t)gridDim.x * blockDim.x)
    w.inv[sorted[k]] = (uint32_t)w.lpos[k];
}

// 5c. `order` and the line lengths in grouped order: line j of run r goes to inv[r] + (j - run_start[r])
__global__ void la_order_kernel(SinkSrc s, LaWork w) {
  const uint64_t m = w.sc[LA_SC_LINES];
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < s.n; j += (uint64_t)gridDim.x * blockDim.x) {
    if (j >= m) {
      w.cnt[j] = 0;  // grouped positions past the last line
      continue;
    }
    const uint32_t r = (uint32_t)w.rpos[j + 1] - 1;  // the run of line j: run flags up to and including j, minus one
    const uint64_t d = w.inv[r] + (j - w.run_start[r]);
    const uint32_t i = w.lrec[j];
    w.order[d] = i;
    w.cnt[d] = (uint32_t)(s.line_off[i + 1] - s.line_off[i]);
  }
}

// 5d. source and destination byte of every sorted run; the group table (n_lines holds the group's first grouped line
// and byte_len 0 until the host turns neighbours into lengths)
__global__ void la_tables_kernel(SinkSrc s, const uint32_t* sorted_keys, const uint32_t* sorted, LaWork w) {
  const uint64_t runs = w.sc[LA_SC_RUNS];
  if (blockIdx.x == 0 && threadIdx.x == 0) w.rdst[runs] = w.sc[LA_SC_BYTES];
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < runs; k += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t r = sorted[k], j0 = w.run_start[r], i0 = w.lrec[j0];
    const uint64_t line = w.lpos[k], dst = w.goff[line];
    w.rsrc[k] = s.line_off[i0];
    w.rdst[k] = dst;
    const uint32_t g = sorted_keys[k];
    if (k == 0 || sorted_keys[k - 1] != g) w.groups[g] = tgi_channel_group{w.lkey[j0], 0, line, i0, dst, 0};
  }
}

// 5e. the gather, mapped from the output side: a thread per 16-byte output vector (data is 256-byte aligned).  A CTA
// takes LA_GATHER_ITEMS * LA_THREADS consecutive vectors per step; a thread's vectors are 4 KiB apart, so its current
// run stays in registers and a later run is found by a few steps forward or by a binary search.  A vector inside one
// run is read with one or two aligned 16-byte loads and funnel shifts (the loads stay within 16 bytes of the run's end,
// inside the PAD bytes every device blob carries); a vector across runs is assembled byte by byte.
__global__ void __launch_bounds__(LA_THREADS) la_gather_kernel(SinkSrc s, LaWork w, uint64_t total) {
  const uint64_t runs = w.sc[LA_SC_RUNS], vecs = (total + 15) / 16;
  uint64_t k = 0, lo = w.rdst[0], hi = w.rdst[1], src = w.rsrc[0];  // the cached run: dest [lo, hi) from jsonl + src
  auto seek = [&](uint64_t q) {  // the run that holds destination byte q
    if (q >= lo && q < hi) return;
    if (q >= hi && k + 4 < runs && q < w.rdst[k + 5]) {
      while (q >= w.rdst[k + 1]) k++;
    } else {
      uint64_t a = q >= hi ? k + 1 : 0, b = runs - 1;  // the last run with rdst <= q
      while (a < b) {
        const uint64_t mid = (a + b + 1) >> 1;
        if (w.rdst[mid] <= q) a = mid;
        else b = mid - 1;
      }
      k = a;
    }
    lo = w.rdst[k];
    hi = w.rdst[k + 1];
    src = w.rsrc[k];
  };
  const uint64_t step = (uint64_t)LA_GATHER_ITEMS * LA_THREADS;
  for (uint64_t v0 = blockIdx.x * step; v0 < vecs; v0 += (uint64_t)gridDim.x * step) {
#pragma unroll 4
    for (int it = 0; it < LA_GATHER_ITEMS; it++) {
      const uint64_t v = v0 + (uint64_t)it * LA_THREADS + threadIdx.x;
      if (v >= vecs) break;
      const uint64_t q = 16 * v;
      const uint32_t nb = total - q < 16 ? (uint32_t)(total - q) : 16u;
      seek(q);
      uint32_t r[4];
      if (q + nb <= hi) {
        // not ld16_unaligned: the second load only when the bytes reach into it, which keeps the config-2 gather 3 %
        // faster (H100 80GB HBM3, 400 W)
        const uintptr_t a = (uintptr_t)(s.jsonl + src + (q - lo));
        const uint4* p = (const uint4*)(a & ~(uintptr_t)15);
        const uint32_t sh = (uint32_t)(a & 15), kw = sh >> 2, bs = 8 * (sh & 3);
        const uint4 v0w = __ldg(p), v1w = sh + nb > 16 ? __ldg(p + 1) : make_uint4(0, 0, 0, 0);
        const uint32_t x[8] = {v0w.x, v0w.y, v0w.z, v0w.w, v1w.x, v1w.y, v1w.z, v1w.w};
        uint32_t y[5];
#pragma unroll
        for (int t = 0; t < 5; t++) y[t] = kw == 0 ? x[t] : kw == 1 ? x[t + 1] : kw == 2 ? x[t + 2] : x[t + 3];
#pragma unroll
        for (int t = 0; t < 4; t++) r[t] = __funnelshift_r(y[t], y[t + 1], bs);
      } else {
        uint64_t b0 = 0, b1 = 0;  // bytes 0-7 and 8-15, little-endian
        for (uint32_t b = 0; b < nb; b++) {
          seek(q + b);
          const uint64_t x = ldb(s.jsonl + src + (q + b - lo));
          if (b < 8) b0 |= x << (8 * b);
          else b1 |= x << (8 * (b - 8));
        }
        r[0] = (uint32_t)b0, r[1] = (uint32_t)(b0 >> 32), r[2] = (uint32_t)b1, r[3] = (uint32_t)(b1 >> 32);
      }
      if (nb == 16) {
        *(uint4*)(w.data + q) = make_uint4(r[0], r[1], r[2], r[3]);
      } else {  // the last vector of the blob
        const uint64_t b0 = r[0] | (uint64_t)r[1] << 32, b1 = r[2] | (uint64_t)r[3] << 32;
        for (uint32_t b = 0; b < nb; b++) w.data[q + b] = (uint8_t)((b < 8 ? b0 >> (8 * b) : b1 >> (8 * (b - 8))) & 0xFF);
      }
    }
  }
}

}  // namespace tgi
