// radix.cuh — the kernels of a stable LSD radix sort of (key, value) pairs (sm_90a): one pass over a digit of `radix`
// (256 or fewer) values is a histogram per tile, an exclusive scan of the counts, digit-major, and a block-local stable
// scatter.  The local sink groups its runs by channel with it, the progress state its live messages by page row; the
// host runs the passes with radix_sort (tgingest.cu).  The pair count is read from the device.
#pragma once
#include "dev_common.cuh"

namespace tgi {

// a tile of RS_TILE pairs per CTA; warp w owns RS_ROUNDS * 32 consecutive pairs of it
constexpr int RS_WARPS = 8, RS_ROUNDS = 8, RS_TILE = RS_WARPS * RS_ROUNDS * 32, RS_RADIX = 256;

// digit counts of one tile of pairs, digit-major: counts[d * ntiles + tile]
__global__ void __launch_bounds__(RS_WARPS * 32) radix_hist_kernel(const uint32_t* keys, const uint64_t* count, uint32_t shift,
                                                                   uint32_t radix, uint32_t ntiles, uint32_t* counts) {
  __shared__ uint32_t h[RS_RADIX];
  for (uint32_t d = threadIdx.x; d < radix; d += blockDim.x) h[d] = 0;
  __syncthreads();
  const uint64_t n = *count, base = (uint64_t)blockIdx.x * RS_TILE;
  for (uint32_t t = threadIdx.x; t < RS_TILE; t += blockDim.x)
    if (base + t < n) atomicAdd(h + ((keys[base + t] >> shift) & (radix - 1)), 1u);
  __syncthreads();
  for (uint32_t d = threadIdx.x; d < radix; d += blockDim.x) counts[(uint64_t)d * ntiles + blockIdx.x] = h[d];
}

// stable scatter of one tile: off[d * ntiles + tile] (the scan of the counts) is where the tile's pairs with digit d
// start.  Warp w walks its pairs in order, 32 at a time: __match_any_sync finds the lanes with the same digit, and a
// pair's rank is the number of such lanes below it plus the pairs of that digit the warp already placed.  The first walk
// counts per warp and digit, the prefix over the warps turns the counts into starts, the second walk places.  Lanes
// past the last pair take the digit 0xFFFFFFFF, which no pair has.
__global__ void __launch_bounds__(RS_WARPS * 32) radix_scatter_kernel(const uint32_t* kin, const uint32_t* vin, uint32_t* kout,
                                                                      uint32_t* vout, const uint64_t* count, uint32_t shift,
                                                                      uint32_t radix, uint32_t ntiles, const uint64_t* off) {
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
    const uint32_t d = ok ? (kk[k] >> shift) & (radix - 1) : 0xFFFFFFFFu;
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
    const uint32_t d = ok ? (kk[k] >> shift) & (radix - 1) : 0xFFFFFFFFu;
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

}  // namespace tgi
