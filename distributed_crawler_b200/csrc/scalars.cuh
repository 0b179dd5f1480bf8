// scalars.cuh — the per-batch scalars block (u64 words) and the device error bits, shared by the kernels that write
// them and the host code that reads them back.
#pragma once

namespace tgi {

// Words of the scalars block.  [SC_CURSOR] holds two 32-bit halves: the link arena's fill (u32), then the error word.
enum {
  SC_CHAN_TOTAL = 0,
  SC_LINE_TOTAL = 1,
  SC_CURSOR = 2,
  SC_NEW = 3,
  SC_FSIZE = 4,
  SC_LINK_TOTAL = 5,
  SC_LONG = 6,
  SC_URL_CURSOR = 7,
  SC_LANE_OUT = 8,
  SC_LANE_IN = 9,
  SC_LISTS = 10,  // 3 x u32
  SC_COUNT = 12,
};
// page kernels: scalars[PAGE_TRACE_AT ..] = phase clock (start, after each barrier, end), then the slowest record of
// each of the three per-record phases
constexpr int PAGE_TRACE_AT = 16, PAGE_PHASES = 7;

// bits of the error word, OR'd in by the kernels
enum : int {
  ERR_ARENA_OVERFLOW = 1,
  ERR_TOO_MANY_REACTIONS = 2,
  ERR_FRONTIER_FULL = 4,
  ERR_TOO_MANY_LINKS = 8,
  ERR_LINE_MISMATCH = 16,  // sized and emitted line lengths disagree: never expected
  ERR_PAGE_OVERFLOW = 64,  // a page kernel's result block or channel blob is too small: the host runs the bulk pipeline
};

}  // namespace tgi
