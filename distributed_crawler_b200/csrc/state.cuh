// state.cuh — the crawl's progress state (state.State: layers of pages, each page with its messages) resident on the
// device (sm_90a): the batched UpdateMessage (state/base.go:182-215) and json.Marshal(GetState()) (base.go:345-372,
// state/storageproviders.go:246-272) over a table that stays in HBM between calls.
//
// Layout (the host keeps the layers and a mirror of the page rows, tgingest.cu):
//   page rows   tgi_state_page[rows], its nine strings in one blob; one row per page id (pageMap), replaced in place.
//   row_gen     [rows] generation of the row's message list: UpdatePage / an overwriting AddLayer bump it, and every
//               message row of an older generation is a tombstone.
//   row_cnt     [rows] live messages of the row.
//   messages    StMsg[n], appended; a row's live messages in storage order ARE its message list in order.
//   table       open-addressed (row, gen, chat_id, message_id) -> lowest message index: the gen in the key keeps
//               tombstones out of every lookup; the table is rebuilt from the live rows when the messages compact.
//
// Render: live messages are compacted and grouped by row with the stable radix sort of radix.cuh (order inside a
// row = storage order); a thread per message sizes it, a warp per entry (a page of a layer, or an empty layer)
// sizes the page around its messages, scans place both, and the emit writes every byte at its final offset: a warp per
// entry for the page's fields, a thread per (entry, message) slot for the messages.
//
// DaprStateManager's side: the exports (daprstate.go:2911-3012, storageproviders.go:550-587) run the same passes with
// st_entry in line mode, one {page}\n per entry; json.Marshal(layerMap) (daprstate.go:947) is a thread per listed id.
//
// Page turns (crawl/runner.go:1132-1211): a thread per fetched key probes the table at the row's current generation and
// records the first fetched index of its message id; the new keys become the row's next generation, and the one page
// renders through the export's line passes over that fresh contiguous segment.  Nothing reads another row's messages.
// The turn's owner keys stay as the row's owner view; the close appends the view as the row's next generation.
//
// Page reads: the rows' fields come from the host mirror; their lists are the live messages of the distinct rows,
// flagged in one pass, grouped by row like the render's and written out in that order.
#pragma once
#include <type_traits>

#include "kernels.cuh"
#include "radix.cuh"

namespace tgi {

constexpr uint32_t ST_NONE = 0xFFFFFFFFu;
constexpr int ST_THREADS = 256;

struct StMsg {  // 32 bytes: one state.Message
  long long chat, msg;
  uint32_t row, gen;  // owning row and the list generation it belongs to
  uint32_t pid;       // row whose id is its pageId
  uint16_t status, platform;  // string-table codes
};

struct StCodes {  // the registered status / platform strings (raw bytes)
  const uint8_t* blob;
  const uint32_t* off;  // [n+1]
};

struct StDev {
  const tgi_state_page* pages;
  const uint8_t* blob;
  uint32_t* row_gen;
  uint32_t* row_cnt;
  StMsg* msgs;
  uint32_t* table;
  uint64_t tmask;
  StCodes codes;
};

DEVI bool st_live(const StDev& d, const StMsg& m) { return m.gen == d.row_gen[m.row]; }

DEVI uint64_t st_hash(uint32_t row, uint32_t gen, long long chat, long long msg) {
  return join_hash(chat ^ (long long)((((uint64_t)row << 32) | gen) * 0x632BE59BD9B4E019ull), msg);
}

// messages [first, end) that are live go into the table; a slot keeps the lowest index of its key (atomicMin)
__global__ void st_table_insert_kernel(StDev d, uint64_t first, uint64_t end) {
  for (uint64_t i = first + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < end; i += (uint64_t)gridDim.x * blockDim.x) {
    const StMsg m = d.msgs[i];
    if (!st_live(d, m)) continue;
    for (uint64_t s = st_hash(m.row, m.gen, m.chat, m.msg) & d.tmask;; s = (s + 1) & d.tmask) {
      const uint32_t cur = atomicCAS(d.table + s, ST_NONE, (uint32_t)i);
      if (cur == ST_NONE) break;
      const StMsg& o = d.msgs[cur];  // an occupant's key never changes
      if (o.row == m.row && o.gen == m.gen && o.chat == m.chat && o.msg == m.msg) {
        atomicMin(d.table + s, (uint32_t)i);
        break;
      }
    }
  }
}

DEVI uint32_t st_lookup(const StDev& d, uint32_t row, uint32_t gen, long long chat, long long msg) {
  for (uint64_t s = st_hash(row, gen, chat, msg) & d.tmask;; s = (s + 1) & d.tmask) {
    const uint32_t cur = d.table[s];
    if (cur == ST_NONE) return ST_NONE;
    const StMsg& o = d.msgs[cur];
    if (o.row == row && o.gen == gen && o.chat == chat && o.msg == msg) return cur;
  }
}

// ---- batched UpdateMessage ------------------------------------------------------------------------------------------
struct StUpd {
  const tgi_state_update* u;  // [n], every row valid (the host drops the unknown-page updates)
  uint64_t n;
  uint32_t* bfirst;  // batch table: lowest update index of the slot's key, ST_NONE = empty
  uint32_t* blast;   // highest update index of the slot's key
  uint64_t bmask;
  uint32_t* slot_of;  // [n] the batch slot of update j
  uint32_t* flag;     // [n] 1: update j leads a key that is not in the page yet (appended)
  uint64_t* pos;      // [n+1] scan of flag
  uint64_t n_msgs;    // message rows before the call
};

DEVI bool st_same_upd(const tgi_state_update& a, const tgi_state_update& b) {
  return a.row == b.row && a.chat_id == b.chat_id && a.message_id == b.message_id;
}

// 1. the batch's distinct (row, chat, message) keys: first occurrence by atomicMin, last writer by atomicMax
__global__ void st_upd_build_kernel(StUpd w) {
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < w.n; j += (uint64_t)gridDim.x * blockDim.x) {
    const tgi_state_update k = w.u[j];
    uint64_t s = st_hash(k.row, 0, k.chat_id, k.message_id) & w.bmask;
    for (;; s = (s + 1) & w.bmask) {
      const uint32_t cur = atomicCAS(w.bfirst + s, ST_NONE, (uint32_t)j);
      if (cur == ST_NONE) break;
      if (st_same_upd(w.u[cur], k)) {
        atomicMin(w.bfirst + s, (uint32_t)j);
        break;
      }
    }
    atomicMax(w.blast + s, (uint32_t)j);  // blast starts at 0
    w.slot_of[j] = (uint32_t)s;
  }
}

// 2. every key's leader (its first update) finds the first live message with the key and gives it the status of the
// key's last update; keys the page does not hold are flagged for appending
__global__ void st_upd_resolve_kernel(StDev d, StUpd w) {
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < w.n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t s = w.slot_of[j];
    uint32_t f = 0;
    if (w.bfirst[s] == (uint32_t)j) {
      const tgi_state_update k = w.u[j];
      const uint32_t hit = st_lookup(d, k.row, d.row_gen[k.row], k.chat_id, k.message_id);
      if (hit != ST_NONE) d.msgs[hit].status = w.u[w.blast[s]].status;
      else f = 1;
    }
    w.flag[j] = f;
  }
}

// 3. the new keys appended in first-occurrence order (pageId = the page itself, no platform) and counted on their row
__global__ void st_upd_append_kernel(StDev d, StUpd w) {
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < w.n; j += (uint64_t)gridDim.x * blockDim.x) {
    if (!w.flag[j]) continue;
    const tgi_state_update k = w.u[j];
    StMsg m;
    m.chat = k.chat_id;
    m.msg = k.message_id;
    m.row = k.row;
    m.gen = d.row_gen[k.row];
    m.pid = k.row;
    m.status = w.u[w.blast[w.slot_of[j]]].status;
    m.platform = 0;
    d.msgs[w.n_msgs + w.pos[j]] = m;
    atomicAdd(d.row_cnt + k.row, 1u);
  }
}

// ---- page turns: processAllMessagesWithProcessor's bookkeeping (crawl/runner.go:1132-1147, 1161-1211) ---------------
// A call covers P pages (distinct rows); page k owns the segment [off[k], off[k+1]) of each of the call's arrays.

// the segment of item i: the last k with off[k] <= i (empty segments share their offset, so this one holds i)
DEVI uint32_t st_seg(const uint64_t* off, uint32_t n_seg, uint64_t i) {
  uint32_t lo = 0, hi = n_seg - 1;
  while (lo < hi) {
    const uint32_t mid = (lo + hi + 1) >> 1;
    if (off[mid] <= i) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

struct StTurn {
  const long long* fetched;  // [n][2] chat_id, message_id in fetch order, page after page
  uint64_t n;
  const uint64_t* foff;      // [P+1] page k's fetched keys
  const uint32_t* prow;      // [P] page k's row
  uint32_t P;
  uint32_t* pg;       // [n] the page of fetched key j
  uint32_t* bfirst;   // batch table keyed by (page, message id): lowest fetched index, ST_NONE = empty
  uint64_t bmask;
  uint32_t* flag;     // [n] 1: fetched key j is not in its page's list (addNewMessages keeps it)
  uint64_t* pos;      // [n+1] scan of flag: the call's new lists, in (page, fetch) order
  uint64_t* woff;     // [P+1] page k's new list is [woff[k], woff[k+1]) of it
  uint64_t n_msgs;    // message rows before the new lists
  long long* keys;    // [n_new][2] the new lists' keys: the turn's owner messages
  uint32_t* work;     // [n_new] fetched index of each owner message's discMessage
  uint32_t* sorted;   // [n_new] message index of each owner message (the render's grouped order)
  uint32_t* rows;     // [n_new] its row
};

DEVI uint64_t st_turn_slot(const StTurn& t, uint32_t k, long long msg) { return st_hash(k, 0, 0, msg) & t.bmask; }
DEVI bool st_turn_same(const StTurn& t, uint32_t k, uint32_t cur, long long msg) {
  return cur >= t.foff[k] && cur < t.foff[k + 1] && t.fetched[2 * cur + 1] == msg;
}

// 1. addNewMessages' test against the page's current list, and the first fetched index of every message id of a page
__global__ void st_turn_probe_kernel(StDev d, StTurn t) {
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < t.n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t k = st_seg(t.foff, t.P, j), row = t.prow[k];
    const long long chat = t.fetched[2 * j], msg = t.fetched[2 * j + 1];
    t.pg[j] = k;
    t.flag[j] = st_lookup(d, row, d.row_gen[row], chat, msg) == ST_NONE;
    for (uint64_t s = st_turn_slot(t, k, msg);; s = (s + 1) & t.bmask) {
      const uint32_t cur = atomicCAS(t.bfirst + s, ST_NONE, (uint32_t)j);
      if (cur == ST_NONE) break;
      if (st_turn_same(t, k, cur, msg)) {
        atomicMin(t.bfirst + s, (uint32_t)j);
        break;
      }
    }
  }
}

// every page's new list in the call's list (woff, nullptr pos: all empty), and every row's message count before the
// call (old, optional)
__global__ void st_turn_meta_kernel(const uint32_t* row_cnt, const uint32_t* prow, uint32_t P, const uint64_t* foff,
                                    const uint64_t* pos, uint64_t* woff, uint32_t* old) {
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k <= P; k += (uint64_t)gridDim.x * blockDim.x) {
    if (woff) woff[k] = pos ? pos[foff[k]] : 0;
    if (k < P && old) old[k] = row_cnt[prow[k]];
  }
}

// 2. the new lists in fetch order, appended as their rows' live messages of the generation the rows now hold: status
// "resample", no platform, pageId = the page; each owner message's discMessage is the first fetched message of its page
// with its message id (the chat id is ignored)
__global__ void st_turn_append_kernel(StDev d, StTurn t) {
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < t.n; j += (uint64_t)gridDim.x * blockDim.x) {
    if (!t.flag[j]) continue;
    const uint64_t p = t.pos[j];
    const uint32_t k = t.pg[j], row = t.prow[k];
    const long long chat = t.fetched[2 * j], msg = t.fetched[2 * j + 1];
    uint64_t s = st_turn_slot(t, k, msg);
    while (!st_turn_same(t, k, t.bfirst[s], msg)) s = (s + 1) & t.bmask;
    t.work[p] = t.bfirst[s];
    t.keys[2 * p] = chat;
    t.keys[2 * p + 1] = msg;
    StMsg m;
    m.chat = chat;
    m.msg = msg;
    m.row = row;
    m.gen = d.row_gen[row];
    m.pid = row;
    m.status = 5;  // "resample"
    m.platform = 0;
    d.msgs[t.n_msgs + p] = m;
    t.sorted[p] = (uint32_t)(t.n_msgs + p);
    t.rows[p] = row;
  }
}

// a row's new fields in one upload: the page row, and with a new list its generation and count; base (ST_NO_BASE: left)
// is its first message in the render's grouped order
constexpr uint64_t ST_NO_BASE = ~0ull;
struct StRowPut {
  tgi_state_page page;
  uint32_t row, gen, cnt, list;
  uint64_t base;
};
__global__ void st_rows_put_kernel(tgi_state_page* pages, uint32_t* row_gen, uint32_t* row_cnt, const StRowPut* in, uint32_t P,
                                   uint64_t* row_base) {
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < P; k += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t r = in[k].row;
    pages[r] = in[k].page;
    if (in[k].list) {
      row_gen[r] = in[k].gen;
      row_cnt[r] = in[k].cnt;
    }
    if (in[k].base != ST_NO_BASE) row_base[r] = in[k].base;
  }
}

// the loop's UpdateMessage calls of every page: update q is owner message woff[k] + (q - uoff[k]) of page k, whose first
// n_done[k] records were processed; it updates the key (message id, chat id), swapped as the reference passes them, with
// "failed" for a record that failed and "fetched" otherwise (status: the turn's records, owner message j at status[j])
struct StEnd {
  const long long* keys;  // [n_work][2] the turn's owner keys
  const uint8_t* status;
  const uint32_t* prow;   // [P]
  const uint64_t* woff;   // [P+1] page k's owner messages
  const uint64_t* uoff;   // [P+1] page k's updates (scan of n_done)
  const uint32_t* live;   // [P] 1: page k's row still holds this turn's owner view
  uint32_t P;
};
__global__ void st_turn_updates_kernel(StEnd e, uint64_t m, tgi_state_update* u) {
  for (uint64_t q = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; q < m; q += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t k = st_seg(e.uoff, e.P, q);
    const uint64_t j = e.woff[k] + (q - e.uoff[k]);
    tgi_state_update v;
    v.chat_id = e.keys[2 * j + 1];
    v.message_id = e.keys[2 * j];
    v.row = e.prow[k];
    v.status = e.status[j] == TGI_ST_FAILED ? 3 : 2;  // "failed" : "fetched"
    v.reserved = 0;
    u[q] = v;
  }
}

// ---- page close: UpdatePage(*owner) (crawl/runner.go:1543-1544) over the row's owner view ---------------------------
// The view is the turn's owner messages of the row: their keys and a status code each, 0 while no hit of the end
// reached the owner (the message is still "resample").  Go's owner shares its backing array with pageMap's page until an
// append reallocates it; the array counts as full, so an UpdateMessage of the end reaches the owner only before the
// end's first append to that page, and then the first owner message of the page with the key takes the status.
struct StView {
  StEnd e;                // the turn's pages, their owner messages and updates
  uint16_t* status;       // [k] the owner messages' statuses
  uint64_t k;             // owner messages of the turn
  uint32_t* vfirst;       // batch table keyed by (page, owner key): lowest owner index, ST_NONE = empty
  uint64_t vmask;
  uint32_t* last;         // [k] 1 + the last update that reached owner message p (0: none)
  uint32_t* app;          // [P] the first update of page k that appended (ST_NONE: none)
};

DEVI uint64_t st_view_slot(const StView& v, uint32_t pg, long long chat, long long msg) {
  return st_hash(pg, 0, chat, msg) & v.vmask;
}

// 1. the owner keys of the pages whose view is the turn's, by first owner index, and each page's first update that
// appended (the lowest flagged leader of its segment)
__global__ void st_view_build_kernel(StView v, const uint32_t* flag, uint64_t n) {
  const uint64_t m = v.k > n ? v.k : n;
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < m; j += (uint64_t)gridDim.x * blockDim.x) {
    if (j < n && flag[j]) atomicMin(v.app + st_seg(v.e.uoff, v.e.P, j), (uint32_t)j);
    if (j >= v.k) continue;
    const uint32_t pg = st_seg(v.e.woff, v.e.P, j);
    if (!v.e.live[pg]) continue;
    const long long chat = v.e.keys[2 * j], msg = v.e.keys[2 * j + 1];
    for (uint64_t s = st_view_slot(v, pg, chat, msg);; s = (s + 1) & v.vmask) {
      const uint32_t cur = atomicCAS(v.vfirst + s, ST_NONE, (uint32_t)j);
      if (cur == ST_NONE) break;
      if (cur >= v.e.woff[pg] && cur < v.e.woff[pg + 1] && v.e.keys[2 * cur] == chat && v.e.keys[2 * cur + 1] == msg) {
        atomicMin(v.vfirst + s, (uint32_t)j);
        break;
      }
    }
  }
}

// 2. every update before its page's first append whose key is an owner key of the page reaches that key's first owner
// message
__global__ void st_view_hit_kernel(StView v, const tgi_state_update* u, uint64_t n) {
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t pg = st_seg(v.e.uoff, v.e.P, j);
    if (j >= v.app[pg] || !v.e.live[pg]) continue;
    const long long chat = u[j].chat_id, msg = u[j].message_id;
    for (uint64_t s = st_view_slot(v, pg, chat, msg);; s = (s + 1) & v.vmask) {
      const uint32_t cur = v.vfirst[s];
      if (cur == ST_NONE) break;
      if (cur >= v.e.woff[pg] && cur < v.e.woff[pg + 1] && v.e.keys[2 * cur] == chat && v.e.keys[2 * cur + 1] == msg) {
        atomicMax(v.last + cur, (uint32_t)j + 1);
        break;
      }
    }
  }
}

// 3. the last such update's status, in update order
__global__ void st_view_status_kernel(StView v, const tgi_state_update* u) {
  for (uint64_t p = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; p < v.k; p += (uint64_t)gridDim.x * blockDim.x)
    if (v.last[p]) v.status[p] = u[v.last[p] - 1].status;
}

// one owner view of a close: its messages are [off, next off) of the close's appended list
struct StViewSeg {
  const long long* keys;   // [k][2]
  const uint16_t* status;  // [k]
  uint64_t off;
  uint32_t row, reserved;
};

// the close: every view's messages appended at n0 as its row's live list of the generation the row now holds (pageId =
// the page, no platform); sorted / rows are the render's grouped order
__global__ void st_view_append_kernel(StDev d, const StViewSeg* seg, uint32_t Q, uint64_t K, uint64_t n0, uint32_t* sorted,
                                      uint32_t* rows) {
  for (uint64_t p = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; p < K; p += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = Q - 1;  // the last view with off <= p
    while (lo < hi) {
      const uint32_t mid = (lo + hi + 1) >> 1;
      if (seg[mid].off <= p) lo = mid;
      else hi = mid - 1;
    }
    const StViewSeg& v = seg[lo];
    const uint64_t i = p - v.off;
    StMsg m;
    m.chat = v.keys[2 * i];
    m.msg = v.keys[2 * i + 1];
    m.row = v.row;
    m.gen = d.row_gen[v.row];
    m.pid = v.row;
    m.status = v.status[i] ? v.status[i] : 5;  // "resample"
    m.platform = 0;
    d.msgs[n0 + p] = m;
    sorted[p] = (uint32_t)(n0 + p);
    rows[p] = v.row;
  }
}

// flag[i] = message i is a live message of one of the rows in set (ascending, n_set > 0)
__global__ void st_rows_flag_kernel(StDev d, uint64_t n, const uint32_t* set, uint32_t n_set, uint32_t* flag) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const StMsg m = d.msgs[i];
    uint32_t lo = 0, hi = n_set - 1;
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (set[mid] < m.row) lo = mid + 1;
      else hi = mid;
    }
    flag[i] = set[lo] == m.row && st_live(d, m);
  }
}

// the first grouped message of every row in rows[0, n) (grouped by row), at base + its position
__global__ void st_row_starts_kernel(const uint32_t* rows, const uint64_t* n, uint64_t base, uint64_t* row_base) {
  const uint64_t m = *n;
  for (uint64_t q = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; q < m; q += (uint64_t)gridDim.x * blockDim.x)
    if (q == 0 || rows[q - 1] != rows[q]) row_base[rows[q]] = base + q;
}

// ---- compaction -------------------------------------------------------------------------------------------------
// flag[i] = message i is live (row == ST_NONE) or a live message of `row`
__global__ void st_live_flag_kernel(StDev d, uint64_t n, uint32_t row, uint32_t* flag) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const StMsg m = d.msgs[i];
    flag[i] = st_live(d, m) && (row == ST_NONE || m.row == row);
  }
}
__global__ void st_compact_kernel(StDev d, uint64_t n, const uint32_t* flag, const uint64_t* pos, StMsg* out) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    if (flag[i]) out[pos[i]] = d.msgs[i];
}

// ---- page reads (tgi_state_read_pages / _read_layer): the message lists of a set of rows -----------------------------
// the live message count of every row of the read set (ascending)
__global__ void st_set_counts_kernel(const uint32_t* row_cnt, const uint32_t* set, uint32_t n_set, uint32_t* cnt) {
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < n_set; k += (uint64_t)gridDim.x * blockDim.x)
    cnt[k] = row_cnt[set[k]];
}
// the set's live messages grouped by row (sorted = their message indices, *n of them) as tgi_state_msg, in that order
__global__ void st_gather_kernel(StDev d, const uint32_t* sorted, const uint64_t* n, tgi_state_msg* out) {
  const uint64_t m = *n;
  for (uint64_t q = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; q < m; q += (uint64_t)gridDim.x * blockDim.x) {
    const StMsg s = d.msgs[sorted[q]];
    tgi_state_msg o;
    o.chat_id = s.chat;
    o.message_id = s.msg;
    o.page_id = s.pid;
    o.status = s.status;
    o.platform = s.platform;
    out[q] = o;
  }
}

// ---- render ---------------------------------------------------------------------------------------------------------
struct StEntry {  // one page of a layer, or an empty layer (row == ST_NONE)
  long long depth;  // the layer's depth
  uint32_t row;
  uint32_t flags;   // ST_E_*
};
enum : uint32_t { ST_E_FIRST = 1, ST_E_LAST = 2, ST_E_FIRST_LAYER = 4 };

struct StRender {
  const StEntry* entries;
  uint64_t n_entries;
  const ZoneEnt* zone;  // time.Local (tgi_set_zone), or the fixed tz when zone_n == 0
  uint32_t zone_n;
  int32_t tz;
  uint64_t* sc;        // ST_SC_*
  uint64_t* row_base;  // [rows+1] scan of row_cnt: first grouped message of every row
  uint32_t* msize;     // [live] bytes of grouped message k (its leading comma included)
  uint64_t* moff;      // [live+1] their scan
  uint32_t* esize_lo;  // [entries] bytes of entry e up to its first message (part A)
  uint32_t* ebytes;    // [entries] bytes of entry e without its messages (parts A and B)
  uint32_t* ecnt;      // [entries] messages of entry e
  uint64_t* eoff;      // [entries+1] scan of the entry sizes with messages
  uint64_t* eslot;     // [entries+1] scan of ecnt
  uint32_t* esz;       // [entries] entry sizes with messages (the scan's input)
  uint8_t* out;        // the layers' bytes
};
// the scalars block: live messages, body bytes, message slots, a timestamp that does not render, an entry, message,
// row or id of 4 GiB or more, message bytes, rows, radix counts
enum { ST_SC_LIVE, ST_SC_BYTES, ST_SC_SLOTS, ST_SC_ERR, ST_SC_BIG, ST_SC_MBYTES, ST_SC_ROWS, ST_SC_RADIX, ST_SC_COUNT };

// The 4 GiB rule: every writer sizes a piece (an entry with its messages, a SQL row, a layer-map id) in 64 bits and flags
// one of 4 GiB or more in ST_SC_BIG, which refuses the call before anything is written; a written piece is under 4 GiB,
// so the emits keep 32-bit offsets within it.
template <bool EMIT>
using StLen = std::conditional_t<EMIT, uint32_t, uint64_t>;
DEVI void st_flag_big(uint64_t* sc, uint64_t bytes) {
  if (bytes > 0xFFFFFFFFull) atomicMax((unsigned long long*)sc + ST_SC_BIG, 1ull);
}

// JSON escape of a short string by one thread (Go's sequential rule, as thread_esc_len measures it)
DEVI uint32_t st_thread_esc(uint8_t* dst, const uint8_t* s, uint32_t n) {
  DstG d{dst};
  uint32_t o = 0;
  for (uint32_t i = 0; i < n;) {
    const uint32_t b = ldb(s + i);
    if (b < 0x80) {
      const uint32_t len = ascii_esc_len(b);
      put_escaped(d, o, b, len);
      o += len;
      i++;
      continue;
    }
    const int need = utf8_valid_lead(s, i, n);
    if (need == 0) {
      put_u(d, o, 'f', 'f', 'f', 'd');
      o += 6;
      i++;
    } else if (need == 3 && b == 0xE2 && ldb(s + i + 1) == 0x80 && (ldb(s + i + 2) | 1u) == 0xA9) {
      put_u(d, o, '2', '0', '2', ldb(s + i + 2) == 0xA8 ? '8' : '9');
      o += 6;
      i += 3;
    } else {
      for (int k = 0; k < need; k++) d.st(o + k, ldb(s + i + k));
      o += (uint32_t)need;
      i += (uint32_t)need;
    }
  }
  return o;
}

DEVI const uint8_t* st_str(const StDev& d, const tgi_state_page& p, int f, uint32_t& len) {
  uint64_t o = p.str_off;
  for (int k = 0; k < f; k++) o += p.str_len[k];
  len = p.str_len[f];
  return d.blob + o;
}

// one message, sized (dst == nullptr) or written: [,]{"chatId":N,"messageId":N,"status":"S","pageId":"P"[,"platform":"X"]}
template <bool EMIT>
DEVI StLen<EMIT> st_message(const StDev& d, const StMsg& m, bool comma, uint8_t* dst) {
  StLen<EMIT> o = 0;
  auto lit = [&](const char* s, uint32_t n) {
    if (EMIT)
      for (uint32_t k = 0; k < n; k++) dst[o + k] = (uint8_t)s[k];
    o += n;
  };
  auto esc = [&](const uint8_t* s, uint32_t n) { o += EMIT ? st_thread_esc(dst + o, s, n) : thread_esc_len<StLen<EMIT>>(s, n); };
  auto num = [&](long long v) { o += EMIT ? (uint32_t)render_i64(dst + o, v) : ndigits_i64(v); };
  if (comma) lit(",", 1);
  lit("{\"chatId\":", 10);
  num(m.chat);
  lit(",\"messageId\":", 13);
  num(m.msg);
  lit(",\"status\":\"", 11);
  esc(d.codes.blob + d.codes.off[m.status], d.codes.off[m.status + 1] - d.codes.off[m.status]);
  lit("\",\"pageId\":\"", 12);
  uint32_t il;
  const uint8_t* id = st_str(d, d.pages[m.pid], TGI_PS_ID, il);
  esc(id, il);
  lit("\"", 1);
  const uint32_t pl = d.codes.off[m.platform + 1] - d.codes.off[m.platform];
  if (pl) {
    lit(",\"platform\":\"", 13);
    esc(d.codes.blob + d.codes.off[m.platform], pl);
    lit("\"", 1);
  }
  lit("}", 1);
  return o;
}

struct StGroup {       // live messages grouped by row (the render, the page reads, the page close)
  const uint32_t* flag;  // [n_msgs] flags of the messages taken
  const uint64_t* pos;   // [n_msgs+1] their scan
  uint32_t* keys[2];     // radix ping-pong: row, message index
  uint32_t* vals[2];
};
// the flagged messages compacted in storage order: the radix sort's input pairs (row, message index)
__global__ void st_render_pairs_kernel(StDev d, uint64_t n, StGroup g) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    if (!g.flag[i]) continue;
    const uint64_t k = g.pos[i];
    g.keys[0][k] = d.msgs[i].row;
    g.vals[0][k] = (uint32_t)i;
  }
}
// size pass, a thread per grouped message k (sorted = the grouped message indices, sorted_rows their rows)
__global__ void st_msg_size_kernel(StDev d, StRender r, const uint32_t* sorted, const uint32_t* sorted_rows, uint64_t live) {
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < live; k += (uint64_t)gridDim.x * blockDim.x) {
    // saturated, not flagged: a message of 4 GiB or more makes its entry one, and only the entries a call writes are
    // checked (a message of a page in no layer list is sized by the render but never written)
    const uint64_t sz = st_message<false>(d, d.msgs[sorted[k]], k != r.row_base[sorted_rows[k]], nullptr);
    r.msize[k] = sz > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)sz;
  }
}

// one entry, sized or written by a warp (lane 0 writes the literals, the warp escapes the strings).  Returns the bytes
// of part A (framing and fields up to the first message) in *a and of the whole entry without messages, in 64 bits
// (part A in 32: when it wraps, so does the whole).  LINE: the
// page alone as one JSONL line, {page}\n, without layer framing (the exports).  A template parameter rather than an
// entry flag: the flag cost the render's emit kernel 8 bytes of spills.
template <bool EMIT, bool LINE = false>
DEVI uint64_t st_entry(const StDev& d, const StRender& r, const StEntry& e, uint32_t cnt, uint8_t* dst, uint64_t msg_bytes,
                       uint32_t* a, bool* bad) {
  const bool l0 = lane_id() == 0;
  uint64_t o = 0;
  auto lit = [&](const char* s, uint32_t n) {
    if (EMIT && l0)
      for (uint32_t k = 0; k < n; k++) dst[o + k] = (uint8_t)s[k];
    o += n;
  };
  auto num = [&](long long v) {
    if (EMIT && l0) render_i64(dst + o, v);
    o += ndigits_i64(v);
  };
  auto str = [&](const tgi_state_page& p, int f) {
    uint32_t n;
    const uint8_t* s = st_str(d, p, f, n);
    o += EMIT ? esc_to_global(dst + o, s, n) : warp_esc_len64(s, n);
  };
  if (LINE) {
  } else if (e.flags & ST_E_FIRST) {
    if (!(e.flags & ST_E_FIRST_LAYER)) lit(",", 1);
    lit("{\"depth\":", 9);
    num(e.depth);
    lit(",\"pages\":[", 10);
  } else {
    lit(",", 1);
  }
  if (e.row != ST_NONE) {
    const tgi_state_page& p = d.pages[e.row];  // read in place: a copy would live across the escaper calls
    auto opt = [&](int f, const char* key, uint32_t kl) {  // an omitempty string
      if (!p.str_len[f]) return;
      lit(key, kl);
      str(p, f);
      lit("\"", 1);
    };
    lit("{\"id\":\"", 7);
    str(p, TGI_PS_ID);
    lit("\",\"url\":\"", 9);
    str(p, TGI_PS_URL);
    lit("\",\"depth\":", 10);
    num(p.depth);
    lit(",\"status\":\"", 11);
    str(p, TGI_PS_STATUS);
    lit("\"", 1);
    opt(TGI_PS_ERROR, ",\"error\":\"", 10);
    lit(",\"timestamp\":", 13);
    {
      uint8_t tb[48];
      int tl = 0;
      if (l0) {
        uint8_t* t = EMIT ? dst + o : tb;
        if (p.ts_off == TGI_STATE_TS_LOCAL) {
          tl = render_zone_time(t, p.ts_sec, p.ts_nsec, r.zone, r.zone_n, r.tz);
        } else {
          tl = render_time(t, p.ts_sec, p.ts_nsec, p.ts_off);
          if (tl && p.ts_off < 0 && p.ts_off > -60) t[tl - 7] = '+';  // Go's minutes-first sign, as render_zone_time
        }
      }
      tl = __shfl_sync(FULL, tl, 0);
      if (!tl) *bad = true;
      o += (uint32_t)tl;
    }
    opt(TGI_PS_PLATFORM, ",\"platform\":\"", 13);
    opt(TGI_PS_PARENT, ",\"parentId\":\"", 13);
    if (cnt) lit(",\"messages\":[", 13);
    *a = (uint32_t)o;
    o += msg_bytes;
    if (cnt) lit("]", 1);
    opt(TGI_PS_CONN, ",\"LastConnectionID\":\"", 21);
    opt(TGI_PS_SEQ, ",\"sequenceId\":\"", 15);
    opt(TGI_PS_CRAWL, ",\"crawlId\":\"", 12);
    lit("}", 1);
  } else {
    *a = (uint32_t)o;
  }
  if (LINE) lit("\n", 1);
  else if (e.flags & ST_E_LAST) lit("]}", 2);
  return o - msg_bytes;
}

constexpr int ST_WARPS = 8;  // warps per CTA of the warp-per-entry kernels

// size pass, a warp per entry: the entry's bytes around its messages, its message count and message bytes
template <bool LINE>
DEVI void st_entry_size(const StDev& d, const StRender& r) {
  const uint64_t w0 = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5, nw = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t e = w0; e < r.n_entries; e += nw) {
    const StEntry en = r.entries[e];
    uint32_t cnt = 0;
    uint64_t mb = 0;
    if (en.row != ST_NONE) {
      cnt = d.row_cnt[en.row];
      const uint64_t b = r.row_base[en.row];
      mb = r.moff[b + cnt] - r.moff[b];
    }
    uint32_t a;
    bool bad = false;
    const uint64_t sz = st_entry<false, LINE>(d, r, en, cnt, nullptr, mb, &a, &bad);
    if (lane_id() == 0) {
      r.esize_lo[e] = a;
      r.ebytes[e] = (uint32_t)sz;
      r.ecnt[e] = cnt;
      r.esz[e] = (uint32_t)(sz + mb);
      st_flag_big(r.sc, sz + mb);
      if (bad) atomicMax((unsigned long long*)r.sc + ST_SC_ERR, 1ull);
    }
  }
}

// emit, a warp per entry: everything but the messages
template <bool LINE>
DEVI void st_entry_emit(const StDev& d, const StRender& r) {
  const uint64_t w0 = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5, nw = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t e = w0; e < r.n_entries; e += nw) {
    const StEntry en = r.entries[e];
    const uint64_t off = r.eoff[e];
    const uint64_t mb = r.eoff[e + 1] - off - r.ebytes[e];
    uint32_t a;
    bool bad = false;
    st_entry<true, LINE>(d, r, en, r.ecnt[e], r.out + off, mb, &a, &bad);
    __syncwarp();
  }
}

__global__ void __launch_bounds__(ST_WARPS * 32) st_entry_size_kernel(StDev d, StRender r) { st_entry_size<false>(d, r); }
__global__ void __launch_bounds__(ST_WARPS * 32) st_entry_emit_kernel(StDev d, StRender r) { st_entry_emit<false>(d, r); }
// the same for the exports' JSONL lines
__global__ void __launch_bounds__(ST_WARPS * 32) st_line_size_kernel(StDev d, StRender r) { st_entry_size<true>(d, r); }
__global__ void __launch_bounds__(ST_WARPS * 32) st_line_emit_kernel(StDev d, StRender r) { st_entry_emit<true>(d, r); }

// emit, a thread per message slot of the output: slot t is message k of entry e (binary search over eslot)
__global__ void st_msg_emit_kernel(StDev d, StRender r, const uint32_t* sorted) {
  const uint64_t slots = r.sc[ST_SC_SLOTS];
  for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < slots; t += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t lo = 0, hi = r.n_entries - 1;  // the last entry with eslot <= t
    while (lo < hi) {
      const uint64_t mid = (lo + hi + 1) >> 1;
      if (r.eslot[mid] <= t) lo = mid;
      else hi = mid - 1;
    }
    const uint64_t e = lo, k = t - r.eslot[e];
    const uint64_t b = r.row_base[r.entries[e].row], q = b + k;
    st_message<true>(d, d.msgs[sorted[q]], k != 0, r.out + r.eoff[e] + r.esize_lo[e] + (r.moff[q] - r.moff[b]));
  }
}

// ---- snowball discovery (crawl/runner.go:1199-1244, standalone/runner.go:835-850, dapr/standalone.go:645-688) -------
struct StCand {      // 48 bytes: one candidate page of the next layer (and one entry of the pending list)
  uint8_t name[32];  // the outlink, zero padded: a key of the resident sets
  uint32_t len;
  uint32_t parent;   // the owner row
  uint32_t span;     // the span that found it (unused in the pending list)
  uint32_t reserved;
};

struct StDisc {
  const tgi_state_span* spans;
  uint32_t n_spans;
  const uint8_t* status;     // the slot's resident result
  const uint32_t* link_off;  // [n+1]
  const tgi_link* links;
  const uint64_t* soff;      // [n_spans+1] scan of the spans' processed link rows
  uint64_t bound;            // gather threads: at least soff[n_spans]
  uint32_t* flag;            // [bound] 1: link row i of the spans is a candidate
  uint32_t* lnk;             // [bound] its link row in the result
  uint32_t* spn;             // [bound] its span
  uint64_t* pos;             // [bound+1] scan of flag
  StCand* out;               // candidate k at out[k]
  uint64_t* coff;            // [n_spans+1] first candidate of every span
};

// the link rows of span k's processed records
__global__ void st_disc_count_kernel(StDisc g, uint32_t* cnt) {
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < g.n_spans; k += (uint64_t)gridDim.x * blockDim.x) {
    const tgi_state_span s = g.spans[k];
    cnt[k] = g.link_off[s.first + s.n_done] - g.link_off[s.first];
  }
}

// a thread per processed link row: a candidate when its record was processed without error (a failed record returned an
// error, a date-skipped one an empty Post) and its name is not byte-equal to the owner's URL (runner.go:1231)
__global__ void st_disc_flag_kernel(StDev d, StDisc g) {
  const uint64_t total = g.soff[g.n_spans];
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < g.bound; i += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t f = 0;
    if (i < total) {
      uint32_t lo = 0, hi = g.n_spans - 1;  // the last span with soff <= i (empty spans share their offset)
      while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (g.soff[mid] <= i) lo = mid;
        else hi = mid - 1;
      }
      const tgi_state_span s = g.spans[lo];
      const uint32_t L = g.link_off[s.first] + (uint32_t)(i - g.soff[lo]);
      uint64_t a = s.first, b = s.first + s.n_done - 1;  // the record that holds link row L
      while (a < b) {
        const uint64_t mid = (a + b + 1) >> 1;
        if (g.link_off[mid] <= L) a = mid;
        else b = mid - 1;
      }
      const uint8_t st = g.status[a];
      if (st == TGI_ST_EMITTED || st == TGI_ST_NOLINE) {
        uint32_t ul;
        const uint8_t* u = st_str(d, d.pages[s.row], TGI_PS_URL, ul);
        const tgi_link& lk = g.links[L];
        bool self = ul == lk.len;
        for (uint32_t k = 0; self && k < ul; k++) self = u[k] == lk.name[k];
        f = !self;
      }
      g.lnk[i] = L;
      g.spn[i] = lo;
    }
    g.flag[i] = f;
  }
}

// the candidates in (span, record, link) order, and every span's first candidate
__global__ void st_disc_emit_kernel(StDisc g) {
  const uint64_t total = g.soff[g.n_spans];
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
    if (!g.flag[i]) continue;
    const tgi_link& lk = g.links[g.lnk[i]];
    StCand& c = g.out[g.pos[i]];
    store_key(c.name, load_key(lk.name));
    c.len = lk.len;
    c.parent = g.spans[g.spn[i]].row;
    c.span = g.spn[i];
    c.reserved = 0;
  }
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k <= g.n_spans; k += (uint64_t)gridDim.x * blockDim.x)
    g.coff[k] = g.pos[g.soff[k]];
}

// first occurrence per URL (per span, or over the list) and Dapr's urlCache test, over candidates [0, *n)
struct StFirst {
  const StCand* c;
  const uint64_t* n;  // device count
  uint64_t bound;     // threads: at least *n
  bool per_span;      // first occurrence within each span (Base rules per page)
  bool dedup;         // false: Dapr's AddLayer keeps a page's repeated URLs
  FrontierDev urls;   // TGI_SET_URLS (table == nullptr: empty, or not tested)
  uint32_t* bfirst;   // batch table: lowest candidate index of the slot's key, ST_NONE = empty
  uint64_t bmask;
  uint32_t* slot_of;  // [bound]
  uint32_t* flag;     // [bound] 1: the candidate survives
  uint64_t* pos;      // [bound+1] scan of flag
  StCand* out;        // the survivors in candidate order
};

DEVI bool st_same_cand(const StFirst& w, const StCand& a, const StCand& b) {
  return (!w.per_span || a.span == b.span) && key_eq(load_key(a.name), load_key(b.name));
}

// a candidate's batch-table hash: its key's, mixed with its span when the candidates of each span are kept apart
DEVI uint64_t st_cand_hash(const Key32& k, uint32_t span, bool per_span) {
  return key_hash(k) ^ (per_span ? span * 0x9E3779B97F4A7C15ull : 0ull);
}

__global__ void st_first_kernel(StFirst w) {
  const uint64_t n = *w.n;
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const StCand& c = w.c[j];
    const uint64_t h = st_cand_hash(load_key(c.name), c.span, w.per_span);
    uint64_t s = (h >> 7) & w.bmask;
    for (;; s = (s + 1) & w.bmask) {
      const uint32_t cur = atomicCAS(w.bfirst + s, ST_NONE, (uint32_t)j);
      if (cur == ST_NONE) break;
      if (st_same_cand(w, w.c[cur], c)) {
        atomicMin(w.bfirst + s, (uint32_t)j);
        break;
      }
    }
    w.slot_of[j] = (uint32_t)s;
  }
}

__global__ void st_keep_kernel(StFirst w) {
  const uint64_t n = *w.n;
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < w.bound; j += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t f = 0;
    if (j < n) {
      f = !w.dedup || w.bfirst[w.slot_of[j]] == (uint32_t)j;
      if (f && w.urls.table) {
        const Key32 k = load_key(w.c[j].name);
        f = set_lookup(w.urls, k, key_hash(k)) < 0;
      }
    }
    w.flag[j] = f;
  }
}

__global__ void st_survivors_kernel(StFirst w) {
  const uint64_t n = *w.n;
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x)
    if (w.flag[j]) w.out[w.pos[j]] = w.c[j];
}

// Philox4x32-10 (Salmon et al., SC'11): ten rounds over the counter, the key bumped between them
DEVI void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
  for (int r = 0; r < 10; r++) {
    if (r) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint32_t lo0 = 0xD2511F53u * c[0], hi0 = __umulhi(0xD2511F53u, c[0]);
    const uint32_t lo1 = 0xCD9E8D57u * c[2], hi1 = __umulhi(0xCD9E8D57u, c[2]);
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
    c[0] = n0;
    c[1] = lo1;
    c[2] = n2;
    c[3] = lo0;
  }
}

// id ctr of the seed in counter domain `domain` (word 2: 0 = pages, 1 = pending-edge batches) as a version-4 uuid
// string of 36 bytes
DEVI void st_uuid(uint64_t seed, uint64_t ctr, uint32_t domain, uint8_t* o) {
  uint32_t c[4] = {(uint32_t)ctr, (uint32_t)(ctr >> 32), domain, 0u};
  philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
  uint8_t b[16];
  for (int q = 0; q < 16; q++) b[q] = (uint8_t)(c[q >> 2] >> (8 * (q & 3)));
  b[6] = (b[6] & 0x0F) | 0x40;
  b[8] = (b[8] & 0x3F) | 0x80;
  for (int q = 0, p = 0; q < 16; q++) {
    if (q == 4 || q == 6 || q == 8 || q == 10) o[p++] = '-';
    o[p++] = "0123456789abcdef"[b[q] >> 4];
    o[p++] = "0123456789abcdef"[b[q] & 15];
  }
}

// page ids n0 .. n0+n-1 of the seed, 36 bytes each
__global__ void st_uuid_kernel(uint64_t seed, uint64_t n0, uint64_t n, uint8_t* out) {
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < n; k += (uint64_t)gridDim.x * blockDim.x)
    st_uuid(seed, n0 + k, 0u, out + 36 * k);
}

// ---- tandem hand-off (crawl/runner.go:1129, 1229-1306, 1414-1455): every page's pending-edge batch -------------------
// The candidates of the discovery gather (owner-URL skip, status, n_done), deduplicated per span by st_first_kernel
// (seenInBatch), then cut by FilterUsername and the invalid set's TTL.  Those two tests depend on the name only, so
// the first occurrence of a name survives exactly when every occurrence in its span would: the order against the
// dedup does not change the edges.
struct StEdges {
  const StCand* c;           // the gather's candidates in (span, record, link) order
  const uint32_t* link;      // [bound] the link row in the result of every candidate
  const uint64_t* coff;      // [n_spans+1] first candidate of every span; coff[n_spans] = the count
  uint64_t bound;            // threads: at least the count
  const uint32_t* bfirst;    // st_first_kernel's batch table (per span) and every candidate's slot in it
  const uint32_t* slot_of;
  const tgi_state_span* spans;
  uint32_t n_spans;
  const uint32_t* link_off;  // the slot's resident result
  const tgi_link* links;
  ExclusionDev x;            // TGI_SET_INVALID with the call's clock, TGI_SET_DISCOVERED
  unsigned long long* n_cand;  // candidates that pass both name tests, before the dedup
  uint32_t* flag;            // [bound] 1: candidate j is an edge
  uint64_t* pos;             // [bound+1] scan of flag: the edge's index
  uint32_t* has;             // [n_spans] 1: the span has an edge
  uint64_t* bpos;            // [n_spans+1] scan of has: the span's batch
  uint64_t seed, batch0;     // the id key, and the counter of the call's first batch
  tgi_state_edge* edges;
  tgi_state_edge_batch* batches;
  uint32_t* span_batch;      // [n_spans]
};

// the link row of every candidate, from the gather's flags and offsets
__global__ void st_edge_link_kernel(StDisc g, uint32_t* link) {
  const uint64_t total = g.soff[g.n_spans];
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x)
    if (g.flag[i]) link[g.pos[i]] = g.lnk[i];
}

__global__ void st_edge_keep_kernel(StEdges e) {
  const uint64_t n = e.coff[e.n_spans];
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < e.bound; j += (uint64_t)gridDim.x * blockDim.x) {
    bool pass = false, f = false;
    if (j < n) {
      const StCand& c = e.c[j];
      const Key32 k = load_key(c.name);
      pass = (e.links[e.link[j]].flags & TGI_LF_FILTER_OK) && !set_invalid_hit(e.x, k, key_hash(k), e.x.now_sec);  // :1247, :1261
      f = pass && e.bfirst[e.slot_of[j]] == (uint32_t)j;  // :1267-1272
    }
    const unsigned am = __activemask(), m = __ballot_sync(am, pass);
    if (m && (threadIdx.x & 31) == (unsigned)__ffs(am) - 1) atomicAdd(e.n_cand, (unsigned long long)__popc(m));
    e.flag[j] = f;
  }
}

__global__ void st_edge_spans_kernel(StEdges e) {
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < e.n_spans; k += (uint64_t)gridDim.x * blockDim.x)
    e.has[k] = e.pos[e.coff[k + 1]] > e.pos[e.coff[k]];
}

// the edges: destination, the record and source of the name's first occurrence in the page, the validator's discovered
// look-up (validator.go:214-226); the batches: one per span with an edge (runner.go:1275-1291), in span order
__global__ void st_edge_emit_kernel(StEdges e) {
  const uint64_t n = e.coff[e.n_spans];
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    if (!e.flag[j]) continue;
    const StCand& c = e.c[j];
    const uint32_t L = e.link[j];
    const tgi_state_span s = e.spans[c.span];
    uint64_t a = s.first, b = s.first + s.n_done - 1;  // the record that holds link row L
    while (a < b) {
      const uint64_t mid = (a + b + 1) >> 1;
      if (e.link_off[mid] <= L) a = mid;
      else b = mid - 1;
    }
    const Key32 k = load_key(c.name);
    tgi_state_edge& o = e.edges[e.pos[j]];
    store_key(o.destination, k);
    o.record = a;
    o.batch = (uint32_t)e.bpos[c.span];
    o.dest_len = (uint8_t)c.len;
    o.source_type = e.links[L].src;
    o.status = set_lookup(e.x.discovered, k, key_hash(k)) >= 0 ? TGI_EDGE_DUPLICATE : TGI_EDGE_PENDING;
    o.reserved = 0;
  }
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < e.n_spans; k += (uint64_t)gridDim.x * blockDim.x) {
    if (!e.has[k]) {
      e.span_batch[k] = TGI_STATE_NO_BATCH;
      continue;
    }
    const uint64_t q = e.bpos[k], f0 = e.pos[e.coff[k]];
    e.span_batch[k] = (uint32_t)q;
    tgi_state_edge_batch& bt = e.batches[q];
    st_uuid(e.seed, e.batch0 + q, 1u, bt.batch_id);
    bt.span = (uint32_t)k;
    bt.first_edge = (uint32_t)f0;
    bt.n_edges = (uint32_t)(e.pos[e.coff[k + 1]] - f0);
  }
}

// ---- tandem hand-off SQL (state/daprstate.go:3643-3678, 3896-3941): the params of every binding call ----------------
// A SQL call's statements: kind i (TGI_SQL_* kind[i]) has rows[i] rows, numbered after the kinds before it; a
// statement holds k[i] consecutive rows of one kind.  A thread per row: a row is ~200 bytes of short strings (uuids, names,
// URLs), which the sequential escaper handles without the warp's 128-byte strips idling most lanes.
constexpr uint32_t ST_SQL_KINDS = 5;  // the most kinds one call renders
struct StSqlPlan {
  uint32_t kind[ST_SQL_KINDS], k[ST_SQL_KINDS];  // each kind's TGI_SQL_* code and rows per statement
  uint64_t rows[ST_SQL_KINDS], m[ST_SQL_KINDS];  // rows and statements of each kind (0 past the call's kinds)
  uint64_t n_stmts;
  uint32_t crawl_len, time_len;
  const uint8_t* crawl;                 // crawl_id as given, then discovery_time rendered with its quotes
  const uint8_t* time;
  uint32_t* size;                       // [rows] bytes of row r
  uint64_t* off;                        // [rows+1] their scan
  uint64_t* sc;                         // ST_SC_*: ST_SC_BIG
  uint8_t* out;
  tgi_state_edge_stmt* stmts;           // [n_stmts]
  uint64_t sql_off[2 * ST_SQL_KINDS], sql_len[2 * ST_SQL_KINDS];  // kind i's texts: [2i] k[i] rows, [2i+1] its last,
                                                                  // shorter statement
  uint64_t base;                        // the params' offset in the output
};

// one row's values, sized (EMIT false) or written at dst: the statement's "[" before its first row and "," before the
// others, quoted escaped strings, page fields, numbers, raw bytes (the rendered clock), "]" after its last row
template <bool EMIT>
struct StSqlRow {
  uint8_t* dst;
  StLen<EMIT> o;
  DEVI void lit(const void* s, uint32_t n) {
    if (EMIT)
      for (uint32_t k = 0; k < n; k++) dst[o + k] = ((const uint8_t*)s)[k];
    o += n;
  }
  DEVI void str(const uint8_t* s, uint32_t n) {
    lit("\"", 1);
    o += EMIT ? st_thread_esc(dst + o, s, n) : thread_esc_len<StLen<EMIT>>(s, n);
    lit("\"", 1);
  }
  DEVI void field(const StDev& d, const tgi_state_page& p, int f) {
    uint32_t n;
    const uint8_t* s = st_str(d, p, f, n);
    str(s, n);
  }
  DEVI void num(long long v) { o += EMIT ? (uint32_t)render_i64(dst + o, v) : ndigits_i64(v); }
  DEVI void open(uint64_t j, uint32_t k) { lit(j % k ? "," : "[", 1); }  // row j of its kind
  DEVI void close(uint64_t j, uint32_t k, uint64_t n) {
    if (j % k == k - 1 || j == n - 1) lit("]", 1);
  }
};

// every statement's entry: its kind, rows, text and params' span
DEVI void st_sql_stmts(const StSqlPlan& q) {
  for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < q.n_stmts; s += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t kind = 0;
    uint64_t j = s, first = 0;
    for (; j >= q.m[kind]; kind++) {
      j -= q.m[kind];
      first += q.rows[kind];
    }
    first += j * q.k[kind];
    const uint32_t rows = (uint32_t)min((uint64_t)q.k[kind], q.rows[kind] - j * q.k[kind]);
    const uint32_t t = 2 * kind + (rows != q.k[kind]);
    tgi_state_edge_stmt& st = q.stmts[s];
    st.kind = q.kind[kind];
    st.rows = rows;
    st.sql_off = q.sql_off[t];
    st.sql_len = q.sql_len[t];
    st.params_off = q.base + q.off[first];
    st.params_len = q.off[first + rows] - q.off[first];
  }
}

// the hand-off's rows: batch inserts [0, nb), edge inserts [nb, nb + ne), batch closes [nb + ne, 2 nb + ne)
struct StSql {
  StSqlPlan p;                          // rows {nb, ne, nb} from TGI_SQL_BATCH_INSERT
  const tgi_state_edge* edges;          // the hand-off, as tgi_state_pending_edges left it on the device
  const tgi_state_edge_batch* batches;
  const tgi_state_span* spans;
};

template <bool EMIT>
DEVI StLen<EMIT> st_sql_row(const StDev& d, const StSql& q, uint64_t r, uint8_t* dst) {
  StSqlRow<EMIT> w{dst, 0};
  const uint64_t nb = q.p.rows[0], ne = q.p.rows[1];
  const uint32_t kind = r < nb ? 0u : r < nb + ne ? 1u : 2u;
  const uint64_t i = kind == 0 ? r : kind == 1 ? r - nb : r - nb - ne;  // the row within its kind
  w.open(i, q.p.k[kind]);
  const tgi_state_edge* e = kind == 1 ? q.edges + i : nullptr;
  const tgi_state_edge_batch& b = q.batches[e ? e->batch : (uint32_t)i];
  w.str(b.batch_id, 36);
  if (kind != 2) {
    const tgi_state_page& p = d.pages[q.spans[b.span].row];  // the owner
    w.lit(",", 1);
    w.str(q.p.crawl, q.p.crawl_len);
    w.lit(",", 1);
    if (kind == 0) {  // CreatePendingBatch (daprstate.go:3897-3906)
      w.field(d, p, TGI_PS_URL);
      w.lit(",", 1);
      w.field(d, p, TGI_PS_ID);
      w.lit(",", 1);
      w.num(p.depth);
      w.lit(",", 1);
      w.field(d, p, TGI_PS_SEQ);
      w.lit(",\"open\"", 7);
    } else {  // InsertPendingEdge (:3915-3926)
      w.str(e->destination, e->dest_len);
      w.lit(",", 1);
      w.field(d, p, TGI_PS_URL);
      w.lit(",", 1);
      w.field(d, p, TGI_PS_SEQ);
      w.lit(",", 1);
      w.lit(q.p.time, q.p.time_len);
      switch (e->source_type) {  // tdutils.go:978-987
        case TGI_SRC_MENTION: w.lit(",\"mention\"", 10); break;
        case TGI_SRC_TEXT_URL: w.lit(",\"text_url\"", 11); break;
        case TGI_SRC_URL: w.lit(",\"url\"", 6); break;
        default: w.lit(",\"plaintext\"", 12); break;
      }
      w.lit(",\"pending\"", 10);
    }
  }
  w.close(i, q.p.k[kind], kind == 1 ? ne : nb);
  return w.o;
}

__global__ void st_sql_size_kernel(StDev d, StSql q) {
  const uint64_t n_rows = q.p.rows[0] + q.p.rows[1] + q.p.rows[2];
  for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n_rows; r += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t sz = st_sql_row<false>(d, q, r, nullptr);
    q.p.size[r] = (uint32_t)sz;
    st_flag_big(q.p.sc, sz);
  }
}

// the rows at their scanned offsets, then the statement table
__global__ void st_sql_emit_kernel(StDev d, StSql q) {
  const uint64_t n_rows = q.p.rows[0] + q.p.rows[1] + q.p.rows[2];
  for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n_rows; r += (uint64_t)gridDim.x * blockDim.x)
    st_sql_row<true>(d, q, r, q.p.out + q.p.off[r]);
  st_sql_stmts(q.p);
}

// ---- tandem forced walkback (crawl/runner.go:115-139, 1425-1455): the pick and the two rows of every edge-less span ---
struct StWalk {
  const uint32_t* spans;           // [n][2] every edge-less span's index and row, in span order
  uint64_t n;
  FrontierDev disc;                // TGI_SET_DISCOVERED (table == nullptr: never allocated)
  uint64_t seed, w0;               // the id key, and the walkback counter of the first span
  tgi_state_walkback_span* out;    // [n]
  uint32_t* ok;                    // [n] 1: TGI_WALK_OK
};

// A walker's draw stream: word 2j and 2j + 1 are Philox block (ctr_lo, ctr_hi, domain, j)'s x0 | x1 << 32 and
// x2 | x3 << 32 under the id key
struct StDraws {
  uint64_t seed, ctr;
  uint32_t domain;
  uint64_t next = 0;
  uint32_t c[4];
  DEVI uint64_t word() {
    if (!(next & 1)) {
      c[0] = (uint32_t)ctr, c[1] = (uint32_t)(ctr >> 32), c[2] = domain, c[3] = (uint32_t)(next >> 1);
      philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
    }
    return (next++ & 1) ? (c[2] | (uint64_t)c[3] << 32) : (c[0] | (uint64_t)c[1] << 32);
  }
  // Lemire's multiply-and-reject: exactly uniform on [0, N), N > 0, as rand.IntN
  DEVI uint64_t below(uint64_t N) {
    uint64_t x = word(), l = x * N;
    if (l < N) {
      const uint64_t t = (0 - N) % N;
      while (l < t) l = (x = word()) * N;
    }
    return __umul64hi(x, N);
  }
};

// key[0, klen) == s[0, n), byte for byte
DEVI bool st_key_eq(const Key32& key, uint32_t klen, const uint8_t* s, uint32_t n) {
  bool eq = klen == n;
  for (uint32_t k = 0; eq && k < n; k++) eq = ((key.w[k >> 2] >> (8 * (k & 3))) & 0xFF) == s[k];
  return eq;
}

// pickWalkbackChannel(sm, source, exclude) (crawl/runner.go:120-139) over the set's keys in first-occurrence order
// (Random() is keys[rand.Intn(len(keys))], state/datamodels.go:152-162): up to 10 draws from r, a draw equal to
// source[0, sl) or excluded(key, klen) retried, over the set's first N keys (N = 0: the set is empty or was never
// allocated).  Returns TGI_WALK_*; key / klen hold the pick when TGI_WALK_OK, else 0.
DEVI uint64_t st_set_count(const FrontierDev& disc) { return disc.table ? *disc.count : 0; }
template <class X>
DEVI uint32_t st_pick_walkback(StDraws& r, const FrontierDev& disc, uint64_t N, const uint8_t* src, uint32_t sl, X&& excluded,
                               Key32& key, uint32_t& klen, uint32_t& draws) {
  uint32_t status = N ? TGI_WALK_EXHAUSTED : TGI_WALK_EMPTY;
  key = Key32{};
  klen = draws = 0;
  while (N && draws < TGI_WALK_MAX_DRAWS) {
    draws++;
    key = load_key(disc.pool + 32 * r.below(N));
    klen = 32;
    while (klen && !((key.w[(klen - 1) >> 2] >> (8 * ((klen - 1) & 3))) & 0xFF)) klen--;
    if (!st_key_eq(key, klen, src, sl) && !excluded(key, klen)) {  // url == sourceURL || exclude[url]
      status = TGI_WALK_OK;
      break;
    }
  }
  if (status != TGI_WALK_OK) key = Key32{}, klen = 0;
  return status;
}

// one span's pickWalkbackChannel(sm, owner.URL, nil) and its two ids
__global__ void st_walk_pick_kernel(StDev d, StWalk w) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < w.n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t wi = w.w0 + i;
    uint32_t ul;
    const uint8_t* u = st_str(d, d.pages[w.spans[2 * i + 1]], TGI_PS_URL, ul);
    tgi_state_walkback_span& o = w.out[i];
    Key32 key;
    uint32_t draws, klen;
    StDraws r{w.seed, wi, 2u};
    const uint32_t status = st_pick_walkback(r, w.disc, st_set_count(w.disc), u, ul, [](const Key32&, uint32_t) { return false; },
                                             key, klen, draws);
    o.span = w.spans[2 * i];
    o.status = status;
    o.draws = draws;
    o.url_len = klen;
    store_key(o.url, key);
    st_uuid(w.seed, wi, 3u, o.page_id);
    st_uuid(w.seed, wi, 4u, o.sequence_id);
    w.ok[i] = status == TGI_WALK_OK;
  }
}

// The SQL of the picks: rows page_buffer [0, n_ok), edge_records [n_ok, 2 n_ok) in span order.  Thread t of [0, 2 n)
// stands for span t % n's row of kind t / n, which it has when the span is TGI_WALK_OK; rank[i] is its place among those.
struct StWalkSql {
  StSqlPlan p;                         // rows {n_ok, n_ok} from TGI_SQL_PAGE_BUFFER_INSERT
  const uint32_t* spans;               // StWalk's
  const tgi_state_walkback_span* wb;   // [n] the picks
  const uint64_t* rank;                // [n+1] scan of StWalk::ok
  uint64_t n;
};

template <bool EMIT>
DEVI StLen<EMIT> st_walk_row(const StDev& d, const StWalkSql& q, uint32_t kind, uint64_t i, uint64_t j, uint8_t* dst) {
  StSqlRow<EMIT> w{dst, 0};
  const tgi_state_walkback_span& b = q.wb[i];
  const tgi_state_page& p = d.pages[q.spans[2 * i + 1]];  // the owner
  w.open(j, q.p.k[kind]);
  if (kind == 0) {  // AddPageToPageBuffer (daprstate.go:3620-3633)
    w.str(b.page_id, 36);
    w.lit(",", 1);
    w.field(d, p, TGI_PS_ID);
    w.lit(",", 1);
    w.num((int64_t)((uint64_t)p.depth + 1));  // owner.Depth + 1 wraps as Go's int
    w.lit(",", 1);
    w.str(b.url, b.url_len);
    w.lit(",", 1);
    w.str(q.p.crawl, q.p.crawl_len);
    w.lit(",", 1);
    w.str(b.sequence_id, 36);
  } else {  // SaveEdgeRecords of the walkback edge (:3176-3184)
    w.str(b.url, b.url_len);
    w.lit(",", 1);
    w.field(d, p, TGI_PS_URL);
    w.lit(",true,false,", 12);
    w.lit(q.p.time, q.p.time_len);
    w.lit(",", 1);
    w.str(q.p.crawl, q.p.crawl_len);
    w.lit(",", 1);
    w.field(d, p, TGI_PS_SEQ);
  }
  w.close(j, q.p.k[kind], q.p.rows[0]);
  return w.o;
}

__global__ void st_walk_size_kernel(StDev d, StWalkSql q) {
  for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < 2 * q.n; t += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t kind = t >= q.n;
    const uint64_t i = t - kind * q.n, j = q.rank[i];
    if (q.rank[i + 1] > j) {
      const uint64_t sz = st_walk_row<false>(d, q, kind, i, j, nullptr);
      q.p.size[kind * q.p.rows[0] + j] = (uint32_t)sz;
      st_flag_big(q.p.sc, sz);
    }
  }
}

// the rows at their scanned offsets, then the statement table
__global__ void st_walk_emit_kernel(StDev d, StWalkSql q) {
  for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < 2 * q.n; t += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t kind = t >= q.n;
    const uint64_t i = t - kind * q.n, j = q.rank[i];
    if (q.rank[i + 1] > j) st_walk_row<true>(d, q, kind, i, j, q.p.out + q.p.off[kind * q.p.rows[0] + j]);
  }
  st_sql_stmts(q.p);
}

// ---- validator walkback (crawl/validator.go:360-489): processWalkbackBatch of every claimed batch -------------------
struct StVw {
  const tgi_claimed_batch* b;      // [n] the claimed batches, their edges and strings as uploaded
  const uint64_t* eoff;            // [n+1]
  const tgi_claimed_edge* e;
  const uint8_t* s;
  uint64_t n;
  int64_t rate;                    // cfg.WalkbackRate
  FrontierDev disc;                // TGI_SET_DISCOVERED (table == nullptr: never allocated)
  uint64_t seed, v0;               // the id key, and the counter of the first batch
  tgi_state_validator_batch* out;  // [n]
  uint32_t* vlist;                 // [n_edges] batch i's valid edges (index within it) at [eoff[i], + n_valid)
  uint32_t* tlist;                 // [n_edges] the first edge of each of its distinct source types at [eoff[i], + d)
  uint32_t* cnt;                   // [3n] per batch: 1 when TGI_WALK_OK; its edge rows; its stats rows
};

// FlushBatchStats' key of an edge: its source_type, "unknown" when empty (daprstate.go:4140-4143)
DEVI const uint8_t* st_vw_type(const StVw& v, const tgi_claimed_edge& e, uint32_t& n) {
  n = e.str_len[TGI_CE_SOURCE_TYPE];
  if (!n) {
    n = 7;
    return (const uint8_t*)"unknown";
  }
  return v.s + e.str_off[TGI_CE_SOURCE_TYPE];
}
DEVI bool st_bytes_eq(const uint8_t* a, uint32_t an, const uint8_t* b, uint32_t bn) {
  bool eq = an == bn;
  for (uint32_t k = 0; eq && k < an; k++) eq = a[k] == b[k];
  return eq;
}

// one batch: its valid edges and distinct source types, the decision, the pick, the two ids and its row counts
__global__ void st_vw_pick_kernel(StVw v) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < v.n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t e0 = v.eoff[i], m = v.eoff[i + 1] - e0, vi = v.v0 + i;
    const tgi_claimed_edge* E = v.e + e0;
    uint32_t nv = 0, nt = 0;
    for (uint32_t q = 0; q < (uint32_t)m; q++) {
      if (E[q].cls == TGI_EDGE_CLASS_VALID) v.vlist[e0 + nv++] = q;
      uint32_t tl, ul;
      const uint8_t* t = st_vw_type(v, E[q], tl);
      bool first = true;
      for (uint32_t r = 0; first && r < nt; r++) first = !st_bytes_eq(t, tl, st_vw_type(v, E[v.tlist[e0 + r]], ul), ul);
      if (first) v.tlist[e0 + nt++] = q;
    }
    StDraws r{v.seed, vi, 5u};
    const tgi_claimed_batch& b = v.b[i];
    int32_t rnd = -1;
    bool walkback = true;
    if (nv) {
      rnd = (int32_t)r.below(100) + 1;
      walkback = v.rate >= rnd;
    }
    Key32 key{};
    uint32_t status = TGI_WALK_OK, draws = 0, klen = 0, fwd = TGI_VW_NO_EDGE;
    if (walkback) {
      const uint32_t* vl = v.vlist + e0;
      auto excluded = [&](const Key32& k, uint32_t kl) {  // exclude[url]: the batch's valid channels
        for (uint32_t x = 0; x < nv; x++) {
          const tgi_claimed_edge& c = E[vl[x]];
          if (st_key_eq(k, kl, v.s + c.str_off[TGI_CE_DESTINATION], c.str_len[TGI_CE_DESTINATION])) return true;
        }
        return false;
      };
      status = st_pick_walkback(r, v.disc, st_set_count(v.disc), v.s + b.str_off[TGI_CB_SOURCE_CHANNEL], b.str_len[TGI_CB_SOURCE_CHANNEL],
                                excluded, key, klen, draws);
    } else {
      fwd = v.vlist[e0 + r.below(nv)];
    }
    tgi_state_validator_batch& o = v.out[i];
    o.status = status;
    o.walkback = walkback;
    o.rnd = rnd;
    o.draws = draws;
    o.n_valid = nv;
    o.forward_edge = fwd;
    o.url_len = klen;
    o.reserved = 0;
    store_key(o.url, key);
    st_uuid(v.seed, vi, 6u, o.page_id);
    st_uuid(v.seed, vi, 7u, o.sequence_id);
    const bool ok = status == TGI_WALK_OK;
    v.cnt[i] = ok;
    v.cnt[v.n + i] = ok ? 1 + nv - !walkback : 0;  // the primary, then the valid channels not followed
    v.cnt[2 * v.n + i] = ok ? nt : 0;
  }
}

// The SQL of the OK batches: rows of page_buffer, edge_records, complete, stats upsert, delete.  Row j of a kind
// belongs to the batch whose rank range holds it: rank (one row per OK batch), erank or srank (scans of StVw::cnt).
struct StVwSql {
  StSqlPlan p;                     // rows {n_ok, edge rows, n_ok, stats rows, n_ok} from TGI_SQL_PAGE_BUFFER_INSERT
  StVw v;
  const uint64_t* rank;            // [3 (n+1)]: the scans of StVw::cnt's three parts
};

// the last batch i with rank[i] <= j: the batch of row j
DEVI uint64_t st_vw_batch(const uint64_t* rank, uint64_t n, uint64_t j) {
  uint64_t a = 0, b = n - 1;
  while (a < b) {
    const uint64_t mid = (a + b + 1) >> 1;
    if (rank[mid] <= j) a = mid;
    else b = mid - 1;
  }
  return a;
}

template <bool EMIT>
DEVI StLen<EMIT> st_vw_row(const StVwSql& q, uint64_t r, uint8_t* dst) {
  uint32_t kind = 0;
  uint64_t j = r;
  while (j >= q.p.rows[kind]) j -= q.p.rows[kind++];
  const StVw& v = q.v;
  const uint64_t* rank = q.rank + (kind == 1 ? 1 : kind == 3 ? 2 : 0) * (v.n + 1);
  const uint64_t i = st_vw_batch(rank, v.n, j), x = j - rank[i];  // the batch, and the row within its rows of the kind
  const tgi_claimed_batch& b = v.b[i];
  const tgi_state_validator_batch& o = v.out[i];
  const tgi_claimed_edge* E = v.e + v.eoff[i];
  StSqlRow<EMIT> w{dst, 0};
  auto bstr = [&](int f) { w.str(v.s + b.str_off[f], b.str_len[f]); };
  auto crawl = [&]() {  // the batch's CrawlID, else the configured one (daprstate.go:3181-3183, 3623-3626)
    if (b.str_len[TGI_CB_CRAWL_ID]) bstr(TGI_CB_CRAWL_ID);
    else w.str(q.p.crawl, q.p.crawl_len);
  };
  auto edge = [&](uint32_t y) { w.str(v.s + E[y].str_off[TGI_CE_DESTINATION], E[y].str_len[TGI_CE_DESTINATION]); };
  auto url = [&]() {  // nextURL
    if (o.walkback) w.str(o.url, o.url_len);
    else edge(o.forward_edge);
  };
  w.open(j, q.p.k[kind]);
  if (kind == 0) {  // AddPageToPageBuffer (daprstate.go:3620-3633) of validator.go:430-438's page
    w.str(o.page_id, 36);
    w.lit(",", 1);
    bstr(TGI_CB_SOURCE_PAGE_ID);
    w.lit(",", 1);
    w.num((int64_t)((uint64_t)b.source_depth + 1));  // SourceDepth + 1 wraps as Go's int
    w.lit(",", 1);
    url();
    w.lit(",", 1);
    crawl();
    w.lit(",", 1);
    if (o.walkback) w.str(o.sequence_id, 36);
    else bstr(TGI_CB_SEQUENCE_ID);
  } else if (kind == 1) {  // SaveEdgeRecords (:3176-3184) of the primary edge, then the skipped ones (validator.go:446-473)
    if (x == 0) {
      url();
    } else {  // the valid channels in edge order without the followed one
      const uint32_t* vl = v.vlist + v.eoff[i];
      const uint32_t y = (uint32_t)x - 1;
      edge(vl[y] < o.forward_edge ? vl[y] : vl[y + 1]);  // a walkback's forward_edge is past every edge
    }
    w.lit(",", 1);
    bstr(TGI_CB_SOURCE_CHANNEL);
    if (x) w.lit(",false,true,", 12);
    else if (o.walkback) w.lit(",true,false,", 12);
    else w.lit(",false,false,", 13);
    w.lit(q.p.time, q.p.time_len);
    w.lit(",", 1);
    crawl();
    w.lit(",", 1);
    bstr(TGI_CB_SEQUENCE_ID);
  } else if (kind == 3) {  // FlushBatchStats' upsert of one source_type (daprstate.go:4137-4166)
    bstr(TGI_CB_CRAWL_ID);
    w.lit(",", 1);
    uint32_t tl, ul;
    const uint8_t* t = st_vw_type(v, E[v.tlist[v.eoff[i] + x]], tl);
    w.str(t, tl);
    long long c[5] = {0, 0, 0, 0, 0};  // total, valid, not_channel, invalid, duplicate
    const uint32_t m = (uint32_t)(v.eoff[i + 1] - v.eoff[i]);
    for (uint32_t e = 0; e < m; e++)
      if (st_bytes_eq(t, tl, st_vw_type(v, E[e], ul), ul)) {
        c[0]++;
#pragma unroll
        for (uint32_t f = 0; f < 4; f++) c[1 + f] += E[e].cls == f;  // the switch's four cases; OTHER is in total only
      }
#pragma unroll
    for (int f = 0; f < 5; f++) {
      w.lit(",", 1);
      w.num(c[f]);
    }
  } else {  // CompletePendingBatch (:4125-4130), FlushBatchStats' delete (:4170-4174)
    bstr(TGI_CB_BATCH_ID);
  }
  w.close(j, q.p.k[kind], q.p.rows[kind]);
  return w.o;
}

__global__ void st_vw_size_kernel(StDev, StVwSql q) {
  const uint64_t n_rows = q.p.rows[0] + q.p.rows[1] + q.p.rows[2] + q.p.rows[3] + q.p.rows[4];
  for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n_rows; r += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t sz = st_vw_row<false>(q, r, nullptr);
    q.p.size[r] = (uint32_t)sz;
    st_flag_big(q.p.sc, sz);
  }
}

// the rows at their scanned offsets, then the statement table
__global__ void st_vw_emit_kernel(StDev, StVwSql q) {
  const uint64_t n_rows = q.p.rows[0] + q.p.rows[1] + q.p.rows[2] + q.p.rows[3] + q.p.rows[4];
  for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n_rows; r += (uint64_t)gridDim.x * blockDim.x)
    st_vw_row<true>(q, r, q.p.out + q.p.off[r]);
  st_sql_stmts(q.p);
}

// ---- standard random walk (crawl/runner.go:1218-1227, 1245-1384, 1458-1540): lookups, then the replay of a step -----
// Every name's candidates depend only on its own history, so only its first candidate of the call acts: skipped when
// the name is invalid or discovered, a seed hit, or a lookup; every later candidate is skipped (the first left the name
// discovered or invalid, or retired the replay).
enum : uint32_t { ST_RW_SKIP = 0, ST_RW_SEED = 1, ST_RW_LOOKUP = 2 };

struct StRw {
  const StCand* c;           // the gather's candidates in (span, record, link) order
  const uint32_t* link;      // [bound] each candidate's link row in the result
  const uint64_t* coff;      // [n_spans+1]; coff[n_spans] = the count
  uint64_t bound;
  const uint32_t* bfirst;    // st_first_kernel's batch table over the call, and every candidate's slot in it
  const uint32_t* slot_of;
  const tgi_state_span* spans;
  uint32_t n_spans;
  const uint32_t* link_off;  // the slot's resident result
  const tgi_link* links;
  ExclusionDev x;            // TGI_SET_INVALID with the call's clock, TGI_SET_DISCOVERED
  FrontierDev seeds;         // TGI_SET_SEEDS
  uint32_t* cls;             // [bound] ST_RW_*
  uint32_t* flag;            // [bound] 1: a lookup
  uint64_t* pos;             // [bound+1] scan of flag: each candidate's lookup index
  tgi_rw_lookup* out;
};

__global__ void st_rw_class_kernel(StRw r) {
  const uint64_t n = r.coff[r.n_spans];
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < r.bound; j += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t cl = ST_RW_SKIP;
    if (j < n && r.bfirst[r.slot_of[j]] == (uint32_t)j) {
      const Key32 k = load_key(r.c[j].name);
      const uint64_t h = key_hash(k);
      if (!set_invalid_hit(r.x, k, h, r.x.now_sec) && set_lookup(r.x.discovered, k, h) < 0)  // :1247, :1310
        cl = set_lookup(r.seeds, k, h) >= 0 ? ST_RW_SEED : ST_RW_LOOKUP;                      // :1312
    }
    r.cls[j] = cl;
    r.flag[j] = cl == ST_RW_LOOKUP;
  }
}

// the lookup rows: name, span, the record that holds the link row, its source
__global__ void st_rw_lookup_kernel(StRw r) {
  const uint64_t n = r.coff[r.n_spans];
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    if (!r.flag[j]) continue;
    const StCand& c = r.c[j];
    const uint32_t L = r.link[j];
    const tgi_state_span s = r.spans[c.span];
    uint64_t a = s.first, b = s.first + s.n_done - 1;  // the record that holds link row L
    while (a < b) {
      const uint64_t mid = (a + b + 1) >> 1;
      if (r.link_off[mid] <= L) a = mid;
      else b = mid - 1;
    }
    tgi_rw_lookup& o = r.out[r.pos[j]];
    store_key(o.name, load_key(c.name));
    o.record = a;
    o.span = c.span;
    o.name_len = (uint8_t)c.len;
    o.source_type = r.links[L].src;
    o.reserved = 0;
  }
}

// The step over the lists of the lookups: lookups [0, nl) apply and so do the candidates before the retiring lookup's
// (of [0, cut)); spans [0, n_dec) decide, and span n_dec is retired when a lookup retires.
struct StRwStep {
  const StCand* c;           // the lookups' lists
  const uint32_t* cls;
  const uint64_t* lpos;
  const uint64_t* coff;
  const tgi_state_span* spans;
  uint32_t n_spans, n_dec;
  const tgi_rw_lookup* lk;
  const tgi_rw_outcome* oc;
  uint64_t nl, cut;          // the lookups before the first retire; the candidates
  uint32_t* flag;            // [2 nl + cut]: found, failed (lookups), discovered insert (candidates)
  uint64_t* pos;             // [3][...+1] their scans: seed upsert rows, invalid upsert rows, discovered inserts
  uint64_t* pos_i;
  uint64_t* pos_d;
  uint32_t* flist;           // [found] the lookup of every seed upsert row = the newChannels of every span
  uint32_t* ilist;           // [failed] the lookup of every invalid upsert row
  uint8_t* fkeys;            // [found][32], [failed][32], [inserts][32]: the three sets' keys in candidate order
  uint8_t* ikeys;
  uint8_t* dkeys;
  const uint32_t* dnew;      // [inserts] 1: the discovered insert added its key
  const uint64_t* npos;      // [inserts+1] its scan
  const uint64_t* n0;        // TGI_SET_DISCOVERED's count before the inserts
  FrontierDev disc;          // TGI_SET_DISCOVERED after them
  int64_t rate;              // cfg.WalkbackRate
  uint64_t seed, u0;         // the id key, and the counter of the first deciding span
  tgi_rw_span* out;          // [n_spans]
  uint32_t* cnt;             // [2 n_spans]: 1 when the span writes its page; its edge rows
};

// every lookup's and applied candidate's effects as flags
__global__ void st_rw_flags_kernel(StRwStep w) {
  const uint64_t m = max(w.nl, w.cut);
  for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < m; t += (uint64_t)gridDim.x * blockDim.x) {
    if (t < w.nl) {
      const uint32_t o = w.oc[t].code;
      w.flag[t] = o == TGI_RW_FOUND;
      w.flag[w.nl + t] = o == TGI_RW_NOT_FOUND || o == TGI_RW_NOT_SUPERGROUP;
    }
    if (t < w.cut) {  // candidate t applies when it comes before the retiring lookup: lpos[t + 1] <= nl
      const uint32_t cl = w.cls[t];
      const bool applies = w.lpos[t] + (cl == ST_RW_LOOKUP) <= w.nl;
      w.flag[2 * w.nl + t] = applies && (cl == ST_RW_SEED || (cl == ST_RW_LOOKUP && w.oc[w.lpos[t]].code == TGI_RW_FOUND));
    }
  }
}

// the flagged rows and keys compacted in candidate order
__global__ void st_rw_compact_kernel(StRwStep w) {
  const uint64_t m = max(w.nl, w.cut);
  for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < m; t += (uint64_t)gridDim.x * blockDim.x) {
    if (t < w.nl && w.flag[t]) {
      w.flist[w.pos[t]] = (uint32_t)t;
      store_key(w.fkeys + 32 * w.pos[t], load_key(w.lk[t].name));
    }
    if (t < w.nl && w.flag[w.nl + t]) {
      w.ilist[w.pos_i[t]] = (uint32_t)t;
      store_key(w.ikeys + 32 * w.pos_i[t], load_key(w.lk[t].name));
    }
    if (t < w.cut && w.flag[2 * w.nl + t]) store_key(w.dkeys + 32 * w.pos_d[t], load_key(w.c[t].name));
  }
}

// MarkChannelInvalid's stamp of every failed lookup's name, the new ones' and the expired ones' alike
__global__ void st_rw_stamp_kernel(FrontierDev inv, const uint8_t* keys, uint64_t n, long long now_sec) {
  for (uint64_t q = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; q < n; q += (uint64_t)gridDim.x * blockDim.x) {
    const Key32 k = load_key(keys + 32 * q);
    const int64_t pi = set_lookup(inv, k, key_hash(k));
    if (pi >= 0) inv.payload[pi] = (uint64_t)now_sec;
  }
}

// the discovered insert's NEW flags as scan input
__global__ void st_rw_new_kernel(const uint8_t* is_new, uint64_t n, uint32_t* out) {
  for (uint64_t q = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; q < n; q += (uint64_t)gridDim.x * blockDim.x)
    out[q] = is_new[q];
}

DEVI const uint8_t* st_rw_name(const StRwStep& w, uint64_t f, uint32_t& len) {  // seed upsert row f's name
  const tgi_rw_lookup& l = w.lk[w.flist[f]];
  len = l.name_len;
  return l.name;
}

// one span: its newChannels, the decision, the pick, the two ids and its row counts
__global__ void st_rw_span_kernel(StDev d, StRwStep w) {
  for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < w.n_spans; s += (uint64_t)gridDim.x * blockDim.x) {
    tgi_rw_span& o = w.out[s];
    Key32 key{};
    uint32_t status = s == w.n_dec ? TGI_RW_RETIRED : TGI_RW_DEFERRED, draws = 0, klen = 0, fwd = TGI_RW_NO_FORWARD;
    uint32_t n_new = 0;
    int32_t rnd = -1;
    bool walkback = false;
    if (s < w.n_dec) {
      const uint64_t ui = w.u0 + s, c1 = w.coff[s + 1];
      const uint64_t f0 = w.pos[w.lpos[w.coff[s]]], f1 = w.pos[w.lpos[c1]];
      n_new = (uint32_t)(f1 - f0);
      StDraws r{w.seed, ui, 8u};
      if (n_new) rnd = (int32_t)r.below(100) + 1;
      walkback = !n_new || w.rate >= rnd;  // :1471-1482
      if (walkback) {
        uint32_t ul;
        const uint8_t* u = st_str(d, d.pages[w.spans[s].row], TGI_PS_URL, ul);
        auto excluded = [&](const Key32& k, uint32_t kl) {  // exclude = newChannels
          for (uint64_t f = f0; f < f1; f++) {
            uint32_t nl;
            const uint8_t* nm = st_rw_name(w, f, nl);
            if (st_key_eq(k, kl, nm, nl)) return true;
          }
          return false;
        };
        const uint64_t N = *w.n0 + w.npos[w.pos_d[c1]];  // the set after this span's candidates
        status = st_pick_walkback(r, w.disc, N, u, ul, excluded, key, klen, draws);
      } else {
        fwd = (uint32_t)r.below(n_new);
        const tgi_rw_lookup& l = w.lk[w.flist[f0 + fwd]];
        key = load_key(l.name);
        klen = l.name_len;
        status = TGI_WALK_OK;
      }
      st_uuid(w.seed, ui, 9u, o.page_id);
      st_uuid(w.seed, ui, 10u, o.sequence_id);
    } else {
      for (int q = 0; q < 36; q++) o.page_id[q] = o.sequence_id[q] = 0;
    }
    o.status = status;
    o.walkback = walkback;
    o.rnd = rnd;
    o.draws = draws;
    o.n_new = n_new;
    o.forward = fwd;
    o.url_len = klen;
    o.reserved = 0;
    store_key(o.url, key);
    const bool ok = status == TGI_WALK_OK;
    w.cnt[s] = ok;
    w.cnt[w.n_spans + s] = ok ? 1 + n_new - !walkback : 0;  // the primary, then the new channels not followed
  }
}

// The SQL of the step: rows of seed upserts, invalid upserts, page_buffer, edge_records.  A page or edge row belongs to
// the span whose rank range holds it (scans of StRwStep::cnt's two parts).
struct StRwSql {
  StSqlPlan p;               // rows {found, failed, pages, edge rows}
  StRwStep w;
  const uint64_t* rank;      // [2 (n_spans+1)]
};

template <bool EMIT>
DEVI StLen<EMIT> st_rw_row(const StDev& d, const StRwSql& q, uint64_t r, uint8_t* dst) {
  uint32_t kind = 0;
  uint64_t j = r;
  while (j >= q.p.rows[kind]) j -= q.p.rows[kind++];
  const StRwStep& w = q.w;
  StSqlRow<EMIT> o{dst, 0};
  o.open(j, q.p.k[kind]);
  if (kind == 0) {  // UpsertSeedChannelChatID (daprstate.go:3395-3402)
    uint32_t nl;
    const uint8_t* nm = st_rw_name(w, j, nl);
    o.str(nm, nl);
    o.lit(",", 1);
    o.num(w.oc[w.flist[j]].chat_id);
  } else if (kind == 1) {  // MarkChannelInvalid (:3569-3578)
    const tgi_rw_lookup& l = w.lk[w.ilist[j]];
    o.str(l.name, l.name_len);
    if (w.oc[w.ilist[j]].code == TGI_RW_NOT_FOUND) o.lit(",\"not_found\"", 12);
    else o.lit(",\"not_supergroup\"", 17);
  } else {
    const uint64_t* rank = q.rank + (kind == 3) * (w.n_spans + 1);
    const uint64_t s = st_vw_batch(rank, w.n_spans, j), x = j - rank[s];  // the span, and the row within its rows
    const tgi_state_page& p = d.pages[w.spans[s].row];  // the owner
    const tgi_rw_span& b = w.out[s];
    if (kind == 2) {  // AddPageToPageBuffer (:3620-3633) of runner.go:1459-1504's page
      o.str(b.page_id, 36);
      o.lit(",", 1);
      o.field(d, p, TGI_PS_ID);
      o.lit(",", 1);
      o.num((int64_t)((uint64_t)p.depth + 1));  // owner.Depth + 1 wraps as Go's int
      o.lit(",", 1);
      o.str(b.url, b.url_len);
      o.lit(",", 1);
      o.str(q.p.crawl, q.p.crawl_len);
      o.lit(",", 1);
      if (b.walkback) o.str(b.sequence_id, 36);
      else o.field(d, p, TGI_PS_SEQ);
    } else {  // SaveEdgeRecords (:3176-3184): the primary edge, then the skipped ones (runner.go:1505-1535)
      if (x == 0) {
        o.str(b.url, b.url_len);
      } else {
        const uint64_t f0 = w.pos[w.lpos[w.coff[s]]], y = x - 1;
        uint32_t nl;
        const uint8_t* nm = st_rw_name(w, f0 + (y < b.forward ? y : y + 1), nl);  // a walkback's forward is past all
        o.str(nm, nl);
      }
      o.lit(",", 1);
      o.field(d, p, TGI_PS_URL);
      if (x) o.lit(",false,true,", 12);
      else if (b.walkback) o.lit(",true,false,", 12);
      else o.lit(",false,false,", 13);
      o.lit(q.p.time, q.p.time_len);
      o.lit(",", 1);
      o.str(q.p.crawl, q.p.crawl_len);
      o.lit(",", 1);
      o.field(d, p, TGI_PS_SEQ);
    }
  }
  o.close(j, q.p.k[kind], q.p.rows[kind]);
  return o.o;
}

__global__ void st_rw_size_kernel(StDev d, StRwSql q) {
  const uint64_t n_rows = q.p.rows[0] + q.p.rows[1] + q.p.rows[2] + q.p.rows[3];
  for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n_rows; r += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t sz = st_rw_row<false>(d, q, r, nullptr);
    q.p.size[r] = (uint32_t)sz;
    st_flag_big(q.p.sc, sz);
  }
}

// the rows at their scanned offsets, then the statement table
__global__ void st_rw_emit_kernel(StDev d, StRwSql q) {
  const uint64_t n_rows = q.p.rows[0] + q.p.rows[1] + q.p.rows[2] + q.p.rows[3];
  for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n_rows; r += (uint64_t)gridDim.x * blockDim.x)
    st_rw_row<true>(d, q, r, q.p.out + q.p.off[r]);
  st_sql_stmts(q.p);
}

// ---- json.Marshal(map[int][]string) of the layer map ----------------------------------------------------------------
struct StLmEntry {  // one id of a layer, or an empty layer (row == ST_NONE)
  uint32_t row;
  uint32_t pre;      // the layer's opening [,]"<depth>":[ in StLm::keys, written by its first entry
  uint32_t pre_len;  // 0: not the layer's first entry
  uint32_t last;     // 1: the entry closes the layer with ]
};
struct StLm {
  const StLmEntry* entries;
  uint64_t n;
  const uint8_t* keys;
  uint32_t* size;  // [n] bytes of entry e
  uint64_t* off;   // [n+1] their scan
  uint64_t* sc;    // ST_SC_*: ST_SC_BIG
  uint8_t* out;
};

// one entry, sized (EMIT false) or written: [opening][,]"<escaped id>"[]]
template <bool EMIT>
DEVI StLen<EMIT> st_lm_entry(const StDev& d, const StLm& L, const StLmEntry& e, uint8_t* dst) {
  StLen<EMIT> o = 0;
  auto ch = [&](uint32_t c) {
    if (EMIT) dst[o] = (uint8_t)c;
    o++;
  };
  if (EMIT)
    for (uint32_t k = 0; k < e.pre_len; k++) dst[k] = L.keys[e.pre + k];
  o += e.pre_len;
  if (e.row != ST_NONE) {
    if (!e.pre_len) ch(',');
    ch('"');
    uint32_t il;
    const uint8_t* id = st_str(d, d.pages[e.row], TGI_PS_ID, il);
    o += EMIT ? st_thread_esc(dst + o, id, il) : thread_esc_len<StLen<EMIT>>(id, il);
    ch('"');
  }
  if (e.last) ch(']');
  return o;
}

__global__ void st_lm_size_kernel(StDev d, StLm L) {
  for (uint64_t e = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; e < L.n; e += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t sz = st_lm_entry<false>(d, L, L.entries[e], nullptr);
    L.size[e] = (uint32_t)sz;
    st_flag_big(L.sc, sz);
  }
}
__global__ void st_lm_emit_kernel(StDev d, StLm L) {
  for (uint64_t e = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; e < L.n; e += (uint64_t)gridDim.x * blockDim.x)
    st_lm_entry<true>(d, L, L.entries[e], L.out + L.off[e]);
}

}  // namespace tgi
