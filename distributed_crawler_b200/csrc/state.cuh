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
// Render: live messages are compacted and grouped by row with the stable radix passes of local_appends.cuh (order
// inside a row = storage order); a thread per message sizes it, a warp per entry (a page of a layer, or an empty layer)
// sizes the page around its messages, scans place both, and the emit writes every byte at its final offset: a warp per
// entry for the page's fields, a thread per (entry, message) slot for the messages.
#pragma once
#include "local_appends.cuh"

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

// ---- compaction / read-back -------------------------------------------------------------------------------------
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
__global__ void st_read_kernel(StDev d, uint64_t n, const uint32_t* flag, const uint64_t* pos, tgi_state_msg* out) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    if (!flag[i]) continue;
    const StMsg m = d.msgs[i];
    tgi_state_msg o;
    o.chat_id = m.chat;
    o.message_id = m.msg;
    o.page_id = m.pid;
    o.status = m.status;
    o.platform = m.platform;
    out[pos[i]] = o;
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
  uint32_t* flag;      // [n_msgs] live flags
  uint64_t* pos;       // [n_msgs+1] their scan
  uint32_t* keys[2];   // radix ping-pong: row, message index
  uint32_t* vals[2];
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
// the scalars block: live messages, body bytes, message slots, a timestamp that does not render, an entry of 4 GiB or
// more, message bytes, rows, radix counts
enum { ST_SC_LIVE, ST_SC_BYTES, ST_SC_SLOTS, ST_SC_ERR, ST_SC_BIG, ST_SC_MBYTES, ST_SC_ROWS, ST_SC_RADIX, ST_SC_COUNT };

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
DEVI uint32_t st_message(const StDev& d, const StMsg& m, bool comma, uint8_t* dst) {
  uint32_t o = 0;
  auto lit = [&](const char* s, uint32_t n) {
    if (EMIT)
      for (uint32_t k = 0; k < n; k++) dst[o + k] = (uint8_t)s[k];
    o += n;
  };
  auto esc = [&](const uint8_t* s, uint32_t n) { o += EMIT ? st_thread_esc(dst + o, s, n) : thread_esc_len(s, n); };
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

// live flags of every message row
__global__ void st_render_flag_kernel(StDev d, uint64_t n, StRender r) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    r.flag[i] = st_live(d, d.msgs[i]);
}
// the live messages compacted in storage order: the radix sort's input pairs (row, message index)
__global__ void st_render_pairs_kernel(StDev d, uint64_t n, StRender r) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    if (!r.flag[i]) continue;
    const uint64_t k = r.pos[i];
    r.keys[0][k] = d.msgs[i].row;
    r.vals[0][k] = (uint32_t)i;
  }
}
// size pass, a thread per grouped message k (sorted = the grouped message indices, sorted_rows their rows)
__global__ void st_msg_size_kernel(StDev d, StRender r, const uint32_t* sorted, const uint32_t* sorted_rows, uint64_t live) {
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < live; k += (uint64_t)gridDim.x * blockDim.x)
    r.msize[k] = st_message<false>(d, d.msgs[sorted[k]], k != r.row_base[sorted_rows[k]], nullptr);
}

// one entry, sized or written by a warp (lane 0 writes the literals, the warp escapes the strings).  Returns the bytes
// of part A (framing and fields up to the first message) in *a and of the whole entry without messages.
template <bool EMIT>
DEVI uint32_t st_entry(const StDev& d, const StRender& r, const StEntry& e, uint32_t cnt, uint8_t* dst, uint64_t msg_bytes,
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
    o += EMIT ? esc_to_global(dst + o, s, n) : warp_esc_len(s, n);
  };
  if (e.flags & ST_E_FIRST) {
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
  if (e.flags & ST_E_LAST) lit("]}", 2);
  return (uint32_t)(o - msg_bytes);
}

constexpr int ST_WARPS = 8;  // warps per CTA of the warp-per-entry kernels

// size pass, a warp per entry: the entry's bytes around its messages, its message count and message bytes
__global__ void __launch_bounds__(ST_WARPS * 32) st_entry_size_kernel(StDev d, StRender r) {
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
    const uint32_t sz = st_entry<false>(d, r, en, cnt, nullptr, mb, &a, &bad);
    if (lane_id() == 0) {
      r.esize_lo[e] = a;
      r.ebytes[e] = sz;
      r.ecnt[e] = cnt;
      r.esz[e] = (uint32_t)(sz + mb);
      if (sz + mb > 0xFFFFFFFFull) atomicMax((unsigned long long*)r.sc + ST_SC_BIG, 1ull);
      if (bad) atomicMax((unsigned long long*)r.sc + ST_SC_ERR, 1ull);
    }
  }
}

// emit, a warp per entry: everything but the messages
__global__ void __launch_bounds__(ST_WARPS * 32) st_entry_emit_kernel(StDev d, StRender r) {
  const uint64_t w0 = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5, nw = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t e = w0; e < r.n_entries; e += nw) {
    const StEntry en = r.entries[e];
    const uint64_t off = r.eoff[e];
    const uint64_t mb = r.eoff[e + 1] - off - r.ebytes[e];
    uint32_t a;
    bool bad = false;
    st_entry<true>(d, r, en, r.ecnt[e], r.out + off, mb, &a, &bad);
    __syncwarp();
  }
}

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

}  // namespace tgi
