// sink_src.cuh — what the result sinks (dapr.cuh, local_appends.cuh, combine.cuh) read of a slot's last Telegram or
// YouTube result that is still resident on the device, and the rules they share (sm_90a).
#pragma once
#include "kernels.cuh"

namespace tgi {

struct SinkSrc {
  uint64_t n;                 // records of the result
  const uint8_t* status;      // its status [n], line offsets [n+1] and lines
  const uint64_t* line_off;
  const uint8_t* jsonl;
  bool yt;
  const tgi_tg_rec* tg_recs;  // the resident batch: records, channel rows and their strings
  const tgi_tg_chan* tg_chans;
  const tgi_yt_rec* yt_recs;
  const tgi_yt_chan* yt_chans;
  const uint8_t* strs;
  const uint8_t* chan_strs;
  uint32_t n_chans;
};

// the channel row of record i
DEVI uint32_t sink_rec_chan(const SinkSrc& s, uint64_t i) { return s.yt ? s.yt_recs[i].chan_idx : s.tg_recs[i].chan_idx; }

// the channelID of channel row `row`: Telegram the row's name (tdutils.go:725), YouTube the row's id
// (youtube_crawler.go:396)
DEVI const uint8_t* sink_chan_id(const SinkSrc& s, uint32_t row, uint32_t& len) {
  if (s.yt) {
    const tgi_yt_chan& ch = s.yt_chans[row];
    len = ch.id_len;
    return s.chan_strs + ch.str_off;
  }
  const tgi_tg_chan& ch = s.tg_chans[row];
  len = ch.name_len;
  return s.chan_strs + ch.str_off + ch.title_len;
}

// one base64 character of a 6-bit value: A-Z a-z 0-9 + / (StdEncoding)
DEVI uint32_t b64_char(uint32_t v) {
  return v + (v < 26 ? 'A' : v < 52 ? 'a' - 26 : v < 62 ? (uint32_t)('0' - 52) : v == 62 ? (uint32_t)('+' - 62) : (uint32_t)('/' - 63));
}

// 4 base64 characters of 3 bytes; n = 1 or 2 valid bytes pad with '=' (the bytes behind them are ignored)
DEVI uint32_t b64_word(uint32_t b0, uint32_t b1, uint32_t b2, uint32_t n) {
  const uint32_t x = (b0 << 16) | (n > 1 ? b1 << 8 : 0u) | (n > 2 ? b2 : 0u);
  const uint32_t c2 = n > 1 ? b64_char((x >> 6) & 63) : '=';
  const uint32_t c3 = n > 2 ? b64_char(x & 63) : '=';
  return b64_char(x >> 18) | (b64_char((x >> 12) & 63) << 8) | (c2 << 16) | (c3 << 24);
}

}  // namespace tgi
