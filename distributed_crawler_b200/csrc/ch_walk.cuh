// ch_walk.cuh — channel record -> model.ChannelData line, the random-walk StoreChannelData output.
//
// Replaces the ChannelData literal of RunForChannel (crawl/runner.go:592-610) followed by json.Marshal+'\n' in
// DaprStateManager.StoreChannelData (state/daprstate.go:3089-3094).  Field order: model/data.go:89-111.  The same small
// templated walk as the generic line (one warp per record, YtSizer for the length pass, YtWriter for the emit pass),
// with the escaper and integer writers they share.
#pragma once
#include "yt_walk.cuh"

namespace tgi {

struct ChBatchDev {
  uint64_t n;
  const tgi_ch_rec* recs;
  const uint8_t* strs;
};

// the largest string length a record may carry: six escaped bytes per input byte keep a line below 2^32 bytes
constexpr uint32_t CH_STR_MAX = (1u << 24) - 1;

// the string ranges of record r are inside strs (the host and ch_validate_kernel apply it before any kernel reads them)
__host__ __device__ inline bool ch_rec_ok(const tgi_ch_rec& v, uint64_t strs_len) {
  if (v.title_len > CH_STR_MAX || v.image_len > CH_STR_MAX || v.url_len > CH_STR_MAX) return false;
  const uint64_t end = v.str_off + (uint64_t)v.title_len + v.image_len + v.url_len;
  return end <= strs_len && end >= v.str_off;
}

template <class W>
DEVI void walk_ch_record(W& w, const ChBatchDev& b, uint64_t r) {
  const tgi_ch_rec v = b.recs[r];
  const uint8_t *title = b.strs + v.str_off, *image = title + v.title_len, *url = image + v.image_len;
  YLIT(w, "{\"channel_id\":\""); w.dec(v.chat_id);                                            // strconv.FormatInt(chat.Id, 10)
  YLIT(w, "\",\"channel_name\":\""); w.esc(title, v.title_len);                               // chat.Title
  YLIT(w, "\",\"channel_description\":\"\",\"channel_profile_image\":\""); w.esc(image, v.image_len);  // chat.Photo.Extra
  YLIT(w, "\",\"channel_engagement_data\":{\"follower_count\":"); w.dec(v.member_count);
  YLIT(w, ",\"following_count\":0,\"like_count\":0,\"post_count\":"); w.dec(v.message_count);
  YLIT(w, ",\"views_count\":"); w.dec(v.total_views);
  // "https://t.me/" is ASCII, so escaping it and p.URL apart is escaping the Sprintf result
  YLIT(w, ",\"comment_count\":0,\"share_count\":0},\"channel_url_external\":\"https://t.me/"); w.esc(url, v.url_len);
  YLIT(w, "\",\"channel_url\":\"https://t.me/"); w.esc(url, v.url_len);
  YLIT(w, "\",\"country_code\":\"\",\"published_at\":\"0001-01-01T00:00:00Z\"}\n");  // the zero time.Time
}

}  // namespace tgi
