// gm_walk.cuh — generic client.Message -> sparse model.Post line (SURVEY §8 a12).
//
// Replaces TelegramCrawler.convertMessageToPost (crawler/telegram/telegram_crawler.go:179-262; the
// message is what TelegramClient.getMessagesWithClient builds, client/clients.go:296-339) followed by
// json.Marshal(post)+'\n'.  A secondary path of the reference: the same small templated walk as the
// YouTube line (one warp per record, YtSizer for the length pass, YtWriter for the emit pass).
#pragma once
#include "tg_walk.cuh"
#include "yt_walk.cuh"

namespace tgi {

struct GmBatchDev {
  uint64_t n;
  const tgi_gm_rec* recs;
  const uint8_t* strs;
  const uint32_t* react_off;
  const tgi_gm_reaction* reacts;
  const uint8_t* aux;
};

// returns false if a time field is not representable (Marshal error -> TGI_ST_NOLINE)
template <class W>
DEVI bool walk_gm_record(W& w, const GmBatchDev& b, const CfgDev& cfg, uint64_t r) {
  const tgi_gm_rec v = b.recs[r];
  const uint8_t *id = b.strs + v.str_off, *chan = id + v.id_len, *text = chan + v.channel_len, *sender = text + v.text_len;
  const int l = lane_id();
  uint32_t tl = 0;
  __syncwarp();
  if (l == 0) tl = (uint32_t)render_zone_time(w.sc->num, v.ts_sec, v.ts_nsec, cfg.zone, cfg.zone_n, cfg.tz);  // :187 GetTimestamp()
  __syncwarp();
  const uint32_t pub_len = __shfl_sync(FULL, tl, 0);
  if (pub_len == 0 || (cfg.flags & CFGDEV_CLOCK_INVALID) || cfg.created_yt_len == 0) return false;
  const uint8_t* created = cfg.blob + cfg.off[2];  // time.Now(), local zone, nanoseconds kept (:188)
  const uint8_t* capture = cfg.blob + cfg.off[3];  // :245

  YLIT(w, "{\"post_link\":\"\",\"channel_id\":\""); w.esc(chan, v.channel_len);  // :184
  YLIT(w, "\",\"post_uid\":\""); w.esc(id, v.id_len);                           // :185
  YLIT(w, "\",\"url\":\"\",\"published_at\":"); w.smem(pub_len);
  YLIT(w, ",\"created_at\":"); w.raw(created, cfg.created_yt_len);
  YLIT(w, ",\"language_code\":\"\",\"engagement\":0,\"view_count\":"); w.dec(v.views);  // :191
  YLIT(w, ",\"like_count\":0,\"share_count\":0,\"comment_count\":0,\"crawl_label\":\"\",\"list_ids\":null,"
          "\"channel_name\":\"");
  w.esc(chan, v.channel_len);  // :197
  YLIT(w, "\",\"search_terms\":null,\"search_term_ids\":null,\"project_ids\":null,\"exercise_ids\":null,"
          "\"label_data\":null,\"labels_metadata\":null,\"project_labeled_post_ids\":null,"
          "\"labeler_ids\":null,\"all_labels\":null,\"label_ids\":null,\"is_ad\":false,"
          "\"transcript_text\":\"\",\"image_text\":\"\",\"video_length\":null,\"is_verified\":null,"
          "\"channel_data\":{\"channel_id\":\"\",\"channel_name\":\"\",\"channel_description\":\"\","
          "\"channel_profile_image\":\"\",\"channel_engagement_data\":{\"follower_count\":0,"
          "\"following_count\":0,\"like_count\":0,\"post_count\":0,\"views_count\":0,\"comment_count\":0,"
          "\"share_count\":0},\"channel_url_external\":\"\",\"channel_url\":\"\",\"country_code\":\"\","
          "\"published_at\":\"0001-01-01T00:00:00Z\"},\"platform_name\":\"telegram\",\"shared_id\":null,"  // :213
          "\"quoted_id\":null,\"replied_id\":null,\"ai_label\":null,\"root_post_id\":null,"
          "\"engagement_steps_count\":0,\"ocr_data\":null,\"performance_scores\":{\"likes\":null,"
          "\"shares\":null,\"comments\":null,\"views\":0},\"has_embed_media\":null,\"description\":\"");
  w.esc(text, v.text_len);  // :223
  YLIT(w, "\",\"repost_channel_data\":null,\"post_type\":null,\"inner_link\":{},\"post_title\":null,"
          "\"media_data\":{\"document_name\":\"\"},\"is_reply\":null,\"ad_fields\":null,\"likes_count\":0,"
          "\"shares_count\":0,\"comments_count\":0,\"views_count\":");
  w.dec(v.views);  // :234
  YLIT(w, ",\"searchable_text\":\""); w.esc(text, v.text_len);  // :235
  YLIT(w, "\",\"all_text\":\""); w.esc(text, v.text_len);       // :236
  YLIT(w, "\",\"contrast_agent_project_ids\":null,\"agent_ids\":null,\"segment_ids\":null,\"thumb_url\":\"\","
          "\"media_url\":\"\",\"comments\":null,\"reactions\":");
  {
    const uint32_t r0 = b.react_off ? b.react_off[r] : 0u, r1 = b.react_off ? b.react_off[r + 1] : 0u;
    if (r1 == r0) {  // :250 nil map
      YLIT(w, "null");
    } else {
      // map[string]int: keys in byte order, the last entry of a key wins.  Every lane runs the same
      // scalar selection (the data is warp-uniform); maps are small.
      w.ch('{');
      int prev = -1;
      for (;;) {
        int best = -1;
        for (uint32_t j = r0; j < r1; j++) {
          const tgi_gm_reaction e = b.reacts[j];
          if (prev >= 0) {
            const tgi_gm_reaction p = b.reacts[prev];
            if (key_cmp(b.aux + e.key_off, e.key_len, b.aux + p.key_off, p.key_len) <= 0) continue;
          }
          if (best >= 0) {
            const tgi_gm_reaction q = b.reacts[best];
            if (key_cmp(b.aux + e.key_off, e.key_len, b.aux + q.key_off, q.key_len) > 0) continue;
          }
          best = (int)j;  // smaller key, or the same key again (later duplicate overwrites)
        }
        if (best < 0) break;
        if (prev >= 0) w.ch(',');
        const tgi_gm_reaction e = b.reacts[best];
        w.ch('"');
        w.esc(b.aux + e.key_off, e.key_len);
        YLIT(w, "\":");
        w.dec(e.count);
        prev = best;
      }
      w.ch('}');
    }
  }
  YLIT(w, ",\"outlinks\":null,\"capture_time\":"); w.raw(capture, cfg.capture_len);
  YLIT(w, ",\"handle\":\""); w.esc(sender, v.sender_len);  // :246
  YLIT(w, "\"}\n");
  return true;
}

}  // namespace tgi
