// tgingest.hpp — C++ host side above the C ABI of include/tgingest.h.
//
// The reference is Go (compiled); there is no Go toolchain in the build image, so the compiled host mirror
// of its interface for this path is C++ (the Go / cgo shim a maintainer would add is in INTEGRATION.md, the
// Python mirror the tests use is distributed_crawler_b200/{pack,engine}.py).  Names follow the reference:
//   Message / FormattedText / TextEntity   go-tdlib's client.Message as ParseMessage reads it
//                                          (telegramhelper/tdutils.go:380-732, SURVEY Appendix B)
//   ChannelInfo                            crawl.channelInfo + the per-channel arguments of ParseMessage
//   MessageProcessor::ProcessMessages      crawl.MessageProcessor (crawl/runner.go:1010-1028), batched:
//                                          one call per slice of fetched messages instead of one per message
// Header-only; link with -ltgingest.
#pragma once
#include <cstdint>
#include <cstring>
#include <optional>
#include <stdexcept>
#include <string>
#include <string_view>
#include <vector>

#include "tgingest.h"

namespace tgingest {

struct TextEntity {  // client.TextEntity
  enum Kind : uint8_t { Other = TGI_ENT_OTHER, TextUrl = TGI_ENT_TEXT_URL, Mention = TGI_ENT_MENTION, UrlEntity = TGI_ENT_URL };
  int32_t Offset = 0, Length = 0;  // UTF-16 code units
  Kind Type = Other;
  std::string Url;                 // TextEntityTypeTextUrl.Url
};
struct FormattedText {  // client.FormattedText
  std::string Text;
  std::vector<TextEntity> Entities;
};
struct Reaction {  // ReactionTypeEmoji + TotalCount (tdutils.go:591-603)
  std::string Emoji;
  int32_t TotalCount = 0;
};
struct Comment {  // model.Comment as GetMessageComments builds it (telegramutils.go:589-635)
  std::string Text;
  std::optional<std::vector<Reaction>> Reactions;  // nullopt = nil map
  int32_t ViewCount = 0, ReplyCount = 0;
  std::string Handle = "unknown";
};
struct Message {  // client.Message + the RPC results the reference resolves per message
  uint8_t ContentType = TGI_CT_TEXT;    // TGI_CT_*: MessageContentType()
  std::optional<FormattedText> Text;    // Text / Caption (nullopt = nil)
  std::string Alt;                      // emoji / poll question / prize type / file name / other type name
  std::string Media;                    // remote file id that becomes media_url
  int64_t Id = 1 << 20, ChatId = 0, MediaAlbumId = 0;
  int32_t Date = 0, ViewCount = 0, ShareCount = 0;
  std::vector<Reaction> Reactions;
  std::optional<std::vector<Comment>> Comments = std::vector<Comment>{};  // nullopt = nil slice
  std::string Handle = "unknown";       // GetPoster
  uint32_t Channel = 0;                 // row of the channel table
  bool Panics = false;                  // the reference's per-message recover() fired upstream
  // messageVideo only, the shape processMessageSafely (tdutils.go:188-199) looks at: Ok = everything there (media_url =
  // the video's remote id); None = no Video / Thumbnail: its error comes before any read, media_url stays ""; Broken = a
  // thumbnail with a nil file / remote / caption: nil dereference, recovered (:395-405), the message is "failed"
  enum class VideoShape { Ok, None, Broken } Video = VideoShape::Ok;
};
struct ChannelInfo {
  std::string Title, Name, Username;    // chat.Title, channelName argument, ActiveUsernames[0] ("" = private)
  int64_t MemberCount = 0, PostCount = 0, ViewCount = 0;
};

// The packed columnar batch of include/tgingest.h, built message by message.
class Batch {
 public:
  void AddChannel(const ChannelInfo& c) {
    tgi_tg_chan row{};
    row.str_off = (uint32_t)chan_strs_.size();
    row.title_len = (uint16_t)c.Title.size();
    row.name_len = (uint16_t)c.Name.size();
    row.user_len = (uint16_t)c.Username.size();
    row.member_count = c.MemberCount;
    row.post_count = c.PostCount;
    row.view_count = c.ViewCount;
    chan_strs_ += c.Title + c.Name + c.Username;
    chans_.push_back(row);
  }
  void Add(const Message& m) {
    tgi_tg_rec r{};
    std::string alt = m.Alt;
    const bool video = m.ContentType == TGI_CT_VIDEO;
    const std::string media = video && m.Video != Message::VideoShape::Ok ? std::string() : m.Media;
    const bool panics = m.Panics || (video && m.Video == Message::VideoShape::Broken);
    r.id = m.Id;
    r.chat_id = m.ChatId;
    r.media_album_id = m.MediaAlbumId;
    r.str_off = strs_.size();
    r.date = m.Date;
    r.view_count = m.ViewCount;
    r.share_count = m.ShareCount;
    r.chan_idx = m.Channel;
    r.text_len = m.Text ? (uint32_t)m.Text->Text.size() : 0u;
    r.alt_len = (uint32_t)alt.size();
    r.media_len = (uint16_t)media.size();
    r.handle_len = (uint16_t)m.Handle.size();
    r.content_type = m.ContentType;
    r.flags = (uint8_t)((m.Text ? TGI_RF_HAS_TEXT : 0) | (m.Comments ? 0 : TGI_RF_COMMENTS_NIL) | (panics ? TGI_RF_PANIC : 0));
    if (m.Text) strs_ += m.Text->Text;
    strs_ += alt + media + m.Handle;
    if (m.Text)
      for (const TextEntity& e : m.Text->Entities) {
        tgi_entity en{};
        en.offset = e.Offset;
        en.length = e.Length;
        en.url_off = (uint32_t)aux_.size();
        en.url_len = (uint16_t)e.Url.size();
        en.type = e.Type;
        aux_ += e.Url;
        ents_.push_back(en);
      }
    for (const Reaction& x : m.Reactions) reacts_.push_back(AddReaction(x));
    if (m.Comments)
      for (const Comment& c : *m.Comments) {
        tgi_comment cm{};
        cm.text_off = (uint32_t)aux_.size();
        cm.text_len = (uint32_t)c.Text.size();
        aux_ += c.Text;
        cm.handle_off = (uint32_t)aux_.size();
        cm.handle_len = (uint16_t)c.Handle.size();
        aux_ += c.Handle;
        cm.flags = c.Reactions ? 1 : 0;
        cm.view_count = c.ViewCount;
        cm.reply_count = c.ReplyCount;
        comment_reacts_.push_back(c.Reactions ? *c.Reactions : std::vector<Reaction>{});
        comments_.push_back(cm);
      }
    recs_.push_back(r);
    ent_off_.push_back((uint32_t)ents_.size());
    react_off_.push_back((uint32_t)reacts_.size());
    comment_off_.push_back((uint32_t)comments_.size());
  }
  size_t Size() const { return recs_.size(); }

  // Valid until the next Add*.  Comment reactions are appended behind the message reactions.
  tgi_tg_batch Descriptor() {
    all_reacts_ = reacts_;
    for (size_t k = 0; k < comments_.size(); k++) {
      comments_[k].react_start = (uint32_t)all_reacts_.size();
      comments_[k].react_count = (uint32_t)comment_reacts_[k].size();
      for (const Reaction& x : comment_reacts_[k]) all_reacts_.push_back(AddReaction(x));
    }
    comment_reacts_.assign(comments_.size(), {});  // their keys now live in aux_
    if (chans_.empty()) AddChannel(ChannelInfo{});
    tgi_tg_batch d{};
    d.n = recs_.size();
    d.recs = recs_.data();
    d.strs = (const uint8_t*)strs_.data();
    d.strs_len = strs_.size();
    d.ent_off = ent_off_.data();
    d.ents = ents_.data();
    d.react_off = react_off_.data();
    d.reacts = all_reacts_.data();
    d.n_reacts = all_reacts_.size();
    d.comment_off = comment_off_.data();
    d.comments = comments_.data();
    d.n_comments = comments_.size();
    d.aux = (const uint8_t*)aux_.data();
    d.aux_len = aux_.size();
    d.n_chans = (uint32_t)chans_.size();
    d.chans = chans_.data();
    d.chan_strs = (const uint8_t*)chan_strs_.data();
    d.chan_strs_len = chan_strs_.size();
    return d;
  }

 private:
  tgi_reaction AddReaction(const Reaction& x) {
    tgi_reaction rc{};
    rc.emoji_off = (uint32_t)aux_.size();
    rc.emoji_len = (uint16_t)x.Emoji.size();
    rc.count = x.TotalCount;
    aux_ += x.Emoji;
    return rc;
  }
  std::vector<tgi_tg_rec> recs_;
  std::string strs_, aux_, chan_strs_;
  std::vector<uint32_t> ent_off_{0}, react_off_{0}, comment_off_{0};
  std::vector<tgi_entity> ents_;
  std::vector<tgi_reaction> reacts_, all_reacts_;
  std::vector<tgi_comment> comments_;
  std::vector<std::vector<Reaction>> comment_reacts_;
  std::vector<tgi_tg_chan> chans_;
};

// One processed batch: views into library-owned pinned memory, released by the destructor.
class Result {
 public:
  Result(tgi_ctx* ctx, const tgi_result& r) : ctx_(ctx), r_(r) {}
  Result(Result&& o) noexcept : ctx_(o.ctx_), r_(o.r_) { o.ctx_ = nullptr; }
  Result(const Result&) = delete;
  ~Result() {
    if (ctx_) tgi_result_release(ctx_, r_.slot);
  }
  uint64_t Size() const { return r_.n; }
  uint8_t Status(uint64_t i) const { return r_.status[i]; }  // TGI_ST_*: emitted / skipped / failed / no line
  std::string_view Line(uint64_t i) const {                  // the JSONL line of message i ('' if none), as StorePost would write it
    return {(const char*)r_.jsonl + r_.line_off[i], (size_t)(r_.line_off[i + 1] - r_.line_off[i])};
  }
  std::vector<std::string> Outlinks(uint64_t i) const {      // what processMessage returns (crawl/runner.go:1720-1809)
    std::vector<std::string> v;
    for (uint32_t k = r_.link_off[i]; k < r_.link_off[i + 1]; k++) v.emplace_back((const char*)r_.links[k].name, r_.links[k].len);
    return v;
  }
  const tgi_result& Raw() const { return r_; }
  // DaprStateManager.StorePost's binding payloads (state/daprstate.go:1141-1181) for every message of this result:
  // base64 of its line and its blob path prefix|channelID|/posts/|PostUID|.jsonl; valid until the next call or the release
  tgi_dapr_payloads_t DaprPayloads(std::string_view path_prefix) const {
    tgi_dapr_payloads_t p{};
    if (tgi_dapr_payloads(ctx_, r_.slot, path_prefix.data(), (uint32_t)path_prefix.size(), &p) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return p;
  }
  // LocalStateManager.StorePost (state/storageproviders.go:275-298) with one append per channel file: this result's lines
  // grouped by channelID on the device, each group's in record order; valid until the next call or the release
  tgi_channel_appends_t ChannelAppends() const {
    tgi_channel_appends_t a{};
    if (tgi_channel_appends(ctx_, r_.slot, &a) != TGI_OK) throw std::runtime_error(tgi_last_error(ctx_));
    return a;
  }

 private:
  tgi_ctx* ctx_;
  tgi_result r_;
};

struct Config {
  int Device = 0;
  std::string CrawlLabel;            // cfg.CrawlLabel
  int TzOffsetSec = 0;               // time.Local as a fixed offset
  std::optional<int64_t> MinPostDate;  // cfg.MinPostDate
};

// crawl.MessageProcessor, batched.  Thread-safe like the C context (TGI_SLOTS calls overlap).
class MessageProcessor {
 public:
  explicit MessageProcessor(const Config& c) {
    tgi_config cfg{};
    cfg.abi_version = TGI_ABI_VERSION;
    cfg.device = c.Device;
    cfg.flags = TGI_CFG_SKIP_MEDIA | (c.MinPostDate ? TGI_CFG_HAS_MIN_POST_DATE : 0);
    cfg.min_post_date = c.MinPostDate.value_or(0);
    cfg.tz_offset_sec = c.TzOffsetSec;
    cfg.crawl_label = c.CrawlLabel.data();
    cfg.crawl_label_len = (uint32_t)c.CrawlLabel.size();
    if (tgi_create(&cfg, &ctx_) != TGI_OK) throw std::runtime_error(tgi_last_error(nullptr));
  }
  ~MessageProcessor() {
    if (ctx_) tgi_destroy(ctx_);
  }
  MessageProcessor(const MessageProcessor&) = delete;
  // Replaces the loop body crawl/runner.go:1161-1244 for one slice of messages.
  Result ProcessMessages(Batch& b, uint32_t run_flags = TGI_RUN_JSONL | TGI_RUN_LINKS | TGI_RUN_FRONTIER | TGI_RUN_SKIP_SELF) {
    const tgi_tg_batch d = b.Descriptor();
    tgi_result r{};
    if (tgi_telegram_batch(ctx_, &d, run_flags, &r) != TGI_OK) throw std::runtime_error(tgi_last_error(ctx_));
    return Result(ctx_, r);
  }
  void SetClock(int64_t created_sec, int32_t created_nsec, int64_t capture_sec, int32_t capture_nsec) {
    tgi_set_clock(ctx_, created_sec, created_nsec, capture_sec, capture_nsec);
  }
  // time.Local as transitions (tgi_set_zone): instant t takes offset_sec[i] of the last start_sec[i] <= t; empty
  // vectors go back to Config::TzOffsetSec.
  void SetZone(const std::vector<int64_t>& start_sec, const std::vector<int32_t>& offset_sec) {
    if (start_sec.size() != offset_sec.size()) throw std::invalid_argument("SetZone: starts and offsets differ in length");
    if (tgi_set_zone(ctx_, start_sec.data(), offset_sec.data(), (uint32_t)start_sec.size()) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
  }
  // Lets the resident sets grow on demand up to max_keys keys each, like the reference's maps (0: fixed capacity).
  void SetGrowth(uint64_t max_keys) {
    if (tgi_set_growth(ctx_, max_keys) != TGI_OK) throw std::runtime_error(tgi_last_error(ctx_));
  }
  // count / capacity / table_slots / grows of one set (TGI_SET_FRONTIER, TGI_SET_INVALID, TGI_SET_DISCOVERED, TGI_SET_OWNED)
  tgi_set_info_t SetInfo(int which) {
    tgi_set_info_t s{};
    if (tgi_set_info(ctx_, which, &s) != TGI_OK) throw std::runtime_error(tgi_last_error(ctx_));
    return s;
  }
  // Combine mode (chunk/main.go:292-421, UploadCombinedFile): the combiner's trigger, hard cap and blob path prefix
  void CombineOpen(uint64_t trigger, uint64_t hard_cap, std::string_view path_prefix) {
    if (tgi_combine_open(ctx_, trigger, hard_cap, path_prefix.data(), (uint32_t)path_prefix.size()) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
  }
  // the lines of a result go to the combiner; the blobs this closes, valid until the next combine call
  tgi_combined_t CombineAdd(const Result& r, int64_t unix_nano) {
    tgi_combined_t o{};
    if (tgi_combine_add(ctx_, r.Raw().slot, unix_nano, &o) != TGI_OK) throw std::runtime_error(tgi_last_error(ctx_));
    return o;
  }
  tgi_combined_t CombineFlush(int64_t unix_nano) {  // Chunker shutdown
    tgi_combined_t o{};
    if (tgi_combine_flush(ctx_, unix_nano, &o) != TGI_OK) throw std::runtime_error(tgi_last_error(ctx_));
    return o;
  }
  // SetState / Initialize on the device-resident crawl state (tgi_state_set): layers[k] takes the next
  // layers[k].n_pages pages, pages[i] the next pages[i].n_msgs messages; returns every page's row
  std::vector<uint32_t> StateSet(const std::vector<tgi_state_layer>& layers, const std::vector<tgi_state_page>& pages,
                                 std::string_view strs, const std::vector<tgi_state_msg>& msgs) {
    std::vector<uint32_t> rows(pages.size());
    if (tgi_state_set(ctx_, layers.data(), (uint32_t)layers.size(), pages.data(), pages.size(), (const uint8_t*)strs.data(),
                      strs.size(), msgs.data(), msgs.size(), rows.data()) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return rows;
  }
  // json.Marshal(GetState()): state.json with the caller's marshalled metadata and lastUpdated spliced in; the view
  // stays valid until the next state call
  std::string_view StateRender(std::string_view metadata_json, std::string_view last_updated_json) {
    tgi_state_json_t o{};
    if (tgi_state_render(ctx_, (const uint8_t*)metadata_json.data(), metadata_json.size(), (const uint8_t*)last_updated_json.data(),
                         last_updated_json.size(), &o) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return std::string_view((const char*)o.data, o.len);
  }
  tgi_ctx* Raw() { return ctx_; }

 private:
  tgi_ctx* ctx_ = nullptr;
};

}  // namespace tgingest
