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

// The channel records of one random-walk step (tgi_ch_batch): what RunForChannel puts in model.ChannelData for each
// channel page it holds (crawl/runner.go:587-607), packed for MessageProcessor::StoreChannelData.
class ChannelBatch {
 public:
  // chat.Id, chat.Title, chat.Photo.Extra ("" when Photo == nil), p.URL and the int32 counts (runner.go:980-982)
  void Add(int64_t chat_id, std::string_view title, std::string_view image, std::string_view url, int32_t member_count,
           int32_t message_count, int32_t total_views) {
    tgi_ch_rec r{};
    r.chat_id = chat_id;
    r.str_off = strs_.size();
    r.member_count = member_count;
    r.message_count = message_count;
    r.total_views = total_views;
    r.title_len = (uint32_t)title.size();
    r.image_len = (uint32_t)image.size();
    r.url_len = (uint32_t)url.size();
    strs_.append(title).append(image).append(url);
    recs_.push_back(r);
  }
  size_t Size() const { return recs_.size(); }
  tgi_ch_batch Descriptor() const {
    return tgi_ch_batch{recs_.size(), recs_.data(), (const uint8_t*)strs_.data(), strs_.size()};
  }

 private:
  std::vector<tgi_ch_rec> recs_;
  std::string strs_;
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
  // The random-walk StoreChannelData lines (daprstate.go:3089-3094) of a step's channel pages; feed the result to
  // Result::DaprPayloads (paths prefix|url|/channel_data.jsonl) or to the combiner.
  Result StoreChannelData(const ChannelBatch& b, uint32_t run_flags = TGI_RUN_JSONL) {
    const tgi_ch_batch d = b.Descriptor();
    tgi_result r{};
    if (tgi_channel_batch(ctx_, &d, run_flags, &r) != TGI_OK) throw std::runtime_error(tgi_last_error(ctx_));
    return Result(ctx_, r);
  }
  void SetClock(int64_t created_sec, int32_t created_nsec, int64_t capture_sec, int32_t capture_nsec) {
    if (tgi_set_clock(ctx_, created_sec, created_nsec, capture_sec, capture_nsec) != TGI_OK) throw std::runtime_error(tgi_last_error(ctx_));
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
  // DaprStateManager.SaveState's json.Marshal(layerMap); the view stays valid until the next state call
  std::string_view StateLayerMap() {
    tgi_state_json_t o{};
    if (tgi_state_layer_map(ctx_, &o) != TGI_OK) throw std::runtime_error(tgi_last_error(ctx_));
    return std::string_view((const char*)o.data, o.len);
  }
  // Dapr's AddLayer for the pages that passed the caller's urlCache test, into the layer `depth` (pages[0].Depth
  // before that test); returns every page's row
  std::vector<uint32_t> StateAddPages(int64_t depth, const std::vector<tgi_state_page>& pages, std::string_view strs) {
    std::vector<uint32_t> rows(pages.size());
    if (tgi_state_add_pages(ctx_, depth, pages.data(), pages.size(), (const uint8_t*)strs.data(), strs.size(), rows.data()) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return rows;
  }
  // ExportPagesToBinding's chunks (TGI_STATE_EXPORT_DAPR: base64, chunk_bytes as exportChunkSizeBytes) or the local
  // export's one raw JSONL chunk; the views stay valid until the next state call.  TGI_E_NOPAGES (Dapr: no page in the
  // layer map) throws like every other error.
  std::vector<std::string_view> StateExport(int mode, uint64_t chunk_bytes) {
    tgi_state_export_t o{};
    if (tgi_state_export(ctx_, mode, chunk_bytes, &o) != TGI_OK) throw std::runtime_error(tgi_last_error(ctx_));
    std::vector<std::string_view> v;
    for (uint64_t k = 0; k < o.n_chunks; k++) v.emplace_back((const char*)o.data + o.off[k], o.len[k]);
    return v;
  }
  // A page turn of processAllMessagesWithProcessor: addNewMessages + resampleMarker + UpdatePage for the fetched
  // (chat_id, message_id) pairs (page: the owner's new fields, or nullptr); pack the batch as fetched[work[i]], run it,
  // then StatePageEnd(turn, slot, n_done) makes the loop's UpdateMessage calls from the slot's result.  work and
  // page_json stay valid until the next state call.
  tgi_state_turn_t StatePageBegin(uint32_t row, const std::vector<int64_t>& fetched, bool page_json,
                                  const tgi_state_page* page = nullptr, std::string_view strs = {}) {
    tgi_state_turn_t t{};
    if (tgi_state_page_begin(ctx_, row, page, (const uint8_t*)strs.data(), strs.size(), fetched.data(), fetched.size() / 2,
                             page_json ? TGI_TURN_PAGE_JSON : 0u, &t) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return t;
  }
  uint64_t StatePageEnd(uint32_t turn, int slot, uint64_t n_done) {
    uint64_t appended = 0;
    if (tgi_state_page_end(ctx_, turn, slot, nullptr, n_done, &appended) != TGI_OK) throw std::runtime_error(tgi_last_error(ctx_));
    return appended;
  }
  // UpdatePage(*owner) after the loop, and the Dapr runner's UpdatePage(page) after it: page's fields replace the
  // row's, and the row's list becomes the last begin's owner view while it holds one.  With page_json the view of
  // json.Marshal(page) stays valid until the next state call; else it is empty.
  std::string_view StatePageClose(uint32_t row, const tgi_state_page& page, std::string_view strs, bool page_json) {
    tgi_state_json_t o{};
    if (tgi_state_page_close(ctx_, row, &page, (const uint8_t*)strs.data(), strs.size(), page_json ? TGI_TURN_PAGE_JSON : 0u,
                             &o) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return page_json ? std::string_view((const char*)o.data, o.len) : std::string_view();
  }
  // Multi-page turns: the pages of many channels in one call per step.  Page k's fetched keys are
  // fetched[2*fetched_off[k] .. 2*fetched_off[k+1]); work indexes the whole fetched array, so the caller packs every
  // page's work into one batch, runs it, and ends the turn from records [first, first + n_work) of that result.  The
  // returned arrays stay valid until the next state call.
  tgi_state_pages_t StatePagesBegin(const std::vector<uint32_t>& rows, const std::vector<int64_t>& fetched,
                                    const std::vector<uint64_t>& fetched_off, bool page_json,
                                    const tgi_state_page* pages = nullptr, std::string_view strs = {}) {
    tgi_state_pages_t t{};
    if (tgi_state_pages_begin(ctx_, rows.data(), (uint32_t)rows.size(), pages, (const uint8_t*)strs.data(), strs.size(),
                              fetched.data(), fetched.size() / 2, fetched_off.data(), page_json ? TGI_TURN_PAGE_JSON : 0u,
                              &t) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return t;
  }
  tgi_state_end_t StatePagesEnd(uint32_t turn, int slot, uint64_t first, const std::vector<uint64_t>& n_done = {}) {
    tgi_state_end_t o{};
    if (tgi_state_pages_end(ctx_, turn, slot, first, nullptr, n_done.empty() ? nullptr : n_done.data(), &o) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return o;
  }
  tgi_state_pages_t StatePagesClose(const std::vector<uint32_t>& rows, const std::vector<tgi_state_page>& pages,
                                    std::string_view strs, bool page_json) {
    tgi_state_pages_t o{};
    if (tgi_state_pages_close(ctx_, rows.data(), (uint32_t)rows.size(), pages.data(), (const uint8_t*)strs.data(), strs.size(),
                              page_json ? TGI_TURN_PAGE_JSON : 0u, &o) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return o;
  }
  // Snowball discovery: the outlinks of the slot's Telegram result as next-layer pages.  StateDiscover with
  // TGI_DISCOVER_NOW is the standalone runner's AddLayer per page; without it the candidates wait in the pending list
  // for StateNextLayer, the Dapr runner's layer end.  The returned arrays stay valid until the next state call.
  void StateIdSeed(uint64_t seed) {
    if (tgi_state_id_seed(ctx_, seed) != TGI_OK) throw std::runtime_error(tgi_last_error(ctx_));
  }
  tgi_state_added_t StateDiscover(int slot, const std::vector<tgi_state_span>& spans, uint32_t flags, int64_t now_sec,
                                  int32_t now_nsec, int64_t max_pages = 0) {
    tgi_state_added_t a{};
    if (tgi_state_discover(ctx_, slot, spans.data(), (uint32_t)spans.size(), flags, now_sec, now_nsec, max_pages, &a) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return a;
  }
  tgi_state_added_t StateNextLayer(int64_t layer_depth, uint32_t flags, int64_t now_sec, int32_t now_nsec, int64_t max_pages = 0) {
    tgi_state_added_t a{};
    if (tgi_state_next_layer(ctx_, layer_depth, flags, now_sec, now_nsec, max_pages, &a) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return a;
  }
  // Tandem hand-off: every span's pending-edge batch from the slot's Telegram result, seenInBatch per page; a span with
  // span_batch[k] == TGI_STATE_NO_BATCH made no batch (the forced walkback).  The arrays stay valid until the next
  // state call.
  tgi_state_edges_t StatePendingEdges(int slot, const std::vector<tgi_state_span>& spans, int64_t now_sec) {
    tgi_state_edges_t a{};
    if (tgi_state_pending_edges(ctx_, slot, spans.data(), (uint32_t)spans.size(), now_sec, &a) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return a;
  }
  // Tandem hand-off SQL: the Postgres binding calls that store the last StatePendingEdges, rows_per_stmt rows per
  // statement; statement k is an exec with metadata {"sql": data[sql_off, +sql_len), "params": data[params_off,
  // +params_len)}.  The arrays stay valid until the next state call.
  tgi_state_edge_sql_t StateEdgeSql(std::string_view crawl_id, int64_t now_sec, int32_t now_nsec, uint32_t rows_per_stmt) {
    tgi_state_edge_sql_t o{};
    if (tgi_state_edge_sql(ctx_, crawl_id.data(), (uint32_t)crawl_id.size(), now_sec, now_nsec, rows_per_stmt, &o) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return o;
  }
  // Tandem forced walkback: for every span of the last StatePendingEdges without edges, a channel picked from the
  // discovered set (walkbacks[k].status TGI_WALK_*), and the exec calls that store the TGI_WALK_OK ones as StateEdgeSql's
  // are read.  A span that is not OK is the reference's random-walk-walkback error for its page.  The arrays stay valid
  // until the next state call.
  tgi_state_walkback_t StateWalkback(std::string_view crawl_id, int64_t now_sec, int32_t now_nsec, uint32_t rows_per_stmt) {
    tgi_state_walkback_t o{};
    if (tgi_state_walkback(ctx_, crawl_id.data(), (uint32_t)crawl_id.size(), now_sec, now_nsec, rows_per_stmt, &o) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return o;
  }
  // Validator walkback: processWalkbackBatch for n claimed batches (batches[k].status TGI_WALK_*; a batch that is not OK
  // is the reference's random-walk-walkback error and stays claimed), and the exec calls of the OK ones as StateEdgeSql's
  // are read.  Ends a live StatePendingEdges hand-off.  The arrays stay valid until the next state call.
  tgi_state_validator_walkback_t StateValidatorWalkback(const tgi_claimed_batches& in, int64_t walkback_rate,
                                                        std::string_view crawl_id, int64_t now_sec, int32_t now_nsec,
                                                        uint32_t rows_per_stmt) {
    tgi_state_validator_walkback_t o{};
    if (tgi_state_validator_walkback(ctx_, &in, walkback_rate, crawl_id.data(), (uint32_t)crawl_id.size(), now_sec,
                                     now_nsec, rows_per_stmt, &o) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return o;
  }
  // Standard random walk: the SearchPublicChat calls of many pages (RwLookups), then, with one outcome per lookup, the
  // step (RwStep): the sets' updates, every page's walkback decision and pick (spans[k].status TGI_WALK_*, or
  // TGI_RW_RETIRED / TGI_RW_DEFERRED past a retiring FLOOD_WAIT) and the exec calls as StateEdgeSql's are read.  The
  // arrays stay valid until the next state call.
  tgi_state_rw_lookups_t RwLookups(int slot, const std::vector<tgi_state_span>& spans, int64_t now_sec) {
    tgi_state_rw_lookups_t o{};
    if (tgi_state_rw_lookups(ctx_, slot, spans.data(), (uint32_t)spans.size(), now_sec, &o) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return o;
  }
  tgi_state_rw_step_t RwStep(const std::vector<tgi_rw_outcome>& outcomes, int64_t walkback_rate, std::string_view crawl_id,
                             int64_t now_sec, int32_t now_nsec, uint32_t rows_per_stmt) {
    tgi_state_rw_step_t o{};
    if (tgi_state_rw_step(ctx_, outcomes.data(), outcomes.size(), walkback_rate, crawl_id.data(), (uint32_t)crawl_id.size(),
                          now_sec, now_nsec, rows_per_stmt, &o) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return o;
  }
  // Layer reads: GetLayerByDepth with a runner's selection (TGI_SELECT_*), GetPage of many rows, and the layer summary
  // (GetMaxDepth, FindIncompleteCrawl's page test).  ReadLayer's selected rows go to StatePagesBegin as they are; with
  // messages each page's list is msgs[msg_first[k] .. + pages[k].n_msgs).  The arrays stay valid until the next state call.
  tgi_state_read_t ReadLayer(int64_t depth, int select, bool messages) {
    tgi_state_read_t o{};
    if (tgi_state_read_layer(ctx_, depth, select, messages ? TGI_READ_MESSAGES : 0u, &o) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return o;
  }
  tgi_state_read_t ReadPages(const std::vector<uint32_t>& rows, bool messages) {
    tgi_state_read_t o{};
    if (tgi_state_read_pages(ctx_, rows.data(), rows.size(), messages ? TGI_READ_MESSAGES : 0u, &o) != TGI_OK)
      throw std::runtime_error(tgi_last_error(ctx_));
    return o;
  }
  // the rows the read's selection processes, in layer order (every row without a selection)
  static std::vector<uint32_t> SelectedRows(const tgi_state_read_t& r) {
    std::vector<uint32_t> out;
    for (uint64_t k = 0; k < r.n_pages; k++)
      if (!r.select || r.select[k]) out.push_back(r.rows[k]);
    return out;
  }
  tgi_state_layers_t Layers() {
    tgi_state_layers_t o{};
    if (tgi_state_layers(ctx_, &o) != TGI_OK) throw std::runtime_error(tgi_last_error(ctx_));
    return o;
  }
  tgi_ctx* Raw() { return ctx_; }

 private:
  tgi_ctx* ctx_ = nullptr;
};

}  // namespace tgingest
