// host_demo.cpp — exercises the C++ host mirror (tgingest.hpp).
//   host_demo --pack   prints an FNV-1a hash of every packed array (no GPU needed): tests/test_host_cpp.py
//                      packs the same messages with pack.py and compares
//   host_demo --run    processes them on the GPU and prints status, outlinks and the JSONL lines
//   host_demo --state  the same, then a one-page crawl state (StateSet) rendered as state.json (StateRender)
//   host_demo --state-dapr  the same state, then a Dapr AddLayer of two pages at depth -1 (StateAddPages), the layer
//                      map (StateLayerMap) and ExportPagesToBinding's base64 chunks of 100 bytes (StateExport)
#include <cstdio>
#include <cstring>

#include "tgingest.hpp"

using namespace tgingest;

static uint64_t fnv(const void* p, size_t n) {
  uint64_t h = 1469598103934665603ull;
  for (size_t i = 0; i < n; i++) h = (h ^ ((const uint8_t*)p)[i]) * 1099511628211ull;
  return h;
}

static Batch fixture() {
  Batch b;
  b.AddChannel({"Test Channel", "testchannel", "testchannel", 1200, 34, 56789});
  b.AddChannel({"Приватный \"канал\"", "private_chan", "", 0, 0, 0});
  Message m1;
  m1.Id = 5ll << 20;
  m1.ChatId = -1001234567890ll;
  m1.Date = 1700000000;
  m1.ViewCount = 1234;
  m1.ShareCount = 7;
  m1.Text = FormattedText{"Join @durov_channel and t.me/some_channel now\nsecond line <b>", {{5, 14, TextEntity::Mention, ""}}};
  m1.Reactions = {{"\xF0\x9F\x91\x8D", 12}, {"\xE2\x9D\xA4\xEF\xB8\x8F", 3}};
  b.Add(m1);
  Message m2;
  m2.Id = 6ll << 20;
  m2.ChatId = -1001234567890ll;
  m2.Date = 1700000100;
  m2.ContentType = TGI_CT_VIDEO;
  m2.MediaAlbumId = 99;
  m2.Media = "BAACAgIAAxkBAAIB";
  m2.Text = FormattedText{"caption with a link", {{15, 4, TextEntity::TextUrl, "https://t.me/linked_channel/42"}}};
  m2.Comments = std::vector<Comment>{{"first!", std::vector<Reaction>{{"\xF0\x9F\x94\xA5", 2}}, 10, 1, "someone"}, {"no reactions", std::nullopt, 0, 0, "unknown"}};
  b.Add(m2);
  Message m3;
  m3.Id = 7ll << 20;
  m3.ChatId = -1009876543210ll;
  m3.Date = 1600000000;
  m3.ContentType = TGI_CT_POLL;
  m3.Alt = "What do you think?";
  m3.Comments = std::nullopt;
  m3.Channel = 1;
  b.Add(m3);
  Message m4;
  m4.Id = 8ll << 20;
  m4.ChatId = -1009876543210ll;
  m4.Date = 1650000000;
  m4.ContentType = TGI_CT_OTHER;
  m4.Alt = "messageDice";
  m4.Channel = 1;
  m4.Panics = true;
  b.Add(m4);
  return b;
}

int main(int argc, char** argv) {
  Batch b = fixture();
  if (argc > 1 && !strcmp(argv[1], "--pack")) {
    const tgi_tg_batch d = b.Descriptor();
    printf("n %llu\n", (unsigned long long)d.n);
    printf("recs %016llx\n", (unsigned long long)fnv(d.recs, d.n * sizeof(tgi_tg_rec)));
    printf("strs %016llx\n", (unsigned long long)fnv(d.strs, d.strs_len));
    printf("ent_off %016llx\n", (unsigned long long)fnv(d.ent_off, (d.n + 1) * 4));
    printf("ents %016llx\n", (unsigned long long)fnv(d.ents, d.ent_off[d.n] * sizeof(tgi_entity)));
    printf("react_off %016llx\n", (unsigned long long)fnv(d.react_off, (d.n + 1) * 4));
    printf("reacts %016llx\n", (unsigned long long)fnv(d.reacts, d.n_reacts * sizeof(tgi_reaction)));
    printf("comment_off %016llx\n", (unsigned long long)fnv(d.comment_off, (d.n + 1) * 4));
    printf("comments %016llx\n", (unsigned long long)fnv(d.comments, d.n_comments * sizeof(tgi_comment)));
    printf("aux %016llx\n", (unsigned long long)fnv(d.aux, d.aux_len));
    printf("chans %016llx\n", (unsigned long long)fnv(d.chans, d.n_chans * sizeof(tgi_tg_chan)));
    printf("chan_strs %016llx\n", (unsigned long long)fnv(d.chan_strs, d.chan_strs_len));
    return 0;
  }
  try {
    Config cfg;
    cfg.CrawlLabel = "demo \"label\"";
    cfg.TzOffsetSec = 3600;
    MessageProcessor proc(cfg);
    proc.SetClock(1750000000, 0, 1750000001, 500);
    Result r = proc.ProcessMessages(b);
    for (uint64_t i = 0; i < r.Size(); i++) {
      printf("status %d links", r.Status(i));
      for (const std::string& l : r.Outlinks(i)) printf(" %s", l.c_str());
      printf("\n");
      fwrite(r.Line(i).data(), 1, r.Line(i).size(), stdout);
    }
    const bool dapr = argc > 1 && !strcmp(argv[1], "--state-dapr");
    if (argc > 1 && (!strcmp(argv[1], "--state") || dapr)) {  // one seed page with one message, as state.json
      tgi_state_page pg{};
      pg.str_len[TGI_PS_ID] = 2, pg.str_len[TGI_PS_URL] = 11, pg.str_len[TGI_PS_STATUS] = 9;
      pg.ts_off = TGI_STATE_TS_LOCAL, pg.ts_sec = 1750000000, pg.n_msgs = 1;
      proc.StateSet({{0, 1}}, {pg}, "p1testchannelunfetched", {{-1001234567890ll, 5ll << 20, 0, 1, 0}});
      const std::string_view js = proc.StateRender("{}", "\"2025-06-15T15:06:40Z\"");
      fwrite(js.data(), 1, js.size(), stdout);
      printf("\n");
    }
    if (dapr) {
      tgi_state_page a{}, b{};
      a.str_len[TGI_PS_ID] = 2, a.str_len[TGI_PS_URL] = 5;
      b = a;
      b.str_off = 7;
      proc.StateAddPages(-1, {a, b}, "p2url-2p3url-3");
      const std::string_view lm = proc.StateLayerMap();
      fwrite(lm.data(), 1, lm.size(), stdout);
      printf("\n");
      for (std::string_view chunk : proc.StateExport(TGI_STATE_EXPORT_DAPR, 100)) {
        fwrite(chunk.data(), 1, chunk.size(), stdout);
        printf("\n");
      }
    }
  } catch (const std::exception& e) {
    fprintf(stderr, "error: %s\n", e.what());
    return 1;
  }
  return 0;
}
