"""CPU tests (no GPU): pin the oracle against the reference's own known-answer vectors and against an
independent restatement of the Go rules (tests/go_rules.py)."""
import random

import numpy as np
import pytest

import go_rules
from distributed_crawler_b200 import abi
from distributed_crawler_b200.corpus import Corpus
from distributed_crawler_b200.pack import Channel, Comment, pack_telegram
from helpers import ALL, TANDEM, msg, names, vector_message
from oracle import pyoracle


def test_channel_link_vectors(vectors, oracle):
    """telegramhelper/channel_links_test.go (24 tests), compared as sets like sortedEqual (:20-32)."""
    msgs = [vector_message(v) for v in vectors["channel_links"]]
    r = oracle.telegram(pack_telegram(msgs), abi.RUN_LINKS)
    for i, v in enumerate(vectors["channel_links"]):
        assert names(r, i) == sorted(v["expected"]), f'{v["name"]} ({v["go_file"]}:{v["go_line"]})'


def test_dedup_vector_is_exactly_one(vectors, oracle):
    v = next(x for x in vectors["channel_links"] if x["name"] == "Deduplication")
    r = oracle.telegram(pack_telegram([vector_message(v)]), abi.RUN_LINKS)
    assert r.record_links(0) == [(b"samechan", "text_url")]  # first (most structured) source wins


def test_filter_username_vectors(vectors):
    for v in vectors["filter_username"]:
        reason = pyoracle.filter_username(v["username"].encode())
        assert (reason == "") == v["valid"], v["name"]
        if not v["valid"]:
            assert reason == v["reason"], v["name"]


def test_tandem_vector(vectors, oracle):
    """crawl/runner_tandem_test.go:15-93: two mention edges pass FilterUsername + seenInBatch."""
    t = vectors["tandem"]["with_edges"]
    m = msg("messageText", t["text"], [tuple(e) for e in t["entities"]])
    b = pack_telegram([m], [Channel(name=t["owner_url"], username=t["owner_url"])])
    r = oracle.telegram(b, TANDEM)
    edges = [l["name"][: l["len"]].tobytes().decode() for l in r.links if l["flags"] & abi.LF_NEW]
    assert edges == t["expected_edges"]
    assert all(l["flags"] & abi.LF_FILTER_OK for l in r.links)


def test_self_reference_and_filter_flags(oracle):
    m = msg("messageText", "t.me/mychannel t.me/some_bot t.me/goodchan t.me/goodchan")
    b = pack_telegram([m], [Channel(name="mychannel")])
    r = oracle.telegram(b, TANDEM)
    got = {l["name"][: l["len"]].tobytes(): int(l["flags"]) for l in r.links}
    assert got[b"mychannel"] & abi.LF_SELF and not got[b"mychannel"] & abi.LF_NEW
    assert not got[b"some_bot"] & abi.LF_FILTER_OK and not got[b"some_bot"] & abi.LF_NEW
    assert got[b"goodchan"] == abi.LF_FILTER_OK | abi.LF_NEW
    assert r.n_new == 1


@pytest.mark.parametrize("text,off,ln", [
    ("Hello @testchan!", 6, 9), ("Привет @testchan", 7, 9), ("😀 @testchan", 3, 9), ("😀 @testchan", 1, 5),
    ("abc", 5, 2), ("abc", 1, 10), ("abc", 1, 0), ("abc", 2, -1), ("", 0, 0), ("😀😀", 2, 2), ("😀😀", 3, 1),
    ("a\xffb", 1, 1)])
def test_utf16_offsets_vs_independent(text, off, ln):
    b = text.encode("utf-8", "surrogateescape") if "\xff" not in text else b"a\xffb"
    assert pyoracle.utf16_offset_to_bytes(b, off, ln) == go_rules.utf16_offset_to_bytes(b, off, ln)


def _random_bytes(rng, n):
    alphabet = [b"a", b"Z", b" ", b"\"", b"\\", b"<", b">", b"&", b"\n", b"\t", b"\x01", b"\x08", b"\x0c", b"\x1f",
                b"\x7f", "é".encode(), "Я".encode(), "中".encode(), "😀".encode(), " ".encode(),
                " ".encode(), b"\xe2\x80", b"\xe2", b"\x80", b"\xff", b"\xc0\x80", b"\xed\xa0\x80",
                b"\xf0\x9f", b"\xf4\x90\x80\x80", b"\xe0\x9f\x80", b"\xe0\xa0\x80", b"\xf0\x8f\x80\x80"]
    return b"".join(rng.choice(alphabet) for _ in range(n))


def test_json_string_vs_independent():
    rng = random.Random(1234)
    for _ in range(600):
        b = _random_bytes(rng, rng.randrange(0, 60))
        assert pyoracle.json_string(b) == go_rules.go_json_string(b), b


def test_json_time_vs_independent():
    rng = random.Random(7)
    for _ in range(400):
        sec = rng.randrange(-2_000_000_000, 4_000_000_000)
        nsec = rng.choice([0, 1, 120_000_000, 999_999_999, 500, 123_456_789])
        tz = rng.choice([0, 3600, -18000, 19800, 12600])
        assert pyoracle.json_time(sec, nsec, tz) == go_rules.go_time_json(sec, nsec, tz)
    assert pyoracle.json_time(-62135596800) == b'"0001-01-01T00:00:00Z"'  # Go zero time
    assert pyoracle.json_time(253402300800) == b""                         # year 10000 -> Marshal error


def test_iso8601_duration():
    cases = [b"PT1H2M3S", b"P1DT2H", b"PT", b"P", b"P0D", b"PT15M", b"", b"PT1H2M3", b"P1D2H", b"PT1M1H",
             b"PT99999999999999999999S", b"XPT1S", b"PT1S "]
    for c in cases:
        assert pyoracle.parse_iso8601_duration(c) == go_rules.parse_iso8601_duration(c), c


def test_float_of_int64():
    for v, want in [(0, b"0"), (10000, b"10000"), (123456789, b"123456789"), (2 ** 53, b"9007199254740992"),
                    (2 ** 53 + 1, b"9007199254740992"), (12345678901234567890 // 2, b"6172839450617283000"),
                    (-42, b"-42"), (9223372036854775807, b"9223372036854775807")]:
        got = pyoracle.json_float_of_int64(v)
        assert float(got) == float(v)
        # shortest round-trip: repr(float) has the same significant digits
        assert got.rstrip(b"0") .lstrip(b"-") == repr(float(v)).replace(".", "").split("e")[0].rstrip("0").lstrip("-").encode() \
            or got == want


def test_links_vs_independent_on_corpus(oracle):
    c = Corpus(3000, profile=3, nthreads=2)
    b = c.batch
    r = oracle.telegram(b, abi.RUN_LINKS)
    src_names = {"text_url": "text_url", "mention": "mention", "url": "url"}
    strs, aux = b.strs.tobytes(), b.aux.tobytes()
    for i in range(b.n):
        rec = b.recs[i]
        so = int(rec["str_off"])
        text = strs[so:so + int(rec["text_len"])] if rec["flags"] & abi.RF_HAS_TEXT else None
        ents = []
        for e in b.ents[int(b.ent_off[i]):int(b.ent_off[i + 1])]:
            typ = {1: "text_url", 2: "mention", 3: "url"}.get(int(e["type"]), "other")
            ents.append((int(e["offset"]), int(e["length"]), typ, aux[int(e["url_off"]):int(e["url_off"]) + int(e["url_len"])]))
        want = go_rules.extract_links(text, ents)
        if rec["flags"] & abi.RF_PANIC:
            continue
        if want is None:
            assert r.status[i] == abi.ST_FAILED, i
        else:
            assert r.record_links(i) == want, i


def test_post_line_is_json_and_roundtrips(oracle):
    import json
    m = [msg("messageText", "hello <b> & \"q\" \\   t.me/abcdef", reactions=[("👍", 3), ("❤", 2), ("👍", 9)],
             comments=[Comment("c1", [("🔥", 1)], 5, 0, "bob"), Comment("c2", None, 0, 1, "al")], id=77 << 20,
             view_count=12, share_count=3, handle="Chan"),
         msg("messageVideo", "cap", media="REMOTEID", media_album_id=5),
         msg("messageDocument", "t.me/docchan", alt="file.pdf", media="DOCID"),
         msg("messageLocation"), msg("none"), msg("messagePoll", alt="why?"), msg("messageText", None, comments=None)]
    r = oracle.telegram(pack_telegram(m, [Channel("T<itle>", "nm", "usr", 10, 20, 30)]))
    d = [json.loads(r.line(i)) for i in range(len(m))]
    assert list(d[0].keys())[:5] == ["post_link", "channel_id", "post_uid", "url", "published_at"]
    assert len(d[0]) == 65
    assert d[0]["post_link"] == "https://t.me/usr/77" and d[0]["post_uid"] == "77-nm"
    assert d[0]["reactions"] == {"❤": 2, "👍": 9} and list(d[0]["reactions"]) == ["❤", "👍"]
    assert d[0]["comments"][1]["reactions"] is None and d[0]["comment_count"] == 2
    assert d[0]["outlinks"] == ["abcdef"] and d[0]["channel_name"] == "T<itle>"
    assert d[0]["channel_data"]["channel_url"] == "https://t.me/c/nm"
    assert d[1]["post_link"].endswith("?single") and d[1]["media_url"] == "REMOTEID" and d[1]["description"] == "cap"
    assert d[2]["description"] == "file.pdf" and d[2]["outlinks"] == ["docchan"] and d[2]["post_type"] == ["messageDocument"]
    assert d[3]["post_type"] == ["messageLocation"] and d[4]["post_type"] == ["unknown"]
    assert d[5]["description"] == "why?" and d[5]["outlinks"] == []
    assert d[6]["comments"] is None and d[6]["description"] == ""
    assert b"\\u003cb\\u003e \\u0026" in r.line(0) and b"\\u2028" in r.line(0)


def test_status_semantics():
    o = pyoracle.Oracle(min_post_date=1_700_000_000)
    m = [msg(date=1_600_000_000, text="t.me/skipped1"), msg(date=1_800_000_000, text="t.me/kept12"),
         msg(text="x", panics=True, date=1_800_000_000),
         msg("messageText", "😀 @testchan", [(1, 5, "mention", "")], date=1_800_000_000)]
    r = o.telegram(pack_telegram(m))
    assert list(r.status) == [abi.ST_SKIPPED, abi.ST_EMITTED, abi.ST_FAILED, abi.ST_FAILED]
    assert [len(r.line(i)) > 0 for i in range(4)] == [False, True, False, False]
    assert r.record_links(0) == [] and r.record_links(1) == [(b"kept12", "plaintext")]


def test_corpus_deterministic_and_shardable():
    a = Corpus(5000, nthreads=1).batch
    b = Corpus(5000, nthreads=4).batch
    for k in a.FIELDS:
        assert np.array_equal(getattr(a, k), getattr(b, k)), k
    sh = Corpus(700, first=1300, nthreads=2).batch
    sl = a.slice(1300, 2000)
    assert np.array_equal(sh.strs, sl.strs)
    for f in sh.recs.dtype.names:
        if f != "chan_idx":  # slice() rebases the channel table, a shard keeps the global one
            assert np.array_equal(sh.recs[f], sl.recs[f]), f
    for f in ("offset", "length", "type", "url_len"):
        assert np.array_equal(sh.ents[f], sl.ents[f]), f
    # same shard -> same oracle output (aux offsets differ, contents do not)
    r1, r2 = pyoracle.Oracle().telegram(sh, ALL), pyoracle.Oracle().telegram(sl, ALL)
    assert np.array_equal(r1.jsonl, r2.jsonl) and np.array_equal(r1.links, r2.links)


def test_youtube_slice_is_a_self_contained_page():
    """YtBatch.slice (bench.py's page-sized calls, tests/test_gpu_page.py): the lines / links of records [a,b) of the whole."""
    from distributed_crawler_b200.corpus import YtCorpus
    from yt_corpus import make_youtube
    F = abi.RUN_JSONL | abi.RUN_LINKS
    for b in (YtCorpus(3000, seed=7, nthreads=2).batch, make_youtube(1500, seed=5)[0]):
        full = pyoracle.Oracle().youtube(b, F)
        for a, e in ((0, 50), (1000, 1050), (b.n - 50, b.n), (17, 18)):
            part = pyoracle.Oracle().youtube(b.slice(a, e), F)
            assert np.array_equal(part.jsonl, full.jsonl[int(full.line_off[a]):int(full.line_off[e])])
            assert np.array_equal(part.status, full.status[a:e])
            assert np.array_equal(part.links, full.links[int(full.link_off[a]):int(full.link_off[e])])


def _random_messages(rnd, n):
    """messages over every content type and every awkward shape the Go code distinguishes"""
    from distributed_crawler_b200.pack import TextEntity, FormattedText, Message
    pieces = [b"hello ", b"t.me/", b"https://t.me/", b"@", b"chan_name1 ", b"SomeChannel ", b"joinchat/x ", b"abcd ", b"\n", b"\t",
              b'"q"', b"\\", b"<b>&", "привет ".encode(), "😀".encode(), "مرحبا ".encode(), b"\xe2\x80\xa8", b"\xe2\x80\xa9",
              b"\xff", b"\xc0\xaf", b"\xed\xa0\x80", b"\xf0\x9f", b"\x01", b"\x7f", b"x" * 40, b"some_bot ", b"a_b_c_d_e "]
    emojis = ["👍", "❤", "🔥", "a", "zz", b"\xff", '"', "k<"]

    def text(maxp):
        return b"".join(rnd.choice(pieces) for _ in range(rnd.randrange(0, maxp)))

    def reacts():
        return [(rnd.choice(emojis), rnd.randrange(-3, 10 ** rnd.randrange(1, 10))) for _ in range(rnd.randrange(0, 6))]

    types = abi.CT_NAMES[:-1] + ["messageLocation", "messageContact"]
    out = []
    for _ in range(n):
        ct = rnd.choice(types)
        t = None if rnd.random() < 0.15 else text(12)
        ents = []
        if t is not None:
            for _ in range(rnd.randrange(0, 4)):
                ents.append(TextEntity(rnd.randrange(-2, 40), rnd.randrange(-2, 30), rnd.choice(["mention", "url", "text_url", "bold"]),
                                       rnd.choice([b"https://t.me/linked_chan", b"http://example.com", b"t.me/x", b""])))
        comments = rnd.choice([None, [], [Comment(text(4), rnd.choice([None, [], reacts()]), rnd.randrange(0, 99), rnd.randrange(0, 9),
                                                  rnd.choice(["bob", b"\xfe", "unknown", ""])) for _ in range(rnd.randrange(1, 4))]])
        out.append(Message(content_type=ct, text=None if t is None else FormattedText(t, ents), alt=text(3), media=rnd.choice([b"", b"REMOTE-id_1", text(2)]),
                           id=rnd.choice([1 << 20, 77 << 20, (5 << 20) + 123, -(3 << 20) - 7, rnd.randrange(0, 1 << 50)]),
                           chat_id=rnd.choice([-1001234567890, 5, -7]), date=rnd.choice([0, 1_600_000_000, 1_700_000_000, 1_800_000_000, 2 ** 31 - 1]),
                           media_album_id=rnd.choice([0, 0, 9]), view_count=rnd.randrange(0, 10 ** rnd.randrange(1, 10)),
                           share_count=rnd.randrange(0, 1000), reactions=reacts(), comments=comments, handle=rnd.choice(["Chan", "", b"\xe9", 'h"x']),
                           channel=rnd.randrange(0, 3), panics=rnd.random() < 0.03, video_shape=rnd.choice(["ok", "ok", "none", "broken"])))
    return out


def test_whole_post_line_vs_independent_restatement():
    """Every byte of the Telegram Post line against tests/go_rules.py:telegram_post_line — a second restatement of
    ParseMessage + json.Marshal written from the Go sources over the host-side message model, not from the oracle."""
    import random
    chans = [Channel("T<itle> \u2028", "nm", "usr", 10, 20, 30), Channel(b"\xff\"t", "name_2", "", 0, 0, 0), Channel("", "", "u3", 2 ** 31 - 1, 7, 2 ** 40)]
    for trial, cfg in enumerate([dict(), dict(tz_offset_sec=19800, crawl_label=b'lab"<el>\xff', capture_nsec=0, created_at_sec=1_760_000_000),
                                 dict(tz_offset_sec=-12600, min_post_date=1_650_000_000, created_at_nsec=999, capture_nsec=120_000_000)]):
        rnd = random.Random(100 + trial)
        ms = _random_messages(rnd, 800)
        r = pyoracle.Oracle(**cfg).telegram(pack_telegram(ms, chans), abi.RUN_JSONL | abi.RUN_LINKS)
        kw = dict(crawl_label=cfg.get("crawl_label", b""), created=(cfg.get("created_at_sec", 1_750_000_000), cfg.get("created_at_nsec", 0)),
                  capture=(1_750_000_000, cfg.get("capture_nsec", 123_456_789)), tz=cfg.get("tz_offset_sec", 0),
                  min_post_date=cfg.get("min_post_date"))
        want_status = {"emitted": abi.ST_EMITTED, "skipped": abi.ST_SKIPPED, "failed": abi.ST_FAILED}
        for i, m in enumerate(ms):
            st, line, links = go_rules.telegram_post_line(m, chans[m.channel], **kw)
            assert r.status[i] == want_status[st], (trial, i, st, m)
            assert r.line(i) == (line or b""), (trial, i, m)
            assert [n for n, _ in r.record_links(i)] == [go_rules._bs(x) for x in links], (trial, i)


def test_whole_youtube_line_vs_independent_restatement():
    """Every byte of the YouTube Post line (and the snowball ids) against tests/go_rules.py:youtube_post_line — a second
    restatement of convertVideoToPost + json.Marshal written from the Go sources, not from the oracle."""
    from yt_corpus import make_youtube, make_youtube_config4
    for mk, n, seed, cfg in ((make_youtube, 1200, 3, dict()), (make_youtube_config4, 500, 5, dict()),
                             (make_youtube, 600, 9, dict(tz_offset_sec=19800, crawl_label=b'yt"<lbl>', created_at_nsec=987_000_000, capture_nsec=0))):
        b, vids, chans = mk(n, seed=seed)
        r = pyoracle.Oracle(**cfg).youtube(b, abi.RUN_JSONL | abi.RUN_LINKS)
        kw = dict(crawl_label=cfg.get("crawl_label", b""), created=(1_750_000_000, cfg.get("created_at_nsec", 0)),
                  capture=(1_750_000_000, cfg.get("capture_nsec", 123_456_789)), tz=cfg.get("tz_offset_sec", 0))
        nolines = 0
        for i, v in enumerate(vids):
            line, _, ids = go_rules.youtube_post_line(v, chans[v.channel], **kw)
            assert r.line(i) == (line or b""), (mk.__name__, i)
            assert r.status[i] == (abi.ST_EMITTED if line else abi.ST_NOLINE)
            assert [x for x, _ in r.record_links(i)] == [x[:32] for x in ids], (mk.__name__, i)  # link rows keep 32 bytes of an id
            nolines += line is None
        assert nolines > 0 or mk is make_youtube_config4  # the adversarial corpus holds unrepresentable dates


def test_oracle_threads_agree():
    c = Corpus(20000, nthreads=2)
    r1 = pyoracle.Oracle().telegram(c.batch, ALL, nthreads=1)
    r4 = pyoracle.Oracle().telegram(c.batch, ALL, nthreads=4)
    assert np.array_equal(r1.jsonl, r4.jsonl) and np.array_equal(r1.links, r4.links) and r1.n_new == r4.n_new


def test_frontier_first_occurrence_order():
    o = pyoracle.Oracle()
    from distributed_crawler_b200.engine import names_to_keys32
    k = names_to_keys32([b"bbbbb", b"aaaaa", b"bbbbb", b"ccccc", b"aaaaa"])
    assert list(o.frontier_insert(k)) == [1, 1, 0, 1, 0]
    assert [bytes(x).rstrip(b"\0") for x in o.frontier_export()] == [b"bbbbb", b"aaaaa", b"ccccc"]
    assert list(o.frontier_insert(names_to_keys32([b"ccccc", b"ddddd"]))) == [0, 1]


def test_oracle_generic_message_sparse_post():
    """SURVEY a12: the sparse Post of convertMessageToPost (crawler/telegram/telegram_crawler.go:179-262),
    cross-checked against an independent restatement built from the Go rules in go_rules.py."""
    import json

    from distributed_crawler_b200.pack import GenericMessage, pack_generic
    from gm_corpus import make_generic
    import go_rules

    batch, msgs = make_generic(300, seed=9)
    tz, cs, cn, ps, pn = 7200, 1_750_000_000, 5_000, 1_750_000_123, 0
    o = pyoracle.Oracle(tz_offset_sec=tz, created_at_sec=cs, created_at_nsec=cn, capture_sec=ps, capture_nsec=pn)
    r = o.generic(batch)
    zero_keys_null = ["list_ids", "search_terms", "search_term_ids", "project_ids", "exercise_ids", "label_data",
                      "labels_metadata", "project_labeled_post_ids", "labeler_ids", "all_labels", "label_ids", "video_length",
                      "is_verified", "shared_id", "quoted_id", "replied_id", "ai_label", "root_post_id", "ocr_data",
                      "has_embed_media", "repost_channel_data", "post_type", "post_title", "is_reply", "ad_fields",
                      "contrast_agent_project_ids", "agent_ids", "segment_ids", "comments", "outlinks"]
    for i, m in enumerate(msgs):
        line = r.line(i)
        assert line == go_rules.generic_post_line(m, created=(cs, cn), capture=(ps, pn), tz=tz), i  # the whole line
        assert line.endswith(b"}\n")
        js = lambda b: go_rules.go_json_string(b if isinstance(b, bytes) else b.encode())
        # the variable parts, byte for byte
        assert line.startswith(b'{"post_link":"","channel_id":' + js(m.channel_id) + b',"post_uid":' + js(m.id) +
                               b',"url":"","published_at":' + go_rules.go_time_json(m.ts_sec, m.ts_nsec, tz) +
                               b',"created_at":' + go_rules.go_time_json(cs, cn, tz) + b',"language_code":"","engagement":0,"view_count":' +
                               str(m.views).encode() + b',')
        assert b',"description":' + js(m.text) + b',"repost_channel_data":null' in line
        assert b',"searchable_text":' + js(m.text) + b',"all_text":' + js(m.text) + b',"contrast_agent_project_ids"' in line
        assert line.endswith(b',"outlinks":null,"capture_time":' + go_rules.go_time_json(ps, pn, tz) + b',"handle":' + js(m.sender_name) + b"}\n")
        if not m.reactions:
            assert b',"reactions":null,' in line
        else:
            d = {}
            for k, v in m.reactions:
                d[k.encode() if isinstance(k, str) else k] = v
            want = b"{" + b",".join(go_rules.go_json_string(k) + b":" + str(d[k]).encode() for k in sorted(d)) + b"}"
            assert b',"reactions":' + want + b',"outlinks"' in line
        # the shape: 65 keys in declaration order, zero values elsewhere (invalid UTF-8 is � by then: valid JSON)
        doc = json.loads(line.decode("utf-8"))
        assert len(doc) == 65 and list(doc)[:4] == ["post_link", "channel_id", "post_uid", "url"] and list(doc)[-1] == "handle"
        assert all(doc[k] is None for k in zero_keys_null)
        assert doc["platform_name"] == "telegram" and doc["channel_name"] == doc["channel_id"] and doc["views_count"] == m.views
        assert doc["channel_data"]["published_at"] == "0001-01-01T00:00:00Z" and doc["inner_link"] == {}
        assert doc["performance_scores"] == {"likes": None, "shares": None, "comments": None, "views": 0}


def test_message_video_shapes(oracle):
    """processMessageSafely (tdutils.go:188-199): no thumbnail -> its error comes before any read, media_url stays "" and
    the description is still the caption; a thumbnail with a nil file / caption -> nil dereference, recovered, "failed"."""
    import json
    from distributed_crawler_b200.pack import FormattedText, Message, pack_telegram
    ms = [Message(content_type="messageVideo", text=FormattedText("cap t.me/fromcaption"), media="VIDEOID", video_shape="ok"),
          Message(content_type="messageVideo", text=FormattedText("cap t.me/fromcaption"), media="VIDEOID", video_shape="none"),
          Message(content_type="messageVideo", text=None, media="VIDEOID", video_shape="broken")]
    r = oracle.telegram(pack_telegram(ms), abi.RUN_JSONL | abi.RUN_LINKS)
    assert list(r.status) == [abi.ST_EMITTED, abi.ST_EMITTED, abi.ST_FAILED]
    a, b = json.loads(r.line(0)), json.loads(r.line(1))
    assert a["media_url"] == "VIDEOID" and b["media_url"] == "" and a["description"] == b["description"] == "cap t.me/fromcaption"
    assert r.line(2) == b"" and [n for n, _ in r.record_links(1)] == [b"fromcaption"]
