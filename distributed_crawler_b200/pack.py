"""Host-side message model + batch packer.

Mirrors the shapes the reference hot path consumes (go-tdlib `client.Message` /
`client.FormattedText` / `client.TextEntity`, SURVEY Appendix B; `youtubemodel.YouTubeVideo`,
model/youtube/types.go:23-36) and lowers them to the packed columnar batch of include/tgingest.h.
This is what the Go shim's packer does (INTEGRATION.md); here it exists so that tests can be
written like the reference's own tests (telegramhelper/channel_links_test.go).
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from . import abi


def _b(s) -> bytes:
    if s is None:
        return b""
    return s if isinstance(s, (bytes, bytearray)) else str(s).encode("utf-8")


@dataclass
class TextEntity:  # client.TextEntity
    offset: int
    length: int
    type: str = "other"  # "mention" | "url" | "text_url" | anything else
    url: str | bytes = ""


@dataclass
class FormattedText:  # client.FormattedText
    text: str | bytes = ""
    entities: list[TextEntity] = field(default_factory=list)


@dataclass
class Comment:  # model.Comment as GetMessageComments builds it (telegramutils.go:589-635)
    text: str | bytes = ""
    reactions: list[tuple[str | bytes, int]] | None = None
    view_count: int = 0
    reply_count: int = 0
    handle: str | bytes = "unknown"


@dataclass
class Message:  # client.Message + pre-resolved RPC results
    content_type: str = "messageText"  # MessageContentType(); "none" = nil content
    text: FormattedText | None = None  # Text / Caption
    alt: str | bytes = ""              # emoji / poll question / prize type / file name / type name
    media: str | bytes = ""            # remote id that becomes media_url
    id: int = 1 << 20
    chat_id: int = -1001234567890
    date: int = 1_700_000_000
    media_album_id: int = 0
    view_count: int = 0
    share_count: int = 0
    reactions: list[tuple[str | bytes, int]] = field(default_factory=list)
    comments: list[Comment] | None = field(default_factory=list)  # None = nil slice
    handle: str | bytes = "unknown"
    channel: int = 0
    panics: bool = False
    # messageVideo only — the shape processMessageSafely (tdutils.go:188-199) looks at.  "ok": Video, Thumbnail, the
    # two files and the caption are all there (media_url = the video's remote id); "none": no Video / no Thumbnail —
    # the function returns its error before reading anything, media_url stays ""; "broken": a thumbnail is present
    # but Thumbnail.File / File.Remote / Video.Video / Video.Video.Remote / Caption is nil — nil dereference, recovered
    # (:395-405), the message is marked "failed"
    video_shape: str = "ok"


@dataclass
class Channel:
    title: str | bytes = "Test Channel"
    name: str | bytes = "testchannel"       # channelName argument (page URL)
    username: str | bytes = "testchannel"   # ActiveUsernames[0]; "" = private
    member_count: int = 0
    post_count: int = 0
    view_count: int = 0


class TgBatch:
    """Owns the numpy arrays of one packed Telegram batch and builds the C descriptor."""

    FIELDS = ("recs", "strs", "ent_off", "ents", "react_off", "reacts", "comment_off", "comments",
              "aux", "chans", "chan_strs")

    def __init__(self, **arrays):
        for k in self.FIELDS:
            setattr(self, k, arrays[k])
        self.n = len(self.recs)

    def descriptor(self) -> abi.TgBatchC:
        d = abi.TgBatchC()
        d.n = self.n
        d.recs = abi.ptr(self.recs)
        d.strs = abi.ptr(self.strs)
        d.strs_len = self.strs.size
        d.ent_off = abi.ptr(self.ent_off)
        d.ents = abi.ptr(self.ents)
        d.react_off = abi.ptr(self.react_off)
        d.reacts = abi.ptr(self.reacts)
        d.n_reacts = len(self.reacts)
        d.comment_off = abi.ptr(self.comment_off)
        d.comments = abi.ptr(self.comments)
        d.n_comments = len(self.comments)
        d.aux = abi.ptr(self.aux)
        d.aux_len = self.aux.size
        d.n_chans = len(self.chans)
        d.chans = abi.ptr(self.chans)
        d.chan_strs = abi.ptr(self.chan_strs)
        d.chan_strs_len = self.chan_strs.size
        return d

    def input_bytes(self) -> int:
        """algorithmic input bytes (DESIGN.md): every input array read once."""
        return sum(getattr(self, k).nbytes for k in self.FIELDS)

    def slice(self, a: int, b: int) -> "TgBatch":
        """records [a,b) as a self-contained batch (every offset rebased; only referenced rows of the
        side arrays are kept) — what a caller packing that range on its own would have produced."""
        recs = self.recs[a:b].copy()
        s0 = int(self.recs["str_off"][a]) if a < self.n else self.strs.size
        s1 = int(self.recs["str_off"][b]) if b < self.n else self.strs.size
        recs["str_off"] -= s0
        e0, e1 = int(self.ent_off[a]), int(self.ent_off[b])
        r0, r1 = int(self.react_off[a]), int(self.react_off[b])
        c0, c1 = int(self.comment_off[a]), int(self.comment_off[b])
        ents = self.ents[e0:e1].copy()
        comments = self.comments[c0:c1].copy()
        # comment reactions sit behind the message reactions: gather the referenced range
        has = (comments["flags"] & 1).astype(bool) & (comments["react_count"] > 0)
        if has.any():
            cr0 = int(comments["react_start"][has].min())
            cr1 = int((comments["react_start"][has] + comments["react_count"][has]).max())
        else:
            cr0 = cr1 = 0
        reacts = np.concatenate([self.reacts[r0:r1], self.reacts[cr0:cr1]]) if (r1 > r0 or cr1 > cr0) else self.reacts[:0].copy()
        comments["react_start"] = np.where(has, comments["react_start"] - cr0 + (r1 - r0), 0)
        # aux: smallest window covering everything referenced
        los, his = [], []
        tu = ents["type"] == abi.ENT_TEXT_URL
        if tu.any():
            los.append(int(ents["url_off"][tu].min())); his.append(int((ents["url_off"][tu] + ents["url_len"][tu]).max()))
        if len(reacts):
            los.append(int(reacts["emoji_off"].min())); his.append(int((reacts["emoji_off"] + reacts["emoji_len"]).max()))
        if len(comments):
            los.append(int(min(comments["text_off"].min(), comments["handle_off"].min())))
            his.append(int(max((comments["text_off"] + comments["text_len"]).max(),
                               (comments["handle_off"] + comments["handle_len"]).max())))
        alo, ahi = (min(los), max(his)) if los else (0, 0)
        ents["url_off"] = np.where(tu, ents["url_off"] - alo, 0)
        reacts = reacts.copy()
        reacts["emoji_off"] -= alo
        comments["text_off"] -= alo
        comments["handle_off"] -= alo
        # channel rows actually referenced
        if len(recs):
            cmin, cmax = int(recs["chan_idx"].min()), int(recs["chan_idx"].max())
        else:
            cmin, cmax = 0, -1
        chans = self.chans[cmin:cmax + 1].copy()
        recs["chan_idx"] -= cmin
        if len(chans):
            clo = int(chans["str_off"].min())
            ln = chans["title_len"].astype(np.int64) + chans["name_len"] + chans["user_len"]
            chi = int((chans["str_off"] + ln).max())
            chans["str_off"] -= clo
        else:
            clo = chi = 0
        return TgBatch(recs=recs, strs=_pad(self.strs[s0:s1]),
                       ent_off=(self.ent_off[a:b + 1] - e0).astype(np.uint32), ents=ents,
                       react_off=(self.react_off[a:b + 1] - r0).astype(np.uint32), reacts=reacts,
                       comment_off=(self.comment_off[a:b + 1] - c0).astype(np.uint32),
                       comments=comments, aux=_pad(self.aux[alo:ahi]), chans=chans,
                       chan_strs=_pad(self.chan_strs[clo:chi]))


def _pad(a: np.ndarray) -> np.ndarray:
    """copy of a uint8 array with 16 readable pad bytes behind it"""
    full = np.zeros(a.size + 16, np.uint8)
    full[: a.size] = a
    return full[: a.size]


_ENT_TYPES = {"text_url": abi.ENT_TEXT_URL, "mention": abi.ENT_MENTION, "url": abi.ENT_URL}


def pack_telegram(messages: list[Message], channels: list[Channel] | None = None) -> TgBatch:
    channels = channels or [Channel()]
    n = len(messages)
    recs = np.zeros(n, abi.TG_REC)
    strs = bytearray()
    aux = bytearray()
    ents, reacts, comments = [], [], []
    ent_off = np.zeros(n + 1, np.uint32)
    react_off = np.zeros(n + 1, np.uint32)
    comment_off = np.zeros(n + 1, np.uint32)
    comment_reacts: list[tuple[int, list]] = []  # (comment index, reactions)
    for i, m in enumerate(messages):
        r = recs[i]
        ct = abi.CT.get(m.content_type, abi.CT["other"])
        alt = _b(m.alt)
        if ct == abi.CT["other"] and not alt:
            alt = _b(m.content_type)
        text = _b(m.text.text) if m.text is not None else b""
        media, handle = _b(m.media), _b(m.handle)
        if m.content_type == "messageVideo" and m.video_shape != "ok":
            media = b""
        flags = 0
        if m.text is not None:
            flags |= abi.RF_HAS_TEXT
        if m.comments is None:
            flags |= abi.RF_COMMENTS_NIL
        if m.panics or (m.content_type == "messageVideo" and m.video_shape == "broken"):
            flags |= abi.RF_PANIC
        r["id"], r["chat_id"], r["media_album_id"] = m.id, m.chat_id, m.media_album_id
        r["str_off"] = len(strs)
        r["date"], r["view_count"], r["share_count"] = m.date, m.view_count, m.share_count
        r["chan_idx"] = m.channel
        r["text_len"], r["alt_len"] = len(text), len(alt)
        r["media_len"], r["handle_len"] = len(media), len(handle)
        r["content_type"], r["flags"] = ct, flags
        strs += text + alt + media + handle
        if m.text is not None:
            for e in m.text.entities:
                url = _b(e.url)
                ents.append((e.offset, e.length, len(aux), len(url), _ENT_TYPES.get(e.type, 0), 0))
                aux += url
        ent_off[i + 1] = len(ents)
        for emoji, cnt in m.reactions:
            eb = _b(emoji)
            reacts.append((len(aux), len(eb), 0, cnt))
            aux += eb
        react_off[i + 1] = len(reacts)
        for c in (m.comments or []):
            tb, hb = _b(c.text), _b(c.handle)
            comments.append([len(aux), len(tb), len(aux) + len(tb), len(hb),
                             1 if c.reactions is not None else 0, 0, c.view_count, c.reply_count,
                             0, 0])
            aux += tb + hb
            comment_reacts.append((len(comments) - 1, c.reactions or []))
        comment_off[i + 1] = len(comments)
    for ci, rl in comment_reacts:  # comment reactions go after all message reactions
        comments[ci][8] = len(reacts)
        comments[ci][9] = len(rl)
        for emoji, cnt in rl:
            eb = _b(emoji)
            reacts.append((len(aux), len(eb), 0, cnt))
            aux += eb
    chans = np.zeros(len(channels), abi.TG_CHAN)
    cstrs = bytearray()
    for i, ch in enumerate(channels):
        t, nm, u = _b(ch.title), _b(ch.name), _b(ch.username)
        chans[i] = (len(cstrs), len(t), len(nm), len(u), 0, 0, ch.member_count, ch.post_count,
                    ch.view_count)
        cstrs += t + nm + u

    def arr(lst, dt):
        a = np.zeros(len(lst), dt)
        for k, row in enumerate(lst):
            a[k] = tuple(row)
        return a

    return TgBatch(recs=recs, strs=_blob(strs), ent_off=ent_off, ents=arr(ents, abi.ENTITY),
                   react_off=react_off, reacts=arr(reacts, abi.REACTION), comment_off=comment_off,
                   comments=arr(comments, abi.COMMENT), aux=_blob(aux), chans=chans,
                   chan_strs=_blob(cstrs))


def _blob(b: bytearray | bytes) -> np.ndarray:
    """uint8 array view with 16 readable pad bytes behind it (kernels may over-read <= 15 bytes)."""
    full = np.frombuffer(bytes(b) + b"\0" * 16, np.uint8).copy()
    return full[: len(b)]


# ---- YouTube ----------------------------------------------------------------------------------
@dataclass
class YouTubeChannel:  # youtubemodel.YouTubeChannel; cached=False -> GetChannelInfo failed
    id: str | bytes = "UCxxxxxxxxxxxxxxxxxxxxxx"
    title: str | bytes = ""
    description: str | bytes = ""
    thumb_default: str | bytes = ""
    country: str | bytes = ""
    subscriber_count: int = 0
    view_count: int = 0
    video_count: int = 0
    published_sec: int = 0
    published_nsec: int = 0
    cached: bool = True


@dataclass
class YouTubeVideo:  # youtubemodel.YouTubeVideo
    id: str | bytes = "dQw4w9WgXcQ"
    title: str | bytes = ""
    description: str | bytes = ""
    published_sec: int = 1_600_000_000
    published_nsec: int = 0
    view_count: int = 0
    like_count: int = 0
    comment_count: int = 0
    duration: str | bytes = ""
    thumbnails: dict[str, str | bytes] = field(default_factory=dict)
    language: str | bytes = ""
    channel: int = 0


class YtBatch:
    FIELDS = ("recs", "strs", "chans", "chan_strs")

    def __init__(self, **arrays):
        for k in self.FIELDS:
            setattr(self, k, arrays[k])
        self.n = len(self.recs)

    def descriptor(self) -> abi.YtBatchC:
        d = abi.YtBatchC()
        d.n = self.n
        d.recs = abi.ptr(self.recs)
        d.strs = abi.ptr(self.strs)
        d.strs_len = self.strs.size
        d.n_chans = len(self.chans)
        d.chans = abi.ptr(self.chans)
        d.chan_strs = abi.ptr(self.chan_strs)
        d.chan_strs_len = self.chan_strs.size
        return d

    def input_bytes(self) -> int:
        return sum(getattr(self, k).nbytes for k in self.FIELDS)

    def slice(self, a: int, b: int) -> "YtBatch":
        """records [a,b) as a self-contained batch (string offsets rebased, only the referenced channel rows kept): what a
        caller packing one page of the Data API on its own would have produced."""
        recs = self.recs[a:b].copy()
        s0 = int(self.recs["str_off"][a]) if a < self.n else self.strs.size
        s1 = int(self.recs["str_off"][b]) if b < self.n else self.strs.size
        recs["str_off"] -= s0
        if len(recs):
            cmin, cmax = int(recs["chan_idx"].min()), int(recs["chan_idx"].max())
        else:
            cmin, cmax = 0, -1
        chans = self.chans[cmin:cmax + 1].copy()
        recs["chan_idx"] -= cmin
        if len(chans):
            clo = int(chans["str_off"].min())
            ln = sum(chans[k].astype(np.int64) for k in ("id_len", "title_len", "desc_len", "thumb_len", "country_len"))
            chi = int((chans["str_off"] + ln).max())
            chans["str_off"] -= clo
        else:
            clo = chi = 0
        return YtBatch(recs=recs, strs=_pad(self.strs[s0:s1]), chans=chans, chan_strs=_pad(self.chan_strs[clo:chi]))


def pack_youtube(videos: list[YouTubeVideo], channels: list[YouTubeChannel] | None = None) -> YtBatch:
    channels = channels or [YouTubeChannel()]
    recs = np.zeros(len(videos), abi.YT_REC)
    strs = bytearray()
    for i, v in enumerate(videos):
        r = recs[i]
        parts = [_b(v.id), _b(v.title), _b(v.description), _b(v.duration), _b(v.language)]
        r["str_off"] = len(strs)
        r["published_sec"], r["published_nsec"] = v.published_sec, v.published_nsec
        r["view_count"], r["like_count"], r["comment_count"] = v.view_count, v.like_count, v.comment_count
        r["id_len"], r["title_len"], r["desc_len"] = len(parts[0]), len(parts[1]), len(parts[2])
        r["duration_len"], r["lang_len"] = len(parts[3]), len(parts[4])
        r["chan_idx"] = v.channel
        for k, key in enumerate(abi.YT_THUMB_KEYS):
            if key in v.thumbnails:
                tb = _b(v.thumbnails[key])
                r["thumb_len"][k] = len(tb)
                parts.append(tb)
            else:
                r["thumb_len"][k] = abi.YT_THUMB_ABSENT
        strs += b"".join(parts)
    chans = np.zeros(len(channels), abi.YT_CHAN)
    cstrs = bytearray()
    for i, ch in enumerate(channels):
        parts = [_b(ch.id), _b(ch.title), _b(ch.description), _b(ch.thumb_default), _b(ch.country)]
        c = chans[i]
        c["str_off"] = len(cstrs)
        c["id_len"], c["title_len"], c["desc_len"] = len(parts[0]), len(parts[1]), len(parts[2])
        c["thumb_len"], c["country_len"] = len(parts[3]), len(parts[4])
        c["subscriber_count"], c["view_count"], c["video_count"] = (
            ch.subscriber_count, ch.view_count, ch.video_count)
        c["published_sec"], c["published_nsec"], c["cached"] = (
            ch.published_sec, ch.published_nsec, 1 if ch.cached else 0)
        cstrs += b"".join(parts)
    return YtBatch(recs=recs, strs=_blob(strs), chans=chans, chan_strs=_blob(cstrs))


# ---- generic client.Message (SURVEY a12) -----------------------------------------------------------
@dataclass
class GenericMessage:  # client.TelegramMessage as getMessagesWithClient fills it (client/clients.go:325-334)
    id: str | bytes = ""
    channel_id: str | bytes = ""
    text: str | bytes = ""
    sender_name: str | bytes = ""
    ts_sec: int = 0
    ts_nsec: int = 0
    views: int = 0
    reactions: list[tuple[str | bytes, int]] = field(default_factory=list)  # map entries (later duplicates overwrite)


class GmBatch:
    FIELDS = ("recs", "strs", "react_off", "reacts", "aux")

    def __init__(self, **arrays):
        for k in self.FIELDS:
            setattr(self, k, arrays[k])
        self.n = len(self.recs)

    def descriptor(self) -> abi.GmBatchC:
        d = abi.GmBatchC()
        d.n = self.n
        d.recs = abi.ptr(self.recs)
        d.strs = abi.ptr(self.strs)
        d.strs_len = self.strs.size
        d.react_off = abi.ptr(self.react_off)
        d.reacts = abi.ptr(self.reacts)
        d.n_reacts = len(self.reacts)
        d.aux = abi.ptr(self.aux)
        d.aux_len = self.aux.size
        return d


def pack_generic(msgs: list[GenericMessage]) -> GmBatch:
    recs = np.zeros(len(msgs), abi.GM_REC)
    react_off = np.zeros(len(msgs) + 1, np.uint32)
    reacts = []
    strs, aux = bytearray(), bytearray()
    for i, m in enumerate(msgs):
        parts = [_b(m.id), _b(m.channel_id), _b(m.text), _b(m.sender_name)]
        r = recs[i]
        r["str_off"] = len(strs)
        r["ts_sec"], r["ts_nsec"], r["views"] = m.ts_sec, m.ts_nsec, m.views
        r["id_len"], r["channel_len"], r["text_len"], r["sender_len"] = (len(parts[0]), len(parts[1]), len(parts[2]), len(parts[3]))
        strs += b"".join(parts)
        for k, cnt in m.reactions:
            kb = _b(k)
            reacts.append((len(aux), len(kb), 0, cnt))
            aux += kb
        react_off[i + 1] = len(reacts)
    ra = np.array(reacts, abi.GM_REACTION) if reacts else np.zeros(0, abi.GM_REACTION)
    return GmBatch(recs=recs, strs=_blob(strs), react_off=react_off, reacts=ra, aux=_blob(aux))


# ---- channel records: the random-walk StoreChannelData line ----------------------------------------------------------
@dataclass
class ChannelRecord:  # what RunForChannel puts in model.ChannelData (crawl/runner.go:592-610)
    chat_id: int = 0                 # chat.Id
    title: str | bytes = ""          # chat.Title
    image: str | bytes = ""          # chat.Photo.Extra ("" when chat.Photo == nil)
    url: str | bytes = ""            # p.URL
    member_count: int = 0            # int32(memberCount), int32(messageCount), int32(totalViews) (runner.go:980-982)
    message_count: int = 0
    total_views: int = 0


class ChBatch:
    FIELDS = ("recs", "strs")

    def __init__(self, **arrays):
        for k in self.FIELDS:
            setattr(self, k, arrays[k])
        self.n = len(self.recs)

    def descriptor(self) -> abi.ChBatchC:
        d = abi.ChBatchC()
        d.n = self.n
        d.recs = abi.ptr(self.recs)
        d.strs = abi.ptr(self.strs)
        d.strs_len = self.strs.size
        return d


def pack_channels(recs_in: list[ChannelRecord]) -> ChBatch:
    """one tgi_ch_rec per channel page; title | image | url of each record back to back in one blob"""
    recs = np.zeros(len(recs_in), abi.CH_REC)
    strs = bytearray()
    for i, c in enumerate(recs_in):
        parts = [_b(c.title), _b(c.image), _b(c.url)]
        r = recs[i]
        r["chat_id"], r["str_off"] = c.chat_id, len(strs)
        r["member_count"], r["message_count"], r["total_views"] = c.member_count, c.message_count, c.total_views
        r["title_len"], r["image_len"], r["url_len"] = (len(p) for p in parts)
        strs += b"".join(parts)
    return ChBatch(recs=recs, strs=_blob(strs))
