"""Independent pure-Python restatement of the random-walk StoreChannelData line, written from crawl/runner.go:587-607
(the model.ChannelData RunForChannel fills: chat.Id through strconv.FormatInt, chat.Title, chat.Photo.Extra or "" without
a photo, the three int32 counts widened to int, "https://t.me/" + p.URL twice), model/data.go:89-111 (field order; the
unset strings "", the unset counts 0, PublishedAt the zero time.Time), encoding/json (tests/go_rules.py) and
state/daprstate.go:3089-3094 (json.Marshal + '\\n') — NOT from tests/channel_oracle.c, so that the two check each
other."""
from __future__ import annotations

from go_rules import _Raw, _bs, _marshal


def channel_data_line(c) -> bytes:
    """-> the line of one pack.ChannelRecord"""
    url = b"https://t.me/" + _bs(c.url)
    data = [
        ("channel_id", str(int(c.chat_id)).encode()), ("channel_name", _bs(c.title)), ("channel_description", b""),
        ("channel_profile_image", _bs(c.image)),
        ("channel_engagement_data", [("follower_count", int(c.member_count)), ("following_count", 0), ("like_count", 0),
                                     ("post_count", int(c.message_count)), ("views_count", int(c.total_views)),
                                     ("comment_count", 0), ("share_count", 0)]),
        ("channel_url_external", url), ("channel_url", url), ("country_code", b""),
        ("published_at", _Raw(b'"0001-01-01T00:00:00Z"')),
    ]
    return _marshal(data) + b"\n"
