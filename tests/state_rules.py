"""A literal Python restatement of BaseStateManager (state/base.go) and of json.Marshal(State) (state/datamodels.go),
the expected output of the tgi_state_* entry points.  Pages and messages are state_pack dicts.

Marshal renders the layers in ascending depth: Go ranges over layerMap in random order, so that is one of its valid
outputs, and the one the engine fixes.  Strings go through go_rules.go_json_string (encoding/json's HTML-safe escaper);
time.Local timestamps use the zone rule of zone_oracle.go_json_time at the instant's offset."""
from __future__ import annotations

import copy

from go_rules import go_json_string
from zone_oracle import go_json_time, go_offset

OMITEMPTY_HEAD = ("error",)  # between status and timestamp
OMITEMPTY_MID = ("platform", "parentId")
OMITEMPTY_TAIL = ("LastConnectionID", "sequenceId", "crawlId")


class MarshalError(Exception):
    """json.Marshal fails: a time.Time whose year is outside [0, 9999]"""


class GoState:
    def __init__(self, max_pages: int = 0):
        self.max_pages = max_pages
        self.page_map: dict[bytes, dict] = {}
        self.layer_map: dict[int, list[bytes]] = {}

    # SetState (base.go:375-398)
    def set_state(self, layers):
        self.layer_map, self.page_map = {}, {}
        for depth, pages in layers:
            self.layer_map[depth] = []
            for p in pages:
                self.page_map[p["id"]] = copy.deepcopy(p)
                self.layer_map[depth].append(p["id"])

    # GetPage (base.go:110-120)
    def get_page(self, pid: bytes):
        return self.page_map.get(pid)

    # UpdatePage (base.go:123-149)
    def update_page(self, page):
        self.page_map[page["id"]] = copy.deepcopy(page)
        for depth, ids in self.layer_map.items():
            if depth == page.get("depth", 0):
                if page["id"] not in ids:
                    self.layer_map[depth] = ids + [page["id"]]
                break

    # UpdateMessage (base.go:182-215): False when the page is unknown (the reference's error)
    def update_message(self, pid: bytes, chat: int, msg: int, status: bytes) -> bool:
        page = self.page_map.get(pid)
        if page is None:
            return False
        msgs = page.setdefault("messages", [])
        for m in msgs:
            if m["chatId"] == chat and m["messageId"] == msg:
                m["status"] = status
                break
        else:
            msgs.append({"chatId": chat, "messageId": msg, "status": status, "pageId": pid})
        return True

    # AddLayer (base.go:219-322); the caller has filled ids and timestamps
    def add_layer(self, pages) -> list[bool]:
        if not pages:
            return []
        total = len(self.page_map)
        deadends = sum(1 for p in self.page_map.values() if p.get("status", b"") == b"deadend")
        reached = self.max_pages > 0 and total >= self.max_pages
        existing = {p.get("url", b""): pid for pid, p in self.page_map.items()}
        depth = pages[0].get("depth", 0)
        self.layer_map.setdefault(depth, [])
        replacements = deadends
        added = []
        for p in pages:
            if p.get("url", b"") in existing:
                added.append(False)
                continue
            if reached:
                if replacements <= 0:
                    added.append(False)
                    continue
                replacements -= 1
            self.page_map[p["id"]] = copy.deepcopy(p)
            existing[p.get("url", b"")] = p["id"]
            self.layer_map[depth].append(p["id"])
            added.append(True)
        return added

    # GetState (base.go:345-372), layers in ascending depth, then json.Marshal
    def marshal(self, metadata: bytes, last_updated: bytes, zone=None, tz: int = 0) -> bytes:
        layers = []
        for depth in sorted(self.layer_map):
            pages = [marshal_page(self.page_map[i], zone, tz) for i in self.layer_map[depth] if i in self.page_map]
            layers.append(b'{"depth":%d,"pages":[%s]}' % (depth, b",".join(pages)))
        return b'{"layers":[%s],"metadata":%s,"lastUpdated":%s}' % (b",".join(layers), metadata, last_updated)


def marshal_time(ts, zone=None, tz: int = 0) -> bytes:
    sec, nsec, off = ts
    if off is None:  # time.Local
        off = go_offset(zone, sec) if zone else tz
    out = go_json_time(sec, nsec, off)
    if not out:
        raise MarshalError(ts)
    return out


def marshal_message(m) -> bytes:
    out = b'{"chatId":%d,"messageId":%d,"status":%s,"pageId":%s' % (
        m["chatId"], m["messageId"], go_json_string(m.get("status", b"")), go_json_string(m.get("pageId", b"")))
    if m.get("platform"):
        out += b',"platform":' + go_json_string(m["platform"])
    return out + b"}"


def marshal_page(p, zone=None, tz: int = 0) -> bytes:
    f = [b'"id":' + go_json_string(p.get("id", b"")), b'"url":' + go_json_string(p.get("url", b"")),
         b'"depth":%d' % p.get("depth", 0), b'"status":' + go_json_string(p.get("status", b""))]
    f += [b'"%s":%s' % (k.encode(), go_json_string(p[k])) for k in OMITEMPTY_HEAD if p.get(k)]
    f.append(b'"timestamp":' + marshal_time(p.get("timestamp", (-62135596800, 0, 0)), zone, tz))
    f += [b'"%s":%s' % (k.encode(), go_json_string(p[k])) for k in OMITEMPTY_MID if p.get(k)]
    if p.get("messages"):
        f.append(b'"messages":[' + b",".join(marshal_message(m) for m in p["messages"]) + b"]")
    f += [b'"%s":%s' % (k.encode(), go_json_string(p[k])) for k in OMITEMPTY_TAIL if p.get(k)]
    return b"{" + b",".join(f) + b"}"
