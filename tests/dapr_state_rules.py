"""A literal Python restatement of DaprStateManager's in-memory AddLayer (state/daprstate.go:625-780), of the
json.Marshal(layerMap) in its SaveState (:947) and of both ExportPagesToBinding (daprstate.go:2911-3012,
storageproviders.go:550-587), on top of state_rules.GoState and marshal_page: the expected output of
tgi_state_add_pages, tgi_state_layer_map and tgi_state_export.

Two orders are Go map orders, so random in the reference and fixed here as the engine fixes them: the Dapr export walks
the layers in ascending depth, and the local export walks pageMap in row order (the order in which the ids first
entered it, which is also a Python dict's order).  A page json.Marshal cannot render (a timestamp year outside
[0, 9999]) raises MarshalError where Go logs it and skips the page: the engine refuses the call, as tgi_state_render
does."""
from __future__ import annotations

import base64
import copy

from go_rules import go_json_string
from state_rules import GoState, marshal_page


class NoPagesFound(Exception):
    """ExportPagesToBinding's "no pages found to export for crawl ID" """


def dapr_add_layer(go: GoState, url_cache: dict, pages, random_walk: bool = False):
    """AddLayer of DaprStateManager: -> (depth, the pages added).  url_cache (URL -> id) spans earlier crawls; it is
    read, not updated, during the filtering, and is skipped in random-walk mode.  The depth is pages[0]'s before the
    filtering; no layer is created when every page was a duplicate."""
    if not pages:
        return 0, []
    depth = pages[0].get("depth", 0)
    to_add = [p for p in pages if random_walk or p.get("url", b"") not in url_cache]
    if not to_add:
        return depth, []
    go.layer_map.setdefault(depth, [])
    for p in to_add:
        go.page_map[p["id"]] = copy.deepcopy(p)
        go.layer_map[depth].append(p["id"])
    for p in to_add:
        url_cache[p.get("url", b"")] = p["id"]
    return depth, to_add


def marshal_layer_map(layer_map: dict[int, list[bytes]]) -> bytes:
    """json.Marshal(map[int][]string): integer keys are sorted as their decimal strings"""
    keys = sorted(layer_map, key=lambda d: str(d))
    return b"{" + b",".join(b'"%d":[%s]' % (d, b",".join(go_json_string(i) for i in layer_map[d])) for d in keys) + b"}"


def export_dapr_chunks(go: GoState, chunk_bytes: int, zone=None, tz: int = 0) -> list[bytes]:
    """the raw JSONL of every InvokeBinding call of DaprStateManager.ExportPagesToBinding"""
    chunks, buf, exported = [], b"", 0
    for depth in sorted(go.layer_map):
        for pid in go.layer_map[depth]:
            if pid not in go.page_map:
                continue  # the reference's GetState fallback: the engine holds every page of its layer map
            buf += marshal_page(go.page_map[pid], zone, tz) + b"\n"
            exported += 1
            if len(buf) >= chunk_bytes:
                chunks.append(buf)
                buf = b""
    if exported == 0:
        raise NoPagesFound
    if buf:
        chunks.append(buf)
    return chunks


def export_dapr(go: GoState, storage_root: str, crawl_cfg_id: str, crawl_id: str, ts: str, chunk_bytes: int,
                zone=None, tz: int = 0) -> list[tuple[str, bytes]]:
    """every InvokeBinding call as (path, base64 data)"""
    return [("%s/%s/analysis/channels/channel-pages-%s-%s-part%d.jsonl" % (storage_root, crawl_cfg_id, crawl_id, ts, k),
             base64.b64encode(c)) for k, c in enumerate(export_dapr_chunks(go, chunk_bytes, zone, tz))]


def export_local(go: GoState, zone=None, tz: int = 0) -> bytes:
    """LocalStateManager.ExportPagesToBinding's file: every page of pageMap once"""
    return b"".join(marshal_page(p, zone, tz) + b"\n" for p in go.page_map.values())
