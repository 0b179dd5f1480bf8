"""A literal Python restatement of snowball discovery over state_rules.GoState and dapr_state_rules: the candidate pages
of processAllMessagesWithProcessor outside random-walk (crawl/runner.go:1199-1244), the standalone runner's AddLayer per
page (standalone/runner.go:835-850), the Dapr runner's layer end (dapr/standalone.go:612-616, 645-688), Dapr's AddLayer
with its urlCache, and the library's page-id generator: the expected output of tgi_state_discover /
tgi_state_next_layer.

Two things are fixed where Go is random.  The outlinks of one message come from a map, so every order is valid; the
library takes the result's link-row order.  uuid.New() is random; the library's ids are Philox4x32-10 of a counter of
added pages under a seed (page_id), and the restatement hands the n-th added page the n-th id.  Every added page gets
the call's one clock reading, in time.Local (a None offset)."""
from __future__ import annotations

import copy

from dapr_state_rules import dapr_add_layer

ST_EMITTED, ST_SKIPPED, ST_FAILED, ST_NOLINE = 0, 1, 2, 3
MASK = 0xFFFFFFFF


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11): four 32-bit counter words and two key words -> four words"""
    c, k0, k1 = list(ctr), key[0], key[1]
    for r in range(10):
        if r:
            k0, k1 = (k0 + 0x9E3779B9) & MASK, (k1 + 0xBB67AE85) & MASK
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k0, p1 & MASK, (p0 >> 32) ^ c[3] ^ k1, p0 & MASK]
    return c


def page_id(seed: int, n: int) -> bytes:
    """the n-th page id under seed: the Philox words little-endian, version 4 and variant 10 bits, 8-4-4-4-12 hex"""
    w = philox4x32_10([n & MASK, n >> 32, 0, 0], [seed & MASK, seed >> 32])
    b = bytearray(b"".join(x.to_bytes(4, "little") for x in w))
    b[6] = b[6] & 0x0F | 0x40
    b[8] = b[8] & 0x3F | 0x80
    h = b.hex()
    return ("%s-%s-%s-%s-%s" % (h[:8], h[8:12], h[12:16], h[16:20], h[20:])).encode()


def outlinks(owner, status, links, n_done: int):
    """runner.go:1199-1244 outside random-walk: the pages built from one owner page's processed records.  status[i] and
    links[i] (outlink names in link-row order) are the result of its i-th record; the loop processed the first n_done.
    A failed record returned an error and a date-skipped one model.Post{}: neither has outlinks.  Ids and timestamps
    are left to AddLayer."""
    pages = []
    for i in range(n_done):
        if status[i] not in (ST_EMITTED, ST_NOLINE):
            continue
        for o in links[i]:
            if o == owner["url"]:  # :1231, byte for byte
                continue
            pages.append({"url": o, "status": b"unfetched", "parentId": owner["id"], "depth": owner.get("depth", 0) + 1})
    return pages


def url_cache_keys(urls):
    """the urlCache as the shim seeds TGI_SET_URLS: a key holds 32 bytes, and an outlink name (5-32 bytes) can never equal
    a longer URL, so those are left out"""
    return [u for u in urls if len(u) <= 32]


class Discovery:
    """the shim's side of both runners: the state, Dapr's urlCache (URL -> id), the id counter and its seed"""

    def __init__(self, go, seed: int, url_cache=None):
        self.go, self.seed, self.n = go, seed, 0
        self.url_cache = {} if url_cache is None else url_cache

    def _stamp(self, pages, added, now):
        """AddLayer's fill of the pages it adds: the next ids in append order, the clock in time.Local"""
        for p, a in zip(pages, added):
            p["timestamp"] = (now[0], now[1], None)
            if a:
                p["id"] = page_id(self.seed, self.n)
                self.n += 1
            else:
                p["id"] = b"not added %d" % id(p)

    def add_layer(self, pages, dapr: bool, now, max_pages: int = 0):
        """one AddLayer call under Base's rules (state/base.go:219-322) or Dapr's (daprstate.go:625-780); returns the
        added pages in append order"""
        pages = copy.deepcopy(pages)
        if dapr:
            for k, p in enumerate(pages):
                p["id"] = b"trial %d" % k
            _, to_add = dapr_add_layer(copy.deepcopy(self.go), dict(self.url_cache), pages)
            chosen = {id(p) for p in to_add}
            self._stamp(pages, [id(p) in chosen for p in pages], now)
            _, to_add = dapr_add_layer(self.go, self.url_cache, pages)
            return to_add
        trial = copy.deepcopy(self.go)
        trial.max_pages = max_pages
        marks = [dict(p, id=b"trial %d" % k) for k, p in enumerate(pages)]
        added = trial.add_layer(marks)
        self._stamp(pages, added, now)
        self.go.max_pages = max_pages
        got = self.go.add_layer(pages)
        return [p for p, a in zip(pages, got) if a]

    def standalone_page(self, owner_id: bytes, status, links, n_done: int, now, dapr: bool = False, max_pages: int = 0):
        """standalone/runner.go:835-850: the page's candidates as one AddLayer; none makes no call"""
        pages = outlinks(self.go.page_map[owner_id], status, links, n_done)
        if not pages:
            return []
        return self.add_layer(pages, dapr, now, max_pages)

    def layer_end(self, discovered, layer_depth: int, now, dapr: bool = True, max_pages: int = 0):
        """dapr/standalone.go:647-688: discovered = the layer's candidate pages in the order its pages reported them;
        the first occurrence of every URL (its ParentID too) at layer_depth + 1, then AddLayer"""
        if not discovered:
            return []
        seen, pages = set(), []
        for ch in discovered:
            if ch["url"] in seen:
                continue
            seen.add(ch["url"])
            pages.append({"url": ch["url"], "depth": layer_depth + 1, "status": b"unfetched",
                          "parentId": ch.get("parentId", b"")})
        return self.add_layer(pages, dapr, now, max_pages)
