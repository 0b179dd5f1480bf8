"""A literal Python restatement of the random-walk tandem branch of processAllMessagesWithProcessor, one page at a time
over state_rules.GoState (crawl/runner.go:1129, 1229-1306, 1414-1455), and of the library's batch-id generator: the
expected output of tgi_state_pending_edges.

Two things are fixed where Go is random.  The outlinks of one message come from a map, so every order is valid; the
library takes the result's link-row order.  uuid.New() is random; the library's batch ids are Philox4x32-10 of a
counter of batches under the page-id seed, with counter word 2 = 1 (batch_id), and the restatement hands the n-th
batch the n-th id."""
from __future__ import annotations

from discover_rules import MASK, ST_EMITTED, ST_NOLINE, philox4x32_10
from go_rules import filter_username

EDGE_PENDING, EDGE_DUPLICATE = 0, 1
TTL = 30 * 24 * 3600  # invalidChannelTTL (state/daprstate.go:3556-3564)


def batch_id(seed: int, n: int) -> bytes:
    """the n-th batch id under seed: page_id's construction with counter word 2 = 1"""
    w = philox4x32_10([n & MASK, n >> 32, 1, 0], [seed & MASK, seed >> 32])
    b = bytearray(b"".join(x.to_bytes(4, "little") for x in w))
    b[6] = b[6] & 0x0F | 0x40
    b[8] = b[8] & 0x3F | 0x80
    h = b.hex()
    return ("%s-%s-%s-%s-%s" % (h[:8], h[8:12], h[12:16], h[16:20], h[20:])).encode()


def is_invalid_channel(invalid: dict, name: bytes, now_sec: int) -> bool:
    """sm.IsInvalidChannel (daprstate.go:3556-3564): invalid = name -> stamp; a stamp of 0 never expires"""
    t = invalid.get(name)
    return t is not None and (t == 0 or now_sec - t < TTL)


class Tandem:
    """the shim's side: the state, the two validator caches and the batch counter with its seed"""

    def __init__(self, go, seed: int):
        self.go, self.seed, self.n = go, seed, 0
        self.invalid: dict[bytes, int] = {}
        self.discovered: set[bytes] = set()

    def page(self, owner_id: bytes, status, links, n_done: int, now_sec: int):
        """one processAllMessagesWithProcessor call in tandem mode.  status[i] and links[i] (the (name, source) pairs of
        the record's link rows) are the result of its i-th record; the loop processed the first n_done.  Returns
        (batch, edges): batch None means no PendingEdgeBatch was made and the crawler walks back (:1425-1455)."""
        owner = self.go.page_map[owner_id]
        seen_in_batch = set()  # :1129, fresh for every page
        batch, edges = None, []
        for i in range(n_done):
            if status[i] not in (ST_EMITTED, ST_NOLINE):  # a failed record returned an error, a date-skipped one model.Post{}
                continue
            for o, src in links[i]:
                if o == owner["url"]:  # :1231, byte for byte
                    continue
                if is_invalid_channel(self.invalid, o, now_sec):  # :1247
                    continue
                if filter_username(o) != "":  # :1261
                    continue
                if o in seen_in_batch:  # :1267-1272
                    continue
                seen_in_batch.add(o)
                if batch is None:  # :1275-1291
                    batch = {"batch_id": batch_id(self.seed, self.n), "source_channel": owner["url"],
                             "source_page_id": owner["id"], "source_depth": owner.get("depth", 0),
                             "sequence_id": owner.get("sequenceId", b""), "status": "open"}
                    self.n += 1
                # :1293-1306, classified as the validator's cache look-ups do (validator.go:214-226)
                edges.append({"destination": o, "record": i, "source_type": src,
                              "status": EDGE_DUPLICATE if o in self.discovered else EDGE_PENDING})
        if batch is not None:  # :1414-1424 ClosePendingBatch
            batch["status"] = "closed"
        return batch, edges
