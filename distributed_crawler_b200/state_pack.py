"""Packer of state.Page / state.Message values for the tgi_state_* entry points.

A page is a dict with the JSON names of state.Page (state/datamodels.go:41-62): the nine strings as bytes ("id", "url",
"status", "error", "platform", "parentId", "LastConnectionID", "sequenceId", "crawlId"; missing = empty), "depth",
"timestamp" = (sec, nsec, offset_sec) with offset_sec None for time.Local, and "messages" = a list of dicts with
"chatId", "messageId", "status", "pageId" and "platform" (bytes).  Missing strings, depth and messages are empty / 0 /
none; a missing timestamp is Go's zero time."""
from __future__ import annotations

import numpy as np

from . import abi

ZERO_TIME = (-62135596800, 0, 0)  # time.Time{}: 0001-01-01T00:00:00Z


def pack_pages(pages, code, msg_page):
    """-> (tgi_state_page array, string blob, tgi_state_msg array).  code(bytes) -> status / platform code;
    msg_page(pageId bytes, index of its page in `pages`) -> the message's page_id field."""
    recs = np.zeros(len(pages), abi.STATE_PAGE)
    blob = bytearray()
    msgs = []
    for i, p in enumerate(pages):
        recs[i]["str_off"] = len(blob)
        for k, name in enumerate(abi.STATE_STRINGS):
            s = p.get(name, b"")
            recs[i]["str_len"][k] = len(s)
            blob += s
        sec, nsec, off = p.get("timestamp", ZERO_TIME)
        recs[i]["ts_sec"], recs[i]["ts_nsec"] = sec, nsec
        recs[i]["ts_off"] = abi.STATE_TS_LOCAL if off is None else off
        recs[i]["depth"] = p.get("depth", 0)
        ms = p.get("messages") or []
        recs[i]["n_msgs"] = len(ms)
        for m in ms:
            msgs.append((m["chatId"], m["messageId"], msg_page(m.get("pageId", b""), i), code(m.get("status", b"")),
                         code(m.get("platform", b""))))
    return recs, np.frombuffer(bytes(blob) + b"\0" * 16, np.uint8).copy(), np.array(msgs, abi.STATE_MSG)


def pack_claimed_batches(batches):
    """-> (tgi_claimed_batch array, edge_off u64[n+1], tgi_claimed_edge array, string blob) of claimed batches, each a
    dict with PendingEdgeBatch's strings as bytes (abi.CLAIMED_BATCH_STRINGS; missing = empty), "source_depth" and
    "edges" = [(destination, source_type, validation_status)], all bytes; the status maps to abi.EDGE_CLASS_* by exact
    match, anything else OTHER.  Equal strings are stored once."""
    recs = np.zeros(len(batches), abi.CLAIMED_BATCH)
    edge_off = np.zeros(len(batches) + 1, np.uint64)
    blob = bytearray()
    at = {}

    def put(s):
        o = at.get(s)
        if o is None:
            o = at[s] = len(blob)
            blob.extend(s)
        return o

    rows = []
    for i, b in enumerate(batches):
        for k, name in enumerate(abi.CLAIMED_BATCH_STRINGS):
            s = b.get(name, b"")
            recs[i]["str_off"][k], recs[i]["str_len"][k] = put(s), len(s)
        recs[i]["source_depth"] = b.get("source_depth", 0)
        for dest, st, status in b.get("edges", ()):
            rows.append((put(dest), put(st), len(dest), len(st), abi.EDGE_CLASS_OF.get(status, abi.EDGE_CLASS_OTHER)))
        edge_off[i + 1] = len(rows)
    edges = np.zeros(len(rows), abi.CLAIMED_EDGE)
    if rows:
        a = np.array(rows, np.uint64)
        edges["str_off"] = a[:, 0:2]
        edges["str_len"] = a[:, 2:4]
        edges["cls"] = a[:, 4]
    return recs, edge_off, edges, np.frombuffer(bytes(blob) + b"\0" * 16, np.uint8).copy()
