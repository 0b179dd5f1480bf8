"""A literal Python restatement of processAllMessagesWithProcessor's message bookkeeping (crawl/runner.go:1132-1147,
1161-1211) over state_rules.GoState: the expected output of tgi_state_page_begin / tgi_state_page_end.

The shim's `owner` is the state's own page: its messages are the state's, with no update in between."""
from __future__ import annotations

import copy

ST_FAILED = 2  # abi.ST_FAILED: ProcessMessage returned an error


# addNewMessages (crawl/runner.go:1650-1697): the map is built from the owner's list only, so a key discovered twice is
# returned twice; the result REPLACES owner.Messages
def add_new_messages(discovered, owner):
    existing = {}
    for m in owner.get("messages") or []:
        existing["%d_%d" % (m["chatId"], m["messageId"])] = True
    return [m for m in discovered if not existing.get("%d_%d" % (m["chatId"], m["messageId"]))]


# resampleMarker (crawl/runner.go:1572-1635)
def resample_marker(messages, discovered):
    dmap = {"%d_%d" % (m["chatId"], m["messageId"]): True for m in discovered}
    for m in messages:
        if m["status"] == b"fetched":
            continue
        m["status"] = b"resample" if dmap.get("%d_%d" % (m["chatId"], m["messageId"])) else b"deleted"
    return messages


def page_begin(go, pid: bytes, fetched, page=None):
    """:1132-1147 and the loop's look-ups (:1161-1176).  fetched = [(chat_id, message_id)] in fetch order; page
    (optional) = the owner's fields.  Returns (owner messages, work): work[i] = the index into fetched of the
    discMessage of the i-th message the loop processes."""
    owner = copy.deepcopy(page if page is not None else go.get_page(pid))
    owner["messages"] = copy.deepcopy(go.get_page(pid).get("messages") or [])
    discovered = [{"chatId": c, "messageId": m, "status": b"unfetched", "pageId": pid} for c, m in fetched]
    owner["messages"] = add_new_messages(discovered, owner)
    owner["messages"] = resample_marker(owner["messages"], discovered)
    go.update_page(owner)
    processed, work = [], []
    for message in owner["messages"]:
        if message["status"] in (b"fetched", b"deleted"):
            continue
        disc = None
        for i, (_, m) in enumerate(fetched):  # the first fetched message with the id; the chat id is not compared
            if m == message["messageId"]:
                disc = i
                break
        # every owner message came from this fetch, so the "deleted" branch (:1185) is unreachable from this flow
        assert disc is not None
        processed.append(copy.deepcopy(message))
        work.append(disc)
    return processed, work


def page_end(go, pid: bytes, processed, statuses, n_done: int):
    """the loop's first n_done UpdateMessage calls (:1201-1209), with the chat and message ids swapped as the
    reference passes them"""
    for message, s in list(zip(processed, statuses))[:n_done]:
        go.update_message(pid, message["messageId"], message["chatId"], b"failed" if s == ST_FAILED else b"fetched")
