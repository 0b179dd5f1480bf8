"""A literal Python restatement of the page close (crawl/runner.go:1543-1544, dapr/standalone.go:589-609) over
state_rules.GoState: the expected output of tgi_state_page_close, with the owner's list tracked across the turn.

In Go the runner's `owner` keeps the slice header page_begin's UpdatePage(*owner) stored: its messages are
runner_rules.page_begin's owner messages.  UpdatePage(*owner) stores that slice again, so whatever the loop's
UpdateMessage calls appended to pageMap's page is gone.  The loop's hits on owner messages reach the owner only while
pageMap's page still shares the owner's backing array; the library counts that array as full (cap == len), so the
first append reallocates it (the one rule Go does not pin: cap comes from growslice and malloc size classes)."""
from __future__ import annotations

import copy

import runner_rules as rr


def page_begin(go, pid: bytes, fetched, page=None):
    """runner_rules.page_begin; returns (owner, processed, work) where owner is the owner's message list (the view)"""
    processed, work = rr.page_begin(go, pid, fetched, page)
    return copy.deepcopy(processed), processed, work


def page_end(go, pid: bytes, owner, processed, statuses, n_done: int) -> int:
    """runner_rules.page_end, and the owner's side of each UpdateMessage (owner None: the row holds no view of this
    turn).  Returns the hits that reached the owner."""
    hits, appended = 0, False
    for message, s in list(zip(processed, statuses))[:n_done]:
        chat, msg = message["messageId"], message["chatId"]  # swapped, as the reference passes them
        status = b"failed" if s == rr.ST_FAILED else b"fetched"
        msgs = go.page_map[pid].get("messages") or []
        first = next((i for i, m in enumerate(msgs) if m["chatId"] == chat and m["messageId"] == msg), None)
        if first is None:
            appended = True  # append reallocates: pageMap's page leaves the owner's array
        elif owner is not None and not appended and first < len(owner):
            owner[first]["status"] = status  # the shared array: the owner sees the write
            hits += 1
        go.update_message(pid, chat, msg, status)
    return hits


def page_close(go, page, owner):
    """UpdatePage(*owner) / UpdatePage(page): page = the fields (no messages); owner = the row's view, or None (no turn
    ran: the list is the one the runner read, the page's list as it is)"""
    p = copy.deepcopy(page)
    p["messages"] = copy.deepcopy(owner if owner is not None else go.page_map[page["id"]].get("messages") or [])
    go.update_page(p)
