"""A literal Python restatement of the reads that begin every layer, over state_rules.GoState: GetLayerByDepth,
GetMaxDepth and FindIncompleteCrawl's in-memory page test (state/base.go), and which pages of a layer each runner
processes (standalone/runner.go, dapr/standalone.go): the expected output of tgi_state_read_layer, tgi_state_read_pages
and tgi_state_layers.  Pages are state_pack dicts."""
from __future__ import annotations


# GetLayerByDepth (base.go:325-342): the listed ids that pageMap holds, in list order; no layer is []
def get_layer_by_depth(go, depth: int):
    ids = go.layer_map.get(depth)
    if ids is None:
        return []
    return [go.page_map[i] for i in ids if i in go.page_map]


# GetMaxDepth (base.go:446-462): None stands for its "no layers found" error
def get_max_depth(go):
    max_depth = -1
    for depth in go.layer_map:
        if depth > max_depth:
            max_depth = depth
    if max_depth == -1:
        return None
    return max_depth


# FindIncompleteCrawl (base.go:482-502): every listed page of pageMap whose status is not "fetched"; the reference
# stops at the first, the library counts them all
def incomplete_pages(go) -> int:
    n = 0
    for ids in go.layer_map.values():
        for i in ids:
            page = go.page_map.get(i)
            if page is not None and page.get("status", b"") != b"fetched":
                n += 1
    return n


# standalone/runner.go:636-694: the startIndex scan, then the loop from startIndex with its own skip
def standalone_selection(layer, resuming: bool) -> list[bool]:
    processed = [False] * len(layer)
    start = 0
    for i, la in enumerate(layer):  # :636-671
        if la.get("status", b"") == b"fetched":
            if resuming:
                start = i + 1
                continue
            break
        break
    for i in range(start, len(layer)):  # :672-694
        la = layer[i]
        if la.get("status", b"") == b"fetched" and resuming:
            continue
        processed[i] = True
    return processed


# processLayerInParallel (dapr/standalone.go:454-498), which sets isResumingSameCrawlExecution to true (:420): fetched
# and errored pages are skipped.  The URL is recorded before the status test.
def dapr_selection(layer, resuming: bool = True) -> list[bool]:
    processed = [False] * len(layer)
    unique_pages = {}
    for k, page in enumerate(layer):
        if unique_pages.get(page.get("url", b"")):  # :459-463
            continue
        unique_pages[page.get("url", b"")] = True
        if page.get("status", b"") in (b"fetched", b"error") and resuming:  # :477-497
            continue
        processed[k] = True
    return processed
