#!/usr/bin/env python3
"""Writes tests/golden/random_walk_vectors.json: the known-answer vectors the reference's OWN tests of the standard
random-walk branch of processAllMessagesWithProcessor hold, transcribed literal by literal with file:line provenance:
  crawl/runner_tandem_test.go      TestNonTandemMode_Unchanged
  crawl/runner_flood_wait_test.go  TestStandardMode_ShortFloodWait, _LongFloodWait, _NotFoundError,
                                   _ShortFloodWait_RetryFailsWithNotFound
The reference is Go and is not executed: these are transcriptions of the test sources, not outputs of a run.  Each
test mocks one message whose only outlink is the name, an owner "source_channel" with SequenceID "seq-1", and caches
that hold nothing of the name; a short FLOOD_WAIT is slept and retried, so only the final outcome is recorded.
"""
import json
import os

STANDARD_WALK = [  # processAllMessagesWithProcessor's standard random-walk branch (owner "source_channel", seq-1, one
    # message whose only outlink is the name; the sets hold nothing of it).  (test name, go file, go line, outlink,
    # walkback rate, SearchPublicChat's final outcome (a short FLOOD_WAIT is slept and retried by the caller) and chat id,
    # the discovered set the walkback reads, and the expectation)
    ("TestNonTandemMode_Unchanged", "crawl/runner_tandem_test.go", 217, "valid_channel", 0, ("found", -100123), [],
     {"error": None, "upsert_seed": [["valid_channel", -100123]], "mark_invalid": [], "added_discovered": ["valid_channel"],
      "page_url": "valid_channel", "walkback": False}),
    ("TestStandardMode_ShortFloodWait", "crawl/runner_flood_wait_test.go", 62, "flood_chan", 0, ("found", -100999), [],
     {"error": None, "upsert_seed": [["flood_chan", -100999]], "mark_invalid": [], "added_discovered": ["flood_chan"],
      "page_url": "flood_chan", "walkback": False}),
    ("TestStandardMode_LongFloodWait", "crawl/runner_flood_wait_test.go", 129, "target_chan", 0, ("retire", 0), [],
     {"error": "ErrFloodWaitRetire", "upsert_seed": [], "mark_invalid": [], "added_discovered": [], "page_url": None,
      "walkback": None}),
    ("TestStandardMode_NotFoundError", "crawl/runner_flood_wait_test.go", 183, "ghost_chan", 0, ("not_found", 0),
     ["walkback_target"],
     {"error": None, "upsert_seed": [], "mark_invalid": [["ghost_chan", "not_found"]], "added_discovered": [],
      "page_url": "walkback_target", "walkback": True}),
    ("TestStandardMode_ShortFloodWait_RetryFailsWithNotFound", "crawl/runner_flood_wait_test.go", 242, "retry_chan", 0,
     ("not_found", 0), ["walkback_target"],
     {"error": None, "upsert_seed": [], "mark_invalid": [["retry_chan", "not_found"]], "added_discovered": [],
      "page_url": "walkback_target", "walkback": True}),
]


def main():
    out = {
        "provenance": "transcribed from the reference's Go test sources; see this script's docstring",
        "standard_walk": [dict(name=n, go_file=f, go_line=ln, outlink=o, walkback_rate=rate, outcome=list(oc), discovered=d,
                               expect=ex) for n, f, ln, o, rate, oc, d, ex in STANDARD_WALK],
    }
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "random_walk_vectors.json")
    with open(path, "w", encoding="utf-8") as f:
        json.dump(out, f, ensure_ascii=False, indent=1)
    print("wrote", path, len(STANDARD_WALK), "standard-walk vectors")


if __name__ == "__main__":
    main()
