#!/usr/bin/env python3
"""Writes tests/golden/validator_edge_vectors.json: the known-answer vectors the reference's OWN tests of the edge
validator hold, transcribed literal by literal with file:line provenance:
  crawl/validator_test.go  TestValidateSingleEdge_Valid, _TransientError, _BlockedError, _NotChannel, _AlreadyInvalid,
                           _AlreadyDiscovered, _ValidButRaceLost (validateSingleEdge, :28-212)
                           TestRunEdgeValidation_EntersBlockedState, _ProbeResumesValidation (runEdgeValidation, :406-546)
The reference is Go and is not executed: these are transcriptions of the test sources, not outputs of a run.  A world
lists the mocks: IsInvalidChannel's true names ("invalid"), IsChannelDiscovered's true names ("discovered"),
ClaimDiscoveredChannel's false names ("raced") and validateFn's answers per name ("script": [status or error kind,
reason]).  Each case is one claim; the probe case is two claims with a successful probe between them.
"""
import json
import os

SINGLE_EDGE = [  # (test name, go line, edge (pending_id, destination, crawl_id), world, expect: status, reason, kind,
    # the DaprStateManager calls made with side effects)
    ("TestValidateSingleEdge_Valid", 28, (1, "testchan", "crawl-1"),
     {"script": {"testchan": [["valid", ""]]}},
     {"status": "valid", "reason": "", "kind": "definitive",
      "calls": [["ClaimDiscoveredChannel", "testchan", "crawl-1"], ["UpsertSeedChannelChatID", "testchan", 0]]}),
    ("TestValidateSingleEdge_TransientError", 58, (1, "testchan", "crawl-1"),
     {"script": {"testchan": [["transient", ""]]}},
     {"status": "pending", "reason": "", "kind": "transient", "calls": []}),
    ("TestValidateSingleEdge_BlockedError", 89, (1, "testchan", "crawl-1"),
     {"script": {"testchan": [["blocked", ""]]}},
     {"status": "pending", "reason": "", "kind": "blocked", "calls": []}),
    ("TestValidateSingleEdge_NotChannel", 120, (3, "userchan", "crawl-1"),
     {"script": {"userchan": [["not_channel", "not_supergroup"]]}},
     {"status": "not_channel", "reason": "not_supergroup", "kind": "definitive",
      "calls": [["MarkChannelInvalid", "userchan", "not_supergroup"]]}),
    ("TestValidateSingleEdge_AlreadyInvalid", 145, (1, "badchan", "crawl-1"),
     {"invalid": ["badchan"]},
     {"status": "invalid", "reason": "cached_invalid", "kind": "definitive", "calls": []}),
    ("TestValidateSingleEdge_AlreadyDiscovered", 167, (2, "known_chan", "crawl-1"),
     {"discovered": ["known_chan"]},
     {"status": "duplicate", "reason": "", "kind": "definitive", "calls": []}),
    ("TestValidateSingleEdge_ValidButRaceLost", 187, (4, "raced_chan", "crawl-1"),
     {"raced": ["raced_chan"], "script": {"raced_chan": [["valid", ""]]}},
     {"status": "duplicate", "reason": "", "kind": "definitive",
      "calls": [["ClaimDiscoveredChannel", "raced_chan", "crawl-1"]]}),
]

BLOCKED = [  # (test name, go line, claims: [edges (pending_id, destination, crawl_id)], world, expect per claim: the
    # UpdatePendingEdge calls [pending_id, status, reason], whether InsertAccessEvent("ip_blocked") ran)
    ("TestRunEdgeValidation_EntersBlockedState", 406,
     [[[i + 1, "chan%d" % i, "crawl-1"] for i in range(6)]],
     {"script": {"chan%d" % i: [["blocked", ""]] for i in range(6)}},
     [{"updates": [[i + 1, "pending", ""] for i in range(6)], "access_event": True}]),
    ("TestRunEdgeValidation_ProbeResumesValidation", 465,
     [[[i + 1, "blocked%d" % i, "crawl-1"] for i in range(5)], [[100, "goodchan", "crawl-1"]]],
     {"script": dict({"blocked%d" % i: [["blocked", ""]] for i in range(5)}, goodchan=[["valid", ""]])},
     [{"updates": [[i + 1, "pending", ""] for i in range(5)], "access_event": True},
      {"updates": [[100, "valid", ""]], "access_event": False}]),
]


def main():
    out = {
        "provenance": "transcribed from the reference's Go test sources; see this script's docstring",
        "single_edge": [dict(name=n, go_file="crawl/validator_test.go", go_line=ln, edge=list(e), world=w, expect=ex)
                        for n, ln, e, w, ex in SINGLE_EDGE],
        "blocked_state": [dict(name=n, go_file="crawl/validator_test.go", go_line=ln, claims=c, world=w, expect=ex)
                          for n, ln, c, w, ex in BLOCKED],
    }
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "validator_edge_vectors.json")
    with open(path, "w", encoding="utf-8") as f:
        json.dump(out, f, ensure_ascii=False, indent=1)
    print("wrote", path, len(SINGLE_EDGE), "single-edge and", len(BLOCKED), "blocked-state vectors")


if __name__ == "__main__":
    main()
