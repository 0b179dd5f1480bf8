"""Expected lines in a local zone given as transitions (tgi_set_zone), for the CPU and GPU zone tests.

The CPU oracle renders time.Local at one fixed offset (tz_offset_sec).  ZonedOracle runs it in UTC and rewrites each
time.Local field of each line with go_json_time at that instant's offset, a Python restatement of Go's
appendFormatRFC3339 / appendStrictRFC3339.  A field whose local year leaves [0, 9999] turns its record into
TGI_ST_NOLINE with an empty line.  Status, links and frontier are otherwise the oracle's.
"""
import bisect
import datetime

import numpy as np

from distributed_crawler_b200 import abi
from oracle import pyoracle
from oracle.pyoracle import Oracle, Result

EPOCH = datetime.datetime(1970, 1, 1)
ERA_SEC = 146097 * 86400  # 400 Gregorian years: five of them move year 0 into datetime's range

# the time.Local fields of each line (tdutils.go:417,715; youtube_crawler.go:704,769; telegram_crawler.go:187-188,245).
# Telegram created_at is UTC (tdutils.go:611) and YouTube published_at keeps the API value's zone.
LOCAL_KEYS = {"telegram": ("published_at", "capture_time"), "youtube": ("created_at", "capture_time"),
              "generic": ("published_at", "created_at", "capture_time")}


def go_offset(zone, t):
    """offset of the last entry with start <= t; entry 0 before the first start"""
    starts, offsets = zone
    return int(offsets[max(bisect.bisect_right(starts, t) - 1, 0)])


def go_json_time(sec, nsec, off):
    """time.Time.MarshalJSON of time.Unix(sec, nsec) at offset `off` (RFC3339Nano, quoted); b"" outside year [0, 9999]"""
    t, shift = sec + off, 0
    if t < 0:
        t, shift = t + 5 * ERA_SEC, 5 * 400
    try:
        d = EPOCH + datetime.timedelta(seconds=t)
    except OverflowError:
        return b""
    year = d.year - shift
    if not 0 <= year <= 9999:
        return b""
    s = f"{year:04d}-{d.month:02d}-{d.day:02d}T{d.hour:02d}:{d.minute:02d}:{d.second:02d}"
    frac = f"{nsec:09d}".rstrip("0")
    if frac:
        s += "." + frac
    if off == 0:
        s += "Z"
    else:
        minutes = abs(off) // 60 * (1 if off > 0 else -1)  # offset / 60 truncated toward zero, sign of the minutes
        s += ("-" if minutes < 0 else "+") + f"{abs(minutes) // 60:02d}:{abs(minutes) % 60:02d}"
    return ('"' + s + '"').encode()


class ZonedOracle:
    """Oracle(**kw) with time.Local = zone (starts, offsets).  kw must leave tz_offset_sec at 0."""

    def __init__(self, zone, **kw):
        assert kw.get("tz_offset_sec", 0) == 0
        self.zone = (list(map(int, zone[0])), list(map(int, zone[1])))
        self.o = Oracle(**kw)
        c = self.o.cfg
        self.clock = (c.created_at_sec, c.created_at_nsec, c.capture_sec, c.capture_nsec)

    def set_clock(self, created_sec, created_nsec, capture_sec, capture_nsec):
        self.o.set_clock(created_sec, created_nsec, capture_sec, capture_nsec)
        self.clock = (created_sec, created_nsec, capture_sec, capture_nsec)

    def telegram(self, batch, run_flags=abi.RUN_JSONL | abi.RUN_LINKS):
        pub = [(int(d), 0) for d in batch.recs["date"]]
        return self._rezone(self.o.telegram(batch, run_flags), "telegram", pub)

    def youtube(self, batch, run_flags=abi.RUN_JSONL | abi.RUN_LINKS):
        return self._rezone(self.o.youtube(batch, run_flags), "youtube", None)

    def generic(self, batch, run_flags=abi.RUN_JSONL):
        pub = [(int(s), int(ns)) for s, ns in zip(batch.recs["ts_sec"], batch.recs["ts_nsec"])]
        return self._rezone(self.o.generic(batch, run_flags), "generic", pub)

    def _rezone(self, r, kind, pub):
        if not r.n or not len(r.jsonl):
            return r
        created, cns, cap, capns = self.clock
        status = r.status.copy()
        lines = []
        for i in range(r.n):
            line = r.line(i)
            if status[i] == abi.ST_EMITTED:
                for key in LOCAL_KEYS[kind]:
                    sec, ns = pub[i] if key == "published_at" else (created, cns) if key == "created_at" else (cap, capns)
                    utc, local = pyoracle.json_time(sec, ns), go_json_time(sec, ns, go_offset(self.zone, sec))
                    k = b'"' + key.encode() + b'":'
                    assert k + utc in line, (kind, i, key)
                    if not local:
                        status[i], line = abi.ST_NOLINE, b""
                        break
                    line = line.replace(k + utc, k + local, 1)
            elif status[i] == abi.ST_NOLINE and pub:  # dropped in UTC: it must be dropped in the zone too to be derived here
                sec, ns = pub[i]
                assert not go_json_time(sec, ns, go_offset(self.zone, sec)), (kind, i)
            lines.append(line)
        off = np.zeros(r.n + 1, np.uint64)
        off[1:] = np.cumsum([len(x) for x in lines], dtype=np.uint64)
        jsonl = np.frombuffer(b"".join(lines), np.uint8).copy()
        return Result(r.n, status, jsonl, off, r.link_off, r.links, r.n_new, r.frontier_size)

    def frontier_export(self):
        return self.o.frontier_export()
