#!/usr/bin/env python3
"""Writes tests/golden/zones.json: transition tables of a few real zones, in the form tgi_set_zone takes.

Each table is built by probing ZoneInfo(name).utcoffset over [-2^31, 2^32) seconds: every 6 hours, and where the offset
differs between two probes, a bisection to the first second of the new offset.  Probing sees what the zone actually
does, including the POSIX-TZ footer rule that slim TZif files use for every year after their last explicit transition.
The first entry starts at -2^31 (the earliest Telegram Date) with the offset in effect there.

Tests read the committed JSON, never the system's tzdata: the machine running them may have none, or another version.
"""
import datetime
import json
import os
import zoneinfo

ZONES = [
    "America/New_York",     # DST
    "Europe/London",        # Z <-> +01:00: the line length changes with the season
    "Europe/Amsterdam",     # +00:19:32 and +01:19:32 before 1937: seconds in the offset
    "Africa/Monrovia",      # -00:44:30 until 1972
    "Australia/Lord_Howe",  # 30-minute DST
    "Asia/Kathmandu",       # +05:45
    "America/St_Johns",     # -03:30 / -02:30
]
LO, HI, STEP = -(1 << 31), 1 << 32, 6 * 3600


def table(name):
    z = zoneinfo.ZoneInfo(name)
    off = lambda t: int(datetime.datetime.fromtimestamp(t, z).utcoffset().total_seconds())
    starts, offsets = [LO], [off(LO)]
    t, o = LO, offsets[0]
    while t < HI - 1:
        u = min(t + STEP, HI - 1)
        ou = off(u)
        if ou != o:
            a, b = t, u  # off(a) == o != off(b): find the first second of the new offset
            while b - a > 1:
                m = (a + b) // 2
                if off(m) == o:
                    a = m
                else:
                    b = m
            starts.append(b)
            offsets.append(off(b))
            o = offsets[-1]
        t = u
    return {"start": starts, "offset": offsets}


def tzdata_version():
    try:
        with open("/usr/share/zoneinfo/tzdata.zi") as f:
            return f.readline().split()[-1]
    except OSError:
        return "unknown"


def main():
    out = {"range": [LO, HI], "tzdata": tzdata_version(), "zones": {n: table(n) for n in ZONES}}
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "zones.json")
    with open(path, "w") as f:
        json.dump(out, f, separators=(",", ":"))
        f.write("\n")
    print(path, {n: len(v["start"]) for n, v in out["zones"].items()})


if __name__ == "__main__":
    main()
