#!/usr/bin/env python
"""Summarise a torch.profiler chrome trace: per-stream busy time and per-kernel durations."""
import collections
import gzip
import json
import sys

tr = json.load(gzip.open(sys.argv[1]))
ev = [e for e in tr["traceEvents"] if e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy") and e.get("ph") == "X"]
ev.sort(key=lambda e: e["ts"])
t0, t1 = ev[0]["ts"], max(e["ts"] + e["dur"] for e in ev)
print("events %d, span %.3f ms" % (len(ev), (t1 - t0) / 1e3))
streams = collections.defaultdict(list)
for e in ev:
    streams[e["args"].get("stream")].append(e)
for sid, es in sorted(streams.items(), key=lambda kv: -sum(e["dur"] for e in kv[1])):
    busy = sum(e["dur"] for e in es)
    names = collections.Counter(e["name"].split("<")[0].split("(")[0].replace("void ", "").replace("gccb::", "") for e in es)
    print("stream %s: %d kernels, busy %.3f ms, top: %s" % (sid, len(es), busy / 1e3, names.most_common(3)))
by = collections.defaultdict(list)
for e in ev:
    by[e["name"].split("(")[0].replace("void ", "").replace("gccb::", "")[:60]].append(e["dur"])
print("%-62s %5s %9s %9s %9s" % ("kernel", "n", "mean_us", "max_us", "total_ms"))
for k, v in sorted(by.items(), key=lambda kv: -sum(kv[1]))[:34]:
    print("%-62s %5d %9.1f %9.1f %9.3f" % (k, len(v), sum(v) / len(v), max(v), sum(v) / 1e3))

if len(sys.argv) > 2:
    def training(e):
        return any(s in e["name"] for s in ("gin_", "infonce", "update_ema", "moco", "gradnorm"))

    def short(e):
        return e["name"].split("(")[0].replace("void ", "").replace("gccb::", "")[:50]

    # one step = between consecutive optimiser kernels (any stream)
    marks = sorted(e["ts"] for e in ev if "update_ema" in e["name"])
    # idle time on a training stream before each of its kernels (end of the stream's previous kernel -> start),
    # over every complete step: waits for SM slots show up here, beside waits for other streams' events
    gaps = collections.defaultdict(list)
    spans = []
    for lo, hi in zip(marks, marks[1:]):
        prev_end = {}
        inside = [e for e in ev if lo < e["ts"] <= hi and training(e)]
        spans.append((max(e["ts"] + e["dur"] for e in inside) - min(e["ts"] for e in inside)) if inside else 0.0)
        for e in inside:
            sid = e["args"].get("stream")
            if sid in prev_end:
                gaps[short(e)].append(e["ts"] - prev_end[sid])
            prev_end[sid] = max(prev_end.get(sid, 0.0), e["ts"] + e["dur"])
    nsteps = max(len(marks) - 1, 1)
    print("%d steps, period %.3f ms, training kernels' span %.3f ms per step; idle gaps before training kernels:" % (
        len(marks) - 1, (marks[-1] - marks[0]) / 1e3 / nsteps, sum(spans) / 1e3 / nsteps))
    print("%-52s %5s %9s %9s %13s" % ("kernel", "n", "mean_us", "max_us", "us_per_step"))
    for k, v in sorted(gaps.items(), key=lambda kv: -sum(kv[1]))[:24]:
        print("%-52s %5d %9.1f %9.1f %13.1f" % (k, len(v), sum(v) / len(v), max(v), sum(v) / nsteps))
    print("all gaps: %.1f us per step" % (sum(sum(v) for v in gaps.values()) / nsteps))
    lo, hi = marks[1], marks[2]
    print("step window %.3f ms; kernels of ALL streams inside it:" % ((hi - lo) / 1e3))
    inside = [e for e in ev if lo < e["ts"] <= hi and training(e)]
    prev_end = {}
    for e in inside:
        sid = e["args"].get("stream")
        gap = e["ts"] - prev_end.get(sid, e["ts"])
        prev_end[sid] = e["ts"] + e["dur"]
        print("%8.1f us  s%-4s dur %7.1f gap %7.1f  %s" % (e["ts"] - lo, sid, e["dur"], gap,
              e["name"].split("(")[0].replace("void ", "").replace("gccb::", "")[:50]))
