#!/usr/bin/env python
"""GPU diagnostic: A/B of library builds that differ in per-SM residency (which CTAs fit beside which), in one
process tree and alternating, so that the builds share the card's state.  Per build and round: `bench.py`
(`value`, `e2e`, `ms_per_step`, `step_time` p50/p95, `phases_ms`, launches per step, eigensolver class counts);
per build once: the training span against the period (`host_cost.py`).  Builds come from `build_variant.py`
(extra -D flags) or another checkout; "default" is the in-tree library.

usage: sm_budget.py [--rounds 3] [--steps 200] [--warmup 20] NAME=LIB [NAME=LIB ...]"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--steps", type=int, default=200)
ap.add_argument("--warmup", type=int, default=20)
ap.add_argument("--no-host-cost", action="store_true")
ap.add_argument("builds", nargs="+", metavar="NAME=LIB")
args = ap.parse_args()
builds = []
for b in args.builds:
    name, lib = b.split("=", 1)
    builds.append((name, None if lib == "default" else os.path.abspath(lib)))


def env_for(lib):
    env = dict(os.environ)
    env.pop("GCCB200_LIB", None)
    if lib:
        env["GCCB200_LIB"] = lib
    return env


card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card:", card, flush=True)
rows = {name: [] for name, _ in builds}
for rnd in range(args.rounds):
    for name, lib in builds:
        out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(args.steps),
                              "--warmup", str(args.warmup), "--no-cpu-baseline"], cwd=ROOT, env=env_for(lib),
                             capture_output=True, text=True)
        line = [x for x in out.stdout.splitlines() if x.startswith("{")]
        if out.returncode or not line:
            print("%s round %d failed (exit %d):\n%s" % (name, rnd, out.returncode, out.stderr[-3000:]), flush=True)
            continue
        r = json.loads(line[-1])
        st, ph, eig = r["step_time"], r["phases_ms"], r["eigensolver"]
        rows[name].append(r)
        print("round %d %-10s value %8.1f  e2e %8.1f  ms/step %.3f  p50 %.3f  p95 %.3f  sampler %.3f  eig %.3f ms  "
              "launches/step %.1f  dense/chfsi %d/%d  chfsi it %.3f  clock %s MHz %s" % (
                  rnd, name, r["value"], r["e2e"]["value"], r["ms_per_step"], st["p50_ms"], st["p95_ms"],
                  ph["sampler_ms"], ph["eigensolver_ms"], r["gpu_launches_per_step"], eig["egonets_dense_solver"],
                  eig["egonets_chfsi"], eig["mean_iterations_chfsi"], r["clocks"]["sm_mhz"], r["clocks"]["reasons"]),
              flush=True)
for name, lib in [] if args.no_host_cost else builds:
    out = subprocess.run([sys.executable, os.path.join(ROOT, "profiles", "host_cost.py")], cwd=ROOT, env=env_for(lib),
                         capture_output=True, text=True)
    m = re.search(r"period .*", out.stdout)
    print("%-10s host_cost: %s" % (name, m.group(0) if m else "failed: " + out.stderr[-2000:]), flush=True)
print("summary (mean over rounds):")
for name, _ in builds:
    rs = rows[name]
    if not rs:
        continue
    mean = lambda f: sum(f(r) for r in rs) / len(rs)  # noqa: E731
    print("%-10s value %8.1f [%s]  e2e %8.1f [%s]  ms/step %.3f" % (
        name, mean(lambda r: r["value"]), " ".join("%.1f" % r["value"] for r in rs),
        mean(lambda r: r["e2e"]["value"]), " ".join("%.1f" % r["e2e"]["value"] for r in rs),
        mean(lambda r: r["ms_per_step"])))
