#!/usr/bin/env python
"""tools/step_timeline.py — where the wall time of one bench.py M2 step goes.

Runs the headline step of bench.py (fused FilterExec -> AggExec(Partial) -> AggExec(Final), one op, input resident in HBM)
with the bench's plan, conf and seeded inputs, and records:

  calls     host wall time of every C-ABI call of a step (release of the previous step's outputs, create, push_device,
            finish, each pull_device, metrics, destroy) over --steps warm steps, profiler off.  Each call is timed as the bench
            makes it: it returns at the op's own synchronisation, nothing is added.
  timeline  a torch.profiler trace (CUDA activities) of --trace-steps warm steps, in a run of its own, written under --out.
            Printed from it: every kernel, memcpy and memset of a step with its duration, every gap between consecutive device
            activities (and before the first / after the last one of the step) with the host call that was running during it,
            and per step the kernel time, the other device time (copies, memsets) and the idle time.

The card's name and power limit are printed and stored beside the numbers (step_timeline.json under --out).
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the plan, conf and inputs of the measured step)

DEVICE_CATS = ("kernel", "gpu_memcpy", "gpu_memset")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception as e:                                       # the numbers are still printed, marked as of an unknown card
        return f"unknown ({e})"


def run_step(r, native, mark, calls):
    """one bench M2 step (Runner.step_device, world 1), every C-ABI call timed on the host clock and wrapped in mark(name)"""
    def call(name, fn):
        with mark(name):
            t0 = time.perf_counter()
            out = fn()
            calls.append((name, 1e3 * (time.perf_counter() - t0)))
        return out
    call("release previous outputs", r._drop_last)
    op = call("create", lambda: native.NativeOp(r.plans["single"], r.conf, r.local))
    call("push_device", lambda: op.push_device(r._input_batch()))
    call("finish", op.finish)
    outs, i = [], 0
    while True:
        o = call(f"pull_device {i}", op.pull_device)
        i += 1
        if o is None:
            break
        outs.append(o)
    r.last = outs
    call("metrics", op.metrics)
    call("destroy", op.close)


def host_calls(torch, r, native, steps):
    from contextlib import nullcontext
    per_step = []
    for _ in range(steps):
        calls = []
        run_step(r, native, lambda name: nullcontext(), calls)
        per_step.append(calls)
    names = [n for n, _ in per_step[0]]
    rows = []
    for j, n in enumerate(names):
        v = sorted(s[j][1] for s in per_step if j < len(s) and s[j][0] == n)
        rows.append({"call": n, "ms_min": v[0], "ms_median": v[len(v) // 2], "ms_max": v[-1]})
    totals = sorted(sum(ms for _, ms in s) for s in per_step)
    return {"calls": rows, "step_ms": totals}


def device_timeline(torch, r, native, steps, out_dir):
    from torch.profiler import ProfilerActivity, profile, record_function, schedule
    sched = schedule(wait=0, warmup=1, active=steps, repeat=1)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], schedule=sched) as prof:
        for i in range(steps + 1):
            with record_function(f"step {i}"):
                run_step(r, native, record_function, [])
            prof.step()
    path = os.path.join(out_dir, "step_timeline.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = json.load(f)["traceEvents"]
    dev = sorted((e for e in ev if e.get("cat") in DEVICE_CATS and "dur" in e), key=lambda e: e["ts"])
    ann = [e for e in ev if e.get("cat") == "user_annotation" and "dur" in e]
    step_ann = sorted((e for e in ann if e["name"].startswith("step ")), key=lambda e: e["ts"])
    call_ann = [e for e in ann if not e["name"].startswith("step ")]
    out = []
    for s in step_ann:
        s0, s1 = s["ts"], s["ts"] + s["dur"]
        acts = [e for e in dev if s0 <= e["ts"] <= s1]
        calls = [c for c in call_ann if s0 <= c["ts"] <= s1]

        def during(a, b):
            best, ov = "-", 0.0
            for c in calls:
                o = min(b, c["ts"] + c["dur"]) - max(a, c["ts"])
                if o > ov:
                    best, ov = c["name"], o
            return best
        items, gaps, cursor = [], [], s0
        kern = other = 0.0
        for e in acts:
            if e["ts"] > cursor:
                gaps.append({"us": e["ts"] - cursor, "before": e["name"][:60], "host_call": during(cursor, e["ts"])})
            items.append({"name": e["name"][:90], "cat": e["cat"], "stream": e.get("args", {}).get("stream"), "us": e["dur"],
                          "host_call": during(e["ts"], e["ts"] + e["dur"])})
            if e["cat"] == "kernel":
                kern += e["dur"]
            else:
                other += e["dur"]
            cursor = max(cursor, e["ts"] + e["dur"])
        if s1 > cursor:
            gaps.append({"us": s1 - cursor, "before": "(end of step)", "host_call": during(cursor, s1)})
        idle = sum(g["us"] for g in gaps)
        by_call = {}
        for g in gaps:
            by_call[g["host_call"]] = by_call.get(g["host_call"], 0.0) + g["us"]
        out.append({"step": s["name"], "wall_us": s1 - s0, "kernel_us": kern, "other_device_us": other, "idle_us": idle,
                    "idle_by_host_call_us": by_call, "activities": items, "gaps": gaps})
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rows", type=int, default=1_000_000_000)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--steps", type=int, default=5, help="warm steps of host call timing")
    ap.add_argument("--trace-steps", type=int, default=3, help="warm steps in the profiler trace")
    ap.add_argument("--gap-us", type=float, default=5.0, help="print gaps at least this long one by one")
    ap.add_argument("--out", required=True, help="directory for the trace and step_timeline.json")
    a = ap.parse_args()
    import torch
    from blaze_b200 import native
    if not torch.cuda.is_available():
        raise SystemExit("step_timeline.py measures a GPU run: no CUDA device is visible")
    os.makedirs(a.out, exist_ok=True)
    torch.cuda.set_device(0)
    r = bench.Runner("M2", torch, None, native, 0, 1, 0, a.rows, None)
    for _ in range(a.warmup):
        r.step_device()
    gpu = card()
    print(f"card: {gpu}   rows: {a.rows}")
    hc = host_calls(torch, r, native, a.steps)
    print(f"\nhost wall time per C-ABI call, {a.steps} warm steps (ms: min / median / max)")
    for c in hc["calls"]:
        print(f"  {c['call']:<26} {c['ms_min']:8.3f} {c['ms_median']:8.3f} {c['ms_max']:8.3f}")
    print("  step total                 " + " ".join(f"{t:.3f}" for t in hc["step_ms"]))
    tl = device_timeline(torch, r, native, a.trace_steps, a.out)
    for s in tl:
        print(f"\n{s['step']}: wall {s['wall_us'] / 1e3:.3f} ms = kernels {s['kernel_us'] / 1e3:.3f} + other device {s['other_device_us'] / 1e3:.3f}"
              f" + idle {s['idle_us'] / 1e3:.3f} ms (profiled: the host side runs slower than in the timing above)")
        for it in s["activities"]:
            print(f"  {it['cat']:<10} {it['us']:9.1f} us  stream {it['stream']}  [{it['host_call']}]  {it['name']}")
        print("  gaps >= %.0f us:" % a.gap_us)
        for g in s["gaps"]:
            if g["us"] >= a.gap_us:
                print(f"    {g['us']:9.1f} us during [{g['host_call']}] before {g['before']}")
        print("  idle by host call: " + ", ".join(f"{k} {v:.1f} us" for k, v in sorted(s["idle_by_host_call_us"].items(), key=lambda kv: -kv[1])))
    r.close()
    with open(os.path.join(a.out, "step_timeline.json"), "w") as f:
        json.dump({"card": gpu, "rows": a.rows, "host_calls": hc, "timeline": tl}, f, indent=1)


if __name__ == "__main__":
    main()
