"""GPU box: the tail of a step, from the end of the persistent solver kernel to the start of the next narrow phase.

    python tools/step_tail_probe.py [pyramid|field|tumbler] [--warmup 12] [--steps 40]

Scenes and step parameters are those of tools/pair_search_probe.py (TGS_Soft, dt = 1/60, 4 sub-steps, 2 relax
iterations). After the warm-up the steps are recorded under torch.profiler (CUDA activities). Every window that opens at
the end of an s2bPersistentSolveT launch and closes at the start of the next s2bUpdateContactsKernel launch holds
finalize (s2bFinalizeBodies, then s2bFinalizeShapes or, on a pass that reuses the hierarchy, s2bFinalizeRefitKernel, which
also refits and collects the moved proxies; the moved-counter copy), the pair search queued behind it for the next step
(refit and movers where finalize did not do them, then one s2bFindPairs launch: the tree walk and the pair rules, survivors,
large movers; the mailbox copy) and the commit of that search at the start of the next step (merge, s2bClearMovedFlags). For each kernel, copy and memset the script prints its mean device
time per window and the mean idle gap in front of it; the gap in front of the first event of the next step includes the
host's per-step synchronisation and the counter read-back of this script. Also printed: the mean moved-proxy count per
step, the pair passes and the contact count.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

OPEN = "s2bPersistentSolveT"
CLOSE = "s2bUpdateContactsKernel"


def _short(name: str) -> str:
    name = name.replace("void ", "")
    if name.startswith("cub::"):
        return "cub::" + name[5:].split("<")[0].split("(")[0].split("::")[-1]
    return name.split("<")[0].split("(")[0][:60]


def tail_windows(events):
    """events: [(start_us, end_us, name)] sorted by start -> list of windows, each [(short, start, end)] between the end of
    the persistent kernel and the start of the next narrow phase (both excluded)."""
    windows, cur = [], None
    for t0, t1, name in events:
        short = _short(name)
        if short == OPEN:
            cur = {"t0": t1, "events": []}
            continue
        if cur is None:
            continue
        if short == CLOSE:
            cur["t1"] = t0
            windows.append(cur)
            cur = None
            continue
        cur["events"].append((short, t0, t1))
    return windows


def report(windows):
    dur, gap, seen = {}, {}, {}
    order = []
    spans, busy = [], []
    for w in windows:
        prev = w["t0"]
        per_d, per_g, times = {}, {}, {}
        for short, t0, t1 in w["events"]:
            # the second and later launches of one name in a window (the D2H copies) are reported apart
            times[short] = times.get(short, 0) + 1
            if times[short] > 1:
                short = f"{short} #{times[short]}"
            if short not in order:
                order.append(short)
            per_d[short] = per_d.get(short, 0.0) + (t1 - t0)
            per_g[short] = per_g.get(short, 0.0) + max(0.0, t0 - prev)
            prev = max(prev, t1)
        for k in per_d:
            dur.setdefault(k, []).append(per_d[k])
            gap.setdefault(k, []).append(per_g[k])
            seen[k] = seen.get(k, 0) + 1
        spans.append(w["t1"] - w["t0"])
        busy.append(sum(t1 - t0 for _, t0, t1 in w["events"]))
    n = len(windows)
    print(f"  {n} windows, span {np.mean(spans):7.1f} us (min {min(spans):.1f} max {max(spans):.1f}), "
          f"device busy {np.mean(busy):7.1f} us, idle {np.mean(spans) - np.mean(busy):7.1f} us")
    print(f"    {'event (first-seen order)':44s} {'mean us':>8s} {'gap before':>10s}  in windows")
    for k in order:
        # means over all windows: an event that is missing from a window counts as 0 there
        d = sum(dur[k]) / n
        g = sum(gap[k]) / n
        print(f"    {k:44s} {d:8.2f} {g:10.2f}  {seen[k]}/{n}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("scene", nargs="?", default="pyramid", choices=["pyramid", "field", "tumbler"])
    ap.add_argument("--warmup", type=int, default=12)
    ap.add_argument("--steps", type=int, default=40)
    args = ap.parse_args()
    assert args.warmup >= 10 and args.steps >= 20

    import torch
    from torch.profiler import ProfilerActivity, profile
    from solver2d_b200 import capi, device, scenes

    torch.cuda.init()
    P = capi.Solver2D(device.LIB_PATH)
    dev = device.Device()
    if args.scene == "pyramid":
        sc = scenes.pyramid(P, "TGS_Soft", base_count=447)
    elif args.scene == "field":
        sc = scenes.pyramid_field(P, "TGS_Soft", count=256, base_count=45)
    else:
        sc = scenes.tumbler(P, "TGS_Soft", grid=100)
    dw = device.DeviceWorld.attach(dev, sc.world)
    for _ in range(args.warmup):
        sc.step(1 / 60, 4, 2, True)
    dw.sync()
    c0 = dw.counters()
    moved = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            sc.step(1 / 60, 4, 2, True)
            dw.sync()
            moved.append(dw.counters().movedCount)
    c1 = dw.counters()
    events = sorted((e.time_range.start, e.time_range.end, e.name) for e in prof.events()
                    if e.device_type == torch.autograd.DeviceType.CUDA)
    print(f"scene {args.scene}: {torch.cuda.get_device_name()}, {args.steps} steps after {args.warmup} warm-up")
    passes = c1.pairPassCount - c0.pairPassCount
    print(f"  moved proxies per step {np.mean(moved):.0f} (min {min(moved)} max {max(moved)}); pair passes {passes}; "
          f"contacts {c1.contactCount}; shapes {c1.shapeCapacity}")
    report(tail_windows(events))
    sc.destroy()


if __name__ == "__main__":
    main()
