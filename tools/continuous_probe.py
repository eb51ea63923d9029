"""Step time with continuous collision off and on (DESIGN.md §3.11), through the public API: CUDA events on the world's
stream (s2World_TimedSteps). Two workloads:

* the bench's headline scene, one TGS_Soft pyramid of base 447 (100 128 boxes), settling: nothing is fast, so the
  difference is the cost of the idle passes (snapshot, classify, an empty sweep launch, clamp);
* a field of about 10 k projectiles (scenes.projectiles with copies), all fast in their first steps: the sweep's cost.

The pyramid is one world whose feature is switched off and on every window of steps (the switch takes effect at the next
step and re-captures nothing), so that both sets of windows see the same, slowly settling scene; medians and the 10th /
90th percentiles of the per-step time of the windows are printed. The projectiles get a fresh world per
window, off and on alternating, each timed over its first three steps. Prints the card's name and power limit
with the numbers. Usage: python tools/continuous_probe.py [--windows N] [--window S] [--warmup W] [--repeats R] [--base B]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from solver2d_b200 import capi, device, scenes  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return out


def alternate(P, dev, sc, windows, window, warmup, results, name):
    """After `warmup` steps, 2 * `windows` windows of `window` steps with the feature switched off and on window by window
    (the switch takes effect at the next step and re-captures nothing): both sets of windows see the same, slowly settling
    scene. Device time per step of every window; medians and the 10th / 90th percentiles."""
    dw = device.DeviceWorld.attach(dev, sc.world)
    for _ in range(warmup):
        sc.step()
    times = {False: [], True: []}
    swept = 0
    for k in range(2 * windows):
        on = k % 2 == 1
        P.s2World_EnableContinuous(sc.world, on)
        times[on].append(P.s2World_TimedSteps(sc.world, window, 1.0 / 60.0, 4, 2, True, 0) / window)
        if on:
            swept = max(swept, dw.counters().continuousShapes)
    for on in (False, True):
        t = np.array(times[on])
        results[f"{name}_{'on' if on else 'off'}_ms"] = {"median": round(float(np.median(t)), 4),
                                                         "p10": round(float(np.percentile(t, 10)), 4),
                                                         "p90": round(float(np.percentile(t, 90)), 4)}
    results[f"{name}_swept_shapes_last_window"] = swept
    results[f"{name}_bodies"] = dw.counters().bodyCapacity


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=20)
    ap.add_argument("--window", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=60)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--base", type=int, default=447)
    args = ap.parse_args()
    dev = device.Device()
    P = capi.Solver2D(device.LIB_PATH)
    P.s2World_TimedSteps = P.lib.s2World_TimedSteps
    P.s2World_TimedSteps.restype = C.c_float
    P.s2World_TimedSteps.argtypes = [capi.WorldId, C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_bool, C.c_int32]
    print("card:", card())
    results = {}
    sc = scenes.pyramid(P, "TGS_Soft", base_count=args.base)
    alternate(P, dev, sc, args.windows, args.window, args.warmup, results, f"pyramid{args.base}")
    sc.destroy()
    # projectiles: 84 x 120 = 10 080, fast in their first steps only, so a fresh world per window (off, on, off, on ...)
    for _ in range(args.repeats):
        for on in (False, True):
            sc = scenes.projectiles(P, "TGS_Soft", copies=84, excluded=False)
            P.s2World_EnableContinuous(sc.world, on)
            ms = P.s2World_TimedSteps(sc.world, 3, 1.0 / 60.0, 4, 2, True, 0) / 3
            results.setdefault(f"projectiles_first3_{'on' if on else 'off'}_ms", []).append(round(ms, 4))
            if on:
                c = device.DeviceWorld.attach(dev, sc.world).counters()
                results["projectiles_swept_shapes_last_step"] = c.continuousShapes
                results["projectiles_clamped_last_step"] = c.continuousHits
            sc.destroy()
    print(json.dumps(results))


if __name__ == "__main__":
    main()
