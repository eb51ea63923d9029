"""Step time with and without bullets (DESIGN.md §3.12), through the public API: CUDA events on the world's stream
(s2World_TimedSteps), continuous collision on throughout. Two workloads:

* idle cost: the bench's headline scene, one TGS_Soft pyramid of base 447 (100 128 boxes), settling, plus one dynamic
  box at rest away from the pile. That box is flagged a bullet and cleared again every window of steps, so both sets of
  windows see the same, slowly settling scene. Flagged, every step adds the bullet pass's refit and launches; nothing is
  fast, so nothing is swept. Medians and the 10th / 90th percentiles of the windows' per-step time;
* K bullets fired into that pile once it has settled: each window adds K circles at 150 m/s, each 2 m left of a row of
  the pile, flagged in every other window, and times the steps in which they reach the pile; the bullets are then
  destroyed and the pile settles for a few untimed steps. Medians and percentiles as above.

Prints the card's name, power limit and maximum SM clock with the numbers. Usage:
python tools/bullet_probe.py [--windows N] [--window S] [--warmup W] [--base B] [--bullets K] [--flight F] [--settle S]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from continuous_probe import card  # noqa: E402
from solver2d_b200 import capi, device, scenes  # noqa: E402


def _body(P, world, x, y, vx, radius=None):
    bd = capi.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    bd.position = capi.Vec2(x, y)
    bd.linearVelocity = capi.Vec2(vx, 0.0)
    bd.gravityScale = 0.0
    bid = P.s2CreateBody(world, C.byref(bd))
    if radius is None:
        P.s2CreatePolygonShape(bid, C.byref(capi.default_shape_def()), C.byref(P.s2MakeBox(0.5, 0.5)))
    else:
        P.s2CreateCircleShape(bid, C.byref(capi.default_shape_def()), C.byref(capi.Circle(capi.Vec2(0.0, 0.0), radius)))
    return bid


def idle(P, dev, args, results):
    sc = scenes.pyramid(P, "TGS_Soft", base_count=args.base)
    P.s2World_EnableContinuous(sc.world, True)
    lone = _body(P, sc.world, 0.0, 2.0 * args.base + 50.0, 0.0)
    dw = device.DeviceWorld.attach(dev, sc.world)
    for _ in range(args.warmup):
        sc.step()
    times = {False: [], True: []}
    for k in range(2 * args.windows):
        on = k % 2 == 1
        P.s2Body_SetBullet(lone, on)
        times[on].append(P.s2World_TimedSteps(sc.world, args.window, 1.0 / 60.0, 4, 2, True, 0) / args.window)
        if on:
            assert dw.counters().bulletShapes == 0
    name = f"pyramid{args.base}_one_idle_bullet"
    for on in (False, True):
        t = np.array(times[on])
        results[f"{name}_{'flagged' if on else 'clear'}_ms"] = {"median": round(float(np.median(t)), 4),
                                                               "p10": round(float(np.percentile(t, 10)), 4),
                                                               "p90": round(float(np.percentile(t, 90)), 4)}
    sc.destroy()


def fired(P, dev, args, results):
    """K bullets fired into the bench's pile once it has settled for --warmup steps: every window creates K circles 2 m
    left of the pile's rows at 150 m/s, flagged in odd windows, times the --flight steps in which they reach the pile, then
    destroys them and lets the pile settle for --settle untimed steps. Both kinds of window pay the same uploads and tree
    rebuild for the new bodies; the flagged ones add the bullet pass with K fast bullets."""
    h = 0.5  # the pyramid's box half size
    sc = scenes.pyramid(P, "TGS_Soft", base_count=args.base)
    P.s2World_EnableContinuous(sc.world, True)
    dw = device.DeviceWorld.attach(dev, sc.world)
    for _ in range(args.warmup):
        sc.step()
    times = {False: [], True: []}
    shapes = hits = 0
    for k in range(2 * args.windows):
        on = k % 2 == 1
        bids = []
        for n in range(args.bullets):
            # row i of the pile starts at x = (i + 1) h - h base: each bullet 2 m left of its row, rows up to 80 % high
            i = int(0.8 * args.base * n / args.bullets)
            bid = _body(P, sc.world, (i + 1) * h - h * args.base - 2.0, (2 * i + 1) * h, 150.0, radius=0.1)
            P.s2Body_SetBullet(bid, on)
            bids.append(bid)
        ms = 0.0
        for _ in range(args.flight):
            ms += P.s2World_TimedSteps(sc.world, 1, 1.0 / 60.0, 4, 2, True, 0)
            if on:
                c = dw.counters()
                shapes, hits = max(shapes, c.bulletShapes), max(hits, c.bulletHits)
        times[on].append(ms / args.flight)
        for bid in bids:
            P.s2DestroyBody(bid)
        for _ in range(args.settle):
            sc.step()
    name = f"pyramid{args.base}_{args.bullets}_bullets_fired"
    for on in (False, True):
        t = np.array(times[on])
        results[f"{name}_{'flagged' if on else 'clear'}_ms"] = {"median": round(float(np.median(t)), 4),
                                                               "p10": round(float(np.percentile(t, 10)), 4),
                                                               "p90": round(float(np.percentile(t, 90)), 4)}
    results["fired_max_bullet_shapes_per_step"] = shapes
    results["fired_max_bullet_hits_per_step"] = hits
    sc.destroy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=20)
    ap.add_argument("--window", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=60)
    ap.add_argument("--base", type=int, default=447)
    ap.add_argument("--bullets", type=int, default=64)
    ap.add_argument("--flight", type=int, default=2)
    ap.add_argument("--settle", type=int, default=5)
    args = ap.parse_args()
    dev = device.Device()
    P = capi.Solver2D(device.LIB_PATH)
    P.s2World_TimedSteps = P.lib.s2World_TimedSteps
    P.s2World_TimedSteps.restype = C.c_float
    P.s2World_TimedSteps.argtypes = [capi.WorldId, C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_bool, C.c_int32]
    print("card:", card())
    results = {}
    idle(P, dev, args, results)
    fired(P, dev, args, results)
    print(json.dumps(results))


if __name__ == "__main__":
    main()
