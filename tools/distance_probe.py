"""Step time of scenes.distance_joints with distance joints and with revolute stand-ins (DESIGN.md §3.16), on the GPU.

About 10 000 bodies (230 copies of the scene). Each variant builds the scene twice: once with its distance joints, once
with every distance joint created as a revolute joint at anchor B's start point (``stand_ins=True``), so the two worlds
have the same bodies, shapes and number of joints. The two are timed alternately (s2World_TimedSteps: CUDA events around
each step, the L2 flushed between steps), for TGS_Soft (soft form) and one variant of each other form: PGS (Baumgarte),
TGS_NGS (rigid velocity) and XPBD. Prints one JSON line with the card name, power limit and maximum SM clock.

    python tools/distance_probe.py [--copies 230] [--steps 60] [--warmup 30] [--out DIR]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from solver2d_b200 import capi, device, scenes  # noqa: E402

DT = 1.0 / 60.0
VARIANTS = ["TGS_Soft", "PGS", "TGS_NGS", "XPBD"]


def _gpu():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def _timer(P):
    L = P.lib
    L.s2World_TimedSteps.restype = C.c_float
    L.s2World_TimedSteps.argtypes = [capi.WorldId, C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_bool, C.c_int32]
    return L.s2World_TimedSteps


def _measure(P, solver, copies, steps, warmup, rounds=3):
    timed = _timer(P)
    worlds = {}
    for kind in ("distance", "stand_ins"):
        sc = scenes.distance_joints(P, solver, copies=copies, stand_ins=kind == "stand_ins")
        for _ in range(warmup):
            sc.step(DT, 4, 2, True)
        worlds[kind] = sc
    ms = {kind: [] for kind in worlds}
    chunk = max(steps // rounds, 1)
    for _ in range(rounds):
        for kind in worlds:
            ms[kind].append(float(timed(worlds[kind].world, chunk, DT, 4, 2, True, 1)) / chunk)
    res = {f"{kind}_ms": ms[kind] for kind in worlds}
    res["bodies"] = len(worlds["distance"].bodies)
    res["joints"] = len(worlds["distance"].joints)
    res["distance_joints"] = len(worlds["distance"].piles["distance"])
    for sc in worlds.values():
        sc.destroy()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--copies", type=int, default=230)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/distance_probe.json")
    args = ap.parse_args()
    P = capi.Solver2D(device.LIB_PATH)
    result = {"gpu": _gpu()}
    for solver in VARIANTS:
        result[solver] = _measure(P, solver, args.copies, args.steps, args.warmup)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "distance_probe.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
