"""Step time of scenes.welded_structures with welds and with their revolute stand-ins (DESIGN.md §3.8), on the GPU.

About 10 000 bodies (330 copies of the scene). Each variant builds the scene twice: once with s2CreateWeldJoint and once
with every weld created as the revolute joint (limits and motor off) the scene uses on a library without welds. The two
are timed alternately (s2World_TimedSteps: CUDA events around each step, the L2 flushed between steps), for TGS_Soft
(soft form) and one variant of each other form: PGS (Baumgarte), TGS_NGS (rigid velocity + NGS position) and XPBD.
Prints one JSON line with the card name and power limit.

    python tools/weld_probe.py [--copies 330] [--steps 60] [--warmup 30] [--out DIR]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from solver2d_b200 import capi, device, scenes  # noqa: E402

DT = 1.0 / 60.0
VARIANTS = ["TGS_Soft", "PGS", "TGS_NGS", "XPBD"]


def _gpu():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def _measure(libs, solver, copies, steps, warmup, rounds=3):
    L = libs["weld"].lib
    L.s2World_TimedSteps.restype = C.c_float
    L.s2World_TimedSteps.argtypes = [capi.WorldId, C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_bool, C.c_int32]
    worlds = {}
    for kind, P in libs.items():
        sc = scenes.welded_structures(P, solver, copies=copies)
        for _ in range(warmup):
            sc.step(DT, 4, 2, True)
        worlds[kind] = sc
    ms = {kind: [] for kind in libs}
    chunk = max(steps // rounds, 1)
    for _ in range(rounds):
        for kind in libs:
            ms[kind].append(float(L.s2World_TimedSteps(worlds[kind].world, chunk, DT, 4, 2, True, 1)) / chunk)
    res = {f"{kind}_ms": ms[kind] for kind in libs}
    res["bodies"] = len(worlds["weld"].bodies)
    res["joints"] = len(worlds["weld"].joints)
    for sc in worlds.values():
        sc.destroy()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--copies", type=int, default=330)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/weld_probe.json")
    args = ap.parse_args()
    weld = capi.Solver2D(device.LIB_PATH)
    standin = capi.Solver2D(device.LIB_PATH)
    standin.missing.append("s2CreateWeldJoint")  # the scene then builds its revolute stand-ins
    result = {"gpu": _gpu()}
    for solver in VARIANTS:
        result[solver] = _measure({"weld": weld, "standin": standin}, solver, args.copies, args.steps, args.warmup)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "weld_probe.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
