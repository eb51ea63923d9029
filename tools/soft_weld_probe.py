"""Step time of scenes.soft_welds with its soft welds soft and with every hertz set to 0 (DESIGN.md §3.15), on the GPU, and of
SURVEY §8d config 4 (scenes.joint_contact_stress: 4 025 revolute joints under a grid of boxes, no welds).

About 10 000 bodies of soft_welds (295 copies of the scene). Each variant builds the scene twice and sets every hertz of
every soft weld to 0 in the second (s2WeldJoint_SetLinearHertz / _SetAngularHertz), so the two worlds have the same bodies
and joints, rigid welds in the second. The two are timed alternately (s2World_TimedSteps: CUDA events around each step, the L2
flushed between steps), for TGS_Soft (soft form) and one variant of each other form: PGS (Baumgarte), TGS_NGS (rigid
velocity) and XPBD. Config 4 is timed under TGS_Soft and PGS_NGS; with --root it times another built checkout's library,
so that a parent and a change can be compared in one session. Prints one JSON line with the card name, power limit and
maximum SM clock.

    python tools/soft_weld_probe.py [--copies 295] [--steps 60] [--warmup 30] [--out DIR]
    python tools/soft_weld_probe.py --config4-only --root OTHER_CHECKOUT   # config 4 on another built checkout's library
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

DT = 1.0 / 60.0
VARIANTS = ["TGS_Soft", "PGS", "TGS_NGS", "XPBD"]
CONFIG4_VARIANTS = ["TGS_Soft", "PGS_NGS"]


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
    for kind in ("soft", "rigid"):
        sc = scenes.soft_welds(P, solver, copies=copies)
        if kind == "rigid":
            for k, *_ in sc.piles["soft_welds"]:
                P.s2WeldJoint_SetLinearHertz(sc.joints[k], 0.0)
                P.s2WeldJoint_SetAngularHertz(sc.joints[k], 0.0)
        for _ in range(warmup):
            sc.step(DT, 4, 2, True)
        worlds[kind] = sc
    ms = {kind: [] for kind in worlds}
    chunk = max(steps // rounds, 1)
    for _ in range(rounds):
        for kind in worlds:
            ms[kind].append(float(timed(worlds[kind].world, chunk, DT, 4, 2, True, 1)) / chunk)
    res = {f"{kind}_ms": ms[kind] for kind in worlds}
    res["bodies"] = len(worlds["soft"].bodies)
    res["joints"] = len(worlds["soft"].joints)
    res["soft_welds"] = len(worlds["soft"].piles["soft_welds"])
    for sc in worlds.values():
        sc.destroy()
    return res


def _config4(P, solver, steps, warmup, rounds=3):
    timed = _timer(P)
    sc = scenes.joint_contact_stress(P, solver)
    for _ in range(warmup):
        sc.step(DT, 4, 2, True)
    chunk = max(steps // rounds, 1)
    ms = [float(timed(sc.world, chunk, DT, 4, 2, True, 1)) / chunk for _ in range(rounds)]
    res = {"ms": ms, "bodies": len(sc.bodies), "joints": len(sc.joints)}
    sc.destroy()
    return res


def main():
    global capi, device, scenes
    ap = argparse.ArgumentParser()
    ap.add_argument("--copies", type=int, default=295)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--config4-only", action="store_true", help="time config 4 only")
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    help="the built checkout whose library and scenes are timed (default: this one)")
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/soft_weld_probe.json")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    from solver2d_b200 import capi, device, scenes  # noqa: E402

    P = capi.Solver2D(device.LIB_PATH)
    result = {"gpu": _gpu(), "root": os.path.abspath(args.root)}
    if not args.config4_only:
        for solver in VARIANTS:
            result[solver] = _measure(P, solver, args.copies, args.steps, args.warmup)
    result["config4"] = {solver: _config4(P, solver, args.steps, args.warmup) for solver in CONFIG4_VARIANTS}
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "soft_weld_probe.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
