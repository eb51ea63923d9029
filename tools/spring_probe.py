"""Step time of scenes.springs with its joint springs on and off (DESIGN.md §3.14), on the GPU, and of SURVEY §8d config 4
(scenes.joint_contact_stress: 4 025 revolute joints under a grid of boxes, no springs).

About 10 000 bodies of springs (340 copies of the scene). Each variant builds the scene twice and switches every spring off
in the second (s2RevoluteJoint_EnableSpring / s2PrismaticJoint_EnableSpring), so the two worlds have the same bodies,
joints, limits and motors. The two are timed alternately (s2World_TimedSteps: CUDA events around each step, the L2
flushed between steps), for TGS_Soft (soft form) and one variant of each other form: PGS (Baumgarte), TGS_NGS (rigid
velocity) and XPBD. Config 4 is timed under TGS_Soft and PGS_NGS; with --root it times another built checkout's library,
so that a parent and a change can be compared in one session. Prints one JSON line with the card name, power limit and
maximum SM clock.

    python tools/spring_probe.py [--copies 340] [--steps 60] [--warmup 30] [--out DIR]
    python tools/spring_probe.py --config4-only --root OTHER_CHECKOUT   # config 4 on another built checkout's library
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
    for kind in ("springs_on", "springs_off"):
        sc = scenes.springs(P, solver, copies=copies)
        if kind == "springs_off":
            for k, _, _ in sc.piles["springs"]:
                # each setter ignores a joint of the other type
                P.s2RevoluteJoint_EnableSpring(sc.joints[k], False)
                P.s2PrismaticJoint_EnableSpring(sc.joints[k], False)
        for _ in range(warmup):
            sc.step(DT, 4, 2, True)
        worlds[kind] = sc
    ms = {kind: [] for kind in worlds}
    chunk = max(steps // rounds, 1)
    for _ in range(rounds):
        for kind in worlds:
            ms[kind].append(float(timed(worlds[kind].world, chunk, DT, 4, 2, True, 1)) / chunk)
    res = {f"{kind}_ms": ms[kind] for kind in worlds}
    res["bodies"] = len(worlds["springs_on"].bodies)
    res["joints"] = len(worlds["springs_on"].joints)
    res["springs"] = len(worlds["springs_on"].piles["springs"])
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
    ap.add_argument("--copies", type=int, default=340)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--config4-only", action="store_true", help="time config 4 only")
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    help="the built checkout whose library and scenes are timed (default: this one)")
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/spring_probe.json")
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
        with open(os.path.join(args.out, "spring_probe.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
