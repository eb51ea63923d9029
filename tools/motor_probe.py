"""Two timings of the motor joint (DESIGN.md §3.10) on the GPU.

1. Step time of scenes.motors at about 10 000 bodies (525 copies: 9 976 bodies and 5 776 joints, 5 775 of them motor
   joints) with motor joints and with their revolute stand-ins, timed alternately with s2World_TimedSteps (CUDA events around each step, the L2 flushed
   between steps), under TGS_Soft, PGS, TGS_NGS and XPBD.
2. Per-frame wall time of re-targeting every motor joint of the same scene and stepping it, under TGS_Soft: through the
   per-joint setters (s2MotorJoint_SetLinearOffset + _SetAngularOffset) against one s2World_SetMotorJointOffsets call.
   Each frame ends with a stream synchronisation, so the time is what a client loop sees.

Prints one JSON line with the card name, power limit and maximum SM clock.

    python tools/motor_probe.py [--copies 525] [--steps 60] [--warmup 30] [--frames 30] [--out DIR]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import time

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


def _measure(libs, solver, copies, steps, warmup, rounds=3):
    timed = _timer(libs["motor"])
    worlds = {}
    for kind, P in libs.items():
        sc = scenes.motors(P, solver, copies=copies)
        for _ in range(warmup):
            sc.step(DT, 4, 2, True)
        worlds[kind] = sc
    ms = {kind: [] for kind in libs}
    chunk = max(steps // rounds, 1)
    for _ in range(rounds):
        for kind in libs:
            ms[kind].append(float(timed(worlds[kind].world, chunk, DT, 4, 2, True, 1)) / chunk)
    res = {f"{kind}_ms": ms[kind] for kind in libs}
    res["bodies"] = len(worlds["motor"].bodies)
    res["joints"] = len(worlds["motor"].joints)
    res["motor_joints"] = len(worlds["motor"].piles["motor"])
    for sc in worlds.values():
        sc.destroy()
    return res


def _retarget(P, copies, frames, warmup):
    """Per-frame wall time (ms) of re-targeting every motor joint and stepping, per-joint setters against the bulk call."""
    dw_sync = P.lib.s2b_sync
    dw_sync.argtypes = [C.c_void_p]
    get_device = P.lib.s2World_GetDevice
    get_device.restype = C.c_void_p
    get_device.argtypes = [capi.WorldId]
    res = {}
    for kind in ("setters", "bulk"):
        sc = scenes.motors(P, "TGS_Soft", copies=copies)
        handle = get_device(sc.world)
        ids = [sc.joints[k] for k in sc.piles["motor"]]
        slots = np.array([j.index for j in ids], dtype=np.int32)
        base = np.array([(d["linearOffset"][0], d["linearOffset"][1], d["angularOffset"]) for d in sc.piles["motor_defs"]],
                        dtype=np.float32)
        times = []
        for frame in range(warmup + frames):
            offsets = base.copy()
            offsets[:, 0] += np.float32(0.01 * math.sin(0.1 * frame))
            t0 = time.perf_counter()
            if kind == "setters":
                for jid, (x, y, a) in zip(ids, offsets):
                    P.s2MotorJoint_SetLinearOffset(jid, capi.Vec2(float(x), float(y)))
                    P.s2MotorJoint_SetAngularOffset(jid, float(a))
            else:
                P.s2World_SetMotorJointOffsets(sc.world, slots.ctypes.data, offsets.ctypes.data, len(slots))
            sc.step(DT, 4, 2, True)
            dw_sync(handle)
            if frame >= warmup:
                times.append(1e3 * (time.perf_counter() - t0))
        res[f"{kind}_ms"] = [float(np.median(times)), float(np.min(times)), float(np.max(times))]
        res["motor_joints"] = len(ids)
        sc.destroy()
    return res


def main():
    global capi, device, scenes, np
    ap = argparse.ArgumentParser()
    ap.add_argument("--copies", type=int, default=525)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/motor_probe.json")
    args = ap.parse_args()
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import numpy as np  # noqa: E402
    from solver2d_b200 import capi, device, scenes  # noqa: E402

    P = capi.Solver2D(device.LIB_PATH)
    standin = capi.Solver2D(device.LIB_PATH)
    standin.missing.append("s2CreateMotorJoint")  # the scene then builds its revolute stand-ins
    result = {"gpu": _gpu()}
    for solver in VARIANTS:
        result[solver] = _measure({"motor": P, "standin": standin}, solver, args.copies, args.steps, args.warmup)
    result["retarget"] = _retarget(P, args.copies, args.frames, 5)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "motor_probe.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
