"""Two timings of breakable joints (DESIGN.md §3.13) on the GPU.

1. Step time of a field of hanging chains (`--chains` chains of `--links` boxes on revolute joints from a static beam) with a
   break threshold on every joint, set so high that none breaks, against the same field without thresholds, timed
   alternately with s2World_TimedSteps (CUDA events around each step, the L2 flushed between steps), under TGS_Soft and
   PGS. The difference is the reaction pass and the wait for its list at the start of each step.
2. Wall time of one s2World_GetJointReactions call on the same field (it synchronises).

Prints one JSON line with the card name, power limit and maximum SM clock.

    python tools/breakable_probe.py [--chains 1000] [--links 10] [--steps 60] [--warmup 30] [--out DIR]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from solver2d_b200 import capi, device  # noqa: E402

DT = 1.0 / 60.0
VARIANTS = ["TGS_Soft", "PGS"]


def _gpu():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def _field(P, solver, chains, links, thresholds):
    wid = P.create_world(solver)
    bd = capi.default_body_def()
    bd.position = capi.Vec2(0.0, 0.0)
    beam = P.s2CreateBody(wid, C.byref(bd))
    sd = capi.default_shape_def()
    sd.density = 1.0
    joints = []
    for c in range(chains):
        prev, anchor = beam, capi.Vec2(2.0 * c, 0.0)
        for k in range(links):
            bd = capi.default_body_def()
            bd.type = capi.DYNAMIC_BODY
            bd.position = capi.Vec2(2.0 * c, -0.5 - k)
            b = P.s2CreateBody(wid, C.byref(bd))
            P.s2CreatePolygonShape(b, C.byref(sd), C.byref(P.s2MakeBox(0.1, 0.5)))
            jd = capi.default_revolute_def()
            jd.bodyIdA, jd.bodyIdB = prev, b
            jd.localAnchorA, jd.localAnchorB = anchor, capi.Vec2(0.0, 0.5)
            j = P.s2CreateRevoluteJoint(wid, C.byref(jd))
            if thresholds:
                P.s2Joint_SetBreakForce(j, 1e9)
            joints.append(j)
            prev, anchor = b, capi.Vec2(0.0, -0.5)
    return wid, joints


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=1000)
    ap.add_argument("--links", type=int, default=10)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    P = capi.Solver2D(device.LIB_PATH)
    timed = P.lib.s2World_TimedSteps
    timed.restype = C.c_float
    timed.argtypes = [capi.WorldId, C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_bool, C.c_int32]
    res = {"gpu": _gpu(), "chains": a.chains, "links": a.links}
    for solver in VARIANTS:
        worlds = {kind: _field(P, solver, a.chains, a.links, kind == "thresholds")[0] for kind in ("plain", "thresholds")}
        for wid in worlds.values():
            for _ in range(a.warmup):
                P.s2World_Step(wid, DT, 4, 2, True)
        ms = {kind: [] for kind in worlds}
        chunk = max(a.steps // 3, 1)
        for _ in range(3):
            for kind, wid in worlds.items():
                ms[kind].append(float(timed(wid, chunk, DT, 4, 2, True, 1)) / chunk)
        res[solver] = {f"{k}_ms": v for k, v in ms.items()}
        cap = a.chains * a.links + 64
        out = np.zeros((cap, 3), dtype=np.float32)
        wid = worlds["thresholds"]
        P.s2World_GetJointReactions(wid, out.ctypes.data, cap)
        calls = []
        for _ in range(20):
            t0 = time.perf_counter()
            P.s2World_GetJointReactions(wid, out.ctypes.data, cap)
            calls.append((time.perf_counter() - t0) * 1e3)
        res[solver]["get_joint_reactions_ms"] = float(np.median(calls))
        assert not np.isnan(out).any()
        for wid in worlds.values():
            P.s2DestroyWorld(wid)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "breakable_probe.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
