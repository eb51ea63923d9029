"""Step time of cars on wheel joints against the same cars built the scenes.springs way (DESIGN.md §3.17), on the GPU.

Each world holds `copies` cars side by side on a flat ground with bumps. A car is a chassis and two circular wheels on
suspension springs (axis up, 4 Hz, damping ratio 0.7, limits +/- 0.25 m) with a motorised rear wheel (-8 rad/s,
12 N-m). The wheel-joint car joins each wheel to the chassis with one wheel joint; the emulated car puts an axle body
between them, a prismatic spring from the chassis to the axle and a revolute joint (carrying the motor) from the axle to
the wheel. The two worlds are timed in alternated rounds (s2World_TimedSteps: CUDA events around each step, the L2
flushed between steps) under TGS_Soft, PGS, TGS_NGS and XPBD. For each world it reports bodies, joints, colours (colour
schedule) and step time. Prints one JSON line with the card name, power limit and maximum SM clock.

    python tools/wheel_probe.py [--copies 2000] [--steps 60] [--warmup 30] [--rounds 3] [--out DIR]
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
from solver2d_b200.capi import Circle, Vec2  # noqa: E402

DT = 1.0 / 60.0
VARIANTS = ["TGS_Soft", "PGS", "TGS_NGS", "XPBD"]
PITCH = 4.0  # m between cars


def _gpu():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def _timer(P):
    L = P.lib
    L.s2World_TimedSteps.restype = C.c_float
    L.s2World_TimedSteps.argtypes = [capi.WorldId, C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_bool, C.c_int32]
    return L.s2World_TimedSteps


def _cars(P, solver, copies, emulated):
    world = P.create_world(solver)
    sc = scenes.Scene(P, world, name=f"cars{copies}")
    sc.bodies.append(scenes._ground(P, world, 0.5 * PITCH * copies + 5.0))

    def body(kind, x, y, hx=0.5, hy=0.1, radius=None, group=0):
        bd = capi.default_body_def()
        bd.type = kind
        bd.position = Vec2(x, y)
        bid = P.s2CreateBody(world, C.byref(bd))
        sd = capi.default_shape_def()
        sd.filter.groupIndex = group
        if radius is not None:
            P.s2CreateCircleShape(bid, C.byref(sd), C.byref(Circle(Vec2(0.0, 0.0), radius)))
        else:
            P.s2CreatePolygonShape(bid, C.byref(sd), C.byref(P.s2MakeBox(hx, hy)))
        sc.bodies.append(bid)
        return bid

    for k in range(copies):
        x0 = -0.5 * PITCH * (copies - 1) + PITCH * k
        body(capi.STATIC_BODY, x0 + 1.8, 0.05, hx=0.3, hy=0.05)
        group = -(k + 1)
        chassis = body(capi.DYNAMIC_BODY, x0, 1.3, hx=1.2, hy=0.2, group=group)
        for dx, motor in ((-0.9, True), (0.9, False)):
            pivot = Vec2(x0 + dx, 0.7)
            tyre = body(capi.DYNAMIC_BODY, pivot.x, pivot.y, radius=0.4, group=group)
            if not emulated:
                jd = capi.default_wheel_def()
                jd.bodyIdA, jd.bodyIdB = chassis, tyre
                jd.localAnchorA, jd.localAnchorB = P.s2Body_GetLocalPoint(chassis, pivot), Vec2(0.0, 0.0)
                jd.hertz, jd.dampingRatio = 4.0, 0.7
                jd.enableLimit, jd.lowerTranslation, jd.upperTranslation = True, -0.25, 0.25
                jd.enableMotor, jd.motorSpeed, jd.maxMotorTorque = motor, -8.0, 12.0
                sc.joints.append(P.s2CreateWheelJoint(world, C.byref(jd)))
                continue
            axle = body(capi.DYNAMIC_BODY, pivot.x, pivot.y, hx=0.1, hy=0.1, group=group)
            pd = capi.default_prismatic_def()
            pd.bodyIdA, pd.bodyIdB = chassis, axle
            pd.localAnchorA, pd.localAnchorB = P.s2Body_GetLocalPoint(chassis, pivot), Vec2(0.0, 0.0)
            pd.localAxisA = Vec2(0.0, 1.0)
            pd.enableSpring, pd.hertz, pd.dampingRatio = True, 4.0, 0.7
            pd.enableLimit, pd.lowerTranslation, pd.upperTranslation = True, -0.25, 0.25
            sc.joints.append(P.s2CreatePrismaticJoint(world, C.byref(pd)))
            rd = capi.default_revolute_def()
            rd.bodyIdA, rd.bodyIdB = axle, tyre
            rd.localAnchorA, rd.localAnchorB = Vec2(0.0, 0.0), Vec2(0.0, 0.0)
            rd.enableMotor, rd.motorSpeed, rd.maxMotorTorque = motor, -8.0, 12.0
            sc.joints.append(P.s2CreateRevoluteJoint(world, C.byref(rd)))
    return sc


def _measure(P, dev, solver, copies, steps, warmup, rounds):
    timed = _timer(P)
    worlds = {}
    for kind in ("wheel", "emulated"):
        sc = _cars(P, solver, copies, kind == "emulated")
        for _ in range(warmup):
            sc.step(DT, 4, 2, True)
        worlds[kind] = sc
    ms = {kind: [] for kind in worlds}
    chunk = max(steps // rounds, 1)
    for _ in range(rounds):
        for kind in worlds:
            ms[kind].append(float(timed(worlds[kind].world, chunk, DT, 4, 2, True, 1)) / chunk)
    res = {}
    for kind, sc in worlds.items():
        dw = device.DeviceWorld.attach(dev, sc.world)
        res[kind] = {"bodies": len(sc.bodies), "joints": len(sc.joints), "colours": int(dw.counters().groupCount),
                     "step_ms": ms[kind]}
        sc.destroy()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--copies", type=int, default=2000)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/wheel_probe.json")
    args = ap.parse_args()
    P = capi.Solver2D(device.LIB_PATH)
    dev = device.Device()
    result = {"gpu": _gpu(), "copies": args.copies}
    for solver in VARIANTS:
        result[solver] = _measure(P, dev, solver, args.copies, args.steps, args.warmup, args.rounds)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "wheel_probe.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
