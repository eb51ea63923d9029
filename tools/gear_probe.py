"""Step time of a large gear-train world against the same world with each gear replaced by a revolute stand-in (DESIGN.md
§3.19), on the GPU.

Both worlds are scenes.gears with `copies` copies side by side (15 bodies and 7 gears each, and a sun with 52 planets on the first
copy; 300 copies is 4 554 bodies and 2 152 gears): the gear world with real gears, the stand-in world (stand_ins=True)
with a revolute joint between the same two bodies in each gear's place. The two hold the same bodies, shapes and joint
graph, so they colour alike at the start; what the comparison isolates is the gear row's solve against the revolute
row's. It does not isolate that alone: the stand-in pins each pair together, so the bodies move differently, and the
contact count and later colourings drift apart; both are reported. The worlds are timed in alternated rounds (s2World_TimedSteps: CUDA events
around each step, the L2 flushed between steps) under TGS_Soft, PGS, TGS_NGS and XPBD. Prints one JSON line with the card
name, power limit and maximum SM clock.

    python tools/gear_probe.py [--copies 300] [--steps 60] [--warmup 30] [--rounds 3] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from solver2d_b200 import capi, device, scenes  # noqa: E402
from wheel_probe import _gpu, _timer  # noqa: E402

DT = 1.0 / 60.0
VARIANTS = ["TGS_Soft", "PGS", "TGS_NGS", "XPBD"]


def _measure(P, dev, solver, copies, steps, warmup, rounds):
    timed = _timer(P)
    worlds = {}
    for kind in ("gear", "stand_in"):
        sc = scenes.gears(P, solver, copies=copies, stand_ins=kind == "stand_in")
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
        c = device.DeviceWorld.attach(dev, sc.world).counters()
        res[kind] = {"bodies": len(sc.bodies), "joints": len(sc.joints), "contacts": int(c.constraintCount),
                     "colours": int(c.groupCount), "step_ms": ms[kind]}
        sc.destroy()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--copies", type=int, default=300)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/gear_probe.json")
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
        with open(os.path.join(args.out, "gear_probe.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
