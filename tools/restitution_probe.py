"""Step time with restitution off and on (DESIGN.md §3.7), on the GPU.

* the bench pyramid (base 447, 100 128 boxes) with restitution 0.5 on every shape: a resting pile, so hardly a point
  qualifies and the difference is the fixed cost of the capture and the extra pass;
* scenes.bouncers at about 20 000 shapes: shapes landing from several heights, the pass doing real work.

Each configuration is built twice, restitution off and on, and the two are timed alternately (s2World_TimedSteps: CUDA
events around each step, the L2 flushed between steps). Prints one JSON line with the card name and power limit.

    python tools/restitution_probe.py [--steps 60] [--warmup 30] [--out DIR]
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


def _gpu():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def _measure(P, make, steps, warmup, rounds=3):
    L = P.lib
    L.s2World_TimedSteps.restype = C.c_float
    L.s2World_TimedSteps.argtypes = [capi.WorldId, C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_bool, C.c_int32]
    worlds = {}
    for on in (False, True):
        sc = make(P)
        P.s2World_EnableRestitution(sc.world, on)
        for _ in range(warmup):
            sc.step(DT, 4, 2, True)
        worlds[on] = sc
    ms = {False: [], True: []}
    chunk = max(steps // rounds, 1)
    for _ in range(rounds):
        for on in (False, True):
            ms[on].append(float(L.s2World_TimedSteps(worlds[on].world, chunk, DT, 4, 2, True, 1)) / chunk)
    counters = device.DeviceWorld.attach(device.Device(), worlds[True].world).counters()
    res = {"off_ms": ms[False], "on_ms": ms[True], "contacts": counters.contactCount, "constraints": counters.constraintCount}
    for sc in worlds.values():
        sc.destroy()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/restitution_probe.json")
    args = ap.parse_args()
    P = capi.Solver2D(device.LIB_PATH)
    result = {"gpu": _gpu()}
    result["pyramid447_e0.5"] = _measure(P, lambda L: scenes.pyramid(L, "TGS_Soft", base_count=447, restitution=0.5), args.steps,
                                         args.warmup)
    result["bouncers_20k"] = _measure(P, lambda L: scenes.bouncers(L, "TGS_Soft", columns=200, rows=100), args.steps, args.warmup)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "restitution_probe.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
