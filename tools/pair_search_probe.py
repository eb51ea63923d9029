"""GPU box: device time of every kernel of the broad-phase pair search (bpSearch in csrc/device/broadphase.cu), per pass.

    python tools/pair_search_probe.py [pyramid|field|tumbler] [--warmup 12] [--steps 48]

Runs the bench workload (TGS_Soft, dt = 1/60, 4 sub-steps, 2 relax iterations) on the chosen scene: `pyramid` is the
100 128-box pyramid of base 447, `field` the bench's config 5 (256 piles of 1 035 boxes in one world), `tumbler` the
hub container of 100 x 100 boxes with four scene-sized walls (large movers). After the warm-up it records the steps
under torch.profiler (CUDA activities), splits the kernel stream into pair-search passes and prints the mean device
time of each kernel, apart for passes that rebuild the hierarchy and passes that only refit it. Also printed: the
"pairs" stage time of the last step (stage_ms()[0]), the moved-proxy count and the binary tree height.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# kernels of a pair-search pass, in launch order; the cub kernels of the Morton sort and the leaf selection run between
# s2bFlagValidShapes and the tree build. On a pass that reuses the hierarchy, the refit and the moved proxies ran inside
# finalize (s2bFinalizeRefitKernel, which also finalizes the shapes); the query launch s2bFindPairs also holds the survivor
# and large-mover scans.
SEARCH_PREFIXES = ("s2bFlagValidShapes", "s2bSceneBounds", "s2bMortonCodes", "s2bBuildRadixTree", "s2bBuildWide",
                   "s2bFinalizeRefitKernel", "s2bRefit", "s2bBuildPairHash", "s2bCollectMovers", "s2bFindPairs")


def _short(name: str) -> str:
    for p in SEARCH_PREFIXES:
        if name.startswith(p) or name.startswith("void " + p):
            return p
    return name.split("(")[0].replace("void ", "")[:60]


def collect_passes(kernels):
    """kernels: [(start_us, end_us, name)] sorted by start. A pass opens at s2bFlagValidShapes (rebuild) or at a refit
    kernel (s2bRefit, s2bFinalizeRefitKernel) that is not preceded by a build in the same pass, and closes at s2bFindPairs."""
    passes, cur, in_build = [], None, False
    for t0, t1, name in kernels:
        short = _short(name)
        if short == "s2bFlagValidShapes":
            cur = {"kernels": [], "rebuild": True, "t0": t0}
            in_build = True
        elif short in ("s2bRefit", "s2bFinalizeRefitKernel") and (cur is None or not in_build):
            cur = {"kernels": [], "rebuild": False, "t0": t0}
        if cur is None:
            continue
        if short in SEARCH_PREFIXES or in_build:
            cur["kernels"].append((short, t1 - t0))
            cur["t1"] = t1
        if short.startswith("s2bRefit"):
            in_build = False
        if short == "s2bFindPairs":
            passes.append(cur)
            cur = None
    return passes


def report(passes, label):
    if not passes:
        print(f"  {label}: none")
        return
    per = {}
    for p in passes:
        seen = {}
        for short, d in p["kernels"]:
            seen[short] = seen.get(short, 0.0) + d
        for k, v in seen.items():
            per.setdefault(k, []).append(v)
    total = [sum(d for _, d in p["kernels"]) for p in passes]
    span = [p["t1"] - p["t0"] for p in passes]
    print(f"  {label}: {len(passes)} passes, kernel sum {np.mean(total):7.1f} us (min {min(total):.1f} max {max(total):.1f}), "
          f"first-to-last kernel span {np.mean(span):7.1f} us")
    for k, v in sorted(per.items(), key=lambda kv: -np.mean(kv[1])):
        print(f"    {k:40s} {np.mean(v):7.2f} us  (min {min(v):6.2f} max {max(v):6.2f}, in {len(v)} passes)")
    tree = sum(np.mean(per.get(k, [0.0])) for k in ("s2bRefit", "s2bFinalizeRefitKernel", "s2bFindPairs"))
    print(f"    refit + queries (s2bRefit or s2bFinalizeRefitKernel, which finalizes the shapes too, + s2bFindPairs): {tree:.1f} us per pass")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("scene", nargs="?", default="pyramid", choices=["pyramid", "field", "tumbler"])
    ap.add_argument("--warmup", type=int, default=12)
    ap.add_argument("--steps", type=int, default=48)
    args = ap.parse_args()
    assert args.warmup >= 10 and args.steps >= 30

    import torch
    from torch.profiler import ProfilerActivity, profile
    from solver2d_b200 import capi, device, scenes

    torch.cuda.init()
    P = capi.Solver2D(device.LIB_PATH)
    dev = device.Device()
    if args.scene == "pyramid":
        sc = scenes.pyramid(P, "TGS_Soft", base_count=447)
    elif args.scene == "field":
        sc = scenes.pyramid_field(P, "TGS_Soft", count=256, base_count=45)
    else:
        sc = scenes.tumbler(P, "TGS_Soft", grid=100)
    dw = device.DeviceWorld.attach(dev, sc.world)
    for _ in range(args.warmup):
        sc.step(1 / 60, 4, 2, True)
    dw.sync()
    moved, pairs_ms = [], []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            sc.step(1 / 60, 4, 2, True)
            dw.sync()
            pairs_ms.append(dw.stage_ms()[0])
            moved.append(dw.counters().movedCount)
    kernels = []
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            kernels.append((e.time_range.start, e.time_range.end, e.name))
    kernels.sort()
    passes = collect_passes(kernels)
    c = dw.counters()
    print(f"scene {args.scene}: {torch.cuda.get_device_name()}, {args.steps} steps after {args.warmup} warm-up")
    print(f"  stage_ms()[0] (pairs) last step {pairs_ms[-1]:.4f} ms, mean {np.mean(pairs_ms):.4f} ms over the recorded steps")
    print(f"  moved proxies (counters().movedCount) last step {c.movedCount}, mean {np.mean(moved):.0f}; "
          f"treeHeight {c.treeHeight}; shapes {c.shapeCapacity}; contacts {c.contactCount}")
    report([p for p in passes if not p["rebuild"]], "refit-only passes")
    report([p for p in passes if p["rebuild"]], "rebuild passes")
    allp = [sum(d for _, d in p["kernels"]) for p in passes]
    if allp:
        print(f"  all passes: {len(allp)}, mean kernel sum {np.mean(allp):.1f} us")
    sc.destroy()


if __name__ == "__main__":
    main()
