"""Regenerate the golden fixtures from the UNMODIFIED reference (needs the reference built into oracle/_ref).

    python tests/golden/make_golden.py          # everything
    python tests/golden/make_golden.py host     # host_reference_sha1.json only

pyramid10_tgs_soft.npz — config 1 (SURVEY §8d): Pyramid baseCount=10, s2_solverTGS_Soft, dt=1/60, 4 sub-steps, 2 relax
iterations, warm starting; per-body origin / rotation / velocity after steps {1, 10, 60, 600}, and for every step the
reference's contact pool order as shape-pair keys (the reference's sequential Gauss-Seidel order, needed to reproduce it
bit for bit with the wavefront schedule).

host_reference_sha1.json — the reference's outputs of the seeded host-function sweeps of tests/test_host_cpu.py (polygon
factories and mass, hull, the nine manifold functions), one truncated sha1 per trial.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref  # noqa: E402
from solver2d_b200 import scenes  # noqa: E402


VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]


def variant_fixture(R, solver, steps=90, marks=(1, 10, 45, 90)):
    """pyramid10_<variant>.npz: the same recipe for every solver variant, 90 steps (the reference's Jacobi has thrown the
    pyramid apart long before that: its fixture simply records that trajectory)."""
    sc = scenes.pyramid(R, solver, base_count=10)
    out = {}
    order_keys, order_offsets = [], [0]
    for step in range(1, steps + 1):
        R.step_collide(sc.world)
        cf, ci = R.contacts(sc.world)
        live = ci[:, 0] == 1
        a, b = ci[live, 1].astype(np.uint64), ci[live, 2].astype(np.uint64)
        keys = (np.minimum(a, b) << np.uint64(32)) | np.maximum(a, b)
        order_keys.append(keys)
        order_offsets.append(order_offsets[-1] + len(keys))
        R.step_solve(sc.world, 1.0 / 60.0, 4, 2, True)
        R.step_finalize(sc.world)
        if step in marks:
            bf, bi = R.bodies(sc.world)
            idx = [b.index for b in sc.bodies]
            out[f"origin_step{step}"] = bf[idx, 0:2].astype(np.float32)
            out[f"rot_step{step}"] = bf[idx, 4:6].astype(np.float32)
            out[f"velocity_step{step}"] = bf[idx, 6:9].astype(np.float32)
    out["order_keys"] = np.concatenate(order_keys)
    out["order_offsets"] = np.array(order_offsets, dtype=np.int64)
    out["marks"] = np.array(marks, dtype=np.int64)
    sc.destroy()
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), f"pyramid10_{solver.lower()}_90.npz")
    np.savez_compressed(path, **out)
    print("wrote", path)


def host_digests(R):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import json
    import test_host_cpu as T
    out = {name: [T.trial_digest(t) for t in sweep(R, True)] for name, sweep in T.SWEEPS.items()}
    with open(T.HOST_GOLDEN, "w") as fh:
        json.dump(out, fh, indent=0)
        fh.write("\n")
    print("wrote", T.HOST_GOLDEN)


def main():
    R = ref.load()
    host_digests(R)
    if sys.argv[1:] == ["host"]:
        return
    for solver in VARIANTS:
        variant_fixture(R, solver)
    sc = scenes.pyramid(R, "TGS_Soft", base_count=10)
    out = {}
    order_keys, order_offsets = [], [0]
    for step in range(1, 601):
        R.step_collide(sc.world)
        cf, ci = R.contacts(sc.world)
        live = ci[:, 0] == 1
        a, b = ci[live, 1].astype(np.uint64), ci[live, 2].astype(np.uint64)
        keys = (np.minimum(a, b) << np.uint64(32)) | np.maximum(a, b)
        order_keys.append(keys)
        order_offsets.append(order_offsets[-1] + len(keys))
        R.step_solve(sc.world, 1.0 / 60.0, 4, 2, True)
        R.step_finalize(sc.world)
        if step in (1, 10, 60, 600):
            bf, bi = R.bodies(sc.world)
            idx = [b.index for b in sc.bodies]
            out[f"origin_step{step}"] = bf[idx, 0:2].astype(np.float32)
            out[f"rot_step{step}"] = bf[idx, 4:6].astype(np.float32)
            out[f"velocity_step{step}"] = bf[idx, 6:9].astype(np.float32)
    out["order_keys"] = np.concatenate(order_keys)
    out["order_offsets"] = np.array(order_offsets, dtype=np.int64)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pyramid10_tgs_soft.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
