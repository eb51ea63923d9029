"""CPU: the weld joint in the joint oracle (tests/joint_oracle.c, DESIGN.md §3.8) on hand-built rows, for all ten variants.

No contacts and every local centre at zero, so finalize is the identity (origin == position) and solver stages chain
directly. The bounds below were measured on these deterministic runs (the largest value over the ten variants, printed
by `python tests/test_weld_cpu.py`) and carry the margin stated next to each.

Mutations each test catches: a bias applied in the relax pass or lambda zeroed at prepare breaks `at rest` (non-zero
impulses) or `spinning pair`; a missing unwind makes `unwind` spin the body round by 2 pi; a weld row that skips its
angular row lets the cantilever and the spinning pair fold at the anchors."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import joint_oracle  # noqa: E402
from solver2d_b200 import capi, device  # noqa: E402

VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]
DT = 1.0 / 60.0
HX, HY = 0.5, 0.125  # box half extents of the beams
MASS = 1.0
INERTIA = MASS * ((2 * HX) ** 2 + (2 * HY) ** 2) / 12.0

# measured maxima over the ten variants (see the module docstring) and the margin each bound keeps
SPIN_ANGLE_BOUND = 1e-5       # measured 0: both bodies turn alike, so the relative angle stays exact
SPIN_GAP_BOUND = 0.02         # measured 8.6e-3 m (Jacobi, PGS_Soft), x ~2.3
SPIN_MOMENTUM_BOUND = 1e-4    # measured 1.2e-5 (XPBD), x ~8: float32 round-off of 60 steps at |p| ~ 2.2
CANTILEVER_SAG_BOUND = 1.5    # measured 0.84 m (PGS_NGS), x ~1.8; TGS_NGS ends 2.7 cm above its rest line
CANTILEVER_RISE_BOUND = 0.05
UNWIND_ANGLE_BOUND = 1e-4     # measured 9.4e-6 rad (TGS_Soft), x ~10, against the 0.2 rad it starts off
UNWIND_TURN_BOUND = 1.0       # measured 0.42 rad of total turn (XPBD); a flip round the seam turns ~2 pi
# PGS solves the weld with Baumgarte rows at the full step (no sub-steps) and 4 iterations: the five-box beam holds for
# about a second, then its oscillation grows and the beam breaks up (tip 8 m down at 2 s). Its bound is taken at 0.5 s.
CANTILEVER_STEPS = {"PGS": 30}


def _bodies(specs):
    """specs: (type, x, y, angle, vx, vy, w) per body."""
    rows = np.zeros(len(specs), dtype=device.BODY_ROW)
    for i, (kind, x, y, angle, vx, vy, w) in enumerate(specs):
        r = rows[i]
        r["index"] = i
        r["flags"] = device.ROW_VALID | (kind << 1)
        r["origin"] = (x, y)
        r["position"] = (x, y)
        r["rot"] = (np.float32(math.sin(angle)), np.float32(math.cos(angle)))
        r["linearVelocity"] = (vx, vy)
        r["angularVelocity"] = w
        r["gravityScale"] = 1.0
        if kind == capi.DYNAMIC_BODY:
            r["mass"], r["invMass"] = MASS, 1.0 / MASS
            r["I"], r["invI"] = INERTIA, 1.0 / INERTIA
        rows[i] = r
    return rows


def _welds(bodies, links):
    """links: (a, b, world pivot, referenceAngle); anchors are the pivot in each body's origin frame."""
    rows = np.zeros(len(links), dtype=device.JOINT_ROW)
    for k, (a, b, pivot, ref) in enumerate(links):
        rows[k]["index"] = k
        rows[k]["flags"] = device.ROW_VALID | (device.JOINT_WELD << 1)
        rows[k]["bodyA"], rows[k]["bodyB"] = a, b
        for name, i in (("localOriginAnchorA", a), ("localOriginAnchorB", b)):
            s, c = bodies["rot"][i]
            d = np.asarray(pivot, dtype=np.float64) - bodies["origin"][i]
            rows[k][name] = (c * d[0] + s * d[1], -s * d[0] + c * d[1])
        rows[k]["referenceAngle"] = ref
    return rows


def _run(solver, bodies, joints, steps, gravity=(0.0, 0.0)):
    O = joint_oracle.load()
    ctx = device.make_context(solver, DT, 4, 2)
    contacts = np.zeros(0, dtype=device.CONTACT_ROW)
    history = []
    for _ in range(steps):
        bodies, _, joints = O.solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, gravity=gravity)
        bodies["origin"] = bodies["position"]
        history.append((bodies.copy(), joints.copy()))
    return history


def _angle(bodies, i):
    return math.atan2(float(bodies["rot"][i][0]), float(bodies["rot"][i][1]))


def _unwind(a):
    return (a + math.pi) % (2.0 * math.pi) - math.pi


def _errors(bodies, joints):
    """Largest angle error and anchor gap over the welds."""
    ang, gap = 0.0, 0.0
    for j in joints:
        a, b = int(j["bodyA"]), int(j["bodyB"])
        ang = max(ang, abs(_unwind(_angle(bodies, b) - _angle(bodies, a) - float(j["referenceAngle"]))))
        p = []
        for i, name in ((a, "localOriginAnchorA"), (b, "localOriginAnchorB")):
            s, c = (float(v) for v in bodies["rot"][i])
            lx, ly = (float(v) for v in j[name])
            p.append(np.array([c * lx - s * ly, s * lx + c * ly]) + bodies["origin"][i].astype(np.float64))
        gap = max(gap, float(np.linalg.norm(p[1] - p[0])))
    return ang, gap


# ---- the scenes ---------------------------------------------------------------------------------------------------------

def _at_rest():
    b = _bodies([(capi.STATIC_BODY, 0.0, 0.0, 0.0, 0, 0, 0), (capi.DYNAMIC_BODY, 1.0, 0.0, 0.0, 0, 0, 0)])
    return b, _welds(b, [(0, 1, (0.5, 0.0), 0.0)])


def _spinning(w=3.0, v=(1.0, 2.0)):
    # a rigid rotation about the pair's centre of mass at the origin, plus a common velocity
    b = _bodies([(capi.DYNAMIC_BODY, -0.5, 0.0, 0.0, v[0], v[1] - 0.5 * w, w),
                 (capi.DYNAMIC_BODY, 0.5, 0.0, 0.0, v[0], v[1] + 0.5 * w, w)])
    return b, _welds(b, [(0, 1, (0.0, 0.0), 0.0)])


def _cantilever(n=5):
    specs = [(capi.STATIC_BODY, 0.0, 0.0, 0.0, 0, 0, 0)]
    specs += [(capi.DYNAMIC_BODY, 0.75 + i, 0.0, 0.0, 0, 0, 0) for i in range(n)]
    b = _bodies(specs)
    return b, _welds(b, [(i, i + 1, (0.25 + i, 0.0), 0.0) for i in range(n)])


def _seam(ref):
    # body B starts 0.2 rad past its reference angle, across the +-pi seam of the relative angle
    b = _bodies([(capi.STATIC_BODY, 0.0, 0.0, 0.0, 0, 0, 0), (capi.DYNAMIC_BODY, 1.0, 0.0, ref + math.copysign(0.2, ref), 0, 0, 0)])
    return b, _welds(b, [(0, 1, (0.5, 0.0), ref)])


# ---- tests --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", VARIANTS)
def test_at_rest_is_exactly_still(solver):
    bodies, joints = _at_rest()
    for b, j in _run(solver, bodies, joints, 5):
        assert np.all(j["impulse"] == 0) and np.all(j["motorImpulse"] == 0)
        assert np.all(b["linearVelocity"] == 0) and np.all(b["angularVelocity"] == 0)
        assert np.array_equal(b["position"], bodies["position"]) and np.array_equal(b["rot"], bodies["rot"])


def _spin_metrics(solver):
    bodies, joints = _spinning()
    p0 = (bodies["linearVelocity"].astype(np.float64) * MASS).sum(axis=0)
    drift, ang, gap = 0.0, 0.0, 0.0
    for b, j in _run(solver, bodies, joints, 60):
        drift = max(drift, float(np.abs((b["linearVelocity"].astype(np.float64) * MASS).sum(axis=0) - p0).max()))
        a, g = _errors(b, j)
        ang, gap = max(ang, a), max(gap, g)
    return drift, ang, gap, b


@pytest.mark.parametrize("solver", VARIANTS)
def test_spinning_pair(solver):
    drift, ang, gap, last = _spin_metrics(solver)
    assert drift < SPIN_MOMENTUM_BOUND, drift
    assert ang < SPIN_ANGLE_BOUND, ang
    assert gap < SPIN_GAP_BOUND, gap
    # it still spins (from 3 rad/s: measured 2.84 to 3.0 after 1 s; TGS_Sticky, which applies its Baumgarte bias to the point
    # row in every pass and starts each step cold, brakes it to 1.23)
    assert np.all(last["angularVelocity"] > 1.0)


def _sag(solver):
    bodies, joints = _cantilever()
    b, _ = _run(solver, bodies, joints, CANTILEVER_STEPS.get(solver, 120), gravity=(0.0, -10.0))[-1]
    return -float(b["position"][-1][1])


@pytest.mark.parametrize("solver", VARIANTS)
def test_cantilever_sag_is_bounded(solver):
    sag = _sag(solver)
    assert -CANTILEVER_RISE_BOUND < sag < CANTILEVER_SAG_BOUND, sag


def _seam_error(solver, ref):
    bodies, joints = _seam(ref)
    hist = _run(solver, bodies, joints, 120)
    b, j = hist[-1]
    err, _ = _errors(b, j)
    # the body turns back by 0.2 rad, never round by 2 pi: track the total turn of its rotation
    turn = sum(abs(_unwind(_angle(h[0], 1) - _angle(p[0], 1))) for p, h in zip([(bodies, joints)] + hist[:-1], hist))
    return err, turn


@pytest.mark.parametrize("ref", [3.0, -3.0])
@pytest.mark.parametrize("solver", VARIANTS)
def test_unwind_across_the_seam(solver, ref):
    err, turn = _seam_error(solver, ref)
    assert err < UNWIND_ANGLE_BOUND, err
    assert turn < UNWIND_TURN_BOUND, turn


if __name__ == "__main__":
    for s in VARIANTS:
        d, a, g, _ = _spin_metrics(s)
        e3, t3 = _seam_error(s, 3.0)
        e_3, t_3 = _seam_error(s, -3.0)
        print(f"{s:14s} spin: dp={d:.2e} angle={a:.2e} gap={g:.2e}  sag={_sag(s):.4f}  seam: {e3:.2e} {e_3:.2e} turn {t3:.3f} {t_3:.3f}")
