"""CPU: the pulley joint in the joint oracle (tests/joint_oracle.c, DESIGN.md §3.18) on hand-built rows, for all ten variants.

No contacts and every local centre at zero, so finalize is the identity (origin == position) and solver stages chain
directly. The bounds below were measured on these deterministic runs (the largest value over the variants a test covers)
and carry the margin stated next to each.

Mutations each test catches: a ratio left out of the mass or of side B's impulse breaks the balance and the acceleration;
a bias with its sign flipped lets lengthA + ratio lengthB drift away; a rope formed from the other body's pose, or from a
start offset left out, breaks the balance; a degenerate rope normalized anyway makes NaNs; an NGS correction without its
clamp closes a large error in one iteration; a pulley branch that takes another type's rows changes the bits
tests/test_joint_oracle_cpu.py pins."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import joint_oracle  # noqa: E402
from solver2d_b200 import capi, device  # noqa: E402

VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]
NGS = {"PGS_NGS": 2, "PGS_NGS_Block": 2, "TGS_NGS": 4}  # NGS position iterations per step at 4 sub-steps, 2 relax
DT = 1.0 / 60.0
G = 10.0
MAX_CORRECTION = 0.2  # s2_maxLinearCorrection

# measured maxima (see the module docstring) and the margin each bound keeps
DRIFT = 1.5e-3              # |lengthA + ratio lengthB - constant| over 4 s: measured 7.1e-4 (Jacobi, PGS_Soft, TGS_Soft),
                            # <= 1.8e-4 under SoftStep, <= 3.9e-6 under the rest, x 2.1
REST_SPEED = 3e-4           # body speed of the balanced pair over 2 s: measured 1.0e-4 (XPBD), <= 5.5e-8 under the rest, x 3
ACCEL_REL = 3e-4            # relative error of both accelerations after 0.5 s: measured 9.3e-5 (XPBD), <= 4.2e-7 under the
                            # rest, x 3.2
DRIVER_SPEED = 2e-4         # |vB - v / ratio| after the first 10 steps: measured 8.3e-5 (XPBD), 3.1e-5 (TGS_Sticky),
                            # <= 3.9e-6 under the rest, x 2.4


def _bodies(specs):
    """specs: (type, x, y, mass[, vy, gravityScale]) per body; boxes with inertia mass / 6 (a unit box's)."""
    rows = np.zeros(len(specs), dtype=device.BODY_ROW)
    for i, spec in enumerate(specs):
        kind, x, y, mass = spec[:4]
        vy = spec[4] if len(spec) > 4 else 0.0
        gs = spec[5] if len(spec) > 5 else 1.0
        r = rows[i]
        r["index"] = i
        r["flags"] = device.ROW_VALID | (kind << 1)
        r["origin"] = (x, y)
        r["position"] = (x, y)
        r["rot"] = (0.0, 1.0)
        r["linearVelocity"] = (0.0, vy)
        r["gravityScale"] = gs
        if kind == capi.DYNAMIC_BODY:
            r["mass"], r["invMass"] = mass, 1.0 / mass
            r["I"], r["invI"] = mass / 6.0, 6.0 / mass
        rows[i] = r
    return rows


def _pulley(a, b, ground_a, ground_b, length_a, length_b, ratio, anchor_a=(0.0, 0.0), anchor_b=(0.0, 0.0), slot=0):
    """One pulley row, laid out as s2FillJointRow lays it out."""
    r = np.zeros(1, dtype=device.JOINT_ROW)[0]
    r["index"] = slot
    r["flags"] = device.ROW_VALID | (device.JOINT_PULLEY << 1) | device.JOINT_COLLIDE_CONNECTED
    r["bodyA"], r["bodyB"] = a, b
    r["localOriginAnchorA"], r["localOriginAnchorB"] = anchor_a, anchor_b
    r["target"], r["localAxisA"] = ground_a, ground_b
    r["referenceAngle"], r["lowerAngle"], r["upperAngle"] = ratio, length_a, length_b
    return r


def _run(solver, bodies, joints, steps, gravity=(0.0, -G)):
    O = joint_oracle.load()
    ctx = device.make_context(solver, DT, 4, 2)
    contacts = np.zeros(0, dtype=device.CONTACT_ROW)
    history = []
    for _ in range(steps):
        bodies, _, joints = O.solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, gravity=gravity)
        bodies["origin"] = bodies["position"]
        history.append((bodies.copy(), joints.copy()))
    return history


def _lengths(b, ground_a, ground_b, ia=1, ib=2):
    pa, pb = b["position"][ia].astype(np.float64), b["position"][ib].astype(np.float64)
    return math.hypot(*(pa - ground_a)), math.hypot(*(pb - ground_b))


# ---- the constraint ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", VARIANTS)
def test_constraint_drift(solver):
    """An unbalanced pair (ratio 1.5, mB = 1.3 mA) with off-centre anchors, so the bodies also turn, runs for 4 s: lengthA
    + ratio lengthB stays within DRIFT of its constant."""
    # anchor A sits 0.3 m above body A's centre and 0.2 m to the side of ground anchor A's vertical, so the rope pulls at an
    # angle and turns body A
    gA, gB = np.array([0.0, 15.0]), np.array([4.0, 15.0])
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0), (capi.DYNAMIC_BODY, 0.2, 0.0, 1.0), (capi.DYNAMIC_BODY, 4.0, 0.1, 1.3)])
    row = _pulley(1, 2, gA, gB, math.hypot(0.2, 14.7), 14.9, 1.5, anchor_a=(0.0, 0.3))
    constant = float(np.float32(row["lowerAngle"]) + np.float32(1.5) * np.float32(row["upperAngle"]))
    worst = 0.0
    for b, _ in _run(solver, bodies, np.array([row]), 240):
        pa = b["position"][1].astype(np.float64) + np.array([-0.3 * b["rot"][1][0], 0.3 * b["rot"][1][1]])
        pb = b["position"][2].astype(np.float64)
        c = math.hypot(*(pa - gA)) + 1.5 * math.hypot(*(pb - gB))
        worst = max(worst, abs(c - constant))
    assert np.isfinite(worst)
    assert worst <= DRIFT, worst


@pytest.mark.parametrize("solver", VARIANTS)
def test_balanced_pair_rests_and_reads_mb_g(solver):
    """ratio 2, mB = 2 mA, anchors at the centres of mass, each body straight below its ground anchor: the pair stays at
    rest, and the reaction on body B reads (0, mB g) (zero under XPBD, which keeps no impulses)."""
    P = capi.Solver2D(device.LIB_PATH)
    gA, gB = (0.0, 5.0), (3.0, 5.0)
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0), (capi.DYNAMIC_BODY, 0.0, 0.0, 1.0), (capi.DYNAMIC_BODY, 3.0, 1.0, 2.0)])
    hist = _run(solver, bodies, np.array([_pulley(1, 2, gA, gB, 5.0, 4.0, 2.0)]), 120)
    b, j = hist[-1]
    speed = max(float(np.abs(h[0]["linearVelocity"][1:]).max()) for h in hist)
    sub = solver in capi.SUBSTEPPING
    rate = np.float32((1.0 / DT) if (solver == "TGS_Sticky" or not sub) else 4.0 / DT)
    # -ratio uB with uB = (0, -1): the axis s2cPulleyJointAxis forms for body B straight below ground anchor B
    r = P.s2ComputeJointReaction(device.JOINT_PULLEY, capi.Vec2(float(j["impulse"][0][0]), float(j["impulse"][0][1])), 0.0, 0.0,
                                 0.0, capi.Rot(0.0, 1.0), capi.Vec2(0.0, 2.0), float(rate))
    assert r.torque == 0.0 and r.force.x == 0.0
    # measured exact under every variant that keeps impulses
    assert r.force.y == (0.0 if solver == "XPBD" else 2.0 * G), r.force.y
    assert speed <= REST_SPEED, speed


@pytest.mark.parametrize("ratio, mass_b", [(1.0, 1.5), (2.0, 1.0), (1.5, 3.5)])
@pytest.mark.parametrize("solver", VARIANTS)
def test_unbalanced_pair_accelerates(solver, ratio, mass_b):
    """Anchors at the centres of mass, ropes vertical, mA = 1: body A accelerates downward at g (mA - mB / ratio) /
    (mA + mB / ratio^2) (with ratio 1, Atwood's g (m1 - m2) / (m1 + m2)), and B upward at that over ratio."""
    mA = 1.0
    expected = G * (mA - mass_b / ratio) / (mA + mass_b / ratio ** 2)
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0), (capi.DYNAMIC_BODY, 0.0, 0.0, mA), (capi.DYNAMIC_BODY, 3.0, 0.0, mass_b)])
    steps = 30
    b, _ = _run(solver, bodies, np.array([_pulley(1, 2, (0.0, 10.0), (3.0, 10.0), 10.0, 10.0, ratio)]), steps)[-1]
    t = steps * DT
    got_a = -float(b["linearVelocity"][1][1]) / t
    got_b = float(b["linearVelocity"][2][1]) / t
    rel = max(abs(got_a - expected), abs(got_b * ratio - expected)) / abs(expected)
    assert rel <= ACCEL_REL, (got_a, got_b, expected)


@pytest.mark.parametrize("solver", VARIANTS)
def test_kinematic_driver_moves_b_at_v_over_ratio(solver):
    """A kinematic body on side A moving down at 0.5 m/s lifts a load on side B (ratio 1.5) at 0.5 / 1.5 m/s."""
    v, ratio = 0.5, 1.5
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0), (capi.KINEMATIC_BODY, 0.0, 0.0, 0.0, -v),
                      (capi.DYNAMIC_BODY, 3.0, 0.0, 1.0)])
    hist = _run(solver, bodies, np.array([_pulley(1, 2, (0.0, 5.0), (3.0, 5.0), 5.0, 5.0, ratio)]), 60)
    worst = max(abs(float(b["linearVelocity"][2][1]) - v / ratio) for b, _ in hist[10:])
    assert worst <= DRIVER_SPEED, worst


@pytest.mark.parametrize("solver", VARIANTS)
def test_degenerate_rope_exerts_nothing(solver):
    """Anchor A within 10 s2_linearSlop of ground anchor A: rope A has no direction, so body A falls as a free body does
    (body 3, no joint) and nothing is NaN; body B still hangs on its rope."""
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0), (capi.DYNAMIC_BODY, 0.0, 4.97, 1.0), (capi.DYNAMIC_BODY, 3.0, 0.0, 1.0),
                      (capi.DYNAMIC_BODY, 6.0, 4.97, 1.0)])
    hist = _run(solver, bodies, np.array([_pulley(1, 2, (0.0, 5.0), (3.0, 5.0), 0.03, 5.0, 1.0)]), 2)
    for b, j in hist:
        assert np.isfinite(b["position"]).all() and np.isfinite(b["linearVelocity"]).all() and np.isfinite(j["impulse"]).all()
        # still within 10 slop after two steps: A moved exactly as the free body
        if solver == "XPBD":
            assert abs(float(b["position"][1][1]) - float(b["position"][3][1])) <= 1e-6
        else:
            assert b["linearVelocity"][1].tobytes() == b["linearVelocity"][3].tobytes()
            assert b["angularVelocity"][1] == 0.0
    # B held on its rope: it did not fall freely
    assert float(hist[-1][0]["position"][2][1]) > float(hist[-1][0]["position"][3][1]) - 4.97 + 1e-3


@pytest.mark.parametrize("sign", [1.0, -1.0])
@pytest.mark.parametrize("solver", sorted(NGS))
def test_large_initial_error_closes_at_most_max_correction_per_iteration(solver, sign):
    """A weightless pair at rest on a pulley created 1 m off its constant: the NGS position pass closes the error by at most
    s2_maxLinearCorrection per iteration, and closes it."""
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0), (capi.DYNAMIC_BODY, 0.0, 0.0, 1.0, 0.0, 0.0),
                      (capi.DYNAMIC_BODY, 3.0, 0.0, 1.0, 0.0, 0.0)])
    constant = 10.0 + sign
    hist = _run(solver, bodies, np.array([_pulley(1, 2, (0.0, 5.0), (3.0, 5.0), 5.0 + sign, 5.0, 1.0)]), 10)
    prev = 1.0
    closed = []
    for b, _ in hist:
        la, lb = _lengths(b, (0.0, 5.0), (3.0, 5.0))
        err = abs(constant - la - lb)
        closed.append(prev - err)
        assert prev - err <= NGS[solver] * MAX_CORRECTION * (1.0 + 1e-5), (prev, err)
        prev = err
    assert closed[0] >= NGS[solver] * MAX_CORRECTION * (1.0 - 1e-5)  # the clamp, not the error, set the first step
    assert prev <= 1e-5


# ---- other joint types and layout -----------------------------------------------------------------------------------------

def test_struct_sizes_unchanged():
    """The pulley row reuses columns: s2bJointRow stays 108 bytes and every other ABI size is the parent's."""
    out = (C.c_int32 * 6)()
    C.CDLL(device.LIB_PATH).s2b_abi_sizes(out)
    assert out[2] == 108 == device.JOINT_ROW.itemsize
    assert (out[0], out[1], out[3]) == (device.BODY_ROW.itemsize, device.SHAPE_ROW.itemsize, device.CONTACT_ROW.itemsize)
