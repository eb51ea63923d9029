"""CPU: the distance joint in the joint oracle (tests/joint_oracle.c, DESIGN.md §3.16) on hand-built rows, for all ten variants.

No contacts and every local centre at zero, so finalize is the identity (origin == position) and solver stages chain
directly. The bounds below were measured on these deterministic runs (the largest value over the variants a test covers,
computed from these same runs) and carry the margin stated next to each.

Mutations each test catches: a rigid row without its bias drifts the pendulum's length; a spring coefficient formed with
another h shifts the frequency or the sag; a limit with its sign flipped lets the rope stretch or pushes it out; a motor
impulse that is not clamped lifts a load it should not; an axis normalised without the degenerate test makes NaNs; an
impulse applied to one body only breaks momentum; a reaction that leaves the rigid impulse out reads zero."""
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
DT = 1.0 / 60.0
G = 10.0
MASS = 2.0
INERTIA = 0.1
SLOP = 0.005

# measured maxima (see the module docstring) and the margin each bound keeps
ROD_DRIFT = 2e-3            # |length - L| of a 1 m rod over 4 s: measured 3.8e-4 (Jacobi, PGS_Soft), <= 8.3e-5 elsewhere, x 5
PERIOD_REL = 5e-3           # small-amplitude period vs 2 pi sqrt(L / g): measured 9.9e-4 under every variant, x 5
SPRING_FREQ_REL = 0.04      # undamped 1 Hz spring over 4 s: measured <= 4.7e-3 (Jacobi, PGS_Soft), 0 elsewhere, at the
                            # resolution of the zero crossings (one step per half period, 1 / 30)
OVERSHOOT = 1e-3            # zeta = 1 from 0.2 m stretched: measured none (the length stays >= rest + 4.8e-7)
SAG_REL = 1e-4              # static sag m g / k against k = m omega^2: measured <= 2.5e-6, x 40
# TGS_Sticky prepares its joints cold once per step and accumulates their impulses over the sub-steps, so its spring is
# softer and more damped than its hertz and damping ratio say (DESIGN.md §3.14). Its spring bounds are its own measured
# values with a margin; no other variant is special-cased.
FREQ_REL_STICKY = 0.6       # measured 0.50 (f = 0.5 Hz for 1 Hz), x 1.2
OVERSHOOT_STICKY = 0.05     # measured 3.3e-2, x 1.5
SAG_REL_STICKY = 4.0        # measured 2.92 (rests at ~3.9 m g / k), x 1.4
ROPE_STRETCH = 2e-3         # a taut rope's length over maxLength: measured <= 2.8e-4; a pushed-out pair's gap short of
                            # minLength: measured <= 9.0e-5
MOTOR_SPEED = 1e-3          # m/s off the set speed after 1 s: measured 0 under every variant but XPBD (no motor there)
MOMENTUM = 1e-4             # free pair, 60 steps: measured <= 4.3e-6, x 20


def _bodies(specs):
    """specs: (type, x, y, vx, vy, w, gravityScale) per body."""
    rows = np.zeros(len(specs), dtype=device.BODY_ROW)
    for i, (kind, x, y, vx, vy, w, gs) in enumerate(specs):
        r = rows[i]
        r["index"] = i
        r["flags"] = device.ROW_VALID | (kind << 1)
        r["origin"] = (x, y)
        r["position"] = (x, y)
        r["rot"] = (0.0, 1.0)
        r["linearVelocity"] = (vx, vy)
        r["angularVelocity"] = w
        r["gravityScale"] = gs
        if kind == capi.DYNAMIC_BODY:
            r["mass"], r["invMass"] = MASS, 1.0 / MASS
            r["I"], r["invI"] = INERTIA, 1.0 / INERTIA
        rows[i] = r
    return rows


def _distance(a, b, anchor_a=(0.0, 0.0), anchor_b=(0.0, 0.0), length=1.0, spring=None, limit=None, motor=None,
              spring_flag=None, slot=0):
    """One distance row. spring = (hertz, dampingRatio); limit = (min, max); motor = (speed, maxForce)."""
    r = np.zeros(1, dtype=device.JOINT_ROW)[0]
    r["index"] = slot
    r["flags"] = device.ROW_VALID | (device.JOINT_DISTANCE << 1)
    r["bodyA"], r["bodyB"] = a, b
    r["localOriginAnchorA"], r["localOriginAnchorB"] = anchor_a, anchor_b
    r["referenceAngle"] = length
    r["lowerAngle"], r["upperAngle"] = SLOP, 100000.0
    if spring is not None or spring_flag:
        r["flags"] |= device.JOINT_ENABLE_SPRING
        r["hertz"], r["dampingRatio"] = spring if spring is not None else (0.0, 0.0)
    if limit is not None:
        r["flags"] |= device.JOINT_ENABLE_LIMIT
        r["lowerAngle"], r["upperAngle"] = limit
    if motor is not None:
        r["flags"] |= device.JOINT_ENABLE_MOTOR
        r["motorSpeed"], r["maxMotorTorque"] = motor
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


def _length(b, i=1):
    return float(np.hypot(*b["position"][i].astype(np.float64)))


def _crossings(xs):
    return [k for k in range(1, len(xs)) if (xs[k - 1] < 0.0) != (xs[k] < 0.0)]


# ---- rod ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", VARIANTS)
def test_rod_pendulum_keeps_length_and_period(solver):
    """A 1 m rod from a static pivot to a box started 0.1 rad off vertical: the length stays within the variant's bound and
    the period is 2 pi sqrt(L / g)."""
    L, a0 = 1.0, 0.1
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 1), (capi.DYNAMIC_BODY, L * math.sin(a0), -L * math.cos(a0), 0, 0, 0, 1)])
    hist = _run(solver, bodies, np.array([_distance(0, 1, length=L)]), 240)
    drift = max(abs(_length(b) - L) for b, _ in hist)
    assert drift <= ROD_DRIFT, drift
    xs = [float(b["position"][1][0]) for b, _ in hist]
    cross = _crossings(xs)
    assert len(cross) >= 4
    period = 2.0 * (cross[-1] - cross[0]) / (len(cross) - 1) * DT
    assert abs(period / (2.0 * math.pi * math.sqrt(L / G)) - 1.0) <= PERIOD_REL, period


# ---- spring ---------------------------------------------------------------------------------------------------------------

def _spring_case(solver, zeta, steps, gravity=(0.0, 0.0), x0=1.2):
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 1), (capi.DYNAMIC_BODY, x0, 0, 0, 0, 0, 1)])
    joint = _distance(0, 1, length=1.0, spring=(1.0, zeta))
    return _run(solver, bodies, np.array([joint]), steps, gravity=gravity)


@pytest.mark.parametrize("solver", VARIANTS)
def test_spring_oscillates_at_hertz(solver):
    hist = _spring_case(solver, 0.0, 240)
    xs = [_length(b) - 1.0 for b, _ in hist]
    cross = _crossings(xs)
    f = (len(cross) - 1) / (2.0 * (cross[-1] - cross[0]) * DT)
    assert abs(f - 1.0) <= (FREQ_REL_STICKY if solver == "TGS_Sticky" else SPRING_FREQ_REL), f


@pytest.mark.parametrize("solver", VARIANTS)
def test_critical_spring_does_not_overshoot(solver):
    hist = _spring_case(solver, 1.0, 240)
    assert min(_length(b) - 1.0 for b, _ in hist) >= -(OVERSHOOT_STICKY if solver == "TGS_Sticky" else OVERSHOOT)


@pytest.mark.parametrize("solver", VARIANTS)
def test_spring_sags_by_mg_over_k(solver):
    """A box hanging on a 1 Hz, zeta = 1 spring of rest length 1 rests at 1 + m g / k, k = m omega^2."""
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 1), (capi.DYNAMIC_BODY, 0, -1.0, 0, 0, 0, 1)])
    hist = _run(solver, bodies, np.array([_distance(0, 1, length=1.0, spring=(1.0, 1.0))]), 600)
    sag = _length(hist[-1][0]) - 1.0
    expect = G / (2.0 * math.pi) ** 2
    assert abs(sag / expect - 1.0) <= (SAG_REL_STICKY if solver == "TGS_Sticky" else SAG_REL), sag


# ---- rope and limits ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", VARIANTS)
def test_rope_is_free_when_slack_and_taut_at_max(solver):
    """A rope (spring on at hertz 0, limit [slop, 2]) from a static point: a box released 1 m below falls freely, then
    hangs at 2 m."""
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 1), (capi.DYNAMIC_BODY, 0, -1.0, 0, 0, 0, 1)])
    joint = _distance(0, 1, length=1.0, spring_flag=True, limit=(SLOP, 2.0))
    hist = _run(solver, bodies, np.array([joint]), 120)
    # free fall for the first 5 steps (the box falls 0.35 m in them)
    vy = float(hist[4][0]["linearVelocity"][1][1])
    assert vy < -0.7
    assert all(float(j["impulse"][0][0]) == 0.0 for _, j in hist)
    stretch = max(_length(b) - 2.0 for b, _ in hist[60:])
    assert stretch <= ROPE_STRETCH, stretch
    assert _length(hist[-1][0]) >= 2.0 - ROPE_STRETCH


@pytest.mark.parametrize("solver", VARIANTS)
def test_min_length_pushes_out(solver):
    """minLength = 1 with the spring on at hertz 0: two boxes pushed together at 0.5 m end apart at >= 1 m - tolerance."""
    bodies = _bodies([(capi.DYNAMIC_BODY, 0, 0, 0, 0, 0, 0), (capi.DYNAMIC_BODY, 0.5, 0, 0, 0, 0, 0)])
    joint = _distance(0, 1, length=1.0, spring_flag=True, limit=(1.0, 3.0))
    hist = _run(solver, bodies, np.array([joint]), 60, gravity=(0.0, 0.0))
    b = hist[-1][0]
    gap = float(b["position"][1][0] - b["position"][0][0])
    assert gap >= 1.0 - ROPE_STRETCH, gap


# ---- motor ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", VARIANTS)
def test_motor_reaches_speed_and_stalls_below_its_load(solver):
    """A winch (spring on at hertz 0, no limit) shortens at 0.5 m/s, lifting a 2 kg box with 100 N; with 10 N (< m g) the
    box sinks. XPBD does not apply the motor (as for the prismatic joint): both boxes fall away."""
    out = []
    for force in (100.0, 10.0):
        bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 1), (capi.DYNAMIC_BODY, 0, -2.0, 0, 0, 0, 1)])
        joint = _distance(0, 1, length=2.0, spring_flag=True, motor=(-0.5, force))
        out.append(_run(solver, bodies, np.array([joint]), 60))
    if solver == "XPBD":
        assert all(_length(o[-1][0]) > 2.0 for o in out)
        return
    vy = float(out[0][-1][0]["linearVelocity"][1][1])
    assert abs(vy - 0.5) <= MOTOR_SPEED, vy
    assert _length(out[0][-1][0]) < 2.0 - 0.3
    assert _length(out[1][-1][0]) > 2.0


# ---- edges ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", VARIANTS)
def test_coincident_anchors_make_no_nan_and_no_impulse(solver):
    """Anchors that coincide exactly (d = 0): the axis is zero, so no impulse reaches the bodies."""
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 1), (capi.DYNAMIC_BODY, 0.0, 0.0, 0, 0, 0, 0)])
    joint = _distance(0, 1, length=1.0, spring=(2.0, 0.5), limit=(0.5, 2.0), motor=(1.0, 10.0))
    hist = _run(solver, bodies, np.array([joint]), 10, gravity=(0.0, 0.0))
    for b, j in hist:
        assert np.all(np.isfinite(b["position"])) and np.all(np.isfinite(j["impulse"]))
        assert np.all(b["linearVelocity"][1] == 0.0) and b["angularVelocity"][1] == 0.0
        assert np.all(b["position"][1] == 0.0)


@pytest.mark.parametrize("solver", VARIANTS)
def test_equal_limits_with_spring_are_the_rigid_joint(solver):
    """minLength == maxLength with the spring on: the rigid row acts, the limits and spring do not, bit for bit."""
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 1), (capi.DYNAMIC_BODY, 0.6, -0.8, 1.0, 0, 0.5, 1)])
    rigid = _distance(0, 1, anchor_b=(0.1, 0.05), length=1.0)
    equal = _distance(0, 1, anchor_b=(0.1, 0.05), length=1.0, spring=(3.0, 0.4), limit=(1.0, 1.0))
    equal["lowerAngle"] = equal["upperAngle"] = 1.0
    a = _run(solver, bodies.copy(), np.array([rigid]), 30)
    b = _run(solver, bodies.copy(), np.array([equal]), 30)
    for (ba, ja), (bb, jb) in zip(a, b):
        assert ba["position"].tobytes() == bb["position"].tobytes()
        assert ba["linearVelocity"].tobytes() == bb["linearVelocity"].tobytes()
        assert ja["impulse"].tobytes() == jb["impulse"].tobytes()


@pytest.mark.parametrize("solver", VARIANTS)
def test_free_pair_conserves_momentum(solver):
    """Two spinning boxes on a sprung, limited, motored distance joint without gravity: linear momentum stays put."""
    bodies = _bodies([(capi.DYNAMIC_BODY, 0, 0, 0.3, 0.1, 1.0, 0), (capi.DYNAMIC_BODY, 1.5, 0.2, -0.2, 0.4, -2.0, 0)])
    joint = _distance(0, 1, anchor_a=(0.1, 0.1), anchor_b=(-0.1, 0.05), length=1.0, spring=(2.0, 0.2), limit=(0.8, 1.6),
                      motor=(0.3, 1.0))
    hist = _run(solver, bodies, np.array([joint]), 60, gravity=(0.0, 0.0))
    p0 = MASS * (bodies["linearVelocity"][0].astype(np.float64) + bodies["linearVelocity"][1])
    for b, _ in hist:
        p = MASS * (b["linearVelocity"][0].astype(np.float64) + b["linearVelocity"][1])
        assert np.abs(p - p0).max() <= MOMENTUM


# ---- reactions ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", VARIANTS)
def test_hanging_load_reads_mg(solver):
    """A 2 kg box hanging at rest on a rod reads exactly (0, m g) under every variant that holds the load (measured: exact,
    as §3.13's rate check), and zero under XPBD."""
    P = capi.Solver2D(device.LIB_PATH)
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 1), (capi.DYNAMIC_BODY, 0.0, -1.0, 0, 0, 0, 1)])
    b, j = _run(solver, bodies, np.array([_distance(0, 1, length=1.0)]), 30)[-1]
    sub = solver in capi.SUBSTEPPING
    rate = (1.0 / DT) if (solver == "TGS_Sticky" or not sub) else 4.0 / DT
    d = b["position"][1].astype(np.float32) - b["position"][0].astype(np.float32)
    n = float(np.hypot(*d.astype(np.float64)))
    axis = capi.Vec2(float(d[0] / np.float32(n)), float(d[1] / np.float32(n)))
    r = P.s2ComputeJointReaction(device.JOINT_DISTANCE, capi.Vec2(float(j["impulse"][0][0]), 0.0), float(j["motorImpulse"][0]),
                                 float(j["lowerImpulse"][0]), float(j["upperImpulse"][0]), capi.Rot(0.0, 1.0), axis,
                                 np.float32(rate))
    if solver == "XPBD":
        assert (r.force.x, r.force.y, r.torque) == (0.0, 0.0, 0.0)
    else:
        assert (r.force.x, r.force.y, r.torque) == (0.0, MASS * G, 0.0)


def test_struct_sizes_unchanged():
    """The distance row reuses columns: s2bJointRow stays 108 bytes and every other ABI size is the parent's."""
    out = (C.c_int32 * 6)()
    C.CDLL(device.LIB_PATH).s2b_abi_sizes(out)
    assert out[2] == 108 == device.JOINT_ROW.itemsize
    assert (out[0], out[1], out[3]) == (device.BODY_ROW.itemsize, device.SHAPE_ROW.itemsize, device.CONTACT_ROW.itemsize)
