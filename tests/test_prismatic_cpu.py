"""CPU: the prismatic joint in the joint oracle (tests/joint_oracle.c, DESIGN.md §3.9) on hand-built rows, for all ten variants.

No contacts and every local centre at zero, so finalize is the identity (origin == position) and solver stages chain
directly. The bounds below were measured on these deterministic runs (the largest value over the ten variants, printed
by `python tests/test_prismatic_cpu.py`) and carry the margin stated next to each.

Mutations each test catches: a bias applied in the relax pass or an impulse kept without its flag breaks `at rest`; a
block that skips its perpendicular or angular row lets the inclined slider and the free pair leave their axis; an axial
mass formed from the revolute's 1 / (iA + iB) or a limit row with the wrong sign breaks the limits; a motor clamped at
the wrong bound or with the wrong sign breaks the motor tests."""
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
HX, HY = 0.5, 0.25  # box half extents
MASS = 1.0
INERTIA = MASS * ((2 * HX) ** 2 + (2 * HY) ** 2) / 12.0
SIN30 = 0.5

# measured maxima over the ten variants (see the module docstring) and the margin each bound keeps
INCLINE_SPEED_REL = 1e-5      # measured 1.0e-6 (TGS_NGS), x ~10: relative error of g sin30 t after 1 s
INCLINE_PERP_BOUND = 1e-3     # measured 2.4e-4 m (Jacobi, PGS_Soft, TGS_Soft), x ~4
INCLINE_ANGLE_BOUND = 1e-6    # measured 4.4e-9 rad: the body does not turn; the bound allows float round-off
LIMIT_BAND = 0.01             # 2 s2_linearSlop; measured < 5e-4 m past a limit hit at 5 m/s (the speculative term)
LIMIT_REST_BAND = 2e-3        # measured 2.8e-4 m under gravity (Jacobi, PGS_Soft, TGS_Soft), x ~7
MOTOR_SPEED_REL = 1e-4        # measured 0 to float round-off
WEAK_ACCEL_REL = 1e-4         # measured 9.1e-6 on g - F/m (SoftStep, TGS_Soft, TGS_NGS), x ~10
WEAK_FORCE_REL = 1e-5         # measured 0: the clamped impulse is h F exactly, up to float round-off
PAIR_MOMENTUM_BOUND = 5e-5    # measured 6.6e-6 (XPBD), x ~7: float32 round-off of 60 steps at |p| ~ 3
PAIR_PERP_BOUND = 5e-3        # measured 1.0e-3 m (Jacobi, PGS_Soft), x ~5
PAIR_ANGLE_BOUND = 5e-3       # measured 7.0e-4 rad (XPBD), x ~7
# TGS_Sticky prepares its joints cold once per step and accumulates their impulses over the sub-steps, so a motor's cap
# h F (h a sub-step) holds for the whole step: a weak motor pushes with F / 4 and the load sinks at g - F / (4 m). The
# motor impulse still sits at its cap, which the force check covers.
WEAK_ACCEL_SKIP = {"TGS_Sticky"}


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


def _local(bodies, i, p):
    s, c = (float(v) for v in bodies["rot"][i])
    d = np.asarray(p, dtype=np.float64) - bodies["origin"][i].astype(np.float64)
    return (c * d[0] + s * d[1], -s * d[0] + c * d[1])


def _prismatic(bodies, a, b, pivot, axis, ref=0.0, limit=None, motor=None):
    """One prismatic row; `axis` in body A's frame (normalized here as the host does), anchors at `pivot`."""
    rows = np.zeros(1, dtype=device.JOINT_ROW)
    r = rows[0]
    r["index"] = 0
    r["flags"] = device.ROW_VALID | (device.JOINT_PRISMATIC << 1)
    r["bodyA"], r["bodyB"] = a, b
    r["localOriginAnchorA"] = _local(bodies, a, pivot)
    r["localOriginAnchorB"] = _local(bodies, b, pivot)
    ax = np.asarray(axis, dtype=np.float32)
    r["localAxisA"] = ax / np.sqrt(ax[0] * ax[0] + ax[1] * ax[1])
    r["referenceAngle"] = ref
    if limit is not None:
        r["flags"] |= device.JOINT_ENABLE_LIMIT
        r["lowerAngle"], r["upperAngle"] = limit
    if motor is not None:
        r["flags"] |= device.JOINT_ENABLE_MOTOR
        r["motorSpeed"], r["maxMotorTorque"] = motor
    rows[0] = r
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
    return history, ctx


def _angle(bodies, i):
    return math.atan2(float(bodies["rot"][i][0]), float(bodies["rot"][i][1]))


def _frame(bodies, joint):
    """(translation, perpendicular offset, angle error, world axis) of one prismatic row, in float64."""
    a, b = int(joint["bodyA"]), int(joint["bodyB"])
    p = []
    for i, name in ((a, "localOriginAnchorA"), (b, "localOriginAnchorB")):
        s, c = (float(v) for v in bodies["rot"][i])
        lx, ly = (float(v) for v in joint[name])
        p.append(np.array([c * lx - s * ly, s * lx + c * ly]) + bodies["origin"][i].astype(np.float64))
    s, c = (float(v) for v in bodies["rot"][a])
    lx, ly = (float(v) for v in joint["localAxisA"])
    axis = np.array([c * lx - s * ly, s * lx + c * ly])
    d = p[1] - p[0]
    err = _angle(bodies, b) - _angle(bodies, a) - float(joint["referenceAngle"])
    err = (err + math.pi) % (2.0 * math.pi) - math.pi
    return float(axis @ d), float(-axis[1] * d[0] + axis[0] * d[1]), err, axis


def _incline():
    # static A at the origin turned by 10 degrees, its axis 20 degrees further: the world axis is at 30 degrees
    b = _bodies([(capi.STATIC_BODY, 0.0, 0.0, math.radians(10.0), 0, 0, 0),
                 (capi.DYNAMIC_BODY, 0.0, 0.0, 0.3, 0, 0, 0)])
    return b, _prismatic(b, 0, 1, (0.0, 0.0), (math.cos(math.radians(20.0)), math.sin(math.radians(20.0))), ref=0.3 - math.radians(10.0))


def _vertical(limit=None, motor=None, v=0.0):
    b = _bodies([(capi.STATIC_BODY, 0.0, 0.0, 0.0, 0, 0, 0), (capi.DYNAMIC_BODY, 0.0, 2.0, 0.0, 0.0, v, 0)])
    return b, _prismatic(b, 0, 1, (0.0, 2.0), (0.0, 2.0), limit=limit, motor=motor)


# ---- the checks ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", VARIANTS)
def test_at_rest(solver):
    """A satisfied joint with limits around it, no gravity and no motion stays exactly where it is, with zero impulses."""
    bodies, joints = _vertical(limit=(-0.5, 0.5))
    history, _ = _run(solver, bodies, joints, 30)
    final, fj = history[-1]
    assert np.array_equal(final["position"], bodies["position"])
    assert np.array_equal(final["rot"], bodies["rot"])
    assert not np.any(final["linearVelocity"]) and not np.any(final["angularVelocity"])
    for name in ("impulse", "motorImpulse", "lowerImpulse", "upperImpulse"):
        assert not np.any(fj[name]), name


@pytest.mark.parametrize("solver", VARIANTS)
def test_free_slider_on_incline(solver):
    """No friction, no limit: the slider accelerates down the 30-degree axis at g sin 30 and stays on the axis."""
    bodies, joints = _incline()
    history, _ = _run(solver, bodies, joints, 60, gravity=(0.0, -G))
    final, _ = history[-1]
    _, _, _, axis = _frame(final, joints[0])
    speed = float(axis @ final["linearVelocity"][1].astype(np.float64))
    expected = -G * SIN30 * 60 * DT
    assert abs(speed - expected) <= INCLINE_SPEED_REL * abs(expected), (speed, expected)
    for b, _ in history:
        _, perp, ang, _ = _frame(b, joints[0])
        assert abs(perp) <= INCLINE_PERP_BOUND and abs(ang) <= INCLINE_ANGLE_BOUND, (perp, ang)


@pytest.mark.parametrize("solver", VARIANTS)
def test_limit_hit_at_speed(solver):
    """Thrown at 5 m/s along the axis with no gravity, the slider stops at the upper limit within the band."""
    bodies, joints = _vertical(limit=(-0.5, 0.5), v=5.0)
    history, _ = _run(solver, bodies, joints, 60)
    worst = max(_frame(b, joints[0])[0] for b, _ in history)
    assert worst <= 0.5 + LIMIT_BAND, worst
    assert _frame(history[-1][0], joints[0])[0] >= -0.5 - LIMIT_BAND


@pytest.mark.parametrize("solver", VARIANTS)
def test_limit_rests_under_gravity(solver):
    """Under gravity the slider falls onto its lower limit and rests there within the band."""
    bodies, joints = _vertical(limit=(-0.5, 0.5))
    history, _ = _run(solver, bodies, joints, 120, gravity=(0.0, -G))
    t = _frame(history[-1][0], joints[0])[0]
    assert abs(t + 0.5) <= LIMIT_REST_BAND, t
    if solver != "XPBD":  # XPBD keeps no impulses
        assert history[-1][1]["lowerImpulse"][0] > 0.0


@pytest.mark.parametrize("solver", [v for v in VARIANTS if v != "XPBD"])
def test_motor_reaches_speed(solver):
    """A motor with force to spare lifts the 10 N load at its speed."""
    bodies, joints = _vertical(motor=(1.0, 50.0))
    history, _ = _run(solver, bodies, joints, 60, gravity=(0.0, -G))
    v = float(history[-1][0]["linearVelocity"][1][1])
    assert abs(v - 1.0) <= MOTOR_SPEED_REL, v


@pytest.mark.parametrize("solver", [v for v in VARIANTS if v != "XPBD"])
def test_weak_motor_sinks(solver):
    """A motor whose 4 N cap is below the 10 N load sinks at g - F/m, pushing with its full force."""
    force = 4.0
    bodies, joints = _vertical(motor=(1.0, force))
    history, ctx = _run(solver, bodies, joints, 60, gravity=(0.0, -G))
    v0 = float(history[29][0]["linearVelocity"][1][1])
    v1 = float(history[59][0]["linearVelocity"][1][1])
    accel = (v1 - v0) / (30 * DT)
    if solver not in WEAK_ACCEL_SKIP:
        assert abs(accel + (G - force / MASS)) <= WEAK_ACCEL_REL * (G - force / MASS), accel
    # the motor impulse is per solver step h (a sub-step for the sub-stepping variants)
    reported = float(history[-1][1]["motorImpulse"][0]) / ctx.h
    assert abs(reported - force) <= WEAK_FORCE_REL * force, reported


@pytest.mark.parametrize("solver", VARIANTS)
def test_free_pair(solver):
    """Two free boxes joined on a tilted axis, thrown apart and spinning with no gravity: linear momentum is conserved
    and B stays on A's axis at the reference angle."""
    b = _bodies([(capi.DYNAMIC_BODY, 0.0, 0.0, 0.2, -1.0, 0.5, 1.0), (capi.DYNAMIC_BODY, 1.0, 0.5, 0.5, 2.0, 1.0, 1.0)])
    joints = _prismatic(b, 0, 1, (1.0, 0.5), (math.cos(0.26), math.sin(0.26)), ref=0.3)
    p0 = b["linearVelocity"].astype(np.float64).sum(axis=0) * MASS
    history, _ = _run(solver, b, joints, 60)
    for bodies, _ in history:
        p = bodies["linearVelocity"].astype(np.float64).sum(axis=0) * MASS
        assert np.abs(p - p0).max() <= PAIR_MOMENTUM_BOUND, p - p0
        _, perp, ang, _ = _frame(bodies, joints[0])
        assert abs(perp) <= PAIR_PERP_BOUND and abs(ang) <= PAIR_ANGLE_BOUND, (perp, ang)


if __name__ == "__main__":
    # print the measured quantities the bounds above come from
    for solver in VARIANTS:
        bodies, joints = _incline()
        h, _ = _run(solver, bodies, joints, 60, gravity=(0.0, -G))
        axis = _frame(h[-1][0], joints[0])[3]
        speed = float(axis @ h[-1][0]["linearVelocity"][1].astype(np.float64))
        inc = (abs(speed / (-G * SIN30) - 1.0), max(abs(_frame(b, joints[0])[1]) for b, _ in h),
               max(abs(_frame(b, joints[0])[2]) for b, _ in h))
        bodies, joints = _vertical(limit=(-0.5, 0.5), v=5.0)
        h, _ = _run(solver, bodies, joints, 60)
        hit = max(_frame(b, joints[0])[0] for b, _ in h) - 0.5
        bodies, joints = _vertical(limit=(-0.5, 0.5))
        h, _ = _run(solver, bodies, joints, 120, gravity=(0.0, -G))
        rest = abs(_frame(h[-1][0], joints[0])[0] + 0.5)
        mot = weak = force = float("nan")
        if solver != "XPBD":
            bodies, joints = _vertical(motor=(1.0, 50.0))
            h, _ = _run(solver, bodies, joints, 60, gravity=(0.0, -G))
            mot = abs(float(h[-1][0]["linearVelocity"][1][1]) - 1.0)
            bodies, joints = _vertical(motor=(1.0, 4.0))
            h, ctx = _run(solver, bodies, joints, 60, gravity=(0.0, -G))
            acc = (float(h[59][0]["linearVelocity"][1][1]) - float(h[29][0]["linearVelocity"][1][1])) / (30 * DT)
            weak = abs(acc / -6.0 - 1.0)
            force = abs(float(h[-1][1]["motorImpulse"][0]) / ctx.h / 4.0 - 1.0)
        b = _bodies([(capi.DYNAMIC_BODY, 0.0, 0.0, 0.2, -1.0, 0.5, 1.0), (capi.DYNAMIC_BODY, 1.0, 0.5, 0.5, 2.0, 1.0, 1.0)])
        joints = _prismatic(b, 0, 1, (1.0, 0.5), (math.cos(0.26), math.sin(0.26)), ref=0.3)
        p0 = b["linearVelocity"].astype(np.float64).sum(axis=0)
        h, _ = _run(solver, b, joints, 60)
        mom = max(float(np.abs(x["linearVelocity"].astype(np.float64).sum(axis=0) - p0).max()) for x, _ in h)
        pp = max(abs(_frame(x, joints[0])[1]) for x, _ in h)
        pa = max(abs(_frame(x, joints[0])[2]) for x, _ in h)
        print(f"{solver:14s} incline {inc[0]:.1e} {inc[1]:.1e} {inc[2]:.1e}  hit {hit:.3f} rest {rest:.1e}  "
              f"motor {mot:.1e} weak {weak:.1e} force {force:.1e}  pair {mom:.1e} {pp:.1e} {pa:.1e}")
