"""CPU: the motor joint in the joint oracle (tests/joint_oracle.c, DESIGN.md §3.10) on hand-built rows, for all ten variants.

No contacts and every local centre at zero, so finalize is the identity (origin == position) and solver stages chain
directly. The bounds below were measured on these deterministic runs (the largest value over the ten variants, printed by
`python tests/test_motor_cpu.py`) and carry the margin stated next to each.

Mutations each test catches: a bias left out of the relax pass or an impulse kept cold breaks `at rest` or the
convergence; a cap applied per component instead of to the length, or at the wrong bound, breaks the weak-motor and
torque-cap tests; an impulse applied to one body only breaks the momentum test; an angle error that is not unwound turns
the seam test the long way round."""
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
ITERS = 4
G = 10.0
HX, HY = 0.5, 0.25  # box half extents
MASS = 1.0
INERTIA = MASS * ((2 * HX) ** 2 + (2 * HY) ** 2) / 12.0

# measured maxima over the ten variants (see the module docstring) and the margin each bound keeps
CONVERGE_LINEAR = 1e-5      # m after 2 s from 2.2 m away; measured 1.4e-7 (the PGS family), x ~70
CONVERGE_ANGULAR = 1e-5     # rad after 2 s from 0.5 rad; measured 1.5e-7, x ~70
WEAK_ACCEL_REL = 1e-4       # relative error of g - F/m; measured 9.1e-6 (SoftStep, TGS_Soft), x ~10
WEAK_FORCE_REL = 1e-5       # the clamped impulse is h F: measured 0, up to float round-off
TORQUE_ACCEL_REL = 1e-5     # relative error of (T - Tmax) / I; measured 1.2e-6 (TGS_Sticky), x ~8
XPBD_TORQUE_REL = 0.05      # XPBD caps a rotation, not an impulse; measured 1.8e-2, x ~3
MOMENTUM_BOUND = 5e-5       # measured 6.4e-6 (XPBD), x ~8: float32 round-off of 60 steps at |p| ~ 3
SEAM_BOUND = 1e-6           # rad: every variant ends within this of the target; measured 5.9e-8, x ~17
# TGS_Sticky prepares its joints cold once per step and accumulates their impulses over the sub-steps, so a cap h F (h a
# sub-step) holds for the whole step: a weak motor pushes with F / ITERS and the load sinks at g - F / (ITERS m). The
# impulse still sits at its cap, which the force check covers.
PER_STEP_CAP = {"TGS_Sticky"}


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


def _motor(a, b, offset=(0.0, 0.0), angle=0.0, max_force=1000.0, max_torque=1000.0, cf=0.3):
    rows = np.zeros(1, dtype=device.JOINT_ROW)
    r = rows[0]
    r["index"] = 0
    r["flags"] = device.ROW_VALID | (device.JOINT_MOTOR << 1)
    r["bodyA"], r["bodyB"] = a, b
    r["localOriginAnchorA"] = offset
    r["referenceAngle"] = angle
    r["maxMotorTorque"] = max_torque
    r["hertz"] = max_force
    r["dampingRatio"] = cf
    rows[0] = r
    return rows


def _run(solver, bodies, joints, steps, gravity=(0.0, 0.0), torque=None):
    O = joint_oracle.load()
    ctx = device.make_context(solver, DT, ITERS, 2)
    contacts = np.zeros(0, dtype=device.CONTACT_ROW)
    history = []
    for _ in range(steps):
        if torque is not None:
            bodies["torque"] = torque
        bodies, _, joints = O.solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, gravity=gravity)
        bodies["origin"] = bodies["position"]
        history.append((bodies.copy(), joints.copy()))
    return history, ctx


def _angle(bodies, i):
    return math.atan2(float(bodies["rot"][i][0]), float(bodies["rot"][i][1]))


def _error(bodies, joint):
    """(linear, angular) pose error of one motor row, in float64: B's origin against A's offset point, and the unwound
    relative angle against the angular offset."""
    a, b = int(joint["bodyA"]), int(joint["bodyB"])
    s, c = (float(v) for v in bodies["rot"][a])
    ox, oy = (float(v) for v in joint["localOriginAnchorA"])
    target = bodies["origin"][a].astype(np.float64) + np.array([c * ox - s * oy, s * ox + c * oy])
    lin = float(np.linalg.norm(bodies["origin"][b].astype(np.float64) - target))
    ang = _angle(bodies, b) - _angle(bodies, a) - float(joint["referenceAngle"])
    ang = (ang + math.pi) % (2.0 * math.pi) - math.pi
    return lin, ang


def _converge_case():
    b = _bodies([(capi.STATIC_BODY, 0.0, 0.0, 0.2, 0, 0, 0), (capi.DYNAMIC_BODY, 0.0, 0.0, 0.0, 0, 0, 0)])
    # caps well above what the drive asks for (cf C / h of up to 160 m/s in a 1/240 s sub-step)
    return b, _motor(0, 1, offset=(2.0, 1.0), angle=0.5, max_force=1e5, max_torque=1e5)


def _hanging_case(max_force):
    b = _bodies([(capi.STATIC_BODY, 0.0, 0.0, 0.0, 0, 0, 0), (capi.DYNAMIC_BODY, 0.0, -1.0, 0.0, 0, 0, 0)])
    return b, _motor(0, 1, offset=(0.0, -1.0), max_force=max_force)


def _weak_accel(history, lo=29, hi=59, axis=1, angular=False):
    if angular:
        v0 = float(history[lo][0]["angularVelocity"][1])
        v1 = float(history[hi][0]["angularVelocity"][1])
    else:
        v0 = float(history[lo][0]["linearVelocity"][1][axis])
        v1 = float(history[hi][0]["linearVelocity"][1][axis])
    return (v1 - v0) / ((hi - lo) * DT)


# ---- the checks ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", VARIANTS)
def test_satisfied_joint_stays_still(solver):
    """B already at the offset with the angle at the angular offset, no gravity and no motion: nothing moves, bit for bit,
    and the impulses stay zero."""
    bodies = _bodies([(capi.STATIC_BODY, 0.0, 0.0, 0.0, 0, 0, 0), (capi.DYNAMIC_BODY, 1.0, 0.5, 0.0, 0, 0, 0)])
    joints = _motor(0, 1, offset=(1.0, 0.5))
    history, _ = _run(solver, bodies, joints, 30)
    final, fj = history[-1]
    assert np.array_equal(final["position"], bodies["position"])
    assert np.array_equal(final["rot"], bodies["rot"])
    assert not np.any(final["linearVelocity"]) and not np.any(final["angularVelocity"])
    for name in ("impulse", "motorImpulse", "lowerImpulse", "upperImpulse"):
        assert not np.any(fj[name]), name


@pytest.mark.parametrize("solver", VARIANTS)
def test_reachable_offset_converges(solver):
    """A free body, no gravity, 2.2 m and 0.5 rad from its target in a turned static frame, with force to spare: it reaches
    the pose. Under the velocity forms the error never grows from one step to the next."""
    bodies, joints = _converge_case()
    history, _ = _run(solver, bodies, joints, 120)
    errors = [_error(b, joints[0]) for b, _ in history]
    lin, ang = errors[-1]
    assert lin <= CONVERGE_LINEAR and abs(ang) <= CONVERGE_ANGULAR, (lin, ang)
    if solver != "XPBD":
        for (l0, a0), (l1, a1) in zip(errors, errors[1:]):
            assert l1 <= l0 and abs(a1) <= abs(a0), (l0, l1, a0, a1)


@pytest.mark.parametrize("solver", VARIANTS)
def test_weak_motor_sinks(solver):
    """A motor capped at 4 N holding a hanging 10 N load sinks at g - F/m, pushing with its full force (TGS_Sticky at its
    per-step cap, XPBD as a position correction of at most h^2 F per sub-step)."""
    force = 4.0
    bodies, joints = _hanging_case(force)
    history, ctx = _run(solver, bodies, joints, 60, gravity=(0.0, -G))
    expected = -(G - force / (ITERS * MASS if solver in PER_STEP_CAP else MASS))
    accel = _weak_accel(history)
    assert abs(accel - expected) <= WEAK_ACCEL_REL * abs(expected), (accel, expected)
    if solver != "XPBD":  # XPBD keeps no impulses
        # the impulse is per solver step h (a sub-step for the sub-stepping variants)
        reported = float(np.linalg.norm(history[-1][1]["impulse"][0].astype(np.float64))) / ctx.h
        assert abs(reported - force) <= WEAK_FORCE_REL * force, reported


@pytest.mark.parametrize("solver", VARIANTS)
def test_torque_cap(solver):
    """A 2 N-m torque on a body whose motor holds its angle with at most 0.5 N-m: it spins up at (T - Tmax) / I."""
    torque, cap = 2.0, 0.5
    bodies = _bodies([(capi.STATIC_BODY, 0.0, 0.0, 0.0, 0, 0, 0), (capi.DYNAMIC_BODY, 0.0, 0.0, 0.0, 0, 0, 0)])
    joints = _motor(0, 1, max_torque=cap)
    history, ctx = _run(solver, bodies, joints, 60, torque=np.array([0.0, torque], dtype=np.float32))
    expected = (torque - cap / (ITERS if solver in PER_STEP_CAP else 1)) / INERTIA
    accel = _weak_accel(history, lo=5, hi=30, angular=True)  # before the angle error wraps past pi and the drive turns
    bound = XPBD_TORQUE_REL if solver == "XPBD" else TORQUE_ACCEL_REL
    assert abs(accel - expected) <= bound * abs(expected), (accel, expected)
    if solver != "XPBD":
        reported = abs(float(history[-1][1]["motorImpulse"][0])) / ctx.h
        assert abs(reported - cap) <= WEAK_FORCE_REL * cap, reported


@pytest.mark.parametrize("solver", VARIANTS)
def test_free_pair_conserves_momentum(solver):
    """Two free boxes driven toward each other's pose with capped effort, thrown apart and spinning with no gravity: the
    motor's impulses are equal and opposite, so linear momentum is conserved."""
    b = _bodies([(capi.DYNAMIC_BODY, 0.0, 0.0, 0.2, -1.0, 0.5, 1.0), (capi.DYNAMIC_BODY, 1.0, 0.5, 0.5, 2.0, 1.0, 1.0)])
    joints = _motor(0, 1, offset=(1.5, -0.5), angle=1.0, max_force=20.0, max_torque=5.0)
    p0 = b["linearVelocity"].astype(np.float64).sum(axis=0) * MASS
    history, _ = _run(solver, b, joints, 60)
    for bodies, _ in history:
        p = bodies["linearVelocity"].astype(np.float64).sum(axis=0) * MASS
        assert np.abs(p - p0).max() <= MOMENTUM_BOUND, p - p0
    assert _error(history[-1][0], joints[0])[0] < _error(b, joints[0])[0]


@pytest.mark.parametrize("solver", VARIANTS)
def test_angular_offset_across_the_seam(solver):
    """B at +3.0 rad with a target of -3.0 rad: the short way is +0.28 rad through pi. The drive turns B that way and never
    the long way (through 0), and it settles at the target."""
    bodies = _bodies([(capi.STATIC_BODY, 0.0, 0.0, 0.0, 0, 0, 0), (capi.DYNAMIC_BODY, 0.0, 0.0, 3.0, 0, 0, 0)])
    joints = _motor(0, 1, angle=-3.0)
    history, _ = _run(solver, bodies, joints, 120)
    assert float(history[0][0]["angularVelocity"][1]) > 0.0
    for b, _ in history:
        assert abs(_angle(b, 1)) > 2.9, _angle(b, 1)
    assert abs(_error(history[-1][0], joints[0])[1]) <= SEAM_BOUND


if __name__ == "__main__":
    # print the measured quantities the bounds above come from
    for solver in VARIANTS:
        bodies, joints = _converge_case()
        h, _ = _run(solver, bodies, joints, 120)
        lin, ang = _error(h[-1][0], joints[0])
        bodies, joints = _hanging_case(4.0)
        h, ctx = _run(solver, bodies, joints, 60, gravity=(0.0, -G))
        exp = -(G - 4.0 / (ITERS if solver in PER_STEP_CAP else 1))
        weak = abs(_weak_accel(h) / exp - 1.0)
        force = abs(float(np.linalg.norm(h[-1][1]["impulse"][0].astype(np.float64))) / ctx.h / 4.0 - 1.0)
        bodies = _bodies([(capi.STATIC_BODY, 0.0, 0.0, 0.0, 0, 0, 0), (capi.DYNAMIC_BODY, 0.0, 0.0, 0.0, 0, 0, 0)])
        h, _ = _run(solver, bodies, _motor(0, 1, max_torque=0.5), 60, torque=np.array([0.0, 2.0], dtype=np.float32))
        texp = (2.0 - 0.5 / (ITERS if solver in PER_STEP_CAP else 1)) / INERTIA
        tq = abs(_weak_accel(h, lo=5, hi=30, angular=True) / texp - 1.0)
        b = _bodies([(capi.DYNAMIC_BODY, 0.0, 0.0, 0.2, -1.0, 0.5, 1.0), (capi.DYNAMIC_BODY, 1.0, 0.5, 0.5, 2.0, 1.0, 1.0)])
        p0 = b["linearVelocity"].astype(np.float64).sum(axis=0)
        h, _ = _run(solver, b, _motor(0, 1, offset=(1.5, -0.5), angle=1.0, max_force=20.0, max_torque=5.0), 60)
        mom = max(float(np.abs(x["linearVelocity"].astype(np.float64).sum(axis=0) - p0).max()) for x, _ in h)
        bodies = _bodies([(capi.STATIC_BODY, 0.0, 0.0, 0.0, 0, 0, 0), (capi.DYNAMIC_BODY, 0.0, 0.0, 3.0, 0, 0, 0)])
        joints = _motor(0, 1, angle=-3.0)
        h, _ = _run(solver, bodies, joints, 120)
        seam = abs(_error(h[-1][0], joints[0])[1])
        print(f"{solver:14s} converge {lin:.1e} {abs(ang):.1e}  weak {weak:.1e} force {force:.1e}  torque {tq:.1e}  "
              f"momentum {mom:.1e}  seam {seam:.1e}")
