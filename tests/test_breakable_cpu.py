"""CPU: joint reactions (s2MakeJointReaction, include/solver2d_b200.h, DESIGN.md §3.13) on oracle rows and hand-built rows.

* Static load: a 2 kg box hangs at rest from a static body on each of the five joint types, solved by the oracle (the joint
  oracle for the weld, prismatic and motor joints) under every variant. The reaction at the rate of the variant must read the
  weight, (0, m g), and no torque. Under XPBD the revolute, weld, prismatic and motor joints are position rows that keep no
  impulses and read exactly zero.
* The mouse joint does not hold a hanging load under TGS_Sticky and XPBD, in the oracle as in the reference: after 3 s the
  box still falls (at 2.5 m/s under TGS_Sticky; at 30 m/s, free fall, under XPBD, whose velocities are derived from the
  positions after the velocity rows ran), so there is no load at rest to read. Under XPBD its impulse still accumulates and
  is reported, so a mouse joint can break there. The test pins that the box is not at rest.
* The sign convention (the force is the one on body B) and the prismatic joint's split along and across its turned axis.
* The exported host function against a float32 numpy statement of the table, bit for bit, on random rows.

The static-load bounds were measured on these deterministic runs (the largest value over the variants, printed by
`python tests/test_breakable_cpu.py`) and keep the margin stated next to each.

Mutations each test catches: a sub-stepping variant read at 1 / dt (or TGS_Sticky at 1 / h) is off by the sub-step count in
the static load; a limit impulse added with the wrong sign, a prismatic axis left in body A's frame or the perpendicular
turned the wrong way fail the table and split checks."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import joint_oracle  # noqa: E402
from oracle import port  # noqa: E402
from solver2d_b200 import capi, device  # noqa: E402

VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]
TYPES = ["revolute", "mouse", "weld", "prismatic", "motor"]
DT = 1.0 / 60.0
ITERS = 4
G = 10.0
MASS = 2.0
HX, HY = 0.5, 0.25
INERTIA = MASS * ((2 * HX) ** 2 + (2 * HY) ** 2) / 12.0
STEPS = 180  # 3 s: the mouse joint's 5 Hz spring has settled

# measured maxima over the variants (see the module docstring) and the margin each bound keeps
LOAD_REL = 1e-5  # |F - (0, m g)| / (m g) of the rigid types; measured 0 (exactly m g) for every variant that holds them
MOUSE_LOAD_REL = 1e-5  # the mouse joint's soft spring after 3 s; measured 8.6e-7 (the sub-stepping variants), x ~10
TORQUE_BOUND = 1e-6  # N-m; measured 0 for every type and variant: the anchor is at B's centre of mass


def _lib():
    return capi.Solver2D(device.LIB_PATH)


def _oracle(kind):
    return port.load() if kind in ("revolute", "mouse") else joint_oracle.load()


def _bodies(a_kind=capi.STATIC_BODY, b_kind=capi.DYNAMIC_BODY, a_y=0.0, b_y=-1.0):
    rows = np.zeros(2, dtype=device.BODY_ROW)
    for i, (kind, y) in enumerate(((a_kind, a_y), (b_kind, b_y))):
        r = rows[i]
        r["index"] = i
        r["flags"] = device.ROW_VALID | (kind << 1)
        r["origin"] = (0.0, y)
        r["position"] = (0.0, y)
        r["rot"] = (0.0, 1.0)
        r["gravityScale"] = 1.0
        if kind == capi.DYNAMIC_BODY:
            r["mass"], r["invMass"] = MASS, 1.0 / MASS
            r["I"], r["invI"] = INERTIA, 1.0 / INERTIA
        rows[i] = r
    return rows


def _joint(kind, a=0, b=1, offset=-1.0):
    """Body B's origin (its centre of mass) `offset` m above body A's origin, joined there."""
    rows = np.zeros(1, dtype=device.JOINT_ROW)
    r = rows[0]
    r["index"] = 0
    code = {"revolute": device.JOINT_REVOLUTE, "mouse": device.JOINT_MOUSE, "weld": device.JOINT_WELD,
            "prismatic": device.JOINT_PRISMATIC, "motor": device.JOINT_MOTOR}[kind]
    r["flags"] = device.ROW_VALID | (code << 1)
    r["bodyA"], r["bodyB"] = a, b
    r["localOriginAnchorA"] = (0.0, offset)
    if kind == "mouse":
        r["target"] = (0.0, offset)
        r["hertz"], r["dampingRatio"] = 5.0, 0.7
    elif kind == "prismatic":
        r["localAxisA"] = (1.0, 0.0)
    elif kind == "motor":
        r["maxMotorTorque"] = 1000.0
        r["hertz"] = 1000.0  # max force
        r["dampingRatio"] = 0.3
    rows[0] = r
    return rows


def _settle(kind, solver, bodies, joints, gravity=(0.0, -G)):
    O = _oracle(kind)
    ctx = device.make_context(solver, DT, ITERS, 2)
    contacts = np.zeros(0, dtype=device.CONTACT_ROW)
    for _ in range(STEPS):
        bodies, _, joints = O.solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, gravity=gravity)
        bodies["origin"] = bodies["position"]
    return bodies, joints, ctx


def _rate(solver, ctx):
    """The table's rate: TGS_Sticky accumulates a step's joint impulses over all sub-steps, the others over one step h."""
    return ctx.inv_dt if solver == "TGS_Sticky" else ctx.inv_h


def _reaction(L, row, rot_a, rate):
    r = L.s2ComputeJointReaction((int(row["flags"]) >> 1) & 7, capi.Vec2(*row["impulse"]), float(row["motorImpulse"]),
                                 float(row["lowerImpulse"]), float(row["upperImpulse"]),
                                 capi.Rot(float(rot_a[0]), float(rot_a[1])), capi.Vec2(*row["localAxisA"]), rate)
    return np.array([r.force.x, r.force.y, r.torque], dtype=np.float32)


def _static_load(kind, solver):
    L = _lib()
    bodies, joints, ctx = _settle(kind, solver, _bodies(), _joint(kind))
    return _reaction(L, joints[0], bodies["rot"][0], _rate(solver, ctx)), bodies


# ---- the checks ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", VARIANTS)
@pytest.mark.parametrize("kind", TYPES)
def test_static_load(kind, solver):
    """A body of mass m hanging at rest reads F = (0, m g) and T = 0 at its variant's rate."""
    got, bodies = _static_load(kind, solver)
    weight = MASS * G
    if kind == "mouse" and solver in ("TGS_Sticky", "XPBD"):
        assert float(bodies["linearVelocity"][1][1]) < -1.0  # (not at rest: see the module docstring)
        assert got[1] > 0.0  # still pulled up
        return
    if solver == "XPBD" and kind != "mouse":
        assert not np.any(got), got  # position rows: no impulses are kept
        return
    assert abs(float(bodies["linearVelocity"][1][1])) < 1e-2  # (at rest)
    bound = MOUSE_LOAD_REL if kind == "mouse" else LOAD_REL
    err = math.hypot(float(got[0]), float(got[1]) - weight) / weight
    assert err <= bound, (got, err)
    assert abs(float(got[2])) <= TORQUE_BOUND, got


@pytest.mark.parametrize("kind", ["revolute", "weld", "motor"])
def test_swapped_bodies_read_the_opposite_force(kind):
    """The force is the one on body B: a body hanging below a static anchor is pulled up (+y); the same joint with the
    bodies swapped (the static anchor is B) reads the opposite force."""
    up, _ = _static_load(kind, "PGS")
    assert up[1] > 0.0
    L = _lib()
    b = _bodies(a_kind=capi.DYNAMIC_BODY, b_kind=capi.STATIC_BODY, a_y=-1.0, b_y=0.0)
    bodies, joints, ctx = _settle(kind, "PGS", b, _joint(kind, a=0, b=1, offset=1.0))
    down = _reaction(L, joints[0], bodies["rot"][0], ctx.inv_h)
    assert down[1] < 0.0
    assert abs(float(down[1]) + float(up[1])) <= LOAD_REL * MASS * G, (up, down)


def test_prismatic_force_splits_along_the_turned_axis():
    """A prismatic row's perpendicular impulse acts along leftPerp(axis) and its axial impulses along axis = qA localAxisA."""
    L = _lib()
    row = _joint("prismatic")[0]
    row["localAxisA"] = (0.6, 0.8)
    row["impulse"] = (2.0, 0.5)  # (perpendicular, angular)
    row["motorImpulse"], row["lowerImpulse"], row["upperImpulse"] = 1.0, 0.25, 0.0
    angle = 0.3
    q = (math.sin(angle), math.cos(angle))
    got = _reaction(L, row, q, 10.0).astype(np.float64)
    axis = np.array([q[1] * 0.6 - q[0] * 0.8, q[0] * 0.6 + q[1] * 0.8])
    perp = np.array([-axis[1], axis[0]])
    assert abs(float(got[:2] @ axis) - 10.0 * 1.25) < 1e-5
    assert abs(float(got[:2] @ perp) - 10.0 * 2.0) < 1e-5
    assert float(got[2]) == np.float32(5.0)


def _table(kind, imp, motor, lower, upper, q, axis, rate):
    """The reaction table in float32 numpy, one rounding per operation in the order of the header."""
    f = np.float32
    imp, q, axis = imp.astype(f), q.astype(f), axis.astype(f)
    motor, lower, upper, rate = f(motor), f(lower), f(upper), f(rate)
    fx, fy, t = imp[0], imp[1], motor
    if kind == device.JOINT_REVOLUTE:
        t = motor + lower - upper
    elif kind == device.JOINT_PRISMATIC:
        ax = q[1] * axis[0] - q[0] * axis[1]
        ay = q[0] * axis[0] + q[1] * axis[1]
        px, py = -ay, ax
        axial = motor + lower - upper
        fx = imp[0] * px + axial * ax
        fy = imp[0] * py + axial * ay
        t = imp[1]
    return np.array([rate * fx, rate * fy, rate * t], dtype=f)


def test_host_function_equals_numpy_table_bit_for_bit():
    L = _lib()
    rng = np.random.default_rng(7)
    for _ in range(2000):
        kind = int(rng.integers(0, 5))
        imp = rng.normal(0.0, 3.0, 2).astype(np.float32)
        motor, lower, upper = (np.float32(v) for v in rng.normal(0.0, 2.0, 3))
        angle = rng.uniform(-math.pi, math.pi)
        q = np.array([math.sin(angle), math.cos(angle)], dtype=np.float32)
        a = rng.uniform(-math.pi, math.pi)
        axis = np.array([math.cos(a), math.sin(a)], dtype=np.float32)
        rate = np.float32(rng.choice([60.0, 240.0, 1.0 / 3.0, 0.0]))
        r = L.s2ComputeJointReaction(kind, capi.Vec2(*imp), float(motor), float(lower), float(upper), capi.Rot(*q),
                                     capi.Vec2(*axis), float(rate))
        got = np.array([r.force.x, r.force.y, r.torque], dtype=np.float32)
        want = _table(kind, imp, motor, lower, upper, q, axis, rate)
        assert got.tobytes() == want.tobytes(), (kind, got, want)


def test_reaction_struct_layout():
    assert C.sizeof(capi.JointReaction) == 12


if __name__ == "__main__":
    # print the measured quantities the bounds above come from
    for kind in TYPES:
        for solver in VARIANTS:
            got, bodies = _static_load(kind, solver)
            err = math.hypot(float(got[0]), float(got[1]) - MASS * G) / (MASS * G)
            print(f"{kind:10s} {solver:14s} F = ({got[0]: .6e}, {got[1]: .6e})  rel {err:.1e}  T {got[2]: .1e}  "
                  f"vy {float(bodies['linearVelocity'][1][1]): .1e}")
