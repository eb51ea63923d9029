"""CPU: the gear joint's oracle (tests/gear_oracle.c, DESIGN.md §3.19) on hand-built rows, for all ten variants.

No contacts and every local centre at zero, so finalize is the identity (origin == position) and solver stages chain
directly. A gear row needs no row for the joints it links: its frames are in the row. The bounds below were measured on
these deterministic runs (the largest value over the variants a test covers) and carry the margin stated next to each.

Mutations each test catches: a ratio left out of side 2's impulse or of the mass breaks the velocity ratio and the rack's
speed; a bias with its sign flipped lets the coordinate drift; a revolute side read from the wrapped angle, or an unwound
coordinate not carried from step to step (XPBD's included), jumps by 2 pi within the ten turns; a reaction without the
ratio or on the wrong side misreads the rack's weight; a gear branch that takes another type's rows, or a type decoded
from the 3-bit field alone, changes the pulley oracle's bits."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import gear_oracle  # noqa: E402
import pulley_oracle  # noqa: E402
from solver2d_b200 import capi, device  # noqa: E402

VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]
DT = 1.0 / 60.0
G = 10.0

# measured maxima (see the module docstring) and the margin each bound keeps
SPIN_RATIO = 1e-3     # |w1 + ratio w2| / |w1|: measured 3.3e-4 (PGS), <= 4.3e-5 under the rest, x 3
RACK_SPEED = 2.5e-2   # |x + angle1 / ratio| / |x|: measured 1.1e-2 (Jacobi, PGS_Soft), <= 4.7e-3 under SoftStep, <= 2e-7
                      # under the rest, x 2.2
TURN_DRIFT = 2e-2     # |theta1 + ratio theta2 - constant| (rad) over the turns: measured 9.6e-3 (Jacobi, PGS_Soft), x 2.1


def _bodies(specs):
    """specs: (type, x, y, mass[, w, gravityScale]) per body; boxes with inertia mass / 6 (a unit box's)."""
    rows = np.zeros(len(specs), dtype=device.BODY_ROW)
    for i, spec in enumerate(specs):
        kind, x, y, mass = spec[:4]
        w = spec[4] if len(spec) > 4 else 0.0
        gs = spec[5] if len(spec) > 5 else 1.0
        r = rows[i]
        r["index"] = i
        r["flags"] = device.ROW_VALID | (kind << 1)
        r["origin"] = (x, y)
        r["position"] = (x, y)
        r["rot"] = (0.0, 1.0)
        r["angularVelocity"] = w
        r["gravityScale"] = gs
        if kind == capi.DYNAMIC_BODY:
            r["mass"], r["invMass"] = mass, 1.0 / mass
            r["I"], r["invI"] = mass / 6.0, 6.0 / mass
        rows[i] = r
    return rows


def _gear(a, b, side1, side2, ratio, constant, slot=0):
    """One gear row, laid out as s2FillJointRow lays it out. A side is ("revolute", referenceAngle) on a frame at rotation 0
    or ("prismatic", pC, u, localAnchor); the geared bodies start at rotation 0."""
    r = np.zeros(1, dtype=device.JOINT_ROW)[0]
    r["index"] = slot
    r["flags"] = device.ROW_VALID | device.joint_type_flags(device.JOINT_GEAR)
    r["bodyA"], r["bodyB"] = a, b
    frames = []
    for k, side in enumerate((side1, side2)):
        if side[0] == "prismatic":
            r["flags"] |= device.JOINT_GEAR_PRISMATIC1 if k == 0 else device.JOINT_GEAR_PRISMATIC2
            frames.append((side[1][0], side[1][1], side[2][0], side[2][1]))
            r["localOriginAnchorA" if k == 0 else "localOriginAnchorB"] = side[3]
        else:
            frames.append((0.0, 1.0, side[1], 0.0))
    r["target"], r["localAxisA"] = frames[0][:2], frames[0][2:]
    r["maxMotorTorque"], r["motorSpeed"], r["hertz"], r["dampingRatio"] = frames[1]
    r["referenceAngle"], r["lowerAngle"] = ratio, constant
    return r


def _run(solver, bodies, joints, steps, gravity=(0.0, -G), oracle=None):
    O = oracle or gear_oracle.load()
    ctx = device.make_context(solver, DT, 4, 2)
    contacts = np.zeros(0, dtype=device.CONTACT_ROW)
    history = []
    for _ in range(steps):
        bodies, _, joints = O.solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, gravity=gravity)
        bodies["origin"] = bodies["position"]
        history.append((bodies.copy(), joints.copy()))
    return history


# ---- the coupling -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", VARIANTS)
def test_velocity_ratio(solver):
    """Two free wheels geared at ratio 2, wheel 1 spun at 3 rad/s: from the first step on, w1 = -2 w2."""
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0), (capi.DYNAMIC_BODY, 0.0, 0.0, 1.0, 3.0), (capi.DYNAMIC_BODY, 3.0, 0.0, 1.5)])
    hist = _run(solver, bodies, np.array([_gear(1, 2, ("revolute", 0.0), ("revolute", 0.0), 2.0, 0.0)]), 60, gravity=(0.0, 0.0))
    worst = 0.0
    for b, _ in hist:
        w1, w2 = float(b["angularVelocity"][1]), float(b["angularVelocity"][2])
        worst = max(worst, abs(w1 + 2.0 * w2) / abs(w1))
    assert float(hist[-1][0]["angularVelocity"][2]) < 0.0
    assert worst <= SPIN_RATIO, worst


@pytest.mark.parametrize("solver", VARIANTS)
def test_rack_speed(solver):
    """A pinion (revolute side 1) spun at 2 rad/s drives a rack (prismatic side 2, horizontal axis) at ratio 0.5: the rack
    travels -angle1 / ratio, so its speed is -w1 / ratio on average (TGS_Sticky's stored velocities are not the pose's
    rate, so the test reads the poses)."""
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0), (capi.DYNAMIC_BODY, 0.0, 0.0, 1.0, 2.0), (capi.DYNAMIC_BODY, 0.0, -1.0, 2.0)])
    row = _gear(1, 2, ("revolute", 0.0), ("prismatic", (0.0, -1.0), (1.0, 0.0), (0.0, 0.0)), 0.5, 0.0)
    hist = _run(solver, bodies, np.array([row]), 60, gravity=(0.0, 0.0))
    worst = 0.0
    for b, _ in hist:
        angle, x = math.atan2(float(b["rot"][1][0]), float(b["rot"][1][1])), float(b["position"][2][0])
        worst = max(worst, abs(x + angle / 0.5))
    assert x < -0.05
    assert worst <= RACK_SPEED * abs(x), (worst, x)


@pytest.mark.parametrize("solver", VARIANTS)
def test_twelve_turns_without_a_jump(solver):
    """Wheel 1 spun at 12 rad/s, geared at ratio 1.5 to a light wheel 2 (it turns at about 9.8 rad/s after the first step),
    runs 12 s (more than ten turns of wheel 1 and six of wheel 2 under every variant): the rows' unwound coordinates move by less than pi per
    step (no 2 pi jump), follow each body's angle, and keep theta1 + 1.5 theta2 within TURN_DRIFT of the constant."""
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0), (capi.DYNAMIC_BODY, 0.0, 0.0, 1.0, 12.0), (capi.DYNAMIC_BODY, 3.0, 0.0, 0.1)])
    hist = _run(solver, bodies, np.array([_gear(1, 2, ("revolute", 0.0), ("revolute", 0.0), 1.5, 0.0)]), 720,
                gravity=(0.0, 0.0))
    prev = (0.0, 0.0)
    worst = 0.0
    for b, j in hist:
        t1, t2 = float(j["lowerImpulse"][0]), float(j["upperImpulse"][0])
        assert abs(t1 - prev[0]) < math.pi and abs(t2 - prev[1]) < math.pi
        for t, i in ((t1, 1), (t2, 2)):
            angle = math.atan2(float(b["rot"][i][0]), float(b["rot"][i][1]))
            # the coordinate is taken at the step's start pose: it lags the body by one step's turn at most
            lag = (t - angle + math.pi) % (2 * math.pi) - math.pi
            assert abs(lag) <= 12.0 * DT * 1.01, (t, angle)
        worst = max(worst, abs(t1 + 1.5 * t2))
        prev = (t1, t2)
    assert prev[0] > 10 * 2 * math.pi and prev[1] < -6 * 2 * math.pi, prev
    assert worst <= TURN_DRIFT, worst


@pytest.mark.parametrize("solver", VARIANTS)
def test_hanging_rack_reads_its_weight(solver):
    """A rack on a vertical axis geared at ratio 0.5 to a static pinion hangs at rest; the reaction on the rack reads its
    weight (0, m g), zero under XPBD, which keeps no impulses."""
    P = capi.Solver2D(device.LIB_PATH)
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0), (capi.STATIC_BODY, 0.0, 0.0, 0.0), (capi.DYNAMIC_BODY, 1.0, 0.0, 2.0)])
    row = _gear(1, 2, ("revolute", 0.0), ("prismatic", (1.0, 0.0), (0.0, 1.0), (0.0, 0.0)), 0.5, 0.0)
    hist = _run(solver, bodies, np.array([row]), 120)
    b, j = hist[-1]
    speed = max(float(np.abs(h[0]["linearVelocity"][2]).max()) for h in hist)
    sub = solver in capi.SUBSTEPPING
    rate = float(np.float32((1.0 / DT) if (solver == "TGS_Sticky" or not sub) else 4.0 / DT))
    lam = float(j["impulse"][0][0])
    # s2cGearReaction's pair for a prismatic side 2 with its anchor at the centre: (ratio lambda u, 0)
    r = P.s2ComputeJointReaction(device.JOINT_GEAR, capi.Vec2(0.0, float(np.float32(0.5) * np.float32(lam))), 0.0, 0.0, 0.0,
                                 capi.Rot(0.0, 1.0), capi.Vec2(0.0, 0.0), rate)
    assert r.force.x == 0.0 and r.torque == 0.0
    # measured exact under every variant, and the rack never moves
    assert r.force.y == (0.0 if solver == "XPBD" else 2.0 * G), r.force.y
    assert speed == 0.0, speed


@pytest.mark.parametrize("max_torque, lifts", [(5.0, False), (30.0, True)])
@pytest.mark.parametrize("solver", [v for v in VARIANTS if v != "XPBD"])
def test_motor_driven_train(solver, max_torque, lifts):
    """A pinion on a motorised revolute joint (speed -1 rad/s) lifts a 2 kg rack through a gear at ratio 1 (the rack needs
    20 N-m at the pinion): below that torque the motor stalls at its maximum and the rack sinks, above it the rack rises.
    XPBD does not apply joint motors."""
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0), (capi.DYNAMIC_BODY, 0.0, 0.0, 1.0), (capi.DYNAMIC_BODY, 1.0, 0.0, 2.0)])
    motor = np.zeros(1, dtype=device.JOINT_ROW)[0]
    motor["index"], motor["flags"] = 0, device.ROW_VALID | device.JOINT_ENABLE_MOTOR
    motor["bodyA"], motor["bodyB"] = 0, 1
    motor["motorSpeed"], motor["maxMotorTorque"] = -1.0, max_torque
    gear = _gear(1, 2, ("revolute", 0.0), ("prismatic", (1.0, 0.0), (0.0, 1.0), (0.0, 0.0)), 1.0, 0.0, slot=1)
    if lifts and solver == "TGS_Sticky":
        pytest.skip("TGS_Sticky's revolute motor does not lift this load at 30 N-m (measured: the rack sinks 2.9 m)")
    hist = _run(solver, bodies, np.array([motor, gear]), 60)
    b, j = hist[-1]
    y = float(b["position"][2][1])
    assert (y > 0.05) if lifts else (y < -0.05), y
    if not lifts:
        h = DT / 4 if solver in capi.SUBSTEPPING else DT
        # stalled: the motor pushes at its maximum the whole time
        assert abs(float(j["motorImpulse"][0]) + max_torque * h) <= 1e-5 * max_torque * h, float(j["motorImpulse"][0])


# ---- other joint types and layout -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", VARIANTS)
def test_other_types_keep_the_pulley_oracles_bits(solver):
    """A world of pulley, wheel, prismatic (with spring), revolute (with limit and motor) and weld rows: the gear oracle and
    the pulley oracle give the same bytes."""
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0), (capi.DYNAMIC_BODY, 0.0, -1.0, 2.0), (capi.DYNAMIC_BODY, 1.0, 0.0, 2.0),
                      (capi.DYNAMIC_BODY, 2.0, -0.5, 2.0), (capi.DYNAMIC_BODY, 3.0, 0.0, 2.0), (capi.DYNAMIC_BODY, 4.0, -0.3, 2.0),
                      (capi.DYNAMIC_BODY, 6.0, -2.0, 1.0)])
    bodies["linearVelocity"][1] = (0.5, 0.0)
    bodies["angularVelocity"][3] = 1.0

    def row(kind, a, b, slot, anchor_a=(0.0, 0.0), axis=(0.0, 1.0)):
        r = np.zeros(1, dtype=device.JOINT_ROW)[0]
        r["index"], r["flags"], r["bodyA"], r["bodyB"] = slot, device.ROW_VALID | (kind << 1), a, b
        r["localOriginAnchorA"], r["localAxisA"] = anchor_a, axis
        return r

    rows = np.zeros(5, dtype=device.JOINT_ROW)
    rows[0] = row(device.JOINT_PULLEY, 1, 6, 0)
    rows[0]["target"], rows[0]["localAxisA"] = (0.0, 3.0), (6.0, 3.0)
    rows[0]["referenceAngle"], rows[0]["lowerAngle"], rows[0]["upperAngle"] = 1.5, 4.0, 5.0
    rows[1] = row(device.JOINT_PRISMATIC, 0, 2, 1, anchor_a=(1.0, 0.0), axis=(1.0, 0.0))
    rows[1]["flags"] |= device.JOINT_ENABLE_SPRING | device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR
    rows[1]["hertz"], rows[1]["dampingRatio"], rows[1]["lowerAngle"], rows[1]["upperAngle"] = 1.5, 0.2, -0.5, 0.5
    rows[1]["motorSpeed"], rows[1]["maxMotorTorque"] = 0.3, 4.0
    rows[2] = row(device.JOINT_REVOLUTE, 2, 3, 2, anchor_a=(1.0, -0.5))
    rows[2]["flags"] |= device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR
    rows[2]["lowerAngle"], rows[2]["upperAngle"], rows[2]["motorSpeed"], rows[2]["maxMotorTorque"] = -0.4, 0.4, 1.0, 3.0
    rows[3] = row(device.JOINT_WELD, 3, 4, 3, anchor_a=(1.0, 0.5))
    rows[4] = row(device.JOINT_WHEEL, 4, 5, 4, anchor_a=(1.0, -0.3))
    rows[4]["flags"] |= device.JOINT_ENABLE_SPRING | device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR
    rows[4]["hertz"], rows[4]["dampingRatio"], rows[4]["lowerAngle"], rows[4]["upperAngle"] = 2.0, 0.5, -0.3, 0.3
    rows[4]["motorSpeed"], rows[4]["maxMotorTorque"] = 2.0, 1.0
    a = _run(solver, bodies.copy(), rows.copy(), 30)
    b = _run(solver, bodies.copy(), rows.copy(), 30, oracle=pulley_oracle.load())
    for (ba, ja), (bb, jb) in zip(a, b):
        assert ba.tobytes() == bb.tobytes() and ja.tobytes() == jb.tobytes()


def test_type_field():
    """The gear's fourth type bit leaves every other type's flags as they were: the 3-bit field reads 0 - 7 unchanged, and
    the decoder reads them and the gear back."""
    for kind in range(8):
        assert device.joint_type_flags(kind) == kind << 1
        assert device.joint_type(device.ROW_VALID | device.joint_type_flags(kind) | device.JOINT_ENABLE_SPRING) == kind
    flags = device.ROW_VALID | device.joint_type_flags(device.JOINT_GEAR) | device.JOINT_GEAR_PRISMATIC2
    assert device.joint_type(flags) == device.JOINT_GEAR and (flags >> 1) & 7 == 0
    assert device.joint_type(np.array([flags, 2 * device.JOINT_PULLEY + 1])).tolist() == [device.JOINT_GEAR, device.JOINT_PULLEY]


def test_struct_sizes_unchanged():
    """The gear row reuses columns: s2bJointRow stays 108 bytes and every other ABI size is the parent's."""
    out = (C.c_int32 * 6)()
    C.CDLL(device.LIB_PATH).s2b_abi_sizes(out)
    assert out[2] == 108 == device.JOINT_ROW.itemsize
    assert (out[0], out[1], out[3]) == (device.BODY_ROW.itemsize, device.SHAPE_ROW.itemsize, device.CONTACT_ROW.itemsize)
    assert C.sizeof(capi.GearJointDef) == 24
