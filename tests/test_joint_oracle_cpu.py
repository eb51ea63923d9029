"""CPU: the joint oracle (tests/joint_oracle.c) gives the bits its types' separate oracles gave, for all ten variants.

The joint types the reference lacks were once defined by one oracle per type, each built on another. Their bytes, recorded
from those oracles on the hand-built worlds below (tests/golden/make_joint_oracle_golden.py, one truncated sha1 per world
and variant over the body and joint rows of every step), are tests/golden/joint_oracle_sha1.json:
  * for each type, a world with every flag of the type on;
  * the worlds where a type's rows once had to leave every other type's bits alone: revolute, prismatic and mouse rows
    without the spring flag; rigid welds (both hertz at 0) beside revolute and mouse rows; distance, prismatic (with
    spring) and revolute (with limit and motor) rows beside wheels, pulleys and gears. Those oracles solved a weld row
    as a revolute row, so these worlds carry that row as the revolute row it was solved as;
  * revolute and mouse rows alone, which are also checked live against the base oracle (oracle/s2o_solver.c).

No contacts and every local centre at zero, so finalize is the identity (origin == position) and solver stages chain
directly."""
import hashlib
import json
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
DT = 1.0 / 60.0
G = 10.0
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "joint_oracle_sha1.json")
S, D = capi.STATIC_BODY, capi.DYNAMIC_BODY
BOX_INERTIA = (1.0 + 0.25) / 12.0  # a 1 kg box of 1 m x 0.5 m


def _bodies(specs, mass=1.0, inertia=BOX_INERTIA):
    """specs: (type, x, y[, angle, vx, vy, w]) per body; every dynamic body of the given mass and rotational inertia."""
    rows = np.zeros(len(specs), dtype=device.BODY_ROW)
    for i, spec in enumerate(specs):
        kind, x, y = spec[:3]
        angle, vx, vy, w = (tuple(spec[3:]) + (0.0, 0.0, 0.0, 0.0))[:4]
        r = rows[i]
        r["index"] = i
        r["flags"] = device.ROW_VALID | (kind << 1)
        r["origin"] = (x, y)
        r["position"] = (x, y)
        r["rot"] = (np.float32(math.sin(angle)), np.float32(math.cos(angle)))
        r["linearVelocity"] = (vx, vy)
        r["angularVelocity"] = w
        r["gravityScale"] = 1.0
        if kind == D:
            r["mass"], r["invMass"] = mass, 1.0 / mass
            r["I"], r["invI"] = inertia, 1.0 / inertia
        rows[i] = r
    return rows


def _local(bodies, i, p):
    s, c = (float(v) for v in bodies["rot"][i])
    d = np.asarray(p, dtype=np.float64) - bodies["origin"][i].astype(np.float64)
    return (c * d[0] + s * d[1], -s * d[0] + c * d[1])


def _row(kind, a, b, slot, flags=0, **fields):
    r = np.zeros(1, dtype=device.JOINT_ROW)[0]
    r["index"], r["flags"], r["bodyA"], r["bodyB"] = slot, device.ROW_VALID | device.joint_type_flags(kind) | flags, a, b
    for name, value in fields.items():
        r[name] = value
    return r


def _pinned(kind, bodies, a, b, pivot, slot, flags=0, **fields):
    """A row with both anchors at the world point `pivot`."""
    return _row(kind, a, b, slot, flags, localOriginAnchorA=_local(bodies, a, pivot), localOriginAnchorB=_local(bodies, b, pivot),
                **fields)


LIMIT_MOTOR = device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR
ALL = LIMIT_MOTOR | device.JOINT_ENABLE_SPRING
UNIT_AXIS = (np.float32(1.0) / np.float32(math.hypot(1.0, 0.3)), np.float32(0.3) / np.float32(math.hypot(1.0, 0.3)))
MOUSE = dict(localOriginAnchorB=(0.1, 0.0), target=(2.5, 0.5), hertz=5.0, dampingRatio=0.7)


def _three_boxes():
    return _bodies([(S, 0, 0), (D, 0.0, 0.0, 0.1, 0.2, 0.0, 1.0), (D, 1.2, 0.1, 0.0, 0.0, 0.3, -0.5)])


def _four_boxes():
    return _bodies([(S, 0, 0), (D, 0.0, 0.0, 0.1, 0.2, 0.0, 1.0), (D, 1.2, 0.1, 0.0, 0.0, 0.3, -0.5), (D, 2.4, 0.1, 3.1, 0.1, 0.0, 0.2)])


# ---- the worlds -----------------------------------------------------------------------------------------------------------

def world_spring_without_flag():
    """Revolute and prismatic rows with limit and motor and a mouse row, none with the spring flag."""
    b = _three_boxes()
    return b, np.array([
        _pinned(device.JOINT_REVOLUTE, b, 0, 1, (0.0, 0.0), 0, LIMIT_MOTOR, lowerAngle=-0.3, upperAngle=0.4, motorSpeed=1.0,
                maxMotorTorque=5.0),
        _pinned(device.JOINT_PRISMATIC, b, 1, 2, (1.0, 0.0), 1, LIMIT_MOTOR, localAxisA=UNIT_AXIS, lowerAngle=-0.2, upperAngle=0.3,
                motorSpeed=-0.5, maxMotorTorque=8.0),
        _row(device.JOINT_MOUSE, 0, 2, 2, **MOUSE)])


def world_rigid_welds():
    """Rigid welds (one at the seam of the angle), a revolute with limit and motor and a mouse row."""
    b = _four_boxes()
    return b, np.array([
        _pinned(device.JOINT_WELD, b, 0, 1, (0.0, 0.0), 0),
        _pinned(device.JOINT_REVOLUTE, b, 1, 2, (0.6, 0.0), 1, LIMIT_MOTOR, lowerAngle=-0.3, upperAngle=0.4, motorSpeed=1.0,
                maxMotorTorque=5.0),
        _pinned(device.JOINT_WELD, b, 2, 3, (1.8, 0.1), 2, referenceAngle=math.pi - 0.01),
        _row(device.JOINT_MOUSE, 0, 3, 3, **MOUSE)])


def _neighbours():
    """Distance (with spring), prismatic (with spring, limit and motor), revolute (with limit and motor) and a revolute row
    in the weld's place, on bodies 0 - 4 and slots 0 - 3."""
    return [
        _row(device.JOINT_DISTANCE, 0, 1, 0, device.JOINT_ENABLE_SPRING, localAxisA=(0.0, 1.0), referenceAngle=1.0, hertz=2.0,
             dampingRatio=0.3, lowerAngle=0.005, upperAngle=100000.0),
        _row(device.JOINT_PRISMATIC, 0, 2, 1, ALL, localOriginAnchorA=(1.0, 0.0), localAxisA=(1.0, 0.0), hertz=1.5, dampingRatio=0.2,
             lowerAngle=-0.5, upperAngle=0.5, motorSpeed=0.3, maxMotorTorque=4.0),
        _row(device.JOINT_REVOLUTE, 2, 3, 2, LIMIT_MOTOR, localOriginAnchorA=(1.0, -0.5), localAxisA=(0.0, 1.0), lowerAngle=-0.4,
             upperAngle=0.4, motorSpeed=1.0, maxMotorTorque=3.0),
        _row(device.JOINT_REVOLUTE, 3, 4, 3, localOriginAnchorA=(1.0, 0.5), localAxisA=(0.0, 1.0))]


def _wheel_row(a, b, slot, anchor_a=(0.0, 0.0)):
    return _row(device.JOINT_WHEEL, a, b, slot, ALL, localOriginAnchorA=anchor_a, localAxisA=(0.0, 1.0), hertz=2.0, dampingRatio=0.5,
                lowerAngle=-0.3, upperAngle=0.3, motorSpeed=2.0, maxMotorTorque=1.0)


def _pulley_row(a, b, slot):
    return _row(device.JOINT_PULLEY, a, b, slot, target=(0.0, 3.0), localAxisA=(6.0, 3.0), referenceAngle=1.5, lowerAngle=4.0,
                upperAngle=5.0)


def world_wheel_neighbours():
    b = _bodies([(S, 0, 0), (D, 0.0, -1.0, 0.0, 0.0, 0.0, 0.5), (D, 1.0, 0.0), (D, 2.0, -0.5, 0.0, 0.0, 0.0, 1.0), (D, 3.0, 0.0)],
                mass=2.0, inertia=0.1)
    b["linearVelocity"][1] = (0.0, 0.3)
    return b, np.array(_neighbours())


def world_pulley_neighbours():
    b = _bodies([(S, 0, 0), (D, 0.0, -1.0, 0.0, 0.5), (D, 1.0, 0.0), (D, 2.0, -0.5, 0.0, 0.0, 0.0, 1.0), (D, 3.0, 0.0), (D, 4.0, -0.3)],
                mass=2.0, inertia=2.0 / 6.0)
    return b, np.array(_neighbours() + [_wheel_row(4, 5, 4, anchor_a=(1.0, -0.3))])


def world_gear_neighbours():
    b = _bodies([(S, 0, 0), (D, 0.0, -1.0, 0.0, 0.5), (D, 1.0, 0.0), (D, 2.0, -0.5, 0.0, 0.0, 0.0, 1.0), (D, 3.0, 0.0), (D, 4.0, -0.3),
                 (D, 6.0, -2.0)], mass=2.0, inertia=2.0 / 6.0)
    rows = _neighbours()[1:] + [_wheel_row(4, 5, 4, anchor_a=(1.0, -0.3))]
    return b, np.array([_pulley_row(1, 6, 0)] + rows)


def world_weld():
    """A cantilever of two rigid welds, the second at an angle across the seam."""
    b = _four_boxes()
    return b, np.array([_pinned(device.JOINT_WELD, b, 0, 1, (0.0, 0.0), 0, referenceAngle=0.1),
                        _pinned(device.JOINT_WELD, b, 1, 2, (0.6, 0.0), 1),
                        _pinned(device.JOINT_WELD, b, 2, 3, (1.8, 0.1), 2, referenceAngle=math.pi - 0.01)])


def world_soft_weld():
    """Welds soft in both parts, in the anchor only and in the angle only."""
    b = _four_boxes()
    return b, np.array([_pinned(device.JOINT_WELD, b, 0, 1, (0.0, 0.0), 0, hertz=1.5, dampingRatio=0.3, maxMotorTorque=2.0,
                                motorSpeed=0.2),
                        _pinned(device.JOINT_WELD, b, 1, 2, (0.6, 0.0), 1, hertz=3.0, dampingRatio=0.7),
                        _pinned(device.JOINT_WELD, b, 2, 3, (1.8, 0.1), 2, referenceAngle=math.pi - 0.01, maxMotorTorque=1.0,
                                motorSpeed=0.0)])


def world_motor():
    """Motor joints driving to offsets, one on the ground with a force cap that binds."""
    b = _three_boxes()
    return b, np.array([
        _row(device.JOINT_MOTOR, 0, 1, 0, localOriginAnchorA=(0.5, 0.5), referenceAngle=0.7, maxMotorTorque=2.0, hertz=6.0,
             dampingRatio=0.3),
        _row(device.JOINT_MOTOR, 1, 2, 1, localOriginAnchorA=(1.0, -0.2), referenceAngle=-0.4, maxMotorTorque=10.0, hertz=50.0,
             dampingRatio=0.8)])


def world_prismatic():
    b = _three_boxes()
    return b, np.array([
        _pinned(device.JOINT_PRISMATIC, b, 0, 1, (0.0, 0.0), 0, LIMIT_MOTOR, localAxisA=(0.0, 1.0), referenceAngle=0.1, lowerAngle=-0.5,
                upperAngle=0.2, motorSpeed=0.4, maxMotorTorque=3.0),
        _pinned(device.JOINT_PRISMATIC, b, 1, 2, (1.0, 0.0), 1, LIMIT_MOTOR, localAxisA=UNIT_AXIS, lowerAngle=-0.2, upperAngle=0.3,
                motorSpeed=-0.5, maxMotorTorque=8.0)])


def world_spring():
    """A sprung revolute and a sprung prismatic joint, each with limit and motor."""
    b = _three_boxes()
    return b, np.array([
        _pinned(device.JOINT_REVOLUTE, b, 0, 1, (0.0, 0.0), 0, ALL, referenceAngle=0.2, hertz=1.5, dampingRatio=0.2, lowerAngle=-0.3,
                upperAngle=0.4, motorSpeed=1.0, maxMotorTorque=0.5),
        _pinned(device.JOINT_PRISMATIC, b, 1, 2, (1.0, 0.0), 1, ALL, localAxisA=UNIT_AXIS, hertz=2.0, dampingRatio=0.5, lowerAngle=-0.2,
                upperAngle=0.3, motorSpeed=-0.5, maxMotorTorque=1.0)])


def world_distance():
    """A sprung rope with limits and motor, and a rigid rod."""
    b = _bodies([(S, 0, 0), (D, 0.0, -1.0, 0.0, 0.5, 0.0, 1.0), (D, 1.0, -1.5)], mass=2.0, inertia=0.1)
    return b, np.array([
        _row(device.JOINT_DISTANCE, 0, 1, 0, ALL, localOriginAnchorB=(0.2, 0.0), referenceAngle=1.2, lowerAngle=0.8, upperAngle=1.5,
             hertz=2.0, dampingRatio=0.3, motorSpeed=0.2, maxMotorTorque=3.0),
        _row(device.JOINT_DISTANCE, 1, 2, 1, localOriginAnchorA=(0.1, 0.0), referenceAngle=1.1, lowerAngle=1.1, upperAngle=1.1)])


def world_wheel():
    b = _bodies([(S, 0, 0), (D, 0.0, -1.0, 0.0, 0.3, 0.0, 0.0), (D, 1.5, -1.0)], mass=2.0, inertia=0.1)
    return b, np.array([_wheel_row(0, 1, 0), _wheel_row(1, 2, 1, anchor_a=(1.5, 0.0))])


def world_pulley():
    b = _bodies([(S, 0, 0), (D, 0.0, -1.0, 0.0, 0.5), (D, 6.0, -2.0)], mass=2.0, inertia=2.0 / 6.0)
    return b, np.array([_row(device.JOINT_PULLEY, 1, 2, 0, localOriginAnchorA=(0.1, 0.2), localOriginAnchorB=(-0.1, 0.0),
                             target=(0.0, 3.0), localAxisA=(6.0, 3.0), referenceAngle=1.5, lowerAngle=4.0, upperAngle=5.0)])


def world_gear():
    """A motorised revolute pinion geared to a second wheel (revolute sides) and to a rack (a prismatic side)."""
    b = _bodies([(S, 0, 0), (D, 0.0, 0.0, 0.0, 0.0, 0.0, 3.0), (D, 3.0, 0.0), (D, 1.0, -1.0)], mass=2.0, inertia=2.0 / 6.0)
    return b, np.array([
        _row(device.JOINT_REVOLUTE, 0, 1, 0, device.JOINT_ENABLE_MOTOR, motorSpeed=-1.0, maxMotorTorque=5.0),
        _row(device.JOINT_GEAR, 1, 2, 1, target=(0.0, 1.0), localAxisA=(0.0, 0.0), maxMotorTorque=0.0, motorSpeed=1.0,
             referenceAngle=2.0),
        _row(device.JOINT_GEAR, 1, 3, 2, device.JOINT_GEAR_PRISMATIC2, target=(0.0, 1.0), localAxisA=(0.0, 0.0), maxMotorTorque=1.0,
             motorSpeed=-1.0, hertz=0.0, dampingRatio=1.0, referenceAngle=0.5)])


def world_revolute_mouse():
    b = _three_boxes()
    return b, np.array([
        _pinned(device.JOINT_REVOLUTE, b, 0, 1, (0.0, 0.0), 0, LIMIT_MOTOR, lowerAngle=-0.3, upperAngle=0.4, motorSpeed=1.0,
                maxMotorTorque=5.0),
        _pinned(device.JOINT_REVOLUTE, b, 1, 2, (0.6, 0.0), 1),
        _row(device.JOINT_MOUSE, 0, 2, 2, **MOUSE)])


# name: (world, steps, the type oracle it was recorded from; "base" = oracle/s2o_solver.c)
WORLDS = {
    "spring_without_flag": (world_spring_without_flag, 40, "prismatic"),
    "rigid_welds": (world_rigid_welds, 40, "weld"),
    "wheel_neighbours": (world_wheel_neighbours, 30, "distance"),
    "pulley_neighbours": (world_pulley_neighbours, 30, "wheel"),
    "gear_neighbours": (world_gear_neighbours, 30, "pulley"),
    "weld": (world_weld, 30, "weld"),
    "soft_weld": (world_soft_weld, 30, "soft_weld"),
    "motor": (world_motor, 30, "motor"),
    "prismatic": (world_prismatic, 30, "prismatic"),
    "spring": (world_spring, 30, "spring"),
    "distance": (world_distance, 30, "distance"),
    "wheel": (world_wheel, 30, "wheel"),
    "pulley": (world_pulley, 30, "pulley"),
    "gear": (world_gear, 30, "gear"),
    "revolute_mouse": (world_revolute_mouse, 30, "base"),
}


def run_digest(O, solver, world, steps):
    """A truncated sha1 of the body and joint rows after each of `steps` steps of `world` under oracle O, in step order."""
    bodies, joints = world()
    ctx = device.make_context(solver, DT, 4, 2)
    contacts = np.zeros(0, dtype=device.CONTACT_ROW)
    h = hashlib.sha1()
    for _ in range(steps):
        bodies, _, joints = O.solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, gravity=(0.0, -G))
        bodies["origin"] = bodies["position"]
        h.update(bodies.tobytes() + joints.tobytes())
    return h.hexdigest()[:16]


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)["worlds"]


@pytest.mark.parametrize("world", sorted(WORLDS))
@pytest.mark.parametrize("solver", VARIANTS)
def test_matches_the_recorded_bits(solver, world):
    build, steps, _ = WORLDS[world]
    assert run_digest(joint_oracle.load(), solver, build, steps) == _golden()[world][solver]


@pytest.mark.parametrize("solver", VARIANTS)
def test_revolute_and_mouse_rows_are_the_base_oracles(solver):
    build, steps, _ = WORLDS["revolute_mouse"]
    assert run_digest(joint_oracle.load(), solver, build, steps) == run_digest(port.load(), solver, build, steps)
