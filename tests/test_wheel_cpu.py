"""CPU: the wheel joint in the joint oracle (tests/joint_oracle.c, DESIGN.md §3.17) on hand-built rows, for all ten variants.

No contacts and every local centre at zero, so finalize is the identity (origin == position) and solver stages chain
directly. The bounds below were measured on these deterministic runs (the largest value over the variants a test covers,
computed from these same runs) and carry the margin stated next to each.

Mutations each test catches: a motor that acts on the axis instead of the rotation never spins the wheel; a motor impulse
that is not clamped lifts a load it should not; a spring coefficient formed with another h shifts the frequency or the
sag; a perpendicular row without its bias lets the anchor drift off the axis; a limit with its sign flipped lets the
translation leave its range; a motor mass formed without the fixed-rotation test makes NaNs; a reaction that leaves the
perpendicular or spring impulse out misreads the hanging load; a wheel branch that takes another type's rows changes the bits
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
DT = 1.0 / 60.0
G = 10.0
MASS = 2.0
INERTIA = 0.1
MOTOR_W = 5.0  # rad/s

# measured maxima (see the module docstring) and the margin each bound keeps
SPRING_FREQ_REL = 0.04      # undamped 1 Hz spring over 4 s: measured <= 5e-3 (Jacobi, PGS_Soft), 0 elsewhere, at the
                            # resolution of the zero crossings (one step per half period, 1 / 30)
OVERSHOOT = 1e-3            # zeta = 1 from 0.2 m stretched: measured none (the translation stays >= -7.5e-9)
SAG_REL = 1e-4              # vertical spring's rest at -g / omega^2: measured <= 7.0e-7, x 140
# TGS_Sticky prepares its joints cold once per step and accumulates their impulses over the sub-steps, so its spring is
# softer and more damped than its hertz and damping ratio say (DESIGN.md §3.14). Its spring bounds are its own measured
# values with a margin; no other variant is special-cased.
FREQ_REL_STICKY = 0.6       # measured 0.50, x 1.2
OVERSHOOT_STICKY = 0.05     # measured 3.26e-2, x 1.5
SAG_REL_STICKY = 4.0        # measured 2.92, x 1.4
PERP_DRIFT = 0.02           # anchor off the axis under a sideways 1 g (2 Hz suspension): measured 5.1e-3 (Jacobi,
                            # PGS_Soft), <= 1.4e-3 under the sub-stepping soft variants, <= 2e-8 under the NGS variants
                            # and XPBD, x 4
LIMIT_OVER = 1.5e-3         # translation past a limit: measured <= 2.8e-4 (Jacobi, PGS_Soft, TGS_Soft), x 5
AXLE = 3e-3                 # |translation| with equal limits, thrown at 1 m/s: measured <= 6.4e-4 (TGS_Soft), x 4.7
MOTOR_SPEED = 1e-3          # rad/s off the set speed after 3 s, unloaded: measured 0 under every variant but XPBD
MOMENTUM = 1e-4             # free pair, 60 steps: measured <= 5.8e-6 (XPBD), x 17
XPBD_SPIN_REL = 1e-4        # XPBD free spin against a free body: measured 1.4e-5, x 7


def _bodies(specs):
    """specs: (type, x, y, vx, vy, w, gravityScale[, fixedRotation]) per body."""
    rows = np.zeros(len(specs), dtype=device.BODY_ROW)
    for i, spec in enumerate(specs):
        kind, x, y, vx, vy, w, gs = spec[:7]
        fixed = len(spec) > 7 and spec[7]
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
            if not fixed:
                r["I"], r["invI"] = INERTIA, 1.0 / INERTIA
        rows[i] = r
    return rows


def _wheel(a, b, anchor_a=(0.0, 0.0), anchor_b=(0.0, 0.0), axis=(0.0, 1.0), spring=None, limit=None, motor=None, slot=0):
    """One wheel row. spring = (hertz, dampingRatio); limit = (lower, upper); motor = (speed, maxTorque)."""
    r = np.zeros(1, dtype=device.JOINT_ROW)[0]
    r["index"] = slot
    r["flags"] = device.ROW_VALID | (device.JOINT_WHEEL << 1)
    r["bodyA"], r["bodyB"] = a, b
    r["localOriginAnchorA"], r["localOriginAnchorB"] = anchor_a, anchor_b
    n = math.hypot(*axis)
    r["localAxisA"] = (np.float32(axis[0]) / np.float32(n), np.float32(axis[1]) / np.float32(n))
    if spring is not None:
        r["flags"] |= device.JOINT_ENABLE_SPRING
        r["hertz"], r["dampingRatio"] = spring
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


def _translation(b, i=1):
    """Along the vertical axis of a static body A at the origin."""
    return float(b["position"][i][1])


def _crossings(xs):
    return [k for k in range(1, len(xs)) if (xs[k - 1] < 0.0) != (xs[k] < 0.0)]


# ---- free spin --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", VARIANTS)
def test_free_spin_keeps_angular_velocity_bit_for_bit(solver):
    """A wheel anchored at its centre on a static body, spinning, with its spring and limits on and no motor, bobbing under
    gravity: nothing acts on its rotation, so its angular velocity stays bit for bit. XPBD forms velocities from poses, and
    its joint rows renormalize the wheel's rotation (a zero-angle s2IntegrateRot), so there it is compared with a free
    spinning body (body 2, no joint) within XPBD_SPIN_REL."""
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 1), (capi.DYNAMIC_BODY, 0.0, 0.1, 0, 0, 7.5, 1),
                      (capi.DYNAMIC_BODY, 5.0, 0.0, 0, 0, 7.5, 1)])
    hist = _run(solver, bodies, np.array([_wheel(0, 1, spring=(2.0, 0.3), limit=(-0.2, 0.2))]), 120)
    for b, _ in hist:
        if solver == "XPBD":
            assert abs(b["angularVelocity"][1] / b["angularVelocity"][2] - 1.0) <= XPBD_SPIN_REL
        else:
            assert b["angularVelocity"][1] == np.float32(7.5)
    assert min(_translation(b) for b, _ in hist) < 0.0  # the spring and gravity moved it along the axis


# ---- spring ---------------------------------------------------------------------------------------------------------------

def _spring_case(solver, zeta, steps, y0=0.2):
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 1), (capi.DYNAMIC_BODY, 0.0, y0, 0, 0, 0, 1)])
    return _run(solver, bodies, np.array([_wheel(0, 1, spring=(1.0, zeta))]), steps, gravity=(0.0, 0.0))


def _sag_case(solver):
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 1), (capi.DYNAMIC_BODY, 0.0, 0.0, 0, 0, 0, 1)])
    return _run(solver, bodies, np.array([_wheel(0, 1, spring=(1.0, 1.0))]), 600)


@pytest.mark.parametrize("solver", VARIANTS)
def test_spring_oscillates_at_hertz(solver):
    hist = _spring_case(solver, 0.0, 240)
    cross = _crossings([_translation(b) for b, _ in hist])
    f = (len(cross) - 1) / (2.0 * (cross[-1] - cross[0]) * DT)
    assert abs(f - 1.0) <= (FREQ_REL_STICKY if solver == "TGS_Sticky" else SPRING_FREQ_REL), f


@pytest.mark.parametrize("solver", VARIANTS)
def test_critical_spring_does_not_overshoot(solver):
    hist = _spring_case(solver, 1.0, 240)
    assert min(_translation(b) for b, _ in hist) >= -(OVERSHOOT_STICKY if solver == "TGS_Sticky" else OVERSHOOT)


@pytest.mark.parametrize("solver", VARIANTS)
def test_vertical_spring_rests_at_g_over_omega_squared(solver):
    """A wheel on a vertical 1 Hz, zeta = 1 suspension rests at -g / omega^2 (the spring's mass is the wheel's)."""
    sag = _translation(_sag_case(solver)[-1][0])
    expect = -G / (2.0 * math.pi) ** 2
    assert abs(sag / expect - 1.0) <= (SAG_REL_STICKY if solver == "TGS_Sticky" else SAG_REL), sag


# ---- perpendicular row and limits -----------------------------------------------------------------------------------------

def _sideways_case(solver):
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 1), (capi.DYNAMIC_BODY, -0.1, 0.0, 0, 0, 2.0, 1)])
    return _run(solver, bodies, np.array([_wheel(0, 1, anchor_b=(0.1, 0.0), spring=(2.0, 0.7))]), 240, gravity=(G, -G))


@pytest.mark.parametrize("solver", VARIANTS)
def test_sideways_load_keeps_the_anchor_on_the_axis(solver):
    """A spinning wheel anchored 0.1 m off its centre, under a 1 g sideways load: anchor B stays on the vertical axis."""
    hist = _sideways_case(solver)
    drift = 0.0
    for b, _ in hist:
        c, s = float(b["rot"][1][1]), float(b["rot"][1][0])
        drift = max(drift, abs(float(b["position"][1][0]) + c * 0.1))
    assert drift <= PERP_DRIFT, drift


def _limit_case(solver, limit, v0):
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 1), (capi.DYNAMIC_BODY, 0.0, 0.0, v0[0], v0[1], 1.0, 1)])
    return _run(solver, bodies, np.array([_wheel(0, 1, limit=limit)]), 120)


@pytest.mark.parametrize("solver", VARIANTS)
def test_translation_stays_inside_its_limits(solver):
    """No spring: the wheel falls to its lower limit and rests there; thrown up at 3 m/s, it stops at its upper limit."""
    lower = max(-0.3 - _translation(b) for b, _ in _limit_case(solver, (-0.3, 0.1), (0.0, 0.0)))
    upper = max(_translation(b) - 0.1 for b, _ in _limit_case(solver, (-0.3, 0.1), (0.0, 3.0)))
    assert lower <= LIMIT_OVER and upper <= LIMIT_OVER, (lower, upper)


@pytest.mark.parametrize("solver", VARIANTS)
def test_equal_limits_are_a_rigid_axle(solver):
    hist = _limit_case(solver, (0.0, 0.0), (0.0, 1.0))
    axle = max(abs(_translation(b)) for b, _ in hist)
    assert axle <= AXLE, axle


# ---- motor ----------------------------------------------------------------------------------------------------------------

def _motor_case(solver, torque, centred):
    """A wheel on a rigid axle (equal limits) of a static body, its motor at MOTOR_W. Centred: no load. Otherwise the
    axle is 0.5 m from the wheel's centre, so gravity loads the motor with up to m g 0.5 = 10 N-m."""
    anchor_b = (0.0, 0.0) if centred else (-0.5, 0.0)
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 1), (capi.DYNAMIC_BODY, 0.0 if centred else 0.5, 0.0, 0, 0, 0, 1)])
    return _run(solver, bodies, np.array([_wheel(0, 1, anchor_b=anchor_b, limit=(0.0, 0.0), motor=(MOTOR_W, torque))]), 180)


def _turned(hist):
    """The wheel's total rotation (rad), unwrapped step by step."""
    total, prev = 0.0, 0.0
    for b, _ in hist:
        angle = math.atan2(float(b["rot"][1][0]), float(b["rot"][1][1]))
        total += math.remainder(angle - prev, 2.0 * math.pi)
        prev = angle
    return total


@pytest.mark.parametrize("solver", VARIANTS)
def test_motor_reaches_speed_and_stalls_under_a_larger_load(solver):
    """Unloaded, the wheel turns at motorSpeed; with the 10 N-m load a 100 N-m motor turns it over the top, a 5 N-m motor
    cannot (its impulse sits at the clamp) and the wheel swings below the axle. XPBD does not apply the motor."""
    free = _motor_case(solver, 100.0, centred=True)
    strong = _motor_case(solver, 100.0, centred=False)
    weak = _motor_case(solver, 5.0, centred=False)
    if solver == "XPBD":
        assert float(free[-1][0]["angularVelocity"][1]) == 0.0
        assert all(float(j["impulse"][0][1]) == 0.0 for _, j in weak)
        return
    w = float(free[-1][0]["angularVelocity"][1])
    assert abs(w - MOTOR_W) <= MOTOR_SPEED, w
    assert _turned(strong) > 2.0 * math.pi
    assert abs(_turned(weak)) < math.pi
    h = DT / 4.0 if solver in capi.SUBSTEPPING else DT
    assert max(abs(float(j["impulse"][0][1])) for _, j in weak) == np.float32(np.float32(h) * np.float32(5.0))


@pytest.mark.parametrize("solver", VARIANTS)
def test_fixed_rotations_with_motor_make_no_nan(solver):
    """Body B with a fixed rotation on a static body: the motor has nothing to turn, so its impulse stays 0."""
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 1), (capi.DYNAMIC_BODY, 0.0, 0.1, 0, 0, 0, 1, True)])
    hist = _run(solver, bodies, np.array([_wheel(0, 1, spring=(2.0, 0.5), limit=(-0.2, 0.2), motor=(3.0, 50.0))]), 60)
    for b, j in hist:
        assert np.all(np.isfinite(b["position"])) and np.all(np.isfinite(b["linearVelocity"]))
        assert np.all(np.isfinite(j["impulse"])) and float(j["impulse"][0][1]) == 0.0
        assert b["angularVelocity"][1] == 0.0


@pytest.mark.parametrize("solver", VARIANTS)
def test_free_pair_conserves_momentum(solver):
    """Two spinning boxes on a sprung, limited, motored wheel joint without gravity: linear momentum stays put."""
    bodies = _bodies([(capi.DYNAMIC_BODY, 0, 0, 0.3, 0.1, 1.0, 0), (capi.DYNAMIC_BODY, 0.2, 0.5, -0.2, 0.4, -2.0, 0)])
    joint = _wheel(0, 1, anchor_a=(0.1, 0.1), anchor_b=(-0.1, 0.05), axis=(1.0, 2.0), spring=(2.0, 0.2), limit=(-0.3, 0.4),
                   motor=(3.0, 1.0))
    hist = _run(solver, bodies, np.array([joint]), 60, gravity=(0.0, 0.0))
    p0 = MASS * (bodies["linearVelocity"][0].astype(np.float64) + bodies["linearVelocity"][1])
    for b, _ in hist:
        p = MASS * (b["linearVelocity"][0].astype(np.float64) + b["linearVelocity"][1])
        assert np.abs(p - p0).max() <= MOMENTUM


# ---- reactions ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", VARIANTS)
def test_hanging_sprung_wheel_reads_mg(solver):
    """A 2 kg wheel at rest on a 2 Hz, zeta = 1 suspension reads (0, m g) (the spring's impulse carries the load), under
    every variant but XPBD, which keeps no impulses. Its torque is rate times the angular motor impulse."""
    P = capi.Solver2D(device.LIB_PATH)
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 1), (capi.DYNAMIC_BODY, 0.0, -G / (4.0 * math.pi) ** 2, 0, 0, 0, 1)])
    joint = _wheel(0, 1, anchor_b=(0.0, 0.0), spring=(2.0, 1.0), motor=(2.0, 0.05))
    b, j = _run(solver, bodies, np.array([joint]), 300)[-1]
    sub = solver in capi.SUBSTEPPING
    rate = np.float32((1.0 / DT) if (solver == "TGS_Sticky" or not sub) else 4.0 / DT)
    spring = float(j["springImpulse"][0])
    r = P.s2ComputeJointReaction(device.JOINT_WHEEL, capi.Vec2(float(j["impulse"][0][0]), float(j["impulse"][0][1])),
                                 float(np.float32(j["motorImpulse"][0]) + np.float32(spring)), float(j["lowerImpulse"][0]),
                                 float(j["upperImpulse"][0]), capi.Rot(float(b["rot"][0][0]), float(b["rot"][0][1])),
                                 capi.Vec2(0.0, 1.0), float(rate))
    assert r.torque == np.float32(rate * np.float32(j["impulse"][0][1]))
    if solver == "XPBD":
        assert (r.force.x, r.force.y, r.torque) == (0.0, 0.0, 0.0)
        return
    assert abs(r.force.x) <= 1e-4 and abs(r.force.y - MASS * G) <= 1e-3 * MASS * G, (r.force.x, r.force.y)
    assert j["impulse"][0][1] != 0.0  # the motor, still accelerating the wheel at its clamp


# ---- other joint types and layout -----------------------------------------------------------------------------------------

def test_struct_sizes_unchanged():
    """The wheel row reuses columns: s2bJointRow stays 108 bytes and every other ABI size is the parent's."""
    out = (C.c_int32 * 6)()
    C.CDLL(device.LIB_PATH).s2b_abi_sizes(out)
    assert out[2] == 108 == device.JOINT_ROW.itemsize
    assert (out[0], out[1], out[3]) == (device.BODY_ROW.itemsize, device.SHAPE_ROW.itemsize, device.CONTACT_ROW.itemsize)
