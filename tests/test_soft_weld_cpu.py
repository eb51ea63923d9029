"""CPU: the soft weld's oracle (tests/soft_weld_oracle.c, DESIGN.md §3.15) on hand-built rows, for all ten variants.

No contacts and every local centre at zero, so finalize is the identity (origin == position) and solver stages chain
directly. Gravity is off unless a test says otherwise. The bounds below were measured on these deterministic runs (the
largest value over the ten variants, printed by `python tests/test_soft_weld_cpu.py`) and carry the margin stated next to
each.

Mutations each test catches: a coefficient formed with the wrong h or the wrong expression shifts the frequency or the sag;
a soft part that is not soft (the error fed back at 1 / h) overshoots with zeta = 1; an impulse applied to one body only
breaks momentum; a missing s2UnwindAngle turns the seam case the long way round; a soft term evaluated on a weld with both
hertz at 0, or on another joint, changes the weld oracle's bits; an angular spring on a body without rotation moves it."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import soft_weld_oracle  # noqa: E402
import weld_oracle  # noqa: E402
from solver2d_b200 import capi, device  # noqa: E402

VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]
DT = 1.0 / 60.0
G = 10.0
HX, HY = 0.5, 0.25  # box half extents
MASS = 1.0
INERTIA = MASS * ((2 * HX) ** 2 + (2 * HY) ** 2) / 12.0

# measured maxima over the ten variants (see the module docstring) and the margin each bound keeps
FREQ_REL = 0.015            # |f - hertz| / hertz of an undamped 1 Hz part over 4 s: measured 5.0e-3, x 3
OVERSHOOT_BOUND = 1e-6      # zeta = 1 from 0.2 (rad or m): measured <= 1.4e-10 (XPBD, linear); 0 elsewhere
UNDAMPED_KEEP = 0.05        # zeta = 0: amplitude after 4 s over the first second's; measured >= 0.073 (Jacobi,
                            # PGS_Soft, whose relax passes damp the soft row), 0.27 (PGS family), >= 0.52 (sub-steppers)
REST_REL = 1e-5             # linear sag -g / omega^2: measured <= 3.4e-7 (PGS family) for every variant but one, x 29
LINEAR_MOMENTUM_BOUND = 1e-5  # free pair, both parts soft, 60 steps: measured <= 1.6e-6 (XPBD; rigid 2.2e-6), x 6
MOMENTUM_SLACK = 5e-5       # angular-only soft pair: drift <= 2 x drift rigid + this; measured 8.0e-6 (TGS_Soft, rigid 2.4e-6)
SEAM_BOUND = 1e-4           # rad: the seam case comes back 0.1 rad across the seam and rests; measured <= 3.3e-6, x 30
# TGS_Sticky prepares its joints cold once per step and accumulates their impulses over the sub-steps, so a soft part's
# impulseScale * lambda term sees the step's running total instead of the sub-step's: the part is softer and more damped
# than its hertz and damping ratio say, as for the springs (§3.14). Its bounds are its own measured values with a margin;
# no other variant is special-cased.
FREQ_REL_STICKY = 0.6       # measured 0.50 (f ~ 0.5 Hz for 1 Hz), x 1.2
OVERSHOOT_STICKY = 0.05     # measured 3.3e-2 (linear), 2.6e-2 (angular), x 1.5
REST_REL_STICKY = 4.0       # measured 2.89 (rests at ~3.9 g / omega^2), x 1.4


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


def weld_row(bodies, a, b, pivot, ref=None, linear=(0.0, 0.0), angular=(0.0, 0.0), slot=0):
    """One weld row with anchors at `pivot`; linear / angular = (hertz, dampingRatio), in the lanes a weld row uses."""
    r = np.zeros(1, dtype=device.JOINT_ROW)[0]
    r["index"] = slot
    r["flags"] = device.ROW_VALID | (device.JOINT_WELD << 1)
    r["bodyA"], r["bodyB"] = a, b
    r["localOriginAnchorA"] = _local(bodies, a, pivot)
    r["localOriginAnchorB"] = _local(bodies, b, pivot)
    r["referenceAngle"] = 0.0 if ref is None else ref
    r["hertz"], r["dampingRatio"] = linear
    r["maxMotorTorque"], r["motorSpeed"] = angular
    return r


def _run(O, solver, bodies, joints, steps, gravity=(0.0, 0.0)):
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


def _angular_error(bodies, joint):
    e = _angle(bodies, int(joint["bodyB"])) - _angle(bodies, int(joint["bodyA"])) - float(joint["referenceAngle"])
    return (e + math.pi) % (2.0 * math.pi) - math.pi


def _separation(bodies, joint):
    """World anchor B - world anchor A."""
    p = []
    for i, name in ((int(joint["bodyA"]), "localOriginAnchorA"), (int(joint["bodyB"]), "localOriginAnchorB")):
        s, c = (float(v) for v in bodies["rot"][i])
        lx, ly = (float(v) for v in joint[name])
        p.append(np.array([c * lx - s * ly, s * lx + c * ly]) + bodies["origin"][i].astype(np.float64))
    return p[1] - p[0]


ANGULAR, LINEAR = "angular", "linear"
PARTS = [ANGULAR, LINEAR]


def _error(part, bodies, joint):
    return _angular_error(bodies, joint) if part == ANGULAR else float(_separation(bodies, joint)[0])


def _oscillator(part, spring, x0=0.2):
    """A box welded at its centre to static body 0: turned by x0 rad (angular spring, rigid anchor) or moved x0 m along x
    (linear spring, rigid angle)."""
    if part == ANGULAR:
        bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 0), (capi.DYNAMIC_BODY, 0, 0, x0, 0, 0, 0)])
        joints = np.array([weld_row(bodies, 0, 1, (0.0, 0.0), angular=spring)])
    else:
        bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 0), (capi.DYNAMIC_BODY, x0, 0, 0, 0, 0, 0)])
        joints = np.array([weld_row(bodies, 0, 1, (0.0, 0.0), linear=spring)])
        joints[0]["localOriginAnchorB"] = (0.0, 0.0)  # anchor B at B's centre: the separation starts at x0
    return bodies, joints


def _errors(part, history):
    return np.array([_error(part, b, j[0]) for b, j in history])


def _frequency(e):
    """Frequency (Hz) from the upward zero crossings of the error history, interpolated."""
    t = []
    for k in range(1, len(e)):
        if e[k - 1] < 0.0 <= e[k]:
            t.append((k - 1 + (-e[k - 1]) / (e[k] - e[k - 1])) * DT)
    assert len(t) >= 2, "fewer than two periods"
    return (len(t) - 1) / (t[-1] - t[0])


def _measure_frequency(solver, part):
    e = _errors(part, _run(soft_weld_oracle.load(), solver, *_oscillator(part, (1.0, 0.0)), 240))
    return abs(_frequency(e) - 1.0)


@pytest.mark.parametrize("part", PARTS)
@pytest.mark.parametrize("solver", VARIANTS)
def test_oscillates_at_hertz(solver, part):
    bound = FREQ_REL_STICKY if solver == "TGS_Sticky" else FREQ_REL
    assert _measure_frequency(solver, part) <= bound


def _measure_overshoot(solver, part):
    e = _errors(part, _run(soft_weld_oracle.load(), solver, *_oscillator(part, (2.0, 1.0)), 180))
    return float(max(0.0, -e.min())), abs(float(e[-1]))


@pytest.mark.parametrize("part", PARTS)
@pytest.mark.parametrize("solver", VARIANTS)
def test_critical_damping_does_not_overshoot(solver, part):
    overshoot, last = _measure_overshoot(solver, part)
    assert overshoot <= (OVERSHOOT_STICKY if solver == "TGS_Sticky" else OVERSHOOT_BOUND)
    assert last < 0.1 * 0.2  # and it returns


def _measure_keep(solver, part):
    e = _errors(part, _run(soft_weld_oracle.load(), solver, *_oscillator(part, (1.0, 0.0)), 300))
    return float(np.abs(e[240:]).max() / np.abs(e[:60]).max())


@pytest.mark.parametrize("part", PARTS)
@pytest.mark.parametrize("solver", VARIANTS)
def test_undamped_amplitude_decay_is_bounded(solver, part):
    assert _measure_keep(solver, part) >= UNDAMPED_KEEP


def _measure_rest(solver):
    """A box hanging from a static body on a linear-only soft weld at its centre: the anchor sags by -g / omega^2."""
    hertz = 2.0
    omega = 2.0 * math.pi * hertz
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 0), (capi.DYNAMIC_BODY, 0, 0, 0, 0, 0, 0)])
    joints = np.array([weld_row(bodies, 0, 1, (0.0, 0.0), linear=(hertz, 0.7))])
    h = _run(soft_weld_oracle.load(), solver, bodies, joints, 300, gravity=(0.0, -G))
    rest = -G / (omega * omega)
    b, j = h[-1]
    return abs(float(_separation(b, j[0])[1]) - rest) / abs(rest)


@pytest.mark.parametrize("solver", VARIANTS)
def test_linear_soft_weld_sags_by_g_over_omega_squared(solver):
    bound = REST_REL_STICKY if solver == "TGS_Sticky" else REST_REL
    assert _measure_rest(solver) <= bound


def _pair(linear=(1.5, 0.3), angular=(2.0, 0.2)):
    """Two free boxes welded at a point between them, both moving."""
    bodies = _bodies([(capi.DYNAMIC_BODY, -0.6, 0.0, 0.0, 0.3, 0.1, 0.5), (capi.DYNAMIC_BODY, 0.6, 0.0, 0.3, -0.2, 0.4, -1.5)])
    joints = np.array([weld_row(bodies, 0, 1, (0.0, 0.0), ref=0.1, linear=linear, angular=angular)])
    return bodies, joints


def _momentum(bodies):
    p = np.zeros(2)
    L = 0.0
    for i in range(len(bodies)):
        m = float(bodies["mass"][i])
        x, y = (float(v) for v in bodies["position"][i])
        vx, vy = (float(v) for v in bodies["linearVelocity"][i])
        p += m * np.array([vx, vy])
        L += m * (x * vy - y * vx) + float(bodies["I"][i]) * float(bodies["angularVelocity"][i])
    return p, L


def _measure_momentum(solver, O, **kw):
    """(linear, angular) worst drift over 60 steps."""
    bodies, joints = _pair(**kw)
    p0, L0 = _momentum(bodies)
    worst_p = worst_L = 0.0
    for b, _ in _run(O, solver, bodies, joints, 60):
        p, L = _momentum(b)
        worst_p = max(worst_p, float(np.abs(p - p0).max()))
        worst_L = max(worst_L, abs(L - L0))
    return worst_p, worst_L


@pytest.mark.parametrize("solver", VARIANTS)
def test_free_pair_conserves_momentum(solver):
    """The soft rows' impulses are equal and opposite: both parts soft keep the pair's linear momentum, and an angular-only
    soft weld drifts in angular momentum no more than the rigid weld does (the position passes of the NGS variants and
    XPBD move it either way). A soft anchor lets the anchors part, and its impulse is not along the line between them, so
    it turns the pair: angular momentum is not a property of a linear soft part (as for Box2D's soft weld)."""
    O = soft_weld_oracle.load()
    rigid_L = _measure_momentum(solver, O, linear=(0.0, 0.0), angular=(0.0, 0.0))[1]
    assert _measure_momentum(solver, O)[0] <= LINEAR_MOMENTUM_BOUND
    assert _measure_momentum(solver, O, linear=(0.0, 0.0))[1] <= 2.0 * rigid_L + MOMENTUM_SLACK


def _measure_seam(solver):
    # rest angle pi - 0.05; B starts at -pi + 0.05, 0.1 rad past the seam: it must come back across it, not go round
    ref = math.pi - 0.05
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 0), (capi.DYNAMIC_BODY, 0, 0, -math.pi + 0.05, 0, 0, 0)])
    joints = np.array([weld_row(bodies, 0, 1, (0.0, 0.0), ref=ref, angular=(2.0, 1.0))])
    travelled = 0.0
    prev = _angle(bodies, 1)
    hist = _run(soft_weld_oracle.load(), solver, bodies, joints, 180)
    for b, _ in hist:
        a = _angle(b, 1)
        travelled += (a - prev + math.pi) % (2.0 * math.pi) - math.pi
        prev = a
    return abs(travelled + 0.1), abs(_angular_error(hist[-1][0], hist[-1][1][0]))


@pytest.mark.parametrize("solver", VARIANTS)
def test_rest_angle_across_the_seam(solver):
    travel_error, rest_error = _measure_seam(solver)
    assert travel_error <= SEAM_BOUND and rest_error <= SEAM_BOUND


def _mixed_rows(bodies):
    """Rigid welds (one at the seam), a revolute with limit and motor, and a mouse row."""
    w0 = weld_row(bodies, 0, 1, (0.0, 0.0), slot=0)
    rev = np.zeros(1, dtype=device.JOINT_ROW)[0]
    rev["index"] = 1
    rev["flags"] = device.ROW_VALID | (device.JOINT_REVOLUTE << 1) | device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR
    rev["bodyA"], rev["bodyB"] = 1, 2
    rev["localOriginAnchorA"] = _local(bodies, 1, (0.6, 0.0))
    rev["localOriginAnchorB"] = _local(bodies, 2, (0.6, 0.0))
    rev["lowerAngle"], rev["upperAngle"] = -0.3, 0.4
    rev["motorSpeed"], rev["maxMotorTorque"] = 1.0, 5.0
    w2 = weld_row(bodies, 2, 3, (1.8, 0.1), ref=math.pi - 0.01, slot=2)
    mouse = np.zeros(1, dtype=device.JOINT_ROW)[0]
    mouse["index"] = 3
    mouse["flags"] = device.ROW_VALID | (device.JOINT_MOUSE << 1)
    mouse["bodyA"], mouse["bodyB"] = 0, 3
    mouse["localOriginAnchorB"] = (0.1, 0.0)
    mouse["target"] = (2.5, 0.5)
    mouse["hertz"], mouse["dampingRatio"] = 5.0, 0.7
    return np.array([w0, rev, w2, mouse])


def _mixed_bodies():
    return _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 0), (capi.DYNAMIC_BODY, 0.0, 0.0, 0.1, 0.2, 0.0, 1.0),
                    (capi.DYNAMIC_BODY, 1.2, 0.1, 0.0, 0.0, 0.3, -0.5), (capi.DYNAMIC_BODY, 2.4, 0.1, 3.1, 0.1, 0.0, 0.2)])


@pytest.mark.parametrize("solver", VARIANTS)
def test_rigid_welds_keep_the_weld_oracle_bits(solver):
    """Both hertz at 0: the soft weld oracle gives the weld oracle's bits, beside revolute and mouse rows."""
    bodies = _mixed_bodies()
    joints = _mixed_rows(bodies)
    a = _run(soft_weld_oracle.load(), solver, bodies, joints, 40, gravity=(0.0, -G))
    b = _run(weld_oracle.load(), solver, bodies, joints, 40, gravity=(0.0, -G))
    for (b1, j1), (b2, j2) in zip(a, b):
        assert b1.tobytes() == b2.tobytes() and j1.tobytes() == j2.tobytes()


@pytest.mark.parametrize("solver", VARIANTS)
def test_soft_welds_act_beside_rigid_rows(solver):
    """The same rows with the welds made soft: the welds move differently and the other rows still solve (no NaN)."""
    bodies = _mixed_bodies()
    joints = _mixed_rows(bodies)
    soft = joints.copy()
    soft[0]["hertz"], soft[0]["dampingRatio"] = 3.0, 0.5
    soft[2]["maxMotorTorque"], soft[2]["motorSpeed"] = 2.0, 0.1
    O = soft_weld_oracle.load()
    a = _run(O, solver, bodies, soft, 40, gravity=(0.0, -G))
    b = _run(O, solver, bodies, joints, 40, gravity=(0.0, -G))
    assert np.isfinite(a[-1][0]["position"]).all()
    assert a[-1][0].tobytes() != b[-1][0].tobytes()


@pytest.mark.parametrize("solver", VARIANTS)
def test_angular_spring_without_rotation_does_nothing(solver):
    """iA + iB == 0: an angular spring gives the rigid weld's bits (the angular row is skipped either way)."""
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 0), (capi.DYNAMIC_BODY, 0.3, 0, 0.2, 0.1, 0, 0)])
    bodies[1]["invI"] = 0.0
    joints = np.array([weld_row(bodies, 0, 1, (0.0, 0.0), angular=(1.0, 0.5))])
    rigid = joints.copy()
    rigid[0]["maxMotorTorque"], rigid[0]["motorSpeed"] = 0.0, 0.0
    O = soft_weld_oracle.load()
    for (b1, j1), (b2, j2) in zip(_run(O, solver, bodies, joints, 10), _run(O, solver, bodies, rigid, 10)):
        assert b1.tobytes() == b2.tobytes()
        assert float(j1[0]["motorImpulse"]) == float(j2[0]["motorImpulse"])


def test_soft_welds_scene_stand_ins(reference):
    """scenes.soft_welds on a library without the extension: every weld becomes a revolute stand-in with the same bodies,
    every soft weld is recorded, and the stand-in world steps with contacts."""
    from solver2d_b200 import scenes
    sc = scenes.soft_welds(reference, "TGS_Soft", copies=2)
    assert "s2CreateWeldJoint" in reference.missing
    assert len(sc.piles["soft_welds"]) > 0 and len(sc.piles["soft_welds"]) % 2 == 0
    assert all(lh > 0.0 or ah > 0.0 for _, lh, _, ah, _ in sc.piles["soft_welds"])
    for _ in range(60):
        sc.step()
    _, ci = reference.contacts(sc.world)
    assert (ci[:, 0] == 1).sum() > 10
    sc.destroy()


def test_sizes():
    """The def grows by four floats at its end, in C and in ctypes; the device row keeps its 108 bytes."""
    out = (C.c_int32 * 6)()
    C.CDLL(device.LIB_PATH).s2b_abi_sizes(out)
    assert out[2] == 108 == device.JOINT_ROW.itemsize
    fields = [f for f, _ in capi.WeldJointDef._fields_]
    assert fields[-4:] == ["linearHertz", "linearDampingRatio", "angularHertz", "angularDampingRatio"]
    assert capi.WeldJointDef.angularDampingRatio.offset == C.sizeof(capi.WeldJointDef) - 4
    d = capi.default_weld_def()
    assert (d.linearHertz, d.linearDampingRatio, d.angularHertz, d.angularDampingRatio) == (0.0, 0.0, 0.0, 0.0)


if __name__ == "__main__":
    for part in PARTS:
        print(part, "frequency rel error", {s: round(_measure_frequency(s, part), 4) for s in VARIANTS})
        print(part, "zeta=1 (overshoot, last)", {s: tuple(f"{v:.1e}" for v in _measure_overshoot(s, part)) for s in VARIANTS})
        print(part, "zeta=0 amplitude kept", {s: round(_measure_keep(s, part), 3) for s in VARIANTS})
    O = soft_weld_oracle.load()
    print("momentum drift (linear both soft, angular angular-only soft, angular rigid)",
          {s: (f"{_measure_momentum(s, O)[0]:.1e}", f"{_measure_momentum(s, O, linear=(0, 0))[1]:.1e}",
               f"{_measure_momentum(s, O, linear=(0, 0), angular=(0, 0))[1]:.1e}") for s in VARIANTS})
    print("rest rel error", {s: f"{_measure_rest(s):.2e}" for s in VARIANTS})
    print("seam (travel err, rest err)", {s: tuple(f"{v:.1e}" for v in _measure_seam(s)) for s in VARIANTS})
