"""CPU: the joint spring in the joint oracle (tests/joint_oracle.c, DESIGN.md §3.14) on hand-built rows, for all ten variants.

No contacts and every local centre at zero, so finalize is the identity (origin == position) and solver stages chain
directly. Gravity is off unless a test says otherwise. The bounds below were measured on these deterministic runs (the
largest value over the ten variants, printed by `python tests/test_spring_cpu.py`) and carry the margin stated next to
each.

Mutations each test catches: a spring coefficient formed with the wrong h or the wrong expression shifts the frequency or
the rest translation; a spring that is not soft (the position error fed back at 1 / h) overshoots with zeta = 1; a spring
impulse applied to one body only breaks momentum; a missing s2UnwindAngle turns the seam case the long way round; a
spring term evaluated on a row without the flag (or with hertz == 0) changes the bits tests/test_joint_oracle_cpu.py
pins."""
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
HX, HY = 0.5, 0.25  # box half extents
MASS = 1.0
INERTIA = MASS * ((2 * HX) ** 2 + (2 * HY) ** 2) / 12.0

# measured maxima over the ten variants (see the module docstring) and the margin each bound keeps
FREQ_REL = 0.015            # |f - hertz| / hertz of an undamped 1 Hz spring over 4 s: measured 5.0e-3 (Jacobi, PGS_Soft), x 3
OVERSHOOT_BOUND = 1e-3      # zeta = 1 from 0.2 (rad or m): measured 0 (the error never changes sign)
UNDAMPED_KEEP = 0.05        # zeta = 0: amplitude after 4 s over the first second's; measured >= 0.073 (Jacobi, PGS_Soft,
                            # whose relax passes damp the soft row), 0.27 (PGS family), >= 0.52 (the sub-stepping variants)
REST_REL = 1e-4             # prismatic rest translation -g / omega^2: measured 0 (exact in float32) for every variant but one
MOMENTUM_SLACK = 5e-5       # free pair, 60 steps: drift with the spring <= 2 x drift with hertz 0 + this; measured <= 1.0x
SEAM_BOUND = 1e-4           # rad: the seam case comes back 0.1 rad across the seam and rests; measured <= 3.3e-6, x ~30
# TGS_Sticky prepares its joints cold once per step and accumulates their impulses over the sub-steps, so its spring's
# impulseScale * lambda term sees the step's running total instead of the sub-step's: the spring is softer and more damped
# than its hertz and damping ratio say. Its bounds are its own measured values with a margin; no other variant is
# special-cased.
FREQ_REL_STICKY = 0.6       # measured 0.50 (f ~ 0.5 Hz for 1 Hz), x 1.2
OVERSHOOT_STICKY = 0.05     # measured 3.3e-2 (prismatic), x 1.5
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


def _joint(bodies, kind, a, b, pivot, axis=(1.0, 0.0), ref=0.0, spring=None, limit=None, motor=None, slot=0):
    """One revolute or prismatic row with anchors at `pivot`; spring = (hertz, dampingRatio)."""
    r = np.zeros(1, dtype=device.JOINT_ROW)[0]
    r["index"] = slot
    r["flags"] = device.ROW_VALID | (kind << 1)
    r["bodyA"], r["bodyB"] = a, b
    r["localOriginAnchorA"] = _local(bodies, a, pivot)
    r["localOriginAnchorB"] = _local(bodies, b, pivot)
    if kind == device.JOINT_PRISMATIC:
        ax = np.asarray(axis, dtype=np.float32)
        r["localAxisA"] = ax / np.sqrt(ax[0] * ax[0] + ax[1] * ax[1])
    r["referenceAngle"] = ref
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


def _error(kind, bodies, joint):
    """The spring's position error: the unwound relative angle, or the translation along the world axis."""
    a, b = int(joint["bodyA"]), int(joint["bodyB"])
    if kind == device.JOINT_REVOLUTE:
        e = _angle(bodies, b) - _angle(bodies, a) - float(joint["referenceAngle"])
        return (e + math.pi) % (2.0 * math.pi) - math.pi
    p = []
    for i, name in ((a, "localOriginAnchorA"), (b, "localOriginAnchorB")):
        s, c = (float(v) for v in bodies["rot"][i])
        lx, ly = (float(v) for v in joint[name])
        p.append(np.array([c * lx - s * ly, s * lx + c * ly]) + bodies["origin"][i].astype(np.float64))
    s, c = (float(v) for v in bodies["rot"][a])
    lx, ly = (float(v) for v in joint["localAxisA"])
    return float(np.array([c * lx - s * ly, s * lx + c * ly]) @ (p[1] - p[0]))


def _oscillator(kind, spring, x0=0.2):
    """Body 1 on a spring to static body 0, displaced by x0 (rad about its centre, or m along x)."""
    if kind == device.JOINT_REVOLUTE:
        bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 0), (capi.DYNAMIC_BODY, 0, 0, x0, 0, 0, 0)])
    else:
        bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 0), (capi.DYNAMIC_BODY, x0, 0, 0, 0, 0, 0)])
    joints = np.array([_joint(bodies, kind, 0, 1, (0.0, 0.0), spring=spring)])
    if kind == device.JOINT_PRISMATIC:
        joints[0]["localOriginAnchorB"] = (0.0, 0.0)  # anchor B at B's centre: the translation starts at x0
    return bodies, joints


def _errors(kind, history):
    return np.array([_error(kind, b, j[0]) for b, j in history])


def _frequency(e):
    """Frequency (Hz) from the upward zero crossings of the error history, interpolated."""
    t = []
    for k in range(1, len(e)):
        if e[k - 1] < 0.0 <= e[k]:
            t.append((k - 1 + (-e[k - 1]) / (e[k] - e[k - 1])) * DT)
    assert len(t) >= 2, "fewer than two periods"
    return (len(t) - 1) / (t[-1] - t[0])


KINDS = [device.JOINT_REVOLUTE, device.JOINT_PRISMATIC]
KIND_IDS = ["revolute", "prismatic"]


def _measure_frequency(solver, kind):
    e = _errors(kind, _run(joint_oracle.load(), solver, *_oscillator(kind, (1.0, 0.0)), 240))
    return abs(_frequency(e) - 1.0)


@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
@pytest.mark.parametrize("solver", VARIANTS)
def test_oscillates_at_hertz(solver, kind):
    bound = FREQ_REL_STICKY if solver == "TGS_Sticky" else FREQ_REL
    assert _measure_frequency(solver, kind) <= bound


def _measure_overshoot(solver, kind):
    e = _errors(kind, _run(joint_oracle.load(), solver, *_oscillator(kind, (2.0, 1.0)), 180))
    return float(max(0.0, -e.min()))


@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
@pytest.mark.parametrize("solver", VARIANTS)
def test_critical_damping_does_not_overshoot(solver, kind):
    e = _errors(kind, _run(joint_oracle.load(), solver, *_oscillator(kind, (2.0, 1.0)), 180))
    assert e.min() >= -(OVERSHOOT_STICKY if solver == "TGS_Sticky" else OVERSHOOT_BOUND)
    assert abs(e[-1]) < 0.1 * 0.2  # and it returns


def _measure_keep(solver, kind):
    e = _errors(kind, _run(joint_oracle.load(), solver, *_oscillator(kind, (1.0, 0.0)), 300))
    first = np.abs(e[:60]).max()
    last = np.abs(e[240:]).max()
    return float(last / first)


@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
@pytest.mark.parametrize("solver", VARIANTS)
def test_undamped_amplitude_decay_is_bounded(solver, kind):
    assert _measure_keep(solver, kind) >= UNDAMPED_KEEP


def _measure_rest(solver):
    hertz = 2.0
    omega = 2.0 * math.pi * hertz
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 0), (capi.DYNAMIC_BODY, 0, 0, 0, 0, 0, 0)])
    joints = np.array([_joint(bodies, device.JOINT_PRISMATIC, 0, 1, (0.0, 0.0), axis=(0.0, 1.0), spring=(hertz, 0.7))])
    h = _run(joint_oracle.load(), solver, bodies, joints, 300, gravity=(0.0, -G))
    rest = -G / (omega * omega)
    b, j = h[-1]
    return abs(_error(device.JOINT_PRISMATIC, b, j[0]) - rest) / abs(rest)


@pytest.mark.parametrize("solver", VARIANTS)
def test_vertical_prismatic_spring_rests_at_g_over_omega_squared(solver):
    bound = REST_REL_STICKY if solver == "TGS_Sticky" else REST_REL
    assert _measure_rest(solver) <= bound


def _pair(kind):
    """Two free boxes joined at a point between them, B turning (revolute) or sliding (prismatic) against A."""
    bodies = _bodies([(capi.DYNAMIC_BODY, -0.6, 0.0, 0.0, 0.3, 0.1, 0.5), (capi.DYNAMIC_BODY, 0.6, 0.0, 0.3, -0.2, 0.4, -1.5)])
    joints = np.array([_joint(bodies, kind, 0, 1, (0.0, 0.0), axis=(1.0, 0.2), spring=(1.5, 0.3))])
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


def _measure_momentum(solver, kind, hertz=None):
    bodies, joints = _pair(kind)
    if hertz is not None:
        joints[0]["hertz"] = hertz
    p0, L0 = _momentum(bodies)
    worst = 0.0
    for b, _ in _run(joint_oracle.load(), solver, bodies, joints, 60):
        p, L = _momentum(b)
        worst = max(worst, float(np.abs(p - p0).max()), abs(L - L0))
    return worst


@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
@pytest.mark.parametrize("solver", VARIANTS)
def test_free_pair_conserves_momentum(solver, kind):
    """The spring's impulses are equal and opposite: the pair drifts no more than the same joint without a spring does
    (the position passes of the NGS variants and XPBD move the pair's angular momentum by up to 1e-2 either way)."""
    assert _measure_momentum(solver, kind) <= 2.0 * _measure_momentum(solver, kind, hertz=0.0) + MOMENTUM_SLACK


@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
@pytest.mark.parametrize("solver", VARIANTS)
def test_zero_hertz_exerts_nothing(solver, kind):
    """hertz == 0 with the flag on gives the same bits as no spring, and its impulse stays 0."""
    bodies, joints = _pair(kind)
    joints[0]["flags"] |= device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR
    joints[0]["lowerAngle"], joints[0]["upperAngle"] = -0.2, 0.25
    joints[0]["motorSpeed"], joints[0]["maxMotorTorque"] = 0.5, 2.0
    off = joints.copy()
    off[0]["flags"] &= ~device.JOINT_ENABLE_SPRING
    joints[0]["hertz"] = 0.0
    O = joint_oracle.load()
    for (b1, j1), (b2, j2) in zip(_run(O, solver, bodies, joints, 30, gravity=(0.0, -G)),
                                  _run(O, solver, bodies, off, 30, gravity=(0.0, -G))):
        assert b1.tobytes() == b2.tobytes()
        assert float(j1[0]["springImpulse"]) == 0.0
        j1 = j1.copy()
        j1[0]["flags"] = j2[0]["flags"]
        j1[0]["hertz"] = j2[0]["hertz"]
        assert j1.tobytes() == j2.tobytes()


def _measure_seam(solver):
    # rest angle pi - 0.05; B starts at -pi + 0.05, 0.1 rad past the seam: it must come back across it, not go round
    ref = math.pi - 0.05
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 0), (capi.DYNAMIC_BODY, 0, 0, -math.pi + 0.05, 0, 0, 0)])
    joints = np.array([_joint(bodies, device.JOINT_REVOLUTE, 0, 1, (0.0, 0.0), ref=ref, spring=(2.0, 1.0))])
    travelled = 0.0
    prev = _angle(bodies, 1)
    hist = _run(joint_oracle.load(), solver, bodies, joints, 180)
    for b, _ in hist:
        a = _angle(b, 1)
        travelled += (a - prev + math.pi) % (2.0 * math.pi) - math.pi
        prev = a
    return abs(travelled + 0.1), abs(_error(device.JOINT_REVOLUTE, hist[-1][0], hist[-1][1][0]))


@pytest.mark.parametrize("solver", VARIANTS)
def test_rest_angle_across_the_seam(solver):
    travel_error, rest_error = _measure_seam(solver)
    assert travel_error <= SEAM_BOUND and rest_error <= SEAM_BOUND


@pytest.mark.parametrize("solver", ["TGS_Soft", "PGS", "TGS_Sticky"])
def test_spring_impulse_is_kept_only_with_the_flag_and_warm_start(solver):
    """The stored spring impulse: nonzero on a loaded spring, 0 once the flag is cleared (the row is re-prepared cold)."""
    bodies, joints = _oscillator(device.JOINT_REVOLUTE, (1.0, 0.2))
    O = joint_oracle.load()
    ctx = device.make_context(solver, DT, 4, 2)
    contacts = np.zeros(0, dtype=device.CONTACT_ROW)
    bodies, _, joints = O.solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, gravity=(0.0, 0.0))
    assert float(joints[0]["springImpulse"]) != 0.0
    joints[0]["flags"] &= ~device.JOINT_ENABLE_SPRING
    bodies["origin"] = bodies["position"]
    bodies, _, joints = O.solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, gravity=(0.0, 0.0))
    assert float(joints[0]["springImpulse"]) == 0.0


def _fixed_rotation_rows():
    bodies = _bodies([(capi.STATIC_BODY, 0, 0, 0, 0, 0, 0), (capi.DYNAMIC_BODY, 0, 0, 0.2, 0.1, 0, 0)])
    bodies[1]["invI"] = 0.0
    return bodies, np.array([_joint(bodies, device.JOINT_REVOLUTE, 0, 1, (0.0, 0.0), spring=(1.0, 0.5))])


@pytest.mark.parametrize("solver", VARIANTS)
def test_revolute_spring_without_rotation_does_nothing(solver):
    bodies, joints = _fixed_rotation_rows()
    off = joints.copy()
    off[0]["flags"] &= ~device.JOINT_ENABLE_SPRING
    O = joint_oracle.load()
    for (b1, j1), (b2, _) in zip(_run(O, solver, bodies, joints, 10), _run(O, solver, bodies, off, 10)):
        assert b1.tobytes() == b2.tobytes() and float(j1[0]["springImpulse"]) == 0.0


def test_springs_scene_stand_ins(reference):
    """scenes.springs on a library without the extension: the prismatic joints become revolute stand-ins with the same
    bodies, no spring is set, and every spring setting is recorded; the stand-in world steps with contacts."""
    from solver2d_b200 import scenes
    sc = scenes.springs(reference, "TGS_Soft", copies=2)
    assert "s2CreatePrismaticJoint" in reference.missing
    assert len(sc.piles["prismatic"]) == 6 and len(sc.piles["springs"]) == 2 * 11
    assert all(hertz > 0.0 for _, hertz, _ in sc.piles["springs"])
    kinds = {k for k, _, _ in sc.piles["springs"]}
    assert set(sc.piles["prismatic"]) <= kinds
    for _ in range(60):
        sc.step()
    _, ci = reference.contacts(sc.world)
    assert (ci[:, 0] == 1).sum() > 10
    sc.destroy()


def test_row_size():
    """s2bJointRow grows by springImpulse at its end (104 -> 108 bytes); the numpy mirror follows."""
    out = (C.c_int32 * 6)()
    C.CDLL(device.LIB_PATH).s2b_abi_sizes(out)
    assert out[2] == 108 == device.JOINT_ROW.itemsize
    assert device.JOINT_ROW.fields["springImpulse"][1] == 104


if __name__ == "__main__":
    for kind, name in zip(KINDS, KIND_IDS):
        print(name, "frequency rel error", {s: round(_measure_frequency(s, kind), 4) for s in VARIANTS})
        print(name, "zeta=1 overshoot", {s: f"{_measure_overshoot(s, kind):.1e}" for s in VARIANTS})
        print(name, "zeta=0 amplitude kept", {s: round(_measure_keep(s, kind), 3) for s in VARIANTS})
        print(name, "momentum drift", {s: f"{_measure_momentum(s, kind):.1e}" for s in VARIANTS})
    print("rest rel error", {s: round(_measure_rest(s), 4) for s in VARIANTS})
    print("seam (travel err, rest err)", {s: tuple(f"{v:.1e}" for v in _measure_seam(s)) for s in VARIANTS})
