"""GPU: the motor joint (DESIGN.md §3.10). The device's motor rows against the joint oracle (tests/joint_oracle.c) bit for
bit, in every schedule, for all ten variants and with the warm-start gather on and off; every step of scenes.motors through
the public API; setter edits between replayed steps; the bulk offset path (s2World_SetMotorJointOffsets) against the
per-joint setters, its precedence rule, its input check and its launch cost; contacts between jointed bodies; the joint's
lifecycle, input checks, getters and debug drawing.

The reference has no motor joint. Its stand-in is the revolute joint that motors creates on a library without
s2CreateMotorJoint: same bodies, anchor A at the linear offset, anchor B at B's origin, and the same collideConnected, so
the reference's collide and finalize stages see the same world. Its rows are turned into motor rows before the oracle runs.

Mutations each test catches: a motor row solved as a revolute (the check against the plain oracle), a cap or correction
factor read from the wrong column, an impulse dropped at prepare or a relax pass that skips the rows fail the stage and
every-step comparisons; a bulk write that misses the host record fails the setter comparison; a bulk write that bumps the
upload epoch fails the launch count; a repeated bulk index whose entries race fails the repeated-index test; motor joints left out of the contact-destroy list fail test_collide_connected."""
import ctypes as C
import math

import numpy as np
import pytest

import joint_oracle
from helpers import (bit_equal, body_rows_from_ref, carry_sticky_friction, contact_rows_from_ref, joint_rows_from_ref,
                     load_bodies_into_ref, ref_delta_positions, store_oracle_bodies)
from oracle import port
from oracle import ref as refmod
from solver2d_b200 import capi, device, scenes
from test_api_lifecycle_gpu import _draw_log

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0
VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]
SUBSTEPPING = {"SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"}
NULL_JOINT = (-1, -1, 0)


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


def _as_motor(joints, slots, defs):
    """Turn the stand-in revolute rows at `slots` into the motor rows `defs` describe."""
    for slot, d in zip(slots, defs):
        r = joints[slot]
        assert r["flags"] & (device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR) == 0
        joints["flags"][slot] = (int(r["flags"]) & ~0xE) | (device.JOINT_MOTOR << 1)
        joints["localOriginAnchorA"][slot] = d["linearOffset"]
        joints["localOriginAnchorB"][slot] = (0.0, 0.0)
        joints["referenceAngle"][slot] = d["angularOffset"]
        joints["maxMotorTorque"][slot] = d["maxTorque"]
        joints["motorSpeed"][slot] = 0.0
        joints["hertz"][slot] = d["maxForce"]
        joints["dampingRatio"][slot] = d["correctionFactor"]
    return joints


def _slots(sc):
    return [sc.joints[k].index for k in sc.piles["motor"]]


def _set_offsets(lib, world, slots, offsets):
    slots = np.ascontiguousarray(slots, dtype=np.int32)
    offsets = np.ascontiguousarray(offsets, dtype=np.float32)
    return bool(lib.s2World_SetMotorJointOffsets(world, slots.ctypes.data, offsets.ctypes.data, len(slots)))


def _apply_offsets(joints, slots, offsets):
    for slot, (x, y, angle) in zip(slots, offsets):
        joints["localOriginAnchorA"][slot] = (x, y)
        joints["referenceAngle"][slot] = angle
    return joints


def _flush(dev, world):
    dev.lib.s2World_Flush.restype = None
    dev.lib.s2World_Flush.argtypes = [capi.WorldId]
    dev.lib.s2World_Flush(world)


def _compare(got, got_contacts, got_joints, ob, oc, oj, bodies, contacts):
    valid = (bodies["flags"] & 1) == 1
    for name in ("position", "rot", "linearVelocity", "angularVelocity"):
        assert bit_equal(got[name][valid], ob[name][valid]), name
    live = contacts["pointCount"] > 0
    for name in ("normalImpulse", "tangentImpulse"):
        assert bit_equal(got_contacts["points"][name][live], oc["points"][name][live]), name
    jv = (oj["flags"] & 1) == 1
    for name in ("impulse", "motorImpulse", "lowerImpulse", "upperImpulse"):
        assert bit_equal(got_joints[name][jv], oj[name][jv]), name


# ---- one solver stage against the oracle --------------------------------------------------------------------------------

@pytest.mark.parametrize("gather", [True, False])
@pytest.mark.parametrize("persistent", [True, False])
@pytest.mark.parametrize("mode", ["wavefront", "color", "regions"])
@pytest.mark.parametrize("solver", VARIANTS)
def test_stage_matches_oracle(reference, dev, solver, mode, persistent, gather):
    """One stage of motors rows (motor joints at and away from their caps, a mouse joint, contacts), the motor joints
    warm-started with random impulses."""
    if not gather and solver not in SUBSTEPPING:
        pytest.skip("the warm-start gather serves the sub-stepping variants only")
    R = reference
    O = joint_oracle.load()
    sc = scenes.motors(R, solver, copies=2)
    for _ in range(30):
        sc.step(DT, 4, 2, True)
    R.step_collide(sc.world)
    bodies = body_rows_from_ref(*R.bodies(sc.world))
    contacts, _ = contact_rows_from_ref(*R.contacts(sc.world))
    joints = _as_motor(joint_rows_from_ref(*R.joints(sc.world)), _slots(sc), sc.piles["motor_defs"])
    sc.destroy()
    motor = (joints["flags"] >> 1 & 0x7) == device.JOINT_MOTOR
    assert motor.sum() >= 20 and len(contacts) > 10
    rng = np.random.default_rng(7)
    n = int(motor.sum())
    joints["impulse"][motor] = rng.uniform(-0.05, 0.05, (n, 2)).astype(np.float32)
    joints["motorImpulse"][motor] = rng.uniform(-0.02, 0.02, n).astype(np.float32)
    ctx = device.make_context(solver, DT, 4, 2)

    dw = dev.create_world(capi.SOLVER[solver])
    dw.upload_bodies(bodies, len(bodies))
    dw.upload_joints(joints, len(joints))
    dw.upload_contacts(contacts)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT if mode == "wavefront" else device.SCHEDULE_COLOR)
    dw.set_regions(2 if mode == "regions" else 0)
    dw.set_persistent(persistent)
    dw.set_warm_gather(gather)
    dw.solve(ctx)
    got = dw.download_all_bodies(len(bodies))
    got_contacts = dw.download_contacts(len(contacts))
    got_joints = dw.download_joints(len(joints))
    order, _ = dw.solve_order(len(contacts) + len(joints))
    dw.destroy()
    order = None if mode == "wavefront" else order
    ob, oc, oj = O.solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, order=order)
    _compare(got, got_contacts, got_joints, ob, oc, oj, bodies, contacts)
    # the motor rows did work: the plain oracle, which solves an unknown joint type as a revolute, ends elsewhere
    pb, _, _ = port.load().solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, order=order)
    valid = (bodies["flags"] & 1) == 1
    assert not bit_equal(pb["position"][valid], ob["position"][valid])


# ---- every step through the public API -----------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", VARIANTS)
def test_motors_every_step(reference, product, dev, solver):
    """Reference collide on the stand-in world, the motor oracle in the device's order, reference finalize; the device runs
    the same steps through s2World_Step with real motor joints, its platforms re-targeted every step through
    s2World_SetMotorJointOffsets. Every step bit for bit: bodies (the kinematic carriage and XPBD's delta positions
    included), contact and joint impulses."""
    R, P = reference, product
    O = joint_oracle.load()
    sr = scenes.motors(R, solver)
    sp = scenes.motors(P, solver)
    assert "s2CreateMotorJoint" in R.missing and "s2CreateMotorJoint" not in P.missing
    slots = _slots(sp)
    assert slots == _slots(sr)
    _flush(dev, sp.world)
    dw = device.DeviceWorld.attach(dev, sp.world)
    ctx = device.make_context(solver, DT, 4, 2, True)
    sticky = solver == "TGS_Sticky"
    solved = {}
    F = refmod.BODY_F
    contacts_seen = 0
    capped = 0
    for step in range(60):
        pslots, poffsets = scenes.motors_platform_offsets(sp, step, DT)
        assert _set_offsets(P, sp.world, pslots, poffsets)
        cap = R.capacities(sr.world)["bodyCap"]
        load_bodies_into_ref(R, sr.world, dw.download_all_bodies(cap))
        R.step_collide(sr.world)
        sp.step(DT, 4, 2, True)

        bodies = body_rows_from_ref(*R.bodies(sr.world))
        cf, ci = R.contacts(sr.world)
        rows_slot, cslots = contact_rows_from_ref(cf, ci)
        keys = (np.minimum(rows_slot["shapeA"], rows_slot["shapeB"]).astype(np.uint64) << np.uint64(32)) | \
            np.maximum(rows_slot["shapeA"], rows_slot["shapeB"]).astype(np.uint64)
        perm = np.argsort(keys, kind="stable")
        rows_key = rows_slot[perm]
        if sticky:
            carry_sticky_friction(rows_key, keys[perm], solved)
        joints = _as_motor(joint_rows_from_ref(*R.joints(sr.world)), slots, sr.piles["motor_defs"])
        joints = _apply_offsets(joints, pslots, poffsets)
        got_contacts = dw.download_contacts(len(rows_key) + 64)
        assert len(got_contacts) == len(rows_key) and np.array_equal(got_contacts["shapeA"], rows_key["shapeA"]), step
        contacts_seen += len(rows_key)

        order, _ = dw.solve_order(len(rows_key) + len(joints) + 16, max_groups=200000)
        ob, oc, oj, odp = O.solve(capi.SOLVER[solver], bodies, rows_key, joints, ctx, order=order,
                                  dp=ref_delta_positions(R, sr.world))
        lam = np.linalg.norm(oj["impulse"][slots].astype(np.float64), axis=1)
        capped += int(np.count_nonzero(np.abs(lam - ctx.h * joints["hertz"][slots]) <= 1e-6 * ctx.h * joints["hertz"][slots]))

        store_oracle_bodies(R, sr.world, ob, odp)
        imp = np.zeros((cf.shape[0], 4), dtype=np.float32)
        imp[cslots[perm], 0] = oc["points"]["normalImpulse"][:, 0]
        imp[cslots[perm], 1] = oc["points"]["tangentImpulse"][:, 0]
        imp[cslots[perm], 2] = oc["points"]["normalImpulse"][:, 1]
        imp[cslots[perm], 3] = oc["points"]["tangentImpulse"][:, 1]
        R.load_contact_impulses(sr.world, imp)
        if sticky:
            solved = dict(zip(keys[perm].tolist(), oc.copy()))
        # the stand-in's impulse columns carry the motor impulses into the next step
        jimp = np.zeros((len(oj), 5), dtype=np.float32)
        jimp[:, 0:2] = oj["impulse"]
        jimp[:, 2] = oj["motorImpulse"]
        jimp[:, 3] = oj["lowerImpulse"]
        jimp[:, 4] = oj["upperImpulse"]
        R.load_joint_impulses(sr.world, jimp)
        R.step_finalize(sr.world)

        post = dw.download_all_bodies(cap)
        rf, ri = R.bodies(sr.world)
        v = ri[:, 0] == 1
        for name, col in (("position", F["position"]), ("rot", F["rot"]), ("linearVelocity", F["v"])):
            assert bit_equal(post[name][v], rf[v, col:col + 2]), f"step {step}: {name}"
        assert bit_equal(post["angularVelocity"][v], rf[v, F["w"]]), f"step {step}: angularVelocity"
        assert bit_equal(dw.download_delta_positions(cap)[v], rf[v, F["dp"]:F["dp"] + 2]), f"step {step}: deltaPosition"
        live = rows_key["pointCount"] > 0
        got_after = dw.download_contacts(len(rows_key) + 64)
        assert bit_equal(got_after["points"]["normalImpulse"][live], oc["points"]["normalImpulse"][live]), f"step {step}"
        gj = dw.download_joints(len(oj))
        jv = (oj["flags"] & 1) == 1
        for name in ("impulse", "motorImpulse", "lowerImpulse", "upperImpulse", "localOriginAnchorA", "referenceAngle"):
            assert bit_equal(gj[name][jv], oj[name][jv]), f"step {step}: joint {name}"
    assert contacts_seen > 100
    if solver != "XPBD":  # XPBD keeps no impulses
        assert capped > 0  # some motor (the weak one, the top-down brakes) worked at its force cap
    sp.destroy()
    sr.destroy()


# ---- a single motor joint: edits, bulk path ------------------------------------------------------------------------------

def _single(L, solver, velocity=(0.0, 0.0)):
    """A static post and a 1 kg box hanging 1.5 m below it on a motor joint (maxForce 20 N): every step is one oracle stage
    (no contacts). `velocity` throws the box; with gravityScale 0 it coasts."""
    wid = L.create_world(solver)
    bd = capi.default_body_def()
    bd.position = capi.Vec2(0.0, 4.0)
    post = L.s2CreateBody(wid, C.byref(bd))
    sd = capi.default_shape_def()
    L.s2CreatePolygonShape(post, C.byref(sd), C.byref(L.s2MakeBox(0.25, 0.25)))
    bd = capi.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    bd.position = capi.Vec2(0.0, 2.5)
    bd.linearVelocity = capi.Vec2(*velocity)
    if velocity != (0.0, 0.0):
        bd.gravityScale = 0.0
    box = L.s2CreateBody(wid, C.byref(bd))
    L.s2CreatePolygonShape(box, C.byref(sd), C.byref(L.s2MakeBox(0.5, 0.5)))
    jd = capi.default_motor_def()
    jd.bodyIdA, jd.bodyIdB = post, box
    jd.linearOffset = capi.Vec2(0.0, -1.5)
    jd.maxForce = 20.0 if velocity == (0.0, 0.0) else 0.0
    jd.maxTorque = 5.0
    return wid, box, L.s2CreateMotorJoint(wid, C.byref(jd))


@pytest.mark.parametrize("solver", ["TGS_Soft", "PGS_NGS", "PGS", "XPBD"])
def test_edits_between_steps(product, dev, solver):
    """Every setter between steps of a captured, replayed step graph: each takes effect at the next step, every step matches
    the oracle run on the rows the host now holds, and the getters return what was set."""
    P = product
    O = joint_oracle.load()
    wid, box, jid = _single(P, solver)
    _flush(dev, wid)
    dw = device.DeviceWorld.attach(dev, wid)
    ctx = device.make_context(solver, DT, 4, 2, True)
    edits = {10: [lambda: P.s2MotorJoint_SetLinearOffset(jid, capi.Vec2(1.0, -1.0))],
             20: [lambda: P.s2MotorJoint_SetAngularOffset(jid, 1.0)],
             30: [lambda: P.s2MotorJoint_SetMaxForce(jid, 4.0)],
             45: [lambda: P.s2MotorJoint_SetMaxForce(jid, 50.0), lambda: P.s2MotorJoint_SetCorrectionFactor(jid, 0.1)],
             55: [lambda: P.s2MotorJoint_SetMaxTorque(jid, 0.05), lambda: P.s2MotorJoint_SetAngularOffset(jid, -1.0)]}
    for step in range(70):
        for edit in edits.get(step, []):
            edit()
        _flush(dev, wid)
        bodies = dw.download_all_bodies(2)
        joints = dw.download_joints(1)
        ob, _, oj = O.solve(capi.SOLVER[solver], bodies, np.zeros(0, dtype=device.CONTACT_ROW), joints, ctx)
        P.s2World_Step(wid, DT, 4, 2, True)
        got = dw.download_all_bodies(2)
        for name in ("position", "rot", "linearVelocity", "angularVelocity"):
            assert bit_equal(got[name], ob[name]), f"step {step}: {name}"
        gj = dw.download_joints(1)
        for name in ("impulse", "motorImpulse"):
            assert bit_equal(gj[name], oj[name]), f"step {step}: {name}"
    assert dw.counters().graphReplays > 0
    r = dw.download_joints(1)[0]
    assert tuple(r["localOriginAnchorA"]) == (1.0, -1.0) and r["referenceAngle"] == np.float32(-1.0)
    assert (r["hertz"], r["dampingRatio"], r["maxMotorTorque"]) == (50.0, np.float32(0.1), np.float32(0.05))
    assert tuple(P.s2MotorJoint_GetLinearOffset(jid)) == (1.0, -1.0)
    assert P.s2MotorJoint_GetAngularOffset(jid) == np.float32(-1.0)
    if solver != "XPBD":
        f = P.s2MotorJoint_GetConstraintForce(jid, 1.0 / ctx.h)
        assert (f.x, f.y) == tuple(np.float32(r["impulse"] * np.float32(1.0 / ctx.h)))
        assert P.s2MotorJoint_GetConstraintTorque(jid, 1.0 / ctx.h) == np.float32(r["motorImpulse"] * np.float32(1.0 / ctx.h))
    P.s2DestroyWorld(wid)


@pytest.mark.parametrize("solver", VARIANTS)
def test_zero_force_cap_matches_oracle(product, dev, solver):
    """A box coasting along x below its post on a motor joint with maxForce 0: every step the linear impulse is scaled back to
    length 0, so its components are zeros whose signs depend on how the total impulse is formed. Every step matches the
    oracle bit for bit, the impulse columns included, through the persistent kernels (the soft variants' shared branches)."""
    P = product
    O = joint_oracle.load()
    wid, _, _ = _single(P, solver, velocity=(3.0, 0.0))
    _flush(dev, wid)
    dw = device.DeviceWorld.attach(dev, wid)
    ctx = device.make_context(solver, DT, 4, 2, True)
    for step in range(30):
        bodies = dw.download_all_bodies(2)
        joints = dw.download_joints(1)
        ob, _, oj = O.solve(capi.SOLVER[solver], bodies, np.zeros(0, dtype=device.CONTACT_ROW), joints, ctx)
        P.s2World_Step(wid, DT, 4, 2, True)
        got = dw.download_all_bodies(2)
        for name in ("position", "rot", "linearVelocity", "angularVelocity"):
            assert bit_equal(got[name], ob[name]), f"step {step}: {name}"
        gj = dw.download_joints(1)
        for name in ("impulse", "motorImpulse"):
            assert bit_equal(gj[name], oj[name]), f"step {step}: {name}"
    P.s2DestroyWorld(wid)


def test_bulk_repeated_index_takes_last(product, dev):
    """A joint named several times in one bulk call takes its last entry, on the device as in the getters, and a joint
    between its repeats keeps its own entry; the same call repeated in a second world gives the same bits."""
    P = product
    results = []
    for _ in range(2):
        wid, box, jid = _single(P, "TGS_Soft")
        md = capi.default_motor_def()
        md.bodyIdA = box
        bd = capi.default_body_def()
        bd.type = capi.DYNAMIC_BODY
        bd.position = capi.Vec2(3.0, 2.5)
        other = P.s2CreateBody(wid, C.byref(bd))
        md.bodyIdB = other
        md.linearOffset = capi.Vec2(3.0, 0.0)
        j2 = P.s2CreateMotorJoint(wid, C.byref(md))
        P.s2World_Step(wid, DT, 4, 2, True)
        dw = device.DeviceWorld.attach(dev, wid)
        slots = [jid.index, j2.index, jid.index, jid.index]
        offsets = [(1.0, -1.0, 0.5), (2.5, 0.25, -0.5), (-1.0, -2.0, 1.0), (0.25, -1.25, -0.25)]
        assert _set_offsets(P, wid, slots, offsets)
        want = np.array(offsets, dtype=np.float32)
        rows = dw.download_joints(max(jid.index, j2.index) + 1)
        for j, w in ((jid, want[3]), (j2, want[1])):
            r = rows[j.index]
            assert bit_equal(r["localOriginAnchorA"], w[:2]) and r["referenceAngle"] == w[2], (j.index, r)
            assert tuple(P.s2MotorJoint_GetLinearOffset(j)) == tuple(w[:2]) and P.s2MotorJoint_GetAngularOffset(j) == w[2]
        for _ in range(10):
            P.s2World_Step(wid, DT, 4, 2, True)
        results.append(dw.download_all_bodies(3))
        P.s2DestroyWorld(wid)
    for name in ("position", "rot", "linearVelocity", "angularVelocity"):
        assert bit_equal(results[0][name], results[1][name]), name


def _targets(step):
    return np.array([[0.5 * math.sin(0.1 * step), -1.5 + 0.25 * math.cos(0.07 * step), 0.02 * step]], dtype=np.float32)


@pytest.mark.parametrize("solver", ["TGS_Soft", "PGS", "TGS_NGS", "XPBD"])
def test_bulk_equals_setters(product, dev, solver):
    """N steps re-targeted by s2World_SetMotorJointOffsets end bit for bit where the same N steps re-targeted by
    s2MotorJoint_SetLinearOffset / _SetAngularOffset end, and the getters agree after each."""
    P = product
    wa, ba, ja = _single(P, solver)
    wb, bb, jb = _single(P, solver)
    da = device.DeviceWorld.attach(dev, wa)
    db = device.DeviceWorld.attach(dev, wb)
    for step in range(60):
        t = _targets(step)
        P.s2MotorJoint_SetLinearOffset(ja, capi.Vec2(float(t[0, 0]), float(t[0, 1])))
        P.s2MotorJoint_SetAngularOffset(ja, float(t[0, 2]))
        assert _set_offsets(P, wb, [jb.index], t)
        assert tuple(P.s2MotorJoint_GetLinearOffset(jb)) == tuple(t[0, :2]) and P.s2MotorJoint_GetAngularOffset(jb) == t[0, 2]
        P.s2World_Step(wa, DT, 4, 2, True)
        P.s2World_Step(wb, DT, 4, 2, True)
        ra, rb = da.download_all_bodies(2), db.download_all_bodies(2)
        for name in ("position", "rot", "linearVelocity", "angularVelocity"):
            assert bit_equal(ra[name], rb[name]), f"step {step}: {name}"
        assert bit_equal(da.download_joints(1)["impulse"], db.download_joints(1)["impulse"]), step
    P.s2DestroyWorld(wa)
    P.s2DestroyWorld(wb)


def test_bulk_last_call_wins(product, dev):
    """Mixed calls before one step: whichever of the setter and the bulk call wrote an offset last is the one the step
    solves with, on the device and in the getters."""
    P = product
    wid, _, jid = _single(P, "TGS_Soft")
    dw = device.DeviceWorld.attach(dev, wid)
    P.s2World_Step(wid, DT, 4, 2, True)
    cases = [
        # (setter first, then bulk) -> bulk
        ([("set", (1.0, -1.0, 0.2)), ("bulk", (2.0, -2.0, 0.3))], (2.0, -2.0, 0.3)),
        # (bulk first, then setter) -> setter
        ([("bulk", (2.5, -1.0, 0.1)), ("set", (-1.0, -0.5, -0.4))], (-1.0, -0.5, -0.4)),
        # bulk, setter, bulk -> the last bulk
        ([("bulk", (0.5, -1.0, 0.0)), ("set", (0.25, -1.25, 0.5)), ("bulk", (0.75, -1.75, -0.5))], (0.75, -1.75, -0.5)),
    ]
    for calls, expected in cases:
        for kind, (x, y, a) in calls:
            if kind == "set":
                P.s2MotorJoint_SetLinearOffset(jid, capi.Vec2(x, y))
                P.s2MotorJoint_SetAngularOffset(jid, a)
            else:
                assert _set_offsets(P, wid, [jid.index], [(x, y, a)])
        P.s2World_Step(wid, DT, 4, 2, True)
        r = dw.download_joints(1)[0]
        want = np.array(expected, dtype=np.float32)
        assert bit_equal(r["localOriginAnchorA"], want[:2]) and r["referenceAngle"] == want[2], (calls, r)
        assert tuple(P.s2MotorJoint_GetLinearOffset(jid)) == tuple(want[:2]) and P.s2MotorJoint_GetAngularOffset(jid) == want[2]
    P.s2DestroyWorld(wid)


def test_bulk_rejects_invalid(product, dev):
    """An index out of range, a free slot, a joint that is not a motor joint or a non-finite value: the call returns false
    and changes no offset, valid entries in the same call included."""
    P = product
    wid, box, jid = _single(P, "TGS_Soft")
    jd = capi.default_revolute_def()
    bd = capi.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    other = P.s2CreateBody(wid, C.byref(bd))
    jd.bodyIdA, jd.bodyIdB = box, other
    rev = P.s2CreateRevoluteJoint(wid, C.byref(jd))
    md = capi.default_motor_def()
    md.bodyIdA, md.bodyIdB = other, box
    gone = P.s2CreateMotorJoint(wid, C.byref(md))
    P.s2DestroyJoint(gone)
    P.s2World_Step(wid, DT, 4, 2, True)
    dw = device.DeviceWorld.attach(dev, wid)
    before = dw.download_joints(3)
    good = (0.25, -1.0, 0.5)
    bad = [([jid.index, 1000], [good, good]), ([jid.index, -1], [good, good]), ([jid.index, rev.index], [good, good]),
           ([jid.index, gone.index], [good, good]), ([jid.index], [(math.nan, 0.0, 0.0)]), ([jid.index], [(0.0, math.inf, 0.0)]),
           ([jid.index], [(0.0, 0.0, -math.inf)])]
    for slots, offsets in bad:
        assert not _set_offsets(P, wid, slots, offsets), slots
        assert tuple(P.s2MotorJoint_GetLinearOffset(jid)) == (0.0, -1.5) and P.s2MotorJoint_GetAngularOffset(jid) == 0.0
    P.s2World_Step(wid, DT, 4, 2, True)
    after = dw.download_joints(3)
    for name in ("localOriginAnchorA", "referenceAngle"):
        assert bit_equal(after[name], before[name]), name
    assert _set_offsets(P, wid, [], np.zeros((0, 3)))
    P.s2DestroyWorld(wid)


def test_bulk_launch_cost(product, dev):
    """Three identical worlds with a coasting box (its proxy leaves its fat box every few steps, so the broad phase has work):
    one unedited, one re-targeted every step through the bulk call with its current offset (the physics stays identical),
    one through the per-joint setters. The bulk world launches exactly one kernel more per step (the scatter) and captures no
    more graphs; the setter world launches more (the row upload's scatter), and each of its uploads discards the pair
    search prefetched behind the previous step, which then runs again inside the step."""
    P = product
    worlds = [_single(P, "TGS_Soft", velocity=(3.0, 0.0)) for _ in range(3)]
    views = [device.DeviceWorld.attach(dev, w) for w, _, _ in worlds]
    offset = np.array([[0.0, -1.5, 0.0]], dtype=np.float32)
    for w, _, _ in worlds:
        P.s2World_Step(w, DT, 4, 2, True)
    base = [v.counters() for v in views]
    per_step = [[], [], []]
    for step in range(40):
        for k, (w, _, j) in enumerate(worlds):
            if k == 2:
                # (the setter's own read-back of the impulses is not counted: only what the step then launches)
                P.s2MotorJoint_SetLinearOffset(j, capi.Vec2(0.0, -1.5))
            before = views[k].counters().kernelLaunches
            if k == 1:
                assert _set_offsets(P, w, [j.index], offset)
            P.s2World_Step(w, DT, 4, 2, True)
            per_step[k].append(views[k].counters().kernelLaunches - before)
    plain, bulk, setter = (np.array(x) for x in per_step)
    assert np.array_equal(bulk, plain + 1), (plain, bulk)
    assert np.all(setter >= plain) and setter.sum() > plain.sum(), (plain, setter)
    assert views[1].counters().graphCaptures == views[0].counters().graphCaptures
    assert views[1].counters().graphCaptures - base[1].graphCaptures == views[0].counters().graphCaptures - base[0].graphCaptures
    r = [v.download_all_bodies(2) for v in views]
    assert bit_equal(r[0]["position"], r[1]["position"]) and bit_equal(r[0]["position"], r[2]["position"])
    for w, _, _ in worlds:
        P.s2DestroyWorld(w)


# ---- contacts between jointed bodies ------------------------------------------------------------------------------------

def _overlapping_pair(L, solver):
    wid = L.create_world(solver)
    bd = capi.default_body_def()
    bd.position = capi.Vec2(0.0, -1.0)
    gid = L.s2CreateBody(wid, C.byref(bd))
    sd = capi.default_shape_def()
    L.s2CreatePolygonShape(gid, C.byref(sd), C.byref(L.s2MakeBox(20.0, 1.0)))
    ids = []
    for x in (0.0, 0.8):
        bd = capi.default_body_def()
        bd.type = capi.DYNAMIC_BODY
        bd.position = capi.Vec2(x, 0.5)
        bid = L.s2CreateBody(wid, C.byref(bd))
        L.s2CreatePolygonShape(bid, C.byref(sd), C.byref(L.s2MakeBox(0.5, 0.5)))
        ids.append(bid)
    return wid, gid, ids


def _create_motor(L, wid, a, b, collide, **kw):
    if "s2CreateMotorJoint" in L.missing:
        jd = capi.default_revolute_def()
        jd.localAnchorA = capi.Vec2(0.8, 0.0)
        fn = L.s2CreateRevoluteJoint
    else:
        jd = capi.default_motor_def()
        jd.linearOffset = capi.Vec2(0.8, 0.0)
        for name, value in kw.items():
            setattr(jd, name, value)
        fn = L.s2CreateMotorJoint
    jd.bodyIdA, jd.bodyIdB = a, b
    jd.collideConnected = collide
    return fn(wid, C.byref(jd))


def _pairs_ref(R, wid):
    _, ci = R.contacts(wid)
    I = refmod.CONTACT_I
    live = ci[ci[:, I["valid"]] == 1]
    return sorted((int(min(a, b)), int(max(a, b))) for a, b in zip(live[:, I["bodyA"]], live[:, I["bodyB"]]))


def _pairs_dev(dw):
    c = dw.download_contacts(256)
    return sorted((int(min(a, b)), int(max(a, b))) for a, b in zip(c["bodyA"], c["bodyB"]))


@pytest.mark.parametrize("collide", [False, True])
def test_collide_connected(reference, product, dev, collide):
    """Two overlapping boxes: the motor joint removes their contact unless collideConnected, and no new one forms while it
    lives; destroying it lets the pair come back. While the joint lives the pair table matches the reference's stand-in."""
    R, P = reference, product
    wr, _, br = _overlapping_pair(R, "TGS_Soft")
    wp, _, bp = _overlapping_pair(P, "TGS_Soft")
    dw = device.DeviceWorld.attach(dev, wp)
    pair = (bp[0].index, bp[1].index)
    for _ in range(3):
        R.s2World_Step(wr, DT, 4, 2, True)
        P.s2World_Step(wp, DT, 4, 2, True)
    assert pair in _pairs_dev(dw)
    jr = _create_motor(R, wr, br[0], br[1], collide)
    jp = _create_motor(P, wp, bp[0], bp[1], collide)
    _flush(dev, wp)
    rows = dw.download_joints(1)
    assert (rows["flags"][0] >> 1 & 0x7) == device.JOINT_MOTOR
    assert bool(rows["flags"][0] & device.JOINT_COLLIDE_CONNECTED) == collide
    back = None
    for step in range(80):
        if step == 20:
            R.s2DestroyJoint(jr)
            P.s2DestroyJoint(jp)
            for L, b in ((R, br[1]), (P, bp[1])):
                L.s2Body_SetLinearVelocity(b, capi.Vec2(0.0, 3.0))
        R.s2World_Step(wr, DT, 4, 2, True)
        P.s2World_Step(wp, DT, 4, 2, True)
        pairs = _pairs_dev(dw)
        if step < 20:
            assert pairs == _pairs_ref(R, wr), step
            assert (pair in pairs) == collide, step
        elif back is None and pair in pairs:
            back = step
    assert back is not None, "the pair did not come back after the joint was destroyed"
    R.s2DestroyWorld(wr)
    P.s2DestroyWorld(wp)


# ---- lifecycle, input checks, drawing -------------------------------------------------------------------------------------

def test_slot_reuse_across_types(product, dev):
    """One joint slot is reused by a motor, a revolute, a weld, a prismatic, a mouse and a motor joint again; the downloaded
    row carries the right type and columns each time, and destroying the joint and its bodies leaves no joint behind."""
    P = product
    wid, gid, (a, b) = _overlapping_pair(P, "TGS_Soft")
    dw = device.DeviceWorld.attach(dev, wid)

    def row(j):
        P.s2World_Step(wid, DT, 4, 2, True)
        return dw.download_joints(j.index + 1)[j.index]

    def kind(r):
        return int(r["flags"]) >> 1 & 0x7

    m = _create_motor(P, wid, a, b, False, angularOffset=0.5, maxForce=7.0, maxTorque=3.0, correctionFactor=0.25)
    r = row(m)
    assert kind(r) == device.JOINT_MOTOR and r["flags"] & (device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR) == 0
    assert tuple(r["localOriginAnchorA"]) == (np.float32(0.8), 0.0) and not np.any(r["localOriginAnchorB"])
    assert (r["referenceAngle"], r["hertz"], r["maxMotorTorque"], r["dampingRatio"]) == (0.5, 7.0, 3.0, 0.25)
    P.s2DestroyJoint(m)
    jd = capi.default_revolute_def()
    jd.bodyIdA, jd.bodyIdB = a, b
    rv = P.s2CreateRevoluteJoint(wid, C.byref(jd))
    assert rv.index == m.index and kind(row(rv)) == device.JOINT_REVOLUTE
    P.s2DestroyJoint(rv)
    wd = capi.default_weld_def()
    wd.bodyIdA, wd.bodyIdB = a, b
    w = P.s2CreateWeldJoint(wid, C.byref(wd))
    assert w.index == m.index and kind(row(w)) == device.JOINT_WELD
    P.s2DestroyJoint(w)
    pd = capi.default_prismatic_def()
    pd.bodyIdA, pd.bodyIdB = a, b
    p = P.s2CreatePrismaticJoint(wid, C.byref(pd))
    assert p.index == m.index and kind(row(p)) == device.JOINT_PRISMATIC
    P.s2DestroyJoint(p)
    md = capi.default_mouse_def()
    md.bodyIdA, md.bodyIdB = gid, b
    md.target = capi.Vec2(1.0, 1.0)
    ms = P.s2CreateMouseJoint(wid, C.byref(md))
    r = row(ms)
    assert ms.index == m.index and kind(r) == device.JOINT_MOUSE and r["hertz"] == 15.0
    P.s2DestroyJoint(ms)
    m2 = _create_motor(P, wid, a, b, True)
    r = row(m2)
    assert m2.index == m.index and kind(r) == device.JOINT_MOTOR and r["flags"] & device.JOINT_COLLIDE_CONNECTED
    assert (r["referenceAngle"], r["hertz"], r["maxMotorTorque"], r["dampingRatio"]) == (0.0, 1.0, 1.0, np.float32(0.3))
    assert not np.any(r["target"]) and not np.any(r["localAxisA"])
    P.s2DestroyJoint(m2)
    P.s2DestroyBody(a)
    P.s2DestroyBody(b)
    for _ in range(3):
        P.s2World_Step(wid, DT, 4, 2, True)
    assert P.s2World_GetStatistics(wid).jointCount == 0
    assert (dw.download_joints(m.index + 1)["flags"] & 1).sum() == 0
    P.s2DestroyWorld(wid)


def test_create_and_setters_reject_bad_input(product, dev):
    """A non-finite offset, a negative or non-finite cap, or a correction factor outside [0, 1] creates nothing and returns
    the null joint id; the setters ignore such input and the joint keeps its values."""
    P = product
    wid, _, (a, b) = _overlapping_pair(P, "TGS_Soft")
    bad = [dict(linearOffset=capi.Vec2(math.nan, 0.0)), dict(linearOffset=capi.Vec2(0.0, math.inf)),
           dict(angularOffset=math.nan), dict(maxForce=-1.0), dict(maxForce=math.inf), dict(maxTorque=-0.5),
           dict(maxTorque=math.nan), dict(correctionFactor=-0.1), dict(correctionFactor=1.5),
           dict(correctionFactor=math.nan)]
    for kw in bad:
        j = _create_motor(P, wid, a, b, False, **kw)
        assert (j.index, j.world, j.revision) == NULL_JOINT, kw
    assert P.s2World_GetStatistics(wid).jointCount == 0
    j = _create_motor(P, wid, a, b, False, maxForce=0.0, maxTorque=0.0, correctionFactor=1.0)
    assert j.index >= 0 and P.s2World_GetStatistics(wid).jointCount == 1
    P.s2MotorJoint_SetLinearOffset(j, capi.Vec2(math.nan, 1.0))
    P.s2MotorJoint_SetAngularOffset(j, math.inf)
    P.s2MotorJoint_SetMaxForce(j, -2.0)
    P.s2MotorJoint_SetMaxTorque(j, math.nan)
    P.s2MotorJoint_SetCorrectionFactor(j, 2.0)
    P.s2World_Step(wid, DT, 4, 2, True)
    r = device.DeviceWorld.attach(dev, wid).download_joints(j.index + 1)[j.index]
    assert tuple(r["localOriginAnchorA"]) == (np.float32(0.8), 0.0) and r["referenceAngle"] == 0.0
    assert (r["hertz"], r["maxMotorTorque"], r["dampingRatio"]) == (0.0, 0.0, 1.0)
    assert tuple(P.s2MotorJoint_GetLinearOffset(j)) == (np.float32(0.8), 0.0) and P.s2MotorJoint_GetAngularOffset(j) == 0.0
    P.s2DestroyWorld(wid)


def test_draw_one_motor(product, dev):
    """s2World_Draw draws a motor joint as the segment from its target point (A's linear offset) to B's origin."""
    P = product
    wid = P.create_world("TGS_Soft")
    bd = capi.default_body_def()
    bd.position = capi.Vec2(1.0, 2.0)
    bd.angle = 0.5 * math.pi
    a = P.s2CreateBody(wid, C.byref(bd))
    bd = capi.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    bd.position = capi.Vec2(-1.0, 3.5)
    b = P.s2CreateBody(wid, C.byref(bd))
    jd = capi.default_motor_def()
    jd.bodyIdA, jd.bodyIdB = a, b
    jd.linearOffset = capi.Vec2(2.0, 0.0)
    P.s2CreateMotorJoint(wid, C.byref(jd))
    log = _draw_log(P, wid)
    segments = [v for name, v in log if name == "DrawSegment"]
    assert len(segments) == 1
    f = np.float32
    s, c = f(math.sin(f(0.5 * math.pi))), f(math.cos(f(0.5 * math.pi)))
    pa = (f(c * f(2.0) - s * f(0.0)) + f(1.0), f(s * f(2.0) + c * f(0.0)) + f(2.0))
    seg = segments[0]
    assert abs(seg[0] - pa[0]) <= 1e-6 and abs(seg[1] - pa[1]) <= 1e-6, seg   # (1, 4): A's offset point
    assert seg[2:4] == (-1.0, 3.5)                                             # B's origin
    assert seg[4:] == tuple(float(f(x)) for x in (0.8, 0.5, 0.9))
    points = [v for name, v in log if name == "DrawPoint"]
    assert any(p[:2] == (-1.0, 3.5) for p in points)
    P.s2DestroyWorld(wid)
