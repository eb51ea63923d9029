"""GPU: joint springs on revolute and prismatic joints (DESIGN.md §3.14). The device's spring rows against the spring oracle
(tests/spring_oracle.c) bit for bit, in every schedule, for all ten variants, persistent and launch by launch, with the
warm-start gather on and off; every step of scenes.springs (cars on suspension springs over bumps, a soft chain falling on a
pile, contacts throughout) through the public API against reference collide and finalize around the spring oracle, with
the kinematic carriage and XPBD's delta positions carried; a contact-free world stepped against the oracle alone; setter
edits between replayed steps; slot reuse across joint types; input
checks; reactions that include the spring's load and a break threshold that the spring's load trips.

Mutations each test catches: a spring coefficient formed with another h or expression order, a spring row placed after
the motor, a warm start or gather that leaves the spring impulse out of the axial sum (or adds it on a row without the
flag), XPBD's start pose read from the wrong column, and a spring impulse dropped at upload, prepare or download all fail
the stage and every-step comparisons; a reaction that leaves the spring impulse out fails the reaction tests."""
import ctypes as C
import math

import numpy as np
import pytest

import prismatic_oracle
import spring_oracle
from helpers import (bit_equal, body_rows_from_ref, carry_sticky_friction, contact_rows_from_ref, joint_rows_from_ref,
                     load_bodies_into_ref, ref_delta_positions, store_oracle_bodies)
from oracle import ref as refmod
from solver2d_b200 import capi, device, scenes
from test_prismatic_gpu import _as_prismatic, _flush, _slots

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0
VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]
SUBSTEPPING = {"SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"}
JOINT_FIELDS = ("impulse", "motorImpulse", "lowerImpulse", "upperImpulse", "springImpulse")


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


def _compare_bodies(got, ob, valid):
    for name in ("position", "rot", "linearVelocity", "angularVelocity"):
        assert bit_equal(got[name][valid], ob[name][valid]), name


def _compare_joints(got, oj):
    jv = (oj["flags"] & 1) == 1
    for name in JOINT_FIELDS:
        assert bit_equal(got[name][jv], oj[name][jv]), name


# ---- one solver stage against the oracle --------------------------------------------------------------------------------

@pytest.mark.parametrize("gather", [True, False])
@pytest.mark.parametrize("persistent", [True, False])
@pytest.mark.parametrize("mode", ["wavefront", "color", "regions"])
@pytest.mark.parametrize("solver", VARIANTS)
def test_stage_matches_oracle(reference, dev, solver, mode, persistent, gather):
    """One stage of sliders rows with a spring on every prismatic and revolute joint (random hertz, damping ratio and
    warm-start impulse, some with hertz 0), beside limits, motors, a mouse joint and contacts."""
    if not gather and solver not in SUBSTEPPING:
        pytest.skip("the warm-start gather serves the sub-stepping variants only")
    R = reference
    sc = scenes.sliders(R, solver, copies=2)
    for _ in range(30):
        sc.step(DT, 4, 2, True)
    R.step_collide(sc.world)
    bodies = body_rows_from_ref(*R.bodies(sc.world))
    contacts, _ = contact_rows_from_ref(*R.contacts(sc.world))
    joints = _as_prismatic(joint_rows_from_ref(*R.joints(sc.world)), _slots(sc), sc.piles["prismatic_defs"])
    sc.destroy()
    kind = joints["flags"] >> 1 & 0x7
    live = (joints["flags"] & 1) == 1
    sprung = live & ((kind == device.JOINT_PRISMATIC) | (kind == device.JOINT_REVOLUTE))
    n = int(sprung.sum())
    assert n >= 20 and len(contacts) > 10
    rng = np.random.default_rng(11)
    joints["flags"][sprung] |= device.JOINT_ENABLE_SPRING
    joints["hertz"][sprung] = np.where(rng.uniform(size=n) < 0.15, 0.0, rng.uniform(0.5, 6.0, n)).astype(np.float32)
    joints["dampingRatio"][sprung] = rng.uniform(0.0, 1.5, n).astype(np.float32)
    joints["springImpulse"][sprung] = rng.uniform(-0.2, 0.2, n).astype(np.float32)
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
    got_joints = dw.download_joints(len(joints))
    order, _ = dw.solve_order(len(contacts) + len(joints))
    dw.destroy()
    order = None if mode == "wavefront" else order
    ob, _, oj = spring_oracle.load().solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, order=order)
    valid = (bodies["flags"] & 1) == 1
    _compare_bodies(got, ob, valid)
    _compare_joints(got_joints, oj)
    # the springs did work: the prismatic oracle, which has no spring, ends elsewhere
    pb, _, _ = prismatic_oracle.load().solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, order=order)
    assert not bit_equal(pb["position"][valid], ob["position"][valid])
    if solver != "XPBD":
        assert np.any(oj["springImpulse"][sprung] != 0.0)


# ---- a world through the public API, every step ---------------------------------------------------------------------------

def _spring_slots(sc):
    return [(sc.joints[k].index, hertz, zeta) for k, hertz, zeta in sc.piles["springs"]]


def _with_springs(joints, springs, carried):
    """Give the stand-in rows their springs and the spring impulses the last step left."""
    for slot, hertz, zeta in springs:
        joints["flags"][slot] |= device.JOINT_ENABLE_SPRING
        joints["hertz"][slot] = hertz
        joints["dampingRatio"][slot] = zeta
        joints["springImpulse"][slot] = carried.get(slot, 0.0)
    return joints


@pytest.mark.parametrize("solver", VARIANTS)
def test_springs_scene_every_step(reference, product, dev, solver):
    """scenes.springs: reference collide on the stand-in world, the spring oracle in the device's order, reference
    finalize; the device runs the same steps through s2World_Step with real springs. Every step bit for bit: bodies, delta
    positions, contact impulses and joint impulses, the spring impulse included."""
    R, P = reference, product
    O = spring_oracle.load()
    sr = scenes.springs(R, solver)
    sp = scenes.springs(P, solver)
    assert "s2CreatePrismaticJoint" in R.missing and "s2CreatePrismaticJoint" not in P.missing
    slots = _slots(sp)
    springs = _spring_slots(sp)
    assert slots == _slots(sr) and springs == _spring_slots(sr) and len(springs) == 11
    _flush(dev, sp.world)
    dw = device.DeviceWorld.attach(dev, sp.world)
    rows = dw.download_joints(len(sp.joints))
    assert all(rows["flags"][slot] & device.JOINT_ENABLE_SPRING for slot, _, _ in springs)
    ctx = device.make_context(solver, DT, 4, 2, True)
    sticky = solver == "TGS_Sticky"
    solved = {}
    carried = {}
    F = refmod.BODY_F
    contacts_seen = 0
    for step in range(90):
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
        joints = _as_prismatic(joint_rows_from_ref(*R.joints(sr.world)), slots, sr.piles["prismatic_defs"])
        joints = _with_springs(joints, springs, carried)
        got_contacts = dw.download_contacts(len(rows_key) + 64)
        assert len(got_contacts) == len(rows_key) and np.array_equal(got_contacts["shapeA"], rows_key["shapeA"]), step
        contacts_seen += int(np.count_nonzero(rows_key["pointCount"]))

        order, _ = dw.solve_order(len(rows_key) + len(joints) + 16, max_groups=200000)
        ob, oc, oj, odp = O.solve(capi.SOLVER[solver], bodies, rows_key, joints, ctx, order=order,
                                  dp=ref_delta_positions(R, sr.world))
        carried = {slot: float(oj["springImpulse"][slot]) for slot, _, _ in springs}

        store_oracle_bodies(R, sr.world, ob, odp)
        imp = np.zeros((cf.shape[0], 4), dtype=np.float32)
        imp[cslots[perm], 0] = oc["points"]["normalImpulse"][:, 0]
        imp[cslots[perm], 1] = oc["points"]["tangentImpulse"][:, 0]
        imp[cslots[perm], 2] = oc["points"]["normalImpulse"][:, 1]
        imp[cslots[perm], 3] = oc["points"]["tangentImpulse"][:, 1]
        R.load_contact_impulses(sr.world, imp)
        if sticky:
            solved = dict(zip(keys[perm].tolist(), oc.copy()))
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
        for name in JOINT_FIELDS:
            assert bit_equal(gj[name][jv], oj[name][jv]), f"step {step}: joint {name}"
    assert contacts_seen > 500
    if solver != "XPBD":
        assert sum(carried[slot] != 0.0 for slot, _, _ in springs) >= len(springs) - 2
    sp.destroy()
    sr.destroy()


def _box(P, wid, kind, x, y, angle=0.0, vx=0.0, vy=0.0, w=0.0, gravity=1.0):
    bd = capi.default_body_def()
    bd.type = kind
    bd.position = capi.Vec2(x, y)
    bd.angle = angle
    bd.linearVelocity = capi.Vec2(vx, vy)
    bd.angularVelocity = w
    bd.gravityScale = gravity
    bid = P.s2CreateBody(wid, C.byref(bd))
    if kind != capi.STATIC_BODY:
        sd = capi.default_shape_def()
        sd.filter.groupIndex = -1  # no contacts: the every-step comparison hands the oracle none
        P.s2CreatePolygonShape(bid, C.byref(sd), C.byref(P.s2MakeBox(0.3, 0.2)))
    return bid


def _revolute(P, wid, a, b, anchor_a, anchor_b, ref=0.0, spring=None, motor=None, limit=None):
    jd = capi.default_revolute_def()
    jd.bodyIdA, jd.bodyIdB = a, b
    jd.localAnchorA, jd.localAnchorB = capi.Vec2(*anchor_a), capi.Vec2(*anchor_b)
    jd.referenceAngle = ref
    if motor is not None:
        jd.enableMotor, jd.motorSpeed, jd.maxMotorTorque = True, motor[0], motor[1]
    if limit is not None:
        jd.enableLimit, jd.lowerAngle, jd.upperAngle = True, limit[0], limit[1]
    j = P.s2CreateRevoluteJoint(wid, C.byref(jd))
    if spring is not None:
        P.s2RevoluteJoint_EnableSpring(j, True)
        P.s2RevoluteJoint_SetSpringHertz(j, spring[0])
        P.s2RevoluteJoint_SetSpringDampingRatio(j, spring[1])
    return j


def _prismatic(P, wid, a, b, anchor_a, anchor_b, axis, spring=None, limit=None, motor=None):
    jd = capi.default_prismatic_def()
    jd.bodyIdA, jd.bodyIdB = a, b
    jd.localAnchorA, jd.localAnchorB = capi.Vec2(*anchor_a), capi.Vec2(*anchor_b)
    jd.localAxisA = capi.Vec2(*axis)
    if spring is not None:
        jd.enableSpring, jd.hertz, jd.dampingRatio = True, spring[0], spring[1]
    if limit is not None:
        jd.enableLimit, jd.lowerTranslation, jd.upperTranslation = True, limit[0], limit[1]
    if motor is not None:
        jd.enableMotor, jd.motorSpeed, jd.maxMotorForce = True, motor[0], motor[1]
    return P.s2CreatePrismaticJoint(wid, C.byref(jd))


def _spring_world(P, solver):
    """Bodies far apart (no contacts): a hanging revolute spring chain, a vertical prismatic suspension with limit and motor,
    a revolute spring with limit and motor whose rest angle sits at the seam, a prismatic spring to a kinematic carriage and
    a mouse joint."""
    wid = P.create_world(solver)
    ground = _box(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    joints = []
    prev = ground
    for k in range(4):  # soft chain hanging from the ground
        b = _box(P, wid, capi.DYNAMIC_BODY, 0.6 * (k + 1), 10.0, w=0.5 * k)
        joints.append(_revolute(P, wid, prev, b, (0.3, 10.0) if k == 0 else (0.3, 0.0), (-0.3, 0.0), spring=(2.0, 0.3)))
        prev = b
    chassis = _box(P, wid, capi.DYNAMIC_BODY, 20.0, 5.0, vx=0.5)
    wheel = _box(P, wid, capi.DYNAMIC_BODY, 20.0, 4.0, w=2.0)
    joints.append(_prismatic(P, wid, chassis, wheel, (0.0, -1.0), (0.0, 0.0), (0.0, 1.0), spring=(4.0, 0.7),
                             limit=(-0.3, 0.3), motor=(0.2, 3.0)))
    seam = _box(P, wid, capi.DYNAMIC_BODY, 40.0, 5.0, angle=-math.pi + 0.05, gravity=0.0)
    joints.append(_revolute(P, wid, ground, seam, (40.0, 5.0), (0.0, 0.0), ref=math.pi - 0.05, spring=(3.0, 0.2),
                            motor=(0.5, 0.05), limit=(-0.5, 0.5)))
    carriage = _box(P, wid, capi.KINEMATIC_BODY, 60.0, 5.0, vx=0.7, w=0.2)
    rider = _box(P, wid, capi.DYNAMIC_BODY, 61.0, 5.0, gravity=0.0)
    joints.append(_prismatic(P, wid, carriage, rider, (0.0, 0.0), (0.0, 0.0), (1.0, 0.0), spring=(1.5, 0.1)))
    dragged = _box(P, wid, capi.DYNAMIC_BODY, 80.0, 5.0)
    md = capi.MouseJointDef()
    md.bodyIdA, md.bodyIdB = ground, dragged
    md.target = capi.Vec2(80.5, 5.5)
    md.hertz, md.dampingRatio = 4.0, 0.7
    joints.append(P.s2CreateMouseJoint(wid, C.byref(md)))
    return wid, joints, (chassis, wheel)


@pytest.mark.parametrize("solver", VARIANTS)
def test_public_world_every_step(product, dev, solver):
    """Each s2World_Step equals the spring oracle's stage on the rows the step started from, bit for bit, delta positions
    included (a kinematic body's grows under XPBD)."""
    P = product
    wid, _, _ = _spring_world(P, solver)
    P.s2World_Step(wid, DT, 4, 2, True)  # uploads the world
    dw = device.DeviceWorld.attach(dev, wid)
    assert dw.body_cap >= 12 and dw.joint_cap >= 8
    dw.set_schedule(device.SCHEDULE_WAVEFRONT)
    O = spring_oracle.load()
    ctx = device.make_context(solver, DT, 4, 2)
    for _ in range(90):
        bodies = dw.download_all_bodies()
        joints = dw.download_joints()
        dp = dw.download_delta_positions()
        P.s2World_Step(wid, DT, 4, 2, True)
        assert dw.counters().constraintCount == 0
        ob, _, oj, odp = O.solve(capi.SOLVER[solver], bodies, np.zeros(0, dtype=device.CONTACT_ROW), joints, ctx, dp=dp)
        valid = (bodies["flags"] & 1) == 1
        _compare_bodies(dw.download_all_bodies(), ob, valid)
        _compare_joints(dw.download_joints(), oj)
        assert bit_equal(dw.download_delta_positions()[valid], odp[valid])
    P.s2DestroyWorld(wid)


@pytest.mark.parametrize("solver", ["TGS_Soft", "PGS", "TGS_NGS", "XPBD"])
def test_setter_edits_between_replayed_steps(product, dev, solver):
    """Springs switched on, retuned and switched off between steps land in the next step's rows (replayed solve graph),
    and each step still equals the oracle."""
    P = product
    wid, joints, _ = _spring_world(P, solver)
    P.s2World_Step(wid, DT, 4, 2, True)
    dw = device.DeviceWorld.attach(dev, wid)
    assert dw.body_cap >= 12 and dw.joint_cap >= 8
    dw.set_schedule(device.SCHEDULE_WAVEFRONT)
    O = spring_oracle.load()
    ctx = device.make_context(solver, DT, 4, 2)
    rev, pri = joints[0], joints[4]
    edits = {5: lambda: P.s2RevoluteJoint_SetSpringHertz(rev, 5.0),
             10: lambda: P.s2PrismaticJoint_SetSpringDampingRatio(pri, 0.05),
             15: lambda: P.s2RevoluteJoint_EnableSpring(rev, False),
             20: lambda: P.s2PrismaticJoint_EnableSpring(pri, False),
             25: lambda: (P.s2RevoluteJoint_EnableSpring(rev, True), P.s2PrismaticJoint_SetSpringHertz(pri, 0.0),
                          P.s2PrismaticJoint_EnableSpring(pri, True))}
    for k in range(30):
        if k in edits:
            edits[k]()
            _flush(dev, wid)  # push the edits, so the rows read below are the ones the step solves
        bodies = dw.download_all_bodies()
        rows = dw.download_joints()
        dp = dw.download_delta_positions()
        P.s2World_Step(wid, DT, 4, 2, True)
        ob, _, oj, _ = O.solve(capi.SOLVER[solver], bodies, np.zeros(0, dtype=device.CONTACT_ROW), rows, ctx, dp=dp)
        _compare_bodies(dw.download_all_bodies(), ob, (bodies["flags"] & 1) == 1)
        _compare_joints(dw.download_joints(), oj)
    r = dw.download_joints()
    assert r["flags"][rev.index] & device.JOINT_ENABLE_SPRING and r["hertz"][rev.index] == np.float32(5.0)
    assert r["flags"][pri.index] & device.JOINT_ENABLE_SPRING and r["hertz"][pri.index] == 0.0
    assert r["dampingRatio"][pri.index] == np.float32(0.05) and r["springImpulse"][pri.index] == 0.0
    P.s2DestroyWorld(wid)


def test_slot_reuse_across_types(product, dev):
    """A slot freed by a sprung joint and taken by a weld, a mouse or a plain revolute joint carries no spring."""
    P = product
    wid, joints, (a, b) = _spring_world(P, "TGS_Soft")
    for _ in range(5):
        P.s2World_Step(wid, DT, 4, 2, True)
    dw = device.DeviceWorld.attach(dev, wid)
    slot = joints[4].index
    P.s2DestroyJoint(joints[4])
    j = _revolute(P, wid, a, b, (0.0, -1.0), (0.0, 0.0))
    assert j.index == slot
    P.s2World_Step(wid, DT, 4, 2, True)
    r = dw.download_joints()[slot]
    assert (r["flags"] & device.JOINT_ENABLE_SPRING) == 0 and r["hertz"] == 0.0 and r["springImpulse"] == 0.0
    P.s2DestroyJoint(j)
    wd = capi.WeldJointDef()
    wd.bodyIdA, wd.bodyIdB = a, b
    j = P.s2CreateWeldJoint(wid, C.byref(wd))
    P.s2RevoluteJoint_EnableSpring(j, True)  # not a revolute joint: ignored
    P.s2World_Step(wid, DT, 4, 2, True)
    r = dw.download_joints()[j.index]
    assert (r["flags"] & device.JOINT_ENABLE_SPRING) == 0 and r["springImpulse"] == 0.0
    P.s2DestroyWorld(wid)


def test_create_and_setters_reject_bad_input(product, dev):
    P = product
    wid = P.create_world("TGS_Soft")
    a = _box(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    b = _box(P, wid, capi.DYNAMIC_BODY, 0.0, 2.0)
    for hz, zeta in ((-1.0, 0.5), (math.nan, 0.5), (math.inf, 0.5), (1.0, -0.1), (1.0, math.nan), (1.0, math.inf)):
        j = _prismatic(P, wid, a, b, (0.0, 0.0), (0.0, 0.0), (0.0, 1.0), spring=(hz, zeta))
        assert (j.index, j.world, j.revision) == (-1, -1, 0), (hz, zeta)
    assert P.s2World_GetStatistics(wid).jointCount == 0
    pj = _prismatic(P, wid, a, b, (0.0, 0.0), (0.0, 0.0), (0.0, 1.0), spring=(2.0, 0.5))
    rj = _revolute(P, wid, a, b, (0.0, 2.0), (0.0, 0.0), spring=(3.0, 0.25))
    for bad in (-1.0, math.nan, math.inf, -math.inf):
        P.s2PrismaticJoint_SetSpringHertz(pj, bad)
        P.s2PrismaticJoint_SetSpringDampingRatio(pj, bad)
        P.s2RevoluteJoint_SetSpringHertz(rj, bad)
        P.s2RevoluteJoint_SetSpringDampingRatio(rj, bad)
    P.s2World_Step(wid, DT, 4, 2, True)
    rows = device.DeviceWorld.attach(dev, wid).download_joints()
    assert (rows["hertz"][pj.index], rows["dampingRatio"][pj.index]) == (np.float32(2.0), np.float32(0.5))
    assert (rows["hertz"][rj.index], rows["dampingRatio"][rj.index]) == (np.float32(3.0), np.float32(0.25))
    P.s2DestroyWorld(wid)


# ---- reactions and break thresholds ---------------------------------------------------------------------------------------

def _rate(solver):
    ctx = device.make_context(solver, DT, 4, 2, True)
    return np.float32(ctx.inv_dt if solver == "TGS_Sticky" else ctx.inv_h)


@pytest.mark.parametrize("solver", ["TGS_Soft", "PGS", "TGS_NGS", "TGS_Sticky", "PGS_NGS_Block"])
def test_reactions_include_the_spring(product, dev, solver):
    """The getters and the bulk read equal s2ComputeJointReaction on the downloaded rows with motorImpulse + springImpulse
    as the motor argument on sprung rows, and differ from the reading without the spring impulse."""
    P = product
    wid, joints, _ = _spring_world(P, solver)
    for _ in range(20):
        P.s2World_Step(wid, DT, 4, 2, True)
    dw = device.DeviceWorld.attach(dev, wid)
    rows = dw.download_joints()
    bodies = dw.download_all_bodies()
    bulk = np.zeros((len(rows), 3), dtype=np.float32)
    dw.L.s2b_download_joint_reactions(dw.h, bulk.ctypes.data, len(rows))
    checked = 0
    for j in joints:
        r = rows[j.index]
        sprung = (int(r["flags"]) & device.JOINT_ENABLE_SPRING) != 0
        motor = np.float32(r["motorImpulse"]) + np.float32(r["springImpulse"]) if sprung else np.float32(r["motorImpulse"])
        q = bodies["rot"][int(r["bodyA"])]
        x = P.s2ComputeJointReaction((int(r["flags"]) >> 1) & 7, capi.Vec2(*r["impulse"]), float(motor),
                                     float(r["lowerImpulse"]), float(r["upperImpulse"]), capi.Rot(float(q[0]), float(q[1])),
                                     capi.Vec2(*r["localAxisA"]), float(_rate(solver)))
        f, t = P.s2Joint_GetReactionForce(j), P.s2Joint_GetReactionTorque(j)
        assert (np.float32(f.x), np.float32(f.y), np.float32(t)) == (np.float32(x.force.x), np.float32(x.force.y),
                                                                     np.float32(x.torque))
        assert bit_equal(bulk[j.index], np.array([x.force.x, x.force.y, x.torque], dtype=np.float32))
        if sprung and r["springImpulse"] != 0.0:
            checked += 1
    assert checked >= 5
    # switching the springs off between steps does not change what the getters report for the step already taken: they
    # pair the synced impulses with the row that produced them, as the device's reaction pass did
    before = [(tuple(P.s2Joint_GetReactionForce(j)), P.s2Joint_GetReactionTorque(j)) for j in joints[:5]]
    P.s2RevoluteJoint_EnableSpring(joints[0], False)
    P.s2PrismaticJoint_EnableSpring(joints[4], False)
    after = [(tuple(P.s2Joint_GetReactionForce(j)), P.s2Joint_GetReactionTorque(j)) for j in joints[:5]]
    assert after == before
    P.s2DestroyWorld(wid)


def test_spring_load_trips_a_break_threshold(product, dev):
    """A stiff revolute spring twisted far from its rest angle: its torque alone passes the threshold, and the joint is
    destroyed by the next step; the same joint without the spring stays."""
    P = product
    kept = []
    for sprung in (True, False):
        wid = P.create_world("TGS_Soft")
        a = _box(P, wid, capi.STATIC_BODY, 0.0, 0.0)
        b = _box(P, wid, capi.DYNAMIC_BODY, 0.0, 0.0, angle=1.0, gravity=0.0)
        j = _revolute(P, wid, a, b, (0.0, 0.0), (0.0, 0.0), spring=(8.0, 0.5) if sprung else None)
        P.s2Joint_SetBreakTorque(j, 0.5)
        P.s2World_Step(wid, DT, 4, 2, True)
        torque = P.s2Joint_GetReactionTorque(j)
        P.s2World_Step(wid, DT, 4, 2, True)
        kept.append(P.s2World_GetStatistics(wid).jointCount)
        if sprung:
            assert abs(torque) > 0.5
        P.s2DestroyWorld(wid)
    assert kept == [0, 1]
