"""GPU: the distance joint (DESIGN.md §3.16). The device against the joint oracle (tests/joint_oracle.c) bit for bit:
every step of scenes.distance_joints (ropes, pendulums, a spring ring over a pile, winches, a kinematic tether, contacts
throughout) through the public API against reference collide and finalize around the oracle, in the wavefront and the
colour schedule; every step of a contact-free world for all ten variants, in both schedules, persistent and launch by
launch, with the warm-start gather on and off; setter edits between replayed steps; slot reuse
across joint types. Also: collideConnected, input checks, GetCurrentLength, the drawn segments, reactions against the
host getters, and a break threshold that breaks a rope.

Mutations each test catches: a row placed in another order, a row that acts where it should not (the rigid row of a rope,
a limit with minLength == maxLength), a warm start or gather that leaves an impulse out of the axial sum, an impulse kept
across a prepare it should not survive, and a frame formed from other poses all fail the every-step comparisons; a
reaction formed from another axis fails the reaction test."""
import ctypes as C
import math

import numpy as np
import pytest

import joint_oracle
from helpers import (bit_equal, body_rows_from_ref, carry_sticky_friction, contact_rows_from_ref, joint_rows_from_ref,
                     load_bodies_into_ref, ref_delta_positions, store_oracle_bodies)
from oracle import ref as refmod
from solver2d_b200 import capi, device, scenes
from test_api_lifecycle_gpu import _draw_log

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0
VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]
SUBSTEPPING = {"SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"}
JOINT_FIELDS = ("impulse", "motorImpulse", "lowerImpulse", "upperImpulse", "springImpulse")


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


def _box(P, wid, kind, x, y, angle=0.0, vx=0.0, vy=0.0, w=0.0, gravity=1.0, group=-1):
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
        sd.filter.groupIndex = group  # -1: no contacts, the every-step comparison hands the oracle none
        P.s2CreatePolygonShape(bid, C.byref(sd), C.byref(P.s2MakeBox(0.3, 0.2)))
    return bid


def _distance(P, wid, a, b, anchor_a, anchor_b, length, spring=None, limit=None, motor=None, collide=False):
    jd = capi.default_distance_def()
    jd.bodyIdA, jd.bodyIdB = a, b
    jd.localAnchorA, jd.localAnchorB = capi.Vec2(*anchor_a), capi.Vec2(*anchor_b)
    jd.length = length
    if spring is not None:
        jd.enableSpring, jd.hertz, jd.dampingRatio = True, spring[0], spring[1]
    if limit is not None:
        jd.enableLimit, jd.minLength, jd.maxLength = True, limit[0], limit[1]
    if motor is not None:
        jd.enableMotor, jd.motorSpeed, jd.maxMotorForce = True, motor[0], motor[1]
    jd.collideConnected = collide
    return P.s2CreateDistanceJoint(wid, C.byref(jd))


def _distance_world(P, solver):
    """Bodies far apart (no contacts): a rod pendulum, a spring, a rope hanging taut, a pushed-out pair on a minLength, a
    winch lifting a load and one set below it, equal limits with the spring on, a tether to a kinematic platform, a
    coincident pair, a revolute link and a mouse joint."""
    wid = P.create_world(solver)
    ground = _box(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    joints = []
    rod = _box(P, wid, capi.DYNAMIC_BODY, 0.8, 9.0, w=0.5)
    joints.append(_distance(P, wid, ground, rod, (0.0, 10.0), (0.1, 0.1), 1.2))
    spring = _box(P, wid, capi.DYNAMIC_BODY, 10.0, 8.5, vx=0.4)
    joints.append(_distance(P, wid, ground, spring, (10.0, 10.0), (0.0, 0.15), 1.0, spring=(2.0, 0.2)))
    rope = _box(P, wid, capi.DYNAMIC_BODY, 20.5, 9.5)
    joints.append(_distance(P, wid, ground, rope, (20.0, 10.0), (0.2, 0.0), 1.0, spring=(0.0, 0.0), limit=(0.0, 1.5)))
    left = _box(P, wid, capi.DYNAMIC_BODY, 30.0, 5.0, gravity=0.0)
    right = _box(P, wid, capi.DYNAMIC_BODY, 30.4, 5.1, w=1.0, gravity=0.0)
    joints.append(_distance(P, wid, left, right, (0.1, 0.0), (-0.1, 0.0), 1.0, spring=(1.0, 0.5), limit=(1.0, 2.0)))
    lift = _box(P, wid, capi.DYNAMIC_BODY, 40.0, 7.0)
    joints.append(_distance(P, wid, ground, lift, (40.0, 10.0), (0.0, 0.0), 3.0, spring=(0.0, 0.0), motor=(-0.5, 60.0)))
    stall = _box(P, wid, capi.DYNAMIC_BODY, 45.0, 7.0)
    joints.append(_distance(P, wid, ground, stall, (45.0, 10.0), (0.0, 0.0), 3.0, spring=(0.0, 0.0), motor=(-0.5, 3.0),
                            limit=(0.5, 4.0)))
    equal = _box(P, wid, capi.DYNAMIC_BODY, 50.5, 9.2)
    joints.append(_distance(P, wid, ground, equal, (50.0, 10.0), (0.0, 0.0), 1.0, spring=(3.0, 0.3), limit=(1.0, 1.0)))
    platform = _box(P, wid, capi.KINEMATIC_BODY, 60.0, 10.0, vx=0.7, w=0.2)
    tethered = _box(P, wid, capi.DYNAMIC_BODY, 60.0, 8.8)
    joints.append(_distance(P, wid, platform, tethered, (0.2, 0.0), (0.0, 0.1), 1.2, spring=(4.0, 0.7), limit=(0.8, 1.5),
                            motor=(0.2, 5.0)))
    same = _box(P, wid, capi.DYNAMIC_BODY, 70.0, 5.0, gravity=0.0)
    joints.append(_distance(P, wid, ground, same, (70.0, 5.0), (0.0, 0.0), 1.0, limit=(0.5, 2.0), motor=(1.0, 10.0)))
    link = _box(P, wid, capi.DYNAMIC_BODY, 80.6, 10.0)
    rd = capi.default_revolute_def()
    rd.bodyIdA, rd.bodyIdB = ground, link
    rd.localAnchorA, rd.localAnchorB = capi.Vec2(80.3, 10.0), capi.Vec2(-0.3, 0.0)
    joints.append(P.s2CreateRevoluteJoint(wid, C.byref(rd)))
    dragged = _box(P, wid, capi.DYNAMIC_BODY, 90.0, 5.0)
    md = capi.MouseJointDef()
    md.bodyIdA, md.bodyIdB = ground, dragged
    md.target = capi.Vec2(90.5, 5.5)
    md.hertz, md.dampingRatio = 4.0, 0.7
    joints.append(P.s2CreateMouseJoint(wid, C.byref(md)))
    return wid, joints, (ground, rod)


def _step_and_compare(P, wid, dw, O, solver, steps, colour=False, edit=None, dt=DT, substeps=4, relax=2):
    ctx = device.make_context(solver, dt, substeps, relax)
    moved = False
    for k in range(steps):
        if edit is not None:
            edit(k)
        P.s2World_Flush(wid)  # the rows the step starts from carry every edit and every created or destroyed joint
        bodies = dw.download_all_bodies()
        joints = dw.download_joints()
        dp = dw.download_delta_positions()
        P.s2World_Step(wid, dt, substeps, relax, True)
        assert dw.counters().constraintCount == 0
        order = None
        if colour:
            order, _ = dw.solve_order(len(joints))
        ob, _, oj, odp = O.solve(capi.SOLVER[solver], bodies, np.zeros(0, dtype=device.CONTACT_ROW), joints, ctx, dp=dp,
                                 order=order)
        valid = (bodies["flags"] & 1) == 1
        got = dw.download_all_bodies()
        for name in ("position", "rot", "linearVelocity", "angularVelocity"):
            assert bit_equal(got[name][valid], ob[name][valid]), (k, name)
        gj = dw.download_joints()
        jv = (oj["flags"] & 1) == 1
        for name in JOINT_FIELDS:
            assert bit_equal(gj[name][jv], oj[name][jv]), (k, name)
        assert bit_equal(dw.download_delta_positions()[valid], odp[valid])
        moved = moved or not bit_equal(got["position"][valid], bodies["position"][valid])
    assert moved


# ---- scenes.distance_joints through the public API against reference collide and finalize ---------------------------------

def _distance_slots(sc):
    return [sc.joints[k].index for k in sc.piles["distance"]]


def _as_distance(joints, slots, defs, carried):
    """Turn the stand-in revolute rows at `slots` into the distance rows `defs` describe, with the spring impulses the last
    step left."""
    for slot, d in zip(slots, defs):
        r = joints[slot]
        assert r["flags"] & (device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR) == 0
        flags = (int(r["flags"]) & ~0xE) | (device.JOINT_DISTANCE << 1)
        flags |= device.JOINT_ENABLE_SPRING if d["enableSpring"] else 0
        flags |= device.JOINT_ENABLE_LIMIT if d["enableLimit"] else 0
        flags |= device.JOINT_ENABLE_MOTOR if d["enableMotor"] else 0
        joints["flags"][slot] = flags
        joints["localOriginAnchorA"][slot] = d["localAnchorA"]
        joints["localOriginAnchorB"][slot] = d["localAnchorB"]
        joints["referenceAngle"][slot] = d["length"]
        joints["lowerAngle"][slot] = d["minLength"]
        joints["upperAngle"][slot] = d["maxLength"]
        joints["maxMotorTorque"][slot] = d["maxMotorForce"]
        joints["motorSpeed"][slot] = d["motorSpeed"]
        joints["hertz"][slot] = d["hertz"]
        joints["dampingRatio"][slot] = d["dampingRatio"]
        joints["springImpulse"][slot] = carried.get(slot, 0.0)
    return joints


@pytest.mark.parametrize("mode", ["wavefront", "color"])
@pytest.mark.parametrize("solver", VARIANTS)
def test_distance_scene_every_step(reference, product, dev, solver, mode):
    """scenes.distance_joints: reference collide on the stand-in world, the distance oracle in the device's order, reference
    finalize; the device runs the same steps through s2World_Step with real distance joints. Every step bit for bit: bodies,
    delta positions, contact impulses and joint impulses, the spring impulse included."""
    R, P = reference, product
    O = joint_oracle.load()
    sr = scenes.distance_joints(R, solver)
    sp = scenes.distance_joints(P, solver)
    assert "s2CreateDistanceJoint" in R.missing and "s2CreateDistanceJoint" not in P.missing
    slots = _distance_slots(sp)
    defs = sp.piles["distance_defs"]
    assert slots == _distance_slots(sr) and defs == sr.piles["distance_defs"] and len(slots) == 29
    P.s2World_Flush(sp.world)
    dw = device.DeviceWorld.attach(dev, sp.world)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT if mode == "wavefront" else device.SCHEDULE_COLOR)
    rows = dw.download_joints(len(sp.joints))
    assert all((rows["flags"][slot] >> 1) & 0x7 == device.JOINT_DISTANCE for slot in slots)
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
        joints = _as_distance(joint_rows_from_ref(*R.joints(sr.world)), slots, defs, carried)
        got_contacts = dw.download_contacts(len(rows_key) + 64)
        assert len(got_contacts) == len(rows_key) and np.array_equal(got_contacts["shapeA"], rows_key["shapeA"]), step
        contacts_seen += int(np.count_nonzero(rows_key["pointCount"]))

        order, _ = dw.solve_order(len(rows_key) + len(joints) + 16, max_groups=200000)
        ob, oc, oj, odp = O.solve(capi.SOLVER[solver], bodies, rows_key, joints, ctx, order=order,
                                  dp=ref_delta_positions(R, sr.world))
        carried = {slot: float(oj["springImpulse"][slot]) for slot in slots}

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
    assert contacts_seen > 400  # manifolds with points over the 90 steps: fewest under Jacobi (454, 476)
    if solver != "XPBD":
        assert sum(oj["impulse"][slot][0] != 0.0 for slot in slots) >= 4
        assert sum(carried[slot] != 0.0 for slot in slots) >= 8
    sp.destroy()
    sr.destroy()


# ---- a contact-free world through the public API, every step ---------------------------------------------------------------

@pytest.mark.parametrize("gather", [True, False])
@pytest.mark.parametrize("persistent", [True, False])
@pytest.mark.parametrize("mode", ["wavefront", "color"])
@pytest.mark.parametrize("solver", VARIANTS)
def test_public_world_every_step(product, dev, solver, mode, persistent, gather):
    """Each s2World_Step equals the distance oracle's stage on the rows the step started from, bit for bit, delta positions
    included (a kinematic body's grows under XPBD)."""
    if not gather and solver not in SUBSTEPPING:
        pytest.skip("the warm-start gather serves the sub-stepping variants only")
    P = product
    wid, _, _ = _distance_world(P, solver)
    P.s2World_Step(wid, DT, 4, 2, True)  # uploads the world
    dw = device.DeviceWorld.attach(dev, wid)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT if mode == "wavefront" else device.SCHEDULE_COLOR)
    dw.set_persistent(persistent)
    dw.set_warm_gather(gather)
    _step_and_compare(P, wid, dw, joint_oracle.load(), solver, 60, colour=mode == "color")
    P.s2DestroyWorld(wid)


@pytest.mark.parametrize("solver", ["TGS_Soft", "PGS", "TGS_NGS", "XPBD"])
def test_setter_edits_between_replayed_steps(product, dev, solver):
    """Lengths, ranges, springs and motors edited between steps land in the next step's rows (replayed solve graph), and
    each step still equals the oracle."""
    P = product
    wid, joints, _ = _distance_world(P, solver)
    P.s2World_Step(wid, DT, 4, 2, True)
    dw = device.DeviceWorld.attach(dev, wid)

    def edit(k):
        if k == 10:
            P.s2DistanceJoint_SetLength(joints[0], 1.5)
            P.s2DistanceJoint_EnableSpring(joints[1], False)
            P.s2DistanceJoint_SetLengthRange(joints[2], 0.5, 1.2)
        elif k == 20:
            P.s2DistanceJoint_SetSpringHertz(joints[3], 5.0)
            P.s2DistanceJoint_SetSpringDampingRatio(joints[3], 0.9)
            P.s2DistanceJoint_SetMotorSpeed(joints[4], 0.5)
            P.s2DistanceJoint_SetMaxMotorForce(joints[5], 100.0)
        elif k == 30:
            P.s2DistanceJoint_EnableLimit(joints[7], False)
            P.s2DistanceJoint_EnableMotor(joints[7], False)
            P.s2DistanceJoint_EnableSpring(joints[1], True)

    replays = dw.counters().graphReplays
    _step_and_compare(P, wid, dw, joint_oracle.load(), solver, 45, colour=True, edit=edit)
    assert dw.counters().graphReplays > replays
    assert P.s2DistanceJoint_GetLength(joints[0]) == np.float32(1.5)
    assert (P.s2DistanceJoint_GetMinLength(joints[2]), P.s2DistanceJoint_GetMaxLength(joints[2])) == (0.5, np.float32(1.2))
    P.s2DestroyWorld(wid)


def test_slot_reuse_across_types(product, dev):
    """A distance joint destroyed and a revolute joint created in its slot, and the other way round: every step equals the
    oracle, so no impulse or marker of the slot's last type survives."""
    P = product
    solver = "TGS_Soft"
    wid, joints, (ground, rod) = _distance_world(P, solver)
    P.s2World_Step(wid, DT, 4, 2, True)
    dw = device.DeviceWorld.attach(dev, wid)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT)
    O = joint_oracle.load()
    _step_and_compare(P, wid, dw, O, solver, 10)
    P.s2DestroyJoint(joints[0])  # the rod
    rd = capi.default_revolute_def()
    rd.bodyIdA, rd.bodyIdB = ground, rod
    rd.localAnchorA, rd.localAnchorB = capi.Vec2(0.0, 10.0), capi.Vec2(0.1, 0.1)
    rev = P.s2CreateRevoluteJoint(wid, C.byref(rd))
    assert rev.index == joints[0].index
    _step_and_compare(P, wid, dw, O, solver, 10)
    P.s2DestroyJoint(rev)
    again = _distance(P, wid, rd.bodyIdA, rd.bodyIdB, (0.0, 10.0), (0.1, 0.1), 0.9, spring=(1.0, 0.1), limit=(0.5, 1.0))
    assert again.index == joints[0].index
    _step_and_compare(P, wid, dw, O, solver, 10)
    P.s2DestroyWorld(wid)


def test_collide_connected(product, dev):
    """Two boxes resting in contact on the ground: a distance joint with collideConnected == false removes their contact,
    one with true keeps it."""
    P = product
    kept = []
    for collide in (False, True):
        wid = P.create_world("TGS_Soft")
        ground = P.s2CreateBody(wid, C.byref(capi.default_body_def()))
        sd = capi.default_shape_def()
        P.s2CreatePolygonShape(ground, C.byref(sd), C.byref(P.s2MakeOffsetBox(20.0, 0.5, capi.Vec2(0.0, -0.5), 0.0)))
        a = _box(P, wid, capi.DYNAMIC_BODY, 0.0, 0.2, group=0)
        b = _box(P, wid, capi.DYNAMIC_BODY, 0.59, 0.2, group=0)
        for _ in range(10):
            P.s2World_Step(wid, DT, 4, 2, True)
        dw = device.DeviceWorld.attach(dev, wid)
        before = dw.counters().constraintCount
        _distance(P, wid, a, b, (0.0, 0.0), (0.0, 0.0), 0.6, collide=collide)
        for _ in range(3):
            P.s2World_Step(wid, DT, 4, 2, True)
        kept.append(dw.counters().constraintCount - before)
        P.s2DestroyWorld(wid)
    assert kept[0] == -1 and kept[1] == 0, kept


def test_create_and_setters_reject_bad_input(product, dev):
    P = product
    wid = P.create_world("TGS_Soft")
    ground = _box(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    body = _box(P, wid, capi.DYNAMIC_BODY, 0.0, -1.0)
    bad = [dict(length=float("nan")), dict(length=-1.0), dict(minLength=-0.1), dict(hertz=-1.0), dict(dampingRatio=float("inf")),
           dict(maxMotorForce=-2.0), dict(minLength=2.0, maxLength=1.0), dict(motorSpeed=float("nan")),
           dict(localAnchorA=capi.Vec2(float("nan"), 0.0))]
    for fields in bad:
        jd = capi.default_distance_def()
        jd.bodyIdA, jd.bodyIdB = ground, body
        for k, v in fields.items():
            setattr(jd, k, v)
        j = P.s2CreateDistanceJoint(wid, C.byref(jd))
        assert j.index == -1, fields  # s2_nullJointId
    jd = capi.default_distance_def()
    jd.bodyIdA, jd.bodyIdB = ground, body
    jd.length, jd.minLength, jd.maxLength = 0.0, 0.0, 1e9
    j = P.s2CreateDistanceJoint(wid, C.byref(jd))
    # clamped into [s2_linearSlop, s2_huge]
    assert (P.s2DistanceJoint_GetLength(j), P.s2DistanceJoint_GetMinLength(j), P.s2DistanceJoint_GetMaxLength(j)) == \
        (np.float32(0.005), np.float32(0.005), 100000.0)
    P.s2DistanceJoint_SetLength(j, -1.0)
    P.s2DistanceJoint_SetLength(j, float("nan"))
    P.s2DistanceJoint_SetLengthRange(j, 2.0, 1.0)
    P.s2DistanceJoint_SetSpringHertz(j, -1.0)
    P.s2DistanceJoint_SetMaxMotorForce(j, float("nan"))
    assert P.s2DistanceJoint_GetLength(j) == np.float32(0.005)
    assert P.s2DistanceJoint_GetMaxLength(j) == 100000.0
    # a joint of another type is ignored and reads 0
    rd = capi.default_revolute_def()
    rd.bodyIdA, rd.bodyIdB = ground, body
    rev = P.s2CreateRevoluteJoint(wid, C.byref(rd))
    P.s2DistanceJoint_SetLength(rev, 3.0)
    P.s2DistanceJoint_SetLengthRange(rev, 1.0, 2.0)
    assert P.s2DistanceJoint_GetLength(rev) == 0.0 and P.s2DistanceJoint_GetCurrentLength(rev) == 0.0
    P.s2World_Step(wid, DT, 4, 2, True)
    rows = device.DeviceWorld.attach(dev, wid).download_joints()
    assert rows["lowerAngle"][rev.index] == 0.0 and rows["referenceAngle"][rev.index] == 0.0
    P.s2DestroyWorld(wid)


def test_current_length_and_draw(product, dev):
    """GetCurrentLength is the distance between the anchors' world points; s2World_Draw draws the anchor segment and, with
    the limit on, a mark at minLength and at maxLength."""
    P = product
    wid = P.create_world("TGS_Soft")
    ground = _box(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    body = _box(P, wid, capi.DYNAMIC_BODY, 0.3, -1.0, angle=0.4)
    j = _distance(P, wid, ground, body, (0.0, 0.0), (0.1, 0.05), 1.0, limit=(0.5, 1.5))
    for _ in range(20):
        P.s2World_Step(wid, DT, 4, 2, True)
    pos, angle = P.s2Body_GetPosition(body), P.s2Body_GetAngle(body)
    c, s_ = math.cos(angle), math.sin(angle)
    pB = (pos.x + c * 0.1 - s_ * 0.05, pos.y + s_ * 0.1 + c * 0.05)
    length = P.s2DistanceJoint_GetCurrentLength(j)
    assert abs(length - math.hypot(*pB)) <= 1e-5
    assert abs(length - 1.0) <= 0.01
    segments = [v for name, v in _draw_log(P, wid) if name == "DrawSegment"]
    assert any(abs(v[0]) < 1e-6 and abs(v[1]) < 1e-6 and abs(v[2] - pB[0]) < 1e-5 and abs(v[3] - pB[1]) < 1e-5 for v in segments)
    # the marks cross the line at 0.5 m and 1.5 m from anchor A
    ux, uy = pB[0] / length, pB[1] / length
    for at in (0.5, 1.5):
        assert any(abs(0.5 * (v[0] + v[2]) - at * ux) < 1e-4 and abs(0.5 * (v[1] + v[3]) - at * uy) < 1e-4 for v in segments), at
    P.s2DestroyWorld(wid)


def test_reactions_and_a_rope_that_breaks(product, dev):
    """A box hanging at rest on a rod reads (0, m g) through the host getter and the device's bulk read alike, bit for bit;
    a rope given a break force below its load breaks."""
    P = product
    wid = P.create_world("TGS_Soft")
    ground = _box(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    body = _box(P, wid, capi.DYNAMIC_BODY, 0.0, -1.0)
    j = _distance(P, wid, ground, body, (0.0, 0.0), (0.0, 0.0), 1.0)
    rope_body = _box(P, wid, capi.DYNAMIC_BODY, 5.0, -1.0)
    rope = _distance(P, wid, ground, rope_body, (5.0, 0.0), (0.0, 0.0), 1.0, spring=(0.0, 0.0), limit=(0.0, 1.0))
    for _ in range(60):
        P.s2World_Step(wid, DT, 4, 2, True)
    f = P.s2Joint_GetReactionForce(j)
    mass = P.s2Body_GetMass(body)
    assert abs(f.x) <= 1e-4 and abs(f.y - mass * 10.0) <= 1e-3 * mass * 10.0, (f.x, f.y, mass)
    assert P.s2Joint_GetReactionTorque(j) == 0.0
    out = np.zeros(3 * 8, dtype=np.float32)
    P.s2World_GetJointReactions(wid, out.ctypes.data, 8)
    assert out[3 * j.index] == np.float32(f.x) and out[3 * j.index + 1] == np.float32(f.y)
    load = P.s2Joint_GetReactionForce(rope)
    assert load.y > 0.5 * mass * 10.0
    P.s2Joint_SetBreakForce(rope, 0.5 * load.y)
    P.s2World_Step(wid, DT, 4, 2, True)
    broken = (capi.JointId * 4)()
    assert P.s2World_GetBrokenJoints(wid, broken, 4) == 1 and broken[0].index == rope.index
    P.s2World_Step(wid, DT, 4, 2, True)
    P.s2DestroyWorld(wid)
