"""GPU: the wheel joint (DESIGN.md §3.17). The device against the wheel oracle (tests/wheel_oracle.c) bit for bit: every
step of scenes.wheels (a motorised car over bumps, a car down a slope, a barrow on a rigid axle, a trolley on a kinematic
rail, contacts throughout) through the public API against reference collide and finalize around the oracle, in the
wavefront and the colour schedule; every step of a contact-free world for all ten variants, in both schedules, persistent
and launch by launch, with the warm-start gather on and off; setter edits between replayed steps; slot reuse across the
wheel, prismatic and distance joints. Also: collideConnected, input checks, GetTranslation, the drawn lines, reactions
against the host getters and GetMotorTorque, and a break threshold that snaps a wheel off.

Mutations each test catches: a row placed in another order, a motor on the axis instead of the rotation, a motor impulse
kept where the motor is off or both rotations are fixed, a warm start or gather that leaves the perpendicular or motor
impulse out, and a frame formed from other poses all fail the every-step comparisons; a reaction that drops the spring's
impulse fails the reaction test."""
import ctypes as C

import numpy as np
import pytest

import wheel_oracle
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


def _body(P, wid, kind, x, y, angle=0.0, vx=0.0, vy=0.0, w=0.0, gravity=1.0, group=-1, radius=None):
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
        if radius is not None:
            P.s2CreateCircleShape(bid, C.byref(sd), C.byref(capi.Circle(capi.Vec2(0.0, 0.0), radius)))
        else:
            P.s2CreatePolygonShape(bid, C.byref(sd), C.byref(P.s2MakeBox(0.3, 0.2)))
    return bid


def _wheel(P, wid, a, b, anchor_a, anchor_b, axis=(0.0, 1.0), spring=None, limit=None, motor=None, collide=False):
    jd = capi.default_wheel_def()
    jd.bodyIdA, jd.bodyIdB = a, b
    jd.localAnchorA, jd.localAnchorB = capi.Vec2(*anchor_a), capi.Vec2(*anchor_b)
    jd.localAxisA = capi.Vec2(*axis)
    jd.enableSpring = spring is not None
    if spring is not None:
        jd.hertz, jd.dampingRatio = spring
    if limit is not None:
        jd.enableLimit, jd.lowerTranslation, jd.upperTranslation = True, limit[0], limit[1]
    if motor is not None:
        jd.enableMotor, jd.motorSpeed, jd.maxMotorTorque = True, motor[0], motor[1]
    jd.collideConnected = collide
    return P.s2CreateWheelJoint(wid, C.byref(jd))


def _wheel_world(P, solver):
    """Bodies far apart (no contacts): a sprung, limited wheel spinning on the ground, a motor lifting an off-centre load on
    a rigid axle and one too weak for it, a free pair on a slanted axis with every row, a trolley on a kinematic rail, a
    motor on a kinematic wheel (both rotations fixed), a spring flag at hertz 0, a revolute link and a mouse joint."""
    wid = P.create_world(solver)
    ground = _body(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    joints = []
    spin = _body(P, wid, capi.DYNAMIC_BODY, 0.0, 9.8, w=6.0, radius=0.3)
    joints.append(_wheel(P, wid, ground, spin, (0.0, 10.0), (0.0, 0.0), spring=(4.0, 0.7), limit=(-0.3, 0.3)))
    for x, torque in ((10.0, 40.0), (15.0, 2.0)):
        load = _body(P, wid, capi.DYNAMIC_BODY, x + 0.5, 10.0)
        joints.append(_wheel(P, wid, ground, load, (x, 10.0), (-0.5, 0.0), limit=(0.0, 0.0), motor=(3.0, torque)))
    left = _body(P, wid, capi.DYNAMIC_BODY, 20.0, 5.0, vx=0.2, w=1.0, gravity=0.0)
    right = _body(P, wid, capi.DYNAMIC_BODY, 20.4, 5.6, w=-2.0, gravity=0.0)
    joints.append(_wheel(P, wid, left, right, (0.1, 0.1), (-0.1, 0.05), axis=(1.0, 2.0), spring=(2.0, 0.2), limit=(-0.2, 0.6),
                         motor=(2.0, 1.0)))
    rail = _body(P, wid, capi.KINEMATIC_BODY, 30.0, 10.0, vx=0.7, w=0.2)
    trolley = _body(P, wid, capi.DYNAMIC_BODY, 30.3, 9.5)
    joints.append(_wheel(P, wid, rail, trolley, (0.3, 0.0), (0.0, 0.5), axis=(1.0, 0.0), spring=(1.0, 0.3), limit=(-1.0, 1.0),
                         motor=(1.0, 5.0)))
    turning = _body(P, wid, capi.KINEMATIC_BODY, 40.0, 5.0, w=1.5)
    joints.append(_wheel(P, wid, ground, turning, (40.0, 5.0), (0.0, 0.0), spring=(3.0, 0.5), motor=(2.0, 10.0)))
    slack = _body(P, wid, capi.DYNAMIC_BODY, 50.0, 9.5, w=0.5)
    joints.append(_wheel(P, wid, ground, slack, (50.0, 10.0), (0.0, 0.5), spring=(0.0, 0.0), limit=(-0.5, 0.5)))
    link = _body(P, wid, capi.DYNAMIC_BODY, 60.6, 10.0)
    rd = capi.default_revolute_def()
    rd.bodyIdA, rd.bodyIdB = ground, link
    rd.localAnchorA, rd.localAnchorB = capi.Vec2(60.3, 10.0), capi.Vec2(-0.3, 0.0)
    joints.append(P.s2CreateRevoluteJoint(wid, C.byref(rd)))
    dragged = _body(P, wid, capi.DYNAMIC_BODY, 70.0, 5.0)
    md = capi.MouseJointDef()
    md.bodyIdA, md.bodyIdB = ground, dragged
    md.target = capi.Vec2(70.5, 5.5)
    md.hertz, md.dampingRatio = 4.0, 0.7
    joints.append(P.s2CreateMouseJoint(wid, C.byref(md)))
    return wid, joints, (ground, spin)


def _step_and_compare(P, wid, dw, O, solver, steps, colour=False, edit=None):
    ctx = device.make_context(solver, DT, 4, 2)
    moved = False
    for k in range(steps):
        if edit is not None:
            edit(k)
        P.s2World_Flush(wid)  # the rows the step starts from carry every edit and every created or destroyed joint
        bodies = dw.download_all_bodies()
        joints = dw.download_joints()
        dp = dw.download_delta_positions()
        P.s2World_Step(wid, DT, 4, 2, True)
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


# ---- scenes.wheels through the public API against reference collide and finalize --------------------------------------------

def _as_wheel(joints, slots, defs, carried):
    """Turn the stand-in revolute rows at `slots` into the wheel rows `defs` describe, with the spring impulses the last step
    left."""
    for slot, d in zip(slots, defs):
        r = joints[slot]
        flags = (int(r["flags"]) & (device.ROW_VALID | device.JOINT_COLLIDE_CONNECTED)) | (device.JOINT_WHEEL << 1)
        flags |= device.JOINT_ENABLE_SPRING if d["enableSpring"] else 0
        flags |= device.JOINT_ENABLE_LIMIT if d["enableLimit"] else 0
        flags |= device.JOINT_ENABLE_MOTOR if d["enableMotor"] else 0
        joints["flags"][slot] = flags
        joints["localOriginAnchorA"][slot] = d["localAnchorA"]
        joints["localOriginAnchorB"][slot] = d["localAnchorB"]
        ax = np.float32(d["localAxisA"])
        n = np.sqrt(ax[0] * ax[0] + ax[1] * ax[1], dtype=np.float32)
        joints["localAxisA"][slot] = (ax[0] / n, ax[1] / n)
        joints["referenceAngle"][slot] = 0.0
        joints["lowerAngle"][slot] = d["lowerTranslation"]
        joints["upperAngle"][slot] = d["upperTranslation"]
        joints["maxMotorTorque"][slot] = d["maxMotorTorque"]
        joints["motorSpeed"][slot] = d["motorSpeed"]
        joints["hertz"][slot] = d["hertz"]
        joints["dampingRatio"][slot] = d["dampingRatio"]
        joints["springImpulse"][slot] = carried.get(slot, 0.0)
    return joints


@pytest.mark.parametrize("mode", ["wavefront", "color"])
@pytest.mark.parametrize("solver", VARIANTS)
def test_wheel_scene_every_step(reference, product, dev, solver, mode):
    """scenes.wheels: reference collide on the stand-in world, the wheel oracle in the device's order, reference finalize;
    the device runs the same steps through s2World_Step with real wheel joints. Every step bit for bit: bodies, delta
    positions, contact impulses and joint impulses, the spring impulse included."""
    R, P = reference, product
    O = wheel_oracle.load()
    sr = scenes.wheels(R, solver)
    sp = scenes.wheels(P, solver)
    assert "s2CreateWheelJoint" in R.missing and "s2CreateWheelJoint" not in P.missing
    slots = [sp.joints[k].index for k in sp.piles["wheel"]]
    defs = sp.piles["wheel_defs"]
    assert slots == [sr.joints[k].index for k in sr.piles["wheel"]] and defs == sr.piles["wheel_defs"] and len(slots) == 6
    P.s2World_Flush(sp.world)
    dw = device.DeviceWorld.attach(dev, sp.world)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT if mode == "wavefront" else device.SCHEDULE_COLOR)
    rows = dw.download_joints(len(sp.joints))
    assert all((rows["flags"][slot] >> 1) & 0x7 == device.JOINT_WHEEL for slot in slots)
    ctx = device.make_context(solver, DT, 4, 2, True)
    sticky = solver == "TGS_Sticky"
    solved = {}
    carried = {}
    F = refmod.BODY_F
    contacts_seen = 0
    motor_seen = False
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
        joints = _as_wheel(joint_rows_from_ref(*R.joints(sr.world)), slots, defs, carried)
        got_contacts = dw.download_contacts(len(rows_key) + 64)
        assert len(got_contacts) == len(rows_key) and np.array_equal(got_contacts["shapeA"], rows_key["shapeA"]), step
        contacts_seen += int(np.count_nonzero(rows_key["pointCount"]))

        order, _ = dw.solve_order(len(rows_key) + len(joints) + 16, max_groups=200000)
        ob, oc, oj, odp = O.solve(capi.SOLVER[solver], bodies, rows_key, joints, ctx, order=order,
                                  dp=ref_delta_positions(R, sr.world))
        carried = {slot: float(oj["springImpulse"][slot]) for slot in slots}
        motor_seen = motor_seen or oj["impulse"][slots[0]][1] != 0.0  # the rear motor

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
    assert contacts_seen > 100
    if solver != "XPBD":
        assert sum(oj["impulse"][slot][0] != 0.0 for slot in slots) >= 4
        assert motor_seen
        assert sum(carried[slot] != 0.0 for slot in slots) >= 4
    sp.destroy()
    sr.destroy()


# ---- a contact-free world through the public API, every step ---------------------------------------------------------------

@pytest.mark.parametrize("gather", [True, False])
@pytest.mark.parametrize("persistent", [True, False])
@pytest.mark.parametrize("mode", ["wavefront", "color"])
@pytest.mark.parametrize("solver", VARIANTS)
def test_public_world_every_step(product, dev, solver, mode, persistent, gather):
    """Each s2World_Step equals the wheel oracle's stage on the rows the step started from, bit for bit, delta positions
    included."""
    if not gather and solver not in SUBSTEPPING:
        pytest.skip("the warm-start gather serves the sub-stepping variants only")
    P = product
    wid, _, _ = _wheel_world(P, solver)
    P.s2World_Step(wid, DT, 4, 2, True)  # uploads the world
    dw = device.DeviceWorld.attach(dev, wid)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT if mode == "wavefront" else device.SCHEDULE_COLOR)
    dw.set_persistent(persistent)
    dw.set_warm_gather(gather)
    _step_and_compare(P, wid, dw, wheel_oracle.load(), solver, 60, colour=mode == "color")
    P.s2DestroyWorld(wid)


@pytest.mark.parametrize("solver", ["TGS_Soft", "PGS", "TGS_NGS", "XPBD"])
def test_setter_edits_between_replayed_steps(product, dev, solver):
    """Springs, limits and motors edited between steps land in the next step's rows (replayed solve graph), and each step
    still equals the oracle."""
    P = product
    wid, joints, _ = _wheel_world(P, solver)
    P.s2World_Step(wid, DT, 4, 2, True)
    dw = device.DeviceWorld.attach(dev, wid)

    def edit(k):
        if k == 10:
            P.s2WheelJoint_SetSpringHertz(joints[0], 6.0)
            P.s2WheelJoint_SetSpringDampingRatio(joints[0], 0.2)
            P.s2WheelJoint_SetLimits(joints[0], -0.1, 0.05)
            P.s2WheelJoint_SetMotorSpeed(joints[1], -2.0)
        elif k == 20:
            P.s2WheelJoint_SetMaxMotorTorque(joints[2], 60.0)
            P.s2WheelJoint_EnableSpring(joints[3], False)
            P.s2WheelJoint_EnableMotor(joints[0], True)
            P.s2WheelJoint_SetMaxMotorTorque(joints[0], 3.0)
        elif k == 30:
            P.s2WheelJoint_EnableLimit(joints[4], False)
            P.s2WheelJoint_EnableMotor(joints[4], False)
            P.s2WheelJoint_EnableSpring(joints[3], True)

    replays = dw.counters().graphReplays
    _step_and_compare(P, wid, dw, wheel_oracle.load(), solver, 45, colour=True, edit=edit)
    assert dw.counters().graphReplays > replays
    P.s2DestroyWorld(wid)


def test_slot_reuse_across_types(product, dev):
    """A wheel joint destroyed and a prismatic joint created in its slot, then a distance joint, then a wheel again: every
    step equals the oracle, so no impulse or marker of the slot's last type survives."""
    P = product
    solver = "TGS_Soft"
    wid, joints, (ground, spin) = _wheel_world(P, solver)
    P.s2World_Step(wid, DT, 4, 2, True)
    dw = device.DeviceWorld.attach(dev, wid)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT)
    O = wheel_oracle.load()
    _step_and_compare(P, wid, dw, O, solver, 10)
    P.s2DestroyJoint(joints[0])
    pd = capi.default_prismatic_def()
    pd.bodyIdA, pd.bodyIdB = ground, spin
    pd.localAnchorA, pd.localAxisA = capi.Vec2(0.0, 10.0), capi.Vec2(0.0, 1.0)
    pd.enableLimit, pd.lowerTranslation, pd.upperTranslation = True, -0.4, 0.4
    pd.enableSpring, pd.hertz, pd.dampingRatio = True, 2.0, 0.5
    prismatic = P.s2CreatePrismaticJoint(wid, C.byref(pd))
    assert prismatic.index == joints[0].index
    _step_and_compare(P, wid, dw, O, solver, 10)
    P.s2DestroyJoint(prismatic)
    dd = capi.default_distance_def()
    dd.bodyIdA, dd.bodyIdB = ground, spin
    dd.localAnchorA, dd.length = capi.Vec2(0.0, 10.0), 0.5
    distance = P.s2CreateDistanceJoint(wid, C.byref(dd))
    assert distance.index == joints[0].index
    _step_and_compare(P, wid, dw, O, solver, 10)
    P.s2DestroyJoint(distance)
    again = _wheel(P, wid, ground, spin, (0.0, 10.0), (0.0, 0.0), spring=(1.0, 0.1), limit=(-0.8, 0.2), motor=(1.0, 1.0))
    assert again.index == joints[0].index
    _step_and_compare(P, wid, dw, O, solver, 10)
    P.s2DestroyWorld(wid)


def test_collide_connected(product, dev):
    """Two boxes resting in contact on the ground: a wheel joint with collideConnected == false removes their contact, one
    with true keeps it."""
    P = product
    kept = []
    for collide in (False, True):
        wid = P.create_world("TGS_Soft")
        ground = P.s2CreateBody(wid, C.byref(capi.default_body_def()))
        sd = capi.default_shape_def()
        P.s2CreatePolygonShape(ground, C.byref(sd), C.byref(P.s2MakeOffsetBox(20.0, 0.5, capi.Vec2(0.0, -0.5), 0.0)))
        a = _body(P, wid, capi.DYNAMIC_BODY, 0.0, 0.2, group=0)
        b = _body(P, wid, capi.DYNAMIC_BODY, 0.59, 0.2, group=0)
        for _ in range(10):
            P.s2World_Step(wid, DT, 4, 2, True)
        dw = device.DeviceWorld.attach(dev, wid)
        before = dw.counters().constraintCount
        _wheel(P, wid, a, b, (0.59, 0.0), (0.0, 0.0), axis=(1.0, 0.0), collide=collide)
        for _ in range(3):
            P.s2World_Step(wid, DT, 4, 2, True)
        kept.append(dw.counters().constraintCount - before)
        P.s2DestroyWorld(wid)
    assert kept[0] == -1 and kept[1] == 0, kept


def test_create_and_setters_reject_bad_input(product, dev):
    P = product
    wid = P.create_world("TGS_Soft")
    ground = _body(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    body = _body(P, wid, capi.DYNAMIC_BODY, 0.0, -1.0)
    nan, inf = float("nan"), float("inf")
    bad = [dict(localAxisA=capi.Vec2(0.0, 0.0)), dict(localAxisA=capi.Vec2(nan, 1.0)), dict(localAxisA=capi.Vec2(inf, 1.0)),
           dict(lowerTranslation=1.0, upperTranslation=0.5), dict(hertz=-1.0), dict(hertz=nan), dict(dampingRatio=-0.1),
           dict(dampingRatio=inf), dict(maxMotorTorque=-2.0), dict(maxMotorTorque=nan), dict(motorSpeed=nan),
           dict(motorSpeed=inf), dict(localAnchorA=capi.Vec2(nan, 0.0))]
    for fields in bad:
        jd = capi.default_wheel_def()
        jd.bodyIdA, jd.bodyIdB = ground, body
        for k, v in fields.items():
            setattr(jd, k, v)
        j = P.s2CreateWheelJoint(wid, C.byref(jd))
        assert j.index == -1, fields  # s2_nullJointId
    j = _wheel(P, wid, ground, body, (0.0, 0.0), (0.0, 0.0), spring=(2.0, 0.5), limit=(-0.5, 0.5), motor=(1.0, 3.0))
    assert j.index >= 0
    P.s2WheelJoint_SetLimits(j, 1.0, 0.0)
    P.s2WheelJoint_SetLimits(j, nan, 1.0)
    P.s2WheelJoint_SetSpringHertz(j, -1.0)
    P.s2WheelJoint_SetSpringDampingRatio(j, nan)
    P.s2WheelJoint_SetMaxMotorTorque(j, -1.0)
    P.s2WheelJoint_SetMotorSpeed(j, inf)
    # a joint of another type is ignored and reads 0
    rd = capi.default_revolute_def()
    rd.bodyIdA, rd.bodyIdB = ground, body
    rev = P.s2CreateRevoluteJoint(wid, C.byref(rd))
    P.s2WheelJoint_SetLimits(rev, -1.0, 2.0)
    P.s2WheelJoint_EnableLimit(rev, True)
    P.s2WheelJoint_SetMaxMotorTorque(rev, 9.0)
    P.s2WheelJoint_EnableSpring(rev, True)
    P.s2World_Step(wid, DT, 4, 2, True)
    assert P.s2WheelJoint_GetTranslation(rev) == 0.0 and P.s2WheelJoint_GetMotorTorque(rev, 60.0) == 0.0
    rows = device.DeviceWorld.attach(dev, wid).download_joints()
    r = rows[j.index]
    assert (r["lowerAngle"], r["upperAngle"], r["hertz"], r["dampingRatio"]) == (-0.5, 0.5, 2.0, 0.5)
    assert (r["maxMotorTorque"], r["motorSpeed"]) == (3.0, 1.0)
    r = rows[rev.index]
    assert r["lowerAngle"] == 0.0 and r["upperAngle"] == 0.0 and r["maxMotorTorque"] == 0.0
    assert r["flags"] & (device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_SPRING) == 0
    # the default definition is Box2D v3's
    d = capi.default_wheel_def()
    assert (d.localAxisA.x, d.localAxisA.y, d.enableSpring, d.hertz, np.float32(d.dampingRatio)) == \
        (0.0, 1.0, True, 1.0, np.float32(0.7))
    assert not d.enableLimit and not d.enableMotor and not d.collideConnected
    P.s2DestroyWorld(wid)


def test_translation_and_draw(product, dev):
    """GetTranslation is anchor B's offset from anchor A along the world axis; s2World_Draw draws the axis through anchor A,
    a mark at each limit and the segment from anchor A to anchor B."""
    P = product
    wid = P.create_world("TGS_Soft")
    ground = _body(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    body = _body(P, wid, capi.DYNAMIC_BODY, 0.3, -0.2, angle=0.4)
    j = _wheel(P, wid, ground, body, (0.3, 0.0), (0.0, 0.0), axis=(0.0, 2.0), spring=(1.0, 0.7), limit=(-0.5, 0.5))
    for _ in range(20):
        P.s2World_Step(wid, DT, 4, 2, True)
    pos = P.s2Body_GetPosition(body)
    t = P.s2WheelJoint_GetTranslation(j)
    assert abs(t - (pos.y - 0.0)) <= 1e-6 and abs(pos.x - 0.3) <= 1e-3
    assert -0.5 - 1e-3 <= t < 0.0
    segments = [v for name, v in _draw_log(P, wid) if name == "DrawSegment"]
    # the axis: drawSize (1 m) each way from anchor A along (0, 1)
    assert any(abs(v[0] - 0.3) < 1e-6 and abs(v[1] + 1.0) < 1e-6 and abs(v[2] - 0.3) < 1e-6 and abs(v[3] - 1.0) < 1e-6
               for v in segments)
    for at in (-0.5, 0.5):
        assert any(abs(0.5 * (v[0] + v[2]) - 0.3) < 1e-5 and abs(0.5 * (v[1] + v[3]) - at) < 1e-5 and abs(v[1] - v[3]) < 1e-6
                   for v in segments), at
    assert any(abs(v[0] - 0.3) < 1e-6 and abs(v[1]) < 1e-6 and abs(v[2] - pos.x) < 1e-5 and abs(v[3] - pos.y) < 1e-5
               for v in segments)
    P.s2DestroyWorld(wid)


def test_reactions_motor_torque_and_a_wheel_that_breaks(product, dev):
    """A wheel hanging at rest on its suspension reads (0, m g) through the host getter and the device's bulk read alike, bit
    for bit, and its reaction torque is GetMotorTorque; a break force below the load snaps the wheel off."""
    P = product
    wid = P.create_world("TGS_Soft")
    ground = _body(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    body = _body(P, wid, capi.DYNAMIC_BODY, 0.0, -1.0, radius=0.3)
    j = _wheel(P, wid, ground, body, (0.0, -1.0), (0.0, 0.0), spring=(2.0, 1.0), motor=(30.0, 0.02))
    for _ in range(180):
        P.s2World_Step(wid, DT, 4, 2, True)
    f = P.s2Joint_GetReactionForce(j)
    mass = P.s2Body_GetMass(body)
    assert abs(f.x) <= 1e-4 and abs(f.y - mass * 10.0) <= 1e-3 * mass * 10.0, (f.x, f.y, mass)
    torque = P.s2Joint_GetReactionTorque(j)
    # GetMotorTorque at the reaction's rate (1 / h) is the reaction torque; at 4 / dt it differs from it by rounding only
    assert torque != 0.0 and abs(torque - P.s2WheelJoint_GetMotorTorque(j, 4.0 / DT)) <= 1e-6 * abs(torque)
    assert abs(torque) <= 0.02 * (1.0 + 1e-6)
    out = np.zeros(3 * 8, dtype=np.float32)
    P.s2World_GetJointReactions(wid, out.ctypes.data, 8)
    assert (out[3 * j.index], out[3 * j.index + 1], out[3 * j.index + 2]) == (np.float32(f.x), np.float32(f.y), np.float32(torque))
    P.s2Joint_SetBreakForce(j, 0.5 * f.y)
    P.s2World_Step(wid, DT, 4, 2, True)
    broken = (capi.JointId * 4)()
    assert P.s2World_GetBrokenJoints(wid, broken, 4) == 1 and broken[0].index == j.index
    P.s2World_Step(wid, DT, 4, 2, True)
    y = P.s2Body_GetPosition(body).y
    for _ in range(10):
        P.s2World_Step(wid, DT, 4, 2, True)
    assert P.s2Body_GetPosition(body).y < y - 0.1  # falling free
    P.s2DestroyWorld(wid)
