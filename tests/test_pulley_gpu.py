"""GPU: the pulley joint (DESIGN.md §3.18). The device against the joint oracle (tests/joint_oracle.c) bit for bit: every
step of scenes.pulleys (Box2D 2.4's testbed pulley, a counterweighted lift on a prismatic joint carrying a pile, a
block-and-tackle at ratio 2, a kinematic driver, contacts throughout) through the public API against reference collide and
finalize around the oracle, in the wavefront and the colour schedule; every step of a contact-free world for all ten
variants, in both schedules, persistent and launch by launch, with the warm-start gather on and off; slot reuse across the
pulley, wheel and distance joints. Also: collideConnected both ways, input checks, the getters, the drawn segments,
reactions against the bulk read, and a break threshold that snaps a pulley.

Mutations each test catches: a rope formed from the other body's pose or without its start offset, a ratio left out of
side B's impulse or of the mass, a warm start or gather that leaves one side out, and an impulse kept without a warm start
all fail the every-step comparisons; a reaction on the wrong side or without -ratio fails the reaction test."""
import ctypes as C

import numpy as np
import pytest

import joint_oracle
from helpers import (bit_equal, body_rows_from_ref, carry_sticky_friction, contact_rows_from_ref, joint_rows_from_ref,
                     load_bodies_into_ref, ref_delta_positions, store_oracle_bodies)
from oracle import ref as refmod
from solver2d_b200 import capi, device, scenes
from test_api_lifecycle_gpu import _draw_log
from test_prismatic_gpu import _as_prismatic
from test_wheel_gpu import _body, _step_and_compare, _wheel

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0
VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]
SUBSTEPPING = {"SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"}
JOINT_FIELDS = ("impulse", "motorImpulse", "lowerImpulse", "upperImpulse", "springImpulse")


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


def _pulley(P, wid, a, b, ground_a, ground_b, anchor_a, anchor_b, length_a, length_b, ratio, collide=True):
    jd = capi.default_pulley_def()
    jd.bodyIdA, jd.bodyIdB = a, b
    jd.groundAnchorA, jd.groundAnchorB = capi.Vec2(*ground_a), capi.Vec2(*ground_b)
    jd.localAnchorA, jd.localAnchorB = capi.Vec2(*anchor_a), capi.Vec2(*anchor_b)
    jd.lengthA, jd.lengthB, jd.ratio = length_a, length_b, ratio
    jd.collideConnected = collide
    return P.s2CreatePulleyJoint(wid, C.byref(jd))


def _world_point(P, body, local):
    p, angle = P.s2Body_GetPosition(body), P.s2Body_GetAngle(body)
    c, s = np.cos(angle), np.sin(angle)
    return p.x + c * local[0] - s * local[1], p.y + s * local[0] + c * local[1]


def _pulley_world(P, solver):
    """Bodies far apart (no contacts): an unbalanced pair at ratio 1.5 with off-centre anchors, a balanced pair at ratio 2,
    a pair created 0.6 m off its constant, a kinematic driver on side A, a rope within 10 s2_linearSlop of its ground
    anchor, a pulley between two dynamic bodies without gravity, spun, a wheel, a revolute link and a mouse joint."""
    wid = P.create_world(solver)
    ground = _body(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    joints = []
    a = _body(P, wid, capi.DYNAMIC_BODY, 0.0, 5.0, w=0.5)
    b = _body(P, wid, capi.DYNAMIC_BODY, 4.0, 5.0, angle=0.3)
    joints.append(_pulley(P, wid, a, b, (0.2, 12.0), (4.0, 12.0), (0.1, 0.2), (-0.2, 0.1), 6.81, 6.9, 1.5))
    light = _body(P, wid, capi.DYNAMIC_BODY, 10.0, 5.0)
    heavy = _body(P, wid, capi.DYNAMIC_BODY, 13.0, 5.0, gravity=2.0)  # twice the weight at the same mass
    joints.append(_pulley(P, wid, light, heavy, (10.0, 12.0), (13.0, 12.0), (0.0, 0.0), (0.0, 0.0), 7.0, 7.0, 2.0))
    off_a = _body(P, wid, capi.DYNAMIC_BODY, 20.0, 5.0)
    off_b = _body(P, wid, capi.DYNAMIC_BODY, 23.0, 5.0)
    joints.append(_pulley(P, wid, off_a, off_b, (20.0, 12.0), (23.0, 12.0), (0.0, 0.0), (0.0, 0.0), 7.6, 7.0, 1.0))
    driver = _body(P, wid, capi.KINEMATIC_BODY, 30.0, 5.0, vy=-0.4, w=0.3)
    load = _body(P, wid, capi.DYNAMIC_BODY, 33.0, 5.0)
    joints.append(_pulley(P, wid, driver, load, (30.0, 12.0), (33.0, 12.0), (0.0, 0.2), (0.0, 0.2), 6.8, 6.8, 1.5))
    tight = _body(P, wid, capi.DYNAMIC_BODY, 40.0, 11.98)
    hung = _body(P, wid, capi.DYNAMIC_BODY, 43.0, 5.0)
    joints.append(_pulley(P, wid, tight, hung, (40.0, 12.0), (43.0, 12.0), (0.0, 0.0), (0.0, 0.0), 0.02, 7.0, 1.0))
    left = _body(P, wid, capi.DYNAMIC_BODY, 50.0, 5.0, vx=0.3, w=1.0, gravity=0.0)
    right = _body(P, wid, capi.DYNAMIC_BODY, 51.0, 4.0, w=-2.0, gravity=0.0)
    joints.append(_pulley(P, wid, left, right, (50.0, 7.0), (52.0, 7.0), (0.2, 0.1), (-0.1, 0.0), 1.8, 3.2, 0.7))
    wheel = _body(P, wid, capi.DYNAMIC_BODY, 60.0, 9.8, w=6.0, radius=0.3)
    joints.append(_wheel(P, wid, ground, wheel, (60.0, 10.0), (0.0, 0.0), spring=(4.0, 0.7), limit=(-0.3, 0.3)))
    link = _body(P, wid, capi.DYNAMIC_BODY, 70.6, 10.0)
    rd = capi.default_revolute_def()
    rd.bodyIdA, rd.bodyIdB = ground, link
    rd.localAnchorA, rd.localAnchorB = capi.Vec2(70.3, 10.0), capi.Vec2(-0.3, 0.0)
    joints.append(P.s2CreateRevoluteJoint(wid, C.byref(rd)))
    dragged = _body(P, wid, capi.DYNAMIC_BODY, 80.0, 5.0)
    md = capi.MouseJointDef()
    md.bodyIdA, md.bodyIdB = ground, dragged
    md.target = capi.Vec2(80.5, 5.5)
    md.hertz, md.dampingRatio = 4.0, 0.7
    joints.append(P.s2CreateMouseJoint(wid, C.byref(md)))
    assert all(j.index >= 0 for j in joints)
    return wid, joints, (ground, a, b)


# ---- scenes.pulleys through the public API against reference collide and finalize -------------------------------------------

def _as_pulley(joints, slots, defs):
    """Turn the stand-in revolute rows at `slots` into the pulley rows `defs` describe."""
    for slot, d in zip(slots, defs):
        r = joints[slot]
        joints["flags"][slot] = (int(r["flags"]) & (device.ROW_VALID | device.JOINT_COLLIDE_CONNECTED)) | (device.JOINT_PULLEY << 1)
        joints["localOriginAnchorA"][slot] = d["localAnchorA"]
        joints["localOriginAnchorB"][slot] = d["localAnchorB"]
        joints["target"][slot] = d["groundAnchorA"]
        joints["localAxisA"][slot] = d["groundAnchorB"]
        joints["referenceAngle"][slot] = d["ratio"]
        joints["lowerAngle"][slot] = d["lengthA"]
        joints["upperAngle"][slot] = d["lengthB"]
    return joints


@pytest.mark.parametrize("mode", ["wavefront", "color"])
@pytest.mark.parametrize("solver", VARIANTS)
def test_pulley_scene_every_step(reference, product, dev, solver, mode):
    """scenes.pulleys: reference collide on the stand-in world, the pulley oracle in the device's order, reference finalize;
    the device runs the same steps through s2World_Step with real pulleys and a real prismatic joint. Every step bit for
    bit: bodies, delta positions, contact impulses and joint impulses."""
    R, P = reference, product
    O = joint_oracle.load()
    sr = scenes.pulleys(R, solver)
    sp = scenes.pulleys(P, solver)
    assert "s2CreatePulleyJoint" in R.missing and "s2CreatePulleyJoint" not in P.missing
    slots = [sp.joints[k].index for k in sp.piles["pulley"]]
    defs = sp.piles["pulley_defs"]
    assert slots == [sr.joints[k].index for k in sr.piles["pulley"]] and defs == sr.piles["pulley_defs"] and len(slots) == 5
    pslots = [sp.joints[k].index for k in sp.piles["prismatic"]]
    assert pslots == [sr.joints[k].index for k in sr.piles["prismatic"]]
    P.s2World_Flush(sp.world)
    dw = device.DeviceWorld.attach(dev, sp.world)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT if mode == "wavefront" else device.SCHEDULE_COLOR)
    rows = dw.download_joints(len(sp.joints))
    assert all((rows["flags"][slot] >> 1) & 0x7 == device.JOINT_PULLEY for slot in slots)
    ctx = device.make_context(solver, DT, 4, 2, True)
    sticky = solver == "TGS_Sticky"
    solved = {}
    F = refmod.BODY_F
    contacts_seen = 0
    shared = False  # a contact on a pulley's body
    pulley_bodies = {int(rows["bodyA"][s]) for s in slots} | {int(rows["bodyB"][s]) for s in slots}
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
        joints = _as_pulley(joint_rows_from_ref(*R.joints(sr.world)), slots, defs)
        joints = _as_prismatic(joints, pslots, sp.piles["prismatic_defs"])
        got_contacts = dw.download_contacts(len(rows_key) + 64)
        assert len(got_contacts) == len(rows_key) and np.array_equal(got_contacts["shapeA"], rows_key["shapeA"]), step
        touching = rows_key["pointCount"] > 0
        contacts_seen += int(np.count_nonzero(touching))
        shared = shared or bool(set(rows_key["bodyA"][touching].tolist() + rows_key["bodyB"][touching].tolist()) & pulley_bodies)

        order, _ = dw.solve_order(len(rows_key) + len(joints) + 16, max_groups=200000)
        ob, oc, oj, odp = O.solve(capi.SOLVER[solver], bodies, rows_key, joints, ctx, order=order,
                                  dp=ref_delta_positions(R, sr.world))

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
    assert contacts_seen > 100 and shared
    if solver != "XPBD":
        assert sum(oj["impulse"][slot][0] != 0.0 for slot in slots) >= 4
    sp.destroy()
    sr.destroy()


# ---- a contact-free world through the public API, every step ---------------------------------------------------------------

@pytest.mark.parametrize("gather", [True, False])
@pytest.mark.parametrize("persistent", [True, False])
@pytest.mark.parametrize("mode", ["wavefront", "color"])
@pytest.mark.parametrize("solver", VARIANTS)
def test_public_world_every_step(product, dev, solver, mode, persistent, gather):
    """Each s2World_Step equals the pulley oracle's stage on the rows the step started from, bit for bit, delta positions
    included."""
    if not gather and solver not in SUBSTEPPING:
        pytest.skip("the warm-start gather serves the sub-stepping variants only")
    P = product
    wid, _, _ = _pulley_world(P, solver)
    P.s2World_Step(wid, DT, 4, 2, True)  # uploads the world
    dw = device.DeviceWorld.attach(dev, wid)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT if mode == "wavefront" else device.SCHEDULE_COLOR)
    dw.set_persistent(persistent)
    dw.set_warm_gather(gather)
    _step_and_compare(P, wid, dw, joint_oracle.load(), solver, 60, colour=mode == "color")
    P.s2DestroyWorld(wid)


def test_slot_reuse_across_types(product, dev):
    """A pulley destroyed and a wheel joint created in its slot, then a distance joint, then a pulley again: every step
    equals the oracle, so no impulse or column of the slot's last type survives."""
    P = product
    solver = "TGS_Soft"
    wid, joints, (ground, a, b) = _pulley_world(P, solver)
    P.s2World_Step(wid, DT, 4, 2, True)
    dw = device.DeviceWorld.attach(dev, wid)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT)
    O = joint_oracle.load()
    _step_and_compare(P, wid, dw, O, solver, 10)
    P.s2DestroyJoint(joints[0])
    wheel = _wheel(P, wid, a, b, (0.0, 0.0), (-4.0, 0.0), axis=(1.0, 0.0), spring=(2.0, 0.5), limit=(-0.4, 0.4), motor=(1.0, 2.0))
    assert wheel.index == joints[0].index
    _step_and_compare(P, wid, dw, O, solver, 10)
    P.s2DestroyJoint(wheel)
    dd = capi.default_distance_def()
    dd.bodyIdA, dd.bodyIdB = ground, a
    dd.localAnchorA, dd.length = capi.Vec2(0.0, 12.0), 5.0
    distance = P.s2CreateDistanceJoint(wid, C.byref(dd))
    assert distance.index == joints[0].index
    _step_and_compare(P, wid, dw, O, solver, 10)
    P.s2DestroyJoint(distance)
    again = _pulley(P, wid, a, b, (0.0, 12.0), (4.0, 12.0), (0.0, 0.0), (0.0, 0.0), 7.0, 7.0, 1.2)
    assert again.index == joints[0].index
    _step_and_compare(P, wid, dw, O, solver, 10)
    P.s2DestroyWorld(wid)


def test_collide_connected(product, dev):
    """Two boxes resting in contact on the ground: a pulley with collideConnected == false removes their contact, one with
    true (the default) keeps it."""
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
        pa, pb = P.s2Body_GetPosition(a), P.s2Body_GetPosition(b)
        _pulley(P, wid, a, b, (0.0, 3.0), (0.59, 3.0), (0.0, 0.0), (0.0, 0.0), 3.0 - pa.y, 3.0 - pb.y, 1.0, collide=collide)
        for _ in range(3):
            P.s2World_Step(wid, DT, 4, 2, True)
        kept.append(dw.counters().constraintCount - before)
        P.s2DestroyWorld(wid)
    assert kept[0] == -1 and kept[1] == 0, kept


def test_create_rejects_bad_input_and_getters(product, dev):
    P = product
    wid = P.create_world("TGS_Soft")
    ground = _body(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    body = _body(P, wid, capi.DYNAMIC_BODY, 0.0, -1.0)
    other = _body(P, wid, capi.DYNAMIC_BODY, 3.0, -2.0, angle=0.5)
    nan, inf = float("nan"), float("inf")
    eps = float(np.finfo(np.float32).eps)
    bad = [dict(groundAnchorA=capi.Vec2(nan, 0.0)), dict(groundAnchorB=capi.Vec2(0.0, inf)),
           dict(localAnchorA=capi.Vec2(inf, 0.0)), dict(localAnchorB=capi.Vec2(0.0, nan)), dict(lengthA=-0.1),
           dict(lengthB=-1.0), dict(lengthA=nan), dict(lengthB=inf), dict(ratio=0.0), dict(ratio=eps), dict(ratio=-1.0),
           dict(ratio=nan), dict(ratio=inf)]
    for fields in bad:
        jd = capi.default_pulley_def()
        jd.bodyIdA, jd.bodyIdB = body, other
        for k, v in fields.items():
            setattr(jd, k, v)
        j = P.s2CreatePulleyJoint(wid, C.byref(jd))
        assert j.index == -1, fields  # s2_nullJointId
    # the default definition is Box2D 2.4's
    d = capi.default_pulley_def()
    assert (d.groundAnchorA.x, d.groundAnchorA.y, d.groundAnchorB.x, d.groundAnchorB.y) == (-1.0, 1.0, 1.0, 1.0)
    assert (d.localAnchorA.x, d.localAnchorA.y, d.localAnchorB.x, d.localAnchorB.y) == (-1.0, 0.0, 1.0, 0.0)
    assert (d.lengthA, d.lengthB, d.ratio, d.collideConnected) == (0.0, 0.0, 1.0, True)
    j = _pulley(P, wid, body, other, (0.0, 4.0), (3.0, 4.0), (0.2, 0.1), (-0.1, 0.3), 5.0, 6.0, 1.25)
    assert j.index >= 0
    ga, gb = P.s2PulleyJoint_GetGroundAnchorA(j), P.s2PulleyJoint_GetGroundAnchorB(j)
    assert (ga.x, ga.y, gb.x, gb.y) == (0.0, 4.0, 3.0, 4.0)
    assert (P.s2PulleyJoint_GetLengthA(j), P.s2PulleyJoint_GetLengthB(j), P.s2PulleyJoint_GetRatio(j)) == (5.0, 6.0, 1.25)
    for _ in range(5):
        P.s2World_Step(wid, DT, 4, 2, True)
    for getter, b, local, g in ((P.s2PulleyJoint_GetCurrentLengthA, body, (0.2, 0.1), (0.0, 4.0)),
                                (P.s2PulleyJoint_GetCurrentLengthB, other, (-0.1, 0.3), (3.0, 4.0))):
        p = _world_point(P, b, local)
        assert abs(getter(j) - np.hypot(p[0] - g[0], p[1] - g[1])) <= 1e-5
    # a joint of another type reads 0
    rd = capi.default_revolute_def()
    rd.bodyIdA, rd.bodyIdB = ground, body
    rev = P.s2CreateRevoluteJoint(wid, C.byref(rd))
    z = P.s2PulleyJoint_GetGroundAnchorA(rev), P.s2PulleyJoint_GetGroundAnchorB(rev)
    assert (z[0].x, z[0].y, z[1].x, z[1].y) == (0.0, 0.0, 0.0, 0.0)
    assert (P.s2PulleyJoint_GetLengthA(rev), P.s2PulleyJoint_GetLengthB(rev), P.s2PulleyJoint_GetRatio(rev),
            P.s2PulleyJoint_GetCurrentLengthA(rev), P.s2PulleyJoint_GetCurrentLengthB(rev)) == (0.0, 0.0, 0.0, 0.0, 0.0)
    rows = device.DeviceWorld.attach(dev, wid).download_joints()
    r = rows[j.index]
    assert (r["flags"] >> 1) & 0x7 == device.JOINT_PULLEY
    assert r["flags"] & (device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR | device.JOINT_ENABLE_SPRING) == 0
    assert (r["referenceAngle"], r["lowerAngle"], r["upperAngle"]) == (np.float32(1.25), 5.0, 6.0)
    assert tuple(r["target"]) == (0.0, 4.0) and tuple(r["localAxisA"]) == (3.0, 4.0)
    P.s2DestroyWorld(wid)


def test_draw_three_segments(product, dev):
    """s2World_Draw draws Box2D 2.4's three segments: anchor A to ground A, anchor B to ground B, ground A to ground B."""
    P = product
    wid = P.create_world("TGS_Soft")
    a = _body(P, wid, capi.DYNAMIC_BODY, 0.0, 0.0, gravity=0.0)
    b = _body(P, wid, capi.DYNAMIC_BODY, 3.0, 0.5, gravity=0.0)
    _pulley(P, wid, a, b, (-0.5, 4.0), (3.5, 4.5), (0.1, 0.2), (0.0, -0.1), 3.8, 4.1, 1.0)
    P.s2World_Step(wid, DT, 4, 2, True)
    pa = _world_point(P, a, (0.1, 0.2))
    pb = _world_point(P, b, (0.0, -0.1))
    segments = [v for name, v in _draw_log(P, wid) if name == "DrawSegment"]

    def drawn(p, q):
        return any(abs(v[0] - p[0]) < 1e-5 and abs(v[1] - p[1]) < 1e-5 and abs(v[2] - q[0]) < 1e-5 and abs(v[3] - q[1]) < 1e-5
                   for v in segments)

    assert drawn((-0.5, 4.0), pa) and drawn((3.5, 4.5), pb) and drawn((-0.5, 4.0), (3.5, 4.5))
    P.s2DestroyWorld(wid)


def test_reactions_and_a_pulley_that_breaks(product, dev):
    """A balanced pair at ratio 2 (mB = 2 mA, anchors at the centres of mass) at rest: the reaction on body B reads
    (0, mB g), the same bits through the host getter and the device's bulk read; a break force below it snaps the pulley and
    both bodies fall."""
    P = product
    wid = P.create_world("TGS_Soft")
    a = _body(P, wid, capi.DYNAMIC_BODY, 0.0, 0.0)
    b = _body(P, wid, capi.DYNAMIC_BODY, 3.0, 1.0, gravity=2.0)  # twice A's weight at the same mass
    j = _pulley(P, wid, a, b, (0.0, 5.0), (3.0, 5.0), (0.0, 0.0), (0.0, 0.0), 5.0, 4.0, 2.0)
    for _ in range(120):
        P.s2World_Step(wid, DT, 4, 2, True)
    weight_b = 2.0 * P.s2Body_GetMass(b) * 10.0
    f = P.s2Joint_GetReactionForce(j)
    assert f.x == 0.0 and abs(f.y - weight_b) <= 1e-4 * weight_b, (f.x, f.y, weight_b)
    assert P.s2Joint_GetReactionTorque(j) == 0.0
    # at rest: the soft row settles 2.8e-4 m from its constant under this load (measured), x 3.5
    assert abs(P.s2Body_GetPosition(a).y) <= 1e-3 and abs(P.s2Body_GetPosition(b).y - 1.0) <= 1e-3
    out = np.zeros(3 * 4, dtype=np.float32)
    P.s2World_GetJointReactions(wid, out.ctypes.data, 4)
    assert (out[3 * j.index], out[3 * j.index + 1], out[3 * j.index + 2]) == (np.float32(f.x), np.float32(f.y), 0.0)
    P.s2Joint_SetBreakForce(j, 0.5 * f.y)
    P.s2World_Step(wid, DT, 4, 2, True)
    broken = (capi.JointId * 4)()
    assert P.s2World_GetBrokenJoints(wid, broken, 4) == 1 and broken[0].index == j.index
    P.s2World_Step(wid, DT, 4, 2, True)
    ya, yb = P.s2Body_GetPosition(a).y, P.s2Body_GetPosition(b).y
    for _ in range(10):
        P.s2World_Step(wid, DT, 4, 2, True)
    assert P.s2Body_GetPosition(a).y < ya - 0.1 and P.s2Body_GetPosition(b).y < yb - 0.1  # falling free
    P.s2DestroyWorld(wid)
