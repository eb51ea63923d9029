"""GPU: the gear joint (DESIGN.md §3.19). The device against the gear oracle (tests/gear_oracle.c) bit for bit on every step of
a contact-free world (revolute-revolute gears, a motor-driven train of three stages, a rack and pinion lifting a load, two
racks, a frame turned away from zero, a wheel geared through more than ten turns, and a sun meshing more planets than
S2B_HUB_DEGREE) for all ten variants, in both schedules, persistent and launch by launch, with the warm-start gather on and
off; slot reuse across the gear, revolute and prismatic joints; a teleported static frame. Also: the cascade on
s2DestroyJoint and on a broken joint 1, every rejected input, the getters and drawing, reactions against the bulk read,
and a break threshold on the gear itself.

Mutations each test catches: a side formed from the other body's pose, a ratio left out of side 2's impulse or of the
mass, a warm start or gather that leaves one side out, an impulse kept without a warm start, an unwound coordinate not
stored back (XPBD's included), a type decoded from the 3-bit field alone and a frame left in place by s2Body_SetTransform
all fail the every-step comparisons; a reaction without the ratio or on the wrong side fails the reaction test; a gear
left behind by its joint's destruction fails the cascade tests."""
import ctypes as C

import numpy as np
import pytest

import gear_oracle
from helpers import (bit_equal, body_rows_from_ref, carry_sticky_friction, contact_rows_from_ref, joint_rows_from_ref,
                     load_bodies_into_ref, ref_delta_positions, store_oracle_bodies)
from oracle import ref as refmod
from solver2d_b200 import capi, device, scenes
from test_api_lifecycle_gpu import _draw_log
from test_prismatic_gpu import _as_prismatic
from test_wheel_gpu import _body, _step_and_compare

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0
VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]
SUBSTEPPING = {"SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"}
HUB_PLANETS = 52  # more than S2B_HUB_DEGREE (48)


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


def _revolute(P, wid, ground, body, anchor, motor=None, reference=0.0):
    rd = capi.default_revolute_def()
    rd.bodyIdA, rd.bodyIdB = ground, body
    rd.localAnchorA = capi.Vec2(*anchor)
    rd.referenceAngle = reference
    if motor is not None:
        rd.enableMotor, rd.motorSpeed, rd.maxMotorTorque = True, motor[0], motor[1]
    return P.s2CreateRevoluteJoint(wid, C.byref(rd))


def _prismatic(P, wid, ground, body, anchor, axis, anchor_b=(0.0, 0.0)):
    pd = capi.default_prismatic_def()
    pd.bodyIdA, pd.bodyIdB = ground, body
    pd.localAnchorA, pd.localAnchorB, pd.localAxisA = capi.Vec2(*anchor), capi.Vec2(*anchor_b), capi.Vec2(*axis)
    return P.s2CreatePrismaticJoint(wid, C.byref(pd))


def _gear(P, wid, j1, j2, ratio, collide=False):
    gd = capi.default_gear_def()
    gd.jointId1, gd.jointId2, gd.ratio, gd.collideConnected = j1, j2, ratio, collide
    return P.s2CreateGearJoint(wid, C.byref(gd))


def _gear_world(P, solver, planets=HUB_PLANETS):
    """Bodies far apart (no contacts). Returns (world, gears, links, frames)."""
    wid = P.create_world(solver)
    ground = _body(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    plate = _body(P, wid, capi.STATIC_BODY, 40.0, 0.0, angle=0.4)  # a frame turned away from zero
    gears, links = [], []
    # Box2D 2.4's Gears: two revolute gears at r2 / r1 and a rack at -1 / r2
    w1 = _body(P, wid, capi.DYNAMIC_BODY, 0.0, 5.0, radius=1.0)
    w2 = _body(P, wid, capi.DYNAMIC_BODY, 3.0, 5.0, radius=2.0)
    rack = _body(P, wid, capi.DYNAMIC_BODY, 5.0, 3.0)
    j1 = _revolute(P, wid, ground, w1, (0.0, 5.0), motor=(2.0, 40.0))
    j2 = _revolute(P, wid, ground, w2, (3.0, 5.0), reference=0.3)
    j3 = _prismatic(P, wid, ground, rack, (5.0, 3.0), (0.0, 1.0), anchor_b=(0.1, 0.0))
    links += [j1, j2, j3]
    gears.append(_gear(P, wid, j1, j2, 2.0))
    gears.append(_gear(P, wid, j2, j3, -0.5))
    # a train of three stages on the turned plate
    train = [_body(P, wid, capi.DYNAMIC_BODY, 40.0 + 2.0 * k, 2.0, radius=0.8) for k in range(4)]
    tj = [_revolute(P, wid, plate, b, (2.0 * k, 2.0), reference=0.1 * k) for k, b in enumerate(train)]
    links += tj
    for k in range(3):
        gears.append(_gear(P, wid, tj[k], tj[k + 1], 1.5 if k % 2 == 0 else -0.75))
    # two racks, one horizontal and one slanted, with gravity on both
    ra = _body(P, wid, capi.DYNAMIC_BODY, 60.0, 2.0)
    rb = _body(P, wid, capi.DYNAMIC_BODY, 63.0, 2.0, w=0.5)
    pa = _prismatic(P, wid, ground, ra, (60.0, 2.0), (1.0, 0.0))
    pb = _prismatic(P, wid, ground, rb, (63.0, 2.0), (0.6, 0.8), anchor_b=(0.0, 0.2))
    links += [pa, pb]
    gears.append(_gear(P, wid, pa, pb, 1.3))
    # a wheel geared through many turns
    fast = _body(P, wid, capi.DYNAMIC_BODY, 80.0, 2.0, w=250.0, radius=0.5)
    slow = _body(P, wid, capi.DYNAMIC_BODY, 82.0, 2.0, radius=0.5)
    fj = _revolute(P, wid, ground, fast, (80.0, 2.0))
    sj = _revolute(P, wid, ground, slow, (82.0, 2.0))
    links += [fj, sj]
    gears.append(_gear(P, wid, fj, sj, 1.0))
    # a sun meshing more planets than S2B_HUB_DEGREE: every planet gear is a constraint on the sun
    if planets:
        sun = _body(P, wid, capi.DYNAMIC_BODY, 120.0, 20.0, w=1.0, radius=3.0)
        sunj = _revolute(P, wid, ground, sun, (120.0, 20.0))
        links.append(sunj)
        for k in range(planets):
            angle = 2.0 * np.pi * k / planets
            x, y = 120.0 + 10.0 * np.cos(angle), 20.0 + 10.0 * np.sin(angle)
            p = _body(P, wid, capi.DYNAMIC_BODY, x, y, radius=0.3)
            pj = _revolute(P, wid, ground, p, (x, y))
            links.append(pj)
            gears.append(_gear(P, wid, sunj, pj, 10.0))
    assert all(g.index >= 0 for g in gears)
    return wid, gears, links, (ground, plate)


# ---- scenes.gears through the public API against reference collide and finalize ---------------------------------------------

JOINT_FIELDS = ("impulse", "motorImpulse", "lowerImpulse", "upperImpulse", "springImpulse")
GEAR_CONFIG = ("flags", "localOriginAnchorA", "localOriginAnchorB", "referenceAngle", "lowerAngle", "upperAngle",
               "maxMotorTorque", "motorSpeed", "hertz", "dampingRatio", "target", "localAxisA")


def _as_gear(joints, slots, config):
    """Turn the stand-in revolute rows at `slots` into the gear rows `config` holds (the device's rows as the host filled
    them: flags, anchors, frames, ratio and constant). The gear's state rides in the stand-in's impulse columns."""
    for slot in slots:
        assert (joints["bodyA"][slot], joints["bodyB"][slot]) == (config["bodyA"][slot], config["bodyB"][slot])
        for name in GEAR_CONFIG:
            joints[name][slot] = config[name][slot]
    return joints


@pytest.mark.parametrize("mode", ["wavefront", "color"])
@pytest.mark.parametrize("solver", VARIANTS)
def test_gear_scene_every_step(reference, product, dev, solver, mode):
    """scenes.gears (Box2D 2.4's Gears, a motor-driven train, a rack and pinion lifting a pile, a wheel through more than ten
    turns, a sun meshing more planets than S2B_HUB_DEGREE): reference collide on the stand-in world, the gear oracle in the
    device's order, reference finalize; the device runs the same steps through s2World_Step with real gears and real
    prismatic joints. Every step bit for bit: bodies, delta positions, contact impulses and joint impulses, the unwound
    coordinates included. The gear rows' configuration is the device's own first upload; their state (impulse and unwound
    coordinates) is carried by the oracle from step to step, seeded at step 0 from that upload.

    Mutations it catches beyond the contact-free world's: a gear row that the colouring, the hub path or the schedules
    treat otherwise than a two-body row while contacts share its bodies."""
    R, P = reference, product
    O = gear_oracle.load()
    sr = scenes.gears(R, solver)
    sp = scenes.gears(P, solver)
    assert "s2CreateGearJoint" in R.missing and "s2CreateGearJoint" not in P.missing
    slots = [sp.joints[k].index for k in sp.piles["gear"]]
    assert slots == [sr.joints[k].index for k in sr.piles["gear"]] and len(slots) == 7 + scenes.GEARS_HUB_PLANETS
    pslots = [sp.joints[k].index for k in sp.piles["prismatic"]]
    assert pslots == [sr.joints[k].index for k in sr.piles["prismatic"]]
    P.s2World_Flush(sp.world)
    dw = device.DeviceWorld.attach(dev, sp.world)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT if mode == "wavefront" else device.SCHEDULE_COLOR)
    config = dw.download_joints(len(sp.joints))
    assert all(device.joint_type(int(config["flags"][slot])) == device.JOINT_GEAR for slot in slots)
    ctx = device.make_context(solver, DT, 4, 2, True)
    sticky = solver == "TGS_Sticky"
    solved = {}
    F = refmod.BODY_F
    contacts_seen = 0
    shared = False  # a contact on a geared body
    gear_bodies = {int(config["bodyA"][s]) for s in slots} | {int(config["bodyB"][s]) for s in slots}
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
        joints = _as_gear(joint_rows_from_ref(*R.joints(sr.world)), slots, config)
        if step == 0:
            for slot in slots:
                joints["lowerImpulse"][slot], joints["upperImpulse"][slot] = config["lowerImpulse"][slot], config["upperImpulse"][slot]
        joints = _as_prismatic(joints, pslots, sp.piles["prismatic_defs"])
        got_contacts = dw.download_contacts(len(rows_key) + 64)
        assert len(got_contacts) == len(rows_key) and np.array_equal(got_contacts["shapeA"], rows_key["shapeA"]), step
        touching = rows_key["pointCount"] > 0
        contacts_seen += int(np.count_nonzero(touching))
        shared = shared or bool(set(rows_key["bodyA"][touching].tolist() + rows_key["bodyB"][touching].tolist()) & gear_bodies)

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
        assert sum(oj["impulse"][slot][0] != 0.0 for slot in slots) >= 6
    # the fast pair (the seventh gear) turned through more than ten turns; XPBD's position row damps the spin
    fast = slots[6]
    turns = 4.0 if solver == "XPBD" else 10.0
    assert oj["lowerImpulse"][fast] > 2.0 * np.pi * turns and oj["upperImpulse"][fast] < -2.0 * np.pi * turns
    sp.destroy()
    sr.destroy()


# ---- a contact-free world through the public API, every step ---------------------------------------------------------------

@pytest.mark.parametrize("gather", [True, False])
@pytest.mark.parametrize("persistent", [True, False])
@pytest.mark.parametrize("mode", ["wavefront", "color"])
@pytest.mark.parametrize("solver", VARIANTS)
def test_public_world_every_step(product, dev, solver, mode, persistent, gather):
    """Each s2World_Step equals the gear oracle's stage on the rows the step started from, bit for bit, delta positions and
    the unwound coordinates included."""
    if not gather and solver not in SUBSTEPPING:
        pytest.skip("the warm-start gather serves the sub-stepping variants only")
    P = product
    wid, gears, _, _ = _gear_world(P, solver)
    P.s2World_Step(wid, DT, 4, 2, True)  # uploads the world
    dw = device.DeviceWorld.attach(dev, wid)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT if mode == "wavefront" else device.SCHEDULE_COLOR)
    dw.set_persistent(persistent)
    dw.set_warm_gather(gather)
    _step_and_compare(P, wid, dw, gear_oracle.load(), solver, 60, colour=mode == "color")
    rows = dw.download_joints()
    assert all(device.joint_type(int(rows["flags"][g.index])) == device.JOINT_GEAR for g in gears)
    # the fast pair turned through more than ten turns in 1 s without a jump in its unwound coordinates; XPBD's position
    # row damps the spin to about four turns (26.6 rad measured; tests/test_gear_cpu.py runs it past ten)
    fast = gears[6].index
    turns = 4.0 if solver == "XPBD" else 10.0
    assert rows["lowerImpulse"][fast] > 2.0 * np.pi * turns and rows["upperImpulse"][fast] < -2.0 * np.pi * turns
    P.s2DestroyWorld(wid)


def test_slot_reuse_across_types(product, dev):
    """A gear destroyed and a revolute joint created in its slot, then a prismatic joint, then a gear again: every step equals
    the oracle, so no column of the slot's last type survives."""
    P = product
    solver = "TGS_Soft"
    wid, gears, links, (ground, _) = _gear_world(P, solver, planets=0)
    P.s2World_Step(wid, DT, 4, 2, True)
    dw = device.DeviceWorld.attach(dev, wid)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT)
    O = gear_oracle.load()
    _step_and_compare(P, wid, dw, O, solver, 10)
    slot = gears[0].index
    P.s2DestroyJoint(gears[0])
    extra = _body(P, wid, capi.DYNAMIC_BODY, 100.0, 5.0)
    rev = _revolute(P, wid, ground, extra, (100.0, 5.0), motor=(1.0, 5.0))
    assert rev.index == slot
    _step_and_compare(P, wid, dw, O, solver, 10)
    P.s2DestroyJoint(rev)
    pri = _prismatic(P, wid, ground, extra, (100.0, 5.0), (1.0, 0.0))
    assert pri.index == slot
    _step_and_compare(P, wid, dw, O, solver, 10)
    P.s2DestroyJoint(pri)
    again = _gear(P, wid, links[0], links[1], 2.0)
    assert again.index == slot
    _step_and_compare(P, wid, dw, O, solver, 10)
    P.s2DestroyWorld(wid)


def test_teleported_static_frame(product, dev):
    """s2Body_SetTransform on the plate under the gear train moves the gears' frames with it: the rows carry the plate's new
    rotation, the constant stays, and every step after the move still equals the oracle."""
    P = product
    solver = "TGS_Soft"
    wid, gears, _, (_, plate) = _gear_world(P, solver, planets=0)
    P.s2World_Step(wid, DT, 4, 2, True)
    dw = device.DeviceWorld.attach(dev, wid)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT)
    before = dw.download_joints()
    train = [g.index for g in gears[2:5]]

    def edit(k):
        if k == 5:
            P.s2Body_SetTransform(plate, capi.Vec2(40.5, 0.2), 1.1)

    _step_and_compare(P, wid, dw, gear_oracle.load(), solver, 20, edit=edit)
    after = dw.download_joints()
    for slot in train:
        # both sides' frames turned with the plate: side 1's rotation in target, side 2's in maxMotorTorque / motorSpeed
        assert np.allclose(after["target"][slot], (np.sin(1.1), np.cos(1.1)), atol=1e-6)
        assert np.allclose((after["maxMotorTorque"][slot], after["motorSpeed"][slot]), (np.sin(1.1), np.cos(1.1)), atol=1e-6)
        assert after["lowerAngle"][slot] == before["lowerAngle"][slot]
    P.s2DestroyWorld(wid)


def test_unwound_coordinate_survives_a_reupload(product, dev):
    """The fast pair turns for 40 steps (several turns); a break-threshold edit on its gear re-uploads the row from the host:
    the unwound coordinates come back with the same bits (not reset into [-pi, pi]), and every step after still equals
    the oracle.

    Mutations it catches: a host that does not mirror lowerImpulse / upperImpulse for a gear, or a row fill that drops them."""
    P = product
    solver = "TGS_Soft"
    wid, gears, _, _ = _gear_world(P, solver, planets=0)
    P.s2World_Step(wid, DT, 4, 2, True)
    dw = device.DeviceWorld.attach(dev, wid)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT)
    O = gear_oracle.load()
    _step_and_compare(P, wid, dw, O, solver, 40)
    fast = gears[6]
    before = dw.download_joints()[fast.index]
    assert before["lowerImpulse"] > 6.0 * np.pi and before["upperImpulse"] < -6.0 * np.pi
    P.s2Joint_SetBreakForce(fast, 1e6)
    P.s2World_Flush(wid)
    after = dw.download_joints()[fast.index]
    assert after["breakForce"] == np.float32(1e6)
    for name in ("impulse", "lowerImpulse", "upperImpulse", "lowerAngle"):
        assert bit_equal(after[name], before[name]), name
    _step_and_compare(P, wid, dw, O, solver, 10)
    assert dw.download_joints()[fast.index]["lowerImpulse"] > before["lowerImpulse"]
    P.s2DestroyWorld(wid)


# ---- lifetime --------------------------------------------------------------------------------------------------------------

def test_destroy_cascade(product, dev):
    """s2DestroyJoint on a linked joint destroys the gears that link it first: joint 2 of the testbed takes both of its
    gears. Destroying those gears' now stale ids afterwards, as a teardown loop would, does nothing: the other gears keep
    their rows and still follow a frame that moves.

    Mutations it catches: a gear left behind by its joint's destruction, and a stale id destroyed twice (which would free
    the slot again and drive the live-gear count to zero, switching off the cascade and the frame updates)."""
    P = product
    wid, gears, links, (_, plate) = _gear_world(P, "TGS_Soft", planets=0)
    P.s2World_Step(wid, DT, 4, 2, True)
    P.s2DestroyJoint(links[1])
    P.s2DestroyJoint(gears[0])
    P.s2DestroyJoint(gears[1])
    P.s2Body_SetTransform(plate, capi.Vec2(40.0, 0.0), 0.9)
    rows = device.DeviceWorld.attach(dev, wid)
    P.s2World_Step(wid, DT, 4, 2, True)
    got = rows.download_joints()
    for g in gears[:2]:
        assert got["flags"][g.index] & 1 == 0
    assert all(got["flags"][g.index] & 1 == 1 for g in gears[2:])
    # the revolute joint 1 and the prismatic joint 3 are still there, and the train's gears followed the plate
    assert got["flags"][links[0].index] & 1 == 1 and got["flags"][links[2].index] & 1 == 1
    for g in gears[2:5]:
        assert np.allclose(got["target"][g.index], (np.sin(0.9), np.cos(0.9)), atol=1e-6)
    P.s2DestroyWorld(wid)


def test_broken_joint1_takes_its_gear(product, dev):
    """A joint 1 broken by its threshold is destroyed with its gear at the next step; s2World_GetBrokenJoints names only the
    joint that went over its threshold."""
    P = product
    wid = P.create_world("TGS_Soft")
    ground = _body(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    pinion = _body(P, wid, capi.DYNAMIC_BODY, 0.0, 0.0, radius=0.5)
    rack = _body(P, wid, capi.DYNAMIC_BODY, 1.0, 0.0)
    j1 = _revolute(P, wid, ground, pinion, (0.0, 0.0))
    j2 = _prismatic(P, wid, ground, rack, (1.0, 0.0), (0.0, 1.0))
    gear = _gear(P, wid, j1, j2, 2.0)
    for _ in range(5):
        P.s2World_Step(wid, DT, 4, 2, True)
    P.s2Joint_SetBreakForce(j1, 1e-3)  # the pinion's pivot carries the rack's weight
    P.s2World_Step(wid, DT, 4, 2, True)
    broken = (capi.JointId * 4)()
    assert P.s2World_GetBrokenJoints(wid, broken, 4) == 1 and broken[0].index == j1.index
    P.s2World_Step(wid, DT, 4, 2, True)
    rows = device.DeviceWorld.attach(dev, wid).download_joints()
    assert rows["flags"][j1.index] & 1 == 0 and rows["flags"][gear.index] & 1 == 0 and rows["flags"][j2.index] & 1 == 1
    P.s2DestroyWorld(wid)


# ---- input, getters, drawing --------------------------------------------------------------------------------------------------

def test_create_rejects_bad_input_and_getters(product, dev):
    """s2CreateGearJoint returns s2_nullJointId for a null, stale or foreign joint id, a joint that is not revolute or
    prismatic, a joint whose body A is not static, two joints with the same body B and a non-finite ratio; the default
    definition is 2.4's; the getters return the linked joints and the ratio, and the null id and 0 for another type; the
    row carries the gear's type bits, side flags, ratio and side 2's frame.

    Mutations it catches: any one rejection left out, a getter reading the wrong field, a type encoded in the 3-bit field
    alone, and a side flag on the wrong side."""
    P = product
    wid = P.create_world("TGS_Soft")
    other_world = P.create_world("TGS_Soft")
    ground = _body(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    a = _body(P, wid, capi.DYNAMIC_BODY, 0.0, 0.0, gravity=0.0)
    b = _body(P, wid, capi.DYNAMIC_BODY, 3.0, 0.0, gravity=0.0)
    c = _body(P, wid, capi.DYNAMIC_BODY, 6.0, 0.0, gravity=0.0)
    ja = _revolute(P, wid, ground, a, (0.0, 0.0))
    jb = _prismatic(P, wid, ground, b, (3.0, 0.0), (1.0, 0.0))
    same_b = _revolute(P, wid, ground, a, (0.5, 0.0))
    dynamic_frame = _revolute(P, wid, a, c, (6.0, 0.0))
    wd = capi.default_wheel_def()
    wd.bodyIdA, wd.bodyIdB = ground, c
    wheel = P.s2CreateWheelJoint(wid, C.byref(wd))
    stale = _revolute(P, wid, ground, c, (6.0, 0.0))
    P.s2DestroyJoint(stale)
    og = _body(P, other_world, capi.STATIC_BODY, 0.0, 0.0)
    ob = _body(P, other_world, capi.DYNAMIC_BODY, 0.0, 0.0)
    foreign = _revolute(P, other_world, og, ob, (0.0, 0.0))
    null = capi.JointId(-1, -1, 0)
    bad = [(null, jb, 1.0), (ja, null, 1.0), (stale, jb, 1.0), (ja, foreign, 1.0), (ja, wheel, 1.0), (wheel, jb, 1.0),
           (dynamic_frame, jb, 1.0), (ja, same_b, 1.0), (ja, jb, float("nan")), (ja, jb, float("inf"))]
    for j1, j2, ratio in bad:
        assert _gear(P, wid, j1, j2, ratio).index == -1, (j1.index, j2.index, ratio)  # s2_nullJointId
    d = capi.default_gear_def()
    assert (d.jointId1.index, d.jointId2.index, d.ratio, d.collideConnected) == (-1, -1, 1.0, False)
    g = _gear(P, wid, ja, jb, -2.5)
    assert g.index >= 0
    g1, g2 = P.s2GearJoint_GetJoint1(g), P.s2GearJoint_GetJoint2(g)
    assert (g1.index, g1.revision, g2.index, g2.revision) == (ja.index, ja.revision, jb.index, jb.revision)
    assert P.s2GearJoint_GetRatio(g) == -2.5
    # a joint of another type reads the null id and 0
    assert P.s2GearJoint_GetJoint1(ja).index == -1 and P.s2GearJoint_GetJoint2(ja).index == -1
    assert P.s2GearJoint_GetRatio(ja) == 0.0
    P.s2World_Step(wid, DT, 4, 2, True)
    r = device.DeviceWorld.attach(dev, wid).download_joints()[g.index]
    assert device.joint_type(int(r["flags"])) == device.JOINT_GEAR and (int(r["flags"]) >> 1) & 7 == 0
    assert r["flags"] & device.JOINT_GEAR_PRISMATIC2 and not r["flags"] & device.JOINT_GEAR_PRISMATIC1
    assert r["flags"] & (device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR | device.JOINT_ENABLE_SPRING) == 0
    assert r["referenceAngle"] == np.float32(-2.5)
    # side 2's frame: the prismatic joint's world anchor and world axis
    assert (r["maxMotorTorque"], r["motorSpeed"], r["hertz"], r["dampingRatio"]) == (3.0, 0.0, 1.0, 0.0)
    P.s2DestroyWorld(wid)
    P.s2DestroyWorld(other_world)


def test_draw_default_lines(product, dev):
    """s2World_Draw draws Box2D 2.4's default joint lines for a gear: each body's origin to its anchor, anchor to anchor."""
    P = product
    wid = P.create_world("TGS_Soft")
    ground = _body(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    a = _body(P, wid, capi.DYNAMIC_BODY, 0.0, 0.0, gravity=0.0)
    b = _body(P, wid, capi.DYNAMIC_BODY, 3.0, 1.0, gravity=0.0)
    ja = _revolute(P, wid, ground, a, (0.0, 0.0))
    jb = _prismatic(P, wid, ground, b, (3.0, 1.0), (0.0, 1.0), anchor_b=(0.2, 0.1))
    _gear(P, wid, ja, jb, 1.0)
    P.s2World_Step(wid, DT, 4, 2, True)
    pb = P.s2Body_GetPosition(b)
    segments = [v for name, v in _draw_log(P, wid) if name == "DrawSegment"]

    def drawn(p, q):
        return any(abs(v[0] - p[0]) < 1e-5 and abs(v[1] - p[1]) < 1e-5 and abs(v[2] - q[0]) < 1e-5 and abs(v[3] - q[1]) < 1e-5
                   for v in segments)

    anchor_b = (pb.x + 0.2, pb.y + 0.1)
    assert drawn((0.0, 0.0), anchor_b) and drawn((pb.x, pb.y), anchor_b)
    P.s2DestroyWorld(wid)


# ---- reactions and breaking ----------------------------------------------------------------------------------------------------

def test_reactions_and_a_gear_that_breaks(product, dev):
    """A rack hanging from a pinion held by its motor through a gear at ratio 0.5: the reaction on the rack reads its weight
    (0, m g),
    the same bits through the host getter and the device's bulk read; a break force below it snaps the gear and the rack
    falls."""
    P = product
    wid = P.create_world("TGS_Soft")
    ground = _body(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    pinion = _body(P, wid, capi.DYNAMIC_BODY, 0.0, 0.0, radius=0.5)
    rack = _body(P, wid, capi.DYNAMIC_BODY, 1.0, 0.0)
    j1 = _revolute(P, wid, ground, pinion, (0.0, 0.0), motor=(0.0, 1000.0))
    j2 = _prismatic(P, wid, ground, rack, (1.0, 0.0), (0.0, 1.0))
    g = _gear(P, wid, j1, j2, 0.5)
    for _ in range(120):
        P.s2World_Step(wid, DT, 4, 2, True)
    weight = P.s2Body_GetMass(rack) * 10.0
    f = P.s2Joint_GetReactionForce(g)
    assert f.x == 0.0 and abs(f.y - weight) <= 1e-3 * weight, (f.x, f.y, weight)
    assert P.s2Joint_GetReactionTorque(g) == 0.0
    out = np.zeros(3 * 8, dtype=np.float32)
    P.s2World_GetJointReactions(wid, out.ctypes.data, 8)
    assert (out[3 * g.index], out[3 * g.index + 1], out[3 * g.index + 2]) == (np.float32(f.x), np.float32(f.y), 0.0)
    y = P.s2Body_GetPosition(rack).y
    P.s2Joint_SetBreakForce(g, 0.5 * f.y)
    P.s2World_Step(wid, DT, 4, 2, True)
    broken = (capi.JointId * 4)()
    assert P.s2World_GetBrokenJoints(wid, broken, 4) == 1 and broken[0].index == g.index
    for _ in range(10):
        P.s2World_Step(wid, DT, 4, 2, True)
    assert P.s2Body_GetPosition(rack).y < y - 0.1  # sliding down its axis
    P.s2DestroyWorld(wid)
