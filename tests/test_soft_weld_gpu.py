"""GPU: soft welds (DESIGN.md §3.15). The device's soft weld rows against the soft weld oracle (tests/soft_weld_oracle.c) bit
for bit, in every schedule, for all ten variants, persistent and launch by launch, with the warm-start gather on and off;
every step of scenes.soft_welds (a donut of capsules on angular springs dropped on a pile, soft and rigid cantilevers, a
box hanging on a linear spring, a box on a kinematic platform, contacts throughout) through the public API against
reference collide and finalize around the soft weld oracle in the device's order, with the kinematic platform and XPBD's
delta positions carried; a contact-free world stepped against the oracle alone; setter edits between replayed steps; slot
reuse; input checks; reactions that include the springs' loads and a break threshold that a soft weld's load trips.

Mutations each test catches: a coefficient formed with another h or expression order, a soft part solved with the rigid
form (or a rigid part with the soft one), the lanes of the two parts swapped, XPBD's start pose read from the wrong column,
a soft part corrected by the NGS position pass, and a marker left on a rigid weld all fail the stage and every-step
comparisons; a reaction that leaves a soft part's impulse out fails the reaction test."""
import ctypes as C
import math

import numpy as np
import pytest

import soft_weld_oracle
import weld_oracle
from helpers import (bit_equal, body_rows_from_ref, carry_sticky_friction, contact_rows_from_ref, joint_rows_from_ref,
                     load_bodies_into_ref, ref_delta_positions, store_oracle_bodies)
from oracle import ref as refmod
from solver2d_b200 import capi, device, scenes
from test_prismatic_gpu import _flush
from test_weld_gpu import _as_welds, _weld_slots

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


def _set_soft(joints, slot, linear, angular):
    """A weld row's soft parts, in the lanes it carries them in."""
    joints["hertz"][slot], joints["dampingRatio"][slot] = linear
    joints["maxMotorTorque"][slot], joints["motorSpeed"][slot] = angular


# ---- one solver stage against the oracle --------------------------------------------------------------------------------

@pytest.mark.parametrize("gather", [True, False])
@pytest.mark.parametrize("persistent", [True, False])
@pytest.mark.parametrize("mode", ["wavefront", "color", "regions"])
@pytest.mark.parametrize("solver", VARIANTS)
def test_stage_matches_oracle(reference, dev, solver, mode, persistent, gather):
    """One stage of soft_welds rows with random soft parts on the welds (some rigid, some linear-only, some angular-only,
    some both; random warm-start impulses), beside rigid welds, revolute and mouse joints and contacts."""
    if not gather and solver not in SUBSTEPPING:
        pytest.skip("the warm-start gather serves the sub-stepping variants only")
    R = reference
    sc = scenes.soft_welds(R, solver, copies=2)
    for _ in range(30):
        sc.step(DT, 4, 2, True)
    R.step_collide(sc.world)
    bodies = body_rows_from_ref(*R.bodies(sc.world))
    contacts, _ = contact_rows_from_ref(*R.contacts(sc.world))
    joints = _as_welds(joint_rows_from_ref(*R.joints(sc.world)), _weld_slots(sc))
    sc.destroy()
    welds = np.flatnonzero((joints["flags"] & 1 == 1) & ((joints["flags"] >> 1 & 0x7) == device.JOINT_WELD))
    assert len(welds) >= 30 and len(contacts) > 10
    rng = np.random.default_rng(17)
    kinds = rng.integers(0, 4, len(welds))  # 0 rigid, 1 linear only, 2 angular only, 3 both
    for slot, kind in zip(welds, kinds):
        linear = (rng.uniform(0.5, 8.0), rng.uniform(0.0, 1.5)) if kind in (1, 3) else (0.0, rng.uniform(0.0, 1.0))
        angular = (rng.uniform(0.5, 8.0), rng.uniform(0.0, 1.5)) if kind in (2, 3) else (0.0, rng.uniform(0.0, 1.0))
        _set_soft(joints, slot, linear, angular)
    joints["impulse"][welds] = rng.uniform(-0.2, 0.2, (len(welds), 2)).astype(np.float32)
    joints["motorImpulse"][welds] = rng.uniform(-0.2, 0.2, len(welds)).astype(np.float32)
    assert set(kinds.tolist()) == {0, 1, 2, 3}
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
    ob, oc, oj = soft_weld_oracle.load().solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, order=order)
    valid = (bodies["flags"] & 1) == 1
    _compare_bodies(got, ob, valid)
    _compare_joints(got_joints, oj)
    live = contacts["pointCount"] > 0
    assert bit_equal(got_contacts["points"]["normalImpulse"][live], oc["points"]["normalImpulse"][live])
    # the soft parts did work: the weld oracle, which reads no hertz, ends elsewhere
    wb, _, _ = weld_oracle.load().solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, order=order)
    assert not bit_equal(wb["position"][valid], ob["position"][valid])


# ---- a world through the public API, every step ---------------------------------------------------------------------------

def _soft_slots(sc):
    return [(sc.joints[k].index,) + tuple(v) for k, *v in sc.piles["soft_welds"]]


@pytest.mark.parametrize("solver", VARIANTS)
def test_soft_welds_scene_every_step(reference, product, dev, solver):
    """scenes.soft_welds: reference collide on the stand-in world, the soft weld oracle in the device's order, reference
    finalize; the device runs the same steps through s2World_Step with real soft welds. Every step bit for bit: bodies,
    delta positions, contact impulses and joint impulses."""
    R, P = reference, product
    O = soft_weld_oracle.load()
    sr = scenes.soft_welds(R, solver)
    sp = scenes.soft_welds(P, solver)
    assert "s2CreateWeldJoint" in R.missing and "s2CreateWeldJoint" not in P.missing
    slots = _weld_slots(sp)
    soft = _soft_slots(sp)
    assert slots == _weld_slots(sr) and soft == _soft_slots(sr) and len(soft) == 14
    _flush(dev, sp.world)
    dw = device.DeviceWorld.attach(dev, sp.world)
    rows = dw.download_joints(len(sp.joints))
    for slot, lh, lz, ah, az in soft:
        assert (rows["hertz"][slot], rows["dampingRatio"][slot]) == (np.float32(lh), np.float32(lz))
        assert (rows["maxMotorTorque"][slot], rows["motorSpeed"][slot]) == (np.float32(ah), np.float32(az))
    ctx = device.make_context(solver, DT, 4, 2, True)
    sticky = solver == "TGS_Sticky"
    solved = {}
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
        joints = _as_welds(joint_rows_from_ref(*R.joints(sr.world)), slots)
        for slot, lh, lz, ah, az in soft:
            _set_soft(joints, slot, (lh, lz), (ah, az))
        got_contacts = dw.download_contacts(len(rows_key) + 64)
        assert len(got_contacts) == len(rows_key) and np.array_equal(got_contacts["shapeA"], rows_key["shapeA"]), step
        contacts_seen += int(np.count_nonzero(rows_key["pointCount"]))

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
        # the stand-in's motorImpulse column carries the weld's angular impulse into the next step
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
        for name in ("impulse", "motorImpulse"):
            assert bit_equal(gj[name][jv], oj[name][jv]), f"step {step}: joint {name}"
    assert contacts_seen > 500
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


def _weld(P, wid, a, b, anchor_a, anchor_b, ref=0.0, linear=(0.0, 0.0), angular=(0.0, 0.0)):
    jd = capi.default_weld_def()
    jd.bodyIdA, jd.bodyIdB = a, b
    jd.localAnchorA, jd.localAnchorB = capi.Vec2(*anchor_a), capi.Vec2(*anchor_b)
    jd.referenceAngle = ref
    jd.linearHertz, jd.linearDampingRatio = linear
    jd.angularHertz, jd.angularDampingRatio = angular
    return P.s2CreateWeldJoint(wid, C.byref(jd))


def _soft_weld_world(P, solver):
    """Bodies far apart (no contacts): a hanging chain of soft welds (both parts), a box on a linear-only soft weld, an
    angular-only soft weld whose rest angle sits at the seam, a soft weld to a kinematic carriage, a rigid weld, a revolute
    joint and a mouse joint."""
    wid = P.create_world(solver)
    ground = _box(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    joints = []
    prev = ground
    for k in range(4):  # soft chain hanging from the ground
        b = _box(P, wid, capi.DYNAMIC_BODY, 0.6 * (k + 1), 10.0, w=0.5 * k)
        joints.append(_weld(P, wid, prev, b, (0.3, 10.0) if k == 0 else (0.3, 0.0), (-0.3, 0.0), linear=(6.0, 0.5),
                            angular=(2.0, 0.3)))
        prev = b
    hanging = _box(P, wid, capi.DYNAMIC_BODY, 20.0, 4.0, w=1.0)
    joints.append(_weld(P, wid, ground, hanging, (20.0, 4.5), (0.0, 0.5), linear=(2.0, 0.1)))
    seam = _box(P, wid, capi.DYNAMIC_BODY, 40.0, 5.0, angle=-math.pi + 0.05, gravity=0.0)
    joints.append(_weld(P, wid, ground, seam, (40.0, 5.0), (0.0, 0.0), ref=math.pi - 0.05, angular=(3.0, 0.2)))
    carriage = _box(P, wid, capi.KINEMATIC_BODY, 60.0, 5.0, vx=0.7, w=0.2)
    rider = _box(P, wid, capi.DYNAMIC_BODY, 61.0, 5.0, gravity=0.0)
    joints.append(_weld(P, wid, carriage, rider, (0.5, 0.0), (-0.5, 0.0), linear=(1.5, 0.1), angular=(1.0, 0.0)))
    rigid = _box(P, wid, capi.DYNAMIC_BODY, 70.0, 5.0, w=0.3)
    joints.append(_weld(P, wid, rider, rigid, (0.5, 0.0), (-8.5, 0.0), ref=0.2))
    swing = _box(P, wid, capi.DYNAMIC_BODY, 75.6, 5.0)
    jd = capi.default_revolute_def()
    jd.bodyIdA, jd.bodyIdB = ground, swing
    jd.localAnchorA, jd.localAnchorB = capi.Vec2(75.0, 5.0), capi.Vec2(-0.6, 0.0)
    joints.append(P.s2CreateRevoluteJoint(wid, C.byref(jd)))
    dragged = _box(P, wid, capi.DYNAMIC_BODY, 80.0, 5.0)
    md = capi.MouseJointDef()
    md.bodyIdA, md.bodyIdB = ground, dragged
    md.target = capi.Vec2(80.5, 5.5)
    md.hertz, md.dampingRatio = 4.0, 0.7
    joints.append(P.s2CreateMouseJoint(wid, C.byref(md)))
    return wid, joints, (ground, hanging)


@pytest.mark.parametrize("solver", VARIANTS)
def test_public_world_every_step(product, dev, solver):
    """Each s2World_Step equals the soft weld oracle's stage on the rows the step started from, bit for bit, delta positions
    included (a kinematic body's grows under XPBD)."""
    P = product
    wid, _, _ = _soft_weld_world(P, solver)
    P.s2World_Step(wid, DT, 4, 2, True)  # uploads the world
    dw = device.DeviceWorld.attach(dev, wid)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT)
    O = soft_weld_oracle.load()
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
    """Soft parts retuned, made rigid and made soft again between steps land in the next step's rows (replayed solve graph),
    and each step still equals the oracle."""
    P = product
    wid, joints, _ = _soft_weld_world(P, solver)
    P.s2World_Step(wid, DT, 4, 2, True)
    dw = device.DeviceWorld.attach(dev, wid)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT)
    O = soft_weld_oracle.load()
    ctx = device.make_context(solver, DT, 4, 2)
    chain, hanging, rigid = joints[1], joints[4], joints[7]
    edits = {5: lambda: P.s2WeldJoint_SetLinearHertz(chain, 9.0),
             10: lambda: P.s2WeldJoint_SetAngularDampingRatio(chain, 0.05),
             15: lambda: (P.s2WeldJoint_SetLinearHertz(hanging, 0.0), P.s2WeldJoint_SetAngularHertz(rigid, 3.0)),
             20: lambda: P.s2WeldJoint_SetAngularHertz(chain, 0.0),
             25: lambda: (P.s2WeldJoint_SetLinearHertz(hanging, 4.0), P.s2WeldJoint_SetLinearDampingRatio(hanging, 1.0))}
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
    assert (r["hertz"][chain.index], r["maxMotorTorque"][chain.index]) == (np.float32(9.0), 0.0)
    assert r["motorSpeed"][chain.index] == np.float32(0.05)
    assert (r["hertz"][hanging.index], r["dampingRatio"][hanging.index]) == (np.float32(4.0), np.float32(1.0))
    assert r["maxMotorTorque"][rigid.index] == np.float32(3.0)
    assert (P.s2WeldJoint_GetLinearHertz(chain), P.s2WeldJoint_GetAngularHertz(chain)) == (9.0, 0.0)
    assert P.s2WeldJoint_GetAngularDampingRatio(chain) == np.float32(0.05)
    assert P.s2WeldJoint_GetLinearDampingRatio(hanging) == 1.0
    P.s2DestroyWorld(wid)


def test_slot_reuse_across_types(product, dev):
    """A slot freed by a soft weld and taken by a revolute joint between the same bodies at the same anchor gives the
    revolute's own bits: its row carries none of the weld's soft lanes and each step equals the oracle's. The slot freed
    again and taken by a prismatic joint carries none either (the soft weld oracle has no prismatic rows, so that step is
    checked by its row only)."""
    P = product
    wid, joints, (a, b) = _soft_weld_world(P, "TGS_Soft")
    for _ in range(5):
        P.s2World_Step(wid, DT, 4, 2, True)
    dw = device.DeviceWorld.attach(dev, wid)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT)
    O = soft_weld_oracle.load()
    ctx = device.make_context("TGS_Soft", DT, 4, 2)
    slot = joints[4].index
    P.s2DestroyJoint(joints[4])
    jd = capi.default_revolute_def()
    jd.bodyIdA, jd.bodyIdB = a, b
    jd.localAnchorA, jd.localAnchorB = capi.Vec2(20.0, 4.5), capi.Vec2(0.0, 0.5)
    rj = P.s2CreateRevoluteJoint(wid, C.byref(jd))
    assert rj.index == slot
    _flush(dev, wid)
    r = dw.download_joints()[slot]
    assert (r["flags"] >> 1 & 0x7) == device.JOINT_REVOLUTE
    assert (r["hertz"], r["dampingRatio"], r["maxMotorTorque"], r["motorSpeed"]) == (0.0, 0.0, 0.0, 0.0)
    assert r["impulse"][0] == 0.0 and r["motorImpulse"] == 0.0
    for _ in range(5):
        bodies, rows, dp = dw.download_all_bodies(), dw.download_joints(), dw.download_delta_positions()
        P.s2World_Step(wid, DT, 4, 2, True)
        ob, _, oj, _ = O.solve(capi.SOLVER["TGS_Soft"], bodies, np.zeros(0, dtype=device.CONTACT_ROW), rows, ctx, dp=dp)
        _compare_bodies(dw.download_all_bodies(), ob, (bodies["flags"] & 1) == 1)
        _compare_joints(dw.download_joints(), oj)
    P.s2DestroyJoint(rj)
    pd = capi.default_prismatic_def()
    pd.bodyIdA, pd.bodyIdB = a, b
    pd.localAnchorA, pd.localAnchorB = capi.Vec2(20.0, 4.5), capi.Vec2(0.0, 0.5)
    pd.localAxisA = capi.Vec2(0.0, 1.0)
    pj = P.s2CreatePrismaticJoint(wid, C.byref(pd))
    assert pj.index == slot
    P.s2World_Step(wid, DT, 4, 2, True)
    r = dw.download_joints()[slot]
    assert (r["flags"] >> 1 & 0x7) == device.JOINT_PRISMATIC
    assert (r["hertz"], r["dampingRatio"], r["maxMotorTorque"], r["motorSpeed"]) == (0.0, 0.0, 0.0, 0.0)
    assert np.isfinite(dw.download_all_bodies()["position"]).all()
    P.s2DestroyWorld(wid)


def test_create_and_setters_reject_bad_input(product, dev):
    P = product
    wid = P.create_world("TGS_Soft")
    a = _box(P, wid, capi.STATIC_BODY, 0.0, 0.0)
    b = _box(P, wid, capi.DYNAMIC_BODY, 0.0, 2.0)
    bad_values = (-1.0, math.nan, math.inf, -math.inf)
    for field in ("linearHertz", "linearDampingRatio", "angularHertz", "angularDampingRatio"):
        for bad in bad_values:
            jd = capi.default_weld_def()
            jd.bodyIdA, jd.bodyIdB = a, b
            setattr(jd, field, bad)
            j = P.s2CreateWeldJoint(wid, C.byref(jd))
            assert (j.index, j.world, j.revision) == (-1, -1, 0), (field, bad)
    assert P.s2World_GetStatistics(wid).jointCount == 0
    wj = _weld(P, wid, a, b, (0.0, 2.0), (0.0, 0.0), linear=(2.0, 0.5), angular=(3.0, 0.25))
    jd = capi.default_revolute_def()
    jd.bodyIdA, jd.bodyIdB = a, b
    rj = P.s2CreateRevoluteJoint(wid, C.byref(jd))
    for bad in bad_values:
        P.s2WeldJoint_SetLinearHertz(wj, bad)
        P.s2WeldJoint_SetLinearDampingRatio(wj, bad)
        P.s2WeldJoint_SetAngularHertz(wj, bad)
        P.s2WeldJoint_SetAngularDampingRatio(wj, bad)
    # a joint of another type is ignored
    P.s2WeldJoint_SetLinearHertz(rj, 5.0)
    P.s2WeldJoint_SetAngularHertz(rj, 5.0)
    P.s2World_Step(wid, DT, 4, 2, True)
    rows = device.DeviceWorld.attach(dev, wid).download_joints()
    assert (rows["hertz"][wj.index], rows["dampingRatio"][wj.index]) == (np.float32(2.0), np.float32(0.5))
    assert (rows["maxMotorTorque"][wj.index], rows["motorSpeed"][wj.index]) == (np.float32(3.0), np.float32(0.25))
    assert (rows["hertz"][rj.index], rows["maxMotorTorque"][rj.index]) == (0.0, 0.0)
    assert (P.s2WeldJoint_GetLinearHertz(wj), P.s2WeldJoint_GetLinearDampingRatio(wj)) == (2.0, 0.5)
    assert (P.s2WeldJoint_GetAngularHertz(wj), P.s2WeldJoint_GetAngularDampingRatio(wj)) == (3.0, 0.25)
    assert P.s2WeldJoint_GetLinearHertz(rj) == 0.0
    P.s2DestroyWorld(wid)


# ---- reactions and break thresholds ---------------------------------------------------------------------------------------

def _rate(solver):
    ctx = device.make_context(solver, DT, 4, 2, True)
    return np.float32(ctx.inv_dt if solver == "TGS_Sticky" else ctx.inv_h)


@pytest.mark.parametrize("solver", ["TGS_Soft", "PGS", "TGS_NGS", "TGS_Sticky", "PGS_NGS_Block"])
def test_reactions_include_the_springs(product, dev, solver):
    """The getters and the bulk read equal s2ComputeJointReaction on the downloaded rows: a soft weld's impulse columns are
    the weld's, so its reaction is its springs' load. The hanging box reads its weight and its centripetal pull."""
    P = product
    wid, joints, _ = _soft_weld_world(P, solver)
    for _ in range(20):
        P.s2World_Step(wid, DT, 4, 2, True)
    dw = device.DeviceWorld.attach(dev, wid)
    rows = dw.download_joints()
    bodies = dw.download_all_bodies()
    bulk = np.zeros((len(rows), 3), dtype=np.float32)
    dw.L.s2b_download_joint_reactions(dw.h, bulk.ctypes.data, len(rows))
    loaded = 0
    for j in joints:
        r = rows[j.index]
        q = bodies["rot"][int(r["bodyA"])]
        x = P.s2ComputeJointReaction((int(r["flags"]) >> 1) & 7, capi.Vec2(*r["impulse"]), float(r["motorImpulse"]),
                                     float(r["lowerImpulse"]), float(r["upperImpulse"]), capi.Rot(float(q[0]), float(q[1])),
                                     capi.Vec2(*r["localAxisA"]), float(_rate(solver)))
        f, t = P.s2Joint_GetReactionForce(j), P.s2Joint_GetReactionTorque(j)
        assert (np.float32(f.x), np.float32(f.y), np.float32(t)) == (np.float32(x.force.x), np.float32(x.force.y),
                                                                     np.float32(x.torque))
        assert bit_equal(bulk[j.index], np.array([x.force.x, x.force.y, x.torque], dtype=np.float32))
        loaded += int(abs(f.x) + abs(f.y) + abs(t) > 0.0)
    assert loaded >= 7
    # the first chain weld carries the chain's weight (four 0.24 kg boxes, g = 10) through its springs
    fy = P.s2Joint_GetReactionForce(joints[0]).y
    assert 0.25 * 9.6 < fy < 4.0 * 9.6
    P.s2DestroyWorld(wid)


def test_soft_weld_load_trips_a_break_threshold(product, dev):
    """A stiff angular spring twisted far from its rest angle: its torque passes the threshold and the joint is destroyed by
    the next step; a soft weld with a weak spring stays."""
    P = product
    kept = []
    for hertz in (8.0, 0.2):
        wid = P.create_world("TGS_Soft")
        a = _box(P, wid, capi.STATIC_BODY, 0.0, 0.0)
        b = _box(P, wid, capi.DYNAMIC_BODY, 0.0, 0.0, angle=1.0, gravity=0.0)
        j = _weld(P, wid, a, b, (0.0, 0.0), (0.0, 0.0), angular=(hertz, 0.5))
        P.s2Joint_SetBreakTorque(j, 0.5)
        P.s2World_Step(wid, DT, 4, 2, True)
        torque = P.s2Joint_GetReactionTorque(j)
        P.s2World_Step(wid, DT, 4, 2, True)
        kept.append(P.s2World_GetStatistics(wid).jointCount)
        if hertz > 1.0:
            assert abs(torque) > 0.5
        P.s2DestroyWorld(wid)
    assert kept == [0, 1]
