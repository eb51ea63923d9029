"""GPU: the weld joint (DESIGN.md §3.8). The device's weld rows against the joint oracle (tests/joint_oracle.c) bit for bit, in
every schedule and for all ten variants; every step of scenes.welded_structures through the public API; contacts between
welded bodies; and the weld's lifecycle.

The reference has no weld. Its stand-in is the revolute joint with limits and motor off that welded_structures creates
on a library without s2CreateWeldJoint: same bodies, anchors, reference angle and collideConnected, so the reference's
collide and finalize stages see the same world. Its rows are turned into weld rows before the oracle runs.

Mutations each test catches: a missing unwind, a bias applied in the soft relax pass, lambda zeroed at prepare or a
weld row solved as a revolute fail the stage and every-step comparisons (the scene has reference angles of +-3 rad and
warm-started welds); welds left out of the contact-destroy list fail test_collide_connected."""
import ctypes as C

import numpy as np
import pytest

import joint_oracle
from helpers import (bit_equal, body_rows_from_ref, carry_sticky_friction, contact_rows_from_ref, joint_rows_from_ref,
                     load_bodies_into_ref, ref_delta_positions, store_oracle_bodies)
from oracle import ref as refmod
from solver2d_b200 import capi, device, scenes

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0
VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


def _as_welds(joints, slots):
    """Turn the stand-in revolute rows at `slots` into weld rows (type bits 1-3; no limit or motor flag)."""
    slots = np.asarray(slots, dtype=np.int64)
    assert np.all((joints["flags"][slots] & (device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR)) == 0)
    joints["flags"][slots] = (joints["flags"][slots] & ~0xE) | (device.JOINT_WELD << 1)
    return joints


def _weld_slots(sc):
    return [sc.joints[k].index for k in sc.piles["welds"]]


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

@pytest.mark.parametrize("persistent", [True, False])
@pytest.mark.parametrize("mode", ["wavefront", "color", "regions"])
@pytest.mark.parametrize("solver", VARIANTS)
def test_stage_matches_oracle(reference, dev, solver, mode, persistent):
    """One stage of welded_structures rows (welds, revolutes with limit and motor, a mouse joint, contacts), the welds
    warm-started with an angular impulse."""
    R = reference
    O = joint_oracle.load()
    sc = scenes.welded_structures(R, solver, copies=2)
    for _ in range(30):
        sc.step(DT, 4, 2, True)
    R.step_collide(sc.world)
    bodies = body_rows_from_ref(*R.bodies(sc.world))
    contacts, _ = contact_rows_from_ref(*R.contacts(sc.world))
    joints = _as_welds(joint_rows_from_ref(*R.joints(sc.world)), _weld_slots(sc))
    sc.destroy()
    welds = (joints["flags"] >> 1 & 0x7) == device.JOINT_WELD
    assert welds.sum() >= 20 and len(contacts) > 10
    assert np.any(np.abs(np.abs(joints["referenceAngle"][welds]) - 3.0) < 1e-6)
    joints["motorImpulse"][welds] = np.random.default_rng(3).uniform(-0.2, 0.2, int(welds.sum())).astype(np.float32)
    ctx = device.make_context(solver, DT, 4, 2)

    dw = dev.create_world(capi.SOLVER[solver])
    dw.upload_bodies(bodies, len(bodies))
    dw.upload_joints(joints, len(joints))
    dw.upload_contacts(contacts)
    dw.set_schedule(device.SCHEDULE_WAVEFRONT if mode == "wavefront" else device.SCHEDULE_COLOR)
    dw.set_regions(2 if mode == "regions" else 0)
    dw.set_persistent(persistent)
    dw.solve(ctx)
    got = dw.download_all_bodies(len(bodies))
    got_contacts = dw.download_contacts(len(contacts))
    got_joints = dw.download_joints(len(joints))
    order, _ = dw.solve_order(len(contacts) + len(joints))
    dw.destroy()
    ob, oc, oj = O.solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, order=None if mode == "wavefront" else order)
    _compare(got, got_contacts, got_joints, ob, oc, oj, bodies, contacts)
    # the welds did work: a weld solved as a revolute would leave motorImpulse where prepare put it
    if solver != "XPBD":
        assert np.any(oj["motorImpulse"][welds] != joints["motorImpulse"][welds])


# ---- every step through the public API -----------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", VARIANTS)
def test_welded_structures_every_step(reference, product, dev, solver):
    """Reference collide on the stand-in world, the weld oracle in the device's order, reference finalize; the device runs
    the same steps through s2World_Step with real welds. Every step bit for bit: bodies, contact and joint impulses."""
    R, P = reference, product
    O = joint_oracle.load()
    sr = scenes.welded_structures(R, solver)
    sp = scenes.welded_structures(P, solver)
    assert "s2CreateWeldJoint" in R.missing and "s2CreateWeldJoint" not in P.missing
    slots = _weld_slots(sp)
    assert slots == _weld_slots(sr)
    # push the freshly built scene to the device now, so that the first step starts from it like any other
    dev.lib.s2World_Flush.restype = None
    dev.lib.s2World_Flush.argtypes = [capi.WorldId]
    dev.lib.s2World_Flush(sp.world)
    dw = device.DeviceWorld.attach(dev, sp.world)
    ctx = device.make_context(solver, DT, 4, 2, True)
    sticky = solver == "TGS_Sticky"
    solved = {}
    F = refmod.BODY_F
    contacts_seen = 0
    for step in range(60):
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
        got_contacts = dw.download_contacts(len(rows_key) + 64)
        assert len(got_contacts) == len(rows_key) and np.array_equal(got_contacts["shapeA"], rows_key["shapeA"]), step
        contacts_seen += len(rows_key)

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
    assert contacts_seen > 100
    sp.destroy()
    sr.destroy()


# ---- contacts between welded bodies -------------------------------------------------------------------------------------

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


def _create_weld(L, wid, a, b, collide):
    if "s2CreateWeldJoint" in L.missing:
        jd = capi.default_revolute_def()
        fn = L.s2CreateRevoluteJoint
    else:
        jd = capi.default_weld_def()
        fn = L.s2CreateWeldJoint
    jd.bodyIdA, jd.bodyIdB = a, b
    jd.localAnchorA = capi.Vec2(0.4, 0.0)
    jd.localAnchorB = capi.Vec2(-0.4, 0.0)
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
    """Two overlapping boxes: the weld removes their contact unless collideConnected, and no new one forms while it lives;
    destroying the weld lets the pair come back. The pair table matches the reference's stand-in every step."""
    R, P = reference, product
    wr, _, br = _overlapping_pair(R, "TGS_Soft")
    wp, _, bp = _overlapping_pair(P, "TGS_Soft")
    dw = device.DeviceWorld.attach(dev, wp)
    pair = (bp[0].index, bp[1].index)
    for _ in range(3):
        R.s2World_Step(wr, DT, 4, 2, True)
        P.s2World_Step(wp, DT, 4, 2, True)
    assert pair in _pairs_dev(dw)
    jr = _create_weld(R, wr, br[0], br[1], collide)
    jp = _create_weld(P, wp, bp[0], bp[1], collide)
    dev.lib.s2World_Flush.restype = None
    dev.lib.s2World_Flush.argtypes = [capi.WorldId]
    dev.lib.s2World_Flush(wp)
    rows = dw.download_joints(1)
    assert (rows["flags"][0] >> 1 & 0x7) == device.JOINT_WELD
    assert bool(rows["flags"][0] & device.JOINT_COLLIDE_CONNECTED) == collide
    back = None
    for step in range(80):
        if step == 20:
            R.s2DestroyJoint(jr)
            P.s2DestroyJoint(jp)
            # the broad phase looks for new pairs only among proxies that moved out of their fat boxes: toss one box up so
            # that it lands on the other again
            for L, b in ((R, br[1]), (P, bp[1])):
                L.s2Body_SetLinearVelocity(b, capi.Vec2(0.0, 3.0))
        R.s2World_Step(wr, DT, 4, 2, True)
        P.s2World_Step(wp, DT, 4, 2, True)
        pairs = _pairs_dev(dw)
        assert pairs == _pairs_ref(R, wr), step
        if step < 20:
            assert (pair in pairs) == collide, step
        elif back is None and pair in pairs:
            back = step
    assert back is not None, "the pair did not come back after the weld was destroyed"
    R.s2DestroyWorld(wr)
    P.s2DestroyWorld(wp)


# ---- lifecycle ----------------------------------------------------------------------------------------------------------

def test_slot_reuse_and_destroy(product, dev):
    """A weld slot is reused by a revolute joint and the other way round, and the downloaded row carries the right type
    and flags each time; destroying a weld and then its bodies leaves no joint behind."""
    P = product
    wid, gid, (a, b) = _overlapping_pair(P, "TGS_Soft")
    dw = device.DeviceWorld.attach(dev, wid)

    def row(j):
        P.s2World_Step(wid, DT, 4, 2, True)
        return dw.download_joints(j.index + 1)[j.index]

    w = _create_weld(P, wid, a, b, False)
    r = row(w)
    assert (r["flags"] >> 1 & 0x7) == device.JOINT_WELD and r["flags"] & (device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR) == 0
    P.s2DestroyJoint(w)
    jd = capi.default_revolute_def()
    jd.bodyIdA, jd.bodyIdB = a, b
    jd.enableLimit, jd.enableMotor = True, True
    jd.lowerAngle, jd.upperAngle, jd.maxMotorTorque = -0.1, 0.1, 1.0
    rv = P.s2CreateRevoluteJoint(wid, C.byref(jd))
    assert rv.index == w.index
    r = row(rv)
    assert (r["flags"] >> 1 & 0x7) == device.JOINT_REVOLUTE
    assert r["flags"] & device.JOINT_ENABLE_LIMIT and r["flags"] & device.JOINT_ENABLE_MOTOR
    P.s2DestroyJoint(rv)
    w2 = _create_weld(P, wid, a, b, True)
    assert w2.index == w.index
    r = row(w2)
    assert (r["flags"] >> 1 & 0x7) == device.JOINT_WELD and r["flags"] & device.JOINT_COLLIDE_CONNECTED
    assert r["flags"] & (device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR) == 0
    P.s2DestroyJoint(w2)
    P.s2DestroyBody(a)
    P.s2DestroyBody(b)
    for _ in range(3):
        P.s2World_Step(wid, DT, 4, 2, True)
    assert P.s2World_GetStatistics(wid).jointCount == 0
    assert (dw.download_joints(w.index + 1)["flags"] & 1).sum() == 0
    P.s2DestroyWorld(wid)
