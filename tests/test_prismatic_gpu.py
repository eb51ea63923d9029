"""GPU: the prismatic joint (DESIGN.md §3.9). The device's prismatic rows against the joint oracle
(tests/joint_oracle.c) bit for bit, in every schedule, for all ten variants and with the warm-start gather on and off;
every step of scenes.sliders through the public API; parameter edits between replayed steps; contacts between jointed
bodies; the joint's lifecycle, input checks, translation getter and debug drawing.

The reference has no prismatic joint. Its stand-in is the revolute joint with limits and motor off that sliders creates on a
library without s2CreatePrismaticJoint: same bodies, anchors, reference angle and collideConnected, so the reference's
collide and finalize stages see the same world. Its rows are turned into prismatic rows before the oracle runs.

Mutations each test catches: a prismatic row solved as a revolute (the check against the plain oracle), a missing axis in
the upload, a gather term of the revolute's shape, the revolute's upper-limit quirk or a dropped impulse at prepare fail
the stage and every-step comparisons; prismatic joints left out of the contact-destroy list fail test_collide_connected."""
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


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


def _unit(axis):
    """The host's normalization (s2CreatePrismaticJoint) in float32: v / sqrtf(v.x * v.x + v.y * v.y)."""
    x, y = np.float32(axis[0]), np.float32(axis[1])
    length = np.sqrt(np.float32(x * x + y * y))
    return np.array([x / length, y / length], dtype=np.float32)


def _as_prismatic(joints, slots, defs):
    """Turn the stand-in revolute rows at `slots` into the prismatic rows `defs` describe."""
    for slot, d in zip(slots, defs):
        r = joints[slot]
        assert r["flags"] & (device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR) == 0
        flags = (int(r["flags"]) & ~0xE) | (device.JOINT_PRISMATIC << 1)
        flags |= device.JOINT_ENABLE_LIMIT if d["enableLimit"] else 0
        flags |= device.JOINT_ENABLE_MOTOR if d["enableMotor"] else 0
        joints["flags"][slot] = flags
        joints["lowerAngle"][slot] = d["lowerTranslation"]
        joints["upperAngle"][slot] = d["upperTranslation"]
        joints["maxMotorTorque"][slot] = d["maxMotorForce"]
        joints["motorSpeed"][slot] = d["motorSpeed"]
        joints["referenceAngle"][slot] = d["referenceAngle"]
        joints["localAxisA"][slot] = _unit(d["localAxisA"])
    return joints


def _slots(sc):
    return [sc.joints[k].index for k in sc.piles["prismatic"]]


def _compare(got, got_contacts, got_joints, ob, oc, oj, bodies, contacts):
    valid = (bodies["flags"] & 1) == 1
    for name in ("position", "rot", "linearVelocity", "angularVelocity"):
        assert bit_equal(got[name][valid], ob[name][valid]), name
    live = contacts["pointCount"] > 0
    for name in ("normalImpulse", "tangentImpulse"):
        assert bit_equal(got_contacts["points"][name][live], oc["points"][name][live]), name
    jv = (oj["flags"] & 1) == 1
    for name in ("impulse", "motorImpulse", "lowerImpulse", "upperImpulse", "localAxisA"):
        assert bit_equal(got_joints[name][jv], oj[name][jv]), name


# ---- one solver stage against the oracle --------------------------------------------------------------------------------

@pytest.mark.parametrize("gather", [True, False])
@pytest.mark.parametrize("persistent", [True, False])
@pytest.mark.parametrize("mode", ["wavefront", "color", "regions"])
@pytest.mark.parametrize("solver", VARIANTS)
def test_stage_matches_oracle(reference, dev, solver, mode, persistent, gather):
    """One stage of sliders rows (prismatic joints with limits and motors, revolute cranks, a mouse joint, contacts), the
    prismatic joints warm-started with random impulses in every column."""
    if not gather and solver not in SUBSTEPPING:
        pytest.skip("the warm-start gather serves the sub-stepping variants only")
    R = reference
    O = joint_oracle.load()
    sc = scenes.sliders(R, solver, copies=2)
    for _ in range(30):
        sc.step(DT, 4, 2, True)
    R.step_collide(sc.world)
    bodies = body_rows_from_ref(*R.bodies(sc.world))
    contacts, _ = contact_rows_from_ref(*R.contacts(sc.world))
    joints = _as_prismatic(joint_rows_from_ref(*R.joints(sc.world)), _slots(sc), sc.piles["prismatic_defs"])
    sc.destroy()
    prism = (joints["flags"] >> 1 & 0x7) == device.JOINT_PRISMATIC
    assert prism.sum() >= 16 and len(contacts) > 10
    rng = np.random.default_rng(5)
    n = int(prism.sum())
    joints["impulse"][prism] = rng.uniform(-0.2, 0.2, (n, 2)).astype(np.float32)
    joints["motorImpulse"][prism] = rng.uniform(-0.1, 0.1, n).astype(np.float32)
    joints["lowerImpulse"][prism] = rng.uniform(0.0, 0.1, n).astype(np.float32)
    joints["upperImpulse"][prism] = rng.uniform(0.0, 0.1, n).astype(np.float32)
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
    # the prismatic rows did work: the plain oracle, which solves an unknown joint type as a revolute, ends elsewhere
    pb, _, _ = port.load().solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, order=order)
    valid = (bodies["flags"] & 1) == 1
    assert not bit_equal(pb["position"][valid], ob["position"][valid])


# ---- every step through the public API -----------------------------------------------------------------------------------

def _flush(dev, world):
    dev.lib.s2World_Flush.restype = None
    dev.lib.s2World_Flush.argtypes = [capi.WorldId]
    dev.lib.s2World_Flush(world)


@pytest.mark.parametrize("solver", VARIANTS)
def test_sliders_every_step(reference, product, dev, solver):
    """Reference collide on the stand-in world, the prismatic oracle in the device's order, reference finalize; the device
    runs the same steps through s2World_Step with real prismatic joints. Every step bit for bit: bodies, contact and joint
    impulses."""
    R, P = reference, product
    O = joint_oracle.load()
    sr = scenes.sliders(R, solver)
    sp = scenes.sliders(P, solver)
    assert "s2CreatePrismaticJoint" in R.missing and "s2CreatePrismaticJoint" not in P.missing
    slots = _slots(sp)
    assert slots == _slots(sr)
    _flush(dev, sp.world)
    dw = device.DeviceWorld.attach(dev, sp.world)
    rows = dw.download_joints(max(slots) + 1)
    assert bit_equal(rows["localAxisA"][slots], np.array([_unit(d["localAxisA"]) for d in sp.piles["prismatic_defs"]]))
    ctx = device.make_context(solver, DT, 4, 2, True)
    sticky = solver == "TGS_Sticky"
    solved = {}
    F = refmod.BODY_F
    contacts_seen = 0
    limits_hit = 0
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
        joints = _as_prismatic(joint_rows_from_ref(*R.joints(sr.world)), slots, sr.piles["prismatic_defs"])
        got_contacts = dw.download_contacts(len(rows_key) + 64)
        assert len(got_contacts) == len(rows_key) and np.array_equal(got_contacts["shapeA"], rows_key["shapeA"]), step
        contacts_seen += len(rows_key)

        order, _ = dw.solve_order(len(rows_key) + len(joints) + 16, max_groups=200000)
        ob, oc, oj, odp = O.solve(capi.SOLVER[solver], bodies, rows_key, joints, ctx, order=order,
                                  dp=ref_delta_positions(R, sr.world))
        limits_hit += int(np.count_nonzero(oj["lowerImpulse"][slots]) + np.count_nonzero(oj["upperImpulse"][slots]))

        store_oracle_bodies(R, sr.world, ob, odp)
        imp = np.zeros((cf.shape[0], 4), dtype=np.float32)
        imp[cslots[perm], 0] = oc["points"]["normalImpulse"][:, 0]
        imp[cslots[perm], 1] = oc["points"]["tangentImpulse"][:, 0]
        imp[cslots[perm], 2] = oc["points"]["normalImpulse"][:, 1]
        imp[cslots[perm], 3] = oc["points"]["tangentImpulse"][:, 1]
        R.load_contact_impulses(sr.world, imp)
        if sticky:
            solved = dict(zip(keys[perm].tolist(), oc.copy()))
        # the stand-in's impulse columns carry the prismatic impulses into the next step
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
        for name in ("impulse", "motorImpulse", "lowerImpulse", "upperImpulse"):
            assert bit_equal(gj[name][jv], oj[name][jv]), f"step {step}: joint {name}"
    assert contacts_seen > 100
    if solver != "XPBD":
        assert limits_hit > 0
    sp.destroy()
    sr.destroy()


# ---- parameter edits between replayed steps -----------------------------------------------------------------------------

def _piston(L, solver):
    """A 1 kg box on a vertical prismatic joint above a static post, nothing else: every step is one oracle stage."""
    wid = L.create_world(solver)
    bd = capi.default_body_def()
    post = L.s2CreateBody(wid, C.byref(bd))
    sd = capi.default_shape_def()
    L.s2CreatePolygonShape(post, C.byref(sd), C.byref(L.s2MakeBox(0.25, 0.25)))
    bd = capi.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    bd.position = capi.Vec2(0.0, 3.0)
    load = L.s2CreateBody(wid, C.byref(bd))
    L.s2CreatePolygonShape(load, C.byref(sd), C.byref(L.s2MakeBox(0.5, 0.5)))
    jd = capi.default_prismatic_def()
    jd.bodyIdA, jd.bodyIdB = post, load
    jd.localAnchorA = capi.Vec2(0.0, 3.0)
    jd.localAxisA = capi.Vec2(0.0, 1.0)
    jd.enableMotor = True
    jd.motorSpeed = 0.5
    jd.maxMotorForce = 100.0
    jd.lowerTranslation, jd.upperTranslation = -1.0, 1.0
    return wid, load, L.s2CreatePrismaticJoint(wid, C.byref(jd))


@pytest.mark.parametrize("solver", ["TGS_Soft", "PGS_NGS", "PGS", "XPBD"])
def test_edits_between_steps(product, dev, solver):
    """SetMotorSpeed, EnableLimit and SetLimits between steps of a captured, replayed step graph: each takes effect at the
    next step and every step matches the oracle run on the rows the host now holds."""
    P = product
    O = joint_oracle.load()
    wid, load, jid = _piston(P, solver)
    _flush(dev, wid)
    dw = device.DeviceWorld.attach(dev, wid)
    ctx = device.make_context(solver, DT, 4, 2, True)
    edits = {10: [lambda: P.s2PrismaticJoint_SetMotorSpeed(jid, -3.0)],
             36: [lambda: P.s2PrismaticJoint_EnableLimit(jid, True)],
             60: [lambda: P.s2PrismaticJoint_SetLimits(jid, -0.25, 0.25), lambda: P.s2PrismaticJoint_SetMotorSpeed(jid, 0.0)]}
    translation = []
    for step in range(90):
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
        for name in ("impulse", "motorImpulse", "lowerImpulse", "upperImpulse"):
            assert bit_equal(gj[name], oj[name]), f"step {step}: {name}"
        translation.append(P.s2PrismaticJoint_GetTranslation(jid))
    assert dw.counters().graphReplays > 0
    t = np.array(translation)
    if solver != "XPBD":  # the motor is not applied under XPBD
        assert t[9] > t[0] + 0.05, t[:10]   # rising at 0.5 m/s
    assert t[35] < -1.05, t[35]             # driven (or, under XPBD, falling) past -1 with the limit off
    assert t[59] >= -1.05, t[59]            # the limit, once on, holds it at -1
    assert -0.3 <= t[89] <= 0.3, t[89]      # and the narrowed limits bring it to -0.25
    P.s2DestroyWorld(wid)


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


def _create_prismatic(L, wid, a, b, collide, **kw):
    if "s2CreatePrismaticJoint" in L.missing:
        jd = capi.default_revolute_def()
        fn = L.s2CreateRevoluteJoint
    else:
        jd = capi.default_prismatic_def()
        jd.localAxisA = capi.Vec2(1.0, 0.0)
        for name, value in kw.items():
            setattr(jd, name, value)
        fn = L.s2CreatePrismaticJoint
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
    """Two overlapping boxes: the prismatic joint removes their contact unless collideConnected, and no new one forms while
    it lives; destroying it lets the pair come back. While the joint lives the pair table matches the reference's stand-in
    every step; after that the boxes, which slid on the prismatic joint and only turned on the stand-in, land elsewhere."""
    R, P = reference, product
    wr, _, br = _overlapping_pair(R, "TGS_Soft")
    wp, _, bp = _overlapping_pair(P, "TGS_Soft")
    dw = device.DeviceWorld.attach(dev, wp)
    pair = (bp[0].index, bp[1].index)
    for _ in range(3):
        R.s2World_Step(wr, DT, 4, 2, True)
        P.s2World_Step(wp, DT, 4, 2, True)
    assert pair in _pairs_dev(dw)
    jr = _create_prismatic(R, wr, br[0], br[1], collide)
    jp = _create_prismatic(P, wp, bp[0], bp[1], collide)
    _flush(dev, wp)
    rows = dw.download_joints(1)
    assert (rows["flags"][0] >> 1 & 0x7) == device.JOINT_PRISMATIC
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
        if step < 20:
            assert pairs == _pairs_ref(R, wr), step
            assert (pair in pairs) == collide, step
        elif back is None and pair in pairs:
            back = step
    assert back is not None, "the pair did not come back after the joint was destroyed"
    R.s2DestroyWorld(wr)
    P.s2DestroyWorld(wp)


# ---- lifecycle, input checks, getters, drawing ---------------------------------------------------------------------------

def test_slot_reuse_across_types(product, dev):
    """One joint slot is reused by a prismatic, a revolute, a weld and a prismatic joint again; the downloaded row carries
    the right type, flags and axis each time, and destroying the joint and its bodies leaves no joint behind."""
    P = product
    wid, gid, (a, b) = _overlapping_pair(P, "TGS_Soft")
    dw = device.DeviceWorld.attach(dev, wid)

    def row(j):
        P.s2World_Step(wid, DT, 4, 2, True)
        return dw.download_joints(j.index + 1)[j.index]

    p = _create_prismatic(P, wid, a, b, False, localAxisA=capi.Vec2(3.0, 4.0), enableLimit=True, lowerTranslation=-0.5,
                          upperTranslation=0.5, enableMotor=True, maxMotorForce=7.0, motorSpeed=0.25)
    r = row(p)
    assert (r["flags"] >> 1 & 0x7) == device.JOINT_PRISMATIC
    assert r["flags"] & device.JOINT_ENABLE_LIMIT and r["flags"] & device.JOINT_ENABLE_MOTOR
    assert bit_equal(r["localAxisA"], _unit((3.0, 4.0)))
    assert (r["lowerAngle"], r["upperAngle"], r["maxMotorTorque"], r["motorSpeed"]) == (-0.5, 0.5, 7.0, 0.25)
    P.s2DestroyJoint(p)
    jd = capi.default_revolute_def()
    jd.bodyIdA, jd.bodyIdB = a, b
    rv = P.s2CreateRevoluteJoint(wid, C.byref(jd))
    assert rv.index == p.index
    r = row(rv)
    assert (r["flags"] >> 1 & 0x7) == device.JOINT_REVOLUTE and not np.any(r["localAxisA"])
    P.s2DestroyJoint(rv)
    wd = capi.default_weld_def()
    wd.bodyIdA, wd.bodyIdB = a, b
    w = P.s2CreateWeldJoint(wid, C.byref(wd))
    assert w.index == p.index
    r = row(w)
    assert (r["flags"] >> 1 & 0x7) == device.JOINT_WELD and not np.any(r["localAxisA"])
    P.s2DestroyJoint(w)
    p2 = _create_prismatic(P, wid, a, b, True)
    assert p2.index == p.index
    r = row(p2)
    assert (r["flags"] >> 1 & 0x7) == device.JOINT_PRISMATIC and r["flags"] & device.JOINT_COLLIDE_CONNECTED
    assert r["flags"] & (device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR) == 0
    P.s2DestroyJoint(p2)
    P.s2DestroyBody(a)
    P.s2DestroyBody(b)
    for _ in range(3):
        P.s2World_Step(wid, DT, 4, 2, True)
    assert P.s2World_GetStatistics(wid).jointCount == 0
    assert (dw.download_joints(p.index + 1)["flags"] & 1).sum() == 0
    P.s2DestroyWorld(wid)


def test_create_rejects_bad_input(product, dev):
    """A zero, NaN or infinite axis, or lower > upper, creates nothing and returns the null joint id; SetLimits with
    lower > upper leaves the limits as they were."""
    P = product
    wid, _, (a, b) = _overlapping_pair(P, "TGS_Soft")
    bad = [dict(localAxisA=capi.Vec2(0.0, 0.0)), dict(localAxisA=capi.Vec2(math.nan, 1.0)),
           dict(localAxisA=capi.Vec2(1.0, math.inf)), dict(lowerTranslation=1.0, upperTranslation=-1.0),
           dict(lowerTranslation=math.nan, upperTranslation=1.0)]
    for kw in bad:
        j = _create_prismatic(P, wid, a, b, False, **kw)
        assert (j.index, j.world, j.revision) == (-1, -1, 0), kw
    assert P.s2World_GetStatistics(wid).jointCount == 0
    j = _create_prismatic(P, wid, a, b, False, localAxisA=capi.Vec2(4.0, 0.0), lowerTranslation=0.5, upperTranslation=0.5)
    assert j.index >= 0 and P.s2World_GetStatistics(wid).jointCount == 1
    P.s2PrismaticJoint_SetLimits(j, 0.3, -0.3)
    P.s2World_Step(wid, DT, 4, 2, True)
    r = device.DeviceWorld.attach(dev, wid).download_joints(j.index + 1)[j.index]
    assert (r["lowerAngle"], r["upperAngle"]) == (0.5, 0.5) and r["localAxisA"][0] == 1.0
    P.s2DestroyWorld(wid)


def test_translation_getter(product, dev):
    """s2PrismaticJoint_GetTranslation against the translation computed from the synced body state."""
    P = product
    sc = scenes.sliders(P, "TGS_Soft")
    for _ in range(40):
        sc.step(DT, 4, 2, True)
    checked = 0
    for k, d in zip(sc.piles["prismatic"], sc.piles["prismatic_defs"]):
        jid = sc.joints[k]
        got = P.s2PrismaticJoint_GetTranslation(jid)
        j = _joint_bodies(sc, k)
        pa = _world_point(P, j[0], d["localAnchorA"])
        pb = _world_point(P, j[1], d["localAnchorB"])
        angle = P.s2Body_GetAngle(j[0])
        u = _unit(d["localAxisA"]).astype(np.float64)
        axis = np.array([math.cos(angle) * u[0] - math.sin(angle) * u[1], math.sin(angle) * u[0] + math.cos(angle) * u[1]])
        assert abs(got - float(axis @ (pb - pa))) <= 1e-5, (k, got)
        checked += 1
    assert checked == len(sc.piles["prismatic"]) and checked > 0
    sc.destroy()


def _joint_bodies(sc, k):
    return sc.piles["prismatic_bodies"][sc.piles["prismatic"].index(k)]


def _world_point(P, body, local):
    p = P.s2Body_GetPosition(body)
    angle = P.s2Body_GetAngle(body)
    c, s = math.cos(angle), math.sin(angle)
    return np.array([p.x + c * local[0] - s * local[1], p.y + s * local[0] + c * local[1]])


def test_draw_one_slider(product, dev):
    """The segments s2World_Draw emits for one slider with limits: the axis through anchor A, a mark at each limit, the
    segment from anchor A to anchor B."""
    P = product
    wid = P.create_world("TGS_Soft")
    bd = capi.default_body_def()
    bd.position = capi.Vec2(1.0, 2.0)
    a = P.s2CreateBody(wid, C.byref(bd))
    bd = capi.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    bd.position = capi.Vec2(1.0, 3.5)
    b = P.s2CreateBody(wid, C.byref(bd))
    jd = capi.default_prismatic_def()
    jd.bodyIdA, jd.bodyIdB = a, b
    jd.localAnchorA = capi.Vec2(0.0, 1.0)
    jd.localAxisA = capi.Vec2(0.0, 2.0)
    jd.enableLimit = True
    jd.lowerTranslation, jd.upperTranslation = -0.5, 1.0
    jd.drawSize = 2.0
    P.s2CreatePrismaticJoint(wid, C.byref(jd))
    segments = [v for name, v in _draw_log(P, wid) if name == "DrawSegment"]
    f = np.float32
    expected = [
        (1.0, 1.0, 1.0, 5.0, f(0.7), f(0.7), f(0.7)),    # the axis: anchor A (1, 3) -/+ 2 * (0, 1)
        (2.0, 2.5, 0.0, 2.5, f(0.3), f(0.9), f(0.3)),    # lower mark at (1, 2.5), half-length 0.5 * drawSize across
        (2.0, 4.0, 0.0, 4.0, f(0.9), f(0.3), f(0.3)),    # upper mark at (1, 4)
        (1.0, 3.0, 1.0, 3.5, f(0.5), f(0.8), f(0.8)),    # anchor A to anchor B
    ]
    assert segments == [tuple(float(x) for x in e) for e in expected]
    P.s2DestroyWorld(wid)
