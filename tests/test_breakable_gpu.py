"""GPU: joint reactions and breakable joints (DESIGN.md §3.13) through the public API and the device ABI.

* The reaction pass: the device's reactions (s2b_download_joint_reactions, s2World_GetJointReactions) and the per-joint
  getters equal s2ComputeJointReaction evaluated on the downloaded joint rows and body A's downloaded rotation, bit for bit,
  under every variant and schedule (colour, wavefront, regions, launch by launch). Its broken list is exactly the joints
  whose reaction exceeds a threshold, in slot order.
* scenes.breakables every step under every variant against the reference: the reference's collide and finalize on the
  stand-in world, the oracle's solve (the weld, prismatic or motor oracle, one extension type per scene) in the device's
  order. The reference destroys with its own s2DestroyJoint, at the start of the next step, exactly the joints whose oracle
  reactions exceed their thresholds. Every step the device's broken list equals the oracle's, the contact set (after each
  break included) equals the reference's, and bodies, contact and joint impulses match bit for bit.
* scenes.breakables every step under every variant, all five types together: the broken list against the same
  restatement on the device's rows; a broken joint is gone at the next step; at least one joint breaks and the joints meant
  to hold never do; under XPBD only the mouse joint breaks.
* Edges: a threshold equal to the reaction; joints to static and kinematic bodies; two joints between the same bodies;
  1 100 joints breaking in one step; thresholds past a capacity growth; a reused slot; a broken joint destroyed by the caller
  first; a short output buffer; a threshold set under graph replay; the launch count with thresholds set and cleared; bad
  input.

Mutations each test catches: a rate taken from the wrong context field, an axis left in body A's frame or a stale pose read
fail the bit-for-bit comparisons; a non-strict comparison fails the equal-threshold test; a list handed out in device order
fails the 1 100-joint test; a deferred destroy without the revision check frees a reused slot in the caller-destroys test; a
pass that runs without thresholds fails the launch-count test."""
import ctypes as C
import math

import numpy as np
import pytest

import motor_oracle
import prismatic_oracle
import weld_oracle
from helpers import (bit_equal, body_rows_from_ref, carry_sticky_friction, contact_rows_from_ref, joint_rows_from_ref,
                     load_bodies_into_ref, ref_delta_positions, store_oracle_bodies)
from oracle import ref as refmod
from solver2d_b200 import capi, device, scenes

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0
VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]
MODES = ["color", "wavefront", "regions", "launch"]


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


@pytest.fixture(scope="module")
def dev():
    return device.Device()


def _rate(solver):
    ctx = device.make_context(solver, DT, 4, 2, True)
    return np.float32(ctx.inv_dt if solver == "TGS_Sticky" else ctx.inv_h)


def _restated(L, joints, bodies, rate):
    """(n, 3) reactions of the downloaded rows through the exported host function; zero for free slots."""
    out = np.zeros((len(joints), 3), dtype=np.float32)
    for i, r in enumerate(joints):
        if (int(r["flags"]) & 1) == 0:
            continue
        q = bodies["rot"][int(r["bodyA"])]
        x = L.s2ComputeJointReaction((int(r["flags"]) >> 1) & 7, capi.Vec2(*r["impulse"]), float(r["motorImpulse"]),
                                     float(r["lowerImpulse"]), float(r["upperImpulse"]), capi.Rot(float(q[0]), float(q[1])),
                                     capi.Vec2(*r["localAxisA"]), float(rate))
        out[i] = (x.force.x, x.force.y, x.torque)
    return out


def _over(joints, reactions):
    """Slots whose reaction exceeds a set threshold, strictly, in float32 as the device compares."""
    f = reactions[:, :2].astype(np.float32)
    force = np.sqrt(f[:, 0] * f[:, 0] + f[:, 1] * f[:, 1])
    valid = (joints["flags"] & 1) == 1
    bf, bt = joints["breakForce"], joints["breakTorque"]
    hit = ((bf > 0) & (force > bf)) | ((bt > 0) & (np.abs(reactions[:, 2]) > bt))
    return np.nonzero(valid & hit)[0].astype(np.int32)


def _broken_ids(L, world, capacity=4096):
    out = (capi.JointId * max(capacity, 1))()
    n = L.s2World_GetBrokenJoints(world, out, capacity)
    return n, [(out[k].index, out[k].revision) for k in range(min(n, capacity))]


def _api_reactions(L, world, cap):
    out = np.zeros((max(cap, 1), 3), dtype=np.float32)
    n = L.s2World_GetJointReactions(world, out.ctypes.data, cap)
    return n, out[:cap]


def _configure(dw, mode):
    if mode == "wavefront":
        dw.set_schedule(device.SCHEDULE_WAVEFRONT)
    elif mode == "regions":
        dw.set_regions(2)
    elif mode == "launch":
        dw.set_persistent(False)


# ---- the reaction pass ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("solver", VARIANTS)
def test_reaction_pass_matches_shared_function(product, dev, solver, mode):
    P = product
    sc = scenes.breakables(P, solver)
    scenes.apply_break_thresholds(sc)
    P.s2World_Flush(sc.world)
    dw = device.DeviceWorld.attach(dev, sc.world)
    _configure(dw, mode)
    rate = _rate(solver)
    live_ids = {j.index: j for j in sc.joints}
    for step in range(24):
        sc.step(DT, 4, 2, True)
        if step % 6 != 5:
            continue
        cap = dw.counters().jointCapacity
        joints = dw.download_joints(cap)
        bodies = dw.download_all_bodies(dw.counters().bodyCapacity)
        want = _restated(P, joints, bodies, rate)
        got = dw.download_joint_reactions(cap)
        assert got.tobytes() == want.tobytes(), f"step {step}"
        n, api = _api_reactions(P, sc.world, cap)
        assert n >= int(np.count_nonzero(joints["flags"] & 1)) and api.tobytes() == want.tobytes(), f"step {step}"
        for slot, jid in live_ids.items():
            if (int(joints["flags"][slot]) & 1) == 1:  # (not yet destroyed by a break)
                f = P.s2Joint_GetReactionForce(jid)
                t = P.s2Joint_GetReactionTorque(jid)
                assert np.array([f.x, f.y, t], dtype=np.float32).tobytes() == want[slot].tobytes(), (step, slot)
        assert np.array_equal(dw.download_broken_joints(), _over(joints, want)), f"step {step}"
    sc.destroy()


# ---- every step against the reference -----------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def reference():
    if not refmod.available():
        pytest.skip("the reference library (oracle/_ref) is not built")
    return refmod.load()


ORACLES = {"weld": weld_oracle, "prismatic": prismatic_oracle, "motor": motor_oracle}


def _own_rows(rows, sc):
    """The stand-in revolute rows of a breakables scene built on the reference, turned into the rows of their own type, with
    the scene's thresholds."""
    for k, kind in enumerate(sc.piles["types"]):
        slot = sc.joints[k].index
        if (int(rows["flags"][slot]) & 1) == 0:
            continue  # (destroyed by a break)
        assert rows["flags"][slot] & (device.JOINT_ENABLE_LIMIT | device.JOINT_ENABLE_MOTOR) == 0
        d = sc.piles["defs"].get(k)
        base = int(rows["flags"][slot]) & ~0xE
        if kind == "weld":
            rows["flags"][slot] = base | (device.JOINT_WELD << 1)
        elif kind == "prismatic":
            rows["flags"][slot] = base | (device.JOINT_PRISMATIC << 1) | device.JOINT_ENABLE_LIMIT
            rows["lowerAngle"][slot], rows["upperAngle"][slot] = d["lowerTranslation"], d["upperTranslation"]
            rows["localAxisA"][slot] = d["localAxisA"]
        elif kind == "motor":
            rows["flags"][slot] = base | (device.JOINT_MOTOR << 1)
            rows["localOriginAnchorA"][slot] = d["linearOffset"]
            rows["localOriginAnchorB"][slot] = (0.0, 0.0)
            rows["maxMotorTorque"][slot] = d["maxTorque"]
            rows["hertz"][slot] = d["maxForce"]
            rows["dampingRatio"][slot] = 0.3  # s2DefaultMotorJointDef's correctionFactor
    for k, force, torque in sc.piles["break"]:
        slot = sc.joints[k].index
        rows["breakForce"][slot], rows["breakTorque"][slot] = force, torque
    return rows


@pytest.mark.parametrize("ext", sorted(ORACLES))
@pytest.mark.parametrize("solver", VARIANTS)
def test_breakables_against_reference(reference, product, dev, solver, ext):
    """Reference collide on the stand-in world, the oracle in the device's order, reference finalize, and the reference's
    s2DestroyJoint on the joints whose oracle reactions exceed their thresholds; the device runs the same steps through
    s2World_Step. Every step: the broken lists, the contact sets and, bit for bit, bodies (XPBD's delta positions included),
    contact and joint impulses."""
    R, P = reference, product
    O = ORACLES[ext].load()
    sr = scenes.breakables(R, solver, parts=(ext,))
    sp = scenes.breakables(P, solver, parts=(ext,))
    assert "s2Joint_SetBreakForce" in R.missing and sr.piles["types"] == sp.piles["types"]
    assert [j.index for j in sr.joints] == [j.index for j in sp.joints]
    scenes.apply_break_thresholds(sp)
    P.s2World_Flush(sp.world)
    dw = device.DeviceWorld.attach(dev, sp.world)
    ctx = device.make_context(solver, DT, 4, 2, True)
    rate = _rate(solver)
    sticky = solver == "TGS_Sticky"
    k_of_slot = {j.index: k for k, j in enumerate(sr.joints)}
    F = refmod.BODY_F
    solved = {}
    ref_broken = []
    broken_total = 0
    broken_kinds = set()
    contacts_after_break = 0
    for step in range(90):
        for slot in ref_broken:  # what s2World_Step does before it flushes
            R.s2DestroyJoint(sr.joints[k_of_slot[slot]])
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
        joints = _own_rows(joint_rows_from_ref(*R.joints(sr.world)), sr)
        got_contacts = dw.download_contacts(len(rows_key) + 64)
        assert len(got_contacts) == len(rows_key), f"step {step}: contact count"
        assert np.array_equal(got_contacts["shapeA"], rows_key["shapeA"]) and \
            np.array_equal(got_contacts["shapeB"], rows_key["shapeB"]), f"step {step}: contact set"
        if broken_total > 0:
            contacts_after_break += len(rows_key)

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
        assert bit_equal(got_after["points"]["tangentImpulse"][live], oc["points"]["tangentImpulse"][live]), f"step {step}"
        gj = dw.download_joints(len(oj))
        jv = (oj["flags"] & 1) == 1
        assert np.array_equal(gj["flags"] & 1, oj["flags"] & 1), f"step {step}: live joints"
        for name in ("impulse", "motorImpulse", "lowerImpulse", "upperImpulse"):
            assert bit_equal(gj[name][jv], oj[name][jv]), f"step {step}: joint {name}"

        # the oracle's reactions, at body A's rotation after the reference's finalize, against the thresholds
        oj["breakForce"], oj["breakTorque"] = joints["breakForce"], joints["breakTorque"]
        ref_broken = _over(oj, _restated(P, oj, body_rows_from_ref(rf, ri), rate)).tolist()
        n, ids = _broken_ids(P, sp.world)
        assert [i for i, _ in ids] == ref_broken, f"step {step}: broken joints"
        broken_total += n
        broken_kinds |= {sr.piles["types"][k_of_slot[slot]] for slot in ref_broken}
    assert contacts_after_break > 0
    if solver == "XPBD":
        assert broken_kinds == {"mouse"}  # the position rows keep no impulses
    else:
        assert broken_kinds == {"revolute", "mouse", ext}, broken_kinds
    sp.destroy()
    sr.destroy()


# ---- every step of the breakables scene ---------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", VARIANTS)
def test_breakables_every_step(product, dev, solver):
    P = product
    sc = scenes.breakables(P, solver)
    scenes.apply_break_thresholds(sc)
    P.s2World_Flush(sc.world)
    dw = device.DeviceWorld.attach(dev, sc.world)
    rate = _rate(solver)
    never = {sc.joints[i].index for i in sc.piles["never"]}
    broken_types = set()
    pending = []
    total = 0
    for step in range(150):
        sc.step(DT, 4, 2, True)
        cap = dw.counters().jointCapacity
        joints = dw.download_joints(cap)
        for slot, rev in pending:  # destroyed at the start of this step
            assert (int(joints["flags"][slot]) & 1) == 0, (step, slot)
        bodies = dw.download_all_bodies(dw.counters().bodyCapacity)
        want = _over(joints, _restated(P, joints, bodies, rate))
        n, ids = _broken_ids(P, sc.world)
        assert n == len(want) and [i for i, _ in ids] == want.tolist(), f"step {step}"
        c = dw.counters()
        assert c.jointsBroken == n and c.jointsChecked == int(np.count_nonzero(
            ((joints["flags"] & 1) == 1) & ((joints["breakForce"] > 0) | (joints["breakTorque"] > 0)))), f"step {step}"
        assert not never & set(want.tolist()), f"step {step}"
        broken_types |= {(int(joints["flags"][s]) >> 1) & 7 for s in want.tolist()}
        total += n
        pending = ids
    assert total > 0
    if solver == "XPBD":
        assert broken_types == {device.JOINT_MOUSE}
    else:
        assert {device.JOINT_REVOLUTE, device.JOINT_MOUSE, device.JOINT_MOTOR} <= broken_types, broken_types
    stats = P.s2World_GetStatistics(sc.world)
    assert stats.jointCount == len(sc.joints) - (total - len(pending))  # (the last step's breaks are destroyed by the next)
    sc.destroy()


# ---- edges --------------------------------------------------------------------------------------------------------------

def _hanging(L, solver="PGS", count=1, kind=capi.STATIC_BODY, joints_per_box=1):
    """`count` 1 m boxes (density 1: 1 kg, 10 N) hanging at rest on revolute joints from one anchor body; with two joints
    per box, from its two top corners."""
    wid = L.create_world(solver)
    bd = capi.default_body_def()
    bd.type = kind
    bd.position = capi.Vec2(0.0, 10.0)
    anchor = L.s2CreateBody(wid, C.byref(bd))
    sd = capi.default_shape_def()
    sd.density = 1.0
    ids = []
    for k in range(count):
        bd = capi.default_body_def()
        bd.type = capi.DYNAMIC_BODY
        bd.position = capi.Vec2(2.0 * k, 9.0)
        b = L.s2CreateBody(wid, C.byref(bd))
        L.s2CreatePolygonShape(b, C.byref(sd), C.byref(L.s2MakeBox(0.5, 0.5)))
        for side in ([0.0] if joints_per_box == 1 else [-0.5, 0.5]):
            jd = capi.default_revolute_def()
            jd.bodyIdA, jd.bodyIdB = anchor, b
            jd.localAnchorA = capi.Vec2(2.0 * k + side, -1.0 + (0.5 if side else 0.0))
            jd.localAnchorB = capi.Vec2(side, 0.5 if side else 0.0)
            ids.append(L.s2CreateRevoluteJoint(wid, C.byref(jd)))
    return wid, anchor, ids


def _force(L, jid):
    f = L.s2Joint_GetReactionForce(jid)
    return np.float32(math.sqrt(np.float32(f.x) * np.float32(f.x) + np.float32(f.y) * np.float32(f.y)))


def test_reads_zero_before_the_first_step(product):
    L = product
    wid, _, ids = _hanging(L)
    f = L.s2Joint_GetReactionForce(ids[0])
    assert (f.x, f.y, L.s2Joint_GetReactionTorque(ids[0])) == (0.0, 0.0, 0.0)
    assert _broken_ids(L, wid)[0] == 0
    L.s2DestroyWorld(wid)


def test_threshold_equal_to_the_reaction_holds(product):
    L = product
    wid, _, ids = _hanging(L)
    for _ in range(60):
        L.s2World_Step(wid, DT, 4, 2, True)
    load = _force(L, ids[0])
    L.s2World_Step(wid, DT, 4, 2, True)
    assert _force(L, ids[0]) == load and load > 0  # (at rest: the same reading every step)
    L.s2Joint_SetBreakForce(ids[0], float(load))
    L.s2World_Step(wid, DT, 4, 2, True)
    assert _broken_ids(L, wid)[0] == 0
    L.s2Joint_SetBreakForce(ids[0], float(np.nextafter(load, np.float32(0))))
    L.s2World_Step(wid, DT, 4, 2, True)
    assert _broken_ids(L, wid)[1] == [(ids[0].index, ids[0].revision)]
    L.s2DestroyWorld(wid)


@pytest.mark.parametrize("kind", [capi.STATIC_BODY, capi.KINEMATIC_BODY])
def test_static_and_kinematic_anchors_and_shared_bodies(product, kind):
    """Two joints between the same pair of bodies, hung from a static or a kinematic body at the box's two top corners,
    break in the same step; the next step destroys both."""
    L = product
    wid, _, ids = _hanging(L, kind=kind, joints_per_box=2)
    for _ in range(30):
        L.s2World_Step(wid, DT, 4, 2, True)
    load = min(float(_force(L, j)) for j in ids)
    assert load > 1.0  # (both carry part of the 10 N)
    for jid in ids:
        L.s2Joint_SetBreakForce(jid, 0.5 * load)
    L.s2World_Step(wid, DT, 4, 2, True)
    n, got = _broken_ids(L, wid)
    assert got == sorted((j.index, j.revision) for j in ids)
    L.s2World_Step(wid, DT, 4, 2, True)
    assert L.s2World_GetStatistics(wid).jointCount == 0
    L.s2DestroyWorld(wid)


def test_many_joints_break_in_slot_order_and_short_buffers(product, dev):
    L = product
    wid, _, ids = _hanging(L, count=1100)
    for jid in ids:
        L.s2Joint_SetBreakForce(jid, 1.0)
    L.s2World_Step(wid, DT, 4, 2, True)
    want = sorted((j.index, j.revision) for j in ids)
    n, got = _broken_ids(L, wid, capacity=2048)
    assert n == 1100 and got == want
    n, got = _broken_ids(L, wid, capacity=10)
    assert n == 1100 and got == want[:10]
    dw = device.DeviceWorld.attach(dev, wid)
    assert dw.download_broken_joints().tolist() == [i for i, _ in want]
    L.s2World_Step(wid, DT, 4, 2, True)
    assert L.s2World_GetStatistics(wid).jointCount == 0
    L.s2DestroyWorld(wid)


def test_thresholds_past_a_capacity_growth(product, dev):
    L = product
    wid, anchor, ids = _hanging(L, count=2)
    L.s2World_Step(wid, DT, 4, 2, True)
    cap0 = device.DeviceWorld.attach(dev, wid).counters().jointCapacity
    sd = capi.default_shape_def()
    sd.density = 1.0
    more = []
    for k in range(200):
        bd = capi.default_body_def()
        bd.type = capi.DYNAMIC_BODY
        bd.position = capi.Vec2(-3.0 - 2.0 * k, 9.0)
        b = L.s2CreateBody(wid, C.byref(bd))
        L.s2CreatePolygonShape(b, C.byref(sd), C.byref(L.s2MakeBox(0.5, 0.5)))
        jd = capi.default_revolute_def()
        jd.bodyIdA, jd.bodyIdB = anchor, b
        jd.localAnchorA = capi.Vec2(-3.0 - 2.0 * k, -1.0)
        more.append(L.s2CreateRevoluteJoint(wid, C.byref(jd)))
    for jid in more[-3:]:
        L.s2Joint_SetBreakForce(jid, 1.0)
    L.s2World_Step(wid, DT, 4, 2, True)
    dw = device.DeviceWorld.attach(dev, wid)
    assert dw.counters().jointCapacity > cap0
    rows = dw.download_joints()
    assert rows["breakForce"][[j.index for j in more[-3:]]].tolist() == [1.0, 1.0, 1.0]
    assert _broken_ids(L, wid)[1] == sorted((j.index, j.revision) for j in more[-3:])
    L.s2DestroyWorld(wid)


def test_caller_destroys_first_and_slot_reuse(product, dev):
    """A broken joint destroyed by the caller before the next step is not destroyed again, and the joint created in its slot
    (a new revision, no threshold) survives the next step."""
    L = product
    wid, anchor, ids = _hanging(L, count=2)
    L.s2Joint_SetBreakForce(ids[0], 1.0)
    L.s2World_Step(wid, DT, 4, 2, True)
    assert _broken_ids(L, wid)[1] == [(ids[0].index, ids[0].revision)]
    L.s2DestroyJoint(ids[0])
    # the same slot, reused: the list still names the joint that broke
    bd = capi.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    bd.position = capi.Vec2(10.0, 9.0)
    b = L.s2CreateBody(wid, C.byref(bd))
    sd = capi.default_shape_def()
    sd.density = 1.0
    L.s2CreatePolygonShape(b, C.byref(sd), C.byref(L.s2MakeBox(0.5, 0.5)))
    jd = capi.default_revolute_def()
    jd.bodyIdA, jd.bodyIdB = anchor, b
    jd.localAnchorA = capi.Vec2(10.0, -1.0)
    fresh = L.s2CreateRevoluteJoint(wid, C.byref(jd))
    assert fresh.index == ids[0].index and fresh.revision != ids[0].revision
    assert L.s2Joint_GetBreakForce(fresh) == 0.0
    assert _broken_ids(L, wid)[1] == [(ids[0].index, ids[0].revision)]
    L.s2World_Step(wid, DT, 4, 2, True)
    assert L.s2World_GetStatistics(wid).jointCount == 2
    rows = device.DeviceWorld.attach(dev, wid).download_joints()
    assert int(rows["flags"][fresh.index]) & 1 == 1 and rows["breakForce"][fresh.index] == 0.0
    L.s2World_Step(wid, DT, 4, 2, True)
    assert L.s2World_GetStatistics(wid).jointCount == 2
    L.s2DestroyWorld(wid)


def test_bad_input_is_ignored(product):
    L = product
    wid, _, ids = _hanging(L)
    j = ids[0]
    L.s2Joint_SetBreakForce(j, 5.0)
    L.s2Joint_SetBreakTorque(j, 7.0)
    for bad in (-1.0, float("nan"), float("inf"), -0.5):
        L.s2Joint_SetBreakForce(j, bad)
        L.s2Joint_SetBreakTorque(j, bad)
    assert (L.s2Joint_GetBreakForce(j), L.s2Joint_GetBreakTorque(j)) == (5.0, 7.0)
    L.s2Joint_SetBreakForce(j, 0.0)
    L.s2Joint_SetBreakTorque(j, 0.0)
    assert (L.s2Joint_GetBreakForce(j), L.s2Joint_GetBreakTorque(j)) == (0.0, 0.0)
    L.s2DestroyWorld(wid)


def _launches_per_step(L, dw, wid, steps=5):
    before = dw.counters().kernelLaunches
    for _ in range(steps):
        L.s2World_Step(wid, DT, 4, 2, True)
    return (dw.counters().kernelLaunches - before) / steps


def test_launch_count_and_graph_captures(product, dev):
    """At rest, a world without thresholds launches what it launched before; a threshold adds the one reaction kernel per
    step; clearing every threshold returns to the first count. A threshold edit under graph replay re-captures the solver
    graph no more often than a motor-speed edit, and takes effect."""
    L = product
    wid, _, ids = _hanging(L, "TGS_Soft", count=4)
    dw = device.DeviceWorld.attach(dev, wid)
    for _ in range(90):
        L.s2World_Step(wid, DT, 4, 2, True)
    base = _launches_per_step(L, dw, wid)
    c0 = dw.counters().graphCaptures
    L.s2RevoluteJoint_SetMotorSpeed(ids[1], 0.0)
    L.s2World_Step(wid, DT, 4, 2, True)
    L.s2World_Step(wid, DT, 4, 2, True)
    motor_edit = dw.counters().graphCaptures - c0
    c1 = dw.counters().graphCaptures
    for jid in ids:
        L.s2Joint_SetBreakForce(jid, 1e6)
    L.s2World_Step(wid, DT, 4, 2, True)
    L.s2World_Step(wid, DT, 4, 2, True)
    assert dw.counters().graphCaptures - c1 <= motor_edit
    assert _launches_per_step(L, dw, wid) == base + 1
    assert dw.counters().jointsChecked == 4
    L.s2Joint_SetBreakForce(ids[2], 1.0)  # takes effect under replay
    L.s2World_Step(wid, DT, 4, 2, True)
    assert _broken_ids(L, wid)[1] == [(ids[2].index, ids[2].revision)]
    L.s2World_Step(wid, DT, 4, 2, True)
    for jid in (ids[0], ids[1], ids[3]):
        L.s2Joint_SetBreakForce(jid, 0.0)
    L.s2World_Step(wid, DT, 4, 2, True)
    assert _launches_per_step(L, dw, wid) == base
    assert dw.counters().jointsChecked == 0 and _broken_ids(L, wid)[0] == 0
    L.s2DestroyWorld(wid)
