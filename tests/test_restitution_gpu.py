"""GPU: the restitution extension (DESIGN.md §3.7) — the device's capture and pass against the oracle (tests/
restitution_oracle.py) bit for bit, in every schedule and for all ten variants; the known answers through the public API;
and restitution turned on but with nothing to bounce leaves every step bit-identical to the production path."""
import ctypes as C

import numpy as np
import pytest

import restitution_oracle as ro
from helpers import (STICKY_FIELDS, bit_equal, body_rows_from_ref, carry_sticky_friction, contact_rows_from_ref,
                     joint_rows_from_ref)
from oracle import port
from oracle import ref as refmod
from solver2d_b200 import capi, device, scenes

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0
VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]
REL = 1e-6  # see test_restitution_cpu.py


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


def _compare(got, got_contacts, ob, oc, bodies, contacts):
    valid = (bodies["flags"] & 1) == 1
    for name in ("position", "rot", "linearVelocity", "angularVelocity"):
        assert bit_equal(got[name][valid], ob[name][valid]), name
    live = contacts["pointCount"] > 0
    for name in ("normalImpulse", "tangentImpulse"):
        assert bit_equal(got_contacts["points"][name][live], oc["points"][name][live]), name


# ---- the solver stage against the oracle ------------------------------------------------------------------------------

@pytest.mark.parametrize("persistent", [True, False])
@pytest.mark.parametrize("mode", ["wavefront", "color", "regions"])
@pytest.mark.parametrize("solver", VARIANTS)
def test_stage_matches_oracle(reference, dev, solver, mode, persistent):
    """One solver stage of a pyramid and of the jointed chains, every contact given e in {0, 0.25, 0.6, 1} and the bodies
    a downward kick, with a low threshold so that many points bounce and many do not."""
    R = reference
    O = port.load()
    bounced = 0
    for recipe, kw, warm in ((scenes.pyramid, dict(base_count=12), 2 if solver == "Jacobi" else 30), (scenes.limited_chains, {}, 40)):
        sc = recipe(R, solver, **kw)
        for _ in range(warm):
            sc.step(DT, 4, 2, True)
        R.step_collide(sc.world)
        bodies = body_rows_from_ref(*R.bodies(sc.world))
        contacts, _ = contact_rows_from_ref(*R.contacts(sc.world))
        joints = joint_rows_from_ref(*R.joints(sc.world))
        sc.destroy()
        rng = np.random.default_rng(7)
        contacts["restitution"] = rng.choice(np.array(scenes.BOUNCER_RESTITUTION, dtype=np.float32), len(contacts))
        moving = bodies["invMass"] != 0
        bodies["linearVelocity"][moving, 1] -= rng.uniform(0.0, 1.5, int(moving.sum())).astype(np.float32)
        ctx = device.make_context(solver, DT, 4, 2)

        dw = dev.create_world(capi.SOLVER[solver])
        dw.upload_bodies(bodies, len(bodies))
        dw.upload_joints(joints, len(joints))
        dw.upload_contacts(contacts)
        dw.set_schedule(device.SCHEDULE_WAVEFRONT if mode == "wavefront" else device.SCHEDULE_COLOR)
        dw.set_regions(2 if mode == "regions" else 0)
        dw.set_persistent(persistent)
        dw.set_restitution(True, 0.3)
        dw.solve(ctx)
        got = dw.download_all_bodies(len(bodies))
        got_contacts = dw.download_contacts(len(contacts))
        order, _ = dw.solve_order(len(contacts) + len(joints))
        counters = dw.counters()
        dw.destroy()
        if mode == "regions" and persistent:
            assert counters.regionCount > 0
        assert bit_equal(got_contacts["restitution"], contacts["restitution"])
        # the wavefront schedule reproduces the natural order: the oracle runs without the device's order there
        ob, oc, oj, n = ro.solve(O, capi.SOLVER[solver], bodies, contacts, joints, ctx, order=None if mode == "wavefront" else order,
                                 threshold=0.3)
        bounced += n
        _compare(got, got_contacts, ob, oc, bodies, contacts)
    assert bounced > 10


# ---- every step of the bouncers scene through the public API -----------------------------------------------------------

def _load_bodies_into_ref(R, wid, rows):
    F = refmod.BODY_F
    bf, bi = R.bodies(wid)
    n = min(len(rows), bf.shape[0])
    valid = bi[:n, 0] == 1
    for name, col, width in (("origin", F["origin"], 2), ("position", F["position"], 2), ("rot", F["rot"], 2),
                             ("linearVelocity", F["v"], 2)):
        bf[:n, col:col + width][valid] = rows[name][:n][valid]
    bf[:n, F["w"]][valid] = rows["angularVelocity"][:n][valid]
    bf[:n, F["dp"]:F["dp"] + 2][valid] = 0.0
    bf[:n, F["force"]:F["force"] + 2][valid] = rows["force"][:n][valid]
    bf[:n, F["torque"]][valid] = rows["torque"][:n][valid]
    R.load_body_state(wid, bf)


@pytest.mark.parametrize("solver", VARIANTS)
def test_bouncers_every_step(reference, product, dev, solver):
    """Reference stages 1-3, then the oracle with restitution in the device's order, then reference finalize; the device runs
    the same steps through s2World_Step with restitution enabled. Every step bit for bit."""
    R, P = reference, product
    O = port.load()
    kw = dict(columns=8, rows=3)
    sr = scenes.bouncers(R, solver, **kw)
    sp = scenes.bouncers(P, solver, **kw)
    P.s2World_EnableRestitution(sp.world, True)
    dev.lib.s2World_Flush.restype = None
    dev.lib.s2World_Flush.argtypes = [capi.WorldId]
    dev.lib.s2World_Flush(sp.world)
    dw = device.DeviceWorld.attach(dev, sp.world)
    ctx = device.make_context(solver, DT, 4, 2, True)
    sticky = solver == "TGS_Sticky"
    solved = {}
    seen = dict(bounced=0, below=0, zero=0, merged_while_bouncing=0)
    jointed = set()
    jf, ji = R.joints(sr.world)
    for row in ji[ji[:, refmod.JOINT_I["valid"]] == 1]:
        jointed.update((int(row[refmod.JOINT_I["bodyA"]]), int(row[refmod.JOINT_I["bodyB"]])))
    jointed_bounced = 0
    prev_keys = None
    F = refmod.BODY_F
    for step in range(90):
        cap = R.capacities(sr.world)["bodyCap"]
        pre = dw.download_all_bodies(cap)
        _load_bodies_into_ref(R, sr.world, pre)
        R.step_collide(sr.world)
        sp.step(DT, 4, 2, True)

        bodies = body_rows_from_ref(*R.bodies(sr.world))
        cf, ci = R.contacts(sr.world)
        rows_slot, slots = contact_rows_from_ref(cf, ci)
        keys = (np.minimum(rows_slot["shapeA"], rows_slot["shapeB"]).astype(np.uint64) << np.uint64(32)) | \
            np.maximum(rows_slot["shapeA"], rows_slot["shapeB"]).astype(np.uint64)
        perm = np.argsort(keys, kind="stable")
        rows_key = rows_slot[perm]
        if sticky:
            carry_sticky_friction(rows_key, keys[perm], solved)
        joints = joint_rows_from_ref(*R.joints(sr.world))
        got_contacts = dw.download_contacts(len(rows_key) + 64)
        assert len(got_contacts) == len(rows_key) and np.array_equal(got_contacts["shapeA"], rows_key["shapeA"])
        # the device mixed each new contact's restitution as max of its shapes' (reference src/contact.c:49-52)
        sf, _ = R.shapes(sr.world)
        e_ref = np.maximum(sf[rows_key["shapeA"], refmod.SHAPE_F["restitution"]], sf[rows_key["shapeB"], refmod.SHAPE_F["restitution"]])
        assert bit_equal(got_contacts["restitution"], e_ref.astype(np.float32)), f"step {step}: mixed restitution"
        rows_key["restitution"] = e_ref

        order, _ = dw.solve_order(len(rows_key) + len(joints) + 16, max_groups=200000)
        cap_rows = ro.capture(bodies, rows_key)
        ob, oc, oj, n = ro.solve(O, capi.SOLVER[solver], bodies, rows_key, joints, ctx, order=order)
        seen["bounced"] += n
        live = rows_key["pointCount"] > 0
        seen["zero"] += int(((rows_key["restitution"] == 0) & live).sum())
        for j in range(2):
            has = (rows_key["pointCount"] > j) & (rows_key["restitution"] > 0)
            seen["below"] += int((has & (cap_rows["vr"][j] < 0) & (cap_rows["vr"][j] > -1.0)).sum())
        if n:
            hit = oc["points"]["normalImpulse"] != _solved_without(O, solver, bodies, rows_key, joints, ctx, order)
            rows_hit = hit.any(axis=1)
            jointed_bounced += int(np.isin(rows_key["bodyA"][rows_hit], list(jointed)).sum()
                                   + np.isin(rows_key["bodyB"][rows_hit], list(jointed)).sum())
            if prev_keys is not None and not np.array_equal(prev_keys, keys[perm]):
                seen["merged_while_bouncing"] += 1
        prev_keys = keys[perm]

        bf, bi = R.bodies(sr.world)
        valid = bi[:, 0] == 1
        bf[:, F["position"]:F["position"] + 2][valid] = ob["position"][valid]
        bf[:, F["rot"]:F["rot"] + 2][valid] = ob["rot"][valid]
        bf[:, F["v"]:F["v"] + 2][valid] = ob["linearVelocity"][valid]
        bf[:, F["w"]][valid] = ob["angularVelocity"][valid]
        bf[:, F["dp"]:F["dp"] + 2][valid] = 0.0
        R.load_body_state(sr.world, bf)
        imp = np.zeros((cf.shape[0], 4), dtype=np.float32)
        imp[slots[perm], 0] = oc["points"]["normalImpulse"][:, 0]
        imp[slots[perm], 1] = oc["points"]["tangentImpulse"][:, 0]
        imp[slots[perm], 2] = oc["points"]["normalImpulse"][:, 1]
        imp[slots[perm], 3] = oc["points"]["tangentImpulse"][:, 1]
        R.load_contact_impulses(sr.world, imp)
        if sticky:
            solved = dict(zip(keys[perm].tolist(), oc.copy()))
        if len(oj):
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
        got_after = dw.download_contacts(len(rows_key) + 64)
        assert bit_equal(got_after["points"]["normalImpulse"][live], oc["points"]["normalImpulse"][live]), f"step {step}: impulses"
    sp.destroy()
    sr.destroy()
    assert seen["bounced"] > 20 and seen["below"] > 0 and seen["zero"] > 0, seen
    assert jointed_bounced > 0, "no jointed body bounced"
    assert seen["merged_while_bouncing"] > 0, seen


def _solved_without(O, solver, bodies, contacts, joints, ctx, order):
    _, oc, _ = O.solve(capi.SOLVER[solver], bodies, contacts, joints, ctx, order=order)
    return oc["points"]["normalImpulse"]


# ---- known answers through the public API ------------------------------------------------------------------------------

def _ball_world(P, solver, e_ball, e_ground, height=3.0):
    wid = P.create_world(solver)
    bd = capi.default_body_def()
    bd.position = capi.Vec2(0.0, -1.0)
    gid = P.s2CreateBody(wid, C.byref(bd))
    sd = capi.default_shape_def()
    sd.restitution = e_ground
    box = P.s2MakeBox(20.0, 1.0)
    P.s2CreatePolygonShape(gid, C.byref(sd), C.byref(box))
    bd = capi.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    bd.position = capi.Vec2(0.0, 0.5 + height)
    bid = P.s2CreateBody(wid, C.byref(bd))
    sd.restitution = e_ball
    P.s2CreateCircleShape(bid, C.byref(sd), C.byref(capi.Circle(capi.Vec2(0.0, 0.0), 0.5)))
    return wid


@pytest.mark.parametrize("solver", VARIANTS)
def test_ball_bounce_known_answer_public_api(product, dev, solver):
    P = product
    for e_ball, e_ground in ((0.6, 0.0), (0.0, 0.6), (0.3, 0.6)):
        e = max(e_ball, e_ground)
        wid = _ball_world(P, solver, e_ball, e_ground)
        P.s2World_EnableRestitution(wid, True)
        dw = device.DeviceWorld.attach(dev, wid)
        bounces = 0
        v0 = np.float32(0.0)
        for step in range(150):
            P.s2World_Step(wid, DT, 4, 2, True)
            rows = dw.download_all_bodies(2)
            c = dw.download_contacts(8)
            v = rows["linearVelocity"][1, 1]
            live = c[c["pointCount"] > 0]
            if len(live):
                assert live["restitution"][0] == np.float32(e)
                lam = live["points"]["normalImpulse"][0, 0]
                if lam > 0 and v0 < -1.0:
                    want = -np.float32(e) * v0
                    assert abs(v - want) <= REL * abs(want), (step, v, want)
                    bounces += 1
            v0 = v
        assert bounces >= 1, f"{solver} e={e}: no bounce"
        P.s2DestroyWorld(wid)


# ---- off is off, and toggling -------------------------------------------------------------------------------------------

def _state(dw):
    rows = dw.download_all_bodies(dw.counters().bodyCapacity)
    assert len(rows) > 1
    return np.concatenate([rows["position"].ravel(), rows["rot"].ravel(), rows["linearVelocity"].ravel(),
                           rows["angularVelocity"].ravel()]).view(np.uint32)


def _twin_steps(P, dev, make, solver, steps, toggle=None):
    """Two copies of a scene, restitution enabled on the second (from the start, or per `toggle(step)`); asserts every step
    bit-identical. Returns the second world's counters."""
    a, b = make(P, solver), make(P, solver)
    P.s2World_EnableRestitution(b.world, toggle is None)
    da, db = device.DeviceWorld.attach(dev, a.world), device.DeviceWorld.attach(dev, b.world)
    for step in range(steps):
        if toggle is not None:
            P.s2World_EnableRestitution(b.world, toggle(step))
        a.step()
        b.step()
        assert np.array_equal(_state(da), _state(db)), f"{solver}: step {step} differs"
    c = db.counters()
    a.destroy()
    b.destroy()
    return c


@pytest.mark.parametrize("solver", VARIANTS)
def test_on_with_nothing_to_bounce_is_bit_identical(product, dev, solver):
    P = product
    # every e = 0: the 5 050-box pyramid and the collision zoo
    _twin_steps(P, dev, lambda L, s: scenes.pyramid(L, s, base_count=100), solver, 12)
    _twin_steps(P, dev, lambda L, s: scenes.collision_zoo(L, s), solver, 40)
    # every e = 1 on a resting pyramid: gravity alone gives approach speeds far below the 1 m/s threshold. (Jacobi blows a
    # pyramid apart within a few steps, test_solver_stage_gpu.py, and its boxes really do bounce; PGS's pyramid settles with
    # approach speeds above 1 m/s from about step 30)
    if solver != "Jacobi":
        _twin_steps(P, dev, lambda L, s: scenes.pyramid(L, s, base_count=20, restitution=1.0), solver, 25)


def test_toggling_recaptures_and_returns_to_the_production_path(product, dev):
    P = product
    # a resting pyramid with e = 0.5: nothing qualifies, so the results stay identical while the graph is re-captured at
    # every change of the setting
    make = lambda L, s: scenes.pyramid(L, s, base_count=20, restitution=0.5)  # noqa: E731
    plain = _twin_steps(P, dev, make, "TGS_Soft", 60, toggle=lambda step: False)
    toggled = _twin_steps(P, dev, make, "TGS_Soft", 60, toggle=lambda step: 20 <= step < 40)
    assert toggled.graphCaptures >= plain.graphCaptures + 2, (plain.graphCaptures, toggled.graphCaptures)
    assert toggled.graphReplays > 0

    # turning it on mid-run changes the very next step of a falling ball
    wa, wb = _ball_world(P, "TGS_Soft", 1.0, 0.0), _ball_world(P, "TGS_Soft", 1.0, 0.0)
    da, db = device.DeviceWorld.attach(dev, wa), device.DeviceWorld.attach(dev, wb)
    differed = None
    for step in range(120):
        if step == 30:
            P.s2World_EnableRestitution(wb, True)
        P.s2World_Step(wa, DT, 4, 2, True)
        P.s2World_Step(wb, DT, 4, 2, True)
        if differed is None and not np.array_equal(_state(da), _state(db)):
            differed = step
    assert differed is not None and differed >= 30
    P.s2DestroyWorld(wa)
    P.s2DestroyWorld(wb)


def test_threshold_validation(product, dev):
    P = product
    wid = _ball_world(P, "TGS_Soft", 1.0, 0.0, height=0.02)  # impact ~0.6 m/s: below the default threshold
    P.s2World_EnableRestitution(wid, True)
    for bad in (-1.0, float("nan"), float("inf")):
        P.s2World_SetRestitutionThreshold(wid, bad)  # rejected: the threshold stays 1 m/s
    dw = device.DeviceWorld.attach(dev, wid)
    top = 0.0
    for _ in range(60):
        P.s2World_Step(wid, DT, 4, 2, True)
        top = max(top, float(dw.download_all_bodies(2)["linearVelocity"][1, 1]))
    assert top < 0.2, "bounced below the default threshold"
    P.s2World_SetRestitutionThreshold(wid, 0.05)
    wid2 = _ball_world(P, "TGS_Soft", 1.0, 0.0, height=0.02)
    P.s2World_EnableRestitution(wid2, True)
    P.s2World_SetRestitutionThreshold(wid2, 0.05)
    dw2 = device.DeviceWorld.attach(dev, wid2)
    top = 0.0
    for _ in range(60):
        P.s2World_Step(wid2, DT, 4, 2, True)
        top = max(top, float(dw2.download_all_bodies(2)["linearVelocity"][1, 1]))
    assert top > 0.3, "did not bounce above a lowered threshold"
    P.s2DestroyWorld(wid)
    P.s2DestroyWorld(wid2)


# ---- batched field with resident regions ---------------------------------------------------------------------------------

def test_field_with_bouncing_piles_matches_oracle(reference, dev):
    """pyramid_field rows (independent piles: resident regions) with every third pile's contacts at e = 1 and a kick,
    one TGS_Soft stage against the oracle in the device's order."""
    R = reference
    O = port.load()
    sc = scenes.pyramid_field(R, "TGS_Soft", count=24, base_count=6)
    for _ in range(20):
        sc.step(DT, 4, 2, True)
    R.step_collide(sc.world)
    bodies = body_rows_from_ref(*R.bodies(sc.world))
    contacts, _ = contact_rows_from_ref(*R.contacts(sc.world))
    joints = joint_rows_from_ref(*R.joints(sc.world))
    sc.destroy()
    pile = contacts["bodyB"] // 21  # 21 boxes per pile of base 6, created pile by pile after the ground
    contacts["restitution"] = np.where(pile % 3 == 0, 1.0, 0.0).astype(np.float32)
    moving = bodies["invMass"] != 0
    bodies["linearVelocity"][moving, 1] -= np.float32(2.0)
    ctx = device.make_context("TGS_Soft", DT, 4, 2)
    dw = dev.create_world(capi.SOLVER["TGS_Soft"])
    dw.upload_bodies(bodies, len(bodies))
    dw.upload_joints(joints, len(joints))
    dw.upload_contacts(contacts)
    dw.set_restitution(True)
    dw.solve(ctx)
    got = dw.download_all_bodies(len(bodies))
    got_contacts = dw.download_contacts(len(contacts))
    order, _ = dw.solve_order(len(contacts) + len(joints))
    counters = dw.counters()
    dw.destroy()
    assert counters.regionCount > 0
    ob, oc, oj, n = ro.solve(O, capi.SOLVER["TGS_Soft"], bodies, contacts, joints, ctx, order=order)
    assert n > 0
    _compare(got, got_contacts, ob, oc, bodies, contacts)
