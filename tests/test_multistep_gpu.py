"""GPU: TIGHT multi-step parity of the free-running PRODUCTION path (public C API, colour schedule, persisted colours,
contact-table merges, feature-id impulse matching, CUDA-graph replay with the schedule skipped while the live constraint
set stands) — every step, every body, every manifold impulse, tolerance 0.

Gauss-Seidel is order sensitive, so the device cannot be compared with the free-running reference directly (SURVEY §7 H1).
Instead every step is checked on its own against the reference pipeline fed with the device's state and order:

    device state before the step  ->  loaded into the unmodified reference world (oracle/_ref, s2ref_load_body_state)
    reference stages 1-3          ->  s2ref_step_collide: pair update, narrow phase, impulse matching   (world.c:123-168)
    device                        ->  one s2World_Step through the public API
    solver stage                  ->  the plain-C oracle (pinned bit for bit to the reference, tests/test_oracle_cpu.py)
                                      replayed in the order the device reports for THIS step
    reference stage 4             ->  s2ref_step_finalize on the oracle's result                         (world.c:258-301)
    compare                       ->  bodies (position, rotation, velocities, origin) and manifold / joint impulses, bitwise

The reference world is advanced with the oracle's result (bodies and warm-start impulses), so its broad phase, contact pool
and manifold ids evolve exactly as if the reference had solved in the device's order."""
import numpy as np
import pytest

from helpers import (STICKY_FIELDS, bit_equal, body_rows_from_ref, carry_sticky_friction, contact_rows_from_ref,
                     joint_rows_from_ref, load_bodies_into_ref, ref_delta_positions, store_oracle_bodies)
from oracle import port
from oracle import ref as refmod
from solver2d_b200 import capi, device, scenes

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


CONTACT_FIELDS = ("normal", "friction", "cacheCount", "cacheIndexA", "cacheIndexB", "cacheMetric")
POINT_FIELDS = ("localAnchorA", "localAnchorB", "separation", "id", "persisted")


def _same(g, w):
    g, w = np.asarray(g), np.asarray(w)
    return bit_equal(g, w) if g.dtype == np.float32 else bool(np.array_equal(g, w))


def _run(R, P, dev, recipe, solver, steps, vel, pos, kw, min_replays=0, setup=None, observe=None, oracle=None,
         as_joints=None, before_step=None, after_step=None):
    """`oracle`: the oracle to replay (default oracle.port's); `as_joints(joints, sc)`: turns the reference's joint rows
    into the device's (stand-ins); `before_step(step, (lib, scene) pairs)`: public-API calls made on both worlds before a
    step; `after_step(dw)`: called after every checked step."""
    O = port.load() if oracle is None else oracle
    sr = recipe(R, solver, **kw)
    sp = recipe(P, solver, **kw)
    # push the freshly built scene to the device now (s2World_Step would do it): the first step is checked like any other
    dev.lib.s2World_Flush.restype = None
    dev.lib.s2World_Flush.argtypes = [capi.WorldId]
    dev.lib.s2World_Flush(sp.world)
    dw = device.DeviceWorld.attach(dev, sp.world)
    if setup is not None:
        setup(dw)
    ctx = device.make_context(solver, DT, vel, pos, True)
    worst = {}
    sticky = solver == "TGS_Sticky"
    solved = {}  # TGS_Sticky: the oracle's rows of the previous step, by pair key
    for step in range(steps):
        if before_step is not None:
            before_step(step, ((R, sr), (P, sp)))
            dev.lib.s2World_Flush(sp.world)
        cap = R.capacities(sr.world)["bodyCap"]
        pre = dw.download_all_bodies(cap)
        load_bodies_into_ref(R, sr.world, pre)
        R.step_collide(sr.world)

        sp.step(DT, vel, pos, True)

        bodies = body_rows_from_ref(*R.bodies(sr.world))
        cf, ci = R.contacts(sr.world)
        rows_slot, slots = contact_rows_from_ref(cf, ci)
        keys = (np.minimum(rows_slot["shapeA"], rows_slot["shapeB"]).astype(np.uint64) << np.uint64(32)) | \
            np.maximum(rows_slot["shapeA"], rows_slot["shapeB"]).astype(np.uint64)
        perm = np.argsort(keys, kind="stable")
        rows_key = rows_slot[perm]
        if sticky:
            carry_sticky_friction(rows_key, keys[perm], solved)
        if observe is not None:
            observe(R, sr.world, rows_key)
        joints = joint_rows_from_ref(*R.joints(sr.world))
        if as_joints is not None:
            joints = as_joints(joints, sr)

        got_contacts = dw.download_contacts(len(rows_key) + 64)
        assert len(got_contacts) == len(rows_key), f"step {step}: contact tables differ in size"
        assert np.array_equal(got_contacts["shapeA"], rows_key["shapeA"]) and np.array_equal(got_contacts["shapeB"], rows_key["shapeB"]), \
            f"step {step}: pair set or (A, B) order differs"
        assert np.array_equal(got_contacts["pointCount"], rows_key["pointCount"]), f"step {step}: manifold point counts differ"

        order, sizes = dw.solve_order(len(rows_key) + len(joints) + 16, max_groups=200000)
        ob, oc, oj, odp = O.solve(capi.SOLVER[solver], bodies, rows_key, joints, ctx, order=order,
                                  dp=ref_delta_positions(R, sr.world))

        # advance the reference world with the oracle's result
        F = refmod.BODY_F
        store_oracle_bodies(R, sr.world, ob, odp)
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

        # compare
        post = dw.download_all_bodies(cap)
        rf, ri = R.bodies(sr.world)
        v = ri[:, 0] == 1
        for name, col, width in (("position", F["position"], 2), ("rot", F["rot"], 2), ("linearVelocity", F["v"], 2),
                                 ("origin", F["origin"], 2)):
            g = np.ascontiguousarray(post[name][v]).reshape(int(v.sum()), -1)
            o = np.ascontiguousarray(rf[v, col:col + width])
            if not bit_equal(g, o):
                worst[name] = max(worst.get(name, 0.0), float(np.abs(g - o).max()))
        if not bit_equal(post["angularVelocity"][v], rf[v, F["w"]]):
            worst["w"] = max(worst.get("w", 0.0), float(np.abs(post["angularVelocity"][v] - rf[v, F["w"]]).max()))
        # the delta position a stage leaves (non-zero for a kinematic body under XPBD)
        got_dp = dw.download_delta_positions(cap)
        if not bit_equal(got_dp[v], rf[v, F["dp"]:F["dp"] + 2]):
            worst["deltaPosition"] = float(np.abs(got_dp[v] - rf[v, F["dp"]:F["dp"] + 2]).max())
        # the contact table as the narrow phase left it (the reference's post-collide rows), and what the solver wrote back
        for name in CONTACT_FIELDS:
            if not _same(got_contacts[name], rows_key[name]):
                worst["contact " + name] = 1.0
        for name in POINT_FIELDS:
            if not _same(got_contacts["points"][name], rows_key["points"][name]):
                worst["contact point " + name] = 1.0
        persisted_want = oc["frictionPersisted"] if sticky else rows_key["frictionPersisted"]
        if not _same(got_contacts["frictionPersisted"], persisted_want):
            worst["contact frictionPersisted"] = 1.0
        if sticky:
            for name in STICKY_FIELDS:
                if not _same(got_contacts["points"][name], oc["points"][name]):
                    worst["contact point " + name] = 1.0
        # shape AABBs and fat AABBs written by the finalize stage (s2bFinalizeShapes)
        sf, si = R.shapes(sr.world)
        aabb, fat, _ = dw.download_shape_boxes(sf.shape[0])
        sv = si[:, refmod.SHAPE_I["valid"]] == 1
        n = min(len(aabb), len(sv))
        assert not sv[n:].any(), f"step {step}: the device holds fewer shape slots than the reference"
        if not _same(aabb[:n][sv[:n]], sf[:n, 0:4][sv[:n]]):
            worst["shape aabb"] = 1.0
        if not _same(fat[:n][sv[:n]], sf[:n, 4:8][sv[:n]]):
            worst["shape fatAABB"] = 1.0
        live = rows_key["pointCount"] > 0
        for name in ("normalImpulse", "tangentImpulse"):
            if not bit_equal(got_contacts["points"][name][live], oc["points"][name][live]):
                worst[name] = max(worst.get(name, 0.0), float(np.abs(got_contacts["points"][name][live] - oc["points"][name][live]).max()))
        if len(oj):
            got_joints = dw.download_joints(len(oj))
            jlive = (joints["flags"] & 1) == 1
            for name in ("impulse", "motorImpulse", "lowerImpulse", "upperImpulse"):
                if not bit_equal(got_joints[name][jlive], oj[name][jlive]):
                    worst["joint " + name] = 1.0
        assert not worst, f"{solver} step {step}: device != reference pipeline replayed in the device's order: {worst}"
        if after_step is not None:
            after_step(dw)
    c = dw.counters()
    assert c.graphReplays >= min_replays, f"the solver stage was replayed as a graph only {c.graphReplays} times"
    sr.destroy()
    sp.destroy()
    return c


def test_config1_every_step_bit_exact(reference, product, dev):
    """BASELINE config 1 (Pyramid, 55 boxes, TGS_Soft, 4 sub-steps), 120 free-running steps."""
    c = _run(reference, product, dev, scenes.pyramid, "TGS_Soft", 120, 4, 2, dict(base_count=10), min_replays=60)
    assert c.constraintCount > 100


def test_pyramid_5k_every_step_bit_exact(reference, product, dev):
    """5 050 boxes / ~15 000 contact constraints, 60 free-running steps: several thread blocks, contact-table changes while
    the pile settles, graph replays with the schedule skipped in between."""
    c = _run(reference, product, dev, scenes.pyramid, "TGS_Soft", 60, 4, 2, dict(base_count=100))
    assert c.constraintCount > 14000


def test_joints_and_contacts_every_step_bit_exact(reference, product, dev):
    """Bridges (revolute chains) with boxes dropped on them: joints and contacts in one colouring, contacts appearing and
    disappearing every few steps."""
    c = _run(reference, product, dev, scenes.joint_contact_stress, "TGS_Soft", 90, 4, 2, dict(bridges=3, planks=24, grid=9))
    assert c.jointCount == 75


def _steps(solver, steps):
    """Jacobi blows scenes apart in the reference as well: a few steps show it, more only measure the explosion."""
    return 12 if solver == "Jacobi" else steps


@pytest.mark.parametrize("solver", ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky",
                                    "TGS_NGS", "XPBD"])
def test_variants_every_step_bit_exact(reference, product, dev, solver):
    """TGS_Sticky also carries the friction anchors and normals its solve writes into the manifolds from step to step
    (helpers.carry_sticky_friction); the device's are compared with the oracle's every step."""
    c = _run(reference, product, dev, scenes.pyramid, solver, _steps(solver, 40), 4, 2, dict(base_count=20))
    assert c.constraintCount > (0 if solver == "Jacobi" else 300)  # Jacobi's pyramid is mostly apart after 12 steps


def _zoo_observer(seen):
    """Records, from the reference's post-collide state, which manifold kinds had points, whether a pair was stored in
    flipped order (primary shape with the higher index) and whether fat AABBs overlapped without a contact where only the
    shape filter can have refused it (different bodies, not both static, not segment against segment)."""
    names = {0: "capsule", 1: "circle", 2: "polygon", 3: "segment"}

    def observe(R, wid, rows):
        sf, si = R.shapes(wid)
        bf, bi = R.bodies(wid)
        I = refmod.SHAPE_I
        types = si[:, I["type"]]
        live = rows["pointCount"] > 0
        for a, b in zip(rows["shapeA"][live], rows["shapeB"][live]):
            seen.setdefault("kinds", set()).add((names[types[a]], names[types[b]]))
        seen["flipped"] = seen.get("flipped", 0) + int((rows["shapeA"] > rows["shapeB"]).sum())
        valid = np.nonzero(si[:, I["valid"]] == 1)[0]
        fat = sf[valid, 4:8]
        over = (fat[:, None, 0] <= fat[None, :, 2]) & (fat[None, :, 0] <= fat[:, None, 2]) & \
               (fat[:, None, 1] <= fat[None, :, 3]) & (fat[None, :, 1] <= fat[:, None, 3])
        body = si[valid, I["body"]]
        static = bi[body, refmod.BODY_I["type"]] == capi.STATIC_BODY
        seg = types[valid] == 3
        cand = over & (body[:, None] != body[None, :]) & ~(static[:, None] & static[None, :]) & ~(seg[:, None] & seg[None, :])
        cand = np.triu(cand, 1)
        pairs = set(zip(np.minimum(rows["shapeA"], rows["shapeB"]).tolist(), np.maximum(rows["shapeA"], rows["shapeB"]).tolist()))
        ia, ib = np.nonzero(cand)
        seen["filtered"] = seen.get("filtered", 0) + sum((int(valid[x]), int(valid[y])) not in pairs for x, y in zip(ia, ib))
    return observe


@pytest.mark.parametrize("solver", capi.SOLVER_TYPES)
def test_collision_zoo_every_step_bit_exact(reference, product, dev, solver):
    """scenes.collision_zoo: all nine manifold kinds, flipped pairs, dynamic segments, rounded polygons and 5-8-gons,
    compound bodies, mixed frictions and every filter rule, under every solver variant."""
    seen = {}
    _run(reference, product, dev, scenes.collision_zoo, solver, _steps(solver, 60), 4, 2, {}, observe=_zoo_observer(seen))
    assert seen["flipped"] > 0, "no pair was stored in flipped order"
    assert seen["filtered"] > 0, "no fat-AABB overlap was refused by the filter"
    if solver != "Jacobi":
        kinds = {("circle", "circle"), ("capsule", "circle"), ("capsule", "capsule"), ("polygon", "circle"),
                 ("polygon", "capsule"), ("polygon", "polygon"), ("segment", "circle"), ("segment", "capsule"),
                 ("segment", "polygon")}
        assert kinds <= seen["kinds"], f"manifold kinds never touching: {sorted(kinds - seen['kinds'])}"


def test_falling_boxes_every_step_bit_exact(reference, product, dev):
    """Boxes thrown sideways: proxies leave their fat AABBs, pairs are created and destroyed, manifolds gain and lose
    points — the schedule is rebuilt on exactly the steps the device flags."""
    def recipe(lib, solver, **kw):
        sc = scenes.vertical_stack(lib, solver, count=5, columns=4)
        for k, bid in enumerate(sc.bodies[1:]):
            if k % 5 >= 3:
                lib.s2Body_SetLinearVelocity(bid, capi.Vec2(3.0 if (k // 5) % 2 == 0 else -3.0, 1.0))
        return sc
    c = _run(reference, product, dev, recipe, "TGS_Soft", 120, 4, 2, {})
    assert c.pairPassCount > 5


def test_kinematic_platforms_under_regions_every_step_bit_exact(reference, product, dev):
    """Piles standing on KINEMATIC platforms that slide sideways, region-local schedule forced. A kinematic body conflicts
    with nothing (no constraint moves it) but its pose changes every sub-step, integrated by the block that owns it: a
    constraint that reads it from another block's region-local phase would race with that pass. Such constraints have to
    run in the device-wide steps (s2bClassifyItemsKernel)."""
    def recipe(lib, solver, **kw):
        import ctypes as C
        world = lib.create_world(solver)
        sc = scenes.Scene(lib, world, name="kinematic_platforms")
        h, base = 0.5, 16
        box = lib.s2MakeSquare(h)
        sd = scenes.default_shape_def()
        sd.density = 1.0
        for k in range(4):
            x0 = k * 30.0
            bd = scenes.default_body_def()
            bd.type = capi.KINEMATIC_BODY
            bd.position = capi.Vec2(x0, -1.0)
            bd.linearVelocity = capi.Vec2(0.6 if k % 2 == 0 else -0.4, 0.0)
            gid = lib.s2CreateBody(world, C.byref(bd))
            plat = lib.s2MakeBox(0.5 * base + 2.0, 1.0)
            lib.s2CreatePolygonShape(gid, C.byref(sd), C.byref(plat))
            sc.bodies.append(gid)
            bd = scenes.default_body_def()
            bd.type = capi.DYNAMIC_BODY
            for i in range(base):
                y = (2.0 * i + 1.0) * h
                for j in range(i, base):
                    x = (i + 1.0) * h + 2.0 * (j - i) * h - h * base
                    bd.position = capi.Vec2(x0 + x, y)
                    bid = lib.s2CreateBody(world, C.byref(bd))
                    lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
                    sc.bodies.append(bid)
        return sc
    c = _run(reference, product, dev, recipe, "TGS_Soft", 40, 4, 2, {}, setup=lambda dw: dw.set_regions(2))
    assert c.regionCount >= 3 and c.cutCount >= 40
