"""GPU: the broad phase's pair table (which pairs have a contact, in which (A, B) order) against the reference's, every
step, on the wide hierarchy the pair search walks (csrc/device/broadphase.cu).

The runs go through the state hand-over of test_multistep_gpu.py: every step the device's body state is loaded into the
reference world, the reference's own collide runs, and the contact tables are compared; the reference is then advanced
with the oracle's solve in the device's order, so both sides keep seeing the same fat AABBs. The hierarchy is rebuilt
every 17th pass (S2B_TREE_REUSE_LIMIT = 16 refit-only passes in between) and whenever shapes are created or destroyed."""
import ctypes as C

import numpy as np
import pytest

from oracle import port
from oracle import ref as refmod
from solver2d_b200 import capi, device, scenes
from test_multistep_gpu import _run
from helpers import (contact_rows_from_ref, body_rows_from_ref, joint_rows_from_ref, bit_equal, load_bodies_into_ref,
                     ref_delta_positions, store_oracle_bodies)

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0
REUSE_LIMIT = 16  # S2B_TREE_REUSE_LIMIT
# passes needed for a run to have refitted a reused hierarchy and rebuilt it at least once after the first build
PASSES_WITH_REBUILD = REUSE_LIMIT + 2


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


def test_pair_table_pyramid_5k_every_step(reference, product, dev):
    """5 050 boxes, 48 steps: refit-only passes and rebuilds while the pile settles."""
    c = _run(reference, product, dev, scenes.pyramid, "TGS_Soft", 48, 4, 2, dict(base_count=100))
    assert c.pairPassCount >= PASSES_WITH_REBUILD


def test_pair_table_bench_pyramid_every_step(reference, product, dev):
    """The bench's 100 128-box pyramid (base 447), 32 steps (the lattice stands still for the first few)."""
    c = _run(reference, product, dev, scenes.pyramid, "TGS_Soft", 32, 4, 2, dict(base_count=447))
    assert c.pairPassCount >= PASSES_WITH_REBUILD
    assert c.contactCount > 290000


def _row(lib, solver, count):
    """`count` shapes: a static ground box and count - 1 unit boxes dropped onto it in two staggered rows (count = 1: one
    box falling on its own)."""
    world = lib.create_world(solver)
    sc = scenes.Scene(lib, world, name=f"row{count}")
    if count > 1:
        sc.bodies.append(scenes._ground(lib, world, 0.5 * count + 2.0))
    bd = scenes.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    sd = scenes.default_shape_def()
    sd.density = 1.0
    box = lib.s2MakeSquare(0.5)
    for k in range(count - 1 if count > 1 else 1):
        bd.position = capi.Vec2(1.05 * (k // 2) + 0.5 * (k % 2), 0.6 + 1.2 * (k % 2))
        bid = lib.s2CreateBody(world, C.byref(bd))
        lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
        sc.bodies.append(bid)
    return sc


@pytest.mark.parametrize("count", [1, 2, 8, 9, 17])
def test_pair_table_few_shapes(reference, product, dev, count):
    """1, 2, W, W + 1 and 2W + 1 shapes (W = 8 children per wide node): a root with few children, a root that is a leaf,
    a second wide level."""
    c = _run(reference, product, dev, lambda lib, solver: _row(lib, solver, count), "TGS_Soft", 40, 4, 2, {})
    if count > 2:
        assert c.contactCount >= count - 1


def _one_spot(lib, solver, count=300):
    """`count` kinematic boxes at one and the same spot (one Morton code), moving together over a row of boxes resting on
    a ground: their fat AABBs all overlap, each of them is a moved proxy whose query walks the whole duplicate-code subtree
    (and makes no pair: a kinematic proxy only pairs with dynamic ones), and the dynamic boxes' queries walk it too."""
    world = lib.create_world(solver)
    sc = scenes.Scene(lib, world, name="one_spot")
    sc.bodies.append(scenes._ground(lib, world, 40.0))
    sd = scenes.default_shape_def()
    sd.density = 1.0
    box = lib.s2MakeSquare(0.5)
    bd = scenes.default_body_def()
    bd.type = capi.KINEMATIC_BODY
    bd.position = capi.Vec2(-20.0, 4.0)
    bd.linearVelocity = capi.Vec2(1.0, 0.0)
    for _ in range(count):
        bid = lib.s2CreateBody(world, C.byref(bd))
        lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
        sc.bodies.append(bid)
    bd = scenes.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    for k in range(40):
        bd.position = capi.Vec2(-30.0 + 1.5 * k, 0.6 + (k % 3))
        bid = lib.s2CreateBody(world, C.byref(bd))
        lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
        sc.bodies.append(bid)
    return sc


def test_pair_table_duplicate_morton_codes(reference, product, dev):
    c = _run(reference, product, dev, _one_spot, "TGS_Soft", 40, 4, 2, {})
    assert c.pairPassCount >= PASSES_WITH_REBUILD
    assert c.contactCount >= 26


def test_pair_table_large_mover(reference, product, dev):
    """The hub container: four scene-sized walls on one rotating body among 400 small boxes. The walls take the
    leaf-side query (s2bFindPairsLarge), which needs the root box of the refit."""
    c = _run(reference, product, dev, scenes.tumbler, "TGS_Soft", 40, 4, 2, dict(grid=20, half_extent=4.0))
    assert c.pairPassCount >= PASSES_WITH_REBUILD


def _moving_mix(lib, solver):
    """Both-moved de-duplication and the body-type rules: falling boxes that pass each other (both proxies moved), a
    kinematic slab sliding through resting boxes (kinematic against dynamic) and over a static box (never a pair)."""
    world = lib.create_world(solver)
    sc = scenes.Scene(lib, world, name="moving_mix")
    ground = scenes._ground(lib, world, 30.0)
    sc.bodies.append(ground)
    sd = scenes.default_shape_def()
    sd.density = 1.0
    bd = scenes.default_body_def()
    bd.position = capi.Vec2(8.0, 3.0)
    static = lib.s2CreateBody(world, C.byref(bd))
    lib.s2CreatePolygonShape(static, C.byref(sd), C.byref(lib.s2MakeBox(0.5, 0.5)))
    sc.bodies.append(static)
    bd = scenes.default_body_def()
    bd.type = capi.KINEMATIC_BODY
    bd.position = capi.Vec2(-10.0, 2.5)
    bd.linearVelocity = capi.Vec2(20.0, 0.0)
    kin = lib.s2CreateBody(world, C.byref(bd))
    lib.s2CreatePolygonShape(kin, C.byref(sd), C.byref(lib.s2MakeBox(1.0, 0.25)))
    sc.bodies.append(kin)
    bd = scenes.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    box = lib.s2MakeSquare(0.4)
    for k in range(24):
        bd.position = capi.Vec2(-6.0 + 0.9 * (k % 12), 0.45 + 5.0 * (k // 12))
        bd.linearVelocity = capi.Vec2(2.0 if k % 2 else -2.0, 0.0) if k >= 12 else capi.Vec2(0.0, 0.0)
        bid = lib.s2CreateBody(world, C.byref(bd))
        lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
        sc.bodies.append(bid)
    return sc


def test_pair_table_both_moved_and_body_types(reference, product, dev):
    c = _run(reference, product, dev, _moving_mix, "TGS_Soft", 60, 4, 2, {})
    assert c.pairPassCount >= PASSES_WITH_REBUILD


def test_pair_table_shapes_destroyed_and_recreated(reference, product, dev):
    """A 36-box pyramid; between steps boxes are destroyed, created in the freed slots elsewhere, and destroyed and
    re-created in the same step, identically in both worlds. Every step the pair table is compared with the reference's."""
    R, P = reference, product
    O = port.load()
    solver = "TGS_Soft"
    sr = scenes.pyramid(R, solver, base_count=8)
    sp = scenes.pyramid(P, solver, base_count=8)
    dev.lib.s2World_Flush.restype = None
    dev.lib.s2World_Flush.argtypes = [capi.WorldId]
    dev.lib.s2World_Flush(sp.world)
    dw = device.DeviceWorld.attach(dev, sp.world)
    ctx = device.make_context(solver, DT, 4, 2, True)

    def create(sc, x, y):
        lib = sc.lib
        bd = scenes.default_body_def()
        bd.type = capi.DYNAMIC_BODY
        bd.position = capi.Vec2(x, y)
        sd = scenes.default_shape_def()
        sd.density = 1.0
        bid = lib.s2CreateBody(sc.world, C.byref(bd))
        lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(lib.s2MakeSquare(0.5)))
        sc.bodies.append(bid)

    def destroy(sc, ks):
        for k in sorted(ks, reverse=True):
            sc.lib.s2DestroyBody(sc.bodies.pop(k))

    edits = {
        8: lambda sc: destroy(sc, [3, 10, 20]),
        12: lambda sc: (create(sc, -2.0, 9.0), create(sc, 0.2, 9.5), create(sc, 6.0, 0.6)),
        20: lambda sc: (destroy(sc, [5]), create(sc, 1.0, 10.0), create(sc, 1.3, 12.0)),
        28: lambda sc: (destroy(sc, [len(sc.bodies) - 1]), create(sc, -5.0, 0.6)),
    }
    F = refmod.BODY_F
    for step in range(48):
        if step in edits:
            edits[step](sr)
            edits[step](sp)
            dev.lib.s2World_Flush(sp.world)
        cap = R.capacities(sr.world)["bodyCap"]
        load_bodies_into_ref(R, sr.world, dw.download_all_bodies(cap))
        R.step_collide(sr.world)
        sp.step(DT, 4, 2, True)

        cf, ci = R.contacts(sr.world)
        rows_slot, slots = contact_rows_from_ref(cf, ci)
        keys = (np.minimum(rows_slot["shapeA"], rows_slot["shapeB"]).astype(np.uint64) << np.uint64(32)) | \
            np.maximum(rows_slot["shapeA"], rows_slot["shapeB"]).astype(np.uint64)
        perm = np.argsort(keys, kind="stable")
        rows_key = rows_slot[perm]
        got = dw.download_contacts(len(rows_key) + 64)
        assert len(got) == len(rows_key), f"step {step}: contact tables differ in size"
        assert np.array_equal(got["shapeA"], rows_key["shapeA"]) and np.array_equal(got["shapeB"], rows_key["shapeB"]), \
            f"step {step}: pair set or (A, B) order differs"

        # advance the reference with the oracle's solve in the device's order (see test_multistep_gpu._run)
        bodies = body_rows_from_ref(*R.bodies(sr.world))
        joints = joint_rows_from_ref(*R.joints(sr.world))
        order, _ = dw.solve_order(len(rows_key) + len(joints) + 16, max_groups=200000)
        ob, oc, _, odp = O.solve(capi.SOLVER[solver], bodies, rows_key, joints, ctx, order=order,
                                 dp=ref_delta_positions(R, sr.world))
        store_oracle_bodies(R, sr.world, ob, odp)
        imp = np.zeros((cf.shape[0], 4), dtype=np.float32)
        imp[slots[perm], 0] = oc["points"]["normalImpulse"][:, 0]
        imp[slots[perm], 1] = oc["points"]["tangentImpulse"][:, 0]
        imp[slots[perm], 2] = oc["points"]["normalImpulse"][:, 1]
        imp[slots[perm], 3] = oc["points"]["tangentImpulse"][:, 1]
        R.load_contact_impulses(sr.world, imp)
        R.step_finalize(sr.world)
        post = dw.download_all_bodies(cap)
        rf, ri = R.bodies(sr.world)
        v = ri[:, 0] == 1
        assert bit_equal(post["position"][v], rf[v, F["position"]:F["position"] + 2]), f"step {step}: bodies diverged"
    c = dw.counters()
    assert c.pairPassCount >= PASSES_WITH_REBUILD
    sr.destroy()
    sp.destroy()


# binary hierarchy height (s2World_GetStatistics().treeHeight) after the first step of a fixed scene, as the binary refit
# reported it before the hierarchy became wide
TREE_HEIGHT_FIXTURE = {"pyramid447": 18, "tumbler100": 16}


@pytest.mark.parametrize("scene", sorted(TREE_HEIGHT_FIXTURE))
def test_tree_height_unchanged(product, dev, scene):
    sc = scenes.pyramid(product, "TGS_Soft", base_count=447) if scene == "pyramid447" else scenes.tumbler(product, "TGS_Soft", grid=100)
    dw = device.DeviceWorld.attach(dev, sc.world)
    sc.step(DT, 4, 2, True)
    dw.sync()
    assert dw.counters().treeHeight == TREE_HEIGHT_FIXTURE[scene]
    sc.destroy()
