"""GPU: the region-local schedule at its edges, every step against the oracle replayed in the device's solve order
(test_multistep_gpu._run: reference collide, oracle, reference finalize, tolerance 0). Every case asserts the edge it
reached through the counters (regionCount, cutCount, maxRegionBodies, residentRegions).

* The whole-island rule of s2bAssignRegionsKernel: an island of at most max(2 * chunk, wholeIslandBodies) bodies stays in
  one region, chunk = ceil(owned bodies / regions). Islands of exactly 2 * chunk and 2 * chunk + 1 bodies under
  S2B_WHOLE_ISLAND=1, sized from the grid the device reached; islands above 2 * chunk with S2B_WHOLE_ISLAND at their size
  and one less; the default of 1 200 with islands of 1 200 and 1 201.
* The grid cap of 511 regions (region ids share a 16-bit sort key with the colour). It cannot be reached on an H100: the
  persistent kernels use 94 to 128 registers per thread at 512 threads per block, so one block fits an SM and the grid stops
  at the SM count (132) whatever S2B_SOLVE_BLOCKS_PER_SM asks for. The test asks for 4 blocks per SM on a world that wants
  more than 511 blocks and asserts the grid it reached.
* Resident regions (TGS_Soft keeps a region's bodies in shared memory when nothing is solved device-wide): the capacity of
  3 072 bodies on both sides, each side also byte for byte against the same scene with S2B_RESIDENT=0; a field of many
  regions near the capacity; a joint, a kinematic body, a hub, an overflow group and a cut set each switching the path off
  on the step they appear and back on after they go, with graph replays in between; warm start off and the ticketed
  (dataflow) passes, which never take it."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from solver2d_b200 import capi, device, scenes
from solver2d_b200.capi import Vec2
from test_multistep_gpu import _run

pytestmark = pytest.mark.gpu
RES_MAX = 3072  # S2B_RES_MAX_BODIES (persistent.cuh)


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


def _with_env(recipe, **env):
    """`recipe` with environment knobs set for the world's creation only."""
    def build(lib, solver, **kw):
        old = {k: os.environ.get(k) for k in env}
        os.environ.update({k: str(v) for k, v in env.items()})
        try:
            return recipe(lib, solver, **kw)
        finally:
            for k, v in old.items():
                if v is None:
                    del os.environ[k]
                else:
                    os.environ[k] = v
    return build


def _box(lib, world, kind, x, y, hx=0.5, hy=0.5):
    bd = capi.default_body_def()
    bd.type = kind
    bd.position = Vec2(x, y)
    bid = lib.s2CreateBody(world, C.byref(bd))
    sd = capi.default_shape_def()
    sd.density = 1.0
    lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(lib.s2MakeBox(hx, hy)))
    return bid


def _pile(lib, sc, x0, n):
    """A pyramid of exactly `n` unit boxes centred on x0, standing at y = 0: rows filled from the bottom, the top row
    partial. One island (every box rests on the row below)."""
    base = 1
    while base * (base + 1) // 2 < n:
        base += 1
    made = 0
    for i in range(base):
        for j in range(i, base):
            if made == n:
                return
            sc.bodies.append(_box(lib, sc.world, capi.DYNAMIC_BODY, x0 + (i + 1.0) * 0.5 + (j - i) - 0.5 * base,
                                  (2.0 * i + 1.0) * 0.5))
            made += 1


def piles(sizes, pitch=None):
    """Recipe: piles of the given sizes side by side on one static ground."""
    def recipe(lib, solver, **kw):
        sc = scenes.Scene(lib, lib.create_world(solver), name="piles")
        width = pitch or (2.0 * np.sqrt(2.0 * max(sizes)) + 8.0)
        sc.bodies.append(scenes._ground(lib, sc.world, 0.5 * width * len(sizes) + 10.0))
        for k, n in enumerate(sizes):
            _pile(lib, sc, (k - 0.5 * (len(sizes) - 1)) * width, n)
        return sc
    return recipe


def _first_step(product, dev, recipe, solver="TGS_Soft", regions=None):
    """Counters and valid body count after one step of the product alone."""
    sc = recipe(product, solver)
    dev.lib.s2World_Flush.restype = None
    dev.lib.s2World_Flush.argtypes = [capi.WorldId]
    dev.lib.s2World_Flush(sc.world)
    dw = device.DeviceWorld.attach(dev, sc.world)
    if regions is not None:
        dw.set_regions(regions)
    sc.step(1.0 / 60.0, 4, 2, True)
    c = dw.counters()
    owned = int(((dw.download_all_bodies(c.bodyCapacity)["flags"] & 1) == 1).sum())
    assert owned > 0
    sc.destroy()
    return c, owned


def _chunk(c, owned):
    return max(-(-owned // c.regionCount), 1)


# ---- the whole-island rule ------------------------------------------------------------------------------------------------

def _field_with_fillers(size, fillers):
    """Recipe: two piles of `size` boxes on a static ground and `fillers` circles spread high in the air (islands of one
    that touch nothing during the run), then 6 000 slots created and freed. The free slots widen the grid (it follows the
    body capacity), the fillers set the owned-body count: together they set the chunk apart from the piles."""
    def recipe(lib, solver, **kw):
        sc = piles([size, size])(lib, solver)
        bd = capi.default_body_def()
        bd.type = capi.DYNAMIC_BODY
        sd = capi.default_shape_def()
        sd.density = 1.0
        for k in range(fillers):
            bd.position = Vec2(-100.0 + 2.0 * (k % 100), 200.0 + 2.0 * (k // 100))
            bid = lib.s2CreateBody(sc.world, C.byref(bd))
            lib.s2CreateCircleShape(bid, C.byref(sd), C.byref(capi.Circle(Vec2(0.0, 0.0), 0.25)))
            sc.bodies.append(bid)
        holes = [lib.s2CreateBody(sc.world, C.byref(bd)) for _ in range(6000)]
        for bid in holes:
            lib.s2DestroyBody(bid)
        return sc
    return recipe


@pytest.mark.parametrize("over", [0, 1])
def test_whole_island_at_two_chunks(reference, product, dev, over):
    """Under S2B_WHOLE_ISLAND=1 only the chunk rule applies: islands of 2 * chunk bodies stay whole (no cut set), islands of
    2 * chunk + 1 are cut. Two piles of 2 * 150 + over boxes; the count of filler bodies is chosen from the grid the device
    reaches so that chunk = ceil(owned / regions) = 150."""
    chunk, size = 150, 2 * 150 + over
    fillers = 1000
    for _ in range(8):
        recipe = _with_env(_field_with_fillers(size, fillers), S2B_WHOLE_ISLAND=1)
        c, owned = _first_step(product, dev, recipe, regions=2)
        assert owned == 2 * size + 1 + fillers
        if _chunk(c, owned) == chunk:
            break
        # the middle of the owned counts that give this chunk on this grid
        fillers = max(c.regionCount * chunk - c.regionCount // 2 - 2 * size - 1, 0)
    assert _chunk(c, owned) == chunk, "no filler count settled on the chunk"
    seen = []

    def after(dw):
        k = dw.counters()
        seen.append((k.regionCount, k.cutCount))

    _run(reference, product, dev, recipe, "TGS_Soft", 8, 4, 2, {}, setup=lambda dw: dw.set_regions(2), after_step=after)
    regions, cut = seen[0]
    assert regions == c.regionCount and -(-owned // regions) == chunk and size == 2 * chunk + over
    assert (cut == 0) == (over == 0), f"islands of {size} bodies, chunk {chunk}: cut set of {cut}"


@pytest.mark.parametrize("size,whole,kept", [(600, 600, True), (600, 599, False), (1200, None, True), (1201, None, False)])
def test_whole_island_limit(reference, product, dev, size, whole, kept):
    """Islands larger than 2 * chunk stay whole up to S2B_WHOLE_ISLAND bodies (default 1 200)."""
    recipe = piles([size, size])
    if whole is not None:
        recipe = _with_env(recipe, S2B_WHOLE_ISLAND=whole)
    seen = []
    _run(reference, product, dev, recipe, "TGS_Soft", 6, 4, 2, {}, setup=lambda dw: dw.set_regions(2),
         after_step=lambda dw: seen.append(dw.counters()))
    c = seen[0]
    owned = 2 * size + 1
    assert c.regionCount > 0 and size > 2 * _chunk(c, owned), "the islands must be larger than two chunks"
    assert (c.cutCount == 0) == kept, f"islands of {size}, limit {whole}: cut set of {c.cutCount}"
    if kept:
        assert c.maxRegionBodies >= size


# ---- the grid cap ---------------------------------------------------------------------------------------------------------

def test_grid_cap(reference, product, dev, monkeypatch):
    """S2B_SOLVE_BLOCKS_PER_SM=4 on a field that asks for more than 511 blocks (over 261 632 constraints). On an H100 the
    occupancy of the persistent kernel (one 512-thread block per SM) stops the grid at the SM count, below the cap."""
    monkeypatch.setenv("S2B_SOLVE_BLOCKS_PER_SM", "4")
    seen = []
    _run(reference, product, dev, scenes.pyramid_field, "TGS_Soft", 2, 4, 2, dict(count=90, base_count=45),
         after_step=lambda dw: seen.append(dw.counters()))
    c = seen[-1]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert c.contactCount > 511 * 512, "the field must ask for more than 511 blocks"
    assert c.regionCount == min(sms, 511) and c.cutCount == 0


# ---- resident regions at their capacity -----------------------------------------------------------------------------------

def _twin_check(product, recipe, seen):
    """setup / after_step hooks that step a twin of the scene built with S2B_RESIDENT=0 beside the checked world and compare
    them byte for byte (bodies and contact rows) every step."""
    twin = {}

    def setup(dw):
        twin["sc"] = _with_env(recipe, S2B_RESIDENT=0)(product, "TGS_Soft")

    def after(dev):
        def check(dw):
            sc = twin["sc"]
            sc.step(1.0 / 60.0, 4, 2, True)
            tw = device.DeviceWorld.attach(dev, sc.world)
            c, t = dw.counters(), tw.counters()
            seen.append(c)
            assert t.residentRegions == 0 and t.maxRegionBodies == c.maxRegionBodies
            assert c.bodyCapacity > 0 and t.bodyCapacity == c.bodyCapacity
            assert np.array_equal(dw.download_all_bodies(c.bodyCapacity).view(np.uint8),
                                  tw.download_all_bodies(c.bodyCapacity).view(np.uint8)), \
                "bodies differ from the S2B_RESIDENT=0 run"
            n = c.contactCount + 64
            assert np.array_equal(dw.download_contacts(n).view(np.uint8), tw.download_contacts(n).view(np.uint8)), \
                "contact rows differ from the S2B_RESIDENT=0 run"
        return check
    return setup, after, twin


def _resident_size(product, dev, whole):
    """Boxes of a single pile for which the largest region holds exactly 3 072 bodies: the static ground lands in the pile's
    region or not depending on its place along the curve."""
    c, _ = _first_step(product, dev, _with_env(piles([RES_MAX]), S2B_WHOLE_ISLAND=whole))
    assert c.maxRegionBodies in (RES_MAX, RES_MAX + 1)
    return RES_MAX - (c.maxRegionBodies - RES_MAX)


@pytest.mark.parametrize("extra", [0, 1])
def test_resident_capacity(reference, product, dev, extra):
    """One island kept whole (S2B_WHOLE_ISLAND above its size), its region holding 3 072 bodies (resident) or 3 073 (not),
    20 steps against the oracle and, byte for byte, against S2B_RESIDENT=0."""
    whole = 4000
    n = _resident_size(product, dev, whole) + extra
    recipe = _with_env(piles([n]), S2B_WHOLE_ISLAND=whole)
    seen = []
    setup, after, twin = _twin_check(product, recipe, seen)
    _run(reference, product, dev, recipe, "TGS_Soft", 20, 4, 2, {}, setup=setup, after_step=after(dev))
    twin["sc"].destroy()
    assert seen[0].maxRegionBodies == RES_MAX + extra and seen[0].residentRegions == 1 - extra
    assert seen[0].regionCount > 1 and seen[0].cutCount == 0
    for c in seen:
        assert c.residentRegions == (1 if c.maxRegionBodies <= RES_MAX else 0)


def test_resident_field_near_capacity(reference, product, dev):
    """Eight islands of 3 071 boxes, each whole in its own region (with the ground, at most 3 072): every region resident."""
    recipe = _with_env(piles([3071] * 8), S2B_WHOLE_ISLAND=4000)
    seen = []
    setup, after, twin = _twin_check(product, recipe, seen)
    _run(reference, product, dev, recipe, "TGS_Soft", 3, 4, 2, {}, setup=setup, after_step=after(dev))
    twin["sc"].destroy()
    for c in seen:
        assert c.residentRegions == 1 and c.maxRegionBodies in (3071, 3072) and c.regionCount >= 8 and c.cutCount == 0


# ---- the resident path switched off and on mid-run ------------------------------------------------------------------------

def test_resident_switches(reference, product, dev):
    """Two piles of 703 boxes, 0.05 m apart at the base (resident). Each of a joint, a kinematic body touching a pile, a hub
    (a slab under 60 boxes, degree above 48), an overflow group (a colour limit of 2) and a cut set (a box bridging the two
    piles into one island of 1 407, above the 1 200 a region keeps whole) switches the resident path off on the step it
    appears and on again after it goes; the graph is replayed in between."""
    base = 37
    half = 0.5 * base

    def recipe(lib, solver, **kw):
        sc = scenes.Scene(lib, lib.create_world(solver), name="switches")
        sc.bodies.append(scenes._ground(lib, sc.world, 150.0))
        _pile(lib, sc, -half - 0.025, base * (base + 1) // 2)
        _pile(lib, sc, half + 0.025, base * (base + 1) // 2)
        return sc

    live = {}
    dwh = {}
    off = {3, 4, 8, 9, 13, 14, 18, 19, 23, 24}

    def before(step, pairs):
        for lib, sc in pairs:
            key = id(lib)
            got = live.setdefault(key, {})
            if step == 3:
                a, b = sc.bodies[1], sc.bodies[2]
                jd = capi.default_revolute_def()
                jd.bodyIdA, jd.bodyIdB = a, b
                pivot = Vec2(-2.0 * half - 0.025 + 1.0, 0.5)
                jd.localAnchorA = lib.s2Body_GetLocalPoint(a, pivot)
                jd.localAnchorB = lib.s2Body_GetLocalPoint(b, pivot)
                got["joint"] = lib.s2CreateRevoluteJoint(sc.world, C.byref(jd))
            elif step == 5:
                lib.s2DestroyJoint(got.pop("joint"))
            elif step == 8:
                left = lib.s2Body_GetPosition(sc.bodies[1])
                got["kin"] = _box(lib, sc.world, capi.KINEMATIC_BODY, float(left.x) - 1.0, float(left.y))
            elif step == 10:
                lib.s2DestroyBody(got.pop("kin"))
            elif step == 13:
                slab = _box(lib, sc.world, capi.DYNAMIC_BODY, 100.0, 0.25, hx=20.0, hy=0.25)
                riders = [_box(lib, sc.world, capi.DYNAMIC_BODY, 100.0 - 18.0 + 0.6 * k, 0.7, hx=0.2, hy=0.2) for k in range(60)]
                got["hub"] = [slab] + riders
            elif step == 15:
                for b in got.pop("hub")[::-1]:
                    lib.s2DestroyBody(b)
            elif step == 23:
                got["bridge"] = _box(lib, sc.world, capi.DYNAMIC_BODY, 0.0, 1.5)
            elif step == 25:
                lib.s2DestroyBody(got.pop("bridge"))
        if step == 18:
            dwh["dw"].set_max_colors(2)
        elif step == 20:
            dwh["dw"].set_max_colors(24)

    seen = []

    def after(dw):
        seen.append(dw.counters())

    def setup(dw):
        dwh["dw"] = dw
        dw.set_regions(2)  # regions always: the default mode drops them for a while after a hub or a wide cut set

    _run(reference, product, dev, recipe, "TGS_Soft", 28, 4, 2, {}, setup=setup, before_step=before, after_step=after)
    resident = [c.residentRegions for c in seen]
    assert resident == [0 if s in off else 1 for s in range(28)], resident
    assert seen[3].jointCount == 1 and seen[8].cutCount > 0 and seen[13].cutCount + seen[13].overflowCount > 0
    assert seen[18].overflowCount > 0 and seen[23].cutCount > 0 and all(c.regionCount > 0 for c in seen)
    # after each switch the stage is replayed as a graph again (the first replays come a few quiet steps into the run)
    replays = [c.graphReplays for c in seen]
    for a, b in ((5, 8), (10, 13), (15, 18), (20, 23), (25, 28)):
        assert replays[b - 1] > replays[a], f"no graph replay between steps {a} and {b - 1}: {replays}"


# ---- what never takes the resident path -----------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["warm_start_off", "dataflow"])
def test_not_resident(reference, product, dev, mode):
    seen = []
    setup = (lambda dw: dw.set_dataflow(True)) if mode == "dataflow" else None
    _run(reference, product, dev, piles([300, 300]), "TGS_Soft", 1, 4, 2, {}, setup=setup,
         after_step=lambda dw: seen.append(dw.counters()), warm_start=mode != "warm_start_off")
    assert seen[0].residentRegions == 0 and seen[0].constraintCount > 0
    if mode == "warm_start_off":
        assert seen[0].regionCount > 0 and seen[0].cutCount == 0
