"""GPU: the step's tail (DESIGN.md §3.3). On a pass that reuses the hierarchy's topology, finalize's shapes, the refit and
the search's moved proxies run as one launch (s2bFinalizeRefitKernel) and the search skips its own refit and
s2bCollectMovers; the survivor and large-mover scans are blocks of the query launch.

* s2bCounters.finalizeRefits shows the fused path ran on the reuse passes of the bench pyramid, the tumbler (large
  movers), shapes recreated in freed slots and a scene with uploads between steps; each of those is checked every step
  against the reference (test_multistep_gpu._run: pair table, manifolds, bodies, boxes).
* The bullets scene with clamps, which the reference cannot run, is checked every step against the same world with the
  fused path off (S2B_FINALIZE_REFIT=0): contact table and body state bit for bit, and every clamped bullet's new pair is
  in the table of the next step."""
import ctypes as C
import os

import pytest

from solver2d_b200 import capi, device, scenes
from test_multistep_gpu import _run

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0
REUSE_LIMIT = 16  # S2B_TREE_REUSE_LIMIT


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


class _Passes:
    """after_step hook: (pair passes, fused passes) after every step."""

    def __init__(self):
        self.seen = []

    def __call__(self, dw):
        c = dw.counters()
        self.seen.append((c.pairPassCount, c.finalizeRefits))

    def fused_steps(self):
        """steps whose pair pass took its refit and moved proxies from the finalize before it"""
        out, prev = [], (0, 0)
        for step, cur in enumerate(self.seen):
            if cur[1] > prev[1]:
                out.append(step)
            prev = cur
        return out

    def after_still(self):
        """passes of a step that follows a step without one: the finalize before them ran the old way (the pass before had
        not been committed), so they refit on their own"""
        out, prev, ran = 0, 0, True
        for cur, _ in self.seen:
            if cur > prev and not ran:
                out += 1
            ran, prev = cur > prev, cur
        return out


def _assert_reuse_passes_fused(c, passes, missed=0):
    """Every pass ran fused but the rebuilds (the first, then about one in REUSE_LIMIT + 1), the passes after a still
    step and `missed` others."""
    rebuilds = (c.pairPassCount + REUSE_LIMIT) // (REUSE_LIMIT + 1) + 1
    assert c.pairPassCount > REUSE_LIMIT + 1
    low = c.pairPassCount - rebuilds - passes.after_still() - missed
    assert low <= c.finalizeRefits < c.pairPassCount, (c.pairPassCount, c.finalizeRefits, low)


def test_bench_pyramid_every_step(reference, product, dev):
    """The bench's 100 128-box pyramid (base 447): the lattice stands still for the first steps, then every pass moves."""
    passes = _Passes()
    c = _run(reference, product, dev, scenes.pyramid, "TGS_Soft", 32, 4, 2, dict(base_count=447), after_step=passes)
    _assert_reuse_passes_fused(c, passes)
    assert c.contactCount > 290000


def test_tumbler_large_movers_every_step(reference, product, dev):
    """The hub container's four scene-sized walls take the large-mover scan, judged against the previous refit's root box."""
    passes = _Passes()
    c = _run(reference, product, dev, scenes.tumbler, "TGS_Soft", 40, 4, 2, dict(grid=20, half_extent=4.0), after_step=passes)
    _assert_reuse_passes_fused(c, passes)


def _create_box(lib, sc, x, y):
    bd = scenes.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    bd.position = capi.Vec2(x, y)
    sd = scenes.default_shape_def()
    sd.density = 1.0
    bid = lib.s2CreateBody(sc.world, C.byref(bd))
    lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(lib.s2MakeSquare(0.5)))
    sc.bodies.append(bid)


def _destroy(lib, sc, ks):
    for k in sorted(ks, reverse=True):
        lib.s2DestroyBody(sc.bodies.pop(k))


def test_shapes_recreated_in_freed_slots_every_step(reference, product, dev):
    """Boxes destroyed, then created in the freed slots elsewhere: the passes after an edit rebuild, the others reuse."""
    edits = {
        6: lambda lib, sc: _destroy(lib, sc, [3, 10, 20]),
        9: lambda lib, sc: (_create_box(lib, sc, -2.0, 9.0), _create_box(lib, sc, 0.2, 9.5), _create_box(lib, sc, 6.0, 0.6)),
        30: lambda lib, sc: (_destroy(lib, sc, [5]), _create_box(lib, sc, 1.0, 10.0)),
    }

    def before_step(step, worlds):
        if step in edits:
            for lib, sc in worlds:
                edits[step](lib, sc)

    passes = _Passes()
    c = _run(reference, product, dev, scenes.pyramid, "TGS_Soft", 48, 4, 2, dict(base_count=8), before_step=before_step,
             after_step=passes)
    fused = passes.fused_steps()
    for step in edits:
        assert step not in fused, f"step {step}: shapes changed, yet the pass reused finalize's refit"
    _assert_reuse_passes_fused(c, passes, missed=2 * len(edits))


def test_uploads_between_steps_every_step(reference, product, dev):
    """Body uploads between steps (velocities): the search started behind the step before is stale, and the
    pass redoes its refit and moved proxies; the passes in between keep the fused path."""
    uploads = set(range(5, 40, 4))

    def before_step(step, worlds):
        for lib, sc in worlds:
            if step in uploads:
                for bid in sc.bodies[2::9]:
                    if lib.s2Body_GetType(bid) == capi.DYNAMIC_BODY:
                        lib.s2Body_SetLinearVelocity(bid, capi.Vec2(0.5, 1.5))
            if step == 21:
                lib.s2Body_SetLinearVelocity(sc.bodies[-1], capi.Vec2(-4.0, 6.0))

    passes = _Passes()
    c = _run(reference, product, dev, scenes.pyramid, "TGS_Soft", 44, 4, 2, dict(base_count=12), before_step=before_step,
             after_step=passes)
    fused = passes.fused_steps()
    for step in uploads | {21}:
        assert step not in fused, f"step {step}: bodies were uploaded, yet the pass reused finalize's refit"
    _assert_reuse_passes_fused(c, passes, missed=len(uploads) + 3)


def _bullet_world(P, D, fused):
    old = os.environ.get("S2B_FINALIZE_REFIT")
    os.environ["S2B_FINALIZE_REFIT"] = "1" if fused else "0"
    try:
        sc = scenes.bullets(P, "TGS_Soft")
        P.s2World_EnableContinuous(sc.world, True)
        P.s2World_Flush(sc.world)
        dw = device.DeviceWorld.attach(D, sc.world)
    finally:
        if old is None:
            del os.environ["S2B_FINALIZE_REFIT"]
        else:
            os.environ["S2B_FINALIZE_REFIT"] = old
    return sc, dw


def _pairs(dw):
    rows = dw.download_contacts(dw.counters().contactCount)
    keys = {(min(int(r["shapeA"]), int(r["shapeB"])), max(int(r["shapeA"]), int(r["shapeB"]))) for r in rows}
    return rows, keys


def _overlap(a, b):
    return a[0] <= b[2] and b[0] <= a[2] and a[1] <= b[3] and b[1] <= a[3]


def test_bullets_with_clamps_against_unfused(product, dev):
    """Clamped bullets: the bullet pass's refit follows the re-finalize, and a bullet that escapes its fat box only there
    joins finalize's moved proxies. Every step the contact table and the bodies equal those of the unfused world, and a
    clamped bullet's new pair (its fat box meets its target's, no contact yet) is in the table of the next step."""
    P = product
    sa, da = _bullet_world(P, dev, True)
    sb, db = _bullet_world(P, dev, False)
    lanes = [lane for lane in sa.piles["lanes"] if not lane["passes"]]
    hits, pending, checked = 0, set(), 0
    for step in range(12):
        sa.step(DT, 4, 2, True)
        sb.step(DT, 4, 2, True)
        ra, ka = _pairs(da)
        rb, _ = _pairs(db)
        assert len(ra) == len(rb) and ra.tobytes() == rb.tobytes(), f"step {step}: contact tables differ"
        ba = da.download_all_bodies(da.counters().bodyCapacity)
        bb = db.download_all_bodies(db.counters().bodyCapacity)
        assert ba.tobytes() == bb.tobytes(), f"step {step}: bodies differ"
        missing = pending - ka
        assert not missing, f"step {step}: pairs of clamped bullets missing: {sorted(missing)}"
        checked += len(pending)
        ca = da.counters()
        hits += ca.bulletHits
        pending = set()
        if ca.bulletHits > 0:
            _, fat, _ = da.download_shape_boxes(ca.shapeCapacity)
            for lane in lanes:
                s = lane["shape"].index
                for _, t in lane["targets"]:
                    key = (min(s, t.index), max(s, t.index))
                    if key not in ka and _overlap(fat[s], fat[t.index]):
                        pending.add(key)
    ca, cb = da.counters(), db.counters()
    assert hits > 0 and checked > 0
    assert ca.finalizeRefits > 0 and cb.finalizeRefits == 0
    assert ca.pairPassCount == cb.pairPassCount
    sa.destroy()
    sb.destroy()
