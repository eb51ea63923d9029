"""GPU: bullets (s2Body_SetBullet, DESIGN.md §3.12), the sweep of fast dynamic bullets against static, kinematic and
non-bullet dynamic shapes at their final poses, after finalize.

* Tunnelling, all ten variants: on scenes.bullets some projectiles end behind their non-static targets with continuous
  collision on and the flag clear; with the flag set none ever does, and the must-pass lanes pass in both modes.
* Bit for bit against the host restatement (test_bullet_cpu.host_bullet_pass), in the colour and wavefront schedules,
  persistent and launch by launch: poses, counters, a clamped bullet's boxes and the moved count.
* float64 (within the bit-for-bit test): a clamped bullet lies at least the target separation, less tolerance and
  round-off, from its target's shapes at their final poses.
* Nothing changes where it should not (flags with continuous off, flags on static and kinematic bodies, flagged bodies
  that are never fast), the next step's pair pass sees a clamped bullet, and the flag's lifecycle."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from solver2d_b200 import capi, device, scenes
from test_bullet_cpu import host_bullet_pass
from test_continuous_gpu import VARIANTS, _attach, _fast, _poses, _rows, _state
from test_toi_reference_cpu import TARGET, TOL, Shape64, Sweep64, sep64

pytestmark = pytest.mark.gpu

DT = 1.0 / 60.0
STEPS = 30
SPEC = np.float32(4.0 * 0.005)  # s2_speculativeDistance
MARGIN = np.float32(0.1)        # s2_aabbMargin
SCHEDULES = [(device.SCHEDULE_COLOR, True), (device.SCHEDULE_COLOR, False), (device.SCHEDULE_WAVEFRONT, True),
             (device.SCHEDULE_WAVEFRONT, False)]


@pytest.fixture(scope="module")
def P():
    return capi.Solver2D(device.LIB_PATH)


@pytest.fixture(scope="module")
def D():
    return device.Device()


def _flag(P, sc, on=True):
    for lane in sc.piles["lanes"]:
        P.s2Body_SetBullet(lane["body"], on)


@pytest.mark.parametrize("solver", VARIANTS)
def test_bullets_stop_at_non_static_targets(P, solver):
    ever = {}
    for flagged in (False, True):
        sc = scenes.bullets(P, solver, flagged=flagged)
        P.s2World_EnableContinuous(sc.world, True)
        lanes = sc.piles["lanes"]
        behind = np.zeros(len(lanes), dtype=bool)
        for _ in range(STEPS):
            sc.step(DT, 4, 2, True)
            behind |= scenes.bullets_behind(P, sc)
        meant = np.array([lane["passes"] for lane in lanes])
        assert behind[meant].all(), f"{solver} flagged={flagged}: a must-pass projectile did not pass"
        # Jacobi does not hold a projectile at the block of boxes: some end behind it within the 30 steps (a stated limit,
        # DESIGN.md §3.12). The pass does stop every one of them at the block's face (test_bullets_reach_the_block_face).
        held = ~meant & ~np.array([solver == "Jacobi" and lane["kind"] == "block" for lane in lanes])
        ever[flagged] = behind[held]
        sc.destroy()
    assert ever[False].sum() >= 1, f"{solver}: nothing tunnels with the flag clear"
    assert ever[True].sum() == 0, f"{solver}: lanes {np.flatnonzero(ever[True]).tolist()} tunnel as bullets"


def _front_local_x(P, lane):
    """x of the projectile's centre in the frame of the block's front middle box (its front face at -BULLET_BLOCK_HALF)"""
    front = lane["targets"][2][0]  # (column 0, row 0: the block is built column by column, rows -2..2)
    return P.s2Body_GetLocalPoint(front, P.s2Body_GetPosition(lane["body"])).x


@pytest.mark.parametrize("solver", VARIANTS)
def test_bullets_reach_the_block_face(P, D, solver):
    """Every block lane, every variant: at the first step that ends with the projectile within 0.4 m of the block's front
    face (the step in which it gets there, at its speed of 0.5-3.3 m per step), its centre is in front of that face, and a
    projectile that would have crossed it in that step was clamped."""
    sc = scenes.bullets(P, solver)
    P.s2World_EnableContinuous(sc.world, True)
    dw = _attach(P, D, sc.world)
    lanes = [lane for lane in sc.piles["lanes"] if lane["kind"] == "block"]
    face = -scenes.BULLET_BLOCK_HALF
    arrived = {}
    for step in range(12):
        sc.step(DT, 4, 2, True)
        hits = dw.counters().bulletHits
        for n, lane in enumerate(lanes):
            if n in arrived:
                continue
            x = _front_local_x(P, lane)
            if x >= face - 0.4:
                arrived[n] = (step, x, hits)
    assert len(arrived) == len(lanes), sorted(set(range(len(lanes))) - set(arrived))
    for n, (step, x, hits) in arrived.items():
        assert x < face, (n, step, x)
        assert hits > 0 or x < face - 0.3, (n, step, x)
    sc.destroy()


def _shapes(sc):
    """host_bullet_pass's shape list and jointed pairs of a bullets scene."""
    shapes, joints = [], set()
    default = (1, 0xFFFFFFFF, 0)
    for lane in sc.piles["lanes"]:
        filtered = lane["exclusion"] == "filter"
        shapes.append(dict(body=lane["body"].index, form=lane["form"], filter=(1, 0xFFFFFFFF & ~2, 0) if filtered else default,
                           segment=False))
        for bid, _ in lane["targets"]:
            shapes.append(dict(body=bid.index, form=lane["target_form"], filter=(2, 0xFFFFFFFF, 0) if filtered else default,
                               segment=False))
        if lane["exclusion"] == "joint":
            joints.add(tuple(sorted((lane["body"].index, lane["target"].index))))
    return shapes, frozenset(joints)


def _finalize_box(form, row):
    """s2bFinalizeShapes' box of a shape at a body row's pose, in float32 operation for operation."""
    f = np.float32
    ox, oy = f(row["origin"][0]), f(row["origin"][1])
    s, c = f(row["rot"][0]), f(row["rot"][1])
    xs, ys = [], []
    for k in range(form.count):
        px, py = f(form.vertices[k].x), f(form.vertices[k].y)
        xs.append((c * px - s * py) + ox)
        ys.append((s * px + c * py) + oy)
    r = f(form.radius)
    return np.array([(min(xs) - r) - SPEC, (min(ys) - r) - SPEC, (max(xs) + r) + SPEC, (max(ys) + r) + SPEC], dtype=f)


def _contains(fat, box):
    return fat[0] <= box[0] and fat[1] <= box[1] and box[2] <= fat[2] and box[3] <= fat[3]


@pytest.mark.parametrize("solver", ["TGS_Soft", "PGS_NGS", "XPBD"])
@pytest.mark.parametrize("schedule,persistent", SCHEDULES, ids=["colour", "colour-launch", "wavefront", "wavefront-launch"])
def test_pass_matches_host_restatement_bit_for_bit(P, D, solver, schedule, persistent):
    hits = 0
    for k in (1, 2, 3):
        # two identical worlds with continuous collision on; k - 1 steps unflagged, then step k with the projectiles of
        # one world flagged. The scene has no static shape, so the unflagged world's end of step is the flagged world's
        # state before its bullet pass.
        worlds = []
        for _ in range(2):
            sc = scenes.bullets(P, solver, flagged=False)
            P.s2World_EnableContinuous(sc.world, True)
            dw = _attach(P, D, sc.world)
            dw.set_schedule(schedule)
            dw.set_persistent(persistent)
            worlds.append((sc, dw))
        (s_off, d_off), (s_on, d_on) = worlds
        for _ in range(k - 1):
            s_off.step(DT, 4, 2, True)
            s_on.step(DT, 4, 2, True)
        cap = d_off.body_cap
        before = d_off.download_all_bodies(cap)
        _, fat_before, _ = d_off.download_shape_boxes()
        _flag(P, s_on)
        s_off.step(DT, 4, 2, True)
        s_on.step(DT, 4, 2, True)
        after = d_off.download_all_bodies(cap)
        got = d_on.download_all_bodies(cap)
        rows = after.copy()
        rows["flags"] = got["flags"]  # the flagged world's bullet bits on the unflagged world's poses
        shapes, joints = _shapes(s_on)
        want = host_bullet_pass(P, shapes, before, rows, joints)
        c_on, c_off = d_on.counters(), d_off.counters()
        # (one shape per projectile)
        fast_shapes = sum(1 for lane in s_on.piles["lanes"] if _fast(before[lane["body"].index], after[lane["body"].index]))
        assert c_on.bulletHits == len(want), k
        assert c_on.bulletShapes == fast_shapes, k
        assert c_on.continuousHits == c_off.continuousHits == 0
        assert c_on.continuousShapes == c_off.continuousShapes - fast_shapes
        assert c_off.bulletShapes == 0 and c_off.bulletHits == 0  # (the bullet plank is never fast)
        for b in range(cap):
            if b in want:
                t, sweep = want[b]
                xf = P.s2GetSweepTransform(C.byref(sweep), t)
                assert np.float32(xf.p.x) == got[b]["origin"][0] and np.float32(xf.p.y) == got[b]["origin"][1], (k, b)
                assert np.float32(xf.q.s) == got[b]["rot"][0] and np.float32(xf.q.c) == got[b]["rot"][1], (k, b)
                assert np.array_equal(got[b]["linearVelocity"], after[b]["linearVelocity"])
            else:
                assert np.array_equal(_poses(got[b:b + 1]), _poses(after[b:b + 1])), (k, b)
        # boxes: a clamped bullet's are finalize's at the clamped pose; its fat box is kept if that box still holds the
        # new one, else re-centred; every other shape's are the unflagged world's
        aabb_on, fat_on, _ = d_on.download_shape_boxes()
        aabb_off, fat_off, _ = d_off.download_shape_boxes()
        clamped_shapes = set()
        for lane in s_on.piles["lanes"]:
            b, s = lane["body"].index, lane["shape"].index
            if b not in want:
                continue
            clamped_shapes.add(s)
            box = _finalize_box(lane["form"], got[b])
            assert np.array_equal(aabb_on[s], box), (k, b)
            fat = fat_off[s] if _contains(fat_off[s], box) else np.array([box[0] - MARGIN, box[1] - MARGIN, box[2] + MARGIN,
                                                                          box[3] + MARGIN], dtype=np.float32)
            assert np.array_equal(fat_on[s], fat), (k, b)
            _check_float64(lane, before, got, b)
        others = np.array([i not in clamped_shapes for i in range(len(aabb_on))])
        assert np.array_equal(aabb_on[others], aabb_off[others]) and np.array_equal(fat_on[others], fat_off[others])
        # every shape the unflagged world's finalize moved, and once more each clamped shape only the re-finalize moved
        again = sum(1 for s in clamped_shapes if np.array_equal(fat_off[s], fat_before[s]) and not np.array_equal(fat_on[s], fat_off[s]))
        assert c_on.movedCount == c_off.movedCount + again
        hits += len(want)
        for sc, _ in worlds:
            sc.destroy()
    assert hits >= 5


def _shape64(form):
    return Shape64([(form.vertices[i].x, form.vertices[i].y) for i in range(form.count)], form.radius)


def _check_float64(lane, before, rows, b):
    """float64: a clamped bullet (rows[b], at its clamped pose) is at least the target separation, less the tolerance and
    round-off, from every shape of its target at the target's final pose, except a shape it already started within
    target + tolerance of (the core rule of DESIGN.md §3.11 then holds it or lets it go, and it stays as deep as it
    started). The pair rules exclude the filtered and jointed lanes' targets and bullet targets; those lanes' projectiles
    are never clamped at them."""
    r, r0 = rows[b], before[b]
    A = _shape64(lane["form"])
    sA = Sweep64(r["localCenter"], r["position"], r["position"], r["rot"], r["rot"])
    sA0 = Sweep64(r0["localCenter"], r0["position"], r0["position"], r0["rot"], r0["rot"])
    O = _shape64(lane["target_form"])
    for bid, _ in lane["targets"]:
        t = rows[bid.index]
        sO = Sweep64(t["localCenter"], t["position"], t["position"], t["rot"], t["rot"])
        if float(sep64(O, sO, A, sA0, [0.0])[0]) <= TARGET + TOL:
            continue
        d = float(sep64(O, sO, A, sA, [0.0])[0])
        big = max(abs(float(x)) for x in (*r["position"], *t["position"]))
        eps = 2e-5 + 8 * float(np.spacing(np.float32(big)))
        assert d >= TARGET - TOL - eps, (lane["kind"], d)


def _launches_and_state(P, D, make, steps, setup):
    sc = make()
    setup(sc)
    dw = _attach(P, D, sc.world)
    start = dw.counters().kernelLaunches
    shapes = 0
    for _ in range(steps):
        sc.step(DT, 4, 2, True)
        shapes += dw.counters().bulletShapes
    out = (dw.counters().kernelLaunches - start, _state(_rows(dw)), shapes)
    sc.destroy()
    return out


def _same_as_unflagged(P, D, make, steps, setup):
    base = _launches_and_state(P, D, make, steps, lambda sc: None)
    other = _launches_and_state(P, D, make, steps, setup)
    assert other[2] == 0
    assert other[0] == base[0], f"{other[0]} launches against {base[0]}"
    assert np.array_equal(other[1], base[1])


def test_flags_without_continuous_change_nothing(P, D):
    _same_as_unflagged(P, D, lambda: scenes.bullets(P, "TGS_Soft", flagged=False), 10, lambda sc: _flag(P, sc))


def test_flag_on_static_and_kinematic_bodies_changes_nothing(P, D):
    def make():
        # (without the must-pass lanes, one of which flags a dynamic plank: no world here has a dynamic bullet)
        sc = scenes.bullets(P, "TGS_Soft", flagged=False, excluded=False)
        P.s2World_EnableContinuous(sc.world, True)
        # a static segment well below the lanes
        bid = P.s2CreateBody(sc.world, C.byref(capi.default_body_def()))
        P.s2CreateSegmentShape(bid, C.byref(capi.default_shape_def()),
                               C.byref(capi.Segment(capi.Vec2(-50.0, -10.0), capi.Vec2(50.0, -10.0))))
        sc.piles["static"] = bid
        return sc

    def setup(sc):
        for lane in sc.piles["lanes"]:
            if lane["kind"] == "kinematic":
                P.s2Body_SetBullet(lane["target"], True)
        P.s2Body_SetBullet(sc.piles["static"], True)

    _same_as_unflagged(P, D, make, 10, setup)

    # the launch count does see the pass: a dynamic bullet at rest adds its five launches to every step
    def one_dynamic(sc):
        setup(sc)
        bd = capi.default_body_def()
        bd.type = capi.DYNAMIC_BODY
        bd.gravityScale = 0.0
        bd.position = capi.Vec2(0.0, -50.0)
        bid = P.s2CreateBody(sc.world, C.byref(bd))
        P.s2CreateCircleShape(bid, C.byref(capi.default_shape_def()), C.byref(capi.Circle(capi.Vec2(0.0, 0.0), 0.1)))
        P.s2Body_SetBullet(bid, True)

    def one_plain(sc):
        setup(sc)
        bd = capi.default_body_def()
        bd.type = capi.DYNAMIC_BODY
        bd.gravityScale = 0.0
        bd.position = capi.Vec2(0.0, -50.0)
        bid = P.s2CreateBody(sc.world, C.byref(bd))
        P.s2CreateCircleShape(bid, C.byref(capi.default_shape_def()), C.byref(capi.Circle(capi.Vec2(0.0, 0.0), 0.1)))

    plain = _launches_and_state(P, D, make, 10, one_plain)
    flagged = _launches_and_state(P, D, make, 10, one_dynamic)
    assert flagged[0] - plain[0] == 10 * 5 and np.array_equal(flagged[1], plain[1])


def test_flagged_bodies_that_are_never_fast_change_nothing(P, D):
    def make():
        sc = scenes.pyramid(P, "TGS_Soft", base_count=20)
        P.s2World_EnableContinuous(sc.world, True)
        return sc

    def setup(sc):
        for bid in sc.bodies[1::7]:
            if P.s2Body_GetType(bid) == capi.DYNAMIC_BODY:
                P.s2Body_SetBullet(bid, True)

    base = _launches_and_state(P, D, make, 20, lambda sc: None)
    other = _launches_and_state(P, D, make, 20, setup)
    assert other[2] == 0 and np.array_equal(other[1], base[1])
    # the refit and four launches per step, and the shape re-finalize: nothing else
    assert other[0] - base[0] == 20 * 5


@pytest.mark.parametrize("env", [None, ("S2B_PREFETCH_PAIRS", "0"), ("S2B_GRAPH", "0")])
def test_next_step_pair_pass_sees_a_clamped_bullet(P, D, env):
    old = os.environ.get(env[0]) if env else None
    if env:
        os.environ[env[0]] = env[1]
    try:
        sc = scenes.bullets(P, "TGS_Soft")
        P.s2World_EnableContinuous(sc.world, True)
        dw = _attach(P, D, sc.world)
        planks = [lane for lane in sc.piles["lanes"] if lane["kind"] == "plank" and not lane["passes"]]
        touching = set()
        for _ in range(6):
            sc.step(DT, 4, 2, True)
            n = dw.counters().contactCount
            rows = dw.download_contacts(n)
            pairs = {tuple(sorted((int(r["bodyA"]), int(r["bodyB"])))) for r in rows}
            for lane in planks:
                if tuple(sorted((lane["body"].index, lane["target"].index))) in pairs:
                    touching.add(lane["body"].index)
        # every projectile fired at a dynamic plank gets its contact with the plank
        assert touching == {lane["body"].index for lane in planks}
        assert not scenes.bullets_behind(P, sc)[[not lane["passes"] for lane in sc.piles["lanes"]]].any()
        sc.destroy()
    finally:
        if env:
            if old is None:
                del os.environ[env[0]]
            else:
                os.environ[env[0]] = old


def test_flag_round_trip_and_slot_reuse(P, D):
    world = P.create_world("TGS_Soft")
    bd = capi.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    body = P.s2CreateBody(world, C.byref(bd))
    P.s2CreateCircleShape(body, C.byref(capi.default_shape_def()), C.byref(capi.Circle(capi.Vec2(0.0, 0.0), 0.1)))
    assert not P.s2Body_IsBullet(body)
    P.s2Body_SetBullet(body, True)
    assert P.s2Body_IsBullet(body)
    dw = _attach(P, D, world)
    assert _rows(dw)[body.index]["flags"] & 0x20
    P.s2DestroyBody(body)
    again = P.s2CreateBody(world, C.byref(bd))
    assert again.index == body.index and not P.s2Body_IsBullet(again)
    P.s2World_Flush(world)
    assert not _rows(dw)[again.index]["flags"] & 0x20
    P.s2DestroyWorld(world)


def _lane_world(P, speed=150.0, target="plank"):
    """A bullet circle fired at a heavy dynamic plank (or a kinematic one) 1.2 m ahead, continuous collision on."""
    world = P.create_world("TGS_Soft")
    td = capi.default_body_def()
    td.type = capi.DYNAMIC_BODY if target == "plank" else capi.KINEMATIC_BODY
    td.gravityScale = 0.0
    plank = P.s2CreateBody(world, C.byref(td))
    sd = capi.default_shape_def()
    sd.density = scenes.BULLET_PLANK_DENSITY
    P.s2CreatePolygonShape(plank, C.byref(sd), C.byref(P.s2MakeBox(0.025, 2.0)))
    bd = capi.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    bd.gravityScale = 0.0
    bd.position = capi.Vec2(-1.2, 0.0)
    bd.linearVelocity = capi.Vec2(speed, 0.0)
    bullet = P.s2CreateBody(world, C.byref(bd))
    P.s2CreateCircleShape(bullet, C.byref(capi.default_shape_def()), C.byref(capi.Circle(capi.Vec2(0.0, 0.0), 0.1)))
    P.s2World_EnableContinuous(world, True)
    return world, plank, bullet


def _past(P, bullet, plank):
    return P.s2Body_GetLocalPoint(plank, P.s2Body_GetPosition(bullet)).x > 0.0


def test_flag_toggled_between_steps(P, D):
    world, plank, bullet = _lane_world(P, speed=40.0)
    dw = _attach(P, D, world)
    P.s2World_Step(world, DT, 4, 2, True)  # 0.67 m: not there yet, unflagged
    assert dw.counters().bulletShapes == 0
    P.s2Body_SetBullet(bullet, True)
    P.s2World_Step(world, DT, 4, 2, True)
    c = dw.counters()
    assert c.bulletShapes == 1 and c.bulletHits == 1
    for _ in range(10):
        P.s2World_Step(world, DT, 4, 2, True)
        assert not _past(P, bullet, plank)
    P.s2Body_SetBullet(bullet, False)
    P.s2World_Step(world, DT, 4, 2, True)
    assert dw.counters().bulletShapes == 0
    P.s2DestroyWorld(world)


@pytest.mark.parametrize("prefetch", ["1", "0"])
def test_target_created_and_destroyed_between_steps(P, D, prefetch):
    old = os.environ.get("S2B_PREFETCH_PAIRS")
    os.environ["S2B_PREFETCH_PAIRS"] = prefetch
    try:
        world, plank, bullet = _lane_world(P, speed=40.0)
        P.s2Body_SetBullet(bullet, True)
        dw = _attach(P, D, world)
        P.s2World_Step(world, DT, 4, 2, True)
        # a second plank created between the bullet and the first: the tree is rebuilt, and the bullet stops at it
        td = capi.default_body_def()
        td.type = capi.DYNAMIC_BODY
        td.gravityScale = 0.0
        td.position = capi.Vec2(-0.3, 0.0)
        near = P.s2CreateBody(world, C.byref(td))
        sd = capi.default_shape_def()
        sd.density = scenes.BULLET_PLANK_DENSITY
        P.s2CreatePolygonShape(near, C.byref(sd), C.byref(P.s2MakeBox(0.025, 2.0)))
        P.s2World_Step(world, DT, 4, 2, True)
        assert dw.counters().bulletHits == 1
        assert P.s2Body_GetPosition(bullet).x < -0.3
        # destroyed again before the next step: nothing to stop at until the first plank
        P.s2DestroyBody(near)
        P.s2Body_SetLinearVelocity(bullet, capi.Vec2(40.0, 0.0))
        for _ in range(8):
            P.s2World_Step(world, DT, 4, 2, True)
            assert not _past(P, bullet, plank)
        assert P.s2Body_GetPosition(bullet).x > -0.3
        P.s2DestroyWorld(world)
    finally:
        if old is None:
            del os.environ["S2B_PREFETCH_PAIRS"]
        else:
            os.environ["S2B_PREFETCH_PAIRS"] = old


def test_destroyed_bullet_slot_reused_by_a_non_bullet(P, D):
    world, plank, bullet = _lane_world(P)
    P.s2Body_SetBullet(bullet, True)
    dw = _attach(P, D, world)
    P.s2World_Step(world, DT, 4, 2, True)
    P.s2DestroyBody(bullet)
    bd = capi.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    bd.gravityScale = 0.0
    bd.position = capi.Vec2(-1.2, 1.0)
    bd.linearVelocity = capi.Vec2(150.0, 0.0)
    other = P.s2CreateBody(world, C.byref(bd))
    assert other.index == bullet.index
    P.s2CreateCircleShape(other, C.byref(capi.default_shape_def()), C.byref(capi.Circle(capi.Vec2(0.0, 0.0), 0.1)))
    assert not P.s2Body_IsBullet(other)
    P.s2World_Step(world, DT, 4, 2, True)
    c = dw.counters()
    assert c.bulletShapes == 0 and c.bulletHits == 0
    assert not _rows(dw)[other.index]["flags"] & 0x20
    assert _past(P, other, plank)  # not a bullet: it tunnels
    P.s2DestroyWorld(world)


def test_jointed_bullet_and_multi_shape_bullet_with_a_segment(P, D):
    world = P.create_world("TGS_Soft")
    td = capi.default_body_def()
    td.type = capi.DYNAMIC_BODY
    td.gravityScale = 0.0
    td.position = capi.Vec2(5.0, 0.0)
    plank = P.s2CreateBody(world, C.byref(td))
    sd = capi.default_shape_def()
    sd.density = scenes.BULLET_PLANK_DENSITY
    P.s2CreatePolygonShape(plank, C.byref(sd), C.byref(P.s2MakeBox(0.025, 3.0)))
    bd = capi.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    bd.gravityScale = 0.0
    bd.position = capi.Vec2(3.0, 0.0)
    bd.linearVelocity = capi.Vec2(150.0, 0.0)
    body = P.s2CreateBody(world, C.byref(bd))
    P.s2CreateCircleShape(body, C.byref(capi.default_shape_def()), C.byref(capi.Circle(capi.Vec2(-0.5, 0.0), 0.1)))
    # the leading shape is a segment 0.6 m ahead of the centre line
    P.s2CreateSegmentShape(body, C.byref(capi.default_shape_def()),
                           C.byref(capi.Segment(capi.Vec2(0.6, 0.9), capi.Vec2(0.6, 1.1))))
    # a small dynamic tag jointed to the bullet (a revolute joint), carried along and never swept against it
    td.position = capi.Vec2(3.0, -1.0)
    tag = P.s2CreateBody(world, C.byref(td))
    P.s2CreateCircleShape(tag, C.byref(capi.default_shape_def()), C.byref(capi.Circle(capi.Vec2(0.0, 0.0), 0.05)))
    jd = capi.default_revolute_def()
    jd.bodyIdA = body
    jd.bodyIdB = tag
    jd.localAnchorA = capi.Vec2(0.0, -1.0)
    jd.localAnchorB = capi.Vec2(0.0, 0.0)
    P.s2CreateRevoluteJoint(world, C.byref(jd))
    P.s2Body_SetBullet(body, True)
    P.s2World_EnableContinuous(world, True)
    dw = _attach(P, D, world)
    P.s2World_Step(world, DT, 4, 2, True)
    c = dw.counters()
    assert c.bulletShapes == 2 and c.bulletHits == 1
    # the body turns as the joint drags the tag along; the clamped segment's midpoint, in the plank's frame, is short of
    # its face
    o, a = P.s2Body_GetPosition(body), P.s2Body_GetAngle(body)
    mid = capi.Vec2(o.x + math.cos(a) * 0.6 - math.sin(a) * 1.0, o.y + math.sin(a) * 0.6 + math.cos(a) * 1.0)
    assert P.s2Body_GetLocalPoint(plank, mid).x < -0.025
    P.s2DestroyWorld(world)
