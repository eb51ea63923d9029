"""GPU: continuous collision of dynamic bodies against static shapes (s2World_EnableContinuous, DESIGN.md §3.11) under all
ten solver variants.

* Tunnelling: on scenes.projectiles some projectiles end behind their walls with the feature off; with it on none is ever
  past its wall's mid-plane, and the filtered and jointed projectiles pass in both modes.
* Bit-exact pass: from identical state one world steps with the feature off and one with it on; the pass is restated on
  the host (s2TimeOfImpact on the downloaded start and end poses, brute force over the static shapes under the same rules)
  and every body's pose must match it bit for bit, in the colour and wavefront schedules, persistent and launch by launch.
* Nothing fast means nothing changes; robustness (teleport, multi-shape body, static and kinematic bodies, toggling,
  S2B_PREFETCH_PAIRS and S2B_GRAPH)."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from solver2d_b200 import capi, device, scenes

pytestmark = pytest.mark.gpu

VARIANTS = ["Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "SoftStep", "TGS_Sticky", "TGS_Soft", "TGS_NGS", "XPBD"]
DT = 1.0 / 60.0
STEPS = 30


@pytest.fixture(scope="module")
def P():
    return capi.Solver2D(device.LIB_PATH)


@pytest.fixture(scope="module")
def D():
    return device.Device()


def _poses(rows):
    return np.concatenate([rows["origin"], rows["position"], rows["rot"]], axis=1)


def _state(rows):
    return np.concatenate([rows["origin"], rows["position"], rows["rot"], rows["linearVelocity"],
                           rows["angularVelocity"][:, None]], axis=1)


@pytest.mark.parametrize("solver", VARIANTS)
def test_projectiles_tunnel_without_and_stop_with_continuous(P, solver):
    ever = {}
    for on in (False, True):
        sc = scenes.projectiles(P, solver)
        P.s2World_EnableContinuous(sc.world, on)
        lanes = sc.piles["lanes"]
        behind = np.zeros(len(lanes), dtype=bool)
        for _ in range(STEPS):
            sc.step(DT, 4, 2, True)
            behind |= scenes.projectiles_behind(P, sc)
        meant = np.array([lane["passes"] for lane in lanes])
        assert behind[meant].all(), f"{solver} on={on}: a filtered or jointed projectile did not pass"
        ever[on] = behind[~meant]
        sc.destroy()
    assert ever[False].sum() >= 1, f"{solver}: nothing tunnels without continuous collision"
    assert ever[True].sum() == 0, f"{solver}: lanes {np.flatnonzero(ever[True]).tolist()} tunnel with continuous collision"


def _attach(P, D, world):
    """Device view of a public-API world, its rows pushed first (so the capacities are known)."""
    P.s2World_Flush(world)
    return device.DeviceWorld.attach(D, world)


def _rows(dw):
    return dw.download_all_bodies(dw.counters().bodyCapacity)


_ATAN2 = None


def _atan2f(y, x):
    """The float atan2 of the device kernels (S2_ATAN2F), evaluated by the host library (s2Atan2Device)."""
    global _ATAN2
    if _ATAN2 is None:
        _ATAN2 = C.CDLL(device.LIB_PATH).s2Atan2Device
        _ATAN2.restype = C.c_float
        _ATAN2.argtypes = [C.c_float, C.c_float]
    return np.float32(_ATAN2(float(y), float(x)))


def _fast(row0, row1):
    """s2bIsFast restated in float32, operation for operation (sqrtf of a float32 is correctly rounded through a double;
    the angle is the device's own atan2)."""
    f = np.float32
    dx = f(row1["position"][0]) - f(row0["position"][0])
    dy = f(row1["position"][1]) - f(row0["position"][1])
    moved = f(math.sqrt(f(dx * dx + dy * dy)))
    s = f(row1["rot"][0] * row0["rot"][1] - row1["rot"][1] * row0["rot"][0])
    c = f(row1["rot"][1] * row0["rot"][1] + row1["rot"][0] * row0["rot"][0])
    return moved + abs(_atan2f(s, c)) * f(row0["maxExtent"]) > f(0.5) * f(row0["minExtent"])


def _sweep(row0, row1):
    return capi.Sweep(capi.Vec2(*row0["localCenter"]), capi.Vec2(*row0["position"]), capi.Vec2(*row1["position"]),
                      capi.Rot(*row0["rot"]), capi.Rot(*row1["rot"]))


def _core_approaches(P, pa, ws, core, sweep):
    """s2cCoreApproaches restated: the core moves toward the static shape by more than the tolerance along their axis."""
    f = np.float32
    inp = capi.DistanceInput(pa, P.s2MakeProxy(core, 1, 0.0), P.s2GetSweepTransform(C.byref(ws), 0.0),
                             P.s2GetSweepTransform(C.byref(sweep), 0.0), False)
    d = P.s2ShapeDistance(C.byref(capi.DistanceCache()), C.byref(inp))
    v = np.array([d.pointB.x - d.pointA.x, d.pointB.y - d.pointA.y], dtype=f)
    length = f(math.sqrt(f(v[0] * v[0] + v[1] * v[1])))
    n = v * (f(1.0) / length) if length >= f(0.001) * f(np.finfo(f).eps) else np.zeros(2, dtype=f)
    dc = np.array([f(sweep.c2.x) - f(sweep.c1.x), f(sweep.c2.y) - f(sweep.c1.y)], dtype=f)
    return -(n[0] * dc[0] + n[1] * dc[1]) > f(0.25 * 0.005)


def _host_pass(P, sc, before, after):
    """The continuous pass restated on the host: body slot -> expected fraction (< 1) for every clamped body."""
    lanes = sc.piles["lanes"]
    walls = [(lane["wall"].index, lane["wall_form"], lane["exclusion"], k) for k, lane in enumerate(lanes)]
    out = {}
    for k, lane in enumerate(lanes):
        b = lane["body"].index
        r0, r1 = before[b], after[b]
        if not _fast(r0, r1):
            continue
        sweep = _sweep(r0, r1)
        form = lane["form"]
        ext = P.s2ComputeShapeExtent(C.byref(form), capi.Vec2(*r0["localCenter"]))
        earliest = 1.0
        for w, wall_form, exclusion, kw in walls:
            if kw == k and exclusion is not None:
                continue  # filtered or jointed: the pair rules drop it
            if lane["exclusion"] == "filter" and exclusion == "filter":
                continue  # a filtered projectile's mask excludes every filtered wall's category
            wr = after[w]
            if np.hypot(*(np.array(wr["position"]) - np.array(r0["position"]))) > 8.0:
                continue
            ws = capi.Sweep(capi.Vec2(*wr["localCenter"]), capi.Vec2(*wr["position"]), capi.Vec2(*wr["position"]),
                            capi.Rot(*wr["rot"]), capi.Rot(*wr["rot"]))
            pa = P.s2MakeProxy(wall_form.vertices, wall_form.count, wall_form.radius)
            pb = P.s2MakeProxy(form.vertices, form.count, form.radius)
            res = P.s2TimeOfImpact(C.byref(capi.TOIInput(pa, pb, ws, sweep, 1.0)))
            if res.state == capi.TOI_OVERLAPPED and ext.minExtent <= 0.0:
                continue  # a segment has no core: touching at the start, it is let go
            if res.state == capi.TOI_OVERLAPPED:
                core = (capi.Vec2 * 1)(ext.center)
                pc = P.s2MakeProxy(core, 1, np.float32(0.25) * np.float32(ext.minExtent))
                res = P.s2TimeOfImpact(C.byref(capi.TOIInput(pa, pc, ws, sweep, 1.0)))
                if res.state == capi.TOI_OVERLAPPED and _core_approaches(P, pa, ws, core, sweep):
                    earliest = 0.0
                    continue
            if res.state in (capi.TOI_HIT, capi.TOI_FAILED):
                earliest = min(earliest, res.fraction)
        if earliest < 1.0:
            out[b] = (earliest, sweep)
    return out


SCHEDULES = [(device.SCHEDULE_COLOR, True), (device.SCHEDULE_COLOR, False), (device.SCHEDULE_WAVEFRONT, True),
             (device.SCHEDULE_WAVEFRONT, False)]


@pytest.mark.parametrize("solver", ["TGS_Soft", "PGS_NGS", "XPBD"])
@pytest.mark.parametrize("schedule,persistent", SCHEDULES, ids=["colour", "colour-launch", "wavefront", "wavefront-launch"])
def test_pass_matches_host_restatement_bit_for_bit(P, D, solver, schedule, persistent):
    hits = 0
    for k in (1, 2, 4):
        # two identical worlds, k - 1 steps with the feature off, then step k: one off, one on
        worlds = []
        for on in (False, True):
            sc = scenes.projectiles(P, solver)
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
        P.s2World_EnableContinuous(s_on.world, True)
        s_off.step(DT, 4, 2, True)
        s_on.step(DT, 4, 2, True)
        after = d_off.download_all_bodies(cap)
        got = d_on.download_all_bodies(cap)
        want = _host_pass(P, s_off, before, after)
        assert d_on.counters().continuousHits == len(want), k
        for b in range(cap):
            if b in want:
                t, sweep = want[b]
                xf = P.s2GetSweepTransform(C.byref(sweep), t)
                assert np.float32(xf.p.x) == got[b]["origin"][0] and np.float32(xf.p.y) == got[b]["origin"][1], (k, b)
                assert np.float32(xf.q.s) == got[b]["rot"][0] and np.float32(xf.q.c) == got[b]["rot"][1], (k, b)
                assert np.array_equal(got[b]["linearVelocity"], after[b]["linearVelocity"])
            else:
                assert np.array_equal(_poses(got[b:b + 1]), _poses(after[b:b + 1])), (k, b)
        hits += len(want)
        for sc, _ in worlds:
            sc.destroy()
    assert hits >= 5


def _compare_on_off(P, D, make, steps, until_clamped=False, no_hold=False):
    """Step a world with the feature off and one with it on; their states must stay bit-identical. With until_clamped,
    up to the first step whose pass clamps a body: there every body that differs must be one the pass moved (as many
    differing bodies as clamped ones, each with the off-world's velocity, which a clamp keeps) and every other body must
    still be bit-equal; the worlds legitimately part from that step on. With no_hold, none of the clamped bodies may be
    held at its start pose (fraction 0). Returns (swept shapes of the last step, the step of the first clamp or None)."""
    a, b = make(), make()
    P.s2World_EnableContinuous(b.world, True)
    da, db = _attach(P, D, a.world), _attach(P, D, b.world)
    first_clamp = None
    rb = _rows(db)
    for step in range(steps):
        before = rb
        a.step(DT, 4, 2, True)
        b.step(DT, 4, 2, True)
        ra, rb = _rows(da), _rows(db)
        hits = db.counters().continuousHits
        if until_clamped and hits > 0:
            differs = ~np.all(_poses(ra) == _poses(rb), axis=1)
            assert differs.sum() == hits, f"step {step}: {differs.sum()} bodies differ, {hits} clamped"
            assert np.array_equal(_state(ra)[~differs], _state(rb)[~differs]), f"step {step}"
            assert np.array_equal(ra["linearVelocity"][differs], rb["linearVelocity"][differs])
            assert np.array_equal(ra["angularVelocity"][differs], rb["angularVelocity"][differs])
            if no_hold:
                held = np.all(_poses(rb)[differs] == _poses(before)[differs], axis=1)
                assert not held.any(), f"step {step}: a body was held at its start pose"
            first_clamp = step
            break
        assert np.array_equal(_state(ra), _state(rb)), f"step {step}"
    shapes = db.counters().continuousShapes
    a.destroy()
    b.destroy()
    return shapes, first_clamp


def _slider_and_wheel(P, solver):
    world = P.create_world(solver)
    sc = scenes.Scene(P, world, name="slide")
    sc.bodies.append(scenes._ground(P, world, 200.0))
    bd = capi.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    bd.position = capi.Vec2(-50.0, 0.25)
    bd.linearVelocity = capi.Vec2(40.0, 0.0)
    bid = P.s2CreateBody(world, C.byref(bd))
    P.s2CreatePolygonShape(bid, C.byref(capi.default_shape_def()), C.byref(P.s2MakeBox(0.25, 0.25)))
    bd.position = capi.Vec2(20.0, 0.3)
    bd.linearVelocity = capi.Vec2(0.0, 0.0)
    bd.angularVelocity = -60.0
    wid = P.s2CreateBody(world, C.byref(bd))
    P.s2CreateCircleShape(wid, C.byref(capi.default_shape_def()), C.byref(capi.Circle(capi.Vec2(0.0, 0.0), 0.3)))
    # a box carrying a segment along its bottom face (minExtent 0: fast whenever it moves; its core is a point at the
    # segment's midpoint, on the ground), sliding
    bd.position = capi.Vec2(-100.0, 0.25)
    bd.linearVelocity = capi.Vec2(15.0, 0.0)
    bd.angularVelocity = 0.0
    sid = P.s2CreateBody(world, C.byref(bd))
    P.s2CreatePolygonShape(sid, C.byref(capi.default_shape_def()), C.byref(P.s2MakeBox(0.5, 0.25)))
    P.s2CreateSegmentShape(sid, C.byref(capi.default_shape_def()),
                           C.byref(capi.Segment(capi.Vec2(-0.5, -0.25), capi.Vec2(0.5, -0.25))))
    sc.bodies += [bid, wid, sid]
    return sc


@pytest.mark.parametrize("solver", VARIANTS)
def test_nothing_fast_nothing_changes(P, D, solver):
    # Jacobi's piles throw boxes fast enough to be swept, and one lands on the ground within a step at step 3: the rigs are
    # identical up to the first clamp there, and for every other variant throughout
    _compare_on_off(P, D, lambda: scenes.kinematic_rigs(P, solver), 60, until_clamped=solver == "Jacobi")
    # fast, but touching the ground from the start: swept, never clamped (nor held, the segment-carrying box included).
    # Jacobi's contacts let the bodies bounce clear of the ground by more than the target separation now and then; a body
    # that comes back down within a step then lands at the target (a clamp at a fraction above 0, never a hold)
    assert _compare_on_off(P, D, lambda: _slider_and_wheel(P, solver), 40, until_clamped=solver == "Jacobi", no_hold=True)[0] > 0


@pytest.mark.parametrize("solver", VARIANTS)
def test_zoo_changes_only_where_the_pass_clamps(P, D, solver):
    """The collision zoo has fast bodies by the rule of DESIGN.md §3.11 (thrown, spinning compounds with a 0.12 m capsule,
    bodies carrying a segment, whose minExtent is 0): a step in which one of them would reach a static shape within the
    step clamps it at the target, where the discrete step lets the speculative contact land it. So the zoo is not
    bit-identical with the feature on: it is up to the first step whose pass clamps a body, and at that step exactly the
    clamped bodies differ."""
    _compare_on_off(P, D, lambda: scenes.collision_zoo(P, solver), 60, until_clamped=True)


def test_pyramid_5050_unchanged(P, D):
    _compare_on_off(P, D, lambda: scenes.pyramid(P, "TGS_Soft", base_count=100), 20)


def test_teleport_across_a_wall_is_not_clamped(P, D):
    sc = scenes.projectiles(P, "TGS_Soft", excluded=False)
    P.s2World_EnableContinuous(sc.world, True)
    lane = sc.piles["lanes"][0]
    sc.step(DT, 4, 2, True)
    cx, cy = lane["center"]
    P.s2Body_SetTransform(lane["body"], capi.Vec2(cx + 1.0, cy), 0.0)
    P.s2Body_SetLinearVelocity(lane["body"], capi.Vec2(1.0, 0.0))
    sc.step(DT, 4, 2, True)
    p = P.s2Body_GetPosition(lane["body"])
    assert p.x > cx + 1.0
    sc.destroy()


def test_multi_shape_body_stops_at_its_earliest_shape_and_static_kinematic_stay(P, D):
    world = P.create_world("TGS_Soft")
    wall = P.s2CreateBody(world, C.byref(capi.default_body_def()))
    P.s2CreatePolygonShape(wall, C.byref(capi.default_shape_def()), C.byref(P.s2MakeOffsetBox(0.025, 3.0, capi.Vec2(5.0, 0.0), 0.0)))
    bd = capi.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    bd.gravityScale = 0.0
    bd.position = capi.Vec2(3.0, 0.0)
    bd.linearVelocity = capi.Vec2(150.0, 0.0)
    body = P.s2CreateBody(world, C.byref(bd))
    sd = capi.default_shape_def()
    P.s2CreateCircleShape(body, C.byref(sd), C.byref(capi.Circle(capi.Vec2(-0.5, 0.0), 0.1)))
    P.s2CreateCircleShape(body, C.byref(sd), C.byref(capi.Circle(capi.Vec2(0.6, 1.0), 0.1)))  # the leading shape
    kd = capi.default_body_def()
    kd.type = capi.KINEMATIC_BODY
    kd.position = capi.Vec2(0.0, 10.0)
    kd.linearVelocity = capi.Vec2(200.0, 0.0)
    kin = P.s2CreateBody(world, C.byref(kd))
    P.s2CreateCircleShape(kin, C.byref(sd), C.byref(capi.Circle(capi.Vec2(0.0, 0.0), 0.1)))
    P.s2World_EnableContinuous(world, True)
    dw = _attach(P, D, world)
    rows = _rows(dw)
    # extents about the centre of mass (the midpoint of the two equal circles)
    lc = np.array([0.05, 0.5])
    assert rows[body.index]["minExtent"] == np.float32(0.1)
    assert abs(rows[body.index]["maxExtent"] - (np.hypot(*(np.array([0.6, 1.0]) - lc)) + 0.1)) < 1e-6
    P.s2World_Step(world, DT, 4, 2, True)
    p = P.s2Body_GetPosition(body)
    # the leading circle stops short of the wall face at x = 4.975: body origin x = 4.975 - 0.1 - slop - 0.6
    assert abs(p.x - (4.975 - 0.1 - 0.005 - 0.6)) < 0.0015
    assert P.s2Body_GetPosition(wall).x == 0.0
    assert abs(P.s2Body_GetPosition(kin).x - 200.0 * DT) < 1e-4
    assert dw.counters().continuousHits == 1
    P.s2DestroyWorld(world)


def test_toggle_takes_effect_next_step_without_recapture(P, D):
    sc = scenes.projectiles(P, "TGS_Soft")
    dw = _attach(P, D, sc.world)
    for _ in range(3):
        sc.step()
    captures = dw.counters().graphCaptures
    P.s2World_EnableContinuous(sc.world, True)
    sc.step()
    c = dw.counters()
    assert c.continuousShapes > 0 and c.continuousHits > 0 and c.graphCaptures == captures
    P.s2World_EnableContinuous(sc.world, False)
    sc.step()
    c = dw.counters()
    assert c.continuousShapes == 0 and c.continuousHits == 0 and c.graphCaptures == captures
    sc.destroy()

    # switched on (nothing to clamp) and off again: the world goes on as one that never had it on
    a, b = _slider_and_wheel(P, "TGS_Soft"), _slider_and_wheel(P, "TGS_Soft")
    da, db = _attach(P, D, a.world), _attach(P, D, b.world)
    for step in range(20):
        P.s2World_EnableContinuous(b.world, 5 <= step < 10)
        a.step()
        b.step()
        assert np.array_equal(_state(_rows(da)), _state(_rows(db))), step
    a.destroy()
    b.destroy()


@pytest.mark.parametrize("env", [("S2B_PREFETCH_PAIRS", "0"), ("S2B_GRAPH", "0")])
def test_results_do_not_depend_on_prefetch_or_graph(P, D, env):
    def run():
        sc = scenes.projectiles(P, "TGS_Soft")
        P.s2World_EnableContinuous(sc.world, True)
        for _ in range(12):
            sc.step()
        rows = _rows(_attach(P, D, sc.world))
        sc.destroy()
        return _state(rows)

    base = run()
    old = os.environ.get(env[0])
    os.environ[env[0]] = env[1]
    try:
        other = run()
    finally:
        if old is None:
            del os.environ[env[0]]
        else:
            os.environ[env[0]] = old
    assert np.array_equal(base, other)
