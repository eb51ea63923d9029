"""GPU: the bullet pass (DESIGN.md §3.12) against static shapes, and against restatements that share its candidates with
the non-bullet pass of §3.11.

* The seeded compound scene of test_continuous_reference_gpu (its builder, imported), with every body it launches (the
  160 fast compound bodies and the arm jointed to a static body) flagged as a bullet:
  - bit for bit: the bullet pass against a brute-force restatement over every static, kinematic and non-bullet dynamic
    shape, under the filter, joint and segment rules;
  - float64: a clamped bullet is at least target - tol - eps from every shape it may collide with, and an unclamped fast
    bullet never came closer over its sweep, but for pairs that start within target + tol and that the rules let go.
* scenes.projectiles with its projectiles flagged: the bullet pass against static walls gives the §3.11 restatement's
  answer (test_continuous_gpu._host_pass), bit for bit.
* Ordering: a bullet fired at a dynamic plank that the §3.11 pass clamps at a static wall in the same step is swept
  against the plank's clamped pose."""
import ctypes as C

import numpy as np
import pytest

import test_continuous_reference_gpu as cref
from solver2d_b200 import capi, device, scenes
from test_bullet_cpu import host_bullet_pass
from test_continuous_gpu import _core_approaches, _fast, _host_pass, _sweep
from test_continuous_reference_gpu import SEGMENT, _bounding_circles, _collide, _eps, _may_reach, _poses, _still
from test_toi_reference_cpu import TARGET, TOL, Sweep64, min_sep64, sep64

pytestmark = pytest.mark.gpu

DT = 1.0 / 60.0
BULLET = 0x20  # S2B_BODY_BULLET


@pytest.fixture(scope="module")
def P():
    return capi.Solver2D(device.LIB_PATH)


@pytest.fixture(scope="module")
def D():
    return device.Device()


class _Recording(cref.World):
    """The reference scene's world, remembering the bodies it launches (dynamic, created with a velocity)."""

    def __init__(self, P, solver):
        super().__init__(P, solver)
        self.movers = []

    def body(self, kind, pos, angle=0.0, v=(0.0, 0.0), w=0.0, gravity=1.0):
        bid = super().body(kind, pos, angle, v, w, gravity)
        if kind == capi.DYNAMIC_BODY and tuple(v) != (0.0, 0.0):
            self.movers.append(bid)
        return bid


def _compound_scene(P, solver, monkeypatch):
    with monkeypatch.context() as m:
        m.setattr(cref, "World", _Recording)
        return cref.reference_scene(P, solver)


def _is_bullet(flags):
    return (flags & 1) != 0 and (flags >> 1) & 3 == capi.DYNAMIC_BODY and (flags & BULLET) != 0


def brute_force_bullets(P, w, before, after):
    """The bullet pass restated by brute force: as test_continuous_reference_gpu.brute_force, over every shape of a body
    that is static, kinematic, or dynamic and not a bullet, each held at its `after` pose. Returns (body slot -> (fraction,
    sweep) for every clamped bullet, shapes of fast bullets, per fast bullet the (shape, other, verdict) pairs swept)."""
    flags = after["flags"]
    valid = [r for r in w.shapes if (flags[r.body] & 1) != 0]
    by_body = {}
    for r in valid:
        by_body.setdefault(r.body, []).append(r)
    joints = set(w.joints)
    out, swept, pairs = {}, 0, {}
    for b, recs in by_body.items():
        if not _is_bullet(int(flags[b])) or not _fast(before[b], after[b]):
            continue
        others = [r for r in valid if r.body != b and not _is_bullet(int(flags[r.body]))]
        centres, radii = _bounding_circles(others, after)
        swept += len(recs)
        sweep = _sweep(before[b], after[b])
        earliest = 1.0
        pairs[b] = []
        for r in recs:
            ext = P.s2ComputeShapeExtent(C.byref(r.form), capi.Vec2(*before[b]["localCenter"]))
            pb = P.s2MakeProxy(r.form.vertices, r.form.count, r.form.radius)
            for j in _may_reach(r, before[b], after[b], centres, radii):
                s = others[j]
                if not _collide(r, s, joints):
                    continue
                sr = after[s.body]
                ws = capi.Sweep(capi.Vec2(*sr["localCenter"]), capi.Vec2(*sr["position"]), capi.Vec2(*sr["position"]),
                                capi.Rot(*sr["rot"]), capi.Rot(*sr["rot"]))
                pa = P.s2MakeProxy(s.form.vertices, s.form.count, s.form.radius)
                res = P.s2TimeOfImpact(C.byref(capi.TOIInput(pa, pb, ws, sweep, 1.0)))
                verdict = "toi"
                if res.state == capi.TOI_OVERLAPPED and ext.minExtent <= 0.0:
                    pairs[b].append((r, s, "segment let go"))
                    continue
                if res.state == capi.TOI_OVERLAPPED:
                    core = (capi.Vec2 * 1)(ext.center)
                    pc = P.s2MakeProxy(core, 1, np.float32(0.25) * np.float32(ext.minExtent))
                    res = P.s2TimeOfImpact(C.byref(capi.TOIInput(pa, pc, ws, sweep, 1.0)))
                    if res.state == capi.TOI_OVERLAPPED and _core_approaches(P, pa, ws, core, sweep):
                        earliest = 0.0
                        pairs[b].append((r, s, "held"))
                        continue
                    verdict = "core" if res.state in (capi.TOI_HIT, capi.TOI_FAILED) else "core let go"
                pairs[b].append((r, s, verdict))
                if res.state in (capi.TOI_HIT, capi.TOI_FAILED):
                    earliest = min(earliest, res.fraction)
        if earliest < 1.0:
            out[b] = (earliest, sweep)
    return out, swept, pairs


def _step_pair(P, D, monkeypatch, solver, schedule, persistent, steps_before):
    """Two identical compound scenes, steps_before steps with continuous collision off; then one step of each: one still
    off, one with it on and every launched body flagged. The first world's end of step is the solver stage's output of
    both. Returns the worlds, the start rows, those end rows (with the flagged world's bullet bits), the flagged world's
    rows and counters, the non-bullet bodies its §3.11 pass must clamp (test_continuous_reference_gpu.brute_force: a
    slow obstacle knocked fast in the steps before) and the rows the bullet pass sees: the solver stage's poses, but the
    §3.11 pass's clamped poses for those bodies (as the flagged world ends them, checked bit for bit by the caller)."""
    worlds = []
    for _ in range(2):
        w = _compound_scene(P, solver, monkeypatch)
        P.s2World_Flush(w.world)
        dw = device.DeviceWorld.attach(D, w.world)
        dw.set_schedule(schedule)
        dw.set_persistent(persistent)
        worlds.append((w, dw))
    (w_off, d_off), (w_on, d_on) = worlds
    for _ in range(steps_before):
        w_off.step()
        w_on.step()
    cap = d_off.body_cap
    before = d_off.download_all_bodies(cap)
    P.s2World_EnableContinuous(w_on.world, True)
    for bid in w_on.movers:
        P.s2Body_SetBullet(bid, True)
    w_off.step()
    w_on.step()
    got = d_on.download_all_bodies(cap)
    after = d_off.download_all_bodies(cap)
    after["flags"] = got["flags"]  # (the flagged world's bullet bits on the other world's poses)
    clamped, _, _ = cref.brute_force(P, w_on, before, after)
    clamped = {b: v for b, v in clamped.items() if not _is_bullet(int(after["flags"][b]))}
    seen = after.copy()
    for b in clamped:
        seen[b] = got[b]
    return worlds, before, after, got, d_on.counters(), clamped, seen


def _check_pose(P, want, got, after, b, k):
    t, sweep = want[b]
    xf = P.s2GetSweepTransform(C.byref(sweep), t)
    assert np.float32(xf.p.x) == got[b]["origin"][0] and np.float32(xf.p.y) == got[b]["origin"][1], (k, b)
    assert np.float32(xf.q.s) == got[b]["rot"][0] and np.float32(xf.q.c) == got[b]["rot"][1], (k, b)
    assert np.array_equal(got[b]["linearVelocity"], after[b]["linearVelocity"])


@pytest.mark.parametrize("solver", ["TGS_Soft", "PGS_NGS", "XPBD"])
@pytest.mark.parametrize("schedule,persistent", cref.SCHEDULES, ids=["persistent", "launch-by-launch"])
def test_compound_bullets_match_brute_force_bit_for_bit(P, D, monkeypatch, solver, schedule, persistent):
    hits = compound = 0
    for k in (0, 2):
        worlds, before, after, got, counters, clamped, seen = _step_pair(P, D, monkeypatch, solver, schedule, persistent, k)
        w = worlds[0][0]
        want, swept, _ = brute_force_bullets(P, w, before, seen)
        assert counters.bulletShapes == swept, k
        assert counters.bulletHits == len(want), k
        assert counters.continuousHits == len(clamped), k
        for b in range(len(got)):
            if b in want:
                _check_pose(P, want, got, after, b, k)
            elif b in clamped:
                _check_pose(P, clamped, got, after, b, k)
            else:
                assert np.array_equal(_poses(got[b:b + 1]), _poses(after[b:b + 1])), (k, b)
        hits += len(want)
        counts = {}
        for r in w.shapes:
            counts[r.body] = counts.get(r.body, 0) + 1
        compound += sum(1 for b in want if counts[b] >= 2)
        for ww, _ in worlds:
            ww.destroy()
    assert hits >= 40 and compound >= 20, (hits, compound)


def test_compound_bullets_float64(P, D, monkeypatch):
    """float64, independent of s2_toi.h: clamped bullets at their clamped pose, and fast bullets left alone over their
    whole sweep, keep target - tol - eps from every shape they may collide with (static, kinematic and non-bullet dynamic,
    at its final pose). The only exceptions are pairs that start within target + tol and that the rules let go (a
    segment, or a core that does not approach), and for a clamped bullet, pairs it started within target + tol of."""
    worlds, before, after, got, counters, _, seen = _step_pair(P, D, monkeypatch, "TGS_Soft", device.SCHEDULE_COLOR, True, 0)
    w = worlds[0][0]
    want, _, pairs = brute_force_bullets(P, w, before, seen)
    assert len(want) >= 20
    checked, exceptions, let_go, kinds = 0, [], set(), set()
    for b, plist in pairs.items():
        if b in want:
            sweep = _still(got[b])
        else:
            sweep = Sweep64(before[b]["localCenter"], before[b]["position"], after[b]["position"], before[b]["rot"],
                            after[b]["rot"])
        for r, s, verdict in plist:
            A, sa = s.shape64(), _still(seen[s.body])
            B = r.shape64()
            eps = _eps(*seen[s.body]["position"], *before[b]["position"], *after[b]["position"]) + 1e-5
            lo = TARGET - TOL - eps
            start = float(sep64(A, sa, B, _still(before[b]), 0.0)[0])
            if verdict in ("segment let go", "core let go"):
                assert start < TARGET + TOL + eps, (b, verdict, start)
                let_go.add((id(r), id(s)))
            if b in want:
                closest = float(sep64(A, sa, B, sweep, 0.0)[0])
            else:
                closest, _ = min_sep64(A, sa, B, sweep, 0.0, 1.0, floor=lo)
            checked += 1
            kinds.add((int(seen[s.body]["flags"]) >> 1) & 3)
            if r.kind == SEGMENT:
                kinds.add("segment")
            if closest < lo:
                exceptions.append((b, verdict, start, closest, (id(r), id(s))))
    assert checked >= 200
    # swept against static and non-bullet dynamic shapes at least, and with segments among the bullets' shapes
    assert {capi.STATIC_BODY, capi.DYNAMIC_BODY, "segment"} <= kinds, kinds
    assert all(e[4] in let_go for e in exceptions if e[0] not in want), [e[:4] for e in exceptions if e[0] not in want]
    assert all(e[2] < TARGET + TOL + 1e-3 for e in exceptions if e[0] in want), [e[:4] for e in exceptions if e[0] in want]
    for ww, _ in worlds:
        ww.destroy()


@pytest.mark.parametrize("solver", ["TGS_Soft", "PGS_NGS", "XPBD"])
@pytest.mark.parametrize("schedule,persistent", cref.SCHEDULES, ids=["persistent", "launch-by-launch"])
def test_bullets_against_static_walls_match_the_continuous_restatement(P, D, solver, schedule, persistent):
    """scenes.projectiles has static walls only: a flagged projectile's bullet pass sweeps exactly the §3.11 pass's
    candidates, so it must give _host_pass's answer bit for bit, counted as bullet hits and not as continuous hits."""
    hits = 0
    for k in (1, 2, 4):
        worlds = []
        for _ in range(2):
            sc = scenes.projectiles(P, solver)
            P.s2World_Flush(sc.world)
            dw = device.DeviceWorld.attach(D, sc.world)
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
        for lane in s_on.piles["lanes"]:
            P.s2Body_SetBullet(lane["body"], True)
        s_off.step(DT, 4, 2, True)
        s_on.step(DT, 4, 2, True)
        after = d_off.download_all_bodies(cap)
        got = d_on.download_all_bodies(cap)
        want = _host_pass(P, s_off, before, after)
        c = d_on.counters()
        assert c.bulletHits == len(want) and c.continuousHits == 0 and c.continuousShapes == 0, k
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


def _ordering_world(P):
    """A static wall at x = 5; a heavy dynamic plank at x = 3 flying at it at 150 m/s (the §3.11 pass clamps it at the
    wall); a bullet circle at x = 1 fired after it at 300 m/s. Returns (world, shapes for host_bullet_pass, plank, bullet)."""
    world = P.create_world("TGS_Soft")
    wall = P.s2CreateBody(world, C.byref(capi.default_body_def()))
    wall_form = P.s2MakeOffsetBox(0.025, 3.0, capi.Vec2(5.0, 0.0), 0.0)
    P.s2CreatePolygonShape(wall, C.byref(capi.default_shape_def()), C.byref(wall_form))
    bd = capi.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    bd.gravityScale = 0.0
    bd.position = capi.Vec2(3.0, 0.0)
    bd.linearVelocity = capi.Vec2(150.0, 0.0)
    plank = P.s2CreateBody(world, C.byref(bd))
    sd = capi.default_shape_def()
    sd.density = scenes.BULLET_PLANK_DENSITY
    plank_form = P.s2MakeBox(0.025, 2.0)
    P.s2CreatePolygonShape(plank, C.byref(sd), C.byref(plank_form))
    bd.position = capi.Vec2(1.0, 0.0)
    bd.linearVelocity = capi.Vec2(300.0, 0.0)
    bullet = P.s2CreateBody(world, C.byref(bd))
    P.s2CreateCircleShape(bullet, C.byref(capi.default_shape_def()), C.byref(capi.Circle(capi.Vec2(0.0, 0.0), 0.1)))
    circle = capi.Polygon()
    circle.count, circle.radius = 1, 0.1
    default = (1, 0xFFFFFFFF, 0)
    shapes = [dict(body=wall.index, form=wall_form, filter=default, segment=False),
              dict(body=plank.index, form=plank_form, filter=default, segment=False),
              dict(body=bullet.index, form=circle, filter=default, segment=False)]
    return world, shapes, plank, bullet


def test_bullet_meets_the_pose_the_continuous_clamp_left(P, D):
    """The bullet pass runs after the §3.11 clamp and finalize: the bullet stops at the plank as clamped at the wall, not
    at the plank's unclamped end pose nor at its start."""
    worlds = []
    for on in (False, True):
        world, shapes, plank, bullet = _ordering_world(P)
        P.s2World_EnableContinuous(world, on)
        if on:
            P.s2Body_SetBullet(bullet, True)
        P.s2World_Flush(world)
        worlds.append((world, device.DeviceWorld.attach(D, world)))
    (w_off, d_off), (w_on, d_on) = worlds
    cap = d_on.body_cap
    before = d_on.download_all_bodies(cap)
    P.s2World_Step(w_off, DT, 4, 2, True)
    P.s2World_Step(w_on, DT, 4, 2, True)
    free = d_off.download_all_bodies(cap)  # the solver stage's poses, nothing clamped
    got = d_on.download_all_bodies(cap)
    c = d_on.counters()
    assert c.continuousHits == 1 and c.bulletHits == 1
    # the plank was clamped at the wall: its face 5 mm short of the wall's
    assert abs(float(got[plank.index]["position"][0]) + 0.025 - (4.975 - 0.005)) < 0.0015
    # the restatement on the final poses of everything but the bullet, whose sweep ends where the solver stage left it
    rows = got.copy()
    rows[bullet.index] = free[bullet.index]
    rows["flags"] = got["flags"]
    want = host_bullet_pass(P, shapes, before, rows)
    assert list(want) == [bullet.index]
    t, sweep = want[bullet.index]
    xf = P.s2GetSweepTransform(C.byref(sweep), t)
    b = got[bullet.index]
    assert np.float32(xf.p.x) == b["origin"][0] and np.float32(xf.p.y) == b["origin"][1]
    assert np.float32(xf.q.s) == b["rot"][0] and np.float32(xf.q.c) == b["rot"][1]
    # in front of the clamped plank: centre 0.1 m + 5 mm short of its face
    assert abs(float(b["position"][0]) - (float(got[plank.index]["position"][0]) - 0.025 - 0.1 - 0.005)) < 0.0015
    for world, _ in worlds:
        P.s2DestroyWorld(world)
