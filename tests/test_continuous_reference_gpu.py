"""GPU: the continuous pass (s2bContinuousSweep / s2bContinuousClamp, DESIGN.md §3.11) on a seeded scene built here, against
a brute-force restatement and against the float64 reference of tests/test_toi_reference_cpu.py.

The scene: a scene-sized ground, a few thousand small static shapes of every kind (rounded polygons and 8-gons included),
rotated static bodies carrying several offset shapes; fast compound bodies of 2-4 shapes, some metres off their centre of
mass, some carrying a segment, spinning at 10-150 rad/s and moving at 10-150 m/s, most aimed to cross a static shape within
the step; kinematic bodies and slow dynamic obstacles in their paths (which never clamp anything); filters (categories and
a negative group) and a revolute joint to a static body.

* Bit for bit: from identical state one world steps with the feature off and one with it on; every dynamic body that is
  fast is swept on the host against every static shape (no distance cut) under the filter, joint and segment rules, the
  earliest fraction over all its shapes taken; every body's pose must match, and both counters.
* float64: a clamped body's pose is at least target - tol - eps from every static shape it may collide with, and a fast
  body left alone never came closer over its sweep, but for pairs that start within target + tol and that the rules let go.
* The bulge: a bar turning 2.5 rad while it moves hits a circle that lies outside both end-pose boxes.
* Tree edges: one fast and one static shape, a single shape, a wall created between steps, a wall destroyed between steps.
* Held bodies: a body turning within 5e-4 rad of a half turn per step (DESIGN.md §3.11, Limits)."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from solver2d_b200 import capi, device
from test_continuous_gpu import _core_approaches, _fast, _sweep
from test_toi_reference_cpu import TARGET, TOL, Shape64, Sweep64, min_sep64, sep64
from test_toi_reference_cpu import _world as world64

pytestmark = pytest.mark.gpu

DT = 1.0 / 60.0
SCHEDULES = [(device.SCHEDULE_COLOR, True), (device.SCHEDULE_COLOR, False)]
CIRCLE, CAPSULE, SEGMENT, POLYGON = "circle", "capsule", "segment", "polygon"


@pytest.fixture(scope="module")
def P():
    return capi.Solver2D(device.LIB_PATH)


@pytest.fixture(scope="module")
def D():
    return device.Device()


class Rec:
    """What the host keeps of a shape: its body, its form in the body frame (a polygon form: 1 vertex for a circle, 2 for
    a capsule or segment), its kind and its filter."""

    def __init__(self, body, form, kind, filt):
        self.body, self.form, self.kind, self.filter = body, form, kind, (filt.categoryBits, filt.maskBits, filt.groupIndex)

    def shape64(self):
        return Shape64([(self.form.vertices[i].x, self.form.vertices[i].y) for i in range(self.form.count)], self.form.radius)


class World:
    def __init__(self, P, solver):
        self.P = P
        self.world = P.create_world(solver)
        self.shapes = []  # Rec
        self.joints = []  # (body index, body index) pairs whose collision a joint turns off

    def body(self, kind, pos, angle=0.0, v=(0.0, 0.0), w=0.0, gravity=1.0):
        bd = capi.default_body_def()
        bd.type = kind
        bd.position = capi.Vec2(*pos)
        bd.angle = angle
        bd.linearVelocity = capi.Vec2(*v)
        bd.angularVelocity = w
        bd.gravityScale = gravity
        return self.P.s2CreateBody(self.world, C.byref(bd))

    def add(self, body, kind, geom, filt=None):
        """geom: ("circle", centre, r) / ("capsule", p1, p2, r) / ("segment", p1, p2) / ("polygon", s2Polygon)"""
        P = self.P
        sd = capi.default_shape_def()
        if filt is not None:
            sd.filter = filt
        if kind == CIRCLE:
            P.s2CreateCircleShape(body, C.byref(sd), C.byref(capi.Circle(capi.Vec2(*geom[0]), geom[1])))
            form = capi.Polygon()
            form.vertices[0] = capi.Vec2(*geom[0])
            form.count, form.radius = 1, geom[1]
        elif kind == CAPSULE:
            P.s2CreateCapsuleShape(body, C.byref(sd), C.byref(capi.Capsule(capi.Vec2(*geom[0]), capi.Vec2(*geom[1]), geom[2])))
            form = P.s2MakeCapsule(capi.Vec2(*geom[0]), capi.Vec2(*geom[1]), geom[2])
        elif kind == SEGMENT:
            P.s2CreateSegmentShape(body, C.byref(sd), C.byref(capi.Segment(capi.Vec2(*geom[0]), capi.Vec2(*geom[1]))))
            form = P.s2MakeCapsule(capi.Vec2(*geom[0]), capi.Vec2(*geom[1]), 0.0)
        else:
            P.s2CreatePolygonShape(body, C.byref(sd), C.byref(geom[0]))
            form = geom[0]
        self.shapes.append(Rec(body.index, form, kind, sd.filter))

    def step(self):
        self.P.s2World_Step(self.world, DT, 4, 2, True)

    def destroy(self):
        self.P.s2DestroyWorld(self.world)


def _filter(cat=1, mask=0xFFFFFFFF, group=0):
    f = capi.Filter()
    f.categoryBits, f.maskBits, f.groupIndex = cat, mask, group
    return f


def _random_geom(P, rng, kind, size, centre=(0.0, 0.0)):
    cx, cy = centre
    a = rng.uniform(-math.pi, math.pi)
    u = np.array([math.cos(a), math.sin(a)]) * size
    if kind == CIRCLE:
        return (centre, size)
    if kind == CAPSULE:
        return ((cx - u[0], cy - u[1]), (cx + u[0], cy + u[1]), size * rng.uniform(0.2, 0.5))
    if kind == SEGMENT:
        return ((cx - u[0], cy - u[1]), (cx + u[0], cy + u[1]))
    n = int(rng.integers(3, 9))
    style = rng.integers(0, 3)
    if style == 0:
        poly = P.s2MakeOffsetBox(size, size * rng.uniform(0.3, 1.0), capi.Vec2(cx, cy), a)
    else:
        ang = np.sort(rng.uniform(0, 2 * math.pi, n)) if n < 8 else np.arange(8) * math.pi / 4
        pts = (capi.Vec2 * n)(*[capi.Vec2(cx + size * math.cos(t), cy + size * math.sin(t)) for t in ang])
        hull = P.s2ComputeHull(pts, n)
        if hull.count < 3:
            poly = P.s2MakeOffsetBox(size, size, capi.Vec2(cx, cy), a)
        else:
            poly = P.s2MakePolygon(C.byref(hull))
    if style == 2 or rng.random() < 0.3:
        poly.radius = size * rng.uniform(0.1, 0.3)
    return (poly,)


KINDS = [CIRCLE, CAPSULE, SEGMENT, POLYGON]
GROUP = -3       # a negative group shared by some fast bodies and some static shapes: never collide
HIDDEN = 0x4     # a category some static shapes carry and some fast bodies mask out


def reference_scene(P, solver, seed=11):
    """The seeded scene of this file (see the module docstring)."""
    rng = np.random.default_rng(seed)
    w = World(P, solver)
    ground = w.body(capi.STATIC_BODY, (0.0, -1.0))
    w.add(ground, POLYGON, (P.s2MakeBox(400.0, 1.0),))
    # a few thousand small static shapes over 200 m x 40 m, one body each, every kind; some in the negative group, some
    # in the hidden category
    statics = []
    field = w.body(capi.STATIC_BODY, (0.0, 0.0))
    for n in range(2400):
        kind = KINDS[n % 4]
        pos = (rng.uniform(-100, 100), rng.uniform(3, 43))
        filt = _filter(cat=HIDDEN) if n % 11 == 0 else _filter(group=GROUP) if n % 13 == 0 else None
        w.add(field, kind, _random_geom(P, rng, kind, rng.uniform(0.05, 0.3), pos), filt)
        statics.append(pos)
    # rotated static bodies carrying 2-3 shapes up to 2 m off their origin
    for n in range(40):
        pos = (rng.uniform(-100, 100), rng.uniform(3, 43))
        body = w.body(capi.STATIC_BODY, pos, angle=rng.uniform(-math.pi, math.pi))
        for m in range(int(rng.integers(2, 4))):
            kind = KINDS[(n + m) % 4]
            w.add(body, kind, _random_geom(P, rng, kind, rng.uniform(0.1, 0.6), tuple(rng.uniform(-2, 2, 2))))
        statics.append(pos)
    # fast compound bodies, each aimed to cross a static shape within the step
    fast = []
    for n in range(160):
        tx, ty = statics[int(rng.integers(len(statics)))]
        speed = rng.uniform(10, 150)
        a = rng.uniform(-math.pi, math.pi)
        d = np.array([math.cos(a), math.sin(a)])
        start = np.array([tx, ty]) - d * speed * DT * rng.uniform(0.3, 0.9)
        spin = rng.uniform(10, 150) * rng.choice([-1.0, 1.0])
        body = w.body(capi.DYNAMIC_BODY, tuple(start), angle=rng.uniform(-math.pi, math.pi), v=tuple(d * speed), w=spin)
        filt = _filter(mask=~HIDDEN & 0xFFFFFFFF) if n % 5 == 0 else _filter(group=GROUP) if n % 7 == 0 else None
        for m in range(int(rng.integers(2, 5))):
            kind = SEGMENT if m == 1 and n % 3 == 0 else KINDS[int(rng.integers(0, 4))]
            off = rng.uniform(-3.0, 3.0, 2) if rng.random() < 0.4 else rng.uniform(-0.4, 0.4, 2)
            w.add(body, kind, _random_geom(P, rng, kind, rng.uniform(0.08, 0.4), tuple(off)), filt)
        fast.append(body)
    # a fast body jointed to a static body (collideConnected false): the static body's shapes never clamp it
    anchor = w.body(capi.STATIC_BODY, (50.0, 20.0))
    w.add(anchor, POLYGON, (P.s2MakeBox(0.5, 0.5),))
    w.add(anchor, SEGMENT, ((-3.0, -1.0), (3.0, -1.0)))
    arm = w.body(capi.DYNAMIC_BODY, (52.0, 20.0), v=(0.0, 60.0), w=80.0)
    w.add(arm, POLYGON, (P.s2MakeOffsetBox(2.5, 0.1, capi.Vec2(0.0, 0.0), 0.0),))
    jd = capi.default_revolute_def()
    jd.bodyIdA, jd.bodyIdB = anchor, arm
    jd.localAnchorA, jd.localAnchorB = capi.Vec2(0.0, 0.0), capi.Vec2(-2.0, 0.0)
    P.s2CreateRevoluteJoint(w.world, C.byref(jd))
    w.joints.append((anchor.index, arm.index))
    # kinematic bodies and slow dynamic obstacles in the field: neither is ever a reason to clamp
    for n in range(12):
        body = w.body(capi.KINEMATIC_BODY, (rng.uniform(-100, 100), rng.uniform(3, 43)), v=tuple(rng.uniform(-150, 150, 2)), w=100.0)
        w.add(body, POLYGON, (P.s2MakeBox(0.3, 0.3),))
    for n in range(40):
        tx, ty = statics[int(rng.integers(len(statics)))]
        body = w.body(capi.DYNAMIC_BODY, (tx + rng.uniform(-2, 2), ty + rng.uniform(-2, 2)), gravity=0.0)
        w.add(body, CIRCLE, ((0.0, 0.0), 0.2))
    return w


# ---------------------------------------------------------------------------------------------------------------------
# the brute-force restatement
# ---------------------------------------------------------------------------------------------------------------------

def _collide(a, b, joints):
    """the broad phase's rules for a fast shape a against a static shape b"""
    (ca, ma, ga), (cb, mb, gb) = a.filter, b.filter
    if ga == gb and ga != 0:
        if ga < 0:
            return False
    elif (ma & cb) == 0 or (ca & mb) == 0:
        return False
    if (a.body, b.body) in joints or (b.body, a.body) in joints:
        return False
    return not (a.kind == SEGMENT and b.kind == SEGMENT)


def _bounding_circles(recs, rows):
    """world centre and radius of a circle holding each shape"""
    centres, radii = np.zeros((len(recs), 2)), np.zeros(len(recs))
    for k, r in enumerate(recs):
        world = _world_verts(r.shape64(), rows[r.body])
        centres[k] = world.mean(axis=0)
        radii[k] = np.hypot(*(world - centres[k]).T).max() + r.form.radius
    return centres, radii


def _may_reach(rec, row0, row1, centres, radii, margin=0.05):
    """Conservative cut by exact geometry (not the device's box): the fast shape stays within its outer extent of the
    centre's path, each static shape within its bounding circle."""
    v = rec.shape64().v
    outer = np.hypot(*(v - row0["localCenter"]).T).max() + rec.form.radius
    c1, c2 = np.asarray(row0["position"], float), np.asarray(row1["position"], float)
    e = c2 - c1
    s = np.clip((centres - c1) @ e / max(float(e @ e), 1e-30), 0.0, 1.0)
    d = np.hypot(*(centres - c1 - s[:, None] * e).T)
    return np.flatnonzero(d <= outer + radii + TARGET + TOL + margin)


def brute_force(P, w, before, after):
    """body slot -> (fraction, sweep) for every body the pass must clamp; the number of shapes on fast bodies; and for
    every fast body the list of (shape rec, static rec, verdict) of the pairs swept ('toi', 'segment let go', 'core let
    go')."""
    flags = after["flags"]
    static = [r for r in w.shapes if (flags[r.body] >> 1) & 3 == capi.STATIC_BODY]
    centres, radii = _bounding_circles(static, after)
    by_body = {}
    for r in w.shapes:
        by_body.setdefault(r.body, []).append(r)
    joints = set(w.joints)
    out, swept, pairs = {}, 0, {}
    for b, recs in by_body.items():
        if (flags[b] & 1) == 0 or (flags[b] >> 1) & 3 != capi.DYNAMIC_BODY or not _fast(before[b], after[b]):
            continue
        swept += len(recs)
        sweep = _sweep(before[b], after[b])
        earliest = 1.0
        pairs[b] = []
        for r in recs:
            ext = P.s2ComputeShapeExtent(C.byref(r.form), capi.Vec2(*before[b]["localCenter"]))
            pb = P.s2MakeProxy(r.form.vertices, r.form.count, r.form.radius)
            for j in _may_reach(r, before[b], after[b], centres, radii):
                s = static[j]
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


def _step_pair(P, D, solver, schedule, persistent, steps_before):
    """two identical worlds, steps_before steps with the feature off, then one step: one off, one on"""
    worlds = []
    for on in (False, True):
        w = reference_scene(P, solver)
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
    w_off.step()
    w_on.step()
    return worlds, before, d_off.download_all_bodies(cap), d_on.download_all_bodies(cap), d_on.counters()


def _rows(dw):
    return dw.download_all_bodies(dw.counters().bodyCapacity)


def _poses(rows):
    return np.concatenate([rows["origin"], rows["position"], rows["rot"]], axis=1)


@pytest.mark.parametrize("solver", ["TGS_Soft", "PGS_NGS", "XPBD"])
@pytest.mark.parametrize("schedule,persistent", SCHEDULES, ids=["persistent", "launch-by-launch"])
def test_pass_matches_brute_force_bit_for_bit(P, D, solver, schedule, persistent):
    hits = compound = 0
    for k in (0, 2):
        worlds, before, after, got, counters = _step_pair(P, D, solver, schedule, persistent, k)
        w = worlds[0][0]
        want, swept, _ = brute_force(P, w, before, after)
        assert counters.continuousShapes == swept, k
        assert counters.continuousHits == len(want), k
        for b in range(len(got)):
            if b in want:
                t, sweep = want[b]
                xf = P.s2GetSweepTransform(C.byref(sweep), t)
                assert np.float32(xf.p.x) == got[b]["origin"][0] and np.float32(xf.p.y) == got[b]["origin"][1], (k, b)
                assert np.float32(xf.q.s) == got[b]["rot"][0] and np.float32(xf.q.c) == got[b]["rot"][1], (k, b)
                assert np.array_equal(got[b]["linearVelocity"], after[b]["linearVelocity"])
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


def _eps(*coords):
    return 2e-5 + 8 * float(np.spacing(np.float32(max(abs(float(c)) for c in coords))))


def _still(row):
    return Sweep64(row["localCenter"], row["position"], row["position"], row["rot"], row["rot"])


def test_float64_no_fast_body_passes_a_static_shape(P, D):
    """float64, independent of s2_toi.h: clamped bodies at their clamped pose, and fast bodies left alone over their whole
    sweep, keep target - tol - eps from every static shape they may collide with. The only exceptions are pairs that
    start within target + tol and that the rules let go (a segment, or a core that does not approach)."""
    worlds, before, after, got, counters = _step_pair(P, D, "TGS_Soft", device.SCHEDULE_COLOR, True, 0)
    w = worlds[0][0]
    want, _, pairs = brute_force(P, w, before, after)
    assert len(want) >= 20
    checked, exceptions, let_go = 0, [], set()
    for b, plist in pairs.items():
        if b in want:
            row = got[b]
            sweep = _still(row)
        else:
            row = after[b]
            sweep = Sweep64(before[b]["localCenter"], before[b]["position"], after[b]["position"], before[b]["rot"], after[b]["rot"])
        for r, s, verdict in plist:
            A, sa = s.shape64(), _still(after[s.body])
            B = r.shape64()
            eps = _eps(*after[s.body]["position"], *before[b]["position"], *after[b]["position"]) + 1e-5
            lo = TARGET - TOL - eps
            start = float(sep64(A, sa, B, Sweep64(before[b]["localCenter"], before[b]["position"], before[b]["position"],
                                                  before[b]["rot"], before[b]["rot"]), 0.0)[0])
            if verdict in ("segment let go", "core let go"):
                assert start < TARGET + TOL + eps, (b, verdict, start)
                let_go.add((id(r), id(s)))
            if b in want:
                closest = float(sep64(A, sa, B, sweep, 0.0)[0])
            else:
                closest, _ = min_sep64(A, sa, B, sweep, 0.0, 1.0, floor=lo)
            checked += 1
            if closest < lo:
                exceptions.append((b, verdict, start, closest, (id(r), id(s))))
    assert checked >= 200
    # a fast body left alone came closer than the target only to a static shape the rules let go (a segment, or a core
    # that does not approach), having started within target + tol; a clamped body is at its pose closer than the target
    # only to a static shape it started within target + tol of (held there, stopped by its core, or let go)
    assert all(e[4] in let_go for e in exceptions if e[0] not in want), [e[:4] for e in exceptions if e[0] not in want]
    assert all(e[2] < TARGET + TOL + 1e-3 for e in exceptions if e[0] in want), [e[:4] for e in exceptions if e[0] in want]
    for ww, _ in worlds:
        ww.destroy()


def _bar_world(P, circle=None):
    w = World(P, "TGS_Soft")
    bar = w.body(capi.DYNAMIC_BODY, (0.0, 10.0), angle=math.radians(18.4), v=(30.0, 0.0), w=173.4, gravity=0.0)
    w.add(bar, POLYGON, (P.s2MakeBox(1.5, 0.05),))
    if circle is not None:
        post = w.body(capi.STATIC_BODY, circle)
        w.add(post, CIRCLE, ((0.0, 0.0), 0.05))
    # something static far away, so that the hierarchy has more than one leaf without the circle
    far = w.body(capi.STATIC_BODY, (0.0, -50.0))
    w.add(far, POLYGON, (P.s2MakeBox(1.0, 1.0),))
    return w, bar


def _aabb(shape, row):
    v = _world_verts(shape, row)
    return v.min(axis=0) - shape.r, v.max(axis=0) + shape.r


def _world_verts(shape, row):
    q = row["rot"]
    return row["origin"] + np.stack([q[1] * shape.v[:, 0] - q[0] * shape.v[:, 1], q[0] * shape.v[:, 0] + q[1] * shape.v[:, 1]], axis=1)


def test_bulge_of_a_turning_bar_is_swept(P, D):
    """A 3 m bar turns about 2.5 rad in one step while it moves 0.5 m; its tip's arc bulges 1 m past the union of its two
    end-pose boxes. A small static circle sits there: the pass must clamp the bar."""
    w, bar = _bar_world(P)
    P.s2World_Flush(w.world)
    dw = device.DeviceWorld.attach(D, w.world)
    r0 = _rows(dw)[bar.index]
    w.step()
    r1 = _rows(dw)[bar.index]
    w.destroy()
    shape = w.shapes[0].shape64()
    sweep = Sweep64(r0["localCenter"], r0["position"], r1["position"], r0["rot"], r1["rot"])
    phi = math.atan2(r0["rot"][1] * r1["rot"][0] - r0["rot"][0] * r1["rot"][1], np.dot(r0["rot"], r1["rot"]))
    assert 2.3 < phi < 2.7
    # the tip at mid-sweep, pulled 3 cm into the bar's path
    tips = world64(shape, sweep, np.array([0.5]))[0]
    tip = tips[np.argmax(tips[:, 1])]
    centre = 0.5 * (sweep.c1 + sweep.c2)
    circle = centre + (tip - centre) * (1.0 - 0.03 / np.hypot(*(tip - centre)))
    post = Shape64([(0.0, 0.0)], 0.05)
    for row in (r0, r1):
        lo, hi = _aabb(shape, row)
        assert np.any(circle + 0.05 < lo) or np.any(circle - 0.05 > hi), row  # misses both end-pose boxes
    post_sweep = Sweep64((0, 0), circle, circle, (0, 1), (0, 1))
    closest, _ = min_sep64(post, post_sweep, shape, sweep, 0.0, 1.0)
    assert closest < 0.0  # the bar passes through the circle
    off, bar_off = _bar_world(P, tuple(circle))
    on, bar_on = _bar_world(P, tuple(circle))
    P.s2World_EnableContinuous(on.world, True)
    d_off, d_on = device.DeviceWorld.attach(D, off.world), device.DeviceWorld.attach(D, on.world)
    off.step()
    on.step()
    a = _rows(d_off)[bar_off.index]
    g = _rows(d_on)[bar_on.index]
    assert np.array_equal(a["rot"], r1["rot"])  # the circle did not touch the bar in the discrete step
    assert d_on.counters().continuousHits == 1
    assert not np.array_equal(g["rot"], a["rot"])
    assert float(sep64(post, post_sweep, shape, _still(g), 0.0)[0]) >= TARGET - TOL - _eps(*circle) - 1e-5
    off.destroy()
    on.destroy()


def _ball(w, pos, v):
    ball = w.body(capi.DYNAMIC_BODY, pos, v=v, gravity=0.0)
    w.add(ball, CIRCLE, ((0.0, 0.0), 0.1))
    return ball


def _wall(w, x):
    wall = w.body(capi.STATIC_BODY, (x, 0.0))
    w.add(wall, POLYGON, (w.P.s2MakeBox(0.025, 2.0),))
    return wall


def test_one_fast_shape_and_one_static_shape(P, D):
    """two leaves in the hierarchy: the smallest tree the sweep walks"""
    w = World(P, "TGS_Soft")
    ball = _ball(w, (-1.0, 0.0), (120.0, 0.0))
    _wall(w, 0.5)
    P.s2World_EnableContinuous(w.world, True)
    dw = device.DeviceWorld.attach(D, w.world)
    w.step()
    assert dw.counters().continuousHits == 1
    assert abs(P.s2Body_GetPosition(ball).x - (0.475 - 0.1 - TARGET)) < 2 * TOL
    w.destroy()


def test_single_shape_world_is_unchanged(P, D):
    rows = []
    for on in (False, True):
        w = World(P, "TGS_Soft")
        _ball(w, (-1.0, 0.0), (120.0, 30.0))
        P.s2World_EnableContinuous(w.world, on)
        dw = device.DeviceWorld.attach(D, w.world)
        for _ in range(3):
            w.step()
        rows.append(_rows(dw))
        assert dw.counters().continuousHits == 0
        w.destroy()
    assert np.array_equal(_poses(rows[0]), _poses(rows[1]))


def _with_env(name, value, fn):
    old = os.environ.get(name)
    os.environ[name] = value
    try:
        return fn()
    finally:
        if old is None:
            del os.environ[name]
        else:
            os.environ[name] = old


@pytest.mark.parametrize("prefetch", ["1", "0"])
def test_wall_created_between_steps_is_swept(P, D, prefetch):
    def run():
        w = World(P, "TGS_Soft")
        ball = _ball(w, (-6.0, 0.0), (120.0, 0.0))
        _wall(w, -40.0)  # (a static shape from the start, so the first steps build a tree)
        P.s2World_EnableContinuous(w.world, True)
        dw = device.DeviceWorld.attach(D, w.world)
        w.step()
        w.step()
        x = P.s2Body_GetPosition(ball).x
        _wall(w, x + 1.0)
        w.step()
        hits = dw.counters().continuousHits
        end = P.s2Body_GetPosition(ball).x
        w.destroy()
        return x, hits, end

    x, hits, end = _with_env("S2B_PREFETCH_PAIRS", prefetch, run)
    assert hits == 1
    assert abs(end - (x + 1.0 - 0.025 - 0.1 - TARGET)) < 2 * TOL


@pytest.mark.parametrize("prefetch", ["1", "0"])
def test_wall_destroyed_between_steps_clamps_nothing(P, D, prefetch):
    def run():
        rows, hits = [], []
        for on in (False, True):
            w = World(P, "TGS_Soft")
            _ball(w, (-6.0, 0.0), (120.0, 0.0))
            wall = _wall(w, -2.0 + 3.0)
            _wall(w, -40.0)
            P.s2World_EnableContinuous(w.world, on)
            dw = device.DeviceWorld.attach(D, w.world)
            w.step()  # the ball ends 5 m short of the wall
            P.s2DestroyBody(wall)
            for _ in range(3):
                w.step()
                hits.append(dw.counters().continuousHits)
            rows.append(_rows(dw))
            w.destroy()
        return rows, hits

    rows, hits = _with_env("S2B_PREFETCH_PAIRS", prefetch, run)
    assert hits == [0] * 6
    assert np.array_equal(_poses(rows[0]), _poses(rows[1]))


def test_half_turn_per_step_is_held(P, D):
    """A free body spinning so that each step turns it within 5e-4 rad of a half turn (4 sub-steps of atan(w h) each) has
    an angular bound of 8e3 or more: the time of impact crawls and fails near 0 against a static shape in its swept box,
    even one off its path. Pinned as a limit (DESIGN.md §3.11): the body is held within a few percent of its start pose
    every step while its velocity is kept."""
    w_h = math.tan(math.pi / 4 - 1e-5 / 4)  # 4 sub-steps of atan(w h) = pi / 4 - 2.5e-6
    omega = w_h * 240.0
    w = World(P, "TGS_Soft")
    body = w.body(capi.DYNAMIC_BODY, (0.0, 0.0), v=(6.0, 0.0), w=omega, gravity=0.0)
    w.add(body, POLYGON, (P.s2MakeBox(1.0, 0.1),))
    # a static box in the swept box (the bar sweeps a disc of radius 1 about its centre; the box's corner reaches 1.4)
    post = w.body(capi.STATIC_BODY, (1.3, 1.3))
    w.add(post, POLYGON, (P.s2MakeBox(0.15, 0.15),))
    P.s2World_EnableContinuous(w.world, True)
    P.s2World_Flush(w.world)
    dw = device.DeviceWorld.attach(D, w.world)
    start = P.s2Body_GetPosition(body)
    for _ in range(4):
        before = _rows(dw)[body.index]
        w.step()
        after = _rows(dw)[body.index]
        assert dw.counters().continuousHits == 1
        assert np.abs(after["position"] - before["position"]).max() <= 0.05 * 6.0 * DT
    assert abs(P.s2Body_GetPosition(body).x - start.x) < 0.05 * 0.4  # of 0.4 m of travel
    assert np.hypot(*after["linearVelocity"]) == pytest.approx(6.0, rel=1e-3)
    w.destroy()
