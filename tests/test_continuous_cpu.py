"""CPU: the time of impact behind continuous collision (s2TimeOfImpact, csrc/shared/s2_toi.h — the same source the device's
continuous pass compiles), the shape extents bodies are classified by, and the projectile scene on the reference.

Known answers: a translating circle against a segment and a box lands at the analytic fraction; a purely rotating box stops
before its corner reaches a wall; a miss is separated at fraction 1; a pair that starts within the target is overlapped.
A seeded property test over every pair of shape kinds checks that a hit lies at the target separation, that no earlier
sample comes closer, that a separated sweep stays clear, and that no case runs out of iterations."""
import ctypes as C
import math

import numpy as np
import pytest

from solver2d_b200 import capi, device, scenes

TARGET = 0.005      # s2_linearSlop
TOL = 0.25 * TARGET  # S2C_TOI_TOLERANCE
# float32 round-off of the GJK distance at coordinates of a few metres
EPS = 2e-5


@pytest.fixture(scope="module")
def lib():
    return capi.Solver2D(device.LIB_PATH)


def rot(a):
    return capi.Rot(math.sin(a), math.cos(a))


def sweep(c1, c2, a1=0.0, a2=0.0, lc=(0.0, 0.0)):
    return capi.Sweep(capi.Vec2(*lc), capi.Vec2(*c1), capi.Vec2(*c2), rot(a1), rot(a2))


def proxy(lib, poly):
    return lib.s2MakeProxy(poly.vertices, poly.count, poly.radius)


def circle_poly(r, c=(0.0, 0.0)):
    p = capi.Polygon()
    p.vertices[0] = capi.Vec2(*c)
    p.count = 1
    p.radius = r
    return p


def toi(lib, pa, sa, pb, sb, t_max=1.0):
    inp = capi.TOIInput(proxy(lib, pa), proxy(lib, pb), sa, sb, t_max)
    return lib.s2TimeOfImpact(C.byref(inp))


def separation(lib, pa, sa, pb, sb, t):
    xa = lib.s2GetSweepTransform(C.byref(sa), t)
    xb = lib.s2GetSweepTransform(C.byref(sb), t)
    inp = capi.DistanceInput(proxy(lib, pa), proxy(lib, pb), xa, xb, False)
    cache = capi.DistanceCache()
    out = lib.s2ShapeDistance(C.byref(cache), C.byref(inp))
    return out.distance - pa.radius - pb.radius


def test_circle_against_segment_at_the_analytic_fraction(lib):
    seg = lib.s2MakeCapsule(capi.Vec2(0.0, -1.0), capi.Vec2(0.0, 1.0), 0.0)
    ball = circle_poly(0.1)
    wall = sweep((0.0, 0.0), (0.0, 0.0))
    shot = sweep((-2.0, 0.3), (2.0, 0.3))  # 4 m per step through a segment
    out = toi(lib, seg, wall, ball, shot)
    assert out.state == capi.TOI_HIT
    want = (2.0 - 0.1 - TARGET) / 4.0
    assert abs(out.fraction - want) * 4.0 <= TOL + EPS
    assert out.iterations <= 2  # head-on: conservative advancement lands in one step


def test_circle_against_box_at_the_analytic_fraction(lib):
    box = lib.s2MakeBox(0.025, 2.0)
    ball = circle_poly(0.1)
    out = toi(lib, box, sweep((0.0, 0.0), (0.0, 0.0)), ball, sweep((-1.5, -0.5), (1.5, -0.5)))
    assert out.state == capi.TOI_HIT
    want = (1.5 - 0.025 - 0.1 - TARGET) / 3.0
    assert abs(out.fraction - want) * 3.0 <= TOL + EPS


def test_rotating_box_stops_before_its_corner_crosses_a_wall(lib):
    # a 1 x 0.2 box spinning about its centre by 1.2 rad next to a wall at x = 0.45: its corner (0.51 from the centre) would
    # cross it
    box = lib.s2MakeBox(0.5, 0.1)
    wall = lib.s2MakeCapsule(capi.Vec2(0.45, -2.0), capi.Vec2(0.45, 2.0), 0.0)
    spin = sweep((0.0, 0.0), (0.0, 0.0), 1.4, 1.4 - 1.2)
    fixed = sweep((0.0, 0.0), (0.0, 0.0))
    out = toi(lib, wall, fixed, box, spin)
    assert out.state == capi.TOI_HIT
    assert 0.0 < out.fraction < 1.0
    assert abs(separation(lib, wall, fixed, box, spin, out.fraction) - TARGET) <= TOL + EPS
    assert separation(lib, wall, fixed, box, spin, 1.0) <= 0.0  # the end pose overlaps the wall


def test_miss_is_separated_at_fraction_one(lib):
    seg = lib.s2MakeCapsule(capi.Vec2(0.0, -1.0), capi.Vec2(0.0, 1.0), 0.0)
    out = toi(lib, seg, sweep((0.0, 0.0), (0.0, 0.0)), circle_poly(0.1), sweep((-2.0, 1.5), (2.0, 1.5)))
    assert out.state == capi.TOI_SEPARATED and out.fraction == 1.0
    out = toi(lib, seg, sweep((0.0, 0.0), (0.0, 0.0)), circle_poly(0.1), sweep((-2.0, 0.0), (-1.0, 0.0)))
    assert out.state == capi.TOI_SEPARATED and out.fraction == 1.0


def test_pair_starting_within_the_target_is_overlapped(lib):
    box = lib.s2MakeBox(1.0, 1.0)
    ball = circle_poly(0.1)
    out = toi(lib, box, sweep((0.0, 0.0), (0.0, 0.0)), ball, sweep((0.0, 1.1 + 0.002), (0.0, 5.0)))
    assert out.state == capi.TOI_OVERLAPPED and out.fraction == 0.0
    out = toi(lib, box, sweep((0.0, 0.0), (0.0, 0.0)), ball, sweep((0.0, 0.5), (0.0, 5.0)))
    assert out.state == capi.TOI_OVERLAPPED


def _shape(lib, kind, rng):
    if kind == "circle":
        return circle_poly(float(rng.uniform(0.05, 0.4)), (float(rng.uniform(-0.2, 0.2)), float(rng.uniform(-0.2, 0.2))))
    if kind == "capsule":
        h = float(rng.uniform(0.1, 0.6))
        return lib.s2MakeCapsule(capi.Vec2(-h, 0.0), capi.Vec2(h, float(rng.uniform(-0.1, 0.1))), float(rng.uniform(0.03, 0.2)))
    if kind == "segment":
        h = float(rng.uniform(0.2, 1.0))
        return lib.s2MakeCapsule(capi.Vec2(-h, float(rng.uniform(-0.2, 0.2))), capi.Vec2(h, 0.0), 0.0)
    if kind == "box":
        p = lib.s2MakeBox(float(rng.uniform(0.05, 0.6)), float(rng.uniform(0.05, 0.6)))
        p.radius = float(rng.choice([0.0, 0.05]))
        return p
    n = int(rng.integers(3, 9))
    pts = (capi.Vec2 * n)(*[capi.Vec2(float(0.4 * math.cos(2 * math.pi * m / n + rng.uniform(-0.2, 0.2))),
                                      float(0.4 * math.sin(2 * math.pi * m / n + rng.uniform(-0.2, 0.2)))) for m in range(n)])
    return lib.s2MakePolygon(C.byref(lib.s2ComputeHull(pts, n)))


KINDS = ["circle", "capsule", "segment", "box", "hull"]
PAIRS = [(a, b) for a in KINDS for b in KINDS if not (a == "segment" and b == "segment")]


@pytest.mark.parametrize("kinds", PAIRS, ids=[f"{a}-{b}" for a, b in PAIRS])
def test_property_seeded_sweeps(lib, kinds):
    rng = np.random.default_rng(KINDS.index(kinds[0]) * 10 + KINDS.index(kinds[1]))
    hits = seps = 0
    for trial in range(40):
        pa, pb = _shape(lib, kinds[0], rng), _shape(lib, kinds[1], rng)
        # A moves little, B crosses its neighbourhood; both rotate
        a0 = float(rng.uniform(-3, 3))
        sa = sweep(tuple(rng.uniform(-0.2, 0.2, 2)), tuple(rng.uniform(-0.2, 0.2, 2)), a0, a0 + float(rng.uniform(-0.6, 0.6)),
                   tuple(rng.uniform(-0.05, 0.05, 2)))
        start = rng.uniform(-1.0, 1.0, 2)
        start = start / np.linalg.norm(start) * 2.5
        end = -start + rng.uniform(-1.2, 1.2, 2)
        a1 = float(rng.uniform(-3, 3))
        sb = sweep(tuple(start), tuple(end), a1, a1 + float(rng.uniform(-1.0, 1.0)), tuple(rng.uniform(-0.05, 0.05, 2)))
        out = toi(lib, pa, sa, pb, sb)
        assert out.iterations < capi.TOI_MAX_ITERATIONS and out.state != capi.TOI_FAILED, (trial, out.iterations)
        if out.state == capi.TOI_OVERLAPPED:
            continue
        end_t = out.fraction if out.state == capi.TOI_HIT else 1.0
        samples = np.linspace(0.0, end_t, 200, endpoint=False)
        closest = min(separation(lib, pa, sa, pb, sb, float(t)) for t in samples)
        if out.state == capi.TOI_HIT:
            hits += 1
            d = separation(lib, pa, sa, pb, sb, out.fraction)
            assert TARGET - TOL - EPS <= d <= TARGET + TOL + EPS, (trial, d)
            assert closest >= TARGET - TOL - EPS, (trial, closest)
        else:
            assert out.state == capi.TOI_SEPARATED and out.fraction == 1.0
            seps += 1
            assert closest >= TARGET - TOL - EPS, (trial, closest)
            assert separation(lib, pa, sa, pb, sb, 1.0) >= TARGET - TOL - EPS
    assert hits >= 5, (hits, seps)


def test_sweep_transform_interpolates_centre_and_rotation(lib):
    s = sweep((0.0, 0.0), (2.0, 4.0), 0.0, 1.0, lc=(0.5, 0.0))
    xf = lib.s2GetSweepTransform(C.byref(s), 0.5)
    q = np.array([0.5 * math.sin(1.0), 0.5 + 0.5 * math.cos(1.0)])
    q /= np.linalg.norm(q)
    assert abs(xf.q.s - q[0]) < 1e-6 and abs(xf.q.c - q[1]) < 1e-6
    # origin = centre - R(q) * localCenter
    assert abs(xf.p.x - (1.0 - 0.5 * q[1])) < 1e-6 and abs(xf.p.y - (2.0 - 0.5 * q[0])) < 1e-6


def test_shape_extents_match_hand_values(lib):
    def ext(poly, lc=(0.0, 0.0)):
        e = lib.s2ComputeShapeExtent(C.byref(poly), capi.Vec2(*lc))
        return e.minExtent, e.maxExtent

    mn, mx = ext(circle_poly(0.3, (0.4, 0.0)), (0.1, 0.0))
    assert mn == pytest.approx(0.3) and mx == pytest.approx(0.6)
    mn, mx = ext(lib.s2MakeCapsule(capi.Vec2(-0.5, 0.0), capi.Vec2(0.5, 0.0), 0.2))
    assert mn == pytest.approx(0.2) and mx == pytest.approx(0.7)
    mn, mx = ext(lib.s2MakeCapsule(capi.Vec2(-1.0, 0.0), capi.Vec2(1.0, 0.0), 0.0), (0.0, 1.0))
    assert mn == 0.0 and mx == pytest.approx(math.sqrt(2.0))
    mn, mx = ext(lib.s2MakeBox(0.5, 0.25))
    assert mn == pytest.approx(0.25) and mx == pytest.approx(math.hypot(0.5, 0.25))
    rounded = lib.s2MakeBox(0.5, 0.25)
    rounded.radius = 0.1
    mn, mx = ext(rounded)
    assert mn == pytest.approx(0.35) and mx == pytest.approx(math.hypot(0.5, 0.25) + 0.1)
    # an offset box: the inner extent is measured from its own centroid, the outer from the body's centre
    mn, mx = ext(lib.s2MakeOffsetBox(0.3, 0.2, capi.Vec2(1.0, 0.0), 0.0))
    assert mn == pytest.approx(0.2) and mx == pytest.approx(math.hypot(1.3, 0.2))


def test_body_extents_match_hand_values(lib):
    """The combination the host stores per body (s2ComputeBodyExtent, called by shape creation): a body of a circle of
    radius 0.1 at (-0.5, 0), a circle of radius 0.1 at (0.6, 1.0) and a 0.4 x 0.2 box centred at (0, -0.3), about the
    centre of mass (0.05, 0.3)."""
    lc = capi.Vec2(0.05, 0.3)
    forms = (capi.Polygon * 3)(circle_poly(0.1, (-0.5, 0.0)), circle_poly(0.1, (0.6, 1.0)),
                               lib.s2MakeOffsetBox(0.2, 0.1, capi.Vec2(0.0, -0.3), 0.0))
    e = lib.s2ComputeBodyExtent(forms, 3, lc)
    # smallest inner extent: the box's half height 0.1 ties the circles' radius 0.1
    assert e.minExtent == pytest.approx(0.1)
    # largest outer extent: the second circle, |(0.6, 1.0) - (0.05, 0.3)| + 0.1
    assert e.maxExtent == pytest.approx(math.hypot(0.55, 0.7) + 0.1)
    # with a segment the inner extent is 0 (such a body is fast whenever it moves)
    forms2 = (capi.Polygon * 2)(forms[2], lib.s2MakeCapsule(capi.Vec2(-1.0, 0.0), capi.Vec2(1.0, 0.0), 0.0))
    e = lib.s2ComputeBodyExtent(forms2, 2, capi.Vec2(0.0, 0.0))
    assert e.minExtent == 0.0 and e.maxExtent == pytest.approx(1.0)
    # no shapes
    e = lib.s2ComputeBodyExtent(forms, 0, capi.Vec2(0.0, 0.0))
    assert e.minExtent == 100000.0 and e.maxExtent == 0.0


def test_reference_tunnels_on_projectiles(reference):
    sc = scenes.projectiles(reference, "TGS_Soft")
    lanes = sc.piles["lanes"]
    ever = np.zeros(len(lanes), dtype=bool)
    for _ in range(30):
        sc.step(1.0 / 60.0, 4, 2, True)
        ever |= scenes.projectiles_behind(reference, sc)
    meant = np.array([lane["passes"] for lane in lanes])
    assert ever[~meant].sum() >= 1  # projectiles that should have hit a wall end behind it
    sc.destroy()
