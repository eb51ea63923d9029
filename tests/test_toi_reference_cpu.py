"""CPU: the time of impact (s2TimeOfImpact, csrc/shared/s2_toi.h, the source the device's continuous pass compiles) and the
shape extents (s2ComputeShapeExtent) against a float64 restatement of what they mean, sharing no code with that header
or the GJK.

The reference (`pose64`, `sep64`, `min_sep64`, below) poses a sweep in float64 (centre linear, rotation by normalised
lerp), measures the exact distance of two convex cores (a separating-axis test for overlap, else the least vertex-edge
distance both ways) minus both radii, and bounds the least separation over an interval by Lipschitz subdivision: between
two samples the separation falls at most at `|dcB - dcA| + wA RA + wB RB`, with `w` the exact float64 maximum of the
lerp's angular speed on that interval. Its results are certified to 1e-5 m, except where the angular speed is unbounded
(a rotation of a float32 half turn, `phi` = pi): there the subdivision runs out of its 2^16 samples and only the samples
are checked (`min_sep64` returns certified = False).

The contract checked (DESIGN.md §3.11, target = s2_linearSlop, tol = target / 4, eps = 2e-5 + 8 ulp32 of the largest
coordinate, the float32 round-off of the inputs and the GJK):
  HIT         sep64(fraction) in [target - tol - eps, target + tol + eps], and the target was never passed before it;
  SEPARATED   fraction == maxFraction, and the separation never fell below target - tol - eps;
  OVERLAPPED  sep64(0) < target + tol + eps;
  FAILED      only for a rotation of at least FAILED_MIN_RATE of angular bound, and the fraction is still safe.
A case whose eps exceeds the tolerance (coordinates near 1e4 m) is held only to "the separation never goes below -eps".
"""
import ctypes as C
import math

import numpy as np
import pytest

from solver2d_b200 import capi, device

TARGET = 0.005      # s2_linearSlop (S2C_TOI_TARGET)
TOL = 0.25 * TARGET  # S2C_TOI_TOLERANCE
RES = 1e-5          # what min_sep64's certified bound may lie below the true minimum
MAX_SAMPLES = 1 << 16
# FAILED (50 iterations without reaching the target or the end) is the answer only of sweeps whose angular bound
# 2 tan(|phi| / 2) is large, so that the advancement crawls. Measured over the seeded families below (x86-64 host build):
# where the round-off is below the tolerance, every FAILED case has a bound of at least 6.02 (phi = 2.5, a 16 m lever
# arm), 28.2 (phi = 3.0) or more; none with |phi| <= pi / 2 (bound 2) fails. At 1e4 m from the origin, where the float32
# round-off of the distance is as large as the tolerance, a sweep with a bound of 0.51 (phi = 0.5) also failed; there
# FAILED is allowed at any rate (its fraction must still be safe).
FAILED_MIN_RATE = 5.0
PHIS = [0.0, 1e-6, 0.5, math.pi / 2, 2.5, 3.0, math.pi - 1e-3, math.pi]


@pytest.fixture(scope="module")
def lib():
    return capi.Solver2D(device.LIB_PATH)


# ---------------------------------------------------------------------------------------------------------------------
# the float64 reference
# ---------------------------------------------------------------------------------------------------------------------

class Shape64:
    """A convex shape in its body frame: 1 (circle), 2 (capsule, segment) or 3-8 (polygon) core vertices and a radius,
    held as the float32 values the library sees, widened exactly to float64."""

    def __init__(self, verts, radius):
        self.v = np.asarray(np.asarray(verts, dtype=np.float32), dtype=np.float64).reshape(-1, 2)
        self.r = float(np.float32(radius))

    def proxy(self, lib):
        pts = (capi.Vec2 * len(self.v))(*[capi.Vec2(float(x), float(y)) for x, y in self.v])
        return lib.s2MakeProxy(pts, len(self.v), self.r)


class Sweep64:
    """A sweep's float32 fields (as in the library's s2Sweep), widened to float64."""

    def __init__(self, lc, c1, c2, q1, q2):
        f = lambda a: np.asarray(np.asarray(a, dtype=np.float32), dtype=np.float64)
        self.lc, self.c1, self.c2, self.q1, self.q2 = f(lc), f(c1), f(c2), f(q1), f(q2)  # q as (s, c)

    def capi(self):
        v = lambda a: capi.Vec2(float(a[0]), float(a[1]))
        return capi.Sweep(v(self.lc), v(self.c1), v(self.c2), capi.Rot(float(self.q1[0]), float(self.q1[1])),
                          capi.Rot(float(self.q2[0]), float(self.q2[1])))

    def reach(self, shape):
        """largest distance of a core vertex from the centre of mass"""
        return float(np.max(np.hypot(*(shape.v - self.lc).T)))

    def max_rate(self, a, b):
        """Exact float64 maximum of |dtheta/dt| of the normalised lerp over [a, b] (arrays): |cross(q1, q2)| / min |m|^2,
        m(t) = (1 - t) q1 + t q2, whose squared length is a quadratic in t."""
        q1, q2 = self.q1, self.q2
        aa, bb, cc = q1 @ q1, q1 @ q2, q2 @ q2
        cross = abs(q1[1] * q2[0] - q1[0] * q2[1])
        if cross == 0.0:
            return np.zeros_like(a)
        m2 = lambda t: aa * (1 - t) ** 2 + 2 * bb * t * (1 - t) + cc * t * t
        lo = np.minimum(m2(a), m2(b))
        k = aa - 2 * bb + cc
        if k > 0:
            ts = (aa - bb) / k
            inside = (a < ts) & (ts < b)
            lo = np.where(inside, np.minimum(lo, m2(ts)), lo)
        with np.errstate(divide="ignore"):
            return np.where(lo > 0, cross / np.maximum(lo, 1e-300), np.inf)


def pose64(sweep, t):
    """Centre (T, 2) and unit rotation (T, 2 as s, c) of a sweep at fractions t (T,): the centre linearly, the rotation by
    normalised lerp."""
    t = np.asarray(t, dtype=np.float64)[:, None]
    c = (1 - t) * sweep.c1 + t * sweep.c2
    m = (1 - t) * sweep.q1 + t * sweep.q2
    n = np.hypot(m[:, 0], m[:, 1])[:, None]
    return c, m / np.where(n > 0, n, 1.0)


def _world(shape, sweep, t):
    c, q = pose64(sweep, t)
    r = shape.v - sweep.lc  # (n, 2) about the centre of mass
    s, co = q[:, 0:1], q[:, 1:2]
    return np.stack([c[:, 0:1] + co * r[:, 0] - s * r[:, 1], c[:, 1:2] + s * r[:, 0] + co * r[:, 1]], axis=-1)  # (T, n, 2)


def _edges(P):
    n = P.shape[1]
    if n == 1:
        return P, P
    if n == 2:
        return P[:, :1], P[:, 1:]
    return P, np.roll(P, -1, axis=1)


def _point_edge(X, E0, E1):
    """distances (T, nX, nE) from points X to the edges E0 -> E1"""
    d = X[:, :, None, :] - E0[:, None, :, :]
    e = (E1 - E0)[:, None, :, :]
    ee = np.sum(e * e, axis=-1)
    s = np.clip(np.sum(d * e, axis=-1) / np.where(ee > 0, ee, 1.0), 0.0, 1.0)
    w = d - s[..., None] * e
    return np.hypot(w[..., 0], w[..., 1])


def _axes(P):
    """separating-axis candidates of a core: the edge normals of a polygon, the normal and the direction of a segment"""
    n = P.shape[1]
    if n == 1:
        return np.zeros((P.shape[0], 0, 2))
    E0, E1 = _edges(P)
    e = E1 - E0
    normals = np.stack([e[..., 1], -e[..., 0]], axis=-1)
    return np.concatenate([normals, e], axis=1) if n == 2 else normals


def core_distance64(PA, PB):
    """Exact distance of the convex hulls of PA (T, nA, 2) and PB (T, nB, 2): 0 where no axis separates them, else the
    least vertex-edge distance in both directions."""
    axes = np.concatenate([_axes(PA), _axes(PB)], axis=1)
    if axes.shape[1]:
        pa = np.einsum("tkd,tnd->tkn", axes, PA)
        pb = np.einsum("tkd,tnd->tkn", axes, PB)
        apart = (pa.max(-1) < pb.min(-1)) | (pb.max(-1) < pa.min(-1))
        overlap = ~apart.any(axis=1)
    else:
        overlap = np.zeros(PA.shape[0], dtype=bool)
    d = np.minimum(_point_edge(PA, *_edges(PB)).min(axis=(1, 2)), _point_edge(PB, *_edges(PA)).min(axis=(1, 2)))
    return np.where(overlap, 0.0, d)


def sep64(A, sweepA, B, sweepB, t):
    """Separation (core distance minus both radii) of two swept shapes at the fractions t."""
    t = np.atleast_1d(np.asarray(t, dtype=np.float64))
    return core_distance64(_world(A, sweepA, t), _world(B, sweepB, t)) - A.r - B.r


def min_sep64(A, sweepA, B, sweepB, t0, t1, floor=np.nan):
    """(bound, certified): a lower bound on the least separation over [t0, t1], within RES of it (or proven >= floor).
    Intervals are split eightfold until the Lipschitz bound of each, (f(a) + f(b) - rate (b - a)) / 2, is within RES of
    the least sample or above the floor. Past MAX_SAMPLES (an unbounded angular speed) only the samples are checked and
    certified is False."""
    dcA, dcB = sweepA.c2 - sweepA.c1, sweepB.c2 - sweepB.c1
    lin = float(np.hypot(*(dcB - dcA)))
    RA, RB = sweepA.reach(A), sweepB.reach(B)
    ts = np.linspace(t0, t1, 257) if t1 > t0 else np.array([t0])
    f = sep64(A, sweepA, B, sweepB, ts)
    best = float(f.min())
    if t1 <= t0:
        return best, True
    a, b, fa, fb = ts[:-1], ts[1:], f[:-1], f[1:]
    bound, used = np.inf, len(ts)
    while len(a):
        rate = lin + sweepA.max_rate(a, b) * RA + sweepB.max_rate(a, b) * RB
        with np.errstate(invalid="ignore"):
            lb = np.where(np.isfinite(rate), 0.5 * (fa + fb - rate * (b - a)), -np.inf)
        done = (lb >= best - RES) | (lb >= floor)  # (never by the floor when none is given: nan compares false)
        if done.any():
            bound = min(bound, float(lb[done].min()))
        a, b, fa, fb = a[~done], b[~done], fa[~done], fb[~done]
        if len(a) == 0:
            break
        if used + 7 * len(a) > MAX_SAMPLES or np.any(b - a < 1e-15):
            return min(bound, best), False
        k = np.arange(1, 8) / 8.0
        mid = a[:, None] + (b - a)[:, None] * k[None, :]
        fm = sep64(A, sweepA, B, sweepB, mid.ravel()).reshape(mid.shape)
        used += mid.size
        best = min(best, float(fm.min()))
        pts = np.concatenate([a[:, None], mid, b[:, None]], axis=1)
        fp = np.concatenate([fa[:, None], fm, fb[:, None]], axis=1)
        a, b = pts[:, :-1].ravel(), pts[:, 1:].ravel()
        fa, fb = fp[:, :-1].ravel(), fp[:, 1:].ravel()
    return min(bound, best), True


def eps_of(A, sweepA, B, sweepB):
    """float32 round-off of a case: 2e-5 + 8 ulp32 of the largest coordinate the sweep reaches"""
    big = 0.0
    for S, sw in ((A, sweepA), (B, sweepB)):
        for t in (0.0, 1.0):
            big = max(big, float(np.abs(_world(S, sw, [t])).max()))
        big = max(big, float(np.abs(sw.c1).max()), float(np.abs(sw.c2).max()))
    return 2e-5 + 8 * float(np.spacing(np.float32(big)))


def angular_bound64(sweep):
    """2 tan(|phi| / 2), phi the angle from q1 to q2 (the float64 value of the bound s2_toi.h uses)"""
    phi = math.atan2(sweep.q1[1] * sweep.q2[0] - sweep.q1[0] * sweep.q2[1], sweep.q1 @ sweep.q2)
    return math.inf if abs(phi) >= math.pi else 2.0 * math.tan(0.5 * abs(phi))


# ---------------------------------------------------------------------------------------------------------------------
# the contract
# ---------------------------------------------------------------------------------------------------------------------

def toi(lib, A, sweepA, B, sweepB, max_fraction=1.0):
    inp = capi.TOIInput(A.proxy(lib), B.proxy(lib), sweepA.capi(), sweepB.capi(), max_fraction)
    return lib.s2TimeOfImpact(C.byref(inp))


def check_contract(lib, A, sweepA, B, sweepB, max_fraction=1.0, what=""):
    """Runs the time of impact and asserts the contract against the float64 reference; returns (state, certified)."""
    out = toi(lib, A, sweepA, B, sweepB, max_fraction)
    mf = float(np.float32(max_fraction))
    eps = eps_of(A, sweepA, B, sweepB)
    strong = eps <= TOL
    lo = TARGET - TOL - eps if strong else -eps
    msg = f"{what} state={out.state} fraction={out.fraction!r} iterations={out.iterations} eps={eps:.2e}"
    assert out.state in (capi.TOI_HIT, capi.TOI_SEPARATED, capi.TOI_OVERLAPPED, capi.TOI_FAILED), msg
    assert 0.0 <= out.fraction <= mf, msg
    certified = True
    if out.state == capi.TOI_OVERLAPPED:
        assert out.fraction == 0.0, msg
        s0 = float(sep64(A, sweepA, B, sweepB, 0.0)[0])
        assert s0 < TARGET + TOL + eps, (msg, s0)
        return out.state, certified
    if out.state == capi.TOI_SEPARATED:
        assert out.fraction == mf, msg
        end = mf
    else:
        end = out.fraction
        if out.state == capi.TOI_FAILED and strong:
            rate = max(angular_bound64(sweepA), angular_bound64(sweepB))
            assert rate >= FAILED_MIN_RATE, (msg, rate)
        s = float(sep64(A, sweepA, B, sweepB, out.fraction)[0])
        assert s >= lo, (msg, s)
        if out.state == capi.TOI_HIT and strong:
            assert s <= TARGET + TOL + eps, (msg, s)
    closest, certified = min_sep64(A, sweepA, B, sweepB, 0.0, end, floor=lo)
    assert closest >= lo, (msg, closest, certified)
    return out.state, certified


# ---------------------------------------------------------------------------------------------------------------------
# the reference checks itself
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("phi", [1e-6, 0.5, math.pi / 2, 2.5, 3.0, math.pi - 1e-3, -2.5, -(math.pi - 1e-3)])
def test_lerp_angular_speed_peaks_at_2_tan_half_phi(phi):
    """The densely sampled float64 angle of the normalised lerp turns fastest at mid-sweep, at 2 tan(|phi| / 2), which
    the time of impact's rotation bound and min_sep64's Lipschitz rate both rest on; at the ends it turns at sin(phi)."""
    a0 = 0.3
    q1, q2 = np.array([math.sin(a0), math.cos(a0)]), np.array([math.sin(a0 + phi), math.cos(a0 + phi)])
    t = np.concatenate([np.linspace(0.0, 1.0, 1 << 16), 0.5 + np.linspace(-1e-3, 1e-3, 4097)])
    bound = 2.0 * math.tan(0.5 * abs(phi))
    h = 1e-4 / max(1.0, bound)  # well inside the width of the mid-sweep peak, (1 + cos phi)^(1/2) / 4

    def m(t):
        return (1 - t)[:, None] * q1 + t[:, None] * q2

    # the angle turned from t - h to t + h, as the angle between the two lerps (no branch cut, no cancellation)
    a, b = m(t - h), m(t + h)
    rate = np.arctan2(a[:, 1] * b[:, 0] - a[:, 0] * b[:, 1], np.sum(a * b, axis=1)) / (2 * h)
    assert np.abs(rate).max() == pytest.approx(bound, rel=1e-5)
    assert np.abs(rate).max() <= bound * (1 + 1e-5)
    sw = Sweep64((0, 0), (0, 0), (0, 0), q1, q2)
    sw.q1, sw.q2 = q1, q2  # (unrounded)
    assert float(sw.max_rate(np.array([0.0]), np.array([1.0]))[0]) == pytest.approx(bound, rel=1e-6)
    assert abs(rate[0]) == pytest.approx(abs(math.sin(phi)), rel=1e-4, abs=1e-9)


def test_reference_distance_against_hand_values():
    box = Shape64([(-1, -1), (1, -1), (1, 1), (-1, 1)], 0.0)
    ball = Shape64([(0, 0)], 0.25)
    seg = Shape64([(-1, 0), (1, 0)], 0.0)
    still = lambda x, y, a=0.0: Sweep64((0, 0), (x, y), (x, y), (math.sin(a), math.cos(a)), (math.sin(a), math.cos(a)))
    assert sep64(box, still(0, 0), ball, still(3, 0), 0.0)[0] == pytest.approx(1.75)
    assert sep64(box, still(0, 0), ball, still(3, 3), 0.0)[0] == pytest.approx(2 * math.sqrt(2) - 0.25)
    assert sep64(box, still(0, 0), ball, still(0.5, 0), 0.0)[0] == -0.25  # overlapping cores: distance 0
    assert sep64(seg, still(0, 0), seg, still(0, 0, math.pi / 2), 0.0)[0] == 0.0  # crossing segments
    assert sep64(seg, still(0, 0), seg, still(3, 0), 0.0)[0] == pytest.approx(1.0)  # collinear, apart
    assert sep64(box, still(0, 0), box, still(1 + math.sqrt(2) + 0.5, 0, math.pi / 4), 0.0)[0] == pytest.approx(0.5)
    # a ball passing over the box at height 1.5: least separation 0.25, at mid-sweep
    over = Sweep64((0, 0), (-5, 1.5), (5, 1.5), (0, 1), (0, 1))
    closest, certified = min_sep64(box, still(0, 0), ball, over, 0, 1, floor=0.25 - 10 * RES)
    assert certified and 0.25 - 10 * RES <= closest <= 0.25
    closest, certified = min_sep64(box, still(0, 0), ball, over, 0, 1, floor=0.25 + RES)
    assert closest < 0.25 + RES
    # a ball passing a box's corner: a single closest point, found to RES without a floor
    corner = Sweep64((0, 0), (-5, -2), (5, 8), (0, 1), (0, 1))  # along y = x + 3, 1 / sqrt(2) from the corner (-1, 1)
    closest, certified = min_sep64(box, still(0, 0), ball, corner, 0, 1)
    assert certified and math.sqrt(0.5) - 0.25 - RES <= closest <= math.sqrt(0.5) - 0.25


# ---------------------------------------------------------------------------------------------------------------------
# shapes and sweeps
# ---------------------------------------------------------------------------------------------------------------------

KINDS = ["circle", "capsule", "segment", "box", "rounded_box", "hull", "rounded_hull"]


def make_shape(lib, kind, size, centre, rng):
    """A shape of the given kind and size (0.01 - 50 m) centred at `centre` of its body frame."""
    g = np.asarray(centre, dtype=np.float64)
    ang = rng.uniform(-math.pi, math.pi)
    u = np.array([math.cos(ang), math.sin(ang)])
    w = np.array([-u[1], u[0]])
    if kind == "circle":
        return Shape64([g], size)
    if kind in ("capsule", "segment"):
        r = rng.uniform(0.1, 0.5) * size if kind == "capsule" else 0.0
        return Shape64([g - size * u, g + size * w * rng.uniform(-0.2, 0.2) + size * u], r)
    if kind in ("box", "rounded_box"):
        hx, hy = size, size * rng.uniform(0.1, 1.0)
        r = rng.uniform(0.05, 0.3) * size if kind == "rounded_box" else 0.0
        return Shape64([g + sx * hx * u + sy * hy * w for sx, sy in ((-1, -1), (1, -1), (1, 1), (-1, 1))], r)
    n = int(rng.integers(3, 9))
    size = max(size, 0.05)  # (the hull welds points closer than s2_linearSlop)
    for _ in range(20):
        ang0 = np.sort(rng.uniform(0, 2 * math.pi, n))
        pts = np.stack([np.cos(ang0), np.sin(ang0)], axis=1) * size * np.array([1.0, rng.uniform(0.3, 1.0)]) + g
        hull = lib.s2ComputeHull((capi.Vec2 * n)(*[capi.Vec2(float(x), float(y)) for x, y in pts]), n)
        if hull.count >= 3:
            break
    else:
        raise AssertionError("no hull")
    verts = [(hull.points[i].x, hull.points[i].y) for i in range(hull.count)]
    r = rng.uniform(0.05, 0.3) * size if kind == "rounded_hull" else 0.0
    return Shape64(verts, r)


def _rot(a):
    return np.array([math.sin(a), math.cos(a)])


def _off_unit(q, rng):
    """a rotation a few ulp off unit length, as s2IntegrateRot leaves them"""
    return np.asarray(np.float32(q) * np.float32(1.0 + int(rng.integers(-4, 5)) * 2.0 ** -23), dtype=np.float64)


def _R(q):
    s, c = q
    return np.array([[c, -s], [s, c]])


def _shape_centre(shape):
    return shape.v.mean(axis=0)


def make_case(lib, kinds, rng):
    """One seeded case: A near `origin`, B swept through its neighbourhood, both with a centre of mass 0.5 - 2 m off the
    shape (B's shape often at its body origin, so that a reach measured from the origin comes out too small)."""
    origin = rng.choice([0.0, 1e2, 1e3, 1e4]) * _rot(rng.uniform(-math.pi, math.pi))
    sizes = np.exp(rng.uniform(math.log(0.01), math.log(50.0), 2))
    shapes, lcs = [], []
    for kind, size in zip(kinds, sizes):
        g = np.zeros(2) if rng.random() < 0.5 else rng.uniform(-3, 3, 2)
        shape = make_shape(lib, kind, size, g, rng)
        lc = _shape_centre(shape) + rng.uniform(0.5, 2.0) * _rot(rng.uniform(-math.pi, math.pi))
        shapes.append(shape)
        lcs.append(lc)
    A, B = shapes
    ext = sizes[0] + sizes[1] + A.r + B.r
    phi = rng.choice(PHIS) * rng.choice([-1.0, 1.0])
    qB1 = _rot(rng.uniform(-math.pi, math.pi))
    qB2 = _rot(math.atan2(qB1[0], qB1[1]) + phi)
    # A: still (as the device pass has it) or moving and rotating as well
    qA1 = _rot(rng.uniform(-math.pi, math.pi))
    if rng.random() < 0.3:
        qA2 = _rot(math.atan2(qA1[0], qA1[1]) + rng.choice(PHIS[:6]) * rng.choice([-1.0, 1.0]))
        dA = rng.uniform(-1, 1, 2) * ext
    else:
        qA2, dA = qA1, np.zeros(2)
    gA, gB = _shape_centre(A) - lcs[0], _shape_centre(B) - lcs[1]
    cA1 = origin - _R(qA1) @ gA
    cA2 = cA1 + dA
    u = _rot(rng.uniform(-math.pi, math.pi))
    w = np.array([-u[1], u[0]])
    if rng.random() < 0.75:
        # B's shape flies from one side of A to the other, passing it at a random miss distance
        start = origin + u * ext * rng.uniform(1.0, 3.0) + w * rng.uniform(-1.0, 1.0) * ext
        end = origin - u * ext * rng.uniform(0.0, 3.0) + w * rng.uniform(-1.0, 1.0) * ext
        cB1, cB2 = start - _R(qB1) @ gB, end - _R(qB2) @ gB
    else:
        # B only turns: A sits near the circle its shape travels on about the centre of mass
        cB1 = origin - _rot(rng.uniform(-math.pi, math.pi)) * (np.hypot(*gB) + rng.uniform(-0.8, 0.8) * ext)
        cB2 = cB1
    sA = Sweep64(lcs[0], cA1, cA2, _off_unit(qA1, rng), _off_unit(qA2, rng))
    sB = Sweep64(lcs[1], cB1, cB2, _off_unit(qB1, rng), _off_unit(qB2, rng))
    max_fraction = float(rng.choice([1.0, 1.0, 0.5, 1e-3]))
    return A, sA, B, sB, max_fraction


PAIRS = [(a, b) for a in KINDS for b in KINDS]


@pytest.mark.parametrize("kinds", PAIRS, ids=[f"{a}-{b}" for a, b in PAIRS])
def test_seeded_families_against_float64(lib, kinds):
    """Every pair of shape kinds: lever arms of 0.5 - 2 m, rotations up to a half turn both ways, both bodies moving,
    maxFraction 1, 0.5 and 1e-3, offsets of 0 - 1e4 m from the origin, sizes of 0.01 - 50 m, rotations a few ulp off
    unit length."""
    rng = np.random.default_rng(1000 + KINDS.index(kinds[0]) * len(KINDS) + KINDS.index(kinds[1]))
    states = []
    for trial in range(24):
        A, sA, B, sB, mf = make_case(lib, kinds, rng)
        state, _ = check_contract(lib, A, sA, B, sB, mf, what=f"trial {trial}")
        states.append(state)
    assert states.count(capi.TOI_HIT) >= 1, states


@pytest.mark.parametrize("phi", [2.5, 3.0, -3.0, math.pi - 1e-3])
@pytest.mark.parametrize("lever", [0.5, 2.0])
@pytest.mark.parametrize("translate", [False, True], ids=["turning", "turning+moving"])
def test_large_rotation_with_a_lever_arm(lib, phi, lever, translate):
    """A box at its body origin, its centre of mass `lever` metres away, turns by `phi` (with or without translation)
    past a wall its shape's arc crosses at mid-sweep. A rotation bound taken at the ends of the sweep (|sin phi|) or a
    reach taken from the body origin lets it through."""
    box = Shape64([(-0.2, -0.1), (0.2, -0.1), (0.2, 0.1), (-0.2, 0.1)], 0.0)
    lc = np.array([lever, 0.0])
    a1 = -0.5 * phi
    q1, q2 = _rot(a1), _rot(a1 + phi)
    # the shape sits on a circle of radius `lever` about the centre; at mid-sweep it points along -x
    # the centre of mass moves from c1 to c2 (or stays at the origin); the shape is at c - R(q) lc, at (-lever, 0) at
    # mid-sweep, 0.2 m into the wall
    c1, c2 = (np.array([0.0, 1.0]), np.array([0.0, -1.0])) if translate else (np.zeros(2), np.zeros(2))
    wall = Shape64([(-lever - 0.15, -3.0), (-lever - 0.1, -3.0), (-lever - 0.1, 3.0), (-lever - 0.15, 3.0)], 0.0)
    still = Sweep64((0, 0), (0, 0), (0, 0), (0, 1), (0, 1))
    sweep = Sweep64(lc, c1, c2, q1, q2)
    # float64: the shape reaches past the wall's face at mid-sweep, and starts clear of it
    assert float(sep64(wall, still, box, sweep, 0.5)[0]) <= 0.0  # (cores overlapping)
    assert float(sep64(wall, still, box, sweep, 0.0)[0]) > TARGET + TOL
    state, _ = check_contract(lib, wall, still, box, sweep)
    assert state in (capi.TOI_HIT, capi.TOI_FAILED)


@pytest.mark.parametrize("k", [-0.5, 0.0, 0.5, 1.0, 2.0])
@pytest.mark.parametrize("kind", ["circle", "box", "rounded_hull"])
@pytest.mark.parametrize("lever", [0.0, 1.5])
def test_grazing_sweeps(lib, k, kind, lever):
    """B passes over a static box at closest approach target + k tol (translation only, so the closest approach is exact
    in float64). Below the target it must stop before the target; two tolerances clear it must be separated."""
    rng = np.random.default_rng(7)
    top = Shape64([(-1, -0.5), (1, -0.5), (1, 0.5), (-1, 0.5)], 0.0)
    B = make_shape(lib, kind, 0.2, (0.0, 0.0), rng)
    low = float(B.v[:, 1].min()) - B.r  # B's lowest point: on a flat path, the closest approach to the top face
    h = 0.5 + TARGET + k * TOL - low
    lc = np.array([0.0, lever])
    still = Sweep64((0, 0), (0, 0), (0, 0), (0, 1), (0, 1))
    sweep = Sweep64(lc, (-3.0, h + lever), (3.0, h + lever), (0, 1), (0, 1))
    want = TARGET + k * TOL
    closest, certified = min_sep64(top, still, B, sweep, 0.0, 1.0, floor=want - 5 * RES)
    assert certified and closest >= want - 5 * RES
    assert abs(float(sep64(top, still, B, sweep, 0.5)[0]) - want) <= 2e-6
    state, _ = check_contract(lib, top, still, B, sweep)
    if k <= -0.5:
        assert state == capi.TOI_HIT
    if k >= 2.0:
        assert state == capi.TOI_SEPARATED


@pytest.mark.parametrize("k", [-1.0, 1.0])
@pytest.mark.parametrize("direction", [1.0, -1.0], ids=["approaching", "leaving"])
def test_start_at_target_plus_minus_tolerance(lib, k, direction):
    top = Shape64([(-1, -0.5), (1, -0.5), (1, 0.5), (-1, 0.5)], 0.0)
    ball = Shape64([(0.0, 0.0)], 0.1)
    h = 0.5 + 0.1 + TARGET + k * TOL
    still = Sweep64((0, 0), (0, 0), (0, 0), (0, 1), (0, 1))
    sweep = Sweep64((0, 0), (0.0, h), (0.3, h - direction * 1.0), (0, 1), (0, 1))
    assert abs(float(sep64(top, still, ball, sweep, 0.0)[0]) - (TARGET + k * TOL)) < 1e-7
    state, _ = check_contract(lib, top, still, ball, sweep)
    if k < 0:
        assert state == capi.TOI_OVERLAPPED


@pytest.mark.parametrize("offset", [1e2, 1e3, 1e4])
@pytest.mark.parametrize("kind", ["circle", "box", "hull"])
def test_far_from_the_origin(lib, offset, kind):
    """A head-on hit and a graze 1e2 - 1e4 m from the origin. Up to 1e3 m the float32 round-off stays below the
    tolerance and the full contract holds; at 1e4 m (ulp 1 mm) only 'never through' does."""
    rng = np.random.default_rng(int(offset) + len(kind))
    o = np.array([offset, -0.7 * offset])
    wall = Shape64([(-0.05, -2), (0.05, -2), (0.05, 2), (-0.05, 2)], 0.0)
    still = Sweep64((0, 0), o, o, (0, 1), (0, 1))
    B = make_shape(lib, kind, 0.2, (0.0, 0.0), rng)
    for y in (0.0, 2.2 + 0.2 + TARGET):
        sweep = Sweep64((0.7, 0.0), o + (-3.0, y), o + (3.0, y), _rot(0.2), _rot(0.9))
        check_contract(lib, wall, still, B, sweep, what=f"y={y}")
    head_on = Sweep64((0.0, 0.0), o + (-3.0, 0.0), o + (3.0, 0.0), (0, 1), (0, 1))
    assert toi(lib, wall, still, B, head_on).state == capi.TOI_HIT


def test_half_turn_sweep_is_held_at_its_start(lib):
    """Within about 5e-4 rad of a half turn the angular bound is at least 8e3 (FLT_MAX at a half turn): the steps are
    too small to get anywhere in 50 iterations, and the sweep fails near fraction 0 against any shape that is not
    touching, even one the shape never comes near (DESIGN.md §3.11, Limits). Pinned: the fraction is safe, and below
    0.05."""
    box = Shape64([(-0.5, -0.1), (0.5, -0.1), (0.5, 0.1), (-0.5, 0.1)], 0.0)
    far = Shape64([(-0.1, -0.1), (0.1, -0.1), (0.1, 0.1), (-0.1, 0.1)], 0.0)
    still = Sweep64((0, 0), (3.0, 3.0), (3.0, 3.0), (0, 1), (0, 1))
    for phi in (math.pi - 2e-4, math.pi, -math.pi + 1e-4):
        sweep = Sweep64((0, 0), (0, 0), (0.5, 0), _rot(0.1), _rot(0.1 + phi))
        closest, _ = min_sep64(far, still, box, sweep, 0.0, 1.0, floor=2.0)
        assert closest >= 2.0  # the box never comes within 2 m of the far shape
        out = toi(lib, far, still, box, sweep)
        assert out.state == capi.TOI_FAILED and out.fraction < 0.05, (phi, out.state, out.fraction)
        check_contract(lib, far, still, box, sweep)
    # a quarter turn (bound 2): the same sweep gets through
    sweep = Sweep64((0, 0), (0, 0), (0.5, 0), _rot(0.1), _rot(0.1 + math.pi / 2))
    assert toi(lib, far, still, box, sweep).state == capi.TOI_SEPARATED


# ---------------------------------------------------------------------------------------------------------------------
# shape extents
# ---------------------------------------------------------------------------------------------------------------------

def _polygon(lib, shape):
    """the library's polygon form of a Shape64 (vertices, normals, radius, count)"""
    p = capi.Polygon()
    n = len(shape.v)
    for i, (x, y) in enumerate(shape.v):
        p.vertices[i] = capi.Vec2(float(x), float(y))
    if n >= 3:
        for i in range(n):
            e = shape.v[(i + 1) % n] - shape.v[i]
            nn = np.array([e[1], -e[0]]) / np.hypot(*e)
            p.normals[i] = capi.Vec2(float(nn[0]), float(nn[1]))
    p.count = n
    p.radius = shape.r
    return p


def _centroid64(v):
    x, y = v[:, 0], v[:, 1]
    x1, y1 = np.roll(x, -1), np.roll(y, -1)
    cr = x * y1 - x1 * y
    area = 0.5 * cr.sum()
    return np.array([((x + x1) * cr).sum(), ((y + y1) * cr).sum()]) / (6.0 * area)


def _edge_distances64(v, p):
    """signed distances (inward positive) of p from the edge lines of the counter-clockwise polygon v"""
    e = np.roll(v, -1, axis=0) - v
    n = np.stack([e[:, 1], -e[:, 0]], axis=1) / np.hypot(e[:, 0], e[:, 1])[:, None]
    return np.sum(n * (v - p), axis=1)


@pytest.mark.parametrize("family", ["hull", "rounded_hull", "thin_hull", "box", "rounded_box", "capsule", "circle",
                                    "segment"])
def test_shape_extent_against_float64(lib, family):
    """outer >= the true largest distance from the centre of mass; inner <= the true distance from the float64 centroid
    to the boundary; and the core circle of radius inner / 4 lies inside the shape (the core rule is sound only so).
    Shapes 0.01 - 50 m, up to 1e3 m from their body's origin, thin hulls 40 - 400 times longer than wide."""
    rng = np.random.default_rng(len(family) * 31)
    for trial in range(60):
        size = float(np.exp(rng.uniform(math.log(0.01), math.log(50.0))))
        g = rng.choice([0.0, 1.0, 1e2, 1e3]) * _rot(rng.uniform(-math.pi, math.pi))
        if family == "thin_hull":
            n = int(rng.integers(3, 9))
            length, width = max(size, 0.5), max(size, 0.5) / rng.uniform(40, 400)
            ang = rng.uniform(-math.pi, math.pi)
            u = np.array([math.cos(ang), math.sin(ang)])
            w = np.array([-u[1], u[0]])
            xs = np.sort(rng.uniform(-1, 1, n)) * length
            xs[0], xs[-1] = -length, length
            side = np.where(np.arange(n) % 2 == 0, 1.0, -1.0) * width
            pts = g + xs[:, None] * u + side[:, None] * w
            hull = lib.s2ComputeHull((capi.Vec2 * n)(*[capi.Vec2(float(x), float(y)) for x, y in pts]), n)
            if hull.count < 3:
                continue
            shape = Shape64([(hull.points[i].x, hull.points[i].y) for i in range(hull.count)], 0.0)
        else:
            shape = make_shape(lib, family, size, g, rng)
        lc = np.asarray(np.float32(_shape_centre(shape) + rng.uniform(0.0, 2.0) * _rot(rng.uniform(-math.pi, math.pi))),
                        dtype=np.float64)
        e = lib.s2ComputeShapeExtent(C.byref(_polygon(lib, shape)), capi.Vec2(float(lc[0]), float(lc[1])))
        inner, outer = float(e.minExtent), float(e.maxExtent)
        core = np.array([e.center.x, e.center.y])
        far = float(np.max(np.hypot(*(shape.v - lc).T))) + shape.r
        # outer: float32 sqrt of a float32 sum, correct to a couple of ulp of itself
        assert outer >= far * (1 - 4 * 2.0 ** -24), (trial, outer, far)
        ulp = float(np.spacing(np.float32(np.abs(shape.v).max())))
        n = len(shape.v)
        if n == 1:
            assert inner == shape.r and np.array_equal(core, shape.v[0])
            continue
        if n == 2:
            assert inner == shape.r
            assert np.abs(core - shape.v.mean(axis=0)).max() <= ulp
            continue
        d_true = _edge_distances64(shape.v, _centroid64(shape.v))
        assert d_true.min() > 0
        assert inner <= d_true.min() + shape.r + 4 * ulp, (trial, inner, d_true.min() + shape.r)
        d_core = _edge_distances64(shape.v, core)
        # the core circle (radius inner / 4) is inside the rounded polygon: the core is inside the core polygon and at
        # least inner / 4 - radius from each edge line
        assert d_core.min() >= 0.0, (trial, d_core.min())
        assert d_core.min() + shape.r >= 0.25 * inner, (trial, d_core.min(), inner)
