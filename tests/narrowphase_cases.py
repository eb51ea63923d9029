"""Seeded narrow-phase cases as plain data, shared by the host sweep `edge_manifold` (test_host_cpu.py) and the per-pair
device test (test_narrowphase_gpu.py).

A case is one shape pair of one of the nine manifold kinds of reference src/contact.c:139-154, in primary (A, B) order:
the shapes, the pose of A, two poses of B (pose 2 is pose 1 moved slightly, as a persistent contact moves between two
steps), an old-state rule for the pose-2 evaluation and seeded warm-start values. Placements are solved in float64 on the
shapes' cores so that the separation lands in the wanted regime; no solver library is consulted while cases are made, so
the cases do not change when the code under test does.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

from solver2d_b200 import capi

LINEAR_SLOP = 0.005
SPECULATIVE = 4.0 * LINEAR_SLOP  # s2_speculativeDistance

# kind -> (shape type of A, shape type of B), primary order of the reference's registry
KINDS = {
    "circles": ("circle", "circle"),
    "capsule_circle": ("capsule", "circle"),
    "capsules": ("capsule", "capsule"),
    "polygon_circle": ("polygon", "circle"),
    "polygon_capsule": ("polygon", "capsule"),
    "polygons": ("polygon", "polygon"),
    "segment_circle": ("segment", "circle"),
    "segment_capsule": ("segment", "capsule"),
    "segment_polygon": ("segment", "polygon"),
}

# separation targets (m); "deep" and "centroid_inside" are scaled by the smaller shape
DISTANCE_REGIMES = ("beyond", "inside", "touching", "shallow", "deep", "coincident", "centroid_inside")
ORIENTATION_REGIMES = ("rel0", "rel0+", "rel90", "rel90+", "rel180", "rel180+", "vertex")
REGIMES = DISTANCE_REGIMES + ORIENTATION_REGIMES

# old manifold states at pose 2, built from the pose-1 result (see old_state)
RULES = ("real", "swap", "dup", "nomatch", "count0", "count1_junk", "count2")

JUNK_ID = 0xA5A0  # larger than any S2_MAKE_ID of two polygon indices (< 0x0808): never a real feature id


def _f32(x):
    return float(np.float32(x))


def _rot(a, v):
    c, s = math.cos(a), math.sin(a)
    return np.array([c * v[0] - s * v[1], s * v[0] + c * v[1]])


# -- shapes --------------------------------------------------------------------------------------------------------------
def _shape(rng, kind, size, k):
    """One shape spec: ("circle", cx, cy, r) | ("capsule", x1, y1, x2, y2, r) | ("segment", x1, y1, x2, y2) |
    ("box", hx, hy, cx, cy, angle, radius) | ("hull", ((x, y), ...), radius)."""
    if kind == "circle":
        off = rng.uniform(-0.5, 0.5, 2) * size if k % 2 else np.zeros(2)
        return ("circle", _f32(off[0]), _f32(off[1]), _f32(size))
    if kind in ("capsule", "segment"):
        a = rng.uniform(-math.pi, math.pi)
        if kind == "capsule" and k % 3 == 0:  # short: longer than s2_linearSlop (s2CreateCapsuleShape) by a little
            half = rng.uniform(0.005, 0.025)
        else:
            half = size * (rng.uniform(0.5, 1.5) if kind == "capsule" else rng.uniform(1.0, 3.0))
        c = rng.uniform(-0.2, 0.2, 2) * size
        p1, p2 = c - _rot(a, (half, 0.0)), c + _rot(a, (half, 0.0))
        if kind == "segment":
            return ("segment", _f32(p1[0]), _f32(p1[1]), _f32(p2[0]), _f32(p2[1]))
        r = size if half < 0.03 else size * rng.uniform(0.2, 0.8)
        return ("capsule", _f32(p1[0]), _f32(p1[1]), _f32(p2[0]), _f32(p2[1]), _f32(r))
    n = 3 + k % 6  # 3 .. 8 vertices
    radius = _f32(size * rng.uniform(0.05, 0.3)) if (k // 6) % 2 else 0.0
    if n == 4 and k % 12 < 6:
        hx, hy = size * rng.uniform(0.4, 1.0), size * rng.uniform(0.4, 1.0)
        off = rng.uniform(-0.3, 0.3, 2) * size if k % 4 else np.zeros(2)
        ang = rng.uniform(-1.0, 1.0) if k % 4 else 0.0
        return ("box", _f32(hx), _f32(hy), _f32(off[0]), _f32(off[1]), _f32(ang), radius)
    # jittered points on a circle: all on the hull, edges longer and corners sharper than the hull's welding and
    # collinearity tolerance (s2_linearSlop) down to the 0.1 m circle an 8-gon needs
    steps = np.sort(rng.uniform(-0.15, 0.15, n) + np.arange(n)) * (2.0 * math.pi / n) + rng.uniform(0, math.pi)
    rad = max(size, 0.1)
    pts = tuple((_f32(rad * math.cos(t)), _f32(rad * math.sin(t))) for t in steps)
    return ("hull", pts, radius)


def core(spec):
    """(vertices as float64 array, radius) of a shape spec: the convex core the manifold functions work on."""
    t = spec[0]
    if t == "circle":
        return np.array([[spec[1], spec[2]]]), spec[3]
    if t in ("capsule", "segment"):
        return np.array([[spec[1], spec[2]], [spec[3], spec[4]]]), (spec[5] if t == "capsule" else 0.0)
    if t == "box":
        hx, hy, cx, cy, a, r = spec[1:]
        v = [np.array([cx, cy]) + _rot(a, (sx * hx, sy * hy)) for sx, sy in ((-1, -1), (1, -1), (1, 1), (-1, 1))]
        return np.array(v), r
    return np.array(spec[1], dtype=np.float64), spec[2]


def _hull(p):
    p = sorted(set(map(tuple, p)))
    if len(p) <= 2:
        return [np.array(q) for q in p]

    def half(pts):
        h = []
        for q in pts:
            while len(h) >= 2 and (h[-1][0] - h[-2][0]) * (q[1] - h[-2][1]) - (h[-1][1] - h[-2][1]) * (q[0] - h[-2][0]) <= 0:
                h.pop()
            h.append(q)
        return h
    lo, hi = half(p), half(p[::-1])
    return [np.array(q) for q in lo[:-1] + hi[:-1]]


def _seg_dist(a, b):
    """Distance from the origin to segment ab."""
    d = b - a
    dd = float(d @ d)
    t = 0.0 if dd == 0.0 else min(1.0, max(0.0, -float(a @ d) / dd))
    return float(np.linalg.norm(a + t * d))


def signed_gap(coreA, rA, coreB, rB):
    """Signed distance between the rounded convex sets (float64): the origin against the Minkowski difference B - A."""
    m = _hull([b - a for a in coreA for b in coreB])
    if len(m) == 1:
        d = float(np.linalg.norm(m[0]))
        return d - rA - rB
    edges = [(m[i], m[(i + 1) % len(m)]) for i in range(len(m) if len(m) > 2 else 1)]
    d = min(_seg_dist(a, b) for a, b in edges)
    inside = len(m) > 2 and all((b[0] - a[0]) * (-a[1]) - (b[1] - a[1]) * (-a[0]) > 0 for a, b in edges)
    return (-d if inside else d) - rA - rB


# -- placement -----------------------------------------------------------------------------------------------------------
def _place(vA, rA, poseA, vB, rB, angB, direction, target):
    """Origin of B, at angle angB, such that B's core centroid starts on A's and moves along `direction` until the gap
    between the shapes is `target` (or stays on A's centroid when `target` is None or deeper than reachable)."""
    wA = np.array([poseA[0], poseA[1]]) + np.array([_rot(poseA[2], v) for v in vA])
    lB = np.array([_rot(angB, v) for v in vB])
    start = wA.mean(axis=0) - lB.mean(axis=0)
    d = np.asarray(direction, dtype=np.float64) / np.linalg.norm(direction)

    def gap(t):
        return signed_gap(wA, rA, start + t * d + lB, rB)
    if target is None or gap(0.0) >= target:
        return start
    lo, hi = 0.0, 1.0
    while gap(hi) < target:
        hi *= 2.0
    for _ in range(60):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if gap(mid) < target else (lo, mid)
    return start + hi * d


def make_cases(seed=20261015, repeats=2):
    """All cases: every kind x regime x placement (near the origin, translated by up to 1e4 m) x `repeats`."""
    rng = np.random.default_rng(seed)
    cases = []
    k = 0
    for kind, (ta, tb) in KINDS.items():
        for regime in REGIMES:
            for far in (False, True):
                for _ in range(repeats):
                    k += 1
                    size_a = float(np.exp(rng.uniform(math.log(0.05), math.log(50.0))))
                    size_b = size_a * float(np.exp(rng.uniform(-1.5, 1.5)))
                    size_b = min(max(size_b, 0.05), 50.0)
                    A = _shape(rng, ta, size_a, k)
                    B = _shape(rng, tb, size_b, k + 1)
                    vA, rA = core(A)
                    vB, rB = core(B)
                    pa = rng.uniform(-1e4, 1e4, 2) if far else rng.uniform(-3.0, 3.0, 2)
                    angA = rng.uniform(-math.pi, math.pi)
                    poseA = (_f32(pa[0]), _f32(pa[1]), _f32(angA))
                    angB = rng.uniform(-math.pi, math.pi)
                    direction = _rot(rng.uniform(-math.pi, math.pi), (1.0, 0.0))
                    small = min(size_a, size_b)
                    target = {"beyond": SPECULATIVE + 0.004, "inside": SPECULATIVE - 0.006, "touching": 0.0,
                              "shallow": -0.6 * LINEAR_SLOP, "deep": -0.4 * small, "coincident": None,
                              "centroid_inside": -1e9}.get(regime, -0.002)
                    if regime.startswith("rel"):
                        # face to face: B moves along the normal of A's first face, at an exact relative angle
                        rel = {"rel0": 0.0, "rel90": 0.5 * math.pi, "rel180": math.pi}[regime.rstrip("+")]
                        angB = poseA[2] + rel + (1e-6 if regime.endswith("+") else 0.0)
                        e = vA[1] - vA[0] if len(vA) > 1 else np.array([0.0, 1.0])
                        direction = _rot(poseA[2], (e[1], -e[0]))
                    elif regime == "vertex":
                        # a vertex of B pointing at a vertex of A, just inside the speculative distance
                        ca, cb = vA.mean(axis=0), vB.mean(axis=0)
                        ua, ub = vA[0] - ca, vB[0] - cb
                        if float(ua @ ua) == 0.0:
                            ua = np.array([1.0, 0.0])
                        if float(ub @ ub) == 0.0:
                            ub = np.array([1.0, 0.0])
                        direction = _rot(poseA[2], ua)
                        phi_d = math.atan2(direction[1], direction[0])
                        angB = phi_d + math.pi - math.atan2(ub[1], ub[0])
                        target = 0.5 * SPECULATIVE
                    angB = math.remainder(angB, 2.0 * math.pi)
                    if regime == "centroid_inside":  # B's centroid inside A, off A's centroid
                        pB = _place(vA, rA, poseA, vB, rB, angB, direction, None) + direction / np.linalg.norm(direction) * 0.3 * small
                    else:
                        pB = _place(vA, rA, poseA, vB, rB, angB, direction, target)
                    poseB1 = (_f32(pB[0]), _f32(pB[1]), _f32(angB))
                    dp = rng.uniform(-0.003, 0.003, 2)
                    poseB2 = (_f32(pB[0] + dp[0]), _f32(pB[1] + dp[1]), _f32(angB + rng.uniform(-0.01, 0.01)))
                    cases.append(dict(
                        kind=kind, regime=regime, far=far, A=A, B=B, poseA=poseA, poseB1=poseB1, poseB2=poseB2,
                        rule=RULES[k % len(RULES)],
                        impulses=tuple(_f32(x) for x in rng.uniform(0.05, 2.0, 4) * np.array([1, -1, 1, 1])),
                        friction=tuple(_f32(x) for x in rng.uniform(-1.0, 1.0, 16)),
                    ))
    return cases


# -- evaluation helpers shared by the host and device tests -------------------------------------------------------------
def geometry(L, spec):
    """The ctypes shape a spec describes, built with library L's own factories."""
    t = spec[0]
    if t == "circle":
        return capi.Circle(capi.Vec2(spec[1], spec[2]), spec[3])
    if t == "capsule":
        return capi.Capsule(capi.Vec2(spec[1], spec[2]), capi.Vec2(spec[3], spec[4]), spec[5])
    if t == "segment":
        return capi.Segment(capi.Vec2(spec[1], spec[2]), capi.Vec2(spec[3], spec[4]))
    if t == "box":
        p = L.s2MakeOffsetBox(spec[1], spec[2], capi.Vec2(spec[3], spec[4]), spec[5])
    else:
        pts = (capi.Vec2 * len(spec[1]))(*[capi.Vec2(x, y) for x, y in spec[1]])
        hull = L.s2ComputeHull(pts, len(spec[1]))
        assert hull.count == len(spec[1]), "a generated hull lost vertices"
        p = L.s2MakePolygon(C.byref(hull))
    p.radius = spec[-1]  # the reference has no s2MakeRoundedBox: a polygon with the radius set is the same shape
    return p


def collide(L, kind, gA, xfA, gB, xfB, cache):
    """The manifold function of `kind` in library L (cache: a capi.DistanceCache, updated in place where used)."""
    fn = {"circles": L.s2CollideCircles, "capsule_circle": L.s2CollideCapsuleAndCircle,
          "polygon_circle": L.s2CollidePolygonAndCircle, "segment_circle": L.s2CollideSegmentAndCircle,
          "capsules": L.s2CollideCapsules, "polygon_capsule": L.s2CollidePolygonAndCapsule,
          "polygons": L.s2CollidePolygons, "segment_capsule": L.s2CollideSegmentAndCapsule,
          "segment_polygon": L.s2CollideSegmentAndPolygon}[kind]
    if kind.endswith("circle") or kind == "circles":
        return fn(C.byref(gA), xfA, C.byref(gB), xfB)
    return fn(C.byref(gA), xfA, C.byref(gB), xfB, C.byref(cache))


def transform(x, y, s, c):
    return capi.Transform(capi.Vec2(x, y), capi.Rot(s, c))


def pose_transform(pose):
    a = np.float32(pose[2])
    return transform(pose[0], pose[1], float(np.sin(a, dtype=np.float32)), float(np.cos(a, dtype=np.float32)))


def copy_cache(cache):
    out = capi.DistanceCache()
    C.memmove(C.byref(out), C.byref(cache), C.sizeof(out))
    return out


def old_state(case, m1):
    """(count, ids) of the old manifold at pose 2, by the case's rule, from the pose-1 manifold m1:

    real         the pose-1 manifold as it is
    swap         two old points, pose-1 ids in swapped slots
    dup          two old points with the same id (the first match must win)
    nomatch      two old points, neither id can occur
    count0       no old point, but real ids in both slots (they must be ignored)
    count1_junk  one old point with a junk id, and a real id in slot 1 (it must be ignored)
    count2       two old points, the second a junk id when pose 1 had one point
    """
    ids = [m1.points[i].id for i in range(m1.pointCount)]
    id0 = ids[0] if ids else JUNK_ID + 2
    id1 = ids[1] if len(ids) > 1 else JUNK_ID + 3
    rule = case["rule"]
    if rule == "real":
        return m1.pointCount, (id0 if ids else 0, id1 if len(ids) > 1 else 0)
    return {"swap": (2, (id1, id0)), "dup": (2, (id0, id0)), "nomatch": (2, (JUNK_ID, JUNK_ID + 1)),
            "count0": (0, (id0, id1)), "count1_junk": (1, (JUNK_ID, id0)), "count2": (2, (id0, id1))}[rule]


def carry(m, old_count, old_ids):
    """s2UpdateContact's id matching (reference src/contact.c:317-358), restated: for each new point, the slot of the
    FIRST old point (of the first old_count) with the same 16-bit id, or -1; and whether friction persists (same point
    count, every point matched)."""
    matched = []
    for i in range(m.pointCount):
        j = next((j for j in range(old_count) if (old_ids[j] & 0xFFFF) == m.points[i].id), -1)
        matched.append(j)
    friction_persisted = m.pointCount == old_count and all(j >= 0 for j in matched)
    return matched, friction_persisted
