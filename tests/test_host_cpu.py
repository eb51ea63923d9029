"""CPU: the product library loads without a GPU, exports every symbol the headers declare, and its host-side geometry and
narrow-phase code (csrc/shared/s2_collide.h — the SAME source the CUDA narrow-phase kernel compiles) is bit-identical to
the unmodified reference on seeded inputs (recorded as digests in tests/golden, and compared live where the reference is
built). No world is created here: s2CreateWorld needs a CUDA device by design."""
import ctypes as C
import hashlib
import json
import os
import re
import struct

import numpy as np
import pytest

from solver2d_b200 import capi, device

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


@pytest.fixture(scope="module")
def reference_if_built():
    """The unmodified reference where oracle/_ref is built, else None (the recorded digests stand in for it)."""
    from oracle import ref
    return ref.load() if ref.available() or ref.build_ref() else None


def test_library_exports_every_declared_symbol(product):
    assert product.missing == []
    lib = C.CDLL(device.LIB_PATH)
    header = open(os.path.join(ROOT, "include", "s2b_device.h")).read()
    declared = re.findall(r"^S2B_API [^;(]*?(s2b_\w+)\(", header, flags=re.M)
    assert len(declared) >= 35
    for name in declared + device.ABI_SYMBOLS:
        assert hasattr(lib, name), name
    ext = open(os.path.join(ROOT, "include", "solver2d_b200.h")).read()
    for name in re.findall(r"^S2B_API [^;(]*?(s2World_\w+)\(", ext, flags=re.M):
        assert hasattr(lib, name), name
    for variant in ("Jacobi", "PGS", "PGS_NGS", "PGS_NGS_Block", "PGS_Soft", "TGS_Soft", "TGS_Sticky", "TGS_NGS", "XPBD",
                    "SoftStep"):
        assert hasattr(lib, f"s2Solve_{variant}")


def test_row_struct_sizes_match_numpy_mirrors():
    lib = C.CDLL(device.LIB_PATH)
    out = (C.c_int32 * 6)()
    lib.s2b_abi_sizes(out)
    assert list(out)[:4] == [device.BODY_ROW.itemsize, device.SHAPE_ROW.itemsize, device.JOINT_ROW.itemsize,
                             device.CONTACT_ROW.itemsize]
    assert out[4] == C.sizeof(device.StepContext) and out[5] == C.sizeof(device.Counters)


# Reference outputs of the three seeded sweeps below, one truncated sha1 per trial (host_digests in tests/golden/make_golden.py):
# the product is checked against them everywhere, and against the reference library itself where oracle/_ref is built.
HOST_GOLDEN = os.path.join(ROOT, "tests", "golden", "host_reference_sha1.json")


def trial_digest(chunks) -> str:
    return hashlib.sha1(b"".join(chunks)).hexdigest()[:16]


def _check(name, product_trials, reference):
    if reference is not None:
        for t, (mine, want) in enumerate(zip(product_trials, SWEEPS[name](reference, True))):
            assert mine == want, f"{name}: trial {t} differs from the reference"
    with open(HOST_GOLDEN) as fh:
        golden = json.load(fh)[name]
    assert len(golden) == len(product_trials)
    for t, (mine, want) in enumerate(zip(product_trials, golden)):
        assert trial_digest(mine) == want, f"{name}: trial {t} differs from the recorded reference"


def _poly(p):
    n = p.count
    return [struct.pack("<if", n, p.radius)] + [struct.pack("<ff", p.vertices[i].x, p.vertices[i].y) for i in range(n)] \
        + [struct.pack("<ff", p.normals[i].x, p.normals[i].y) for i in range(n)]


def polygon_sweep(L, is_reference):
    rng = np.random.default_rng(7)
    trials = []
    for _ in range(50):
        out = []
        hx, hy = rng.uniform(0.05, 3.0, 2)
        ang = rng.uniform(-3, 3)
        c = capi.Vec2(*rng.uniform(-2, 2, 2))
        out += _poly(L.s2MakeBox(hx, hy))
        a = L.s2MakeOffsetBox(hx, hy, c, ang)
        out += _poly(a)
        for dens in (1.0, 20.0):
            out.append(bytes(L.s2ComputePolygonMass(C.byref(a), dens)))
        if is_reference:  # the reference has no s2MakeRoundedBox: a box with the radius set is the same polygon
            rb = L.s2MakeBox(hx, hy)
            rb.radius = 0.1
        else:
            rb = L.s2MakeRoundedBox(hx, hy, 0.1)
        out.append(bytes(L.s2ComputePolygonMass(C.byref(rb), 2.0)))
        p1, p2 = capi.Vec2(*rng.uniform(-1, 1, 2)), capi.Vec2(*rng.uniform(1.5, 3, 2))
        out += _poly(L.s2MakeCapsule(p1, p2, 0.3))
        cap = capi.Capsule(p1, p2, 0.3)
        out.append(bytes(L.s2ComputeCapsuleMass(C.byref(cap), 1.5)))
        xf = capi.Transform(c, capi.Rot(np.float32(np.sin(ang)), np.float32(np.cos(ang))))
        out.append(bytes(L.s2ComputePolygonAABB(C.byref(a), xf)))
        trials.append(out)
    return trials


def test_polygon_factories_and_mass_match_reference(reference_if_built, product):
    _check("polygon", polygon_sweep(product, False), reference_if_built)


def hull_sweep(L, is_reference):
    rng = np.random.default_rng(11)
    trials = []
    for trial in range(200):
        n = int(rng.integers(3, 9))
        pts = (capi.Vec2 * n)(*[capi.Vec2(*rng.uniform(-1.5, 1.5, 2)) for _ in range(n)])
        if trial % 5 == 0:  # welded / collinear inputs
            pts[1] = capi.Vec2(pts[0].x + 0.001, pts[0].y)
        h = L.s2ComputeHull(pts, n)
        out = [struct.pack("<i", h.count)] + [struct.pack("<ff", h.points[i].x, h.points[i].y) for i in range(h.count)]
        if h.count >= 3:
            out += _poly(L.s2MakePolygon(C.byref(h)))
        trials.append(out)
    return trials


def test_hull_matches_reference(reference_if_built, product):
    _check("hull", hull_sweep(product, False), reference_if_built)


def _manifold(m):
    out = [struct.pack("<i", m.pointCount)]
    if m.pointCount > 0:
        out.append(struct.pack("<ff", m.normal.x, m.normal.y))
    for i in range(m.pointCount):
        p = m.points[i]
        out.append(struct.pack("<5fI", p.localAnchorA.x, p.localAnchorA.y, p.localAnchorB.x, p.localAnchorB.y, p.separation,
                               p.id & 0xFFFFFFFF))
    return out


def manifold_sweep(L, is_reference):
    rng = np.random.default_rng(2024)

    def xf(x, y, ang):
        return capi.Transform(capi.Vec2(x, y), capi.Rot(np.float32(np.sin(ang)), np.float32(np.cos(ang))))

    trials = []
    for trial in range(400):
        out = []
        boxA = L.s2MakeBox(*rng.uniform(0.3, 1.2, 2))
        pts = (capi.Vec2 * 6)(*[capi.Vec2(*rng.uniform(-0.8, 0.8, 2)) for _ in range(6)])
        hull = L.s2ComputeHull(pts, 6)
        polyB = L.s2MakePolygon(C.byref(hull)) if hull.count >= 3 else L.s2MakeBox(0.5, 0.4)
        polyB.radius = 0.05 if trial % 3 == 0 else 0.0
        circ = capi.Circle(capi.Vec2(*rng.uniform(-0.2, 0.2, 2)), float(rng.uniform(0.2, 0.6)))
        circ2 = capi.Circle(capi.Vec2(0.0, 0.0), float(rng.uniform(0.2, 0.6)))
        cap = capi.Capsule(capi.Vec2(-0.5, 0.0), capi.Vec2(0.5, float(rng.uniform(-0.2, 0.2))), float(rng.uniform(0.1, 0.4)))
        cap2 = capi.Capsule(capi.Vec2(0.0, -0.4), capi.Vec2(0.1, 0.5), 0.25)
        seg = capi.Segment(capi.Vec2(-1.0, 0.0), capi.Vec2(1.0, float(rng.uniform(-0.3, 0.3))))
        d = rng.uniform(0.6, 1.9)
        th = rng.uniform(0, 2 * np.pi)
        cache = [capi.DistanceCache() for _ in range(5)]
        for it in range(3):  # persistent cache across slightly moved poses
            A = xf(*rng.uniform(-0.01, 0.01, 2), rng.uniform(-0.02, 0.02) + 0.3 * trial)
            B = xf(d * np.cos(th) + rng.uniform(-0.01, 0.01), d * np.sin(th) + rng.uniform(-0.01, 0.01), rng.uniform(-3, 3) if it == 0 else 0.1 * it)
            for m in (L.s2CollideCircles(C.byref(circ), A, C.byref(circ2), B),
                      L.s2CollideCapsuleAndCircle(C.byref(cap), A, C.byref(circ), B),
                      L.s2CollideSegmentAndCircle(C.byref(seg), A, C.byref(circ), B),
                      L.s2CollidePolygonAndCircle(C.byref(boxA), A, C.byref(circ), B),
                      L.s2CollidePolygons(C.byref(boxA), A, C.byref(polyB), B, C.byref(cache[0])),
                      L.s2CollideCapsules(C.byref(cap), A, C.byref(cap2), B, C.byref(cache[1])),
                      L.s2CollidePolygonAndCapsule(C.byref(boxA), A, C.byref(cap), B, C.byref(cache[2])),
                      L.s2CollideSegmentAndCapsule(C.byref(seg), A, C.byref(cap), B, C.byref(cache[3])),
                      L.s2CollideSegmentAndPolygon(C.byref(seg), A, C.byref(polyB), B, C.byref(cache[4]))):
                out += _manifold(m)
            for c in cache:
                out.append(struct.pack("<i", c.count) + bytes(c.indexA) + bytes(c.indexB))
        trials.append(out)
    return trials


def test_manifold_functions_match_reference_bitwise(reference_if_built, product):
    """All nine shape-pair manifold functions (reference src/contact.c:139-154) on random near-contact configurations,
    with the GJK cache carried over several perturbed calls as a persistent contact does."""
    trials = manifold_sweep(product, False)
    _check("manifold", trials, reference_if_built)
    hits = sum(struct.unpack_from("<i", chunk)[0] > 0 for t in trials for chunk in t if len(chunk) == 4)  # pointCounts
    assert hits > 1500  # the sweep actually produced contacts


def edge_manifold_sweep(L, is_reference):
    """The cases of tests/narrowphase_cases.py (also run through the device kernel by test_narrowphase_gpu.py): each pair
    from an empty cache at pose 1, then at pose 2 with the cache carried over."""
    import narrowphase_cases as N
    trials = []
    for case in N.make_cases():
        gA, gB = N.geometry(L, case["A"]), N.geometry(L, case["B"])
        xfA = N.pose_transform(case["poseA"])
        cache = capi.DistanceCache()
        out = []
        for pose in ("poseB1", "poseB2"):
            out += _manifold(N.collide(L, case["kind"], gA, xfA, gB, N.pose_transform(case[pose]), cache))
            out.append(struct.pack("<fi", cache.metric, cache.count) + bytes(cache.indexA) + bytes(cache.indexB))
        trials.append(out)
    return trials


def test_edge_manifold_cases_match_reference_bitwise(reference_if_built, product):
    """Separations around the speculative distance, touching, shallow and deep overlap, coincident centres, exact
    relative angles with and without a 1e-6 rad offset, vertex against vertex, 3-8-gons with and without radius, offset
    circles, short capsules, sizes 0.05-50 m, near the origin and 1e4 m away."""
    _check("edge_manifold", edge_manifold_sweep(product, False), reference_if_built)


SWEEPS = {"polygon": polygon_sweep, "hull": hull_sweep, "manifold": manifold_sweep, "edge_manifold": edge_manifold_sweep}


def _atan2_inputs(n, seed):
    rng = np.random.default_rng(seed)
    # (sin, cos)-like pairs as s2RelativeAngle produces them, raw bit patterns, and the special values
    a = rng.uniform(-np.pi, np.pi, n)
    y = [np.sin(a).astype(np.float32), rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32).view(np.float32),
         np.array([0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, 1e-40, -1e-40, 3e38, 0.4375, 0.6875, 1.1875, 2.4375] * 13, np.float32)]
    x = [np.cos(a).astype(np.float32), rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32).view(np.float32),
         np.repeat(np.array([0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, 1e-40, -1e-40, 3e38, 0.4375, 0.6875, 1.1875, 2.4375],
                            np.float32), 13)]
    return np.concatenate(y), np.concatenate(x)


def test_device_atan2_restatement_equals_libm_on_host():
    """include/solver2d/atan2_f32.h (what the kernels call) against the C library atan2f the reference is linked with."""
    import ctypes.util
    lib = C.CDLL(device.LIB_PATH)
    lib.s2Atan2Device.restype = C.c_float
    lib.s2Atan2Device.argtypes = [C.c_float, C.c_float]
    libm = C.CDLL(ctypes.util.find_library("m"))
    libm.atan2f.restype = C.c_float
    libm.atan2f.argtypes = [C.c_float, C.c_float]
    y, x = _atan2_inputs(150000, 11)
    mine = np.array([lib.s2Atan2Device(float(a), float(b)) for a, b in zip(y, x)], np.float32)
    want = np.array([libm.atan2f(float(a), float(b)) for a, b in zip(y, x)], np.float32)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(mine), nan)
    assert np.array_equal(mine[~nan].view(np.uint32), want[~nan].view(np.uint32))
