"""GPU: the device narrow phase (s2bUpdateContactsKernel, csrc/device/narrowphase.cu) pinned pair by pair to the reference,
bit for bit.

The scene tests reach this kernel only through whole worlds of mostly boxes. Here every case of tests/narrowphase_cases.py
(all nine manifold kinds of reference src/contact.c:139-154 across distance, orientation, geometry and placement regimes)
is one contact row of a world built through the public API, so the kernel's own code runs: shapes read from the polygon
form of the shape columns, polygon B moved into A's frame while it loads, dispatch by shape type, the GJK cache packed
into 20 bits, 16-bit ids, impulses matched by id, frictionPersisted, and (TGS_Sticky) friction anchors and normals carried
by id. The broad phase plays no part: s2World_Step is never called.

Each case is evaluated at pose 1 from an empty old manifold and at pose 2 with an old state derived from the pose-1 result
(narrowphase_cases.old_state: the real result, swapped ids, duplicate ids, no match, old point count 0 / 1 / 2 with ids
that must be ignored) carrying seeded impulses, friction anchors and normals. The expected rows are the reference library's
s2Collide* on the transforms the device holds, followed by a restatement of s2UpdateContact's id matching."""
import ctypes as C
import collections

import numpy as np
import pytest

import narrowphase_cases as N
from helpers import bit_equal
from solver2d_b200 import capi, device

pytestmark = pytest.mark.gpu

CREATE = {"circle": "s2CreateCircleShape", "capsule": "s2CreateCapsuleShape", "segment": "s2CreateSegmentShape",
          "box": "s2CreatePolygonShape", "hull": "s2CreatePolygonShape"}


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


@pytest.fixture(scope="module")
def cases():
    return N.make_cases()


def _add_body(P, world, pose, spec):
    bd = capi.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    bd.position = capi.Vec2(pose[0], pose[1])
    bd.angle = pose[2]
    bid = P.s2CreateBody(world, C.byref(bd))
    sd = capi.default_shape_def()
    g = N.geometry(P, spec)
    sid = getattr(P, CREATE[spec[0]])(bid, C.byref(sd), C.byref(g))
    assert sid.index >= 0, f"shape {spec} was refused"
    return bid.index, sid.index


def _expected(R, case, xfA, xfB1, xfB2):
    """Reference rows at pose 1 (empty old manifold) and pose 2 (old state by the case's rule), as device contact rows
    without the pair columns, plus the old pose-2 row the device is given."""
    gA, gB = N.geometry(R, case["A"]), N.geometry(R, case["B"])
    cache1 = capi.DistanceCache()
    m1 = N.collide(R, case["kind"], gA, xfA, gB, xfB1, cache1)
    old_count, old_ids = N.old_state(case, m1)
    imp = np.array(case["impulses"], np.float32).reshape(2, 2)
    fr = np.array(case["friction"], np.float32).reshape(2, 2, 4)  # point, (anchor, normal), 4 floats

    old = np.zeros(1, device.CONTACT_ROW)[0]
    old["pointCount"] = old_count
    old["frictionPersisted"] = 1
    old["friction"] = 0.6
    old["normal"] = (0.25, -0.5)  # everything the kernel recomputes starts as junk
    for j in range(2):
        p = old["points"][j]
        p["id"] = old_ids[j]
        p["persisted"] = 1
        p["normalImpulse"], p["tangentImpulse"] = imp[j]
        p["separation"] = 7.0
        p["localAnchorA"] = (3.0, -3.0)
        p["localAnchorB"] = (-2.0, 2.0)
        p["frictionAnchorA"], p["frictionAnchorB"] = fr[j, 0, 0:2], fr[j, 0, 2:4]
        p["frictionNormalA"], p["frictionNormalB"] = fr[j, 1, 0:2], fr[j, 1, 2:4]
    old["cacheCount"] = cache1.count
    old["cacheIndexA"][:3] = list(cache1.indexA)
    old["cacheIndexB"][:3] = list(cache1.indexB)
    old["cacheMetric"] = cache1.metric

    cache2 = N.copy_cache(cache1)
    m2 = N.collide(R, case["kind"], gA, xfA, gB, xfB2, cache2)
    matched, fp = N.carry(m2, old_count, old_ids)

    def row(m, cache, matched, fp, friction_old):
        r = np.zeros(1, device.CONTACT_ROW)[0]
        r["pointCount"] = m.pointCount
        r["frictionPersisted"] = 1 if fp else 0
        r["friction"] = 0.6
        r["normal"] = (m.normal.x, m.normal.y)
        for i in range(2):
            q, p = m.points[i], r["points"][i]
            p["localAnchorA"] = (q.localAnchorA.x, q.localAnchorA.y)
            p["localAnchorB"] = (q.localAnchorB.x, q.localAnchorB.y)
            p["separation"] = q.separation
            p["id"] = q.id if i < m.pointCount else 0
            j = matched[i] if i < len(matched) else -1
            if j >= 0:
                p["persisted"] = 1
                p["normalImpulse"], p["tangentImpulse"] = imp[j]
                p["frictionAnchorA"], p["frictionAnchorB"] = friction_old[j, 0, 0:2], friction_old[j, 0, 2:4]
                p["frictionNormalA"], p["frictionNormalB"] = friction_old[j, 1, 0:2], friction_old[j, 1, 2:4]
        r["cacheCount"] = cache.count
        r["cacheIndexA"][:3] = list(cache.indexA)
        r["cacheIndexB"][:3] = list(cache.indexB)
        r["cacheMetric"] = cache.metric
        return r

    want1 = row(m1, cache1, [-1] * m1.pointCount, m1.pointCount == 0, fr)
    want2 = row(m2, cache2, matched, fp, fr)
    return want1, old, want2


FIELDS = ("pointCount", "frictionPersisted", "friction", "normal", "cacheCount", "cacheMetric")
POINT_FIELDS = ("localAnchorA", "localAnchorB", "separation", "normalImpulse", "tangentImpulse", "id", "persisted")
STICKY_FIELDS = ("frictionAnchorA", "frictionAnchorB", "frictionNormalA", "frictionNormalB")


def _same(g, w):
    g, w = np.asarray(g), np.asarray(w)
    return bit_equal(g, w) if g.dtype == np.float32 else np.array_equal(g, w)


def _differences(got, want, sticky):
    bad = [f for f in FIELDS if not _same(got[f], want[f])]
    if not (_same(got["cacheIndexA"][:3], want["cacheIndexA"][:3]) and _same(got["cacheIndexB"][:3], want["cacheIndexB"][:3])):
        bad.append("cache indices")
    for i in range(2):
        for f in POINT_FIELDS + (STICKY_FIELDS if sticky else ()):
            if not _same(got["points"][i][f], want["points"][i][f]):
                bad.append(f"point {i} {f}")
    return bad


@pytest.mark.parametrize("solver", ["TGS_Soft", "TGS_Sticky"])
def test_narrowphase_matches_reference_per_pair(reference, product, dev, cases, solver):
    R, P = reference, product
    world = P.create_world(solver)
    try:
        # one body per shape: A, B at pose 1, B at pose 2
        ids = []
        for case in cases:
            a = _add_body(P, world, case["poseA"], case["A"])
            b1 = _add_body(P, world, case["poseB1"], case["B"])
            b2 = _add_body(P, world, case["poseB2"], case["B"])
            ids.append((a, b1, b2))
        dev.lib.s2World_Flush.restype = None
        dev.lib.s2World_Flush.argtypes = [capi.WorldId]
        dev.lib.s2World_Flush(world)
        dw = device.DeviceWorld.attach(dev, world)
        bodies = dw.download_all_bodies()

        def xf(body):  # the origin and rotation bits the device holds
            o, q = bodies["origin"][body], bodies["rot"][body]
            return N.transform(float(o[0]), float(o[1]), float(q[0]), float(q[1]))

        rows, wants, labels = [], [], []
        for case, (a, b1, b2) in zip(cases, ids):
            want1, old2, want2 = _expected(R, case, xf(a[0]), xf(b1[0]), xf(b2[0]))
            for (body, shape), old, want, pose in ((b1, None, want1, 1), (b2, old2, want2, 2)):
                r = np.zeros(1, device.CONTACT_ROW)[0] if old is None else old.copy()
                if old is None:
                    r["friction"] = 0.6
                r["shapeA"], r["shapeB"], r["bodyA"], r["bodyB"] = a[1], shape, a[0], body
                rows.append(r)
                wants.append(want)
                labels.append((case, pose))
        rows = np.array(rows, dtype=device.CONTACT_ROW)
        keys = (np.minimum(rows["shapeA"], rows["shapeB"]).astype(np.uint64) << np.uint64(32)) | \
            np.maximum(rows["shapeA"], rows["shapeB"]).astype(np.uint64)
        perm = np.argsort(keys, kind="stable")
        dw.upload_contacts(rows[perm])
        dw.update_contacts()
        got = dw.download_contacts(len(rows) + 8)
        assert len(got) == len(rows)

        sticky = solver == "TGS_Sticky"
        failures = []
        coverage = collections.Counter()
        for k, p in enumerate(perm):
            case, pose = labels[p]
            want = wants[p]
            assert got[k]["shapeA"] == rows[p]["shapeA"] and got[k]["shapeB"] == rows[p]["shapeB"]
            bad = _differences(got[k], want, sticky)
            if bad:
                failures.append(f"{case['kind']} {case['regime']} far={case['far']} rule={case['rule']} pose {pose}: {bad}")
            coverage[(case["kind"], case["far"], int(want["pointCount"]))] += 1
            if pose == 2 and want["points"]["persisted"].any():
                coverage[(case["kind"], "carried")] += 1
        assert not failures, f"{len(failures)} of {len(rows)} rows differ from the reference, e.g. {failures[:8]}"
    finally:
        P.s2DestroyWorld(world)

    # the cases really reach every kind with 0, 1 and (where the kind has two) 2 points, near and far, and carry impulses
    for kind, (ta, tb) in N.KINDS.items():
        for far in (False, True):
            for n in (0, 1) if tb == "circle" else (0, 1, 2):
                assert coverage[(kind, far, n)] >= 2, f"{kind} far={far}: only {coverage[(kind, far, n)]} rows with {n} points"
        assert coverage[(kind, "carried")] >= 10, f"{kind}: impulses carried in only {coverage[(kind, 'carried')]} rows"
