"""GPU: island labels (s2b_download_islands) against a graph reference, scipy's connected components over an edge list
built on the host.

The edges are the contacts with at least one manifold point and the live joints. An endpoint drops out when it cannot be
moved by a constraint: a static or kinematic body, or one with zero inverse mass and zero inverse inertia; a mouse joint's
body A always drops out, and so does a self-edge (s2bItemEndpoints). The label of a body is the smallest slot of its
component, -1 for a free slot, and the island count is the number of distinct labels over the valid slots. Both must equal
the device's exactly.

The scenes are seeded and each is checked after its first step and after several more: debris of boxes, circles and
capsules (with the edges also taken from the reference library's own contact table, every step checked against the oracle
on the way), two piles on one kinematic platform and the kinematic rigs, every joint type with mouse joints on a static
and on a dynamic body A and a self-joint, a contact pair with no points, slot churn (freed slots, a new body in a freed low
slot that becomes its island's label), a 20 000-link revolute chain whose slots run in scrambled order, where the
lock-free hooks race, the 100 128-box pyramid, and the tumbler's hub."""
import ctypes as C

import numpy as np
import pytest
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from solver2d_b200 import capi, device, scenes
from solver2d_b200.capi import Vec2
from test_multistep_gpu import _run

pytestmark = pytest.mark.gpu
DT = 1.0 / 60.0
DYNAMIC = 2  # body type in flags bits 1-2 (s2b_internal.cuh)


@pytest.fixture(scope="module")
def product():
    return capi.Solver2D(device.LIB_PATH)


def reference_islands(bodies, a, b, joints=None):
    """(labels, island count) of the constraint graph: `a`, `b` are the body slots of the contacts with points."""
    cap = len(bodies)
    valid = (bodies["flags"] & 1) == 1
    movable = valid & (((bodies["flags"] >> 1) & 3) == DYNAMIC) & ((bodies["invMass"] != 0) | (bodies["invI"] != 0))
    ea, eb = [np.asarray(a, np.int64)], [np.asarray(b, np.int64)]
    if joints is not None and len(joints):
        live = (joints["flags"] & 1) == 1
        mouse = ((joints["flags"] >> 1) & 7) == device.JOINT_MOUSE
        ea.append(np.where(mouse, -1, joints["bodyA"])[live].astype(np.int64))
        eb.append(joints["bodyB"][live].astype(np.int64))
    ea, eb = np.concatenate(ea), np.concatenate(eb)
    keep = (ea >= 0) & (eb >= 0) & (ea != eb)
    ea, eb = ea[keep], eb[keep]
    keep = movable[ea] & movable[eb]
    ea, eb = ea[keep], eb[keep]
    graph = coo_matrix((np.ones(len(ea)), (ea, eb)), shape=(cap, cap))
    _, comp = connected_components(graph, directed=False)
    smallest = np.full(cap, cap, dtype=np.int64)
    np.minimum.at(smallest, comp, np.arange(cap))
    labels = np.where(valid, smallest[comp], -1).astype(np.int32)
    return labels, int((labels[valid] == np.nonzero(valid)[0]).sum())


def check(dw, rows=None):
    """Compare the device's labels with the reference's over the device's own contact rows (or `rows`); returns labels."""
    c = dw.counters()
    bodies = dw.download_all_bodies(c.bodyCapacity)
    if rows is None:
        rows = dw.download_contacts(c.contactCount + 64)
    live = rows["pointCount"] >= 1
    want, want_n = reference_islands(bodies, rows["bodyA"][live], rows["bodyB"][live], dw.download_joints(c.jointCapacity))
    got, n = dw.islands(len(bodies))
    assert len(bodies) > 0 and want_n > 0
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, f"labels differ at slots {bad[:8].tolist()}: device {got[bad[:8]].tolist()} reference {want[bad[:8]].tolist()}"
    assert n == want_n
    return got


def _attach(dev, sc):
    dev.lib.s2World_Flush.restype = None
    dev.lib.s2World_Flush.argtypes = [capi.WorldId]
    dev.lib.s2World_Flush(sc.world)
    return device.DeviceWorld.attach(dev, sc.world)


def _body(lib, sc, kind, x, y, shape="box", hx=0.5, hy=0.5, angle=0.0, vx=0.0, w=0.0):
    bd = capi.default_body_def()
    bd.type = kind
    bd.position = Vec2(x, y)
    bd.angle = angle
    bd.linearVelocity = Vec2(vx, 0.0)
    bd.angularVelocity = w
    bid = lib.s2CreateBody(sc.world, C.byref(bd))
    sd = capi.default_shape_def()
    sd.density = 1.0
    if shape == "circle":
        lib.s2CreateCircleShape(bid, C.byref(sd), C.byref(capi.Circle(Vec2(0.0, 0.0), hx)))
    elif shape == "capsule":
        lib.s2CreateCapsuleShape(bid, C.byref(sd), C.byref(capi.Capsule(Vec2(-hx, 0.0), Vec2(hx, 0.0), hy)))
    else:
        lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(lib.s2MakeBox(hx, hy)))
    sc.bodies.append(bid)
    return bid


def _steps(sc, dw, n, rows=None):
    for _ in range(n):
        sc.step(DT, 4, 2, True)
    return check(dw, rows)


# ---- debris ---------------------------------------------------------------------------------------------------------------

def debris(lib, solver="TGS_Soft", seed=5, clusters=14):
    """Clusters of boxes, circles and capsules dropped on a static ground among static posts: many islands of mixed sizes,
    singletons in the air."""
    rng = np.random.default_rng(seed)
    sc = scenes.Scene(lib, lib.create_world(solver), name="debris")
    sc.bodies.append(scenes._ground(lib, sc.world, 60.0))
    for k in range(6):
        _body(lib, sc, capi.STATIC_BODY, -50.0 + 20.0 * k, 1.0, hx=0.3, hy=1.0)
    for k in range(clusters):
        # a cluster of touching shapes three wide, 1 to 40 of them, and one shape alone in the air
        x0 = -55.0 + 8.0 * k + rng.uniform(-1.0, 1.0)
        for n in range(int(rng.integers(1, 40))):
            kind = ("box", "circle", "capsule")[int(rng.integers(0, 3))]
            _body(lib, sc, capi.DYNAMIC_BODY, x0 + 0.8 * (n % 3), 0.45 + 0.7 * (n // 3), kind,
                  hx=float(rng.uniform(0.3, 0.45)), hy=float(rng.uniform(0.2, 0.35)), angle=float(rng.uniform(-0.5, 0.5)))
        _body(lib, sc, capi.DYNAMIC_BODY, x0, 40.0 + rng.uniform(0.0, 5.0), "circle", hx=0.3)
    return sc


def test_debris_labels_from_the_reference_contact_table(reference, product, dev):
    """Every step checked against the oracle (test_multistep_gpu._run), and the labels against the components of the
    reference library's post-collide contact table of the same step, and of the device's."""
    seen = {}

    def observe(R, wid, rows):
        seen["rows"] = rows

    def after(dw):
        labels = check(dw, seen["rows"])
        check(dw)
        valid = labels >= 0
        sizes = np.bincount(labels[valid])
        seen.setdefault("sizes", set()).update(sizes[sizes > 0].tolist())

    _run(reference, product, dev, debris, "TGS_Soft", 40, 4, 2, {}, observe=observe, after_step=after)
    assert 1 in seen["sizes"] and max(seen["sizes"]) >= 10 and len(seen["sizes"]) >= 5, sorted(seen["sizes"])


# ---- kinematic bodies -----------------------------------------------------------------------------------------------------

def test_two_piles_on_one_kinematic_platform(product, dev):
    lib = product
    sc = scenes.Scene(lib, lib.create_world("TGS_Soft"), name="platform")
    plat = _body(lib, sc, capi.KINEMATIC_BODY, 0.0, -1.0, hx=20.0, hy=0.5, vx=0.5)
    piles = []
    for x0 in (-10.0, 10.0):
        pile = []
        for i in range(4):
            for j in range(i, 4):
                pile.append(_body(lib, sc, capi.DYNAMIC_BODY, x0 + (i + 1.0) * 0.5 + (j - i) - 2.0, (2.0 * i + 1.0) * 0.5 - 0.5))
        piles.append([b.index for b in pile])
    dw = _attach(dev, sc)
    for n in (1, 10):
        labels = _steps(sc, dw, n)
        assert labels[plat.index] == plat.index, "a kinematic body is an island of its own"
        assert [set(labels[p].tolist()) for p in piles] == [{min(p)} for p in piles], "one island per pile"
    sc.destroy()


def test_kinematic_rigs(product, dev):
    sc = scenes.kinematic_rigs(product, "TGS_Soft", platforms=3, base_count=6)
    dw = _attach(dev, sc)
    for n in (1, 12):
        labels = _steps(sc, dw, n)
        kin = [b.index for b in sc.piles["kinematic"]]
        assert (labels[kin] == kin).all()
    sc.destroy()


# ---- every joint type -----------------------------------------------------------------------------------------------------

def _joint_scene(lib):
    sc = scenes.Scene(lib, lib.create_world("TGS_Soft"), name="joints")
    ground = scenes._ground(lib, sc.world, 60.0, y=-30.0)
    sc.bodies.append(ground)
    D = capi.DYNAMIC_BODY
    chains = {}
    for c, kind in enumerate(("revolute", "weld", "prismatic", "motor")):
        links = [_body(lib, sc, D, -30.0 + 12.0 * c + 1.2 * k, 10.0, hx=0.5, hy=0.1) for k in range(6)]
        for a, b in zip(links, links[1:]):
            pivot = Vec2(float(lib.s2Body_GetPosition(a).x) + 0.6, 10.0)
            if kind == "revolute":
                jd = capi.default_revolute_def()
            elif kind == "weld":
                jd = capi.default_weld_def()
            elif kind == "prismatic":
                jd = capi.default_prismatic_def()
                jd.localAxisA = Vec2(1.0, 0.0)
            else:
                jd = capi.default_motor_def()
            jd.bodyIdA, jd.bodyIdB = a, b
            if kind != "motor":
                jd.localAnchorA = lib.s2Body_GetLocalPoint(a, pivot)
                jd.localAnchorB = lib.s2Body_GetLocalPoint(b, pivot)
            else:
                jd.linearOffset = Vec2(1.2, 0.0)
            create = {"revolute": lib.s2CreateRevoluteJoint, "weld": lib.s2CreateWeldJoint,
                      "prismatic": lib.s2CreatePrismaticJoint, "motor": lib.s2CreateMotorJoint}[kind]
            sc.joints.append(create(sc.world, C.byref(jd)))
        chains[kind] = [b.index for b in links]
    # mouse joints: body A static (the ground), and body A dynamic, which the joint never moves
    dragged = _body(lib, sc, D, 25.0, 10.0)
    puller = _body(lib, sc, D, 28.0, 10.0)
    dragged2 = _body(lib, sc, D, 31.0, 10.0)
    for a, b in ((ground, dragged), (puller, dragged2)):
        md = capi.default_mouse_def()
        md.bodyIdA, md.bodyIdB = a, b
        p = lib.s2Body_GetPosition(b)
        md.target = Vec2(p.x + 1.0, p.y + 1.0)
        md.hertz, md.dampingRatio = 3.0, 0.7
        sc.joints.append(lib.s2CreateMouseJoint(sc.world, C.byref(md)))
    # a self-joint connects nothing
    lone = _body(lib, sc, D, 36.0, 10.0)
    jd = capi.default_revolute_def()
    jd.bodyIdA = jd.bodyIdB = lone
    sc.joints.append(lib.s2CreateRevoluteJoint(sc.world, C.byref(jd)))
    return sc, chains, (dragged.index, puller.index, dragged2.index, lone.index)


def test_every_joint_type(product, dev):
    sc, chains, (dragged, puller, dragged2, lone) = _joint_scene(product)
    dw = _attach(dev, sc)
    for n in (1, 8):
        labels = _steps(sc, dw, n)
        for kind, ids in chains.items():
            assert set(labels[ids].tolist()) == {min(ids)}, f"the {kind} chain is not one island"
        assert labels[dragged] == dragged and labels[puller] == puller and labels[dragged2] == dragged2
        assert labels[lone] == lone
    sc.destroy()


# ---- contacts without points ----------------------------------------------------------------------------------------------

def test_pair_without_points_does_not_connect(product, dev):
    """Two piles whose bottom boxes are 0.05 m apart: inside each other's fat AABBs (margin 0.1 m), beyond the speculative
    distance (0.02 m), so the pair exists with no point. A plank laid across the two piles then merges them."""
    lib = product
    sc = scenes.Scene(lib, lib.create_world("TGS_Soft"), name="gap")
    sc.bodies.append(scenes._ground(lib, sc.world, 20.0))
    left = [_body(lib, sc, capi.DYNAMIC_BODY, -0.525, 0.5 + k) for k in range(2)]
    right = [_body(lib, sc, capi.DYNAMIC_BODY, 0.525, 0.5 + k) for k in range(2)]
    L, Rt = [b.index for b in left], [b.index for b in right]
    dw = _attach(dev, sc)
    for n in (1, 6):
        labels = _steps(sc, dw, n)
        rows = dw.download_contacts(dw.counters().contactCount + 64)
        gap = ((rows["bodyA"] == L[0]) & (rows["bodyB"] == Rt[0])) | ((rows["bodyA"] == Rt[0]) & (rows["bodyB"] == L[0]))
        assert gap.sum() == 1 and rows["pointCount"][gap][0] == 0, "the pair across the gap must exist without points"
        assert set(labels[L].tolist()) == {min(L)} and set(labels[Rt].tolist()) == {min(Rt)}
    plank = _body(lib, sc, capi.DYNAMIC_BODY, 0.0, 2.1, hx=1.5, hy=0.1)
    for n in (1, 6):
        labels = _steps(sc, dw, n)
        assert set(labels[L + Rt + [plank.index]].tolist()) == {min(L)}
    sc.destroy()


# ---- slot churn -----------------------------------------------------------------------------------------------------------

def test_slot_churn(product, dev):
    """Three piles of 21 boxes (slots: ground 22 k, boxes 22 k + 1 ...). Freed slots are labelled -1; a new box on the
    second pile takes a freed slot below the pile's label and becomes its label."""
    lib = product
    sc = scenes.pyramid_field(lib, "TGS_Soft", count=3, base_count=6)
    ids = [b.index for b in sc.bodies]
    assert ids == list(range(66))
    dw = _attach(dev, sc)
    _steps(sc, dw, 1)
    # the tops of piles 0 and 2, then the bottom-left box of pile 1 (its label)
    victims = [sc.bodies[21], sc.bodies[65], sc.bodies[23]]
    for v in victims:
        lib.s2DestroyBody(v)
    freed = [21, 65, 23]
    pile1 = list(range(24, 44))
    for n in (1, 5):
        labels = _steps(sc, dw, n)
        assert (labels[freed] == -1).all() and set(labels[pile1].tolist()) == {24}
    p = lib.s2Body_GetPosition(sc.bodies[43])
    new = _body(lib, sc, capi.DYNAMIC_BODY, float(p.x), float(p.y) + 1.0)
    assert new.index in (21, 23), new.index
    for n in (1, 10):
        labels = _steps(sc, dw, n)
        assert set(labels[pile1 + [new.index]].tolist()) == {new.index}
        assert (labels[[f for f in freed if f != new.index]] == -1).all()
    sc.destroy()


# ---- hooks that race ------------------------------------------------------------------------------------------------------

def test_long_chain_in_scrambled_slots(product, dev):
    """A 20 000-link revolute chain hanging from the ground, its links created in slots freed in shuffled and in reverse
    order: the hooks meet roots in every order."""
    lib = product
    n = 20000
    rng = np.random.default_rng(3)
    sc = scenes.Scene(lib, lib.create_world("TGS_Soft"), name="chain")
    ground = scenes._ground(lib, sc.world, 10.0, y=-50.0)
    sc.bodies.append(ground)
    bd = capi.default_body_def()
    bd.type = capi.DYNAMIC_BODY
    fillers = [lib.s2CreateBody(sc.world, C.byref(bd)) for _ in range(n)]
    order = np.concatenate([rng.permutation(n // 2), np.arange(n // 2, n)[::-1]])
    for k in order:
        lib.s2DestroyBody(fillers[int(k)])
    links = [_body(lib, sc, capi.DYNAMIC_BODY, 0.5 + k, 0.0, hx=0.5, hy=0.05) for k in range(n)]
    prev = ground
    for k, link in enumerate(links):
        jd = capi.default_revolute_def()
        jd.bodyIdA, jd.bodyIdB = prev, link
        pivot = Vec2(float(k), 0.0)
        jd.localAnchorA = lib.s2Body_GetLocalPoint(prev, pivot)
        jd.localAnchorB = lib.s2Body_GetLocalPoint(link, pivot)
        sc.joints.append(lib.s2CreateRevoluteJoint(sc.world, C.byref(jd)))
        prev = link
    slots = np.array([b.index for b in links])
    assert (np.diff(slots) < 0).sum() > n // 4, "the chain's slots are not scrambled"
    dw = _attach(dev, sc)
    for m in (1, 3):
        labels = _steps(sc, dw, m)
        assert set(labels[slots].tolist()) == {int(slots.min())}
    sc.destroy()


def test_bench_pyramid_is_one_island(product, dev):
    sc = scenes.pyramid(product, "TGS_Soft", base_count=447)
    dw = _attach(dev, sc)
    for n in (1, 3):
        labels = _steps(sc, dw, n)
        boxes = np.array([b.index for b in sc.bodies[1:]])
        assert len(boxes) == 100128 and set(labels[boxes].tolist()) == {int(boxes.min())}
    sc.destroy()


# ---- a hub ----------------------------------------------------------------------------------------------------------------

def test_tumbler_hub(product, dev):
    """The container (one dynamic body of four walls, jointed to the ground) and every box touching it: one island."""
    sc = scenes.tumbler(product, "TGS_Soft", grid=60, half_extent=10.0)
    dw = _attach(dev, sc)
    container = sc.bodies[1].index
    _steps(sc, dw, 1)
    for n in (40, 10):
        labels = _steps(sc, dw, n)
        rows = dw.download_contacts(dw.counters().contactCount + 64)
        touching = rows["pointCount"] > 0
        on = np.concatenate([rows["bodyB"][touching & (rows["bodyA"] == container)],
                             rows["bodyA"][touching & (rows["bodyB"] == container)]])
        assert len(on) > 48, "the container should be a hub"
        assert (labels[on] == labels[container]).all() and labels[container] == container
    sc.destroy()
