"""Scenes of tests/test_pair_edges_gpu.py, each built to drive the device's pair search (csrc/device/broadphase.cu) onto
one of its capacity edges, and a brute-force restatement of the pair table. The CPU companion
tests/test_pair_edges_cpu.py checks on the reference's own tables, without a GPU, that the restatement equals the
reference's pair table and that every scene reaches its edge.

The edges (DESIGN.md §3.3):

* the candidate-pair buffer: a search that finds more new pairs than the buffer holds is run again with a larger one,
  in the synchronous loop and when the search was started behind the previous step (S2B_PAIR_BUFFER sets the initial
  capacity; the default is 8 per shape slot + 1024, taken once, on the first pass);
* the large-mover route: with at least 256 leaves, a moved proxy whose fat box covers more than 1/256 of the root box
  is tested against every leaf instead of walking the hierarchy, at most 64 of them (S2B_MAX_LARGE_MOVERS);
* the contact table emptying and refilling, and the pair-key hash crossing a power of two (>= 1024 slots and
  >= 2 x contacts: 512 contacts fit 1024 slots, 513 need 2048);
* fat boxes that touch exactly (the overlap test is closed) and a neighbour one float32 ulp away;
* the large-mover decision on the fused path (previous refit's root box) and the unfused one (the pass's own);
* the radix tree's height over degenerate Morton inputs, restated in float32 (tree_height);
* rebuilds mixed with refits, and finalize refits that no search takes over.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import ref as refmod
from solver2d_b200 import capi, scenes

DT = 1.0 / 60.0
MAX_LARGE_MOVERS = 64   # S2B_MAX_LARGE_MOVERS
LARGE_MIN_LEAVES = 256  # fewer leaves: every moved proxy walks the hierarchy
SEGMENT = 3             # shape type of a segment (reference s2ShapeType)


def _overlap_pairs(fat):
    """Unordered index pairs (i < j) of the boxes `fat` (n, 4: min x, min y, max x, max y) that overlap under the closed
    test of s2AABB_Overlaps: a sweep and prune along x in numpy."""
    n = len(fat)
    if n < 2:
        return np.zeros((0, 2), np.int64)
    order = np.argsort(fat[:, 0], kind="stable")
    x0 = fat[order, 0]
    # candidates of the k-th box in sweep order: the boxes after it that start at or before its end
    end = np.searchsorted(x0, fat[order, 2], side="right")
    counts = np.maximum(end - np.arange(n) - 1, 0)
    a = np.repeat(np.arange(n), counts)
    first = np.cumsum(counts) - counts
    b = a + 1 + np.arange(len(a)) - np.repeat(first, counts)
    a, b = order[a], order[b]
    keep = (fat[b, 0] <= fat[a, 2]) & (fat[a, 0] <= fat[b, 2]) & (fat[b, 1] <= fat[a, 3]) & (fat[a, 1] <= fat[b, 3])
    a, b = a[keep], b[keep]
    return np.stack([np.minimum(a, b), np.maximum(a, b)], axis=1)


def brute_pairs(fat, body, body_type, filter=None, shape_type=None, joint_pairs=()):
    """The shape pairs the pair table must hold, as a set of (lower shape slot, higher shape slot).

    `fat`: (n, 4) float32 fat boxes by shape slot; `body`: body slot of every shape slot, < 0 for a free slot;
    `body_type`: body type by body slot (capi.STATIC_BODY ...); `filter`: (n, 3) category bits, mask bits, group index
    by shape slot (None: the default filter); `shape_type`: reference shape type by shape slot (None: no segments);
    `joint_pairs`: body pairs joined by a joint with collideConnected == false.

    A pair is kept when the fat boxes overlap (closed test), the shapes are on different bodies, at least one body is
    dynamic, s2ShouldShapesCollide passes (group, then category / mask), no such joint joins the bodies and the pair is
    not segment against segment.

    This is the reference's pair table only while no static shape was created over a shape that does not move: the
    reference buffers no move for a new static proxy (reference src/broad_phase.c:94-104), so such an overlap never
    becomes a pair there. The scenes here never do that."""
    fat = np.asarray(fat, np.float32)
    body = np.asarray(body, np.int64)
    live = np.nonzero(body >= 0)[0]
    p = _overlap_pairs(fat[live])
    a, b = live[p[:, 0]], live[p[:, 1]]
    btype = np.asarray(body_type)
    keep = body[a] != body[b]
    keep &= (btype[body[a]] == capi.DYNAMIC_BODY) | (btype[body[b]] == capi.DYNAMIC_BODY)
    if filter is not None:
        f = np.asarray(filter, np.int64)
        cat, mask, group = f[:, 0] & 0xFFFFFFFF, f[:, 1] & 0xFFFFFFFF, f[:, 2]
        same = (group[a] == group[b]) & (group[a] != 0)
        bits = ((mask[a] & cat[b]) != 0) & ((cat[a] & mask[b]) != 0)
        keep &= np.where(same, group[a] > 0, bits)
    if shape_type is not None:
        t = np.asarray(shape_type)
        keep &= ~((t[a] == SEGMENT) & (t[b] == SEGMENT))
    blocked = {(min(x, y), max(x, y)) for x, y in joint_pairs}
    out = set()
    for x, y, ok in zip(a.tolist(), b.tolist(), keep.tolist()):
        if ok and (min(body[x], body[y]), max(body[x], body[y])) not in blocked:
            out.add((x, y))
    return out


def ref_pairs(R, wid):
    """(brute-force pairs over the reference's fat boxes, the reference's contact table as a key set)."""
    sf, si = R.shapes(wid)
    _, bi = R.bodies(wid)
    I = refmod.SHAPE_I
    body = np.where(si[:, I["valid"]] == 1, si[:, I["body"]], -1)
    want = brute_pairs(sf[:, 4:8], body, bi[:, refmod.BODY_I["type"]], None, si[:, I["type"]])
    _, ci = R.contacts(wid)
    live = ci[:, 0] == 1
    a, b = ci[live, 1], ci[live, 2]
    got = set(zip(np.minimum(a, b).tolist(), np.maximum(a, b).tolist()))
    return want, got


def device_fat(dw):
    """(fat boxes, live flags) of every device shape slot."""
    _, fat, flags = dw.download_shape_boxes(dw.counters().shapeCapacity)
    return fat, (flags & 1) == 1


def device_pairs(lib, sc, dw, fat):
    """(brute-force pairs over `fat`, the device's contact table as a key set). `fat` are the device's fat boxes the
    step's pair pass saw: those its finalize left the step before, or those uploaded since (device_fat). Bodies and
    their types come through the public API (s2Shape_GetBody, s2Body_GetType)."""
    shapes = sc.piles["shapes"]
    n = max(s.index for s, _ in shapes) + 1
    body = np.full(len(fat), -1, np.int64)
    shape_type = np.zeros(len(fat), np.int64)
    types = {}
    for sid, kind in shapes:
        bid = lib.s2Shape_GetBody(sid)
        body[sid.index] = bid.index
        types[bid.index] = lib.s2Body_GetType(bid)
        shape_type[sid.index] = kind
    btype = np.zeros(max(types) + 1, np.int64)
    for k, t in types.items():
        btype[k] = t
    assert n <= len(fat)
    want = brute_pairs(fat, body, btype, None, shape_type)
    rows = dw.download_contacts(dw.counters().contactCount)
    got = set(zip(np.minimum(rows["shapeA"], rows["shapeB"]).tolist(), np.maximum(rows["shapeA"], rows["shapeB"]).tolist()))
    return want, got


def large_movers(fat, body, moved, root=None):
    """How many moved proxies take the large-mover route (uncapped), restated from the fat boxes in float32 as
    s2bCollectMovers decides it; `root` defaults to the union of every live fat box (the refit's root box)."""
    fat = np.asarray(fat, np.float32)
    live = np.asarray(body) >= 0
    if int(live.sum()) < LARGE_MIN_LEAVES:
        return 0
    if root is None:
        root = root_box(fat, body)
    f32 = np.float32
    area = (fat[:, 2] - fat[:, 0]).astype(f32) * (fat[:, 3] - fat[:, 1]).astype(f32)
    scene = f32(f32(root[2] - root[0]) * f32(root[3] - root[1]))
    return int((live & moved & (area * f32(256.0) > scene)).sum())


def root_box(fat, body):
    live = np.asarray(body) >= 0
    f = np.asarray(fat, np.float32)[live]
    return np.array([f[:, 0].min(), f[:, 1].min(), f[:, 2].max(), f[:, 3].max()], np.float32)


def expand_bits(v):
    v = np.asarray(v, np.uint64) & np.uint64(0xFFFF)
    for shift, mask in ((8, 0x00FF00FF), (4, 0x0F0F0F0F), (2, 0x33333333), (1, 0x55555555)):
        v = (v | (v << np.uint64(shift))) & np.uint64(mask)
    return v


def morton_codes(fat):
    """The 31-bit Morton code of every box, in float32 as s2bMortonCodes computes it (the device build uses
    -fmad=false -prec-div=true -ftz=false): box centres, scene bounds of the centres, a zero-width axis clamped to 1e-6,
    16-bit quantisation."""
    f32 = np.float32
    fat = np.asarray(fat, f32)
    cx = f32(0.5) * (fat[:, 0] + fat[:, 2])
    cy = f32(0.5) * (fat[:, 1] + fat[:, 3])
    minx, maxx, miny, maxy = cx.min(), cx.max(), cy.min(), cy.max()
    ex = max(f32(maxx - minx), f32(1.0e-6))
    ey = max(f32(maxy - miny), f32(1.0e-6))
    ux = np.clip((cx - minx) / ex, f32(0.0), f32(1.0)).astype(f32)
    uy = np.clip((cy - miny) / ey, f32(0.0), f32(1.0)).astype(f32)
    qx = (ux * f32(32767.0)).astype(np.uint64)
    qy = (uy * f32(32767.0)).astype(np.uint64)
    return (expand_bits(qx) | (expand_bits(qy) << np.uint64(1))) & np.uint64(0x7FFFFFFF)


def tree_height(codes):
    """Height of the binary radix tree the device builds over `codes` (leaf order): leaves sorted stably by code (cub's
    radix sort), keys (code, sorted position) of 63 bits, every internal node split on the highest bit in which its
    range's first and last keys differ. The root is at depth 0; the height is the depth of the deepest leaf."""
    codes = np.asarray(codes, np.uint64)
    order = np.argsort(codes, kind="stable")
    keys = [(int(c) << 32) | k for k, c in enumerate(codes[order])]

    def height(lo, hi):
        if hi - lo == 1:
            return 0
        bit = (keys[lo] ^ keys[hi - 1]).bit_length() - 1
        split = next(i for i in range(lo + 1, hi) if (keys[i] >> bit) & 1)
        return 1 + max(height(lo, split), height(split, hi))

    return height(0, len(keys))


def restated_height(fat, valid):
    """treeHeight of a hierarchy built over the live shapes' fat boxes (leaves in shape-slot order)."""
    return tree_height(morton_codes(np.asarray(fat, np.float32)[np.asarray(valid, bool)]))


# ---------------------------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------------------------

POLYGON, CIRCLE = 2, 1  # reference shape types


def _world(lib, solver, name):
    sc = scenes.Scene(lib, lib.create_world(solver), name=name)
    sc.piles["shapes"] = []
    return sc


def _body(lib, sc, kind, x, y, vx=0.0, vy=0.0, gravity=1.0):
    bd = scenes.default_body_def()
    bd.type = kind
    bd.position = capi.Vec2(x, y)
    bd.linearVelocity = capi.Vec2(vx, vy)
    bd.gravityScale = gravity
    bid = lib.s2CreateBody(sc.world, C.byref(bd))
    sc.bodies.append(bid)
    return bid


def _box(lib, sc, kind, x, y, hx=0.5, hy=0.5, **kw):
    bid = _body(lib, sc, kind, x, y, **kw)
    sd = scenes.default_shape_def()
    sd.density = 1.0
    sid = lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(lib.s2MakeBox(hx, hy)))
    sc.piles["shapes"].append((sid, POLYGON))
    return bid


def _circle(lib, sc, x, y, r, **kw):
    bid = _body(lib, sc, capi.DYNAMIC_BODY, x, y, **kw)
    sd = scenes.default_shape_def()
    sd.density = 1.0
    circle = capi.Circle(capi.Vec2(0.0, 0.0), r)
    sid = lib.s2CreateCircleShape(bid, C.byref(sd), C.byref(circle))
    sc.piles["shapes"].append((sid, CIRCLE))
    return bid


def _slider(lib, sc, x=-60.0, y=60.0):
    """A weightless box sliding at 9 m/s through empty space: its proxy leaves its fat box every step, so a pair pass runs
    every step (and one is started behind every step) whatever the rest of the scene does."""
    _box(lib, sc, capi.DYNAMIC_BODY, x, y, vx=9.0, gravity=0.0)


def _ground(lib, sc, half_width):
    _box(lib, sc, capi.STATIC_BODY, 0.0, -1.0, half_width, 1.0)


def lattice_burst(lib, solver, rows=30, cols=50):
    """A ground and the slider; lattice_burst_create adds rows x cols unit boxes in a touching lattice in one go."""
    sc = _world(lib, solver, "lattice_burst")
    _ground(lib, sc, 40.0)
    _slider(lib, sc)
    return sc


def lattice_burst_create(lib, sc, rows=30, cols=50):
    for i in range(rows):
        for j in range(cols):
            _box(lib, sc, capi.DYNAMIC_BODY, 1.02 * j - 0.51 * cols, 0.5 + 1.0 * i)


LATTICE_STEP = 3  # the lattice is created before this step


def interleaving_clouds(lib, solver, lanes=12, per_lane=12):
    """Two clouds of weightless circles (radius 0.25) in lanes 2 m apart, 2 m apart along a lane, moving at 9 m/s against
    each other; cloud B's lanes sit 0.6 m above cloud A's and its circles start half-way between A's. Inside a cloud no
    fat boxes meet; the clouds' circles never touch (0.6 m > 0.5 m), but their fat boxes meet lane by lane, and every
    column of one cloud lines up with a column of the other on the same step: bursts of new pairs, a step apart, with no
    upload in between."""
    sc = _world(lib, solver, "interleaving_clouds")
    _slider(lib, sc)
    for k in range(lanes):
        for i in range(per_lane):
            _circle(lib, sc, 2.0 * i, 2.0 * k, 0.25, vx=9.0, gravity=0.0)
            _circle(lib, sc, 2.0 * i + 1.0, 2.0 * k + 0.6, 0.25, vx=-9.0, gravity=0.0)
    return sc


CLOUD_BUFFER = 64  # S2B_PAIR_BUFFER of the interleaving clouds


def large_glide(lib, solver, large=65, bed=300):
    """`large` weightless boxes of half-extent 1.5, 3.2 m apart, gliding at 9 m/s 0.1 m above a row of `bed` static
    boxes (half-extent 0.25, 0.7 m apart). Each large box's fat box covers more than 1/256 of the root box, and each
    leaves its fat box on every step, so every pass has `large` large movers; each one's fat box always overlaps static
    boxes (which never query), so a large mover whose query is lost loses pairs on the first pass and whenever it
    reaches a new static box."""
    sc = _world(lib, solver, f"large_glide{large}")
    for k in range(bed):
        _box(lib, sc, capi.STATIC_BODY, -105.0 + 0.7 * k, 0.0, 0.25, 0.25)
    for k in range(large):
        _box(lib, sc, capi.DYNAMIC_BODY, -104.0 + 3.2 * k, 1.85, 1.5, 1.5, vx=9.0, gravity=0.0)
    return sc


def one_big(lib, solver, leaves=256):
    """`leaves` shapes in all: a ground, one box big enough to be a large mover and small boxes on the ground."""
    sc = _world(lib, solver, f"one_big{leaves}")
    _ground(lib, sc, 20.0)
    _box(lib, sc, capi.DYNAMIC_BODY, 0.0, 8.0, 4.0, 4.0)
    for k in range(leaves - 2):
        _box(lib, sc, capi.DYNAMIC_BODY, -19.0 + 0.6 * (k % 64), 0.25 + 0.6 * (k // 64), 0.25, 0.25)
    return sc


TOUCH_A = (-1.28, -1.28)
TOUCH_B = (0.0, -1.28)              # fat box touches A's along A's right edge
TOUCH_D = (0.0, 0.0)                # touches A's at A's upper right corner
TOUCH_C = (-1.28, 2.0 ** -24)       # one float32 ulp above A's fat box


def exact_touch(lib, solver):
    """Weightless unit boxes at rest whose fat boxes (made at creation: box +- 0.02 + 0.12) touch exactly in float32:
    B along A's edge, D at A's corner (and at B's and C's edges); C sits one ulp of 0.64 above A and never pairs with
    it. Nothing touches, so nothing moves; the slider keeps a pass (and the survivor scan) running every step."""
    sc = _world(lib, solver, "exact_touch")
    _slider(lib, sc)
    for x, y in (TOUCH_A, TOUCH_B, TOUCH_C, TOUCH_D):
        _box(lib, sc, capi.DYNAMIC_BODY, x, y, gravity=0.0)
    return sc


def launched_row(lib, solver, count=16):
    """`count` boxes resting 2 m apart on a ground; launched_row_launch throws them up until every fat box is clear of
    the ground, and they fall back."""
    sc = _world(lib, solver, "launched_row")
    _ground(lib, sc, 20.0)
    for k in range(count):
        _box(lib, sc, capi.DYNAMIC_BODY, -16.0 + 2.0 * k, 0.5)
    return sc


LAUNCH_STEP = 4


def launched_row_launch(lib, sc):
    for bid in sc.bodies[1:]:
        lib.s2Body_SetLinearVelocity(bid, capi.Vec2(0.0, 5.0))


def ground_row(lib, solver, count=512):
    """`count` boxes resting 1.5 m apart on a ground (exactly `count` contacts) and the slider."""
    sc = _world(lib, solver, f"ground_row{count}")
    _ground(lib, sc, 0.75 * count + 4.0)
    _slider(lib, sc)
    for k in range(count):
        _box(lib, sc, capi.DYNAMIC_BODY, -0.75 * count + 1.5 * k, 0.5)
    return sc


def root_flip(lib, solver):
    """A weightless box of half-extent 1 sliding at 9 m/s 0.1 m above a row of 300 small boxes resting on a 160 m ground
    (its fat box meets theirs), and a weightless marker thrown straight up at 30 m/s far to the side. The marker raises
    the root box every step; the slider leaves its fat box every step. On ROOT_FLIP_STEP the slider is a large mover
    under the root box of the pass before (which the fused path uses) and not under the pass's own (which the unfused
    search uses)."""
    sc = _world(lib, solver, "root_flip")
    _ground(lib, sc, 80.0)
    for k in range(300):
        _box(lib, sc, capi.DYNAMIC_BODY, -75.0 + 0.5 * k, 0.2, 0.2, 0.2)
    _box(lib, sc, capi.DYNAMIC_BODY, -70.0, 1.5, 1.0, 1.0, vx=9.0, gravity=0.0)
    _box(lib, sc, capi.DYNAMIC_BODY, 78.0, 3.0, vy=30.0, gravity=0.0)
    return sc


def line_row(lib, solver, count=300):
    """`count` weightless boxes on one horizontal line, 1.1 m apart, all moving at 9 m/s: every centre has the same y, so
    the Morton build clamps the zero-height scene axis to 1e-6."""
    sc = _world(lib, solver, "line_row")
    for k in range(count):
        _box(lib, sc, capi.DYNAMIC_BODY, 1.1 * k, 0.0, vx=9.0, gravity=0.0)
    return sc


def far_pile(lib, solver):
    """A ground and three rows of boxes dropped onto it about 1e4 m from the origin, and the slider beside them."""
    sc = _world(lib, solver, "far_pile")
    _box(lib, sc, capi.STATIC_BODY, 1.0e4, 1.0e4 - 1.0, 20.0, 1.0)
    for k in range(60):
        _box(lib, sc, capi.DYNAMIC_BODY, 1.0e4 - 15.0 + 1.5 * (k % 20) + 0.25 * (k // 20), 1.0e4 + 0.6 + 1.2 * (k // 20))
    _slider(lib, sc, 1.0e4 - 40.0, 1.0e4 + 30.0)
    return sc


def cluster(lib, solver, depth=40):
    """Kinematic boxes moving together at 1 m/s on a staircase that halves its distance to one point in x, then in y
    (x = 32 * 2^-ceil(k/2), y = 8 * 2^-floor(k/2) from it), the lowest 0.1 m above a row of boxes on a ground: the
    centres crowd geometrically, and once the steps fall below the Morton quantum the deepest boxes share a code."""
    sc = _world(lib, solver, "cluster")
    _ground(lib, sc, 40.0)
    for k in range(depth):
        _box(lib, sc, capi.KINEMATIC_BODY, -10.0 + 32.0 * 2.0 ** -((k + 1) // 2), 1.6 + 8.0 * 2.0 ** -(k // 2), vx=1.0)
    for k in range(40):
        _box(lib, sc, capi.DYNAMIC_BODY, -20.0 + 1.5 * k, 0.5)
    return sc


ROOT_FLIP_STEP = 5  # root_flip: the previous root makes the slider a large mover, the pass's own root does not

CADENCE_PERIOD = 6  # the cadence slider moves for half of every period and stands for the other half


def cadence_toggle(lib, sc, step):
    """Stop the slider at the start of every period, start it half-way: passes run on half of the steps, and the
    finalize refits of the still steps are never taken up."""
    slider = sc.bodies[1]
    if step % CADENCE_PERIOD == 0:
        lib.s2Body_SetLinearVelocity(slider, capi.Vec2(0.0, 0.0))
    elif step % CADENCE_PERIOD == CADENCE_PERIOD // 2:
        lib.s2Body_SetLinearVelocity(slider, capi.Vec2(9.0, 0.0))


def before_step_for(name):
    """Public-API calls a scene makes between steps, as _run's before_step hook (None: none)."""
    if name == "lattice_burst":
        def hook(step, worlds):
            if step == LATTICE_STEP:
                for lib, sc in worlds:
                    lattice_burst_create(lib, sc)
        return hook
    if name == "cadence":
        def hook(step, worlds):
            if step % CADENCE_PERIOD in (0, CADENCE_PERIOD // 2):
                for lib, sc in worlds:
                    cadence_toggle(lib, sc, step)
        return hook
    if name == "launched_row":
        def hook(step, worlds):
            if step == LAUNCH_STEP:
                for lib, sc in worlds:
                    launched_row_launch(lib, sc)
        return hook
    return None


# name -> (builder, steps)
SCENES = {
    "lattice_burst": (lattice_burst, 8),
    "interleaving_clouds": (interleaving_clouds, 24),
    "large_glide64": (lambda L, s: large_glide(L, s, large=64), 12),
    "large_glide65": (lambda L, s: large_glide(L, s, large=65), 12),
    "root_flip": (root_flip, 14),
    "line_row": (line_row, 6),
    "far_pile": (far_pile, 6),
    "cluster": (cluster, 6),
    "cadence": (lambda L, s: ground_row(L, s, 64), 60),
    "one_big255": (lambda L, s: one_big(L, s, leaves=255), 6),
    "one_big256": (lambda L, s: one_big(L, s, leaves=256), 6),
    "exact_touch": (exact_touch, 20),
    "launched_row": (launched_row, 80),
    "ground_row512": (lambda L, s: ground_row(L, s, 512), 4),
    "ground_row513": (lambda L, s: ground_row(L, s, 513), 4),
}
