"""Headless scene recipes, written only against the public C API (so they run on either library, see capi.py).

Each recipe restates one of the reference's sample scenes or one of the synthetic configs of SURVEY.md §8(d):

* :func:`pyramid`         — ``Pyramid`` (reference samples/collection/sample_contact.cpp:499-561), ground widened
                            for baseCount > 200 (SURVEY §8d config 2 / headline).
* :func:`vertical_stack`  — small stack of boxes (quick contact test).
* :func:`bridge`          — ``Bridge`` (reference samples/collection/sample_joints.cpp:15-90).
* :func:`joint_contact_stress` — config 4: stacked bridges + a grid of boxes dropped on them.
* :func:`tumbler`         — config 3: motorised hollow container with a grid of small boxes.
* :func:`mixed_shapes`    — circles/capsules/polygons/segments on a ground, exercising all nine manifold functions.
* :func:`collision_zoo`   — every manifold kind, flipped pairs, dynamic segments, compound bodies, mixed frictions and
                            shape filters, thrown sideways.
* :func:`bouncers`        — shapes with restitution dropped from several heights (the restitution extension).
* :func:`welded_structures` — cantilevers, welded assemblies, a welded platform rider and a chain (the weld joint).
* :func:`sliders`         — pistons, an elevator, an inclined slider, a kinematic carriage, a slider-crank and a mouse
                            joint on a slider (the prismatic joint).
* :func:`kinematic_rigs`  — piles on sliding kinematic platforms and a turntable, joints hanging from moving kinematic
                            carriages (kinematic bodies under every solver variant).

All scenes are deterministic lattices (no RNG). A recipe returns a :class:`Scene` holding the world id and the
body ids in creation order.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, field

from . import capi
from .capi import (BodyId, Capsule, Circle, Segment, Vec2, default_body_def, default_mouse_def, default_revolute_def,
                   default_shape_def)


@dataclass
class Scene:
    lib: capi.Solver2D
    world: capi.WorldId
    bodies: list = field(default_factory=list)
    joints: list = field(default_factory=list)
    name: str = ""
    piles: dict = field(default_factory=dict)

    def step(self, dt=1.0 / 60.0, vel_iters=4, pos_iters=2, warm_start=True):
        self.lib.s2World_Step(self.world, dt, vel_iters, pos_iters, warm_start)

    def destroy(self):
        self.lib.s2DestroyWorld(self.world)


def _ground(lib, world, half_width, half_height=1.0, y=-1.0, restitution=0.0):
    bd = default_body_def()
    bd.position = Vec2(0.0, y)
    gid = lib.s2CreateBody(world, C.byref(bd))
    box = lib.s2MakeBox(half_width, half_height)
    sd = default_shape_def()
    sd.restitution = restitution
    lib.s2CreatePolygonShape(gid, C.byref(sd), C.byref(box))
    return gid


def pyramid(lib: capi.Solver2D, solver="TGS_Soft", base_count=10, restitution=0.0) -> Scene:
    """Pyramid recipe, reference samples/collection/sample_contact.cpp:511-552.

    The reference ground is ``s2MakeBox(100, 1)``; for base_count > 200 the ground half-width is widened to
    ``0.5*N + 50`` so the base row still rests on it (SURVEY §8d config 2). ``restitution`` is given to every shape (the
    sample's 0 by default).
    """
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"pyramid{base_count}")
    half_width = 100.0 if base_count <= 200 else 0.5 * base_count + 50.0
    sc.bodies.append(_ground(lib, world, half_width, restitution=restitution))

    bd = default_body_def()
    bd.type = capi.DYNAMIC_BODY
    sd = default_shape_def()
    sd.density = 1.0
    sd.restitution = restitution
    h = 0.5
    box = lib.s2MakeSquare(h)
    shift = 1.0 * h
    for i in range(base_count):
        # all terms are exactly representable in float32, so Python floats reproduce the sample's float math
        y = (2.0 * i + 1.0) * shift
        for j in range(i, base_count):
            x = (i + 1.0) * shift + 2.0 * (j - i) * shift - h * base_count
            bd.position = Vec2(x, y)
            bid = lib.s2CreateBody(world, C.byref(bd))
            lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
            sc.bodies.append(bid)
    return sc


def vertical_stack(lib, solver="TGS_Soft", count=8, columns=1) -> Scene:
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"stack{count}x{columns}")
    sc.bodies.append(_ground(lib, world, 40.0))
    bd = default_body_def()
    bd.type = capi.DYNAMIC_BODY
    sd = default_shape_def()
    box = lib.s2MakeSquare(0.5)
    for c in range(columns):
        for i in range(count):
            bd.position = Vec2(-2.0 * (columns - 1) + 4.0 * c, 0.5 + 1.0 * i)
            bid = lib.s2CreateBody(world, C.byref(bd))
            lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
            sc.bodies.append(bid)
    return sc


def _add_bridge(lib, sc, ground_id, count, xbase, y):
    box = lib.s2MakeBox(0.5, 0.125)
    sd = default_shape_def()
    sd.density = 20.0
    jd = default_revolute_def()
    jd.drawSize = 0.1
    prev = ground_id
    for i in range(count):
        bd = default_body_def()
        bd.type = capi.DYNAMIC_BODY
        bd.position = Vec2(xbase + 0.5 + 1.0 * i, y)
        bd.linearDamping = 0.1
        bd.angularDamping = 0.1
        bid = lib.s2CreateBody(sc.world, C.byref(bd))
        lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
        sc.bodies.append(bid)
        pivot = Vec2(xbase + 1.0 * i, y)
        jd.bodyIdA = prev
        jd.bodyIdB = bid
        jd.localAnchorA = lib.s2Body_GetLocalPoint(prev, pivot)
        jd.localAnchorB = lib.s2Body_GetLocalPoint(bid, pivot)
        sc.joints.append(lib.s2CreateRevoluteJoint(sc.world, C.byref(jd)))
        prev = bid
    pivot = Vec2(xbase + 1.0 * count, y)
    jd.bodyIdA = prev
    jd.bodyIdB = ground_id
    jd.localAnchorA = lib.s2Body_GetLocalPoint(prev, pivot)
    jd.localAnchorB = lib.s2Body_GetLocalPoint(ground_id, pivot)
    sc.joints.append(lib.s2CreateRevoluteJoint(sc.world, C.byref(jd)))


def bridge(lib, solver="TGS_Soft", count=160) -> Scene:
    """Bridge recipe, reference samples/collection/sample_joints.cpp:39-80."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"bridge{count}")
    bd = default_body_def()
    gid = lib.s2CreateBody(world, C.byref(bd))
    sc.bodies.append(gid)
    _add_bridge(lib, sc, gid, count, -0.5 * count, 20.0)
    return sc


def joint_contact_stress(lib, solver="TGS_Soft", bridges=25, planks=160, grid=73) -> Scene:
    """SURVEY §8d config 4: ``bridges`` suspension bridges stacked 4 m apart plus a grid x grid lattice of boxes
    dropped from above (≈4k revolute joints, ≈16k contacts in steady state at the defaults)."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"jointstress{bridges}x{planks}")
    gid = _ground(lib, world, 0.5 * planks + 50.0)
    sc.bodies.append(gid)
    for b in range(bridges):
        _add_bridge(lib, sc, gid, planks, -0.5 * planks, 4.0 + 4.0 * b)
    bd = default_body_def()
    bd.type = capi.DYNAMIC_BODY
    sd = default_shape_def()
    box = lib.s2MakeSquare(0.25)
    top = 4.0 + 4.0 * bridges
    pitch = 0.75
    for i in range(grid):
        for j in range(grid):
            bd.position = Vec2((j - 0.5 * (grid - 1)) * pitch, top + 1.0 + i * pitch)
            bid = lib.s2CreateBody(world, C.byref(bd))
            lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
            sc.bodies.append(bid)
    return sc


def tumbler(lib, solver="TGS_Soft", grid=100, half_extent=30.0) -> Scene:
    """SURVEY §8d config 3: hollow motorised container (four offset-box walls on one dynamic body, pattern of
    reference samples/collection/sample_contact.cpp:323-336 and sample_joints.cpp:266-276) holding a grid x grid
    lattice of 0.25 m boxes."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"tumbler{grid}")
    bd = default_body_def()
    gid = lib.s2CreateBody(world, C.byref(bd))
    sc.bodies.append(gid)

    bd = default_body_def()
    bd.type = capi.DYNAMIC_BODY
    bd.position = Vec2(0.0, half_extent)
    cid = lib.s2CreateBody(world, C.byref(bd))
    sc.bodies.append(cid)
    sd = default_shape_def()
    sd.density = 5.0
    t = 0.5
    e = half_extent
    for (hx, hy, cx, cy) in ((t, e, e, 0.0), (t, e, -e, 0.0), (e, t, 0.0, e), (e, t, 0.0, -e)):
        wall = lib.s2MakeOffsetBox(hx, hy, Vec2(cx, cy), 0.0)
        lib.s2CreatePolygonShape(cid, C.byref(sd), C.byref(wall))

    jd = default_revolute_def()
    jd.bodyIdA = gid
    jd.bodyIdB = cid
    jd.localAnchorA = Vec2(0.0, half_extent)
    jd.localAnchorB = Vec2(0.0, 0.0)
    jd.enableMotor = True
    jd.motorSpeed = 0.05 * math.pi
    jd.maxMotorTorque = 1.0e8
    sc.joints.append(lib.s2CreateRevoluteJoint(world, C.byref(jd)))

    bd = default_body_def()
    bd.type = capi.DYNAMIC_BODY
    sd = default_shape_def()
    box = lib.s2MakeSquare(0.125)
    pitch = 0.3
    for i in range(grid):
        for j in range(grid):
            bd.position = Vec2((j - 0.5 * (grid - 1)) * pitch, half_extent + (i - 0.5 * (grid - 1)) * pitch)
            bid = lib.s2CreateBody(world, C.byref(bd))
            lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
            sc.bodies.append(bid)
    return sc


def limited_chains(lib, solver="TGS_Soft", chains=3, links=6) -> Scene:
    """Joint feature coverage: hanging capsule chains whose revolute joints have angle limits (every joint), a motor
    (every other joint), collideConnected on one chain, and a mouse joint dragging the last link of the first chain
    (s2DefaultMouseJointDef pattern of reference samples/sample.cpp). The chains swing into a pile of boxes on the
    ground so that joints and contacts share bodies."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"chains{chains}x{links}")
    gid = _ground(lib, world, 30.0)
    sc.bodies.append(gid)
    sd = default_shape_def()
    sd.density = 2.0
    cap = Capsule(Vec2(-0.4, 0.0), Vec2(0.4, 0.0), 0.12)
    for c in range(chains):
        x0 = -6.0 + 6.0 * c
        y0 = 6.0
        prev = gid
        for i in range(links):
            bd = default_body_def()
            bd.type = capi.DYNAMIC_BODY
            bd.position = Vec2(x0 + 0.5 + 1.0 * i, y0)
            bid = lib.s2CreateBody(world, C.byref(bd))
            lib.s2CreateCapsuleShape(bid, C.byref(sd), C.byref(cap))
            sc.bodies.append(bid)
            jd = default_revolute_def()
            pivot = Vec2(x0 + 1.0 * i, y0)
            jd.bodyIdA = prev
            jd.bodyIdB = bid
            jd.localAnchorA = lib.s2Body_GetLocalPoint(prev, pivot)
            jd.localAnchorB = lib.s2Body_GetLocalPoint(bid, pivot)
            jd.enableLimit = True
            jd.lowerAngle = -0.25 * math.pi if i > 0 else -0.6 * math.pi
            jd.upperAngle = 0.15 * math.pi if i > 0 else 0.1 * math.pi
            if i % 2 == 1:
                jd.enableMotor = True
                jd.motorSpeed = 0.5 if c % 2 == 0 else -0.5
                jd.maxMotorTorque = 30.0
            jd.collideConnected = c == 1
            sc.joints.append(lib.s2CreateRevoluteJoint(world, C.byref(jd)))
            prev = bid
        if c == 0:
            md = default_mouse_def()
            md.bodyIdA = gid
            md.bodyIdB = prev
            md.target = Vec2(x0 + links + 1.0, y0 - 1.0)
            md.hertz = 5.0
            md.dampingRatio = 0.7
            sc.joints.append(lib.s2CreateMouseJoint(world, C.byref(md)))
    bd = default_body_def()
    bd.type = capi.DYNAMIC_BODY
    box = lib.s2MakeSquare(0.3)
    for i in range(4):
        for j in range(10):
            bd.position = Vec2(-8.0 + 1.7 * j + 0.1 * i, 0.35 + 0.65 * i)
            bid = lib.s2CreateBody(world, C.byref(bd))
            lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
            sc.bodies.append(bid)
    return sc


def mixed_shapes(lib, solver="TGS_Soft", rows=6, cols=8) -> Scene:
    """Every shape-pair manifold function of reference src/contact.c:139-154 in one pile: polygons, rounded
    polygons, circles and capsules dropped on a polygon ground bordered by two segment walls."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"mixed{rows}x{cols}")
    gid = _ground(lib, world, 30.0)
    sc.bodies.append(gid)
    sd = default_shape_def()
    for x in (-14.0, 14.0):
        seg = Segment(Vec2(x, 0.0), Vec2(x * 1.2, 12.0))
        lib.s2CreateSegmentShape(gid, C.byref(sd), C.byref(seg))
    bd = default_body_def()
    bd.type = capi.DYNAMIC_BODY
    k = 0
    for i in range(rows):
        for j in range(cols):
            bd.position = Vec2(-10.0 + 2.6 * j + 0.35 * (i % 3), 1.0 + 2.2 * i)
            bd.angle = 0.17 * ((i * cols + j) % 7) - 0.5
            bid = lib.s2CreateBody(world, C.byref(bd))
            kind = k % 4
            if kind == 0:
                box = lib.s2MakeBox(0.6, 0.4)
                lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
            elif kind == 1:
                circle = Circle(Vec2(0.1, 0.0), 0.5)
                lib.s2CreateCircleShape(bid, C.byref(sd), C.byref(circle))
            elif kind == 2:
                cap = Capsule(Vec2(-0.5, 0.0), Vec2(0.5, 0.1), 0.3)
                lib.s2CreateCapsuleShape(bid, C.byref(sd), C.byref(cap))
            else:
                pts = (Vec2 * 5)(Vec2(-0.6, -0.4), Vec2(0.5, -0.5), Vec2(0.8, 0.1), Vec2(0.1, 0.7), Vec2(-0.7, 0.3))
                hull = lib.s2ComputeHull(pts, 5)
                poly = lib.s2MakePolygon(C.byref(hull))
                poly.radius = 0.05 if (k % 8) == 3 else 0.0
                lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(poly))
            sc.bodies.append(bid)
            k += 1
    return sc


def collision_zoo(lib, solver="TGS_Soft", rows=5, cols=7) -> Scene:
    """Every manifold kind, both pair orders, every friction mix and every filter rule in one small scene that keeps
    changing: a static ground (box, two inward-leaning segment walls the bodies reach, a circle bump) under a lattice of
    dynamic circles with offset centres, boxes, 5-8-gons, rounded boxes, capsules, compound bodies (2-3 shapes of
    different kinds, local centre off the origin) and bodies carrying a segment next to a box, thrown sideways and spinning
    so that pairs form and break and manifolds change point count.

    * shape frictions cycle through {0, 0.2, 0.6, 1.0};
    * categories 0x2 and 0x4 exclude each other by mask; column 2 shares a negative group (never collides within it),
      column 4 a positive group of stacked capsules and circles whose masks exclude each other (collides within it all
      the same);
    * each row starts at a different kind, so circles are created before some of the polygons they land on: the pair's
      primary shape (reference src/contact.c:139-154) then has the higher shape index (flipped pairs);
    * the outer columns start just inside the walls and are thrown at them."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"zoo{rows}x{cols}")
    bd = default_body_def()
    bd.position = Vec2(0.0, -1.0)
    gid = lib.s2CreateBody(world, C.byref(bd))
    sc.bodies.append(gid)
    sd = default_shape_def()
    ground = lib.s2MakeBox(12.0, 1.0)
    lib.s2CreatePolygonShape(gid, C.byref(sd), C.byref(ground))
    for x in (-9.0, 9.0):
        wall = Segment(Vec2(x, 1.0), Vec2(0.7 * x, 8.0))
        lib.s2CreateSegmentShape(gid, C.byref(sd), C.byref(wall))
    bump = Circle(Vec2(0.5, 1.2), 0.6)
    lib.s2CreateCircleShape(gid, C.byref(sd), C.byref(bump))

    frictions = (0.0, 0.2, 0.6, 1.0)
    nshape = 0

    def shape_def(col, k):
        nonlocal nshape
        d = default_shape_def()
        d.friction = frictions[nshape % 4]
        nshape += 1
        if k % 9 == 2:
            d.filter = capi.Filter(0x0002, 0xFFFFFFFF & ~0x0004, 0)
        elif k % 9 == 3:
            d.filter = capi.Filter(0x0004, 0xFFFFFFFF, 0)
        if col == 2:
            d.filter = capi.Filter(0x0001, 0xFFFFFFFF, -1)
        elif col == 4:
            d.filter = capi.Filter(0x0008, 0xFFFFFFFF & ~0x0008, 1)
        return d

    for i in range(rows):
        for j in range(cols):
            k = i * cols + j
            bd = default_body_def()
            bd.type = capi.DYNAMIC_BODY
            # the filtered columns start closer together than any shapes could rest: only the filter keeps them apart
            y = 1.0 + (0.95 if j in (2, 4) else 1.4) * i
            if j in (0, cols - 1):  # outer columns just inside the walls, thrown at them
                side = -1.0 if j == 0 else 1.0
                bd.position = Vec2(side * (8.1 - 2.7 * y / 7.0), y)
                bd.linearVelocity = Vec2(3.0 * side, 0.0)
            else:
                bd.position = Vec2(2.0 * (j - 0.5 * (cols - 1)) + 0.3 * (i % 2), y)
                bd.linearVelocity = Vec2(2.5 if i % 2 == 0 else -2.5, 0.5 * (j % 3) - 0.5)
            bd.angle = 0.37 * ((k * 3) % 5) - 0.7
            if j == 4:  # the positive group: level capsules and circles stacked 0.02 m apart, touching from the start
                bd.position = Vec2(bd.position.x, (1.0, 1.6, 2.48, 3.15, 4.03)[i % 5] + 4.0 * (i // 5))
                bd.angle = 0.0
            bd.angularVelocity = 1.5 if k % 2 == 0 else -2.0
            bid = lib.s2CreateBody(world, C.byref(bd))
            sc.bodies.append(bid)
            kind = (j + 3 * i) % 7  # every kind in every row but the positive group's: capsules and circles stacked
            if j == 4:
                kind = (4, 4, 0, 4, 0)[i % 5]
            if kind == 0:
                circle = Circle(Vec2(0.12, -0.05), 0.45)
                lib.s2CreateCircleShape(bid, C.byref(shape_def(j, k)), C.byref(circle))
            elif kind == 1:
                box = lib.s2MakeBox(0.55, 0.35)
                lib.s2CreatePolygonShape(bid, C.byref(shape_def(j, k)), C.byref(box))
            elif kind == 2:
                n = 5 + k % 4
                pts = (Vec2 * n)(*[Vec2(0.55 * math.cos(2.0 * math.pi * (m + 0.1 * (m % 2)) / n),
                                        0.5 * math.sin(2.0 * math.pi * (m + 0.1 * (m % 2)) / n)) for m in range(n)])
                hull = lib.s2ComputeHull(pts, n)
                poly = lib.s2MakePolygon(C.byref(hull))
                lib.s2CreatePolygonShape(bid, C.byref(shape_def(j, k)), C.byref(poly))
            elif kind == 3:
                rounded = lib.s2MakeBox(0.4, 0.25)  # the reference has no s2MakeRoundedBox: a box with the radius set
                rounded.radius = 0.12
                lib.s2CreatePolygonShape(bid, C.byref(shape_def(j, k)), C.byref(rounded))
            elif kind == 4:
                cap = Capsule(Vec2(-0.45, 0.0), Vec2(0.45, 0.08), 0.25)
                lib.s2CreateCapsuleShape(bid, C.byref(shape_def(j, k)), C.byref(cap))
            elif kind == 5:
                box = lib.s2MakeOffsetBox(0.3, 0.25, Vec2(0.35, 0.05), 0.2)
                lib.s2CreatePolygonShape(bid, C.byref(shape_def(j, k)), C.byref(box))
                circle = Circle(Vec2(-0.35, 0.1), 0.28)
                lib.s2CreateCircleShape(bid, C.byref(shape_def(j, k)), C.byref(circle))
                if k % 2 == 0:
                    cap = Capsule(Vec2(-0.2, 0.45), Vec2(0.3, 0.5), 0.12)
                    lib.s2CreateCapsuleShape(bid, C.byref(shape_def(j, k)), C.byref(cap))
            else:
                box = lib.s2MakeOffsetBox(0.4, 0.2, Vec2(0.0, 0.15), 0.0)
                lib.s2CreatePolygonShape(bid, C.byref(shape_def(j, k)), C.byref(box))
                seg = Segment(Vec2(-0.6, -0.2), Vec2(0.6, -0.25))
                lib.s2CreateSegmentShape(bid, C.byref(shape_def(j, k)), C.byref(seg))
    return sc


RECIPES = {
    "pyramid": pyramid,
    "vertical_stack": vertical_stack,
    "bridge": bridge,
    "joint_contact_stress": joint_contact_stress,
    "tumbler": tumbler,
    "mixed_shapes": mixed_shapes,
    "collision_zoo": collision_zoo,
}


BOUNCER_RESTITUTION = (0.0, 0.25, 0.6, 1.0)
# drop heights above the ground (m): impact speeds sqrt(2 g h) of about 0.45, 1.4, 3.2 and 6.3 m/s, on both sides of the
# default 1 m/s restitution threshold
BOUNCER_DROPS = (0.01, 0.1, 0.5, 2.0)


def bouncers(lib: capi.Solver2D, solver="TGS_Soft", columns=16, rows=4, joints=True, platform=True) -> Scene:
    """Restitution coverage. A ground of boxes (restitution 0 and 0.5 alternating) and segments, bordered by two walls; above
    it `rows` x `columns` circles, boxes, capsules and rounded polygons with restitution 0, 0.25, 0.6 and 1, each column
    dropped from one of BOUNCER_DROPS. With `joints`: the three revolute-jointed boxes of restitution 1 of the reference's
    "Ragdoll Stress" sample (samples/collection/sample_joints.cpp:261 sets shapeDef.restitution = 1). With `platform`: a
    kinematic platform moving up and down under the last columns. Shape count ~ columns x rows + columns / 2 + 8."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"bouncers{rows}x{columns}")
    pitch = 1.6
    half = 0.5 * pitch * columns + 4.0
    bd = default_body_def()
    bd.position = Vec2(0.0, -1.0)
    gid = lib.s2CreateBody(world, C.byref(bd))
    sc.bodies.append(gid)
    sd = default_shape_def()
    tiles = max(2, columns // 2)
    tile = 2.0 * half / tiles
    for t in range(tiles):
        sd.restitution = 0.5 if t % 2 == 1 else 0.0
        box = lib.s2MakeOffsetBox(0.5 * tile, 1.0, Vec2(-half + (t + 0.5) * tile, 0.0), 0.0)
        lib.s2CreatePolygonShape(gid, C.byref(sd), C.byref(box))
    sd.restitution = 0.0
    for x in (-half, half):
        lib.s2CreateSegmentShape(gid, C.byref(sd), C.byref(Segment(Vec2(x, 1.0), Vec2(x, 30.0))))
    # a segment strip lying on the ground under the first columns (segment-vs-shape manifolds)
    sd.restitution = 0.5
    lib.s2CreateSegmentShape(gid, C.byref(sd), C.byref(Segment(Vec2(-half + 1.0, 1.0), Vec2(-half + 6.0, 1.0))))

    bd = default_body_def()
    bd.type = capi.DYNAMIC_BODY
    for j in range(columns):
        drop = BOUNCER_DROPS[j % len(BOUNCER_DROPS)]
        for i in range(rows):
            k = i * columns + j
            # each row falls as a layer: lower rows land first, the layers do not start in contact
            bd.position = Vec2(-0.5 * pitch * (columns - 1) + pitch * j, 1.0 + 0.6 + drop + 1.6 * i)
            bd.angle = 0.0
            bid = lib.s2CreateBody(world, C.byref(bd))
            sd.restitution = BOUNCER_RESTITUTION[(j + i) % len(BOUNCER_RESTITUTION)]
            kind = (i + j // 4) % 4
            if kind == 0:
                lib.s2CreateCircleShape(bid, C.byref(sd), C.byref(Circle(Vec2(0.0, 0.0), 0.5)))
            elif kind == 1:
                box = lib.s2MakeBox(0.5, 0.4)
                lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
            elif kind == 2:
                lib.s2CreateCapsuleShape(bid, C.byref(sd), C.byref(Capsule(Vec2(-0.3, 0.0), Vec2(0.3, 0.0), 0.3)))
            else:
                rounded = lib.s2MakeBox(0.4, 0.3)  # a box with the radius set: rounded polygon
                rounded.radius = 0.1
                lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(rounded))
            sc.bodies.append(bid)
    if joints:
        # Ragdoll Stress: boxes joined by revolute joints, every shape with restitution 1
        sd.restitution = 1.0
        prev = None
        box = lib.s2MakeBox(0.5, 0.25)
        x0, y0 = -3.0, 1.0 + 0.6 + 1.6 * rows + 3.0
        for n in range(3):
            bd.position = Vec2(x0 + 1.0 * n, y0)
            bid = lib.s2CreateBody(world, C.byref(bd))
            lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
            sc.bodies.append(bid)
            if prev is not None:
                jd = default_revolute_def()
                pivot = Vec2(x0 + 1.0 * n - 0.5, y0)
                jd.bodyIdA = prev
                jd.bodyIdB = bid
                jd.localAnchorA = lib.s2Body_GetLocalPoint(prev, pivot)
                jd.localAnchorB = lib.s2Body_GetLocalPoint(bid, pivot)
                sc.joints.append(lib.s2CreateRevoluteJoint(world, C.byref(jd)))
            prev = bid
    if platform:
        kd = default_body_def()
        kd.type = capi.KINEMATIC_BODY
        kd.position = Vec2(0.5 * pitch * (columns - 1) - 1.0, 1.0 + 0.6 + 1.6 * rows + 6.0)
        kd.linearVelocity = Vec2(0.0, -1.5)
        pid = lib.s2CreateBody(world, C.byref(kd))
        sd.restitution = 0.6
        box = lib.s2MakeBox(1.5, 0.2)
        lib.s2CreatePolygonShape(pid, C.byref(sd), C.byref(box))
        sc.bodies.append(pid)
        sc.piles["platform"] = pid
    return sc


WELDED_PITCH = 30.0  # width of one copy of welded_structures (m)


def welded_structures(lib: capi.Solver2D, solver="TGS_Soft", copies=1, platform=True) -> Scene:
    """Weld joint coverage, `copies` side by side (about 30 bodies each). Per copy:

    * two cantilever beams of five boxes welded end to end to a static wall; in the second, the boxes alternate between
      angle 0 and 3 rad, so its welds have reference angles of +3 and -3 rad (near +-pi: the unwind is exercised);
    * an L and a T of welded boxes dropped onto a small pile, the L pulled by a mouse joint (first copy only);
    * with `platform`: a dynamic box welded onto a kinematic platform that moves sideways;
    * a hanging chain of three revolute links (limits on the first, a motor on the second) ending in a welded pair, whose
      weld keeps collideConnected.

    On a library without s2CreateWeldJoint (the reference) every weld is created as a revolute joint with limits and
    motor off, with the same bodies, anchors, reference angle and collideConnected: the broad phase treats every joint
    alike, so both libraries see the same pairs. ``sc.piles["welds"]`` lists the indices into ``sc.joints`` of the welds."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"welded{copies}")
    sc.piles["welds"] = []
    has_weld = "s2CreateWeldJoint" not in lib.missing
    gid = _ground(lib, world, 0.5 * WELDED_PITCH * copies + 5.0)
    sc.bodies.append(gid)
    sd = default_shape_def()

    def body(kind, x, y, angle=0.0, hx=0.5, hy=0.125, vx=0.0):
        bd = default_body_def()
        bd.type = kind
        bd.position = Vec2(x, y)
        bd.angle = angle
        bd.linearVelocity = Vec2(vx, 0.0)
        bid = lib.s2CreateBody(world, C.byref(bd))
        box = lib.s2MakeBox(hx, hy)
        lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
        sc.bodies.append(bid)
        return bid

    def weld(a, b, pivot, reference_angle, collide=False):
        if has_weld:
            jd = capi.default_weld_def()
        else:
            jd = default_revolute_def()
        jd.bodyIdA = a
        jd.bodyIdB = b
        jd.localAnchorA = lib.s2Body_GetLocalPoint(a, pivot)
        jd.localAnchorB = lib.s2Body_GetLocalPoint(b, pivot)
        jd.referenceAngle = reference_angle
        jd.collideConnected = collide
        create = lib.s2CreateWeldJoint if has_weld else lib.s2CreateRevoluteJoint
        sc.piles["welds"].append(len(sc.joints))
        sc.joints.append(create(world, C.byref(jd)))

    D, S, K = capi.DYNAMIC_BODY, capi.STATIC_BODY, capi.KINEMATIC_BODY
    for k in range(copies):
        x0 = -0.5 * WELDED_PITCH * (copies - 1) + WELDED_PITCH * k - 12.0
        # cantilevers
        for beam, y in enumerate((6.0, 9.0)):
            wall = body(S, x0, y, hx=0.25, hy=1.0)
            prev, prev_angle = wall, 0.0
            for i in range(5):
                angle = 3.0 if beam == 1 and i % 2 == 0 else 0.0
                bid = body(D, x0 + 0.75 + 1.0 * i, y, angle=angle)
                weld(prev, bid, Vec2(x0 + 0.25 + 1.0 * i, y), angle - prev_angle)
                prev, prev_angle = bid, angle
        # a small pile, an L and a T dropped onto it
        for i in range(3):
            for j in range(2):
                body(D, x0 + 7.0 + 1.05 * i, 0.25 + 0.5 * j, hx=0.5, hy=0.25)
        a = body(D, x0 + 7.5, 3.0)
        b = body(D, x0 + 8.0 - 0.125, 3.0 + 0.375, angle=0.5 * math.pi, hx=0.5, hy=0.125)
        weld(a, b, Vec2(x0 + 8.0 - 0.125, 3.0), 0.5 * math.pi)
        ell = a
        a = body(D, x0 + 8.0, 5.0)
        b = body(D, x0 + 8.0, 5.0 - 0.625, angle=0.5 * math.pi)
        weld(a, b, Vec2(x0 + 8.0, 5.0 - 0.125), 0.5 * math.pi)
        c = body(D, x0 + 8.0, 5.0 + 0.375, hx=0.25, hy=0.25)
        weld(a, c, Vec2(x0 + 8.0, 5.0 + 0.125), 0.0)
        if k == 0:
            md = default_mouse_def()
            md.bodyIdA = gid
            md.bodyIdB = ell
            md.target = Vec2(x0 + 6.0, 4.0)
            md.hertz = 3.0
            md.dampingRatio = 0.7
            sc.joints.append(lib.s2CreateMouseJoint(world, C.byref(md)))
        if platform:
            p = body(K, x0 + 12.0, 2.0, hx=1.0, hy=0.125, vx=0.5)
            q = body(D, x0 + 12.0, 2.0 + 0.375, hx=0.25, hy=0.25)
            weld(p, q, Vec2(x0 + 12.0, 2.0 + 0.125), 0.0)
        # revolute chain ending in a welded pair
        anchor = body(S, x0 + 17.0, 10.0, hx=0.25, hy=0.25)
        prev = anchor
        for i in range(3):
            bid = body(D, x0 + 17.5 + 1.0 * i, 10.0)
            jd = default_revolute_def()
            pivot = Vec2(x0 + 17.0 + 1.0 * i, 10.0)
            jd.bodyIdA = prev
            jd.bodyIdB = bid
            jd.localAnchorA = lib.s2Body_GetLocalPoint(prev, pivot)
            jd.localAnchorB = lib.s2Body_GetLocalPoint(bid, pivot)
            if i == 0:
                jd.enableLimit = True
                jd.lowerAngle = -0.5 * math.pi
                jd.upperAngle = 0.25 * math.pi
            elif i == 1:
                jd.enableMotor = True
                jd.motorSpeed = 0.5
                jd.maxMotorTorque = 5.0
            sc.joints.append(lib.s2CreateRevoluteJoint(world, C.byref(jd)))
            prev = bid
        end = body(D, x0 + 20.75, 10.0, hx=0.25, hy=0.25)
        weld(prev, end, Vec2(x0 + 20.5, 10.0), 0.0, collide=True)
    return sc


SLIDERS_PITCH = 32.0  # width of one copy of sliders (m)


def sliders(lib: capi.Solver2D, solver="TGS_Soft", copies=1, kinematic=True) -> Scene:
    """Prismatic joint coverage, `copies` side by side (about 20 bodies each). Per copy:

    * three pistons on static posts, motors driving boxes up against gravity: one with force to spare, one capped by an
      upper limit, and one whose maxMotorForce (4 N) is below its 10 N load, so it sinks onto the ground;
    * an elevator platform with both limits and a motor, carrying a small pile of boxes;
    * a slider on an axis inclined at 0.5 rad in a body turned by 0.2 rad, with referenceAngle 0.4 - 0.2, thrown along the
      axis into its upper limit and falling back onto its lower one;
    * with `kinematic`: a box sliding on a kinematic body that moves sideways (limits and a weak motor);
    * a slider-crank: a motorised revolute crank on a static hub, a connecting rod, and a piston on a prismatic joint;
    * a horizontal slider with limits, pulled off its axis by a mouse joint (first copy only).

    On a library without s2CreatePrismaticJoint (the reference) every prismatic joint is created as a revolute joint with
    limits and motor off, with the same bodies, anchors, reference angle and collideConnected: the broad phase treats every
    joint alike, so both libraries see the same pairs. ``sc.piles["prismatic"]`` lists the indices into ``sc.joints`` of the
    prismatic joints, ``sc.piles["prismatic_defs"]`` their definitions (dicts of s2PrismaticJointDef fields, the axis as
    given) and ``sc.piles["prismatic_bodies"]`` their (bodyIdA, bodyIdB), so that a test can turn the stand-in rows into
    prismatic rows."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"sliders{copies}")
    sc.piles["prismatic"] = []
    sc.piles["prismatic_defs"] = []
    sc.piles["prismatic_bodies"] = []
    has_prismatic = "s2CreatePrismaticJoint" not in lib.missing
    gid = _ground(lib, world, 0.5 * SLIDERS_PITCH * copies + 5.0)
    sc.bodies.append(gid)
    sd = default_shape_def()

    def body(kind, x, y, angle=0.0, hx=0.5, hy=0.125, vx=0.0, vy=0.0):
        bd = default_body_def()
        bd.type = kind
        bd.position = Vec2(x, y)
        bd.angle = angle
        bd.linearVelocity = Vec2(vx, vy)
        bid = lib.s2CreateBody(world, C.byref(bd))
        box = lib.s2MakeBox(hx, hy)
        lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
        sc.bodies.append(bid)
        return bid

    def prismatic(a, b, pivot, axis, reference_angle=0.0, limit=None, motor=None, collide=False):
        d = dict(localAnchorA=tuple(lib.s2Body_GetLocalPoint(a, pivot)), localAnchorB=tuple(lib.s2Body_GetLocalPoint(b, pivot)),
                 localAxisA=axis, referenceAngle=reference_angle, enableLimit=limit is not None,
                 lowerTranslation=limit[0] if limit else 0.0, upperTranslation=limit[1] if limit else 0.0,
                 enableMotor=motor is not None, motorSpeed=motor[0] if motor else 0.0,
                 maxMotorForce=motor[1] if motor else 0.0, collideConnected=collide)
        if has_prismatic:
            jd = capi.default_prismatic_def()
            for name, value in d.items():
                setattr(jd, name, Vec2(*value) if isinstance(value, tuple) else value)
            create = lib.s2CreatePrismaticJoint
        else:
            jd = default_revolute_def()
            jd.localAnchorA = Vec2(*d["localAnchorA"])
            jd.localAnchorB = Vec2(*d["localAnchorB"])
            jd.referenceAngle = reference_angle
            jd.collideConnected = collide
            create = lib.s2CreateRevoluteJoint
        jd.bodyIdA = a
        jd.bodyIdB = b
        sc.piles["prismatic"].append(len(sc.joints))
        sc.piles["prismatic_defs"].append(d)
        sc.piles["prismatic_bodies"].append((a, b))
        jid = create(world, C.byref(jd))
        sc.joints.append(jid)
        return jid

    def revolute(a, b, pivot, motor=None):
        jd = default_revolute_def()
        jd.bodyIdA = a
        jd.bodyIdB = b
        jd.localAnchorA = lib.s2Body_GetLocalPoint(a, pivot)
        jd.localAnchorB = lib.s2Body_GetLocalPoint(b, pivot)
        if motor is not None:
            jd.enableMotor = True
            jd.motorSpeed, jd.maxMotorTorque = motor
        sc.joints.append(lib.s2CreateRevoluteJoint(world, C.byref(jd)))

    D, S, K = capi.DYNAMIC_BODY, capi.STATIC_BODY, capi.KINEMATIC_BODY
    up = (0.0, 1.0)
    for k in range(copies):
        x0 = -0.5 * SLIDERS_PITCH * (copies - 1) + SLIDERS_PITCH * k - 14.0
        # pistons: 1 kg boxes (10 N) on static posts
        for i, (limit, motor) in enumerate((((-1.0, 3.0), (0.5, 200.0)), ((-1.0, 0.5), (1.0, 200.0)), (None, (0.5, 4.0)))):
            x = x0 + 1.5 * i
            post = body(S, x, 0.25, hx=0.25, hy=0.25)
            load = body(D, x, 1.5, hx=0.5, hy=0.5)
            prismatic(post, load, Vec2(x, 1.5), up, limit=limit, motor=motor)
        # elevator with a small pile
        base = body(S, x0 + 7.0, 0.25, hx=0.25, hy=0.25)
        deck = body(D, x0 + 7.0, 1.5, hx=1.5, hy=0.125)
        prismatic(base, deck, Vec2(x0 + 7.0, 1.5), up, limit=(-1.0, 1.5), motor=(1.0, 100.0))
        for i in range(3):
            body(D, x0 + 6.3 + 0.7 * i, 1.875, hx=0.25, hy=0.25)
        body(D, x0 + 6.65, 2.375, hx=0.25, hy=0.25)
        # inclined slider, thrown into its limits
        frame = body(S, x0 + 11.0, 3.0, angle=0.2, hx=0.25, hy=0.25)
        c, s = math.cos(0.7), math.sin(0.7)  # world direction of the axis: 0.2 + 0.5 rad
        slider = body(D, x0 + 11.0 + c, 3.0 + s, angle=0.4, hx=0.375, hy=0.125, vx=4.0 * c, vy=4.0 * s)
        prismatic(frame, slider, Vec2(x0 + 11.0 + c, 3.0 + s), (2.0 * math.cos(0.5), 2.0 * math.sin(0.5)),
                  reference_angle=0.4 - 0.2, limit=(0.0, 2.0))
        # a box riding a kinematic carriage
        if kinematic:
            carriage = body(K, x0 + 15.0, 2.0, hx=1.0, hy=0.125, vx=0.5)
            rider = body(D, x0 + 15.0, 2.375, hx=0.25, hy=0.25)
            prismatic(carriage, rider, Vec2(x0 + 15.0, 2.375), (1.0, 0.0), limit=(-0.75, 0.75), motor=(0.3, 5.0))
        # slider-crank
        hub = body(S, x0 + 20.0, 3.0, hx=0.1, hy=0.1)
        crank = body(D, x0 + 20.5, 3.0, hx=0.5, hy=0.1)
        revolute(hub, crank, Vec2(x0 + 20.0, 3.0), motor=(2.0, 50.0))
        rod = body(D, x0 + 22.0, 3.0, hx=1.0, hy=0.1)
        revolute(crank, rod, Vec2(x0 + 21.0, 3.0))
        piston = body(D, x0 + 23.0, 3.0, hx=0.25, hy=0.25)
        revolute(rod, piston, Vec2(x0 + 23.0, 3.0))
        prismatic(hub, piston, Vec2(x0 + 23.0, 3.0), (1.0, 0.0))
        # horizontal slider pulled by a mouse joint
        rail = body(S, x0 + 27.0, 1.0, hx=0.25, hy=0.25)
        carriage = body(D, x0 + 27.0, 1.5, hx=0.5, hy=0.125)
        prismatic(rail, carriage, Vec2(x0 + 27.0, 1.5), (1.0, 0.0), limit=(-1.0, 1.0), collide=True)
        if k == 0:
            md = default_mouse_def()
            md.bodyIdA = gid
            md.bodyIdB = carriage
            md.target = Vec2(x0 + 29.0, 2.5)
            md.hertz = 3.0
            md.dampingRatio = 0.7
            sc.joints.append(lib.s2CreateMouseJoint(world, C.byref(md)))
    return sc


KINEMATIC_RIGS_PITCH = 24.0  # width of one platform of kinematic_rigs (m)


def kinematic_rigs(lib: capi.Solver2D, solver="TGS_Soft", platforms=4, base_count=12, prismatic=True, turning=True) -> Scene:
    """Kinematic bodies carrying dynamic ones, `platforms` side by side. Per platform:

    * a kinematic platform sliding sideways (alternate platforms left and right), a pyramid of `base_count` boxes on it;
    * a kinematic carriage above it, moving sideways and turning slowly, with a pendulum on a revolute joint (limits on), a
      slider on a prismatic joint (limits and a weak motor) and a box on a second revolute joint (motor on).
    Beside them a kinematic turntable turning at 0.25 rad/s with a small pyramid on it, and a mouse joint pulling the
    first pendulum.

    With `turning` False the carriages and the turntable keep their angle. On a library without s2CreatePrismaticJoint,
    or with `prismatic` False on either library, each prismatic joint is a
    revolute joint with limits and motor off (the stand-in of :func:`sliders`). ``sc.piles`` holds "kinematic" (the ids of
    the kinematic bodies), "prismatic" / "prismatic_defs" / "prismatic_bodies" as :func:`sliders` does."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"kinematic_rigs{platforms}")
    sc.piles.update(kinematic=[], prismatic=[], prismatic_defs=[], prismatic_bodies=[])
    has_prismatic = prismatic and "s2CreatePrismaticJoint" not in lib.missing
    gid = _ground(lib, world, 0.5 * KINEMATIC_RIGS_PITCH * (platforms + 1) + 5.0, y=-12.0)
    sc.bodies.append(gid)
    sd = default_shape_def()
    sd.density = 1.0
    D, K = capi.DYNAMIC_BODY, capi.KINEMATIC_BODY

    def body(kind, x, y, hx, hy, vx=0.0, w=0.0, angle=0.0):
        bd = default_body_def()
        bd.type = kind
        bd.position = Vec2(x, y)
        bd.angle = angle
        bd.linearVelocity = Vec2(vx, 0.0)
        bd.angularVelocity = w
        bid = lib.s2CreateBody(world, C.byref(bd))
        lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(lib.s2MakeBox(hx, hy)))
        sc.bodies.append(bid)
        if kind == K:
            sc.piles["kinematic"].append(bid)
        return bid

    def pile(x0, y0, base, h=0.5):
        for i in range(base):
            for j in range(i, base):
                body(D, x0 + (i + 1.0) * h + 2.0 * (j - i) * h - h * base, y0 + (2.0 * i + 1.0) * h, h, h)

    def revolute(a, b, pivot, limit=None, motor=None):
        jd = default_revolute_def()
        jd.bodyIdA, jd.bodyIdB = a, b
        jd.localAnchorA = lib.s2Body_GetLocalPoint(a, pivot)
        jd.localAnchorB = lib.s2Body_GetLocalPoint(b, pivot)
        if limit is not None:
            jd.enableLimit = True
            jd.lowerAngle, jd.upperAngle = limit
        if motor is not None:
            jd.enableMotor = True
            jd.motorSpeed, jd.maxMotorTorque = motor
        jid = lib.s2CreateRevoluteJoint(world, C.byref(jd))
        sc.joints.append(jid)
        return jid

    def slider(a, b, pivot, axis, limit, motor):
        d = dict(localAnchorA=tuple(lib.s2Body_GetLocalPoint(a, pivot)), localAnchorB=tuple(lib.s2Body_GetLocalPoint(b, pivot)),
                 localAxisA=axis, referenceAngle=0.0, enableLimit=True, lowerTranslation=limit[0],
                 upperTranslation=limit[1], enableMotor=True, motorSpeed=motor[0], maxMotorForce=motor[1],
                 collideConnected=False)
        if has_prismatic:
            jd = capi.default_prismatic_def()
            for name, value in d.items():
                setattr(jd, name, Vec2(*value) if isinstance(value, tuple) else value)
            create = lib.s2CreatePrismaticJoint
        else:
            jd = default_revolute_def()
            jd.localAnchorA = Vec2(*d["localAnchorA"])
            jd.localAnchorB = Vec2(*d["localAnchorB"])
            create = lib.s2CreateRevoluteJoint
        jd.bodyIdA, jd.bodyIdB = a, b
        sc.piles["prismatic"].append(len(sc.joints))
        sc.piles["prismatic_defs"].append(d)
        sc.piles["prismatic_bodies"].append((a, b))
        sc.joints.append(create(world, C.byref(jd)))

    first = None
    for k in range(platforms):
        x0 = -0.5 * KINEMATIC_RIGS_PITCH * platforms + KINEMATIC_RIGS_PITCH * k
        body(K, x0, -1.0, 0.5 * base_count + 1.5, 0.5, vx=0.6 if k % 2 == 0 else -0.4)
        pile(x0, -0.5, base_count)
        carriage = body(K, x0, base_count + 4.0, 3.0, 0.2, vx=0.5 if k % 2 == 0 else -0.5,
                        w=(0.1 if k % 2 == 0 else -0.1) if turning else 0.0)
        pendulum = body(D, x0 - 2.0, base_count + 2.5, 0.15, 0.75)
        revolute(carriage, pendulum, Vec2(x0 - 2.0, base_count + 3.25), limit=(-0.6, 0.6))
        rider = body(D, x0 + 0.5, base_count + 4.45, 0.25, 0.25)
        slider(carriage, rider, Vec2(x0 + 0.5, base_count + 4.45), (1.0, 0.0), (-1.0, 1.0), (0.4, 3.0))
        crank = body(D, x0 + 2.0, base_count + 3.0, 0.6, 0.1, angle=0.3)
        revolute(carriage, crank, Vec2(x0 + 2.0, base_count + 3.8), motor=(1.5, 20.0))
        first = pendulum if first is None else first
    x0 = 0.5 * KINEMATIC_RIGS_PITCH * platforms + 2.0
    body(K, x0, -1.0, 4.5, 0.5, w=0.25 if turning else 0.0)
    pile(x0, -0.5, 6)
    md = default_mouse_def()
    md.bodyIdA, md.bodyIdB = gid, first
    p = lib.s2Body_GetPosition(first)
    md.target = Vec2(p.x + 1.5, p.y + 0.5)
    md.hertz = 3.0
    md.dampingRatio = 0.7
    sc.joints.append(lib.s2CreateMouseJoint(world, C.byref(md)))
    return sc


def pyramid_rows(base_count: int):
    """The Pyramid recipe (see ``pyramid``) as device rows built with numpy instead of one API call per box: bodies and
    shapes for ``Device.create_world().upload_*``. For worlds too large to author through ctypes in reasonable time
    (the per-colour kernel roofline probe builds 3 M boxes this way). Values are what the host library would produce for
    s2MakeSquare(0.5) boxes of density 1 on a static ground."""
    import numpy as np
    from . import device as dv
    n = base_count
    nb = n * (n + 1) // 2
    i_idx = np.repeat(np.arange(n), n - np.arange(n))
    j_idx = np.concatenate([np.arange(i, n) for i in range(n)])
    h = np.float32(0.5)
    x = ((i_idx + 1) * 0.5 + 2.0 * (j_idx - i_idx) * 0.5 - 0.5 * n).astype(np.float32)
    y = ((2.0 * i_idx + 1.0) * 0.5).astype(np.float32)
    bodies = np.zeros(nb + 1, dtype=dv.BODY_ROW)
    bodies["index"] = np.arange(nb + 1)
    bodies["flags"] = dv.ROW_VALID | (capi.DYNAMIC_BODY << 1)
    bodies["flags"][0] = dv.ROW_VALID | (capi.STATIC_BODY << 1)
    bodies["origin"][1:, 0] = x
    bodies["origin"][1:, 1] = y
    bodies["origin"][0] = (0.0, -1.0)
    bodies["position"] = bodies["origin"]
    bodies["rot"][:, 1] = 1.0
    bodies["mass"][1:] = 1.0
    bodies["invMass"][1:] = 1.0
    bodies["I"][1:] = np.float32(1.0 / 6.0)
    bodies["invI"][1:] = np.float32(6.0)
    bodies["gravityScale"] = 1.0
    shapes = np.zeros(nb + 1, dtype=dv.SHAPE_ROW)
    shapes["index"] = np.arange(nb + 1)
    polygon = 2  # s2_polygonShape
    shapes["flags"] = dv.ROW_VALID | (polygon << 1) | dv.SHAPE_MOVED | 0x20  # + FRESH
    shapes["flags"][0] = dv.ROW_VALID | (polygon << 1) | 0x20
    shapes["body"] = np.arange(nb + 1)
    shapes["proxyKey"] = np.arange(nb + 1)
    shapes["categoryBits"] = 1
    shapes["maskBits"] = 0xFFFFFFFF
    shapes["friction"] = 0.6
    shapes["count"] = 4
    hw = np.full(nb + 1, h, dtype=np.float32)
    hh = np.full(nb + 1, h, dtype=np.float32)
    hw[0] = max(100.0, 0.5 * n + 50.0)
    hh[0] = 1.0
    verts = np.stack([-hw, -hh, hw, -hh, hw, hh, -hw, hh], axis=1)
    shapes["vertices"][:, :8] = verts
    shapes["normals"][:, :8] = np.array([0.0, -1.0, 1.0, 0.0, 0.0, 1.0, -1.0, 0.0], dtype=np.float32)
    cx, cy = bodies["origin"][:, 0], bodies["origin"][:, 1]
    shapes["aabb"] = np.stack([cx - hw, cy - hh, cx + hw, cy + hh], axis=1)
    m = np.float32(0.1)  # s2_aabbMargin
    shapes["fatAABB"] = np.stack([cx - hw - m, cy - hh - m, cx + hw + m, cy + hh + m], axis=1)
    return bodies, shapes


def pyramid_field_interleaved(lib: capi.Solver2D, solver="TGS_Soft", count=12, base_count=8, pitch=None, only=None) -> Scene:
    """The same piles as :func:`pyramid_field`, but created ROUND-ROBIN — body k of every pile before body k + 1 of any — so
    that the islands are thoroughly interleaved in every pool and table (slots, proxy ids, contact keys). Within one pile
    the creation order is the pyramid recipe's, so each pile evolves bit for bit like a world that holds it alone
    (``only=k`` builds exactly that world, at the same position). ``Scene.bodies`` lists pile 0's bodies first (ground,
    then boxes), then pile 1's ... — ``Scene.piles[k]`` is the slice of pile k."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"field{count}x{base_count}i")
    h = 0.5
    if pitch is None:
        pitch = float(base_count + 6)
    box = lib.s2MakeSquare(h)
    ground = lib.s2MakeBox(0.5 * base_count + 2.0, 1.0)
    sd = default_shape_def()
    sd.density = 1.0
    which = list(range(count)) if only is None else [only]
    cells = [(i, j) for i in range(base_count) for j in range(i, base_count)]
    per_pile = {k: [] for k in which}
    for k in which:
        bd = default_body_def()
        bd.position = Vec2(k * pitch, -1.0)
        gid = lib.s2CreateBody(world, C.byref(bd))
        lib.s2CreatePolygonShape(gid, C.byref(sd), C.byref(ground))
        per_pile[k].append(gid)
    bd = default_body_def()
    bd.type = capi.DYNAMIC_BODY
    for (i, j) in cells:
        y = (2.0 * i + 1.0) * h
        x = (i + 1.0) * h + 2.0 * (j - i) * h - h * base_count
        for k in which:
            bd.position = Vec2(k * pitch + x, y)
            bid = lib.s2CreateBody(world, C.byref(bd))
            lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
            per_pile[k].append(bid)
    sc.piles = {}
    for k in which:
        sc.piles[k] = slice(len(sc.bodies), len(sc.bodies) + len(per_pile[k]))
        sc.bodies.extend(per_pile[k])
    return sc


def pyramid_field(lib: capi.Solver2D, solver="TGS_Soft", count=256, base_count=45, first=0, pitch=None) -> Scene:
    """SURVEY §8d config 5, batched: ``count`` independent Pyramid worlds (each with its own static ground) laid side by
    side in ONE s2World, ``pitch`` metres apart, so that a single set of launches steps them all — independent worlds are
    disconnected islands of one constraint graph, which is what makes small worlds big enough for the GPU. ``first`` offsets
    the world indices (rank r of an N-rank run builds worlds r, r + N, ... by passing the right slice)."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"field{count}x{base_count}")
    h = 0.5
    if pitch is None:
        pitch = float(base_count + 6)
    box = lib.s2MakeSquare(h)
    sd = default_shape_def()
    sd.density = 1.0
    for k in range(count):
        x0 = (first + k) * pitch
        bd = default_body_def()
        bd.position = Vec2(x0, -1.0)
        gid = lib.s2CreateBody(world, C.byref(bd))
        ground = lib.s2MakeBox(0.5 * base_count + 2.0, 1.0)
        lib.s2CreatePolygonShape(gid, C.byref(sd), C.byref(ground))
        sc.bodies.append(gid)
        bd = default_body_def()
        bd.type = capi.DYNAMIC_BODY
        for i in range(base_count):
            y = (2.0 * i + 1.0) * h
            for j in range(i, base_count):
                x = (i + 1.0) * h + 2.0 * (j - i) * h - h * base_count
                bd.position = Vec2(x0 + x, y)
                bid = lib.s2CreateBody(world, C.byref(bd))
                lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
                sc.bodies.append(bid)
    return sc
