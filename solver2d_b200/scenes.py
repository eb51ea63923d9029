"""Headless scene recipes, written only against the public C API (so they run on either library, see capi.py).

Each recipe restates one of the reference's sample scenes or one of the synthetic configs of SURVEY.md §8(d):

* :func:`pyramid`         — ``Pyramid`` (reference samples/collection/sample_contact.cpp:499-561), ground widened
                            for baseCount > 200 (SURVEY §8d config 2 / headline).
* :func:`vertical_stack`  — small stack of boxes (quick contact test).
* :func:`bridge`          — ``Bridge`` (reference samples/collection/sample_joints.cpp:15-90).
* :func:`joint_contact_stress` — config 4: stacked bridges + a grid of boxes dropped on them.
* :func:`tumbler`         — config 3: motorised hollow container with a grid of small boxes.
* :func:`damped_mix`      — a pile, thrown bodies and unconstrained bodies with body damping and gravity scales, and
                            optionally a damped revolute chain.
* :func:`mixed_shapes`    — circles/capsules/polygons/segments on a ground, exercising all nine manifold functions.
* :func:`collision_zoo`   — every manifold kind, flipped pairs, dynamic segments, compound bodies, mixed frictions and
                            shape filters, thrown sideways.
* :func:`bouncers`        — shapes with restitution dropped from several heights (the restitution extension).
* :func:`welded_structures` — cantilevers, welded assemblies, a welded platform rider and a chain (the weld joint).
* :func:`sliders`         — pistons, an elevator, an inclined slider, a kinematic carriage, a slider-crank and a mouse
                            joint on a slider (the prismatic joint).
* :func:`distance_joints` — ropes of boxes, rigid-rod pendulums, a spring ring of circles over a pile, winches, a tether
                            to a kinematic platform, a revolute chain and a mouse joint (the distance joint).
* :func:`wheels`          — a motorised car over bumps, a car rolling down a slope, a barrow on a rigid axle, a trolley
                            hanging from a kinematic rail and a mouse joint (the wheel joint).
* :func:`motors`          — top-down friction, a driven platform with a pile, a weak motor under its load, a dynamic
                            pair, a rider on a kinematic carriage, a drive across the angle seam and a mouse joint
                            (the motor joint).
* :func:`kinematic_rigs`  — piles on sliding kinematic platforms and a turntable, joints hanging from moving kinematic
                            carriages (kinematic bodies under every solver variant).
* :func:`projectiles`     — circles, capsules, boxes and hulls fired at 30-200 m/s at thin static boxes and segments
                            (continuous collision).
* :func:`hub_trays`       — trays carrying spaced riders of 1-60 shapes, and riders on the ground: hub bodies with exact
                            contact counts (the solver's hub-body capacity limits).
* :func:`hub_beam`        — a beam hanging N pendulums: a hub body with exact joint counts.

All scenes are deterministic lattices (no RNG). A recipe returns a :class:`Scene` holding the world id and the
body ids in creation order.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, field

import numpy as np

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


DAMPED_LINEAR = (0.0, 0.1, 0.5, 2.0)
DAMPED_ANGULAR = (0.0, 0.3, 5.0)
DAMPED_GRAVITY = (1.0, 0.5, 0.0, -0.25)


def damped_mix(lib, solver="TGS_Soft", joints=False) -> Scene:
    """Body damping and gravity scale coverage. Every dynamic body k gets linearDamping DAMPED_LINEAR[k % 4] and
    angularDamping DAMPED_ANGULAR[k % 3] (all twelve pairs), and a gravityScale from DAMPED_GRAVITY:

    * a pile of 24 boxes on the ground (gravity scale 1 or 0.5, so it stays a pile);
    * eight circles, capsules and boxes thrown at the pile, spinning (every gravity scale);
    * eight spinning bodies high above the ground and 3 m apart, drifting apart: they touch nothing during a test run, so
      they are integrated as unconstrained bodies (every gravity scale, one rising);
    * with `joints`: a chain of six capsules on revolute joints hanging from the ground, damped like the rest.

    Without `joints` the world has no joints and no kinematic bodies."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name="damped_mix" + ("_joints" if joints else ""))
    gid = _ground(lib, world, 30.0)
    sc.bodies.append(gid)
    sd = default_shape_def()
    k = 0

    def body(x, y, gravity, kind, vx=0.0, vy=0.0, w=0.0, angle=0.0):
        nonlocal k
        bd = default_body_def()
        bd.type = capi.DYNAMIC_BODY
        bd.position = Vec2(x, y)
        bd.angle = angle
        bd.linearVelocity = Vec2(vx, vy)
        bd.angularVelocity = w
        bd.linearDamping = DAMPED_LINEAR[k % 4]
        bd.angularDamping = DAMPED_ANGULAR[k % 3]
        bd.gravityScale = gravity
        k += 1
        bid = lib.s2CreateBody(world, C.byref(bd))
        if kind == 0:
            box = lib.s2MakeBox(0.4, 0.3)
            lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
        elif kind == 1:
            lib.s2CreateCircleShape(bid, C.byref(sd), C.byref(Circle(Vec2(0.05, 0.0), 0.35)))
        else:
            lib.s2CreateCapsuleShape(bid, C.byref(sd), C.byref(Capsule(Vec2(-0.35, 0.0), Vec2(0.35, 0.0), 0.2)))
        sc.bodies.append(bid)
        return bid

    for i in range(4):
        for j in range(6):
            body(-10.0 + 0.85 * j + 0.2 * (i % 2), 0.3 + 0.6 * i, DAMPED_GRAVITY[(i + j) % 2], 0)
    for n in range(8):
        body(-1.0 + 0.9 * n, 1.0 + 0.5 * (n % 3), DAMPED_GRAVITY[n % 4], n % 3, vx=-6.0 - 0.5 * n, vy=1.5,
             w=4.0 if n % 2 == 0 else -3.0, angle=0.3 * n)
    for n in range(8):
        body(10.0 + 3.0 * n, 40.0, DAMPED_GRAVITY[n % 4], n % 3, vx=0.5 * (n - 3.5), vy=0.8, w=2.0 + n, angle=0.2 * n)
    if joints:
        prev = gid
        for i in range(6):
            bid = body(2.5 + 1.0 * i, 10.0, DAMPED_GRAVITY[i % 2], 2)
            jd = default_revolute_def()
            pivot = Vec2(2.0 + 1.0 * i, 10.0)
            jd.bodyIdA = prev
            jd.bodyIdB = bid
            jd.localAnchorA = lib.s2Body_GetLocalPoint(prev, pivot)
            jd.localAnchorB = lib.s2Body_GetLocalPoint(bid, pivot)
            sc.joints.append(lib.s2CreateRevoluteJoint(world, C.byref(jd)))
            prev = bid
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


SOFT_WELDS_PITCH = 30.0  # width of one copy of soft_welds (m)


def soft_welds(lib: capi.Solver2D, solver="TGS_Soft", copies=1, kinematic=True) -> Scene:
    """Soft weld coverage (DESIGN.md §3.15), `copies` side by side (34 bodies each). Per copy:

    * a donut: a ring of eight capsules welded end to end with angular springs (and a stiff anchor spring on one weld),
      dropped onto a small pile;
    * two cantilevers of four boxes welded to a static wall: one soft (angular springs), one rigid; in the soft one the
      boxes alternate between angle 0 and 3 rad, so its welds have reference angles of +3 and -3 rad (near +-pi);
    * a box hanging from a static body on a linear-only soft weld;
    * with `kinematic`: a box on a platform that moves sideways, held by a soft weld (both parts);
    * a hanging chain of three revolute links, and (first copy only) a mouse joint pulling the donut.

    On a library without s2CreateWeldJoint (the reference) every weld is created as a revolute joint with limits and
    motor off, with the same bodies, anchors, reference angle and collideConnected, as ``welded_structures`` does.
    ``sc.piles["welds"]`` lists the indices into ``sc.joints`` of every weld, soft or rigid; ``sc.piles["soft_welds"]``
    lists one (joint index, linearHertz, linearDampingRatio, angularHertz, angularDampingRatio) per soft weld, so that a
    test can turn the stand-in rows into soft weld rows."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"soft_welds{copies}")
    sc.piles["welds"] = []
    sc.piles["soft_welds"] = []
    has_weld = "s2CreateWeldJoint" not in lib.missing
    gid = _ground(lib, world, 0.5 * SOFT_WELDS_PITCH * copies + 5.0)
    sc.bodies.append(gid)
    sd = default_shape_def()

    def body(kind, x, y, angle=0.0, hx=0.5, hy=0.125, vx=0.0, capsule=None):
        bd = default_body_def()
        bd.type = kind
        bd.position = Vec2(x, y)
        bd.angle = angle
        bd.linearVelocity = Vec2(vx, 0.0)
        bid = lib.s2CreateBody(world, C.byref(bd))
        if capsule is not None:
            cap = Capsule(Vec2(-capsule[0], 0.0), Vec2(capsule[0], 0.0), capsule[1])
            lib.s2CreateCapsuleShape(bid, C.byref(sd), C.byref(cap))
        else:
            box = lib.s2MakeBox(hx, hy)
            lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
        sc.bodies.append(bid)
        return bid

    def weld(a, b, pivot, reference_angle, linear=(0.0, 0.0), angular=(0.0, 0.0)):
        jd = capi.default_weld_def() if has_weld else default_revolute_def()
        jd.bodyIdA = a
        jd.bodyIdB = b
        jd.localAnchorA = lib.s2Body_GetLocalPoint(a, pivot)
        jd.localAnchorB = lib.s2Body_GetLocalPoint(b, pivot)
        jd.referenceAngle = reference_angle
        if has_weld:
            jd.linearHertz, jd.linearDampingRatio = linear
            jd.angularHertz, jd.angularDampingRatio = angular
        create = lib.s2CreateWeldJoint if has_weld else lib.s2CreateRevoluteJoint
        sc.piles["welds"].append(len(sc.joints))
        if linear[0] > 0.0 or angular[0] > 0.0:
            sc.piles["soft_welds"].append((len(sc.joints),) + tuple(linear) + tuple(angular))
        sc.joints.append(create(world, C.byref(jd)))

    D, S, K = capi.DYNAMIC_BODY, capi.STATIC_BODY, capi.KINEMATIC_BODY
    for k in range(copies):
        x0 = -0.5 * SOFT_WELDS_PITCH * (copies - 1) + SOFT_WELDS_PITCH * k - 10.0
        # a small pile with a donut above it: eight capsules on a ring of radius 1.2, each welded to the next at their
        # shared end point with an angular spring
        for i in range(4):
            for j in range(2):
                body(D, x0 + 0.5 + 1.05 * i, 0.25 + 0.5 * j, hx=0.5, hy=0.25)
        n, radius, cx, cy = 8, 1.2, x0 + 2.0, 4.0
        half = radius * math.sin(math.pi / n)
        ring = []
        for i in range(n):
            t = 2.0 * math.pi * (i + 0.5) / n
            ring.append(body(D, cx + radius * math.cos(math.pi / n) * math.cos(t), cy + radius * math.cos(math.pi / n) * math.sin(t),
                             angle=t + 0.5 * math.pi, capsule=(half, 0.15)))
        for i in range(n):
            t = 2.0 * math.pi * (i + 1) / n
            pivot = Vec2(cx + radius * math.cos(t), cy + radius * math.sin(t))
            weld(ring[i], ring[(i + 1) % n], pivot, 2.0 * math.pi / n if i < n - 1 else 2.0 * math.pi / n - 2.0 * math.pi,
                 linear=(15.0, 1.0) if i == 0 else (0.0, 0.0), angular=(4.0, 0.3))
        # cantilevers: the soft one at y = 9 with reference angles near +-pi, the rigid one at y = 7
        for beam, y in enumerate((9.0, 7.0)):
            wall = body(S, x0 + 6.0, y, hx=0.25, hy=1.0)
            prev, prev_angle = wall, 0.0
            for i in range(4):
                angle = 3.0 if beam == 0 and i % 2 == 0 else 0.0
                bid = body(D, x0 + 6.75 + 1.0 * i, y, angle=angle)
                weld(prev, bid, Vec2(x0 + 6.25 + 1.0 * i, y), angle - prev_angle,
                     angular=(3.0 + 0.5 * i, 0.2) if beam == 0 else (0.0, 0.0))
                prev, prev_angle = bid, angle
        # a box hanging on a linear-only soft weld
        hook = body(S, x0 + 13.0, 8.0, hx=0.25, hy=0.25)
        box = body(D, x0 + 13.0, 7.25, hx=0.25, hy=0.25)
        weld(hook, box, Vec2(x0 + 13.0, 7.5), 0.0, linear=(2.0, 0.1))
        if kinematic:
            p = body(K, x0 + 16.0, 2.0, hx=1.0, hy=0.125, vx=0.5)
            q = body(D, x0 + 16.0, 2.0 + 0.375, hx=0.25, hy=0.25)
            weld(p, q, Vec2(x0 + 16.0, 2.0 + 0.125), 0.0, linear=(5.0, 0.5), angular=(2.0, 0.7))
        # revolute chain
        anchor = body(S, x0 + 19.0, 10.0, hx=0.25, hy=0.25)
        prev = anchor
        for i in range(3):
            bid = body(D, x0 + 19.5 + 1.0 * i, 10.0)
            jd = default_revolute_def()
            pivot = Vec2(x0 + 19.0 + 1.0 * i, 10.0)
            jd.bodyIdA = prev
            jd.bodyIdB = bid
            jd.localAnchorA = lib.s2Body_GetLocalPoint(prev, pivot)
            jd.localAnchorB = lib.s2Body_GetLocalPoint(bid, pivot)
            sc.joints.append(lib.s2CreateRevoluteJoint(world, C.byref(jd)))
            prev = bid
        if k == 0:
            md = default_mouse_def()
            md.bodyIdA = gid
            md.bodyIdB = ring[0]
            md.target = Vec2(cx + 1.5, cy + 1.0)
            md.hertz = 2.0
            md.dampingRatio = 0.7
            sc.joints.append(lib.s2CreateMouseJoint(world, C.byref(md)))
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


SPRINGS_PITCH = 40.0  # width of one copy of springs (m)


def springs(lib: capi.Solver2D, solver="TGS_Soft", copies=1, kinematic=True) -> Scene:
    """Joint spring coverage (DESIGN.md §3.14), `copies` side by side (about 25 bodies each). Per copy:

    * a car driving over bumps: a chassis on two prismatic suspension springs with limits (axis up, 4 Hz, damping ratio
      0.7), each holding an axle, and a circular wheel on each axle on a motorised revolute joint (the car's parts share a
      negative collision group, so only the wheels and the chassis touch the world);
    * a soft chain of six links on revolute springs (3 Hz, 0.3), hung from a post, falling onto a pile of boxes;
    * a flipper: a revolute joint with a spring (5 Hz, 0.2), limits and a weak motor on one plank;
    * with `kinematic`: a box on a prismatic spring (2 Hz, 0.1) along a kinematic carriage that moves sideways;
    * a revolute spring (2 Hz, 0.5) whose rest angle, pi - 0.05, sits at the seam: its body starts at -pi + 0.1, so the
      spring turns it back across the seam;
    * a box pulled by a mouse joint (first copy only).

    On a library without s2CreatePrismaticJoint (the reference) every prismatic joint is created as a revolute joint with
    limits and motor off, and no spring is set, as ``sliders`` does. ``sc.piles["prismatic"]``, ``["prismatic_defs"]`` and
    ``["prismatic_bodies"]`` describe the prismatic joints as in ``sliders``; ``sc.piles["springs"]`` lists
    (index into ``sc.joints``, hertz, dampingRatio) of every sprung joint, so that a test can give the stand-in rows their
    springs."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"springs{copies}")
    sc.piles["prismatic"] = []
    sc.piles["prismatic_defs"] = []
    sc.piles["prismatic_bodies"] = []
    sc.piles["springs"] = []
    has_prismatic = "s2CreatePrismaticJoint" not in lib.missing
    gid = _ground(lib, world, 0.5 * SPRINGS_PITCH * copies + 5.0)
    sc.bodies.append(gid)

    def body(kind, x, y, angle=0.0, hx=0.5, hy=0.125, vx=0.0, vy=0.0, radius=None, group=0):
        bd = default_body_def()
        bd.type = kind
        bd.position = Vec2(x, y)
        bd.angle = angle
        bd.linearVelocity = Vec2(vx, vy)
        bid = lib.s2CreateBody(world, C.byref(bd))
        sd = default_shape_def()
        sd.filter.groupIndex = group
        if radius is not None:
            lib.s2CreateCircleShape(bid, C.byref(sd), C.byref(Circle(Vec2(0.0, 0.0), radius)))
        else:
            lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(lib.s2MakeBox(hx, hy)))
        sc.bodies.append(bid)
        return bid

    def spring(jid, hertz, zeta, prismatic_joint):
        sc.piles["springs"].append((len(sc.joints) - 1, hertz, zeta))
        if not has_prismatic:
            return  # the reference has no spring
        if prismatic_joint:
            return  # set in the definition
        lib.s2RevoluteJoint_EnableSpring(jid, True)
        lib.s2RevoluteJoint_SetSpringHertz(jid, hertz)
        lib.s2RevoluteJoint_SetSpringDampingRatio(jid, zeta)

    def prismatic(a, b, pivot, axis, limit=None, hertz=0.0, zeta=0.0):
        d = dict(localAnchorA=tuple(lib.s2Body_GetLocalPoint(a, pivot)), localAnchorB=tuple(lib.s2Body_GetLocalPoint(b, pivot)),
                 localAxisA=axis, referenceAngle=0.0, enableLimit=limit is not None,
                 lowerTranslation=limit[0] if limit else 0.0, upperTranslation=limit[1] if limit else 0.0,
                 enableMotor=False, motorSpeed=0.0, maxMotorForce=0.0, collideConnected=False)
        if has_prismatic:
            jd = capi.default_prismatic_def()
            for name, value in d.items():
                setattr(jd, name, Vec2(*value) if isinstance(value, tuple) else value)
            jd.enableSpring, jd.hertz, jd.dampingRatio = True, hertz, zeta
            create = lib.s2CreatePrismaticJoint
        else:
            jd = default_revolute_def()
            jd.localAnchorA = Vec2(*d["localAnchorA"])
            jd.localAnchorB = Vec2(*d["localAnchorB"])
            create = lib.s2CreateRevoluteJoint
        jd.bodyIdA = a
        jd.bodyIdB = b
        sc.piles["prismatic"].append(len(sc.joints))
        sc.piles["prismatic_defs"].append(d)
        sc.piles["prismatic_bodies"].append((a, b))
        jid = create(world, C.byref(jd))
        sc.joints.append(jid)
        spring(jid, hertz, zeta, True)
        return jid

    def revolute(a, b, pivot, reference_angle=0.0, motor=None, limit=None, hertz=None, zeta=0.0):
        jd = default_revolute_def()
        jd.bodyIdA = a
        jd.bodyIdB = b
        jd.localAnchorA = lib.s2Body_GetLocalPoint(a, pivot)
        jd.localAnchorB = lib.s2Body_GetLocalPoint(b, pivot)
        jd.referenceAngle = reference_angle
        if motor is not None:
            jd.enableMotor = True
            jd.motorSpeed, jd.maxMotorTorque = motor
        if limit is not None:
            jd.enableLimit = True
            jd.lowerAngle, jd.upperAngle = limit
        jid = lib.s2CreateRevoluteJoint(world, C.byref(jd))
        sc.joints.append(jid)
        if hertz is not None:
            spring(jid, hertz, zeta, False)
        return jid

    D, S, K = capi.DYNAMIC_BODY, capi.STATIC_BODY, capi.KINEMATIC_BODY
    up = (0.0, 1.0)
    for k in range(copies):
        x0 = -0.5 * SPRINGS_PITCH * (copies - 1) + SPRINGS_PITCH * k - 18.0
        # bumps on the ground, then the car
        for i in range(4):
            body(S, x0 + 4.0 + 2.5 * i, 0.05, hx=0.4, hy=0.05 + 0.05 * (i % 2))
        group = -(k + 1)
        chassis = body(D, x0, 1.5, hx=1.2, hy=0.2, group=group)
        for dx in (-0.9, 0.9):
            axle = body(D, x0 + dx, 0.9, hx=0.1, hy=0.1, group=group)
            prismatic(chassis, axle, Vec2(x0 + dx, 0.9), up, limit=(-0.25, 0.25), hertz=4.0, zeta=0.7)
            wheel = body(D, x0 + dx, 0.9, radius=0.4, group=group)
            revolute(axle, wheel, Vec2(x0 + dx, 0.9), motor=(-8.0, 12.0))
        # a soft chain falling onto a pile
        post = body(S, x0 + 16.0, 6.0, hx=0.1, hy=0.1)
        prev = post
        for i in range(6):
            link = body(D, x0 + 16.5 + 1.0 * i, 6.0, hx=0.5, hy=0.1)
            revolute(prev, link, Vec2(x0 + 16.0 + 1.0 * i, 6.0), hertz=3.0, zeta=0.3)
            prev = link
        for i in range(3):
            for j in range(3 - i):
                body(D, x0 + 18.0 + 0.55 * j + 0.275 * i, 0.25 + 0.5 * i, hx=0.25, hy=0.25)
        # a flipper: spring, limits and a weak motor together
        hinge = body(S, x0 + 25.0, 1.0, hx=0.1, hy=0.1)
        plank = body(D, x0 + 26.0, 1.0, hx=1.0, hy=0.1)
        revolute(hinge, plank, Vec2(x0 + 25.0, 1.0), motor=(1.0, 2.0), limit=(-0.5, 0.5), hertz=5.0, zeta=0.2)
        # a box on a prismatic spring along a kinematic carriage
        if kinematic:
            carriage = body(K, x0 + 30.0, 3.0, hx=1.0, hy=0.125, vx=0.7)
            rider = body(D, x0 + 30.5, 3.375, hx=0.25, hy=0.25)
            prismatic(carriage, rider, Vec2(x0 + 30.5, 3.375), (1.0, 0.0), limit=(-0.75, 0.75), hertz=2.0, zeta=0.1)
        # a revolute spring whose rest angle sits at the seam
        pin = body(S, x0 + 34.0, 4.0, hx=0.1, hy=0.1)
        arm = body(D, x0 + 34.0, 4.0, angle=-math.pi + 0.1, hx=0.6, hy=0.1)
        revolute(pin, arm, Vec2(x0 + 34.0, 4.0), reference_angle=math.pi - 0.05, hertz=2.0, zeta=0.5)
        if k == 0:
            dragged = body(D, x0 + 37.0, 0.25, hx=0.25, hy=0.25)
            md = default_mouse_def()
            md.bodyIdA = gid
            md.bodyIdB = dragged
            md.target = Vec2(x0 + 37.5, 1.5)
            md.hertz = 3.0
            md.dampingRatio = 0.7
            sc.joints.append(lib.s2CreateMouseJoint(world, C.byref(md)))
    return sc


DISTANCE_PITCH = 40.0  # width of one copy of distance_joints (m)


def distance_joints(lib: capi.Solver2D, solver="TGS_Soft", copies=1, kinematic=True, stand_ins=None) -> Scene:
    """Distance joint coverage (DESIGN.md §3.16), `copies` side by side (about 60 bodies each). Per copy:

    * two hanging ropes of five boxes each (every link a rope: spring on at hertz 0, limit [slop, 0.6]) from a beam;
    * a row of four rigid-rod pendulums (1.5 m) started at different angles, so the bobs hit one another;
    * a soft ring of eight circles on springs (neighbours 6 Hz, opposite pairs 3 Hz) dropped on a pile of boxes;
    * a winch (rope with a motor shortening at 0.5 m/s) lifting a box with 60 N, and one set below its load (3 N);
    * with `kinematic`: a box on a sprung, limited tether below a kinematic platform that moves sideways;
    * a revolute chain of four links hung from a post;
    * a box pulled by a mouse joint (first copy only).

    On a library without s2CreateDistanceJoint (the reference), or with `stand_ins` true, every distance joint is created as
    a revolute joint at anchor B's start point with limits and motor off. ``sc.piles["distance"]`` lists the index into
    ``sc.joints`` of every distance joint and ``sc.piles["distance_defs"]`` its definition (anchors relative to the body
    origins, lengths clamped as s2CreateDistanceJoint clamps them), so that a test can turn the stand-in rows into distance
    rows."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"distance_joints{copies}")
    sc.piles["distance"] = []
    sc.piles["distance_defs"] = []
    real = "s2CreateDistanceJoint" not in lib.missing and not stand_ins
    gid = _ground(lib, world, 0.5 * DISTANCE_PITCH * copies + 5.0)
    sc.bodies.append(gid)

    def body(kind, x, y, hx=0.25, hy=0.25, vx=0.0, radius=None, group=0):
        bd = default_body_def()
        bd.type = kind
        bd.position = Vec2(x, y)
        bd.linearVelocity = Vec2(vx, 0.0)
        bid = lib.s2CreateBody(world, C.byref(bd))
        sd = default_shape_def()
        sd.filter.groupIndex = group
        if radius is not None:
            lib.s2CreateCircleShape(bid, C.byref(sd), C.byref(Circle(Vec2(0.0, 0.0), radius)))
        else:
            lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(lib.s2MakeBox(hx, hy)))
        sc.bodies.append(bid)
        return bid

    def clamp(length):
        return float(np.clip(np.float32(length), np.float32(0.005), np.float32(100000.0)))

    def distance(a, b, pa, pb, length, spring=None, limit=None, motor=None):
        """pa, pb: the anchors' world points at creation."""
        d = dict(localAnchorA=tuple(lib.s2Body_GetLocalPoint(a, pa)), localAnchorB=tuple(lib.s2Body_GetLocalPoint(b, pb)),
                 length=clamp(length), enableSpring=spring is not None, hertz=spring[0] if spring else 0.0,
                 dampingRatio=spring[1] if spring else 0.0, enableLimit=limit is not None,
                 minLength=clamp(limit[0] if limit else 0.0), maxLength=clamp(limit[1] if limit else 100000.0),
                 enableMotor=motor is not None, motorSpeed=motor[0] if motor else 0.0, maxMotorForce=motor[1] if motor else 0.0)
        if real:
            jd = capi.default_distance_def()
            for name, value in d.items():
                setattr(jd, name, Vec2(*value) if isinstance(value, tuple) else value)
            create = lib.s2CreateDistanceJoint
        else:
            jd = default_revolute_def()
            jd.localAnchorA = lib.s2Body_GetLocalPoint(a, pb)
            jd.localAnchorB = lib.s2Body_GetLocalPoint(b, pb)
            create = lib.s2CreateRevoluteJoint
        jd.bodyIdA = a
        jd.bodyIdB = b
        sc.piles["distance"].append(len(sc.joints))
        sc.piles["distance_defs"].append(d)
        jid = create(world, C.byref(jd))
        sc.joints.append(jid)
        return jid

    def revolute(a, b, pivot):
        jd = default_revolute_def()
        jd.bodyIdA = a
        jd.bodyIdB = b
        jd.localAnchorA = lib.s2Body_GetLocalPoint(a, pivot)
        jd.localAnchorB = lib.s2Body_GetLocalPoint(b, pivot)
        sc.joints.append(lib.s2CreateRevoluteJoint(world, C.byref(jd)))

    D, S, K = capi.DYNAMIC_BODY, capi.STATIC_BODY, capi.KINEMATIC_BODY
    rope = (0.0, 0.0)
    for k in range(copies):
        x0 = -0.5 * DISTANCE_PITCH * (copies - 1) + DISTANCE_PITCH * k - 18.0
        # two hanging ropes of boxes from a beam, the second started swinging
        beam = body(S, x0 + 1.5, 9.0, hx=1.5, hy=0.1)
        for r, dx in enumerate((0.5, 2.5)):
            prev, prev_at = beam, Vec2(x0 + dx, 8.9)
            for i in range(5):
                x = x0 + dx + 0.5 * (i + 1) * r
                y = 8.9 - 0.55 * (i + 1)
                box = body(D, x, y, hx=0.15, hy=0.15)
                distance(prev, box, prev_at, Vec2(x, y + 0.15), 0.5, spring=rope, limit=(0.0, 0.6))
                prev, prev_at = box, Vec2(x, y - 0.15)
        # a row of rigid-rod pendulums that hit one another
        for i in range(4):
            pivot = Vec2(x0 + 5.0 + 0.6 * i, 6.0)
            angle = 0.8 if i == 0 else 0.05 * i
            bob = body(D, pivot.x - 1.5 * math.sin(angle), 6.0 - 1.5 * math.cos(angle), hx=0.25, hy=0.25)
            distance(gid, bob, pivot, Vec2(pivot.x - 1.5 * math.sin(angle), 6.0 - 1.5 * math.cos(angle)), 1.5)
        # a pile of boxes and a soft ring of circles falling onto it
        for i in range(4):
            for j in range(4 - i):
                body(D, x0 + 11.0 + 0.55 * j + 0.275 * i, 0.25 + 0.5 * i, hx=0.25, hy=0.25)
        ring = []
        for i in range(8):
            a = 2.0 * math.pi * i / 8
            ring.append((body(D, x0 + 11.8 + math.cos(a), 5.0 + math.sin(a), radius=0.2), Vec2(x0 + 11.8 + math.cos(a), 5.0 + math.sin(a))))
        for i in range(8):
            (a, pa), (b, pb) = ring[i], ring[(i + 1) % 8]
            distance(a, b, pa, pb, math.hypot(pb.x - pa.x, pb.y - pa.y), spring=(6.0, 0.5))
        for i in range(4):
            (a, pa), (b, pb) = ring[i], ring[i + 4]
            distance(a, b, pa, pb, 2.0, spring=(3.0, 0.3), limit=(1.0, 2.5))
        # a winch lifting its load, and one set below its load
        for dx, force in ((17.0, 60.0), (19.0, 3.0)):
            load = body(D, x0 + dx, 5.0, hx=0.3, hy=0.3)
            distance(gid, load, Vec2(x0 + dx, 9.0), Vec2(x0 + dx, 5.3), 3.7, spring=rope, limit=(0.5, 4.0),
                     motor=(-0.5, force))
        # a sprung tether below a kinematic platform
        if kinematic:
            platform = body(K, x0 + 23.0, 7.0, hx=1.0, hy=0.125, vx=0.7)
            rider = body(D, x0 + 23.0, 5.5, hx=0.25, hy=0.25)
            distance(platform, rider, Vec2(x0 + 23.0, 6.875), Vec2(x0 + 23.0, 5.75), 1.2, spring=(2.0, 0.2), limit=(0.6, 1.6))
        # a revolute chain
        post = body(S, x0 + 27.0, 6.0, hx=0.1, hy=0.1)
        prev = post
        for i in range(4):
            link = body(D, x0 + 27.5 + 1.0 * i, 6.0, hx=0.5, hy=0.1)
            revolute(prev, link, Vec2(x0 + 27.0 + 1.0 * i, 6.0))
            prev = link
        if k == 0:
            dragged = body(D, x0 + 33.0, 0.25)
            md = default_mouse_def()
            md.bodyIdA = gid
            md.bodyIdB = dragged
            md.target = Vec2(x0 + 33.5, 1.5)
            md.hertz = 3.0
            md.dampingRatio = 0.7
            sc.joints.append(lib.s2CreateMouseJoint(world, C.byref(md)))
    return sc


WHEELS_PITCH = 40.0  # width of one copy of wheels (m)


def wheels(lib: capi.Solver2D, solver="TGS_Soft", copies=1, kinematic=True, stand_ins=None) -> Scene:
    """Wheel joint coverage (DESIGN.md §3.17), `copies` side by side (about 20 bodies each). Per copy:

    * a car driving over bumps: a chassis on two wheel joints (axis up, spring 4 Hz, damping ratio 0.7, limits +/- 0.25 m),
      the rear one motorised (-8 rad/s, 12 N-m); the car's parts share a negative collision group, so only the wheels and
      the chassis touch the world;
    * a car without a motor rolling down a slope (spring 3 Hz, 0.5, limits +/- 0.2 m);
    * a barrow: a plank on one wheel with equal limits (a rigid axle), its other end on the ground;
    * with `kinematic`: a trolley hanging from a kinematic rail that moves sideways, on a wheel joint along the rail
      (spring 1 Hz, 0.3, limits +/- 1.5 m), free to swing about its anchor;
    * a box pulled by a mouse joint (first copy only).

    On a library without s2CreateWheelJoint (the reference), or with `stand_ins` true, every wheel joint is created as a
    revolute joint at the wheel's anchor that carries the same motor. ``sc.piles["wheel"]`` lists the index into
    ``sc.joints`` of every wheel joint and ``sc.piles["wheel_defs"]`` its definition (anchors relative to the body origins),
    so that a test can turn the stand-in rows into wheel rows."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"wheels{copies}")
    sc.piles["wheel"] = []
    sc.piles["wheel_defs"] = []
    real = "s2CreateWheelJoint" not in lib.missing and not stand_ins
    gid = _ground(lib, world, 0.5 * WHEELS_PITCH * copies + 5.0)
    sc.bodies.append(gid)

    def body(kind, x, y, angle=0.0, hx=0.5, hy=0.125, vx=0.0, radius=None, group=0):
        bd = default_body_def()
        bd.type = kind
        bd.position = Vec2(x, y)
        bd.angle = angle
        bd.linearVelocity = Vec2(vx, 0.0)
        bid = lib.s2CreateBody(world, C.byref(bd))
        sd = default_shape_def()
        sd.filter.groupIndex = group
        if radius is not None:
            lib.s2CreateCircleShape(bid, C.byref(sd), C.byref(Circle(Vec2(0.0, 0.0), radius)))
        else:
            lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(lib.s2MakeBox(hx, hy)))
        sc.bodies.append(bid)
        return bid

    def wheel(a, b, pivot, axis, spring=None, limit=None, motor=None):
        """pivot: the anchors' world point at creation."""
        d = dict(localAnchorA=tuple(lib.s2Body_GetLocalPoint(a, pivot)), localAnchorB=tuple(lib.s2Body_GetLocalPoint(b, pivot)),
                 localAxisA=axis, enableSpring=spring is not None, hertz=spring[0] if spring else 0.0,
                 dampingRatio=spring[1] if spring else 0.0, enableLimit=limit is not None,
                 lowerTranslation=limit[0] if limit else 0.0, upperTranslation=limit[1] if limit else 0.0,
                 enableMotor=motor is not None, motorSpeed=motor[0] if motor else 0.0, maxMotorTorque=motor[1] if motor else 0.0)
        if real:
            jd = capi.default_wheel_def()
            for name, value in d.items():
                setattr(jd, name, Vec2(*value) if isinstance(value, tuple) else value)
            create = lib.s2CreateWheelJoint
        else:
            jd = default_revolute_def()
            jd.localAnchorA = Vec2(*d["localAnchorA"])
            jd.localAnchorB = Vec2(*d["localAnchorB"])
            jd.enableMotor = d["enableMotor"]
            jd.motorSpeed, jd.maxMotorTorque = d["motorSpeed"], d["maxMotorTorque"]
            create = lib.s2CreateRevoluteJoint
        jd.bodyIdA = a
        jd.bodyIdB = b
        sc.piles["wheel"].append(len(sc.joints))
        sc.piles["wheel_defs"].append(d)
        jid = create(world, C.byref(jd))
        sc.joints.append(jid)
        return jid

    D, S, K = capi.DYNAMIC_BODY, capi.STATIC_BODY, capi.KINEMATIC_BODY
    up = (0.0, 1.0)
    for k in range(copies):
        x0 = -0.5 * WHEELS_PITCH * (copies - 1) + WHEELS_PITCH * k - 18.0
        group = -(k + 1)
        # bumps on the ground, then a car with a rear motor driving over them
        for i in range(4):
            body(S, x0 + 4.0 + 2.5 * i, 0.05, hx=0.4, hy=0.05 + 0.05 * (i % 2))
        chassis = body(D, x0, 1.3, hx=1.2, hy=0.2, group=group)
        for dx, motor in ((-0.9, (-8.0, 12.0)), (0.9, None)):
            tyre = body(D, x0 + dx, 0.7, radius=0.4, group=group)
            wheel(chassis, tyre, Vec2(x0 + dx, 0.7), up, spring=(4.0, 0.7), limit=(-0.25, 0.25), motor=motor)
        # a car without a motor rolling down a slope
        body(S, x0 + 20.0, 2.0, angle=-0.25, hx=4.0, hy=0.2)
        body2 = body(D, x0 + 18.0, 3.5, angle=-0.25, hx=0.9, hy=0.15, group=group)
        for dx in (-0.6, 0.6):
            c, s_ = math.cos(-0.25), math.sin(-0.25)
            at = Vec2(x0 + 18.0 + c * dx + s_ * 0.45, 3.5 + s_ * dx - c * 0.45)
            tyre = body(D, at.x, at.y, radius=0.3, group=group)
            wheel(body2, tyre, at, up, spring=(3.0, 0.5), limit=(-0.2, 0.2))
        # a barrow: a plank on one wheel with equal limits, its other end on the ground
        plank = body(D, x0 + 27.0, 0.7, angle=0.3, hx=1.0, hy=0.1, group=group)
        c, s_ = math.cos(0.3), math.sin(0.3)
        at = Vec2(x0 + 27.0 + c * 0.9, 0.7 + s_ * 0.9 - 0.1)
        tyre = body(D, at.x, at.y, radius=0.35, group=group)
        wheel(plank, tyre, at, up, limit=(0.0, 0.0))
        # a trolley hanging from a kinematic rail, along the rail
        if kinematic:
            rail = body(K, x0 + 32.0, 5.0, hx=2.0, hy=0.1, vx=0.5, group=group)
            trolley = body(D, x0 + 32.3, 4.5, hx=0.25, hy=0.5, group=group)
            wheel(rail, trolley, Vec2(x0 + 32.3, 5.0), (1.0, 0.0), spring=(1.0, 0.3), limit=(-1.5, 1.5))
        if k == 0:
            dragged = body(D, x0 + 36.0, 0.25, hx=0.25, hy=0.25)
            md = default_mouse_def()
            md.bodyIdA = gid
            md.bodyIdB = dragged
            md.target = Vec2(x0 + 36.5, 1.5)
            md.hertz = 3.0
            md.dampingRatio = 0.7
            sc.joints.append(lib.s2CreateMouseJoint(world, C.byref(md)))
    return sc


PULLEYS_PITCH = 40.0  # width of one copy of pulleys (m)


def pulleys(lib: capi.Solver2D, solver="TGS_Soft", copies=1, kinematic=True, stand_ins=None) -> Scene:
    """Pulley joint coverage (DESIGN.md §3.18), `copies` side by side (18 bodies each). Per copy:

    * Box2D 2.4's testbed pulley: two equal boxes hung from ground anchors 6 m apart, ratio 1.5, so box A sinks;
    * a counterweighted lift: a platform on a vertical prismatic joint (limits -1.5 m and 3 m) hung over a pulley against a
      counterweight, with a pile of boxes dropped onto it, so contacts share the pulley's bodies;
    * a block-and-tackle at ratio 2: a load on side A that balances one twice its mass on side B, and the same with a side B
      1.1 times as heavy again, which lifts its load;
    * with `kinematic`: a kinematic body on side A moving down at 0.4 m/s, raising the load on side B (ratio 1.5);
    * a revolute chain of three links hung from a post, and a box pulled by a mouse joint (first copy only).

    Every pulley keeps s2DefaultPulleyJointDef's collideConnected = true. On a library without s2CreatePulleyJoint (the
    reference), or with `stand_ins` true, every pulley is created as a revolute joint between the same two bodies at anchor
    B's start point, with the same collideConnected; on a library without s2CreatePrismaticJoint the lift's prismatic joint
    is such a stand-in too. ``sc.piles["pulley"]`` lists the index into ``sc.joints`` of every pulley and
    ``sc.piles["pulley_defs"]`` its definition (anchors relative to the body origins, rest lengths as the float32 values the
    row carries); ``sc.piles["prismatic"]`` and ``["prismatic_defs"]`` describe the prismatic joint as ``sliders`` does, so
    that a test can turn the stand-in rows into pulley and prismatic rows."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"pulleys{copies}")
    sc.piles["pulley"] = []
    sc.piles["pulley_defs"] = []
    sc.piles["prismatic"] = []
    sc.piles["prismatic_defs"] = []
    real = "s2CreatePulleyJoint" not in lib.missing and not stand_ins
    has_prismatic = "s2CreatePrismaticJoint" not in lib.missing
    gid = _ground(lib, world, 0.5 * PULLEYS_PITCH * copies + 5.0)
    sc.bodies.append(gid)

    def body(kind, x, y, hx=0.25, hy=0.25, vy=0.0):
        bd = default_body_def()
        bd.type = kind
        bd.position = Vec2(x, y)
        bd.linearVelocity = Vec2(0.0, vy)
        bid = lib.s2CreateBody(world, C.byref(bd))
        lib.s2CreatePolygonShape(bid, C.byref(default_shape_def()), C.byref(lib.s2MakeBox(hx, hy)))
        sc.bodies.append(bid)
        return bid

    def pulley(a, b, ga, gb, pa, pb, ratio):
        """ga, gb: the ground anchors; pa, pb: the anchors' world points at creation."""
        f32 = np.float32
        d = dict(groundAnchorA=ga, groundAnchorB=gb, localAnchorA=tuple(lib.s2Body_GetLocalPoint(a, Vec2(*pa))),
                 localAnchorB=tuple(lib.s2Body_GetLocalPoint(b, Vec2(*pb))),
                 lengthA=float(f32(math.hypot(pa[0] - ga[0], pa[1] - ga[1]))),
                 lengthB=float(f32(math.hypot(pb[0] - gb[0], pb[1] - gb[1]))), ratio=float(f32(ratio)), collideConnected=True)
        if real:
            jd = capi.default_pulley_def()
            for name, value in d.items():
                setattr(jd, name, Vec2(*value) if isinstance(value, tuple) else value)
            create = lib.s2CreatePulleyJoint
        else:
            jd = default_revolute_def()
            jd.localAnchorA = lib.s2Body_GetLocalPoint(a, Vec2(*pb))
            jd.localAnchorB = Vec2(*d["localAnchorB"])
            jd.collideConnected = True
            create = lib.s2CreateRevoluteJoint
        jd.bodyIdA = a
        jd.bodyIdB = b
        sc.piles["pulley"].append(len(sc.joints))
        sc.piles["pulley_defs"].append(d)
        jid = create(world, C.byref(jd))
        sc.joints.append(jid)
        return jid

    def prismatic(a, b, pivot, limit):
        d = dict(localAnchorA=tuple(lib.s2Body_GetLocalPoint(a, pivot)), localAnchorB=tuple(lib.s2Body_GetLocalPoint(b, pivot)),
                 localAxisA=(0.0, 1.0), referenceAngle=0.0, enableLimit=True, lowerTranslation=limit[0],
                 upperTranslation=limit[1], enableMotor=False, motorSpeed=0.0, maxMotorForce=0.0, collideConnected=False)
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
        jd.bodyIdA = a
        jd.bodyIdB = b
        sc.piles["prismatic"].append(len(sc.joints))
        sc.piles["prismatic_defs"].append(d)
        sc.joints.append(create(world, C.byref(jd)))

    def revolute(a, b, pivot):
        jd = default_revolute_def()
        jd.bodyIdA = a
        jd.bodyIdB = b
        jd.localAnchorA = lib.s2Body_GetLocalPoint(a, pivot)
        jd.localAnchorB = lib.s2Body_GetLocalPoint(b, pivot)
        sc.joints.append(lib.s2CreateRevoluteJoint(world, C.byref(jd)))

    D, S, K = capi.DYNAMIC_BODY, capi.STATIC_BODY, capi.KINEMATIC_BODY
    for k in range(copies):
        x0 = -0.5 * PULLEYS_PITCH * (copies - 1) + PULLEYS_PITCH * k - 18.0
        # Box2D 2.4's testbed pulley (scaled): anchors at the boxes' tops, ratio 1.5
        a = body(D, x0 - 3.0, 5.0, hx=0.5, hy=1.0)
        b = body(D, x0 + 3.0, 5.0, hx=0.5, hy=1.0)
        pulley(a, b, (x0 - 3.0, 10.0), (x0 + 3.0, 10.0), (x0 - 3.0, 6.0), (x0 + 3.0, 6.0), 1.5)
        # a counterweighted lift carrying a pile dropped onto it
        platform = body(D, x0 + 9.0, 2.0, hx=1.2, hy=0.1)
        prismatic(gid, platform, Vec2(x0 + 9.0, 2.0), (-1.5, 3.0))
        weight = body(D, x0 + 12.0, 5.0, hx=0.4, hy=0.5)
        pulley(platform, weight, (x0 + 9.0, 9.0), (x0 + 12.0, 9.0), (x0 + 9.0, 2.1), (x0 + 12.0, 5.5), 1.0)
        for i in range(4):
            body(D, x0 + 8.3 + 0.45 * i, 3.5 + 0.6 * i)
        # block-and-tackle at ratio 2: balanced, then a side B 1.1 times heavier again
        for dx, hxB in ((15.0, 0.6), (20.0, 0.66)):
            load = body(D, x0 + dx, 5.0, hx=0.3, hy=0.3)
            heavy = body(D, x0 + dx + 2.0, 5.0, hx=hxB, hy=0.3)
            pulley(load, heavy, (x0 + dx, 9.0), (x0 + dx + 2.0, 9.0), (x0 + dx, 5.0), (x0 + dx + 2.0, 5.0), 2.0)
        # a kinematic driver on side A raising the load on side B
        if kinematic:
            driver = body(K, x0 + 26.0, 6.0, hx=0.3, hy=0.3, vy=-0.4)
            lifted = body(D, x0 + 28.0, 4.0, hx=0.3, hy=0.3)
            pulley(driver, lifted, (x0 + 26.0, 10.0), (x0 + 28.0, 10.0), (x0 + 26.0, 6.3), (x0 + 28.0, 4.3), 1.5)
        # a revolute chain
        post = body(S, x0 + 31.0, 6.0, hx=0.1, hy=0.1)
        prev = post
        for i in range(3):
            link = body(D, x0 + 31.5 + 1.0 * i, 6.0, hx=0.5, hy=0.1)
            revolute(prev, link, Vec2(x0 + 31.0 + 1.0 * i, 6.0))
            prev = link
        if k == 0:
            dragged = body(D, x0 + 36.0, 0.25)
            md = default_mouse_def()
            md.bodyIdA = gid
            md.bodyIdB = dragged
            md.target = Vec2(x0 + 36.5, 1.5)
            md.hertz = 3.0
            md.dampingRatio = 0.7
            sc.joints.append(lib.s2CreateMouseJoint(world, C.byref(md)))
    return sc


GEARS_PITCH = 60.0  # width of one copy of gears (m)
GEARS_HUB_PLANETS = 52  # planets on the first copy's sun: more than S2B_HUB_DEGREE (48)


def gears(lib: capi.Solver2D, solver="TGS_Soft", copies=1, stand_ins=None, hub=True) -> Scene:
    """Gear joint coverage (DESIGN.md §3.19), `copies` side by side. Per copy:

    * Box2D 2.4's testbed Gears: two wheels (radius 1 and 2) on revolute joints geared at r2 / r1 = 2, and a rack on a
      vertical prismatic joint geared to the second wheel at -1 / r2;
    * a gear train of four wheels (three stages, ratios 1.5, -0.75, 1.5) driven by a motor on the first wheel's joint;
    * a rack and pinion lifting a pile: a motorised pinion geared to a platform on a vertical prismatic joint, with boxes
      dropped onto the platform, so contacts share a geared body;
    * a wheel spun at 150 rad/s geared at ratio 1 to another, so both turn through more than ten turns in 90 steps;
    * with `hub` (first copy only): a sun geared to GEARS_HUB_PLANETS planets at ratio 10, more than S2B_HUB_DEGREE.

    Every linked joint hangs off the static ground; every gear keeps s2DefaultGearJointDef's collideConnected = false. On
    a library without s2CreateGearJoint (the reference), or with `stand_ins` true, every gear is created as a revolute joint
    between its two bodies at body B's origin, with collideConnected false; on a library without s2CreatePrismaticJoint
    the racks' prismatic joints are such stand-ins too. ``sc.piles["gear"]`` lists the index into ``sc.joints`` of every gear
    and ``sc.piles["prismatic"]`` / ``["prismatic_defs"]`` describe the prismatic joints as ``sliders`` does, so that a test
    can turn the stand-in rows into gear and prismatic rows."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"gears{copies}")
    sc.piles["gear"] = []
    sc.piles["prismatic"] = []
    sc.piles["prismatic_defs"] = []
    real = "s2CreateGearJoint" not in lib.missing and not stand_ins
    has_prismatic = "s2CreatePrismaticJoint" not in lib.missing
    gid = _ground(lib, world, 0.5 * GEARS_PITCH * copies + 5.0)
    sc.bodies.append(gid)

    def body(x, y, radius=None, hx=0.25, hy=0.25, w=0.0):
        bd = default_body_def()
        bd.type = capi.DYNAMIC_BODY
        bd.position = Vec2(x, y)
        bd.angularVelocity = w
        bid = lib.s2CreateBody(world, C.byref(bd))
        if radius is not None:
            lib.s2CreateCircleShape(bid, C.byref(default_shape_def()), C.byref(capi.Circle(Vec2(0.0, 0.0), radius)))
        else:
            lib.s2CreatePolygonShape(bid, C.byref(default_shape_def()), C.byref(lib.s2MakeBox(hx, hy)))
        sc.bodies.append(bid)
        return bid

    def revolute(b, pivot, motor=None):
        jd = default_revolute_def()
        jd.bodyIdA = gid
        jd.bodyIdB = b
        jd.localAnchorA = lib.s2Body_GetLocalPoint(gid, Vec2(*pivot))
        jd.localAnchorB = lib.s2Body_GetLocalPoint(b, Vec2(*pivot))
        if motor is not None:
            jd.enableMotor, jd.motorSpeed, jd.maxMotorTorque = True, motor[0], motor[1]
        jid = lib.s2CreateRevoluteJoint(world, C.byref(jd))
        sc.joints.append(jid)
        return jid

    def prismatic(b, pivot, limit):
        d = dict(localAnchorA=tuple(lib.s2Body_GetLocalPoint(gid, Vec2(*pivot))),
                 localAnchorB=tuple(lib.s2Body_GetLocalPoint(b, Vec2(*pivot))), localAxisA=(0.0, 1.0), referenceAngle=0.0,
                 enableLimit=True, lowerTranslation=limit[0], upperTranslation=limit[1], enableMotor=False, motorSpeed=0.0,
                 maxMotorForce=0.0, collideConnected=False)
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
        jd.bodyIdA = gid
        jd.bodyIdB = b
        sc.piles["prismatic"].append(len(sc.joints))
        sc.piles["prismatic_defs"].append(d)
        jid = create(world, C.byref(jd))
        sc.joints.append(jid)
        return jid

    def gear(j1, b1, j2, b2, ratio):
        """j1 / j2 link the ground to b1 / b2."""
        if real:
            gd = capi.default_gear_def()
            gd.jointId1, gd.jointId2, gd.ratio = j1, j2, ratio
            jid = lib.s2CreateGearJoint(world, C.byref(gd))
        else:
            jd = default_revolute_def()
            jd.bodyIdA = b1
            jd.bodyIdB = b2
            jd.localAnchorA = lib.s2Body_GetLocalPoint(b1, lib.s2Body_GetPosition(b2))
            jid = lib.s2CreateRevoluteJoint(world, C.byref(jd))
        sc.piles["gear"].append(len(sc.joints))
        sc.joints.append(jid)
        return jid

    for k in range(copies):
        x0 = -0.5 * GEARS_PITCH * (copies - 1) + GEARS_PITCH * k - 25.0
        # Box2D 2.4's testbed Gears
        w1 = body(x0, 8.0, radius=1.0)
        w2 = body(x0 + 4.0, 8.0, radius=2.0)
        rack = body(x0 + 7.0, 8.0, hx=0.5, hy=2.0)
        j1 = revolute(w1, (x0, 8.0))
        j2 = revolute(w2, (x0 + 4.0, 8.0))
        j3 = prismatic(rack, (x0 + 7.0, 8.0), (-3.0, 3.0))
        gear(j1, w1, j2, w2, 2.0)
        gear(j2, w2, j3, rack, -0.5)
        # a gear train of three stages driven by the first wheel's motor
        wheels = [body(x0 + 11.0 + 2.5 * i, 8.0, radius=1.0) for i in range(4)]
        joints = [revolute(wheels[0], (x0 + 11.0, 8.0), motor=(1.5, 50.0))]
        joints += [revolute(wheels[i], (x0 + 11.0 + 2.5 * i, 8.0)) for i in range(1, 4)]
        for i, ratio in enumerate((1.5, -0.75, 1.5)):
            gear(joints[i], wheels[i], joints[i + 1], wheels[i + 1], ratio)
        # a rack and pinion lifting a pile
        pinion = body(x0 + 23.0, 6.0, radius=0.5)
        platform = body(x0 + 26.0, 2.0, hx=1.2, hy=0.1)
        jp = revolute(pinion, (x0 + 23.0, 6.0), motor=(-1.0, 200.0))
        jl = prismatic(platform, (x0 + 26.0, 2.0), (-1.5, 4.0))
        gear(jp, pinion, jl, platform, 2.0)
        for i in range(4):
            body(x0 + 25.3 + 0.45 * i, 3.0 + 0.6 * i)
        # a wheel geared through many turns
        fast = body(x0 + 31.0, 8.0, radius=0.5, w=150.0)
        slow = body(x0 + 33.0, 8.0, radius=0.5)
        gear(revolute(fast, (x0 + 31.0, 8.0)), fast, revolute(slow, (x0 + 33.0, 8.0)), slow, 1.0)
        # a sun meshing more planets than S2B_HUB_DEGREE
        if hub and k == 0:
            cx, cy = x0 + 45.0, 14.0
            sun = body(cx, cy, radius=2.0, w=1.0)
            js = revolute(sun, (cx, cy))
            for i in range(GEARS_HUB_PLANETS):
                angle = 2.0 * math.pi * i / GEARS_HUB_PLANETS
                px, py = cx + 9.0 * math.cos(angle), cy + 9.0 * math.sin(angle)
                planet = body(px, py, radius=0.3)
                gear(js, sun, revolute(planet, (px, py)), planet, 10.0)
    return sc


MOTORS_PITCH = 30.0  # width of one copy of motors (m)


def motors(lib: capi.Solver2D, solver="TGS_Soft", copies=1, kinematic=True) -> Scene:
    """Motor joint coverage, `copies` side by side (about 25 bodies each). Per copy:

    * top-down friction: six boxes that ignore gravity (gravityScale 0), motor-jointed to the ground at their start
      position with correctionFactor 0 and small caps, thrown with initial velocities and spins so that the caps brake them;
    * a dynamic platform driven by a changing linear offset (see :func:`motors_platform_offsets`), carrying a small pile;
    * a hanging 1 kg box held by a motor whose 4 N cap is below its 10 N weight, so it sinks onto the ground;
    * a motor joint between two dynamic boxes, the upper one thrown sideways;
    * with `kinematic`: a box held above a kinematic carriage that moves sideways;
    * a box started at +3.0 rad, driven to -3.0 rad across the +/-pi seam;
    * a mouse joint pulling the upper box of the dynamic pair (first copy only).

    On a library without s2CreateMotorJoint (the reference) every motor joint is created as a revolute joint with the same
    bodies, anchor A at the linear offset, anchor B at B's origin, the angular offset as its reference angle and the same
    collideConnected: the broad phase treats every joint alike, so both libraries see the same pairs.
    ``sc.piles["motor"]`` lists the indices into ``sc.joints`` of the motor joints, ``sc.piles["motor_defs"]`` their
    definitions (dicts of s2MotorJointDef fields) and ``sc.piles["platform"]`` the indices of the platform joints among
    ``sc.piles["motor"]``, so that a test can turn the stand-in rows into motor rows and drive the platforms."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"motors{copies}")
    sc.piles["motor"] = []
    sc.piles["motor_defs"] = []
    sc.piles["platform"] = []
    has_motor = "s2CreateMotorJoint" not in lib.missing
    gid = _ground(lib, world, 0.5 * MOTORS_PITCH * copies + 5.0)
    sc.bodies.append(gid)
    sd = default_shape_def()

    def body(kind, x, y, angle=0.0, hx=0.5, hy=0.5, vx=0.0, vy=0.0, w=0.0, gravity_scale=1.0):
        bd = default_body_def()
        bd.type = kind
        bd.position = Vec2(x, y)
        bd.angle = angle
        bd.linearVelocity = Vec2(vx, vy)
        bd.angularVelocity = w
        bd.gravityScale = gravity_scale
        bid = lib.s2CreateBody(world, C.byref(bd))
        box = lib.s2MakeBox(hx, hy)
        lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(box))
        sc.bodies.append(bid)
        return bid

    def motor(a, b, offset, angle=0.0, max_force=1.0, max_torque=1.0, cf=0.3, collide=False):
        d = dict(linearOffset=(float(offset[0]), float(offset[1])), angularOffset=angle, maxForce=max_force, maxTorque=max_torque,
                 correctionFactor=cf, collideConnected=collide)
        if has_motor:
            jd = capi.default_motor_def()
            for name, value in d.items():
                setattr(jd, name, Vec2(*value) if isinstance(value, tuple) else value)
            create = lib.s2CreateMotorJoint
        else:
            jd = default_revolute_def()
            jd.localAnchorA = Vec2(*d["linearOffset"])
            jd.localAnchorB = Vec2(0.0, 0.0)
            jd.referenceAngle = angle
            jd.collideConnected = collide
            create = lib.s2CreateRevoluteJoint
        jd.bodyIdA = a
        jd.bodyIdB = b
        sc.piles["motor"].append(len(sc.joints))
        sc.piles["motor_defs"].append(d)
        jid = create(world, C.byref(jd))
        sc.joints.append(jid)
        return jid

    D, S, K = capi.DYNAMIC_BODY, capi.STATIC_BODY, capi.KINEMATIC_BODY
    ground_y = -1.0  # the ground body's origin: offsets to it are relative to (0, -1)
    for k in range(copies):
        x0 = -0.5 * MOTORS_PITCH * (copies - 1) + MOTORS_PITCH * k - 14.0
        # top-down friction: clear of the ground (y = 3), no gravity, braked by the caps alone
        for i in range(6):
            x, y = x0 + 1.5 * i, 3.0
            box = body(D, x, y, hx=0.25, hy=0.25, vx=2.0 - 0.8 * i, vy=0.5 * (i % 3) - 0.5, w=1.0 - 0.4 * i, gravity_scale=0.0)
            motor(gid, box, (x, y - ground_y), max_force=2.0, max_torque=0.2, cf=0.0)
        # a dynamic platform, driven sideways by its offset, carrying a pile
        px, py = x0 + 11.0, 1.0
        deck = body(D, px, py, hx=2.0, hy=0.125)
        sc.piles["platform"].append(len(sc.piles["motor"]))
        motor(gid, deck, (px, py - ground_y), max_force=500.0, max_torque=200.0, cf=0.3)
        for i in range(3):
            body(D, px - 0.7 + 0.7 * i, py + 0.375, hx=0.25, hy=0.25)
        body(D, px - 0.35, py + 0.875, hx=0.25, hy=0.25)
        # a motor weaker than its hanging load
        post = body(S, x0 + 15.0, 4.0, hx=0.25, hy=0.25)
        load = body(D, x0 + 15.0, 2.5)
        motor(post, load, (0.0, -1.5), max_force=4.0, max_torque=5.0)
        # a motor between two dynamic bodies
        lower = body(D, x0 + 18.0, 0.5)
        upper = body(D, x0 + 18.0, 2.5, hx=0.4, hy=0.2, vx=2.0)
        motor(lower, upper, (0.0, 1.5), angle=0.3, max_force=30.0, max_torque=10.0)
        # a box held above a moving kinematic carriage
        if kinematic:
            carriage = body(K, x0 + 22.0, 2.0, hx=1.0, hy=0.125, vx=0.5)
            rider = body(D, x0 + 22.0, 3.0, hx=0.25, hy=0.25)
            motor(carriage, rider, (0.0, 1.0), max_force=40.0, max_torque=5.0)
        # an angular offset across the seam: from +3.0 rad to -3.0 rad is 0.28 rad through pi
        pivot = body(S, x0 + 26.0, 3.0, hx=0.1, hy=0.1)
        spinner = body(D, x0 + 26.0, 4.0, angle=3.0, hx=0.6, hy=0.1)
        motor(pivot, spinner, (0.0, 1.0), angle=-3.0, max_force=50.0, max_torque=2.0)
        if k == 0:
            md = default_mouse_def()
            md.bodyIdA = gid
            md.bodyIdB = upper
            md.target = Vec2(x0 + 19.0, 3.0)
            md.hertz = 3.0
            md.dampingRatio = 0.7
            sc.joints.append(lib.s2CreateMouseJoint(world, C.byref(md)))
    return sc


def motors_platform_offsets(sc: Scene, step: int, dt: float = 1.0 / 60.0):
    """(joint slots, offsets) that drive every platform of a :func:`motors` scene at `step`: the deck swings 1.5 m either side
    of its start with a 4 s period. `offsets` is float32 (x, y, angle) per joint, the layout of
    s2World_SetMotorJointOffsets."""
    slots, offsets = [], []
    t = step * dt
    for m in sc.piles["platform"]:
        d = sc.piles["motor_defs"][m]
        slots.append(sc.joints[sc.piles["motor"][m]].index)
        offsets.append((d["linearOffset"][0] + 1.5 * math.sin(0.5 * math.pi * t), d["linearOffset"][1], d["angularOffset"]))
    return np.array(slots, dtype=np.int32), np.array(offsets, dtype=np.float32).reshape(-1, 3)


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


PROJECTILE_SPEEDS = (30.0, 55.0, 90.0, 140.0, 200.0)  # m/s
PROJECTILE_TILTS = (0.0, 0.3, -0.45)  # rad: wall turned away from facing the projectile head-on
PROJECTILE_WALL_HALF_LENGTH = 2.0
PROJECTILE_WALL_HALF_THICKNESS = 0.025  # a 0.05 m thick box


def projectiles(lib: capi.Solver2D, solver="TGS_Soft", copies=1, excluded=True) -> Scene:
    """Continuous-collision coverage: lanes on a grid, each a static wall (its own body: a box 0.05 m thick or a segment,
    4 m long, tilted by one of PROJECTILE_TILTS) and a projectile without gravity fired at it along +x (a circle, capsule,
    box or hexagon at each of PROJECTILE_SPEEDS). At 60 Hz a projectile moves 0.5-3.3 m per step, so without continuous
    collision many pass through. With `excluded`, four more lanes whose projectile must pass: two whose filter excludes the
    wall and two jointed to the wall's body by a prismatic joint along the flight (the joint rule creates no contact; the
    reference has no prismatic joint and builds these lanes without it). `copies` repeats the lane set.

    sc.piles["lanes"]: per lane a dict with the projectile's and the wall's body ids, the wall's centre, unit normal
    (pointing away from the projectile's side) and half length, `passes` (the projectile is meant to pass), `exclusion`
    ("filter", "joint" or None) and both shapes in polygon form (`form`, `wall_form`)."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"projectiles{copies}")
    specs = [(kind, v, wall, tilt, None) for kind in range(4) for v in PROJECTILE_SPEEDS for wall in ("box", "segment")
             for tilt in PROJECTILE_TILTS] * copies
    if excluded:
        specs += [(0, 90.0, "box", 0.0, "filter"), (2, 140.0, "segment", 0.0, "filter"), (1, 90.0, "box", 0.0, "joint"),
                  (3, 140.0, "segment", 0.0, "joint")]
    cols = int(math.ceil(math.sqrt(len(specs))))
    lanes = []
    hexagon = lib.s2MakePolygon(C.byref(lib.s2ComputeHull(
        (Vec2 * 6)(*[Vec2(0.12 * math.cos(math.pi * m / 3.0), 0.12 * math.sin(math.pi * m / 3.0)) for m in range(6)]), 6)))
    for n, (kind, speed, wall, tilt, exclusion) in enumerate(specs):
        i, j = divmod(n, cols)
        cx, cy = 12.0 * j + 6.0 * (i % 2), 10.0 * i
        bd = default_body_def()
        bd.position = Vec2(cx, cy)
        bd.angle = tilt
        wid = lib.s2CreateBody(world, C.byref(bd))
        sd = default_shape_def()
        if exclusion == "filter":
            sd.filter = capi.Filter(0x0002, 0xFFFFFFFF, 0)
        if wall == "box":
            wall_form = lib.s2MakeBox(PROJECTILE_WALL_HALF_THICKNESS, PROJECTILE_WALL_HALF_LENGTH)
            lib.s2CreatePolygonShape(wid, C.byref(sd), C.byref(wall_form))
        else:
            seg = Segment(Vec2(0.0, -PROJECTILE_WALL_HALF_LENGTH), Vec2(0.0, PROJECTILE_WALL_HALF_LENGTH))
            lib.s2CreateSegmentShape(wid, C.byref(sd), C.byref(seg))
            wall_form = lib.s2MakeCapsule(seg.point1, seg.point2, 0.0)

        pd = default_body_def()
        pd.type = capi.DYNAMIC_BODY
        start = Vec2(cx - 2.5 - 0.17 * (n % 5), cy)
        pd.position = start
        pd.gravityScale = 0.0
        pd.linearVelocity = Vec2(speed, 0.0)
        pd.angle = 0.3 * (n % 4)
        pd.angularVelocity = 2.0 if n % 3 == 0 else 0.0
        pid = lib.s2CreateBody(world, C.byref(pd))
        ps = default_shape_def()
        if exclusion == "filter":
            ps.filter = capi.Filter(0x0001, 0xFFFFFFFF & ~0x0002, 0)
        if kind == 0:
            lib.s2CreateCircleShape(pid, C.byref(ps), C.byref(Circle(Vec2(0.0, 0.0), 0.1)))
            form = capi.Polygon()
            form.count, form.radius = 1, 0.1
        elif kind == 1:
            lib.s2CreateCapsuleShape(pid, C.byref(ps), C.byref(Capsule(Vec2(-0.15, 0.0), Vec2(0.15, 0.0), 0.05)))
            form = lib.s2MakeCapsule(Vec2(-0.15, 0.0), Vec2(0.15, 0.0), 0.05)
        elif kind == 2:
            form = lib.s2MakeBox(0.1, 0.1)
            lib.s2CreatePolygonShape(pid, C.byref(ps), C.byref(form))
        else:
            form = hexagon
            lib.s2CreatePolygonShape(pid, C.byref(ps), C.byref(hexagon))
        if exclusion == "joint" and "s2CreatePrismaticJoint" not in lib.missing:
            jd = capi.default_prismatic_def()
            jd.bodyIdA = wid
            jd.bodyIdB = pid
            jd.localAnchorA = lib.s2Body_GetLocalPoint(wid, start)
            jd.localAnchorB = Vec2(0.0, 0.0)
            jd.localAxisA = Vec2(math.cos(tilt), -math.sin(tilt))
            jd.referenceAngle = pd.angle - tilt
            sc.joints.append(lib.s2CreatePrismaticJoint(world, C.byref(jd)))
        sc.bodies.append(pid)
        lanes.append(dict(body=pid, wall=wid, center=(cx, cy), normal=(math.cos(tilt), math.sin(tilt)),
                          half_length=PROJECTILE_WALL_HALF_LENGTH, passes=exclusion is not None, exclusion=exclusion,
                          form=form, wall_form=wall_form))
    sc.piles["lanes"] = lanes
    return sc


def projectiles_behind(lib: capi.Solver2D, sc: Scene) -> np.ndarray:
    """Per lane of a :func:`projectiles` scene: True where the projectile's centre of mass is past its wall's mid-plane
    within the wall's span, half a metre in from either end."""
    out = []
    for lane in sc.piles["lanes"]:
        p = lib.s2Body_GetPosition(lane["body"])
        dx, dy = p.x - lane["center"][0], p.y - lane["center"][1]
        nx, ny = lane["normal"]
        depth = dx * nx + dy * ny
        along = -dx * ny + dy * nx
        # (half a metre in from the ends: a projectile that slides off a tilted wall and rounds its end is not through it)
        out.append(depth > 0.0 and abs(along) <= lane["half_length"] - 0.5)
    return np.array(out, dtype=bool)


BULLET_TARGETS = ("plank", "kinematic", "block")
BULLET_PLANK_HALF_LENGTH = 2.0
BULLET_PLANK_HALF_THICKNESS = 0.025  # a 0.05 m thick plank
BULLET_PLANK_DENSITY = 2000.0        # 400 kg: a projectile (at most 0.15 kg) stopped at it moves it by mm/s
BULLET_KINEMATIC_SPEED = 0.5         # m/s along the kinematic plank's own length
BULLET_BLOCK_HALF = 0.15             # boxes of the block: 0.3 m, 3 deep and 5 high, touching
BULLET_BLOCK_DENSITY = 2000.0
BULLET_LANE_PITCH = 6.0              # m between lanes: each lane has a row of its own, free past its target


def bullets(lib: capi.Solver2D, solver="TGS_Soft", copies=1, flagged=True, excluded=True) -> Scene:
    """Bullet coverage (s2Body_SetBullet, DESIGN.md §3.12): lanes stacked along y, each a projectile without gravity fired
    along +x (a circle, capsule, box or hexagon at each of PROJECTILE_SPEEDS) at a non-static target, in the manner of
    :func:`projectiles`. Targets (BULLET_TARGETS): a heavy dynamic plank 0.05 m thick without gravity; a kinematic plank of
    the same shape sliding slowly along its own length; a small block of heavy boxes without gravity (3 deep, 5 high), the
    projectile aimed at its middle row. With `flagged` every projectile is a bullet. With `excluded`, three more lanes
    whose projectile must pass its plank in both modes: the plank is itself a bullet (bullet against bullet is not swept), a filter excludes
    the plank, or the projectile is jointed to the plank by a prismatic joint along the flight (the reference has no
    prismatic joint and builds that lane without it). `copies` repeats the lane set.

    sc.piles["lanes"]: per lane a dict with the projectile's body and shape ids (`body`, `shape`), its target's body id
    (`target`; the back middle box of a block), every (body id, shape id) of the target (`targets`), `kind` (one of
    BULLET_TARGETS), `passes`, `exclusion` ("bullet", "filter", "joint" or None),
    `span` (half the extent of the target face that counts, in the target's frame) and the shapes in polygon form (`form`,
    `target_form`)."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"bullets{copies}")
    specs = [(kind, v, target, None) for target in BULLET_TARGETS for kind in range(4) for v in PROJECTILE_SPEEDS] * copies
    if excluded:
        specs += [(0, 140.0, "plank", "bullet"), (2, 140.0, "plank", "filter"), (1, 140.0, "plank", "joint")]
    hexagon = lib.s2MakePolygon(C.byref(lib.s2ComputeHull(
        (Vec2 * 6)(*[Vec2(0.12 * math.cos(math.pi * m / 3.0), 0.12 * math.sin(math.pi * m / 3.0)) for m in range(6)]), 6)))
    lanes = []
    for n, (kind, speed, target, exclusion) in enumerate(specs):
        cy = BULLET_LANE_PITCH * n
        tilt = 0.2 if n % 2 else 0.0
        sd = default_shape_def()
        if exclusion == "filter":
            sd.filter = capi.Filter(0x0002, 0xFFFFFFFF, 0)
        td = default_body_def()
        td.gravityScale = 0.0
        if target == "block":
            td.type = capi.DYNAMIC_BODY
            sd.density = BULLET_BLOCK_DENSITY
            target_form = lib.s2MakeBox(BULLET_BLOCK_HALF, BULLET_BLOCK_HALF)
            tid, targets = None, []
            for col in range(3):
                for row in range(-2, 3):
                    td.position = Vec2(2.0 * BULLET_BLOCK_HALF * col, cy + 2.0 * BULLET_BLOCK_HALF * row)
                    bid = lib.s2CreateBody(world, C.byref(td))
                    targets.append((bid, lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(target_form))))
                    sc.bodies.append(bid)
                    if col == 2 and row == 0:
                        tid = bid  # (the back middle box: a projectile past it went through the whole block)
            span = BULLET_BLOCK_HALF
        else:
            td.position = Vec2(0.0, cy)
            td.angle = tilt
            if target == "plank":
                td.type = capi.DYNAMIC_BODY
                sd.density = BULLET_PLANK_DENSITY
            else:
                td.type = capi.KINEMATIC_BODY
                td.linearVelocity = Vec2(-math.sin(tilt) * BULLET_KINEMATIC_SPEED, math.cos(tilt) * BULLET_KINEMATIC_SPEED)
            tid = lib.s2CreateBody(world, C.byref(td))
            target_form = lib.s2MakeBox(BULLET_PLANK_HALF_THICKNESS, BULLET_PLANK_HALF_LENGTH)
            targets = [(tid, lib.s2CreatePolygonShape(tid, C.byref(sd), C.byref(target_form)))]
            sc.bodies.append(tid)
            # (half a metre in from the ends: a projectile that slides off a tilted plank and rounds its end is not through it)
            span = BULLET_PLANK_HALF_LENGTH - 0.5
        if exclusion == "bullet" and "s2Body_SetBullet" not in lib.missing:
            lib.s2Body_SetBullet(tid, True)

        pd = default_body_def()
        pd.type = capi.DYNAMIC_BODY
        # far enough from the target that no step starts with the two within contact reach: 1.2 m, or more for slow shots
        start = Vec2(-1.2 - 0.17 * (n % 5), cy)
        pd.position = start
        pd.gravityScale = 0.0
        pd.linearVelocity = Vec2(speed, 0.0)
        pd.angle = 0.3 * (n % 4)
        pd.angularVelocity = 2.0 if n % 3 == 0 else 0.0
        pid = lib.s2CreateBody(world, C.byref(pd))
        ps = default_shape_def()
        if exclusion == "filter":
            ps.filter = capi.Filter(0x0001, 0xFFFFFFFF & ~0x0002, 0)
        if kind == 0:
            shape = lib.s2CreateCircleShape(pid, C.byref(ps), C.byref(Circle(Vec2(0.0, 0.0), 0.1)))
            form = capi.Polygon()
            form.count, form.radius = 1, 0.1
        elif kind == 1:
            shape = lib.s2CreateCapsuleShape(pid, C.byref(ps), C.byref(Capsule(Vec2(-0.15, 0.0), Vec2(0.15, 0.0), 0.05)))
            form = lib.s2MakeCapsule(Vec2(-0.15, 0.0), Vec2(0.15, 0.0), 0.05)
        elif kind == 2:
            form = lib.s2MakeBox(0.1, 0.1)
            shape = lib.s2CreatePolygonShape(pid, C.byref(ps), C.byref(form))
        else:
            form = hexagon
            shape = lib.s2CreatePolygonShape(pid, C.byref(ps), C.byref(hexagon))
        if flagged and "s2Body_SetBullet" not in lib.missing:
            lib.s2Body_SetBullet(pid, True)
        if exclusion == "joint" and "s2CreatePrismaticJoint" not in lib.missing:
            jd = capi.default_prismatic_def()
            jd.bodyIdA = tid
            jd.bodyIdB = pid
            jd.localAnchorA = lib.s2Body_GetLocalPoint(tid, start)
            jd.localAnchorB = Vec2(0.0, 0.0)
            jd.localAxisA = Vec2(math.cos(tilt), -math.sin(tilt))
            jd.referenceAngle = pd.angle - tilt
            sc.joints.append(lib.s2CreatePrismaticJoint(world, C.byref(jd)))
        sc.bodies.append(pid)
        lanes.append(dict(body=pid, shape=shape, target=tid, targets=targets, kind=target, passes=exclusion is not None,
                          exclusion=exclusion, span=span, form=form, target_form=target_form))
    sc.piles["lanes"] = lanes
    return sc


def bullets_behind(lib: capi.Solver2D, sc: Scene) -> np.ndarray:
    """Per lane of a :func:`bullets` scene: True where the projectile's centre of mass is past the mid-plane of its target
    at the target's current pose, within the lane's span of that plane."""
    out = []
    for lane in sc.piles["lanes"]:
        p = lib.s2Body_GetPosition(lane["body"])
        local = lib.s2Body_GetLocalPoint(lane["target"], p)
        out.append(local.x > 0.0 and abs(local.y) <= lane["span"])
    return np.array(out, dtype=bool)


HUB_RIDER_PITCH = 0.25  # m between the shapes of one rider
HUB_RIDER_GAP = 0.4     # m between neighbouring riders: their fat boxes (0.1 m margin) stay apart, so they never touch
HUB_LANE_LENGTH = 150.0  # m of riders on one ground lane (on_ground)


def hub_trays(lib: capi.Solver2D, solver="TGS_Soft", trays=(), on_ground=()) -> Scene:
    """Hub bodies with contact counts set exactly, on static ground lanes 4 m apart (each lane its own static box, top face
    at y = -4 * lane), so that no coordinate grows past about half the longest tray:

    * one lane per entry of `trays`: a dynamic tray (a 0.5 m thick box) resting on the lane, with one spaced layer of
      riders on top. An entry lists the riders' shape counts: a rider with k shapes is one body with k shapes in a row,
      0.25 m apart, so it touches its tray k times and nothing else. Riders at even positions are 0.1 m circles created after
      their tray; riders at odd positions are 0.2 m boxes created before it, so the tray is body A of some contacts and
      body B of others. A tray's incidence list is then 1 (its lane) + the sum of its entry.
    * then `on_ground`: one rider per entry resting on the lanes themselves (up to HUB_LANE_LENGTH per lane), each a body
      with exactly that many incident contacts (the static lane does not count).

    ``sc.piles["trays"]`` holds the trays' body ids, ``sc.piles["riders"]`` per tray the riders' ids and
    ``sc.piles["on_ground"]`` those of `on_ground`."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name="hub_trays")
    r, thick = 0.1, 0.25
    sc.piles["trays"], sc.piles["riders"], sc.piles["on_ground"] = [], [], []

    def width(k):
        return HUB_RIDER_PITCH * (k - 1) + 2.0 * r

    def lane(n, length):
        bd = default_body_def()
        bd.position = Vec2(0.0, -4.0 * n - 1.0)
        gid = lib.s2CreateBody(world, C.byref(bd))
        sd = default_shape_def()
        lib.s2CreatePolygonShape(gid, C.byref(sd), C.byref(lib.s2MakeBox(0.5 * length + 1.0, 1.0)))
        sc.bodies.append(gid)

    def rider(x_left, y, k, box):
        bd = default_body_def()
        bd.type = capi.DYNAMIC_BODY
        bd.position = Vec2(x_left + 0.5 * width(k), y + r)
        bid = lib.s2CreateBody(world, C.byref(bd))
        sd = default_shape_def()
        for m in range(k):
            cx = -0.5 * width(k) + r + HUB_RIDER_PITCH * m
            if box:
                poly = lib.s2MakeOffsetBox(r, r, Vec2(cx, 0.0), 0.0)
                lib.s2CreatePolygonShape(bid, C.byref(sd), C.byref(poly))
            else:
                lib.s2CreateCircleShape(bid, C.byref(sd), C.byref(Circle(Vec2(cx, 0.0), r)))
        sc.bodies.append(bid)
        return bid

    n = 0
    for entry in trays:
        span = sum(width(k) + HUB_RIDER_GAP for k in entry) + HUB_RIDER_GAP
        lane(n, span)
        y0 = -4.0 * n
        lefts = []
        cursor = -0.5 * span + HUB_RIDER_GAP
        for k in entry:
            lefts.append(cursor)
            cursor += width(k) + HUB_RIDER_GAP
        ids = [None] * len(entry)
        for m in range(1, len(entry), 2):
            ids[m] = rider(lefts[m], y0 + 2.0 * thick, entry[m], True)
        bd = default_body_def()
        bd.type = capi.DYNAMIC_BODY
        bd.position = Vec2(0.0, y0 + thick)
        tid = lib.s2CreateBody(world, C.byref(bd))
        sd = default_shape_def()
        sd.density = 5.0
        lib.s2CreatePolygonShape(tid, C.byref(sd), C.byref(lib.s2MakeBox(0.5 * span, thick)))
        sc.bodies.append(tid)
        for m in range(0, len(entry), 2):
            ids[m] = rider(lefts[m], y0 + 2.0 * thick, entry[m], False)
        sc.piles["trays"].append(tid)
        sc.piles["riders"].append(ids)
        n += 1
    rows, row = [], []
    for k in on_ground:
        if row and sum(width(j) + HUB_RIDER_GAP for j in row) + width(k) > HUB_LANE_LENGTH:
            rows.append(row)
            row = []
        row.append(k)
    if row:
        rows.append(row)
    for row in rows:
        span = sum(width(k) + HUB_RIDER_GAP for k in row) + HUB_RIDER_GAP
        lane(n, span)
        cursor = -0.5 * span + HUB_RIDER_GAP
        for k in row:
            sc.piles["on_ground"].append(rider(cursor, -4.0 * n, k, False))
            cursor += width(k) + HUB_RIDER_GAP
        n += 1
    return sc


def hub_beam(lib: capi.Solver2D, solver="TGS_Soft", pendulums=8, limits_motor=False, mouse=True) -> Scene:
    """A dynamic beam hung from a static anchor by a revolute joint at each end, with `pendulums` boxes hanging 1 m below it
    on revolute joints, 0.5 m apart (the beam is body A of the even ones and body B of the odd ones), and with `mouse` a
    mouse joint pulling the beam. The beam's incidence list is pendulums + 2 (+ 1); nothing touches anything. No two bobs
    share mass, inertia and centre of mass (half sizes 0.05-0.08 m, densities 0.5-2, centres up to 0.02 m off the origin;
    neighbours stay 0.3 m apart, so their fat boxes never overlap),
    and the beam is created after them, so a row that reads another body's columns reads different values. With
    `limits_motor` the pendulum joints have angle limits and a motor. ``sc.piles["pendulum"]`` holds the indices into
    ``sc.joints`` of the pendulum joints, ``sc.piles["beam"]`` the beam's id."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name=f"hub_beam{pendulums}")
    bd = default_body_def()
    anchor = lib.s2CreateBody(world, C.byref(bd))
    sc.bodies.append(anchor)
    half = 0.25 * pendulums + 0.5
    y = 10.0
    bobs, xs = [], []
    for n in range(pendulums):
        px = -half + 0.5 + 0.5 * n
        bd = default_body_def()
        bd.type = capi.DYNAMIC_BODY
        bd.position = Vec2(px, y - 1.0)
        bob = lib.s2CreateBody(world, C.byref(bd))
        sd = default_shape_def()
        sd.density = 0.5 + 0.25 * (n % 7)
        h = 0.05 + 0.01 * (n % 4)
        lib.s2CreatePolygonShape(bob, C.byref(sd), C.byref(lib.s2MakeOffsetBox(h, h, Vec2(0.01 * (n % 5 - 2), 0.0), 0.0)))
        sc.bodies.append(bob)
        bobs.append(bob)
        xs.append(px)
    bd = default_body_def()
    bd.type = capi.DYNAMIC_BODY
    bd.position = Vec2(0.0, y)
    beam = lib.s2CreateBody(world, C.byref(bd))
    sd = default_shape_def()
    lib.s2CreatePolygonShape(beam, C.byref(sd), C.byref(lib.s2MakeBox(half, 0.1)))
    sc.bodies.append(beam)
    sc.piles["beam"] = beam
    for end, (a, b) in ((-1.0, (anchor, beam)), (1.0, (beam, anchor))):
        jd = default_revolute_def()
        pivot = Vec2(end * half, y)
        jd.bodyIdA, jd.bodyIdB = a, b
        jd.localAnchorA = lib.s2Body_GetLocalPoint(a, pivot)
        jd.localAnchorB = lib.s2Body_GetLocalPoint(b, pivot)
        sc.joints.append(lib.s2CreateRevoluteJoint(world, C.byref(jd)))
    sc.piles["pendulum"] = []
    for n, (bob, px) in enumerate(zip(bobs, xs)):
        a, b = (beam, bob) if n % 2 == 0 else (bob, beam)
        jd = default_revolute_def()
        pivot = Vec2(px, y)
        jd.bodyIdA, jd.bodyIdB = a, b
        jd.localAnchorA = lib.s2Body_GetLocalPoint(a, pivot)
        jd.localAnchorB = lib.s2Body_GetLocalPoint(b, pivot)
        if limits_motor:
            jd.enableLimit = True
            jd.lowerAngle, jd.upperAngle = -0.05, 0.05
            jd.enableMotor = True
            jd.motorSpeed = 0.5 if n % 3 == 0 else -0.25
            jd.maxMotorTorque = 0.5
        sc.piles["pendulum"].append(len(sc.joints))
        sc.joints.append(lib.s2CreateRevoluteJoint(world, C.byref(jd)))
    if mouse:
        md = default_mouse_def()
        md.bodyIdA = anchor
        md.bodyIdB = beam
        md.target = Vec2(0.5, y + 0.25)
        md.hertz = 4.0
        md.dampingRatio = 0.7
        sc.joints.append(lib.s2CreateMouseJoint(world, C.byref(md)))
    return sc


def breakables(lib: capi.Solver2D, solver="TGS_Soft", parts=("weld", "prismatic", "motor")) -> Scene:
    """Breakable joints (DESIGN.md §3.13), about 40 bodies:

    * a plank bridge: ten planks on revolute joints (collideConnected false) between two static posts, a heavy ball
      (15.7 kg) dropped on its middle; breakForce 400 N on every bridge joint;
    * a shelf welded to a static wall (breakTorque 25 N-m), loaded by a growing pile of boxes that rain onto it;
    * a piston on a vertical prismatic joint, thrown up at 20 m/s into its upper limit (breakForce 200 N);
    * a motor joint with a 500 N cap driving its box towards a pose 5 m away (breakForce 100 N: under TGS_Sticky the cap
      holds for the whole step, so the reading is a quarter of it), and a mouse joint whose 5 Hz spring is pulled 5 m off
      its box (breakForce 300 N);
    * one joint of each type holding a box at rest, with thresholds it never reaches (1e6).

    `parts` names the extension joint types the scene contains (the shelf, the piston and the motor joints with their
    held boxes); the revolute and mouse joints are always there. On a library without the extensions (the reference) each weld, prismatic and motor joint is a revolute joint with the
    same bodies, anchors and collideConnected, as in :func:`sliders` and :func:`motors`, so both libraries see the same pairs.
    Thresholds are not applied here: ``sc.piles["break"]`` lists (index into ``sc.joints``, breakForce, breakTorque) and
    :func:`apply_break_thresholds` sets them; ``sc.piles["never"]`` lists the indices of the joints that must hold;
    ``sc.piles["types"]`` names the type of every joint and ``sc.piles["defs"]`` maps the index of each prismatic and motor
    joint to its definition (dicts of s2PrismaticJointDef / s2MotorJointDef fields), so that a test can turn the stand-in
    rows into rows of their own type."""
    world = lib.create_world(solver)
    sc = Scene(lib, world, name="breakables")
    sc.piles.update({"break": [], "never": [], "types": [], "defs": {}})
    has_ext = "s2CreateWeldJoint" not in lib.missing
    gid = _ground(lib, world, 40.0)
    sc.bodies.append(gid)
    sd = default_shape_def()
    sd.density = 1.0

    def body(x, y, hx=0.5, hy=0.5, vy=0.0, radius=0.0, density=1.0, kind=capi.DYNAMIC_BODY):
        bd = default_body_def()
        bd.type = kind
        bd.position = Vec2(x, y)
        bd.linearVelocity = Vec2(0.0, vy)
        bid = lib.s2CreateBody(world, C.byref(bd))
        d = default_shape_def()
        d.density = density
        if radius > 0.0:
            lib.s2CreateCircleShape(bid, C.byref(d), C.byref(Circle(Vec2(0.0, 0.0), radius)))
        else:
            lib.s2CreatePolygonShape(bid, C.byref(d), C.byref(lib.s2MakeBox(hx, hy)))
        sc.bodies.append(bid)
        return bid

    def add(kind, jid, force=0.0, torque=0.0, never=False):
        sc.piles["types"].append(kind)
        if never:
            sc.piles["never"].append(len(sc.joints))
        sc.piles["break"].append((len(sc.joints), force, torque))
        sc.joints.append(jid)

    def revolute(a, b, anchor_a, anchor_b, collide=False):
        jd = default_revolute_def()
        jd.bodyIdA, jd.bodyIdB = a, b
        jd.localAnchorA, jd.localAnchorB = Vec2(*anchor_a), Vec2(*anchor_b)
        jd.collideConnected = collide
        return lib.s2CreateRevoluteJoint(world, C.byref(jd))

    def weld(a, b, anchor_a, anchor_b):
        if not has_ext:
            return revolute(a, b, anchor_a, anchor_b)
        jd = capi.default_weld_def()
        jd.bodyIdA, jd.bodyIdB = a, b
        jd.localAnchorA, jd.localAnchorB = Vec2(*anchor_a), Vec2(*anchor_b)
        return lib.s2CreateWeldJoint(world, C.byref(jd))

    def prismatic(a, b, anchor_a, lower, upper):
        sc.piles["defs"][len(sc.joints)] = dict(lowerTranslation=lower, upperTranslation=upper, localAxisA=(0.0, 1.0))
        if not has_ext:
            return revolute(a, b, anchor_a, (0.0, 0.0))
        jd = capi.default_prismatic_def()
        jd.bodyIdA, jd.bodyIdB = a, b
        jd.localAnchorA = Vec2(*anchor_a)
        jd.localAxisA = Vec2(0.0, 1.0)
        jd.enableLimit = True
        jd.lowerTranslation, jd.upperTranslation = lower, upper
        return lib.s2CreatePrismaticJoint(world, C.byref(jd))

    def motor(a, b, offset, max_force):
        sc.piles["defs"][len(sc.joints)] = dict(linearOffset=offset, maxForce=max_force, maxTorque=max_force)
        if not has_ext:
            return revolute(a, b, offset, (0.0, 0.0))
        jd = capi.default_motor_def()
        jd.bodyIdA, jd.bodyIdB = a, b
        jd.linearOffset = Vec2(*offset)
        jd.maxForce, jd.maxTorque = max_force, max_force
        return lib.s2CreateMotorJoint(world, C.byref(jd))

    def mouse(b, at, target):
        # a mouse joint is anchored where it is created: created on the box, then pulled to its target
        jd = default_mouse_def()
        jd.bodyIdA, jd.bodyIdB = gid, b
        jd.target = Vec2(*at)
        jd.hertz, jd.dampingRatio = 5.0, 0.7
        jid = lib.s2CreateMouseJoint(world, C.byref(jd))
        lib.s2MouseJoint_SetTarget(jid, Vec2(*target))
        return jid

    # the plank bridge between two posts: post tops at y = 4, planks 1 m long
    left, right = body(-16.5, 2.0, 0.5, 2.0, kind=capi.STATIC_BODY), body(-5.5, 2.0, 0.5, 2.0, kind=capi.STATIC_BODY)
    prev, prev_anchor = left, (0.5, 2.0)
    for k in range(10):
        plank = body(-15.5 + k, 4.0, 0.5, 0.125)
        add("revolute", revolute(prev, plank, prev_anchor, (-0.5, 0.0)), force=400.0)
        prev, prev_anchor = plank, (0.5, 0.0)
    add("revolute", revolute(prev, right, prev_anchor, (-0.5, 2.0)), force=400.0)
    body(-11.0, 9.0, radius=0.5, density=20.0)

    if "weld" in parts:
        # the welded shelf on a wall, and its pile
        wall = body(-1.0, 3.0, 0.25, 3.0, kind=capi.STATIC_BODY)
        shelf = body(0.75, 3.0, 1.5, 0.1)
        add("weld", weld(wall, shelf, (0.25, 0.0), (-1.5, 0.0)), torque=25.0)
        for k in range(6):
            body(1.25, 4.0 + 1.5 * k, 0.3, 0.3, density=2.0)

    if "prismatic" in parts:
        # the piston: a static guide, a 1 kg block thrown up into its upper limit
        guide = body(5.0, 1.0, 0.25, 1.0, kind=capi.STATIC_BODY)
        block = body(6.0, 1.0, 0.5, 0.5, vy=20.0)
        add("prismatic", prismatic(guide, block, (1.0, 0.0), -0.5, 1.5), force=200.0)

    if "motor" in parts:
        # the motor joint driving its box 5 m off
        post = body(10.0, 1.0, 0.25, 1.0, kind=capi.STATIC_BODY)
        driven = body(11.0, 3.0, 0.5, 0.5)
        add("motor", motor(post, driven, (6.0, 2.0), 500.0), force=100.0)
    # the mouse joint pulled 5 m off its box
    pulled = body(14.0, 2.0, 0.5, 0.5)
    add("mouse", mouse(pulled, (14.0, 2.0), (19.0, 2.0)), force=300.0)

    # one joint of each type holding a box at rest, far below its thresholds
    hanger = body(25.0, 8.0, 4.0, 0.25, kind=capi.STATIC_BODY)
    boxes = [body(22.0 + 1.5 * k, 6.5, 0.25, 0.25) for k in range(5)]
    add("revolute", revolute(hanger, boxes[0], (-3.0, -1.5), (0.0, 0.0)), force=1e6, torque=1e6, never=True)
    if "weld" in parts:
        add("weld", weld(hanger, boxes[1], (-1.5, -1.5), (0.0, 0.0)), force=1e6, torque=1e6, never=True)
    if "prismatic" in parts:
        add("prismatic", prismatic(hanger, boxes[2], (0.0, -1.5), -0.5, 0.5), force=1e6, torque=1e6, never=True)
    if "motor" in parts:
        add("motor", motor(hanger, boxes[3], (1.5, -1.5), 100.0), force=1e6, torque=1e6, never=True)
    add("mouse", mouse(boxes[4], (28.0, 6.5), (28.0, 6.5)), force=1e6, torque=1e6, never=True)
    return sc


def apply_break_thresholds(sc: Scene):
    """Sets the thresholds :func:`breakables` recorded (a library without s2Joint_SetBreakForce is left as it is)."""
    if "s2Joint_SetBreakForce" in sc.lib.missing:
        return
    for index, force, torque in sc.piles["break"]:
        if force > 0.0:
            sc.lib.s2Joint_SetBreakForce(sc.joints[index], force)
        if torque > 0.0:
            sc.lib.s2Joint_SetBreakTorque(sc.joints[index], torque)
