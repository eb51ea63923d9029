"""ctypes mirror of the solver2d public C API (reference include/solver2d/solver2d.h:22-70, types.h, id.h,
joint_types.h, geometry.h).

The same binding drives both libraries, because both export the same C API:

* ``solver2d_b200/libsolver2d.so`` — this repo's GPU library (host C + CUDA behind it), and
* ``oracle/_ref/libsolver2d_ref.so`` — the unmodified reference compiled by ``oracle/Makefile`` (tests/bench only).

That is the drop-in claim in executable form: a scene script written against :class:`Solver2D` runs unchanged on
either. Nothing in this module computes anything; it only marshals arguments.
"""
from __future__ import annotations

import ctypes as C
import os

# --------------------------------------------------------------------------------------------------------------
# POD types (layout-compatible with reference include/solver2d/types.h:31-163, id.h:12-47)
# --------------------------------------------------------------------------------------------------------------


class Vec2(C.Structure):
    _fields_ = [("x", C.c_float), ("y", C.c_float)]

    def __iter__(self):
        yield self.x
        yield self.y


class Rot(C.Structure):
    _fields_ = [("s", C.c_float), ("c", C.c_float)]


class Box(C.Structure):
    _fields_ = [("lowerBound", Vec2), ("upperBound", Vec2)]


class WorldId(C.Structure):
    _fields_ = [("index", C.c_int16), ("revision", C.c_uint16)]


class BodyId(C.Structure):
    _fields_ = [("index", C.c_int32), ("world", C.c_int16), ("revision", C.c_uint16)]


class ShapeId(C.Structure):
    _fields_ = [("index", C.c_int32), ("world", C.c_int16), ("revision", C.c_uint16)]


class JointId(C.Structure):
    _fields_ = [("index", C.c_int32), ("world", C.c_int16), ("revision", C.c_uint16)]


class WorldDef(C.Structure):
    _fields_ = [("solverType", C.c_int)]


class BodyDef(C.Structure):
    _fields_ = [
        ("type", C.c_int),
        ("position", Vec2),
        ("angle", C.c_float),
        ("linearVelocity", Vec2),
        ("angularVelocity", C.c_float),
        ("linearDamping", C.c_float),
        ("angularDamping", C.c_float),
        ("gravityScale", C.c_float),
        ("userData", C.c_void_p),
    ]


class Filter(C.Structure):
    _fields_ = [("categoryBits", C.c_uint32), ("maskBits", C.c_uint32), ("groupIndex", C.c_int32)]


class ShapeDef(C.Structure):
    _fields_ = [
        ("userData", C.c_void_p),
        ("friction", C.c_float),
        ("restitution", C.c_float),
        ("density", C.c_float),
        ("filter", Filter),
    ]


MAX_POLYGON_VERTICES = 8


class Polygon(C.Structure):
    _fields_ = [
        ("vertices", Vec2 * MAX_POLYGON_VERTICES),
        ("normals", Vec2 * MAX_POLYGON_VERTICES),
        ("radius", C.c_float),
        ("count", C.c_int32),
    ]


class Circle(C.Structure):
    _fields_ = [("point", Vec2), ("radius", C.c_float)]


class Capsule(C.Structure):
    _fields_ = [("point1", Vec2), ("point2", Vec2), ("radius", C.c_float)]


class Segment(C.Structure):
    _fields_ = [("point1", Vec2), ("point2", Vec2)]


class Hull(C.Structure):
    _fields_ = [("points", Vec2 * MAX_POLYGON_VERTICES), ("count", C.c_int32)]


class MouseJointDef(C.Structure):
    _fields_ = [
        ("bodyIdA", BodyId),
        ("bodyIdB", BodyId),
        ("target", Vec2),
        ("hertz", C.c_float),
        ("dampingRatio", C.c_float),
    ]


class RevoluteJointDef(C.Structure):
    _fields_ = [
        ("bodyIdA", BodyId),
        ("bodyIdB", BodyId),
        ("localAnchorA", Vec2),
        ("localAnchorB", Vec2),
        ("referenceAngle", C.c_float),
        ("enableLimit", C.c_bool),
        ("lowerAngle", C.c_float),
        ("upperAngle", C.c_float),
        ("enableMotor", C.c_bool),
        ("motorSpeed", C.c_float),
        ("maxMotorTorque", C.c_float),
        ("drawSize", C.c_float),
        ("collideConnected", C.c_bool),
    ]


class Statistics(C.Structure):
    _fields_ = [
        ("bodyCount", C.c_int32),
        ("contactCount", C.c_int32),
        ("jointCount", C.c_int32),
        ("proxyCount", C.c_int32),
        ("treeHeight", C.c_int32),
        ("stackCapacity", C.c_int32),
        ("stackUsed", C.c_int32),
    ]


# s2SolverType (reference include/solver2d/types.h:75-88) — enum order is ABI.
SOLVER_TYPES = [
    "Jacobi",
    "PGS",
    "PGS_NGS",
    "PGS_NGS_Block",
    "PGS_Soft",
    "SoftStep",
    "TGS_Sticky",
    "TGS_Soft",
    "TGS_NGS",
    "XPBD",
]
SOLVER = {name: i for i, name in enumerate(SOLVER_TYPES)}

STATIC_BODY, KINEMATIC_BODY, DYNAMIC_BODY = 0, 1, 2

# substepping variants use h = dt / iterations (reference src/world.c:186-201)
SUBSTEPPING = {"XPBD", "TGS_Soft", "TGS_Sticky", "TGS_NGS", "SoftStep"}


def default_body_def() -> BodyDef:
    """s2_defaultBodyDef (reference include/solver2d/types.h:120-130)."""
    d = BodyDef()
    d.type = STATIC_BODY
    d.gravityScale = 1.0
    return d


def default_shape_def() -> ShapeDef:
    """s2_defaultShapeDef (reference include/solver2d/types.h:150-156)."""
    d = ShapeDef()
    d.friction = 0.6
    d.restitution = 0.0
    d.density = 1.0
    d.filter = Filter(0x00000001, 0xFFFFFFFF, 0)
    return d


def default_revolute_def() -> RevoluteJointDef:
    """s2DefaultRevoluteJointDef (reference include/solver2d/joint_types.h:80-97)."""
    d = RevoluteJointDef()
    d.bodyIdA = BodyId(-1, -1, 0)
    d.bodyIdB = BodyId(-1, -1, 0)
    d.drawSize = 1.0
    return d


def default_mouse_def() -> MouseJointDef:
    """s2DefaultMouseJointDef (reference include/solver2d/joint_types.h:28-37)."""
    d = MouseJointDef()
    d.bodyIdA = BodyId(-1, -1, 0)
    d.bodyIdB = BodyId(-1, -1, 0)
    d.hertz = 15.0
    d.dampingRatio = 1.0
    return d


_API = {
    # name: (restype, [argtypes])
    "s2CreateWorld": (WorldId, [C.POINTER(WorldDef)]),
    "s2DestroyWorld": (None, [WorldId]),
    "s2World_Step": (None, [WorldId, C.c_float, C.c_int32, C.c_int32, C.c_bool]),
    "s2World_GetStatistics": (Statistics, [WorldId]),
    "s2CreateBody": (BodyId, [WorldId, C.POINTER(BodyDef)]),
    "s2DestroyBody": (None, [BodyId]),
    "s2Body_GetPosition": (Vec2, [BodyId]),
    "s2Body_GetAngle": (C.c_float, [BodyId]),
    "s2Body_GetLocalPoint": (Vec2, [BodyId, Vec2]),
    "s2Body_SetLinearVelocity": (None, [BodyId, Vec2]),
    "s2Body_SetAngularVelocity": (None, [BodyId, C.c_float]),
    "s2Body_ApplyForceToCenter": (None, [BodyId, Vec2]),
    "s2Body_ApplyLinearImpulse": (None, [BodyId, Vec2, Vec2]),
    "s2Body_GetType": (C.c_int, [BodyId]),
    "s2Body_GetMass": (C.c_float, [BodyId]),
    "s2CreateCircleShape": (ShapeId, [BodyId, C.POINTER(ShapeDef), C.POINTER(Circle)]),
    "s2CreateSegmentShape": (ShapeId, [BodyId, C.POINTER(ShapeDef), C.POINTER(Segment)]),
    "s2CreateCapsuleShape": (ShapeId, [BodyId, C.POINTER(ShapeDef), C.POINTER(Capsule)]),
    "s2CreatePolygonShape": (ShapeId, [BodyId, C.POINTER(ShapeDef), C.POINTER(Polygon)]),
    "s2Shape_GetBody": (BodyId, [ShapeId]),
    "s2Shape_TestPoint": (C.c_bool, [ShapeId, Vec2]),
    "s2CreateMouseJoint": (JointId, [WorldId, C.POINTER(MouseJointDef)]),
    "s2CreateRevoluteJoint": (JointId, [WorldId, C.POINTER(RevoluteJointDef)]),
    "s2DestroyJoint": (None, [JointId]),
    "s2MouseJoint_SetTarget": (None, [JointId, Vec2]),
    "s2RevoluteJoint_EnableLimit": (None, [JointId, C.c_bool]),
    "s2RevoluteJoint_EnableMotor": (None, [JointId, C.c_bool]),
    "s2RevoluteJoint_SetMotorSpeed": (None, [JointId, C.c_float]),
    "s2RevoluteJoint_GetMotorTorque": (C.c_float, [JointId, C.c_float]),
    "s2MakeBox": (Polygon, [C.c_float, C.c_float]),
    "s2MakeSquare": (Polygon, [C.c_float]),
    "s2MakeOffsetBox": (Polygon, [C.c_float, C.c_float, Vec2, C.c_float]),
    "s2MakeCapsule": (Polygon, [Vec2, Vec2, C.c_float]),
    "s2MakePolygon": (Polygon, [C.POINTER(Hull)]),
    "s2ComputeHull": (Hull, [C.POINTER(Vec2), C.c_int32]),
    # extensions (include/solver2d_b200.h): restitution is off unless a world enables it
    "s2World_EnableRestitution": (None, [WorldId, C.c_bool]),
    "s2World_SetRestitutionThreshold": (None, [WorldId, C.c_float]),
}

class Transform(C.Structure):
    _fields_ = [("p", Vec2), ("q", Rot)]


class ManifoldPoint(C.Structure):
    _fields_ = [("localAnchorA", Vec2), ("localAnchorB", Vec2), ("frictionAnchorA", Vec2), ("frictionAnchorB", Vec2),
                ("frictionNormalA", Vec2), ("frictionNormalB", Vec2), ("separation", C.c_float),
                ("normalImpulse", C.c_float), ("tangentImpulse", C.c_float), ("id", C.c_uint16), ("persisted", C.c_bool)]


class Manifold(C.Structure):
    _fields_ = [("points", ManifoldPoint * 2), ("normal", Vec2), ("pointCount", C.c_int32),
                ("constraintIndex", C.c_int32), ("frictionPersisted", C.c_bool)]


class DistanceCache(C.Structure):
    _fields_ = [("metric", C.c_float), ("count", C.c_uint16), ("indexA", C.c_uint8 * 3), ("indexB", C.c_uint8 * 3)]


class MassData(C.Structure):
    _fields_ = [("mass", C.c_float), ("center", Vec2), ("I", C.c_float)]


# host-callable geometry / narrow-phase API (reference include/solver2d/manifold.h, geometry.h)
_API.update({
    "s2CollideCircles": (Manifold, [C.POINTER(Circle), Transform, C.POINTER(Circle), Transform]),
    "s2CollideCapsuleAndCircle": (Manifold, [C.POINTER(Capsule), Transform, C.POINTER(Circle), Transform]),
    "s2CollideSegmentAndCircle": (Manifold, [C.POINTER(Segment), Transform, C.POINTER(Circle), Transform]),
    "s2CollidePolygonAndCircle": (Manifold, [C.POINTER(Polygon), Transform, C.POINTER(Circle), Transform]),
    "s2CollideCapsules": (Manifold, [C.POINTER(Capsule), Transform, C.POINTER(Capsule), Transform, C.POINTER(DistanceCache)]),
    "s2CollideSegmentAndCapsule": (Manifold, [C.POINTER(Segment), Transform, C.POINTER(Capsule), Transform,
                                              C.POINTER(DistanceCache)]),
    "s2CollidePolygonAndCapsule": (Manifold, [C.POINTER(Polygon), Transform, C.POINTER(Capsule), Transform,
                                              C.POINTER(DistanceCache)]),
    "s2CollidePolygons": (Manifold, [C.POINTER(Polygon), Transform, C.POINTER(Polygon), Transform, C.POINTER(DistanceCache)]),
    "s2CollideSegmentAndPolygon": (Manifold, [C.POINTER(Segment), Transform, C.POINTER(Polygon), Transform,
                                              C.POINTER(DistanceCache)]),
    "s2ComputePolygonMass": (MassData, [C.POINTER(Polygon), C.c_float]),
    "s2ComputeCapsuleMass": (MassData, [C.POINTER(Capsule), C.c_float]),
    "s2ComputeCircleMass": (MassData, [C.POINTER(Circle), C.c_float]),
    "s2ComputePolygonAABB": (Box, [C.POINTER(Polygon), Transform]),
    "s2PointInPolygon": (C.c_bool, [Vec2, C.POINTER(Polygon)]),
    "s2MakeRoundedBox": (Polygon, [C.c_float, C.c_float, C.c_float]),
})

QUERY_CALLBACK = C.CFUNCTYPE(C.c_bool, ShapeId, C.c_void_p)


class Solver2D:
    """A loaded solver2d-API library (ours or the reference)."""

    def __init__(self, path: str):
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.path = path
        self.lib = C.CDLL(path, mode=C.RTLD_GLOBAL if False else C.RTLD_LOCAL)
        self.missing = []
        for name, (res, args) in _API.items():
            try:
                fn = getattr(self.lib, name)
            except AttributeError:
                self.missing.append(name)
                continue
            fn.restype = res
            fn.argtypes = args
            setattr(self, name, fn)
        try:
            fn = self.lib.s2World_QueryAABB
            fn.restype = None
            fn.argtypes = [WorldId, Box, QUERY_CALLBACK, C.c_void_p]
            self.s2World_QueryAABB = fn
        except AttributeError:
            self.missing.append("s2World_QueryAABB")

    # -- small conveniences used by the scene recipes ---------------------------------------------------------
    def create_world(self, solver: str | int) -> WorldId:
        d = WorldDef()
        d.solverType = SOLVER[solver] if isinstance(solver, str) else int(solver)
        wid = self.s2CreateWorld(C.byref(d))
        if wid.index < 0:
            raise RuntimeError("s2CreateWorld: no free world slot")
        return wid

    def step(self, wid: WorldId, dt: float, vel_iters: int, pos_iters: int, warm_start: bool = True) -> None:
        self.s2World_Step(wid, dt, vel_iters, pos_iters, warm_start)
