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


class WeldJointDef(C.Structure):
    """s2WeldJointDef (include/solver2d_b200.h): an extension, absent from the reference."""
    _fields_ = [
        ("bodyIdA", BodyId),
        ("bodyIdB", BodyId),
        ("localAnchorA", Vec2),
        ("localAnchorB", Vec2),
        ("referenceAngle", C.c_float),
        ("drawSize", C.c_float),
        ("collideConnected", C.c_bool),
        ("linearHertz", C.c_float),
        ("linearDampingRatio", C.c_float),
        ("angularHertz", C.c_float),
        ("angularDampingRatio", C.c_float),
    ]


class PrismaticJointDef(C.Structure):
    """s2PrismaticJointDef (include/solver2d_b200.h): an extension, absent from the reference."""
    _fields_ = [
        ("bodyIdA", BodyId),
        ("bodyIdB", BodyId),
        ("localAnchorA", Vec2),
        ("localAnchorB", Vec2),
        ("localAxisA", Vec2),
        ("referenceAngle", C.c_float),
        ("enableLimit", C.c_bool),
        ("lowerTranslation", C.c_float),
        ("upperTranslation", C.c_float),
        ("enableMotor", C.c_bool),
        ("motorSpeed", C.c_float),
        ("maxMotorForce", C.c_float),
        ("drawSize", C.c_float),
        ("collideConnected", C.c_bool),
        ("enableSpring", C.c_bool),
        ("hertz", C.c_float),
        ("dampingRatio", C.c_float),
    ]


class DistanceJointDef(C.Structure):
    """s2DistanceJointDef (include/solver2d_b200.h): an extension, absent from the reference."""
    _fields_ = [
        ("bodyIdA", BodyId),
        ("bodyIdB", BodyId),
        ("localAnchorA", Vec2),
        ("localAnchorB", Vec2),
        ("length", C.c_float),
        ("enableSpring", C.c_bool),
        ("hertz", C.c_float),
        ("dampingRatio", C.c_float),
        ("enableLimit", C.c_bool),
        ("minLength", C.c_float),
        ("maxLength", C.c_float),
        ("enableMotor", C.c_bool),
        ("maxMotorForce", C.c_float),
        ("motorSpeed", C.c_float),
        ("collideConnected", C.c_bool),
    ]


class WheelJointDef(C.Structure):
    """s2WheelJointDef (include/solver2d_b200.h): an extension, absent from the reference."""
    _fields_ = [
        ("bodyIdA", BodyId),
        ("bodyIdB", BodyId),
        ("localAnchorA", Vec2),
        ("localAnchorB", Vec2),
        ("localAxisA", Vec2),
        ("enableSpring", C.c_bool),
        ("hertz", C.c_float),
        ("dampingRatio", C.c_float),
        ("enableLimit", C.c_bool),
        ("lowerTranslation", C.c_float),
        ("upperTranslation", C.c_float),
        ("enableMotor", C.c_bool),
        ("maxMotorTorque", C.c_float),
        ("motorSpeed", C.c_float),
        ("collideConnected", C.c_bool),
    ]


class PulleyJointDef(C.Structure):
    """s2PulleyJointDef (include/solver2d_b200.h): an extension, absent from the reference."""
    _fields_ = [
        ("bodyIdA", BodyId),
        ("bodyIdB", BodyId),
        ("groundAnchorA", Vec2),
        ("groundAnchorB", Vec2),
        ("localAnchorA", Vec2),
        ("localAnchorB", Vec2),
        ("lengthA", C.c_float),
        ("lengthB", C.c_float),
        ("ratio", C.c_float),
        ("collideConnected", C.c_bool),
    ]


class GearJointDef(C.Structure):
    """s2GearJointDef (include/solver2d_b200.h): an extension, absent from the reference."""
    _fields_ = [
        ("jointId1", JointId),
        ("jointId2", JointId),
        ("ratio", C.c_float),
        ("collideConnected", C.c_bool),
    ]


class MotorJointDef(C.Structure):
    """s2MotorJointDef (include/solver2d_b200.h): an extension, absent from the reference."""
    _fields_ = [
        ("bodyIdA", BodyId),
        ("bodyIdB", BodyId),
        ("linearOffset", Vec2),
        ("angularOffset", C.c_float),
        ("maxForce", C.c_float),
        ("maxTorque", C.c_float),
        ("correctionFactor", C.c_float),
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


def default_weld_def() -> WeldJointDef:
    """s2DefaultWeldJointDef (include/solver2d_b200.h)."""
    d = WeldJointDef()
    d.bodyIdA = BodyId(-1, -1, 0)
    d.bodyIdB = BodyId(-1, -1, 0)
    d.drawSize = 1.0
    # a rigid weld: hertz 0 on both parts (DESIGN.md §3.15)
    d.linearHertz = d.linearDampingRatio = d.angularHertz = d.angularDampingRatio = 0.0
    return d


def default_prismatic_def() -> PrismaticJointDef:
    """s2DefaultPrismaticJointDef (include/solver2d_b200.h)."""
    d = PrismaticJointDef()
    d.bodyIdA = BodyId(-1, -1, 0)
    d.bodyIdB = BodyId(-1, -1, 0)
    d.localAxisA = Vec2(1.0, 0.0)
    d.drawSize = 1.0
    return d


def default_distance_def() -> DistanceJointDef:
    """s2DefaultDistanceJointDef (include/solver2d_b200.h)."""
    d = DistanceJointDef()
    d.bodyIdA = BodyId(-1, -1, 0)
    d.bodyIdB = BodyId(-1, -1, 0)
    d.length = 1.0
    d.maxLength = 100000.0  # s2_huge
    return d


def default_wheel_def() -> WheelJointDef:
    """s2DefaultWheelJointDef (include/solver2d_b200.h): Box2D v3's defaults."""
    d = WheelJointDef()
    d.bodyIdA = BodyId(-1, -1, 0)
    d.bodyIdB = BodyId(-1, -1, 0)
    d.localAxisA = Vec2(0.0, 1.0)
    d.enableSpring = True
    d.hertz = 1.0
    d.dampingRatio = 0.7
    return d


def default_pulley_def() -> PulleyJointDef:
    """s2DefaultPulleyJointDef (include/solver2d_b200.h): Box2D 2.4's defaults, collideConnected on."""
    d = PulleyJointDef()
    d.bodyIdA = BodyId(-1, -1, 0)
    d.bodyIdB = BodyId(-1, -1, 0)
    d.groundAnchorA = Vec2(-1.0, 1.0)
    d.groundAnchorB = Vec2(1.0, 1.0)
    d.localAnchorA = Vec2(-1.0, 0.0)
    d.localAnchorB = Vec2(1.0, 0.0)
    d.ratio = 1.0
    d.collideConnected = True
    return d


def default_gear_def() -> GearJointDef:
    """s2DefaultGearJointDef (include/solver2d_b200.h): Box2D 2.4's defaults, ratio 1, collideConnected off."""
    d = GearJointDef()
    d.jointId1 = JointId(-1, -1, 0)
    d.jointId2 = JointId(-1, -1, 0)
    d.ratio = 1.0
    return d


def default_motor_def() -> MotorJointDef:
    """s2DefaultMotorJointDef (include/solver2d_b200.h)."""
    d = MotorJointDef()
    d.bodyIdA = BodyId(-1, -1, 0)
    d.bodyIdB = BodyId(-1, -1, 0)
    d.maxForce = 1.0
    d.maxTorque = 1.0
    d.correctionFactor = 0.3
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
    "s2CreateWeldJoint": (JointId, [WorldId, C.POINTER(WeldJointDef)]),
    # soft weld (DESIGN.md §3.15)
    "s2WeldJoint_SetLinearHertz": (None, [JointId, C.c_float]),
    "s2WeldJoint_SetLinearDampingRatio": (None, [JointId, C.c_float]),
    "s2WeldJoint_SetAngularHertz": (None, [JointId, C.c_float]),
    "s2WeldJoint_SetAngularDampingRatio": (None, [JointId, C.c_float]),
    "s2WeldJoint_GetLinearHertz": (C.c_float, [JointId]),
    "s2WeldJoint_GetLinearDampingRatio": (C.c_float, [JointId]),
    "s2WeldJoint_GetAngularHertz": (C.c_float, [JointId]),
    "s2WeldJoint_GetAngularDampingRatio": (C.c_float, [JointId]),
    "s2CreatePrismaticJoint": (JointId, [WorldId, C.POINTER(PrismaticJointDef)]),
    "s2PrismaticJoint_EnableLimit": (None, [JointId, C.c_bool]),
    "s2PrismaticJoint_SetLimits": (None, [JointId, C.c_float, C.c_float]),
    "s2PrismaticJoint_EnableMotor": (None, [JointId, C.c_bool]),
    "s2PrismaticJoint_SetMotorSpeed": (None, [JointId, C.c_float]),
    "s2PrismaticJoint_GetMotorForce": (C.c_float, [JointId, C.c_float]),
    "s2PrismaticJoint_GetTranslation": (C.c_float, [JointId]),
    # distance joint (DESIGN.md §3.16)
    "s2CreateDistanceJoint": (JointId, [WorldId, C.POINTER(DistanceJointDef)]),
    "s2DistanceJoint_SetLength": (None, [JointId, C.c_float]),
    "s2DistanceJoint_GetLength": (C.c_float, [JointId]),
    "s2DistanceJoint_EnableLimit": (None, [JointId, C.c_bool]),
    "s2DistanceJoint_SetLengthRange": (None, [JointId, C.c_float, C.c_float]),
    "s2DistanceJoint_GetMinLength": (C.c_float, [JointId]),
    "s2DistanceJoint_GetMaxLength": (C.c_float, [JointId]),
    "s2DistanceJoint_EnableSpring": (None, [JointId, C.c_bool]),
    "s2DistanceJoint_SetSpringHertz": (None, [JointId, C.c_float]),
    "s2DistanceJoint_SetSpringDampingRatio": (None, [JointId, C.c_float]),
    "s2DistanceJoint_EnableMotor": (None, [JointId, C.c_bool]),
    "s2DistanceJoint_SetMotorSpeed": (None, [JointId, C.c_float]),
    "s2DistanceJoint_SetMaxMotorForce": (None, [JointId, C.c_float]),
    "s2DistanceJoint_GetMotorForce": (C.c_float, [JointId, C.c_float]),
    "s2DistanceJoint_GetCurrentLength": (C.c_float, [JointId]),
    # wheel joint (DESIGN.md §3.17)
    "s2CreateWheelJoint": (JointId, [WorldId, C.POINTER(WheelJointDef)]),
    "s2WheelJoint_EnableSpring": (None, [JointId, C.c_bool]),
    "s2WheelJoint_SetSpringHertz": (None, [JointId, C.c_float]),
    "s2WheelJoint_SetSpringDampingRatio": (None, [JointId, C.c_float]),
    "s2WheelJoint_EnableLimit": (None, [JointId, C.c_bool]),
    "s2WheelJoint_SetLimits": (None, [JointId, C.c_float, C.c_float]),
    "s2WheelJoint_EnableMotor": (None, [JointId, C.c_bool]),
    "s2WheelJoint_SetMotorSpeed": (None, [JointId, C.c_float]),
    "s2WheelJoint_SetMaxMotorTorque": (None, [JointId, C.c_float]),
    "s2WheelJoint_GetMotorTorque": (C.c_float, [JointId, C.c_float]),
    "s2WheelJoint_GetTranslation": (C.c_float, [JointId]),
    # pulley joint (DESIGN.md §3.18)
    "s2CreatePulleyJoint": (JointId, [WorldId, C.POINTER(PulleyJointDef)]),
    "s2PulleyJoint_GetGroundAnchorA": (Vec2, [JointId]),
    "s2PulleyJoint_GetGroundAnchorB": (Vec2, [JointId]),
    "s2PulleyJoint_GetLengthA": (C.c_float, [JointId]),
    "s2PulleyJoint_GetLengthB": (C.c_float, [JointId]),
    "s2PulleyJoint_GetRatio": (C.c_float, [JointId]),
    "s2PulleyJoint_GetCurrentLengthA": (C.c_float, [JointId]),
    "s2PulleyJoint_GetCurrentLengthB": (C.c_float, [JointId]),
    # gear joint (DESIGN.md §3.19)
    "s2CreateGearJoint": (JointId, [WorldId, C.POINTER(GearJointDef)]),
    "s2GearJoint_GetJoint1": (JointId, [JointId]),
    "s2GearJoint_GetJoint2": (JointId, [JointId]),
    "s2GearJoint_GetRatio": (C.c_float, [JointId]),
    # joint springs (DESIGN.md §3.14)
    "s2PrismaticJoint_EnableSpring": (None, [JointId, C.c_bool]),
    "s2PrismaticJoint_SetSpringHertz": (None, [JointId, C.c_float]),
    "s2PrismaticJoint_SetSpringDampingRatio": (None, [JointId, C.c_float]),
    "s2RevoluteJoint_EnableSpring": (None, [JointId, C.c_bool]),
    "s2RevoluteJoint_SetSpringHertz": (None, [JointId, C.c_float]),
    "s2RevoluteJoint_SetSpringDampingRatio": (None, [JointId, C.c_float]),
    "s2CreateMotorJoint": (JointId, [WorldId, C.POINTER(MotorJointDef)]),
    "s2MotorJoint_SetLinearOffset": (None, [JointId, Vec2]),
    "s2MotorJoint_GetLinearOffset": (Vec2, [JointId]),
    "s2MotorJoint_SetAngularOffset": (None, [JointId, C.c_float]),
    "s2MotorJoint_GetAngularOffset": (C.c_float, [JointId]),
    "s2MotorJoint_SetMaxForce": (None, [JointId, C.c_float]),
    "s2MotorJoint_SetMaxTorque": (None, [JointId, C.c_float]),
    "s2MotorJoint_SetCorrectionFactor": (None, [JointId, C.c_float]),
    "s2MotorJoint_GetConstraintForce": (Vec2, [JointId, C.c_float]),
    "s2MotorJoint_GetConstraintTorque": (C.c_float, [JointId, C.c_float]),
    # indices (int32 per joint), offsets (x, y, angle per joint), count
    "s2World_SetMotorJointOffsets": (C.c_bool, [WorldId, C.c_void_p, C.c_void_p, C.c_int32]),
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


class DistanceProxy(C.Structure):
    _fields_ = [("vertices", Vec2 * MAX_POLYGON_VERTICES), ("count", C.c_int32), ("radius", C.c_float)]


class DistanceInput(C.Structure):
    _fields_ = [("proxyA", DistanceProxy), ("proxyB", DistanceProxy), ("transformA", Transform),
                ("transformB", Transform), ("useRadii", C.c_bool)]


class DistanceOutput(C.Structure):
    _fields_ = [("pointA", Vec2), ("pointB", Vec2), ("distance", C.c_float), ("iterations", C.c_int32)]


class Sweep(C.Structure):
    """s2Sweep (include/solver2d_b200.h): centre c1 -> c2 linearly, rotation q1 -> q2 by normalised lerp."""
    _fields_ = [("localCenter", Vec2), ("c1", Vec2), ("c2", Vec2), ("q1", Rot), ("q2", Rot)]


class TOIInput(C.Structure):
    _fields_ = [("proxyA", DistanceProxy), ("proxyB", DistanceProxy), ("sweepA", Sweep), ("sweepB", Sweep),
                ("maxFraction", C.c_float)]


class TOIOutput(C.Structure):
    _fields_ = [("state", C.c_int), ("fraction", C.c_float), ("iterations", C.c_int32)]


class ShapeExtent(C.Structure):
    _fields_ = [("minExtent", C.c_float), ("maxExtent", C.c_float), ("center", Vec2)]


# s2TOIState (include/solver2d_b200.h)
TOI_UNKNOWN, TOI_FAILED, TOI_OVERLAPPED, TOI_HIT, TOI_SEPARATED = range(5)
TOI_MAX_ITERATIONS = 50  # S2_TOI_MAX_ITERATIONS


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
    "s2MakeProxy": (DistanceProxy, [C.POINTER(Vec2), C.c_int32, C.c_float]),
    "s2ShapeDistance": (DistanceOutput, [C.POINTER(DistanceCache), C.POINTER(DistanceInput)]),
    # continuous collision (include/solver2d_b200.h): extensions, absent from the reference
    "s2World_EnableContinuous": (None, [WorldId, C.c_bool]),
    "s2Body_SetTransform": (None, [BodyId, Vec2, C.c_float]),
    "s2World_Flush": (None, [WorldId]),
    "s2GetSweepTransform": (Transform, [C.POINTER(Sweep), C.c_float]),
    "s2TimeOfImpact": (TOIOutput, [C.POINTER(TOIInput)]),
    "s2ComputeShapeExtent": (ShapeExtent, [C.POINTER(Polygon), Vec2]),
    "s2ComputeBodyExtent": (ShapeExtent, [C.POINTER(Polygon), C.c_int32, Vec2]),
    # bullets (include/solver2d_b200.h): extensions, absent from the reference
    "s2Body_SetBullet": (None, [BodyId, C.c_bool]),
    "s2Body_IsBullet": (C.c_bool, [BodyId]),
})

class JointReaction(C.Structure):
    """s2JointReaction (include/solver2d_b200.h): force on body B (N, world frame) and torque on B (N-m)."""
    _fields_ = [("force", Vec2), ("torque", C.c_float)]


# breakable joints (include/solver2d_b200.h, DESIGN.md §3.13): extensions, absent from the reference
_API.update({
    "s2ComputeJointReaction": (JointReaction, [C.c_int32, Vec2, C.c_float, C.c_float, C.c_float, Rot, Vec2, C.c_float]),
    "s2Joint_GetReactionForce": (Vec2, [JointId]),
    "s2Joint_GetReactionTorque": (C.c_float, [JointId]),
    "s2Joint_SetBreakForce": (None, [JointId, C.c_float]),
    "s2Joint_GetBreakForce": (C.c_float, [JointId]),
    "s2Joint_SetBreakTorque": (None, [JointId, C.c_float]),
    "s2Joint_GetBreakTorque": (C.c_float, [JointId]),
    # out (s2JointId per entry), capacity; returns the count
    "s2World_GetBrokenJoints": (C.c_int32, [WorldId, C.c_void_p, C.c_int32]),
    # out (fx, fy, torque per slot), capacity; returns the joint capacity
    "s2World_GetJointReactions": (C.c_int32, [WorldId, C.c_void_p, C.c_int32]),
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
