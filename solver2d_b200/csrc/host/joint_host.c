// solver2d-b200 — joints behind the public API (behaviour of reference src/joint.c:154-292, src/revolute_joint.c:825-888,
// src/mouse_joint.c:18-29). Host bookkeeping only: the joint solvers run on the device.
#include "s2_host.h"
#include "shared/s2_distance_joint.h"
#include "shared/s2_gear_joint.h"
#include "solver2d_b200.h"

#include <float.h>
#include <string.h>

static s2Joint* s2AllocJoint(s2World* world, s2Body* bodyA, s2Body* bodyB)
{
	s2FetchBrokenJoints(world); // (the slot may be one the last step broke)
	s2Joint* joint = (s2Joint*)s2AllocObject(&world->jointPool);
	world->joints = (s2Joint*)world->jointPool.memory;
	bool rowDirty = joint->rowDirty;
	s2Object object = joint->object;
	memset(joint, 0, sizeof(*joint));
	joint->object = object;
	joint->rowDirty = rowDirty; // a reused slot may already sit in the dirty list
	joint->bodyIndexA = bodyA->object.index;
	joint->bodyIndexB = bodyB->object.index;
	bodyA->jointCount += 1;
	bodyB->jointCount += 1;
	world->jointPairsDirty = true;
	s2MarkJointDirty(world, joint);
	return joint;
}

// reference src/joint.c:154-179
s2JointId s2CreateMouseJoint(s2WorldId worldId, const s2MouseJointDef* def)
{
	s2World* world = s2GetWorldFromId(worldId);
	s2SyncStateToHost(world);
	s2Body* bodyA = world->bodies + def->bodyIdA.index;
	s2Body* bodyB = world->bodies + def->bodyIdB.index;

	s2Joint* joint = s2AllocJoint(world, bodyA, bodyB);
	joint->type = s2_mouseJoint;
	joint->drawSize = 1.0f;
	s2Transform xfA = {bodyA->origin, bodyA->rot};
	s2Transform xfB = {bodyB->origin, bodyB->rot};
	joint->localOriginAnchorA = s2InvTransformPoint(xfA, def->target);
	joint->localOriginAnchorB = s2InvTransformPoint(xfB, def->target);
	joint->targetA = def->target;
	joint->hertz = def->hertz;
	joint->dampingRatio = def->dampingRatio;
	// the reference never initialises collideConnected for mouse joints and never removes existing contacts for them
	joint->collideConnected = true;

	s2JointId jointId = {joint->object.index, world->index, joint->object.revision};
	return jointId;
}

// reference src/joint.c:181-223
s2JointId s2CreateRevoluteJoint(s2WorldId worldId, const s2RevoluteJointDef* def)
{
	s2World* world = s2GetWorldFromId(worldId);
	s2Body* bodyA = world->bodies + def->bodyIdA.index;
	s2Body* bodyB = world->bodies + def->bodyIdB.index;

	s2Joint* joint = s2AllocJoint(world, bodyA, bodyB);
	joint->type = s2_revoluteJoint;
	joint->drawSize = def->drawSize;
	joint->localOriginAnchorA = def->localAnchorA;
	joint->localOriginAnchorB = def->localAnchorB;
	joint->referenceAngle = def->referenceAngle;
	joint->lowerAngle = def->lowerAngle;
	joint->upperAngle = def->upperAngle;
	joint->maxMotorTorque = def->maxMotorTorque;
	joint->motorSpeed = def->motorSpeed;
	joint->enableLimit = def->enableLimit;
	joint->enableMotor = def->enableMotor;
	// collideConnected == false removes the contacts that already exist between the two bodies (the pair pass does it on
	// the device); new contacts between jointed bodies are never created either way
	joint->collideConnected = def->collideConnected;

	s2JointId jointId = {joint->object.index, world->index, joint->object.revision};
	return jointId;
}

static bool s2IsValidSpringValue(float value)
{
	return s2IsValid(value) && value >= 0.0f;
}

// The weld has no counterpart in the reference. Its row carries no limit or motor flags; like a revolute joint created
// with collideConnected == false it removes the contacts that already exist between its bodies. A negative or non-finite
// hertz or damping ratio creates nothing and returns s2_nullJointId.
s2JointId s2CreateWeldJoint(s2WorldId worldId, const s2WeldJointDef* def)
{
	if (s2IsValidSpringValue(def->linearHertz) == false || s2IsValidSpringValue(def->linearDampingRatio) == false ||
		s2IsValidSpringValue(def->angularHertz) == false || s2IsValidSpringValue(def->angularDampingRatio) == false)
	{
		return s2_nullJointId;
	}
	s2World* world = s2GetWorldFromId(worldId);
	s2Body* bodyA = world->bodies + def->bodyIdA.index;
	s2Body* bodyB = world->bodies + def->bodyIdB.index;

	s2Joint* joint = s2AllocJoint(world, bodyA, bodyB);
	joint->type = s2_weldJoint;
	joint->drawSize = def->drawSize;
	joint->localOriginAnchorA = def->localAnchorA;
	joint->localOriginAnchorB = def->localAnchorB;
	joint->referenceAngle = def->referenceAngle;
	joint->collideConnected = def->collideConnected;
	joint->linearHertz = def->linearHertz;
	joint->linearDampingRatio = def->linearDampingRatio;
	joint->angularHertz = def->angularHertz;
	joint->angularDampingRatio = def->angularDampingRatio;

	s2JointId jointId = {joint->object.index, world->index, joint->object.revision};
	return jointId;
}

// reference src/joint.c:225-292
void s2DestroyJoint(s2JointId jointId)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	s2FetchBrokenJoints(world); // (the slot may be one the last step broke)
	s2Joint* joint = world->joints + jointId.index;
	if (jointId.index < 0 || jointId.index >= world->jointPool.capacity || s2ObjectValid(&joint->object) == false ||
		joint->object.revision != jointId.revision)
	{
		// a stale id, such as a gear that the destruction of a joint it links already took (DESIGN.md §3.19): nothing to do
		return;
	}
	if (joint->breakForce > 0.0f || joint->breakTorque > 0.0f)
	{
		world->breakableCount -= 1;
	}
	if (world->gearCount > 0 && joint->type != s2_gearJoint)
	{
		// the gears that link this joint go first (DESIGN.md §3.19)
		for (int32_t i = 0; i < world->jointPool.capacity; ++i)
		{
			const s2Joint* gear = world->joints + i;
			if (s2ObjectValid(&gear->object) && gear->type == s2_gearJoint &&
				((gear->gearJoint1.index == jointId.index && gear->gearJoint1.revision == jointId.revision) ||
				 (gear->gearJoint2.index == jointId.index && gear->gearJoint2.revision == jointId.revision)))
			{
				s2JointId gearId = {i, world->index, gear->object.revision};
				s2DestroyJoint(gearId);
			}
		}
	}
	if (joint->type == s2_gearJoint)
	{
		world->gearCount -= 1;
	}
	world->bodies[joint->bodyIndexA].jointCount -= 1;
	world->bodies[joint->bodyIndexB].jointCount -= 1;
	s2FreeObject(&world->jointPool, &joint->object);
	s2MarkJointDirty(world, joint);
	world->jointPairsDirty = true;
}

static s2Joint* s2GetJointForEdit(s2JointId jointId, s2World** worldOut)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	// the row carries the accumulated impulses: make the host copy current before it is re-uploaded
	s2SyncStateToHost(world);
	s2Joint* joint = world->joints + jointId.index;
	S2_ASSERT(s2ObjectValid(&joint->object));
	S2_ASSERT(joint->object.revision == jointId.revision);
	*worldOut = world;
	return joint;
}

void s2MouseJoint_SetTarget(s2JointId jointId, s2Vec2 target)
{
	s2World* world;
	s2Joint* joint = s2GetJointForEdit(jointId, &world);
	joint->targetA = target;
	s2MarkJointDirty(world, joint);
}

void s2RevoluteJoint_EnableLimit(s2JointId jointId, bool enableLimit)
{
	s2World* world;
	s2Joint* joint = s2GetJointForEdit(jointId, &world);
	joint->enableLimit = enableLimit;
	s2MarkJointDirty(world, joint);
}

void s2RevoluteJoint_EnableMotor(s2JointId jointId, bool enableMotor)
{
	s2World* world;
	s2Joint* joint = s2GetJointForEdit(jointId, &world);
	joint->enableMotor = enableMotor;
	s2MarkJointDirty(world, joint);
}

void s2RevoluteJoint_SetMotorSpeed(s2JointId jointId, float motorSpeed)
{
	s2World* world;
	s2Joint* joint = s2GetJointForEdit(jointId, &world);
	joint->motorSpeed = motorSpeed;
	s2MarkJointDirty(world, joint);
}

float s2RevoluteJoint_GetMotorTorque(s2JointId jointId, float inverseTimeStep)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	s2SyncStateToHost(world);
	return inverseTimeStep * world->joints[jointId.index].motorImpulse;
}

// ---- joint springs (DESIGN.md §3.14): revolute, prismatic, distance and wheel joints; hertz and dampingRatio carry the spring

static void s2EnableJointSpring(s2JointId jointId, s2JointType type, bool enableSpring)
{
	s2World* world;
	s2Joint* joint = s2GetJointForEdit(jointId, &world);
	if (joint->type != type)
	{
		return; // only revolute, prismatic, distance and wheel joints have a spring
	}
	joint->enableSpring = enableSpring;
	s2MarkJointDirty(world, joint);
}

static void s2SetJointSpringValue(s2JointId jointId, s2JointType type, float value, bool dampingRatio)
{
	if (s2IsValidSpringValue(value) == false)
	{
		return; // rejected: the joint keeps its value
	}
	s2World* world;
	s2Joint* joint = s2GetJointForEdit(jointId, &world);
	if (joint->type != type)
	{
		return; // only revolute, prismatic, distance and wheel joints have a spring
	}
	if (dampingRatio)
	{
		joint->dampingRatio = value;
	}
	else
	{
		joint->hertz = value;
	}
	s2MarkJointDirty(world, joint);
}

void s2RevoluteJoint_EnableSpring(s2JointId jointId, bool enableSpring)
{
	s2EnableJointSpring(jointId, s2_revoluteJoint, enableSpring);
}

void s2RevoluteJoint_SetSpringHertz(s2JointId jointId, float hertz)
{
	s2SetJointSpringValue(jointId, s2_revoluteJoint, hertz, false);
}

void s2RevoluteJoint_SetSpringDampingRatio(s2JointId jointId, float dampingRatio)
{
	s2SetJointSpringValue(jointId, s2_revoluteJoint, dampingRatio, true);
}

void s2PrismaticJoint_EnableSpring(s2JointId jointId, bool enableSpring)
{
	s2EnableJointSpring(jointId, s2_prismaticJoint, enableSpring);
}

void s2PrismaticJoint_SetSpringHertz(s2JointId jointId, float hertz)
{
	s2SetJointSpringValue(jointId, s2_prismaticJoint, hertz, false);
}

void s2PrismaticJoint_SetSpringDampingRatio(s2JointId jointId, float dampingRatio)
{
	s2SetJointSpringValue(jointId, s2_prismaticJoint, dampingRatio, true);
}

// ---- soft weld (DESIGN.md §3.15): the weld's anchor and angle springs ------------------------------------------------------

enum
{
	s2_weldLinearHertz,
	s2_weldLinearDampingRatio,
	s2_weldAngularHertz,
	s2_weldAngularDampingRatio,
};

static float* s2WeldSpringField(s2Joint* joint, int field)
{
	switch (field)
	{
		case s2_weldLinearHertz:
			return &joint->linearHertz;
		case s2_weldLinearDampingRatio:
			return &joint->linearDampingRatio;
		case s2_weldAngularHertz:
			return &joint->angularHertz;
		default:
			return &joint->angularDampingRatio;
	}
}

static void s2SetWeldSpringValue(s2JointId jointId, int field, float value)
{
	if (s2IsValidSpringValue(value) == false)
	{
		return; // rejected: the joint keeps its value
	}
	s2World* world;
	s2Joint* joint = s2GetJointForEdit(jointId, &world);
	if (joint->type != s2_weldJoint)
	{
		return;
	}
	*s2WeldSpringField(joint, field) = value;
	s2MarkJointDirty(world, joint);
}

static float s2GetWeldSpringValue(s2JointId jointId, int field)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	s2Joint* joint = world->joints + jointId.index;
	S2_ASSERT(s2ObjectValid(&joint->object) && joint->object.revision == jointId.revision);
	return joint->type == s2_weldJoint ? *s2WeldSpringField(joint, field) : 0.0f;
}

void s2WeldJoint_SetLinearHertz(s2JointId jointId, float hertz)
{
	s2SetWeldSpringValue(jointId, s2_weldLinearHertz, hertz);
}

void s2WeldJoint_SetLinearDampingRatio(s2JointId jointId, float dampingRatio)
{
	s2SetWeldSpringValue(jointId, s2_weldLinearDampingRatio, dampingRatio);
}

void s2WeldJoint_SetAngularHertz(s2JointId jointId, float hertz)
{
	s2SetWeldSpringValue(jointId, s2_weldAngularHertz, hertz);
}

void s2WeldJoint_SetAngularDampingRatio(s2JointId jointId, float dampingRatio)
{
	s2SetWeldSpringValue(jointId, s2_weldAngularDampingRatio, dampingRatio);
}

float s2WeldJoint_GetLinearHertz(s2JointId jointId)
{
	return s2GetWeldSpringValue(jointId, s2_weldLinearHertz);
}

float s2WeldJoint_GetLinearDampingRatio(s2JointId jointId)
{
	return s2GetWeldSpringValue(jointId, s2_weldLinearDampingRatio);
}

float s2WeldJoint_GetAngularHertz(s2JointId jointId)
{
	return s2GetWeldSpringValue(jointId, s2_weldAngularHertz);
}

float s2WeldJoint_GetAngularDampingRatio(s2JointId jointId)
{
	return s2GetWeldSpringValue(jointId, s2_weldAngularDampingRatio);
}

// The prismatic joint has no counterpart in the reference (DESIGN.md §3.9). Degenerate input creates nothing and returns
// s2_nullJointId: an axis that cannot be normalized, lowerTranslation > upperTranslation, or a spring hertz or damping ratio
// that is negative or not finite.
s2JointId s2CreatePrismaticJoint(s2WorldId worldId, const s2PrismaticJointDef* def)
{
	s2Vec2 axis = def->localAxisA;
	float length = s2Length(axis);
	if (s2IsValidVec2(axis) == false || s2IsValid(length) == false || length == 0.0f ||
		(def->lowerTranslation <= def->upperTranslation) == false || s2IsValidSpringValue(def->hertz) == false ||
		s2IsValidSpringValue(def->dampingRatio) == false)
	{
		return s2_nullJointId;
	}

	s2World* world = s2GetWorldFromId(worldId);
	s2Body* bodyA = world->bodies + def->bodyIdA.index;
	s2Body* bodyB = world->bodies + def->bodyIdB.index;

	s2Joint* joint = s2AllocJoint(world, bodyA, bodyB);
	joint->type = s2_prismaticJoint;
	joint->drawSize = def->drawSize;
	joint->localOriginAnchorA = def->localAnchorA;
	joint->localOriginAnchorB = def->localAnchorB;
	joint->localAxisA = s2MakeVec2(axis.x / length, axis.y / length);
	joint->referenceAngle = def->referenceAngle;
	joint->lowerAngle = def->lowerTranslation;
	joint->upperAngle = def->upperTranslation;
	joint->maxMotorTorque = def->maxMotorForce;
	joint->motorSpeed = def->motorSpeed;
	joint->enableLimit = def->enableLimit;
	joint->enableMotor = def->enableMotor;
	joint->collideConnected = def->collideConnected;
	joint->enableSpring = def->enableSpring;
	joint->hertz = def->hertz;
	joint->dampingRatio = def->dampingRatio;

	s2JointId jointId = {joint->object.index, world->index, joint->object.revision};
	return jointId;
}

void s2PrismaticJoint_EnableLimit(s2JointId jointId, bool enableLimit)
{
	s2World* world;
	s2Joint* joint = s2GetJointForEdit(jointId, &world);
	joint->enableLimit = enableLimit;
	s2MarkJointDirty(world, joint);
}

void s2PrismaticJoint_SetLimits(s2JointId jointId, float lower, float upper)
{
	if ((lower <= upper) == false)
	{
		return; // rejected: the joint keeps its limits
	}
	s2World* world;
	s2Joint* joint = s2GetJointForEdit(jointId, &world);
	joint->lowerAngle = lower;
	joint->upperAngle = upper;
	s2MarkJointDirty(world, joint);
}

void s2PrismaticJoint_EnableMotor(s2JointId jointId, bool enableMotor)
{
	s2World* world;
	s2Joint* joint = s2GetJointForEdit(jointId, &world);
	joint->enableMotor = enableMotor;
	s2MarkJointDirty(world, joint);
}

void s2PrismaticJoint_SetMotorSpeed(s2JointId jointId, float motorSpeed)
{
	s2World* world;
	s2Joint* joint = s2GetJointForEdit(jointId, &world);
	joint->motorSpeed = motorSpeed;
	s2MarkJointDirty(world, joint);
}

float s2PrismaticJoint_GetMotorForce(s2JointId jointId, float inverseTimeStep)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	s2SyncStateToHost(world);
	return inverseTimeStep * world->joints[jointId.index].motorImpulse;
}

// The motor joint has no counterpart in the reference (DESIGN.md §3.10). Its row has no limit or motor flag; its offsets, caps
// and correction factor sit in the columns s2_host.h lists. Invalid input creates nothing and returns s2_nullJointId.
s2JointId s2CreateMotorJoint(s2WorldId worldId, const s2MotorJointDef* def)
{
	if (s2IsValidVec2(def->linearOffset) == false || s2IsValid(def->angularOffset) == false || s2IsValid(def->maxForce) == false ||
		def->maxForce < 0.0f || s2IsValid(def->maxTorque) == false || def->maxTorque < 0.0f ||
		(def->correctionFactor >= 0.0f && def->correctionFactor <= 1.0f) == false)
	{
		return s2_nullJointId;
	}

	s2World* world = s2GetWorldFromId(worldId);
	s2Body* bodyA = world->bodies + def->bodyIdA.index;
	s2Body* bodyB = world->bodies + def->bodyIdB.index;

	s2Joint* joint = s2AllocJoint(world, bodyA, bodyB);
	joint->type = s2_motorJoint;
	joint->drawSize = 1.0f;
	joint->localOriginAnchorA = def->linearOffset;
	joint->localOriginAnchorB = s2Vec2_zero;
	joint->referenceAngle = def->angularOffset;
	joint->maxMotorTorque = def->maxTorque;
	joint->hertz = def->maxForce;
	joint->dampingRatio = def->correctionFactor;
	joint->collideConnected = def->collideConnected;

	s2JointId jointId = {joint->object.index, world->index, joint->object.revision};
	return jointId;
}

void s2MotorJoint_SetLinearOffset(s2JointId jointId, s2Vec2 linearOffset)
{
	if (s2IsValidVec2(linearOffset) == false)
	{
		return; // rejected: the joint keeps its offset
	}
	s2World* world;
	s2Joint* joint = s2GetJointForEdit(jointId, &world);
	joint->localOriginAnchorA = linearOffset;
	s2MarkJointDirty(world, joint);
}

s2Vec2 s2MotorJoint_GetLinearOffset(s2JointId jointId)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	return world->joints[jointId.index].localOriginAnchorA;
}

void s2MotorJoint_SetAngularOffset(s2JointId jointId, float angularOffset)
{
	if (s2IsValid(angularOffset) == false)
	{
		return;
	}
	s2World* world;
	s2Joint* joint = s2GetJointForEdit(jointId, &world);
	joint->referenceAngle = angularOffset;
	s2MarkJointDirty(world, joint);
}

float s2MotorJoint_GetAngularOffset(s2JointId jointId)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	return world->joints[jointId.index].referenceAngle;
}

void s2MotorJoint_SetMaxForce(s2JointId jointId, float maxForce)
{
	if (s2IsValid(maxForce) == false || maxForce < 0.0f)
	{
		return;
	}
	s2World* world;
	s2Joint* joint = s2GetJointForEdit(jointId, &world);
	joint->hertz = maxForce;
	s2MarkJointDirty(world, joint);
}

void s2MotorJoint_SetMaxTorque(s2JointId jointId, float maxTorque)
{
	if (s2IsValid(maxTorque) == false || maxTorque < 0.0f)
	{
		return;
	}
	s2World* world;
	s2Joint* joint = s2GetJointForEdit(jointId, &world);
	joint->maxMotorTorque = maxTorque;
	s2MarkJointDirty(world, joint);
}

void s2MotorJoint_SetCorrectionFactor(s2JointId jointId, float correctionFactor)
{
	if ((correctionFactor >= 0.0f && correctionFactor <= 1.0f) == false)
	{
		return;
	}
	s2World* world;
	s2Joint* joint = s2GetJointForEdit(jointId, &world);
	joint->dampingRatio = correctionFactor;
	s2MarkJointDirty(world, joint);
}

s2Vec2 s2MotorJoint_GetConstraintForce(s2JointId jointId, float inverseTimeStep)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	s2SyncStateToHost(world);
	return s2MulSV(inverseTimeStep, world->joints[jointId.index].impulse);
}

float s2MotorJoint_GetConstraintTorque(s2JointId jointId, float inverseTimeStep)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	s2SyncStateToHost(world);
	return inverseTimeStep * world->joints[jointId.index].motorImpulse;
}

float s2PrismaticJoint_GetTranslation(s2JointId jointId)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	s2SyncStateToHost(world);
	const s2Joint* joint = world->joints + jointId.index;
	const s2Body* bodyA = world->bodies + joint->bodyIndexA;
	const s2Body* bodyB = world->bodies + joint->bodyIndexB;
	s2Transform xfA = {bodyA->origin, bodyA->rot};
	s2Transform xfB = {bodyB->origin, bodyB->rot};
	s2Vec2 pA = s2TransformPoint(xfA, joint->localOriginAnchorA);
	s2Vec2 pB = s2TransformPoint(xfB, joint->localOriginAnchorB);
	s2Vec2 axis = s2RotateVector(bodyA->rot, joint->localAxisA);
	return s2Dot(axis, s2Sub(pB, pA));
}

// ---- distance joint (DESIGN.md §3.16) ------------------------------------------------------------------------------------

static float s2ClampDistanceLength(float length)
{
	return S2_CLAMP(length, s2_linearSlop, s2_huge);
}

static bool s2IsValidDistanceValue(float value)
{
	return s2IsValid(value) && value >= 0.0f;
}

// The distance joint has no counterpart in the reference. Invalid input creates nothing and returns s2_nullJointId; the lengths
// are clamped into [s2_linearSlop, s2_huge] as Box2D clamps them.
s2JointId s2CreateDistanceJoint(s2WorldId worldId, const s2DistanceJointDef* def)
{
	if (s2IsValidVec2(def->localAnchorA) == false || s2IsValidVec2(def->localAnchorB) == false ||
		s2IsValidDistanceValue(def->length) == false || s2IsValidDistanceValue(def->minLength) == false ||
		s2IsValidDistanceValue(def->maxLength) == false || (def->minLength <= def->maxLength) == false ||
		s2IsValidDistanceValue(def->hertz) == false || s2IsValidDistanceValue(def->dampingRatio) == false ||
		s2IsValidDistanceValue(def->maxMotorForce) == false || s2IsValid(def->motorSpeed) == false)
	{
		return s2_nullJointId;
	}

	s2World* world = s2GetWorldFromId(worldId);
	s2Body* bodyA = world->bodies + def->bodyIdA.index;
	s2Body* bodyB = world->bodies + def->bodyIdB.index;

	s2Joint* joint = s2AllocJoint(world, bodyA, bodyB);
	joint->type = s2_distanceJoint;
	joint->drawSize = 1.0f;
	joint->localOriginAnchorA = def->localAnchorA;
	joint->localOriginAnchorB = def->localAnchorB;
	joint->referenceAngle = s2ClampDistanceLength(def->length);
	joint->lowerAngle = s2ClampDistanceLength(def->minLength);
	joint->upperAngle = s2ClampDistanceLength(def->maxLength);
	joint->enableSpring = def->enableSpring;
	joint->hertz = def->hertz;
	joint->dampingRatio = def->dampingRatio;
	joint->enableLimit = def->enableLimit;
	joint->enableMotor = def->enableMotor;
	joint->maxMotorTorque = def->maxMotorForce;
	joint->motorSpeed = def->motorSpeed;
	joint->collideConnected = def->collideConnected;

	s2JointId jointId = {joint->object.index, world->index, joint->object.revision};
	return jointId;
}

// the joint to edit, or NULL for a joint of another type
static s2Joint* s2GetDistanceJointForEdit(s2JointId jointId, s2World** worldOut)
{
	s2Joint* joint = s2GetJointForEdit(jointId, worldOut);
	return joint->type == s2_distanceJoint ? joint : NULL;
}

static const s2Joint* s2GetDistanceJoint(s2JointId jointId)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	const s2Joint* joint = world->joints + jointId.index;
	S2_ASSERT(s2ObjectValid(&joint->object) && joint->object.revision == jointId.revision);
	return joint->type == s2_distanceJoint ? joint : NULL;
}

void s2DistanceJoint_SetLength(s2JointId jointId, float length)
{
	if (s2IsValidDistanceValue(length) == false)
	{
		return;
	}
	s2World* world;
	s2Joint* joint = s2GetDistanceJointForEdit(jointId, &world);
	if (joint != NULL)
	{
		joint->referenceAngle = s2ClampDistanceLength(length);
		s2MarkJointDirty(world, joint);
	}
}

float s2DistanceJoint_GetLength(s2JointId jointId)
{
	const s2Joint* joint = s2GetDistanceJoint(jointId);
	return joint != NULL ? joint->referenceAngle : 0.0f;
}

void s2DistanceJoint_EnableLimit(s2JointId jointId, bool enableLimit)
{
	s2World* world;
	s2Joint* joint = s2GetDistanceJointForEdit(jointId, &world);
	if (joint != NULL)
	{
		joint->enableLimit = enableLimit;
		s2MarkJointDirty(world, joint);
	}
}

void s2DistanceJoint_SetLengthRange(s2JointId jointId, float minLength, float maxLength)
{
	if (s2IsValidDistanceValue(minLength) == false || s2IsValidDistanceValue(maxLength) == false || (minLength <= maxLength) == false)
	{
		return;
	}
	s2World* world;
	s2Joint* joint = s2GetDistanceJointForEdit(jointId, &world);
	if (joint != NULL)
	{
		joint->lowerAngle = s2ClampDistanceLength(minLength);
		joint->upperAngle = s2ClampDistanceLength(maxLength);
		s2MarkJointDirty(world, joint);
	}
}

float s2DistanceJoint_GetMinLength(s2JointId jointId)
{
	const s2Joint* joint = s2GetDistanceJoint(jointId);
	return joint != NULL ? joint->lowerAngle : 0.0f;
}

float s2DistanceJoint_GetMaxLength(s2JointId jointId)
{
	const s2Joint* joint = s2GetDistanceJoint(jointId);
	return joint != NULL ? joint->upperAngle : 0.0f;
}

void s2DistanceJoint_EnableSpring(s2JointId jointId, bool enableSpring)
{
	s2EnableJointSpring(jointId, s2_distanceJoint, enableSpring);
}

void s2DistanceJoint_SetSpringHertz(s2JointId jointId, float hertz)
{
	s2SetJointSpringValue(jointId, s2_distanceJoint, hertz, false);
}

void s2DistanceJoint_SetSpringDampingRatio(s2JointId jointId, float dampingRatio)
{
	s2SetJointSpringValue(jointId, s2_distanceJoint, dampingRatio, true);
}

void s2DistanceJoint_EnableMotor(s2JointId jointId, bool enableMotor)
{
	s2World* world;
	s2Joint* joint = s2GetDistanceJointForEdit(jointId, &world);
	if (joint != NULL)
	{
		joint->enableMotor = enableMotor;
		s2MarkJointDirty(world, joint);
	}
}

void s2DistanceJoint_SetMotorSpeed(s2JointId jointId, float motorSpeed)
{
	if (s2IsValid(motorSpeed) == false)
	{
		return;
	}
	s2World* world;
	s2Joint* joint = s2GetDistanceJointForEdit(jointId, &world);
	if (joint != NULL)
	{
		joint->motorSpeed = motorSpeed;
		s2MarkJointDirty(world, joint);
	}
}

void s2DistanceJoint_SetMaxMotorForce(s2JointId jointId, float maxMotorForce)
{
	if (s2IsValidDistanceValue(maxMotorForce) == false)
	{
		return;
	}
	s2World* world;
	s2Joint* joint = s2GetDistanceJointForEdit(jointId, &world);
	if (joint != NULL)
	{
		joint->maxMotorTorque = maxMotorForce;
		s2MarkJointDirty(world, joint);
	}
}

float s2DistanceJoint_GetMotorForce(s2JointId jointId, float inverseTimeStep)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	s2SyncStateToHost(world);
	const s2Joint* joint = s2GetDistanceJoint(jointId);
	return joint != NULL ? inverseTimeStep * joint->motorImpulse : 0.0f;
}

// the line from anchor A to anchor B at the lazily synced poses
static s2Vec2 s2DistanceJointAxis(s2World* world, const s2Joint* joint, float* length)
{
	const s2Body* bodyA = world->bodies + joint->bodyIndexA;
	const s2Body* bodyB = world->bodies + joint->bodyIndexB;
	return s2cDistanceJointAxis(length, bodyA->position, bodyA->rot, s2Sub(joint->localOriginAnchorA, bodyA->localCenter),
								bodyB->position, bodyB->rot, s2Sub(joint->localOriginAnchorB, bodyB->localCenter));
}

float s2DistanceJoint_GetCurrentLength(s2JointId jointId)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	s2SyncStateToHost(world);
	const s2Joint* joint = s2GetDistanceJoint(jointId);
	if (joint == NULL)
	{
		return 0.0f;
	}
	float length;
	s2DistanceJointAxis(world, joint, &length);
	return length;
}

// ---- wheel joint (DESIGN.md §3.17) ---------------------------------------------------------------------------------------

// The wheel joint has no counterpart in the reference. Invalid input creates nothing and returns s2_nullJointId.
s2JointId s2CreateWheelJoint(s2WorldId worldId, const s2WheelJointDef* def)
{
	s2Vec2 axis = def->localAxisA;
	float length = s2Length(axis);
	if (s2IsValidVec2(def->localAnchorA) == false || s2IsValidVec2(def->localAnchorB) == false || s2IsValidVec2(axis) == false ||
		s2IsValid(length) == false || length == 0.0f || s2IsValid(def->lowerTranslation) == false ||
		s2IsValid(def->upperTranslation) == false || (def->lowerTranslation <= def->upperTranslation) == false ||
		s2IsValidSpringValue(def->hertz) == false || s2IsValidSpringValue(def->dampingRatio) == false ||
		s2IsValidSpringValue(def->maxMotorTorque) == false || s2IsValid(def->motorSpeed) == false)
	{
		return s2_nullJointId;
	}

	s2World* world = s2GetWorldFromId(worldId);
	s2Body* bodyA = world->bodies + def->bodyIdA.index;
	s2Body* bodyB = world->bodies + def->bodyIdB.index;

	s2Joint* joint = s2AllocJoint(world, bodyA, bodyB);
	joint->type = s2_wheelJoint;
	joint->drawSize = 1.0f;
	joint->localOriginAnchorA = def->localAnchorA;
	joint->localOriginAnchorB = def->localAnchorB;
	joint->localAxisA = s2MakeVec2(axis.x / length, axis.y / length);
	joint->lowerAngle = def->lowerTranslation;
	joint->upperAngle = def->upperTranslation;
	joint->maxMotorTorque = def->maxMotorTorque;
	joint->motorSpeed = def->motorSpeed;
	joint->enableLimit = def->enableLimit;
	joint->enableMotor = def->enableMotor;
	joint->enableSpring = def->enableSpring;
	joint->hertz = def->hertz;
	joint->dampingRatio = def->dampingRatio;
	joint->collideConnected = def->collideConnected;

	s2JointId jointId = {joint->object.index, world->index, joint->object.revision};
	return jointId;
}

// the joint to edit, or NULL for a joint of another type
static s2Joint* s2GetWheelJointForEdit(s2JointId jointId, s2World** worldOut)
{
	s2Joint* joint = s2GetJointForEdit(jointId, worldOut);
	return joint->type == s2_wheelJoint ? joint : NULL;
}

void s2WheelJoint_EnableSpring(s2JointId jointId, bool enableSpring)
{
	s2EnableJointSpring(jointId, s2_wheelJoint, enableSpring);
}

void s2WheelJoint_SetSpringHertz(s2JointId jointId, float hertz)
{
	s2SetJointSpringValue(jointId, s2_wheelJoint, hertz, false);
}

void s2WheelJoint_SetSpringDampingRatio(s2JointId jointId, float dampingRatio)
{
	s2SetJointSpringValue(jointId, s2_wheelJoint, dampingRatio, true);
}

void s2WheelJoint_EnableLimit(s2JointId jointId, bool enableLimit)
{
	s2World* world;
	s2Joint* joint = s2GetWheelJointForEdit(jointId, &world);
	if (joint != NULL)
	{
		joint->enableLimit = enableLimit;
		s2MarkJointDirty(world, joint);
	}
}

void s2WheelJoint_SetLimits(s2JointId jointId, float lower, float upper)
{
	if (s2IsValid(lower) == false || s2IsValid(upper) == false || (lower <= upper) == false)
	{
		return;
	}
	s2World* world;
	s2Joint* joint = s2GetWheelJointForEdit(jointId, &world);
	if (joint != NULL)
	{
		joint->lowerAngle = lower;
		joint->upperAngle = upper;
		s2MarkJointDirty(world, joint);
	}
}

void s2WheelJoint_EnableMotor(s2JointId jointId, bool enableMotor)
{
	s2World* world;
	s2Joint* joint = s2GetWheelJointForEdit(jointId, &world);
	if (joint != NULL)
	{
		joint->enableMotor = enableMotor;
		s2MarkJointDirty(world, joint);
	}
}

void s2WheelJoint_SetMotorSpeed(s2JointId jointId, float motorSpeed)
{
	if (s2IsValid(motorSpeed) == false)
	{
		return;
	}
	s2World* world;
	s2Joint* joint = s2GetWheelJointForEdit(jointId, &world);
	if (joint != NULL)
	{
		joint->motorSpeed = motorSpeed;
		s2MarkJointDirty(world, joint);
	}
}

void s2WheelJoint_SetMaxMotorTorque(s2JointId jointId, float maxMotorTorque)
{
	if (s2IsValidSpringValue(maxMotorTorque) == false)
	{
		return;
	}
	s2World* world;
	s2Joint* joint = s2GetWheelJointForEdit(jointId, &world);
	if (joint != NULL)
	{
		joint->maxMotorTorque = maxMotorTorque;
		s2MarkJointDirty(world, joint);
	}
}

float s2WheelJoint_GetMotorTorque(s2JointId jointId, float inverseTimeStep)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	s2SyncStateToHost(world);
	const s2Joint* joint = world->joints + jointId.index;
	S2_ASSERT(s2ObjectValid(&joint->object) && joint->object.revision == jointId.revision);
	// the angular motor's impulse rides in impulse.y (the row's impulse[1])
	return joint->type == s2_wheelJoint ? inverseTimeStep * joint->impulse.y : 0.0f;
}

float s2WheelJoint_GetTranslation(s2JointId jointId)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	const s2Joint* joint = world->joints + jointId.index;
	S2_ASSERT(s2ObjectValid(&joint->object) && joint->object.revision == jointId.revision);
	return joint->type == s2_wheelJoint ? s2PrismaticJoint_GetTranslation(jointId) : 0.0f;
}

// ---- pulley joint (DESIGN.md §3.18) --------------------------------------------------------------------------------------

// The pulley joint has no counterpart in the reference. Invalid input creates nothing and returns s2_nullJointId.
s2JointId s2CreatePulleyJoint(s2WorldId worldId, const s2PulleyJointDef* def)
{
	if (s2IsValidVec2(def->groundAnchorA) == false || s2IsValidVec2(def->groundAnchorB) == false ||
		s2IsValidVec2(def->localAnchorA) == false || s2IsValidVec2(def->localAnchorB) == false ||
		s2IsValidDistanceValue(def->lengthA) == false || s2IsValidDistanceValue(def->lengthB) == false ||
		s2IsValid(def->ratio) == false || (def->ratio > FLT_EPSILON) == false)
	{
		return s2_nullJointId;
	}

	s2World* world = s2GetWorldFromId(worldId);
	s2Body* bodyA = world->bodies + def->bodyIdA.index;
	s2Body* bodyB = world->bodies + def->bodyIdB.index;

	s2Joint* joint = s2AllocJoint(world, bodyA, bodyB);
	joint->type = s2_pulleyJoint;
	joint->drawSize = 1.0f;
	joint->localOriginAnchorA = def->localAnchorA;
	joint->localOriginAnchorB = def->localAnchorB;
	joint->targetA = def->groundAnchorA;
	joint->localAxisA = def->groundAnchorB;
	joint->referenceAngle = def->ratio;
	joint->lowerAngle = def->lengthA;
	joint->upperAngle = def->lengthB;
	joint->collideConnected = def->collideConnected;

	s2JointId jointId = {joint->object.index, world->index, joint->object.revision};
	return jointId;
}

// the joint, or NULL for a joint of another type
static const s2Joint* s2GetPulleyJoint(s2JointId jointId)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	const s2Joint* joint = world->joints + jointId.index;
	S2_ASSERT(s2ObjectValid(&joint->object) && joint->object.revision == jointId.revision);
	return joint->type == s2_pulleyJoint ? joint : NULL;
}

s2Vec2 s2PulleyJoint_GetGroundAnchorA(s2JointId jointId)
{
	const s2Joint* joint = s2GetPulleyJoint(jointId);
	return joint != NULL ? joint->targetA : s2Vec2_zero;
}

s2Vec2 s2PulleyJoint_GetGroundAnchorB(s2JointId jointId)
{
	const s2Joint* joint = s2GetPulleyJoint(jointId);
	return joint != NULL ? joint->localAxisA : s2Vec2_zero;
}

float s2PulleyJoint_GetLengthA(s2JointId jointId)
{
	const s2Joint* joint = s2GetPulleyJoint(jointId);
	return joint != NULL ? joint->lowerAngle : 0.0f;
}

float s2PulleyJoint_GetLengthB(s2JointId jointId)
{
	const s2Joint* joint = s2GetPulleyJoint(jointId);
	return joint != NULL ? joint->upperAngle : 0.0f;
}

float s2PulleyJoint_GetRatio(s2JointId jointId)
{
	const s2Joint* joint = s2GetPulleyJoint(jointId);
	return joint != NULL ? joint->referenceAngle : 0.0f;
}

// -ratio uB (sideB) or -uA, and the rope's length, at the lazily synced poses
static s2Vec2 s2PulleyJointAxis(s2World* world, const s2Joint* joint, bool sideB, float* length)
{
	const s2Body* body = world->bodies + (sideB ? joint->bodyIndexB : joint->bodyIndexA);
	s2Vec2 local = s2Sub(sideB ? joint->localOriginAnchorB : joint->localOriginAnchorA, body->localCenter);
	return s2cPulleyJointAxis(length, sideB ? joint->localAxisA : joint->targetA, body->position, body->rot, local,
							  sideB ? joint->referenceAngle : 1.0f);
}

static float s2PulleyJointCurrentLength(s2JointId jointId, bool sideB)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	s2SyncStateToHost(world);
	const s2Joint* joint = s2GetPulleyJoint(jointId);
	if (joint == NULL)
	{
		return 0.0f;
	}
	float length;
	s2PulleyJointAxis(world, joint, sideB, &length);
	return length;
}

float s2PulleyJoint_GetCurrentLengthA(s2JointId jointId)
{
	return s2PulleyJointCurrentLength(jointId, false);
}

float s2PulleyJoint_GetCurrentLengthB(s2JointId jointId)
{
	return s2PulleyJointCurrentLength(jointId, true);
}

// ---- gear joint (DESIGN.md §3.19) ----------------------------------------------------------------------------------------

// the live joint `jointId` names in `world`, or NULL for a stale, null or foreign id
static s2Joint* s2FindJoint(s2World* world, s2JointId jointId)
{
	if (jointId.world != world->index || jointId.index < 0 || jointId.index >= world->jointPool.capacity)
	{
		return NULL;
	}
	s2Joint* joint = world->joints + jointId.index;
	return s2ObjectValid(&joint->object) && joint->object.revision == jointId.revision ? joint : NULL;
}

// a linked joint's frame in the four row lanes of its side: a revolute joint's frame rotation (s, c) and reference angle, a
// prismatic joint's world anchor and world axis
static void s2GearFrame(const s2World* world, const s2Joint* link, float frame[4])
{
	const s2Body* body = world->bodies + link->bodyIndexA;
	if (link->type == s2_prismaticJoint)
	{
		s2Vec2 p = s2Add(body->origin, s2RotateVector(body->rot, link->localOriginAnchorA));
		s2Vec2 u = s2RotateVector(body->rot, link->localAxisA);
		frame[0] = p.x;
		frame[1] = p.y;
		frame[2] = u.x;
		frame[3] = u.y;
	}
	else
	{
		frame[0] = body->rot.s;
		frame[1] = body->rot.c;
		frame[2] = link->referenceAngle;
		frame[3] = 0.0f;
	}
}

static void s2SetGearFrames(s2World* world, s2Joint* gear)
{
	float f1[4], f2[4];
	s2GearFrame(world, world->joints + gear->gearJoint1.index, f1);
	s2GearFrame(world, world->joints + gear->gearJoint2.index, f2);
	gear->targetA = s2MakeVec2(f1[0], f1[1]);
	gear->localAxisA = s2MakeVec2(f1[2], f1[3]);
	gear->maxMotorTorque = f2[0];
	gear->motorSpeed = f2[1];
	gear->hertz = f2[2];
	gear->dampingRatio = f2[3];
}

// one side at the host's body state; a revolute side is unwound from its stored coordinate
static s2cGearSide s2GearSideAt(const s2World* world, const s2Joint* gear, bool side2)
{
	const s2Body* body = world->bodies + (side2 ? gear->bodyIndexB : gear->bodyIndexA);
	s2Vec2 local = s2Sub(side2 ? gear->localOriginAnchorB : gear->localOriginAnchorA, body->localCenter);
	float f[4] = {gear->targetA.x, gear->targetA.y, gear->localAxisA.x, gear->localAxisA.y};
	if (side2)
	{
		f[0] = gear->maxMotorTorque;
		f[1] = gear->motorSpeed;
		f[2] = gear->hertz;
		f[3] = gear->dampingRatio;
	}
	if (side2 ? gear->gearPrismatic2 : gear->gearPrismatic1)
	{
		return s2cGearPrismatic(s2Sub(body->position, s2MakeVec2(f[0], f[1])), s2MakeVec2(f[2], f[3]), s2Vec2_zero, body->rot,
								local);
	}
	return s2cGearRevolute(f[0], f[1], f[2], side2 ? gear->upperImpulse : gear->lowerImpulse, body->rot);
}

static bool s2IsGearInput(const s2World* world, const s2Joint* joint)
{
	return joint != NULL && (joint->type == s2_revoluteJoint || joint->type == s2_prismaticJoint) &&
		   world->bodies[joint->bodyIndexA].type == s2_staticBody;
}

// The gear joint has no counterpart in the reference. Invalid input creates nothing and returns s2_nullJointId.
s2JointId s2CreateGearJoint(s2WorldId worldId, const s2GearJointDef* def)
{
	s2World* world = s2GetWorldFromId(worldId);
	s2Joint* joint1 = s2FindJoint(world, def->jointId1);
	s2Joint* joint2 = s2FindJoint(world, def->jointId2);
	if (s2IsGearInput(world, joint1) == false || s2IsGearInput(world, joint2) == false ||
		joint1->bodyIndexB == joint2->bodyIndexB || s2IsValid(def->ratio) == false)
	{
		return s2_nullJointId;
	}

	// the constant is taken at the current poses
	s2SyncStateToHost(world);
	s2Joint* joint = s2AllocJoint(world, world->bodies + joint1->bodyIndexB, world->bodies + joint2->bodyIndexB);
	// (the allocation may have moved the joint array)
	joint1 = world->joints + def->jointId1.index;
	joint2 = world->joints + def->jointId2.index;
	joint->type = s2_gearJoint;
	joint->drawSize = 1.0f;
	joint->localOriginAnchorA = joint1->localOriginAnchorB;
	joint->localOriginAnchorB = joint2->localOriginAnchorB;
	joint->gearJoint1 = def->jointId1;
	joint->gearJoint2 = def->jointId2;
	joint->gearPrismatic1 = joint1->type == s2_prismaticJoint;
	joint->gearPrismatic2 = joint2->type == s2_prismaticJoint;
	joint->referenceAngle = def->ratio;
	joint->collideConnected = def->collideConnected;
	s2SetGearFrames(world, joint);
	s2cGearSide side1 = s2GearSideAt(world, joint, false);
	s2cGearSide side2 = s2GearSideAt(world, joint, true);
	joint->lowerImpulse = joint->gearPrismatic1 ? 0.0f : side1.coordinate;
	joint->upperImpulse = joint->gearPrismatic2 ? 0.0f : side2.coordinate;
	joint->lowerAngle = side1.coordinate + def->ratio * side2.coordinate;
	world->gearCount += 1;

	s2JointId jointId = {joint->object.index, world->index, joint->object.revision};
	return jointId;
}

void s2MoveGearFrames(s2World* world, int32_t bodyIndex)
{
	if (world->gearCount == 0 || world->bodies[bodyIndex].type != s2_staticBody)
	{
		return;
	}
	for (int32_t i = 0; i < world->jointPool.capacity; ++i)
	{
		s2Joint* gear = world->joints + i;
		if (s2ObjectValid(&gear->object) && gear->type == s2_gearJoint &&
			(world->joints[gear->gearJoint1.index].bodyIndexA == bodyIndex ||
			 world->joints[gear->gearJoint2.index].bodyIndexA == bodyIndex))
		{
			s2SetGearFrames(world, gear);
			s2MarkJointDirty(world, gear);
		}
	}
}

// the joint, or NULL for a joint of another type
static const s2Joint* s2GetGearJoint(s2JointId jointId)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	const s2Joint* joint = world->joints + jointId.index;
	S2_ASSERT(s2ObjectValid(&joint->object) && joint->object.revision == jointId.revision);
	return joint->type == s2_gearJoint ? joint : NULL;
}

s2JointId s2GearJoint_GetJoint1(s2JointId jointId)
{
	const s2Joint* joint = s2GetGearJoint(jointId);
	return joint != NULL ? joint->gearJoint1 : s2_nullJointId;
}

s2JointId s2GearJoint_GetJoint2(s2JointId jointId)
{
	const s2Joint* joint = s2GetGearJoint(jointId);
	return joint != NULL ? joint->gearJoint2 : s2_nullJointId;
}

float s2GearJoint_GetRatio(s2JointId jointId)
{
	const s2Joint* joint = s2GetGearJoint(jointId);
	return joint != NULL ? joint->referenceAngle : 0.0f;
}

// ---- reactions and break thresholds (DESIGN.md §3.13) -----------------------------------------------------------------

// s2JointType and the device's S2B_JOINT_* number the joint types alike
_Static_assert((int)s2_revoluteJoint == S2B_JOINT_REVOLUTE && (int)s2_mouseJoint == S2B_JOINT_MOUSE &&
				   (int)s2_weldJoint == S2B_JOINT_WELD && (int)s2_prismaticJoint == S2B_JOINT_PRISMATIC &&
				   (int)s2_motorJoint == S2B_JOINT_MOTOR && (int)s2_distanceJoint == S2B_JOINT_DISTANCE &&
				   (int)s2_wheelJoint == S2B_JOINT_WHEEL && (int)s2_pulleyJoint == S2B_JOINT_PULLEY &&
				   (int)s2_gearJoint == S2B_JOINT_GEAR,
			   "joint type numbering");

s2JointReaction s2ComputeJointReaction(int32_t type, s2Vec2 impulse, float motorImpulse, float lowerImpulse, float upperImpulse,
									   s2Rot qA, s2Vec2 localAxisA, float rate)
{
	return s2MakeJointReaction(type, impulse, motorImpulse, lowerImpulse, upperImpulse, qA, localAxisA, rate);
}

// from the lazily synced impulses and body A's rotation, at the rate of the last step: the numbers the device's pass tested
static s2JointReaction s2GetJointReaction(s2JointId jointId)
{
	s2World* world = s2GetWorldFromIndex(jointId.world);
	s2SyncStateToHost(world);
	const s2Joint* joint = world->joints + jointId.index;
	S2_ASSERT(s2ObjectValid(&joint->object) && joint->object.revision == jointId.revision);
	// a spring acts on the motor's axis: its impulse joins the motor argument (DESIGN.md §3.14). The flag is the one of the
	// row the device last solved, so the getters read what the device's reaction and break pass read for that step even
	// after s2*Joint_EnableSpring has changed the joint and before the next step uploads it.
	if (joint->type == s2_gearJoint)
	{
		// (lambda Jv2, lambda Jw2) through the generic branch, as the device's pass forms them (DESIGN.md §3.19)
		float angular;
		s2Vec2 linear = s2cGearReaction(&angular, joint->impulse.x, joint->referenceAngle, s2GearSideAt(world, joint, true));
		return s2MakeJointReaction(S2B_JOINT_GEAR, linear, angular, 0.0f, 0.0f, world->bodies[joint->bodyIndexA].rot,
								   s2Vec2_zero, world->reactionRate);
	}
	float motorImpulse = joint->springUploaded ? joint->motorImpulse + joint->springImpulse : joint->motorImpulse;
	// a distance joint passes its world axis at the end of the step (DESIGN.md §3.16), a pulley -ratio uB (§3.18)
	float length;
	s2Vec2 axis = joint->localAxisA;
	if (joint->type == s2_distanceJoint)
	{
		axis = s2DistanceJointAxis(world, joint, &length);
	}
	else if (joint->type == s2_pulleyJoint)
	{
		axis = s2PulleyJointAxis(world, joint, true, &length);
	}
	return s2MakeJointReaction((int32_t)joint->type, joint->impulse, motorImpulse, joint->lowerImpulse, joint->upperImpulse,
							   world->bodies[joint->bodyIndexA].rot, axis, world->reactionRate);
}

s2Vec2 s2Joint_GetReactionForce(s2JointId jointId)
{
	return s2GetJointReaction(jointId).force;
}

float s2Joint_GetReactionTorque(s2JointId jointId)
{
	return s2GetJointReaction(jointId).torque;
}

// a positive finite threshold sets it, 0 removes it; anything else is ignored
static void s2SetBreakThreshold(s2JointId jointId, float value, bool torque)
{
	if ((value >= 0.0f && value <= FLT_MAX) == false)
	{
		return; // rejected (negative, NaN or infinite): the joint keeps its threshold
	}
	s2World* world;
	s2Joint* joint = s2GetJointForEdit(jointId, &world);
	bool had = joint->breakForce > 0.0f || joint->breakTorque > 0.0f;
	if (torque)
	{
		joint->breakTorque = value;
	}
	else
	{
		joint->breakForce = value;
	}
	bool has = joint->breakForce > 0.0f || joint->breakTorque > 0.0f;
	world->breakableCount += (int32_t)has - (int32_t)had;
	s2MarkJointDirty(world, joint);
}

void s2Joint_SetBreakForce(s2JointId jointId, float breakForce)
{
	s2SetBreakThreshold(jointId, breakForce, false);
}

float s2Joint_GetBreakForce(s2JointId jointId)
{
	return s2GetWorldFromIndex(jointId.world)->joints[jointId.index].breakForce;
}

void s2Joint_SetBreakTorque(s2JointId jointId, float breakTorque)
{
	s2SetBreakThreshold(jointId, breakTorque, true);
}

float s2Joint_GetBreakTorque(s2JointId jointId)
{
	return s2GetWorldFromIndex(jointId.world)->joints[jointId.index].breakTorque;
}
