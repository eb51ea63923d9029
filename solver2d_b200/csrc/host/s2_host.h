// solver2d-b200 — host-side object model behind the public C API.
//
// The host keeps what clients author and read: body / shape / joint definitions, id + revision pools with the same
// reuse semantics as the reference (src/pool.c:108-159: LIFO free list, revision bumped on reuse, growth by 1.5x) and a
// lazily refreshed copy of the simulation state. Everything s2World_Step computes lives on the device (s2b_device.h);
// the host only (a) uploads rows that changed since the last step and (b) pulls state back the first time a client
// reads it after a step.
#pragma once

#include "s2b_device.h"

// everything declared by the public headers is exported from the shared library; the rest of the host code is
// compiled with -fvisibility=hidden
#pragma GCC visibility push(default)
#include "solver2d/solver2d.h"

#include "solver2d/aabb.h"
#include "solver2d/constants.h"
#include "solver2d/debug_draw.h"
#include "solver2d/distance.h"
#include "solver2d/geometry.h"
#include "solver2d/hull.h"
#include "solver2d/manifold.h"
#include "solver2d/math.h"
#pragma GCC visibility pop

#include <stdbool.h>
#include <stdint.h>

#define S2_EXPORT __attribute__((visibility("default")))

#if defined(_DEBUG)
	#include <assert.h>
	#define S2_ASSERT(c) assert(c)
#else
	#define S2_ASSERT(...) ((void)0)
#endif

// ---- pools ------------------------------------------------------------------------------------------------------

// first member of every pooled struct; a live object has next == index
typedef struct s2Object
{
	int32_t index;
	int32_t next;
	uint16_t revision;
} s2Object;

typedef struct s2Pool
{
	char* memory;
	int32_t objectSize;
	int32_t capacity;
	int32_t count;
	int32_t freeList;
} s2Pool;

s2Pool s2CreatePool(int32_t objectSize, int32_t capacity);
void s2DestroyPool(s2Pool* pool);
s2Object* s2AllocObject(s2Pool* pool);
void s2FreeObject(s2Pool* pool, s2Object* object);

static inline bool s2ObjectValid(const s2Object* object)
{
	return object->index == object->next;
}

static inline bool s2IsFree(const s2Object* object)
{
	return object->index != object->next;
}

// ---- objects ----------------------------------------------------------------------------------------------------

typedef enum s2ShapeType
{
	s2_capsuleShape,
	s2_circleShape,
	s2_polygonShape,
	s2_segmentShape,
	s2_shapeTypeCount
} s2ShapeType;

typedef enum s2JointType
{
	s2_revoluteJoint,
	s2_mouseJoint,
	s2_weldJoint,
	s2_prismaticJoint,
} s2JointType;

typedef struct s2Body
{
	s2Object object;
	enum s2BodyType type;

	// simulation state (a cache of the device columns, see s2World.stateFresh)
	s2Vec2 origin;
	s2Vec2 position; // centre of mass
	s2Rot rot;
	s2Vec2 linearVelocity;
	float angularVelocity;
	s2Vec2 force;
	float torque;

	// authored / derived
	s2Vec2 localCenter;
	float mass, invMass;
	float I, invI;
	float linearDamping;
	float angularDamping;
	float gravityScale;

	int32_t shapeList;
	int32_t jointCount;
	void* userData;
	int16_t world;

	// dirty bookkeeping
	bool rowDirty;	 // whole row must be re-uploaded
	bool forceDirty; // only force / torque changed
	bool teleported; // moved by s2Body_SetTransform since the last upload: the device resets its delta position
	bool onDevice;	 // the device already holds a row for this body: uploads add its pending force instead of setting it
} s2Body;

typedef struct s2Shape
{
	s2Object object;
	int32_t bodyIndex;
	int32_t nextShapeIndex;
	enum s2ShapeType type;
	float density;
	float friction;
	float restitution;
	s2Filter filter;
	s2Box aabb;
	s2Box fatAABB;
	int32_t proxyKey;
	void* userData;
	bool rowDirty;
	bool fresh; // created since the last upload

	union
	{
		s2Capsule capsule;
		s2Circle circle;
		s2Polygon polygon;
		s2Segment segment;
	};
} s2Shape;

typedef struct s2Joint
{
	s2Object object;
	s2JointType type;
	int32_t bodyIndexA, bodyIndexB;
	s2Vec2 localOriginAnchorA;
	s2Vec2 localOriginAnchorB;
	float drawSize;
	bool collideConnected;

	// revolute; a prismatic joint keeps its translation limits in lowerAngle / upperAngle and its maximum motor force in
	// maxMotorTorque, as its device row does
	bool enableMotor, enableLimit;
	float maxMotorTorque, motorSpeed;
	float referenceAngle, lowerAngle, upperAngle;
	// prismatic
	s2Vec2 localAxisA;
	// mouse
	float hertz, dampingRatio;
	s2Vec2 targetA;
	// accumulated impulses (cache of the device columns)
	s2Vec2 impulse;
	float motorImpulse, lowerImpulse, upperImpulse;

	bool rowDirty;
} s2Joint;

// Emulation of the node-id allocator of one reference dynamic tree (src/dynamic_tree.c:105-167) so that proxy keys —
// which decide the (A, B) order of every contact (reference src/broad_phase.c:196-205) — match the reference.
typedef struct s2ProxyIds
{
	int32_t* freeStack; // freed ids, LIFO; -1 marks a freed internal node
	int32_t freeCount, freeCapacity;
	int32_t nextFresh;
	int32_t proxyCount;
} s2ProxyIds;

typedef struct s2IndexList
{
	int32_t* data;
	int32_t count, capacity;
} s2IndexList;

typedef struct s2World
{
	int16_t index;
	uint16_t revision;
	bool inUse;
	s2SolverType solverType;

	s2Pool bodyPool, shapePool, jointPool;
	s2Body* bodies;
	s2Shape* shapes;
	s2Joint* joints;

	s2ProxyIds proxyIds[s2_bodyTypeCount];

	s2bWorld* device;
	s2IndexList dirtyBodies, dirtyForces, dirtyShapes, dirtyJoints;
	bool jointPairsDirty;
	// restitution (include/solver2d_b200.h): pushed to the device by the next flush when restitutionDirty
	bool enableRestitution;
	float restitutionThreshold;
	bool restitutionDirty;
	bool stateFresh;	 // host body / joint state mirrors the device
	bool boxesFresh;	 // host shape AABBs mirror the device
	uint64_t stepId;
	int32_t bodyHighWater; // one past the largest body slot ever used
	s2Vec2 gravity;

	// row staging (pinned host memory owned by the device library)
	void* staging;
	size_t stagingBytes;
} s2World;

// mirrors s2StepContext (reference src/solvers.h:13-24); `bodies` is unused because the solver runs on the device
typedef struct s2StepContext
{
	float dt;
	float inv_dt;
	float h;
	float inv_h;
	int32_t iterations;
	int32_t extraIterations;
	s2Body* bodies;
	int32_t bodyCapacity;
	bool warmStart;
} s2StepContext;

s2World* s2GetWorldFromId(s2WorldId id);
s2World* s2GetWorldFromIndex(int16_t index);
s2Body* s2GetBody(s2World* world, s2BodyId id);

// make the host copy of the simulation state current (lazy read-back after a step)
void s2SyncStateToHost(s2World* world);
void s2SyncBoxesToHost(s2World* world);
// push every dirty row to the device
void s2FlushToDevice(s2World* world);

void s2MarkBodyDirty(s2World* world, s2Body* body);
void s2MarkBodyForceDirty(s2World* world, s2Body* body);
void s2MarkShapeDirty(s2World* world, s2Shape* shape);
void s2MarkJointDirty(s2World* world, s2Joint* joint);
void s2IndexListPush(s2IndexList* list, int32_t value);

int32_t s2AllocProxyId(s2ProxyIds* ids);
void s2FreeProxyId(s2ProxyIds* ids, int32_t proxyId);

s2Box s2Shape_ComputeAABB(const s2Shape* shape, s2Transform xf);
s2MassData s2Shape_ComputeMass(const s2Shape* shape);

// per-variant solver entry points (names and shape of reference src/solvers.h:70-79); each enqueues the variant's
// kernel schedule on the world's device
S2_EXPORT void s2Solve_Jacobi(s2World* world, s2StepContext* stepContext);
S2_EXPORT void s2Solve_PGS(s2World* world, s2StepContext* stepContext);
S2_EXPORT void s2Solve_PGS_NGS(s2World* world, s2StepContext* context);
S2_EXPORT void s2Solve_PGS_NGS_Block(s2World* world, s2StepContext* stepContext);
S2_EXPORT void s2Solve_PGS_Soft(s2World* world, s2StepContext* stepContext);
S2_EXPORT void s2Solve_TGS_Soft(s2World* world, s2StepContext* stepContext);
S2_EXPORT void s2Solve_TGS_Sticky(s2World* world, s2StepContext* stepContext);
S2_EXPORT void s2Solve_TGS_NGS(s2World* world, s2StepContext* stepContext);
S2_EXPORT void s2Solve_XPBD(s2World* world, s2StepContext* stepContext);
S2_EXPORT void s2Solve_SoftStep(s2World* world, s2StepContext* stepContext);
