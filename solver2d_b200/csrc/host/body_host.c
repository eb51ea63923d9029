// solver2d-b200 — bodies and shapes behind the public API (behaviour of reference src/body.c, src/shape.c).
// All of this is host bookkeeping: it edits the host copy of an object and marks its row dirty; the next s2World_Step
// uploads the row. Reads of simulation state first make the host copy current (s2SyncStateToHost).
#include "s2_host.h"

#include <string.h>

s2Body* s2GetBody(s2World* world, s2BodyId id)
{
	S2_ASSERT(0 <= id.index && id.index < world->bodyPool.capacity);
	s2Body* body = world->bodies + id.index;
	S2_ASSERT(s2ObjectValid(&body->object));
	S2_ASSERT(id.revision == body->object.revision);
	return body;
}

// A new body slot (behaviour of reference src/body.c:17-63): state from the definition, no shapes and hence no mass yet.
s2BodyId s2CreateBody(s2WorldId worldId, const s2BodyDef* def)
{
	s2World* world = s2GetWorldFromId(worldId);
	s2Body* slot = (s2Body*)s2AllocObject(&world->bodyPool);
	world->bodies = (s2Body*)world->bodyPool.memory; // the pool may have moved
	int32_t used = slot->object.index + 1;
	world->bodyHighWater = used > world->bodyHighWater ? used : world->bodyHighWater;

	// what the definition prescribes
	slot->type = def->type;
	slot->userData = def->userData;
	slot->world = worldId.index;
	slot->rot = s2MakeRot(def->angle);
	slot->origin = slot->position = def->position; // centre of mass == origin until a shape with density arrives
	slot->linearVelocity = def->linearVelocity;
	slot->angularVelocity = def->angularVelocity;
	slot->linearDamping = def->linearDamping;
	slot->angularDamping = def->angularDamping;
	slot->gravityScale = def->gravityScale;
	// what a body without shapes is
	slot->localCenter = slot->force = s2Vec2_zero;
	slot->torque = 0.0f;
	slot->mass = slot->invMass = slot->I = slot->invI = 0.0f;
	slot->shapeList = S2_NULL_INDEX;
	slot->jointCount = 0;
	// device mirror: not there yet (rowDirty / forceDirty keep their value — a reused slot may already sit in the dirty list)
	slot->onDevice = false;
	slot->teleported = false;
	s2MarkBodyDirty(world, slot);

	return (s2BodyId){slot->object.index, worldId.index, slot->object.revision};
}

static void s2DestroyShapeProxy(s2World* world, s2Shape* shape)
{
	int type = shape->proxyKey & 0xF;
	s2FreeProxyId(world->proxyIds + type, shape->proxyKey >> 4);
	shape->proxyKey = S2_NULL_INDEX;
}

// reference src/body.c:75-150. Contacts of the body live on the device: invalidating its shape rows makes the next pair
// pass drop them.
void s2DestroyBody(s2BodyId bodyId)
{
	s2World* world = s2GetWorldFromIndex(bodyId.world);
	s2Body* body = world->bodies + bodyId.index;
	S2_ASSERT(body->jointCount == 0);

	int32_t shapeIndex = body->shapeList;
	while (shapeIndex != S2_NULL_INDEX)
	{
		s2Shape* shape = world->shapes + shapeIndex;
		shapeIndex = shape->nextShapeIndex;
		s2DestroyShapeProxy(world, shape);
		s2FreeObject(&world->shapePool, &shape->object);
		s2MarkShapeDirty(world, shape);
	}
	s2FreeObject(&world->bodyPool, &body->object);
	body->onDevice = false;
	s2MarkBodyDirty(world, body);
}

// per shape kind: tight box and mass properties, dispatched through tables indexed by s2ShapeType
typedef s2Box s2ShapeBoxFcn(const void* geometry, s2Transform xf);
typedef s2MassData s2ShapeMassFcn(const void* geometry, float density);

static s2Box s2BoxOfCapsule(const void* g, s2Transform xf)
{
	return s2ComputeCapsuleAABB((const s2Capsule*)g, xf);
}
static s2Box s2BoxOfCircle(const void* g, s2Transform xf)
{
	return s2ComputeCircleAABB((const s2Circle*)g, xf);
}
static s2Box s2BoxOfPolygon(const void* g, s2Transform xf)
{
	return s2ComputePolygonAABB((const s2Polygon*)g, xf);
}
static s2Box s2BoxOfSegment(const void* g, s2Transform xf)
{
	return s2ComputeSegmentAABB((const s2Segment*)g, xf);
}
static s2MassData s2MassOfCapsule(const void* g, float density)
{
	return s2ComputeCapsuleMass((const s2Capsule*)g, density);
}
static s2MassData s2MassOfCircle(const void* g, float density)
{
	return s2ComputeCircleMass((const s2Circle*)g, density);
}
static s2MassData s2MassOfPolygon(const void* g, float density)
{
	return s2ComputePolygonMass((const s2Polygon*)g, density);
}

static s2ShapeBoxFcn* const s2_shapeBox[s2_shapeTypeCount] = {
	[s2_capsuleShape] = s2BoxOfCapsule, [s2_circleShape] = s2BoxOfCircle, [s2_polygonShape] = s2BoxOfPolygon, [s2_segmentShape] = s2BoxOfSegment};
// (a segment has no area: no entry, no mass)
static s2ShapeMassFcn* const s2_shapeMass[s2_shapeTypeCount] = {
	[s2_capsuleShape] = s2MassOfCapsule, [s2_circleShape] = s2MassOfCircle, [s2_polygonShape] = s2MassOfPolygon};

s2Box s2Shape_ComputeAABB(const s2Shape* shape, s2Transform xf)
{
	if ((unsigned)shape->type < (unsigned)s2_shapeTypeCount && s2_shapeBox[shape->type] != NULL)
	{
		return s2_shapeBox[shape->type](&shape->capsule, xf); // the geometry union starts at its first member
	}
	return (s2Box){xf.p, xf.p};
}

s2MassData s2Shape_ComputeMass(const s2Shape* shape)
{
	if ((unsigned)shape->type < (unsigned)s2_shapeTypeCount && s2_shapeMass[shape->type] != NULL)
	{
		return s2_shapeMass[shape->type](&shape->capsule, shape->density);
	}
	return (s2MassData){0};
}

// Mass, centre of mass and inertia about it of a body from the shapes attached to it (behaviour of reference
// src/body.c:152-218; sums run over the shape list in list order, the float operations are the reference's).
typedef struct s2MassSum
{
	float mass;		 // sum of the shape masses
	s2Vec2 moment;	 // sum of mass x centre (body frame)
	float inertia;	 // sum of the shape inertias about the body origin
} s2MassSum;

static s2MassSum s2SumShapeMasses(const s2World* world, const s2Body* body)
{
	s2MassSum sum = {0.0f, {0.0f, 0.0f}, 0.0f};
	int32_t next = body->shapeList;
	while (next != S2_NULL_INDEX)
	{
		const s2Shape* shape = world->shapes + next;
		next = shape->nextShapeIndex;
		if (shape->density != 0.0f)
		{
			s2MassData part = s2Shape_ComputeMass(shape);
			sum.mass += part.mass;
			sum.moment = s2MulAdd(sum.moment, part.mass, part.center);
			sum.inertia += part.I;
		}
	}
	return sum;
}

static void s2UpdateBodyMass(s2World* world, s2Body* b)
{
	b->mass = b->invMass = b->I = b->invI = 0.0f;
	b->localCenter = s2Vec2_zero;
	if (b->type != s2_dynamicBody)
	{
		// static and kinematic bodies have no mass: the "centre of mass" is the origin
		b->position = b->origin;
		return;
	}

	s2MassSum sum = s2SumShapeMasses(world, b);
	s2Vec2 center = sum.moment;
	b->mass = sum.mass;
	if (sum.mass > 0.0f)
	{
		b->invMass = 1.0f / sum.mass;
		center = s2MulSV(b->invMass, center);
	}
	if (sum.inertia > 0.0f)
	{
		// from the body origin to the centre of mass (parallel axes)
		b->I = sum.inertia - b->mass * s2Dot(center, center);
		b->invI = 1.0f / b->I;
	}

	// the centre of mass moved inside the body: keep the velocity of the material (v refers to the centre of mass)
	s2Vec2 before = b->position;
	b->localCenter = center;
	b->position = s2Add(s2RotateVector(b->rot, center), b->origin);
	b->linearVelocity = s2Add(b->linearVelocity, s2CrossSV(b->angularVelocity, s2Sub(b->position, before)));
}

// reference src/body.c:220-280 + s2Shape_CreateProxy (src/shape.c:48-67)
static s2ShapeId s2CreateShape(s2BodyId bodyId, const s2ShapeDef* def, const void* geometry, s2ShapeType shapeType)
{
	s2World* world = s2GetWorldFromIndex(bodyId.world);
	s2SyncStateToHost(world); // the body's transform and velocity are read below

	s2Shape* shape = (s2Shape*)s2AllocObject(&world->shapePool);
	world->shapes = (s2Shape*)world->shapePool.memory;
	s2Body* body = world->bodies + bodyId.index;

	switch (shapeType)
	{
		case s2_capsuleShape:
			shape->capsule = *(const s2Capsule*)geometry;
			break;
		case s2_circleShape:
			shape->circle = *(const s2Circle*)geometry;
			break;
		case s2_polygonShape:
			shape->polygon = *(const s2Polygon*)geometry;
			break;
		case s2_segmentShape:
			shape->segment = *(const s2Segment*)geometry;
			break;
		default:
			break;
	}

	shape->bodyIndex = body->object.index;
	shape->type = shapeType;
	shape->density = def->density;
	shape->friction = def->friction;
	S2_ASSERT(s2IsValid(def->restitution) && def->restitution >= 0.0f);
	shape->restitution = def->restitution;
	shape->userData = def->userData;
	shape->filter = def->filter;
	shape->fresh = true; // rowDirty keeps its value: a reused slot may already sit in the dirty list

	// tight AABB + speculative margin; fat AABB adds the move margin for movable bodies
	s2Transform xf = {body->origin, body->rot};
	shape->aabb = s2Shape_ComputeAABB(shape, xf);
	shape->aabb.lowerBound.x -= s2_speculativeDistance;
	shape->aabb.lowerBound.y -= s2_speculativeDistance;
	shape->aabb.upperBound.x += s2_speculativeDistance;
	shape->aabb.upperBound.y += s2_speculativeDistance;
	float margin = body->type == s2_staticBody ? s2_speculativeDistance : s2_aabbMargin + s2_speculativeDistance;
	shape->fatAABB.lowerBound.x = shape->aabb.lowerBound.x - margin;
	shape->fatAABB.lowerBound.y = shape->aabb.lowerBound.y - margin;
	shape->fatAABB.upperBound.x = shape->aabb.upperBound.x + margin;
	shape->fatAABB.upperBound.y = shape->aabb.upperBound.y + margin;

	// proxy key of the reference broad phase: (tree node id << 4) | body type (reference src/broad_phase.h:18-20)
	int32_t proxyId = s2AllocProxyId(world->proxyIds + body->type);
	shape->proxyKey = (proxyId << 4) | (int32_t)body->type;

	shape->nextShapeIndex = body->shapeList;
	body->shapeList = shape->object.index;

	if (shape->density)
	{
		s2UpdateBodyMass(world, body);
	}

	s2MarkShapeDirty(world, shape);
	s2MarkBodyDirty(world, body);

	s2ShapeId id = {shape->object.index, bodyId.world, shape->object.revision};
	return id;
}

s2ShapeId s2CreateCircleShape(s2BodyId bodyId, const s2ShapeDef* def, const s2Circle* circle)
{
	return s2CreateShape(bodyId, def, circle, s2_circleShape);
}

s2ShapeId s2CreatePolygonShape(s2BodyId bodyId, const s2ShapeDef* def, const s2Polygon* polygon)
{
	return s2CreateShape(bodyId, def, polygon, s2_polygonShape);
}

s2ShapeId s2CreateSegmentShape(s2BodyId bodyId, const s2ShapeDef* def, const s2Segment* segment)
{
	if (s2DistanceSquared(segment->point1, segment->point2) <= s2_linearSlop * s2_linearSlop)
	{
		return s2_nullShapeId;
	}
	return s2CreateShape(bodyId, def, segment, s2_segmentShape);
}

s2ShapeId s2CreateCapsuleShape(s2BodyId bodyId, const s2ShapeDef* def, const s2Capsule* capsule)
{
	if (s2DistanceSquared(capsule->point1, capsule->point2) <= s2_linearSlop * s2_linearSlop)
	{
		return s2_nullShapeId;
	}
	return s2CreateShape(bodyId, def, capsule, s2_capsuleShape);
}

// ---- accessors (reference src/body.c:313-384) ---------------------------------------------------------------------

s2Vec2 s2Body_GetPosition(s2BodyId bodyId)
{
	s2World* world = s2GetWorldFromIndex(bodyId.world);
	s2SyncStateToHost(world);
	return world->bodies[bodyId.index].origin;
}

float s2Body_GetAngle(s2BodyId bodyId)
{
	s2World* world = s2GetWorldFromIndex(bodyId.world);
	s2SyncStateToHost(world);
	return s2Rot_GetAngle(world->bodies[bodyId.index].rot);
}

s2Vec2 s2Body_GetLocalPoint(s2BodyId bodyId, s2Vec2 globalPoint)
{
	s2World* world = s2GetWorldFromIndex(bodyId.world);
	s2SyncStateToHost(world);
	s2Body* body = s2GetBody(world, bodyId);
	s2Transform xf = {body->origin, body->rot};
	return s2InvTransformPoint(xf, globalPoint);
}

// Declared by the reference API (solver2d.h:38) but never defined there; provided here as a teleport.
void s2Body_SetTransform(s2BodyId bodyId, s2Vec2 position, float angle)
{
	s2World* world = s2GetWorldFromIndex(bodyId.world);
	s2SyncStateToHost(world);
	s2SyncBoxesToHost(world);
	s2Body* body = s2GetBody(world, bodyId);
	body->origin = position;
	body->rot = s2MakeRot(angle);
	body->position = s2Add(s2RotateVector(body->rot, body->localCenter), body->origin);
	// the body is placed exactly where asked: the delta position XPBD carries for a kinematic body goes (DESIGN.md §3.8)
	body->teleported = true;
	s2MarkBodyDirty(world, body);
	s2Transform xf = {body->origin, body->rot};
	for (int32_t si = body->shapeList; si != S2_NULL_INDEX;)
	{
		s2Shape* shape = world->shapes + si;
		si = shape->nextShapeIndex;
		shape->aabb = s2Shape_ComputeAABB(shape, xf);
		shape->aabb.lowerBound.x -= s2_speculativeDistance;
		shape->aabb.lowerBound.y -= s2_speculativeDistance;
		shape->aabb.upperBound.x += s2_speculativeDistance;
		shape->aabb.upperBound.y += s2_speculativeDistance;
		float margin = body->type == s2_staticBody ? s2_speculativeDistance : s2_aabbMargin + s2_speculativeDistance;
		shape->fatAABB.lowerBound.x = shape->aabb.lowerBound.x - margin;
		shape->fatAABB.lowerBound.y = shape->aabb.lowerBound.y - margin;
		shape->fatAABB.upperBound.x = shape->aabb.upperBound.x + margin;
		shape->fatAABB.upperBound.y = shape->aabb.upperBound.y + margin;
		shape->fresh = true; // re-buffer the proxy as moved
		s2MarkShapeDirty(world, shape);
	}
}

void s2Body_SetLinearVelocity(s2BodyId bodyId, s2Vec2 linearVelocity)
{
	s2World* world = s2GetWorldFromIndex(bodyId.world);
	s2SyncStateToHost(world);
	s2Body* body = world->bodies + bodyId.index;
	body->linearVelocity = linearVelocity;
	s2MarkBodyDirty(world, body);
}

void s2Body_SetAngularVelocity(s2BodyId bodyId, float angularVelocity)
{
	s2World* world = s2GetWorldFromIndex(bodyId.world);
	s2SyncStateToHost(world);
	s2Body* body = world->bodies + bodyId.index;
	body->angularVelocity = angularVelocity;
	s2MarkBodyDirty(world, body);
}

// Forces are host-authoritative between steps (the device zeroes them at the end of every step, reference
// src/world.c:275-276), so accumulating one needs no read-back: only the 16-byte force row travels.
void s2Body_ApplyForceToCenter(s2BodyId bodyId, s2Vec2 force)
{
	s2World* world = s2GetWorldFromIndex(bodyId.world);
	s2Body* body = s2GetBody(world, bodyId);
	// the host copy is zeroed whenever it is uploaded (s2FlushToDevice), mirroring the reset at the end of the step
	body->force = s2Add(body->force, force);
	s2MarkBodyForceDirty(world, body);
}

void s2Body_ApplyLinearImpulse(s2BodyId bodyId, s2Vec2 impulse, s2Vec2 point)
{
	s2World* world = s2GetWorldFromIndex(bodyId.world);
	s2SyncStateToHost(world);
	s2Body* body = s2GetBody(world, bodyId);
	if (body->type != s2_dynamicBody)
	{
		return;
	}
	body->linearVelocity = s2MulAdd(body->linearVelocity, body->invMass, impulse);
	body->angularVelocity += body->invI * s2Cross(s2Sub(point, body->position), impulse);
	s2MarkBodyDirty(world, body);
}

s2BodyType s2Body_GetType(s2BodyId bodyId)
{
	s2World* world = s2GetWorldFromIndex(bodyId.world);
	return world->bodies[bodyId.index].type;
}

float s2Body_GetMass(s2BodyId bodyId)
{
	s2World* world = s2GetWorldFromIndex(bodyId.world);
	return world->bodies[bodyId.index].mass;
}

// ---- shapes (reference src/shape.c:91-137) ------------------------------------------------------------------------

s2BodyId s2Shape_GetBody(s2ShapeId shapeId)
{
	s2World* world = s2GetWorldFromIndex(shapeId.world);
	s2Shape* shape = world->shapes + shapeId.index;
	s2Body* body = world->bodies + shape->bodyIndex;
	s2BodyId bodyId = {body->object.index, shapeId.world, body->object.revision};
	return bodyId;
}

bool s2Shape_TestPoint(s2ShapeId shapeId, s2Vec2 point)
{
	s2World* world = s2GetWorldFromIndex(shapeId.world);
	s2SyncStateToHost(world);
	s2Shape* shape = world->shapes + shapeId.index;
	s2Body* body = world->bodies + shape->bodyIndex;
	s2Transform xf = {body->origin, body->rot};
	s2Vec2 localPoint = s2InvTransformPoint(xf, point);
	switch (shape->type)
	{
		case s2_capsuleShape:
			return s2PointInCapsule(localPoint, &shape->capsule);
		case s2_circleShape:
			return s2PointInCircle(localPoint, &shape->circle);
		case s2_polygonShape:
			return s2PointInPolygon(localPoint, &shape->polygon);
		default:
			return false;
	}
}
