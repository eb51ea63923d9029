// solver2d-b200 — world registry and the step driver behind s2CreateWorld / s2World_Step (reference src/world.c).
//
// s2World_Step keeps the reference's stage order (world.c:120-306) but every stage is an enqueue on the world's CUDA
// stream:
//     flush dirty rows  ->  s2b_update_pairs  ->  s2b_update_contacts  ->  s2Solve_<variant>  ->  s2b_finalize
// The host does not wait for the step; the first API read after it (s2Body_GetPosition, s2World_Draw, ...) pulls the
// state back once (s2SyncStateToHost).
#include "s2_host.h"

#include <stdio.h>
#include <stdlib.h>
#include <string.h>

static s2World s2_worlds[s2_maxWorlds];

s2World* s2GetWorldFromId(s2WorldId id)
{
	S2_ASSERT(0 <= id.index && id.index < s2_maxWorlds);
	s2World* world = s2_worlds + id.index;
	S2_ASSERT(id.revision == world->revision);
	return world;
}

s2World* s2GetWorldFromIndex(int16_t index)
{
	S2_ASSERT(0 <= index && index < s2_maxWorlds);
	return s2_worlds + index;
}

// ---- small containers -------------------------------------------------------------------------------------------

void s2IndexListPush(s2IndexList* list, int32_t value)
{
	if (list->count == list->capacity)
	{
		list->capacity = list->capacity ? 2 * list->capacity : 64;
		list->data = (int32_t*)realloc(list->data, sizeof(int32_t) * (size_t)list->capacity);
	}
	list->data[list->count++] = value;
}

static void s2IndexListFree(s2IndexList* list)
{
	free(list->data);
	memset(list, 0, sizeof(*list));
}

// node-id allocator of a reference dynamic tree: pops the free list (LIFO), else the next never-used id
int32_t s2AllocProxyId(s2ProxyIds* ids)
{
	int32_t leaf = -1;
	while (ids->freeCount > 0 && leaf < 0)
	{
		leaf = ids->freeStack[--ids->freeCount];
	}
	if (leaf < 0)
	{
		leaf = ids->nextFresh++;
	}
	if (ids->proxyCount > 0)
	{
		// inserting into a non-empty tree also allocates the new parent node (reference src/dynamic_tree.c:625)
		if (ids->freeCount > 0)
		{
			ids->freeCount -= 1;
		}
		else
		{
			ids->nextFresh += 1;
		}
	}
	ids->proxyCount += 1;
	return leaf;
}

static void s2ProxyPush(s2ProxyIds* ids, int32_t value)
{
	if (ids->freeCount == ids->freeCapacity)
	{
		ids->freeCapacity = ids->freeCapacity ? 2 * ids->freeCapacity : 64;
		ids->freeStack = (int32_t*)realloc(ids->freeStack, sizeof(int32_t) * (size_t)ids->freeCapacity);
	}
	ids->freeStack[ids->freeCount++] = value;
}

void s2FreeProxyId(s2ProxyIds* ids, int32_t proxyId)
{
	// removing a leaf frees its parent node first (unless it was the root), then the leaf itself
	// (reference src/dynamic_tree.c:686-783)
	if (ids->proxyCount > 1)
	{
		s2ProxyPush(ids, -1);
	}
	s2ProxyPush(ids, proxyId);
	ids->proxyCount -= 1;
}

// ---- dirty tracking ---------------------------------------------------------------------------------------------

void s2MarkBodyDirty(s2World* world, s2Body* body)
{
	if (body->rowDirty == false)
	{
		body->rowDirty = true;
		s2IndexListPush(&world->dirtyBodies, body->object.index);
	}
}

void s2MarkBodyForceDirty(s2World* world, s2Body* body)
{
	if (body->rowDirty == false && body->forceDirty == false)
	{
		body->forceDirty = true;
		s2IndexListPush(&world->dirtyForces, body->object.index);
	}
}

void s2MarkShapeDirty(s2World* world, s2Shape* shape)
{
	if (shape->rowDirty == false)
	{
		shape->rowDirty = true;
		s2IndexListPush(&world->dirtyShapes, shape->object.index);
	}
}

void s2MarkJointDirty(s2World* world, s2Joint* joint)
{
	if (joint->rowDirty == false)
	{
		joint->rowDirty = true;
		s2IndexListPush(&world->dirtyJoints, joint->object.index);
	}
}

static void* s2Staging(s2World* world, size_t bytes)
{
	if (bytes > world->stagingBytes)
	{
		if (world->staging)
		{
			s2b_host_free(world->staging);
		}
		world->stagingBytes = bytes + bytes / 2 + 4096;
		world->staging = s2b_host_alloc(world->stagingBytes);
	}
	return world->staging;
}

static void s2FillBodyRow(s2bBodyRow* r, const s2Body* b)
{
	r->index = b->object.index;
	r->flags = s2IsFree(&b->object) ? 0 : (S2B_ROW_VALID | ((int32_t)b->type << 1) | (b->onDevice ? S2B_BODY_ADD_FORCE : 0) |
											 (b->teleported ? S2B_BODY_TELEPORT : 0));
	r->origin[0] = b->origin.x;
	r->origin[1] = b->origin.y;
	r->position[0] = b->position.x;
	r->position[1] = b->position.y;
	r->rot[0] = b->rot.s;
	r->rot[1] = b->rot.c;
	r->linearVelocity[0] = b->linearVelocity.x;
	r->linearVelocity[1] = b->linearVelocity.y;
	r->angularVelocity = b->angularVelocity;
	r->localCenter[0] = b->localCenter.x;
	r->localCenter[1] = b->localCenter.y;
	r->mass = b->mass;
	r->invMass = b->invMass;
	r->I = b->I;
	r->invI = b->invI;
	r->force[0] = b->force.x;
	r->force[1] = b->force.y;
	r->torque = b->torque;
	r->linearDamping = b->linearDamping;
	r->angularDamping = b->angularDamping;
	r->gravityScale = b->gravityScale;
}

static void s2FillShapeRow(s2bShapeRow* r, const s2Shape* s)
{
	memset(r, 0, sizeof(*r));
	r->index = s->object.index;
	if (s2IsFree(&s->object))
	{
		return;
	}
	r->flags = S2B_ROW_VALID | ((int32_t)s->type << 1);
	r->body = s->bodyIndex;
	r->proxyKey = s->proxyKey;
	r->categoryBits = s->filter.categoryBits;
	r->maskBits = s->filter.maskBits;
	r->groupIndex = s->filter.groupIndex;
	r->friction = s->friction;
	r->restitution = s->restitution;
	r->aabb[0] = s->aabb.lowerBound.x;
	r->aabb[1] = s->aabb.lowerBound.y;
	r->aabb[2] = s->aabb.upperBound.x;
	r->aabb[3] = s->aabb.upperBound.y;
	r->fatAABB[0] = s->fatAABB.lowerBound.x;
	r->fatAABB[1] = s->fatAABB.lowerBound.y;
	r->fatAABB[2] = s->fatAABB.upperBound.x;
	r->fatAABB[3] = s->fatAABB.upperBound.y;

	// polygon form of every shape kind (see s2b_device.h)
	s2Polygon poly;
	switch (s->type)
	{
		case s2_circleShape:
			memset(&poly, 0, sizeof(poly));
			poly.vertices[0] = s->circle.point;
			poly.count = 1;
			poly.radius = s->circle.radius;
			break;
		case s2_capsuleShape:
			poly = s2MakeCapsule(s->capsule.point1, s->capsule.point2, s->capsule.radius);
			break;
		case s2_segmentShape:
			poly = s2MakeCapsule(s->segment.point1, s->segment.point2, 0.0f);
			break;
		default:
			poly = s->polygon;
			break;
	}
	r->radius = poly.radius;
	r->count = poly.count;
	for (int i = 0; i < poly.count && i < s2_maxPolygonVertices; ++i)
	{
		r->vertices[2 * i] = poly.vertices[i].x;
		r->vertices[2 * i + 1] = poly.vertices[i].y;
		r->normals[2 * i] = poly.normals[i].x;
		r->normals[2 * i + 1] = poly.normals[i].y;
	}
}

static void s2FillJointRow(s2bJointRow* r, const s2Joint* j)
{
	memset(r, 0, sizeof(*r));
	r->index = j->object.index;
	if (s2IsFree(&j->object))
	{
		return;
	}
	int type = S2B_JOINT_REVOLUTE;
	switch (j->type)
	{
		case s2_revoluteJoint:
			type = S2B_JOINT_REVOLUTE;
			break;
		case s2_mouseJoint:
			type = S2B_JOINT_MOUSE;
			break;
		case s2_weldJoint:
			type = S2B_JOINT_WELD;
			break;
		case s2_prismaticJoint:
			type = S2B_JOINT_PRISMATIC;
			break;
	}
	r->flags = S2B_ROW_VALID | (type << 1);
	// a weld is created with enableLimit == enableMotor == false, so its row never carries either flag
	r->flags |= j->enableLimit ? S2B_JOINT_ENABLE_LIMIT : 0;
	r->flags |= j->enableMotor ? S2B_JOINT_ENABLE_MOTOR : 0;
	r->flags |= j->collideConnected ? S2B_JOINT_COLLIDE_CONNECTED : 0;
	r->bodyA = j->bodyIndexA;
	r->bodyB = j->bodyIndexB;
	r->localOriginAnchorA[0] = j->localOriginAnchorA.x;
	r->localOriginAnchorA[1] = j->localOriginAnchorA.y;
	r->localOriginAnchorB[0] = j->localOriginAnchorB.x;
	r->localOriginAnchorB[1] = j->localOriginAnchorB.y;
	r->referenceAngle = j->referenceAngle;
	r->lowerAngle = j->lowerAngle;
	r->upperAngle = j->upperAngle;
	r->maxMotorTorque = j->maxMotorTorque;
	r->motorSpeed = j->motorSpeed;
	r->hertz = j->hertz;
	r->dampingRatio = j->dampingRatio;
	r->target[0] = j->targetA.x;
	r->target[1] = j->targetA.y;
	r->impulse[0] = j->impulse.x;
	r->impulse[1] = j->impulse.y;
	r->motorImpulse = j->motorImpulse;
	r->lowerImpulse = j->lowerImpulse;
	r->upperImpulse = j->upperImpulse;
	r->localAxisA[0] = j->localAxisA.x;
	r->localAxisA[1] = j->localAxisA.y;
}

static int s2CompareU64(const void* a, const void* b)
{
	uint64_t x = *(const uint64_t*)a, y = *(const uint64_t*)b;
	return x < y ? -1 : (x > y ? 1 : 0);
}

void s2FlushToDevice(s2World* world)
{
	s2bWorld* dev = world->device;

	if (world->dirtyBodies.count > 0)
	{
		int n = world->dirtyBodies.count;
		s2bBodyRow* rows = (s2bBodyRow*)s2Staging(world, sizeof(s2bBodyRow) * (size_t)n);
		for (int i = 0; i < n; ++i)
		{
			s2Body* b = world->bodies + world->dirtyBodies.data[i];
			s2FillBodyRow(rows + i, b);
			b->rowDirty = false;
			b->forceDirty = false;
			b->onDevice = s2IsFree(&b->object) == false;
			b->teleported = false;
			// the pending force now lives on the device, which zeroes it at the end of the step (reference src/world.c:275-276)
			b->force = s2Vec2_zero;
			b->torque = 0.0f;
		}
		s2b_upload_bodies(dev, rows, n, world->bodyPool.capacity);
		world->dirtyBodies.count = 0;
	}

	if (world->dirtyForces.count > 0)
	{
		int n = 0;
		s2bForceRow* rows = (s2bForceRow*)s2Staging(world, sizeof(s2bForceRow) * (size_t)world->dirtyForces.count);
		for (int i = 0; i < world->dirtyForces.count; ++i)
		{
			s2Body* b = world->bodies + world->dirtyForces.data[i];
			if (b->forceDirty == false)
			{
				continue; // already covered by a full row
			}
			rows[n].index = b->object.index;
			rows[n].force[0] = b->force.x;
			rows[n].force[1] = b->force.y;
			rows[n].torque = b->torque;
			b->forceDirty = false;
			b->force = s2Vec2_zero;
			b->torque = 0.0f;
			n += 1;
		}
		if (n > 0)
		{
			s2b_upload_forces(dev, rows, n);
		}
		world->dirtyForces.count = 0;
	}

	if (world->dirtyShapes.count > 0)
	{
		int n = world->dirtyShapes.count;
		s2bShapeRow* rows = (s2bShapeRow*)s2Staging(world, sizeof(s2bShapeRow) * (size_t)n);
		for (int i = 0; i < n; ++i)
		{
			s2Shape* s = world->shapes + world->dirtyShapes.data[i];
			s2FillShapeRow(rows + i, s);
			if (s2ObjectValid(&s->object) && s->fresh)
			{
				rows[i].flags |= S2B_SHAPE_FRESH;
				// new proxies of movable bodies are buffered as moved (reference src/broad_phase.c:104-107)
				if (world->bodies[s->bodyIndex].type != s2_staticBody)
				{
					rows[i].flags |= S2B_SHAPE_MOVED;
				}
				s->fresh = false;
			}
			s->rowDirty = false;
		}
		s2b_upload_shapes(dev, rows, n, world->shapePool.capacity);
		world->dirtyShapes.count = 0;
	}

	if (world->dirtyJoints.count > 0)
	{
		int n = world->dirtyJoints.count;
		s2bJointRow* rows = (s2bJointRow*)s2Staging(world, sizeof(s2bJointRow) * (size_t)n);
		for (int i = 0; i < n; ++i)
		{
			s2Joint* j = world->joints + world->dirtyJoints.data[i];
			s2FillJointRow(rows + i, j);
			j->rowDirty = false;
		}
		s2b_upload_joints(dev, rows, n, world->jointPool.capacity);
		world->dirtyJoints.count = 0;
	}

	if (world->restitutionDirty)
	{
		s2b_set_restitution(dev, world->enableRestitution ? 1 : 0, world->restitutionThreshold);
		world->restitutionDirty = false;
	}

	if (world->jointPairsDirty)
	{
		// Two key lists (body pair = lo << 32 | hi):
		//   block   — every live joint: s2ShouldBodiesCollide (reference src/body.c:386-417) vetoes a new contact between
		//             jointed bodies and does not look at collideConnected;
		//   destroy — revolute, weld and prismatic joints created with collideConnected == false: contacts that already
		//             exist between the two bodies are removed (reference src/joint.c:214-217).
		int cap = world->jointPool.capacity;
		uint64_t* block = (uint64_t*)malloc(sizeof(uint64_t) * (size_t)(cap > 0 ? cap : 1));
		uint64_t* destroy = (uint64_t*)malloc(sizeof(uint64_t) * (size_t)(cap > 0 ? cap : 1));
		int nBlock = 0, nDestroy = 0;
		for (int i = 0; i < cap; ++i)
		{
			s2Joint* j = world->joints + i;
			if (s2IsFree(&j->object))
			{
				continue;
			}
			uint64_t lo = (uint64_t)(j->bodyIndexA < j->bodyIndexB ? j->bodyIndexA : j->bodyIndexB);
			uint64_t hi = (uint64_t)(j->bodyIndexA < j->bodyIndexB ? j->bodyIndexB : j->bodyIndexA);
			block[nBlock++] = (lo << 32) | hi;
			if ((j->type == s2_revoluteJoint || j->type == s2_weldJoint || j->type == s2_prismaticJoint) && j->collideConnected == false)
			{
				destroy[nDestroy++] = (lo << 32) | hi;
			}
		}
		qsort(block, (size_t)nBlock, sizeof(uint64_t), s2CompareU64);
		qsort(destroy, (size_t)nDestroy, sizeof(uint64_t), s2CompareU64);
		s2b_upload_joint_pairs(dev, block, nBlock, destroy, nDestroy);
		free(block);
		free(destroy);
		world->jointPairsDirty = false;
	}
}

void s2SyncStateToHost(s2World* world)
{
	if (world->stateFresh)
	{
		return;
	}
	int cap = world->bodyPool.capacity;
	const float* state = s2b_sync_body_state(world->device, cap);
	for (int i = 0; i < cap; ++i)
	{
		s2Body* b = world->bodies + i;
		if (s2IsFree(&b->object) || b->rowDirty)
		{
			continue; // free slot, or the host copy is newer than the device's
		}
		const float* r = state + 12 * (size_t)i;
		b->origin = s2MakeVec2(r[0], r[1]);
		b->position = s2MakeVec2(r[2], r[3]);
		b->rot.s = r[4];
		b->rot.c = r[5];
		b->linearVelocity = s2MakeVec2(r[6], r[7]);
		b->angularVelocity = r[8];
		// force / torque are not mirrored: on the host they only hold what has not been uploaded yet
	}

	int jcap = world->jointPool.capacity;
	if (world->jointPool.count > 0)
	{
		s2bJointRow* rows = (s2bJointRow*)malloc(sizeof(s2bJointRow) * (size_t)jcap);
		s2b_download_joints(world->device, rows, jcap);
		for (int i = 0; i < jcap; ++i)
		{
			s2Joint* j = world->joints + i;
			if (s2IsFree(&j->object) || j->rowDirty)
			{
				continue;
			}
			j->impulse = s2MakeVec2(rows[i].impulse[0], rows[i].impulse[1]);
			j->motorImpulse = rows[i].motorImpulse;
			j->lowerImpulse = rows[i].lowerImpulse;
			j->upperImpulse = rows[i].upperImpulse;
		}
		free(rows);
	}
	world->stateFresh = true;
}

void s2SyncBoxesToHost(s2World* world)
{
	if (world->boxesFresh)
	{
		return;
	}
	int cap = world->shapePool.capacity;
	float* aabb = (float*)malloc(sizeof(float) * 4 * (size_t)cap);
	float* fat = (float*)malloc(sizeof(float) * 4 * (size_t)cap);
	s2b_download_shape_boxes(world->device, aabb, fat, NULL, cap);
	for (int i = 0; i < cap; ++i)
	{
		s2Shape* s = world->shapes + i;
		if (s2IsFree(&s->object) || s->rowDirty)
		{
			continue;
		}
		s->aabb.lowerBound = s2MakeVec2(aabb[4 * i], aabb[4 * i + 1]);
		s->aabb.upperBound = s2MakeVec2(aabb[4 * i + 2], aabb[4 * i + 3]);
		s->fatAABB.lowerBound = s2MakeVec2(fat[4 * i], fat[4 * i + 1]);
		s->fatAABB.upperBound = s2MakeVec2(fat[4 * i + 2], fat[4 * i + 3]);
	}
	free(aabb);
	free(fat);
	world->boxesFresh = true;
}

// ---- lifecycle --------------------------------------------------------------------------------------------------

// reference src/world.c:47-103
s2WorldId s2CreateWorld(const s2WorldDef* def)
{
	s2WorldId id = s2_nullWorldId;
	for (int16_t i = 0; i < s2_maxWorlds; ++i)
	{
		if (s2_worlds[i].inUse == false)
		{
			id.index = i;
			break;
		}
	}
	if (id.index == s2_nullWorldId.index)
	{
		return id;
	}

	s2World* world = s2_worlds + id.index;
	uint16_t revision = world->revision;
	memset(world, 0, sizeof(*world));
	world->index = id.index;
	world->inUse = true;
	world->solverType = def->solverType;
	world->bodyPool = s2CreatePool(sizeof(s2Body), 4);
	world->bodies = (s2Body*)world->bodyPool.memory;
	world->shapePool = s2CreatePool(sizeof(s2Shape), 4);
	world->shapes = (s2Shape*)world->shapePool.memory;
	world->jointPool = s2CreatePool(sizeof(s2Joint), 4);
	world->joints = (s2Joint*)world->jointPool.memory;
	world->gravity = s2MakeVec2(0.0f, -10.0f);
	world->restitutionThreshold = 1.0f; // reference src/world.c:98
	world->stepId = 0;
	world->revision = (uint16_t)(revision + 1);
	world->stateFresh = true;
	world->boxesFresh = true;

	// no CUDA device -> s2b_world_create reports and aborts: there is no CPU path
	// S2B_DEVICE selects the CUDA device of new worlds (one process per GPU sets it to its local rank)
	const char* deviceEnv = getenv("S2B_DEVICE");
	world->device = s2b_world_create(deviceEnv != NULL ? atoi(deviceEnv) : -1, (int)def->solverType);
	s2b_set_gravity(world->device, world->gravity.x, world->gravity.y);

	const char* schedule = getenv("S2B_SCHEDULE");
	if (schedule != NULL && strcmp(schedule, "wavefront") == 0)
	{
		s2b_set_schedule(world->device, S2B_SCHEDULE_WAVEFRONT);
	}

	id.revision = world->revision;
	return id;
}

void s2DestroyWorld(s2WorldId id)
{
	s2World* world = s2GetWorldFromId(id);
	s2b_world_destroy(world->device);
	if (world->staging)
	{
		s2b_host_free(world->staging);
	}
	s2DestroyPool(&world->jointPool);
	s2DestroyPool(&world->shapePool);
	s2DestroyPool(&world->bodyPool);
	s2IndexListFree(&world->dirtyBodies);
	s2IndexListFree(&world->dirtyForces);
	s2IndexListFree(&world->dirtyShapes);
	s2IndexListFree(&world->dirtyJoints);
	for (int i = 0; i < s2_bodyTypeCount; ++i)
	{
		free(world->proxyIds[i].freeStack);
	}
	uint16_t revision = world->revision;
	memset(world, 0, sizeof(*world));
	world->revision = revision;
}

// ---- the step ---------------------------------------------------------------------------------------------------

static bool s2IsSubstepping(s2SolverType type)
{
	return type == s2_solverXPBD || type == s2_solverTGS_Soft || type == s2_solverTGS_Sticky || type == s2_solverTGS_NGS ||
		   type == s2_solverSoftStep;
}

void s2World_Step(s2WorldId worldId, float timeStep, int32_t velIters, int32_t posIters, bool warmStart)
{
	s2World* world = s2GetWorldFromId(worldId);
	world->stepId += 1;

	s2FlushToDevice(world);

	// stages 1-3 (reference src/world.c:125-168)
	s2b_update_pairs(world->device);
	s2b_update_contacts(world->device);

	// step context (reference src/world.c:171-202)
	s2StepContext context = {0};
	context.dt = timeStep;
	context.iterations = velIters;
	context.extraIterations = posIters;
	context.warmStart = warmStart;
	context.inv_dt = timeStep > 0.0f ? 1.0f / timeStep : 0.0f;
	if (s2IsSubstepping(world->solverType))
	{
		context.h = context.dt / context.iterations;
		context.inv_h = context.inv_dt * context.iterations;
	}
	else
	{
		context.h = context.dt;
		context.inv_h = context.inv_dt;
	}
	context.bodies = world->bodies;
	context.bodyCapacity = world->bodyPool.capacity;

	// solver dispatch through the per-variant entry points (reference src/world.c:206-256)
	switch (world->solverType)
	{
		case s2_solverJacobi:
			s2Solve_Jacobi(world, &context);
			break;
		case s2_solverPGS:
			s2Solve_PGS(world, &context);
			break;
		case s2_solverPGS_NGS:
			s2Solve_PGS_NGS(world, &context);
			break;
		case s2_solverPGS_NGS_Block:
			s2Solve_PGS_NGS_Block(world, &context);
			break;
		case s2_solverPGS_Soft:
			s2Solve_PGS_Soft(world, &context);
			break;
		case s2_solverTGS_Sticky:
			s2Solve_TGS_Sticky(world, &context);
			break;
		case s2_solverTGS_Soft:
			s2Solve_TGS_Soft(world, &context);
			break;
		case s2_solverTGS_NGS:
			s2Solve_TGS_NGS(world, &context);
			break;
		case s2_solverXPBD:
			s2Solve_XPBD(world, &context);
			break;
		case s2_solverSoftStep:
			s2Solve_SoftStep(world, &context);
			break;
		default:
			break;
	}

	// stage 4 (reference src/world.c:258-301); also zeroes the applied forces on the device
	s2b_finalize(world->device);
	// the pair search of the NEXT step (reference src/broad_phase.c:309-367: s2UpdateBroadPhasePairs) only needs what finalize
	// has just produced: start it now, so that the next step finds its counters waiting instead of stopping mid-pass
	s2b_prefetch_pairs(world->device);

	// forces are consumed by the step (reference src/world.c:275-276)
	world->stateFresh = false;
	world->boxesFresh = false;
}

// ---- solver entry points ----------------------------------------------------------------------------------------

static void s2SolveOnDevice(s2World* world, s2StepContext* context, s2SolverType type)
{
	s2bStepContext ctx;
	ctx.dt = context->dt;
	ctx.inv_dt = context->inv_dt;
	ctx.h = context->h;
	ctx.inv_h = context->inv_h;
	ctx.iterations = context->iterations;
	ctx.extraIterations = context->extraIterations;
	ctx.warmStart = context->warmStart ? 1 : 0;
	s2b_solve(world->device, (int)type, &ctx);
}

void s2Solve_Jacobi(s2World* world, s2StepContext* context)
{
	s2SolveOnDevice(world, context, s2_solverJacobi);
}

void s2Solve_PGS(s2World* world, s2StepContext* context)
{
	s2SolveOnDevice(world, context, s2_solverPGS);
}

void s2Solve_PGS_NGS(s2World* world, s2StepContext* context)
{
	s2SolveOnDevice(world, context, s2_solverPGS_NGS);
}

void s2Solve_PGS_NGS_Block(s2World* world, s2StepContext* context)
{
	s2SolveOnDevice(world, context, s2_solverPGS_NGS_Block);
}

void s2Solve_PGS_Soft(s2World* world, s2StepContext* context)
{
	s2SolveOnDevice(world, context, s2_solverPGS_Soft);
}

void s2Solve_TGS_Soft(s2World* world, s2StepContext* context)
{
	s2SolveOnDevice(world, context, s2_solverTGS_Soft);
}

void s2Solve_TGS_Sticky(s2World* world, s2StepContext* context)
{
	s2SolveOnDevice(world, context, s2_solverTGS_Sticky);
}

void s2Solve_TGS_NGS(s2World* world, s2StepContext* context)
{
	s2SolveOnDevice(world, context, s2_solverTGS_NGS);
}

void s2Solve_XPBD(s2World* world, s2StepContext* context)
{
	s2SolveOnDevice(world, context, s2_solverXPBD);
}

void s2Solve_SoftStep(s2World* world, s2StepContext* context)
{
	s2SolveOnDevice(world, context, s2_solverSoftStep);
}

// ---- queries ----------------------------------------------------------------------------------------------------

// reference src/world.c:565-579
struct s2Statistics s2World_GetStatistics(s2WorldId worldId)
{
	s2World* world = s2GetWorldFromId(worldId);
	s2Statistics stats = {0};
	s2bCounters counters;
	s2b_get_counters(world->device, &counters);
	stats.bodyCount = world->bodyPool.count;
	stats.contactCount = counters.contactCount;
	stats.jointCount = world->jointPool.count;
	stats.proxyCount = world->shapePool.count;
	stats.treeHeight = counters.treeHeight;
	stats.stackCapacity = (int32_t)(counters.scratchBytes > 0x7FFFFFFF ? 0x7FFFFFFF : counters.scratchBytes);
	stats.stackUsed = stats.stackCapacity;
	return stats;
}

// reference src/world.c:581-615: every proxy whose fat AABB overlaps the query box (the reference walks its trees; the
// host mirror is scanned linearly here — this is an editor / picking query, not on the step path)
void s2World_QueryAABB(s2WorldId worldId, s2Box aabb, s2QueryCallbackFcn* fcn, void* context)
{
	s2World* world = s2GetWorldFromId(worldId);
	s2SyncBoxesToHost(world);
	int cap = world->shapePool.capacity;
	for (int i = 0; i < cap; ++i)
	{
		s2Shape* shape = world->shapes + i;
		if (s2IsFree(&shape->object))
		{
			continue;
		}
		if (s2AABB_Overlaps(shape->fatAABB, aabb))
		{
			s2ShapeId id = {shape->object.index, world->index, shape->object.revision};
			if (fcn(id, context) == false)
			{
				return;
			}
		}
	}
}

// ---- extensions (include/solver2d_b200.h) -----------------------------------------------------------------------

#include "solver2d_b200.h"

s2bWorld* s2World_GetDevice(s2WorldId worldId)
{
	return s2GetWorldFromId(worldId)->device;
}

void s2World_EnableRestitution(s2WorldId worldId, bool enable)
{
	s2World* world = s2GetWorldFromId(worldId);
	world->enableRestitution = enable;
	world->restitutionDirty = true;
}

void s2World_SetRestitutionThreshold(s2WorldId worldId, float threshold)
{
	s2World* world = s2GetWorldFromId(worldId);
	S2_ASSERT(s2IsValid(threshold) && threshold >= 0.0f);
	if (s2IsValid(threshold) == false || threshold < 0.0f)
	{
		return; // rejected: the world keeps its threshold
	}
	world->restitutionThreshold = threshold;
	world->restitutionDirty = true;
}

void s2World_Flush(s2WorldId worldId)
{
	s2FlushToDevice(s2GetWorldFromId(worldId));
}

void s2World_ApplyForcesToCenters(s2WorldId worldId, const int32_t* bodyIndices, const float* forcesXY, int32_t count)
{
	// bulk s2Body_ApplyForceToCenter: the forces go straight to the device accumulators. Rows that are still dirty on the
	// host are uploaded first so that a body created since the last step exists before it receives its force.
	s2World* world = s2GetWorldFromId(worldId);
	if (world->dirtyBodies.count > 0)
	{
		s2FlushToDevice(world);
	}
	s2b_add_forces(world->device, bodyIndices, forcesXY, count);
}

float s2World_TimedSteps(s2WorldId worldId, int32_t steps, float timeStep, int32_t velIters, int32_t posIters, bool warmStart,
						 int32_t flushL2)
{
	s2World* world = s2GetWorldFromId(worldId);
	float total = 0.0f;
	for (int32_t i = 0; i < steps; ++i)
	{
		if (flushL2)
		{
			s2b_flush_l2(world->device);
		}
		s2b_mark_time(world->device, 0);
		s2World_Step(worldId, timeStep, velIters, posIters, warmStart);
		s2b_mark_time(world->device, 1);
		total += s2b_elapsed_ms(world->device);
	}
	return total;
}

int32_t s2World_GetBodyTransforms(s2WorldId worldId, float* out, int32_t capacity)
{
	// transforms straight from the device columns: one gather + one D2H of 16 B per used slot; the host body structs are not
	// refreshed (their lazy read-back stays pending for whoever asks for velocities etc.)
	s2World* world = s2GetWorldFromId(worldId);
	if (world->dirtyBodies.count > 0)
	{
		s2FlushToDevice(world); // a transform set through the API since the last step wins
	}
	int32_t n = world->bodyHighWater < capacity ? world->bodyHighWater : capacity;
	s2b_download_transforms(world->device, out, n);
	return world->bodyPool.capacity;
}

float s2Atan2Device(float y, float x)
{
	return s2Atan2F32(y, x);
}
