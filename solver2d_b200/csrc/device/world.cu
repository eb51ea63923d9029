// solver2d-b200 — device world lifecycle, row scatter (host -> SoA) and row gather (SoA -> host).
//
// Replaces the reference's AoS pools (s2Body 184 B, s2Shape 240 B, s2Joint 188 B, s2Contact 216 B; reference
// src/body.h, shape.h, joint.h, contact.h) with 128-bit aligned SoA columns resident in HBM. The host only ever
// moves *rows that changed*; a scatter kernel writes them into the columns, so a stale host copy of an untouched
// neighbour can never overwrite device state.
#include "s2b_internal.cuh"

// ---------------------------------------------------------------------------------------------------------------
// scatter kernels
// ---------------------------------------------------------------------------------------------------------------

__global__ void s2bScatterBodies(const s2bBodyRow* __restrict__ rows, int count, BodyView b, int* schedDirty)
{
	int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= count)
	{
		return;
	}
	s2bBodyRow r = rows[t];
	int i = r.index;
	{
		// the solve schedule (conflict graph, regions) depends on which bodies exist and which of them can move
		bool wasValid = (b.flags[i] & S2B_BODY_VALID) != 0, isValid = (r.flags & S2B_BODY_VALID) != 0;
		bool wasMovable = b.vel[i].w != 0.0f || b.prm[i].w != 0.0f, isMovable = r.invMass != 0.0f || r.invI != 0.0f;
		if (wasValid != isValid || (isValid && wasMovable != isMovable))
		{
			*schedDirty = 1;
		}
	}
	b.vel[i] = make_float4(r.linearVelocity[0], r.linearVelocity[1], r.angularVelocity, r.invMass);
	// a body the device already holds keeps its delta position (reference src/body.c:337-350 set only the velocity; XPBD
	// carries a kinematic body's from step to step); a new body, a reused slot or a teleported body starts at zero
	bool keepDelta = (r.flags & (S2B_BODY_ADD_FORCE | S2B_BODY_TELEPORT)) == S2B_BODY_ADD_FORCE;
	float4 pose = b.pose[i];
	b.pose[i] = make_float4(keepDelta ? pose.x : 0.0f, keepDelta ? pose.y : 0.0f, r.rot[0], r.rot[1]);
	b.pos[i] = make_float4(r.position[0], r.position[1], r.invI, r.I);
	b.org[i] = make_float4(r.origin[0], r.origin[1], r.localCenter[0], r.localCenter[1]);
	if (r.flags & S2B_BODY_ADD_FORCE)
	{
		float4 f = b.frc[i];
		b.frc[i] = make_float4(f.x + r.force[0], f.y + r.force[1], f.z + r.torque, r.mass);
	}
	else
	{
		b.frc[i] = make_float4(r.force[0], r.force[1], r.torque, r.mass);
	}
	b.prm[i] = make_float4(r.linearDamping, r.angularDamping, r.gravityScale, r.invI);
	b.flags[i] = (uint8_t)(r.flags & 0x7);
}

__global__ void s2bScatterShapes(const s2bShapeRow* __restrict__ rows, int count, ShapeView s)
{
	int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= count)
	{
		return;
	}
	const s2bShapeRow* r = rows + t;
	int i = r->index;
	s.head[i] = make_int4(r->flags, r->body, r->proxyKey, r->count);
	s.filter[i] = make_int4((int)r->categoryBits, (int)r->maskBits, r->groupIndex, 0);
	s.aabb[i] = make_float4(r->aabb[0], r->aabb[1], r->aabb[2], r->aabb[3]);
	s.fat[i] = make_float4(r->fatAABB[0], r->fatAABB[1], r->fatAABB[2], r->fatAABB[3]);
	s.fr[i] = make_float2(r->friction, r->radius);
	s.restitution[i] = r->restitution;
	for (int k = 0; k < 8; ++k)
	{
		s.verts[i * 8 + k] = make_float2(r->vertices[2 * k], r->vertices[2 * k + 1]);
		s.normals[i * 8 + k] = make_float2(r->normals[2 * k], r->normals[2 * k + 1]);
	}
}

__global__ void s2bScatterJoints(const s2bJointRow* __restrict__ rows, int count, JointView j, int* schedDirty)
{
	int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= count)
	{
		return;
	}
	const s2bJointRow* r = rows + t;
	int i = r->index;
	{
		// a joint that appears, disappears or changes its bodies / kind changes the solve schedule; a new target, motor
		// speed or limit does not
		int4 old = j.head[i];
		if (((old.x ^ r->flags) & (S2B_ROW_VALID | 0xE)) != 0 || ((r->flags & S2B_ROW_VALID) != 0 && (old.y != r->bodyA || old.z != r->bodyB)))
		{
			*schedDirty = 1;
			j.color[i] = -1; // (an unchanged joint keeps the colour it was last solved with)
		}
	}
	j.head[i] = make_int4(r->flags, r->bodyA, r->bodyB, 0);
	j.anchors[i] = make_float4(r->localOriginAnchorA[0], r->localOriginAnchorA[1], r->localOriginAnchorB[0],
							   r->localOriginAnchorB[1]);
	j.lim[i] = make_float4(r->referenceAngle, r->lowerAngle, r->upperAngle, 0.0f);
	j.motor[i] = make_float4(r->maxMotorTorque, r->motorSpeed, r->hertz, r->dampingRatio);
	j.target[i] = make_float4(r->target[0], r->target[1], r->localAxisA[0], r->localAxisA[1]);
	j.imp[i] = make_float4(r->impulse[0], r->impulse[1], r->motorImpulse, 0.0f);
	j.limp[i] = make_float4(r->lowerImpulse, r->upperImpulse, 0.0f, 0.0f);
}

__device__ __forceinline__ int s2bPackCache(const s2bContactRow* r)
{
	// count (2 bits) | indexA[0..2] (3 bits each) | indexB[0..2] (3 bits each)
	int bits = r->cacheCount & 0x3;
	for (int k = 0; k < 3; ++k)
	{
		bits |= (r->cacheIndexA[k] & 0x7) << (2 + 3 * k);
		bits |= (r->cacheIndexB[k] & 0x7) << (11 + 3 * k);
	}
	return bits;
}

__global__ void s2bScatterContacts(const s2bContactRow* __restrict__ rows, int count, ContactView c, int sticky)
{
	int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= count)
	{
		return;
	}
	const s2bContactRow* r = rows + t;
	unsigned long long lo = (unsigned long long)(r->shapeA < r->shapeB ? r->shapeA : r->shapeB);
	unsigned long long hi = (unsigned long long)(r->shapeA < r->shapeB ? r->shapeB : r->shapeA);
	c.key[t] = (lo << 32) | hi;
	c.shapes[t] = make_int2(r->shapeA, r->shapeB);
	c.bodies[t] = make_int2(r->bodyA, r->bodyB);
	int flags = (r->pointCount & 0x3) | (r->frictionPersisted ? S2B_CI_FRICTION_PERSISTED : 0) |
				(r->points[0].persisted ? S2B_CI_PERSISTED0 : 0) | (r->points[1].persisted ? S2B_CI_PERSISTED1 : 0);
	int ids = (r->points[0].id & 0xFFFF) | ((r->points[1].id & 0xFFFF) << 16);
	c.info[t] = make_int4(flags, ids, s2bPackCache(r), __float_as_int(r->cacheMetric));
	c.nf[t] = make_float4(r->normal[0], r->normal[1], r->friction, r->restitution);
	c.color[t] = -1;
	for (int p = 0; p < 2; ++p)
	{
		const s2bContactPoint* q = r->points + p;
		c.anchor[p][t] = make_float4(q->localAnchorA[0], q->localAnchorA[1], q->localAnchorB[0], q->localAnchorB[1]);
		c.impulse[p][t] = make_float4(q->separation, q->normalImpulse, q->tangentImpulse, 0.0f);
		if (sticky)
		{
			c.fanchor[p][t] =
				make_float4(q->frictionAnchorA[0], q->frictionAnchorA[1], q->frictionAnchorB[0], q->frictionAnchorB[1]);
			c.fnormal[p][t] =
				make_float4(q->frictionNormalA[0], q->frictionNormalA[1], q->frictionNormalB[0], q->frictionNormalB[1]);
		}
	}
}

// ---------------------------------------------------------------------------------------------------------------
// gather kernels
// ---------------------------------------------------------------------------------------------------------------

__global__ void s2bGatherBodies(s2bBodyRow* rows, int count, BodyView b, int useRowIndex)
{
	int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= count)
	{
		return;
	}
	int i = useRowIndex ? rows[t].index : t;
	s2bBodyRow r;
	float4 vel = b.vel[i], pose = b.pose[i], pos = b.pos[i], org = b.org[i], frc = b.frc[i], prm = b.prm[i];
	r.index = i;
	r.flags = b.flags[i];
	r.origin[0] = org.x;
	r.origin[1] = org.y;
	r.position[0] = pos.x;
	r.position[1] = pos.y;
	r.rot[0] = pose.z;
	r.rot[1] = pose.w;
	r.linearVelocity[0] = vel.x;
	r.linearVelocity[1] = vel.y;
	r.angularVelocity = vel.z;
	r.localCenter[0] = org.z;
	r.localCenter[1] = org.w;
	r.mass = frc.w;
	r.invMass = vel.w;
	r.I = pos.w;
	r.invI = pos.z;
	r.force[0] = frc.x;
	r.force[1] = frc.y;
	r.torque = frc.z;
	r.linearDamping = prm.x;
	r.angularDamping = prm.y;
	r.gravityScale = prm.z;
	rows[t] = r;
}

__global__ void s2bGatherJoints(s2bJointRow* rows, int count, JointView j)
{
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= count)
	{
		return;
	}
	s2bJointRow r;
	int4 head = j.head[i];
	float4 a = j.anchors[i], lim = j.lim[i], motor = j.motor[i], target = j.target[i], imp = j.imp[i], limp = j.limp[i];
	r.index = i;
	r.flags = head.x;
	r.bodyA = head.y;
	r.bodyB = head.z;
	r.localOriginAnchorA[0] = a.x;
	r.localOriginAnchorA[1] = a.y;
	r.localOriginAnchorB[0] = a.z;
	r.localOriginAnchorB[1] = a.w;
	r.referenceAngle = lim.x;
	r.lowerAngle = lim.y;
	r.upperAngle = lim.z;
	r.maxMotorTorque = motor.x;
	r.motorSpeed = motor.y;
	r.hertz = motor.z;
	r.dampingRatio = motor.w;
	r.target[0] = target.x;
	r.target[1] = target.y;
	r.localAxisA[0] = target.z;
	r.localAxisA[1] = target.w;
	r.impulse[0] = imp.x;
	r.impulse[1] = imp.y;
	r.motorImpulse = imp.z;
	r.lowerImpulse = limp.x;
	r.upperImpulse = limp.y;
	rows[i] = r;
}

__global__ void s2bGatherContacts(s2bContactRow* rows, int count, ContactView c, int sticky)
{
	int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= count)
	{
		return;
	}
	s2bContactRow r;
	memset(&r, 0, sizeof(r));
	int2 sh = c.shapes[t], bo = c.bodies[t];
	int4 info = c.info[t];
	float4 nf = c.nf[t];
	r.shapeA = sh.x;
	r.shapeB = sh.y;
	r.bodyA = bo.x;
	r.bodyB = bo.y;
	r.pointCount = S2B_CI_COUNT(info.x);
	r.frictionPersisted = (info.x & S2B_CI_FRICTION_PERSISTED) ? 1 : 0;
	r.friction = nf.z;
	r.restitution = nf.w;
	r.normal[0] = nf.x;
	r.normal[1] = nf.y;
	for (int p = 0; p < 2; ++p)
	{
		s2bContactPoint* q = r.points + p;
		float4 a = c.anchor[p][t], m = c.impulse[p][t];
		q->localAnchorA[0] = a.x;
		q->localAnchorA[1] = a.y;
		q->localAnchorB[0] = a.z;
		q->localAnchorB[1] = a.w;
		q->separation = m.x;
		q->normalImpulse = m.y;
		q->tangentImpulse = m.z;
		q->id = (info.y >> (16 * p)) & 0xFFFF;
		q->persisted = (info.x & (p == 0 ? S2B_CI_PERSISTED0 : S2B_CI_PERSISTED1)) ? 1 : 0;
		if (sticky)
		{
			float4 fa = c.fanchor[p][t], fn = c.fnormal[p][t];
			q->frictionAnchorA[0] = fa.x;
			q->frictionAnchorA[1] = fa.y;
			q->frictionAnchorB[0] = fa.z;
			q->frictionAnchorB[1] = fa.w;
			q->frictionNormalA[0] = fn.x;
			q->frictionNormalA[1] = fn.y;
			q->frictionNormalB[0] = fn.z;
			q->frictionNormalB[1] = fn.w;
		}
	}
	r.cacheCount = info.z & 0x3;
	for (int k = 0; k < 3; ++k)
	{
		r.cacheIndexA[k] = (uint8_t)((info.z >> (2 + 3 * k)) & 0x7);
		r.cacheIndexB[k] = (uint8_t)((info.z >> (11 + 3 * k)) & 0x7);
	}
	r.cacheMetric = __int_as_float(info.w);
	rows[t] = r;
}

__global__ void s2bPackBodyState(BodyView b, int first, int count, float4* out)
{
	int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= count)
	{
		return;
	}
	int i = first + t;
	float4 org = b.org[i], pose = b.pose[i], vel = b.vel[i];
	out[2 * t + 0] = make_float4(org.x, org.y, pose.z, pose.w);
	out[2 * t + 1] = make_float4(vel.x, vel.y, vel.z, 0.0f);
}

__global__ void s2bFlushKernel(char* buf, size_t n, int value)
{
	size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	size_t stride = (size_t)gridDim.x * blockDim.x;
	int4* p = (int4*)buf;
	size_t n4 = n / sizeof(int4);
	for (; i < n4; i += stride)
	{
		p[i] = make_int4(value, value, value, value);
	}
}

// ---------------------------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------------------------

static void* stageRows(s2bWorld* w, const void* hostRows, size_t bytes)
{
	// stream-ordered staging buffer: allocate, copy, free after the scatter kernel
	void* d = nullptr;
	S2B_CHECK(cudaMallocAsync(&d, bytes, w->stream));
	S2B_CHECK(cudaMemcpyAsync(d, hostRows, bytes, cudaMemcpyHostToDevice, w->stream));
	return d;
}

extern "C" s2bWorld* s2b_world_create(int cudaDevice, int solverType)
{
	int deviceCount = 0;
	cudaError_t err = cudaGetDeviceCount(&deviceCount);
	if (err != cudaSuccess || deviceCount == 0)
	{
		fprintf(stderr, "solver2d-b200: no CUDA device available (%s) — this library has no CPU fallback\n",
				cudaGetErrorString(err));
		abort();
	}
	s2bWorld* w = new s2bWorld();
	if (cudaDevice < 0)
	{
		S2B_CHECK(cudaGetDevice(&cudaDevice));
	}
	w->device = cudaDevice;
	S2B_CHECK(cudaSetDevice(cudaDevice));
	S2B_CHECK(cudaStreamCreateWithFlags(&w->stream, cudaStreamNonBlocking));
	cudaDeviceProp prop;
	S2B_CHECK(cudaGetDeviceProperties(&prop, cudaDevice));
	w->smCount = prop.multiProcessorCount;
	w->coopSupported = prop.cooperativeLaunch;
	{
		const char* env = getenv("S2B_WARM_GATHER");
		if (env != nullptr)
		{
			w->gatherWarm = atoi(env) != 0 ? 1 : 0;
		}
		env = getenv("S2B_GRAPH");
		if (env != nullptr)
		{
			w->useGraph = atoi(env) != 0 ? 1 : 0;
		}
		env = getenv("S2B_PREFETCH_PAIRS");
		if (env != nullptr)
		{
			w->prefetchPairs = atoi(env);
		}
		env = getenv("S2B_FUSE_POSITIONS");
		if (env != nullptr)
		{
			w->fusePositions = atoi(env);
		}
		env = getenv("S2B_HUB_DEGREE");
		if (env != nullptr)
		{
			w->hubDegree = atoi(env);
		}
		env = getenv("S2B_RESIDENT");
		if (env != nullptr)
		{
			w->residentRegions = atoi(env);
		}
		env = getenv("S2B_SIDE_COPIES");
		if (env != nullptr)
		{
			w->sideCopies = atoi(env);
		}
		env = getenv("S2B_WHOLE_ISLAND");
		if (env != nullptr)
		{
			w->wholeIslandBodies = atoi(env);
		}
		env = getenv("S2B_KEMPE");
		if (env != nullptr)
		{
			w->kempe = atoi(env);
		}
		env = getenv("S2B_PERSISTENT");
		if (env != nullptr)
		{
			w->persistent = atoi(env) != 0 ? 1 : 0;
		}
		env = getenv("S2B_REGIONS");
		if (env != nullptr)
		{
			w->useRegions = atoi(env) < 0 ? 0 : (atoi(env) > 2 ? 2 : atoi(env));
		}
		env = getenv("S2B_REGION_CUT_LIMIT");
		if (env != nullptr)
		{
			w->regionCutLimit = atoi(env) < 0 ? 0 : (atoi(env) > 64 ? 64 : atoi(env));
		}
		env = getenv("S2B_DATAFLOW");
		if (env != nullptr)
		{
			w->dataflow = atoi(env) != 0 ? 1 : 0;
		}
		env = getenv("S2B_NEIGHBOUR_SYNC");
		if (env != nullptr)
		{
			w->neighbourSync = atoi(env) != 0 ? 1 : 0;
		}
		env = getenv("S2B_NARROWPHASE_PREPARE");
		if (env != nullptr)
		{
			w->narrowphasePrepare = atoi(env) != 0 ? 1 : 0;
		}
		env = getenv("S2B_BLOCK_WARM");
		if (env != nullptr)
		{
			w->blockWarm = atoi(env) != 0 ? 1 : 0;
		}
		env = getenv("S2B_BLOCK_WARM_BYTES");
		if (env != nullptr)
		{
			w->blockWarmBytes = atoi(env) < 0 ? 0 : atoi(env);
		}
	}
	w->solverType = solverType;
	w->sticky = (solverType == 6); // s2_solverTGS_Sticky
	w->schedDirty.reserve(8, w->stream, true, true); // S2B_SCHED_WORDS
	w->solveBarrier.reserve(64, w->stream, true, true);
	S2B_CHECK(cudaMallocHost((void**)&w->hostMail, MAIL_COUNT * sizeof(int)));
	memset(w->hostMail, 0, MAIL_COUNT * sizeof(int));
	S2B_CHECK(cudaMalloc((void**)&w->devMail, MAIL_COUNT * sizeof(int)));
	S2B_CHECK(cudaMemset(w->devMail, 0, MAIL_COUNT * sizeof(int)));
	for (int i = 0; i < 5; ++i)
	{
		S2B_CHECK(cudaEventCreate(&w->timer.ev[i]));
	}
	// keep freed stream-ordered allocations cached in the pool (per-step scratch is recycled, not re-malloc'ed)
	cudaMemPool_t pool;
	S2B_CHECK(cudaDeviceGetDefaultMemPool(&pool, cudaDevice));
	unsigned long long threshold = ~0ull;
	S2B_CHECK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &threshold));
	return w;
}

extern "C" void s2b_world_destroy(s2bWorld* w)
{
	if (w == nullptr)
	{
		return;
	}
	S2B_CHECK(cudaSetDevice(w->device));
	S2B_CHECK(cudaStreamSynchronize(w->stream));
	s2bFreeSolverScratch(w);
	s2bFreeBroadScratch(w);
	w->bVel.release();
	w->bPose.release();
	w->bPos.release();
	w->bOrg.release();
	w->bFrc.release();
	w->bPrm.release();
	w->bAux0.release();
	w->bAux1.release();
	w->bFlags.release();
	w->sHead.release();
	w->sFilter.release();
	w->sAabb.release();
	w->sFat.release();
	w->sFr.release();
	w->sRestitution.release();
	w->sVerts.release();
	w->sNormals.release();
	w->jHead.release();
	w->jAnchors.release();
	w->jLim.release();
	w->jMotor.release();
	w->jTarget.release();
	w->jImp.release();
	w->jLimp.release();
	w->jColor.release();
	w->jointPairKeys.release();
	w->jointDestroyKeys.release();
	w->dState.release();
	if (w->hostState != nullptr)
	{
		cudaFreeHost(w->hostState);
	}
	w->contacts[0].release();
	w->contacts[1].release();
	w->dMovedFlag.release();
	w->solveBarrier.release();
	w->schedDirty.release();
	w->l2Flush.release();
	w->dWork.release();
	if (w->solveKernelStart != nullptr)
	{
		cudaEventDestroy(w->solveKernelStart);
		cudaEventDestroy(w->solveKernelEnd);
	}
	if (w->copyStream != nullptr)
	{
		cudaStreamSynchronize(w->copyStream); // (its copies write into the pinned mailbox freed below)
		cudaStreamDestroy(w->copyStream);
		w->copyStream = nullptr;
	}
	if (w->movedEvent != nullptr)
	{
		cudaEventDestroy(w->movedEvent);
		cudaEventDestroy(w->finalizedEvent);
	}
	for (int i = 0; i < 2; ++i)
	{
		if (w->markEvents[i] != nullptr)
		{
			cudaEventDestroy(w->markEvents[i]);
		}
		if (w->bulkEvent[i] != nullptr)
		{
			cudaEventDestroy(w->bulkEvent[i]);
		}
		if (w->bulkHost[i] != nullptr)
		{
			cudaFreeHost(w->bulkHost[i]);
		}
	}
	if (w->hostXf != nullptr)
	{
		cudaFreeHost(w->hostXf);
	}
	w->dBulk.release();
	w->dXf.release();
	cudaFreeHost(w->hostMail);
	cudaFree(w->devMail);
	for (int i = 0; i < 5; ++i)
	{
		cudaEventDestroy(w->timer.ev[i]);
	}
	cudaStreamDestroy(w->stream);
	delete w;
}

extern "C" void s2b_set_gravity(s2bWorld* w, float gx, float gy)
{
	w->gravity = make_float2(gx, gy);
}

extern "C" void s2b_set_schedule(s2bWorld* w, int schedule)
{
	w->schedule = schedule;
	w->scheduleEpoch += 1;
}

extern "C" void s2b_set_max_colors(s2bWorld* w, int maxColors)
{
	w->maxColors = maxColors < 1 ? 1 : (maxColors > 64 ? 64 : maxColors);
	w->scheduleEpoch += 1;
}

extern "C" void s2b_set_persistent(s2bWorld* w, int enable)
{
	w->persistent = enable;
	w->scheduleEpoch += 1;
}

extern "C" void s2b_set_warm_gather(s2bWorld* w, int enable)
{
	w->gatherWarm = enable;
	w->scheduleEpoch += 1;
}

extern "C" void s2b_set_graph(s2bWorld* w, int enable)
{
	w->useGraph = enable;
	w->scheduleEpoch += 1;
}

extern "C" void s2b_set_dataflow(s2bWorld* w, int enable)
{
	w->dataflow = enable;
	w->scheduleEpoch += 1;
}

extern "C" void s2b_set_regions(s2bWorld* w, int enable)
{
	w->useRegions = enable;
	w->scheduleEpoch += 1;
}

extern "C" void s2b_set_restitution(s2bWorld* w, int enable, float threshold)
{
	// a threshold that is not a finite, non-negative speed is ignored (the previous one stays)
	if (isfinite(threshold) && threshold >= 0.0f)
	{
		w->restitutionThreshold = threshold;
	}
	w->restitution = enable != 0 ? 1 : 0;
}

static void reserveBodies(s2bWorld* w, int cap)
{
	if (cap <= w->bodyCap)
	{
		return;
	}
	cudaStream_t s = w->stream;
	w->bVel.reserve(cap, s);
	w->bPose.reserve(cap, s);
	w->bPos.reserve(cap, s);
	w->bOrg.reserve(cap, s);
	w->bFrc.reserve(cap, s);
	w->bPrm.reserve(cap, s);
	w->bAux0.reserve(cap, s);
	w->bAux1.reserve(cap, s);
	w->bFlags.reserve(cap, s);
	w->bodyCap = (int)w->bVel.cap;
}

static void reserveShapes(s2bWorld* w, int cap)
{
	if (cap <= w->shapeCap)
	{
		return;
	}
	cudaStream_t s = w->stream;
	w->sHead.reserve(cap, s);
	w->sFilter.reserve(cap, s);
	w->sAabb.reserve(cap, s);
	w->sFat.reserve(cap, s);
	w->sFr.reserve(cap, s);
	w->sRestitution.reserve(cap, s);
	w->shapeCap = (int)w->sHead.cap;
	w->sVerts.reserve((size_t)w->shapeCap * 8, s);
	w->sNormals.reserve((size_t)w->shapeCap * 8, s);
}

static void reserveJoints(s2bWorld* w, int cap)
{
	if (cap <= w->jointCap)
	{
		return;
	}
	cudaStream_t s = w->stream;
	w->jHead.reserve(cap, s);
	w->jAnchors.reserve(cap, s);
	w->jLim.reserve(cap, s);
	w->jMotor.reserve(cap, s);
	w->jTarget.reserve(cap, s);
	w->jImp.reserve(cap, s);
	w->jLimp.reserve(cap, s);
	w->jColor.reserve(cap, s);
	w->jointCap = (int)w->jHead.cap;
}

extern "C" void s2b_upload_bodies(s2bWorld* w, const s2bBodyRow* rows, int count, int bodyCapacity)
{
	S2B_CHECK(cudaSetDevice(w->device));
	w->xfSeq += 1; // (rows or the columns themselves may change: the next transform read-back orders itself behind this stream)
	reserveBodies(w, bodyCapacity);
	if (count <= 0)
	{
		return;
	}
	w->uploadEpoch += 1; // rows changed: a pair search started behind the previous step is stale now
	s2bBodyRow* d = (s2bBodyRow*)stageRows(w, rows, sizeof(s2bBodyRow) * (size_t)count);
	S2B_LAUNCH(w, s2bScatterBodies, gridFor(count, 128), 128, 0, d, count, bodyView(w), w->schedDirty.p);
	S2B_CHECK(cudaFreeAsync(d, w->stream));
	// the staging copy reads pageable host memory: make sure it is consumed before the caller reuses the buffer
	S2B_CHECK(cudaStreamSynchronize(w->stream));
}

extern "C" void s2b_upload_shapes(s2bWorld* w, const s2bShapeRow* rows, int count, int shapeCapacity)
{
	S2B_CHECK(cudaSetDevice(w->device));
	reserveShapes(w, shapeCapacity);
	if (count <= 0)
	{
		return;
	}
	w->uploadEpoch += 1; // rows changed: a pair search started behind the previous step is stale now
	s2bShapeRow* d = (s2bShapeRow*)stageRows(w, rows, sizeof(s2bShapeRow) * (size_t)count);
	S2B_LAUNCH(w, s2bScatterShapes, gridFor(count, 128), 128, 0, d, count, shapeView(w));
	S2B_CHECK(cudaFreeAsync(d, w->stream));
	S2B_CHECK(cudaStreamSynchronize(w->stream));
	w->pairsDirty = true;
}

extern "C" void s2b_upload_joints(s2bWorld* w, const s2bJointRow* rows, int count, int jointCapacity)
{
	S2B_CHECK(cudaSetDevice(w->device));
	reserveJoints(w, jointCapacity);
	if (count <= 0)
	{
		return;
	}
	w->uploadEpoch += 1; // rows changed: a pair search started behind the previous step is stale now
	s2bJointRow* d = (s2bJointRow*)stageRows(w, rows, sizeof(s2bJointRow) * (size_t)count);
	S2B_LAUNCH(w, s2bScatterJoints, gridFor(count, 128), 128, 0, d, count, jointView(w), w->schedDirty.p);
	S2B_CHECK(cudaFreeAsync(d, w->stream));
	S2B_CHECK(cudaStreamSynchronize(w->stream));
}

extern "C" void s2b_upload_contacts(s2bWorld* w, const s2bContactRow* rows, int count)
{
	w->uploadEpoch += 1; // a pair search started behind the previous step is stale now
	S2B_CHECK(cudaSetDevice(w->device));
	ContactColumns& c = w->contacts[w->cur];
	c.reserve((size_t)(count > 0 ? count : 1), w->stream, w->sticky, false);
	w->contactCount = count;
	w->contactTableVersion += 1;
	if (count <= 0)
	{
		return;
	}
	s2bContactRow* d = (s2bContactRow*)stageRows(w, rows, sizeof(s2bContactRow) * (size_t)count);
	S2B_LAUNCH(w, s2bScatterContacts, gridFor(count, 128), 128, 0, d, count, makeView(c), w->sticky ? 1 : 0);
	S2B_CHECK(cudaFreeAsync(d, w->stream));
	S2B_CHECK(cudaStreamSynchronize(w->stream));
}

extern "C" void s2b_upload_joint_pairs(s2bWorld* w, const uint64_t* blockKeys, int blockCount, const uint64_t* destroyKeys,
									   int destroyCount)
{
	w->uploadEpoch += 1; // a pair search started behind the previous step is stale now
	S2B_CHECK(cudaSetDevice(w->device));
	w->jointPairKeys.reserve((size_t)(blockCount > 0 ? blockCount : 1), w->stream, false);
	w->jointDestroyKeys.reserve((size_t)(destroyCount > 0 ? destroyCount : 1), w->stream, false);
	w->jointPairCount = blockCount;
	w->jointDestroyCount = destroyCount;
	if (blockCount > 0)
	{
		S2B_CHECK(cudaMemcpyAsync(w->jointPairKeys.p, blockKeys, sizeof(uint64_t) * (size_t)blockCount, cudaMemcpyHostToDevice,
								  w->stream));
	}
	if (destroyCount > 0)
	{
		S2B_CHECK(cudaMemcpyAsync(w->jointDestroyKeys.p, destroyKeys, sizeof(uint64_t) * (size_t)destroyCount,
								  cudaMemcpyHostToDevice, w->stream));
	}
	S2B_CHECK(cudaStreamSynchronize(w->stream));
	w->pairsDirty = true;
}

__global__ void s2bScatterForces(const s2bForceRow* __restrict__ rows, int count, BodyView b)
{
	int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= count)
	{
		return;
	}
	s2bForceRow r = rows[t];
	float4 f = b.frc[r.index];
	b.frc[r.index] = make_float4(f.x + r.force[0], f.y + r.force[1], f.z + r.torque, f.w);
}

__global__ void s2bAddForcesKernel(const int* __restrict__ indices, const float2* __restrict__ forces, int count, BodyView b)
{
	int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= count)
	{
		return;
	}
	int i = indices[t];
	// a body index may appear several times in one call (each entry adds, like repeated s2Body_ApplyForceToCenter calls):
	// atomic adds; out-of-range or dead slots are ignored
	if (i < 0 || i >= b.capacity || (b.flags[i] & S2B_BODY_VALID) == 0)
	{
		return;
	}
	float2 add = forces[t];
	float* f = reinterpret_cast<float*>(b.frc + i);
	atomicAdd(f + 0, add.x);
	atomicAdd(f + 1, add.y);
}

__global__ void s2bGatherTransforms(BodyView b, int count, float4* out)
{
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= count)
	{
		return;
	}
	float4 org = b.org[i];
	float4 pose = b.pose[i];
	out[i] = make_float4(org.x, org.y, pose.z, pose.w);
}

extern "C" void s2b_upload_forces(s2bWorld* w, const s2bForceRow* rows, int count)
{
	if (count <= 0)
	{
		return;
	}
	S2B_CHECK(cudaSetDevice(w->device));
	s2bForceRow* d = (s2bForceRow*)stageRows(w, rows, sizeof(s2bForceRow) * (size_t)count);
	S2B_LAUNCH(w, s2bScatterForces, gridFor(count, 128), 128, 0, d, count, bodyView(w));
	S2B_CHECK(cudaFreeAsync(d, w->stream));
	S2B_CHECK(cudaStreamSynchronize(w->stream));
}

// page-locked staging for the bulk paths: two buffers used alternately, each guarded by an event so that the host never
// overwrites a buffer whose H2D copy is still in flight and never has to synchronise the stream
static void* bulkStaging(s2bWorld* w, size_t bytes)
{
	int k = w->bulkNext;
	w->bulkNext ^= 1;
	if (w->bulkEvent[k] == nullptr)
	{
		S2B_CHECK(cudaEventCreateWithFlags(&w->bulkEvent[k], cudaEventDisableTiming));
	}
	else
	{
		S2B_CHECK(cudaEventSynchronize(w->bulkEvent[k]));
	}
	if (bytes > w->bulkBytes[k])
	{
		if (w->bulkHost[k] != nullptr)
		{
			cudaFreeHost(w->bulkHost[k]);
		}
		w->bulkBytes[k] = bytes + bytes / 2;
		S2B_CHECK(cudaMallocHost(&w->bulkHost[k], w->bulkBytes[k]));
	}
	w->bulkCurrent = k;
	return w->bulkHost[k];
}

extern "C" void s2b_add_forces(s2bWorld* w, const int32_t* bodyIndices, const float* forcesXY, int count)
{
	S2bEpochFreeze freeze; // transfer / flush buffers are not part of any captured graph

	if (count <= 0)
	{
		return;
	}
	S2B_CHECK(cudaSetDevice(w->device));
	size_t idxBytes = sizeof(int32_t) * (size_t)count;
	size_t idxPadded = (idxBytes + 15) & ~(size_t)15;
	size_t bytes = idxPadded + sizeof(float) * 2 * (size_t)count;
	char* host = (char*)bulkStaging(w, bytes);
	memcpy(host, bodyIndices, idxBytes);
	memcpy(host + idxPadded, forcesXY, sizeof(float) * 2 * (size_t)count);
	w->dBulk.reserve(bytes, w->stream, false, false);
	S2B_CHECK(cudaMemcpyAsync(w->dBulk.p, host, bytes, cudaMemcpyHostToDevice, w->stream));
	S2B_CHECK(cudaEventRecord(w->bulkEvent[w->bulkCurrent], w->stream));
	S2B_LAUNCH(w, s2bAddForcesKernel, gridFor(count, 256), 256, 0, (const int*)w->dBulk.p, (const float2*)(w->dBulk.p + idxPadded), count,
			   bodyView(w));
}

// one thread per entry: a motor joint's linear offset (anchors.xy) and angular offset (lim.x), nothing else of the row.
// Entries that do not name a live motor joint are skipped; the host validates before it calls.
__global__ void s2bSetMotorOffsetsKernel(const int* __restrict__ indices, const float* __restrict__ offsets, int count, JointView j)
{
	int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= count)
	{
		return;
	}
	int i = indices[t];
	if (i < 0 || i >= j.capacity)
	{
		return;
	}
	int flags = j.head[i].x;
	if ((flags & S2B_ROW_VALID) == 0 || ((flags >> 1) & 0x7) != S2B_JOINT_MOTOR)
	{
		return;
	}
	float* anchors = reinterpret_cast<float*>(j.anchors + i);
	anchors[0] = offsets[3 * t + 0];
	anchors[1] = offsets[3 * t + 1];
	reinterpret_cast<float*>(j.lim + i)[0] = offsets[3 * t + 2];
}

extern "C" void s2b_set_motor_offsets(s2bWorld* w, const int32_t* jointIndices, const float* offsets, int count)
{
	S2bEpochFreeze freeze; // transfer buffers are not part of any captured graph

	if (count <= 0)
	{
		return;
	}
	S2B_CHECK(cudaSetDevice(w->device));
	// no uploadEpoch bump, no schedDirty and no synchronisation: the offsets are solver inputs only, so the prefetched pair
	// search and the captured step graph stay valid
	size_t idxBytes = sizeof(int32_t) * (size_t)count;
	size_t idxPadded = (idxBytes + 15) & ~(size_t)15;
	size_t bytes = idxPadded + sizeof(float) * 3 * (size_t)count;
	char* host = (char*)bulkStaging(w, bytes);
	memcpy(host, jointIndices, idxBytes);
	memcpy(host + idxPadded, offsets, sizeof(float) * 3 * (size_t)count);
	w->dBulk.reserve(bytes, w->stream, false, false);
	S2B_CHECK(cudaMemcpyAsync(w->dBulk.p, host, bytes, cudaMemcpyHostToDevice, w->stream));
	S2B_CHECK(cudaEventRecord(w->bulkEvent[w->bulkCurrent], w->stream));
	S2B_LAUNCH(w, s2bSetMotorOffsetsKernel, gridFor(count, 256), 256, 0, (const int*)w->dBulk.p,
			   (const float*)(w->dBulk.p + idxPadded), count, jointView(w));
}

extern "C" void s2b_download_transforms(s2bWorld* w, float* out, int count)
{
	S2bEpochFreeze freeze; // transfer / flush buffers are not part of any captured graph

	S2B_CHECK(cudaSetDevice(w->device));
	if (count > w->bodyCap)
	{
		count = w->bodyCap;
	}
	if (count <= 0)
	{
		return;
	}
	size_t floats = 4 * (size_t)count;
	if (floats > w->hostXfFloats)
	{
		if (w->hostXf != nullptr)
		{
			cudaFreeHost(w->hostXf);
		}
		w->hostXfFloats = floats + floats / 2;
		S2B_CHECK(cudaMallocHost((void**)&w->hostXf, sizeof(float) * w->hostXfFloats));
	}
	// finalize was the last writer of the transforms (nothing uploaded, no solver stage since): gather and copy on the side
	// stream, behind finalize only — not behind what the world's stream has queued after it
	bool side = w->sideCopies != 0 && w->movedEvent != nullptr && w->finalizeSeq == w->xfSeq && w->dXf.cap >= (size_t)count;
	w->dXf.reserve((size_t)count, w->stream, false, false);
	cudaStream_t cs = w->stream;
	if (side)
	{
		if (w->copyStream == nullptr)
		{
			S2B_CHECK(cudaStreamCreateWithFlags(&w->copyStream, cudaStreamNonBlocking));
		}
		cs = w->copyStream;
		S2B_CHECK(cudaStreamWaitEvent(cs, w->movedEvent, 0));
	}
	s2bGatherTransforms<<<gridFor(count, 256), 256, 0, cs>>>(bodyView(w), count, w->dXf.p);
	S2B_CHECK(cudaGetLastError());
	w->kernelLaunches += 1;
	// a page-locked destination (s2b_host_alloc / cudaHostRegister) takes the DMA directly; pageable memory goes through the
	// world's own pinned buffer and one host copy
	cudaPointerAttributes attr;
	bool pinned = cudaPointerGetAttributes(&attr, out) == cudaSuccess && attr.type == cudaMemoryTypeHost;
	(void)cudaGetLastError();
	float* dst = pinned ? out : w->hostXf;
	S2B_CHECK(cudaMemcpyAsync(dst, w->dXf.p, sizeof(float) * floats, cudaMemcpyDeviceToHost, cs));
	S2B_CHECK(cudaStreamSynchronize(cs));
	if (pinned == false)
	{
		memcpy(out, w->hostXf, sizeof(float) * floats);
	}
}

extern "C" void* s2b_host_alloc(size_t bytes)
{
	void* p = nullptr;
	S2B_CHECK(cudaMallocHost(&p, bytes));
	return p;
}

extern "C" void s2b_host_free(void* p)
{
	if (p != nullptr)
	{
		cudaFreeHost(p);
	}
}

__global__ void s2bGatherBodyState(BodyView b, int count, float4* out)
{
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= count)
	{
		return;
	}
	float4 org = b.org[i], pos = b.pos[i], pose = b.pose[i], vel = b.vel[i], frc = b.frc[i];
	out[3 * i + 0] = make_float4(org.x, org.y, pos.x, pos.y);
	out[3 * i + 1] = make_float4(pose.z, pose.w, vel.x, vel.y);
	out[3 * i + 2] = make_float4(vel.z, frc.x, frc.y, frc.z);
}

extern "C" const float* s2b_sync_body_state(s2bWorld* w, int capacity)
{
	S2bEpochFreeze freeze; // transfer / flush buffers are not part of any captured graph

	S2B_CHECK(cudaSetDevice(w->device));
	if (capacity > w->bodyCap)
	{
		capacity = w->bodyCap;
	}
	size_t floats = 12 * (size_t)(capacity > 0 ? capacity : 1);
	if (floats > w->hostStateFloats)
	{
		if (w->hostState != nullptr)
		{
			cudaFreeHost(w->hostState);
		}
		w->hostStateFloats = floats + floats / 2;
		S2B_CHECK(cudaMallocHost((void**)&w->hostState, sizeof(float) * w->hostStateFloats));
	}
	if (capacity > 0)
	{
		w->dState.reserve(3 * (size_t)capacity, w->stream, false, false);
		S2B_LAUNCH(w, s2bGatherBodyState, gridFor(capacity, 256), 256, 0, bodyView(w), capacity, w->dState.p);
		S2B_CHECK(cudaMemcpyAsync(w->hostState, w->dState.p, sizeof(float) * 12 * (size_t)capacity, cudaMemcpyDeviceToHost,
								  w->stream));
	}
	S2B_CHECK(cudaStreamSynchronize(w->stream));
	return w->hostState;
}

extern "C" void s2b_mark_pairs_dirty(s2bWorld* w)
{
	w->pairsDirty = true;
}

extern "C" void s2b_set_contact_order(s2bWorld* w, const uint64_t* pairKeys, int count)
{
	w->orderHint.assign(pairKeys, pairKeys + (count > 0 ? count : 0));
}

extern "C" void* s2b_get_stream(s2bWorld* w)
{
	return (void*)w->stream;
}

extern "C" void s2b_sync(s2bWorld* w)
{
	S2B_CHECK(cudaSetDevice(w->device));
	S2B_CHECK(cudaStreamSynchronize(w->stream));
}

extern "C" void s2b_download_bodies(s2bWorld* w, s2bBodyRow* rows, int count)
{
	if (count <= 0)
	{
		return;
	}
	S2B_CHECK(cudaSetDevice(w->device));
	s2bBodyRow* d = (s2bBodyRow*)stageRows(w, rows, sizeof(s2bBodyRow) * (size_t)count);
	S2B_LAUNCH(w, s2bGatherBodies, gridFor(count, 128), 128, 0, d, count, bodyView(w), 1);
	S2B_CHECK(cudaMemcpyAsync(rows, d, sizeof(s2bBodyRow) * (size_t)count, cudaMemcpyDeviceToHost, w->stream));
	S2B_CHECK(cudaFreeAsync(d, w->stream));
	S2B_CHECK(cudaStreamSynchronize(w->stream));
}

extern "C" void s2b_download_all_bodies(s2bWorld* w, s2bBodyRow* rows, int capacity)
{
	if (capacity <= 0)
	{
		return;
	}
	S2B_CHECK(cudaSetDevice(w->device));
	if (capacity > w->bodyCap)
	{
		capacity = w->bodyCap;
	}
	s2bBodyRow* d = nullptr;
	S2B_CHECK(cudaMallocAsync((void**)&d, sizeof(s2bBodyRow) * (size_t)capacity, w->stream));
	S2B_LAUNCH(w, s2bGatherBodies, gridFor(capacity, 128), 128, 0, d, capacity, bodyView(w), 0);
	S2B_CHECK(cudaMemcpyAsync(rows, d, sizeof(s2bBodyRow) * (size_t)capacity, cudaMemcpyDeviceToHost, w->stream));
	S2B_CHECK(cudaFreeAsync(d, w->stream));
	S2B_CHECK(cudaStreamSynchronize(w->stream));
}

__global__ void s2bGatherDeltaPositions(float2* out, int count, BodyView b)
{
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < count)
	{
		float4 pose = b.pose[i];
		out[i] = make_float2(pose.x, pose.y);
	}
}

extern "C" void s2b_download_delta_positions(s2bWorld* w, float* xy, int capacity)
{
	S2B_CHECK(cudaSetDevice(w->device));
	if (capacity > w->bodyCap)
	{
		memset(xy + 2 * (size_t)w->bodyCap, 0, sizeof(float2) * (size_t)(capacity - w->bodyCap));
		capacity = w->bodyCap;
	}
	if (capacity <= 0)
	{
		return;
	}
	float2* d = nullptr;
	S2B_CHECK(cudaMallocAsync((void**)&d, sizeof(float2) * (size_t)capacity, w->stream));
	S2B_LAUNCH(w, s2bGatherDeltaPositions, gridFor(capacity, 128), 128, 0, d, capacity, bodyView(w));
	S2B_CHECK(cudaMemcpyAsync(xy, d, sizeof(float2) * (size_t)capacity, cudaMemcpyDeviceToHost, w->stream));
	S2B_CHECK(cudaFreeAsync(d, w->stream));
	S2B_CHECK(cudaStreamSynchronize(w->stream));
}

extern "C" void s2b_download_shape_boxes(s2bWorld* w, float* aabb4, float* fat4, int32_t* flags, int capacity)
{
	S2B_CHECK(cudaSetDevice(w->device));
	if (capacity > w->shapeCap)
	{
		capacity = w->shapeCap;
	}
	if (capacity <= 0)
	{
		return;
	}
	S2B_CHECK(cudaStreamSynchronize(w->stream));
	if (aabb4)
	{
		S2B_CHECK(cudaMemcpy(aabb4, w->sAabb.p, sizeof(float4) * (size_t)capacity, cudaMemcpyDeviceToHost));
	}
	if (fat4)
	{
		S2B_CHECK(cudaMemcpy(fat4, w->sFat.p, sizeof(float4) * (size_t)capacity, cudaMemcpyDeviceToHost));
	}
	if (flags)
	{
		std::vector<int4> head((size_t)capacity);
		S2B_CHECK(cudaMemcpy(head.data(), w->sHead.p, sizeof(int4) * (size_t)capacity, cudaMemcpyDeviceToHost));
		for (int i = 0; i < capacity; ++i)
		{
			flags[i] = head[i].x;
		}
	}
}

extern "C" void s2b_download_joints(s2bWorld* w, s2bJointRow* rows, int capacity)
{
	S2B_CHECK(cudaSetDevice(w->device));
	if (capacity > w->jointCap)
	{
		capacity = w->jointCap;
	}
	if (capacity <= 0)
	{
		return;
	}
	s2bJointRow* d = nullptr;
	S2B_CHECK(cudaMallocAsync((void**)&d, sizeof(s2bJointRow) * (size_t)capacity, w->stream));
	S2B_LAUNCH(w, s2bGatherJoints, gridFor(capacity, 128), 128, 0, d, capacity, jointView(w));
	S2B_CHECK(cudaMemcpyAsync(rows, d, sizeof(s2bJointRow) * (size_t)capacity, cudaMemcpyDeviceToHost, w->stream));
	S2B_CHECK(cudaFreeAsync(d, w->stream));
	S2B_CHECK(cudaStreamSynchronize(w->stream));
}

extern "C" int s2b_download_contacts(s2bWorld* w, s2bContactRow* rows, int maxCount)
{
	S2B_CHECK(cudaSetDevice(w->device));
	S2B_CHECK(cudaStreamSynchronize(w->stream));
	int count = w->contactCount < maxCount ? w->contactCount : maxCount;
	if (count <= 0)
	{
		return 0;
	}
	s2bContactRow* d = nullptr;
	S2B_CHECK(cudaMallocAsync((void**)&d, sizeof(s2bContactRow) * (size_t)count, w->stream));
	S2B_LAUNCH(w, s2bGatherContacts, gridFor(count, 128), 128, 0, d, count, makeView(w->contacts[w->cur]),
			   w->sticky ? 1 : 0);
	S2B_CHECK(cudaMemcpyAsync(rows, d, sizeof(s2bContactRow) * (size_t)count, cudaMemcpyDeviceToHost, w->stream));
	S2B_CHECK(cudaFreeAsync(d, w->stream));
	S2B_CHECK(cudaStreamSynchronize(w->stream));
	return count;
}

extern "C" void s2b_pack_body_state(s2bWorld* w, int first, int count, void* deviceOut)
{
	if (count <= 0)
	{
		return;
	}
	S2B_CHECK(cudaSetDevice(w->device));
	S2B_LAUNCH(w, s2bPackBodyState, gridFor(count, 128), 128, 0, bodyView(w), first, count, (float4*)deviceOut);
}

extern "C" void s2b_flush_l2(s2bWorld* w)
{
	S2bEpochFreeze freeze; // transfer / flush buffers are not part of any captured graph

	S2B_CHECK(cudaSetDevice(w->device));
	const size_t bytes = (size_t)128 << 20; // more than twice the 50 MB L2 of an H100
	w->l2Flush.reserve(bytes, w->stream, false, false);
	static int value = 0;
	value += 1;
	S2B_LAUNCH(w, s2bFlushKernel, w->smCount * 8, 256, 0, w->l2Flush.p, bytes, value);
}

// Each stage stamps its start on the world's stream (ev[0..3]); finalize also stamps the end (ev[4]).
extern "C" void s2b_update_pairs(s2bWorld* w)
{
	S2B_CHECK(cudaSetDevice(w->device));
	s2bBroadphaseUpdatePairs(w); // may synchronise on the previous step before it enqueues anything
}

extern "C" void s2b_update_contacts(s2bWorld* w)
{
	S2B_CHECK(cudaSetDevice(w->device));
	S2B_CHECK(cudaEventRecord(w->timer.ev[1], w->stream));
	s2bNarrowphaseUpdate(w);
}

extern "C" void s2b_solve(s2bWorld* w, int solverType, const s2bStepContext* context)
{
	S2B_CHECK(cudaSetDevice(w->device));
	w->xfSeq += 1;
	S2B_CHECK(cudaEventRecord(w->timer.ev[2], w->stream));
	s2bSolve(w, solverType, context);
}

extern "C" void s2b_finalize(s2bWorld* w)
{
	S2B_CHECK(cudaSetDevice(w->device));
	S2B_CHECK(cudaEventRecord(w->timer.ev[3], w->stream));
	s2bFinalize(w);
	w->xfSeq += 1;
	w->finalizeSeq = w->xfSeq;
	S2B_CHECK(cudaEventRecord(w->timer.ev[4], w->stream));
	w->timer.recorded = true;
}

extern "C" void s2b_prefetch_pairs(s2bWorld* w)
{
	S2B_CHECK(cudaSetDevice(w->device));
	s2bPrefetchPairSearch(w);
}

extern "C" void s2b_step(s2bWorld* w, int solverType, const s2bStepContext* context)
{
	s2b_update_pairs(w);
	s2b_update_contacts(w);
	s2b_solve(w, solverType, context);
	s2b_finalize(w);
	s2b_prefetch_pairs(w);
}

extern "C" void s2b_last_stage_ms(s2bWorld* w, float out[4])
{
	S2B_CHECK(cudaSetDevice(w->device));
	for (int i = 0; i < 4; ++i)
	{
		out[i] = 0.0f;
	}
	if (w->timer.recorded == false)
	{
		return;
	}
	S2B_CHECK(cudaEventSynchronize(w->timer.ev[4]));
	for (int i = 0; i < 4; ++i)
	{
		S2B_CHECK(cudaEventElapsedTime(out + i, w->timer.ev[i], w->timer.ev[i + 1]));
	}
	// the search half of the pair pass runs behind finalize (s2b_prefetch_pairs): the last finished one is charged to "pairs"
	out[0] += s2bLastPairSearchMs(w);
}

extern "C" float s2b_timed_steps(s2bWorld* w, int solverType, const s2bStepContext* context, int steps)
{
	S2B_CHECK(cudaSetDevice(w->device));
	cudaEvent_t e0, e1;
	S2B_CHECK(cudaEventCreate(&e0));
	S2B_CHECK(cudaEventCreate(&e1));
	S2B_CHECK(cudaStreamSynchronize(w->stream));
	S2B_CHECK(cudaEventRecord(e0, w->stream));
	for (int i = 0; i < steps; ++i)
	{
		s2b_step(w, solverType, context);
	}
	S2B_CHECK(cudaEventRecord(e1, w->stream));
	S2B_CHECK(cudaEventSynchronize(e1));
	float ms = 0.0f;
	S2B_CHECK(cudaEventElapsedTime(&ms, e0, e1));
	cudaEventDestroy(e0);
	cudaEventDestroy(e1);
	return ms;
}

// user stop-watch on the world's stream: mark(0) ... mark(1), then elapsed
static cudaEvent_t s2bMarkEvent(s2bWorld* w, int slot)
{
	static_assert(sizeof(cudaEvent_t) == sizeof(void*), "event handle size");
	if (w->markEvents[slot] == nullptr)
	{
		S2B_CHECK(cudaEventCreate(&w->markEvents[slot]));
	}
	return w->markEvents[slot];
}

extern "C" void s2b_mark_time(s2bWorld* w, int slot)
{
	S2B_CHECK(cudaSetDevice(w->device));
	S2B_CHECK(cudaEventRecord(s2bMarkEvent(w, slot & 1), w->stream));
}

extern "C" float s2b_elapsed_ms(s2bWorld* w)
{
	S2B_CHECK(cudaSetDevice(w->device));
	S2B_CHECK(cudaEventSynchronize(s2bMarkEvent(w, 1)));
	float ms = 0.0f;
	S2B_CHECK(cudaEventElapsedTime(&ms, s2bMarkEvent(w, 0), s2bMarkEvent(w, 1)));
	return ms;
}

extern "C" void s2b_abi_sizes(int32_t out[6])
{
	out[0] = (int32_t)sizeof(s2bBodyRow);
	out[1] = (int32_t)sizeof(s2bShapeRow);
	out[2] = (int32_t)sizeof(s2bJointRow);
	out[3] = (int32_t)sizeof(s2bContactRow);
	out[4] = (int32_t)sizeof(s2bStepContext);
	out[5] = (int32_t)sizeof(s2bCounters);
}

extern "C" const char* s2b_version(void)
{
	return "solver2d-b200 0.1 (sm_90a)";
}

__global__ void s2bEvalAtan2Kernel(const float* y, const float* x, float* out, int n)
{
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n)
	{
		out[i] = S2_ATAN2F(y[i], x[i]);
	}
}

extern "C" void s2b_eval_atan2(const float* y, const float* x, float* out, int32_t count)
{
	if (count <= 0)
	{
		return;
	}
	float *dy = nullptr, *dx = nullptr, *dout = nullptr;
	size_t bytes = sizeof(float) * (size_t)count;
	S2B_CHECK(cudaMalloc(&dy, bytes));
	S2B_CHECK(cudaMalloc(&dx, bytes));
	S2B_CHECK(cudaMalloc(&dout, bytes));
	S2B_CHECK(cudaMemcpy(dy, y, bytes, cudaMemcpyHostToDevice));
	S2B_CHECK(cudaMemcpy(dx, x, bytes, cudaMemcpyHostToDevice));
	s2bEvalAtan2Kernel<<<(count + 255) / 256, 256>>>(dy, dx, dout, count);
	S2B_CHECK(cudaGetLastError());
	S2B_CHECK(cudaMemcpy(out, dout, bytes, cudaMemcpyDeviceToHost));
	cudaFree(dy);
	cudaFree(dx);
	cudaFree(dout);
}
