// solver2d-b200 — stage 4 of s2World_Step on the device: body origins, force reset, shape AABB refit, fat-AABB
// "enlarge" + move buffering (reference src/world.c:258-301, src/shape.c:48-67).
//
// Both kernels are pure streaming passes (bandwidth-bound): bodies 64 B read + 32 B written, shapes ~190 B read
// (geometry) + 16-32 B written.
#include "s2b_internal.cuh"

__global__ void s2bFinalizeBodies(BodyView b)
{
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= b.capacity)
	{
		return;
	}
	unsigned f = b.flags[i];
	if ((f & S2B_BODY_VALID) == 0 || S2B_BODY_TYPE(f) == S2B_BODY_STATIC)
	{
		return;
	}
	float4 pos = b.pos[i];
	float4 pose = b.pose[i];
	float4 org = b.org[i];
	float4 frc = b.frc[i];
	s2Rot q = {pose.z, pose.w};
	s2Vec2 lc = {org.z, org.w};
	s2Vec2 p = {pos.x, pos.y};
	// origin = position - R * localCenter  (reference src/world.c:274)
	s2Vec2 o = s2Sub(p, s2RotateVector(q, lc));
	b.org[i] = make_float4(o.x, o.y, org.z, org.w);
	b.frc[i] = make_float4(0.0f, 0.0f, 0.0f, frc.w);
}

// All four shape kinds are stored in polygon form (count vertices + radius), for which the per-kind AABB functions of
// the reference (src/geometry.c:288-341) reduce to the same float operations: min/max over the transformed
// vertices, then -/+ radius.
//
// Once finalize has run, the bullet pass (DESIGN.md §3.12) redoes a clamped bullet's shapes with `again`: a shape that is
// already flagged MOVED is not counted a second time.
template <bool again> __device__ __forceinline__ void s2bFinalizeShape(const ShapeView& s, const BodyView& b, int i, int4 head,
																		 int* movedCounter)
{
	int body = head.y;
	float4 org = b.org[body];
	float4 pose = b.pose[body];
	s2Transform xf;
	xf.p.x = org.x;
	xf.p.y = org.y;
	xf.q.s = pose.z;
	xf.q.c = pose.w;

	int count = head.w;
	float radius = s.fr[i].y;
	float2 v0 = s.verts[i * 8];
	s2Vec2 p0 = {v0.x, v0.y};
	s2Vec2 lower = s2TransformPoint(xf, p0);
	s2Vec2 upper = lower;
	for (int k = 1; k < count; ++k)
	{
		float2 vk = s.verts[i * 8 + k];
		s2Vec2 pk = {vk.x, vk.y};
		s2Vec2 v = s2TransformPoint(xf, pk);
		lower = s2Min(lower, v);
		upper = s2Max(upper, v);
	}
	s2Vec2 r = {radius, radius};
	lower = s2Sub(lower, r);
	upper = s2Add(upper, r);

	s2Box aabb;
	aabb.lowerBound.x = lower.x - s2_speculativeDistance;
	aabb.lowerBound.y = lower.y - s2_speculativeDistance;
	aabb.upperBound.x = upper.x + s2_speculativeDistance;
	aabb.upperBound.y = upper.y + s2_speculativeDistance;
	s.aabb[i] = make_float4(aabb.lowerBound.x, aabb.lowerBound.y, aabb.upperBound.x, aabb.upperBound.y);

	float4 fat4 = s.fat[i];
	s2Box fat;
	fat.lowerBound.x = fat4.x;
	fat.lowerBound.y = fat4.y;
	fat.upperBound.x = fat4.z;
	fat.upperBound.y = fat4.w;
	if (s2AABB_Contains(fat, aabb) == false)
	{
		// the proxy escaped its fat box: re-centre it and buffer a move for the next pair update
		// (reference src/world.c:291-296 -> s2BroadPhase_EnlargeProxy -> s2BufferMove)
		s.fat[i] = make_float4(aabb.lowerBound.x - s2_aabbMargin, aabb.lowerBound.y - s2_aabbMargin,
							   aabb.upperBound.x + s2_aabbMargin, aabb.upperBound.y + s2_aabbMargin);
		s.head[i] = make_int4(head.x | S2B_SHAPE_MOVED, head.y, head.z, head.w);
		if (again == false || (head.x & S2B_SHAPE_MOVED) == 0)
		{
			atomicAdd(movedCounter, 1);
		}
	}
}

__global__ void s2bFinalizeShapes(ShapeView s, BodyView b, int* movedCounter)
{
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= s.capacity)
	{
		return;
	}
	int4 head = s.head[i];
	if ((head.x & S2B_ROW_VALID) == 0)
	{
		return;
	}
	unsigned f = b.flags[head.y];
	if (S2B_BODY_TYPE(f) == S2B_BODY_STATIC)
	{
		return;
	}
	s2bFinalizeShape<false>(s, b, i, head, movedCounter);
}

// The listed shapes (list[0, count[0])) of the bodies the bullet pass clamped (fraction below 1): boxes and fat-box moves
// for the clamped pose, as finalize derives them.
__global__ void s2bRefinalizeShapes(ShapeView s, BodyView b, const int* list, const int* count, const unsigned* fraction,
									int* movedCounter)
{
	int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= count[0])
	{
		return;
	}
	int i = list[k];
	int4 head = s.head[i];
	if (fraction[head.y] >= S2B_FRACTION_ONE) // (not clamped)
	{
		return;
	}
	s2bFinalizeShape<true>(s, b, i, head, movedCounter);
}

void s2bRefinalizeBulletShapes(s2bWorld* w, const int* list, const int* count, const unsigned* fraction)
{
	S2B_LAUNCH(w, s2bRefinalizeShapes, gridFor(w->shapeCap, 256), 256, 0, shapeView(w), bodyView(w), list, count, fraction,
			   w->dMovedFlag.p);
}

void s2bFinalize(s2bWorld* w)
{
	cudaStream_t st = w->stream;
	w->dMovedFlag.reserve(4, st, true);
	if (w->bodyCap > 0)
	{
		S2B_LAUNCH(w, s2bFinalizeBodies, gridFor(w->bodyCap, 256), 256, 0, bodyView(w));
	}
	if (w->shapeCap > 0)
	{
		S2B_LAUNCH(w, s2bFinalizeShapes, gridFor(w->shapeCap, 256), 256, 0, shapeView(w), bodyView(w), w->dMovedFlag.p);
	}
	// bullets are swept once every other body is final, and their boxes and moves redone where they were clamped: all of it
	// before the moved counter is copied, so that the transform read-back and the pair search behind it see the clamped poses
	if (w->continuous != 0 && w->bulletCount > 0)
	{
		s2bBulletPass(w);
	}
	// publish the moved-proxy counter to the pinned mailbox; the next step reads it after this step has drained. The copy
	// runs on the side stream, behind finalize only: on the world's stream the device-to-host copy (and the counter memset
	// after it) between finalize and the pair search queued behind it left the device idle for ~20 us per step (H100). Until
	// movedEvent has passed, the counter must not be reset (s2bBroadphaseUpdatePairs waits for it) and the mailbox slot
	// must not be read (s2bBroadphaseUpdatePairs, s2b_get_counters).
	if (w->movedEvent == nullptr)
	{
		S2B_CHECK(cudaEventCreateWithFlags(&w->movedEvent, cudaEventDisableTiming));
		S2B_CHECK(cudaEventCreateWithFlags(&w->finalizedEvent, cudaEventDisableTiming));
	}
	cudaStream_t cs = st;
	if (w->sideCopies != 0)
	{
		if (w->copyStream == nullptr)
		{
			S2B_CHECK(cudaStreamCreateWithFlags(&w->copyStream, cudaStreamNonBlocking));
		}
		cs = w->copyStream;
		S2B_CHECK(cudaEventRecord(w->finalizedEvent, st));
		S2B_CHECK(cudaStreamWaitEvent(cs, w->finalizedEvent, 0));
	}
	S2B_CHECK(cudaMemcpyAsync(w->hostMail + MAIL_MOVED, w->dMovedFlag.p, sizeof(int), cudaMemcpyDeviceToHost, cs));
	S2B_CHECK(cudaEventRecord(w->movedEvent, cs));
}
