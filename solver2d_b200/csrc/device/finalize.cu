// solver2d-b200 — stage 4 of s2World_Step on the device: body origins, force reset, shape AABB refit, fat-AABB
// "enlarge" + move buffering (reference src/world.c:258-301, src/shape.c:48-67).
//
// Both kernels are pure streaming passes (bandwidth-bound): bodies 64 B read + 32 B written, shapes ~190 B read
// (geometry) + 16-32 B written.
#include "finalize.cuh"

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
// for the clamped pose, as finalize derives them. When finalize has already collected this pass's moved proxies
// (s2bFinalizeRefit), `movedLeaves` is set: a shape that escapes its fat box only now (the one that is counted) is appended to
// them, at its sorted leaf (`shapeLeaf`).
__global__ void s2bRefinalizeShapes(ShapeView s, BodyView b, const int* list, const int* count, const unsigned* fraction,
									int* movedCounter, const int* shapeLeaf, int* movedLeaves, int* movedLeafCount)
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
	int before = head.x;
	s2bFinalizeShape<true>(s, b, i, head, movedCounter);
	if (movedLeaves != nullptr && (head.x & S2B_SHAPE_MOVED) != 0 && (before & S2B_SHAPE_MOVED) == 0)
	{
		movedLeaves[atomicAdd(movedLeafCount, 1)] = shapeLeaf[i];
	}
}

void s2bRefinalizeBulletShapes(s2bWorld* w, const int* list, const int* count, const unsigned* fraction, const int* shapeLeaf,
							   int* movedLeaves, int* movedLeafCount)
{
	S2B_LAUNCH(w, s2bRefinalizeShapes, gridFor(w->shapeCap, 256), 256, 0, shapeView(w), bodyView(w), list, count, fraction,
			   w->dMovedFlag.p, shapeLeaf, movedLeaves, movedLeafCount);
}

void s2bFinalize(s2bWorld* w)
{
	cudaStream_t st = w->stream;
	w->dMovedFlag.reserve(4, st, true);
	if (w->bodyCap > 0)
	{
		S2B_LAUNCH(w, s2bFinalizeBodies, gridFor(w->bodyCap, 256), 256, 0, bodyView(w));
	}
	// when the next pair search will reuse the hierarchy's topology, the shapes are finalized by the kernel that also refits
	// it and collects the search's moved proxies (DESIGN.md §3.3)
	if (w->shapeCap > 0 && s2bFinalizeRefit(w) == false)
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
	// joint reactions against their break thresholds, on the impulses just solved and the final poses; a world without
	// thresholds launches nothing here (DESIGN.md §3.13)
	if (w->breakCount > 0 && w->jointCap > 0)
	{
		s2bJointBreakPass(w, cs);
	}
	else
	{
		w->brokenPending = false;
		w->jointsChecked = 0;
	}
}
