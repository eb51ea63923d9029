// solver2d-b200 — joint reactions and break thresholds (DESIGN.md §3.13).
//
// One thread per joint slot evaluates s2MakeJointReaction (include/solver2d_b200.h) on the impulses the last solve stored,
// body A's final rotation (a distance joint: the line between its anchors at both bodies' final poses; a pulley: -ratio times
// rope B's direction at body B's final pose; a gear: its impulse times side 2's Jacobian at body B's final pose) and the rate
// of that
// solve. After finalize (s2bFinalize) it compares the reaction with the
// slot's thresholds and appends the slots over one to a list; on demand (s2b_download_joint_reactions) it writes the
// reactions instead. The solver kernels are not touched: everything it reads is already in the joint and body columns.
#include "s2b_internal.cuh"
#include "shared/s2_distance_joint.h"
#include "shared/s2_gear_joint.h"
#include "solver2d_b200.h"

#include <algorithm>

__global__ void s2bJointReactionKernel(JointView j, const float2* __restrict__ brk, const float4* __restrict__ pose,
									   const float4* __restrict__ pos, const float4* __restrict__ org, float rate, float* reactions,
									   int* broken)
{
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= j.capacity)
	{
		return;
	}
	int4 head = j.head[i];
	if ((head.x & S2B_ROW_VALID) == 0)
	{
		if (reactions != nullptr)
		{
			reactions[3 * i] = 0.0f;
			reactions[3 * i + 1] = 0.0f;
			reactions[3 * i + 2] = 0.0f;
		}
		return;
	}
	float2 thresholds = make_float2(0.0f, 0.0f);
	if (broken != nullptr)
	{
		thresholds = brk[i];
		if (thresholds.x <= 0.0f && thresholds.y <= 0.0f)
		{
			return; // nothing to test: no load is read
		}
	}
	float4 imp = j.imp[i], limp = j.limp[i], target = j.target[i];
	float4 qa = pose[head.y];
	s2Rot qA = {qa.z, qa.w};
	// a spring acts on the motor's axis: its impulse joins the motor argument (DESIGN.md §3.14)
	float motorImpulse = (head.x & S2B_JOINT_ENABLE_SPRING) != 0 ? imp.z + imp.w : imp.z;
	int type = s2bJointType(head.x);
	s2Vec2 axis = s2MakeVec2(target.z, target.w);
	if (type == S2B_JOINT_DISTANCE)
	{
		// the world axis from anchor A to anchor B at the end of the step (DESIGN.md §3.16), as the host getters form it
		float4 anchors = j.anchors[i];
		float4 pa = pos[head.y], pb = pos[head.z], qb = pose[head.z], oa = org[head.y], ob = org[head.z];
		float length;
		axis = s2cDistanceJointAxis(&length, s2MakeVec2(pa.x, pa.y), qA, s2Sub(s2MakeVec2(anchors.x, anchors.y), s2MakeVec2(oa.z, oa.w)),
									s2MakeVec2(pb.x, pb.y), s2Rot{qb.z, qb.w},
									s2Sub(s2MakeVec2(anchors.z, anchors.w), s2MakeVec2(ob.z, ob.w)));
	}
	else if (type == S2B_JOINT_PULLEY)
	{
		// -ratio uB at the end of the step (DESIGN.md §3.18): ground anchor B rides in target.zw, the ratio in lim.x
		float4 anchors = j.anchors[i];
		float4 pb = pos[head.z], qb = pose[head.z], ob = org[head.z];
		float length;
		axis = s2cPulleyJointAxis(&length, axis, s2MakeVec2(pb.x, pb.y), s2Rot{qb.z, qb.w},
								  s2Sub(s2MakeVec2(anchors.z, anchors.w), s2MakeVec2(ob.z, ob.w)), j.lim[i].x);
	}
	else if (type == S2B_JOINT_GEAR)
	{
		// (lambda Jv2, lambda Jw2) at the end of the step through the generic branch (DESIGN.md §3.19): side 2's frame rides
		// in motor, the ratio in lim.x. Only the Jacobian is read, so the revolute side's coordinate is formed at theta 0.
		float4 anchors = j.anchors[i], frame = j.motor[i];
		float4 pb = pos[head.z], qb = pose[head.z], ob = org[head.z];
		s2Rot qB = {qb.z, qb.w};
		s2cGearSide side2 = (head.x & S2B_JOINT_GEAR_PRISMATIC2) != 0
								? s2cGearPrismatic(s2Sub(s2MakeVec2(pb.x, pb.y), s2MakeVec2(frame.x, frame.y)), s2MakeVec2(frame.z, frame.w),
												   s2MakeVec2(0.0f, 0.0f), qB, s2Sub(s2MakeVec2(anchors.z, anchors.w), s2MakeVec2(ob.z, ob.w)))
								: s2cGearRevolute(frame.x, frame.y, frame.z, 0.0f, qB);
		float angular;
		s2Vec2 linear = s2cGearReaction(&angular, imp.x, j.lim[i].x, side2);
		imp = make_float4(linear.x, linear.y, 0.0f, 0.0f);
		motorImpulse = angular;
		limp = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
	}
	s2JointReaction r = s2MakeJointReaction(type, s2MakeVec2(imp.x, imp.y), motorImpulse, limp.x, limp.y, qA, axis, rate);
	if (reactions != nullptr)
	{
		reactions[3 * i] = r.force.x;
		reactions[3 * i + 1] = r.force.y;
		reactions[3 * i + 2] = r.torque;
	}
	if (broken != nullptr)
	{
		// strict comparisons, each only where its threshold is set
		float force = sqrtf(r.force.x * r.force.x + r.force.y * r.force.y);
		if ((thresholds.x > 0.0f && force > thresholds.x) || (thresholds.y > 0.0f && fabsf(r.torque) > thresholds.y))
		{
			broken[1 + atomicAdd(broken, 1)] = i;
		}
	}
}

void s2bJointBreakPass(s2bWorld* w, cudaStream_t cs)
{
	cudaStream_t st = w->stream;
	int cap = w->jointCap;
	if (w->brokenEvent == nullptr)
	{
		S2B_CHECK(cudaEventCreateWithFlags(&w->brokenEvent, cudaEventDisableTiming));
	}
	if (w->hostBrokenCap < cap + 1)
	{
		// the previous step's copy may still be writing the old buffer
		S2B_CHECK(cudaEventSynchronize(w->brokenEvent));
		if (w->hostBroken != nullptr)
		{
			S2B_CHECK(cudaFreeHost(w->hostBroken));
		}
		S2B_CHECK(cudaMallocHost((void**)&w->hostBroken, sizeof(int) * (size_t)(cap + 1)));
		w->hostBrokenCap = cap + 1;
	}
	{
		S2bEpochFreeze freeze; // the list is written outside the captured solver graph
		w->dBroken.reserve((size_t)cap + 1, st, false, false);
	}
	S2B_CHECK(cudaMemsetAsync(w->dBroken.p, 0, sizeof(int), st));
	S2B_LAUNCH(w, s2bJointReactionKernel, gridFor(cap, 128), 128, 0, jointView(w), w->jBreak.p, w->bPose.p, w->bPos.p, w->bOrg.p,
			   w->reactionRate, (float*)nullptr, w->dBroken.p);
	if (cs != st)
	{
		S2B_CHECK(cudaEventRecord(w->finalizedEvent, st));
		S2B_CHECK(cudaStreamWaitEvent(cs, w->finalizedEvent, 0));
	}
	S2B_CHECK(cudaMemcpyAsync(w->hostBroken, w->dBroken.p, sizeof(int) * (size_t)(cap + 1), cudaMemcpyDeviceToHost, cs));
	S2B_CHECK(cudaEventRecord(w->brokenEvent, cs));
	w->brokenPending = true;
	w->jointsChecked = w->breakCount;
}

extern "C" void s2b_download_joint_reactions(s2bWorld* w, float* out, int capacity)
{
	S2B_CHECK(cudaSetDevice(w->device));
	int n = capacity < w->jointCap ? capacity : w->jointCap;
	for (int i = n > 0 ? 3 * n : 0; i < 3 * capacity; ++i)
	{
		out[i] = 0.0f; // slots past the device's capacity have never held a joint
	}
	if (n <= 0)
	{
		return;
	}
	S2bEpochFreeze freeze; // transfer buffers are not part of any captured graph
	float* d = nullptr;
	S2B_CHECK(cudaMallocAsync((void**)&d, sizeof(float) * 3 * (size_t)w->jointCap, w->stream));
	S2B_LAUNCH(w, s2bJointReactionKernel, gridFor(w->jointCap, 128), 128, 0, jointView(w), w->jBreak.p, w->bPose.p, w->bPos.p,
			   w->bOrg.p, w->reactionRate, d, (int*)nullptr);
	S2B_CHECK(cudaMemcpyAsync(out, d, sizeof(float) * 3 * (size_t)n, cudaMemcpyDeviceToHost, w->stream));
	S2B_CHECK(cudaFreeAsync(d, w->stream));
	S2B_CHECK(cudaStreamSynchronize(w->stream));
}

extern "C" int s2b_download_broken_joints(s2bWorld* w, int32_t* slots, int capacity)
{
	S2B_CHECK(cudaSetDevice(w->device));
	if (w->brokenPending == false)
	{
		return 0;
	}
	// waits for the copy behind the last finalize's pass only, not for the pair search queued after it
	S2B_CHECK(cudaEventSynchronize(w->brokenEvent));
	int count = w->hostBroken[0];
	// the device appends in whatever order its threads arrive: the list is handed out in slot order
	std::sort(w->hostBroken + 1, w->hostBroken + 1 + count);
	for (int k = 0; k < count && k < capacity; ++k)
	{
		slots[k] = w->hostBroken[1 + k];
	}
	return count;
}
