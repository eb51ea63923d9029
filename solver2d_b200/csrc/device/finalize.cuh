// solver2d-b200 — one shape's box and fat-box move at its body's final pose (stage 4 of s2World_Step). Shared by finalize's
// kernels (finalize.cu) and by the finalize that refits the pair search's hierarchy on the way (broadphase.cu).
#pragma once

#include "s2b_internal.cuh"

// All four shape kinds are stored in polygon form (count vertices + radius), for which the per-kind AABB functions of
// the reference (src/geometry.c:288-341) reduce to the same float operations: min/max over the transformed
// vertices, then -/+ radius.
//
// Once finalize has run, the bullet pass (DESIGN.md §3.12) redoes a clamped bullet's shapes with `again`: a shape that is
// already flagged MOVED is not counted a second time.
//
// `head` is the shape's header as read; it comes back as written (MOVED set when the proxy escaped its fat box), and the
// shape's fat box is returned.
template <bool again> __device__ __forceinline__ float4 s2bFinalizeShape(const ShapeView& s, const BodyView& b, int i, int4& head,
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
		fat4 = make_float4(aabb.lowerBound.x - s2_aabbMargin, aabb.lowerBound.y - s2_aabbMargin, aabb.upperBound.x + s2_aabbMargin,
						   aabb.upperBound.y + s2_aabbMargin);
		s.fat[i] = fat4;
		int4 moved = make_int4(head.x | S2B_SHAPE_MOVED, head.y, head.z, head.w);
		s.head[i] = moved;
		if (again == false || (head.x & S2B_SHAPE_MOVED) == 0)
		{
			atomicAdd(movedCounter, 1);
		}
		head = moved;
	}
	return fat4;
}
