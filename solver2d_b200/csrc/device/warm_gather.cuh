// solver2d-b200 — warm starting as a per-body GATHER fused with s2IntegrateVelocities.
//
// The sub-stepping variants warm start every sub-step (reference src/solve_tgs_soft.c:217-233,
// src/solve_soft_step.c:246-262, src/solve_tgs_ngs.c:270-286). Run constraint by constraint that costs one grid
// barrier per colour. But a warm start only ADDS terms to v and w that do not depend on v and w themselves:
//     contact:  P = ln * n + lt * t ;  w -/+= invI * cross(r, P) ;  v = v -/+ invM * P        (r from the rotation, which
//     joint:    P = impulse        ;  w -/+= invI * (cross(r, P) + axial) ;  v = v -/+ invM * P   no warm start changes)
// so each body can collect its own terms. Float addition is not associative, therefore the terms are added in exactly
// the order the constraint-by-constraint pass would have produced them: the incidence list of every movable body is
// sorted by position in the solve order (group-major; joints before contacts inside a group; serial order inside
// the overflow group). The result is bit-identical to the grouped pass, with no barrier between colours and the
// integrate-velocities body pass folded in.
#pragma once

#include "joint_kernels.cuh"

// incidence entry: (t << 2) | (side << 1) | isContact — t = position in the contact / joint constraint stream
#define S2B_INC_CONTACT 1
#define S2B_INC_SIDE_B 2
// bodies with more incident constraints than this are gathered by a whole block instead of one thread
#define S2B_HEAVY_DEGREE 48

// the terms one incidence entry contributes to its body: (tw0, tv0) of point 0 / the joint, (tw1, tv1) of point 1
struct GatherTerms
{
	int np;
	float tw0, tw1;
	s2Vec2 tv0, tv1;
};

// anchorRow: this side's anchors when the caller holds them (a block's shared-memory copy); null = warmAnchor
template <bool FIXED>
__device__ __forceinline__ GatherTerms s2bGatherTermsOf(const SolveArgs& a, int e, s2Rot q, float invMass, float invI,
														const float4* anchorRow = nullptr)
{
	GatherTerms g;
	g.np = 0;
	g.tw0 = g.tw1 = 0.0f;
	g.tv0 = g.tv1 = V2(0.0f, 0.0f);
	int t = e >> 2;
	bool sideB = (e & S2B_INC_SIDE_B) != 0;
	if (e & S2B_INC_CONTACT)
	{
		// two 16-byte rows: the impulse vectors of both points, this side's anchors (contact_kernels.cuh, s2bWriteWarm*)
		float4 imp = a.cc.warmP[t];
		float4 anchors = anchorRow != nullptr ? *anchorRow : a.cc.warmAnchor[(size_t)t * 2 + (sideB ? 1 : 0)];
		g.np = imp.z == imp.z ? 2 : 1;
#pragma unroll
		for (int j = 0; j < 2; ++j)
		{
			if (j < g.np)
			{
				s2Vec2 local = j == 0 ? V2(anchors.x, anchors.y) : V2(anchors.z, anchors.w);
				s2Vec2 r = FIXED ? local : s2RotateVector(q, local);
				s2Vec2 P = j == 0 ? V2(imp.x, imp.y) : V2(imp.z, imp.w);
				float c = invI * s2Cross(r, P);
				float tw = sideB ? c : -c;
				s2Vec2 tv = s2MulSV(sideB ? invMass : -invMass, P);
				if (j == 0)
				{
					g.tw0 = tw;
					g.tv0 = tv;
				}
				else
				{
					g.tw1 = tw;
					g.tv1 = tv;
				}
			}
		}
	}
	else
	{
		int4 head = a.jc.head[t];
		float4 anchor = a.jc.anchor[t];
		float4 imp = a.jc.imp[t];
		s2Vec2 P = V2(imp.x, imp.y);
		g.np = 1;
		if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_MOUSE)
		{
			s2Vec2 rB = s2RotateVector(q, V2(anchor.z, anchor.w));
			g.tv0 = s2MulSV(invMass, P);
			g.tw0 = invI * (s2Cross(rB, P) + imp.z);
		}
		else if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_PRISMATIC)
		{
			// P and L depend on both poses (DESIGN.md §3.9); poses are not written during the gather
			PrismaticWarm pw = s2bPrismaticWarmTerms(a, t);
			s2Vec2 mp = s2MulSV(invMass, pw.P);
			g.tv0 = sideB ? mp : V2(-mp.x, -mp.y);
			g.tw0 = sideB ? invI * pw.LB : -(invI * pw.LA);
		}
		else
		{
			float4 limp = a.jc.limp[t];
			float axialImpulse = imp.z + limp.x - limp.y;
			if (sideB)
			{
				s2Vec2 rB = s2RotateVector(q, V2(anchor.z, anchor.w));
				g.tv0 = s2MulSV(invMass, P);
				g.tw0 = invI * (s2Cross(rB, P) + axialImpulse);
			}
			else
			{
				s2Vec2 rA = s2RotateVector(q, V2(anchor.x, anchor.y));
				s2Vec2 mp = s2MulSV(invMass, P);
				g.tv0 = V2(-mp.x, -mp.y);
				g.tw0 = -(invI * (s2Cross(rA, P) + axialImpulse));
			}
		}
	}
	return g;
}

// what the gather needs of a body before it can look at its incidence list: loaded in one go (and, in the grid-stride loop
// of the body pass, one body AHEAD: the next body's first round trip overlaps this body's dependent chain)
struct GatherHead
{
	unsigned f;
	float4 vel, prm, frc, pose;
	int begin, end;
};

__device__ __forceinline__ GatherHead s2bLoadGatherHead(const SolveArgs& a, int i)
{
	GatherHead hd;
	hd.f = a.bodies.flags[i];
	hd.vel = a.bodies.vel[i];
	hd.prm = a.bodies.prm[i];
	hd.frc = a.bodies.frc[i];
	hd.pose = a.bodies.pose[i];
	hd.begin = a.incStart[i];
	hd.end = a.incStart[i + 1];
	return hd;
}

// four incidence entries: their (independent) load chains — entry -> constraint row — in flight together, then added to
// v, w in list order (same float operations, same order as the constraint-by-constraint pass, and the same code as the
// block-wide hub gather below)
template <bool FIXED>
__device__ __forceinline__ void s2bGatherFour(const SolveArgs& a, const int (&e)[4], s2Rot q, float invMass, float invI, s2Vec2& v, float& w,
											  const float4* anchors = nullptr)
{
	GatherTerms g[4];
#pragma unroll
	for (int u = 0; u < 4; ++u)
	{
		g[u].np = 0;
		g[u].tw0 = g[u].tw1 = 0.0f;
		g[u].tv0 = g[u].tv1 = V2(0.0f, 0.0f);
		if (e[u] != -1)
		{
			g[u] = s2bGatherTermsOf<FIXED>(a, e[u], q, invMass, invI, anchors != nullptr ? anchors + u : nullptr);
		}
	}
#pragma unroll
	for (int u = 0; u < 4; ++u)
	{
		if (g[u].np >= 1)
		{
			w = w + g[u].tw0;
			v = V2(v.x + g[u].tv0.x, v.y + g[u].tv0.y);
		}
		if (g[u].np == 2)
		{
			w = w + g[u].tw1;
			v = V2(v.x + g[u].tv1.x, v.y + g[u].tv1.y);
		}
	}
}

// FIXED = false: anchors rotated by the current rotation (s2WarmStartContacts, reference src/solve_common.c:276-326)
// FIXED = true : prepare-time anchors (s2WarmStartContacts_Fixed, reference src/solve_soft_step.c:16-63)
// alsoPosition: the bias sweep integrates the positions of the bodies it touches (ConstraintView::lastTouch); a body
// without any constraint is touched by nobody, so its position is integrated here, right after its velocity (nothing in
// between changes either). Only where this pass still runs beside the folded position integration: when a constraint reads
// a kinematic body (persistent.cuh, S2bLaunchInfo::firstTouch); otherwise the finalize pass sub-steps such bodies.
// velOut: where the new velocity goes (the region's shared-memory copy in a resident launch); null = the body's row
// list, listAnchors: where hd.begin / hd.end point, the entries and their side's anchors (a block's shared-memory copy of its
// first-touched bodies' lists); null = incList, warmAnchor
template <bool FIXED>
__device__ __forceinline__ void s2bIntegrateVelocityWarmHead(const SolveArgs& a, int i, float h, const GatherHead& hd, bool alsoPosition = false,
															 float4* velOut = nullptr, const int* list = nullptr,
															 const float4* listAnchors = nullptr)
{
	const int* inc = list != nullptr ? list : a.incList;
	float4* out = velOut != nullptr ? velOut : a.bodies.vel + i;
	unsigned f = hd.f;
	if ((f & S2B_BODY_VALID) == 0)
	{
		return;
	}
	float4 vel = hd.vel;
	float4 prm = hd.prm;
	float invMass = vel.w, invI = prm.w;
	s2Vec2 v = V2(vel.x, vel.y);
	float w = vel.z;
	bool dynamic = S2B_BODY_TYPE(f) == S2B_BODY_DYNAMIC;

	// s2IntegrateVelocities (reference src/solve_common.c:10-45)
	if (dynamic)
	{
		float4 frc = hd.frc;
		s2Vec2 gravity = V2(a.gravity.x, a.gravity.y);
		v = s2Add(v, s2MulSV(h * invMass, s2MulAdd(V2(frc.x, frc.y), frc.w * prm.z, gravity)));
		w = w + h * invI * frc.z;
		v = s2MulSV(1.0f / (1.0f + h * prm.x), v);
		w *= 1.0f / (1.0f + h * prm.y);
	}

	int begin = hd.begin, end = hd.end;
	if (begin == end)
	{
		if (dynamic)
		{
			*out = make_float4(v.x, v.y, w, invMass);
		}
		if (alsoPosition && S2B_BODY_TYPE(f) != S2B_BODY_STATIC)
		{
			// s2IntegratePositions (reference src/solve_common.c:47-68)
			s2Vec2 dp = s2MulAdd(V2(hd.pose.x, hd.pose.y), h, v);
			s2Rot qn = s2IntegrateRot(R2(hd.pose.z, hd.pose.w), h * w);
			a.bodies.pose[i] = make_float4(dp.x, dp.y, qn.s, qn.c);
		}
		return;
	}
	if (a.heavyBodies != nullptr && end - begin > S2B_HEAVY_DEGREE)
	{
		return; // a hub body (container wall ...): gathered by a whole block, s2bGatherHeavyBodies
	}

	s2Rot q = R2(hd.pose.z, hd.pose.w);
	// the first eight entries of the list in one round trip (a box in a pile has six neighbours), then four at a time
	int e0[4], e1[4];
#pragma unroll
	for (int u = 0; u < 4; ++u)
	{
		e0[u] = begin + u < end ? inc[begin + u] : -1;
		e1[u] = begin + 4 + u < end ? inc[begin + 4 + u] : -1;
	}
	s2bGatherFour<FIXED>(a, e0, q, invMass, invI, v, w, listAnchors != nullptr ? listAnchors + begin : nullptr);
	if (end - begin > 4)
	{
		s2bGatherFour<FIXED>(a, e1, q, invMass, invI, v, w, listAnchors != nullptr ? listAnchors + begin + 4 : nullptr);
	}
	for (int k0 = begin + 8; k0 < end; k0 += 4)
	{
		int e[4];
#pragma unroll
		for (int u = 0; u < 4; ++u)
		{
			e[u] = k0 + u < end ? inc[k0 + u] : -1;
		}
		s2bGatherFour<FIXED>(a, e, q, invMass, invI, v, w, listAnchors != nullptr ? listAnchors + k0 : nullptr);
	}
	*out = make_float4(v.x, v.y, w, invMass);
}

template <bool FIXED> __device__ __forceinline__ void s2bIntegrateVelocityWarm(const SolveArgs& a, int i, float h)
{
	s2bIntegrateVelocityWarmHead<FIXED>(a, i, h, s2bLoadGatherHead(a, i));
}

// ---- first-touch warm start (TGS_Soft, persistent.cuh) -----------------------------------------------------------------
// The warm start of a body reads its own row, its rotation and the warm rows of its constraints. Between the end of a
// sub-step's last sweep and the body's FIRST constraint in the next bias sweep none of them changes, so the thread that
// solves that constraint runs the gather of the body right before the solve (S2B_TOUCH_FIRST_* marks), with the same
// operations in the same order as the body pass, instead of a device-wide body pass before the sweep.

// before the colour step's wait: the read-only part of the marked bodies' heads into L2 (an L1 prefetch would be lost: the
// acquire of the wait invalidates L1)
__device__ __forceinline__ void s2bPrefetchL2(const void* ptr)
{
	asm volatile("prefetch.global.L2 [%0];" ::"l"(ptr));
}

__device__ __forceinline__ void s2bFirstTouchPrefetch(const SolveArgs& a, int i)
{
	s2bPrefetchL2(a.bodies.flags + i);
	s2bPrefetchL2(a.bodies.prm + i);
	s2bPrefetchL2(a.bodies.frc + i);
	s2bPrefetchL2(a.incStart + i);
}

// after the wait, before the solve: s2IntegrateVelocities + the gathered warm start of the marked bodies, one after the other
// (one inlined copy of the gather; two heads held at once spilled)
__device__ __forceinline__ void s2bFirstTouchWarm(const SolveArgs& a, int2 idx, int marks)
{
#pragma unroll 1
	for (int side = 0; side < 2; ++side)
	{
		if (marks & (side == 0 ? S2B_TOUCH_FIRST_A : S2B_TOUCH_FIRST_B))
		{
			int i = side == 0 ? idx.x : idx.y & S2B_CF_INDEX_MASK;
			s2bIntegrateVelocityWarmHead<false>(a, i, a.ctx.h, s2bLoadGatherHead(a, i));
		}
	}
}

// A body no constraint touches, in a launch whose bias sweeps warm-start at the first touch: nothing in the launch reads it,
// so the finalize pass runs all its sub-steps at once — s2IntegrateVelocities, then s2IntegratePositions, `substeps` times:
// the operations the per-sub-step body passes applied to it, in their order.
__device__ __forceinline__ void s2bSubstepFreeBody(const SolveArgs& a, int i, float h, int substeps)
{
	unsigned f = a.bodies.flags[i];
	if ((f & S2B_BODY_VALID) == 0 || S2B_BODY_TYPE(f) == S2B_BODY_STATIC || a.incStart[i] != a.incStart[i + 1])
	{
		return;
	}
	for (int s = 0; s < substeps; ++s)
	{
		s2bIntegrateVelocityWarm<false>(a, i, h); // (an empty incidence list: the velocity part only)
		s2bIntegratePosition(a, i, h);
	}
}

// the body pass of the persistent kernel without regions: every body slot, grid-stride, the next body's head loaded ahead
template <bool FIXED> __device__ __forceinline__ void s2bIntegrateVelocityWarmAll(const SolveArgs& a, float h, bool alsoPosition = false)
{
	int stride = gridDim.x * blockDim.x;
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= a.bodies.capacity)
	{
		return;
	}
	GatherHead hd = s2bLoadGatherHead(a, i);
	for (; i < a.bodies.capacity; i += stride)
	{
		GatherHead next = hd;
		if (i + stride < a.bodies.capacity)
		{
			next = s2bLoadGatherHead(a, i + stride);
		}
		s2bIntegrateVelocityWarmHead<FIXED>(a, i, h, hd, alsoPosition);
		hd = next;
	}
}

// ---- hub bodies -----------------------------------------------------------------------------------------------------
// A container touching hundreds of boxes has hundreds of incident constraints; one thread walking them pays a dependent round trip per entry.
// The terms tw = -/+ invI * (cross(r, P) [+ axial]) and tv = (-/+ invM) * P do not involve v or w, so a whole block forms them
// in parallel (shared memory) and ONE thread then adds them to v, w in list order: the same float operations in the same
// order as the serial walk, hence the same bits.
// called by every block of the persistent kernel after the per-thread gather; block b takes hub bodies b, b + gridDim, ...
template <bool FIXED> __device__ __forceinline__ void s2bGatherHeavyBodies(const SolveArgs& a, float h)
{
	__shared__ float sTw0[S2B_BLOCK], sTw1[S2B_BLOCK], sX0[S2B_BLOCK], sY0[S2B_BLOCK], sX1[S2B_BLOCK], sY1[S2B_BLOCK];
	__shared__ int sNp[S2B_BLOCK];
	int heavy = a.heavyBodies[0];
	for (int hb = blockIdx.x; hb < heavy; hb += gridDim.x)
	{
		int i = a.heavyBodies[1 + hb];
		unsigned f = a.bodies.flags[i];
		float4 vel = a.bodies.vel[i];
		float4 prm = a.bodies.prm[i];
		float invMass = vel.w, invI = prm.w;
		s2Vec2 v = V2(vel.x, vel.y);
		float w = vel.z;
		if (S2B_BODY_TYPE(f) == S2B_BODY_DYNAMIC)
		{
			// s2IntegrateVelocities (reference src/solve_common.c:10-45), computed redundantly by every thread
			float4 frc = a.bodies.frc[i];
			s2Vec2 gravity = V2(a.gravity.x, a.gravity.y);
			v = s2Add(v, s2MulSV(h * invMass, s2MulAdd(V2(frc.x, frc.y), frc.w * prm.z, gravity)));
			w = w + h * invI * frc.z;
			v = s2MulSV(1.0f / (1.0f + h * prm.x), v);
			w *= 1.0f / (1.0f + h * prm.y);
		}
		float4 pose = a.bodies.pose[i];
		s2Rot q = R2(pose.z, pose.w);
		int begin = a.incStart[i], end = a.incStart[i + 1];
		for (int k0 = begin; k0 < end; k0 += blockDim.x)
		{
			int k = k0 + threadIdx.x;
			GatherTerms g;
			g.np = 0;
			g.tw0 = g.tw1 = 0.0f;
			g.tv0 = g.tv1 = V2(0.0f, 0.0f);
			if (k < end)
			{
				g = s2bGatherTermsOf<FIXED>(a, a.incList[k], q, invMass, invI);
			}
			sNp[threadIdx.x] = g.np;
			sTw0[threadIdx.x] = g.tw0;
			sTw1[threadIdx.x] = g.tw1;
			sX0[threadIdx.x] = g.tv0.x;
			sY0[threadIdx.x] = g.tv0.y;
			sX1[threadIdx.x] = g.tv1.x;
			sY1[threadIdx.x] = g.tv1.y;
			__syncthreads();
			if (threadIdx.x == 0)
			{
				int count = min((int)blockDim.x, end - k0);
				for (int u = 0; u < count; ++u)
				{
					int np = sNp[u];
					if (np >= 1)
					{
						w = w + sTw0[u];
						v = V2(v.x + sX0[u], v.y + sY0[u]);
					}
					if (np == 2)
					{
						w = w + sTw1[u];
						v = V2(v.x + sX1[u], v.y + sY1[u]);
					}
				}
			}
			__syncthreads();
		}
		if (threadIdx.x == 0)
		{
			a.bodies.vel[i] = make_float4(v.x, v.y, w, invMass);
		}
	}
}
