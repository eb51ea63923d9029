// solver2d-b200 — per-body and per-contact-constraint device functions of the solver stage.
//
// One thread owns one constraint (both manifold points are solved sequentially by that thread, as the points of a
// manifold are coupled through the two bodies). Within a group (colour / wavefront level) no two constraints share a
// movable body, so the read-modify-write of the body velocity columns is race-free without atomics.
//
// Float expressions follow the reference op for op (compiled with -fmad=false), see the citations on each function.
#pragma once

#include "solver_state.cuh"

__device__ __forceinline__ s2Vec2 V2(float x, float y)
{
	s2Vec2 v = {x, y};
	return v;
}

__device__ __forceinline__ s2Rot R2(float s, float c)
{
	s2Rot q = {s, c};
	return q;
}

// ---------------------------------------------------------------------------------------------------------------
// body phases
// ---------------------------------------------------------------------------------------------------------------

// s2IntegrateVelocities (reference src/solve_common.c:10-45): dynamic bodies only; gravity, forces, implicit damping.
// Algorithmic traffic: read vel, frc, prm (48 B) + flag, write vel (16 B).
__device__ __forceinline__ void s2bIntegrateVelocity(const SolveArgs& a, int i, float h)
{
	unsigned f = a.bodies.flags[i];
	if ((f & S2B_BODY_VALID) == 0 || S2B_BODY_TYPE(f) != S2B_BODY_DYNAMIC)
	{
		return;
	}
	float4 vel = a.bodies.vel[i];
	float4 frc = a.bodies.frc[i];
	float4 prm = a.bodies.prm[i];
	float invMass = vel.w, invI = prm.w, mass = frc.w;
	s2Vec2 v = V2(vel.x, vel.y);
	float w = vel.z;
	s2Vec2 gravity = V2(a.gravity.x, a.gravity.y);

	v = s2Add(v, s2MulSV(h * invMass, s2MulAdd(V2(frc.x, frc.y), mass * prm.z, gravity)));
	w = w + h * invI * frc.z;

	v = s2MulSV(1.0f / (1.0f + h * prm.x), v);
	w *= 1.0f / (1.0f + h * prm.y);

	a.bodies.vel[i] = make_float4(v.x, v.y, w, invMass);
}

// s2IntegratePositions (reference src/solve_common.c:47-68): every non-static body (kinematic bodies move too).
__device__ __forceinline__ void s2bIntegratePosition(const SolveArgs& a, int i, float h)
{
	unsigned f = a.bodies.flags[i];
	if ((f & S2B_BODY_VALID) == 0 || S2B_BODY_TYPE(f) == S2B_BODY_STATIC)
	{
		return;
	}
	float4 vel = a.bodies.vel[i];
	float4 pose = a.bodies.pose[i];
	s2Vec2 dp = s2MulAdd(V2(pose.x, pose.y), h, V2(vel.x, vel.y));
	s2Rot q = s2IntegrateRot(R2(pose.z, pose.w), h * vel.z);
	a.bodies.pose[i] = make_float4(dp.x, dp.y, q.s, q.c);
}

// s2FinalizePositions (reference src/solve_common.c:70-91)
__device__ __forceinline__ void s2bFinalizePosition(const SolveArgs& a, int i)
{
	unsigned f = a.bodies.flags[i];
	if ((f & S2B_BODY_VALID) == 0 || S2B_BODY_TYPE(f) == S2B_BODY_STATIC)
	{
		return;
	}
	float4 pos = a.bodies.pos[i];
	float4 pose = a.bodies.pose[i];
	s2Vec2 p = s2Add(V2(pos.x, pos.y), V2(pose.x, pose.y));
	a.bodies.pos[i] = make_float4(p.x, p.y, pos.z, pos.w);
	a.bodies.pose[i] = make_float4(0.0f, 0.0f, pose.z, pose.w);
}

// ---------------------------------------------------------------------------------------------------------------
// The warm-start rows of one constraint (ConstraintView::warmP / warmAnchor, read by the per-body gather).
// s2bWriteWarmImpulses: by whichever pass leaves the impulses the next gather applies — prepare, and the last solve /
// relax pass of a sub-step. s2bWriteWarmAnchors: by prepare; anchors[j] = side A anchor in .xy, side B in .zw.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void s2bWriteWarmImpulses(const SolveArgs& a, int t, s2Vec2 normal, s2Vec2 tangent, int pointCount, float2 lam0,
													 float2 lam1)
{
	s2Vec2 P0 = s2Add(s2MulSV(lam0.x, normal), s2MulSV(lam0.y, tangent));
	s2Vec2 P1 = s2Add(s2MulSV(lam1.x, normal), s2MulSV(lam1.y, tangent));
	if (pointCount != 2)
	{
		P1.x = __int_as_float(0x7FC00000); // NaN: no second point
	}
	a.cc.warmP[t] = make_float4(P0.x, P0.y, P1.x, P1.y);
}

__device__ __forceinline__ void s2bWriteWarmAnchors(const SolveArgs& a, int t, float4 anchors0, float4 anchors1)
{
	a.cc.warmAnchor[(size_t)t * 2] = make_float4(anchors0.x, anchors0.y, anchors1.x, anchors1.y);
	a.cc.warmAnchor[(size_t)t * 2 + 1] = make_float4(anchors0.z, anchors0.w, anchors1.z, anchors1.w);
}

// ---------------------------------------------------------------------------------------------------------------
// contact constraints: prepare
// ---------------------------------------------------------------------------------------------------------------

enum PrepareKind
{
	PREPARE_PGS = 0,  // s2PrepareContacts_PGS  (reference src/solve_common.c:93-168)
	PREPARE_SOFT = 1, // s2PrepareContacts_Soft (reference src/solve_common.c:188-274)
	PREPARE_COLD = 2, // s2PrepareContacts_XPBD (reference src/solve_xpbd.c:18-86): never warm starts
};

// The points of a manifold in the contact table: its local anchors and separation + stored impulses, read where used.
struct S2bTablePoints
{
	const ContactView& c;
	int slot;
	__device__ __forceinline__ float4 anchor(int j) const
	{
		return c.anchor[j][slot];
	}
	__device__ __forceinline__ float4 impulse(int j) const
	{
		return c.impulse[j][slot];
	}
};

// Writes row t of the constraint stream from one manifold and its two bodies: the manifold's normal / friction (mnf), its
// points (POINTS::anchor(j) / impulse(j) = the table's anchor[j] / impulse[j] columns, asked for j < pointCount only), and
// per body the local centre (org.zw), the rotation (pose.zw), the inverse mass (vel.w) and the inverse inertia (prm.w).
// Writes are coalesced (row t). Called by the solver's prepare pass, which gathers these values through src[t], and by the
// narrow phase, which has them in registers when the solve schedule stands (narrowphase.cu): the row format lives here only.
template <int KIND, typename POINTS>
__device__ __forceinline__ void s2bWriteContactRow(const SolveArgs& a, int t, int2 bodies, int pointCount, float4 mnf, const POINTS& points,
												   float4 orgA, float4 orgB, float4 poseA, float4 poseB, float mA, float mB, float iA, float iB)
{
	const ConstraintView& cc = a.cc;
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	s2Vec2 normal = V2(mnf.x, mnf.y);
	s2Vec2 tangent = s2RightPerp(normal);
	bool warmStart = KIND == PREPARE_COLD ? false : a.ctx.warmStart != 0;

	// contact stiffness is doubled against a body of infinite mass (reference solve_common.c:219)
	unsigned flags = 0;
	if (mA == 0.0f || mB == 0.0f)
	{
		flags |= S2B_CF_STATIC_SOFT;
	}
	if (pointCount == 2)
	{
		flags |= S2B_CF_TWO_POINTS;
	}
	int rowA = bodies.x, rowB = bodies.y;
	if (a.bodyLocal != nullptr && a.counts[CNT_RESIDENT] != 0)
	{
		// resident regions: the sweeps address the bodies through the region's shared-memory copy
		rowA = (mA != 0.0f || iA != 0.0f) ? a.bodyLocal[rowA] : (rowA | S2B_RES_GLOBAL);
		rowB = (mB != 0.0f || iB != 0.0f) ? a.bodyLocal[rowB] : (rowB | S2B_RES_GLOBAL);
	}
	cc.idx[t] = make_int2(rowA, (int)((unsigned)rowB | flags));
	cc.nf[t] = make_float4(normal.x, normal.y, mnf.z, iA);
	float2 warmLam[2] = {make_float2(0.0f, 0.0f), make_float2(0.0f, 0.0f)};
	float4 warmAnchor[2] = {make_float4(0.0f, 0.0f, 0.0f, 0.0f), make_float4(0.0f, 0.0f, 0.0f, 0.0f)};

#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < pointCount)
		{
			float4 la = points.anchor(j);
			float4 mi = points.impulse(j);
			float separation = mi.x;
			// PGS prepare tests cp->separation <= 0 on the zero-filled scratch, i.e. always true (SURVEY §8a N1), so
			// both prepare flavours take the stored impulses whenever warm starting is on.
			float normalImpulse = warmStart ? mi.y : 0.0f;
			float tangentImpulse = warmStart ? mi.z : 0.0f;

			s2Vec2 lA = s2Sub(V2(la.x, la.y), V2(orgA.z, orgA.w));
			s2Vec2 lB = s2Sub(V2(la.z, la.w), V2(orgB.z, orgB.w));
			s2Vec2 rA = s2RotateVector(qA, lA);
			s2Vec2 rB = s2RotateVector(qB, lB);

			float adjustedSeparation = separation - s2Dot(s2Sub(rB, rA), normal);

			float rnA = s2Cross(rA, normal);
			float rnB = s2Cross(rB, normal);
			float kNormal = mA + mB + iA * rnA * rnA + iB * rnB * rnB;
			float normalMass = kNormal > 0.0f ? 1.0f / kNormal : 0.0f;

			float rtA = s2Cross(rA, tangent);
			float rtB = s2Cross(rB, tangent);
			float kTangent = mA + mB + iA * rtA * rtA + iB * rtB * rtB;
			float tangentMass = kTangent > 0.0f ? 1.0f / kTangent : 0.0f;

			cc.anchor[j][t] = make_float4(lA.x, lA.y, lB.x, lB.y);
			cc.pm[j][t] = make_float4(adjustedSeparation, normalMass, tangentMass, j == 0 ? iB : 0.0f);
			cc.lambda[j][t] = make_float2(normalImpulse, tangentImpulse);
			warmLam[j] = make_float2(normalImpulse, tangentImpulse);
			// SoftStep warm starts at the prepare-time world anchors (reference src/solve_soft_step.c:16-63)
			warmAnchor[j] = a.solverType == 5 ? make_float4(rA.x, rA.y, rB.x, rB.y) : make_float4(lA.x, lA.y, lB.x, lB.y);
			if (cc.r0[j] != nullptr)
			{
				cc.r0[j][t] = make_float4(rA.x, rA.y, rB.x, rB.y);
			}
			if (cc.sep[j] != nullptr)
			{
				cc.sep[j][t] = separation;
			}
		}
		else
		{
			cc.anchor[j][t] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
			cc.pm[j][t] = make_float4(0.0f, 0.0f, 0.0f, j == 0 ? iB : 0.0f);
			cc.lambda[j][t] = make_float2(0.0f, 0.0f);
			if (cc.r0[j] != nullptr)
			{
				cc.r0[j][t] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
			}
			if (cc.sep[j] != nullptr)
			{
				cc.sep[j][t] = 0.0f;
			}
		}
	}
	if (cc.warmP != nullptr)
	{
		s2bWriteWarmImpulses(a, t, normal, tangent, pointCount, warmLam[0], warmLam[1]);
		s2bWriteWarmAnchors(a, t, warmAnchor[0], warmAnchor[1]);
	}
}

// Builds row t of the constraint stream from contact slot src[t]: gathers the persistent manifold and the two bodies.
// Skipped on the steps whose rows the narrow phase has already written (CNT_ROWS_READY, persistent.cuh).
template <int KIND> __device__ __forceinline__ void s2bPrepareContact(const SolveArgs& a, int t)
{
	int slot = a.cc.src[t];
	int2 bodies = a.contacts.bodies[slot];
	int4 info = a.contacts.info[slot];
	float4 mnf = a.contacts.nf[slot];
	int pointCount = S2B_CI_COUNT(info.x);

	float4 velA = a.bodies.vel[bodies.x], velB = a.bodies.vel[bodies.y];
	float4 poseA = a.bodies.pose[bodies.x], poseB = a.bodies.pose[bodies.y];
	float4 orgA = a.bodies.org[bodies.x], orgB = a.bodies.org[bodies.y];
	float iA = a.bodies.prm[bodies.x].w, iB = a.bodies.prm[bodies.y].w;
	S2bTablePoints points = {a.contacts, slot};
	s2bWriteContactRow<KIND>(a, t, bodies, pointCount, mnf, points, orgA, orgB, poseA, poseB, velA.w, velB.w, iA, iB);
}

// s2StoreContactImpulses (reference src/solve_common.c:396-410): scatter accumulated impulses back to the manifolds.
__device__ __forceinline__ void s2bStoreContactImpulses(const SolveArgs& a, int t, float scale)
{
	const ConstraintView& cc = a.cc;
	int slot = cc.src[t];
	int pointCount = (cc.idx[t].y & S2B_CF_TWO_POINTS) ? 2 : 1;
#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < pointCount)
		{
			float2 l = cc.lambda[j][t];
			float4 mi = a.contacts.impulse[j][slot];
			mi.y = scale == 1.0f ? l.x : l.x * scale;
			mi.z = scale == 1.0f ? l.y : l.y * scale;
			a.contacts.impulse[j][slot] = mi;
		}
	}
}

// ---------------------------------------------------------------------------------------------------------------
// contact constraints: shared load / store of the two bodies
// ---------------------------------------------------------------------------------------------------------------

struct BodyPair
{
	int ia, ib;
	float4 velA, velB;
	bool movA, movB;
};

__device__ __forceinline__ void s2bStoreVelocities(const SolveArgs& a, const BodyPair& bp, s2Vec2 vA, float wA, s2Vec2 vB,
												   float wB)
{
	// bodies of infinite mass and inertia (static, kinematic) are never written: the reference writes them back
	// unchanged (SURVEY §8a N7), and skipping the store keeps every group free of write conflicts on them.
	if (bp.movA)
	{
		a.bodies.vel[bp.ia] = make_float4(vA.x, vA.y, wA, bp.velA.w);
	}
	if (bp.movB)
	{
		a.bodies.vel[bp.ib] = make_float4(vB.x, vB.y, wB, bp.velB.w);
	}
}

// ---------------------------------------------------------------------------------------------------------------
// restitution
// ---------------------------------------------------------------------------------------------------------------
// The restitution pass (an extension, DESIGN.md §3.7; the reference stores restitution and never applies it). Runs after
// the variant's whole program, once per contact constraint in the stage's solve order. A point bounces when its approach
// speed at the start of the stage, vr (SolveArgs::restVr), was faster than the threshold and it carries a normal impulse:
// the impulse that takes its current normal velocity to -e * vr is added, clamped so that the accumulated impulse stays
// >= 0, at the anchors captured with vr. Works on the manifold and the body columns directly (body slots from the contact
// table): by now every body is back in global memory and the constraint rows may address a region's shared copy.
__device__ __forceinline__ void s2bApplyRestitution(const SolveArgs& a, int t)
{
	int slot = a.cc.src[t];
	float4 mnf = a.contacts.nf[slot];
	float e = mnf.w;
	if (e == 0.0f)
	{
		return;
	}
	int2 bodies = a.contacts.bodies[slot];
	int pointCount = S2B_CI_COUNT(a.contacts.info[slot].x);
	float4 velA = a.bodies.vel[bodies.x], velB = a.bodies.vel[bodies.y];
	float mA = velA.w, mB = velB.w;
	float iA = a.bodies.prm[bodies.x].w, iB = a.bodies.prm[bodies.y].w;
	s2Vec2 vA = V2(velA.x, velA.y), vB = V2(velB.x, velB.y);
	float wA = velA.z, wB = velB.z;
	s2Vec2 normal = V2(mnf.x, mnf.y);
	float4 captured = a.restVr[slot];
	float vr[2] = {captured.x, captured.y};
	float normalMass[2] = {captured.z, captured.w};
	bool applied = false;

#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < pointCount)
		{
			float4 mi = a.contacts.impulse[j][slot];
			if (vr[j] > -a.restitutionThreshold || mi.y == 0.0f)
			{
				continue;
			}
			float4 r = a.restR[j][slot];
			s2Vec2 rA = V2(r.x, r.y), rB = V2(r.z, r.w);
			s2Vec2 vrB = s2Add(vB, s2CrossSV(wB, rB));
			s2Vec2 vrA = s2Add(vA, s2CrossSV(wA, rA));
			float vn = s2Dot(s2Sub(vrB, vrA), normal);
			float impulse = -normalMass[j] * (vn + e * vr[j]);
			float newImpulse = S2_MAX(mi.y + impulse, 0.0f);
			impulse = newImpulse - mi.y;
			mi.y = newImpulse;
			a.contacts.impulse[j][slot] = mi;
			s2Vec2 P = s2MulSV(impulse, normal);
			vA = s2MulSub(vA, mA, P);
			wA -= iA * s2Cross(rA, P);
			vB = s2MulAdd(vB, mB, P);
			wB += iB * s2Cross(rB, P);
			applied = true;
		}
	}

	if (applied)
	{
		BodyPair bp = {bodies.x, bodies.y, velA, velB, (mA != 0.0f) || (iA != 0.0f), (mB != 0.0f) || (iB != 0.0f)};
		s2bStoreVelocities(a, bp, vA, wA, vB, wB);
	}
}

// ---------------------------------------------------------------------------------------------------------------
// s2WarmStartContacts (reference src/solve_common.c:276-326): impulses applied at the current anchors.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void s2bWarmStartContact(const SolveArgs& a, int t)
{
	const ConstraintView& cc = a.cc;
	int2 idx = cc.idx[t];
	int ia = idx.x, ib = idx.y & S2B_CF_INDEX_MASK;
	int pointCount = (idx.y & S2B_CF_TWO_POINTS) ? 2 : 1;
	float4 nf = cc.nf[t];
	float4 velA = a.bodies.vel[ia], velB = a.bodies.vel[ib];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	float mA = velA.w, mB = velB.w, iA = nf.w, iB = cc.pm[0][t].w;
	s2Vec2 vA = V2(velA.x, velA.y), vB = V2(velB.x, velB.y);
	float wA = velA.z, wB = velB.z;
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	s2Vec2 normal = V2(nf.x, nf.y);
	s2Vec2 tangent = s2RightPerp(normal);

#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < pointCount)
		{
			float4 la = cc.anchor[j][t];
			float2 l = cc.lambda[j][t];
			s2Vec2 rA = s2RotateVector(qA, V2(la.x, la.y));
			s2Vec2 rB = s2RotateVector(qB, V2(la.z, la.w));
			s2Vec2 P = s2Add(s2MulSV(l.x, normal), s2MulSV(l.y, tangent));
			wA -= iA * s2Cross(rA, P);
			vA = s2MulAdd(vA, -mA, P);
			wB += iB * s2Cross(rB, P);
			vB = s2MulAdd(vB, mB, P);
		}
	}

	BodyPair bp = {ia, ib, velA, velB, (mA != 0.0f) || (iA != 0.0f), (mB != 0.0f) || (iB != 0.0f)};
	s2bStoreVelocities(a, bp, vA, wA, vB, wB);
}

// ---------------------------------------------------------------------------------------------------------------
// s2SolveContacts_TGS_Soft (reference src/solve_tgs_soft.c:17-135): THE inner kernel of the headline variant.
// Soft normal constraint evaluated at the current (sub-stepped) anchors, then Coulomb friction.
// Algorithmic traffic per 2-point constraint: stream idx 8 + nf 16 + 2 x (anchor 16 + pm 16 + lambda 8 r + 8 w)
// = 120 B, bodies 2 x (vel 16 + pose 16 r, vel 16 w) = 96 B.
// ---------------------------------------------------------------------------------------------------------------
// the constraint-stream part of a contact constraint: everything a solve pass reads that no other thread writes. Kept
// apart from the body loads so that a caller can stage it differently (the TMA bulk-copy variant of the colour kernel
// reads it from shared memory)
struct ContactStream
{
	int2 idx;
	float4 nf;
	float4 la0, la1, pm0, pm1;
	float2 l0, l1;
	int slot; // contact slot of the row (only loaded by the sweep that also stores the impulses to the manifold)
	int last; // ConstraintView::lastTouch marks (only loaded by a bias sweep that also integrates positions)
};

__device__ __forceinline__ ContactStream s2bLoadContactStream(const SolveArgs& a, int t, bool withSlot = false)
{
	const ConstraintView& cc = a.cc;
	ContactStream cs;
	cs.last = 0;
	cs.slot = withSlot ? cc.src[t] : -1;
	cs.idx = cc.idx[t];
	cs.nf = cc.nf[t];
	cs.la0 = cc.anchor[0][t];
	cs.pm0 = cc.pm[0][t];
	cs.l0 = cc.lambda[0][t];
	cs.la1 = cc.anchor[1][t];
	cs.pm1 = cc.pm[1][t];
	cs.l1 = cc.lambda[1][t];
	return cs;
}

// storeManifold: this is the last sweep of the step — the accumulated impulses also go to the persistent manifold
// (s2StoreContactImpulses, reference src/solve_common.c:396-410, folded into the sweep: the values are in registers here and
// a separate pass would cost a device-wide barrier plus a dependent slot -> manifold round trip per constraint).
// RES: resident regions — a.bodies.vel / .pose point at the region's shared-memory copy and the row's indices are positions
// in it, except indices flagged S2B_RES_GLOBAL, which are body slots of the global arrays gVel / gPose (immovable bodies).
template <bool RES = false>
__device__ __forceinline__ void s2bSolveContactTgsSoftStream(const SolveArgs& a, int t, const ContactStream& cs, float inv_h, bool useBias,
															 bool writeWarm = false, bool storeManifold = false, const float4* gVel = nullptr,
															 const float4* gPose = nullptr, float4* lVel = nullptr, float4* lPose = nullptr)
{
	// (RES: the region's copy is addressed through lVel / lPose, handed over as plain arguments)
	float4* velRows = RES ? lVel : a.bodies.vel;
	float4* poseRows = RES ? lPose : a.bodies.pose;
	const ConstraintView& cc = a.cc;
	int2 idx = cs.idx;
	int ia = idx.x, ib = idx.y & S2B_CF_INDEX_MASK;
	int pointCount = (idx.y & S2B_CF_TWO_POINTS) ? 2 : 1;
	const SoftCoef soft = ((unsigned)idx.y & S2B_CF_STATIC_SOFT) ? a.softStatic : a.softDynamic;

	float4 nf = cs.nf;
	float4 la0 = cs.la0, pm0 = cs.pm0;
	float2 l0 = cs.l0;
	float4 la1 = cs.la1, pm1 = cs.pm1;
	float2 l1 = cs.l1;

	float4 velA, velB, poseA, poseB;
	if (RES && (ia & S2B_RES_GLOBAL))
	{
		ia &= ~S2B_RES_GLOBAL;
		velA = gVel[ia];
		poseA = gPose[ia];
	}
	else
	{
		velA = velRows[ia];
		poseA = poseRows[ia];
	}
	if (RES && (ib & S2B_RES_GLOBAL))
	{
		ib &= ~S2B_RES_GLOBAL;
		velB = gVel[ib];
		poseB = gPose[ib];
	}
	else
	{
		velB = velRows[ib];
		poseB = poseRows[ib];
	}

	float mA = velA.w, mB = velB.w, iA = nf.w, iB = pm0.w;
	s2Vec2 vA = V2(velA.x, velA.y), vB = V2(velB.x, velB.y);
	float wA = velA.z, wB = velB.z;
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);

	s2Vec2 normal = V2(nf.x, nf.y);
	s2Vec2 tangent = s2RightPerp(normal);
	float friction = nf.z;

	float4 la[2] = {la0, la1};
	float4 pm[2] = {pm0, pm1};
	float2 lam[2] = {l0, l1};

	// non-penetration
#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < pointCount)
		{
			s2Vec2 rA = s2RotateVector(qA, V2(la[j].x, la[j].y));
			s2Vec2 rB = s2RotateVector(qB, V2(la[j].z, la[j].w));

			// separation at the current sub-step pose
			s2Vec2 ds = s2Add(s2Sub(dcB, dcA), s2Sub(rB, rA));
			float s = s2Dot(ds, normal) + pm[j].x;

			float bias = 0.0f;
			float massScale = 1.0f;
			float impulseScale = 0.0f;
			if (s > 0.0f)
			{
				// speculative: allow approach up to the gap
				bias = s * inv_h;
			}
			else if (useBias)
			{
				bias = S2_MAX(soft.bias * s, -s2_maxBaumgarteVelocity);
				massScale = soft.mass;
				impulseScale = soft.impulse;
			}

			s2Vec2 vrB = s2Add(vB, s2CrossSV(wB, rB));
			s2Vec2 vrA = s2Add(vA, s2CrossSV(wA, rA));
			float vn = s2Dot(s2Sub(vrB, vrA), normal);

			float impulse = -pm[j].y * massScale * (vn + bias) - impulseScale * lam[j].x;

			float newImpulse = S2_MAX(lam[j].x + impulse, 0.0f);
			impulse = newImpulse - lam[j].x;
			lam[j].x = newImpulse;

			s2Vec2 P = s2MulSV(impulse, normal);
			vA = s2MulSub(vA, mA, P);
			wA -= iA * s2Cross(rA, P);
			vB = s2MulAdd(vB, mB, P);
			wB += iB * s2Cross(rB, P);
		}
	}

	// friction
#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < pointCount)
		{
			s2Vec2 rA = s2RotateVector(qA, V2(la[j].x, la[j].y));
			s2Vec2 rB = s2RotateVector(qB, V2(la[j].z, la[j].w));

			s2Vec2 vrB = s2Add(vB, s2CrossSV(wB, rB));
			s2Vec2 vrA = s2Add(vA, s2CrossSV(wA, rA));
			float vt = s2Dot(s2Sub(vrB, vrA), tangent);

			float impulse = -pm[j].z * vt;

			float maxFriction = friction * lam[j].x;
			float newImpulse = S2_CLAMP(lam[j].y + impulse, -maxFriction, maxFriction);
			impulse = newImpulse - lam[j].y;
			lam[j].y = newImpulse;

			s2Vec2 P = s2MulSV(impulse, tangent);
			vA = s2MulSub(vA, mA, P);
			wA -= iA * s2Cross(rA, P);
			vB = s2MulAdd(vB, mB, P);
			wB += iB * s2Cross(rB, P);
		}
	}

	cc.lambda[0][t] = lam[0];
	if (pointCount == 2)
	{
		cc.lambda[1][t] = lam[1];
	}
	if (writeWarm && cc.warmP != nullptr)
	{
		s2bWriteWarmImpulses(a, t, normal, tangent, pointCount, lam[0], lam[1]);
	}
	if (storeManifold)
	{
		// (.x separation and .w stay as the narrow phase left them: two scalar stores instead of a read-modify-write)
		float* m0 = reinterpret_cast<float*>(a.contacts.impulse[0] + cs.slot);
		m0[1] = lam[0].x;
		m0[2] = lam[0].y;
		if (pointCount == 2)
		{
			float* m1 = reinterpret_cast<float*>(a.contacts.impulse[1] + cs.slot);
			m1[1] = lam[1].x;
			m1[2] = lam[1].y;
		}
	}
	// bodies of infinite mass and inertia are never written (s2bStoreVelocities)
	if ((mA != 0.0f) || (iA != 0.0f))
	{
		velRows[ia] = make_float4(vA.x, vA.y, wA, velA.w);
	}
	if ((mB != 0.0f) || (iB != 0.0f))
	{
		velRows[ib] = make_float4(vB.x, vB.y, wB, velB.w);
	}
	// s2IntegratePositions (reference src/solve_common.c:47-68) of the bodies this constraint is the last of the sweep to
	// touch: the same arithmetic on the values just stored as s2bIntegratePosition applies after a device-wide barrier
	// (cs.last is only ever non-zero in a bias sweep of the persistent kernel that folds the position pass; marked bodies
	// are movable, hence valid and not static)
	if (cs.last & S2B_TOUCH_LAST_A)
	{
		s2Vec2 dp = s2MulAdd(dcA, a.ctx.h, vA);
		s2Rot q = s2IntegrateRot(qA, a.ctx.h * wA);
		poseRows[ia] = make_float4(dp.x, dp.y, q.s, q.c);
	}
	if (cs.last & S2B_TOUCH_LAST_B)
	{
		s2Vec2 dp = s2MulAdd(dcB, a.ctx.h, vB);
		s2Rot q = s2IntegrateRot(qB, a.ctx.h * wB);
		poseRows[ib] = make_float4(dp.x, dp.y, q.s, q.c);
	}
}

// writeWarm: this is the last pass that changes the impulses before the next sub-step's warm-start gather
__device__ __forceinline__ void s2bSolveContactTgsSoft(const SolveArgs& a, int t, float inv_h, bool useBias, bool writeWarm = false,
													   bool storeManifold = false)
{
	ContactStream cs = s2bLoadContactStream(a, t, storeManifold);
	s2bSolveContactTgsSoftStream(a, t, cs, inv_h, useBias, writeWarm, storeManifold);
}

// ===============================================================================================================
// The other variants. Every function keeps the structure "load both bodies - normal rows - friction rows - store" and
// differs in the switches of SURVEY.md §8a: anchors (fixed r0 | current), separation (prepare-time | current), bias
// law, row order, and what is written back (v,w | dv,dw | dp,q).
// ===============================================================================================================

struct ContactLoad
{
	int ia, ib, pointCount;
	bool staticSoft;
	float4 nf;
	float4 velA, velB;
	float mA, mB, iA, iB;
};

__device__ __forceinline__ ContactLoad s2bLoadContact(const SolveArgs& a, int t)
{
	ContactLoad c;
	int2 idx = a.cc.idx[t];
	c.ia = idx.x;
	c.ib = idx.y & S2B_CF_INDEX_MASK;
	c.pointCount = (idx.y & S2B_CF_TWO_POINTS) ? 2 : 1;
	c.staticSoft = ((unsigned)idx.y & S2B_CF_STATIC_SOFT) != 0;
	c.nf = a.cc.nf[t];
	c.velA = a.bodies.vel[c.ia];
	c.velB = a.bodies.vel[c.ib];
	c.mA = c.velA.w;
	c.mB = c.velB.w;
	c.iA = c.nf.w;
	c.iB = a.cc.pm[0][t].w;
	return c;
}

__device__ __forceinline__ void s2bStoreContactVelocities(const SolveArgs& a, const ContactLoad& c, s2Vec2 vA, float wA, s2Vec2 vB, float wB)
{
	if ((c.mA != 0.0f) || (c.iA != 0.0f))
	{
		a.bodies.vel[c.ia] = make_float4(vA.x, vA.y, wA, c.velA.w);
	}
	if ((c.mB != 0.0f) || (c.iB != 0.0f))
	{
		a.bodies.vel[c.ib] = make_float4(vB.x, vB.y, wB, c.velB.w);
	}
}

// s2WarmStartContacts_Fixed (reference src/solve_soft_step.c:16-63): prepare-time anchors
__device__ __forceinline__ void s2bWarmStartContactFixed(const SolveArgs& a, int t)
{
	ContactLoad c = s2bLoadContact(a, t);
	s2Vec2 vA = V2(c.velA.x, c.velA.y), vB = V2(c.velB.x, c.velB.y);
	float wA = c.velA.z, wB = c.velB.z;
	s2Vec2 normal = V2(c.nf.x, c.nf.y);
	s2Vec2 tangent = s2RightPerp(normal);
#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < c.pointCount)
		{
			float4 r0 = a.cc.r0[j][t];
			float2 l = a.cc.lambda[j][t];
			s2Vec2 rA = V2(r0.x, r0.y), rB = V2(r0.z, r0.w);
			s2Vec2 P = s2Add(s2MulSV(l.x, normal), s2MulSV(l.y, tangent));
			wA -= c.iA * s2Cross(rA, P);
			vA = s2MulAdd(vA, -c.mA, P);
			wB += c.iB * s2Cross(rB, P);
			vB = s2MulAdd(vB, c.mB, P);
		}
	}
	s2bStoreContactVelocities(a, c, vA, wA, vB, wB);
}

// Velocity solves with FIXED anchors and the PREPARE-time separation:
//   KIND 0  s2SolveContacts_PGS_Baumgarte (reference src/solve_pgs.c:17-122)
//   KIND 1  s2SolveContacts_PGS_Soft      (reference src/solve_pgs_soft.c:16-125), bias clamp -0.5 * maxBaumgarteVelocity
//   KIND 2  s2SolveContacts_Jacobi_Soft   (reference src/solve_jacobi.c:21-132), clamp -maxBaumgarteVelocity, writes dv/dw
template <int KIND> __device__ __forceinline__ void s2bSolveContactFixed(const SolveArgs& a, int t, float inv_h, bool useBias)
{
	ContactLoad c = s2bLoadContact(a, t);
	const SoftCoef soft = c.staticSoft ? a.softStatic : a.softDynamic;
	s2Vec2 vA = V2(c.velA.x, c.velA.y), vB = V2(c.velB.x, c.velB.y);
	float wA = c.velA.z, wB = c.velB.z;
	s2Vec2 normal = V2(c.nf.x, c.nf.y);
	s2Vec2 tangent = s2RightPerp(normal);
	float friction = c.nf.z;
	float2 lam[2] = {a.cc.lambda[0][t], a.cc.lambda[1][t]};
	float4 r0[2] = {a.cc.r0[0][t], a.cc.r0[1][t]};
	float4 pm[2] = {a.cc.pm[0][t], a.cc.pm[1][t]};
	float sep[2] = {a.cc.sep[0][t], a.cc.sep[1][t]};

#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < c.pointCount)
		{
			float bias = 0.0f, massScale = 1.0f, impulseScale = 0.0f;
			if (KIND == 0)
			{
				if (sep[j] > 0.0f)
				{
					bias = sep[j] * inv_h;
				}
				else
				{
					bias = S2_MAX(s2_baumgarte * inv_h * S2_MIN(0.0f, sep[j] + s2_linearSlop), -s2_maxBaumgarteVelocity);
				}
			}
			else
			{
				if (sep[j] > 0.0f)
				{
					bias = sep[j] * inv_h;
				}
				else if (useBias)
				{
					bias = KIND == 1 ? S2_MAX(soft.bias * sep[j], -0.5f * s2_maxBaumgarteVelocity)
									 : S2_MAX(soft.bias * sep[j], -s2_maxBaumgarteVelocity);
					massScale = soft.mass;
					impulseScale = soft.impulse;
				}
			}
			s2Vec2 rA = V2(r0[j].x, r0[j].y), rB = V2(r0[j].z, r0[j].w);
			s2Vec2 vrB = s2Add(vB, s2CrossSV(wB, rB));
			s2Vec2 vrA = s2Add(vA, s2CrossSV(wA, rA));
			float vn = s2Dot(s2Sub(vrB, vrA), normal);
			float impulse = KIND == 0 ? -pm[j].y * (vn + bias) : -pm[j].y * massScale * (vn + bias) - impulseScale * lam[j].x;
			float newImpulse = S2_MAX(lam[j].x + impulse, 0.0f);
			impulse = newImpulse - lam[j].x;
			lam[j].x = newImpulse;
			s2Vec2 P = s2MulSV(impulse, normal);
			vA = s2MulSub(vA, c.mA, P);
			wA -= c.iA * s2Cross(rA, P);
			vB = s2MulAdd(vB, c.mB, P);
			wB += c.iB * s2Cross(rB, P);
		}
	}

#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < c.pointCount)
		{
			s2Vec2 rA = V2(r0[j].x, r0[j].y), rB = V2(r0[j].z, r0[j].w);
			s2Vec2 vrB = s2Add(vB, s2CrossSV(wB, rB));
			s2Vec2 vrA = s2Add(vA, s2CrossSV(wA, rA));
			s2Vec2 dv = s2Sub(vrB, vrA);
			float vt = s2Dot(dv, tangent);
			float lambda = pm[j].z * (-vt);
			float maxFriction = friction * lam[j].x;
			float newImpulse = S2_CLAMP(lam[j].y + lambda, -maxFriction, maxFriction);
			lambda = newImpulse - lam[j].y;
			lam[j].y = newImpulse;
			s2Vec2 P = s2MulSV(lambda, tangent);
			vA = s2MulSub(vA, c.mA, P);
			wA -= c.iA * s2Cross(rA, P);
			vB = s2MulAdd(vB, c.mB, P);
			wB += c.iB * s2Cross(rB, P);
		}
	}

	a.cc.lambda[0][t] = lam[0];
	if (c.pointCount == 2)
	{
		a.cc.lambda[1][t] = lam[1];
	}
	if (KIND == 2)
	{
		// Jacobi: accumulate the velocity change instead of applying it (reference src/solve_jacobi.c:126-130). Bodies of
		// infinite mass receive an exact zero in the reference; they are skipped here.
		if ((c.mA != 0.0f) || (c.iA != 0.0f))
		{
			float4 d = a.bodies.aux0[c.ia];
			s2Vec2 dvA = s2Add(V2(d.x, d.y), s2Sub(vA, V2(c.velA.x, c.velA.y)));
			a.bodies.aux0[c.ia] = make_float4(dvA.x, dvA.y, d.z + (wA - c.velA.z), 0.0f);
		}
		if ((c.mB != 0.0f) || (c.iB != 0.0f))
		{
			float4 d = a.bodies.aux0[c.ib];
			s2Vec2 dvB = s2Add(V2(d.x, d.y), s2Sub(vB, V2(c.velB.x, c.velB.y)));
			a.bodies.aux0[c.ib] = make_float4(dvB.x, dvB.y, d.z + (wB - c.velB.z), 0.0f);
		}
	}
	else
	{
		s2bStoreContactVelocities(a, c, vA, wA, vB, wB);
	}
}

// s2SolveContacts_PGS (reference src/solve_pgs_ngs.c:16-124): Box2D-2.4 order — friction rows first, then normal rows;
// speculative points (prepare-time separation > 0) are skipped and their impulse zeroed.
__device__ __forceinline__ void s2bSolveContactPgs(const SolveArgs& a, int t)
{
	ContactLoad c = s2bLoadContact(a, t);
	s2Vec2 vA = V2(c.velA.x, c.velA.y), vB = V2(c.velB.x, c.velB.y);
	float wA = c.velA.z, wB = c.velB.z;
	s2Vec2 normal = V2(c.nf.x, c.nf.y);
	s2Vec2 tangent = s2CrossVS(normal, 1.0f);
	float friction = c.nf.z;
	float2 lam[2] = {a.cc.lambda[0][t], a.cc.lambda[1][t]};
	float4 r0[2] = {a.cc.r0[0][t], a.cc.r0[1][t]};
	float4 pm[2] = {a.cc.pm[0][t], a.cc.pm[1][t]};
	float sep[2] = {a.cc.sep[0][t], a.cc.sep[1][t]};

#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < c.pointCount)
		{
			if (sep[j] > 0.0f)
			{
				lam[j].y = 0.0f;
				continue;
			}
			s2Vec2 rA = V2(r0[j].x, r0[j].y), rB = V2(r0[j].z, r0[j].w);
			s2Vec2 vrB = s2Add(vB, s2CrossSV(wB, rB));
			s2Vec2 vrA = s2Add(vA, s2CrossSV(wA, rA));
			float vt = s2Dot(s2Sub(vrB, vrA), tangent);
			float lambda = pm[j].z * (-vt);
			float maxFriction = friction * lam[j].x;
			float newImpulse = S2_CLAMP(lam[j].y + lambda, -maxFriction, maxFriction);
			lambda = newImpulse - lam[j].y;
			lam[j].y = newImpulse;
			s2Vec2 P = s2MulSV(lambda, tangent);
			vA = s2MulSub(vA, c.mA, P);
			wA -= c.iA * s2Cross(rA, P);
			vB = s2MulAdd(vB, c.mB, P);
			wB += c.iB * s2Cross(rB, P);
		}
	}

#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < c.pointCount)
		{
			if (sep[j] > 0.0f)
			{
				lam[j].x = 0.0f;
				continue;
			}
			s2Vec2 rA = V2(r0[j].x, r0[j].y), rB = V2(r0[j].z, r0[j].w);
			s2Vec2 vrB = s2Add(vB, s2CrossSV(wB, rB));
			s2Vec2 vrA = s2Add(vA, s2CrossSV(wA, rA));
			float vn = s2Dot(s2Sub(vrB, vrA), normal);
			float impulse = -pm[j].y * vn;
			float newImpulse = S2_MAX(lam[j].x + impulse, 0.0f);
			impulse = newImpulse - lam[j].x;
			lam[j].x = newImpulse;
			s2Vec2 P = s2MulSV(impulse, normal);
			vA = s2MulSub(vA, c.mA, P);
			wA -= c.iA * s2Cross(rA, P);
			vB = s2MulAdd(vB, c.mB, P);
			wB += c.iB * s2Cross(rB, P);
		}
	}

	a.cc.lambda[0][t] = lam[0];
	if (c.pointCount == 2)
	{
		a.cc.lambda[1][t] = lam[1];
	}
	s2bStoreContactVelocities(a, c, vA, wA, vB, wB);
}

// Velocity solves that evaluate the separation at the CURRENT sub-step pose:
//   KIND 0  s2SolveContacts_TGS_Fixed (reference src/solve_soft_step.c:66-177): soft, clamp -0.5*maxBaumgarte, velocity
//           and impulse applied at the FIXED prepare-time anchors
//   KIND 1  s2SolveContacts_TGS       (reference src/solve_tgs_ngs.c:91-201): rigid, speculative bias only, current anchors
template <int KIND>
__device__ __forceinline__ void s2bSolveContactSubstep(const SolveArgs& a, int t, float inv_h, bool useBias, bool writeWarm = false)
{
	ContactLoad c = s2bLoadContact(a, t);
	const SoftCoef soft = c.staticSoft ? a.softStatic : a.softDynamic;
	float4 poseA = a.bodies.pose[c.ia], poseB = a.bodies.pose[c.ib];
	s2Vec2 vA = V2(c.velA.x, c.velA.y), vB = V2(c.velB.x, c.velB.y);
	float wA = c.velA.z, wB = c.velB.z;
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	s2Vec2 normal = V2(c.nf.x, c.nf.y);
	s2Vec2 tangent = s2RightPerp(normal);
	float friction = c.nf.z;
	float2 lam[2] = {a.cc.lambda[0][t], a.cc.lambda[1][t]};
	float4 la[2] = {a.cc.anchor[0][t], a.cc.anchor[1][t]};
	float4 pm[2] = {a.cc.pm[0][t], a.cc.pm[1][t]};
	float4 r0[2];
	if (KIND == 0)
	{
		r0[0] = a.cc.r0[0][t];
		r0[1] = a.cc.r0[1][t];
	}

#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < c.pointCount)
		{
			s2Vec2 rAc = s2RotateVector(qA, V2(la[j].x, la[j].y));
			s2Vec2 rBc = s2RotateVector(qB, V2(la[j].z, la[j].w));
			s2Vec2 rA, rB;
			float s;
			float bias = 0.0f, massScale = 1.0f, impulseScale = 0.0f;
			if (KIND == 0)
			{
				s2Vec2 ds = s2Add(s2Sub(dcB, dcA), s2Sub(rBc, rAc));
				s = s2Dot(ds, normal) + pm[j].x;
				if (s > 0.0f)
				{
					bias = s * inv_h;
				}
				else if (useBias)
				{
					bias = S2_MAX(soft.bias * s, -0.5f * s2_maxBaumgarteVelocity);
					massScale = soft.mass;
					impulseScale = soft.impulse;
				}
				rA = V2(r0[j].x, r0[j].y);
				rB = V2(r0[j].z, r0[j].w);
			}
			else
			{
				s2Vec2 d = s2Add(s2Sub(dcB, dcA), s2Sub(rBc, rAc));
				s = s2Dot(d, normal) + pm[j].x;
				bias = s > 0.0f ? s * inv_h : 0.0f;
				rA = rAc;
				rB = rBc;
			}
			s2Vec2 vrB = s2Add(vB, s2CrossSV(wB, rB));
			s2Vec2 vrA = s2Add(vA, s2CrossSV(wA, rA));
			float vn = s2Dot(s2Sub(vrB, vrA), normal);
			float impulse = KIND == 0 ? -pm[j].y * massScale * (vn + bias) - impulseScale * lam[j].x : -pm[j].y * (vn + bias);
			float newImpulse = S2_MAX(lam[j].x + impulse, 0.0f);
			impulse = newImpulse - lam[j].x;
			lam[j].x = newImpulse;
			s2Vec2 P = s2MulSV(impulse, normal);
			vA = s2MulSub(vA, c.mA, P);
			wA -= c.iA * s2Cross(rA, P);
			vB = s2MulAdd(vB, c.mB, P);
			wB += c.iB * s2Cross(rB, P);
		}
	}

#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < c.pointCount)
		{
			s2Vec2 rA, rB;
			if (KIND == 0)
			{
				rA = V2(r0[j].x, r0[j].y);
				rB = V2(r0[j].z, r0[j].w);
			}
			else
			{
				rA = s2RotateVector(qA, V2(la[j].x, la[j].y));
				rB = s2RotateVector(qB, V2(la[j].z, la[j].w));
			}
			s2Vec2 vrB = s2Add(vB, s2CrossSV(wB, rB));
			s2Vec2 vrA = s2Add(vA, s2CrossSV(wA, rA));
			float vt = s2Dot(s2Sub(vrB, vrA), tangent);
			float impulse = -pm[j].z * vt;
			float maxFriction = friction * lam[j].x;
			float newImpulse = S2_CLAMP(lam[j].y + impulse, -maxFriction, maxFriction);
			impulse = newImpulse - lam[j].y;
			lam[j].y = newImpulse;
			s2Vec2 P = s2MulSV(impulse, tangent);
			vA = s2MulSub(vA, c.mA, P);
			wA -= c.iA * s2Cross(rA, P);
			vB = s2MulAdd(vB, c.mB, P);
			wB += c.iB * s2Cross(rB, P);
		}
	}

	a.cc.lambda[0][t] = lam[0];
	if (c.pointCount == 2)
	{
		a.cc.lambda[1][t] = lam[1];
	}
	if (writeWarm && a.cc.warmP != nullptr)
	{
		s2bWriteWarmImpulses(a, t, normal, tangent, c.pointCount, lam[0], lam[1]);
	}
	s2bStoreContactVelocities(a, c, vA, wA, vB, wB);
}

// s2SolveContact_NGS (reference src/solve_common.c:328-394): non-linear Gauss-Seidel position pass. Reads and writes
// deltaPosition and rotation of both bodies; points that were speculative at prepare time are skipped.
__device__ __forceinline__ void s2bSolveContactNgs(const SolveArgs& a, int t)
{
	ContactLoad c = s2bLoadContact(a, t);
	float4 poseA = a.bodies.pose[c.ia], poseB = a.bodies.pose[c.ib];
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	s2Vec2 normal = V2(c.nf.x, c.nf.y);

#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < c.pointCount)
		{
			if (a.cc.sep[j][t] > 0.0f)
			{
				continue;
			}
			float4 la = a.cc.anchor[j][t];
			float adjustedSeparation = a.cc.pm[j][t].x;
			s2Vec2 rA = s2RotateVector(qA, V2(la.x, la.y));
			s2Vec2 rB = s2RotateVector(qB, V2(la.z, la.w));
			s2Vec2 d = s2Add(s2Sub(dcB, dcA), s2Sub(rB, rA));
			float separation = s2Dot(d, normal) + adjustedSeparation;
			float C = S2_CLAMP(s2_baumgarte * (separation + s2_linearSlop), -s2_maxLinearCorrection, 0.0f);
			float rnA = s2Cross(rA, normal);
			float rnB = s2Cross(rB, normal);
			float K = c.mA + c.mB + c.iA * rnA * rnA + c.iB * rnB * rnB;
			float impulse = K > 0.0f ? -C / K : 0.0f;
			s2Vec2 P = s2MulSV(impulse, normal);
			dcA = s2MulSub(dcA, c.mA, P);
			qA = s2IntegrateRot(qA, -c.iA * s2Cross(rA, P));
			dcB = s2MulAdd(dcB, c.mB, P);
			qB = s2IntegrateRot(qB, c.iB * s2Cross(rB, P));
		}
	}

	if ((c.mA != 0.0f) || (c.iA != 0.0f))
	{
		a.bodies.pose[c.ia] = make_float4(dcA.x, dcA.y, qA.s, qA.c);
	}
	if ((c.mB != 0.0f) || (c.iB != 0.0f))
	{
		a.bodies.pose[c.ib] = make_float4(dcB.x, dcB.y, qB.s, qB.c);
	}
}

// ---------------------------------------------------------------------------------------------------------------
// PGS_NGS_Block (reference src/solve_pgs_ngs_block.c): Box2D-2.4 style block solver — the two normal rows of a 2-point
// manifold are solved together as a 2x2 LCP by total enumeration. Optional stream columns used here:
//   r0[j]      prepare-time anchors rA.xy rB.xy (the velocity rows never move their anchors)
//   fanchor[0] K      = {k11, k12, k12, k22}   (cx.x cx.y cy.x cy.y)
//   fanchor[1] K^-1   (s2GetInverse22)
//   tsep[j].x  velocityBias of point j = -max(0, separation * inv_dt)
// ---------------------------------------------------------------------------------------------------------------

// s2CreateContactSolver, the per-constraint part (reference src/solve_pgs_ngs_block.c:135-262): the PGS prepare plus the
// speculative velocity bias and the 2x2 block; a manifold whose two rows are nearly dependent (condition number guard
// 1000) is solved, warm started AND stored as a 1-point manifold from here on.
__device__ __forceinline__ void s2bPrepareContactBlock(const SolveArgs& a, int t)
{
	s2bPrepareContact<PREPARE_PGS>(a, t);
	const ConstraintView& cc = a.cc;
	int2 idx = cc.idx[t];
	int slot = cc.src[t];
	float4 nf = cc.nf[t];
	s2Vec2 normal = V2(nf.x, nf.y);
	float mA = a.bodies.vel[idx.x].w, mB = a.bodies.vel[idx.y & S2B_CF_INDEX_MASK].w;
	float iA = nf.w, iB = cc.pm[0][t].w;
	int pointCount = (idx.y & S2B_CF_TWO_POINTS) ? 2 : 1;
#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		float separation = j < pointCount ? a.contacts.impulse[j][slot].x : 0.0f;
		cc.tsep[j][t] = make_float2(-S2_MAX(0.0f, separation * a.ctx.inv_dt), 0.0f);
	}
	s2Mat22 K = s2Mat22_zero, invK = s2Mat22_zero;
	if (pointCount == 2)
	{
		float4 r1 = cc.r0[0][t], r2 = cc.r0[1][t];
		float rn1A = s2Cross(V2(r1.x, r1.y), normal);
		float rn1B = s2Cross(V2(r1.z, r1.w), normal);
		float rn2A = s2Cross(V2(r2.x, r2.y), normal);
		float rn2B = s2Cross(V2(r2.z, r2.w), normal);
		float k11 = mA + mB + iA * rn1A * rn1A + iB * rn1B * rn1B;
		float k22 = mA + mB + iA * rn2A * rn2A + iB * rn2B * rn2B;
		float k12 = mA + mB + iA * rn1A * rn2A + iB * rn1B * rn2B;
		const float k_maxConditionNumber = 1000.0f;
		if (k11 * k11 < k_maxConditionNumber * (k11 * k22 - k12 * k12))
		{
			K.cx = V2(k11, k12);
			K.cy = V2(k12, k22);
			invK = s2GetInverse22(K);
		}
		else
		{
			cc.idx[t] = make_int2(idx.x, (int)((unsigned)idx.y & ~(unsigned)S2B_CF_TWO_POINTS));
		}
	}
	cc.fanchor[0][t] = make_float4(K.cx.x, K.cx.y, K.cy.x, K.cy.y);
	cc.fanchor[1][t] = make_float4(invK.cx.x, invK.cx.y, invK.cy.x, invK.cy.y);
}

// s2BlockSolveVelocity, one constraint (reference src/solve_pgs_ngs_block.c:329-658)
__device__ __forceinline__ void s2bSolveContactBlockVelocity(const SolveArgs& a, int t)
{
	ContactLoad c = s2bLoadContact(a, t);
	s2Vec2 vA = V2(c.velA.x, c.velA.y), vB = V2(c.velB.x, c.velB.y);
	float wA = c.velA.z, wB = c.velB.z;
	s2Vec2 normal = V2(c.nf.x, c.nf.y);
	s2Vec2 tangent = s2CrossVS(normal, 1.0f);
	float friction = c.nf.z;
	float mA = c.mA, mB = c.mB, iA = c.iA, iB = c.iB;
	float2 lam[2] = {a.cc.lambda[0][t], a.cc.lambda[1][t]};
	float4 r0[2] = {a.cc.r0[0][t], a.cc.r0[1][t]};
	float4 pm[2] = {a.cc.pm[0][t], a.cc.pm[1][t]};
	float bias[2] = {a.cc.tsep[0][t].x, a.cc.tsep[1][t].x};

	// friction rows first
#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < c.pointCount)
		{
			s2Vec2 rA = V2(r0[j].x, r0[j].y), rB = V2(r0[j].z, r0[j].w);
			s2Vec2 vrB = s2Add(vB, s2CrossSV(wB, rB));
			s2Vec2 vrA = s2Add(vA, s2CrossSV(wA, rA));
			s2Vec2 dv = s2Sub(vrB, vrA);
			float vt = s2Dot(dv, tangent);
			float lambda = pm[j].z * (-vt);
			float maxFriction = friction * lam[j].x;
			float newImpulse = S2_CLAMP(lam[j].y + lambda, -maxFriction, maxFriction);
			lambda = newImpulse - lam[j].y;
			lam[j].y = newImpulse;
			s2Vec2 P = s2MulSV(lambda, tangent);
			vA = s2MulSub(vA, mA, P);
			wA -= iA * s2Cross(rA, P);
			vB = s2MulAdd(vB, mB, P);
			wB += iB * s2Cross(rB, P);
		}
	}

	if (c.pointCount == 1)
	{
		s2Vec2 rA = V2(r0[0].x, r0[0].y), rB = V2(r0[0].z, r0[0].w);
		s2Vec2 vrB = s2Add(vB, s2CrossSV(wB, rB));
		s2Vec2 vrA = s2Add(vA, s2CrossSV(wA, rA));
		s2Vec2 dv = s2Sub(vrB, vrA);
		float vn = s2Dot(dv, normal);
		float lambda = -pm[0].y * (vn - bias[0]);
		float newImpulse = S2_MAX(lam[0].x + lambda, 0.0f);
		lambda = newImpulse - lam[0].x;
		lam[0].x = newImpulse;
		s2Vec2 P = s2MulSV(lambda, normal);
		vA = s2MulSub(vA, mA, P);
		wA -= iA * s2Cross(rA, P);
		vB = s2MulAdd(vB, mB, P);
		wB += iB * s2Cross(rB, P);
	}
	else
	{
		// 2x2 LCP:  vn = K x + b',  vn >= 0, x >= 0, vn_i x_i = 0, with b' = b - K a (a = accumulated impulses)
		float4 kk = a.cc.fanchor[0][t], ik = a.cc.fanchor[1][t];
		s2Mat22 K, normalMass;
		K.cx = V2(kk.x, kk.y);
		K.cy = V2(kk.z, kk.w);
		normalMass.cx = V2(ik.x, ik.y);
		normalMass.cy = V2(ik.z, ik.w);
		s2Vec2 rA1 = V2(r0[0].x, r0[0].y), rB1 = V2(r0[0].z, r0[0].w);
		s2Vec2 rA2 = V2(r0[1].x, r0[1].y), rB2 = V2(r0[1].z, r0[1].w);
		s2Vec2 acc = V2(lam[0].x, lam[1].x);
		s2Vec2 vrA = s2Add(vA, s2CrossSV(wA, rA1));
		s2Vec2 vrB = s2Add(vB, s2CrossSV(wB, rB1));
		s2Vec2 dv1 = s2Sub(vrB, vrA);
		vrA = s2Add(vA, s2CrossSV(wA, rA2));
		vrB = s2Add(vB, s2CrossSV(wB, rB2));
		s2Vec2 dv2 = s2Sub(vrB, vrA);
		float vn1 = s2Dot(dv1, normal);
		float vn2 = s2Dot(dv2, normal);
		s2Vec2 b = V2(vn1 - bias[0], vn2 - bias[1]);
		b = s2Sub(b, s2MulMV(K, acc));

		bool solved = false;
		s2Vec2 x = s2Neg(s2MulMV(normalMass, b));
		if (x.x >= 0.0f && x.y >= 0.0f)
		{
			solved = true; // case 1: both rows active
		}
		if (solved == false)
		{
			x.x = -pm[0].y * b.x;
			x.y = 0.0f;
			vn2 = K.cx.y * x.x + b.y;
			if (x.x >= 0.0f && vn2 >= 0.0f)
			{
				solved = true; // case 2: row 1 active, row 2 separating
			}
		}
		if (solved == false)
		{
			x.x = 0.0f;
			x.y = -pm[1].y * b.y;
			vn1 = K.cy.x * x.y + b.x;
			if (x.y >= 0.0f && vn1 >= 0.0f)
			{
				solved = true; // case 3: row 2 active
			}
		}
		if (solved == false)
		{
			x.x = 0.0f;
			x.y = 0.0f;
			if (b.x >= 0.0f && b.y >= 0.0f)
			{
				solved = true; // case 4: both separating
			}
		}
		if (solved)
		{
			s2Vec2 d = s2Sub(x, acc);
			s2Vec2 P1 = s2MulSV(d.x, normal);
			s2Vec2 P2 = s2MulSV(d.y, normal);
			vA = s2MulSub(vA, mA, s2Add(P1, P2));
			wA -= iA * (s2Cross(rA1, P1) + s2Cross(rA2, P2));
			vB = s2MulAdd(vB, mB, s2Add(P1, P2));
			wB += iB * (s2Cross(rB1, P1) + s2Cross(rB2, P2));
			lam[0].x = x.x;
			lam[1].x = x.y;
		}
		// no case holds (numerically inconsistent): the impulses stay as they are (reference :653-654)
	}

	a.cc.lambda[0][t] = lam[0];
	if (c.pointCount == 2)
	{
		a.cc.lambda[1][t] = lam[1];
	}
	s2bStoreContactVelocities(a, c, vA, wA, vB, wB);
}

// s2BlockSolvePosition, one constraint (reference src/solve_pgs_ngs_block.c:679-890): non-linear Gauss-Seidel on the
// positions with the block re-linearised at the current pose (condition number guard 10000, else point by point)
__device__ __forceinline__ void s2bSolveContactBlockPosition(const SolveArgs& a, int t)
{
	ContactLoad c = s2bLoadContact(a, t);
	float4 poseA = a.bodies.pose[c.ia], poseB = a.bodies.pose[c.ib];
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	s2Vec2 normal = V2(c.nf.x, c.nf.y);
	float mA = c.mA, mB = c.mB, iA = c.iA, iB = c.iB;
	float slop = s2_linearSlop;
	float4 la[2] = {a.cc.anchor[0][t], a.cc.anchor[1][t]};
	float adj[2] = {a.cc.pm[0][t].x, a.cc.pm[1][t].x};

	bool pointwise = c.pointCount != 2;
	if (c.pointCount == 2)
	{
		s2Vec2 rA1 = s2RotateVector(qA, V2(la[0].x, la[0].y));
		s2Vec2 rB1 = s2RotateVector(qB, V2(la[0].z, la[0].w));
		s2Vec2 rA2 = s2RotateVector(qA, V2(la[1].x, la[1].y));
		s2Vec2 rB2 = s2RotateVector(qB, V2(la[1].z, la[1].w));
		s2Vec2 dc = s2Sub(dcB, dcA);
		s2Vec2 d1 = s2Add(dc, s2Sub(rB1, rA1));
		float separation1 = s2Dot(d1, normal) + adj[0];
		s2Vec2 d2 = s2Add(dc, s2Sub(rB2, rA2));
		float separation2 = s2Dot(d2, normal) + adj[1];
		float C1 = S2_CLAMP(s2_baumgarte * (separation1 + slop), -s2_maxLinearCorrection, 0.0f);
		float C2 = S2_CLAMP(s2_baumgarte * (separation2 + slop), -s2_maxLinearCorrection, 0.0f);
		s2Vec2 b = V2(C1, C2);
		float rn1A = s2Cross(rA1, normal);
		float rn1B = s2Cross(rB1, normal);
		float rn2A = s2Cross(rA2, normal);
		float rn2B = s2Cross(rB2, normal);
		float k11 = mA + mB + iA * rn1A * rn1A + iB * rn1B * rn1B;
		float k22 = mA + mB + iA * rn2A * rn2A + iB * rn2B * rn2B;
		float k12 = mA + mB + iA * rn1A * rn2A + iB * rn1B * rn2B;
		const float k_maxConditionNumber = 10000.0f;
		if (k11 * k11 < k_maxConditionNumber * (k11 * k22 - k12 * k12))
		{
			s2Mat22 K;
			K.cx = V2(k11, k12);
			K.cy = V2(k12, k22);
			s2Mat22 invK = s2GetInverse22(K);
			bool solved = false;
			s2Vec2 x = s2Neg(s2MulMV(invK, b));
			if (x.x >= 0.0f && x.y >= 0.0f)
			{
				solved = true;
			}
			if (solved == false)
			{
				x.x = -b.x / k11;
				x.y = 0.0f;
				float vn2 = K.cx.y * x.x + b.y;
				if (x.x >= 0.0f && vn2 >= 0.0f)
				{
					solved = true;
				}
			}
			if (solved == false)
			{
				x.x = 0.0f;
				x.y = -b.y / k22;
				float vn1 = K.cy.x * x.y + b.x;
				if (x.y >= 0.0f && vn1 >= 0.0f)
				{
					solved = true;
				}
			}
			// the fourth case (both rows satisfied) moves nothing
			if (solved)
			{
				s2Vec2 P1 = s2MulSV(x.x, normal);
				s2Vec2 P2 = s2MulSV(x.y, normal);
				dcA = s2MulSub(dcA, mA, s2Add(P1, P2));
				qA = s2IntegrateRot(qA, -iA * (s2Cross(rA1, P1) + s2Cross(rA2, P2)));
				dcB = s2MulAdd(dcB, mB, s2Add(P1, P2));
				qB = s2IntegrateRot(qB, iB * (s2Cross(rB1, P1) + s2Cross(rB2, P2)));
			}
		}
		else
		{
			pointwise = true; // manifold_degenerate
		}
	}
	if (pointwise)
	{
#pragma unroll
		for (int j = 0; j < 2; ++j)
		{
			if (j < c.pointCount)
			{
				s2Vec2 rA = s2RotateVector(qA, V2(la[j].x, la[j].y));
				s2Vec2 rB = s2RotateVector(qB, V2(la[j].z, la[j].w));
				s2Vec2 d = s2Add(s2Sub(dcB, dcA), s2Sub(rB, rA));
				float separation = s2Dot(d, normal) + adj[j];
				float C = S2_CLAMP(s2_baumgarte * (separation + slop), -s2_maxLinearCorrection, 0.0f);
				float rnA = s2Cross(rA, normal);
				float rnB = s2Cross(rB, normal);
				float K = mA + mB + iA * rnA * rnA + iB * rnB * rnB;
				float impulse = K > 0.0f ? -C / K : 0.0f;
				s2Vec2 P = s2MulSV(impulse, normal);
				dcA = s2MulSub(dcA, mA, P);
				qA = s2IntegrateRot(qA, -iA * s2Cross(rA, P));
				dcB = s2MulAdd(dcB, mB, P);
				qB = s2IntegrateRot(qB, iB * s2Cross(rB, P));
			}
		}
	}

	if ((mA != 0.0f) || (iA != 0.0f))
	{
		a.bodies.pose[c.ia] = make_float4(dcA.x, dcA.y, qA.s, qA.c);
	}
	if ((mB != 0.0f) || (iB != 0.0f))
	{
		a.bodies.pose[c.ib] = make_float4(dcB.x, dcB.y, qB.s, qB.c);
	}
}

// ---------------------------------------------------------------------------------------------------------------
// TGS_Sticky (reference src/solve_tgs_sticky.c)
// ---------------------------------------------------------------------------------------------------------------

// s2PrepareContacts_Sticky (reference src/solve_tgs_sticky.c:19-165): no warm starting; friction acts at anchors that
// persist across steps while the pair keeps its manifold and the bodies have not rotated / separated too far. Reads and
// WRITES the persistent manifold (friction anchors, friction normals, frictionPersisted).
__device__ __forceinline__ void s2bPrepareContactSticky(const SolveArgs& a, int t)
{
	const ConstraintView& cc = a.cc;
	int slot = cc.src[t];
	int2 bodies = a.contacts.bodies[slot];
	int4 info = a.contacts.info[slot];
	float4 mnf = a.contacts.nf[slot];
	int pointCount = S2B_CI_COUNT(info.x);

	float4 velA = a.bodies.vel[bodies.x], velB = a.bodies.vel[bodies.y];
	float4 poseA = a.bodies.pose[bodies.x], poseB = a.bodies.pose[bodies.y];
	float4 orgA = a.bodies.org[bodies.x], orgB = a.bodies.org[bodies.y];
	float4 posA = a.bodies.pos[bodies.x], posB = a.bodies.pos[bodies.y];
	float mA = velA.w, mB = velB.w, iA = posA.z, iB = posB.z;
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	s2Vec2 lcA = V2(orgA.z, orgA.w), lcB = V2(orgB.z, orgB.w);
	s2Vec2 normal = V2(mnf.x, mnf.y);
	s2Vec2 tangent = s2RightPerp(normal);

	unsigned flags = pointCount == 2 ? S2B_CF_TWO_POINTS : 0;
	cc.idx[t] = make_int2(bodies.x, (int)((unsigned)bodies.y | flags));
	cc.nf[t] = make_float4(normal.x, normal.y, mnf.z, iA);

	s2Vec2 lA[2], lB[2], rA0[2], rB0[2];
	float adjSep[2], normalMass[2], tangentMass[2], tangentSeparation[2];
	s2Vec2 lfA[2], lfB[2];
	float4 manifoldAnchor[2];
	for (int j = 0; j < 2; ++j)
	{
		lA[j] = lB[j] = rA0[j] = rB0[j] = lfA[j] = lfB[j] = V2(0.0f, 0.0f);
		adjSep[j] = normalMass[j] = tangentMass[j] = tangentSeparation[j] = 0.0f;
		manifoldAnchor[j] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		if (j < pointCount)
		{
			float4 la = a.contacts.anchor[j][slot];
			manifoldAnchor[j] = la;
			float separation = a.contacts.impulse[j][slot].x;
			lA[j] = s2Sub(V2(la.x, la.y), lcA);
			lB[j] = s2Sub(V2(la.z, la.w), lcB);
			s2Vec2 rA = s2RotateVector(qA, lA[j]);
			s2Vec2 rB = s2RotateVector(qB, lB[j]);
			rA0[j] = rA;
			rB0[j] = rB;
			adjSep[j] = separation - s2Dot(s2Sub(rB, rA), normal);
			float rtA = s2Cross(rA, tangent);
			float rtB = s2Cross(rB, tangent);
			float kTangent = mA + mB + iA * rtA * rtA + iB * rtB * rtB;
			tangentMass[j] = kTangent > 0.0f ? 1.0f / kTangent : 0.0f;
			float rnA = s2Cross(rA, normal);
			float rnB = s2Cross(rB, normal);
			float kNormal = mA + mB + iA * rnA * rnA + iB * rnB * rnB;
			normalMass[j] = kNormal > 0.0f ? 1.0f / kNormal : 0.0f;
		}
	}

	s2Vec2 cA = V2(posA.x, posA.y), cB = V2(posB.x, posB.y);
	bool frictionConfirmed = false;
	if (info.x & S2B_CI_FRICTION_PERSISTED)
	{
		int confirmCount = 0;
		for (int j = 0; j < pointCount; ++j)
		{
			float4 fa = a.contacts.fanchor[j][slot];
			float4 fn = a.contacts.fnormal[j][slot];
			s2Vec2 normalA = s2RotateVector(qA, V2(fn.x, fn.y));
			s2Vec2 normalB = s2RotateVector(qB, V2(fn.z, fn.w));
			float nn = s2Dot(normalA, normalB);
			if (nn < 0.98f)
			{
				break; // relative rotation invalidated the cached anchors
			}
			lfA[j] = s2Sub(V2(fa.x, fa.y), lcA);
			lfB[j] = s2Sub(V2(fa.z, fa.w), lcB);
			s2Vec2 rAf = s2RotateVector(qA, lfA[j]);
			s2Vec2 rBf = s2RotateVector(qB, lfB[j]);
			s2Vec2 offset = s2Add(s2Sub(cB, cA), s2Sub(rBf, rAf));
			float normalSeparation = s2Dot(offset, normalA);
			if (S2_ABS(normalSeparation) > 2.0f * s2_linearSlop)
			{
				break; // normal separation invalidated the cached anchors
			}
			tangentSeparation[j] = s2Dot(s2Sub(cB, cA), tangent);
			float rtA = s2Cross(rAf, tangent);
			float rtB = s2Cross(rBf, tangent);
			float kTangent = mA + mB + iA * rtA * rtA + iB * rtB * rtB;
			tangentMass[j] = kTangent > 0.0f ? 1.0f / kTangent : 0.0f;
			confirmCount += 1;
		}
		frictionConfirmed = confirmCount == pointCount;
	}

	if (frictionConfirmed == false)
	{
		for (int j = 0; j < pointCount; ++j)
		{
			s2Vec2 fnA = s2InvRotateVector(qA, normal);
			s2Vec2 fnB = s2InvRotateVector(qB, normal);
			a.contacts.fnormal[j][slot] = make_float4(fnA.x, fnA.y, fnB.x, fnB.y);
			a.contacts.fanchor[j][slot] = manifoldAnchor[j];
			lfA[j] = lA[j];
			lfB[j] = lB[j];
			tangentSeparation[j] = s2Dot(s2Sub(cB, cA), tangent);
			float rtA = s2Cross(rA0[j], tangent);
			float rtB = s2Cross(rB0[j], tangent);
			float kTangent = mA + mB + iA * rtA * rtA + iB * rtB * rtB;
			tangentMass[j] = kTangent > 0.0f ? 1.0f / kTangent : 0.0f;
		}
	}
	a.contacts.info[slot] = make_int4(info.x | S2B_CI_FRICTION_PERSISTED, info.y, info.z, info.w);

	for (int j = 0; j < 2; ++j)
	{
		cc.anchor[j][t] = make_float4(lA[j].x, lA[j].y, lB[j].x, lB[j].y);
		cc.pm[j][t] = make_float4(adjSep[j], normalMass[j], tangentMass[j], j == 0 ? iB : 0.0f);
		cc.lambda[j][t] = make_float2(0.0f, 0.0f);
		cc.fanchor[j][t] = make_float4(lfA[j].x, lfA[j].y, lfB[j].x, lfB[j].y);
		cc.tsep[j][t] = make_float2(tangentSeparation[j], 0.0f);
	}
}

// s2SolveContacts_TGS_Sticky (reference src/solve_tgs_sticky.c:167-310): Baumgarte normal rows at the current anchors
// (factor 0.8), then friction as a *position-level* constraint at the persistent friction anchors (factor 0.5) limited by
// half the friction coefficient times the sum of the normal impulses; hitting the limit un-persists the anchors.
__device__ __forceinline__ void s2bSolveContactSticky(const SolveArgs& a, int t, float inv_h, bool useBias)
{
	ContactLoad c = s2bLoadContact(a, t);
	const float contactBaumgarte = 0.8f;
	const float frictionBaumgarte = 0.5f;
	float4 poseA = a.bodies.pose[c.ia], poseB = a.bodies.pose[c.ib];
	s2Vec2 vA = V2(c.velA.x, c.velA.y), vB = V2(c.velB.x, c.velB.y);
	float wA = c.velA.z, wB = c.velB.z;
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	s2Vec2 normal = V2(c.nf.x, c.nf.y);
	s2Vec2 tangent = s2RightPerp(normal);
	float friction = c.nf.z;
	float2 lam[2] = {a.cc.lambda[0][t], a.cc.lambda[1][t]};
	float totalNormalImpulse = 0.0f;
	bool unpersist = false;

#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < c.pointCount)
		{
			float4 la = a.cc.anchor[j][t];
			float4 pm = a.cc.pm[j][t];
			s2Vec2 rA = s2RotateVector(qA, V2(la.x, la.y));
			s2Vec2 rB = s2RotateVector(qB, V2(la.z, la.w));
			s2Vec2 d = s2Add(s2Sub(dcB, dcA), s2Sub(rB, rA));
			float separation = s2Dot(d, normal) + pm.x;
			float bias = 0.0f;
			if (separation > 0.0f)
			{
				bias = separation * inv_h;
			}
			else if (useBias)
			{
				bias = S2_MAX(-s2_maxBaumgarteVelocity, contactBaumgarte * separation * inv_h);
			}
			s2Vec2 vrA = s2Add(vA, s2CrossSV(wA, rA));
			s2Vec2 vrB = s2Add(vB, s2CrossSV(wB, rB));
			float vn = s2Dot(s2Sub(vrB, vrA), normal);
			float impulse = -pm.y * (vn + bias);
			float newImpulse = S2_MAX(lam[j].x + impulse, 0.0f);
			impulse = newImpulse - lam[j].x;
			lam[j].x = newImpulse;
			totalNormalImpulse += lam[j].x;
			s2Vec2 P = s2MulSV(impulse, normal);
			vA = s2MulSub(vA, c.mA, P);
			wA -= c.iA * s2Cross(rA, P);
			vB = s2MulAdd(vB, c.mB, P);
			wB += c.iB * s2Cross(rB, P);
		}
	}

#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < c.pointCount)
		{
			float4 lf = a.cc.fanchor[j][t];
			float tangentMass = a.cc.pm[j][t].z;
			float tangentSeparation = a.cc.tsep[j][t].x;
			s2Vec2 rAf = s2RotateVector(qA, V2(lf.x, lf.y));
			s2Vec2 rBf = s2RotateVector(qB, V2(lf.z, lf.w));
			s2Vec2 d = s2Add(s2Sub(dcB, dcA), s2Sub(rBf, rAf));
			float separation = s2Dot(d, tangent) + tangentSeparation;
			float bias = useBias ? frictionBaumgarte * separation * inv_h : 0.0f;
			s2Vec2 vrA = s2Add(vA, s2CrossSV(wA, rAf));
			s2Vec2 vrB = s2Add(vB, s2CrossSV(wB, rBf));
			float vt = s2Dot(s2Sub(vrB, vrA), tangent);
			float impulse = -tangentMass * (vt + bias);
			float maxFriction = 0.5f * friction * totalNormalImpulse;
			float newImpulse = lam[j].y + impulse;
			if (newImpulse < -maxFriction)
			{
				newImpulse = -maxFriction;
				unpersist = true;
			}
			else if (newImpulse > maxFriction)
			{
				newImpulse = maxFriction;
				unpersist = true;
			}
			impulse = newImpulse - lam[j].y;
			lam[j].y = newImpulse;
			s2Vec2 P = s2MulSV(impulse, tangent);
			vA = s2MulSub(vA, c.mA, P);
			wA -= c.iA * s2Cross(rAf, P);
			vB = s2MulAdd(vB, c.mB, P);
			wB += c.iB * s2Cross(rBf, P);
		}
	}

	a.cc.lambda[0][t] = lam[0];
	if (c.pointCount == 2)
	{
		a.cc.lambda[1][t] = lam[1];
	}
	if (unpersist)
	{
		int slot = a.cc.src[t];
		int4 info = a.contacts.info[slot];
		a.contacts.info[slot] = make_int4(info.x & ~S2B_CI_FRICTION_PERSISTED, info.y, info.z, info.w);
	}
	s2bStoreContactVelocities(a, c, vA, wA, vB, wB);
}

// ---------------------------------------------------------------------------------------------------------------
// XPBD (reference src/solve_xpbd.c)
// ---------------------------------------------------------------------------------------------------------------

// s2SolveContactPositions_XPBD (reference src/solve_xpbd.c:88-216): position-level non-penetration and static friction.
__device__ __forceinline__ void s2bSolveContactXpbdPositions(const SolveArgs& a, int t, float h)
{
	ContactLoad c = s2bLoadContact(a, t);
	const float baseCompliance = 0.0f;
	float compliance = (c.mA == 0.0f || c.mB == 0.0f) ? 0.25f * baseCompliance : baseCompliance;
	float4 poseA = a.bodies.pose[c.ia], poseB = a.bodies.pose[c.ib];
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	s2Vec2 normal = V2(c.nf.x, c.nf.y);
	s2Vec2 tangent = s2CrossVS(normal, 1.0f);
	float friction = c.nf.z;
	float2 lam[2] = {a.cc.lambda[0][t], a.cc.lambda[1][t]};

#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < c.pointCount)
		{
			float4 la = a.cc.anchor[j][t];
			float4 r0 = a.cc.r0[j][t];
			s2Vec2 rA = s2RotateVector(qA, V2(la.x, la.y));
			s2Vec2 rB = s2RotateVector(qB, V2(la.z, la.w));
			s2Vec2 drA = s2Sub(rA, V2(r0.x, r0.y));
			s2Vec2 drB = s2Sub(rB, V2(r0.z, r0.w));
			s2Vec2 ds = s2Add(s2Sub(dcB, dcA), s2Sub(drB, drA));
			float C = s2Dot(ds, normal) + a.cc.sep[j][t];
			if (C > 0)
			{
				lam[j].x = 0.0f;
				continue;
			}
			C = S2_MAX(-s2_maxBaumgarteVelocity * h, C);
			float rnA = s2Cross(rA, normal);
			float rnB = s2Cross(rB, normal);
			float kA = c.mA + c.iA * rnA * rnA;
			float kB = c.mB + c.iB * rnB * rnB;
			float lambda = -C / (kA + kB + compliance);
			lam[j].x = lambda;
			s2Vec2 P = s2MulSV(lambda, normal);
			dcA = s2MulSub(dcA, c.mA, P);
			qA = s2IntegrateRot(qA, -c.iA * s2Cross(rA, P));
			dcB = s2MulAdd(dcB, c.mB, P);
			qB = s2IntegrateRot(qB, c.iB * s2Cross(rB, P));
		}
	}

#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < c.pointCount)
		{
			float4 la = a.cc.anchor[j][t];
			float4 r0 = a.cc.r0[j][t];
			s2Vec2 rA = s2RotateVector(qA, V2(la.x, la.y));
			s2Vec2 rB = s2RotateVector(qB, V2(la.z, la.w));
			s2Vec2 drA = s2Sub(rA, V2(r0.x, r0.y));
			s2Vec2 drB = s2Sub(rB, V2(r0.z, r0.w));
			s2Vec2 dp = s2Add(s2Sub(dcB, dcA), s2Sub(drB, drA));
			float C = s2Dot(dp, tangent);
			float rtA = s2Cross(rA, tangent);
			float rtB = s2Cross(rB, tangent);
			float kA = c.mA + c.iA * rtA * rtA;
			float kB = c.mB + c.iB * rtB * rtB;
			float lambda = -C / (kA + kB);
			float maxLambda = friction * lam[j].x;
			if (lambda < -maxLambda || maxLambda < lambda)
			{
				lam[j].y = 0.0f; // beyond the static friction cone: skipped, not clamped (reference :190-194)
				continue;
			}
			lam[j].y = lambda;
			s2Vec2 P = s2MulSV(lambda, tangent);
			dcA = s2MulSub(dcA, c.mA, P);
			qA = s2IntegrateRot(qA, -c.iA * s2Cross(rA, P));
			dcB = s2MulAdd(dcB, c.mB, P);
			qB = s2IntegrateRot(qB, c.iB * s2Cross(rB, P));
		}
	}

	a.cc.lambda[0][t] = lam[0];
	if (c.pointCount == 2)
	{
		a.cc.lambda[1][t] = lam[1];
	}
	if ((c.mA != 0.0f) || (c.iA != 0.0f))
	{
		a.bodies.pose[c.ia] = make_float4(dcA.x, dcA.y, qA.s, qA.c);
	}
	if ((c.mB != 0.0f) || (c.iB != 0.0f))
	{
		a.bodies.pose[c.ib] = make_float4(dcB.x, dcB.y, qB.s, qB.c);
	}
}

// s2SolveContactVelocities_XPBD (reference src/solve_xpbd.c:218-338): velocity relaxation + kinetic friction
__device__ __forceinline__ void s2bSolveContactXpbdVelocities(const SolveArgs& a, int t, float h)
{
	ContactLoad c = s2bLoadContact(a, t);
	float inv_h = h > 0.0f ? 1.0f / h : 0.0f;
	float4 poseA = a.bodies.pose[c.ia], poseB = a.bodies.pose[c.ib];
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	s2Vec2 vA = V2(c.velA.x, c.velA.y), vB = V2(c.velB.x, c.velB.y);
	float wA = c.velA.z, wB = c.velB.z;
	s2Vec2 normal = V2(c.nf.x, c.nf.y);
	s2Vec2 tangent = s2CrossVS(normal, 1.0f);
	float friction = c.nf.z;
	float2 lam[2] = {a.cc.lambda[0][t], a.cc.lambda[1][t]};

#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < c.pointCount)
		{
			if (lam[j].x == 0.0f)
			{
				continue;
			}
			float4 la = a.cc.anchor[j][t];
			s2Vec2 rA = s2RotateVector(qA, V2(la.x, la.y));
			s2Vec2 rB = s2RotateVector(qB, V2(la.z, la.w));
			s2Vec2 vrB = s2Add(vB, s2CrossSV(wB, rB));
			s2Vec2 vrA = s2Add(vA, s2CrossSV(wA, rA));
			s2Vec2 dv = s2Sub(vrB, vrA);
			float rnA = s2Cross(rA, normal);
			float rnB = s2Cross(rB, normal);
			float kA = c.mA + c.iA * rnA * rnA;
			float kB = c.mB + c.iB * rnB * rnB;
			float vn = s2Dot(dv, normal);
			float lambda = -vn / (kA + kB);
			s2Vec2 P = s2MulSV(lambda, normal);
			vA = s2MulSub(vA, c.mA, P);
			wA -= c.iA * s2Cross(rA, P);
			vB = s2MulAdd(vB, c.mB, P);
			wB += c.iB * s2Cross(rB, P);
		}
	}

#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		if (j < c.pointCount)
		{
			float4 la = a.cc.anchor[j][t];
			s2Vec2 rA = s2RotateVector(qA, V2(la.x, la.y));
			s2Vec2 rB = s2RotateVector(qB, V2(la.z, la.w));
			s2Vec2 vrB = s2Add(vB, s2CrossSV(wB, rB));
			s2Vec2 vrA = s2Add(vA, s2CrossSV(wA, rA));
			s2Vec2 dv = s2Sub(vrB, vrA);
			float vt = s2Dot(dv, tangent);
			if (vt == 0.0f)
			{
				continue;
			}
			float rtA = s2Cross(rA, tangent);
			float rtB = s2Cross(rB, tangent);
			float kA = c.mA + c.iA * rtA * rtA;
			float kB = c.mB + c.iB * rtB * rtB;
			float maxFrictionImpulse = friction * lam[j].x;
			float huf = (maxFrictionImpulse * inv_h) * (kA + kB);
			float abs_vt = S2_ABS(vt);
			float Cdot = (vt / abs_vt) * S2_MIN(huf, abs_vt);
			float lambda = -Cdot / (kA + kB);
			lam[j].y = lambda;
			s2Vec2 P = s2MulSV(lambda, tangent);
			vA = s2MulSub(vA, c.mA, P);
			wA -= c.iA * s2Cross(rA, P);
			vB = s2MulAdd(vB, c.mB, P);
			wB += c.iB * s2Cross(rB, P);
		}
	}

	a.cc.lambda[0][t] = lam[0];
	if (c.pointCount == 2)
	{
		a.cc.lambda[1][t] = lam[1];
	}
	s2bStoreContactVelocities(a, c, vA, wA, vB, wB);
}

// ---------------------------------------------------------------------------------------------------------------
// body passes of the Jacobi and XPBD variants
// ---------------------------------------------------------------------------------------------------------------

// reset of dv / dw (reference src/solve_jacobi.c:176-186)
__device__ __forceinline__ void s2bJacobiReset(const SolveArgs& a, int i)
{
	if (a.bodies.flags[i] & S2B_BODY_VALID)
	{
		a.bodies.aux0[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
	}
}

// apply and clear the accumulated velocity change of one sweep (reference src/solve_jacobi.c:233-245)
__device__ __forceinline__ void s2bJacobiApply(const SolveArgs& a, int i)
{
	if ((a.bodies.flags[i] & S2B_BODY_VALID) == 0)
	{
		return;
	}
	float4 vel = a.bodies.vel[i];
	float4 d = a.bodies.aux0[i];
	s2Vec2 v = s2Add(V2(vel.x, vel.y), V2(d.x, d.y));
	float w = vel.z + d.z;
	a.bodies.vel[i] = make_float4(v.x, v.y, w, vel.w);
	a.bodies.aux0[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}

// XPBD integrates velocities AND positions up front and remembers the previous pose (reference src/solve_xpbd.c:408-443);
// every non-static body, kinematic ones included
__device__ __forceinline__ void s2bXpbdIntegrate(const SolveArgs& a, int i, float h)
{
	unsigned f = a.bodies.flags[i];
	if ((f & S2B_BODY_VALID) == 0 || S2B_BODY_TYPE(f) == S2B_BODY_STATIC)
	{
		return;
	}
	float4 vel = a.bodies.vel[i];
	float4 frc = a.bodies.frc[i];
	float4 prm = a.bodies.prm[i];
	float4 pose = a.bodies.pose[i];
	float invMass = vel.w, invI = prm.w, mass = frc.w;
	s2Vec2 v = V2(vel.x, vel.y);
	float w = vel.z;
	s2Vec2 gravity = V2(a.gravity.x, a.gravity.y);
	v = s2Add(v, s2MulSV(h * invMass, s2MulAdd(V2(frc.x, frc.y), mass * prm.z, gravity)));
	w = w + h * invI * frc.z;
	v = s2MulSV(1.0f / (1.0f + h * prm.x), v);
	w *= 1.0f / (1.0f + h * prm.y);
	a.bodies.vel[i] = make_float4(v.x, v.y, w, invMass);
	a.bodies.aux0[i] = pose; // deltaPosition0, rot0
	s2Vec2 dp = s2MulAdd(V2(pose.x, pose.y), h, v);
	s2Rot q = s2IntegrateRot(R2(pose.z, pose.w), h * w);
	a.bodies.pose[i] = make_float4(dp.x, dp.y, q.s, q.c);
}

// velocities from the position change of the sub-step (reference src/solve_xpbd.c:457-483); dynamic bodies only
__device__ __forceinline__ void s2bXpbdProjectVelocity(const SolveArgs& a, int i, float inv_h)
{
	unsigned f = a.bodies.flags[i];
	if ((f & S2B_BODY_VALID) == 0 || S2B_BODY_TYPE(f) != S2B_BODY_DYNAMIC)
	{
		return;
	}
	float4 vel = a.bodies.vel[i];
	float4 pose = a.bodies.pose[i];
	float4 pose0 = a.bodies.aux0[i];
	s2Vec2 v = s2MulSV(inv_h, s2Sub(V2(pose.x, pose.y), V2(pose0.x, pose0.y)));
	float w = s2ComputeAngularVelocity(R2(pose0.z, pose0.w), R2(pose.z, pose.w), inv_h);
	a.bodies.vel[i] = make_float4(v.x, v.y, w, vel.w);
}

// XPBD finalises dynamic bodies only (reference src/solve_xpbd.c:497-511, SURVEY §8a N6)
__device__ __forceinline__ void s2bXpbdFinalize(const SolveArgs& a, int i)
{
	unsigned f = a.bodies.flags[i];
	if ((f & S2B_BODY_VALID) == 0 || S2B_BODY_TYPE(f) != S2B_BODY_DYNAMIC)
	{
		return;
	}
	float4 pos = a.bodies.pos[i];
	float4 pose = a.bodies.pose[i];
	s2Vec2 p = s2Add(V2(pos.x, pos.y), V2(pose.x, pose.y));
	a.bodies.pos[i] = make_float4(p.x, p.y, pos.z, pos.w);
	a.bodies.pose[i] = make_float4(0.0f, 0.0f, pose.z, pose.w);
}
