// solver2d-b200 — stage 3 of s2World_Step on the device: one thread per contact recomputes the manifold of its shape
// pair and carries the accumulated impulses over by feature id.
//
// Replaces the contact loop of s2World_Step (reference src/world.c:138-168) + s2UpdateContact (reference
// src/contact.c:296-359) + the manifold functions it dispatches to (src/manifold.c via the table at contact.c:139-154).
// The geometry itself lives in csrc/shared/s2_collide.h and is shared with the host-callable s2Collide* API.
//
// Traffic per polygon-polygon contact: 2 shape headers + 2 x (count x 16 B) geometry + 2 x 32 B body transform read,
// ~112 B of manifold columns read and written. Arithmetic (GJK + clip) dominates; the kernel is latency/ALU bound,
// not bandwidth bound.
//
// While the solve schedule stands, each thread also writes its constraint's row of the solver's constraint stream
// (s2bWriteContactRow): it holds the manifold and both bodies' transforms already, and the solver's prepare pass, which
// would gather them all again, is skipped (DESIGN.md §3.4).
#include "contact_kernels.cuh"

#include "shared/s2_collide.h"

// Polygons live in shared memory while a thread works on its pair: GJK / SAT / clipping index them dynamically, so as
// automatic variables they end up in local memory, and 300 k threads x ~400 B of touched stack is written back to HBM when
// the lines are evicted (several times the bytes of the manifold columns themselves). Two polygons per thread,
// thread stride 69 words (odd: same-field accesses of a warp fall in 32 different banks).
#define S2B_NP_BLOCK 128
#define S2B_NP_POLY_WORDS 34
#define S2B_NP_THREAD_WORDS (2 * S2B_NP_POLY_WORDS + 1)
static_assert(sizeof(s2Polygon) == 4 * S2B_NP_POLY_WORDS, "s2Polygon layout");

// the points of a manifold just computed, for s2bWriteContactRow: what the table's anchor / impulse columns now hold
struct S2bFreshPoints
{
	float4 anchor0, anchor1, impulse0, impulse1;
	__device__ __forceinline__ float4 anchor(int j) const
	{
		return j == 0 ? anchor0 : anchor1;
	}
	__device__ __forceinline__ float4 impulse(int j) const
	{
		return j == 0 ? impulse0 : impulse1;
	}
};

__device__ __forceinline__ void s2bLoadPolygon(s2Polygon* poly, const ShapeView& s, int shape, int count, float radius)
{
	for (int k = 0; k < count; ++k)
	{
		float2 v = s.verts[shape * 8 + k];
		float2 n = s.normals[shape * 8 + k];
		poly->vertices[k].x = v.x;
		poly->vertices[k].y = v.y;
		poly->normals[k].x = n.x;
		poly->normals[k].y = n.y;
	}
	poly->count = count;
	poly->radius = radius;
}

// polyB of a pair, moved into polyA's frame while it is loaded (s2cMakeLocalPolygon, same arithmetic)
__device__ __forceinline__ void s2bLoadLocalPolygon(s2Polygon* poly, const ShapeView& s, int shape, int count, float radius,
													s2Transform xf)
{
	for (int k = 0; k < count; ++k)
	{
		float2 v = s.verts[shape * 8 + k];
		float2 n = s.normals[shape * 8 + k];
		s2Vec2 lv = {v.x, v.y}, ln = {n.x, n.y};
		poly->vertices[k] = s2TransformPoint(xf, lv);
		poly->normals[k] = s2RotateVector(xf.q, ln);
	}
	poly->count = count;
	poly->radius = radius;
}

// KIND < 0: the manifolds only. KIND = PREPARE_SOFT / PREPARE_COLD: also row rowOf[i] of the constraint stream of `a` for every
// manifold with points that has a row. Thread 0 says which in *rowsReady (CNT_ROWS_READY of the solver's counts; null before
// the first solve), for the schedule gate.
template <int KIND>
__global__ void __launch_bounds__(S2B_NP_BLOCK) s2bUpdateContactsKernel(ContactView c, int contactCount, ShapeView s, BodyView b, int sticky,
																		  int* schedDirty, SolveArgs a, const int* rowOf, int* rowsReady)
{
	__shared__ float polyStore[S2B_NP_BLOCK * S2B_NP_THREAD_WORDS];
	s2Polygon* polyA = reinterpret_cast<s2Polygon*>(polyStore + threadIdx.x * S2B_NP_THREAD_WORDS);
	s2Polygon* polyB = reinterpret_cast<s2Polygon*>(polyStore + threadIdx.x * S2B_NP_THREAD_WORDS + S2B_NP_POLY_WORDS);

	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i == 0 && rowsReady != nullptr)
	{
		*rowsReady = KIND >= 0 ? 1 : 0;
	}
	if (i >= contactCount)
	{
		return;
	}

	int2 shapes = c.shapes[i];
	int4 headA = s.head[shapes.x], headB = s.head[shapes.y];
	int typeA = (headA.x >> 1) & 0x7, typeB = (headB.x >> 1) & 0x7;
	int bodyA = headA.y, bodyB = headB.y;
	float radiusA = s.fr[shapes.x].y, radiusB = s.fr[shapes.y].y;

	float4 orgA = b.org[bodyA], orgB = b.org[bodyB];
	float4 poseA = b.pose[bodyA], poseB = b.pose[bodyB];
	s2Transform xfA, xfB;
	xfA.p.x = orgA.x;
	xfA.p.y = orgA.y;
	xfA.q.s = poseA.z;
	xfA.q.c = poseA.w;
	xfB.p.x = orgB.x;
	xfB.p.y = orgB.y;
	xfB.q.s = poseB.z;
	xfB.q.c = poseB.w;

	// previous manifold state (scalars, not arrays: a dynamically indexed array would live on the local stack)
	int4 info = c.info[i];
	int oldCount = S2B_CI_COUNT(info.x);
	int oldId0 = info.y & 0xFFFF, oldId1 = (info.y >> 16) & 0xFFFF;
	float4 oldImp0 = c.impulse[0][i], oldImp1 = c.impulse[1][i];

	s2DistanceCache cache;
	cache.metric = __int_as_float(info.w);
	cache.count = (uint16_t)(info.z & 0x3);
	for (int k = 0; k < 3; ++k)
	{
		cache.indexA[k] = (uint8_t)((info.z >> (2 + 3 * k)) & 0x7);
		cache.indexB[k] = (uint8_t)((info.z >> (11 + 3 * k)) & 0x7);
	}

	s2Manifold m;
	if (typeB == S2B_SHAPE_CIRCLE)
	{
		float2 cB = s.verts[shapes.y * 8];
		s2Vec2 centerB = {cB.x, cB.y};
		if (typeA == S2B_SHAPE_CIRCLE)
		{
			float2 cA = s.verts[shapes.x * 8];
			s2Vec2 centerA = {cA.x, cA.y};
			s2cCollideCircles(&m, centerA, radiusA, xfA, centerB, radiusB, xfB);
		}
		else if (typeA == S2B_SHAPE_CAPSULE || typeA == S2B_SHAPE_SEGMENT)
		{
			float2 a1 = s.verts[shapes.x * 8], a2 = s.verts[shapes.x * 8 + 1];
			s2Vec2 p1 = {a1.x, a1.y}, p2 = {a2.x, a2.y};
			s2cCollideCapsuleAndCircle(&m, p1, p2, typeA == S2B_SHAPE_SEGMENT ? 0.0f : radiusA, xfA, centerB, radiusB, xfB);
		}
		else
		{
			s2bLoadPolygon(polyA, s, shapes.x, headA.w, radiusA);
			s2cCollidePolygonAndCircle(&m, polyA->vertices, polyA->normals, polyA->count, polyA->radius, xfA, centerB, radiusB, xfB);
		}
	}
	else
	{
		// polygon / capsule / segment pairs all go through the polygon path (capsules and segments are 2-gons)
		s2Transform xf = s2InvMulTransforms(xfA, xfB);
		s2bLoadPolygon(polyA, s, shapes.x, headA.w, typeA == S2B_SHAPE_SEGMENT ? 0.0f : radiusA);
		s2bLoadLocalPolygon(polyB, s, shapes.y, headB.w, typeB == S2B_SHAPE_SEGMENT ? 0.0f : radiusB, xf);
		s2cCollidePolygonsLocal(&m, polyA, xfA, polyB, xf, &cache);
	}

	// s2UpdateContact: match old ids to new ids and carry the impulses (reference src/contact.c:317-358). A new point takes
	// the impulses of the FIRST old point with the same feature id.
	int pointCount = m.pointCount;
	int newId0 = pointCount > 0 ? m.points[0].id : 0, newId1 = pointCount > 1 ? m.points[1].id : 0;
	int matched0 = pointCount > 0 ? ((oldCount > 0 && oldId0 == newId0) ? 0 : ((oldCount > 1 && oldId1 == newId0) ? 1 : -1)) : -1;
	int matched1 = pointCount > 1 ? ((oldCount > 0 && oldId0 == newId1) ? 0 : ((oldCount > 1 && oldId1 == newId1) ? 1 : -1)) : -1;
	float4 newImp0 = make_float4(0.0f, 0.0f, 0.0f, 0.0f), newImp1 = newImp0;
	if (pointCount > 0)
	{
		newImp0.x = m.points[0].separation;
		if (matched0 >= 0)
		{
			newImp0.y = matched0 == 0 ? oldImp0.y : oldImp1.y;
			newImp0.z = matched0 == 0 ? oldImp0.z : oldImp1.z;
		}
	}
	if (pointCount > 1)
	{
		newImp1.x = m.points[1].separation;
		if (matched1 >= 0)
		{
			newImp1.y = matched1 == 0 ? oldImp0.y : oldImp1.y;
			newImp1.z = matched1 == 0 ? oldImp0.z : oldImp1.z;
		}
	}
	int flags = pointCount & 0x3;
	flags |= matched0 >= 0 ? S2B_CI_PERSISTED0 : 0;
	flags |= matched1 >= 0 ? S2B_CI_PERSISTED1 : 0;
	// friction anchors persist only when the point count is unchanged and every point was matched
	bool frictionPersisted = pointCount == oldCount && (pointCount < 1 || matched0 >= 0) && (pointCount < 2 || matched1 >= 0);
	if (frictionPersisted)
	{
		flags |= S2B_CI_FRICTION_PERSISTED;
	}

	if (sticky)
	{
		// friction anchors / normals follow their point (reference src/contact.c:339-342); unmatched points start at 0
		float4 zero = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		float4 oldFA0 = c.fanchor[0][i], oldFA1 = c.fanchor[1][i];
		float4 oldFN0 = c.fnormal[0][i], oldFN1 = c.fnormal[1][i];
		c.fanchor[0][i] = matched0 < 0 ? zero : (matched0 == 0 ? oldFA0 : oldFA1);
		c.fnormal[0][i] = matched0 < 0 ? zero : (matched0 == 0 ? oldFN0 : oldFN1);
		c.fanchor[1][i] = matched1 < 0 ? zero : (matched1 == 0 ? oldFA0 : oldFA1);
		c.fnormal[1][i] = matched1 < 0 ? zero : (matched1 == 0 ? oldFN0 : oldFN1);
	}

	int cacheBits = cache.count & 0x3;
	for (int k = 0; k < 3; ++k)
	{
		cacheBits |= (cache.indexA[k] & 0x7) << (2 + 3 * k);
		cacheBits |= (cache.indexB[k] & 0x7) << (11 + 3 * k);
	}
	c.info[i] = make_int4(flags, (newId0 & 0xFFFF) | ((newId1 & 0xFFFF) << 16), cacheBits, __float_as_int(cache.metric));
	float4 nf = c.nf[i];
	c.nf[i] = make_float4(m.normal.x, m.normal.y, nf.z, nf.w);
	if (pointCount == 0)
	{
		c.color[i] = -1; // not a constraint this step: its colour is free again
	}
	if ((pointCount > 0) != (oldCount > 0))
	{
		*schedDirty = 1; // the set of live constraints changed: the solve schedule has to be rebuilt (solver.cu, s2bScheduleGate)
	}
	c.anchor[0][i] = make_float4(m.points[0].localAnchorA.x, m.points[0].localAnchorA.y, m.points[0].localAnchorB.x, m.points[0].localAnchorB.y);
	c.anchor[1][i] = make_float4(m.points[1].localAnchorA.x, m.points[1].localAnchorA.y, m.points[1].localAnchorB.x, m.points[1].localAnchorB.y);
	c.impulse[0][i] = newImp0;
	c.impulse[1][i] = newImp1;

	if constexpr (KIND >= 0)
	{
		// the row prepare would build from what was just stored: a manifold without points has no row, a manifold that gained
		// its first point has none yet (both raised schedDirty above: the rebuilt schedule's prepare writes every row)
		int t = pointCount > 0 ? rowOf[i] : -1;
		if (t >= 0)
		{
			int2 bodies = c.bodies[i];
			if (bodies.x != bodyA || bodies.y != bodyB)
			{
				*schedDirty = 1; // (never seen: the table's bodies are its shapes' bodies) prepare gathers the table's bodies
			}
			else
			{
				float mA = b.vel[bodyA].w, mB = b.vel[bodyB].w;
				float iA = b.prm[bodyA].w, iB = b.prm[bodyB].w;
				S2bFreshPoints points = {
					make_float4(m.points[0].localAnchorA.x, m.points[0].localAnchorA.y, m.points[0].localAnchorB.x, m.points[0].localAnchorB.y),
					make_float4(m.points[1].localAnchorA.x, m.points[1].localAnchorA.y, m.points[1].localAnchorB.x, m.points[1].localAnchorB.y),
					newImp0, newImp1};
				s2bWriteContactRow<KIND>(a, t, bodies, pointCount, make_float4(m.normal.x, m.normal.y, nf.z, nf.w), points, orgA, orgB, poseA, poseB,
										 mA, mB, iA, iB);
			}
		}
	}
}

void s2bNarrowphaseUpdate(s2bWorld* w)
{
	if (w->contactCount <= 0)
	{
		return;
	}
	SolveArgs a;
	memset(&a, 0, sizeof(a));
	const int* rowOf = nullptr;
	int* rowsReady = nullptr;
	int kind = s2bNarrowphaseRows(w, &a, &rowOf, &rowsReady);
	ContactView c = makeView(w->contacts[w->cur]);
	int grid = gridFor(w->contactCount, S2B_NP_BLOCK);
	int sticky = w->sticky ? 1 : 0;
	if (kind == PREPARE_SOFT)
	{
		S2B_LAUNCH(w, s2bUpdateContactsKernel<PREPARE_SOFT>, grid, S2B_NP_BLOCK, 0, c, w->contactCount, shapeView(w), bodyView(w), sticky,
				   w->schedDirty.p, a, rowOf, rowsReady);
	}
	else if (kind == PREPARE_COLD)
	{
		S2B_LAUNCH(w, s2bUpdateContactsKernel<PREPARE_COLD>, grid, S2B_NP_BLOCK, 0, c, w->contactCount, shapeView(w), bodyView(w), sticky,
				   w->schedDirty.p, a, rowOf, rowsReady);
	}
	else
	{
		S2B_LAUNCH(w, s2bUpdateContactsKernel<-1>, grid, S2B_NP_BLOCK, 0, c, w->contactCount, shapeView(w), bodyView(w), sticky, w->schedDirty.p, a,
				   rowOf, rowsReady);
	}
}
