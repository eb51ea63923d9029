// solver2d-b200 — time of impact and shape extents for continuous collision (DESIGN.md §3.11), written once as plain-C
// inline functions that compile for the host (public s2TimeOfImpact / s2GetSweepTransform / s2ComputeShapeExtent,
// csrc/host/geometry_host.c) and for the device (the continuous pass, csrc/device/broadphase.cu). Both sides are compiled
// without FMA contraction, so they give the same bits on the same inputs.
#pragma once

#include "shared/s2_collide.h"
#include "solver2d_b200.h"

// Target separation of a time of impact (radii included) and the tolerance it is reached within. The target stays below
// s2_speculativeDistance, so the narrow phase of the next step gives the pair a speculative point.
#define S2C_TOI_TARGET s2_linearSlop
#define S2C_TOI_TOLERANCE (0.25f * s2_linearSlop)

// centre of mass and rotation of a sweep at fraction t: the centre linearly, the rotation by normalised lerp
S2C_FN void s2cSweepPose(const s2Sweep* sweep, float t, s2Vec2* c, s2Rot* q)
{
	float u = 1.0f - t;
	c->x = u * sweep->c1.x + t * sweep->c2.x;
	c->y = u * sweep->c1.y + t * sweep->c2.y;
	s2Rot r = {u * sweep->q1.s + t * sweep->q2.s, u * sweep->q1.c + t * sweep->q2.c};
	*q = s2NormalizeRot(r);
}

// the body transform (origin, rotation) of a sweep at fraction t; origin = centre - R * localCenter, the expression
// finalize derives body origins with
S2C_FN s2Transform s2cGetSweepTransform(const s2Sweep* sweep, float t)
{
	s2Transform xf;
	s2cSweepPose(sweep, t, &xf.p, &xf.q);
	xf.p = s2Sub(xf.p, s2RotateVector(xf.q, sweep->localCenter));
	return xf;
}

// Bound on the angular speed d(theta)/dt of the normalised lerp from q1 to q2 over t in [0, 1] (DESIGN.md §3.11):
// |q1 - q2|^2 / |cross(q1, q2)|, which is 2 tan(|phi| / 2) for unit rotations (phi the angle from q1 to q2) and stays an
// upper bound for rotations a few ulp off unit length (as s2IntegrateRot leaves them). Unbounded for a half turn. (The
// form 2 |sin phi| / (1 + cos phi) is not: at a half turn of rotations shorter than unit, 1 + cos phi is a few ulp and
// sin phi round-off, and the bound came out near 0.)
S2C_FN float s2cSweepAngularBound(const s2Sweep* sweep)
{
	float sinPhi = sweep->q1.c * sweep->q2.s - sweep->q1.s * sweep->q2.c;
	float cosPhi = sweep->q1.c * sweep->q2.c + sweep->q1.s * sweep->q2.s;
	float dc = sweep->q1.c - sweep->q2.c, ds = sweep->q1.s - sweep->q2.s;
	float chordSq = dc * dc + ds * ds;
	if (sinPhi == 0.0f)
	{
		return cosPhi > 0.0f ? 0.0f : FLT_MAX;
	}
	return S2_MIN(chordSq / S2_ABS(sinPhi), FLT_MAX);
}

// largest distance of a vertex from the body's centre of mass (vertices in the body frame)
S2C_FN float s2cMaxVertexDistance(const s2Vec2* vertices, int count, s2Vec2 localCenter)
{
	float maxSq = 0.0f;
	for (int i = 0; i < count; ++i)
	{
		maxSq = S2_MAX(maxSq, s2DistanceSquared(vertices[i], localCenter));
	}
	return sqrtf(maxSq);
}

// Time of impact of two convex shapes in polygon form (vertices in their body frames) by conservative advancement on the
// GJK distance of their cores. At each iterate t the closest points give a unit axis n from A to B; the shapes' separation
// along n can only fall at the rate mu = -n . (dcB - dcA) + wA RA + wB RB (dc: centre displacement over the sweep, w: the
// angular bound above, R: largest vertex distance from the centre), so advancing by (separation - target) / mu never
// passes the target. A rate mu <= 0 means the separation cannot fall again before the end.
#define S2C_TOI_MAX_ITERATIONS S2_TOI_MAX_ITERATIONS

S2C_FN s2TOIOutput s2cTimeOfImpact(const s2Vec2* vertsA, int countA, float radiusA, const s2Sweep* sweepA, const s2Vec2* vertsB,
								   int countB, float radiusB, const s2Sweep* sweepB, float maxFraction)
{
	s2TOIOutput output;
	output.state = s2_toiStateUnknown;
	output.fraction = maxFraction;
	output.iterations = 0;

	float totalRadius = radiusA + radiusB;
	const float target = S2C_TOI_TARGET;
	const float tolerance = S2C_TOI_TOLERANCE;
	s2Vec2 dc = s2Sub(s2Sub(sweepB->c2, sweepB->c1), s2Sub(sweepA->c2, sweepA->c1));
	float rotation = s2cSweepAngularBound(sweepA) * s2cMaxVertexDistance(vertsA, countA, sweepA->localCenter) +
					 s2cSweepAngularBound(sweepB) * s2cMaxVertexDistance(vertsB, countB, sweepB->localCenter);

	s2DistanceCache cache = {0};
	float t = 0.0f;
	for (int iter = 0; iter < S2C_TOI_MAX_ITERATIONS; ++iter)
	{
		output.iterations = iter + 1;
		s2Transform xfA = s2cGetSweepTransform(sweepA, t);
		s2Transform xfB = s2cGetSweepTransform(sweepB, t);
		s2DistanceOutput d = s2cShapeDistance(&cache, vertsA, countA, radiusA, xfA, vertsB, countB, radiusB, xfB, false);
		float separation = d.distance - totalRadius;
		if (separation < target + tolerance)
		{
			output.state = iter == 0 ? s2_toiStateOverlapped : s2_toiStateHit;
			output.fraction = t;
			return output;
		}
		s2Vec2 n = s2cNormalize(s2Sub(d.pointB, d.pointA));
		float mu = rotation - s2Dot(n, dc);
		t = mu > 0.0f ? t + (separation - target) / mu : maxFraction;
		if (t >= maxFraction)
		{
			output.state = s2_toiStateSeparated;
			output.fraction = maxFraction;
			return output;
		}
	}
	// out of iterations: t is still a time the shapes are apart
	output.state = s2_toiStateFailed;
	output.fraction = t;
	return output;
}

// Inner and outer extent of a shape in polygon form (circle: 1 vertex; capsule: 2 vertices and its radius; segment: 2
// vertices, radius 0), the quantities a body is classified as fast by:
//   core    — where the core proxy of a shape that starts a step touching a static shape sits: the vertex of a circle, the
//             midpoint of a capsule or segment, the centroid of a polygon;
//   inner   — circle and capsule: the radius; segment: 0; polygon: the smallest distance from the centroid to an edge's
//             line, plus the rounding radius;
//   outer   — the largest distance of a vertex from the body's centre of mass, plus the radius.
typedef struct s2cShapeExtent
{
	s2Vec2 core;
	float inner, outer;
} s2cShapeExtent;

S2C_FN s2cShapeExtent s2cComputeShapeExtent(const s2Vec2* vertices, const s2Vec2* normals, int count, float radius, s2Vec2 localCenter)
{
	s2cShapeExtent e;
	e.outer = s2cMaxVertexDistance(vertices, count, localCenter) + radius;
	if (count == 1)
	{
		e.core = vertices[0];
		e.inner = radius;
		return e;
	}
	if (count == 2)
	{
		e.core = s2cVec(0.5f * (vertices[0].x + vertices[1].x), 0.5f * (vertices[0].y + vertices[1].y));
		e.inner = radius;
		return e;
	}
	// centroid by a triangle fan from the first vertex (reference src/geometry.c:30-58)
	s2Vec2 center = s2cVec(0.0f, 0.0f);
	float area = 0.0f;
	s2Vec2 origin = vertices[0];
	const float inv3 = 1.0f / 3.0f;
	for (int i = 1; i < count - 1; ++i)
	{
		s2Vec2 e1 = s2Sub(vertices[i], origin);
		s2Vec2 e2 = s2Sub(vertices[i + 1], origin);
		float a = 0.5f * s2Cross(e1, e2);
		center = s2MulAdd(center, a * inv3, s2Add(e1, e2));
		area += a;
	}
	float invArea = 1.0f / area;
	e.core = s2cVec(center.x * invArea + origin.x, center.y * invArea + origin.y);
	float inner = FLT_MAX;
	for (int i = 0; i < count; ++i)
	{
		inner = S2_MIN(inner, s2Dot(normals[i], s2Sub(vertices[i], e.core)));
	}
	e.inner = inner + radius;
	return e;
}

// A core (see s2cComputeShapeExtent) that starts a sweep within the target of a static shape is held where it is if it
// moves toward that shape by more than the tolerance over the sweep: its body is already a quarter of its inner extent
// deep, and letting it go on would carry it through a thin wall (a solver that ignores speculative points lets a body
// that was stopped at the target run on). Coincident cores (no axis) and cores moving along or away are let go.
S2C_FN bool s2cCoreApproaches(const s2Vec2* vertsA, int countA, const s2Sweep* sweepA, s2Vec2 core, const s2Sweep* sweepB)
{
	s2DistanceCache cache = {0};
	s2DistanceOutput d = s2cShapeDistance(&cache, vertsA, countA, 0.0f, s2cGetSweepTransform(sweepA, 0.0f), &core, 1, 0.0f,
										  s2cGetSweepTransform(sweepB, 0.0f), false);
	s2Vec2 n = s2cNormalize(s2Sub(d.pointB, d.pointA));
	s2Vec2 dc = s2Sub(s2Sub(sweepB->c2, sweepB->c1), s2Sub(sweepA->c2, sweepA->c1));
	return -s2Dot(n, dc) > S2C_TOI_TOLERANCE;
}
