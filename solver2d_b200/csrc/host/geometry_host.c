// solver2d-b200 — host geometry helpers of the public API (behaviour of reference src/geometry.c, src/math.c,
// src/aabb.c). Set-up time only: shapes are authored here, mass properties and the first AABB are computed here, and
// the result is mirrored once into the device shape / body tables. Mass and AABB arithmetic follows the reference
// expression for expression because it feeds the solver (invMass, invI, localCenter) and the pair set (fat AABBs).
#include "s2_host.h"

#include "shared/s2_collide.h"
#include "shared/s2_toi.h"

#include <float.h>
#include <string.h>
#include <math.h>

// ---- math.h out-of-line part (reference src/math.c) --------------------------------------------------------------

bool s2IsValid(float a)
{
	return isnan(a) == 0 && isinf(a) == 0;
}

bool s2IsValidVec2(s2Vec2 v)
{
	return s2IsValid(v.x) && s2IsValid(v.y);
}

s2Vec2 s2Normalize(s2Vec2 v)
{
	return s2cNormalize(v);
}

s2Vec2 s2NormalizeChecked(s2Vec2 v)
{
	S2_ASSERT(s2Length(v) >= FLT_EPSILON);
	return s2cNormalizeChecked(v);
}

s2Vec2 s2GetLengthAndNormalize(float* length, s2Vec2 v)
{
	return s2cGetLengthAndNormalize(length, v);
}

// ---- aabb.h out-of-line part (reference src/aabb.c) --------------------------------------------------------------

bool s2AABB_IsValid(s2Box a)
{
	s2Vec2 d = s2Sub(a.upperBound, a.lowerBound);
	return d.x >= 0.0f && d.y >= 0.0f && s2IsValidVec2(a.lowerBound) && s2IsValidVec2(a.upperBound);
}

// slab test (Ericson, Real-Time Collision Detection 5.3.3); hit only for entry fractions in [0, 1]
s2RayCastOutput s2AABB_RayCast(s2Box a, s2Vec2 p1, s2Vec2 p2)
{
	s2RayCastOutput out = {0};
	float tmin = -FLT_MAX, tmax = FLT_MAX;
	s2Vec2 d = s2Sub(p2, p1);
	s2Vec2 normal = {0.0f, 0.0f};
	const float lo[2] = {a.lowerBound.x, a.lowerBound.y};
	const float hi[2] = {a.upperBound.x, a.upperBound.y};
	const float p[2] = {p1.x, p1.y};
	const float dd[2] = {d.x, d.y};
	for (int axis = 0; axis < 2; ++axis)
	{
		if (S2_ABS(dd[axis]) < FLT_EPSILON)
		{
			if (p[axis] < lo[axis] || hi[axis] < p[axis])
			{
				return out;
			}
			continue;
		}
		float inv = 1.0f / dd[axis];
		float t1 = (lo[axis] - p[axis]) * inv;
		float t2 = (hi[axis] - p[axis]) * inv;
		float sign = -1.0f;
		if (t1 > t2)
		{
			float tmp = t1;
			t1 = t2;
			t2 = tmp;
			sign = 1.0f;
		}
		if (t1 > tmin)
		{
			normal.x = axis == 0 ? sign : 0.0f;
			normal.y = axis == 1 ? sign : 0.0f;
			tmin = t1;
		}
		tmax = S2_MIN(tmax, t2);
		if (tmin > tmax)
		{
			return out;
		}
	}
	if (tmin < 0.0f || 1.0f < tmin)
	{
		return out;
	}
	out.fraction = tmin;
	out.normal = normal;
	out.point = s2Lerp(p1, p2, tmin);
	out.hit = true;
	return out;
}

// ---- polygon factories ------------------------------------------------------------------------------------------

bool s2IsValidRay(const s2RayCastInput* input)
{
	return s2IsValidVec2(input->p1) && s2IsValidVec2(input->p2) && s2IsValid(input->maxFraction) && 0.0f <= input->maxFraction &&
		   input->maxFraction < s2_huge;
}

// reference src/geometry.c:23-47: outward normals = normalised right-perpendicular of each edge
s2Polygon s2MakePolygon(const s2Hull* hull)
{
	s2Polygon shape;
	shape.count = hull->count;
	shape.radius = 0.0f;
	for (int32_t i = 0; i < shape.count; ++i)
	{
		shape.vertices[i] = hull->points[i];
	}
	for (int32_t i = 0; i < shape.count; ++i)
	{
		int32_t next = i + 1 < shape.count ? i + 1 : 0;
		s2Vec2 edge = s2Sub(shape.vertices[next], shape.vertices[i]);
		shape.normals[i] = s2cNormalize(s2CrossVS(edge, 1.0f));
	}
	return shape;
}

// reference src/geometry.c:54-71
s2Polygon s2MakeBox(float hx, float hy)
{
	s2Polygon shape = {0};
	shape.count = 4;
	shape.vertices[0] = s2MakeVec2(-hx, -hy);
	shape.vertices[1] = s2MakeVec2(hx, -hy);
	shape.vertices[2] = s2MakeVec2(hx, hy);
	shape.vertices[3] = s2MakeVec2(-hx, hy);
	shape.normals[0] = s2MakeVec2(0.0f, -1.0f);
	shape.normals[1] = s2MakeVec2(1.0f, 0.0f);
	shape.normals[2] = s2MakeVec2(0.0f, 1.0f);
	shape.normals[3] = s2MakeVec2(-1.0f, 0.0f);
	shape.radius = 0.0f;
	return shape;
}

s2Polygon s2MakeSquare(float h)
{
	return s2MakeBox(h, h);
}

s2Polygon s2MakeRoundedBox(float hx, float hy, float radius)
{
	s2Polygon shape = s2MakeBox(hx, hy);
	shape.radius = radius;
	return shape;
}

// reference src/geometry.c:80-94
s2Polygon s2MakeOffsetBox(float hx, float hy, s2Vec2 center, float angle)
{
	s2Transform xf;
	xf.p = center;
	xf.q = s2MakeRot(angle);
	s2Polygon shape = {0};
	shape.count = 4;
	shape.vertices[0] = s2TransformPoint(xf, s2MakeVec2(-hx, -hy));
	shape.vertices[1] = s2TransformPoint(xf, s2MakeVec2(hx, -hy));
	shape.vertices[2] = s2TransformPoint(xf, s2MakeVec2(hx, hy));
	shape.vertices[3] = s2TransformPoint(xf, s2MakeVec2(-hx, hy));
	shape.normals[0] = s2RotateVector(xf.q, s2MakeVec2(0.0f, -1.0f));
	shape.normals[1] = s2RotateVector(xf.q, s2MakeVec2(1.0f, 0.0f));
	shape.normals[2] = s2RotateVector(xf.q, s2MakeVec2(0.0f, 1.0f));
	shape.normals[3] = s2RotateVector(xf.q, s2MakeVec2(-1.0f, 0.0f));
	shape.radius = 0.0f;
	return shape;
}

s2Polygon s2MakeCapsule(s2Vec2 p1, s2Vec2 p2, float radius)
{
	s2Polygon shape;
	s2cMakeCapsule(&shape, p1, p2, radius);
	return shape;
}

// ---- mass properties --------------------------------------------------------------------------------------------

// reference src/geometry.c:113-124
s2MassData s2ComputeCircleMass(const s2Circle* shape, float density)
{
	float rr = shape->radius * shape->radius;
	s2MassData md;
	md.mass = density * s2_pi * rr;
	md.center = shape->point;
	md.I = md.mass * (0.5f * rr + s2Dot(shape->point, shape->point));
	return md;
}

// reference src/geometry.c:126-150: rectangle plus two half discs
s2MassData s2ComputeCapsuleMass(const s2Capsule* shape, float density)
{
	float radius = shape->radius;
	float rr = radius * radius;
	s2Vec2 p1 = shape->point1;
	s2Vec2 p2 = shape->point2;
	float length = s2Length(s2Sub(p2, p1));
	float ll = length * length;

	s2MassData md;
	md.mass = density * (s2_pi * radius + 2.0f * length) * radius;
	md.center.x = 0.5f * (p1.x + p2.x);
	md.center.y = 0.5f * (p1.y + p2.y);

	float circleInertia = 0.5f * (rr + ll);
	float boxInertia = (4.0f * rr + ll) / 12.0f;
	md.I = md.mass * (circleInertia + boxInertia);
	return md;
}

// Outline whose area a (possibly rounded) polygon is given the mass of: the polygon itself, or — radius > 0 — every corner
// moved outwards along the bisector of its two edge normals until the straight edges have moved out by `radius`.
static void s2MassOutline(const s2Polygon* poly, s2Vec2* outline)
{
	int32_t n = poly->count;
	if (poly->radius <= 0.0f)
	{
		memcpy(outline, poly->vertices, sizeof(s2Vec2) * (size_t)n);
		return;
	}
	for (int32_t corner = 0, before = n - 1; corner < n; before = corner++)
	{
		s2Vec2 nIn = poly->normals[before], nOut = poly->normals[corner];
		s2Vec2 bisector = s2cNormalize(s2Add(nIn, nOut));
		s2Vec2 alongIn = {-nIn.y, nIn.x};
		// sine of half the corner's exterior angle; a straight "corner" keeps the plain radius
		float s = s2Cross(bisector, alongIn);
		float push = s > FLT_EPSILON ? poly->radius / s : poly->radius;
		outline[corner] = s2MulAdd(poly->vertices[corner], push, bisector);
	}
}

// Mass properties of a convex polygon (behaviour of reference src/geometry.c:152-286, whose arithmetic is kept operation
// for operation — the body masses of a scene have to come out bit-identical). Degenerate polygons are the round shapes
// they stand for; everything else is summed as a fan of triangles spanned from the first outline vertex.
s2MassData s2ComputePolygonMass(const s2Polygon* shape, float density)
{
	if (shape->count <= 2)
	{
		if (shape->count == 1)
		{
			s2Circle disc = {shape->vertices[0], shape->radius};
			return s2ComputeCircleMass(&disc, density);
		}
		s2Capsule pill = {shape->vertices[0], shape->vertices[1], shape->radius};
		return s2ComputeCapsuleMass(&pill, density);
	}

	s2Vec2 outline[s2_maxPolygonVertices];
	s2MassOutline(shape, outline);

	// zeroth, first and second moments about the fan's apex
	const s2Vec2 apex = outline[0];
	const float third = 1.0f / 3.0f;
	float areaSum = 0.0f, secondMoment = 0.0f;
	s2Vec2 firstMoment = {0.0f, 0.0f};
	for (const s2Vec2* v = outline + 1; v + 1 < outline + shape->count; ++v)
	{
		s2Vec2 a = s2Sub(v[0], apex), b = s2Sub(v[1], apex);
		float twiceArea = s2Cross(a, b);
		float wedge = 0.5f * twiceArea;
		areaSum += wedge;
		firstMoment = s2MulAdd(firstMoment, wedge * third, s2Add(a, b));
		float xx = a.x * a.x + b.x * a.x + b.x * b.x;
		float yy = a.y * a.y + b.y * a.y + b.y * b.y;
		secondMoment += (0.25f * third * twiceArea) * (xx + yy);
	}

	s2MassData out;
	out.mass = density * areaSum;
	float perArea = 1.0f / areaSum;
	s2Vec2 centroidFromApex = {firstMoment.x * perArea, firstMoment.y * perArea};
	out.center = s2Add(apex, centroidFromApex);
	// inertia about the apex, shifted to the shape's origin (parallel axes, through the centroid)
	out.I = density * secondMoment;
	out.I += out.mass * (s2Dot(out.center, out.center) - s2Dot(centroidFromApex, centroidFromApex));
	return out;
}

// ---- bounding boxes (reference src/geometry.c:288-341) ------------------------------------------------------------

s2Box s2ComputeCircleAABB(const s2Circle* shape, s2Transform xf)
{
	s2Vec2 p = s2TransformPoint(xf, shape->point);
	float r = shape->radius;
	s2Box aabb = {{p.x - r, p.y - r}, {p.x + r, p.y + r}};
	return aabb;
}

s2Box s2ComputeCapsuleAABB(const s2Capsule* shape, s2Transform xf)
{
	s2Vec2 v1 = s2TransformPoint(xf, shape->point1);
	s2Vec2 v2 = s2TransformPoint(xf, shape->point2);
	s2Vec2 r = {shape->radius, shape->radius};
	s2Box aabb;
	aabb.lowerBound = s2Sub(s2Min(v1, v2), r);
	aabb.upperBound = s2Add(s2Max(v1, v2), r);
	return aabb;
}

s2Box s2ComputePolygonAABB(const s2Polygon* shape, s2Transform xf)
{
	s2Vec2 lower = s2TransformPoint(xf, shape->vertices[0]);
	s2Vec2 upper = lower;
	for (int32_t i = 1; i < shape->count; ++i)
	{
		s2Vec2 v = s2TransformPoint(xf, shape->vertices[i]);
		lower = s2Min(lower, v);
		upper = s2Max(upper, v);
	}
	s2Vec2 r = {shape->radius, shape->radius};
	s2Box aabb;
	aabb.lowerBound = s2Sub(lower, r);
	aabb.upperBound = s2Add(upper, r);
	return aabb;
}

s2Box s2ComputeSegmentAABB(const s2Segment* shape, s2Transform xf)
{
	s2Vec2 v1 = s2TransformPoint(xf, shape->point1);
	s2Vec2 v2 = s2TransformPoint(xf, shape->point2);
	s2Box aabb;
	aabb.lowerBound = s2Min(v1, v2);
	aabb.upperBound = s2Max(v1, v2);
	return aabb;
}

// ---- point tests (reference src/geometry.c:343-391) ---------------------------------------------------------------

bool s2PointInCircle(s2Vec2 point, const s2Circle* shape)
{
	return s2DistanceSquared(point, shape->point) <= shape->radius * shape->radius;
}

bool s2PointInCapsule(s2Vec2 point, const s2Capsule* shape)
{
	float rr = shape->radius * shape->radius;
	s2Vec2 p1 = shape->point1;
	s2Vec2 d = s2Sub(shape->point2, p1);
	float dd = s2Dot(d, d);
	if (dd == 0.0f)
	{
		return s2DistanceSquared(point, p1) <= rr;
	}
	float t = s2Dot(s2Sub(point, p1), d) / dd;
	t = S2_CLAMP(t, 0.0f, 1.0f);
	s2Vec2 c = s2MulAdd(p1, t, d);
	return s2DistanceSquared(point, c) <= rr;
}

bool s2PointInPolygon(s2Vec2 point, const s2Polygon* shape)
{
	s2DistanceCache cache = {0};
	int count = S2_MIN(shape->count, s2_maxPolygonVertices);
	s2DistanceOutput output = s2cShapeDistance(&cache, shape->vertices, count, 0.0f, s2Transform_identity, &point, 1, 0.0f,
											   s2Transform_identity, false);
	return output.distance <= shape->radius;
}

// ---- ray casts in shape space -----------------------------------------------------------------------------------
// Contract (reference src/geometry.c:393-730): fraction in [0, maxFraction], outward normal, a ray that starts inside
// the shape misses.

s2RayCastOutput s2RayCastCircle(const s2RayCastInput* input, const s2Circle* shape)
{
	s2RayCastOutput out = {0};
	s2Vec2 center = shape->point;
	s2Vec2 s = s2Sub(input->p1, center);
	float length;
	s2Vec2 dir = s2GetLengthAndNormalize(&length, s2Sub(input->p2, input->p1));
	if (length == 0.0f)
	{
		return out;
	}
	// closest approach of the line to the centre, then Pythagoras for the entry point
	float t = -s2Dot(s, dir);
	s2Vec2 c = s2MulAdd(s, t, dir);
	float cc = s2Dot(c, c);
	float rr = shape->radius * shape->radius;
	if (cc > rr)
	{
		return out;
	}
	float fraction = t - sqrtf(rr - cc);
	if (fraction < 0.0f || input->maxFraction * length < fraction)
	{
		return out;
	}
	s2Vec2 hit = s2MulAdd(s, fraction, dir);
	out.fraction = fraction / length;
	out.normal = s2Normalize(hit);
	out.point = s2MulAdd(center, shape->radius, out.normal);
	out.hit = true;
	return out;
}

s2RayCastOutput s2RayCastCapsule(const s2RayCastInput* input, const s2Capsule* shape)
{
	s2RayCastOutput out = {0};
	s2Vec2 v1 = shape->point1, v2 = shape->point2;
	float capsuleLength;
	s2Vec2 axis = s2GetLengthAndNormalize(&capsuleLength, s2Sub(v2, v1));
	s2Circle cap1 = {v1, shape->radius}, cap2 = {v2, shape->radius};
	if (capsuleLength < FLT_EPSILON)
	{
		return s2RayCastCircle(input, &cap1);
	}

	s2Vec2 p1 = input->p1, p2 = input->p2;
	s2Vec2 q = s2Sub(p1, v1);
	float qa = s2Dot(q, axis);
	s2Vec2 qp = s2MulAdd(q, -qa, axis);
	float radius = shape->radius;

	if (s2Dot(qp, qp) < radius * radius)
	{
		// the ray starts inside the infinite slab of the capsule
		if (qa < 0.0f)
		{
			return s2RayCastCircle(input, &cap1);
		}
		if (qa > 1.0f)
		{
			return s2RayCastCircle(input, &cap2);
		}
		return out;
	}

	s2Vec2 n = {axis.y, -axis.x};
	float rayLength;
	s2Vec2 u = s2GetLengthAndNormalize(&rayLength, s2Sub(p2, p1));

	// intersect with the two side lines: v1 +/- radius n + s1 axis = p1 + s2 u   (Cramer)
	float den = -axis.x * u.y + u.x * axis.y;
	if (-FLT_EPSILON < den && den < FLT_EPSILON)
	{
		return out;
	}
	s2Vec2 bNeg = s2MulSub(q, radius, n);
	s2Vec2 bPos = s2MulAdd(q, radius, n);
	float invDen = 1.0f / den;
	float sNeg = (axis.x * bNeg.y - bNeg.x * axis.y) * invDen;
	float sPos = (axis.x * bPos.y - bPos.x * axis.y) * invDen;

	float s2;
	s2Vec2 b;
	if (sNeg < sPos)
	{
		s2 = sNeg;
		b = bNeg;
	}
	else
	{
		s2 = sPos;
		b = bPos;
		n = s2Neg(n);
	}
	if (s2 < 0.0f || input->maxFraction * rayLength < s2)
	{
		return out;
	}
	float s1 = (-b.x * u.y + u.x * b.y) * invDen;
	if (s1 < 0.0f)
	{
		return s2RayCastCircle(input, &cap1);
	}
	if (capsuleLength < s1)
	{
		return s2RayCastCircle(input, &cap2);
	}
	out.fraction = s2 / rayLength;
	out.point = s2Add(s2Lerp(v1, v2, s1 / capsuleLength), s2MulSV(shape->radius, n));
	out.normal = n;
	out.hit = true;
	return out;
}

s2RayCastOutput s2RayCastSegment(const s2RayCastInput* input, const s2Segment* shape)
{
	s2RayCastOutput out = {0};
	s2Vec2 p1 = input->p1;
	s2Vec2 d = s2Sub(input->p2, p1);
	s2Vec2 v1 = shape->point1;
	float length;
	s2Vec2 eUnit = s2GetLengthAndNormalize(&length, s2Sub(shape->point2, v1));
	if (length == 0.0f)
	{
		return out;
	}
	s2Vec2 normal = {eUnit.y, -eUnit.x};
	float numerator = s2Dot(normal, s2Sub(v1, p1));
	float denominator = s2Dot(normal, d);
	if (denominator == 0.0f)
	{
		return out;
	}
	float t = numerator / denominator;
	if (t < 0.0f || input->maxFraction < t)
	{
		return out;
	}
	s2Vec2 p = s2MulAdd(p1, t, d);
	float s = s2Dot(s2Sub(p, v1), eUnit);
	if (s < 0.0f || length < s)
	{
		return out;
	}
	if (numerator > 0.0f)
	{
		normal = s2Neg(normal);
	}
	out.fraction = t;
	out.normal = normal;
	out.hit = true;
	return out;
}

// clip the ray against every edge half-plane (Cyrus-Beck)
s2RayCastOutput s2RayCastPolygon(const s2RayCastInput* input, const s2Polygon* shape)
{
	s2RayCastOutput out = {0};
	s2Vec2 p1 = input->p1, p2 = input->p2;
	s2Vec2 d = s2Sub(p2, p1);
	float lower = 0.0f, upper = input->maxFraction;
	int32_t index = -1;
	for (int32_t i = 0; i < shape->count; ++i)
	{
		float numerator = s2Dot(shape->normals[i], s2Sub(shape->vertices[i], p1));
		float denominator = s2Dot(shape->normals[i], d);
		if (denominator == 0.0f)
		{
			if (numerator < 0.0f)
			{
				return out;
			}
		}
		else if (denominator < 0.0f && numerator < lower * denominator)
		{
			lower = numerator / denominator;
			index = i;
		}
		else if (denominator > 0.0f && numerator < upper * denominator)
		{
			upper = numerator / denominator;
		}
		if (upper < lower)
		{
			return out;
		}
	}
	if (index >= 0)
	{
		out.fraction = lower;
		out.normal = shape->normals[index];
		out.point = s2Lerp(p1, p2, out.fraction);
		out.hit = true;
	}
	return out;
}

// ---- public narrow-phase API (shared implementation, csrc/shared/s2_collide.h) -----------------------------------

s2SegmentDistanceResult s2SegmentDistance(s2Vec2 p1, s2Vec2 q1, s2Vec2 p2, s2Vec2 q2)
{
	return s2cSegmentDistance(p1, q1, p2, q2);
}

s2DistanceProxy s2MakeProxy(const s2Vec2* vertices, int32_t count, float radius)
{
	count = S2_MIN(count, s2_maxPolygonVertices);
	s2DistanceProxy proxy;
	for (int32_t i = 0; i < count; ++i)
	{
		proxy.vertices[i] = vertices[i];
	}
	proxy.count = count;
	proxy.radius = radius;
	return proxy;
}

s2DistanceOutput s2ShapeDistance(s2DistanceCache* cache, const s2DistanceInput* input)
{
	return s2cShapeDistance(cache, input->proxyA.vertices, input->proxyA.count, input->proxyA.radius, input->transformA,
							input->proxyB.vertices, input->proxyB.count, input->proxyB.radius, input->transformB,
							input->useRadii);
}

s2Manifold s2CollideCircles(const s2Circle* circleA, s2Transform xfA, const s2Circle* circleB, s2Transform xfB)
{
	s2Manifold m;
	s2cCollideCircles(&m, circleA->point, circleA->radius, xfA, circleB->point, circleB->radius, xfB);
	return m;
}

s2Manifold s2CollideCapsuleAndCircle(const s2Capsule* capsuleA, s2Transform xfA, const s2Circle* circleB, s2Transform xfB)
{
	s2Manifold m;
	s2cCollideCapsuleAndCircle(&m, capsuleA->point1, capsuleA->point2, capsuleA->radius, xfA, circleB->point, circleB->radius, xfB);
	return m;
}

s2Manifold s2CollideSegmentAndCircle(const s2Segment* segmentA, s2Transform xfA, const s2Circle* circleB, s2Transform xfB)
{
	s2Manifold m;
	s2cCollideCapsuleAndCircle(&m, segmentA->point1, segmentA->point2, 0.0f, xfA, circleB->point, circleB->radius, xfB);
	return m;
}

s2Manifold s2CollidePolygonAndCircle(const s2Polygon* polygonA, s2Transform xfA, const s2Circle* circleB, s2Transform xfB)
{
	s2Manifold m;
	s2cCollidePolygonAndCircle(&m, polygonA->vertices, polygonA->normals, polygonA->count, polygonA->radius, xfA, circleB->point,
							   circleB->radius, xfB);
	return m;
}

s2Manifold s2CollidePolygons(const s2Polygon* polyA, s2Transform xfA, const s2Polygon* polyB, s2Transform xfB, s2DistanceCache* cache)
{
	s2Manifold m;
	s2cCollidePolygons(&m, polyA, xfA, polyB, xfB, cache);
	return m;
}

s2Manifold s2CollideCapsules(const s2Capsule* capsuleA, s2Transform xfA, const s2Capsule* capsuleB, s2Transform xfB,
							 s2DistanceCache* cache)
{
	s2Polygon polyA = s2MakeCapsule(capsuleA->point1, capsuleA->point2, capsuleA->radius);
	s2Polygon polyB = s2MakeCapsule(capsuleB->point1, capsuleB->point2, capsuleB->radius);
	return s2CollidePolygons(&polyA, xfA, &polyB, xfB, cache);
}

s2Manifold s2CollideSegmentAndCapsule(const s2Segment* segmentA, s2Transform xfA, const s2Capsule* capsuleB, s2Transform xfB,
									  s2DistanceCache* cache)
{
	s2Polygon polyA = s2MakeCapsule(segmentA->point1, segmentA->point2, 0.0f);
	s2Polygon polyB = s2MakeCapsule(capsuleB->point1, capsuleB->point2, capsuleB->radius);
	return s2CollidePolygons(&polyA, xfA, &polyB, xfB, cache);
}

s2Manifold s2CollidePolygonAndCapsule(const s2Polygon* polygonA, s2Transform xfA, const s2Capsule* capsuleB, s2Transform xfB,
									  s2DistanceCache* cache)
{
	s2Polygon polyB = s2MakeCapsule(capsuleB->point1, capsuleB->point2, capsuleB->radius);
	return s2CollidePolygons(polygonA, xfA, &polyB, xfB, cache);
}

s2Manifold s2CollideSegmentAndPolygon(const s2Segment* segmentA, s2Transform xfA, const s2Polygon* polygonB, s2Transform xfB,
									  s2DistanceCache* cache)
{
	s2Polygon polyA = s2MakeCapsule(segmentA->point1, segmentA->point2, 0.0f);
	return s2CollidePolygons(&polyA, xfA, polygonB, xfB, cache);
}

// ---- continuous collision (shared implementation, csrc/shared/s2_toi.h) --------------------------------------------

s2Transform s2GetSweepTransform(const s2Sweep* sweep, float fraction)
{
	return s2cGetSweepTransform(sweep, fraction);
}

s2TOIOutput s2TimeOfImpact(const s2TOIInput* input)
{
	return s2cTimeOfImpact(input->proxyA.vertices, input->proxyA.count, input->proxyA.radius, &input->sweepA, input->proxyB.vertices,
						   input->proxyB.count, input->proxyB.radius, &input->sweepB, input->maxFraction);
}

s2ShapeExtent s2ComputeShapeExtent(const s2Polygon* polygonForm, s2Vec2 localCenter)
{
	s2cShapeExtent e = s2cComputeShapeExtent(polygonForm->vertices, polygonForm->normals, polygonForm->count, polygonForm->radius,
											 localCenter);
	s2ShapeExtent out = {e.inner, e.outer, e.core};
	return out;
}

s2ShapeExtent s2ComputeBodyExtent(const s2Polygon* polygonForms, int32_t count, s2Vec2 localCenter)
{
	s2ShapeExtent out = {s2_huge, 0.0f, localCenter};
	for (int32_t i = 0; i < count; ++i)
	{
		s2ShapeExtent e = s2ComputeShapeExtent(polygonForms + i, localCenter);
		out.minExtent = S2_MIN(out.minExtent, e.minExtent);
		out.maxExtent = S2_MAX(out.maxExtent, e.maxExtent);
	}
	return out;
}
