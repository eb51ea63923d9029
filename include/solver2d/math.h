// solver2d-b200 — vector / rotation / transform inlines (API of reference include/solver2d/math.h).
//
// These are the float expressions every stage of s2World_Step is built from. Host C, the sm_90a kernels (compiled
// with -fmad=false) and the test oracle all include this one header, so each of them evaluates the same IEEE-754
// single-precision operations in the same order as the reference CPU solver — that is what makes bit-exact
// per-stage parity possible (SURVEY.md §7 H4). Two deliberate details:
//   * S2_MIN / S2_MAX / S2_CLAMP are comparisons-and-selects (reference math.h:10-13), never fminf/fmaxf: the NaN
//     and signed-zero behaviour differs;
//   * s2NormalizeRot guards on mag > 0 and multiplies by 1.0f/mag instead of dividing (reference math.h:201-207).
#pragma once

#include "solver2d/atan2_f32.h"
#include "solver2d/constants.h"
#include "solver2d/types.h"

#include <math.h>

// atan2f as the reference's C library computes it: libm on the host, the bit-identical restatement on the device
// (see solver2d/atan2_f32.h for why CUDA's own atan2f will not do)
#if defined(__CUDA_ARCH__)
	#define S2_ATAN2F(Y, X) s2Atan2F32((Y), (X))
#else
	#define S2_ATAN2F(Y, X) atan2f((Y), (X))
#endif

#define S2_MIN(A, B) ((A) < (B) ? (A) : (B))
#define S2_MAX(A, B) ((A) > (B) ? (A) : (B))
#define S2_ABS(A) ((A) > 0.0f ? (A) : -(A))
#define S2_CLAMP(A, B, C) S2_MIN(S2_MAX(A, B), C)

static const s2Vec2 s2Vec2_zero = {0.0f, 0.0f};
static const s2Rot s2Rot_identity = {0.0f, 1.0f};
static const s2Transform s2Transform_identity = {{0.0f, 0.0f}, {0.0f, 1.0f}};
static const s2Mat22 s2Mat22_zero = {{0.0f, 0.0f}, {0.0f, 0.0f}};

#ifdef __cplusplus
extern "C"
{
#endif

// out-of-line helpers (host library)
bool s2IsValid(float a);
bool s2IsValidVec2(s2Vec2 v);
s2Vec2 s2Normalize(s2Vec2 v);
s2Vec2 s2NormalizeChecked(s2Vec2 v);
s2Vec2 s2GetLengthAndNormalize(float* length, s2Vec2 v);

#ifdef __cplusplus
}
#endif

// ---- construction ---------------------------------------------------------------------------------------------

S2_INLINE s2Vec2 s2MakeVec2(float x, float y)
{
	s2Vec2 v = {x, y};
	return v;
}

// ---- products ---------------------------------------------------------------------------------------------------

S2_INLINE float s2Dot(s2Vec2 a, s2Vec2 b)
{
	return a.x * b.x + a.y * b.y;
}

// z-component of the 3D cross product
S2_INLINE float s2Cross(s2Vec2 a, s2Vec2 b)
{
	return a.x * b.y - a.y * b.x;
}

// v x (s k)
S2_INLINE s2Vec2 s2CrossVS(s2Vec2 v, float s)
{
	s2Vec2 r = {s * v.y, -s * v.x};
	return r;
}

// (s k) x v
S2_INLINE s2Vec2 s2CrossSV(float s, s2Vec2 v)
{
	s2Vec2 r = {-s * v.y, s * v.x};
	return r;
}

// clockwise quarter turn, equals s2CrossVS(v, 1)
S2_INLINE s2Vec2 s2RightPerp(s2Vec2 v)
{
	s2Vec2 r = {v.y, -v.x};
	return r;
}

// counter-clockwise quarter turn, equals s2CrossSV(1, v)
S2_INLINE s2Vec2 s2LeftPerp(s2Vec2 v)
{
	s2Vec2 r = {-v.y, v.x};
	return r;
}

// ---- arithmetic -------------------------------------------------------------------------------------------------

S2_INLINE s2Vec2 s2Add(s2Vec2 a, s2Vec2 b)
{
	s2Vec2 r = {a.x + b.x, a.y + b.y};
	return r;
}

S2_INLINE s2Vec2 s2Sub(s2Vec2 a, s2Vec2 b)
{
	s2Vec2 r = {a.x - b.x, a.y - b.y};
	return r;
}

S2_INLINE s2Vec2 s2Neg(s2Vec2 a)
{
	s2Vec2 r = {-a.x, -a.y};
	return r;
}

S2_INLINE s2Vec2 s2Lerp(s2Vec2 a, s2Vec2 b, float t)
{
	s2Vec2 r = {a.x + t * (b.x - a.x), a.y + t * (b.y - a.y)};
	return r;
}

S2_INLINE s2Vec2 s2Mul(s2Vec2 a, s2Vec2 b)
{
	s2Vec2 r = {a.x * b.x, a.y * b.y};
	return r;
}

S2_INLINE s2Vec2 s2MulSV(float s, s2Vec2 v)
{
	s2Vec2 r = {s * v.x, s * v.y};
	return r;
}

// a + s b
S2_INLINE s2Vec2 s2MulAdd(s2Vec2 a, float s, s2Vec2 b)
{
	s2Vec2 r = {a.x + s * b.x, a.y + s * b.y};
	return r;
}

// a - s b
S2_INLINE s2Vec2 s2MulSub(s2Vec2 a, float s, s2Vec2 b)
{
	s2Vec2 r = {a.x - s * b.x, a.y - s * b.y};
	return r;
}

S2_INLINE s2Vec2 s2Abs(s2Vec2 a)
{
	s2Vec2 r;
	r.x = S2_ABS(a.x);
	r.y = S2_ABS(a.y);
	return r;
}

S2_INLINE s2Vec2 s2Min(s2Vec2 a, s2Vec2 b)
{
	s2Vec2 r;
	r.x = S2_MIN(a.x, b.x);
	r.y = S2_MIN(a.y, b.y);
	return r;
}

S2_INLINE s2Vec2 s2Max(s2Vec2 a, s2Vec2 b)
{
	s2Vec2 r;
	r.x = S2_MAX(a.x, b.x);
	r.y = S2_MAX(a.y, b.y);
	return r;
}

S2_INLINE s2Vec2 s2Clamp(s2Vec2 v, s2Vec2 lo, s2Vec2 hi)
{
	s2Vec2 r;
	r.x = S2_CLAMP(v.x, lo.x, hi.x);
	r.y = S2_CLAMP(v.y, lo.y, hi.y);
	return r;
}

// ---- norms ------------------------------------------------------------------------------------------------------

S2_INLINE float s2Length(s2Vec2 v)
{
	return sqrtf(v.x * v.x + v.y * v.y);
}

S2_INLINE float s2LengthSquared(s2Vec2 v)
{
	return v.x * v.x + v.y * v.y;
}

S2_INLINE float s2Distance(s2Vec2 a, s2Vec2 b)
{
	float dx = b.x - a.x;
	float dy = b.y - a.y;
	return sqrtf(dx * dx + dy * dy);
}

S2_INLINE float s2DistanceSquared(s2Vec2 a, s2Vec2 b)
{
	float dx = b.x - a.x;
	float dy = b.y - a.y;
	return dx * dx + dy * dy;
}

// ---- rotations --------------------------------------------------------------------------------------------------

S2_INLINE s2Rot s2MakeRot(float angle)
{
	s2Rot q = {sinf(angle), cosf(angle)};
	return q;
}

S2_INLINE s2Rot s2NormalizeRot(s2Rot q)
{
	float mag = sqrtf(q.s * q.s + q.c * q.c);
	// the reference writes `mag > 0.0` (a double compare); float->double is exact, so `> 0.0f` selects identically
	float invMag = mag > 0.0f ? 1.0f / mag : 0.0f;
	s2Rot qn = {q.s * invMag, q.c * invMag};
	return qn;
}

// One explicit Euler step of (sin, cos) by the angle increment omega*h, then renormalise
// (reference math.h:209-223; one sqrtf and one divide).
S2_INLINE s2Rot s2IntegrateRot(s2Rot q1, float omegah)
{
	s2Rot q2 = {q1.s + omegah * q1.c, q1.c - omegah * q1.s};
	return s2NormalizeRot(q2);
}

// inverse of s2IntegrateRot to first order: sin(a2 - a1) / h
S2_INLINE float s2ComputeAngularVelocity(s2Rot q1, s2Rot q2, float inv_h)
{
	return inv_h * (q2.s * q1.c - q2.c * q1.s);
}

S2_INLINE float s2Rot_GetAngle(s2Rot q)
{
	return S2_ATAN2F(q.s, q.c);
}

S2_INLINE s2Vec2 s2Rot_GetXAxis(s2Rot q)
{
	s2Vec2 v = {q.c, q.s};
	return v;
}

S2_INLINE s2Vec2 s2Rot_GetYAxis(s2Rot q)
{
	s2Vec2 v = {-q.s, q.c};
	return v;
}

// composition b * a (angle addition)
S2_INLINE s2Rot s2MulRot(s2Rot b, s2Rot a)
{
	s2Rot r;
	r.s = b.s * a.c + b.c * a.s;
	r.c = b.c * a.c - b.s * a.s;
	return r;
}

// inverse(b) * a (angle subtraction a - b)
S2_INLINE s2Rot s2InvMulRot(s2Rot b, s2Rot a)
{
	s2Rot r;
	r.s = b.c * a.s - b.s * a.c;
	r.c = b.c * a.c + b.s * a.s;
	return r;
}

// angle of b relative to a
S2_INLINE float s2RelativeAngle(s2Rot b, s2Rot a)
{
	float s = b.s * a.c - b.c * a.s;
	float c = b.c * a.c + b.s * a.s;
	return S2_ATAN2F(s, c);
}

// Brings an angle difference into [-pi, pi] with one add or subtract of 2 pi: enough for the difference of two angles
// in [-pi, pi], such as the weld joint's relative angle minus its reference angle.
S2_INLINE float s2UnwindAngle(float angle)
{
	if (angle < -s2_pi)
	{
		return angle + 2.0f * s2_pi;
	}
	if (angle > s2_pi)
	{
		return angle - 2.0f * s2_pi;
	}
	return angle;
}

// v scaled back to length maxLength when it is longer, else v itself: the unit vector is formed as s2Normalize forms it
// (one sqrtf, then a multiply by 1 / length), so host and device agree bit for bit. Caps the motor joint's linear impulse.
S2_INLINE s2Vec2 s2ClampLength(s2Vec2 v, float maxLength)
{
	float lengthSquared = v.x * v.x + v.y * v.y;
	if (lengthSquared > maxLength * maxLength)
	{
		float invLength = 1.0f / sqrtf(lengthSquared);
		s2Vec2 n = {invLength * v.x, invLength * v.y};
		s2Vec2 r = {maxLength * n.x, maxLength * n.y};
		return r;
	}
	return v;
}

S2_INLINE s2Vec2 s2RotateVector(s2Rot q, s2Vec2 v)
{
	s2Vec2 r = {q.c * v.x - q.s * v.y, q.s * v.x + q.c * v.y};
	return r;
}

S2_INLINE s2Vec2 s2InvRotateVector(s2Rot q, s2Vec2 v)
{
	s2Vec2 r = {q.c * v.x + q.s * v.y, -q.s * v.x + q.c * v.y};
	return r;
}

// ---- transforms -------------------------------------------------------------------------------------------------

S2_INLINE s2Vec2 s2TransformPoint(s2Transform xf, const s2Vec2 p)
{
	float x = (xf.q.c * p.x - xf.q.s * p.y) + xf.p.x;
	float y = (xf.q.s * p.x + xf.q.c * p.y) + xf.p.y;
	s2Vec2 r = {x, y};
	return r;
}

S2_INLINE s2Vec2 s2InvTransformPoint(s2Transform xf, const s2Vec2 p)
{
	float vx = p.x - xf.p.x;
	float vy = p.y - xf.p.y;
	s2Vec2 r = {xf.q.c * vx + xf.q.s * vy, -xf.q.s * vx + xf.q.c * vy};
	return r;
}

// A * B : first B, then A
S2_INLINE s2Transform s2MulTransforms(s2Transform A, s2Transform B)
{
	s2Transform C;
	C.q = s2MulRot(A.q, B.q);
	C.p = s2Add(s2RotateVector(A.q, B.p), A.p);
	return C;
}

// inverse(A) * B : B expressed in A's frame
S2_INLINE s2Transform s2InvMulTransforms(s2Transform A, s2Transform B)
{
	s2Transform C;
	C.q = s2InvMulRot(A.q, B.q);
	C.p = s2InvRotateVector(A.q, s2Sub(B.p, A.p));
	return C;
}

// ---- 2x2 --------------------------------------------------------------------------------------------------------

S2_INLINE s2Vec2 s2MulMV(s2Mat22 A, s2Vec2 v)
{
	s2Vec2 u = {A.cx.x * v.x + A.cy.x * v.y, A.cx.y * v.x + A.cy.y * v.y};
	return u;
}

// inverse; a singular matrix yields the adjugate scaled by its zero determinant (reference math.h:386-402)
S2_INLINE s2Mat22 s2GetInverse22(s2Mat22 A)
{
	float a = A.cx.x, b = A.cy.x, c = A.cx.y, d = A.cy.y;
	float det = a * d - b * c;
	if (det != 0.0f)
	{
		det = 1.0f / det;
	}
	s2Mat22 B;
	B.cx.x = det * d;
	B.cy.x = -det * b;
	B.cx.y = -det * c;
	B.cy.y = det * a;
	return B;
}

// solve A x = b by Cramer's rule (reference math.h:406-420)
S2_INLINE s2Vec2 s2Solve22(s2Mat22 A, s2Vec2 b)
{
	float a11 = A.cx.x, a12 = A.cy.x, a21 = A.cx.y, a22 = A.cy.y;
	float det = a11 * a22 - a12 * a21;
	if (det != 0.0f)
	{
		det = 1.0f / det;
	}
	s2Vec2 x = {det * (a22 * b.x - a12 * b.y), det * (a11 * b.y - a21 * b.x)};
	return x;
}
