// solver2d-b200 — the distance joint's line and the pulley joint's ropes at given poses (DESIGN.md §3.16, §3.18), one plain-C
// definition for the host (reaction getters, current lengths) and the device (reaction pass, pulley frame), both compiled
// without FMA contraction.
#pragma once

#include "s2_collide.h"

// d = (pB + qB lB) - (pA + qA lA) with p a centre of mass and l a centre-of-mass-relative anchor; returns the unit vector
// along d (zero when |d| < FLT_EPSILON) and its length
S2C_FN s2Vec2 s2cDistanceJointAxis(float* length, s2Vec2 pA, s2Rot qA, s2Vec2 lA, s2Vec2 pB, s2Rot qB, s2Vec2 lB)
{
	s2Vec2 rA = s2RotateVector(qA, lA);
	s2Vec2 rB = s2RotateVector(qB, lB);
	return s2cGetLengthAndNormalize(length, s2Sub(s2Add(pB, rB), s2Add(pA, rA)));
}

// the pulley joint's rope direction (DESIGN.md §3.18, Box2D 2.4's rule): u = d / |d|, zero when |d| <= 10 s2_linearSlop, and
// |d| in *length. The device's frame, the oracle and the host getters all form u this way.
S2C_FN s2Vec2 s2cPulleyRope(float* length, s2Vec2 d)
{
	*length = s2Length(d);
	return *length > 10.0f * s2_linearSlop ? s2MulSV(1.0f / *length, d) : s2cVec(0.0f, 0.0f);
}

// the pulley's reaction axis at given poses: -ratio uB with uB the rope direction from ground anchor B to anchor B
// = pB + qB lB (p a centre of mass, l a centre-of-mass-relative anchor); the rope's length in *length. The reaction pass
// and the host getters pass it to s2MakeJointReaction as localAxisA; with ratio 1 and side A's values it gives rope A.
S2C_FN s2Vec2 s2cPulleyJointAxis(float* length, s2Vec2 ground, s2Vec2 p, s2Rot q, s2Vec2 l, float ratio)
{
	s2Vec2 u = s2cPulleyRope(length, s2Sub(s2Add(p, s2RotateVector(q, l)), ground));
	return s2cVec(-ratio * u.x, -ratio * u.y);
}
