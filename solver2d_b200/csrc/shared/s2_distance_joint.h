// solver2d-b200 — the distance joint's line at given poses (DESIGN.md §3.16), one plain-C definition for the host (reaction
// getters, current length) and the device (reaction pass), both compiled without FMA contraction.
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
