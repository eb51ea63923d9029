// solver2d-b200 — the gear joint's two sides at given poses (DESIGN.md §3.19), one plain-C definition for the device (solver
// rows, reaction pass), the host (constant at creation, reaction getters) and the test oracle, all compiled without FMA
// contraction, so all three agree bit for bit.
//
// A side is the linked joint's coordinate as a function of the geared body alone, its frame body being static:
//   revolute   angle(q) - angle(qC) - referenceAngle, unwound: it does not wrap at +/- pi. Jv = 0, Jw = 1.
//   prismatic  (c + q l - pC) . u with pC the world anchor and u the world axis. Jv = u, Jw = (q l) x u.
#pragma once

#include "s2_collide.h"

#include <math.h>

typedef struct s2cGearSide
{
	s2Vec2 Jv;
	float Jw;
	float coordinate;
} s2cGearSide;

// any angle brought into [-pi, pi] (s2UnwindAngle adds or subtracts 2 pi once, too little for a difference of unwound angles)
S2C_FN float s2cGearUnwind(float angle)
{
	return angle - (2.0f * s2_pi) * rintf(angle * (0.5f / s2_pi));
}

// A revolute side: the frame's rotation (qs, qc), its reference angle and theta, the side's unwound coordinate at the start
// of the step. The coordinate is the relative angle at q taken to the turn nearest theta.
S2C_FN s2cGearSide s2cGearRevolute(float qs, float qc, float referenceAngle, float theta, s2Rot q)
{
	s2Rot qC;
	qC.s = qs;
	qC.c = qc;
	s2cGearSide side;
	side.Jv = s2cVec(0.0f, 0.0f);
	side.Jw = 1.0f;
	side.coordinate = theta + s2cGearUnwind(s2RelativeAngle(q, qC) - referenceAngle - theta);
	return side;
}

// A prismatic side: d0 = the body's centre at the start of the step minus the world anchor, u the world axis, dc the
// body's centre moved since the start, l its centre-of-mass-relative anchor. (The host passes dc = 0 and d0 = c - pC.)
S2C_FN s2cGearSide s2cGearPrismatic(s2Vec2 d0, s2Vec2 u, s2Vec2 dc, s2Rot q, s2Vec2 l)
{
	s2Vec2 r = s2RotateVector(q, l);
	s2cGearSide side;
	side.Jv = u;
	side.Jw = s2Cross(r, u);
	side.coordinate = s2Dot(s2Add(s2Add(dc, r), d0), u);
	return side;
}

// a side's share of the row's inverse mass before the ratio: m Jv.Jv + i Jw^2
S2C_FN float s2cGearSideMass(s2cGearSide side, float m, float i)
{
	return m * s2Dot(side.Jv, side.Jv) + i * (side.Jw * side.Jw);
}

// The gear's impulse lambda on body B as (lambda Jv2, lambda Jw2), side 2's Jacobian scaled by the ratio: the force in the
// return value and the torque in *angular. The reaction pass and the host getters pass them to s2MakeJointReaction.
S2C_FN s2Vec2 s2cGearReaction(float* angular, float lambda, float ratio, s2cGearSide side2)
{
	float s = ratio * lambda;
	*angular = s * side2.Jw;
	return s2cVec(s * side2.Jv.x, s * side2.Jv.y);
}
