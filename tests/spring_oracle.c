// TEST INFRASTRUCTURE — the joint spring's oracle (DESIGN.md §3.14). The reference has no joint spring, so this file is its
// definition: plain, sequential C that the device must match bit for bit.
//
// It is the prismatic oracle (tests/prismatic_oracle.c, itself built on oracle/s2o_solver.c) with a spring row added to
// revolute and prismatic joints, built from both files unmodified. The prismatic oracle routes the oracle's s2oJointOp and
// s2oPrepareJointSoft to its own functions by the preprocessor; this file routes those two in turn, the same way: each
// macro below pastes the first token of its first argument onto a prefix. The prismatic file's declaration and definition
// start with a type name (struct, s2oSolve, s2oJoint) and select its own function, renamed ..._Inner; every call passes a
// plain variable (s, j) and selects the spring function, which then hands the joint on to the prismatic function, which
// hands every joint that is not prismatic on to the base oracle.
//
// The spring acts on a row with S2B_JOINT_ENABLE_SPRING, a positive hertz and, on a revolute row, a rotation to act on
// (invIA + invIB > 0). Its state lives beside the oracle's joint struct, in a table indexed by joint slot, and its
// accumulated impulse is written back to the row's springImpulse as it changes.
//   * prepare: the velocity coefficients from hertz and dampingRatio for the context's h, in the mouse joint's expression
//     order (oracle/s2o_solver.c, s2oPrepareJointSoft); the impulse kept exactly when the point impulse is, else 0.
//   * every velocity op (soft, Baumgarte, rigid, biased and relax passes): the spring row, then the joint's own rows.
//   * the warm start: the joint's own, with the spring impulse added to the axial sum (spring + motor + lower - upper).
//   * the NGS position op: nothing more.
//   * XPBD: a compliant row with damping on the sub-step's start pose, then the joint's own rows.
//
// Compiled with the oracle's flags (gcc -std=gnu17 -O2, no FMA contraction) by tests/spring_oracle.py.

#include "s2b_device.h"

#include <stdlib.h>

struct s2oSolve;
struct s2oJoint;
struct s2oBody;
static void s2oSpringJointOp(struct s2oSolve* s, int op, struct s2oJoint* j);
static void s2oSpringPrepareJointSoft(struct s2oJoint* j, const s2bJointRow* row, const struct s2oBody* bodies, float contextH,
									  float h, float hertz, int warmStart);

#define s2oPrismaticJointOp(first, ...) S2OS_JOINT_OP_##first, __VA_ARGS__)
#define S2OS_JOINT_OP_struct s2oPrismaticJointOp_Inner(struct
#define S2OS_JOINT_OP_s2oSolve s2oPrismaticJointOp_Inner(s2oSolve
#define S2OS_JOINT_OP_s s2oSpringJointOp(s

#define s2oPrismaticPrepareJointSoft(first, ...) S2OS_PREPARE_##first, __VA_ARGS__)
#define S2OS_PREPARE_struct s2oPrismaticPrepareJointSoft_Inner(struct
#define S2OS_PREPARE_s2oJoint s2oPrismaticPrepareJointSoft_Inner(s2oJoint
#define S2OS_PREPARE_j s2oSpringPrepareJointSoft(j

#include "prismatic_oracle.c"

#undef s2oPrismaticJointOp
#undef s2oPrismaticPrepareJointSoft

// ---- state -----------------------------------------------------------------------------------------------------------

typedef struct s2oSpring
{
	int active;
	float bias, massScale, impulseScale; // the velocity rows' coefficients
	float lambda;						 // accumulated impulse
} s2oSpring;

static s2oSpring* s2oSprings = NULL;
static int s2oSpringCapacity = 0;

static s2oSpring* s2oSpringOf(int slot)
{
	if (slot >= s2oSpringCapacity)
	{
		int capacity = slot + 1 > 2 * s2oSpringCapacity ? slot + 1 : 2 * s2oSpringCapacity;
		s2oSprings = (s2oSpring*)realloc(s2oSprings, sizeof(s2oSpring) * (size_t)capacity);
		for (int i = s2oSpringCapacity; i < capacity; ++i)
		{
			s2oSprings[i] = (s2oSpring){0};
		}
		s2oSpringCapacity = capacity;
	}
	return s2oSprings + slot;
}

// ---- prepare ---------------------------------------------------------------------------------------------------------

static void s2oSpringPrepareJointSoft(s2oJoint* j, const s2bJointRow* row, const s2oBody* bodies, float contextH, float h,
									  float hertz, int warmStart)
{
	s2oPrismaticPrepareJointSoft_Inner(j, row, bodies, contextH, h, hertz, warmStart);
	s2oSpring* sp = s2oSpringOf(j->slot);
	*sp = (s2oSpring){0};
	int type = j->type;
	sp->active = (row->flags & S2B_JOINT_ENABLE_SPRING) != 0 && (type == S2B_JOINT_REVOLUTE || type == S2B_JOINT_PRISMATIC) &&
				 row->hertz > 0.0f && (type == S2B_JOINT_PRISMATIC || j->invIA + j->invIB != 0.0f);
	if (sp->active)
	{
		float zeta = row->dampingRatio;
		float omega = 2.0f * s2_pi * row->hertz;
		sp->bias = omega / (2.0f * zeta + contextH * omega);
		float c = contextH * omega * (2.0f * zeta + contextH * omega);
		sp->impulseScale = 1.0f / (1.0f + c);
		sp->massScale = c * sp->impulseScale;
		sp->lambda = warmStart ? row->springImpulse : 0.0f;
	}
	// the rows the driver hands in are the caller's (s2oSolve.jointRows): the impulse is stored as it changes
	((s2bJointRow*)row)->springImpulse = sp->lambda;
}

// ---- rows ------------------------------------------------------------------------------------------------------------

static float s2oSpringImpulse(float k, float C, float Cdot, const s2oSpring* sp)
{
	return -k * sp->massScale * (Cdot + sp->bias * C) - sp->impulseScale * sp->lambda;
}

static float s2oSpringXpbdImpulse(float w, float C, float C0, float omegaH, float zeta)
{
	float alphaTilde = w / (omegaH * omegaH);
	float gamma = 2.0f * zeta / omegaH;
	return -(C + gamma * (C - C0)) / ((1.0f + gamma) * w + alphaTilde);
}

// A body's new state is stored only when it has mass or inertia: the joint's own rows then read the bodies as the device's
// do after its spring row has stored them.
static void s2oSpringStore(const s2oJoint* j, s2oBody* bodyA, s2oBody* bodyB, s2oBody a, s2oBody b)
{
	if (j->invMassA != 0.0f || j->invIA != 0.0f)
	{
		*bodyA = a;
	}
	if (j->invMassB != 0.0f || j->invIB != 0.0f)
	{
		*bodyB = b;
	}
}

static void s2oSpringVelocity(s2oSolve* s, s2oJoint* j, s2oSpring* sp)
{
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2oBody a = *bodyA, b = *bodyB;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;
	if (j->type == S2B_JOINT_REVOLUTE)
	{
		float C = s2UnwindAngle(s2RelativeAngle(b.q, a.q) - j->referenceAngle);
		float impulse = s2oSpringImpulse(j->axialMass, C, b.w - a.w, sp);
		sp->lambda += impulse;
		a.w -= iA * impulse;
		b.w += iB * impulse;
	}
	else
	{
		s2oPrismaticFrame f = s2oPrismaticFrameAt(s, j, a.dp, a.q, b.dp, b.q);
		s2Vec2 axis = f.axis;
		s2Vec2 dA = s2Add(f.d, f.rA);
		float translation = s2Dot(axis, f.d);
		float a1 = s2Cross(dA, axis), a2 = s2Cross(f.rB, axis);
		float k = mA + mB + iA * a1 * a1 + iB * a2 * a2;
		float axialMass = k > 0.0f ? 1.0f / k : 0.0f;
		float Cdot = s2Dot(axis, s2Sub(b.v, a.v)) + a2 * b.w - a1 * a.w;
		float impulse = s2oSpringImpulse(axialMass, translation, Cdot, sp);
		sp->lambda += impulse;
		s2Vec2 P = s2MulSV(impulse, axis);
		a.v = s2MulSub(a.v, mA, P);
		a.w -= iA * (impulse * a1);
		b.v = s2MulAdd(b.v, mB, P);
		b.w += iB * (impulse * a2);
	}
	s2oSpringStore(j, bodyA, bodyB, a, b);
	s->jointRows[j->slot].springImpulse = sp->lambda;
}

// rotations are integrated only where they can change (s2IntegrateRot renormalizes even by a zero angle)
static void s2oSpringXpbd(s2oSolve* s, s2oJoint* j)
{
	const s2bJointRow* row = s->jointRows + j->slot;
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2oBody a = *bodyA, b = *bodyB;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;
	float omegaH = 2.0f * s2_pi * row->hertz * s->ctx->h;
	float zeta = row->dampingRatio;
	if (j->type == S2B_JOINT_REVOLUTE)
	{
		float C = s2UnwindAngle(s2RelativeAngle(b.q, a.q) - j->referenceAngle);
		float C0 = s2UnwindAngle(s2RelativeAngle(b.q0, a.q0) - j->referenceAngle);
		float p = s2oSpringXpbdImpulse(iA + iB, C, C0, omegaH, zeta);
		if (iA != 0.0f)
		{
			a.q = s2IntegrateRot(a.q, -iA * p);
		}
		if (iB != 0.0f)
		{
			b.q = s2IntegrateRot(b.q, iB * p);
		}
		s2oSpringStore(j, bodyA, bodyB, a, b);
		return;
	}
	s2oPrismaticFrame f0 = s2oPrismaticFrameAt(s, j, a.dp0, a.q0, b.dp0, b.q0);
	s2oPrismaticFrame f = s2oPrismaticFrameAt(s, j, a.dp, a.q, b.dp, b.q);
	float a1 = s2Cross(s2Add(f.d, f.rA), f.axis), a2 = s2Cross(f.rB, f.axis);
	float k = mA + mB + iA * a1 * a1 + iB * a2 * a2;
	if (k > 0.0f)
	{
		float lambda = s2oSpringXpbdImpulse(k, s2Dot(f.axis, f.d), s2Dot(f0.axis, f0.d), omegaH, zeta);
		s2Vec2 P = s2MulSV(lambda, f.axis);
		a.dp = s2MulSub(a.dp, mA, P);
		b.dp = s2MulAdd(b.dp, mB, P);
		if (iA != 0.0f)
		{
			a.q = s2IntegrateRot(a.q, -iA * (lambda * a1));
		}
		if (iB != 0.0f)
		{
			b.q = s2IntegrateRot(b.q, iB * (lambda * a2));
		}
		s2oSpringStore(j, bodyA, bodyB, a, b);
	}
}

// the joint's warm start with axial = spring + motor + lower - upper
static void s2oSpringWarmStart(s2oSolve* s, s2oJoint* j, const s2oSpring* sp)
{
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	float axialImpulse = sp->lambda + j->motorImpulse + j->lowerImpulse - j->upperImpulse;
	if (j->type == S2B_JOINT_REVOLUTE)
	{
		s2Vec2 rA = s2RotateVector(bodyA->q, j->localAnchorA);
		s2Vec2 rB = s2RotateVector(bodyB->q, j->localAnchorB);
		s2Vec2 P = j->impulse;
		bodyA->v = s2MulSub(bodyA->v, j->invMassA, P);
		bodyA->w -= j->invIA * (s2Cross(rA, P) + axialImpulse);
		bodyB->v = s2MulAdd(bodyB->v, j->invMassB, P);
		bodyB->w += j->invIB * (s2Cross(rB, P) + axialImpulse);
		return;
	}
	s2oPrismaticFrame f = s2oPrismaticFrameAt(s, j, bodyA->dp, bodyA->q, bodyB->dp, bodyB->q);
	s2Vec2 perp = s2LeftPerp(f.axis);
	s2Vec2 dA = s2Add(f.d, f.rA);
	s2Vec2 P = s2Add(s2MulSV(axialImpulse, f.axis), s2MulSV(j->impulse.x, perp));
	float LA = axialImpulse * s2Cross(dA, f.axis) + j->impulse.x * s2Cross(dA, perp) + j->impulse.y;
	float LB = axialImpulse * s2Cross(f.rB, f.axis) + j->impulse.x * s2Cross(f.rB, perp) + j->impulse.y;
	bodyA->v = s2MulSub(bodyA->v, j->invMassA, P);
	bodyA->w = bodyA->w - j->invIA * LA;
	bodyB->v = s2MulAdd(bodyB->v, j->invMassB, P);
	bodyB->w = bodyB->w + j->invIB * LB;
}

// ---- dispatch --------------------------------------------------------------------------------------------------------

static void s2oSpringJointOp(s2oSolve* s, int op, s2oJoint* j)
{
	s2oSpring* sp = s2oSpringOf(j->slot);
	if (sp->active)
	{
		switch (op)
		{
			case S2O_J_WARM:
				s2oSpringWarmStart(s, j, sp);
				return;
			case S2O_J_SOFT_BIAS:
			case S2O_J_SOFT_RELAX:
			case S2O_J_BAUMGARTE_BIAS:
			case S2O_J_BAUMGARTE_RELAX:
			case S2O_J_RIGID:
				s2oSpringVelocity(s, j, sp);
				break;
			case S2O_J_XPBD:
				s2oSpringXpbd(s, j);
				break;
			default:
				break;
		}
	}
	s2oPrismaticJointOp_Inner(s, op, j);
}
