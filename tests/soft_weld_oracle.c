// TEST INFRASTRUCTURE — the soft weld's oracle (DESIGN.md §3.15). The reference has no weld, soft or rigid, so this file is
// the soft weld's definition: plain, sequential C that the device must match bit for bit.
//
// It is the weld oracle (tests/weld_oracle.c, itself built on oracle/s2o_solver.c) with the weld's anchor and angle
// constraints made springs where their hertz is positive, built from both files unmodified. The weld oracle routes the
// oracle's s2oJointOp and s2oPrepareJointSoft to its own functions by the preprocessor; this file routes those two in turn,
// the same way: each macro below pastes the first token of its first argument onto a prefix. The weld file's declaration
// and definition start with a type name (struct, s2oSolve, s2oJoint) and select its own function, renamed ..._Inner; every
// call passes a plain variable (s, j) and selects the soft weld function, which hands every joint that is not a soft weld
// (every other type, and a weld with both hertz at 0) to the weld function unchanged.
//
// A weld row carries its soft parts in lanes it leaves free: the linear (anchor) pair in hertz / dampingRatio, the angular
// pair in maxMotorTorque / motorSpeed. A part with a positive hertz is soft:
//   * prepare: its velocity coefficients for the context's h, in the mouse joint's expression order (bias = omega / (2 zeta +
//     h omega), c = h omega (2 zeta + h omega), impulseScale = 1 / (1 + c), massScale = c impulseScale). The impulses are
//     the weld's (angular motorImpulse, point impulse) and are kept or dropped as the weld's.
//   * every velocity op (soft, Baumgarte, rigid; biased and relax passes): the angular row, then the point row, as the weld;
//     a soft part is impulse = -k massScale (Cdot + bias C) - impulseScale lambda, k the axial mass for the angle and, for the
//     anchor, the 2x2 effective mass of the flavour's point row (fresh in the soft and Baumgarte ops, the prepare-time pivot
//     in the rigid op). A rigid part is the weld's row of that op.
//   * the warm start: the weld's.
//   * the NGS position op: nothing for a soft part, the weld's correction for a rigid part.
//   * XPBD: a soft part is p = -(C + gamma (C - C0)) / ((1 + gamma) w + alphaTilde), alphaTilde = w / (omega h)^2,
//     gamma = 2 zeta / (omega h), C0 the error at the sub-step's start pose (dp0, q0); the anchor's acts along
//     n = separation / |separation| with C = |separation|, C0 = n . separation0 and the weld's w = kA + kB.
//
// Compiled with the oracle's flags (gcc -std=gnu17 -O2, no FMA contraction) by tests/soft_weld_oracle.py.

#include "s2b_device.h"

#include <stdlib.h>

struct s2oSolve;
struct s2oJoint;
struct s2oBody;
static void s2oSoftWeldJointOp(struct s2oSolve* s, int op, struct s2oJoint* j);
static void s2oSoftWeldPrepareJointSoft(struct s2oJoint* j, const s2bJointRow* row, const struct s2oBody* bodies, float contextH,
										float h, float hertz, int warmStart);

#define s2oWeldJointOp(first, ...) S2OSW_JOINT_OP_##first, __VA_ARGS__)
#define S2OSW_JOINT_OP_struct s2oWeldJointOp_Inner(struct
#define S2OSW_JOINT_OP_s2oSolve s2oWeldJointOp_Inner(s2oSolve
#define S2OSW_JOINT_OP_s s2oSoftWeldJointOp(s

#define s2oWeldPrepareJointSoft(first, ...) S2OSW_PREPARE_##first, __VA_ARGS__)
#define S2OSW_PREPARE_struct s2oWeldPrepareJointSoft_Inner(struct
#define S2OSW_PREPARE_s2oJoint s2oWeldPrepareJointSoft_Inner(s2oJoint
#define S2OSW_PREPARE_j s2oSoftWeldPrepareJointSoft(j

#include "weld_oracle.c"

#undef s2oWeldJointOp
#undef s2oWeldPrepareJointSoft

// ---- state -----------------------------------------------------------------------------------------------------------

typedef struct s2oSoftPart
{
	int active;
	float hertz, zeta;					 // XPBD reads these
	float bias, massScale, impulseScale; // the velocity rows' coefficients
} s2oSoftPart;

typedef struct s2oSoftWeld
{
	s2oSoftPart angular, linear;
} s2oSoftWeld;

static s2oSoftWeld* s2oSoftWelds = NULL;
static int s2oSoftWeldCapacity = 0;

static s2oSoftWeld* s2oSoftWeldOf(int slot)
{
	if (slot >= s2oSoftWeldCapacity)
	{
		int capacity = slot + 1 > 2 * s2oSoftWeldCapacity ? slot + 1 : 2 * s2oSoftWeldCapacity;
		s2oSoftWelds = (s2oSoftWeld*)realloc(s2oSoftWelds, sizeof(s2oSoftWeld) * (size_t)capacity);
		for (int i = s2oSoftWeldCapacity; i < capacity; ++i)
		{
			s2oSoftWelds[i] = (s2oSoftWeld){0};
		}
		s2oSoftWeldCapacity = capacity;
	}
	return s2oSoftWelds + slot;
}

// ---- prepare ---------------------------------------------------------------------------------------------------------

static s2oSoftPart s2oSoftPartOf(float hertz, float zeta, float contextH)
{
	s2oSoftPart p = {0};
	p.active = hertz > 0.0f;
	if (p.active)
	{
		p.hertz = hertz;
		p.zeta = zeta;
		float omega = 2.0f * s2_pi * hertz;
		p.bias = omega / (2.0f * zeta + contextH * omega);
		float c = contextH * omega * (2.0f * zeta + contextH * omega);
		p.impulseScale = 1.0f / (1.0f + c);
		p.massScale = c * p.impulseScale;
	}
	return p;
}

static void s2oSoftWeldPrepareJointSoft(s2oJoint* j, const s2bJointRow* row, const s2oBody* bodies, float contextH, float h,
										float hertz, int warmStart)
{
	s2oWeldPrepareJointSoft_Inner(j, row, bodies, contextH, h, hertz, warmStart);
	s2oSoftWeld* sw = s2oSoftWeldOf(j->slot);
	*sw = (s2oSoftWeld){0};
	if (j->type == S2B_JOINT_WELD)
	{
		sw->angular = s2oSoftPartOf(row->maxMotorTorque, row->motorSpeed, contextH);
		sw->linear = s2oSoftPartOf(row->hertz, row->dampingRatio, contextH);
	}
}

// ---- velocity rows ---------------------------------------------------------------------------------------------------

static void s2oSoftWeldAngular(s2oJoint* j, s2oBody* bodies, const s2oSoftPart* sp)
{
	s2oBody* bodyA = bodies + j->indexA;
	s2oBody* bodyB = bodies + j->indexB;
	float C = s2oWeldAngle(j, bodyA->q, bodyB->q);
	float Cdot = bodyB->w - bodyA->w;
	float impulse = -j->axialMass * sp->massScale * (Cdot + sp->bias * C) - sp->impulseScale * j->motorImpulse;
	s2oWeldApplyAngular(j, bodies, impulse);
}

// the point row as a spring; `pivot` selects the prepare-time effective mass (the rigid op) over a fresh one
static void s2oSoftWeldPoint(s2oJoint* j, s2oBody* bodies, const s2oSoftPart* sp, int pivot)
{
	s2oBody* bodyA = bodies + j->indexA;
	s2oBody* bodyB = bodies + j->indexB;
	s2Vec2 vA = bodyA->v, vB = bodyB->v;
	float wA = bodyA->w, wB = bodyB->w;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;
	s2Vec2 rA = s2RotateVector(bodyA->q, j->localAnchorA);
	s2Vec2 rB = s2RotateVector(bodyB->q, j->localAnchorB);
	s2Vec2 Cdot = s2Sub(s2Add(vB, s2CrossSV(wB, rB)), s2Add(vA, s2CrossSV(wA, rA)));
	s2Vec2 separation = s2Add(s2Add(s2Sub(bodyB->dp, bodyA->dp), s2Sub(rB, rA)), j->centerDiff0);
	s2Vec2 bias = s2MulSV(sp->bias, separation);
	s2Vec2 b;
	if (pivot)
	{
		b = s2MulMV(j->pivotMass, s2Add(Cdot, bias));
	}
	else
	{
		s2Mat22 K;
		K.cx.x = mA + mB + rA.y * rA.y * iA + rB.y * rB.y * iB;
		K.cy.x = -rA.y * rA.x * iA - rB.y * rB.x * iB;
		K.cx.y = K.cy.x;
		K.cy.y = mA + mB + rA.x * rA.x * iA + rB.x * rB.x * iB;
		b = s2Solve22(K, s2Add(Cdot, bias));
	}
	s2Vec2 impulse;
	impulse.x = -sp->massScale * b.x - sp->impulseScale * j->impulse.x;
	impulse.y = -sp->massScale * b.y - sp->impulseScale * j->impulse.y;
	j->impulse.x += impulse.x;
	j->impulse.y += impulse.y;
	bodyA->v = s2MulSub(vA, mA, impulse);
	bodyA->w = wA - iA * s2Cross(rA, impulse);
	bodyB->v = s2MulAdd(vB, mB, impulse);
	bodyB->w = wB + iB * s2Cross(rB, impulse);
}

// ---- position rows ---------------------------------------------------------------------------------------------------

// the NGS position op: the weld's correction of each rigid part (s2oWeldPosition), nothing for a soft part
static void s2oSoftWeldPosition(s2oJoint* j, s2oBody* bodies, const s2oSoftWeld* sw)
{
	if (sw->angular.active && sw->linear.active)
	{
		return;
	}
	s2oBody* bodyA = bodies + j->indexA;
	s2oBody* bodyB = bodies + j->indexB;
	s2Vec2 dcA = bodyA->dp, dcB = bodyB->dp;
	s2Rot qA = bodyA->q, qB = bodyB->q;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;

	if (sw->angular.active == 0)
	{
		if (iA + iB != 0.0f)
		{
			float C = s2oWeldAngle(j, qA, qB);
			float p = -j->axialMass * S2_CLAMP(C, -s2_maxAngularCorrection, s2_maxAngularCorrection);
			qA = s2IntegrateRot(qA, -iA * p);
			qB = s2IntegrateRot(qB, iB * p);
		}
	}
	else
	{
		s2Vec2 rA = s2RotateVector(qA, j->localAnchorA);
		s2Vec2 rB = s2RotateVector(qB, j->localAnchorB);
		s2Vec2 C = s2Add(s2Add(s2Sub(dcB, dcA), s2Sub(rB, rA)), j->centerDiff0);
		s2Mat22 K;
		K.cx.x = mA + mB + iA * rA.y * rA.y + iB * rB.y * rB.y;
		K.cx.y = -iA * rA.x * rA.y - iB * rB.x * rB.y;
		K.cy.x = K.cx.y;
		K.cy.y = mA + mB + iA * rA.x * rA.x + iB * rB.x * rB.x;
		s2Vec2 impulse = s2Solve22(K, s2Neg(C));
		dcA = s2MulSub(dcA, mA, impulse);
		qA = s2IntegrateRot(qA, -iA * s2Cross(rA, impulse));
		dcB = s2MulAdd(dcB, mB, impulse);
		qB = s2IntegrateRot(qB, iB * s2Cross(rB, impulse));
	}

	if (mA != 0.0f || iA != 0.0f)
	{
		bodyA->dp = dcA;
		bodyA->q = qA;
	}
	if (mB != 0.0f || iB != 0.0f)
	{
		bodyB->dp = dcB;
		bodyB->q = qB;
	}
}

static float s2oSoftWeldXpbdImpulse(float w, float C, float C0, float omegaH, float zeta)
{
	float alphaTilde = w / (omegaH * omegaH);
	float gamma = 2.0f * zeta / omegaH;
	return -(C + gamma * (C - C0)) / ((1.0f + gamma) * w + alphaTilde);
}

// XPBD: the weld's rows (s2oWeldXpbd) with each soft part compliant and damped
static void s2oSoftWeldXpbd(s2oSolve* s, s2oJoint* j, const s2oSoftWeld* sw)
{
	const float compliance = 0.0f;
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2Vec2 dcA = bodyA->dp, dcB = bodyB->dp;
	s2Rot qA = bodyA->q, qB = bodyB->q;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;
	float h = s->ctx->h;

	if (iA + iB != 0.0f)
	{
		float C = s2oWeldAngle(j, qA, qB);
		float p;
		if (sw->angular.active)
		{
			float omegaH = 2.0f * s2_pi * sw->angular.hertz * h;
			float C0 = s2oWeldAngle(j, bodyA->q0, bodyB->q0);
			p = s2oSoftWeldXpbdImpulse(iA + iB, C, C0, omegaH, sw->angular.zeta);
		}
		else
		{
			p = -C / (iA + iB);
		}
		qA = s2IntegrateRot(qA, -iA * p);
		qB = s2IntegrateRot(qB, iB * p);
	}

	s2Vec2 rA = s2RotateVector(qA, j->localAnchorA);
	s2Vec2 rB = s2RotateVector(qB, j->localAnchorB);
	s2Vec2 separation = s2Add(s2Add(s2Sub(dcB, dcA), s2Sub(rB, rA)), j->centerDiff0);
	float c = s2Length(separation);
	s2Vec2 n = s2Vec2_zero;
	if (c >= 0.001f * 1.1920929e-07f)
	{
		float invLength = 1.0f / c;
		n = s2MakeVec2(invLength * separation.x, invLength * separation.y);
	}
	if (mA == 0.0f && mB == 0.0f)
	{
		return;
	}
	float rnA = s2Cross(rA, n);
	float rnB = s2Cross(rB, n);
	float kA = mA + iA * rnA * rnA;
	float kB = mB + iB * rnB * rnB;
	float lambda;
	if (sw->linear.active)
	{
		float omegaH = 2.0f * s2_pi * sw->linear.hertz * h;
		s2Vec2 rA0 = s2RotateVector(bodyA->q0, j->localAnchorA);
		s2Vec2 rB0 = s2RotateVector(bodyB->q0, j->localAnchorB);
		s2Vec2 separation0 = s2Add(s2Add(s2Sub(bodyB->dp0, bodyA->dp0), s2Sub(rB0, rA0)), j->centerDiff0);
		lambda = s2oSoftWeldXpbdImpulse(kA + kB, c, s2Dot(n, separation0), omegaH, sw->linear.zeta);
	}
	else
	{
		lambda = -c / (kA + kB + compliance);
	}
	s2Vec2 p = s2MulSV(lambda, n);
	dcA = s2MulSub(dcA, mA, p);
	qA = s2IntegrateRot(qA, -iA * s2Cross(rA, p));
	dcB = s2MulAdd(dcB, mB, p);
	qB = s2IntegrateRot(qB, iB * s2Cross(rB, p));
	if (mA != 0.0f || iA != 0.0f)
	{
		bodyA->dp = dcA;
		bodyA->q = qA;
	}
	if (mB != 0.0f || iB != 0.0f)
	{
		bodyB->dp = dcB;
		bodyB->q = qB;
	}
}

// ---- dispatch --------------------------------------------------------------------------------------------------------

static void s2oSoftWeldJointOp(s2oSolve* s, int op, s2oJoint* j)
{
	s2oSoftWeld* sw = s2oSoftWeldOf(j->slot);
	if (j->type != S2B_JOINT_WELD || (sw->angular.active == 0 && sw->linear.active == 0))
	{
		s2oWeldJointOp_Inner(s, op, j);
		return;
	}
	int angular = j->invIA + j->invIB != 0.0f;
	int pivot = 0;
	switch (op)
	{
		case S2O_J_SOFT_BIAS:
		case S2O_J_SOFT_RELAX:
			if (angular)
			{
				if (sw->angular.active)
				{
					s2oSoftWeldAngular(j, s->bodies, &sw->angular);
				}
				else
				{
					s2oWeldAngularSoft(j, s->bodies, op == S2O_J_SOFT_BIAS);
				}
			}
			break;
		case S2O_J_BAUMGARTE_BIAS:
		case S2O_J_BAUMGARTE_RELAX:
			if (angular)
			{
				if (sw->angular.active)
				{
					s2oSoftWeldAngular(j, s->bodies, &sw->angular);
				}
				else
				{
					s2oWeldAngularBaumgarte(j, s->bodies, s->inv_h);
				}
			}
			break;
		case S2O_J_RIGID:
			if (angular)
			{
				if (sw->angular.active)
				{
					s2oSoftWeldAngular(j, s->bodies, &sw->angular);
				}
				else
				{
					s2oWeldAngularRigid(j, s->bodies);
				}
			}
			pivot = 1;
			break;
		case S2O_J_POSITION:
			s2oSoftWeldPosition(j, s->bodies, sw);
			return;
		case S2O_J_XPBD:
			s2oSoftWeldXpbd(s, j, sw);
			return;
		default:
			// the warm start is the weld's
			s2oJointOp_Base(s, op, j);
			return;
	}
	// the point row: a spring, or the op's rigid row (the base oracle's revolute rows solve exactly their point row for a
	// weld, which has no limit or motor flag)
	if (sw->linear.active)
	{
		s2oSoftWeldPoint(j, s->bodies, &sw->linear, pivot);
	}
	else
	{
		s2oJointOp_Base(s, op, j);
	}
}
