// TEST INFRASTRUCTURE — the weld joint's oracle (DESIGN.md §3.8). The reference has no weld, so this file is the weld's
// definition: plain, sequential C that the device must match bit for bit.
//
// It is the oracle of oracle/s2o_solver.c with weld rows (S2B_JOINT_WELD) added, built from that file unmodified so that
// the revolute and mouse paths stay exactly the ones tests/test_oracle_cpu.py pins to the reference. Two oracle functions
// are routed through the weld functions below, by the preprocessor:
//   * s2oJointOp, the per-constraint dispatch of every driver;
//   * s2oPrepareJointSoft, which every joint prepare runs (the rigid and XPBD prepares call it first).
// Each macro pastes the first token of its first argument onto a prefix. A definition's first parameter starts with a
// type name (s2oSolve*, s2oJoint*), which selects the oracle's own function, renamed ..._Base; every call passes a
// plain variable (s, j), which selects the weld function. The weld functions handle welds and hand every other joint
// to the _Base function.
//
// Compiled with the oracle's flags (gcc -std=gnu17 -O2, no FMA contraction) by tests/weld_oracle.py.

#include "s2b_device.h"
#include "solver2d/constants.h"
#include "solver2d/math.h"

struct s2oSolve;
struct s2oJoint;
struct s2oBody;
static void s2oWeldJointOp(struct s2oSolve* s, int op, struct s2oJoint* j);
static void s2oWeldPrepareJointSoft(struct s2oJoint* j, const s2bJointRow* row, const struct s2oBody* bodies, float contextH,
									float h, float hertz, int warmStart);

#define s2oJointOp(first, ...) S2OW_JOINT_OP_##first, __VA_ARGS__)
#define S2OW_JOINT_OP_s2oSolve s2oJointOp_Base(s2oSolve
#define S2OW_JOINT_OP_s s2oWeldJointOp(s

#define s2oPrepareJointSoft(first, ...) S2OW_PREPARE_##first, __VA_ARGS__)
#define S2OW_PREPARE_s2oJoint s2oPrepareJointSoft_Base(s2oJoint
#define S2OW_PREPARE_j s2oWeldPrepareJointSoft(j

#include "../oracle/s2o_solver.c"

#undef s2oJointOp
#undef s2oPrepareJointSoft

// ---- prepare -------------------------------------------------------------------------------------------------------

// The revolute prepare, except that the angular impulse (motorImpulse) is kept or zeroed exactly when the point
// impulse is. The XPBD prepare zeroes both afterwards.
static void s2oWeldPrepareJointSoft(s2oJoint* j, const s2bJointRow* row, const s2oBody* bodies, float contextH, float h,
									float hertz, int warmStart)
{
	s2oPrepareJointSoft_Base(j, row, bodies, contextH, h, hertz, warmStart);
	if (j->type == S2B_JOINT_WELD)
	{
		j->motorImpulse = warmStart ? row->motorImpulse : 0.0f;
	}
}

// ---- the angular row -----------------------------------------------------------------------------------------------

static float s2oWeldAngle(const s2oJoint* j, s2Rot qA, s2Rot qB)
{
	return s2UnwindAngle(s2RelativeAngle(qB, qA) - j->referenceAngle);
}

static void s2oWeldApplyAngular(s2oJoint* j, s2oBody* bodies, float impulse)
{
	j->motorImpulse += impulse;
	bodies[j->indexA].w -= j->invIA * impulse;
	bodies[j->indexB].w += j->invIB * impulse;
}

// soft (Jacobi, PGS_Soft, SoftStep, TGS_Soft): the revolute's soft angular rows with the joint softness
static void s2oWeldAngularSoft(s2oJoint* j, s2oBody* bodies, int useBias)
{
	s2oBody* bodyA = bodies + j->indexA;
	s2oBody* bodyB = bodies + j->indexB;
	float C = s2oWeldAngle(j, bodyA->q, bodyB->q);
	float bias = 0.0f, massScale = 1.0f, impulseScale = 0.0f;
	if (useBias)
	{
		bias = j->biasCoefficient * C;
		massScale = j->massCoefficient;
		impulseScale = j->impulseCoefficient;
	}
	float Cdot = bodyB->w - bodyA->w;
	float impulse = -j->axialMass * massScale * (Cdot + bias) - impulseScale * j->motorImpulse;
	s2oWeldApplyAngular(j, bodies, impulse);
}

// Baumgarte (PGS, TGS_Sticky): the bias is applied in every pass, as for this flavour's point row
static void s2oWeldAngularBaumgarte(s2oJoint* j, s2oBody* bodies, float inv_h)
{
	s2oBody* bodyA = bodies + j->indexA;
	s2oBody* bodyB = bodies + j->indexB;
	float C = s2oWeldAngle(j, bodyA->q, bodyB->q);
	float bias = s2_baumgarte * inv_h * C;
	float Cdot = bodyB->w - bodyA->w;
	float impulse = -j->axialMass * (Cdot + bias);
	s2oWeldApplyAngular(j, bodies, impulse);
}

// rigid velocity (PGS_NGS, PGS_NGS_Block, TGS_NGS): the angle error is left to the position pass
static void s2oWeldAngularRigid(s2oJoint* j, s2oBody* bodies)
{
	float Cdot = bodies[j->indexB].w - bodies[j->indexA].w;
	float impulse = -j->axialMass * Cdot;
	s2oWeldApplyAngular(j, bodies, impulse);
}

// ---- position forms: the angular row corrects the rotations the point row then uses ------------------------------

// NGS position (PGS_NGS, PGS_NGS_Block, TGS_NGS); the point row is s2oSolveRevolutePosition's
static void s2oWeldPosition(s2oJoint* j, s2oBody* bodies)
{
	s2oBody* bodyA = bodies + j->indexA;
	s2oBody* bodyB = bodies + j->indexB;
	s2Vec2 dcA = bodyA->dp, dcB = bodyB->dp;
	s2Rot qA = bodyA->q, qB = bodyB->q;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;

	if (iA + iB != 0.0f)
	{
		float C = s2oWeldAngle(j, qA, qB);
		float p = -j->axialMass * S2_CLAMP(C, -s2_maxAngularCorrection, s2_maxAngularCorrection);
		qA = s2IntegrateRot(qA, -iA * p);
		qB = s2IntegrateRot(qB, iB * p);
	}

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

// XPBD: zero compliance; the point row is s2oSolveRevoluteXpbd's
static void s2oWeldXpbd(s2oJoint* j, s2oBody* bodies)
{
	const float compliance = 0.0f;
	s2oBody* bodyA = bodies + j->indexA;
	s2oBody* bodyB = bodies + j->indexB;
	s2Vec2 dcA = bodyA->dp, dcB = bodyB->dp;
	s2Rot qA = bodyA->q, qB = bodyB->q;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;

	if (iA + iB != 0.0f)
	{
		float C = s2oWeldAngle(j, qA, qB);
		float p = -C / (iA + iB);
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
	float lambda = -c / (kA + kB + compliance);
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

// Velocity forms: the angular row, then the revolute's point row (a weld row has no limit or motor flag, so the revolute
// functions solve exactly their point row). Position forms replace the revolute's.
static void s2oWeldJointOp(s2oSolve* s, int op, s2oJoint* j)
{
	if (j->type != S2B_JOINT_WELD)
	{
		s2oJointOp_Base(s, op, j);
		return;
	}
	int angular = j->invIA + j->invIB != 0.0f;
	switch (op)
	{
		case S2O_J_SOFT_BIAS:
		case S2O_J_SOFT_RELAX:
			if (angular)
			{
				s2oWeldAngularSoft(j, s->bodies, op == S2O_J_SOFT_BIAS);
			}
			break;
		case S2O_J_BAUMGARTE_BIAS:
		case S2O_J_BAUMGARTE_RELAX:
			if (angular)
			{
				s2oWeldAngularBaumgarte(j, s->bodies, s->inv_h);
			}
			break;
		case S2O_J_RIGID:
			if (angular)
			{
				s2oWeldAngularRigid(j, s->bodies);
			}
			break;
		case S2O_J_POSITION:
			s2oWeldPosition(j, s->bodies);
			return;
		case S2O_J_XPBD:
			s2oWeldXpbd(j, s->bodies);
			return;
		default:
			break;
	}
	s2oJointOp_Base(s, op, j);
}
