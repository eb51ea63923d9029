// TEST INFRASTRUCTURE — the motor joint's oracle (DESIGN.md §3.10). The reference has no motor joint, so this file is its
// definition: plain, sequential C that the device must match bit for bit.
//
// It is the oracle of oracle/s2o_solver.c with motor rows (S2B_JOINT_MOTOR) added, built from that file unmodified so that
// the revolute and mouse paths stay exactly the ones tests/test_oracle_cpu.py pins to the reference. Two oracle functions
// are routed through the motor functions below by the preprocessor, as tests/prismatic_oracle.c does for the prismatic
// joint:
//   * s2oJointOp, the per-constraint dispatch of every driver;
//   * s2oPrepareJointSoft, which every joint prepare runs (the rigid and XPBD prepares call it first).
// Each macro pastes the first token of its first argument onto a prefix. A definition's first parameter starts with a
// type name (s2oSolve*, s2oJoint*), which selects the oracle's own function, renamed ..._Base; every call passes a plain
// variable (s, j), which selects the motor function. The motor functions handle motor rows and hand every other joint to
// the _Base function.
//
// A motor row reuses the revolute's fields: localOriginAnchorA is the linear offset and localOriginAnchorB is zero (so the
// revolute prepare forms the anchors lA = offset - localCenterA, lB = -localCenterB), referenceAngle is the angular
// offset, maxMotorTorque the maximum torque, impulse the linear impulse and motorImpulse the angular impulse. The maximum
// force (hertz) and the correction factor (dampingRatio) are read from the joint's row.
//
// Compiled with the oracle's flags (gcc -std=gnu17 -O2, no FMA contraction) by tests/motor_oracle.py.

#include "s2b_device.h"
#include "solver2d/constants.h"
#include "solver2d/math.h"

struct s2oSolve;
struct s2oJoint;
struct s2oBody;
static void s2oMotorJointOp(struct s2oSolve* s, int op, struct s2oJoint* j);
static void s2oMotorPrepareJointSoft(struct s2oJoint* j, const s2bJointRow* row, const struct s2oBody* bodies, float contextH,
									 float h, float hertz, int warmStart);

#define s2oJointOp(first, ...) S2OM_JOINT_OP_##first, __VA_ARGS__)
#define S2OM_JOINT_OP_s2oSolve s2oJointOp_Base(s2oSolve
#define S2OM_JOINT_OP_s s2oMotorJointOp(s

#define s2oPrepareJointSoft(first, ...) S2OM_PREPARE_##first, __VA_ARGS__)
#define S2OM_PREPARE_s2oJoint s2oPrepareJointSoft_Base(s2oJoint
#define S2OM_PREPARE_j s2oMotorPrepareJointSoft(j

#include "../oracle/s2o_solver.c"

#undef s2oJointOp
#undef s2oPrepareJointSoft

// ---- prepare -------------------------------------------------------------------------------------------------------

// The revolute prepare, then the motor's impulse policy: the linear and the angular impulse are both kept exactly when the
// revolute point impulse would be (a warm start); the limit impulses are zero. (The revolute's fixedRotation zeroing of the
// angular impulse does not apply: the angular row is skipped instead.) The XPBD prepare zeroes all of them afterwards.
static void s2oMotorPrepareJointSoft(s2oJoint* j, const s2bJointRow* row, const s2oBody* bodies, float contextH, float h,
									 float hertz, int warmStart)
{
	s2oPrepareJointSoft_Base(j, row, bodies, contextH, h, hertz, warmStart);
	if (j->type == S2B_JOINT_MOTOR)
	{
		j->impulse = warmStart ? s2MakeVec2(row->impulse[0], row->impulse[1]) : s2Vec2_zero;
		j->motorImpulse = warmStart ? row->motorImpulse : 0.0f;
		j->lowerImpulse = 0.0f;
		j->upperImpulse = 0.0f;
	}
}

static float s2oMotorMaxForce(const s2oSolve* s, const s2oJoint* j)
{
	return s->jointRows[j->slot].hertz;
}

static float s2oMotorCorrection(const s2oSolve* s, const s2oJoint* j)
{
	return s->jointRows[j->slot].dampingRatio;
}

// ---- velocity rows -----------------------------------------------------------------------------------------------------

// The same two rows in every velocity pass (soft, Baumgarte and rigid; biased and relax): the bias is the drive.
//   angular: impulse = -(wB - wA + cf / h * C) / (iA + iB), the accumulated impulse clamped to +/- h maxTorque; skipped
//            when iA + iB == 0;
//   linear:  impulse = -K^-1 (Cdot + cf / h * C) with the revolute's 2x2 mass at the current anchors, the accumulated
//            impulse scaled back to length h maxForce.
static void s2oMotorVelocity(s2oSolve* s, s2oJoint* j)
{
	float h = s->h, inv_h = s->inv_h;
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2Vec2 vA = bodyA->v, vB = bodyB->v;
	float wA = bodyA->w, wB = bodyB->w;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;
	s2Rot qA = bodyA->q, qB = bodyB->q;
	float biasScale = s2oMotorCorrection(s, j) * inv_h;

	if (iA + iB != 0.0f)
	{
		float k = 1.0f / (iA + iB);
		float C = s2UnwindAngle(s2RelativeAngle(qB, qA) - j->referenceAngle);
		float impulse = -k * (wB - wA + biasScale * C);
		float oldImpulse = j->motorImpulse;
		float maxImpulse = h * j->maxMotorTorque;
		j->motorImpulse = S2_CLAMP(oldImpulse + impulse, -maxImpulse, maxImpulse);
		impulse = j->motorImpulse - oldImpulse;
		wA -= iA * impulse;
		wB += iB * impulse;
	}

	{
		s2Vec2 rA = s2RotateVector(qA, j->localAnchorA);
		s2Vec2 rB = s2RotateVector(qB, j->localAnchorB);
		s2Vec2 Cdot = s2Sub(s2Add(vB, s2CrossSV(wB, rB)), s2Add(vA, s2CrossSV(wA, rA)));
		s2Vec2 C = s2Add(s2Add(s2Sub(bodyB->dp, bodyA->dp), s2Sub(rB, rA)), j->centerDiff0);
		s2Mat22 K;
		K.cx.x = mA + mB + rA.y * rA.y * iA + rB.y * rB.y * iB;
		K.cy.x = -rA.y * rA.x * iA - rB.y * rB.x * iB;
		K.cx.y = K.cy.x;
		K.cy.y = mA + mB + rA.x * rA.x * iA + rB.x * rB.x * iB;
		s2Vec2 b = s2Solve22(K, s2Add(Cdot, s2MulSV(biasScale, C)));
		s2Vec2 oldImpulse = j->impulse;
		j->impulse = s2ClampLength(s2Sub(oldImpulse, b), h * s2oMotorMaxForce(s, j));
		s2Vec2 impulse = s2Sub(j->impulse, oldImpulse);
		vA = s2MulSub(vA, mA, impulse);
		wA -= iA * s2Cross(rA, impulse);
		vB = s2MulAdd(vB, mB, impulse);
		wB += iB * s2Cross(rB, impulse);
	}

	bodyA->v = vA;
	bodyA->w = wA;
	bodyB->v = vB;
	bodyB->w = wB;
}

// ---- XPBD ----------------------------------------------------------------------------------------------------------------

// Zero compliance. The angular correction p = -cf C / (iA + iB), clamped to +/- h^2 maxTorque; then the revolute's XPBD row
// along the current separation with lambda = -cf |C| / (kA + kB), clamped to h^2 maxForce in magnitude.
static void s2oMotorXpbd(s2oSolve* s, s2oJoint* j)
{
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2Vec2 dcA = bodyA->dp, dcB = bodyB->dp;
	s2Rot qA = bodyA->q, qB = bodyB->q;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;
	float h = s->h;
	float cf = s2oMotorCorrection(s, j);

	if (iA + iB != 0.0f)
	{
		float C = s2UnwindAngle(s2RelativeAngle(qB, qA) - j->referenceAngle);
		float maxP = h * h * j->maxMotorTorque;
		float p = S2_CLAMP(-cf * C / (iA + iB), -maxP, maxP);
		qA = s2IntegrateRot(qA, -iA * p);
		qB = s2IntegrateRot(qB, iB * p);
	}

	if (mA != 0.0f || mB != 0.0f)
	{
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
		float rnA = s2Cross(rA, n);
		float rnB = s2Cross(rB, n);
		float kA = mA + iA * rnA * rnA;
		float kB = mB + iB * rnB * rnB;
		float lambda = S2_MAX(-cf * c / (kA + kB), -(h * h * s2oMotorMaxForce(s, j)));
		s2Vec2 p = s2MulSV(lambda, n);
		dcA = s2MulSub(dcA, mA, p);
		qA = s2IntegrateRot(qA, -iA * s2Cross(rA, p));
		dcB = s2MulAdd(dcB, mB, p);
		qB = s2IntegrateRot(qB, iB * s2Cross(rB, p));
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

// ---- dispatch --------------------------------------------------------------------------------------------------------

static void s2oMotorJointOp(s2oSolve* s, int op, s2oJoint* j)
{
	if (j->type != S2B_JOINT_MOTOR)
	{
		s2oJointOp_Base(s, op, j);
		return;
	}
	switch (op)
	{
		case S2O_J_WARM:
			// the revolute's warm start: P = impulse at rA / rB, axial = motorImpulse (the limit impulses are zero)
			s2oJointOp_Base(s, op, j);
			break;
		case S2O_J_SOFT_BIAS:
		case S2O_J_SOFT_RELAX:
		case S2O_J_BAUMGARTE_BIAS:
		case S2O_J_BAUMGARTE_RELAX:
		case S2O_J_RIGID:
			s2oMotorVelocity(s, j);
			break;
		case S2O_J_XPBD:
			s2oMotorXpbd(s, j);
			break;
		default:
			// S2O_J_POSITION: no NGS position row, as for the mouse joint
			break;
	}
}
