// TEST INFRASTRUCTURE — the prismatic joint's oracle (DESIGN.md §3.9). The reference has no prismatic joint, so this file
// is its definition: plain, sequential C that the device must match bit for bit.
//
// It is the oracle of oracle/s2o_solver.c with prismatic rows (S2B_JOINT_PRISMATIC) added, built from that file unmodified
// so that the revolute and mouse paths stay exactly the ones tests/test_oracle_cpu.py pins to the reference. Two oracle
// functions are routed through the prismatic functions below by the preprocessor, as tests/weld_oracle.c does for the weld:
//   * s2oJointOp, the per-constraint dispatch of every driver (its S2O_J_WARM is the joint warm start);
//   * s2oPrepareJointSoft, which every joint prepare runs (the rigid and XPBD prepares call it first).
// Each macro pastes the first token of its first argument onto a prefix. A definition's first parameter starts with a
// type name (s2oSolve*, s2oJoint*), which selects the oracle's own function, renamed ..._Base; every call passes a
// plain variable (s, j), which selects the prismatic function. The prismatic functions handle prismatic rows and hand
// every other joint to the _Base function.
//
// A prismatic row reuses the revolute's fields: lowerAngle / upperAngle are the translation limits, maxMotorTorque the
// maximum motor force, impulse the (perpendicular, angular) block impulse, motorImpulse / lowerImpulse / upperImpulse the
// axial impulses. The oracle's joint struct has no axis; the prismatic functions read localAxisA from the joint's row.
//
// Compiled with the oracle's flags (gcc -std=gnu17 -O2, no FMA contraction) by tests/prismatic_oracle.py.

#include "s2b_device.h"
#include "solver2d/constants.h"
#include "solver2d/math.h"

struct s2oSolve;
struct s2oJoint;
struct s2oBody;
static void s2oPrismaticJointOp(struct s2oSolve* s, int op, struct s2oJoint* j);
static void s2oPrismaticPrepareJointSoft(struct s2oJoint* j, const s2bJointRow* row, const struct s2oBody* bodies, float contextH,
										 float h, float hertz, int warmStart);

#define s2oJointOp(first, ...) S2OP_JOINT_OP_##first, __VA_ARGS__)
#define S2OP_JOINT_OP_s2oSolve s2oJointOp_Base(s2oSolve
#define S2OP_JOINT_OP_s s2oPrismaticJointOp(s

#define s2oPrepareJointSoft(first, ...) S2OP_PREPARE_##first, __VA_ARGS__)
#define S2OP_PREPARE_s2oJoint s2oPrepareJointSoft_Base(s2oJoint
#define S2OP_PREPARE_j s2oPrismaticPrepareJointSoft(j

#include "../oracle/s2o_solver.c"

#undef s2oJointOp
#undef s2oPrepareJointSoft

// ---- prepare -------------------------------------------------------------------------------------------------------

// The revolute prepare, then the prismatic's impulse policy: the block impulse is kept exactly when the point impulse
// would be, the limit impulses only with the limit flag and a warm start, the motor impulse only with the motor flag and a
// warm start. (The revolute's fixedRotation zeroing does not apply: the axial rows are linear.) The XPBD prepare zeroes
// all of them afterwards.
static void s2oPrismaticPrepareJointSoft(s2oJoint* j, const s2bJointRow* row, const s2oBody* bodies, float contextH, float h,
										 float hertz, int warmStart)
{
	s2oPrepareJointSoft_Base(j, row, bodies, contextH, h, hertz, warmStart);
	if (j->type == S2B_JOINT_PRISMATIC)
	{
		j->impulse = warmStart ? s2MakeVec2(row->impulse[0], row->impulse[1]) : s2Vec2_zero;
		j->motorImpulse = warmStart && j->enableMotor ? row->motorImpulse : 0.0f;
		j->lowerImpulse = warmStart && j->enableLimit ? row->lowerImpulse : 0.0f;
		j->upperImpulse = warmStart && j->enableLimit ? row->upperImpulse : 0.0f;
	}
}

// ---- the joint frame -------------------------------------------------------------------------------------------------

// centre-of-mass-relative anchors, d = (dcB - dcA) + (rB - rA) + centerDiff0 and the world axis at the given poses
typedef struct s2oPrismaticFrame
{
	s2Vec2 rA, rB, d, axis;
} s2oPrismaticFrame;

static s2oPrismaticFrame s2oPrismaticFrameAt(const s2oSolve* s, const s2oJoint* j, s2Vec2 dcA, s2Rot qA, s2Vec2 dcB, s2Rot qB)
{
	const s2bJointRow* row = s->jointRows + j->slot;
	s2oPrismaticFrame f;
	f.rA = s2RotateVector(qA, j->localAnchorA);
	f.rB = s2RotateVector(qB, j->localAnchorB);
	f.d = s2Add(s2Add(s2Sub(dcB, dcA), s2Sub(f.rB, f.rA)), j->centerDiff0);
	f.axis = s2RotateVector(qA, s2MakeVec2(row->localAxisA[0], row->localAxisA[1]));
	return f;
}

// ---- warm start --------------------------------------------------------------------------------------------------------

// P = axial * axis + lambdaPerp * perp, L = axial * a + lambdaPerp * s + lambdaAngle on each side (axial = motor + lower - upper)
static void s2oPrismaticWarmStart(s2oSolve* s, s2oJoint* j)
{
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2oPrismaticFrame f = s2oPrismaticFrameAt(s, j, bodyA->dp, bodyA->q, bodyB->dp, bodyB->q);
	s2Vec2 perp = s2LeftPerp(f.axis);
	s2Vec2 dA = s2Add(f.d, f.rA);
	float axialImpulse = j->motorImpulse + j->lowerImpulse - j->upperImpulse;
	s2Vec2 P = s2Add(s2MulSV(axialImpulse, f.axis), s2MulSV(j->impulse.x, perp));
	float LA = axialImpulse * s2Cross(dA, f.axis) + j->impulse.x * s2Cross(dA, perp) + j->impulse.y;
	float LB = axialImpulse * s2Cross(f.rB, f.axis) + j->impulse.x * s2Cross(f.rB, perp) + j->impulse.y;
	bodyA->v = s2MulSub(bodyA->v, j->invMassA, P);
	bodyA->w = bodyA->w - j->invIA * LA;
	bodyB->v = s2MulAdd(bodyB->v, j->invMassB, P);
	bodyB->w = bodyB->w + j->invIB * LB;
}

// ---- velocity rows -----------------------------------------------------------------------------------------------------

enum
{
	S2OP_SOFT = 0,		// Jacobi, PGS_Soft, SoftStep, TGS_Soft
	S2OP_BAUMGARTE = 1, // PGS, TGS_Sticky
	S2OP_RIGID = 2,		// PGS_NGS, PGS_NGS_Block, TGS_NGS
};

typedef struct s2oRowScale
{
	float bias, massScale, impulseScale;
} s2oRowScale;

// soft: a limit not reached is speculative (C / h); otherwise the soft bias and scales in the biased pass, nothing in the
// relax pass. Baumgarte: as soft, with s2_baumgarte * inv_h * C in every pass. Rigid: max(C, 0) / h on the limits only.
static s2oRowScale s2oPrismaticScale(int kind, const s2oJoint* j, float C, int limit, float h, float inv_h, int useBias)
{
	s2oRowScale r = {0.0f, 1.0f, 0.0f};
	if (kind == S2OP_RIGID)
	{
		r.bias = limit ? S2_MAX(C, 0.0f) / h : 0.0f;
	}
	else if (limit && C > 0.0f)
	{
		r.bias = C * inv_h;
	}
	else if (kind == S2OP_BAUMGARTE)
	{
		r.bias = s2_baumgarte * inv_h * C;
	}
	else if (useBias)
	{
		r.bias = j->biasCoefficient * C;
		r.massScale = j->massCoefficient;
		r.impulseScale = j->impulseCoefficient;
	}
	return r;
}

// motor, lower limit, upper limit (each along the axis, with a fresh axial mass), then the 2x2 block of the perpendicular
// separation and the relative angle
static void s2oPrismaticVelocity(s2oSolve* s, s2oJoint* j, int kind, int useBias)
{
	float h = s->h, inv_h = s->inv_h;
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2Vec2 vA = bodyA->v, vB = bodyB->v;
	float wA = bodyA->w, wB = bodyB->w;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;
	s2oPrismaticFrame f = s2oPrismaticFrameAt(s, j, bodyA->dp, bodyA->q, bodyB->dp, bodyB->q);
	s2Vec2 axis = f.axis;
	s2Vec2 dA = s2Add(f.d, f.rA);
	float translation = s2Dot(axis, f.d);
	float a1 = s2Cross(dA, axis), a2 = s2Cross(f.rB, axis);
	float k = mA + mB + iA * a1 * a1 + iB * a2 * a2;
	float axialMass = k > 0.0f ? 1.0f / k : 0.0f;

	if (j->enableMotor)
	{
		float Cdot = s2Dot(axis, s2Sub(vB, vA)) + a2 * wB - a1 * wA;
		float impulse = axialMass * (j->motorSpeed - Cdot);
		float oldImpulse = j->motorImpulse;
		float maxImpulse = h * j->maxMotorTorque;
		j->motorImpulse = S2_CLAMP(oldImpulse + impulse, -maxImpulse, maxImpulse);
		impulse = j->motorImpulse - oldImpulse;
		s2Vec2 P = s2MulSV(impulse, axis);
		vA = s2MulSub(vA, mA, P);
		wA -= iA * (impulse * a1);
		vB = s2MulAdd(vB, mB, P);
		wB += iB * (impulse * a2);
	}

	if (j->enableLimit)
	{
		{
			s2oRowScale r = s2oPrismaticScale(kind, j, translation - j->lowerAngle, 1, h, inv_h, useBias);
			float Cdot = s2Dot(axis, s2Sub(vB, vA)) + a2 * wB - a1 * wA;
			float impulse = -axialMass * r.massScale * (Cdot + r.bias) - r.impulseScale * j->lowerImpulse;
			float oldImpulse = j->lowerImpulse;
			j->lowerImpulse = S2_MAX(oldImpulse + impulse, 0.0f);
			impulse = j->lowerImpulse - oldImpulse;
			s2Vec2 P = s2MulSV(impulse, axis);
			vA = s2MulSub(vA, mA, P);
			wA -= iA * (impulse * a1);
			vB = s2MulAdd(vB, mB, P);
			wB += iB * (impulse * a2);
		}
		{
			// the upper limit relaxes with its own impulse (the revolute's reference quirk is not carried over)
			s2oRowScale r = s2oPrismaticScale(kind, j, j->upperAngle - translation, 1, h, inv_h, useBias);
			float Cdot = s2Dot(axis, s2Sub(vA, vB)) + a1 * wA - a2 * wB;
			float impulse = -axialMass * r.massScale * (Cdot + r.bias) - r.impulseScale * j->upperImpulse;
			float oldImpulse = j->upperImpulse;
			j->upperImpulse = S2_MAX(oldImpulse + impulse, 0.0f);
			impulse = j->upperImpulse - oldImpulse;
			s2Vec2 P = s2MulSV(impulse, axis);
			vA = s2MulAdd(vA, mA, P);
			wA += iA * (impulse * a1);
			vB = s2MulSub(vB, mB, P);
			wB -= iB * (impulse * a2);
		}
	}

	{
		s2Vec2 perp = s2LeftPerp(axis);
		float sA = s2Cross(dA, perp), sB = s2Cross(f.rB, perp);
		s2Vec2 Cdot = s2MakeVec2(s2Dot(perp, s2Sub(vB, vA)) + sB * wB - sA * wA, wB - wA);
		s2Vec2 C = s2MakeVec2(s2Dot(perp, f.d), s2UnwindAngle(s2RelativeAngle(bodyB->q, bodyA->q) - j->referenceAngle));
		s2oRowScale rx = s2oPrismaticScale(kind, j, C.x, 0, h, inv_h, useBias);
		s2oRowScale ry = s2oPrismaticScale(kind, j, C.y, 0, h, inv_h, useBias);
		float k11 = mA + mB + iA * sA * sA + iB * sB * sB;
		float k12 = iA * sA + iB * sB;
		float k22 = iA + iB;
		if (k22 == 0.0f)
		{
			k22 = 1.0f;
		}
		s2Mat22 K;
		K.cx = s2MakeVec2(k11, k12);
		K.cy = s2MakeVec2(k12, k22);
		s2Vec2 b = s2Solve22(K, s2MakeVec2(Cdot.x + rx.bias, Cdot.y + ry.bias));
		s2Vec2 impulse = s2MakeVec2(-rx.massScale * b.x - rx.impulseScale * j->impulse.x,
									-ry.massScale * b.y - ry.impulseScale * j->impulse.y);
		j->impulse.x += impulse.x;
		j->impulse.y += impulse.y;
		s2Vec2 P = s2MulSV(impulse.x, perp);
		float LA = impulse.x * sA + impulse.y;
		float LB = impulse.x * sB + impulse.y;
		vA = s2MulSub(vA, mA, P);
		wA -= iA * LA;
		vB = s2MulAdd(vB, mB, P);
		wB += iB * LB;
	}

	bodyA->v = vA;
	bodyA->w = wA;
	bodyB->v = vB;
	bodyB->w = wB;
}

// ---- position forms ----------------------------------------------------------------------------------------------------

static void s2oPrismaticStorePoses(s2oJoint* j, s2oBody* bodyA, s2oBody* bodyB, s2Vec2 dcA, s2Rot qA, s2Vec2 dcB, s2Rot qB)
{
	if (j->invMassA != 0.0f || j->invIA != 0.0f)
	{
		bodyA->dp = dcA;
		bodyA->q = qA;
	}
	if (j->invMassB != 0.0f || j->invIB != 0.0f)
	{
		bodyB->dp = dcB;
		bodyB->q = qB;
	}
}

// NGS position (PGS_NGS, PGS_NGS_Block, TGS_NGS): the block with clamped corrections, then the limit row on the corrected
// poses (slop s2_linearSlop; equal limits within 2 * s2_linearSlop are held both ways)
static void s2oPrismaticPosition(s2oSolve* s, s2oJoint* j)
{
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2Vec2 dcA = bodyA->dp, dcB = bodyB->dp;
	s2Rot qA = bodyA->q, qB = bodyB->q;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;

	{
		s2oPrismaticFrame f = s2oPrismaticFrameAt(s, j, dcA, qA, dcB, qB);
		s2Vec2 perp = s2LeftPerp(f.axis);
		s2Vec2 dA = s2Add(f.d, f.rA);
		float sA = s2Cross(dA, perp), sB = s2Cross(f.rB, perp);
		s2Vec2 C;
		C.x = S2_CLAMP(s2Dot(perp, f.d), -s2_maxLinearCorrection, s2_maxLinearCorrection);
		C.y = S2_CLAMP(s2UnwindAngle(s2RelativeAngle(qB, qA) - j->referenceAngle), -s2_maxAngularCorrection, s2_maxAngularCorrection);
		float k11 = mA + mB + iA * sA * sA + iB * sB * sB;
		float k12 = iA * sA + iB * sB;
		float k22 = iA + iB;
		if (k22 == 0.0f)
		{
			k22 = 1.0f;
		}
		s2Mat22 K;
		K.cx = s2MakeVec2(k11, k12);
		K.cy = s2MakeVec2(k12, k22);
		s2Vec2 impulse = s2Solve22(K, s2Neg(C));
		s2Vec2 P = s2MulSV(impulse.x, perp);
		float LA = impulse.x * sA + impulse.y;
		float LB = impulse.x * sB + impulse.y;
		dcA = s2MulSub(dcA, mA, P);
		qA = s2IntegrateRot(qA, -iA * LA);
		dcB = s2MulAdd(dcB, mB, P);
		qB = s2IntegrateRot(qB, iB * LB);
	}

	if (j->enableLimit)
	{
		s2oPrismaticFrame f = s2oPrismaticFrameAt(s, j, dcA, qA, dcB, qB);
		s2Vec2 dA = s2Add(f.d, f.rA);
		float a1 = s2Cross(dA, f.axis), a2 = s2Cross(f.rB, f.axis);
		float translation = s2Dot(f.axis, f.d);
		float lower = j->lowerAngle, upper = j->upperAngle;
		float C = 0.0f;
		if (S2_ABS(upper - lower) < 2.0f * s2_linearSlop)
		{
			C = S2_CLAMP(translation - lower, -s2_maxLinearCorrection, s2_maxLinearCorrection);
		}
		else if (translation <= lower)
		{
			C = S2_CLAMP(translation - lower + s2_linearSlop, -s2_maxLinearCorrection, 0.0f);
		}
		else if (translation >= upper)
		{
			C = S2_CLAMP(translation - upper - s2_linearSlop, 0.0f, s2_maxLinearCorrection);
		}
		float k = mA + mB + iA * a1 * a1 + iB * a2 * a2;
		float impulse = k > 0.0f ? -C / k : 0.0f;
		s2Vec2 P = s2MulSV(impulse, f.axis);
		dcA = s2MulSub(dcA, mA, P);
		qA = s2IntegrateRot(qA, -iA * (impulse * a1));
		dcB = s2MulAdd(dcB, mB, P);
		qB = s2IntegrateRot(qB, iB * (impulse * a2));
	}

	s2oPrismaticStorePoses(j, bodyA, bodyB, dcA, qA, dcB, qB);
}

// XPBD, zero compliance: the angle row (as the weld's), the perpendicular row, then the limits as position inequalities.
// The motor is not applied, as the revolute joint's XPBD form ignores its motor.
static void s2oPrismaticXpbd(s2oSolve* s, s2oJoint* j)
{
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2Vec2 dcA = bodyA->dp, dcB = bodyB->dp;
	s2Rot qA = bodyA->q, qB = bodyB->q;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;

	if (iA + iB != 0.0f)
	{
		float C = s2UnwindAngle(s2RelativeAngle(qB, qA) - j->referenceAngle);
		float p = -C / (iA + iB);
		qA = s2IntegrateRot(qA, -iA * p);
		qB = s2IntegrateRot(qB, iB * p);
	}

	{
		s2oPrismaticFrame f = s2oPrismaticFrameAt(s, j, dcA, qA, dcB, qB);
		s2Vec2 perp = s2LeftPerp(f.axis);
		float sA = s2Cross(s2Add(f.d, f.rA), perp), sB = s2Cross(f.rB, perp);
		float k = mA + mB + iA * sA * sA + iB * sB * sB;
		if (k > 0.0f)
		{
			float lambda = -s2Dot(perp, f.d) / k;
			s2Vec2 P = s2MulSV(lambda, perp);
			dcA = s2MulSub(dcA, mA, P);
			qA = s2IntegrateRot(qA, -iA * (lambda * sA));
			dcB = s2MulAdd(dcB, mB, P);
			qB = s2IntegrateRot(qB, iB * (lambda * sB));
		}
	}

	if (j->enableLimit)
	{
		s2oPrismaticFrame f = s2oPrismaticFrameAt(s, j, dcA, qA, dcB, qB);
		float a1 = s2Cross(s2Add(f.d, f.rA), f.axis), a2 = s2Cross(f.rB, f.axis);
		float translation = s2Dot(f.axis, f.d);
		float C = 0.0f;
		if (translation < j->lowerAngle)
		{
			C = translation - j->lowerAngle;
		}
		else if (translation > j->upperAngle)
		{
			C = translation - j->upperAngle;
		}
		float k = mA + mB + iA * a1 * a1 + iB * a2 * a2;
		if (C != 0.0f && k > 0.0f)
		{
			float lambda = -C / k;
			s2Vec2 P = s2MulSV(lambda, f.axis);
			dcA = s2MulSub(dcA, mA, P);
			qA = s2IntegrateRot(qA, -iA * (lambda * a1));
			dcB = s2MulAdd(dcB, mB, P);
			qB = s2IntegrateRot(qB, iB * (lambda * a2));
		}
	}

	s2oPrismaticStorePoses(j, bodyA, bodyB, dcA, qA, dcB, qB);
}

// ---- dispatch --------------------------------------------------------------------------------------------------------

static void s2oPrismaticJointOp(s2oSolve* s, int op, s2oJoint* j)
{
	if (j->type != S2B_JOINT_PRISMATIC)
	{
		s2oJointOp_Base(s, op, j);
		return;
	}
	switch (op)
	{
		case S2O_J_WARM:
			s2oPrismaticWarmStart(s, j);
			break;
		case S2O_J_SOFT_BIAS:
		case S2O_J_SOFT_RELAX:
			s2oPrismaticVelocity(s, j, S2OP_SOFT, op == S2O_J_SOFT_BIAS);
			break;
		case S2O_J_BAUMGARTE_BIAS:
		case S2O_J_BAUMGARTE_RELAX:
			s2oPrismaticVelocity(s, j, S2OP_BAUMGARTE, op == S2O_J_BAUMGARTE_BIAS);
			break;
		case S2O_J_RIGID:
			s2oPrismaticVelocity(s, j, S2OP_RIGID, 0);
			break;
		case S2O_J_POSITION:
			s2oPrismaticPosition(s, j);
			break;
		case S2O_J_XPBD:
			s2oPrismaticXpbd(s, j);
			break;
		default:
			break;
	}
}
