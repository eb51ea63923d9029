// TEST INFRASTRUCTURE — the wheel joint's oracle (DESIGN.md §3.17). The reference has no wheel joint, so this file is its
// definition: plain, sequential C that the device must match bit for bit.
//
// It is the distance joint's oracle (tests/distance_oracle.c, itself built on the spring, prismatic and base oracles) with
// wheel rows (S2B_JOINT_WHEEL) added, built from that file unmodified by the same preprocessor routing: the distance oracle's
// s2oDistanceJointOp and s2oDistancePrepareJointSoft are routed to the functions below, which handle wheel rows and hand
// every other joint on. One oracle so covers wheel, distance, revolute (with spring), prismatic (with spring), weld, motor and
// mouse rows.
//
// A wheel row holds its axis in localAxisA, its translation limits in lowerAngle / upperAngle, its maximum motor torque in
// maxMotorTorque, its motor speed in motorSpeed and its spring in hertz / dampingRatio. The frame is the prismatic joint's:
// d = (dcB - dcA) + (rB - rA) + centerDiff0, axis = qA localAxisA, perp = leftPerp(axis), a = (d + rA) x axis, s = (d + rA) x
// perp on body A and rB x axis, rB x perp on body B, all formed from the current poses in every solve.
//   * rows, in this order: spring along the axis toward translation 0 (enableSpring, hertz > 0; the spring oracle's row),
//     motor on the relative rotation (enableMotor, iA + iB > 0: the revolute motor's form, mass 1 / (iA + iB), clamped to
//     +/- h maxMotorTorque), lower and upper limit (enableLimit: the prismatic's rows), the perpendicular row C = perp . d
//     (mass 1 / (mA + mB + iA sA^2 + iB sB^2)). A row that does not act keeps a zero impulse.
//   * impulses: impulse.x the perpendicular row's, impulse.y the motor's; motorImpulse stays 0.
//   * velocity forms: the prismatic's per flavour (soft, Baumgarte, rigid), the perpendicular row as the prismatic's block
//     row with its own scalar mass; the motor is the same in every flavour.
//   * warm start: the prismatic's, P = axial axis + impulse.x perp, L = axial a + impulse.x s + impulse.y, axial = [spring +]
//     motorImpulse + lower - upper.
//   * NGS position: the perpendicular row (C clamped to +/- s2_maxLinearCorrection, impulse -C / k), then the prismatic's
//     limit correction on the corrected poses.
//   * XPBD: the spring as §3.14's compliant row with damping, then the perpendicular row and a violated limit at zero
//     compliance; the motor is not applied and the impulses stay zero.
//
// Compiled with the oracle's flags (gcc -std=gnu17 -O2, no FMA contraction) by tests/wheel_oracle.py.

#include "s2b_device.h"

struct s2oSolve;
struct s2oJoint;
struct s2oBody;
static void s2oWheelJointOp(struct s2oSolve* s, int op, struct s2oJoint* j);
static void s2oWheelPrepareJointSoft(struct s2oJoint* j, const s2bJointRow* row, const struct s2oBody* bodies, float contextH,
									 float h, float hertz, int warmStart);

#define s2oDistanceJointOp(first, ...) S2OW_JOINT_OP_##first, __VA_ARGS__)
#define S2OW_JOINT_OP_struct s2oDistanceJointOp_Inner(struct
#define S2OW_JOINT_OP_s2oSolve s2oDistanceJointOp_Inner(s2oSolve
#define S2OW_JOINT_OP_s s2oWheelJointOp(s

#define s2oDistancePrepareJointSoft(first, ...) S2OW_PREPARE_##first, __VA_ARGS__)
#define S2OW_PREPARE_struct s2oDistancePrepareJointSoft_Inner(struct
#define S2OW_PREPARE_s2oJoint s2oDistancePrepareJointSoft_Inner(s2oJoint
#define S2OW_PREPARE_j s2oWheelPrepareJointSoft(j

#include "distance_oracle.c"

#undef s2oDistanceJointOp
#undef s2oDistancePrepareJointSoft

// ---- state -----------------------------------------------------------------------------------------------------------

typedef struct s2oWheel
{
	int motor, spring; // which rows act (the limits act exactly with enableLimit)
	float motorMass;   // 1 / (iA + iB)
} s2oWheel;

static s2oWheel* s2oWheels = NULL;
static int s2oWheelCapacity = 0;

static s2oWheel* s2oWheelOf(int slot)
{
	if (slot >= s2oWheelCapacity)
	{
		int capacity = slot + 1 > 2 * s2oWheelCapacity ? slot + 1 : 2 * s2oWheelCapacity;
		s2oWheels = (s2oWheel*)realloc(s2oWheels, sizeof(s2oWheel) * (size_t)capacity);
		for (int i = s2oWheelCapacity; i < capacity; ++i)
		{
			s2oWheels[i] = (s2oWheel){0};
		}
		s2oWheelCapacity = capacity;
	}
	return s2oWheels + slot;
}

// ---- prepare ---------------------------------------------------------------------------------------------------------

// The base prepare (anchors, masses, centerDiff0, the limits in the revolute fields), then the wheel joint's rows and impulse
// policy: each impulse is kept only with a warm start and where its row acts. The spring's coefficients and impulse go in
// the spring oracle's per-slot state, so its rows serve the wheel unchanged. The XPBD prepare zeroes the impulses after.
static void s2oWheelPrepareJointSoft(s2oJoint* j, const s2bJointRow* row, const s2oBody* bodies, float contextH, float h, float hertz,
									 int warmStart)
{
	// the spring oracle's prepare zeroes the springImpulse of every row it has no spring for, a wheel row's included
	float springImpulse = row->springImpulse;
	s2oDistancePrepareJointSoft_Inner(j, row, bodies, contextH, h, hertz, warmStart);
	if (j->type != S2B_JOINT_WHEEL)
	{
		return;
	}
	s2oWheel* wj = s2oWheelOf(j->slot);
	*wj = (s2oWheel){0};
	float k = j->invIA + j->invIB;
	wj->motor = j->enableMotor && k > 0.0f;
	wj->motorMass = k > 0.0f ? 1.0f / k : 0.0f;
	wj->spring = (row->flags & S2B_JOINT_ENABLE_SPRING) != 0 && row->hertz > 0.0f;
	j->impulse = s2MakeVec2(warmStart ? row->impulse[0] : 0.0f, warmStart && wj->motor ? row->impulse[1] : 0.0f);
	j->motorImpulse = 0.0f;
	j->lowerImpulse = warmStart && j->enableLimit ? row->lowerImpulse : 0.0f;
	j->upperImpulse = warmStart && j->enableLimit ? row->upperImpulse : 0.0f;
	s2oSpring* sp = s2oSpringOf(j->slot);
	*sp = (s2oSpring){0};
	if (wj->spring)
	{
		float zeta = row->dampingRatio;
		float omega = 2.0f * s2_pi * row->hertz;
		sp->bias = omega / (2.0f * zeta + contextH * omega);
		float c = contextH * omega * (2.0f * zeta + contextH * omega);
		sp->impulseScale = 1.0f / (1.0f + c);
		sp->massScale = c * sp->impulseScale;
		sp->lambda = warmStart ? springImpulse : 0.0f;
	}
	((s2bJointRow*)row)->springImpulse = sp->lambda;
}

// ---- velocity rows -----------------------------------------------------------------------------------------------------

// motor (on the rotation), lower limit, upper limit, then the perpendicular row
static void s2oWheelVelocity(s2oSolve* s, s2oJoint* j, const s2oWheel* wj, int kind, int useBias)
{
	float h = s->h, inv_h = s->inv_h;
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2oBody a = *bodyA, b = *bodyB;
	s2Vec2 vA = a.v, vB = b.v;
	float wA = a.w, wB = b.w;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;
	s2oPrismaticFrame f = s2oPrismaticFrameAt(s, j, a.dp, a.q, b.dp, b.q);
	s2Vec2 axis = f.axis;
	s2Vec2 dA = s2Add(f.d, f.rA);
	float translation = s2Dot(axis, f.d);
	float a1 = s2Cross(dA, axis), a2 = s2Cross(f.rB, axis);
	float k = mA + mB + iA * a1 * a1 + iB * a2 * a2;
	float axialMass = k > 0.0f ? 1.0f / k : 0.0f;

	if (wj->motor)
	{
		float Cdot = wB - wA - j->motorSpeed;
		float impulse = -wj->motorMass * Cdot;
		float oldImpulse = j->impulse.y;
		float maxImpulse = h * j->maxMotorTorque;
		j->impulse.y = S2_CLAMP(oldImpulse + impulse, -maxImpulse, maxImpulse);
		impulse = j->impulse.y - oldImpulse;
		wA -= iA * impulse;
		wB += iB * impulse;
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
		s2oRowScale r = s2oPrismaticScale(kind, j, s2Dot(perp, f.d), 0, h, inv_h, useBias);
		float Cdot = s2Dot(perp, s2Sub(vB, vA)) + sB * wB - sA * wA;
		float kp = mA + mB + iA * sA * sA + iB * sB * sB;
		float perpMass = kp > 0.0f ? 1.0f / kp : 0.0f;
		float impulse = -perpMass * r.massScale * (Cdot + r.bias) - r.impulseScale * j->impulse.x;
		j->impulse.x += impulse;
		s2Vec2 P = s2MulSV(impulse, perp);
		vA = s2MulSub(vA, mA, P);
		wA -= iA * (impulse * sA);
		vB = s2MulAdd(vB, mB, P);
		wB += iB * (impulse * sB);
	}

	a.v = vA;
	a.w = wA;
	b.v = vB;
	b.w = wB;
	s2oSpringStore(j, bodyA, bodyB, a, b);
}

// ---- position forms ----------------------------------------------------------------------------------------------------

// NGS position (PGS_NGS, PGS_NGS_Block, TGS_NGS): the perpendicular row, then the prismatic's limit correction on the
// corrected poses (slop s2_linearSlop; equal limits within 2 * s2_linearSlop are held both ways)
static void s2oWheelPosition(s2oSolve* s, s2oJoint* j)
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
		float C = S2_CLAMP(s2Dot(perp, f.d), -s2_maxLinearCorrection, s2_maxLinearCorrection);
		float k = mA + mB + iA * sA * sA + iB * sB * sB;
		float impulse = k > 0.0f ? -C / k : 0.0f;
		s2Vec2 P = s2MulSV(impulse, perp);
		dcA = s2MulSub(dcA, mA, P);
		qA = s2IntegrateRot(qA, -iA * (impulse * sA));
		dcB = s2MulAdd(dcB, mB, P);
		qB = s2IntegrateRot(qB, iB * (impulse * sB));
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

// XPBD, after the spring: the perpendicular row, then a violated limit, both at zero compliance
static void s2oWheelXpbd(s2oSolve* s, s2oJoint* j)
{
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2Vec2 dcA = bodyA->dp, dcB = bodyB->dp;
	s2Rot qA = bodyA->q, qB = bodyB->q;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;

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

static void s2oWheelJointOp(s2oSolve* s, int op, s2oJoint* j)
{
	if (j->type != S2B_JOINT_WHEEL)
	{
		s2oDistanceJointOp_Inner(s, op, j);
		return;
	}
	const s2oWheel* wj = s2oWheelOf(j->slot);
	s2oSpring* sp = s2oSpringOf(j->slot);
	switch (op)
	{
		case S2O_J_WARM:
			// the prismatic's warm start, with the spring's impulse in the axial sum where the spring acts
			if (wj->spring)
			{
				s2oSpringWarmStart(s, j, sp);
			}
			else
			{
				s2oPrismaticWarmStart(s, j);
			}
			break;
		case S2O_J_SOFT_BIAS:
		case S2O_J_SOFT_RELAX:
		case S2O_J_BAUMGARTE_BIAS:
		case S2O_J_BAUMGARTE_RELAX:
		case S2O_J_RIGID:
		{
			if (wj->spring)
			{
				s2oSpringVelocity(s, j, sp);
			}
			int kind = op == S2O_J_RIGID ? S2OP_RIGID : (op == S2O_J_SOFT_BIAS || op == S2O_J_SOFT_RELAX ? S2OP_SOFT : S2OP_BAUMGARTE);
			s2oWheelVelocity(s, j, wj, kind, op == S2O_J_SOFT_BIAS || op == S2O_J_BAUMGARTE_BIAS);
			break;
		}
		case S2O_J_POSITION:
			s2oWheelPosition(s, j);
			break;
		case S2O_J_XPBD:
			if (wj->spring)
			{
				s2oSpringXpbd(s, j);
			}
			s2oWheelXpbd(s, j);
			break;
		default:
			break;
	}
}
