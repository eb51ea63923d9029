// TEST INFRASTRUCTURE — the distance joint's oracle (DESIGN.md §3.16). The reference has no distance joint, so this file is
// its definition: plain, sequential C that the device must match bit for bit.
//
// It is the joint spring's oracle (tests/spring_oracle.c, itself built on the prismatic oracle and oracle/s2o_solver.c) with
// distance rows (S2B_JOINT_DISTANCE) added, built from that file unmodified by the same preprocessor routing: the spring
// oracle's s2oSpringJointOp and s2oSpringPrepareJointSoft are routed to the functions below, which handle distance rows and
// hand every other joint on. One oracle so covers distance, revolute (with spring), prismatic (with spring), weld, motor and
// mouse rows.
//
// A distance row holds its rest length in referenceAngle, its min / max length in lowerAngle / upperAngle, its maximum motor
// force in maxMotorTorque and its spring in hertz / dampingRatio. Every quantity is formed from the current poses in every
// solve: d = (dcB - dcA) + (rB - rA) + centerDiff0, length and axis = s2cGetLengthAndNormalize(d), crA = rA x axis,
// crB = rB x axis, k = 1 / (mA + mB + iA crA^2 + iB crB^2) (0 when the sum is 0).
//   * rows, in this order: spring (enableSpring, minLength < maxLength, hertz > 0), motor (enableMotor), lower and upper
//     limit (enableLimit, minLength < maxLength), rigid (the spring off or minLength == maxLength). A row that does not act
//     keeps a zero impulse.
//   * velocity forms: the prismatic's per flavour (soft, Baumgarte, rigid); the spring is §3.14's force law.
//   * warm start: P = axial axis, L = axial (r x axis), axial = [rigid +] (spring + motor + lower - upper).
//   * NGS position: a rigid length corrects length - rest; otherwise only a violated limit (length - min or length - max).
//     Clamped to +/- s2_maxLinearCorrection, impulse = -k C.
//   * XPBD: the spring as §3.14's compliant row with damping, then a violated limit, then the rigid row, both at zero
//     compliance; the motor is not applied and the impulses stay zero.
//
// Compiled with the oracle's flags (gcc -std=gnu17 -O2, no FMA contraction) by tests/distance_oracle.py.

#include "s2b_device.h"

struct s2oSolve;
struct s2oJoint;
struct s2oBody;
static void s2oDistanceJointOp(struct s2oSolve* s, int op, struct s2oJoint* j);
static void s2oDistancePrepareJointSoft(struct s2oJoint* j, const s2bJointRow* row, const struct s2oBody* bodies, float contextH,
										float h, float hertz, int warmStart);

#define s2oSpringJointOp(first, ...) S2OD_JOINT_OP_##first, __VA_ARGS__)
#define S2OD_JOINT_OP_struct s2oSpringJointOp_Inner(struct
#define S2OD_JOINT_OP_s2oSolve s2oSpringJointOp_Inner(s2oSolve
#define S2OD_JOINT_OP_s s2oDistanceJointOp(s

#define s2oSpringPrepareJointSoft(first, ...) S2OD_PREPARE_##first, __VA_ARGS__)
#define S2OD_PREPARE_struct s2oSpringPrepareJointSoft_Inner(struct
#define S2OD_PREPARE_s2oJoint s2oSpringPrepareJointSoft_Inner(s2oJoint
#define S2OD_PREPARE_j s2oDistancePrepareJointSoft(j

#include "spring_oracle.c"

#undef s2oSpringJointOp
#undef s2oSpringPrepareJointSoft

#include "../solver2d_b200/csrc/shared/s2_collide.h"

// ---- state -----------------------------------------------------------------------------------------------------------

typedef struct s2oDistance
{
	int rigid, limit, spring;			 // which rows act
	float bias, massScale, impulseScale; // the spring's velocity coefficients
} s2oDistance;

static s2oDistance* s2oDistances = NULL;
static int s2oDistanceCapacity = 0;

static s2oDistance* s2oDistanceOf(int slot)
{
	if (slot >= s2oDistanceCapacity)
	{
		int capacity = slot + 1 > 2 * s2oDistanceCapacity ? slot + 1 : 2 * s2oDistanceCapacity;
		s2oDistances = (s2oDistance*)realloc(s2oDistances, sizeof(s2oDistance) * (size_t)capacity);
		for (int i = s2oDistanceCapacity; i < capacity; ++i)
		{
			s2oDistances[i] = (s2oDistance){0};
		}
		s2oDistanceCapacity = capacity;
	}
	return s2oDistances + slot;
}

// ---- prepare ---------------------------------------------------------------------------------------------------------

// The base prepare (anchors, masses, centerDiff0, the lengths in the revolute fields), then the distance joint's rows and
// impulse policy: each impulse is kept only with a warm start and where its row acts. The XPBD prepare zeroes them after.
static void s2oDistancePrepareJointSoft(s2oJoint* j, const s2bJointRow* row, const s2oBody* bodies, float contextH, float h,
										float hertz, int warmStart)
{
	// the spring oracle's prepare zeroes the springImpulse of every row it has no spring for, a distance row's included
	float springImpulse = row->springImpulse;
	s2oSpringPrepareJointSoft_Inner(j, row, bodies, contextH, h, hertz, warmStart);
	if (j->type != S2B_JOINT_DISTANCE)
	{
		return;
	}
	s2oDistance* dj = s2oDistanceOf(j->slot);
	*dj = (s2oDistance){0};
	int range = j->lowerAngle < j->upperAngle;
	int enableSpring = (row->flags & S2B_JOINT_ENABLE_SPRING) != 0;
	dj->rigid = !(enableSpring && range);
	dj->limit = j->enableLimit && range;
	dj->spring = enableSpring && range && row->hertz > 0.0f;
	j->impulse = s2MakeVec2(warmStart && dj->rigid ? row->impulse[0] : 0.0f, 0.0f);
	j->motorImpulse = warmStart && j->enableMotor ? row->motorImpulse : 0.0f;
	j->lowerImpulse = warmStart && dj->limit ? row->lowerImpulse : 0.0f;
	j->upperImpulse = warmStart && dj->limit ? row->upperImpulse : 0.0f;
	float lambda = 0.0f;
	if (dj->spring)
	{
		float zeta = row->dampingRatio;
		float omega = 2.0f * s2_pi * row->hertz;
		dj->bias = omega / (2.0f * zeta + contextH * omega);
		float c = contextH * omega * (2.0f * zeta + contextH * omega);
		dj->impulseScale = 1.0f / (1.0f + c);
		dj->massScale = c * dj->impulseScale;
		lambda = warmStart ? springImpulse : 0.0f;
	}
	((s2bJointRow*)row)->springImpulse = lambda;
}

// ---- the frame -------------------------------------------------------------------------------------------------------

typedef struct s2oDistanceFrame
{
	s2Vec2 rA, rB, axis;
	float length;
} s2oDistanceFrame;

static s2oDistanceFrame s2oDistanceFrameAt(const s2oJoint* j, s2Vec2 dcA, s2Rot qA, s2Vec2 dcB, s2Rot qB)
{
	s2oDistanceFrame f;
	f.rA = s2RotateVector(qA, j->localAnchorA);
	f.rB = s2RotateVector(qB, j->localAnchorB);
	s2Vec2 d = s2Add(s2Add(s2Sub(dcB, dcA), s2Sub(f.rB, f.rA)), j->centerDiff0);
	f.axis = s2cGetLengthAndNormalize(&f.length, d);
	return f;
}

// ---- warm start ------------------------------------------------------------------------------------------------------

static void s2oDistanceWarmStart(s2oSolve* s, s2oJoint* j, const s2oDistance* dj)
{
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	const s2bJointRow* row = s->jointRows + j->slot;
	s2oDistanceFrame f = s2oDistanceFrameAt(j, bodyA->dp, bodyA->q, bodyB->dp, bodyB->q);
	float axialImpulse = (dj->spring ? row->springImpulse + j->motorImpulse : j->motorImpulse) + j->lowerImpulse - j->upperImpulse;
	axialImpulse = dj->rigid ? j->impulse.x + axialImpulse : axialImpulse;
	s2Vec2 P = s2MulSV(axialImpulse, f.axis);
	float LA = axialImpulse * s2Cross(f.rA, f.axis);
	float LB = axialImpulse * s2Cross(f.rB, f.axis);
	s2oBody a = *bodyA, b = *bodyB;
	a.v = s2MulSub(a.v, j->invMassA, P);
	a.w = a.w - j->invIA * LA;
	b.v = s2MulAdd(b.v, j->invMassB, P);
	b.w = b.w + j->invIB * LB;
	s2oSpringStore(j, bodyA, bodyB, a, b);
}

// ---- velocity rows -----------------------------------------------------------------------------------------------------

// the spring row (§3.14's force law along the current line), stored through the bodies as the device's spring row is
static void s2oDistanceSpring(s2oSolve* s, s2oJoint* j, const s2oDistance* dj)
{
	s2bJointRow* row = s->jointRows + j->slot;
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2oBody a = *bodyA, b = *bodyB;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;
	s2oDistanceFrame f = s2oDistanceFrameAt(j, a.dp, a.q, b.dp, b.q);
	float a1 = s2Cross(f.rA, f.axis), a2 = s2Cross(f.rB, f.axis);
	float k = mA + mB + iA * a1 * a1 + iB * a2 * a2;
	float axialMass = k > 0.0f ? 1.0f / k : 0.0f;
	float Cdot = s2Dot(f.axis, s2Sub(b.v, a.v)) + a2 * b.w - a1 * a.w;
	float impulse = -axialMass * dj->massScale * (Cdot + dj->bias * (f.length - j->referenceAngle)) - dj->impulseScale * row->springImpulse;
	row->springImpulse += impulse;
	s2Vec2 P = s2MulSV(impulse, f.axis);
	a.v = s2MulSub(a.v, mA, P);
	a.w -= iA * (impulse * a1);
	b.v = s2MulAdd(b.v, mB, P);
	b.w += iB * (impulse * a2);
	s2oSpringStore(j, bodyA, bodyB, a, b);
}

// motor, lower limit, upper limit (the prismatic's axial rows with the length as the coordinate), then the rigid row
static void s2oDistanceVelocity(s2oSolve* s, s2oJoint* j, const s2oDistance* dj, int kind, int useBias)
{
	float h = s->h, inv_h = s->inv_h;
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2oBody a = *bodyA, b = *bodyB;
	s2Vec2 vA = a.v, vB = b.v;
	float wA = a.w, wB = b.w;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;
	s2oDistanceFrame f = s2oDistanceFrameAt(j, a.dp, a.q, b.dp, b.q);
	s2Vec2 axis = f.axis;
	float a1 = s2Cross(f.rA, axis), a2 = s2Cross(f.rB, axis);
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

	if (dj->limit)
	{
		{
			s2oRowScale r = s2oPrismaticScale(kind, j, f.length - j->lowerAngle, 1, h, inv_h, useBias);
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
			s2oRowScale r = s2oPrismaticScale(kind, j, j->upperAngle - f.length, 1, h, inv_h, useBias);
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

	if (dj->rigid)
	{
		s2oRowScale r = s2oPrismaticScale(kind, j, f.length - j->referenceAngle, 0, h, inv_h, useBias);
		float Cdot = s2Dot(axis, s2Sub(vB, vA)) + a2 * wB - a1 * wA;
		float impulse = -axialMass * r.massScale * (Cdot + r.bias) - r.impulseScale * j->impulse.x;
		j->impulse.x += impulse;
		s2Vec2 P = s2MulSV(impulse, axis);
		vA = s2MulSub(vA, mA, P);
		wA -= iA * (impulse * a1);
		vB = s2MulAdd(vB, mB, P);
		wB += iB * (impulse * a2);
	}

	a.v = vA;
	a.w = wA;
	b.v = vB;
	b.w = wB;
	s2oSpringStore(j, bodyA, bodyB, a, b);
}

// ---- position forms ----------------------------------------------------------------------------------------------------

static void s2oDistanceCorrect(const s2oJoint* j, const s2oDistanceFrame* f, float C, s2Vec2* dcA, s2Rot* qA, s2Vec2* dcB, s2Rot* qB)
{
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;
	float crA = s2Cross(f->rA, f->axis), crB = s2Cross(f->rB, f->axis);
	float k = mA + mB + iA * crA * crA + iB * crB * crB;
	float axialMass = k > 0.0f ? 1.0f / k : 0.0f;
	float impulse = -axialMass * C;
	s2Vec2 P = s2MulSV(impulse, f->axis);
	*dcA = s2MulSub(*dcA, mA, P);
	*qA = s2IntegrateRot(*qA, -iA * (impulse * crA));
	*dcB = s2MulAdd(*dcB, mB, P);
	*qB = s2IntegrateRot(*qB, iB * (impulse * crB));
}

static void s2oDistancePosition(s2oSolve* s, s2oJoint* j, const s2oDistance* dj)
{
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2Vec2 dcA = bodyA->dp, dcB = bodyB->dp;
	s2Rot qA = bodyA->q, qB = bodyB->q;
	s2oDistanceFrame f = s2oDistanceFrameAt(j, dcA, qA, dcB, qB);
	float C;
	if (dj->rigid)
	{
		C = f.length - j->referenceAngle;
	}
	else if (dj->limit && f.length < j->lowerAngle)
	{
		C = f.length - j->lowerAngle;
	}
	else if (dj->limit && f.length > j->upperAngle)
	{
		C = f.length - j->upperAngle;
	}
	else
	{
		return;
	}
	C = S2_CLAMP(C, -s2_maxLinearCorrection, s2_maxLinearCorrection);
	s2oDistanceCorrect(j, &f, C, &dcA, &qA, &dcB, &qB);
	s2oPrismaticStorePoses(j, bodyA, bodyB, dcA, qA, dcB, qB);
}

// XPBD, after the spring: a violated limit, then the rigid row on the corrected poses, both at zero compliance
static void s2oDistanceXpbd(s2oSolve* s, s2oJoint* j, const s2oDistance* dj)
{
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2Vec2 dcA = bodyA->dp, dcB = bodyB->dp;
	s2Rot qA = bodyA->q, qB = bodyB->q;
	if (dj->limit)
	{
		s2oDistanceFrame f = s2oDistanceFrameAt(j, dcA, qA, dcB, qB);
		float C = 0.0f;
		if (f.length < j->lowerAngle)
		{
			C = f.length - j->lowerAngle;
		}
		else if (f.length > j->upperAngle)
		{
			C = f.length - j->upperAngle;
		}
		if (C != 0.0f)
		{
			s2oDistanceCorrect(j, &f, C, &dcA, &qA, &dcB, &qB);
		}
	}
	if (dj->rigid)
	{
		s2oDistanceFrame f = s2oDistanceFrameAt(j, dcA, qA, dcB, qB);
		s2oDistanceCorrect(j, &f, f.length - j->referenceAngle, &dcA, &qA, &dcB, &qB);
	}
	s2oPrismaticStorePoses(j, bodyA, bodyB, dcA, qA, dcB, qB);
}

// the spring's XPBD row (§3.14) along the current line: C and C0 = length - rest at the current and the sub-step's start pose
static void s2oDistanceSpringXpbd(s2oSolve* s, s2oJoint* j)
{
	const s2bJointRow* row = s->jointRows + j->slot;
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2oBody a = *bodyA, b = *bodyB;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;
	float omegaH = 2.0f * s2_pi * row->hertz * s->ctx->h;
	float zeta = row->dampingRatio;
	s2oDistanceFrame f0 = s2oDistanceFrameAt(j, a.dp0, a.q0, b.dp0, b.q0);
	s2oDistanceFrame f = s2oDistanceFrameAt(j, a.dp, a.q, b.dp, b.q);
	float a1 = s2Cross(f.rA, f.axis), a2 = s2Cross(f.rB, f.axis);
	float k = mA + mB + iA * a1 * a1 + iB * a2 * a2;
	if (k > 0.0f)
	{
		float lambda = s2oSpringXpbdImpulse(k, f.length - j->referenceAngle, f0.length - j->referenceAngle, omegaH, zeta);
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

// ---- dispatch --------------------------------------------------------------------------------------------------------

static void s2oDistanceJointOp(s2oSolve* s, int op, s2oJoint* j)
{
	if (j->type != S2B_JOINT_DISTANCE)
	{
		s2oSpringJointOp_Inner(s, op, j);
		return;
	}
	const s2oDistance* dj = s2oDistanceOf(j->slot);
	switch (op)
	{
		case S2O_J_WARM:
			s2oDistanceWarmStart(s, j, dj);
			break;
		case S2O_J_SOFT_BIAS:
		case S2O_J_SOFT_RELAX:
		case S2O_J_BAUMGARTE_BIAS:
		case S2O_J_BAUMGARTE_RELAX:
		case S2O_J_RIGID:
		{
			if (dj->spring)
			{
				s2oDistanceSpring(s, j, dj);
			}
			int kind = op == S2O_J_RIGID ? S2OP_RIGID : (op == S2O_J_SOFT_BIAS || op == S2O_J_SOFT_RELAX ? S2OP_SOFT : S2OP_BAUMGARTE);
			s2oDistanceVelocity(s, j, dj, kind, op == S2O_J_SOFT_BIAS || op == S2O_J_BAUMGARTE_BIAS);
			break;
		}
		case S2O_J_POSITION:
			s2oDistancePosition(s, j, dj);
			break;
		case S2O_J_XPBD:
			if (dj->spring)
			{
				s2oDistanceSpringXpbd(s, j);
			}
			s2oDistanceXpbd(s, j, dj);
			break;
		default:
			break;
	}
}
