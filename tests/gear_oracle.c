// TEST INFRASTRUCTURE — the gear joint's oracle (DESIGN.md §3.19). The reference has no gear joint, so this file is its
// definition: plain, sequential C that the device must match bit for bit.
//
// It is the pulley joint's oracle (tests/pulley_oracle.c, itself built on the wheel, distance, spring, prismatic and base
// oracles) with gear rows (S2B_JOINT_GEAR) added, built from that file unmodified by the same preprocessor routing: the
// pulley oracle's s2oPulleyJointOp and s2oPulleyPrepareJointSoft are routed to the functions below, which handle gear rows
// and hand every other joint on. One oracle so covers every joint type. Gear rows are intercepted before any inner oracle
// decodes them: the inner prepare sees a bare revolute copy of the row (for the anchors, masses and soft coefficients), and
// no inner op sees a gear row.
//
// A gear row holds side 1's frame in target / localAxisA and side 2's in maxMotorTorque / motorSpeed / hertz / dampingRatio
// (a revolute side: the frame rotation (s, c) and the reference angle; a prismatic side: the world anchor pC and the world
// axis u), flags S2B_JOINT_GEAR_PRISMATIC1 / 2 for a prismatic side, its ratio in referenceAngle and its constant in
// lowerAngle; lowerImpulse / upperImpulse are the revolute sides' unwound coordinates. Prepare turns a prismatic side's pC
// into d0 = c - pC at the start poses and moves each revolute side's coordinate theta to the start pose,
// theta <- theta + unwind(relAngle(q, qC) - ref - theta) (s2cGearRevolute). Every other quantity is formed from the
// current poses in every solve, each side from its own body's pose (s2cGearRevolute / s2cGearPrismatic):
//   * the row: C = coordinate1 + ratio coordinate2 - constant, Cdot = (Jv1 . vA + Jw1 wA) + ratio (Jv2 . vB + Jw2 wB),
//     k = 1 / (mass1 + ratio^2 mass2) with mass = m Jv.Jv + i Jw^2 (0 when the sum is 0), impulse applied as
//     v += m (impulse Jv1), w += i (impulse Jw1) on side 1 and the same with ratio impulse on side 2.
//   * impulses: impulse.x the gear's, kept with the variant's warm start (never under XPBD); every other impulse stays 0.
//   * velocity forms: the soft bias in the biased pass, Baumgarte in every pass, no bias under the rigid flavour.
//   * warm start: P = lambda Jv1, L = lambda Jw1 on side 1, P = (ratio lambda) Jv2, L = (ratio lambda) Jw2 on side 2.
//   * NGS position: Box2D 2.4's gear correction, impulse -k C, with C clamped to +/- s2_maxAngularCorrection for a
//     revolute side 1, +/- s2_maxLinearCorrection for a prismatic side 1.
//   * XPBD: the same C and gradients at zero compliance, lambda = -C / (1 / k), nothing when 1 / k is 0. The XPBD prepare
//     zeroes every joint impulse after this prepare, so the XPBD op puts the unwound coordinates back for the store.
//
// Compiled with the oracle's flags (gcc -std=gnu17 -O2, no FMA contraction) by tests/gear_oracle.py.

#include "s2b_device.h"

struct s2oSolve;
struct s2oJoint;
struct s2oBody;
static void s2oGearJointOp(struct s2oSolve* s, int op, struct s2oJoint* j);
static void s2oGearPrepareJointSoft(struct s2oJoint* j, const s2bJointRow* row, const struct s2oBody* bodies, float contextH,
									float h, float hertz, int warmStart);

#define s2oPulleyJointOp(first, ...) S2OGR_JOINT_OP_##first, __VA_ARGS__)
#define S2OGR_JOINT_OP_struct s2oPulleyJointOp_Inner(struct
#define S2OGR_JOINT_OP_s2oSolve s2oPulleyJointOp_Inner(s2oSolve
#define S2OGR_JOINT_OP_s s2oGearJointOp(s

#define s2oPulleyPrepareJointSoft(first, ...) S2OGR_PREPARE_##first, __VA_ARGS__)
#define S2OGR_PREPARE_struct s2oPulleyPrepareJointSoft_Inner(struct
#define S2OGR_PREPARE_s2oJoint s2oPulleyPrepareJointSoft_Inner(s2oJoint
#define S2OGR_PREPARE_j s2oGearPrepareJointSoft(j

#include "pulley_oracle.c"

#undef s2oPulleyJointOp
#undef s2oPulleyPrepareJointSoft

#include "../solver2d_b200/csrc/shared/s2_gear_joint.h"

// ---- state -----------------------------------------------------------------------------------------------------------

typedef struct s2oGear
{
	int prismatic1, prismatic2;
	float frame1[4], frame2[4]; // revolute: qC.s, qC.c, ref; prismatic: c - pC at the start poses, u
	float theta1, theta2;		// the revolute sides' unwound coordinates at the start poses
	float constant, ratio;
} s2oGear;

static s2oGear* s2oGears = NULL;
static int s2oGearCapacity = 0;

static s2oGear* s2oGearOf(int slot)
{
	if (slot >= s2oGearCapacity)
	{
		int capacity = slot + 1 > 2 * s2oGearCapacity ? slot + 1 : 2 * s2oGearCapacity;
		s2oGears = (s2oGear*)realloc(s2oGears, sizeof(s2oGear) * (size_t)capacity);
		for (int i = s2oGearCapacity; i < capacity; ++i)
		{
			s2oGears[i] = (s2oGear){0};
		}
		s2oGearCapacity = capacity;
	}
	return s2oGears + slot;
}

// ---- prepare ---------------------------------------------------------------------------------------------------------

static void s2oGearPrepareJointSoft(s2oJoint* j, const s2bJointRow* row, const s2oBody* bodies, float contextH, float h,
									float hertz, int warmStart)
{
	if (s2bJointType(row->flags) != S2B_JOINT_GEAR)
	{
		s2oPulleyPrepareJointSoft_Inner(j, row, bodies, contextH, h, hertz, warmStart);
		return;
	}
	// the base prepare's anchors, masses and soft coefficients, from a copy that reads as a bare revolute row
	s2bJointRow base = *row;
	base.flags = S2B_ROW_VALID;
	s2oPulleyPrepareJointSoft_Inner(j, &base, bodies, contextH, h, hertz, warmStart);
	j->type = S2B_JOINT_GEAR;

	const s2oBody* bodyA = bodies + j->indexA;
	const s2oBody* bodyB = bodies + j->indexB;
	s2oGear* g = s2oGearOf(j->slot);
	g->prismatic1 = (row->flags & S2B_JOINT_GEAR_PRISMATIC1) != 0;
	g->prismatic2 = (row->flags & S2B_JOINT_GEAR_PRISMATIC2) != 0;
	float f1[4] = {row->target[0], row->target[1], row->localAxisA[0], row->localAxisA[1]};
	float f2[4] = {row->maxMotorTorque, row->motorSpeed, row->hertz, row->dampingRatio};
	g->theta1 = 0.0f;
	g->theta2 = 0.0f;
	if (g->prismatic1)
	{
		f1[0] = bodyA->position.x - f1[0];
		f1[1] = bodyA->position.y - f1[1];
	}
	else
	{
		g->theta1 = s2cGearRevolute(f1[0], f1[1], f1[2], row->lowerImpulse, bodyA->q).coordinate;
	}
	if (g->prismatic2)
	{
		f2[0] = bodyB->position.x - f2[0];
		f2[1] = bodyB->position.y - f2[1];
	}
	else
	{
		g->theta2 = s2cGearRevolute(f2[0], f2[1], f2[2], row->upperImpulse, bodyB->q).coordinate;
	}
	memcpy(g->frame1, f1, sizeof(f1));
	memcpy(g->frame2, f2, sizeof(f2));
	g->ratio = row->referenceAngle;
	g->constant = row->lowerAngle;
	j->impulse = s2MakeVec2(warmStart ? row->impulse[0] : 0.0f, 0.0f);
	j->motorImpulse = 0.0f;
	j->lowerImpulse = g->theta1;
	j->upperImpulse = g->theta2;
}

// ---- the sides -------------------------------------------------------------------------------------------------------

static s2cGearSide s2oGearSide(const s2oJoint* j, const s2oGear* g, int side2, s2Vec2 dc, s2Rot q)
{
	const float* f = side2 ? g->frame2 : g->frame1;
	if (side2 ? g->prismatic2 : g->prismatic1)
	{
		return s2cGearPrismatic(s2MakeVec2(f[0], f[1]), s2MakeVec2(f[2], f[3]), dc, q, side2 ? j->localAnchorB : j->localAnchorA);
	}
	return s2cGearRevolute(f[0], f[1], f[2], side2 ? g->theta2 : g->theta1, q);
}

static float s2oGearInvMass(const s2oJoint* j, const s2cGearSide* A, const s2cGearSide* B, float ratio)
{
	return s2cGearSideMass(*A, j->invMassA, j->invIA) + ratio * ratio * s2cGearSideMass(*B, j->invMassB, j->invIB);
}

// ---- warm start ------------------------------------------------------------------------------------------------------

static void s2oGearWarmStart(s2oSolve* s, s2oJoint* j, const s2oGear* g)
{
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2oBody a = *bodyA, b = *bodyB;
	s2cGearSide A = s2oGearSide(j, g, 0, a.dp, a.q);
	s2cGearSide B = s2oGearSide(j, g, 1, b.dp, b.q);
	float lambda = j->impulse.x;
	float lambdaB = g->ratio * lambda;
	a.v = s2MulAdd(a.v, j->invMassA, s2MulSV(lambda, A.Jv));
	a.w = a.w + j->invIA * (lambda * A.Jw);
	b.v = s2MulAdd(b.v, j->invMassB, s2MulSV(lambdaB, B.Jv));
	b.w = b.w + j->invIB * (lambdaB * B.Jw);
	s2oSpringStore(j, bodyA, bodyB, a, b);
}

// ---- velocity row ------------------------------------------------------------------------------------------------------

static void s2oGearVelocity(s2oSolve* s, s2oJoint* j, const s2oGear* g, int kind, int useBias)
{
	float h = s->h, inv_h = s->inv_h;
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2oBody a = *bodyA, b = *bodyB;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;
	float ratio = g->ratio;
	s2cGearSide A = s2oGearSide(j, g, 0, a.dp, a.q);
	s2cGearSide B = s2oGearSide(j, g, 1, b.dp, b.q);
	float kInv = s2oGearInvMass(j, &A, &B, ratio);
	float k = kInv > 0.0f ? 1.0f / kInv : 0.0f;

	s2oRowScale r = s2oPrismaticScale(kind, j, A.coordinate + ratio * B.coordinate - g->constant, 0, h, inv_h, useBias);
	float Cdot = (s2Dot(A.Jv, a.v) + A.Jw * a.w) + ratio * (s2Dot(B.Jv, b.v) + B.Jw * b.w);
	float impulse = -k * r.massScale * (Cdot + r.bias) - r.impulseScale * j->impulse.x;
	j->impulse.x += impulse;
	float impulseB = ratio * impulse;
	a.v = s2MulAdd(a.v, mA, s2MulSV(impulse, A.Jv));
	a.w += iA * (impulse * A.Jw);
	b.v = s2MulAdd(b.v, mB, s2MulSV(impulseB, B.Jv));
	b.w += iB * (impulseB * B.Jw);
	s2oSpringStore(j, bodyA, bodyB, a, b);
}

// ---- position forms ----------------------------------------------------------------------------------------------------

// NGS (xpbd == 0): Box2D 2.4's gear position solve, impulse -k C, with C clamped in side 1's units. XPBD (xpbd == 1):
// lambda = -C / (1 / k) at zero compliance, nothing when 1 / k is 0.
static void s2oGearPosition(s2oSolve* s, s2oJoint* j, const s2oGear* g, int xpbd)
{
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2Vec2 dcA = bodyA->dp, dcB = bodyB->dp;
	s2Rot qA = bodyA->q, qB = bodyB->q;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;
	float ratio = g->ratio;
	s2cGearSide A = s2oGearSide(j, g, 0, dcA, qA);
	s2cGearSide B = s2oGearSide(j, g, 1, dcB, qB);
	float kInv = s2oGearInvMass(j, &A, &B, ratio);
	float C = A.coordinate + ratio * B.coordinate - g->constant;
	float impulse;
	if (xpbd)
	{
		if ((kInv > 0.0f) == false)
		{
			return;
		}
		impulse = -C / kInv;
	}
	else
	{
		float maxC = g->prismatic1 ? s2_maxLinearCorrection : s2_maxAngularCorrection;
		float k = kInv > 0.0f ? 1.0f / kInv : 0.0f;
		impulse = -k * S2_CLAMP(C, -maxC, maxC);
	}
	float impulseB = ratio * impulse;
	dcA = s2MulAdd(dcA, mA, s2MulSV(impulse, A.Jv));
	qA = s2IntegrateRot(qA, iA * (impulse * A.Jw));
	dcB = s2MulAdd(dcB, mB, s2MulSV(impulseB, B.Jv));
	qB = s2IntegrateRot(qB, iB * (impulseB * B.Jw));
	s2oPrismaticStorePoses(j, bodyA, bodyB, dcA, qA, dcB, qB);
}

// ---- dispatch --------------------------------------------------------------------------------------------------------

static void s2oGearJointOp(s2oSolve* s, int op, s2oJoint* j)
{
	if (j->type != S2B_JOINT_GEAR)
	{
		s2oPulleyJointOp_Inner(s, op, j);
		return;
	}
	const s2oGear* g = s2oGearOf(j->slot);
	switch (op)
	{
		case S2O_J_WARM:
			s2oGearWarmStart(s, j, g);
			break;
		case S2O_J_SOFT_BIAS:
		case S2O_J_SOFT_RELAX:
		case S2O_J_BAUMGARTE_BIAS:
		case S2O_J_BAUMGARTE_RELAX:
		case S2O_J_RIGID:
		{
			int kind = op == S2O_J_RIGID ? S2OP_RIGID : (op == S2O_J_SOFT_BIAS || op == S2O_J_SOFT_RELAX ? S2OP_SOFT : S2OP_BAUMGARTE);
			s2oGearVelocity(s, j, g, kind, op == S2O_J_SOFT_BIAS || op == S2O_J_BAUMGARTE_BIAS);
			break;
		}
		case S2O_J_POSITION:
			s2oGearPosition(s, j, g, 0);
			break;
		case S2O_J_XPBD:
			// the unwound coordinates are state: back in the joint after the XPBD prepare zeroed its impulses
			j->lowerImpulse = g->theta1;
			j->upperImpulse = g->theta2;
			s2oGearPosition(s, j, g, 1);
			break;
		default:
			break;
	}
}
