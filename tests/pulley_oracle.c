// TEST INFRASTRUCTURE — the pulley joint's oracle (DESIGN.md §3.18). The reference has no pulley joint, so this file is its
// definition: plain, sequential C that the device must match bit for bit.
//
// It is the wheel joint's oracle (tests/wheel_oracle.c, itself built on the distance, spring, prismatic and base oracles) with
// pulley rows (S2B_JOINT_PULLEY) added, built from that file unmodified by the same preprocessor routing: the wheel oracle's
// s2oWheelJointOp and s2oWheelPrepareJointSoft are routed to the functions below, which handle pulley rows and hand every
// other joint on. One oracle so covers every joint type: pulley, wheel, distance, revolute (with spring), prismatic (with
// spring), weld, motor and mouse rows.
//
// A pulley row holds ground anchor A in target, ground anchor B in localAxisA, its ratio in referenceAngle and its rest
// lengths lengthA / lengthB in lowerAngle / upperAngle. Prepare forms constant = lengthA + ratio lengthB and, at the start
// poses, d0A = cA - groundA and d0B = cB - groundB. Every other quantity is formed from the current poses in every solve, each
// rope from its own body's pose: rA = qA lA, uA = s2cPulleyRope((dcA + rA) + d0A) (Box2D 2.4's rule: zero when the rope is no
// longer than 10 s2_linearSlop), lengthA its length; the same for B.
//   * the row: C = constant - lengthA - ratio lengthB, Cdot = -uA . vpA - ratio uB . vpB, k = 1 / (mA + iA ruA^2 + ratio^2
//     (mB + iB ruB^2)) (0 when the sum is 0), impulse applied as PA = -lambda uA, PB = -(ratio lambda) uB (v += m P,
//     w += i r x P). It is an equality row: the rope can push.
//   * impulses: impulse.x the rope's, kept with the variant's warm start; every other impulse stays 0.
//   * velocity forms: the distance joint's rigid row per flavour (soft bias in the biased pass, Baumgarte in every pass, no
//     bias under the rigid flavour).
//   * warm start: PA = -lambda uA, PB = -(ratio lambda) uB, L = r x P on each side.
//   * NGS position: Box2D 2.4's pulley correction, impulse -k C, with C clamped to +/- s2_maxLinearCorrection.
//   * XPBD: the same C and gradients at zero compliance, lambda = -C / (1 / k), nothing when 1 / k is 0; the impulse stays 0.
//
// Compiled with the oracle's flags (gcc -std=gnu17 -O2, no FMA contraction) by tests/pulley_oracle.py.

#include "s2b_device.h"

struct s2oSolve;
struct s2oJoint;
struct s2oBody;
static void s2oPulleyJointOp(struct s2oSolve* s, int op, struct s2oJoint* j);
static void s2oPulleyPrepareJointSoft(struct s2oJoint* j, const s2bJointRow* row, const struct s2oBody* bodies, float contextH,
									  float h, float hertz, int warmStart);

#define s2oWheelJointOp(first, ...) S2OPL_JOINT_OP_##first, __VA_ARGS__)
#define S2OPL_JOINT_OP_struct s2oWheelJointOp_Inner(struct
#define S2OPL_JOINT_OP_s2oSolve s2oWheelJointOp_Inner(s2oSolve
#define S2OPL_JOINT_OP_s s2oPulleyJointOp(s

#define s2oWheelPrepareJointSoft(first, ...) S2OPL_PREPARE_##first, __VA_ARGS__)
#define S2OPL_PREPARE_struct s2oWheelPrepareJointSoft_Inner(struct
#define S2OPL_PREPARE_s2oJoint s2oWheelPrepareJointSoft_Inner(s2oJoint
#define S2OPL_PREPARE_j s2oPulleyPrepareJointSoft(j

#include "wheel_oracle.c"

#undef s2oWheelJointOp
#undef s2oWheelPrepareJointSoft

#include "../solver2d_b200/csrc/shared/s2_distance_joint.h"

// ---- state -----------------------------------------------------------------------------------------------------------

typedef struct s2oPulley
{
	s2Vec2 d0A, d0B; // cA - groundA, cB - groundB at the start poses
	float constant, ratio;
} s2oPulley;

static s2oPulley* s2oPulleys = NULL;
static int s2oPulleyCapacity = 0;

static s2oPulley* s2oPulleyOf(int slot)
{
	if (slot >= s2oPulleyCapacity)
	{
		int capacity = slot + 1 > 2 * s2oPulleyCapacity ? slot + 1 : 2 * s2oPulleyCapacity;
		s2oPulleys = (s2oPulley*)realloc(s2oPulleys, sizeof(s2oPulley) * (size_t)capacity);
		for (int i = s2oPulleyCapacity; i < capacity; ++i)
		{
			s2oPulleys[i] = (s2oPulley){0};
		}
		s2oPulleyCapacity = capacity;
	}
	return s2oPulleys + slot;
}

// ---- prepare ---------------------------------------------------------------------------------------------------------

// The base prepare (anchors, masses), then the pulley's constant, ratio and start offsets and its impulse policy: the rope
// impulse is kept only with a warm start. The XPBD prepare zeroes it after.
static void s2oPulleyPrepareJointSoft(s2oJoint* j, const s2bJointRow* row, const s2oBody* bodies, float contextH, float h,
									  float hertz, int warmStart)
{
	s2oWheelPrepareJointSoft_Inner(j, row, bodies, contextH, h, hertz, warmStart);
	if (j->type != S2B_JOINT_PULLEY)
	{
		return;
	}
	s2oPulley* pj = s2oPulleyOf(j->slot);
	pj->ratio = row->referenceAngle;
	pj->constant = row->lowerAngle + row->referenceAngle * row->upperAngle;
	pj->d0A = s2Sub(bodies[j->indexA].position, s2MakeVec2(row->target[0], row->target[1]));
	pj->d0B = s2Sub(bodies[j->indexB].position, s2MakeVec2(row->localAxisA[0], row->localAxisA[1]));
	j->impulse = s2MakeVec2(warmStart ? row->impulse[0] : 0.0f, 0.0f);
	j->motorImpulse = 0.0f;
	j->lowerImpulse = 0.0f;
	j->upperImpulse = 0.0f;
}

// ---- the ropes -------------------------------------------------------------------------------------------------------

typedef struct s2oRope
{
	s2Vec2 r, u;
	float length;
} s2oRope;

static s2oRope s2oRopeAt(s2Vec2 localAnchor, s2Vec2 d0, s2Vec2 dc, s2Rot q)
{
	s2oRope p;
	p.r = s2RotateVector(q, localAnchor);
	p.u = s2cPulleyRope(&p.length, s2Add(s2Add(dc, p.r), d0));
	return p;
}

static float s2oPulleyInvMass(const s2oJoint* j, const s2oRope* A, const s2oRope* B, float ratio)
{
	float ruA = s2Cross(A->r, A->u), ruB = s2Cross(B->r, B->u);
	return j->invMassA + j->invIA * ruA * ruA + ratio * ratio * (j->invMassB + j->invIB * ruB * ruB);
}

// ---- warm start ------------------------------------------------------------------------------------------------------

static void s2oPulleyWarmStart(s2oSolve* s, s2oJoint* j, const s2oPulley* pj)
{
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2oBody a = *bodyA, b = *bodyB;
	s2oRope A = s2oRopeAt(j->localAnchorA, pj->d0A, a.dp, a.q);
	s2oRope B = s2oRopeAt(j->localAnchorB, pj->d0B, b.dp, b.q);
	float lambda = j->impulse.x;
	s2Vec2 PA = s2MulSV(-lambda, A.u);
	s2Vec2 PB = s2MulSV(-(pj->ratio * lambda), B.u);
	a.v = s2MulAdd(a.v, j->invMassA, PA);
	a.w = a.w + j->invIA * s2Cross(A.r, PA);
	b.v = s2MulAdd(b.v, j->invMassB, PB);
	b.w = b.w + j->invIB * s2Cross(B.r, PB);
	s2oSpringStore(j, bodyA, bodyB, a, b);
}

// ---- velocity row ------------------------------------------------------------------------------------------------------

static void s2oPulleyVelocity(s2oSolve* s, s2oJoint* j, const s2oPulley* pj, int kind, int useBias)
{
	float h = s->h, inv_h = s->inv_h;
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2oBody a = *bodyA, b = *bodyB;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;
	float ratio = pj->ratio;
	s2oRope A = s2oRopeAt(j->localAnchorA, pj->d0A, a.dp, a.q);
	s2oRope B = s2oRopeAt(j->localAnchorB, pj->d0B, b.dp, b.q);
	float kInv = s2oPulleyInvMass(j, &A, &B, ratio);
	float k = kInv > 0.0f ? 1.0f / kInv : 0.0f;

	s2oRowScale r = s2oPrismaticScale(kind, j, pj->constant - A.length - ratio * B.length, 0, h, inv_h, useBias);
	s2Vec2 vpA = s2Add(a.v, s2CrossSV(a.w, A.r));
	s2Vec2 vpB = s2Add(b.v, s2CrossSV(b.w, B.r));
	float Cdot = -s2Dot(A.u, vpA) - ratio * s2Dot(B.u, vpB);
	float impulse = -k * r.massScale * (Cdot + r.bias) - r.impulseScale * j->impulse.x;
	j->impulse.x += impulse;
	s2Vec2 PA = s2MulSV(-impulse, A.u);
	s2Vec2 PB = s2MulSV(-(ratio * impulse), B.u);
	a.v = s2MulAdd(a.v, mA, PA);
	a.w += iA * s2Cross(A.r, PA);
	b.v = s2MulAdd(b.v, mB, PB);
	b.w += iB * s2Cross(B.r, PB);
	s2oSpringStore(j, bodyA, bodyB, a, b);
}

// ---- position forms ----------------------------------------------------------------------------------------------------

// NGS (xpbd == 0): Box2D 2.4's pulley position solve, impulse -k C, with C clamped to +/- s2_maxLinearCorrection (2.4 does
// not clamp). XPBD (xpbd == 1): lambda = -C / (1 / k) at zero compliance, nothing when 1 / k is 0.
static void s2oPulleyPosition(s2oSolve* s, s2oJoint* j, const s2oPulley* pj, int xpbd)
{
	s2oBody* bodyA = s->bodies + j->indexA;
	s2oBody* bodyB = s->bodies + j->indexB;
	s2Vec2 dcA = bodyA->dp, dcB = bodyB->dp;
	s2Rot qA = bodyA->q, qB = bodyB->q;
	float mA = j->invMassA, mB = j->invMassB, iA = j->invIA, iB = j->invIB;
	float ratio = pj->ratio;
	s2oRope A = s2oRopeAt(j->localAnchorA, pj->d0A, dcA, qA);
	s2oRope B = s2oRopeAt(j->localAnchorB, pj->d0B, dcB, qB);
	float kInv = s2oPulleyInvMass(j, &A, &B, ratio);
	float C = pj->constant - A.length - ratio * B.length;
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
		float k = kInv > 0.0f ? 1.0f / kInv : 0.0f;
		impulse = -k * S2_CLAMP(C, -s2_maxLinearCorrection, s2_maxLinearCorrection);
	}
	s2Vec2 PA = s2MulSV(-impulse, A.u);
	s2Vec2 PB = s2MulSV(-(ratio * impulse), B.u);
	dcA = s2MulAdd(dcA, mA, PA);
	qA = s2IntegrateRot(qA, iA * s2Cross(A.r, PA));
	dcB = s2MulAdd(dcB, mB, PB);
	qB = s2IntegrateRot(qB, iB * s2Cross(B.r, PB));
	s2oPrismaticStorePoses(j, bodyA, bodyB, dcA, qA, dcB, qB);
}

// ---- dispatch --------------------------------------------------------------------------------------------------------

static void s2oPulleyJointOp(s2oSolve* s, int op, s2oJoint* j)
{
	if (j->type != S2B_JOINT_PULLEY)
	{
		s2oWheelJointOp_Inner(s, op, j);
		return;
	}
	const s2oPulley* pj = s2oPulleyOf(j->slot);
	switch (op)
	{
		case S2O_J_WARM:
			s2oPulleyWarmStart(s, j, pj);
			break;
		case S2O_J_SOFT_BIAS:
		case S2O_J_SOFT_RELAX:
		case S2O_J_BAUMGARTE_BIAS:
		case S2O_J_BAUMGARTE_RELAX:
		case S2O_J_RIGID:
		{
			int kind = op == S2O_J_RIGID ? S2OP_RIGID : (op == S2O_J_SOFT_BIAS || op == S2O_J_SOFT_RELAX ? S2OP_SOFT : S2OP_BAUMGARTE);
			s2oPulleyVelocity(s, j, pj, kind, op == S2O_J_SOFT_BIAS || op == S2O_J_BAUMGARTE_BIAS);
			break;
		}
		case S2O_J_POSITION:
			s2oPulleyPosition(s, j, pj, 0);
			break;
		case S2O_J_XPBD:
			s2oPulleyPosition(s, j, pj, 1);
			break;
		default:
			break;
	}
}
