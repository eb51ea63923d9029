// solver2d-b200 — per-joint-constraint device functions (revolute + mouse), one thread per joint.
// Joints take part in the same colouring as contacts: a body appears at most once per group across both kinds.
// Float expressions follow the reference op for op; citations on each function. Reference quirks that parity
// depends on are kept on purpose (SURVEY.md §8a N2-N4).
#pragma once

#include "contact_kernels.cuh"
#include "shared/s2_collide.h"
#include "shared/s2_distance_joint.h"
#include "shared/s2_gear_joint.h"

#define S2B_JOINT_TYPE(flags) s2bJointType(flags)
// row flags of the joint-constraint stream only (jc.head.x): an XPBD spring row's body A / B is static, so its sub-step start
// pose is its pose (a static body's aux0 row is never written)
#define S2B_JC_STATIC_A 0x100
#define S2B_JC_STATIC_B 0x200
// row flags of the joint-constraint stream only: a weld row's angle / anchor constraint is a spring (DESIGN.md §3.15). XPBD
// soft weld rows also carry S2B_JC_STATIC_A / _B.
#define S2B_JC_SOFT_ANGULAR 0x400
#define S2B_JC_SOFT_LINEAR 0x800
#define S2B_JC_SOFT_WELD (S2B_JC_SOFT_ANGULAR | S2B_JC_SOFT_LINEAR)
// on a distance row (DESIGN.md §3.16), S2B_JC_SOFT_LINEAR marks a length that is not rigid: enableSpring with
// minLength < maxLength, whatever the hertz (a rope at hertz 0)

struct JointBodies
{
	int ia, ib;
	float4 velA, velB;
};

__device__ __forceinline__ void s2bStoreJointVelocities(const SolveArgs& a, int ia, int ib, float4 velA, float4 velB,
														s2Vec2 vA, float wA, s2Vec2 vB, float wB, float mA, float iA,
														float mB, float iB)
{
	if ((mA != 0.0f) | (iA != 0.0f))
	{
		a.bodies.vel[ia] = make_float4(vA.x, vA.y, wA, velA.w);
	}
	if ((mB != 0.0f) | (iB != 0.0f))
	{
		a.bodies.vel[ib] = make_float4(vB.x, vB.y, wB, velB.w);
	}
}

// ---------------------------------------------------------------------------------------------------------------
// prepare
// ---------------------------------------------------------------------------------------------------------------

enum JointPrepareKind
{
	JPREP_RIGID = 0, // s2PrepareRevolute       (reference src/revolute_joint.c:30-105)
	JPREP_SOFT = 1,	 // s2PrepareRevolute_Soft  (reference src/revolute_joint.c:421-506)
	JPREP_XPBD = 2,	 // s2PrepareRevolute_XPBD  (reference src/revolute_joint.c:792-823)
};

// a weld row's soft parts (DESIGN.md §3.15), run at the end of the weld's prepare; defined with the soft weld below
template <int KIND> __device__ __forceinline__ void s2bPrepareSoftWeld(const SolveArgs& a, int t, int slot);

// Builds row t of the joint-constraint stream from joint slot `slot`. `warmStart` is the flag the *variant* passes
// (TGS_Soft and SoftStep pass true regardless of the step flag, TGS_Sticky false; SURVEY §8a N3).
template <int KIND> __device__ __forceinline__ void s2bPrepareJointRows(const SolveArgs& a, int t, int slot, bool warmStart)
{
	const JointConstraintView& jc = a.jc;
	int4 head = a.joints.head[slot];
	int flags = head.x;
	int ia = head.y, ib = head.z;
	float4 anchors = a.joints.anchors[slot];
	float4 imp = a.joints.imp[slot];
	float4 limp = a.joints.limp[slot];

	float4 orgA = a.bodies.org[ia], orgB = a.bodies.org[ib];
	float4 posA = a.bodies.pos[ia], posB = a.bodies.pos[ib];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	float mA = a.bodies.vel[ia].w, mB = a.bodies.vel[ib].w;
	float iA = posA.z, iB = posB.z;

	jc.head[t] = make_int4(flags, ia, ib, slot);

	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_MOUSE)
	{
		// s2PrepareMouse (reference src/mouse_joint.c:31-83); the same function serves every variant
		float4 motor = a.joints.motor[slot];
		float4 target = a.joints.target[slot];
		s2Vec2 lB = s2Sub(V2(anchors.z, anchors.w), V2(orgB.z, orgB.w));
		float h = a.ctx.h;
		float zeta = motor.w;
		float omega = 2.0f * s2_pi * motor.z;
		float biasCoefficient = omega / (2.0f * zeta + h * omega);
		float c = h * omega * (2.0f * zeta + h * omega);
		float impulseCoefficient = 1.0f / (1.0f + c);
		float massCoefficient = c * impulseCoefficient;

		s2Vec2 rB = s2RotateVector(R2(poseB.z, poseB.w), lB);
		s2Mat22 K;
		K.cx.x = mB + iB * rB.y * rB.y;
		K.cx.y = -iB * rB.x * rB.y;
		K.cy.x = K.cx.y;
		K.cy.y = mB + iB * rB.x * rB.x;
		s2Mat22 pivot = s2GetInverse22(K);
		s2Vec2 centerDiff0 = s2Sub(V2(posB.x, posB.y), V2(target.x, target.y));

		jc.anchor[t] = make_float4(0.0f, 0.0f, lB.x, lB.y);
		jc.mass[t] = make_float4(0.0f, 0.0f, mB, iB);
		jc.d0ax[t] = make_float4(centerDiff0.x, centerDiff0.y, 0.0f, posB.w /* I of body B */);
		jc.lim[t] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		jc.motor[t] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		jc.coef[t] = make_float4(biasCoefficient, massCoefficient, impulseCoefficient, 0.0f);
		jc.pivot[t] = make_float4(pivot.cx.x, pivot.cx.y, pivot.cy.x, pivot.cy.y);
		jc.imp[t] = imp;
		jc.limp[t] = limp;
		return;
	}

	// revolute
	float4 lim = a.joints.lim[slot];
	float4 motor = a.joints.motor[slot];
	s2Vec2 lA = s2Sub(V2(anchors.x, anchors.y), V2(orgA.z, orgA.w));
	s2Vec2 lB = s2Sub(V2(anchors.z, anchors.w), V2(orgB.z, orgB.w));
	s2Vec2 centerDiff0 = s2Sub(V2(posB.x, posB.y), V2(posA.x, posA.y));

	jc.anchor[t] = make_float4(lA.x, lA.y, lB.x, lB.y);
	jc.mass[t] = make_float4(mA, iA, mB, iB);
	jc.lim[t] = lim;
	jc.coef[t] = make_float4(a.softJoint.bias, a.softJoint.mass, a.softJoint.impulse, 0.0f);

	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_GEAR)
	{
		// DESIGN.md §3.19: side 1's frame (the row's target) goes to d0ax and side 2's (the row's motor) to pivot, a prismatic
		// side's world anchor pC becoming the body's start offset c - pC; lim = (constant, ratio). Each revolute side's
		// unwound coordinate moves to the start pose in limp.xy under every variant (it is state, not an impulse). The gear
		// impulse is kept only with the variant's warm start, and never under XPBD.
		float4 f1 = a.joints.target[slot], f2 = a.joints.motor[slot];
		float theta1 = 0.0f, theta2 = 0.0f;
		if ((flags & S2B_JOINT_GEAR_PRISMATIC1) != 0)
		{
			f1 = make_float4(posA.x - f1.x, posA.y - f1.y, f1.z, f1.w);
		}
		else
		{
			theta1 = s2cGearRevolute(f1.x, f1.y, f1.z, limp.x, R2(poseA.z, poseA.w)).coordinate;
		}
		if ((flags & S2B_JOINT_GEAR_PRISMATIC2) != 0)
		{
			f2 = make_float4(posB.x - f2.x, posB.y - f2.y, f2.z, f2.w);
		}
		else
		{
			theta2 = s2cGearRevolute(f2.x, f2.y, f2.z, limp.y, R2(poseB.z, poseB.w)).coordinate;
		}
		jc.lim[t] = make_float4(lim.y, lim.x, 0.0f, 0.0f);
		jc.d0ax[t] = f1;
		jc.pivot[t] = f2;
		jc.motor[t] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		jc.imp[t] = make_float4(KIND != JPREP_XPBD && warmStart ? imp.x : 0.0f, 0.0f, 0.0f, 0.0f);
		jc.limp[t] = make_float4(theta1, theta2, 0.0f, 0.0f);
		return;
	}
	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_PULLEY)
	{
		// DESIGN.md §3.18: the row's lim = (ratio, lengthA, lengthB) and target = (groundA, groundB) become lim = (constant,
		// ratio) and d0ax = (cA - groundA, cB - groundB) at the start poses; the frame and the mass are formed fresh in each
		// solve. The rope impulse is kept only with the variant's warm start, and never under XPBD.
		float4 ground = a.joints.target[slot];
		jc.lim[t] = make_float4(lim.y + lim.x * lim.z, lim.x, 0.0f, 0.0f);
		jc.d0ax[t] = make_float4(posA.x - ground.x, posA.y - ground.y, posB.x - ground.z, posB.y - ground.w);
		jc.motor[t] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		jc.pivot[t] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		jc.imp[t] = make_float4(KIND != JPREP_XPBD && warmStart ? imp.x : 0.0f, 0.0f, 0.0f, 0.0f);
		jc.limp[t] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		return;
	}
	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_DISTANCE)
	{
		// DESIGN.md §3.16: lim = (rest length, min, max), motor = (maxMotorForce, motorSpeed); the frame and the axial mass
		// are formed fresh in each solve. A row that does not act keeps no impulse: the limits need the flag and
		// min < max, the rigid row needs the spring off or min == max.
		bool range = lim.y < lim.z;
		bool soft = (flags & S2B_JOINT_ENABLE_SPRING) != 0 && range;
		flags = (range ? flags : flags & ~S2B_JOINT_ENABLE_LIMIT) | (soft ? S2B_JC_SOFT_LINEAR : 0);
		jc.head[t] = make_int4(flags, ia, ib, slot);
		jc.motor[t] = make_float4(motor.x, motor.y, 0.0f, 0.0f);
		jc.d0ax[t] = make_float4(centerDiff0.x, centerDiff0.y, 0.0f, 0.0f);
		jc.pivot[t] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		if (KIND == JPREP_XPBD || warmStart == false)
		{
			imp = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
			limp = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		}
		if ((flags & S2B_JOINT_ENABLE_LIMIT) == 0)
		{
			limp.x = 0.0f;
			limp.y = 0.0f;
		}
		if ((flags & S2B_JOINT_ENABLE_MOTOR) == 0)
		{
			imp.z = 0.0f;
		}
		if (soft)
		{
			imp.x = 0.0f;
		}
		imp.y = 0.0f;
		jc.imp[t] = imp;
		jc.limp[t] = limp;
		return;
	}
	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_PRISMATIC || S2B_JOINT_TYPE(flags) == S2B_JOINT_MOTOR ||
		S2B_JOINT_TYPE(flags) == S2B_JOINT_WHEEL)
	{
		// DESIGN.md §3.9: the local axis rides in the motor row's spare zw; every mass is formed fresh in each solve.
		// Limit and motor impulses are kept only with their flag and a warm start, the block impulse with the warm start.
		// A motor joint (§3.10) carries its maximum force and correction factor in those zw instead, never has either
		// flag, and keeps its angular impulse (imp.z) exactly when it keeps its linear one. A wheel joint (§3.17) keeps its
		// perpendicular impulse in imp.x and its angular motor impulse in imp.y; imp.z stays 0.
		bool motorJoint = S2B_JOINT_TYPE(flags) == S2B_JOINT_MOTOR;
		bool wheel = S2B_JOINT_TYPE(flags) == S2B_JOINT_WHEEL;
		float4 axis = a.joints.target[slot];
		jc.motor[t] = motorJoint ? motor : make_float4(motor.x, motor.y, axis.z, axis.w);
		// a motor joint's angular row and a wheel joint's motor use the revolute's axial mass, 1 / (iA + iB) (0 when both
		// rotations are fixed)
		float motorAxialMass = (motorJoint || wheel) && iA + iB > 0.0f ? 1.0f / (iA + iB) : 0.0f;
		jc.d0ax[t] = make_float4(centerDiff0.x, centerDiff0.y, motorAxialMass, 0.0f);
		jc.pivot[t] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		if (KIND == JPREP_XPBD || warmStart == false)
		{
			imp = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
			limp = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		}
		if ((flags & S2B_JOINT_ENABLE_LIMIT) == 0)
		{
			limp.x = 0.0f;
			limp.y = 0.0f;
		}
		if ((flags & S2B_JOINT_ENABLE_MOTOR) == 0 && motorJoint == false)
		{
			imp.z = 0.0f;
		}
		if (wheel)
		{
			imp.y = (flags & S2B_JOINT_ENABLE_MOTOR) != 0 && motorAxialMass > 0.0f ? imp.y : 0.0f;
			imp.z = 0.0f;
		}
		jc.imp[t] = imp;
		jc.limp[t] = limp;
		return;
	}
	jc.motor[t] = make_float4(motor.x, motor.y, 0.0f, 0.0f);

	if (KIND == JPREP_XPBD)
	{
		jc.d0ax[t] = make_float4(centerDiff0.x, centerDiff0.y, 0.0f, 0.0f);
		jc.pivot[t] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		jc.imp[t] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		jc.limp[t] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		s2bPrepareSoftWeld<KIND>(a, t, slot);
		return;
	}

	s2Vec2 rA = s2RotateVector(R2(poseA.z, poseA.w), lA);
	s2Vec2 rB = s2RotateVector(R2(poseB.z, poseB.w), lB);
	s2Mat22 K;
	K.cx.x = mA + mB + rA.y * rA.y * iA + rB.y * rB.y * iB;
	K.cy.x = -rA.y * rA.x * iA - rB.y * rB.x * iB;
	K.cx.y = K.cy.x;
	K.cy.y = mA + mB + rA.x * rA.x * iA + rB.x * rB.x * iB;
	s2Mat22 pivot = s2GetInverse22(K);
	jc.pivot[t] = make_float4(pivot.cx.x, pivot.cx.y, pivot.cy.x, pivot.cy.y);

	float axialMass = iA + iB;
	bool fixedRotation;
	if (axialMass > 0.0f)
	{
		axialMass = 1.0f / axialMass;
		fixedRotation = false;
	}
	else
	{
		fixedRotation = true;
	}
	jc.d0ax[t] = make_float4(centerDiff0.x, centerDiff0.y, axialMass, 0.0f);

	bool enableLimit = (flags & S2B_JOINT_ENABLE_LIMIT) != 0;
	bool enableMotor = (flags & S2B_JOINT_ENABLE_MOTOR) != 0;
	bool weld = S2B_JOINT_TYPE(flags) == S2B_JOINT_WELD;
	if (enableLimit == false || fixedRotation || warmStart == false)
	{
		limp.x = 0.0f;
		limp.y = 0.0f;
	}
	// a weld's angular impulse (imp.z) is kept or dropped together with its point impulse
	if (weld ? warmStart == false : (enableMotor == false || fixedRotation || warmStart == false))
	{
		imp.z = 0.0f;
	}
	if (warmStart == false)
	{
		imp.x = 0.0f;
		imp.y = 0.0f;
	}
	jc.imp[t] = imp;
	jc.limp[t] = limp;
	if (weld)
	{
		s2bPrepareSoftWeld<KIND>(a, t, slot);
	}
}

// write the accumulated joint impulses back to the persistent joint columns
__device__ __forceinline__ void s2bStoreJointImpulses(const SolveArgs& a, int t)
{
	int slot = a.jc.head[t].w;
	a.joints.imp[slot] = a.jc.imp[t];
	a.joints.limp[slot] = a.jc.limp[t];
}

// ---------------------------------------------------------------------------------------------------------------
// joint spring (extension, DESIGN.md §3.14; definition: tests/spring_oracle.c). One soft row on the joint's axis toward zero
// error, solved before the joint's own rows in every velocity pass of every variant: the revolute's relative angle, the
// prismatic's translation. XPBD solves it as a compliant position row with damping instead. The spring is kept in functions
// of its own, run ahead of the joint's rows through memory (the bodies' velocity and pose rows, jc.imp.w), so the joint
// rows' code and register allocation stay as they are without it.
// Stream lanes: jc.coef.w = bias, jc.lim.w = mass scale, jc.d0ax.w = impulse scale (XPBD: 2 pi hertz h, damping ratio);
// jc.imp.w = accumulated spring impulse.
// ---------------------------------------------------------------------------------------------------------------

// the spring's part of prepare. A spring acts only on a revolute, prismatic, distance or wheel row with a positive hertz
// and, on a revolute row, a rotation to act on, on a distance row minLength < maxLength; every other row loses the flag in
// jc.head, so no solve or warm start evaluates a spring term for it, and gets a zero spring impulse.
template <int KIND> __device__ __forceinline__ void s2bPrepareSpring(const SolveArgs& a, int t, int slot, bool warmStart)
{
	const JointConstraintView& jc = a.jc;
	float* lambda = reinterpret_cast<float*>(jc.imp + t) + 3;
	int4 head = jc.head[t];
	int flags = head.x;
	if ((flags & S2B_JOINT_ENABLE_SPRING) == 0)
	{
		*lambda = 0.0f;
		return;
	}
	float4 motor = a.joints.motor[slot]; // hertz, damping ratio in zw
	float iA = a.bodies.pos[head.y].z, iB = a.bodies.pos[head.z].z;
	int type = S2B_JOINT_TYPE(flags);
	if ((type != S2B_JOINT_REVOLUTE && type != S2B_JOINT_PRISMATIC && type != S2B_JOINT_DISTANCE && type != S2B_JOINT_WHEEL) ||
		(motor.z > 0.0f) == false ||
		(type == S2B_JOINT_REVOLUTE && iA + iB == 0.0f) || (type == S2B_JOINT_DISTANCE && (flags & S2B_JC_SOFT_LINEAR) == 0))
	{
		jc.head[t] = make_int4(flags & ~S2B_JOINT_ENABLE_SPRING, head.y, head.z, head.w);
		*lambda = 0.0f;
		return;
	}
	// the mouse joint's coefficients and expression order, for the step h every variant passes to its joint solve
	float h = a.ctx.h;
	float zeta = motor.w;
	float omega = 2.0f * s2_pi * motor.z;
	if (KIND == JPREP_XPBD)
	{
		flags |= (S2B_BODY_TYPE(a.bodies.flags[head.y]) == S2B_BODY_STATIC ? S2B_JC_STATIC_A : 0) |
				 (S2B_BODY_TYPE(a.bodies.flags[head.z]) == S2B_BODY_STATIC ? S2B_JC_STATIC_B : 0);
		jc.head[t] = make_int4(flags, head.y, head.z, head.w);
		reinterpret_cast<float*>(jc.coef + t)[3] = omega * h;
		reinterpret_cast<float*>(jc.lim + t)[3] = zeta;
		*lambda = 0.0f;
		return;
	}
	float biasCoefficient = omega / (2.0f * zeta + h * omega);
	float c = h * omega * (2.0f * zeta + h * omega);
	float impulseCoefficient = 1.0f / (1.0f + c);
	float massCoefficient = c * impulseCoefficient;
	reinterpret_cast<float*>(jc.coef + t)[3] = biasCoefficient;
	reinterpret_cast<float*>(jc.lim + t)[3] = massCoefficient;
	reinterpret_cast<float*>(jc.d0ax + t)[3] = impulseCoefficient;
	// kept exactly when the variant's warm-start flag keeps the point impulse
	*lambda = warmStart ? a.joints.imp[slot].w : 0.0f;
}

// ---------------------------------------------------------------------------------------------------------------
// soft weld (extension, DESIGN.md §3.15; definition: tests/soft_weld_oracle.c). A weld row whose anchor or angle constraint
// has a positive hertz replaces the rigid form of that row with a force law, the same in every velocity flavour and pass;
// the NGS position pass skips a soft part and XPBD solves it as a compliant row with damping. Its impulse columns and warm
// start are the weld's (angular imp.z, point imp.xy). A weld row with both hertz at 0 gets no marker and takes the weld's
// own rows. Row lanes (s2bJointRow): the linear pair in hertz / dampingRatio, the angular pair in maxMotorTorque /
// motorSpeed, so joints.motor = (angularHertz, angularDampingRatio, linearHertz, linearDampingRatio).
// Stream lanes: jc.motor.xyz = the angular part's bias, mass scale, impulse scale (XPBD: 2 pi hertz h, damping ratio in
// xy); jc.lim.yzw = the linear part's (XPBD: yz).
// ---------------------------------------------------------------------------------------------------------------

template <int KIND> __device__ __forceinline__ void s2bPrepareSoftWeld(const SolveArgs& a, int t, int slot)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	if (S2B_JOINT_TYPE(head.x) != S2B_JOINT_WELD)
	{
		return;
	}
	float4 motor = a.joints.motor[slot];
	bool softAngular = motor.x > 0.0f, softLinear = motor.z > 0.0f;
	if (softAngular == false && softLinear == false)
	{
		return;
	}
	// the mouse joint's coefficients and expression order, for the step h every variant passes to its joint solve
	float h = a.ctx.h;
	float4 lim = jc.lim[t];
	float4 coefA = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
	int flags = head.x | (softAngular ? S2B_JC_SOFT_ANGULAR : 0) | (softLinear ? S2B_JC_SOFT_LINEAR : 0);
	for (int part = 0; part < 2; ++part)
	{
		float hertz = part == 0 ? motor.x : motor.z;
		float zeta = part == 0 ? motor.y : motor.w;
		if ((hertz > 0.0f) == false)
		{
			continue;
		}
		float omega = 2.0f * s2_pi * hertz;
		float x, y, z = 0.0f;
		if (KIND == JPREP_XPBD)
		{
			x = omega * h;
			y = zeta;
		}
		else
		{
			x = omega / (2.0f * zeta + h * omega);
			float c = h * omega * (2.0f * zeta + h * omega);
			z = 1.0f / (1.0f + c);
			y = c * z;
		}
		if (part == 0)
		{
			coefA = make_float4(x, y, z, 0.0f);
		}
		else
		{
			lim = make_float4(lim.x, x, y, z);
		}
	}
	if (KIND == JPREP_XPBD)
	{
		flags |= (S2B_BODY_TYPE(a.bodies.flags[head.y]) == S2B_BODY_STATIC ? S2B_JC_STATIC_A : 0) |
				 (S2B_BODY_TYPE(a.bodies.flags[head.z]) == S2B_BODY_STATIC ? S2B_JC_STATIC_B : 0);
	}
	jc.head[t] = make_int4(flags, head.y, head.z, head.w);
	jc.motor[t] = coefA;
	jc.lim[t] = lim;
}

// Builds row t of the joint-constraint stream from joint slot `slot`: the joint's rows (a weld's with its soft parts), then
// its spring.
template <int KIND> __device__ __forceinline__ void s2bPrepareJoint(const SolveArgs& a, int t, int slot, bool warmStart)
{
	s2bPrepareJointRows<KIND>(a, t, slot, warmStart);
	s2bPrepareSpring<KIND>(a, t, slot, warmStart);
}

// ---------------------------------------------------------------------------------------------------------------
// prismatic joint (extension, DESIGN.md §3.9; definition: tests/prismatic_oracle.c). Body B slides along an axis fixed
// in body A: rows motor, lower limit, upper limit (along the axis), then a 2x2 block holding the perpendicular
// separation and the relative angle. Every mass depends on the current separation d, so each solve forms it fresh.
// Row columns: lim = (referenceAngle, lowerTranslation, upperTranslation), motor = (maxMotorForce, motorSpeed,
// localAxisA.xy), imp = (perpendicular, angular, motor), limp = (lower, upper).
// ---------------------------------------------------------------------------------------------------------------

// the joint frame at the given poses: centre-of-mass-relative anchors, d = (dcB - dcA) + (rB - rA) + centerDiff0 and
// the world axis
struct PrismaticFrame
{
	s2Vec2 rA, rB, d, axis;
};

__device__ __forceinline__ PrismaticFrame s2bPrismaticFrame(float4 anchor, float4 d0, float4 motor, s2Vec2 dcA, s2Rot qA, s2Vec2 dcB,
															s2Rot qB)
{
	PrismaticFrame f;
	f.rA = s2RotateVector(qA, V2(anchor.x, anchor.y));
	f.rB = s2RotateVector(qB, V2(anchor.z, anchor.w));
	f.d = s2Add(s2Add(s2Sub(dcB, dcA), s2Sub(f.rB, f.rA)), V2(d0.x, d0.y));
	f.axis = s2RotateVector(qA, V2(motor.z, motor.w));
	return f;
}

// the distance joint's frame at the given poses (DESIGN.md §3.16): centre-of-mass-relative anchors, the length of
// d = (dcB - dcA) + (rB - rA) + centerDiff0 and the unit axis along d (zero for a degenerate d)
struct DistanceFrame
{
	s2Vec2 rA, rB, axis;
	float length;
};

__device__ __forceinline__ DistanceFrame s2bDistanceFrame(float4 anchor, float4 d0, s2Vec2 dcA, s2Rot qA, s2Vec2 dcB, s2Rot qB)
{
	DistanceFrame f;
	f.rA = s2RotateVector(qA, V2(anchor.x, anchor.y));
	f.rB = s2RotateVector(qB, V2(anchor.z, anchor.w));
	s2Vec2 d = s2Add(s2Add(s2Sub(dcB, dcA), s2Sub(f.rB, f.rA)), V2(d0.x, d0.y));
	f.axis = s2cGetLengthAndNormalize(&f.length, d);
	return f;
}

// what warm starting adds to each body: v -/+= m * P, w -/+= i * L. Shared by the constraint-by-constraint warm start and
// the per-body gather (warm_gather.cuh), so both add the same bits. Prismatic, distance and wheel rows; a wheel row's imp.y
// is its angular motor impulse, which enters L as the prismatic's angular impulse does (DESIGN.md §3.17).
struct PrismaticWarm
{
	s2Vec2 P;
	float LA, LB;
};

__device__ __forceinline__ PrismaticWarm s2bPrismaticWarmTerms(const SolveArgs& a, int t)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	float4 imp = jc.imp[t];
	float4 limp = jc.limp[t];
	float4 poseA = a.bodies.pose[head.y], poseB = a.bodies.pose[head.z];
	// axial = spring + motor + lower - upper (DESIGN.md §3.14); a row without a spring adds no spring term
	float axialImpulse = ((head.x & S2B_JOINT_ENABLE_SPRING) != 0 ? imp.w + imp.z : imp.z) + limp.x - limp.y;
	PrismaticWarm w;
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_DISTANCE)
	{
		// DESIGN.md §3.16: the rigid row's impulse joins the sum only where that row acts
		DistanceFrame f = s2bDistanceFrame(jc.anchor[t], jc.d0ax[t], V2(poseA.x, poseA.y), R2(poseA.z, poseA.w),
										   V2(poseB.x, poseB.y), R2(poseB.z, poseB.w));
		axialImpulse = (head.x & S2B_JC_SOFT_LINEAR) == 0 ? imp.x + axialImpulse : axialImpulse;
		w.P = s2MulSV(axialImpulse, f.axis);
		w.LA = axialImpulse * s2Cross(f.rA, f.axis);
		w.LB = axialImpulse * s2Cross(f.rB, f.axis);
		return w;
	}
	PrismaticFrame f = s2bPrismaticFrame(jc.anchor[t], jc.d0ax[t], jc.motor[t], V2(poseA.x, poseA.y), R2(poseA.z, poseA.w),
										 V2(poseB.x, poseB.y), R2(poseB.z, poseB.w));
	s2Vec2 perp = s2LeftPerp(f.axis);
	s2Vec2 dA = s2Add(f.d, f.rA);
	w.P = s2Add(s2MulSV(axialImpulse, f.axis), s2MulSV(imp.x, perp));
	w.LA = axialImpulse * s2Cross(dA, f.axis) + imp.x * s2Cross(dA, perp) + imp.y;
	w.LB = axialImpulse * s2Cross(f.rB, f.axis) + imp.x * s2Cross(f.rB, perp) + imp.y;
	return w;
}

enum PrismaticSolveKind
{
	PSOLVE_SOFT = 0,	  // Jacobi, PGS_Soft, SoftStep, TGS_Soft
	PSOLVE_BAUMGARTE = 1, // PGS, TGS_Sticky
	PSOLVE_RIGID = 2,	  // PGS_NGS, PGS_NGS_Block, TGS_NGS
};

// the bias, mass scale and impulse scale of one row with position error C (a limit row when `limit`: speculative when
// the limit is not reached)
template <int KIND>
__device__ __forceinline__ float3 s2bPrismaticBias(float C, bool limit, float4 coef, float h, float inv_h, bool useBias)
{
	float bias = 0.0f, massScale = 1.0f, impulseScale = 0.0f;
	if (KIND == PSOLVE_RIGID)
	{
		bias = limit ? S2_MAX(C, 0.0f) / h : 0.0f;
	}
	else if (limit && C > 0.0f)
	{
		bias = C * inv_h;
	}
	else if (KIND == PSOLVE_BAUMGARTE)
	{
		bias = s2_baumgarte * inv_h * C;
	}
	else if (useBias)
	{
		bias = coef.x * C;
		massScale = coef.y;
		impulseScale = coef.z;
	}
	return make_float3(bias, massScale, impulseScale);
}

// the axial rows the prismatic and distance joints share (DESIGN.md §3.9, §3.16): the motor, then the lower and upper limit,
// each along `axis` with lever arms a1 (body A) and a2 (body B) and the axial mass. x is the joint's coordinate along the
// axis (the prismatic's translation, the distance joint's length), lim.yz its limits, motor.xy the maximum force and the
// speed; imp.z is the motor impulse and limp.xy the limit impulses.
template <int KIND>
__device__ __forceinline__ void s2bSolveAxialRows(int flags, s2Vec2 axis, float a1, float a2, float axialMass, float x, float4 lim,
												  float4 motor, float4 coef, float h, float inv_h, bool useBias, float mA, float iA,
												  float mB, float iB, float4& imp, float4& limp, s2Vec2& vA, float& wA, s2Vec2& vB,
												  float& wB)
{
	if (flags & S2B_JOINT_ENABLE_MOTOR)
	{
		float Cdot = s2Dot(axis, s2Sub(vB, vA)) + a2 * wB - a1 * wA;
		float impulse = axialMass * (motor.y - Cdot);
		float oldImpulse = imp.z;
		float maxImpulse = h * motor.x;
		imp.z = S2_CLAMP(oldImpulse + impulse, -maxImpulse, maxImpulse);
		impulse = imp.z - oldImpulse;
		s2Vec2 P = s2MulSV(impulse, axis);
		vA = s2MulSub(vA, mA, P);
		wA -= iA * (impulse * a1);
		vB = s2MulAdd(vB, mB, P);
		wB += iB * (impulse * a2);
	}

	if (flags & S2B_JOINT_ENABLE_LIMIT)
	{
		// lower limit
		{
			float3 s = s2bPrismaticBias<KIND>(x - lim.y, true, coef, h, inv_h, useBias);
			float Cdot = s2Dot(axis, s2Sub(vB, vA)) + a2 * wB - a1 * wA;
			float impulse = -axialMass * s.y * (Cdot + s.x) - s.z * limp.x;
			float oldImpulse = limp.x;
			limp.x = S2_MAX(oldImpulse + impulse, 0.0f);
			impulse = limp.x - oldImpulse;
			s2Vec2 P = s2MulSV(impulse, axis);
			vA = s2MulSub(vA, mA, P);
			wA -= iA * (impulse * a1);
			vB = s2MulAdd(vB, mB, P);
			wB += iB * (impulse * a2);
		}
		// upper limit (signs flipped so C stays positive when satisfied); it relaxes with its own impulse
		{
			float3 s = s2bPrismaticBias<KIND>(lim.z - x, true, coef, h, inv_h, useBias);
			float Cdot = s2Dot(axis, s2Sub(vA, vB)) + a1 * wA - a2 * wB;
			float impulse = -axialMass * s.y * (Cdot + s.x) - s.z * limp.y;
			float oldImpulse = limp.y;
			limp.y = S2_MAX(oldImpulse + impulse, 0.0f);
			impulse = limp.y - oldImpulse;
			s2Vec2 P = s2MulSV(impulse, axis);
			vA = s2MulAdd(vA, mA, P);
			wA += iA * (impulse * a1);
			vB = s2MulSub(vB, mB, P);
			wB -= iB * (impulse * a2);
		}
	}
}

template <int KIND>
__device__ __forceinline__ void s2bSolvePrismaticVelocity(const SolveArgs& a, int t, float h, float inv_h, bool useBias)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 mass = jc.mass[t];
	float4 lim = jc.lim[t];
	float4 motor = jc.motor[t];
	float4 coef = jc.coef[t];
	float4 imp = jc.imp[t];
	float4 limp = jc.limp[t];
	float4 velA = a.bodies.vel[ia], velB = a.bodies.vel[ib];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 vA = V2(velA.x, velA.y), vB = V2(velB.x, velB.y);
	float wA = velA.z, wB = velB.z;
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	PrismaticFrame f = s2bPrismaticFrame(jc.anchor[t], jc.d0ax[t], motor, V2(poseA.x, poseA.y), qA, V2(poseB.x, poseB.y), qB);
	s2Vec2 axis = f.axis;
	s2Vec2 dA = s2Add(f.d, f.rA);
	float translation = s2Dot(axis, f.d);
	float a1 = s2Cross(dA, axis), a2 = s2Cross(f.rB, axis);
	float k = mA + mB + iA * a1 * a1 + iB * a2 * a2;
	float axialMass = k > 0.0f ? 1.0f / k : 0.0f;

	s2bSolveAxialRows<KIND>(head.x, axis, a1, a2, axialMass, translation, lim, motor, coef, h, inv_h, useBias, mA, iA, mB, iB, imp,
							limp, vA, wA, vB, wB);

	// the 2x2 block: perpendicular separation and relative angle
	{
		s2Vec2 perp = s2LeftPerp(axis);
		float sA = s2Cross(dA, perp), sB = s2Cross(f.rB, perp);
		s2Vec2 Cdot = V2(s2Dot(perp, s2Sub(vB, vA)) + sB * wB - sA * wA, wB - wA);
		s2Vec2 C = V2(s2Dot(perp, f.d), s2UnwindAngle(s2RelativeAngle(qB, qA) - lim.x));
		float3 sx = s2bPrismaticBias<KIND>(C.x, false, coef, h, inv_h, useBias);
		float3 sy = s2bPrismaticBias<KIND>(C.y, false, coef, h, inv_h, useBias);
		float k11 = mA + mB + iA * sA * sA + iB * sB * sB;
		float k12 = iA * sA + iB * sB;
		float k22 = iA + iB;
		if (k22 == 0.0f)
		{
			k22 = 1.0f; // both rotations fixed: keeps K invertible
		}
		s2Mat22 K;
		K.cx = V2(k11, k12);
		K.cy = V2(k12, k22);
		s2Vec2 b = s2Solve22(K, V2(Cdot.x + sx.x, Cdot.y + sy.x));
		s2Vec2 impulse = V2(-sx.y * b.x - sx.z * imp.x, -sy.y * b.y - sy.z * imp.y);
		imp.x += impulse.x;
		imp.y += impulse.y;
		s2Vec2 P = s2MulSV(impulse.x, perp);
		float LA = impulse.x * sA + impulse.y;
		float LB = impulse.x * sB + impulse.y;
		vA = s2MulSub(vA, mA, P);
		wA -= iA * LA;
		vB = s2MulAdd(vB, mB, P);
		wB += iB * LB;
	}

	jc.imp[t] = imp;
	jc.limp[t] = limp;
	s2bStoreJointVelocities(a, ia, ib, velA, velB, vA, wA, vB, wB, mA, iA, mB, iB);
}

// the prismatic's NGS limit correction along its axis, on the given poses (slop s2_linearSlop; equal limits within
// 2 s2_linearSlop are held both ways). The wheel joint's NGS pass runs it too (DESIGN.md §3.17).
__device__ __forceinline__ void s2bAxialLimitPosition(float4 anchor, float4 d0, float4 motor, float4 lim, float mA, float iA, float mB,
													  float iB, s2Vec2& dcA, s2Rot& qA, s2Vec2& dcB, s2Rot& qB)
{
	PrismaticFrame f = s2bPrismaticFrame(anchor, d0, motor, dcA, qA, dcB, qB);
	s2Vec2 dA = s2Add(f.d, f.rA);
	float a1 = s2Cross(dA, f.axis), a2 = s2Cross(f.rB, f.axis);
	float translation = s2Dot(f.axis, f.d);
	float C = 0.0f;
	if (S2_ABS(lim.z - lim.y) < 2.0f * s2_linearSlop)
	{
		C = S2_CLAMP(translation - lim.y, -s2_maxLinearCorrection, s2_maxLinearCorrection);
	}
	else if (translation <= lim.y)
	{
		C = S2_CLAMP(translation - lim.y + s2_linearSlop, -s2_maxLinearCorrection, 0.0f);
	}
	else if (translation >= lim.z)
	{
		C = S2_CLAMP(translation - lim.z - s2_linearSlop, 0.0f, s2_maxLinearCorrection);
	}
	float k = mA + mB + iA * a1 * a1 + iB * a2 * a2;
	float impulse = k > 0.0f ? -C / k : 0.0f;
	s2Vec2 P = s2MulSV(impulse, f.axis);
	dcA = s2MulSub(dcA, mA, P);
	qA = s2IntegrateRot(qA, -iA * (impulse * a1));
	dcB = s2MulAdd(dcB, mB, P);
	qB = s2IntegrateRot(qB, iB * (impulse * a2));
}

// XPBD, zero compliance: the perpendicular row, C = perp . d, on the given poses. The prismatic's and the wheel's.
__device__ __forceinline__ void s2bPerpendicularXpbd(float4 anchor, float4 d0, float4 motor, float mA, float iA, float mB, float iB,
													 s2Vec2& dcA, s2Rot& qA, s2Vec2& dcB, s2Rot& qB)
{
	PrismaticFrame f = s2bPrismaticFrame(anchor, d0, motor, dcA, qA, dcB, qB);
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

// XPBD, zero compliance: a violated translation limit as a position inequality, on the given poses. The prismatic's and
// the wheel's.
__device__ __forceinline__ void s2bAxialLimitXpbd(float4 anchor, float4 d0, float4 motor, float4 lim, float mA, float iA, float mB,
												  float iB, s2Vec2& dcA, s2Rot& qA, s2Vec2& dcB, s2Rot& qB)
{
	PrismaticFrame f = s2bPrismaticFrame(anchor, d0, motor, dcA, qA, dcB, qB);
	float a1 = s2Cross(s2Add(f.d, f.rA), f.axis), a2 = s2Cross(f.rB, f.axis);
	float translation = s2Dot(f.axis, f.d);
	float C = 0.0f;
	if (translation < lim.y)
	{
		C = translation - lim.y;
	}
	else if (translation > lim.z)
	{
		C = translation - lim.z;
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

// NGS position pass: the block on the current poses (corrections clamped), then the limit row on the corrected poses
__device__ __forceinline__ void s2bSolvePrismaticPosition(const SolveArgs& a, int t)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 lim = jc.lim[t];
	float4 motor = jc.motor[t];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;

	{
		PrismaticFrame f = s2bPrismaticFrame(anchor, d0, motor, dcA, qA, dcB, qB);
		s2Vec2 perp = s2LeftPerp(f.axis);
		s2Vec2 dA = s2Add(f.d, f.rA);
		float sA = s2Cross(dA, perp), sB = s2Cross(f.rB, perp);
		s2Vec2 C;
		C.x = S2_CLAMP(s2Dot(perp, f.d), -s2_maxLinearCorrection, s2_maxLinearCorrection);
		C.y = S2_CLAMP(s2UnwindAngle(s2RelativeAngle(qB, qA) - lim.x), -s2_maxAngularCorrection, s2_maxAngularCorrection);
		float k11 = mA + mB + iA * sA * sA + iB * sB * sB;
		float k12 = iA * sA + iB * sB;
		float k22 = iA + iB;
		if (k22 == 0.0f)
		{
			k22 = 1.0f;
		}
		s2Mat22 K;
		K.cx = V2(k11, k12);
		K.cy = V2(k12, k22);
		s2Vec2 impulse = s2Solve22(K, s2Neg(C));
		s2Vec2 P = s2MulSV(impulse.x, perp);
		float LA = impulse.x * sA + impulse.y;
		float LB = impulse.x * sB + impulse.y;
		dcA = s2MulSub(dcA, mA, P);
		qA = s2IntegrateRot(qA, -iA * LA);
		dcB = s2MulAdd(dcB, mB, P);
		qB = s2IntegrateRot(qB, iB * LB);
	}

	if (head.x & S2B_JOINT_ENABLE_LIMIT)
	{
		s2bAxialLimitPosition(anchor, d0, motor, lim, mA, iA, mB, iB, dcA, qA, dcB, qB);
	}

	if ((mA != 0.0f) || (iA != 0.0f))
	{
		a.bodies.pose[ia] = make_float4(dcA.x, dcA.y, qA.s, qA.c);
	}
	if ((mB != 0.0f) || (iB != 0.0f))
	{
		a.bodies.pose[ib] = make_float4(dcB.x, dcB.y, qB.s, qB.c);
	}
}

// XPBD, zero compliance: the angle row (as the weld's), the perpendicular row, then the limits as position inequalities.
// The motor is not applied, as the revolute joint's XPBD form ignores its motor.
__device__ __forceinline__ void s2bSolvePrismaticXpbd(const SolveArgs& a, int t)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 lim = jc.lim[t];
	float4 motor = jc.motor[t];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;

	if (iA + iB != 0.0f)
	{
		float C = s2UnwindAngle(s2RelativeAngle(qB, qA) - lim.x);
		float p = -C / (iA + iB);
		qA = s2IntegrateRot(qA, -iA * p);
		qB = s2IntegrateRot(qB, iB * p);
	}

	s2bPerpendicularXpbd(anchor, d0, motor, mA, iA, mB, iB, dcA, qA, dcB, qB);

	if (head.x & S2B_JOINT_ENABLE_LIMIT)
	{
		s2bAxialLimitXpbd(anchor, d0, motor, lim, mA, iA, mB, iB, dcA, qA, dcB, qB);
	}

	if ((mA != 0.0f) || (iA != 0.0f))
	{
		a.bodies.pose[ia] = make_float4(dcA.x, dcA.y, qA.s, qA.c);
	}
	if ((mB != 0.0f) || (iB != 0.0f))
	{
		a.bodies.pose[ib] = make_float4(dcB.x, dcB.y, qB.s, qB.c);
	}
}

// ---------------------------------------------------------------------------------------------------------------
// distance joint (extension, DESIGN.md §3.16; definition: tests/distance_oracle.c). Holds anchor B at a distance from
// anchor A along the line between them: rows spring (s2bSolveSpringVelocity, ahead of these), motor, lower limit, upper
// limit (the prismatic's axial rows, s2bSolveAxialRows) and the rigid length row, each along the axis of the current d.
// Row columns: lim = (rest length, minLength, maxLength), motor = (maxMotorForce, motorSpeed), imp = (rigid, 0, motor,
// spring), limp = (lower, upper). Prepare drops the limit flag where minLength == maxLength and marks a row whose length
// is not rigid with S2B_JC_SOFT_LINEAR.
// ---------------------------------------------------------------------------------------------------------------
template <int KIND>
__device__ __forceinline__ void s2bSolveDistanceVelocity(const SolveArgs& a, int t, float h, float inv_h, bool useBias)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 mass = jc.mass[t];
	float4 lim = jc.lim[t];
	float4 motor = jc.motor[t];
	float4 coef = jc.coef[t];
	float4 imp = jc.imp[t];
	float4 limp = jc.limp[t];
	float4 velA = a.bodies.vel[ia], velB = a.bodies.vel[ib];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 vA = V2(velA.x, velA.y), vB = V2(velB.x, velB.y);
	float wA = velA.z, wB = velB.z;
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	DistanceFrame f = s2bDistanceFrame(jc.anchor[t], jc.d0ax[t], V2(poseA.x, poseA.y), R2(poseA.z, poseA.w), V2(poseB.x, poseB.y),
									   R2(poseB.z, poseB.w));
	s2Vec2 axis = f.axis;
	float crA = s2Cross(f.rA, axis), crB = s2Cross(f.rB, axis);
	float k = mA + mB + iA * crA * crA + iB * crB * crB;
	float axialMass = k > 0.0f ? 1.0f / k : 0.0f;

	s2bSolveAxialRows<KIND>(head.x, axis, crA, crB, axialMass, f.length, lim, motor, coef, h, inv_h, useBias, mA, iA, mB, iB, imp,
							limp, vA, wA, vB, wB);

	if ((head.x & S2B_JC_SOFT_LINEAR) == 0)
	{
		// the rigid row: the flavour's bilateral form of C = length - rest length
		float3 s = s2bPrismaticBias<KIND>(f.length - lim.x, false, coef, h, inv_h, useBias);
		float Cdot = s2Dot(axis, s2Sub(vB, vA)) + crB * wB - crA * wA;
		float impulse = -axialMass * s.y * (Cdot + s.x) - s.z * imp.x;
		imp.x += impulse;
		s2Vec2 P = s2MulSV(impulse, axis);
		vA = s2MulSub(vA, mA, P);
		wA -= iA * (impulse * crA);
		vB = s2MulAdd(vB, mB, P);
		wB += iB * (impulse * crB);
	}

	jc.imp[t] = imp;
	jc.limp[t] = limp;
	s2bStoreJointVelocities(a, ia, ib, velA, velB, vA, wA, vB, wB, mA, iA, mB, iB);
}

// one axial position correction along the frame's axis: lambda = -C / k (0 when k is 0), applied to the poses
__device__ __forceinline__ void s2bDistanceCorrect(const DistanceFrame& f, float C, float mA, float iA, float mB, float iB, s2Vec2& dcA,
												   s2Rot& qA, s2Vec2& dcB, s2Rot& qB)
{
	float crA = s2Cross(f.rA, f.axis), crB = s2Cross(f.rB, f.axis);
	float k = mA + mB + iA * crA * crA + iB * crB * crB;
	float axialMass = k > 0.0f ? 1.0f / k : 0.0f;
	float impulse = -axialMass * C;
	s2Vec2 P = s2MulSV(impulse, f.axis);
	dcA = s2MulSub(dcA, mA, P);
	qA = s2IntegrateRot(qA, -iA * (impulse * crA));
	dcB = s2MulAdd(dcB, mB, P);
	qB = s2IntegrateRot(qB, iB * (impulse * crB));
}

// NGS position pass (Box2D 2.4's distance position solve): a rigid length corrects length - rest length; a length that is
// not rigid corrects only a violated limit. Clamped to +/- s2_maxLinearCorrection. The spring and the motor do nothing.
__device__ __forceinline__ void s2bSolveDistancePosition(const SolveArgs& a, int t)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 mass = jc.mass[t];
	float4 lim = jc.lim[t];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	DistanceFrame f = s2bDistanceFrame(jc.anchor[t], jc.d0ax[t], dcA, qA, dcB, qB);
	float C;
	if ((head.x & S2B_JC_SOFT_LINEAR) == 0)
	{
		C = f.length - lim.x;
	}
	else if ((head.x & S2B_JOINT_ENABLE_LIMIT) && f.length < lim.y)
	{
		C = f.length - lim.y;
	}
	else if ((head.x & S2B_JOINT_ENABLE_LIMIT) && f.length > lim.z)
	{
		C = f.length - lim.z;
	}
	else
	{
		return;
	}
	C = S2_CLAMP(C, -s2_maxLinearCorrection, s2_maxLinearCorrection);
	s2bDistanceCorrect(f, C, mA, iA, mB, iB, dcA, qA, dcB, qB);
	if ((mA != 0.0f) || (iA != 0.0f))
	{
		a.bodies.pose[ia] = make_float4(dcA.x, dcA.y, qA.s, qA.c);
	}
	if ((mB != 0.0f) || (iB != 0.0f))
	{
		a.bodies.pose[ib] = make_float4(dcB.x, dcB.y, qB.s, qB.c);
	}
}

// XPBD, zero compliance: a violated limit as a position inequality, then the rigid length row on the corrected poses. The
// spring (s2bSolveSpringXpbd) runs ahead; the motor is not applied, as the prismatic's XPBD form ignores its motor.
__device__ __forceinline__ void s2bSolveDistanceXpbd(const SolveArgs& a, int t)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 lim = jc.lim[t];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;

	if (head.x & S2B_JOINT_ENABLE_LIMIT)
	{
		DistanceFrame f = s2bDistanceFrame(anchor, d0, dcA, qA, dcB, qB);
		float C = 0.0f;
		if (f.length < lim.y)
		{
			C = f.length - lim.y;
		}
		else if (f.length > lim.z)
		{
			C = f.length - lim.z;
		}
		if (C != 0.0f)
		{
			s2bDistanceCorrect(f, C, mA, iA, mB, iB, dcA, qA, dcB, qB);
		}
	}

	if ((head.x & S2B_JC_SOFT_LINEAR) == 0)
	{
		DistanceFrame f = s2bDistanceFrame(anchor, d0, dcA, qA, dcB, qB);
		s2bDistanceCorrect(f, f.length - lim.x, mA, iA, mB, iB, dcA, qA, dcB, qB);
	}

	if ((mA != 0.0f) || (iA != 0.0f))
	{
		a.bodies.pose[ia] = make_float4(dcA.x, dcA.y, qA.s, qA.c);
	}
	if ((mB != 0.0f) || (iB != 0.0f))
	{
		a.bodies.pose[ib] = make_float4(dcB.x, dcB.y, qB.s, qB.c);
	}
}

// ---------------------------------------------------------------------------------------------------------------
// wheel joint (extension, DESIGN.md §3.17; definition: tests/wheel_oracle.c). Body B's anchor slides along an axis fixed in
// body A and B turns freely: rows spring (s2bSolveSpringVelocity, ahead of these), the motor on the relative rotation (the
// revolute's form, axial mass 1 / (iA + iB) in jc.d0ax.z), lower and upper translation limit (s2bSolveAxialRows with the
// motor flag masked off) and the perpendicular point-on-line row. The frame is the prismatic's. Row columns: lim =
// (unused, lowerTranslation, upperTranslation), motor = (maxMotorTorque, motorSpeed, localAxisA.xy), imp = (perpendicular,
// angular motor, 0, spring), limp = (lower, upper).
// ---------------------------------------------------------------------------------------------------------------
template <int KIND>
__device__ __forceinline__ void s2bSolveWheelVelocity(const SolveArgs& a, int t, float h, float inv_h, bool useBias)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 lim = jc.lim[t];
	float4 motor = jc.motor[t];
	float4 coef = jc.coef[t];
	float4 imp = jc.imp[t];
	float4 limp = jc.limp[t];
	float4 velA = a.bodies.vel[ia], velB = a.bodies.vel[ib];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 vA = V2(velA.x, velA.y), vB = V2(velB.x, velB.y);
	float wA = velA.z, wB = velB.z;
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	PrismaticFrame f = s2bPrismaticFrame(jc.anchor[t], d0, motor, V2(poseA.x, poseA.y), R2(poseA.z, poseA.w), V2(poseB.x, poseB.y),
										 R2(poseB.z, poseB.w));
	s2Vec2 axis = f.axis;
	s2Vec2 dA = s2Add(f.d, f.rA);
	float translation = s2Dot(axis, f.d);
	float a1 = s2Cross(dA, axis), a2 = s2Cross(f.rB, axis);
	float k = mA + mB + iA * a1 * a1 + iB * a2 * a2;
	float axialMass = k > 0.0f ? 1.0f / k : 0.0f;

	if ((head.x & S2B_JOINT_ENABLE_MOTOR) && d0.z > 0.0f)
	{
		float Cdot = wB - wA - motor.y;
		float impulse = -d0.z * Cdot;
		float oldImpulse = imp.y;
		float maxImpulse = h * motor.x;
		imp.y = S2_CLAMP(oldImpulse + impulse, -maxImpulse, maxImpulse);
		impulse = imp.y - oldImpulse;
		wA -= iA * impulse;
		wB += iB * impulse;
	}

	s2bSolveAxialRows<KIND>(head.x & ~S2B_JOINT_ENABLE_MOTOR, axis, a1, a2, axialMass, translation, lim, motor, coef, h, inv_h,
							useBias, mA, iA, mB, iB, imp, limp, vA, wA, vB, wB);

	// the point-on-line row: C = perp . d
	{
		s2Vec2 perp = s2LeftPerp(axis);
		float sA = s2Cross(dA, perp), sB = s2Cross(f.rB, perp);
		float3 s = s2bPrismaticBias<KIND>(s2Dot(perp, f.d), false, coef, h, inv_h, useBias);
		float Cdot = s2Dot(perp, s2Sub(vB, vA)) + sB * wB - sA * wA;
		float kp = mA + mB + iA * sA * sA + iB * sB * sB;
		float perpMass = kp > 0.0f ? 1.0f / kp : 0.0f;
		float impulse = -perpMass * s.y * (Cdot + s.x) - s.z * imp.x;
		imp.x += impulse;
		s2Vec2 P = s2MulSV(impulse, perp);
		vA = s2MulSub(vA, mA, P);
		wA -= iA * (impulse * sA);
		vB = s2MulAdd(vB, mB, P);
		wB += iB * (impulse * sB);
	}

	jc.imp[t] = imp;
	jc.limp[t] = limp;
	s2bStoreJointVelocities(a, ia, ib, velA, velB, vA, wA, vB, wB, mA, iA, mB, iB);
}

// NGS position pass: the perpendicular row on the current poses (C clamped to +/- s2_maxLinearCorrection, impulse -C / k),
// then the prismatic's limit correction on the corrected poses. The spring and the motor do nothing.
__device__ __forceinline__ void s2bSolveWheelPosition(const SolveArgs& a, int t)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 lim = jc.lim[t];
	float4 motor = jc.motor[t];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;

	{
		PrismaticFrame f = s2bPrismaticFrame(anchor, d0, motor, dcA, qA, dcB, qB);
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

	if (head.x & S2B_JOINT_ENABLE_LIMIT)
	{
		s2bAxialLimitPosition(anchor, d0, motor, lim, mA, iA, mB, iB, dcA, qA, dcB, qB);
	}

	if ((mA != 0.0f) || (iA != 0.0f))
	{
		a.bodies.pose[ia] = make_float4(dcA.x, dcA.y, qA.s, qA.c);
	}
	if ((mB != 0.0f) || (iB != 0.0f))
	{
		a.bodies.pose[ib] = make_float4(dcB.x, dcB.y, qB.s, qB.c);
	}
}

// XPBD, zero compliance: the perpendicular row, then a violated limit. The spring (s2bSolveSpringXpbd) runs ahead; the
// motor is not applied, as no joint's XPBD form applies its motor.
__device__ __forceinline__ void s2bSolveWheelXpbd(const SolveArgs& a, int t)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 lim = jc.lim[t];
	float4 motor = jc.motor[t];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;

	s2bPerpendicularXpbd(anchor, d0, motor, mA, iA, mB, iB, dcA, qA, dcB, qB);

	if (head.x & S2B_JOINT_ENABLE_LIMIT)
	{
		s2bAxialLimitXpbd(anchor, d0, motor, lim, mA, iA, mB, iB, dcA, qA, dcB, qB);
	}

	if ((mA != 0.0f) || (iA != 0.0f))
	{
		a.bodies.pose[ia] = make_float4(dcA.x, dcA.y, qA.s, qA.c);
	}
	if ((mB != 0.0f) || (iB != 0.0f))
	{
		a.bodies.pose[ib] = make_float4(dcB.x, dcB.y, qB.s, qB.c);
	}
}

// ---------------------------------------------------------------------------------------------------------------
// pulley joint (extension, DESIGN.md §3.18; definition: tests/pulley_oracle.c). Anchor A hangs on a rope from ground anchor
// A, anchor B on one from ground anchor B, and one equality row holds C = constant - lengthA - ratio lengthB at zero with
// J = (-uA, -ratio uB). Each rope is formed from its own body's pose alone, so the per-body gather can form its side's
// warm-start term without the other body. Row columns: lim = (constant, ratio), d0ax = (cA - groundA, cB - groundB) at the
// start poses, imp.x = the rope impulse.
// ---------------------------------------------------------------------------------------------------------------

// one rope at its body's pose: r = q anchor, and the length and unit direction u of (dc + r) + d0, the vector from the
// ground anchor to the body anchor (u is zero within 10 s2_linearSlop)
struct PulleyRope
{
	s2Vec2 r, u;
	float length;
};

__device__ __forceinline__ PulleyRope s2bPulleyRope(float ax, float ay, float d0x, float d0y, s2Vec2 dc, s2Rot q)
{
	PulleyRope p;
	p.r = s2RotateVector(q, V2(ax, ay));
	p.u = s2cPulleyRope(&p.length, s2Add(s2Add(dc, p.r), V2(d0x, d0y)));
	return p;
}

// the row's inverse effective mass, mA + iA ruA^2 + ratio^2 (mB + iB ruB^2)
__device__ __forceinline__ float s2bPulleyInvMass(const PulleyRope& A, const PulleyRope& B, float ratio, float mA, float iA, float mB,
												  float iB)
{
	float ruA = s2Cross(A.r, A.u), ruB = s2Cross(B.r, B.u);
	return mA + iA * ruA * ruA + ratio * ratio * (mB + iB * ruB * ruB);
}

// what warm starting adds to one side (v += m P, w += i L): P = -lambda uA on side A, -(ratio lambda) uB on side B,
// L = r x P. Shared by the constraint-by-constraint warm start and the per-body gather, so both add the same bits.
struct PulleyWarm
{
	s2Vec2 P;
	float L;
};

__device__ __forceinline__ PulleyWarm s2bPulleyWarmTerm(const SolveArgs& a, int t, bool sideB)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	float4 anchor = jc.anchor[t], d0 = jc.d0ax[t];
	float4 pose = a.bodies.pose[sideB ? head.z : head.y];
	float lambda = jc.imp[t].x;
	PulleyRope rope = sideB ? s2bPulleyRope(anchor.z, anchor.w, d0.z, d0.w, V2(pose.x, pose.y), R2(pose.z, pose.w))
							: s2bPulleyRope(anchor.x, anchor.y, d0.x, d0.y, V2(pose.x, pose.y), R2(pose.z, pose.w));
	PulleyWarm w;
	w.P = s2MulSV(sideB ? -(jc.lim[t].y * lambda) : -lambda, rope.u);
	w.L = s2Cross(rope.r, w.P);
	return w;
}

// the velocity row in each flavour: the distance joint's rigid row (soft bias in the biased pass, Baumgarte in every pass,
// none under the rigid flavour)
template <int KIND>
__device__ __forceinline__ void s2bSolvePulleyVelocity(const SolveArgs& a, int t, float h, float inv_h, bool useBias)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 lim = jc.lim[t];
	float4 imp = jc.imp[t];
	float4 velA = a.bodies.vel[ia], velB = a.bodies.vel[ib];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 vA = V2(velA.x, velA.y), vB = V2(velB.x, velB.y);
	float wA = velA.z, wB = velB.z;
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	float ratio = lim.y;
	PulleyRope A = s2bPulleyRope(anchor.x, anchor.y, d0.x, d0.y, V2(poseA.x, poseA.y), R2(poseA.z, poseA.w));
	PulleyRope B = s2bPulleyRope(anchor.z, anchor.w, d0.z, d0.w, V2(poseB.x, poseB.y), R2(poseB.z, poseB.w));
	float kInv = s2bPulleyInvMass(A, B, ratio, mA, iA, mB, iB);
	float k = kInv > 0.0f ? 1.0f / kInv : 0.0f;

	float3 s = s2bPrismaticBias<KIND>(lim.x - A.length - ratio * B.length, false, jc.coef[t], h, inv_h, useBias);
	s2Vec2 vpA = s2Add(vA, s2CrossSV(wA, A.r));
	s2Vec2 vpB = s2Add(vB, s2CrossSV(wB, B.r));
	float Cdot = -s2Dot(A.u, vpA) - ratio * s2Dot(B.u, vpB);
	float impulse = -k * s.y * (Cdot + s.x) - s.z * imp.x;
	imp.x += impulse;
	s2Vec2 PA = s2MulSV(-impulse, A.u);
	s2Vec2 PB = s2MulSV(-(ratio * impulse), B.u);
	vA = s2MulAdd(vA, mA, PA);
	wA += iA * s2Cross(A.r, PA);
	vB = s2MulAdd(vB, mB, PB);
	wB += iB * s2Cross(B.r, PB);

	jc.imp[t] = imp;
	s2bStoreJointVelocities(a, ia, ib, velA, velB, vA, wA, vB, wB, mA, iA, mB, iB);
}

// one position correction of the row on the given poses: impulse = -k C with C clamped (NGS) or -C / (1 / k) (XPBD at zero
// compliance, skipped when 1 / k is 0), applied as PA = -impulse uA, PB = -(ratio impulse) uB
template <bool XPBD>
__device__ __forceinline__ void s2bSolvePulleyPositionT(const SolveArgs& a, int t)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 lim = jc.lim[t];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	float ratio = lim.y;
	PulleyRope A = s2bPulleyRope(anchor.x, anchor.y, d0.x, d0.y, dcA, qA);
	PulleyRope B = s2bPulleyRope(anchor.z, anchor.w, d0.z, d0.w, dcB, qB);
	float kInv = s2bPulleyInvMass(A, B, ratio, mA, iA, mB, iB);
	float C = lim.x - A.length - ratio * B.length;
	if (XPBD && (kInv > 0.0f) == false)
	{
		return;
	}
	// NGS: C clamped as every NGS row here is (DESIGN.md §3.18; Box2D 2.4 does not clamp the pulley)
	float impulse = XPBD ? -C / kInv
						 : -(kInv > 0.0f ? 1.0f / kInv : 0.0f) * S2_CLAMP(C, -s2_maxLinearCorrection, s2_maxLinearCorrection);
	s2Vec2 PA = s2MulSV(-impulse, A.u);
	s2Vec2 PB = s2MulSV(-(ratio * impulse), B.u);
	dcA = s2MulAdd(dcA, mA, PA);
	qA = s2IntegrateRot(qA, iA * s2Cross(A.r, PA));
	dcB = s2MulAdd(dcB, mB, PB);
	qB = s2IntegrateRot(qB, iB * s2Cross(B.r, PB));
	if ((mA != 0.0f) || (iA != 0.0f))
	{
		a.bodies.pose[ia] = make_float4(dcA.x, dcA.y, qA.s, qA.c);
	}
	if ((mB != 0.0f) || (iB != 0.0f))
	{
		a.bodies.pose[ib] = make_float4(dcB.x, dcB.y, qB.s, qB.c);
	}
}

// ---------------------------------------------------------------------------------------------------------------
// gear joint (extension, DESIGN.md §3.19; definition: tests/gear_oracle.c). Couples two revolute or prismatic joints whose
// frame bodies are static: one equality row holds C = coordinate1 + ratio coordinate2 - constant at zero, each side's
// coordinate and Jacobian formed by s2cGearRevolute / s2cGearPrismatic from its own body's pose alone, so the per-body
// gather can form its side's warm-start term without the other body. Row columns: lim = (constant, ratio), d0ax = side
// 1's frame, pivot = side 2's frame (revolute: qC.s, qC.c, referenceAngle; prismatic: c - pC at the start poses, u),
// limp.xy = the revolute sides' unwound coordinates at the start poses, imp.x = the gear impulse.
// ---------------------------------------------------------------------------------------------------------------

// one side at the body's current pose: frame and theta as the row keeps them, (lx, ly) the side's local anchor
__device__ __forceinline__ s2cGearSide s2bGearSide(bool prismatic, float4 frame, float theta, float4 pose, float lx, float ly)
{
	s2Rot q = R2(pose.z, pose.w);
	return prismatic ? s2cGearPrismatic(V2(frame.x, frame.y), V2(frame.z, frame.w), V2(pose.x, pose.y), q, V2(lx, ly))
					 : s2cGearRevolute(frame.x, frame.y, frame.z, theta, q);
}

__device__ __forceinline__ s2cGearSide s2bGearSideOf(const SolveArgs& a, int t, bool sideB, float4 pose)
{
	const JointConstraintView& jc = a.jc;
	int flags = jc.head[t].x;
	float4 anchor = jc.anchor[t];
	float4 limp = jc.limp[t];
	return sideB ? s2bGearSide((flags & S2B_JOINT_GEAR_PRISMATIC2) != 0, jc.pivot[t], limp.y, pose, anchor.z, anchor.w)
				 : s2bGearSide((flags & S2B_JOINT_GEAR_PRISMATIC1) != 0, jc.d0ax[t], limp.x, pose, anchor.x, anchor.y);
}

// what warm starting adds to one side (v += m P, w += i L): P = s Jv, L = s Jw with s = lambda on side 1 and ratio lambda
// on side 2. Shared by the constraint-by-constraint warm start and the per-body gather, so both add the same bits.
struct GearWarm
{
	s2Vec2 P;
	float L;
};

__device__ __forceinline__ GearWarm s2bGearWarmTerm(const SolveArgs& a, int t, bool sideB)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	float4 pose = a.bodies.pose[sideB ? head.z : head.y];
	s2cGearSide side = s2bGearSideOf(a, t, sideB, pose);
	float lambda = jc.imp[t].x;
	float s = sideB ? jc.lim[t].y * lambda : lambda;
	GearWarm w;
	w.P = s2MulSV(s, side.Jv);
	w.L = s * side.Jw;
	return w;
}

// the constraint-by-constraint warm start: each side's term from s2bGearWarmTerm
__device__ __forceinline__ void s2bWarmStartGear(const SolveArgs& a, int t)
{
	int4 head = a.jc.head[t];
	int ia = head.y, ib = head.z;
	float4 mass = a.jc.mass[t];
	float4 velA = a.bodies.vel[ia], velB = a.bodies.vel[ib];
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	GearWarm wa = s2bGearWarmTerm(a, t, false);
	GearWarm wb = s2bGearWarmTerm(a, t, true);
	s2Vec2 vA = s2MulAdd(V2(velA.x, velA.y), mA, wa.P);
	float wA = velA.z + iA * wa.L;
	s2Vec2 vB = s2MulAdd(V2(velB.x, velB.y), mB, wb.P);
	float wB = velB.z + iB * wb.L;
	s2bStoreJointVelocities(a, ia, ib, velA, velB, vA, wA, vB, wB, mA, iA, mB, iB);
}

// the velocity row in each flavour: soft bias in the biased pass, Baumgarte in every pass, none under the rigid flavour
template <int KIND>
__device__ __forceinline__ void s2bSolveGearVelocity(const SolveArgs& a, int t, float h, float inv_h, bool useBias)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 mass = jc.mass[t];
	float4 lim = jc.lim[t];
	float4 imp = jc.imp[t];
	float4 velA = a.bodies.vel[ia], velB = a.bodies.vel[ib];
	s2cGearSide A = s2bGearSideOf(a, t, false, a.bodies.pose[ia]);
	s2cGearSide B = s2bGearSideOf(a, t, true, a.bodies.pose[ib]);
	s2Vec2 vA = V2(velA.x, velA.y), vB = V2(velB.x, velB.y);
	float wA = velA.z, wB = velB.z;
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	float ratio = lim.y;
	float kInv = s2cGearSideMass(A, mA, iA) + ratio * ratio * s2cGearSideMass(B, mB, iB);
	float k = kInv > 0.0f ? 1.0f / kInv : 0.0f;

	float3 s = s2bPrismaticBias<KIND>(A.coordinate + ratio * B.coordinate - lim.x, false, jc.coef[t], h, inv_h, useBias);
	float Cdot = (s2Dot(A.Jv, vA) + A.Jw * wA) + ratio * (s2Dot(B.Jv, vB) + B.Jw * wB);
	float impulse = -k * s.y * (Cdot + s.x) - s.z * imp.x;
	imp.x += impulse;
	float impulseB = ratio * impulse;
	vA = s2MulAdd(vA, mA, s2MulSV(impulse, A.Jv));
	wA += iA * (impulse * A.Jw);
	vB = s2MulAdd(vB, mB, s2MulSV(impulseB, B.Jv));
	wB += iB * (impulseB * B.Jw);

	jc.imp[t] = imp;
	s2bStoreJointVelocities(a, ia, ib, velA, velB, vA, wA, vB, wB, mA, iA, mB, iB);
}

// one position correction of the row on the given poses: impulse = -k C with C clamped in side 1's units (NGS: Box2D 2.4's
// gear correction) or -C / (1 / k) (XPBD at zero compliance, skipped when 1 / k is 0)
template <bool XPBD>
__device__ __forceinline__ void s2bSolveGearPositionT(const SolveArgs& a, int t)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 mass = jc.mass[t];
	float4 lim = jc.lim[t];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2cGearSide A = s2bGearSideOf(a, t, false, poseA);
	s2cGearSide B = s2bGearSideOf(a, t, true, poseB);
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	float ratio = lim.y;
	float kInv = s2cGearSideMass(A, mA, iA) + ratio * ratio * s2cGearSideMass(B, mB, iB);
	float C = A.coordinate + ratio * B.coordinate - lim.x;
	if (XPBD && (kInv > 0.0f) == false)
	{
		return;
	}
	float maxC = (head.x & S2B_JOINT_GEAR_PRISMATIC1) != 0 ? s2_maxLinearCorrection : s2_maxAngularCorrection;
	float impulse = XPBD ? -C / kInv : -(kInv > 0.0f ? 1.0f / kInv : 0.0f) * S2_CLAMP(C, -maxC, maxC);
	float impulseB = ratio * impulse;
	dcA = s2MulAdd(dcA, mA, s2MulSV(impulse, A.Jv));
	qA = s2IntegrateRot(qA, iA * (impulse * A.Jw));
	dcB = s2MulAdd(dcB, mB, s2MulSV(impulseB, B.Jv));
	qB = s2IntegrateRot(qB, iB * (impulseB * B.Jw));
	if ((mA != 0.0f) || (iA != 0.0f))
	{
		a.bodies.pose[ia] = make_float4(dcA.x, dcA.y, qA.s, qA.c);
	}
	if ((mB != 0.0f) || (iB != 0.0f))
	{
		a.bodies.pose[ib] = make_float4(dcB.x, dcB.y, qB.s, qB.c);
	}
}

// ---------------------------------------------------------------------------------------------------------------
// motor joint (extension, DESIGN.md §3.10; definition: tests/motor_oracle.c). Drives body B toward a pose relative to body
// A with capped effort: an angular row toward angle(B) - angle(A) = angularOffset, its accumulated impulse clamped to
// +/- h maxTorque, then a point row that takes B's origin to the linear offset in A's frame, its accumulated impulse scaled
// back to length h maxForce. Both rows are biased by correctionFactor / h times their position error in every velocity
// pass: the bias is the drive, and there is no rigid part. Row columns: anchor = (offset - localCenterA, -localCenterB),
// lim.x = angularOffset, motor = (maxTorque, 0, maxForce, correctionFactor), imp = (linear impulse, angular impulse).
// The warm start is the revolute's (P = linear impulse at rA / rB, axial = angular impulse).
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void s2bSolveMotorVelocity(const SolveArgs& a, int t, float h, float inv_h)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 motor = jc.motor[t];
	float angularOffset = jc.lim[t].x;
	float4 imp = jc.imp[t];
	float4 velA = a.bodies.vel[ia], velB = a.bodies.vel[ib];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 vA = V2(velA.x, velA.y), vB = V2(velB.x, velB.y);
	float wA = velA.z, wB = velB.z;
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	float biasScale = motor.w * inv_h;

	if (iA + iB != 0.0f)
	{
		float k = 1.0f / (iA + iB);
		float C = s2UnwindAngle(s2RelativeAngle(qB, qA) - angularOffset);
		float impulse = -k * (wB - wA + biasScale * C);
		float oldImpulse = imp.z;
		float maxImpulse = h * motor.x;
		imp.z = S2_CLAMP(oldImpulse + impulse, -maxImpulse, maxImpulse);
		impulse = imp.z - oldImpulse;
		wA -= iA * impulse;
		wB += iB * impulse;
	}

	{
		s2Vec2 rA = s2RotateVector(qA, V2(anchor.x, anchor.y));
		s2Vec2 rB = s2RotateVector(qB, V2(anchor.z, anchor.w));
		s2Vec2 Cdot = s2Sub(s2Add(vB, s2CrossSV(wB, rB)), s2Add(vA, s2CrossSV(wA, rA)));
		s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
		s2Vec2 C = s2Add(s2Add(s2Sub(dcB, dcA), s2Sub(rB, rA)), V2(d0.x, d0.y));
		s2Mat22 K;
		K.cx.x = mA + mB + rA.y * rA.y * iA + rB.y * rB.y * iB;
		K.cy.x = -rA.y * rA.x * iA - rB.y * rB.x * iB;
		K.cx.y = K.cy.x;
		K.cy.y = mA + mB + rA.x * rA.x * iA + rB.x * rB.x * iB;
		s2Vec2 b = s2Solve22(K, s2Add(Cdot, s2MulSV(biasScale, C)));
		s2Vec2 oldImpulse = V2(imp.x, imp.y);
		s2Vec2 total = s2ClampLength(s2Sub(oldImpulse, b), h * motor.z);
		s2Vec2 impulse = s2Sub(total, oldImpulse);
		imp.x = total.x;
		imp.y = total.y;
		vA = s2MulSub(vA, mA, impulse);
		wA -= iA * s2Cross(rA, impulse);
		vB = s2MulAdd(vB, mB, impulse);
		wB += iB * s2Cross(rB, impulse);
	}

	jc.imp[t] = imp;
	s2bStoreJointVelocities(a, ia, ib, velA, velB, vA, wA, vB, wB, mA, iA, mB, iB);
}

// XPBD, zero compliance: the angular row, then the revolute's XPBD row along the current separation. Each removes the
// fraction correctionFactor of its error, its correction capped at h^2 times the maximum torque or force.
__device__ __forceinline__ void s2bSolveMotorXpbd(const SolveArgs& a, int t)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 motor = jc.motor[t];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	float h = a.ctx.h;
	float cf = motor.w;

	if (iA + iB != 0.0f)
	{
		float C = s2UnwindAngle(s2RelativeAngle(qB, qA) - jc.lim[t].x);
		float maxP = h * h * motor.x;
		float p = S2_CLAMP(-cf * C / (iA + iB), -maxP, maxP);
		qA = s2IntegrateRot(qA, -iA * p);
		qB = s2IntegrateRot(qB, iB * p);
	}

	if (mA != 0.0f || mB != 0.0f)
	{
		s2Vec2 rA = s2RotateVector(qA, V2(anchor.x, anchor.y));
		s2Vec2 rB = s2RotateVector(qB, V2(anchor.z, anchor.w));
		s2Vec2 separation = s2Add(s2Add(s2Sub(dcB, dcA), s2Sub(rB, rA)), V2(d0.x, d0.y));
		float c = s2Length(separation);
		s2Vec2 n = V2(0.0f, 0.0f);
		if (c >= 0.001f * 1.1920929e-07f)
		{
			float invLength = 1.0f / c;
			n = V2(invLength * separation.x, invLength * separation.y);
		}
		float rnA = s2Cross(rA, n);
		float rnB = s2Cross(rB, n);
		float kA = mA + iA * rnA * rnA;
		float kB = mB + iB * rnB * rnB;
		float lambda = S2_MAX(-cf * c / (kA + kB), -(h * h * motor.z));
		s2Vec2 p = s2MulSV(lambda, n);
		dcA = s2MulSub(dcA, mA, p);
		qA = s2IntegrateRot(qA, -iA * s2Cross(rA, p));
		dcB = s2MulAdd(dcB, mB, p);
		qB = s2IntegrateRot(qB, iB * s2Cross(rB, p));
	}

	if ((mA != 0.0f) || (iA != 0.0f))
	{
		a.bodies.pose[ia] = make_float4(dcA.x, dcA.y, qA.s, qA.c);
	}
	if ((mB != 0.0f) || (iB != 0.0f))
	{
		a.bodies.pose[ib] = make_float4(dcB.x, dcB.y, qB.s, qB.c);
	}
}

// ---------------------------------------------------------------------------------------------------------------
// joint spring rows (DESIGN.md §3.14), run ahead of the joint's own rows by the dispatchers below
// ---------------------------------------------------------------------------------------------------------------

// the velocity row, the same in every velocity flavour (a force law, not an error correction):
// impulse = -k massScale (Cdot + bias C) - impulseScale lambda, k the axis's effective mass
__device__ __forceinline__ void s2bSolveSpringVelocity(const SolveArgs& a, int t)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 lim = jc.lim[t];
	float bias = jc.coef[t].w, massScale = lim.w, impulseScale = d0.w;
	float4 imp = jc.imp[t];
	float4 velA = a.bodies.vel[ia], velB = a.bodies.vel[ib];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 vA = V2(velA.x, velA.y), vB = V2(velB.x, velB.y);
	float wA = velA.z, wB = velB.z;
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_REVOLUTE)
	{
		// C = the weld's angular error (§3.8), k = 1 / (iA + iB)
		float k = 1.0f / (iA + iB);
		float C = s2UnwindAngle(s2RelativeAngle(qB, qA) - lim.x);
		float impulse = -k * massScale * (wB - wA + bias * C) - impulseScale * imp.w;
		imp.w += impulse;
		wA -= iA * impulse;
		wB += iB * impulse;
	}
	else
	{
		// prismatic and wheel (§3.17): C = the translation, k = the axial mass §3.9 forms in every solve; distance (§3.16):
		// C = length - rest length along the current line
		s2Vec2 axis;
		float a1, a2, C;
		if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_DISTANCE)
		{
			DistanceFrame f = s2bDistanceFrame(jc.anchor[t], d0, V2(poseA.x, poseA.y), qA, V2(poseB.x, poseB.y), qB);
			axis = f.axis;
			a1 = s2Cross(f.rA, axis);
			a2 = s2Cross(f.rB, axis);
			C = f.length - lim.x;
		}
		else
		{
			PrismaticFrame f = s2bPrismaticFrame(jc.anchor[t], d0, jc.motor[t], V2(poseA.x, poseA.y), qA, V2(poseB.x, poseB.y), qB);
			axis = f.axis;
			a1 = s2Cross(s2Add(f.d, f.rA), axis);
			a2 = s2Cross(f.rB, axis);
			C = s2Dot(axis, f.d);
		}
		float k = mA + mB + iA * a1 * a1 + iB * a2 * a2;
		float axialMass = k > 0.0f ? 1.0f / k : 0.0f;
		float Cdot = s2Dot(axis, s2Sub(vB, vA)) + a2 * wB - a1 * wA;
		float impulse = -axialMass * massScale * (Cdot + bias * C) - impulseScale * imp.w;
		imp.w += impulse;
		s2Vec2 P = s2MulSV(impulse, axis);
		vA = s2MulSub(vA, mA, P);
		wA -= iA * (impulse * a1);
		vB = s2MulAdd(vB, mB, P);
		wB += iB * (impulse * a2);
	}
	reinterpret_cast<float*>(jc.imp + t)[3] = imp.w;
	s2bStoreJointVelocities(a, ia, ib, velA, velB, vA, wA, vB, wB, mA, iA, mB, iB);
}

// XPBD with damping (Macklin et al. 2016), one solve per sub-step from a zero multiplier: w = the axis's generalized inverse
// mass, C and C0 the error now and at the sub-step's start pose (aux0: dp0, q0; a static body's own pose), omegaH = 2 pi
// hertz h. A rotation is integrated only where it can change (s2IntegrateRot renormalizes even by a zero angle).
__device__ __forceinline__ void s2bSolveSpringXpbd(const SolveArgs& a, int t)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 mass = jc.mass[t];
	float4 lim = jc.lim[t];
	float omegaH = jc.coef[t].w, zeta = lim.w;
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	float4 p0A = (head.x & S2B_JC_STATIC_A) != 0 ? poseA : a.bodies.aux0[ia];
	float4 p0B = (head.x & S2B_JC_STATIC_B) != 0 ? poseB : a.bodies.aux0[ib];
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	float w, C, C0, LA, LB;
	s2Vec2 axis = V2(0.0f, 0.0f);
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_REVOLUTE)
	{
		w = iA + iB;
		C = s2UnwindAngle(s2RelativeAngle(qB, qA) - lim.x);
		C0 = s2UnwindAngle(s2RelativeAngle(R2(p0B.z, p0B.w), R2(p0A.z, p0A.w)) - lim.x);
		LA = 1.0f;
		LB = 1.0f;
	}
	else
	{
		float4 anchor = jc.anchor[t], d0 = jc.d0ax[t];
		if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_DISTANCE)
		{
			DistanceFrame f0 = s2bDistanceFrame(anchor, d0, V2(p0A.x, p0A.y), R2(p0A.z, p0A.w), V2(p0B.x, p0B.y), R2(p0B.z, p0B.w));
			DistanceFrame f = s2bDistanceFrame(anchor, d0, dcA, qA, dcB, qB);
			axis = f.axis;
			LA = s2Cross(f.rA, f.axis);
			LB = s2Cross(f.rB, f.axis);
			C = f.length - lim.x;
			C0 = f0.length - lim.x;
		}
		else
		{
			float4 motor = jc.motor[t];
			PrismaticFrame f0 =
				s2bPrismaticFrame(anchor, d0, motor, V2(p0A.x, p0A.y), R2(p0A.z, p0A.w), V2(p0B.x, p0B.y), R2(p0B.z, p0B.w));
			PrismaticFrame f = s2bPrismaticFrame(anchor, d0, motor, dcA, qA, dcB, qB);
			axis = f.axis;
			LA = s2Cross(s2Add(f.d, f.rA), f.axis);
			LB = s2Cross(f.rB, f.axis);
			C = s2Dot(f.axis, f.d);
			C0 = s2Dot(f0.axis, f0.d);
		}
		w = mA + mB + iA * LA * LA + iB * LB * LB;
		if ((w > 0.0f) == false)
		{
			return;
		}
	}
	float alphaTilde = w / (omegaH * omegaH);
	float gamma = 2.0f * zeta / omegaH;
	float p = -(C + gamma * (C - C0)) / ((1.0f + gamma) * w + alphaTilde);
	if (S2B_JOINT_TYPE(head.x) != S2B_JOINT_REVOLUTE)
	{
		s2Vec2 P = s2MulSV(p, axis);
		dcA = s2MulSub(dcA, mA, P);
		dcB = s2MulAdd(dcB, mB, P);
		LA = p * LA;
		LB = p * LB;
	}
	else
	{
		LA = p;
		LB = p;
	}
	if (iA != 0.0f)
	{
		qA = s2IntegrateRot(qA, -iA * LA);
	}
	if (iB != 0.0f)
	{
		qB = s2IntegrateRot(qB, iB * LB);
	}
	if ((mA != 0.0f) || (iA != 0.0f))
	{
		a.bodies.pose[ia] = make_float4(dcA.x, dcA.y, qA.s, qA.c);
	}
	if ((mB != 0.0f) || (iB != 0.0f))
	{
		a.bodies.pose[ib] = make_float4(dcB.x, dcB.y, qB.s, qB.c);
	}
}

// ---------------------------------------------------------------------------------------------------------------
// warm start: s2WarmStartRevolute (reference src/revolute_joint.c:107-150), s2WarmStartMouse (mouse_joint.c:85-107)
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void s2bWarmStartJoint(const SolveArgs& a, int t)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 imp = jc.imp[t];

	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_MOUSE)
	{
		float4 velB = a.bodies.vel[ib];
		float4 poseB = a.bodies.pose[ib];
		s2Vec2 rB = s2RotateVector(R2(poseB.z, poseB.w), V2(anchor.z, anchor.w));
		s2Vec2 vB = V2(velB.x, velB.y);
		float wB = velB.z;
		s2Vec2 impulse = V2(imp.x, imp.y);
		vB = s2MulAdd(vB, mass.z, impulse);
		wB += mass.w * (s2Cross(rB, impulse) + imp.z);
		if ((mass.z != 0.0f) | (mass.w != 0.0f))
		{
			a.bodies.vel[ib] = make_float4(vB.x, vB.y, wB, velB.w);
		}
		return;
	}

	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_PRISMATIC || S2B_JOINT_TYPE(head.x) == S2B_JOINT_DISTANCE ||
		S2B_JOINT_TYPE(head.x) == S2B_JOINT_WHEEL)
	{
		float4 velA = a.bodies.vel[ia], velB = a.bodies.vel[ib];
		float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
		PrismaticWarm pw = s2bPrismaticWarmTerms(a, t);
		s2Vec2 vA = s2MulSub(V2(velA.x, velA.y), mA, pw.P);
		float wA = velA.z - iA * pw.LA;
		s2Vec2 vB = s2MulAdd(V2(velB.x, velB.y), mB, pw.P);
		float wB = velB.z + iB * pw.LB;
		s2bStoreJointVelocities(a, ia, ib, velA, velB, vA, wA, vB, wB, mA, iA, mB, iB);
		return;
	}

	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_GEAR)
	{
		s2bWarmStartGear(a, t);
		return;
	}
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_PULLEY)
	{
		float4 velA = a.bodies.vel[ia], velB = a.bodies.vel[ib];
		float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
		PulleyWarm wa = s2bPulleyWarmTerm(a, t, false);
		PulleyWarm wb = s2bPulleyWarmTerm(a, t, true);
		s2Vec2 vA = s2MulAdd(V2(velA.x, velA.y), mA, wa.P);
		float wA = velA.z + iA * wa.L;
		s2Vec2 vB = s2MulAdd(V2(velB.x, velB.y), mB, wb.P);
		float wB = velB.z + iB * wb.L;
		s2bStoreJointVelocities(a, ia, ib, velA, velB, vA, wA, vB, wB, mA, iA, mB, iB);
		return;
	}

	float4 limp = jc.limp[t];
	float4 velA = a.bodies.vel[ia], velB = a.bodies.vel[ib];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 vA = V2(velA.x, velA.y), vB = V2(velB.x, velB.y);
	float wA = velA.z, wB = velB.z;
	s2Vec2 rA = s2RotateVector(R2(poseA.z, poseA.w), V2(anchor.x, anchor.y));
	s2Vec2 rB = s2RotateVector(R2(poseB.z, poseB.w), V2(anchor.z, anchor.w));
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;

	// axial = spring + motor + lower - upper (DESIGN.md §3.14); a row without a spring adds no spring term
	float axialImpulse = ((head.x & S2B_JOINT_ENABLE_SPRING) != 0 ? imp.w + imp.z : imp.z) + limp.x - limp.y;
	s2Vec2 P = V2(imp.x, imp.y);

	vA = s2MulSub(vA, mA, P);
	wA -= iA * (s2Cross(rA, P) + axialImpulse);
	vB = s2MulAdd(vB, mB, P);
	wB += iB * (s2Cross(rB, P) + axialImpulse);

	s2bStoreJointVelocities(a, ia, ib, velA, velB, vA, wA, vB, wB, mA, iA, mB, iB);
}

// ---------------------------------------------------------------------------------------------------------------
// s2SolveMouse (reference src/mouse_joint.c:109-167): ad-hoc angular damper + soft point constraint on body B.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void s2bSolveMouse(const SolveArgs& a, int t)
{
	const JointConstraintView& jc = a.jc;
	int ib = jc.head[t].z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 coef = jc.coef[t];
	float4 pv = jc.pivot[t];
	float4 imp = jc.imp[t];
	float4 velB = a.bodies.vel[ib];
	float4 poseB = a.bodies.pose[ib];

	s2Vec2 vB = V2(velB.x, velB.y);
	float wB = velB.z;
	float mB = mass.z, iB = mass.w;

	{
		float h = a.ctx.h;
		float zeta = 0.1f;
		float omega = 2.0f * s2_pi * 0.5f;
		float c = h * omega * (2.0f * zeta + h * omega);
		float impulseScale = 1.0f / (1.0f + c);
		float massScale = c * impulseScale;
		float impulse = -massScale * d0.w * wB - impulseScale * imp.z;
		imp.z += impulse;
		wB += iB * impulse;
	}

	{
		s2Vec2 rB = s2RotateVector(R2(poseB.z, poseB.w), V2(anchor.z, anchor.w));
		s2Vec2 Cdot = s2Add(vB, s2CrossSV(wB, rB));
		s2Vec2 dcB = V2(poseB.x, poseB.y);
		s2Vec2 separation = s2Add(s2Add(dcB, rB), V2(d0.x, d0.y));
		s2Vec2 bias = s2MulSV(coef.x, separation);
		float massScale = coef.y;
		float impulseScale = coef.z;
		s2Mat22 pivot;
		pivot.cx = V2(pv.x, pv.y);
		pivot.cy = V2(pv.z, pv.w);
		s2Vec2 b = s2MulMV(pivot, s2Add(Cdot, bias));
		s2Vec2 impulse;
		impulse.x = -massScale * b.x - impulseScale * imp.x;
		impulse.y = -massScale * b.y - impulseScale * imp.y;
		imp.x += impulse.x;
		imp.y += impulse.y;
		vB = s2MulAdd(vB, mB, impulse);
		wB += iB * s2Cross(rB, impulse);
	}

	jc.imp[t] = imp;
	if ((mB != 0.0f) | (iB != 0.0f))
	{
		a.bodies.vel[ib] = make_float4(vB.x, vB.y, wB, velB.w);
	}
}

// ---------------------------------------------------------------------------------------------------------------
// s2SolveRevolute_Soft (reference src/revolute_joint.c:508-657) and s2SolveRevolute_Baumgarte (:660-790):
// motor, lower / upper limit, point-to-point with a fresh 2x2 effective mass (S2_FRESH_PIVOT_MASS == 1).
// ---------------------------------------------------------------------------------------------------------------
enum JointSolveKind
{
	JSOLVE_SOFT = 0,
	JSOLVE_BAUMGARTE = 1,
};

// MOTOR_ROWS: the soft flavour also solves motor joints (see below); the Baumgarte flavour never does.
template <int KIND, bool MOTOR_ROWS>
__device__ __forceinline__ void s2bSolveRevoluteVelocity(const SolveArgs& a, int t, float h, float inv_h, bool useBias)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 lim = jc.lim[t];
	float4 motor = jc.motor[t];
	float4 coef = jc.coef[t];
	float4 imp = jc.imp[t];
	float4 limp = jc.limp[t];

	float4 velA = a.bodies.vel[ia], velB = a.bodies.vel[ib];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 vA = V2(velA.x, velA.y), vB = V2(velB.x, velB.y);
	float wA = velA.z, wB = velB.z;
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	float axialMass = d0.z;
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);

	bool fixedRotation = (iA + iB == 0.0f);
	bool enableLimit = (head.x & S2B_JOINT_ENABLE_LIMIT) != 0;
	bool enableMotor = (head.x & S2B_JOINT_ENABLE_MOTOR) != 0;

	// A weld has no motor: its one bilateral angular row (DESIGN.md §3.8) takes the motor row's place and column (imp.z).
	// The rotations do not change in a velocity pass. The soft flavour evaluates the angle once for the weld and the
	// limits; the Baumgarte flavour evaluates it where each row needs it. Both give the same bits; each choice is the
	// one that keeps its kernels' stack frame and spills at what they are without the weld (DESIGN.md §3.8).
	bool weld = S2B_JOINT_TYPE(head.x) == S2B_JOINT_WELD;
	// With MOTOR_ROWS the soft flavour also solves the motor joint (DESIGN.md §3.10), whose two rows are this function's
	// motor row and point row with a drive bias: its angular row is the motor row at the speed -cf / h * C, its point row is
	// biased by cf / h times the separation in every pass and its accumulated impulse is capped in length. The same bits as
	// s2bSolveMotorVelocity; sharing the branches keeps TGS_Soft's stack frame and spills where they are without the motor
	// joint.
	bool motorJoint = KIND == JSOLVE_SOFT && MOTOR_ROWS && S2B_JOINT_TYPE(head.x) == S2B_JOINT_MOTOR;
	float jointAngle = 0.0f;
	if (KIND == JSOLVE_SOFT && (enableLimit || weld || motorJoint) && fixedRotation == false)
	{
		jointAngle = s2RelativeAngle(qB, qA) - lim.x;
	}
	if ((enableMotor || weld || motorJoint) && fixedRotation == false)
	{
		float impulse;
		if (weld)
		{
			float C = s2UnwindAngle(KIND == JSOLVE_SOFT ? jointAngle : s2RelativeAngle(qB, qA) - lim.x);
			float bias = 0.0f;
			float massScale = 1.0f;
			float impulseScale = 0.0f;
			if (KIND == JSOLVE_SOFT)
			{
				if (head.x & S2B_JC_SOFT_ANGULAR)
				{
					// a soft weld's angle spring (DESIGN.md §3.15): its own coefficients, in every pass
					bias = motor.x * C;
					massScale = motor.y;
					impulseScale = motor.z;
				}
				else if (useBias)
				{
					bias = coef.x * C;
					massScale = coef.y;
					impulseScale = coef.z;
				}
			}
			else
			{
				// as this flavour's point row, the Baumgarte bias is applied in every pass
				bias = s2_baumgarte * inv_h * C;
			}
			float Cdot = wB - wA;
			impulse = KIND == JSOLVE_SOFT ? -axialMass * massScale * (Cdot + bias) - impulseScale * imp.z
										  : -axialMass * (Cdot + bias);
			imp.z += impulse;
		}
		else
		{
			// a motor joint's speed -(cf / h * C) makes Cdot = wB - wA + cf / h * C exactly
			float speed = motorJoint ? -((motor.w * inv_h) * s2UnwindAngle(jointAngle)) : motor.y;
			float Cdot = wB - wA - speed;
			impulse = -axialMass * Cdot;
			float oldImpulse = imp.z;
			float maxImpulse = h * motor.x;
			imp.z = S2_CLAMP(imp.z + impulse, -maxImpulse, maxImpulse);
			impulse = imp.z - oldImpulse;
		}
		wA -= iA * impulse;
		wB += iB * impulse;
	}

	if (enableLimit && fixedRotation == false)
	{
		if (KIND != JSOLVE_SOFT)
		{
			jointAngle = s2RelativeAngle(qB, qA) - lim.x;
		}

		// lower limit
		{
			float C = jointAngle - lim.y;
			float bias = 0.0f;
			float massScale = 1.0f;
			float impulseScale = 0.0f;
			if (C > 0.0f)
			{
				bias = C * inv_h;
			}
			else if (useBias)
			{
				if (KIND == JSOLVE_SOFT)
				{
					bias = coef.x * C;
					massScale = coef.y;
					impulseScale = coef.z;
				}
				else
				{
					bias = s2_baumgarte * inv_h * C;
				}
			}
			float Cdot = wB - wA;
			float impulse = KIND == JSOLVE_SOFT ? -axialMass * massScale * (Cdot + bias) - impulseScale * limp.x
												: -axialMass * (Cdot + bias);
			float oldImpulse = limp.x;
			limp.x = S2_MAX(limp.x + impulse, 0.0f);
			impulse = limp.x - oldImpulse;
			wA -= iA * impulse;
			wB += iB * impulse;
		}

		// upper limit (signs flipped so C stays positive when satisfied)
		{
			float C = lim.z - jointAngle;
			float bias = 0.0f;
			float massScale = 1.0f;
			float impulseScale = 0.0f;
			if (C > 0.0f)
			{
				bias = C * inv_h;
			}
			else if (useBias)
			{
				if (KIND == JSOLVE_SOFT)
				{
					bias = coef.x * C;
					massScale = coef.y;
					impulseScale = coef.z;
				}
				else
				{
					bias = s2_baumgarte * inv_h * C;
				}
			}
			float Cdot = wA - wB;
			// the soft flavour relaxes with the *lower* impulse here: a reference quirk kept for parity
			// (reference src/revolute_joint.c:595, SURVEY §8a N2)
			float impulse = KIND == JSOLVE_SOFT ? -axialMass * massScale * (Cdot + bias) - impulseScale * limp.x
												: -axialMass * (Cdot + bias);
			float oldImpulse = limp.y;
			limp.y = S2_MAX(limp.y + impulse, 0.0f);
			impulse = limp.y - oldImpulse;
			wA += iA * impulse;
			wB -= iB * impulse;
		}
	}

	// point-to-point
	{
		s2Vec2 rA = s2RotateVector(qA, V2(anchor.x, anchor.y));
		s2Vec2 rB = s2RotateVector(qB, V2(anchor.z, anchor.w));
		s2Vec2 Cdot = s2Sub(s2Add(vB, s2CrossSV(wB, rB)), s2Add(vA, s2CrossSV(wA, rA)));

		s2Vec2 bias = V2(0.0f, 0.0f);
		float massScale = 1.0f;
		float impulseScale = 0.0f;
		if (KIND == JSOLVE_SOFT)
		{
			// a soft weld's anchor spring (DESIGN.md §3.15) takes its own coefficients in every pass
			bool softLinear = (head.x & S2B_JC_SOFT_LINEAR) != 0;
			if (useBias || motorJoint || softLinear)
			{
				s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
				s2Vec2 separation = s2Add(s2Add(s2Sub(dcB, dcA), s2Sub(rB, rA)), V2(d0.x, d0.y));
				bias = s2MulSV(softLinear ? lim.y : (motorJoint ? motor.w * inv_h : coef.x), separation);
				massScale = softLinear ? lim.z : (motorJoint ? 1.0f : coef.y);
				impulseScale = softLinear ? lim.w : (motorJoint ? 0.0f : coef.z);
			}
		}
		else
		{
			// the Baumgarte flavour always applies its bias (reference src/revolute_joint.c:757-758)
			s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
			s2Vec2 separation = s2Add(s2Add(s2Sub(dcB, dcA), s2Sub(rB, rA)), V2(d0.x, d0.y));
			bias = s2MulSV(s2_baumgarte * inv_h, separation);
		}

		s2Mat22 K;
		K.cx.x = mA + mB + rA.y * rA.y * iA + rB.y * rB.y * iB;
		K.cy.x = -rA.y * rA.x * iA - rB.y * rB.x * iB;
		K.cx.y = K.cy.x;
		K.cy.y = mA + mB + rA.x * rA.x * iA + rB.x * rB.x * iB;
		s2Vec2 b = s2Solve22(K, s2Add(Cdot, bias));

		s2Vec2 impulse;
		if (KIND == JSOLVE_SOFT)
		{
			impulse.x = -massScale * b.x - impulseScale * imp.x;
			impulse.y = -massScale * b.y - impulseScale * imp.y;
		}
		else
		{
			impulse.x = -b.x;
			impulse.y = -b.y;
		}
		s2Vec2 oldImpulse = V2(imp.x, imp.y);
		imp.x += impulse.x;
		imp.y += impulse.y;
		if (motorJoint)
		{
			// the total is formed as oldImpulse - b, as s2bSolveMotorVelocity forms it: oldImpulse + (-1 * b - 0 * imp) has
			// the same value but can differ in the sign of a zero
			s2Vec2 total = s2ClampLength(s2Sub(oldImpulse, b), h * motor.z);
			impulse = s2Sub(total, oldImpulse);
			imp.x = total.x;
			imp.y = total.y;
		}

		vA = s2MulSub(vA, mA, impulse);
		wA -= iA * s2Cross(rA, impulse);
		vB = s2MulAdd(vB, mB, impulse);
		wB += iB * s2Cross(rB, impulse);
	}

	jc.imp[t] = imp;
	jc.limp[t] = limp;
	s2bStoreJointVelocities(a, ia, ib, velA, velB, vA, wA, vB, wB, mA, iA, mB, iB);
}

// ---------------------------------------------------------------------------------------------------------------
// soft weld rows (DESIGN.md §3.15): a weld row with S2B_JC_SOFT_ANGULAR or S2B_JC_SOFT_LINEAR. The angular row, then the
// point row, as the weld's; a soft part is the force law impulse = -k massScale (Cdot + bias C) - impulseScale lambda in
// every velocity pass, a rigid part is the flavour's weld row, op for op. k is the weld's axial mass for the angular row
// and, for the point row, the 2x2 effective mass the flavour's point row uses: fresh in the Baumgarte flavour, the
// prepare-time pivot in the rigid flavour. The soft flavour needs no function of its own: its weld rows already have the
// force law's form, and s2bSolveRevoluteVelocity gives them the soft parts' coefficients. The other two are kept apart
// from s2bSolveRevoluteVelocity / s2bSolveRevoluteRigid, whose weld rows have another form, so that those rows' code
// stays as it is.
// ---------------------------------------------------------------------------------------------------------------
enum SoftWeldForm
{
	SWELD_BAUMGARTE = 1, // PGS, TGS_Sticky
	SWELD_RIGID = 2,	 // PGS_NGS, PGS_NGS_Block, TGS_NGS
};

template <int FORM> __device__ __forceinline__ void s2bSolveSoftWeldVelocity(const SolveArgs& a, int t, float inv_h)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 lim = jc.lim[t];
	float4 imp = jc.imp[t];
	float4 velA = a.bodies.vel[ia], velB = a.bodies.vel[ib];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 vA = V2(velA.x, velA.y), vB = V2(velB.x, velB.y);
	float wA = velA.z, wB = velB.z;
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	float axialMass = d0.z;
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	bool softLinear = (head.x & S2B_JC_SOFT_LINEAR) != 0;

	// angular row
	if (iA + iB != 0.0f)
	{
		float impulse;
		if (head.x & S2B_JC_SOFT_ANGULAR)
		{
			float4 sc = jc.motor[t]; // bias, mass scale, impulse scale
			float C = s2UnwindAngle(s2RelativeAngle(qB, qA) - lim.x);
			float Cdot = wB - wA;
			impulse = -axialMass * sc.y * (Cdot + sc.x * C) - sc.z * imp.z;
		}
		else if (FORM == SWELD_BAUMGARTE)
		{
			float C = s2UnwindAngle(s2RelativeAngle(qB, qA) - lim.x);
			float bias = s2_baumgarte * inv_h * C;
			float Cdot = wB - wA;
			impulse = -axialMass * (Cdot + bias);
		}
		else
		{
			impulse = -axialMass * (wB - wA);
		}
		imp.z += impulse;
		wA -= iA * impulse;
		wB += iB * impulse;
	}

	// point row
	{
		s2Vec2 rA = s2RotateVector(qA, V2(anchor.x, anchor.y));
		s2Vec2 rB = s2RotateVector(qB, V2(anchor.z, anchor.w));
		s2Vec2 Cdot = s2Sub(s2Add(vB, s2CrossSV(wB, rB)), s2Add(vA, s2CrossSV(wA, rA)));
		s2Vec2 bias = V2(0.0f, 0.0f);
		float massScale = 1.0f;
		float impulseScale = 0.0f;
		if (softLinear || FORM == SWELD_BAUMGARTE)
		{
			s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
			s2Vec2 separation = s2Add(s2Add(s2Sub(dcB, dcA), s2Sub(rB, rA)), V2(d0.x, d0.y));
			if (softLinear)
			{
				bias = s2MulSV(lim.y, separation);
				massScale = lim.z;
				impulseScale = lim.w;
			}
			else
			{
				bias = s2MulSV(s2_baumgarte * inv_h, separation);
			}
		}

		s2Vec2 b;
		if (FORM == SWELD_RIGID)
		{
			float4 pv = jc.pivot[t];
			s2Mat22 pivot;
			pivot.cx = V2(pv.x, pv.y);
			pivot.cy = V2(pv.z, pv.w);
			b = s2MulMV(pivot, softLinear ? s2Add(Cdot, bias) : s2Neg(Cdot));
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
		if (softLinear)
		{
			impulse.x = -massScale * b.x - impulseScale * imp.x;
			impulse.y = -massScale * b.y - impulseScale * imp.y;
		}
		else if (FORM == SWELD_BAUMGARTE)
		{
			impulse.x = -b.x;
			impulse.y = -b.y;
		}
		else
		{
			impulse = b; // pivot (-Cdot)
		}
		imp.x += impulse.x;
		imp.y += impulse.y;
		vA = s2MulSub(vA, mA, impulse);
		wA -= iA * s2Cross(rA, impulse);
		vB = s2MulAdd(vB, mB, impulse);
		wB += iB * s2Cross(rB, impulse);
	}

	jc.imp[t] = imp;
	s2bStoreJointVelocities(a, ia, ib, velA, velB, vA, wA, vB, wB, mA, iA, mB, iB);
}

// The NGS position pass: a soft part has no position row (as the mouse joint and the springs); a rigid part is the weld's
// correction (s2bSolveJointPosition), the angle first.
__device__ __forceinline__ void s2bSolveSoftWeldPosition(const SolveArgs& a, int t)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	if ((head.x & S2B_JC_SOFT_WELD) == S2B_JC_SOFT_WELD)
	{
		return;
	}
	int ia = head.y, ib = head.z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;

	// at least one part is soft: a rigid angle (then the anchor is soft) or a rigid anchor (then the angle is soft)
	if ((head.x & S2B_JC_SOFT_ANGULAR) == 0)
	{
		if (iA + iB != 0.0f)
		{
			float C = s2UnwindAngle(s2RelativeAngle(qB, qA) - jc.lim[t].x);
			float p = -d0.z * S2_CLAMP(C, -s2_maxAngularCorrection, s2_maxAngularCorrection);
			qA = s2IntegrateRot(qA, -iA * p);
			qB = s2IntegrateRot(qB, iB * p);
		}
	}
	else
	{
		s2Vec2 rA = s2RotateVector(qA, V2(anchor.x, anchor.y));
		s2Vec2 rB = s2RotateVector(qB, V2(anchor.z, anchor.w));
		s2Vec2 C = s2Add(s2Add(s2Sub(dcB, dcA), s2Sub(rB, rA)), V2(d0.x, d0.y));
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

	if ((mA != 0.0f) || (iA != 0.0f))
	{
		a.bodies.pose[ia] = make_float4(dcA.x, dcA.y, qA.s, qA.c);
	}
	if ((mB != 0.0f) || (iB != 0.0f))
	{
		a.bodies.pose[ib] = make_float4(dcB.x, dcB.y, qB.s, qB.c);
	}
}

// XPBD with damping (Macklin et al. 2016), as the springs' (§3.14): w the row's generalized inverse mass, C and C0 the error
// now and at the sub-step's start pose, omegaH = 2 pi hertz h
__device__ __forceinline__ float s2bSoftWeldXpbdImpulse(float w, float C, float C0, float omegaH, float zeta)
{
	float alphaTilde = w / (omegaH * omegaH);
	float gamma = 2.0f * zeta / omegaH;
	return -(C + gamma * (C - C0)) / ((1.0f + gamma) * w + alphaTilde);
}

// XPBD: the weld's rows (s2bSolveJointXpbd), a soft part compliant with damping. The start pose is aux0 (dp0, q0), or a
// static body's own pose. The linear row acts along n = separation / |separation| with C = |separation| and C0 = n . the
// separation at the start pose.
__device__ __forceinline__ void s2bSolveSoftWeldXpbd(const SolveArgs& a, int t)
{
	const float compliance = 0.0f;
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 lim = jc.lim[t];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	float4 p0A = (head.x & S2B_JC_STATIC_A) != 0 ? poseA : a.bodies.aux0[ia];
	float4 p0B = (head.x & S2B_JC_STATIC_B) != 0 ? poseB : a.bodies.aux0[ib];
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	s2Rot q0A = R2(p0A.z, p0A.w), q0B = R2(p0B.z, p0B.w);
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	if (iA + iB != 0.0f)
	{
		float C = s2UnwindAngle(s2RelativeAngle(qB, qA) - lim.x);
		float p;
		if (head.x & S2B_JC_SOFT_ANGULAR)
		{
			float4 sc = jc.motor[t]; // 2 pi hertz h, damping ratio
			float C0 = s2UnwindAngle(s2RelativeAngle(q0B, q0A) - lim.x);
			p = s2bSoftWeldXpbdImpulse(iA + iB, C, C0, sc.x, sc.y);
		}
		else
		{
			p = -C / (iA + iB);
		}
		qA = s2IntegrateRot(qA, -iA * p);
		qB = s2IntegrateRot(qB, iB * p);
	}
	s2Vec2 rA = s2RotateVector(qA, V2(anchor.x, anchor.y));
	s2Vec2 rB = s2RotateVector(qB, V2(anchor.z, anchor.w));
	s2Vec2 separation = s2Add(s2Add(s2Sub(dcB, dcA), s2Sub(rB, rA)), V2(d0.x, d0.y));
	float c = s2Length(separation);
	s2Vec2 n = V2(0.0f, 0.0f);
	if (c >= 0.001f * 1.1920929e-07f)
	{
		float invLength = 1.0f / c;
		n = V2(invLength * separation.x, invLength * separation.y);
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
	if (head.x & S2B_JC_SOFT_LINEAR)
	{
		s2Vec2 rA0 = s2RotateVector(q0A, V2(anchor.x, anchor.y));
		s2Vec2 rB0 = s2RotateVector(q0B, V2(anchor.z, anchor.w));
		s2Vec2 separation0 = s2Add(s2Add(s2Sub(V2(p0B.x, p0B.y), V2(p0A.x, p0A.y)), s2Sub(rB0, rA0)), V2(d0.x, d0.y));
		lambda = s2bSoftWeldXpbdImpulse(kA + kB, c, s2Dot(n, separation0), lim.y, lim.z);
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
	if ((mA != 0.0f) || (iA != 0.0f))
	{
		a.bodies.pose[ia] = make_float4(dcA.x, dcA.y, qA.s, qA.c);
	}
	if ((mB != 0.0f) || (iB != 0.0f))
	{
		a.bodies.pose[ib] = make_float4(dcB.x, dcB.y, qB.s, qB.c);
	}
}

// s2SolveJoint_Soft dispatch (reference src/joint.c:385-405): the mouse joint is solved only in the biased pass. A motor
// joint is solved in every pass, by the revolute's soft rows when SHARED_MOTOR (the persistent kernels), else by
// s2bSolveMotorVelocity (the launch-by-launch kernel, whose every-op build spills less that way). Both give the same bits.
template <bool SHARED_MOTOR>
__device__ __forceinline__ void s2bSolveJointSoft(const SolveArgs& a, int t, float h, float inv_h, bool useBias)
{
	int flags = a.jc.head[t].x;
	if (flags & S2B_JOINT_ENABLE_SPRING)
	{
		s2bSolveSpringVelocity(a, t);
	}
	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_MOUSE)
	{
		if (useBias)
		{
			s2bSolveMouse(a, t);
		}
		return;
	}
	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_PRISMATIC)
	{
		s2bSolvePrismaticVelocity<PSOLVE_SOFT>(a, t, h, inv_h, useBias);
		return;
	}
	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_DISTANCE)
	{
		s2bSolveDistanceVelocity<PSOLVE_SOFT>(a, t, h, inv_h, useBias);
		return;
	}
	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_WHEEL)
	{
		s2bSolveWheelVelocity<PSOLVE_SOFT>(a, t, h, inv_h, useBias);
		return;
	}
	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_GEAR)
	{
		s2bSolveGearVelocity<PSOLVE_SOFT>(a, t, h, inv_h, useBias);
		return;
	}
	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_PULLEY)
	{
		s2bSolvePulleyVelocity<PSOLVE_SOFT>(a, t, h, inv_h, useBias);
		return;
	}
	if (SHARED_MOTOR == false && S2B_JOINT_TYPE(flags) == S2B_JOINT_MOTOR)
	{
		s2bSolveMotorVelocity(a, t, h, inv_h);
		return;
	}
	// a soft weld's rows are the revolute soft rows with its own coefficients (DESIGN.md §3.15)
	s2bSolveRevoluteVelocity<JSOLVE_SOFT, SHARED_MOTOR>(a, t, h, inv_h, useBias);
}

// s2SolveJoint_Baumgarte dispatch (reference src/joint.c:409-425)
__device__ __forceinline__ void s2bSolveJointBaumgarte(const SolveArgs& a, int t, float h, float inv_h, bool useBias)
{
	int flags = a.jc.head[t].x;
	if (flags & S2B_JOINT_ENABLE_SPRING)
	{
		s2bSolveSpringVelocity(a, t);
	}
	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_MOUSE)
	{
		s2bSolveMouse(a, t);
		return;
	}
	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_PRISMATIC)
	{
		s2bSolvePrismaticVelocity<PSOLVE_BAUMGARTE>(a, t, h, inv_h, useBias);
		return;
	}
	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_DISTANCE)
	{
		s2bSolveDistanceVelocity<PSOLVE_BAUMGARTE>(a, t, h, inv_h, useBias);
		return;
	}
	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_WHEEL)
	{
		s2bSolveWheelVelocity<PSOLVE_BAUMGARTE>(a, t, h, inv_h, useBias);
		return;
	}
	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_GEAR)
	{
		s2bSolveGearVelocity<PSOLVE_BAUMGARTE>(a, t, h, inv_h, useBias);
		return;
	}
	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_PULLEY)
	{
		s2bSolvePulleyVelocity<PSOLVE_BAUMGARTE>(a, t, h, inv_h, useBias);
		return;
	}
	if (S2B_JOINT_TYPE(flags) == S2B_JOINT_MOTOR)
	{
		s2bSolveMotorVelocity(a, t, h, inv_h);
		return;
	}
	if (flags & S2B_JC_SOFT_WELD)
	{
		s2bSolveSoftWeldVelocity<SWELD_BAUMGARTE>(a, t, inv_h);
		return;
	}
	s2bSolveRevoluteVelocity<JSOLVE_BAUMGARTE, false>(a, t, h, inv_h, useBias);
}

// ---------------------------------------------------------------------------------------------------------------
// s2SolveRevolute (reference src/revolute_joint.c:152-303): rigid velocity solve used by PGS_NGS and TGS_NGS — motor,
// limits with a speculative max(C, 0)/h term, point-to-point with the pivot mass computed at prepare time.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void s2bSolveRevoluteRigid(const SolveArgs& a, int t, float h)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	int ia = head.y, ib = head.z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 lim = jc.lim[t];
	float4 motor = jc.motor[t];
	float4 pv = jc.pivot[t];
	float4 imp = jc.imp[t];
	float4 limp = jc.limp[t];
	float4 velA = a.bodies.vel[ia], velB = a.bodies.vel[ib];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 vA = V2(velA.x, velA.y), vB = V2(velB.x, velB.y);
	float wA = velA.z, wB = velB.z;
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	float axialMass = d0.z;
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	bool fixedRotation = (iA + iB == 0.0f);

	if ((head.x & S2B_JOINT_ENABLE_MOTOR) && fixedRotation == false)
	{
		float Cdot = wB - wA - motor.y;
		float impulse = -axialMass * Cdot;
		float oldImpulse = imp.z;
		float maxImpulse = h * motor.x;
		imp.z = S2_CLAMP(imp.z + impulse, -maxImpulse, maxImpulse);
		impulse = imp.z - oldImpulse;
		wA -= iA * impulse;
		wB += iB * impulse;
	}
	else if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_WELD && fixedRotation == false)
	{
		// weld angular row, rigid (DESIGN.md §3.8): the position error is left to the NGS position pass
		float impulse = -axialMass * (wB - wA);
		imp.z += impulse;
		wA -= iA * impulse;
		wB += iB * impulse;
	}

	if ((head.x & S2B_JOINT_ENABLE_LIMIT) && fixedRotation == false)
	{
		float angle = s2RelativeAngle(qB, qA) - lim.x;
		{
			float C = angle - lim.y;
			float Cdot = wB - wA;
			float impulse = -axialMass * (Cdot + S2_MAX(C, 0.0f) / h);
			float oldImpulse = limp.x;
			limp.x = S2_MAX(limp.x + impulse, 0.0f);
			impulse = limp.x - oldImpulse;
			wA -= iA * impulse;
			wB += iB * impulse;
		}
		{
			float C = lim.z - angle;
			float Cdot = wA - wB;
			float impulse = -axialMass * (Cdot + S2_MAX(C, 0.0f) / h);
			float oldImpulse = limp.y;
			limp.y = S2_MAX(limp.y + impulse, 0.0f);
			impulse = limp.y - oldImpulse;
			wA += iA * impulse;
			wB -= iB * impulse;
		}
	}

	{
		s2Vec2 rA = s2RotateVector(qA, V2(anchor.x, anchor.y));
		s2Vec2 rB = s2RotateVector(qB, V2(anchor.z, anchor.w));
		s2Vec2 Cdot = s2Sub(s2Add(vB, s2CrossSV(wB, rB)), s2Add(vA, s2CrossSV(wA, rA)));
		s2Mat22 pivot;
		pivot.cx = V2(pv.x, pv.y);
		pivot.cy = V2(pv.z, pv.w);
		s2Vec2 impulse = s2MulMV(pivot, s2Neg(Cdot));
		imp.x += impulse.x;
		imp.y += impulse.y;
		vA = s2MulSub(vA, mA, impulse);
		wA -= iA * s2Cross(rA, impulse);
		vB = s2MulAdd(vB, mB, impulse);
		wB += iB * s2Cross(rB, impulse);
	}

	jc.imp[t] = imp;
	jc.limp[t] = limp;
	s2bStoreJointVelocities(a, ia, ib, velA, velB, vA, wA, vB, wB, mA, iA, mB, iB);
}

// s2SolveJoint dispatch (reference src/joint.c:329-345)
__device__ __forceinline__ void s2bSolveJointRigid(const SolveArgs& a, int t, float h)
{
	if (a.jc.head[t].x & S2B_JOINT_ENABLE_SPRING)
	{
		s2bSolveSpringVelocity(a, t);
	}
	if (S2B_JOINT_TYPE(a.jc.head[t].x) == S2B_JOINT_MOUSE)
	{
		s2bSolveMouse(a, t);
		return;
	}
	if (S2B_JOINT_TYPE(a.jc.head[t].x) == S2B_JOINT_PRISMATIC)
	{
		s2bSolvePrismaticVelocity<PSOLVE_RIGID>(a, t, h, 0.0f /* inv_h: unused by the rigid rows */, false);
		return;
	}
	if (S2B_JOINT_TYPE(a.jc.head[t].x) == S2B_JOINT_DISTANCE)
	{
		s2bSolveDistanceVelocity<PSOLVE_RIGID>(a, t, h, 0.0f /* inv_h: unused by the rigid rows */, false);
		return;
	}
	if (S2B_JOINT_TYPE(a.jc.head[t].x) == S2B_JOINT_WHEEL)
	{
		s2bSolveWheelVelocity<PSOLVE_RIGID>(a, t, h, 0.0f /* inv_h: unused by the rigid rows */, false);
		return;
	}
	if (S2B_JOINT_TYPE(a.jc.head[t].x) == S2B_JOINT_GEAR)
	{
		s2bSolveGearVelocity<PSOLVE_RIGID>(a, t, h, 0.0f /* inv_h: unused by the rigid row */, false);
		return;
	}
	if (S2B_JOINT_TYPE(a.jc.head[t].x) == S2B_JOINT_PULLEY)
	{
		s2bSolvePulleyVelocity<PSOLVE_RIGID>(a, t, h, 0.0f /* inv_h: unused by the rigid row */, false);
		return;
	}
	if (S2B_JOINT_TYPE(a.jc.head[t].x) == S2B_JOINT_MOTOR)
	{
		s2bSolveMotorVelocity(a, t, h, a.ctx.inv_h);
		return;
	}
	if (a.jc.head[t].x & S2B_JC_SOFT_WELD)
	{
		s2bSolveSoftWeldVelocity<SWELD_RIGID>(a, t, 0.0f /* inv_h: unused by the rigid rows */);
		return;
	}
	s2bSolveRevoluteRigid(a, t, h);
}

// ---------------------------------------------------------------------------------------------------------------
// s2SolveRevolutePosition (reference src/revolute_joint.c:305-419): NGS position pass for the revolute joint (angular
// limit + point-to-point with a fresh 2x2 mass); s2SolveJointPosition does nothing for a mouse joint (joint.c:349-361).
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void s2bSolveJointPosition(const SolveArgs& a, int t)
{
	const JointConstraintView& jc = a.jc;
	int4 head = jc.head[t];
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_MOUSE || S2B_JOINT_TYPE(head.x) == S2B_JOINT_MOTOR)
	{
		return; // a motor joint, like a mouse joint, has no NGS position row (DESIGN.md §3.10)
	}
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_PRISMATIC)
	{
		s2bSolvePrismaticPosition(a, t);
		return;
	}
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_DISTANCE)
	{
		s2bSolveDistancePosition(a, t);
		return;
	}
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_WHEEL)
	{
		s2bSolveWheelPosition(a, t);
		return;
	}
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_GEAR)
	{
		s2bSolveGearPositionT<false>(a, t);
		return;
	}
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_PULLEY)
	{
		s2bSolvePulleyPositionT<false>(a, t);
		return;
	}
	if (head.x & S2B_JC_SOFT_WELD)
	{
		s2bSolveSoftWeldPosition(a, t);
		return;
	}
	int ia = head.y, ib = head.z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 lim = jc.lim[t];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	float axialMass = d0.z;
	bool fixedRotation = (iA + iB == 0.0f);

	if ((head.x & S2B_JOINT_ENABLE_LIMIT) && fixedRotation == false)
	{
		float angle = s2RelativeAngle(qB, qA) - lim.x;
		float C = 0.0f;
		if (S2_ABS(lim.z - lim.y) < 2.0f * s2_angularSlop)
		{
			C = S2_CLAMP(angle - lim.y, -s2_maxAngularCorrection, s2_maxAngularCorrection);
		}
		else if (angle <= lim.y)
		{
			C = S2_CLAMP(angle - lim.y + s2_angularSlop, -s2_maxAngularCorrection, 0.0f);
		}
		else if (angle >= lim.z)
		{
			C = S2_CLAMP(angle - lim.z - s2_angularSlop, 0.0f, s2_maxAngularCorrection);
		}
		float limitImpulse = -axialMass * C;
		qA = s2IntegrateRot(qA, -iA * limitImpulse);
		qB = s2IntegrateRot(qB, iB * limitImpulse);
	}
	else if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_WELD && fixedRotation == false)
	{
		// weld angular row (DESIGN.md §3.8); the point row below then runs on the corrected rotations
		float C = s2UnwindAngle(s2RelativeAngle(qB, qA) - lim.x);
		float p = -axialMass * S2_CLAMP(C, -s2_maxAngularCorrection, s2_maxAngularCorrection);
		qA = s2IntegrateRot(qA, -iA * p);
		qB = s2IntegrateRot(qB, iB * p);
	}

	{
		s2Vec2 rA = s2RotateVector(qA, V2(anchor.x, anchor.y));
		s2Vec2 rB = s2RotateVector(qB, V2(anchor.z, anchor.w));
		s2Vec2 C = s2Add(s2Add(s2Sub(dcB, dcA), s2Sub(rB, rA)), V2(d0.x, d0.y));
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

	if ((mA != 0.0f) || (iA != 0.0f))
	{
		a.bodies.pose[ia] = make_float4(dcA.x, dcA.y, qA.s, qA.c);
	}
	if ((mB != 0.0f) || (iB != 0.0f))
	{
		a.bodies.pose[ib] = make_float4(dcB.x, dcB.y, qB.s, qB.c);
	}
}

// ---------------------------------------------------------------------------------------------------------------
// s2SolveJoint_XPBD (reference src/joint.c:447-463): mouse -> s2SolveMouse; revolute -> s2SolveRevolute_XPBD
// (src/revolute_joint.c:825-888): distance constraint along the current separation, zero compliance.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void s2bSolveJointXpbd(const SolveArgs& a, int t)
{
	const JointConstraintView& jc = a.jc;
	if (jc.head[t].x & S2B_JOINT_ENABLE_SPRING)
	{
		s2bSolveSpringXpbd(a, t);
	}
	int4 head = jc.head[t];
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_MOUSE)
	{
		s2bSolveMouse(a, t);
		return;
	}
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_PRISMATIC)
	{
		s2bSolvePrismaticXpbd(a, t);
		return;
	}
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_DISTANCE)
	{
		s2bSolveDistanceXpbd(a, t);
		return;
	}
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_WHEEL)
	{
		s2bSolveWheelXpbd(a, t);
		return;
	}
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_GEAR)
	{
		s2bSolveGearPositionT<true>(a, t);
		return;
	}
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_PULLEY)
	{
		s2bSolvePulleyPositionT<true>(a, t);
		return;
	}
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_MOTOR)
	{
		s2bSolveMotorXpbd(a, t);
		return;
	}
	if (head.x & S2B_JC_SOFT_WELD)
	{
		s2bSolveSoftWeldXpbd(a, t);
		return;
	}
	const float compliance = 0.0f;
	int ia = head.y, ib = head.z;
	float4 anchor = jc.anchor[t];
	float4 mass = jc.mass[t];
	float4 d0 = jc.d0ax[t];
	float4 poseA = a.bodies.pose[ia], poseB = a.bodies.pose[ib];
	s2Vec2 dcA = V2(poseA.x, poseA.y), dcB = V2(poseB.x, poseB.y);
	s2Rot qA = R2(poseA.z, poseA.w), qB = R2(poseB.z, poseB.w);
	float mA = mass.x, iA = mass.y, mB = mass.z, iB = mass.w;
	if (S2B_JOINT_TYPE(head.x) == S2B_JOINT_WELD && iA + iB != 0.0f)
	{
		// weld angular row, zero compliance (DESIGN.md §3.8); the point row below then runs on the corrected rotations
		float C = s2UnwindAngle(s2RelativeAngle(qB, qA) - jc.lim[t].x);
		float p = -C / (iA + iB);
		qA = s2IntegrateRot(qA, -iA * p);
		qB = s2IntegrateRot(qB, iB * p);
	}
	s2Vec2 rA = s2RotateVector(qA, V2(anchor.x, anchor.y));
	s2Vec2 rB = s2RotateVector(qB, V2(anchor.z, anchor.w));
	s2Vec2 separation = s2Add(s2Add(s2Sub(dcB, dcA), s2Sub(rB, rA)), V2(d0.x, d0.y));
	float c = s2Length(separation);
	// s2Normalize (reference src/math.c:40-51)
	s2Vec2 n = V2(0.0f, 0.0f);
	if (c >= 0.001f * 1.1920929e-07f)
	{
		float invLength = 1.0f / c;
		n = V2(invLength * separation.x, invLength * separation.y);
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
	if ((mA != 0.0f) || (iA != 0.0f))
	{
		a.bodies.pose[ia] = make_float4(dcA.x, dcA.y, qA.s, qA.c);
	}
	if ((mB != 0.0f) || (iB != 0.0f))
	{
		a.bodies.pose[ib] = make_float4(dcB.x, dcB.y, qB.s, qB.c);
	}
}
