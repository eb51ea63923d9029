// solver2d-b200 — extensions to the solver2d C API that only make sense for the GPU library.
// A client that sticks to include/solver2d/solver2d.h never needs this header.
#pragma once

#include "s2b_device.h"
#include "solver2d/constants.h"
#include "solver2d/distance.h"
#include "solver2d/geometry.h"
#include "solver2d/id.h"
#include "solver2d/types.h"

#ifdef __cplusplus
extern "C"
{
#endif

// The device world behind a public world id, for the stage-level entry points of s2b_device.h (schedule selection,
// counters, NCCL packing). The handle is owned by the world.
S2B_API s2bWorld* s2World_GetDevice(s2WorldId worldId);

// Bounce contacts by their shapes' restitution (default off: restitution is ignored, as in the reference). A contact's
// restitution is the larger of its two shapes' s2ShapeDef.restitution. Takes effect at the next s2World_Step.
S2B_API void s2World_EnableRestitution(s2WorldId worldId, bool enable);
// Approach speed (m/s) below which a contact does not bounce. Default 1 m/s, the reference's world->restitutionThreshold.
// A threshold that is not finite or is negative is rejected (the world keeps its threshold). Takes effect at the next
// s2World_Step.
S2B_API void s2World_SetRestitutionThreshold(s2WorldId worldId, float threshold);

// Weld joint: holds body B to body A, the anchor points together and angle(B) - angle(A) at referenceAngle. With both
// hertz at 0 it is rigid: as rigid as the solver variant makes a revolute joint's point constraint (DESIGN.md §3.8). A
// positive linearHertz makes the anchor constraint a spring, a positive angularHertz the angle constraint (a soft weld,
// DESIGN.md §3.15). Anchors are relative to each body's origin. Destroy it with s2DestroyJoint.
typedef struct s2WeldJointDef
{
	s2BodyId bodyIdA;
	s2BodyId bodyIdB;
	s2Vec2 localAnchorA;
	s2Vec2 localAnchorB;
	float referenceAngle; // angle(B) - angle(A) at rest
	float drawSize;
	bool collideConnected;	   // keep the contacts the two bodies already have
	float linearHertz;		   // the anchor spring's stiffness as a frequency (Hz), >= 0; 0 = rigid
	float linearDampingRatio;  // the anchor spring's damping ratio, >= 0 (1 = critical)
	float angularHertz;		   // the angle spring's stiffness as a frequency (Hz), >= 0; 0 = rigid
	float angularDampingRatio; // the angle spring's damping ratio, >= 0 (1 = critical)
} s2WeldJointDef;

S2_INLINE struct s2WeldJointDef s2DefaultWeldJointDef(void)
{
	s2WeldJointDef def = S2_ZERO_INIT;
	def.bodyIdA = s2_nullBodyId;
	def.bodyIdB = s2_nullBodyId;
	def.drawSize = 1.0f;
	return def;
}

// Returns s2_nullJointId (and creates nothing) for a negative or non-finite hertz or damping ratio.
S2B_API s2JointId s2CreateWeldJoint(s2WorldId worldId, const s2WeldJointDef* def);
// The soft weld (DESIGN.md §3.15). A setter ignores a negative or non-finite value (the joint keeps its value) and a joint
// that is not a weld; a change takes effect at the next step. A getter returns 0 for a joint that is not a weld.
S2B_API void s2WeldJoint_SetLinearHertz(s2JointId jointId, float hertz);
S2B_API void s2WeldJoint_SetLinearDampingRatio(s2JointId jointId, float dampingRatio);
S2B_API void s2WeldJoint_SetAngularHertz(s2JointId jointId, float hertz);
S2B_API void s2WeldJoint_SetAngularDampingRatio(s2JointId jointId, float dampingRatio);
S2B_API float s2WeldJoint_GetLinearHertz(s2JointId jointId);
S2B_API float s2WeldJoint_GetLinearDampingRatio(s2JointId jointId);
S2B_API float s2WeldJoint_GetAngularHertz(s2JointId jointId);
S2B_API float s2WeldJoint_GetAngularDampingRatio(s2JointId jointId);

// Prismatic (slider) joint: body B slides along an axis fixed in body A, keeps angle(B) - angle(A) at referenceAngle and
// may have translation limits, a linear motor (DESIGN.md §3.9) and a spring toward translation 0 (DESIGN.md §3.14). Anchors
// are relative to each body's origin; the translation is measured along the axis from anchor A to anchor B. Under XPBD the
// motor is not applied. Destroy it with s2DestroyJoint.
typedef struct s2PrismaticJointDef
{
	s2BodyId bodyIdA;
	s2BodyId bodyIdB;
	s2Vec2 localAnchorA;
	s2Vec2 localAnchorB;
	s2Vec2 localAxisA;	  // the sliding axis in body A's frame; normalized at creation
	float referenceAngle; // angle(B) - angle(A) at rest
	bool enableLimit;
	float lowerTranslation; // m
	float upperTranslation; // m
	bool enableMotor;
	float motorSpeed;	 // m/s
	float maxMotorForce; // N
	float drawSize;
	bool collideConnected; // keep the contacts the two bodies already have
	bool enableSpring;	   // a spring along the axis that pulls the translation toward 0
	float hertz;		   // the spring's stiffness as a frequency (Hz), >= 0; 0 exerts nothing
	float dampingRatio;	   // the spring's damping ratio, >= 0 (1 = critical)
} s2PrismaticJointDef;

S2_INLINE struct s2PrismaticJointDef s2DefaultPrismaticJointDef(void)
{
	s2PrismaticJointDef def = S2_ZERO_INIT;
	def.bodyIdA = s2_nullBodyId;
	def.bodyIdB = s2_nullBodyId;
	def.localAxisA.x = 1.0f;
	def.drawSize = 1.0f;
	return def;
}

// Returns s2_nullJointId (and creates nothing) for an axis of zero length or with a non-finite component, for
// lowerTranslation > upperTranslation, or for a negative or non-finite hertz or dampingRatio.
S2B_API s2JointId s2CreatePrismaticJoint(s2WorldId worldId, const s2PrismaticJointDef* def);
S2B_API void s2PrismaticJoint_EnableLimit(s2JointId jointId, bool enableLimit);
// Ignored when lower > upper (the joint keeps its limits).
S2B_API void s2PrismaticJoint_SetLimits(s2JointId jointId, float lower, float upper);
S2B_API void s2PrismaticJoint_EnableMotor(s2JointId jointId, bool enableMotor);
S2B_API void s2PrismaticJoint_SetMotorSpeed(s2JointId jointId, float motorSpeed);
// The motor force of the last step (N): inverseTimeStep times the motor impulse.
S2B_API float s2PrismaticJoint_GetMotorForce(s2JointId jointId, float inverseTimeStep);
// The current translation (m) along the world axis, from anchor A to anchor B.
S2B_API float s2PrismaticJoint_GetTranslation(s2JointId jointId);
// The spring (DESIGN.md §3.14). A negative or non-finite hertz or damping ratio is ignored (the joint keeps its value).
S2B_API void s2PrismaticJoint_EnableSpring(s2JointId jointId, bool enableSpring);
S2B_API void s2PrismaticJoint_SetSpringHertz(s2JointId jointId, float hertz);
S2B_API void s2PrismaticJoint_SetSpringDampingRatio(s2JointId jointId, float dampingRatio);

// Revolute joint spring (DESIGN.md §3.14): pulls angle(B) - angle(A) toward referenceAngle with stiffness hertz (Hz) and
// damping ratio dampingRatio, before the motor and the limits. s2RevoluteJointDef is the reference's and has no spring
// fields: a revolute joint starts without a spring (hertz 0, damping ratio 0). A negative or non-finite hertz or damping
// ratio is ignored (the joint keeps its value). A spring on a joint whose two rotations are fixed exerts nothing.
S2B_API void s2RevoluteJoint_EnableSpring(s2JointId jointId, bool enableSpring);
S2B_API void s2RevoluteJoint_SetSpringHertz(s2JointId jointId, float hertz);
S2B_API void s2RevoluteJoint_SetSpringDampingRatio(s2JointId jointId, float dampingRatio);

// Motor joint: drives body B toward a pose relative to body A with bounded effort (DESIGN.md §3.10). Each solver step h it
// removes the fraction correctionFactor of the pose error, with an impulse of at most h * maxForce (linear) and
// h * maxTorque (angular). It has no spring and no rigid part. Uses: top-down friction (a joint to the ground with zero
// offsets and small caps), platforms that a heavy load can stall, force-limited characters and pose controllers.
// Re-target it every frame with s2World_SetMotorJointOffsets. Destroy it with s2DestroyJoint.
typedef struct s2MotorJointDef
{
	s2BodyId bodyIdA;
	s2BodyId bodyIdB;
	s2Vec2 linearOffset;	// target position of body B's origin in body A's frame, relative to A's origin (m)
	float angularOffset;	// target angle(B) - angle(A) (rad), within [-pi, pi]
	float maxForce;			// N, >= 0
	float maxTorque;		// N-m, >= 0
	float correctionFactor; // in [0, 1]: fraction of the pose error removed per solver step h
	bool collideConnected;	// keep the contacts the two bodies already have
} s2MotorJointDef;

S2_INLINE struct s2MotorJointDef s2DefaultMotorJointDef(void)
{
	s2MotorJointDef def = S2_ZERO_INIT;
	def.bodyIdA = s2_nullBodyId;
	def.bodyIdB = s2_nullBodyId;
	def.maxForce = 1.0f;
	def.maxTorque = 1.0f;
	def.correctionFactor = 0.3f;
	return def;
}

// Returns s2_nullJointId (and creates nothing) for a non-finite offset, a negative or non-finite maxForce or maxTorque, or
// a correctionFactor outside [0, 1]. The setters ignore such input (the joint keeps its value).
S2B_API s2JointId s2CreateMotorJoint(s2WorldId worldId, const s2MotorJointDef* def);
S2B_API void s2MotorJoint_SetLinearOffset(s2JointId jointId, s2Vec2 linearOffset);
S2B_API s2Vec2 s2MotorJoint_GetLinearOffset(s2JointId jointId);
S2B_API void s2MotorJoint_SetAngularOffset(s2JointId jointId, float angularOffset);
S2B_API float s2MotorJoint_GetAngularOffset(s2JointId jointId);
S2B_API void s2MotorJoint_SetMaxForce(s2JointId jointId, float maxForce);
S2B_API void s2MotorJoint_SetMaxTorque(s2JointId jointId, float maxTorque);
S2B_API void s2MotorJoint_SetCorrectionFactor(s2JointId jointId, float correctionFactor);
// The linear impulse of the last step times inverseTimeStep (N); the impulse is per solver step h.
S2B_API s2Vec2 s2MotorJoint_GetConstraintForce(s2JointId jointId, float inverseTimeStep);
// The angular impulse of the last step times inverseTimeStep (N-m).
S2B_API float s2MotorJoint_GetConstraintTorque(s2JointId jointId, float inverseTimeStep);

// Distance joint (DESIGN.md §3.16; Box2D v3's semantics): holds anchor B at a distance from anchor A along the line between
// them, which turns as the bodies move. Rows, all along that line: a spring toward `length` (enableSpring, acts when
// minLength < maxLength and hertz > 0), a motor (enableMotor: drives the rate of change of the length to motorSpeed with at
// most maxMotorForce), a lower and an upper limit (enableLimit, when minLength < maxLength) and a rigid row toward `length`
// (whenever the spring is off or minLength == maxLength). A rope is enableSpring with hertz 0 and a limit: free inside
// [minLength, maxLength], taut at maxLength. Anchors are relative to each body's origin. Under XPBD the motor is not applied.
// Destroy it with s2DestroyJoint.
typedef struct s2DistanceJointDef
{
	s2BodyId bodyIdA;
	s2BodyId bodyIdB;
	s2Vec2 localAnchorA;
	s2Vec2 localAnchorB;
	float length; // rest length (m)
	bool enableSpring;
	float hertz;		// the spring's stiffness as a frequency (Hz), >= 0; 0 exerts nothing
	float dampingRatio; // the spring's damping ratio, >= 0 (1 = critical)
	bool enableLimit;
	float minLength; // m
	float maxLength; // m
	bool enableMotor;
	float maxMotorForce; // N, >= 0
	float motorSpeed;	 // m/s, positive lengthens
	bool collideConnected; // keep the contacts the two bodies already have
} s2DistanceJointDef;

S2_INLINE struct s2DistanceJointDef s2DefaultDistanceJointDef(void)
{
	s2DistanceJointDef def = S2_ZERO_INIT;
	def.bodyIdA = s2_nullBodyId;
	def.bodyIdB = s2_nullBodyId;
	def.length = 1.0f;
	def.maxLength = s2_huge;
	return def;
}

// Returns s2_nullJointId (and creates nothing) for any non-finite value, a negative length, minLength, hertz, dampingRatio or
// maxMotorForce, or minLength > maxLength. Otherwise length, minLength and maxLength are each clamped into
// [s2_linearSlop, s2_huge], as Box2D does: a rest length below the slop would leave the line between the anchors undefined.
S2B_API s2JointId s2CreateDistanceJoint(s2WorldId worldId, const s2DistanceJointDef* def);
// The setters ignore a non-finite or negative value (the joint keeps its value) and a joint that is not a distance joint;
// lengths are clamped as at creation. A change takes effect at the next step. The getters return 0 for another type.
S2B_API void s2DistanceJoint_SetLength(s2JointId jointId, float length);
S2B_API float s2DistanceJoint_GetLength(s2JointId jointId);
S2B_API void s2DistanceJoint_EnableLimit(s2JointId jointId, bool enableLimit);
// Ignored when minLength > maxLength.
S2B_API void s2DistanceJoint_SetLengthRange(s2JointId jointId, float minLength, float maxLength);
S2B_API float s2DistanceJoint_GetMinLength(s2JointId jointId);
S2B_API float s2DistanceJoint_GetMaxLength(s2JointId jointId);
S2B_API void s2DistanceJoint_EnableSpring(s2JointId jointId, bool enableSpring);
S2B_API void s2DistanceJoint_SetSpringHertz(s2JointId jointId, float hertz);
S2B_API void s2DistanceJoint_SetSpringDampingRatio(s2JointId jointId, float dampingRatio);
S2B_API void s2DistanceJoint_EnableMotor(s2JointId jointId, bool enableMotor);
// Any finite speed.
S2B_API void s2DistanceJoint_SetMotorSpeed(s2JointId jointId, float motorSpeed);
S2B_API void s2DistanceJoint_SetMaxMotorForce(s2JointId jointId, float maxMotorForce);
// The motor force of the last step (N): inverseTimeStep times the motor impulse.
S2B_API float s2DistanceJoint_GetMotorForce(s2JointId jointId, float inverseTimeStep);
// The current distance between the two anchors (m).
S2B_API float s2DistanceJoint_GetCurrentLength(s2JointId jointId);

// Wheel joint (DESIGN.md §3.17; Box2D v3's semantics): body B's anchor slides along an axis fixed in body A, and body B
// turns freely about it. Rows: a spring along the axis toward translation 0 (enableSpring, acts when hertz > 0), a motor on
// the relative rotation (enableMotor: drives angularVelocity(B) - angularVelocity(A) to motorSpeed with at most
// maxMotorTorque; nothing when both rotations are fixed), a lower and an upper translation limit (enableLimit) and the
// point-on-line row that keeps anchor B on the axis. Equal limits make a rigid axle. Anchors are relative to each body's
// origin; the translation is measured along the axis from anchor A to anchor B. Under XPBD the motor is not applied.
// Destroy it with s2DestroyJoint.
typedef struct s2WheelJointDef
{
	s2BodyId bodyIdA;
	s2BodyId bodyIdB;
	s2Vec2 localAnchorA;
	s2Vec2 localAnchorB;
	s2Vec2 localAxisA; // the suspension axis in body A's frame; normalized at creation
	bool enableSpring;
	float hertz;		// the spring's stiffness as a frequency (Hz), >= 0; 0 exerts nothing
	float dampingRatio; // the spring's damping ratio, >= 0 (1 = critical)
	bool enableLimit;
	float lowerTranslation; // m
	float upperTranslation; // m
	bool enableMotor;
	float maxMotorTorque;  // N-m, >= 0
	float motorSpeed;	   // rad/s
	bool collideConnected; // keep the contacts the two bodies already have
} s2WheelJointDef;

S2_INLINE struct s2WheelJointDef s2DefaultWheelJointDef(void)
{
	s2WheelJointDef def = S2_ZERO_INIT;
	def.bodyIdA = s2_nullBodyId;
	def.bodyIdB = s2_nullBodyId;
	def.localAxisA.y = 1.0f;
	def.enableSpring = true;
	def.hertz = 1.0f;
	def.dampingRatio = 0.7f;
	return def;
}

// Returns s2_nullJointId (and creates nothing) for an axis of zero length or with a non-finite component, a non-finite
// anchor, lowerTranslation > upperTranslation, a negative or non-finite hertz, dampingRatio or maxMotorTorque, or a
// non-finite motorSpeed.
S2B_API s2JointId s2CreateWheelJoint(s2WorldId worldId, const s2WheelJointDef* def);
// The setters ignore bad input (the joint keeps its value) and a joint that is not a wheel joint. A change takes effect at
// the next step. The spring setters are the revolute and prismatic joints' (a negative or non-finite value is ignored).
S2B_API void s2WheelJoint_EnableSpring(s2JointId jointId, bool enableSpring);
S2B_API void s2WheelJoint_SetSpringHertz(s2JointId jointId, float hertz);
S2B_API void s2WheelJoint_SetSpringDampingRatio(s2JointId jointId, float dampingRatio);
S2B_API void s2WheelJoint_EnableLimit(s2JointId jointId, bool enableLimit);
// Ignored when lower > upper or either is not finite.
S2B_API void s2WheelJoint_SetLimits(s2JointId jointId, float lower, float upper);
S2B_API void s2WheelJoint_EnableMotor(s2JointId jointId, bool enableMotor);
// Any finite speed (rad/s).
S2B_API void s2WheelJoint_SetMotorSpeed(s2JointId jointId, float motorSpeed);
// Ignored when negative or not finite.
S2B_API void s2WheelJoint_SetMaxMotorTorque(s2JointId jointId, float maxMotorTorque);
// The motor torque of the last step (N-m): inverseTimeStep times the angular motor impulse. 0 for another joint type.
S2B_API float s2WheelJoint_GetMotorTorque(s2JointId jointId, float inverseTimeStep);
// The current translation (m) along the world axis, from anchor A to anchor B. 0 for another joint type.
S2B_API float s2WheelJoint_GetTranslation(s2JointId jointId);

// Pulley joint (DESIGN.md §3.18; Box2D 2.4's b2PulleyJoint): anchor A hangs on a rope from the fixed world point
// groundAnchorA, anchor B on a rope from groundAnchorB, and the joint holds lengthA + ratio lengthB at its value for the
// rest lengths, lengthA + ratio lengthB, where each length is the distance from the ground anchor to the body anchor. Moving
// anchor A by d along its rope moves anchor B by d / ratio along its own. It is an equality constraint, as in Box2D 2.4: the
// ropes can push as well as pull (there is no slack, tension-only pulley). A rope whose anchor comes within
// 10 s2_linearSlop of its ground anchor exerts nothing on its body. Anchors are relative to each body's origin. Destroy it
// with s2DestroyJoint.
typedef struct s2PulleyJointDef
{
	s2BodyId bodyIdA;
	s2BodyId bodyIdB;
	s2Vec2 groundAnchorA; // world
	s2Vec2 groundAnchorB; // world
	s2Vec2 localAnchorA;
	s2Vec2 localAnchorB;
	float lengthA; // the rest length of rope A (m), >= 0
	float lengthB; // the rest length of rope B (m), >= 0
	float ratio;   // > FLT_EPSILON
	bool collideConnected;
} s2PulleyJointDef;

// Box2D 2.4's defaults, collideConnected = true included
S2_INLINE struct s2PulleyJointDef s2DefaultPulleyJointDef(void)
{
	s2PulleyJointDef def = S2_ZERO_INIT;
	def.bodyIdA = s2_nullBodyId;
	def.bodyIdB = s2_nullBodyId;
	def.groundAnchorA.x = -1.0f;
	def.groundAnchorA.y = 1.0f;
	def.groundAnchorB.x = 1.0f;
	def.groundAnchorB.y = 1.0f;
	def.localAnchorA.x = -1.0f;
	def.localAnchorB.x = 1.0f;
	def.ratio = 1.0f;
	def.collideConnected = true;
	return def;
}

// Returns s2_nullJointId (and creates nothing) for a non-finite anchor or length, a negative length, or a ratio that is not
// finite or is <= FLT_EPSILON.
S2B_API s2JointId s2CreatePulleyJoint(s2WorldId worldId, const s2PulleyJointDef* def);
// The getters return 0 (or a zero vector) for a joint of another type.
S2B_API s2Vec2 s2PulleyJoint_GetGroundAnchorA(s2JointId jointId);
S2B_API s2Vec2 s2PulleyJoint_GetGroundAnchorB(s2JointId jointId);
// the rest lengths (m)
S2B_API float s2PulleyJoint_GetLengthA(s2JointId jointId);
S2B_API float s2PulleyJoint_GetLengthB(s2JointId jointId);
S2B_API float s2PulleyJoint_GetRatio(s2JointId jointId);
// the current distance (m) from each ground anchor to its body anchor
S2B_API float s2PulleyJoint_GetCurrentLengthA(s2JointId jointId);
S2B_API float s2PulleyJoint_GetCurrentLengthB(s2JointId jointId);

// Gear joint (DESIGN.md §3.19; Box2D 2.4's b2GearJoint): couples two revolute or prismatic joints whose body A (the frame)
// is static. The gear's body A is joint 1's body B and its body B is joint 2's body B, and it holds
// coordinate1 + ratio coordinate2 at the value it has when created, where a revolute joint's coordinate is its angle
// (angle(B) - angle(A) - referenceAngle, unwound: it does not wrap at +/- pi, so a gear train may turn any number of times)
// and a prismatic joint's its translation along its axis. Turning joint 1 by d turns joint 2 by -d / ratio. The linked
// joints keep acting on their own. s2DestroyJoint on a linked joint (a break included) destroys the gears that link it
// first, so their ids go stale (s2DestroyJoint on a stale id does nothing); s2Body_SetTransform on a frame body moves the gear's frames with it and keeps its constant. Destroy it with
// s2DestroyJoint.
typedef struct s2GearJointDef
{
	s2JointId jointId1;
	s2JointId jointId2;
	float ratio; // finite; the sign sets the direction of the coupling
	bool collideConnected;
} s2GearJointDef;

// Box2D 2.4's defaults: ratio 1, collideConnected false
S2_INLINE struct s2GearJointDef s2DefaultGearJointDef(void)
{
	s2GearJointDef def = S2_ZERO_INIT;
	def.jointId1 = s2_nullJointId;
	def.jointId2 = s2_nullJointId;
	def.ratio = 1.0f;
	return def;
}

// Returns s2_nullJointId (and creates nothing) for a stale, null or foreign joint id, a joint that is not revolute or
// prismatic, a joint whose body A is not static, two joints with the same body B, or a non-finite ratio.
S2B_API s2JointId s2CreateGearJoint(s2WorldId worldId, const s2GearJointDef* def);
// The getters return s2_nullJointId or 0 for a joint of another type.
S2B_API s2JointId s2GearJoint_GetJoint1(s2JointId jointId);
S2B_API s2JointId s2GearJoint_GetJoint2(s2JointId jointId);
S2B_API float s2GearJoint_GetRatio(s2JointId jointId);

// ---- joint reactions and breakable joints (DESIGN.md §3.13) --------------------------------------------------------

// What a joint exerts on body B over the last step: force (N, world frame) and torque (N-m).
typedef struct s2JointReaction
{
	s2Vec2 force;
	float torque;
} s2JointReaction;

// The one definition of a joint's reaction, used by the device's reaction pass, the host getters and the tests. `type` is
// an S2B_JOINT_* value; the impulses are the columns of s2bJointRow; qA is body A's rotation at the end of the step (only the
// prismatic and wheel joints read it, with localAxisA). `rate` is 1 / (the interval the solver variant accumulates the
// impulses over): 1 / dt under TGS_Sticky, 1 / h under every other variant (h = dt for the variants that do not sub-step).
// A revolute, prismatic or wheel joint with its spring enabled passes motorImpulse + springImpulse as `motorImpulse` (the
// spring acts on the same axis: the revolute's torque, the prismatic's and the wheel's axial force), so its reaction and
// break test include the spring's load; every other joint passes motorImpulse.
//   revolute   force = rate impulse    torque = rate (motorImpulse + lowerImpulse - upperImpulse)
//   mouse, weld, motor                 force = rate impulse    torque = rate motorImpulse
//   prismatic  force = rate (impulse.x perp + (motorImpulse + lowerImpulse - upperImpulse) axis), torque = rate impulse.y,
//              axis = qA localAxisA, perp = leftPerp(axis)
//   wheel      as prismatic: impulse.x is the perpendicular impulse, impulse.y the angular motor's and motorImpulse (0 in
//              the row) carries the spring, so force = rate (impulse.x perp + (spring + lower - upper) axis) and
//              torque = rate impulse.y
//   distance   force = rate (impulse.x + motorImpulse + lowerImpulse - upperImpulse) axis, torque = 0. Here localAxisA is the
//              WORLD axis, the unit vector from anchor A to anchor B at the end of the step (zero when they coincide), and
//              qA is not read; a distance joint with its spring enabled also passes motorImpulse + springImpulse.
//   pulley     the distance branch with localAxisA = -ratio uB, uB the unit vector from ground anchor B to anchor B at the end
//              of the step (zero within 10 s2_linearSlop), and impulse.x the rope impulse: force = rate impulse.x (-ratio uB),
//              torque = 0
//   gear       the generic branch: impulse = (lambda Jv2) and motorImpulse = lambda Jw2, side 2's Jacobian at the end of
//              the step scaled by the ratio (s2cGearReaction), so force = rate lambda Jv2, torque = rate lambda Jw2
// Every operation is a separate float32 rounding, so the host and the device (built without contraction) agree bit for bit.
S2_INLINE s2JointReaction s2MakeJointReaction(int32_t type, s2Vec2 impulse, float motorImpulse, float lowerImpulse,
											  float upperImpulse, s2Rot qA, s2Vec2 localAxisA, float rate)
{
	s2JointReaction r;
	s2Vec2 f = impulse;
	float t = motorImpulse;
	if (type == S2B_JOINT_REVOLUTE)
	{
		t = motorImpulse + lowerImpulse - upperImpulse;
	}
	else if (type == S2B_JOINT_DISTANCE || type == S2B_JOINT_PULLEY)
	{
		float axial = impulse.x + motorImpulse + lowerImpulse - upperImpulse;
		f.x = axial * localAxisA.x;
		f.y = axial * localAxisA.y;
		t = 0.0f;
	}
	else if (type == S2B_JOINT_PRISMATIC || type == S2B_JOINT_WHEEL)
	{
		s2Vec2 axis = s2RotateVector(qA, localAxisA);
		s2Vec2 perp = s2LeftPerp(axis);
		float axial = motorImpulse + lowerImpulse - upperImpulse;
		f.x = impulse.x * perp.x + axial * axis.x;
		f.y = impulse.x * perp.y + axial * axis.y;
		t = impulse.y;
	}
	r.force.x = rate * f.x;
	r.force.y = rate * f.y;
	r.torque = rate * t;
	return r;
}

// s2MakeJointReaction as an exported host function, for bindings and CPU tests that evaluate oracle rows with the same
// arithmetic.
S2B_API s2JointReaction s2ComputeJointReaction(int32_t type, s2Vec2 impulse, float motorImpulse, float lowerImpulse,
											   float upperImpulse, s2Rot qA, s2Vec2 localAxisA, float rate);

// The reaction of the last s2World_Step (zero before the first step), from the same impulses and rate the break test used.
// Every joint type. XPBD keeps no impulses for its revolute, weld, prismatic and motor rows, so they read zero under XPBD.
// Under XPBD a mouse joint reads its running impulse (carried across steps without a warm start or reset) times 1 / h:
// not a measured load, since XPBD's mouse joint does not hold a load at rest (DESIGN.md §3.13).
S2B_API s2Vec2 s2Joint_GetReactionForce(s2JointId jointId);
S2B_API float s2Joint_GetReactionTorque(s2JointId jointId);
// Break thresholds (default: none). A positive finite value sets one, 0 removes it, a negative or NaN value is ignored (the
// joint keeps its value). A joint breaks when |force| > breakForce or |torque| > breakTorque, each test applying only when
// its threshold is set. A joint that exceeds a threshold at the end of a step acted in that step; the next s2World_Step
// destroys it, exactly as s2DestroyJoint, before it pushes edits to the device. Until then it exists, its getters report the
// load that broke it, and it may be destroyed by the caller.
S2B_API void s2Joint_SetBreakForce(s2JointId jointId, float breakForce);
S2B_API float s2Joint_GetBreakForce(s2JointId jointId);
S2B_API void s2Joint_SetBreakTorque(s2JointId jointId, float breakTorque);
S2B_API float s2Joint_GetBreakTorque(s2JointId jointId);
// The joints that went over a threshold in the last step, in slot order, with the ids they had then. Returns the count and
// writes at most `capacity` ids.
S2B_API int32_t s2World_GetBrokenJoints(s2WorldId worldId, s2JointId* out, int32_t capacity);
// Bulk s2Joint_GetReactionForce + _GetReactionTorque, computed on the device: {fx, fy, torque} for joint slots
// [0, min(capacity, joint capacity)) into out[3 * capacity]; free slots read zero. Returns the joint capacity.
S2B_API int32_t s2World_GetJointReactions(s2WorldId worldId, float* out, int32_t capacity);

// Continuous collision of dynamic bodies against static shapes (default off: collision is discrete, as in the reference).
// When on, a dynamic body that moved more than half its smallest inner extent in a step is swept from its pose at the
// start of the step to its pose at the end against the static shapes its shapes may collide with, and stopped at the
// first time of impact, s2_linearSlop short of the surface; its velocity is kept. Bodies that start the step touching a
// static shape are held back only if a small core inside the shape would hit it, or starts touching it and moves toward
// it (the body is then already a quarter of its inner extent deep). Dynamic against dynamic or kinematic bodies is swept
// only for bullets (s2Body_SetBullet). Takes effect at the next s2World_Step.
S2B_API void s2World_EnableContinuous(s2WorldId worldId, bool enable);

// Bullets (DESIGN.md §3.12; default off). While continuous collision is on, a fast dynamic bullet (fast by the rule above)
// is swept once every other body has its final pose for the step: against the shapes of static, kinematic and non-bullet
// dynamic bodies, each held still at that final pose, under the same pair rules. It stops at the first time of impact,
// s2_linearSlop short of the surface, and keeps its velocity, so the next step's contact does the stopping. Bullet against
// bullet is not swept, and a target's own motion within the step is not swept either. No effect on static and kinematic
// bodies, nor while continuous collision is off. Takes effect at the next s2World_Step.
S2B_API void s2Body_SetBullet(s2BodyId bodyId, bool flag);
S2B_API bool s2Body_IsBullet(s2BodyId bodyId);

// Motion of a body over one step, for s2TimeOfImpact: the centre of mass moves linearly from c1 to c2 and the rotation is
// the normalised linear interpolation of q1 and q2.
typedef struct s2Sweep
{
	s2Vec2 localCenter; // centre of mass in the body frame
	s2Vec2 c1, c2;		// centre of mass in the world at fractions 0 and 1
	s2Rot q1, q2;		// rotation at fractions 0 and 1
} s2Sweep;

typedef struct s2TOIInput
{
	s2DistanceProxy proxyA; // vertices in body A's frame
	s2DistanceProxy proxyB; // vertices in body B's frame
	s2Sweep sweepA;
	s2Sweep sweepB;
	float maxFraction; // sweep interval [0, maxFraction], maxFraction <= 1
} s2TOIInput;

typedef enum s2TOIState
{
	s2_toiStateUnknown,
	s2_toiStateFailed,	   // the iteration cap was reached: fraction is a time the shapes are still apart
	s2_toiStateOverlapped, // the shapes are within the target separation at fraction 0
	s2_toiStateHit,		   // the shapes reach the target separation at fraction
	s2_toiStateSeparated   // the shapes stay apart over the whole interval: fraction = maxFraction
} s2TOIState;

typedef struct s2TOIOutput
{
	s2TOIState state;
	float fraction;
	int32_t iterations; // conservative-advancement iterations taken
} s2TOIOutput;

// The body transform of a sweep at `fraction`.
S2B_API s2Transform s2GetSweepTransform(const s2Sweep* sweep, float fraction);
// Time of impact by conservative advancement: the first fraction at which the shapes' separation (radii included) falls to
// s2_linearSlop, within a tolerance of s2_linearSlop / 4. The same function runs in the device's continuous pass.
S2B_API s2TOIOutput s2TimeOfImpact(const s2TOIInput* input);
// iteration cap of s2TimeOfImpact (s2TOIOutput.iterations never exceeds it)
#define S2_TOI_MAX_ITERATIONS 50

// The extents a body is classified as fast by, for one shape given in polygon form (circle: 1 vertex; capsule:
// s2MakeCapsule; segment: s2MakeCapsule with radius 0): minExtent = the radius for a circle or capsule, 0 for a segment,
// the smallest distance from the centroid to an edge plus the radius for a polygon; maxExtent = the largest distance of a
// vertex from localCenter (the body's centre of mass, body frame) plus the radius. A body's extents are the smallest
// minExtent and the largest maxExtent of its shapes. center: where the shape's core proxy sits (a circle of radius
// minExtent / 4 that continuous collision sweeps for a shape that starts a step touching a static shape): the vertex of a
// circle, the midpoint of a capsule or segment, the centroid of a polygon.
typedef struct s2ShapeExtent
{
	float minExtent, maxExtent;
	s2Vec2 center;
} s2ShapeExtent;
S2B_API s2ShapeExtent s2ComputeShapeExtent(const s2Polygon* polygonForm, s2Vec2 localCenter);
// The extents of a body with `count` shapes in polygon form about its centre of mass localCenter: the smallest minExtent
// and the largest maxExtent of the shapes (s2_huge and 0 without shapes), center = localCenter. What the host stores in
// s2bBodyRow.minExtent / maxExtent whenever a shape is added to a body.
S2B_API s2ShapeExtent s2ComputeBodyExtent(const s2Polygon* polygonForms, int32_t count, s2Vec2 localCenter);

// Push every pending host-side edit to the device now (s2World_Step does this itself).
S2B_API void s2World_Flush(s2WorldId worldId);

// Bulk forms of the per-body calls, for clients that touch every body every frame (one FFI call instead of Nb):
//   s2World_ApplyForcesToCenters == s2Body_ApplyForceToCenter for bodyIndices[i] with force (forcesXY[2i], forcesXY[2i+1]);
//   s2World_GetBodyTransforms    == s2Body_GetPosition + rotation for every body slot: {origin.x, origin.y, rot.s, rot.c}
//                                   into out[4 * capacity]; returns the body capacity.
S2B_API void s2World_ApplyForcesToCenters(s2WorldId worldId, const int32_t* bodyIndices, const float* forcesXY, int32_t count);
S2B_API int32_t s2World_GetBodyTransforms(s2WorldId worldId, float* out, int32_t capacity);
// Bulk s2MotorJoint_SetLinearOffset + _SetAngularOffset: offsets[3i .. 3i+2] = (linear x, linear y, angular) for the motor
// joint in slot jointIndices[i] (its s2JointId.index). All entries are checked first: an index out of range, a free slot, a
// joint that is not a motor joint or a non-finite value rejects the call, which then changes nothing and returns false.
// A joint named more than once takes its last entry.
// Unlike the per-joint setters it writes only the offset columns on the device, asynchronously, and keeps the pair search
// prefetched behind the last step. Whichever of the two wrote an offset last before a step wins.
S2B_API bool s2World_SetMotorJointOffsets(s2WorldId worldId, const int32_t* jointIndices, const float* offsets, int32_t count);

// Run `steps` calls of s2World_Step back to back and return the summed device time of the steps in milliseconds, each
// step bracketed by CUDA events on the world's stream. With flushL2 != 0 the L2 (50 MB on an H100) is evicted between steps
// (outside the timed intervals) so every step starts from HBM.
S2B_API float s2World_TimedSteps(s2WorldId worldId, int32_t steps, float timeStep, int32_t velIters, int32_t posIters,
								 bool warmStart, int32_t flushL2);

// The float atan2 the device kernels use (include/solver2d/atan2_f32.h), evaluated on the host: lets a CPU-only test
// pin it to the C library's atan2f.
S2B_API float s2Atan2Device(float y, float x);

#ifdef __cplusplus
}
#endif
