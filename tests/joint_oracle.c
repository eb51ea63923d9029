// TEST INFRASTRUCTURE — the joint oracle: oracle/s2o_solver.c with every joint type the reference lacks (DESIGN.md §3.8 -
// §3.10, §3.14 - §3.19). The reference has none of these joints, so this file and the per-type files under
// tests/joint_oracle/ are their definition: plain, sequential C that the device must match bit for bit.
//
// It is built from oracle/s2o_solver.c unmodified, so that the revolute and mouse paths stay exactly the ones
// tests/test_oracle_cpu.py pins to the reference. Two oracle functions are routed to the dispatch at the end of this file
// by the preprocessor:
//   * s2oJointOp, the per-constraint dispatch of every driver;
//   * s2oPrepareJointSoft, which every joint prepare runs (the rigid and XPBD prepares call it first).
// Each macro pastes the first token of its first argument onto a prefix. A definition's first parameter starts with a
// type name (s2oSolve*, s2oJoint*), which selects the oracle's own function, renamed ..._Base; every call passes a
// plain variable (s, j), which selects the dispatch.
//
// Compiled with the oracle's flags (gcc -std=gnu17 -O2, no FMA contraction) by tests/joint_oracle.py.

#include "s2b_device.h"
#include "solver2d/constants.h"
#include "solver2d/math.h"

#include <stdlib.h>

struct s2oSolve;
struct s2oJoint;
struct s2oBody;
static void s2oJointDispatchOp(struct s2oSolve* s, int op, struct s2oJoint* j);
static void s2oJointDispatchPrepare(struct s2oJoint* j, const s2bJointRow* row, const struct s2oBody* bodies, float contextH,
									float h, float hertz, int warmStart);

#define s2oJointOp(first, ...) S2OJ_JOINT_OP_##first, __VA_ARGS__)
#define S2OJ_JOINT_OP_s2oSolve s2oJointOp_Base(s2oSolve
#define S2OJ_JOINT_OP_s s2oJointDispatchOp(s

#define s2oPrepareJointSoft(first, ...) S2OJ_PREPARE_##first, __VA_ARGS__)
#define S2OJ_PREPARE_s2oJoint s2oPrepareJointSoft_Base(s2oJoint
#define S2OJ_PREPARE_j s2oJointDispatchPrepare(j

#include "../oracle/s2o_solver.c"

#undef s2oJointOp
#undef s2oPrepareJointSoft

// each type's rows, in dependency order
#include "joint_oracle/weld.inc"
#include "joint_oracle/soft_weld.inc"
#include "joint_oracle/motor.inc"
#include "joint_oracle/prismatic.inc"
#include "joint_oracle/spring.inc"
#include "../solver2d_b200/csrc/shared/s2_collide.h"
#include "joint_oracle/distance.inc"
#include "joint_oracle/wheel.inc"
#include "../solver2d_b200/csrc/shared/s2_distance_joint.h"
#include "joint_oracle/pulley.inc"
#include "../solver2d_b200/csrc/shared/s2_gear_joint.h"
#include "joint_oracle/gear.inc"

// ---- per-slot state --------------------------------------------------------------------------------------------------

// What a joint keeps beside the oracle's joint struct, by joint slot. Every prepare resets its slot's record, so a reused
// slot never carries another type's state.
typedef struct s2oJointState
{
	s2oSpring spring; // a revolute or prismatic row's spring, a wheel's spring
	s2oSoftWeld softWeld;
	s2oDistance distance;
	s2oWheel wheel;
	s2oPulley pulley;
	s2oGear gear;
} s2oJointState;

static s2oJointState* s2oJointStates = NULL;
static int s2oJointStateCapacity = 0;

static s2oJointState* s2oJointStateOf(int slot)
{
	if (slot >= s2oJointStateCapacity)
	{
		int capacity = slot + 1 > 2 * s2oJointStateCapacity ? slot + 1 : 2 * s2oJointStateCapacity;
		s2oJointStates = (s2oJointState*)realloc(s2oJointStates, sizeof(s2oJointState) * (size_t)capacity);
		s2oJointStateCapacity = capacity;
	}
	return s2oJointStates + slot;
}

// ---- dispatch --------------------------------------------------------------------------------------------------------
//
// Prepare, every row: the base prepare (a gear row's of a copy that reads as a bare revolute row, for the anchors, masses
// and soft coefficients; the joint is then typed as a gear), then the spring's prepare, then the type's own:
//   revolute, mouse   nothing more
//   prismatic         the prismatic's impulse policy
//   weld              the weld's impulse policy, then the soft weld's parts
//   motor             the motor's impulse policy
//   distance, wheel, pulley, gear   their own prepare
//
// Ops:
//   revolute          the spring's row when it is active, then the base's
//   prismatic         the spring's row when it is active, then the prismatic's
//   weld              the soft weld's rows when either hertz is positive, otherwise the weld's
//   motor, distance, wheel, pulley, gear   their own rows
//   mouse             the base's
// An active spring's warm start replaces the joint's own (it adds the spring impulse to the axial sum).
//
// springImpulse: every row leaves prepare with its spring's impulse there, 0 for a row without an active spring (a mouse,
// weld, motor, pulley or gear row, and a revolute or prismatic row without the flag), as the device's s2bPrepareSpring
// leaves it. The distance and wheel prepares store their own spring's impulse, from the value the row came in with.

static void s2oJointDispatchPrepare(s2oJoint* j, const s2bJointRow* row, const s2oBody* bodies, float contextH, float h,
									float hertz, int warmStart)
{
	int type = s2bJointType(row->flags);
	float springImpulse = row->springImpulse;
	if (type == S2B_JOINT_GEAR)
	{
		s2bJointRow base = *row;
		base.flags = S2B_ROW_VALID;
		s2oPrepareJointSoft_Base(j, &base, bodies, contextH, h, hertz, warmStart);
		j->type = S2B_JOINT_GEAR;
	}
	else
	{
		s2oPrepareJointSoft_Base(j, row, bodies, contextH, h, hertz, warmStart);
	}

	s2oJointState* st = s2oJointStateOf(j->slot);
	*st = (s2oJointState){0};
	s2oSpringPrepare(&st->spring, j, row, contextH, warmStart);
	switch (type)
	{
		case S2B_JOINT_PRISMATIC:
			s2oPrismaticPrepare(j, row, warmStart);
			break;
		case S2B_JOINT_WELD:
			s2oWeldPrepare(j, row, warmStart);
			s2oSoftWeldPrepare(&st->softWeld, row, contextH);
			break;
		case S2B_JOINT_MOTOR:
			s2oMotorPrepare(j, row, warmStart);
			break;
		case S2B_JOINT_DISTANCE:
			s2oDistancePrepare(&st->distance, j, row, contextH, warmStart, springImpulse);
			break;
		case S2B_JOINT_WHEEL:
			s2oWheelPrepare(&st->wheel, &st->spring, j, row, contextH, warmStart, springImpulse);
			break;
		case S2B_JOINT_PULLEY:
			s2oPulleyPrepare(&st->pulley, j, row, bodies, warmStart);
			break;
		case S2B_JOINT_GEAR:
			s2oGearPrepare(&st->gear, j, row, bodies, warmStart);
			break;
		default:
			break;
	}
}

static void s2oJointDispatchOp(s2oSolve* s, int op, s2oJoint* j)
{
	s2oJointState* st = s2oJointStateOf(j->slot);
	switch (j->type)
	{
		case S2B_JOINT_REVOLUTE:
			if (st->spring.active == 0 || s2oSpringOp(s, op, j, &st->spring) == 0)
			{
				s2oJointOp_Base(s, op, j);
			}
			break;
		case S2B_JOINT_PRISMATIC:
			if (st->spring.active == 0 || s2oSpringOp(s, op, j, &st->spring) == 0)
			{
				s2oPrismaticOp(s, op, j);
			}
			break;
		case S2B_JOINT_WELD:
			if (st->softWeld.angular.active || st->softWeld.linear.active)
			{
				s2oSoftWeldOp(s, op, j, &st->softWeld);
			}
			else
			{
				s2oWeldOp(s, op, j);
			}
			break;
		case S2B_JOINT_MOTOR:
			s2oMotorOp(s, op, j);
			break;
		case S2B_JOINT_DISTANCE:
			s2oDistanceOp(s, op, j, &st->distance);
			break;
		case S2B_JOINT_WHEEL:
			s2oWheelOp(s, op, j, &st->wheel, &st->spring);
			break;
		case S2B_JOINT_PULLEY:
			s2oPulleyOp(s, op, j, &st->pulley);
			break;
		case S2B_JOINT_GEAR:
			s2oGearOp(s, op, j, &st->gear);
			break;
		default:
			s2oJointOp_Base(s, op, j);
			break;
	}
}
