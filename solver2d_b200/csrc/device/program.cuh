// solver2d-b200 — the vocabulary of solver PROGRAMS (passes and per-pass operations) and the per-variant dispatchers.
//
// Every solver variant is a short list of passes over bodies, joint constraints and contact constraints, built on the host
// from the variant's driver in the reference (buildProgram in solver.cu cites each one). The persistent kernel is
// instantiated once per variant: s2bUses*Op(SOLVER, op) prunes every operation the variant never schedules, so each
// instantiation only carries its own five or six per-constraint functions (registers and code size of the variant, not of
// the union of all ten). SOLVER = -1 keeps everything (the launch-by-launch cross-check kernels).
#pragma once

#include "joint_kernels.cuh"
#include "warm_gather.cuh"

// ---------------------------------------------------------------------------------------------------------------
// Programs: every solver variant is a short list of PASSES over bodies, joint constraints and contact constraints.
// The list is built on the host from the variant's driver in the reference (citations in buildProgram) and executed
// either by ONE persistent cooperative kernel (grid barrier after every dependent phase) or launch by launch.
// ---------------------------------------------------------------------------------------------------------------

enum PassKind
{
	PASS_BODY = 0,	// every body slot, no ordering
	PASS_FLAT = 1,	// every joint / contact constraint, no ordering between them (prepare, store)
	PASS_GROUP = 2, // Gauss-Seidel: groups in order, a barrier after each, then the serial overflow group
};

enum BodyOp
{
	BOP_NONE = 0,
	BOP_INTEGRATE_VELOCITIES,
	BOP_INTEGRATE_POSITIONS,
	BOP_FINALIZE_POSITIONS,
	BOP_JACOBI_RESET,
	BOP_JACOBI_APPLY,
	BOP_XPBD_INTEGRATE,
	BOP_XPBD_PROJECT,
	BOP_XPBD_FINALIZE,
	BOP_INTEGRATE_VELOCITIES_WARM,		 // s2IntegrateVelocities + warm start gathered per body (warm_gather.cuh)
	BOP_INTEGRATE_VELOCITIES_WARM_FIXED, // same with the prepare-time anchors of SoftStep
};

enum ContactOp
{
	COP_NONE = 0,
	COP_PREPARE,		// s2PrepareContacts_PGS / _Soft / local TGS_NGS flavour: same arithmetic, optional columns differ
	COP_PREPARE_COLD,	// XPBD: impulses always start at zero
	COP_PREPARE_STICKY,
	COP_PREPARE_BLOCK,
	COP_WARM_START,
	COP_WARM_START_FIXED,
	COP_TGS_SOFT_BIAS,
	COP_TGS_SOFT_RELAX,
	COP_PGS_BAUMGARTE,
	COP_PGS,
	COP_PGS_SOFT_BIAS,
	COP_PGS_SOFT_RELAX,
	COP_JACOBI_BIAS,
	COP_JACOBI_RELAX,
	COP_SOFTSTEP_BIAS,
	COP_SOFTSTEP_RELAX,
	COP_TGS,
	COP_NGS,
	COP_STICKY_BIAS,
	COP_STICKY_RELAX,
	COP_XPBD_POSITIONS,
	COP_XPBD_VELOCITIES,
	COP_BLOCK_VELOCITY,
	COP_BLOCK_POSITION,
	COP_STORE,
	COP_STORE_SCALED, // XPBD stores impulse * inv_h
	COP_TGS_SOFT_RELAX_STORE, // the LAST relax sweep of TGS_Soft: also writes the impulses to the manifolds (no separate store pass)
	COP_RESTITUTION,		  // the restitution pass (s2bApplyRestitution): only in the program of S2B_RESTITUTION_PROGRAM
};

enum JointOp
{
	JOP_NONE = 0,
	JOP_PREPARE_SOFT_WARM,	// s2PrepareJoint_Soft(..., warmStart = true)
	JOP_PREPARE_SOFT_FLAG,	// s2PrepareJoint_Soft(..., context->warmStart)
	JOP_PREPARE_RIGID_FLAG, // s2PrepareJoint(..., context->warmStart)
	JOP_PREPARE_RIGID_COLD, // s2PrepareJoint(..., false)
	JOP_PREPARE_XPBD,
	JOP_WARM_START,
	JOP_SOFT_BIAS,
	JOP_SOFT_RELAX,
	JOP_BAUMGARTE_BIAS,
	JOP_BAUMGARTE_RELAX,
	JOP_RIGID,
	JOP_POSITION,
	JOP_XPBD,
	JOP_STORE,
};

// The instantiation of the persistent kernel that runs the restitution pass after a variant's program (solver.cu): its
// program is one Gauss-Seidel pass of COP_RESTITUTION and it carries no other operation.
#define S2B_RESTITUTION_PROGRAM 10

struct PassDesc
{
	unsigned char kind, bodyOp, jointOp, contactOp;
};

#define S2B_MAX_SEGMENTS 6
#define S2B_MAX_SEGMENT_PASSES 8

// a program = segments executed in order, each a list of passes repeated `repeat` times
struct Program
{
	int segmentCount;
	int repeat[S2B_MAX_SEGMENTS];
	int passCount[S2B_MAX_SEGMENTS];
	PassDesc passes[S2B_MAX_SEGMENTS][S2B_MAX_SEGMENT_PASSES];
};

struct PassPtrs
{
	const int* jointSlots;
	const int* jPerm;
};

// which operations a variant's program can contain (s2bSolve verifies every built program against these tables)
__host__ __device__ constexpr bool s2bUsesBodyOp(int solver, int op)
{
	if (solver < 0)
	{
		return true;
	}
	if (solver == S2B_RESTITUTION_PROGRAM)
	{
		return false;
	}
	switch (op)
	{
		case BOP_INTEGRATE_VELOCITIES:
		case BOP_INTEGRATE_POSITIONS:
		case BOP_FINALIZE_POSITIONS:
			return solver != 9;
		case BOP_JACOBI_RESET:
		case BOP_JACOBI_APPLY:
			return solver == 0;
		case BOP_XPBD_INTEGRATE:
		case BOP_XPBD_PROJECT:
		case BOP_XPBD_FINALIZE:
			return solver == 9;
		case BOP_INTEGRATE_VELOCITIES_WARM:
			return solver == 7 || solver == 8;
		case BOP_INTEGRATE_VELOCITIES_WARM_FIXED:
			return solver == 5;
		default:
			return false;
	}
}

__host__ __device__ constexpr bool s2bUsesContactOp(int solver, int op)
{
	if (solver < 0)
	{
		return true;
	}
	if (solver == S2B_RESTITUTION_PROGRAM)
	{
		return op == COP_RESTITUTION;
	}
	switch (op)
	{
		case COP_PREPARE:
			return solver == 0 || solver == 1 || solver == 2 || solver == 4 || solver == 5 || solver == 7 || solver == 8;
		case COP_PREPARE_COLD:
			return solver == 9;
		case COP_PREPARE_STICKY:
			return solver == 6;
		case COP_PREPARE_BLOCK:
			return solver == 3;
		case COP_WARM_START:
			return solver == 0 || solver == 1 || solver == 2 || solver == 4 || solver == 7 || solver == 8;
		case COP_WARM_START_FIXED:
			return solver == 3 || solver == 5;
		case COP_TGS_SOFT_BIAS:
		case COP_TGS_SOFT_RELAX:
		case COP_TGS_SOFT_RELAX_STORE:
			return solver == 7;
		case COP_PGS_BAUMGARTE:
			return solver == 1;
		case COP_PGS:
			return solver == 2;
		case COP_PGS_SOFT_BIAS:
		case COP_PGS_SOFT_RELAX:
			return solver == 4;
		case COP_JACOBI_BIAS:
		case COP_JACOBI_RELAX:
			return solver == 0;
		case COP_SOFTSTEP_BIAS:
		case COP_SOFTSTEP_RELAX:
			return solver == 5;
		case COP_TGS:
			return solver == 8;
		case COP_NGS:
			return solver == 2 || solver == 8;
		case COP_STICKY_BIAS:
		case COP_STICKY_RELAX:
			return solver == 6;
		case COP_XPBD_POSITIONS:
		case COP_XPBD_VELOCITIES:
		case COP_STORE_SCALED:
			return solver == 9;
		case COP_BLOCK_VELOCITY:
		case COP_BLOCK_POSITION:
			return solver == 3;
		case COP_STORE:
			return solver != 9;
		default:
			return false;
	}
}

__host__ __device__ constexpr bool s2bUsesJointOp(int solver, int op)
{
	if (solver < 0)
	{
		return true;
	}
	if (solver == S2B_RESTITUTION_PROGRAM)
	{
		return false;
	}
	switch (op)
	{
		case JOP_PREPARE_SOFT_WARM:
			return solver == 5 || solver == 7;
		case JOP_PREPARE_SOFT_FLAG:
			return solver == 0 || solver == 4;
		case JOP_PREPARE_RIGID_FLAG:
			return solver == 1 || solver == 2 || solver == 3 || solver == 8;
		case JOP_PREPARE_RIGID_COLD:
			return solver == 6;
		case JOP_PREPARE_XPBD:
		case JOP_XPBD:
			return solver == 9;
		case JOP_WARM_START:
			return solver != 6 && solver != 9;
		case JOP_SOFT_BIAS:
		case JOP_SOFT_RELAX:
			return solver == 0 || solver == 4 || solver == 5 || solver == 7;
		case JOP_BAUMGARTE_BIAS:
			return solver == 1 || solver == 6;
		case JOP_BAUMGARTE_RELAX:
			return solver == 6;
		case JOP_RIGID:
		case JOP_POSITION:
			return solver == 2 || solver == 3 || solver == 8;
		case JOP_STORE:
			return true;
		default:
			return false;
	}
}

template <int SOLVER> __device__ __forceinline__ void s2bRunBodyOpT(int op, const SolveArgs& a, int i)
{
	switch (op)
	{
		case BOP_INTEGRATE_VELOCITIES:
			if constexpr (s2bUsesBodyOp(SOLVER, BOP_INTEGRATE_VELOCITIES))
			{
				s2bIntegrateVelocity(a, i, a.ctx.h);
			}
			break;
		case BOP_INTEGRATE_POSITIONS:
			if constexpr (s2bUsesBodyOp(SOLVER, BOP_INTEGRATE_POSITIONS))
			{
				s2bIntegratePosition(a, i, a.ctx.h);
			}
			break;
		case BOP_FINALIZE_POSITIONS:
			if constexpr (s2bUsesBodyOp(SOLVER, BOP_FINALIZE_POSITIONS))
			{
				s2bFinalizePosition(a, i);
			}
			break;
		case BOP_JACOBI_RESET:
			if constexpr (s2bUsesBodyOp(SOLVER, BOP_JACOBI_RESET))
			{
				s2bJacobiReset(a, i);
			}
			break;
		case BOP_JACOBI_APPLY:
			if constexpr (s2bUsesBodyOp(SOLVER, BOP_JACOBI_APPLY))
			{
				s2bJacobiApply(a, i);
			}
			break;
		case BOP_XPBD_INTEGRATE:
			if constexpr (s2bUsesBodyOp(SOLVER, BOP_XPBD_INTEGRATE))
			{
				s2bXpbdIntegrate(a, i, a.ctx.h);
			}
			break;
		case BOP_XPBD_PROJECT:
			if constexpr (s2bUsesBodyOp(SOLVER, BOP_XPBD_PROJECT))
			{
				s2bXpbdProjectVelocity(a, i, a.xpbdInvH);
			}
			break;
		case BOP_INTEGRATE_VELOCITIES_WARM:
			if constexpr (s2bUsesBodyOp(SOLVER, BOP_INTEGRATE_VELOCITIES_WARM))
			{
				s2bIntegrateVelocityWarm<false>(a, i, a.ctx.h);
			}
			break;
		case BOP_INTEGRATE_VELOCITIES_WARM_FIXED:
			if constexpr (s2bUsesBodyOp(SOLVER, BOP_INTEGRATE_VELOCITIES_WARM_FIXED))
			{
				s2bIntegrateVelocityWarm<true>(a, i, a.ctx.h);
			}
			break;
		case BOP_XPBD_FINALIZE:
			if constexpr (s2bUsesBodyOp(SOLVER, BOP_XPBD_FINALIZE))
			{
				s2bXpbdFinalize(a, i);
			}
			break;
		default:
			break;
	}
}


template <int SOLVER> __device__ __forceinline__ void s2bRunContactOpT(int op, const SolveArgs& a, int t)
{
	float inv_h = a.ctx.inv_h;
	switch (op)
	{
		case COP_PREPARE:
			if constexpr (s2bUsesContactOp(SOLVER, COP_PREPARE))
			{
				s2bPrepareContact<PREPARE_SOFT>(a, t);
			}
			break;
		case COP_PREPARE_COLD:
			if constexpr (s2bUsesContactOp(SOLVER, COP_PREPARE_COLD))
			{
				s2bPrepareContact<PREPARE_COLD>(a, t);
			}
			break;
		case COP_PREPARE_STICKY:
			if constexpr (s2bUsesContactOp(SOLVER, COP_PREPARE_STICKY))
			{
				s2bPrepareContactSticky(a, t);
			}
			break;
		case COP_PREPARE_BLOCK:
			if constexpr (s2bUsesContactOp(SOLVER, COP_PREPARE_BLOCK))
			{
				s2bPrepareContactBlock(a, t);
			}
			break;
		case COP_BLOCK_VELOCITY:
			if constexpr (s2bUsesContactOp(SOLVER, COP_BLOCK_VELOCITY))
			{
				s2bSolveContactBlockVelocity(a, t);
			}
			break;
		case COP_BLOCK_POSITION:
			if constexpr (s2bUsesContactOp(SOLVER, COP_BLOCK_POSITION))
			{
				s2bSolveContactBlockPosition(a, t);
			}
			break;
		case COP_WARM_START:
			if constexpr (s2bUsesContactOp(SOLVER, COP_WARM_START))
			{
				s2bWarmStartContact(a, t);
			}
			break;
		case COP_WARM_START_FIXED:
			if constexpr (s2bUsesContactOp(SOLVER, COP_WARM_START_FIXED))
			{
				s2bWarmStartContactFixed(a, t);
			}
			break;
		case COP_TGS_SOFT_BIAS:
			if constexpr (s2bUsesContactOp(SOLVER, COP_TGS_SOFT_BIAS))
			{
				s2bSolveContactTgsSoft(a, t, inv_h, true, a.ctx.extraIterations == 0);
			}
			break;
		case COP_TGS_SOFT_RELAX:
			if constexpr (s2bUsesContactOp(SOLVER, COP_TGS_SOFT_RELAX))
			{
				s2bSolveContactTgsSoft(a, t, inv_h, false, true);
			}
			break;
		case COP_TGS_SOFT_RELAX_STORE:
			if constexpr (s2bUsesContactOp(SOLVER, COP_TGS_SOFT_RELAX_STORE))
			{
				s2bSolveContactTgsSoft(a, t, inv_h, false, true, true);
			}
			break;
		case COP_PGS_BAUMGARTE:
			if constexpr (s2bUsesContactOp(SOLVER, COP_PGS_BAUMGARTE))
			{
				s2bSolveContactFixed<0>(a, t, inv_h, true);
			}
			break;
		case COP_PGS:
			if constexpr (s2bUsesContactOp(SOLVER, COP_PGS))
			{
				s2bSolveContactPgs(a, t);
			}
			break;
		case COP_PGS_SOFT_BIAS:
			if constexpr (s2bUsesContactOp(SOLVER, COP_PGS_SOFT_BIAS))
			{
				s2bSolveContactFixed<1>(a, t, inv_h, true);
			}
			break;
		case COP_PGS_SOFT_RELAX:
			if constexpr (s2bUsesContactOp(SOLVER, COP_PGS_SOFT_RELAX))
			{
				s2bSolveContactFixed<1>(a, t, inv_h, false);
			}
			break;
		case COP_JACOBI_BIAS:
			if constexpr (s2bUsesContactOp(SOLVER, COP_JACOBI_BIAS))
			{
				s2bSolveContactFixed<2>(a, t, inv_h, true);
			}
			break;
		case COP_JACOBI_RELAX:
			if constexpr (s2bUsesContactOp(SOLVER, COP_JACOBI_RELAX))
			{
				s2bSolveContactFixed<2>(a, t, inv_h, false);
			}
			break;
		case COP_SOFTSTEP_BIAS:
			if constexpr (s2bUsesContactOp(SOLVER, COP_SOFTSTEP_BIAS))
			{
				s2bSolveContactSubstep<0>(a, t, inv_h, true, a.ctx.extraIterations == 0);
			}
			break;
		case COP_SOFTSTEP_RELAX:
			if constexpr (s2bUsesContactOp(SOLVER, COP_SOFTSTEP_RELAX))
			{
				s2bSolveContactSubstep<0>(a, t, inv_h, false, true);
			}
			break;
		case COP_TGS:
			if constexpr (s2bUsesContactOp(SOLVER, COP_TGS))
			{
				s2bSolveContactSubstep<1>(a, t, inv_h, true, true);
			}
			break;
		case COP_NGS:
			if constexpr (s2bUsesContactOp(SOLVER, COP_NGS))
			{
				s2bSolveContactNgs(a, t);
			}
			break;
		case COP_STICKY_BIAS:
			if constexpr (s2bUsesContactOp(SOLVER, COP_STICKY_BIAS))
			{
				s2bSolveContactSticky(a, t, inv_h, true);
			}
			break;
		case COP_STICKY_RELAX:
			if constexpr (s2bUsesContactOp(SOLVER, COP_STICKY_RELAX))
			{
				s2bSolveContactSticky(a, t, inv_h, false);
			}
			break;
		case COP_XPBD_POSITIONS:
			if constexpr (s2bUsesContactOp(SOLVER, COP_XPBD_POSITIONS))
			{
				s2bSolveContactXpbdPositions(a, t, a.ctx.h);
			}
			break;
		case COP_XPBD_VELOCITIES:
			if constexpr (s2bUsesContactOp(SOLVER, COP_XPBD_VELOCITIES))
			{
				s2bSolveContactXpbdVelocities(a, t, a.ctx.h);
			}
			break;
		case COP_STORE:
			if constexpr (s2bUsesContactOp(SOLVER, COP_STORE))
			{
				s2bStoreContactImpulses(a, t, 1.0f);
			}
			break;
		case COP_STORE_SCALED:
			if constexpr (s2bUsesContactOp(SOLVER, COP_STORE_SCALED))
			{
				s2bStoreContactImpulses(a, t, a.xpbdInvH);
			}
			break;
		case COP_RESTITUTION:
			if constexpr (s2bUsesContactOp(SOLVER, COP_RESTITUTION))
			{
				s2bApplyRestitution(a, t);
			}
			break;
		default:
			break;
	}
}


template <int SOLVER> __device__ __forceinline__ void s2bRunJointOpT(int op, const SolveArgs& a, int t, const PassPtrs& p)
{
	switch (op)
	{
		case JOP_PREPARE_SOFT_WARM:
			if constexpr (s2bUsesJointOp(SOLVER, JOP_PREPARE_SOFT_WARM))
			{
				s2bPrepareJoint<JPREP_SOFT>(a, t, p.jointSlots[p.jPerm[t]], true);
			}
			break;
		case JOP_PREPARE_SOFT_FLAG:
			if constexpr (s2bUsesJointOp(SOLVER, JOP_PREPARE_SOFT_FLAG))
			{
				s2bPrepareJoint<JPREP_SOFT>(a, t, p.jointSlots[p.jPerm[t]], a.ctx.warmStart != 0);
			}
			break;
		case JOP_PREPARE_RIGID_FLAG:
			if constexpr (s2bUsesJointOp(SOLVER, JOP_PREPARE_RIGID_FLAG))
			{
				s2bPrepareJoint<JPREP_RIGID>(a, t, p.jointSlots[p.jPerm[t]], a.ctx.warmStart != 0);
			}
			break;
		case JOP_PREPARE_RIGID_COLD:
			if constexpr (s2bUsesJointOp(SOLVER, JOP_PREPARE_RIGID_COLD))
			{
				s2bPrepareJoint<JPREP_RIGID>(a, t, p.jointSlots[p.jPerm[t]], false);
			}
			break;
		case JOP_PREPARE_XPBD:
			if constexpr (s2bUsesJointOp(SOLVER, JOP_PREPARE_XPBD))
			{
				s2bPrepareJoint<JPREP_XPBD>(a, t, p.jointSlots[p.jPerm[t]], false);
			}
			break;
		case JOP_WARM_START:
			if constexpr (s2bUsesJointOp(SOLVER, JOP_WARM_START))
			{
				s2bWarmStartJoint(a, t);
			}
			break;
		case JOP_SOFT_BIAS:
			if constexpr (s2bUsesJointOp(SOLVER, JOP_SOFT_BIAS))
			{
				s2bSolveJointSoft<(SOLVER >= 0)>(a, t, a.ctx.h, a.ctx.inv_h, true);
			}
			break;
		case JOP_SOFT_RELAX:
			if constexpr (s2bUsesJointOp(SOLVER, JOP_SOFT_RELAX))
			{
				s2bSolveJointSoft<(SOLVER >= 0)>(a, t, a.ctx.h, a.ctx.inv_h, false);
			}
			break;
		case JOP_BAUMGARTE_BIAS:
			if constexpr (s2bUsesJointOp(SOLVER, JOP_BAUMGARTE_BIAS))
			{
				s2bSolveJointBaumgarte(a, t, a.ctx.h, a.ctx.inv_h, true);
			}
			break;
		case JOP_BAUMGARTE_RELAX:
			if constexpr (s2bUsesJointOp(SOLVER, JOP_BAUMGARTE_RELAX))
			{
				s2bSolveJointBaumgarte(a, t, a.ctx.h, a.ctx.inv_h, false);
			}
			break;
		case JOP_RIGID:
			if constexpr (s2bUsesJointOp(SOLVER, JOP_RIGID))
			{
				s2bSolveJointRigid(a, t, a.ctx.h);
			}
			break;
		case JOP_POSITION:
			if constexpr (s2bUsesJointOp(SOLVER, JOP_POSITION))
			{
				s2bSolveJointPosition(a, t);
			}
			break;
		case JOP_XPBD:
			if constexpr (s2bUsesJointOp(SOLVER, JOP_XPBD))
			{
				s2bSolveJointXpbd(a, t);
			}
			break;
		case JOP_STORE:
			if constexpr (s2bUsesJointOp(SOLVER, JOP_STORE))
			{
				s2bStoreJointImpulses(a, t);
			}
			break;
		default:
			break;
	}
}


// everything (launch-by-launch kernels, serial cross-checks)
__device__ __forceinline__ void s2bRunBodyOp(int op, const SolveArgs& a, int i)
{
	s2bRunBodyOpT<-1>(op, a, i);
}

__device__ __forceinline__ void s2bRunContactOp(int op, const SolveArgs& a, int t)
{
	s2bRunContactOpT<-1>(op, a, t);
}

__device__ __forceinline__ void s2bRunJointOp(int op, const SolveArgs& a, int t, const PassPtrs& p)
{
	s2bRunJointOpT<-1>(op, a, t, p);
}
