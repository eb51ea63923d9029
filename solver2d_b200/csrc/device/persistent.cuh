// solver2d-b200 — the persistent cooperative solver kernel: one launch executes a variant's whole program (prepare ...
// store) for one step. Instantiated once per solver variant (program.cuh prunes the operations a variant never uses).
//
// REGION-LOCAL SCHEDULE (DESIGN.md §3.1). A dependent colour step costs about as much as the device-wide barrier
// behind it whatever it holds (tools/barrier_lab.cu; not measured on H100), so what bounds a 100 k-body scene is the NUMBER of device-wide steps,
// not bytes. The bodies are therefore partitioned into one spatially compact REGION per thread block (Hilbert order,
// solver.cu). A constraint whose movable bodies all belong to one region is INTERIOR to it: the block that owns the region
// runs the interior constraints of ALL colours with __syncthreads() between colours — no other block touches those bodies.
// Only the constraints that straddle two regions (the CUT set, a few per cent, coloured among themselves into a handful
// of cut colours) run as device-wide steps. One Gauss-Seidel sweep costs 1 + (cut colours) grid barriers instead of one
// per colour, and body passes (integrate, finalize, warm-start gather) are region-local as well.
// The serial order this corresponds to — region by region, colour by colour inside a region, then the cut colours, then
// the serial overflow group — is what s2b_download_solve_order reports and the order-permuted oracle replays bit for bit.
#pragma once

#include "program.cuh"

// Shared-memory staging of the serial overflow group (block 0 only; dynamic shared memory of the kernel): the bodies its
// constraints touch — a hub such as a container wall plus everything resting against it — and the body indices of its
// rows re-mapped to that staging. The serial walk then runs at shared-memory latency instead of an L2 round trip per
// body access (every item reads the hub's velocity the previous item has just written).
#define S2B_OV_MAX_BODIES 1024
#define S2B_OV_MAX_CONTACTS 2048
#define S2B_OV_MAX_JOINTS 256
#define S2B_OV_SHARED_BYTES (S2B_OV_MAX_BODIES * 48 + S2B_OV_MAX_CONTACTS * 8 + S2B_OV_MAX_JOINTS * 16)
// Resident regions: when nothing has to be solved device-wide (no cut set, no overflow group, no hub, no joints — batched
// independent worlds, a small scene) every block keeps the velocity and pose rows of its region's bodies in shared memory from
// prepare to finalize: 32 B per body in the same dynamic shared memory (the overflow staging is not needed then).
#define S2B_RES_MAX_BODIES 3072
#define S2B_RES_SHARED_BYTES (S2B_RES_MAX_BODIES * 32)
#define S2B_DYN_SHARED_BYTES (S2B_RES_SHARED_BYTES > S2B_OV_SHARED_BYTES ? S2B_RES_SHARED_BYTES : S2B_OV_SHARED_BYTES)

// stride of the per-region offset tables: entry c = first stream row of (region, colour c), entry S2B_MAX_COLORS = end
#define S2B_REG_STRIDE (S2B_MAX_COLORS + 1)

// ---- diagnostics -------------------------------------------------------------------------------------------------

// time stamps (s2b_set_solve_trace): code = what just finished (pass kind << 8 | op), stamped by one thread
__device__ __forceinline__ void s2bTrace(const SolveArgs& a, int code)
{
	if (a.trace != nullptr && blockIdx.x == 0 && threadIdx.x == 0)
	{
		unsigned long long now;
		asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
		unsigned long long n = a.trace[0];
		if ((int)n + 1 < a.traceCap)
		{
			a.trace[1 + n] = ((unsigned long long)code << 48) | (now & 0xFFFFFFFFFFFFull);
			a.trace[0] = n + 1;
		}
	}
}

// ---- synchronisation ---------------------------------------------------------------------------------------------
// Grid barrier on a monotonic arrival counter: one red.release per block, thread 0 polls with ld.acquire (which also
// invalidates the SM's L1: CCTL.IVALL), __syncthreads() on both sides. Compared with cooperative_groups' grid.sync()
// in tools/barrier_lab.cu: same bare cost, less per dependent colour step (not measured on H100). The counter is never
// reset: every launch starts from the base the previous launch left in barrier[32].

struct S2bSync
{
	unsigned base;	   // arrival count at kernel start
	unsigned arrivals; // arrivals expected since then (barriers passed x blocks)
	int pending;	   // what ran since the last synchronisation: 0 nothing, 1 region-local work, 2 device-wide work
	int code;		   // trace code of the last phase executed (pass kind << 8 | op; kind byte bit 7: device-wide step, bits 7+6:
					   // overflow group, bit 6 alone: neighbour-synchronised colour step)
};

#define S2B_PENDING_NONE 0
#define S2B_PENDING_LOCAL 1
#define S2B_PENDING_GLOBAL 2
#define S2B_PENDING_FLOW 3 // a ticketed pass: orders itself against the next ticketed pass, anything else needs the barrier
#define S2B_PENDING_NEIGHBOURS 4 // a neighbour-synchronised colour step: orders itself against the next one, anything else needs the barrier

__device__ __forceinline__ unsigned s2bLdAcquireU32(const unsigned* p)
{
	unsigned v;
	asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
	return v;
}

__device__ __forceinline__ void s2bGridBarrier(const SolveArgs& a, S2bSync& s)
{
	__syncthreads();
	if (gridDim.x > 1)
	{
		s.arrivals += gridDim.x;
		if (threadIdx.x == 0)
		{
			asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(a.barrier), "r"(1u) : "memory");
			unsigned target = s.base + s.arrivals;
			while ((int)(s2bLdAcquireU32(a.barrier) - target) < 0)
			{
			}
		}
		__syncthreads();
	}
	s.pending = S2B_PENDING_NONE;
}

// before region-local work: data of this block's region only — written by this block (block barrier) unless a device-wide
// phase ran in between
__device__ __forceinline__ void s2bSyncBeforeLocal(const SolveArgs& a, S2bSync& s)
{
	if (s.pending == S2B_PENDING_GLOBAL || s.pending == S2B_PENDING_NEIGHBOURS)
	{
		s2bGridBarrier(a, s);
		s2bTrace(a, s.code);
	}
	else if (s.pending == S2B_PENDING_LOCAL)
	{
		__syncthreads();
	}
}

__device__ __forceinline__ void s2bSyncBeforeGlobal(const SolveArgs& a, S2bSync& s)
{
	if (s.pending != S2B_PENDING_NONE)
	{
		s2bGridBarrier(a, s);
		s2bTrace(a, s.code);
	}
}

// ---- neighbour-synchronised colour steps (DESIGN.md §3.1) -----------------------------------------------------------
// Block b runs the b-th share of every device-wide colour (s2bGroupShare). Two blocks are neighbours when constraints they
// run share a movable body (solver.cu, s2bBlockEdgesKernel). Between two colour steps a block therefore only has to wait for
// its neighbours to finish the previous step, not for the whole grid: each block owns an epoch word (one 128-byte line),
// counts its neighbour-synchronised steps in it with a release store, and before step e waits with acquire loads until every
// neighbour has published e - 1 (the acquire also invalidates the SM's L1, as the grid barrier's does). Body passes, flat
// passes and the overflow group still take the grid barrier (`pending` says a neighbour step ran).
// Why the order is the serial one: any two constraints that share a movable body run on the same block or on neighbours, so
// every read-after-write and write-after-read between colours is ordered by the epochs; inside a colour no two constraints
// share a movable body, so they commute.
// Why it cannot deadlock: the launch is cooperative (every block is resident), every block runs the same steps, and a block
// only ever waits for a neighbour (a symmetric relation) to reach an epoch lower than the one it is about to publish. The block
// whose published epoch is the smallest therefore always finds its wait satisfied and moves on.
// Epochs are monotonic across launches (as barrier[0]): every block of a launch publishes the same sequence base + 1, base + 2,
// ..., and block 0 leaves the final value in barrier[S2B_EPOCH_BASE_WORD] for the next launch (the restitution kernel
// continues it). A block the previous launches did not run holds an older, smaller value, which no wait accepts.

// sNbr: the block's neighbour count, its neighbours, then (S2B_NBR_EPOCH) the epoch of its last colour step, written by thread 0
// only (kept in shared memory rather than in every thread's registers: only warp 0 reads it)
#define S2B_NBR_EPOCH S2B_NSYNC_STRIDE

__device__ __forceinline__ void s2bNeighbourWait(const SolveArgs& a, S2bSync& s, int* sNbr)
{
	// lanes 0 .. n-1 of warp 0 poll one neighbour each, all at once
	__syncwarp();
	if (threadIdx.x < sNbr[0])
	{
		const unsigned* flag = a.barrier + S2B_EPOCH_WORD(sNbr[1 + threadIdx.x]);
		unsigned epoch = (unsigned)sNbr[S2B_NBR_EPOCH];
		while ((int)(s2bLdAcquireU32(flag) - epoch) < 0)
		{
		}
	}
	__syncthreads();
	s2bTrace(a, s.code);
}

// the colour step is done in this block: publish its epoch
__device__ __forceinline__ void s2bPublishEpoch(const SolveArgs& a, S2bSync& s, int* sNbr)
{
	__syncthreads();
	if (threadIdx.x == 0)
	{
		unsigned epoch = (unsigned)sNbr[S2B_NBR_EPOCH] + 1u;
		sNbr[S2B_NBR_EPOCH] = (int)epoch;
		asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(a.barrier + S2B_EPOCH_WORD(blockIdx.x)), "r"(epoch) : "memory");
	}
	s.pending = S2B_PENDING_NEIGHBOURS;
}

// ---- passes ------------------------------------------------------------------------------------------------------

// what does not change during the launch, read once
struct S2bLaunchInfo
{
	int nJ, nC;		  // live joint / contact constraints
	int primary;	  // colours used inside regions
	int groups;		  // device-wide groups: cut colours (colour schedule) or wavefront levels
	int ovJ, ovC;	  // serial overflow group
	int hubs;		  // hub bodies (body passes run over them grid-wide)
	int bodyBegin, bodyEnd; // this block's range of regBodies
	bool regions;
	bool neighbours;	// device-wide colour steps are neighbour-synchronised (grid-uniform)
	bool foldPositions; // TGS_Soft: the bias sweep integrates positions (ConstraintView::lastTouch), the body pass is skipped
	bool firstTouch;	// TGS_Soft, with foldPositions: the bias sweep also warm-starts velocities (S2B_TOUCH_FIRST_*), the
						// warm-start body pass is skipped and finalize sub-steps the bodies without constraints
	bool resident;		// TGS_Soft: the region's velocity / pose rows live in shared memory for the whole launch
};

template <int SOLVER> __device__ __forceinline__ void s2bBodyPass(int bodyOp, const SolveArgs& a, const S2bLaunchInfo& li)
{
	if (li.regions)
	{
		for (int k = li.bodyBegin + threadIdx.x; k < li.bodyEnd; k += blockDim.x)
		{
			s2bRunBodyOpT<SOLVER>(bodyOp, a, a.regBodies[k]);
		}
		if (li.hubs > 0)
		{
			// hub bodies belong to no region: all their constraints are in the cut set, so nothing region-local touches them
			if (s2bUsesBodyOp(SOLVER, BOP_INTEGRATE_VELOCITIES_WARM) && bodyOp == BOP_INTEGRATE_VELOCITIES_WARM)
			{
				s2bGatherHeavyBodies<false>(a, a.ctx.h);
			}
			else if (s2bUsesBodyOp(SOLVER, BOP_INTEGRATE_VELOCITIES_WARM_FIXED) && bodyOp == BOP_INTEGRATE_VELOCITIES_WARM_FIXED)
			{
				s2bGatherHeavyBodies<true>(a, a.ctx.h);
			}
			else
			{
				int stride = gridDim.x * blockDim.x;
				for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < li.hubs; k += stride)
				{
					s2bRunBodyOpT<SOLVER>(bodyOp, a, a.heavyBodies[1 + k]);
				}
			}
		}
		return;
	}
	if (s2bUsesBodyOp(SOLVER, BOP_INTEGRATE_VELOCITIES_WARM) && bodyOp == BOP_INTEGRATE_VELOCITIES_WARM)
	{
		s2bIntegrateVelocityWarmAll<false>(a, a.ctx.h, li.foldPositions);
	}
	else if (s2bUsesBodyOp(SOLVER, BOP_INTEGRATE_VELOCITIES_WARM_FIXED) && bodyOp == BOP_INTEGRATE_VELOCITIES_WARM_FIXED)
	{
		s2bIntegrateVelocityWarmAll<true>(a, a.ctx.h);
	}
	else
	{
		int stride = gridDim.x * blockDim.x;
		for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.bodies.capacity; i += stride)
		{
			if (SOLVER == 7 && li.firstTouch && bodyOp == BOP_FINALIZE_POSITIONS)
			{
				// (no warm-start pass ran: the sub-steps of a body without constraints are still owed)
				s2bSubstepFreeBody(a, i, a.ctx.h, a.ctx.iterations);
			}
			s2bRunBodyOpT<SOLVER>(bodyOp, a, i);
		}
	}
	if (a.heavyBodies != nullptr)
	{
		if (s2bUsesBodyOp(SOLVER, BOP_INTEGRATE_VELOCITIES_WARM) && bodyOp == BOP_INTEGRATE_VELOCITIES_WARM)
		{
			s2bGatherHeavyBodies<false>(a, a.ctx.h);
		}
		else if (s2bUsesBodyOp(SOLVER, BOP_INTEGRATE_VELOCITIES_WARM_FIXED) && bodyOp == BOP_INTEGRATE_VELOCITIES_WARM_FIXED)
		{
			s2bGatherHeavyBodies<true>(a, a.ctx.h);
		}
	}
}

template <int SOLVER>
__device__ __forceinline__ void s2bFlatPass(int jointOp, int contactOp, const SolveArgs& a, const PassPtrs& p, const S2bLaunchInfo& li)
{
	int stride = gridDim.x * blockDim.x;
	for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < li.nJ + li.nC; t += stride)
	{
		if (t < li.nJ)
		{
			if (jointOp != JOP_NONE)
			{
				s2bRunJointOpT<SOLVER>(jointOp, a, t, p);
			}
		}
		else if (contactOp != COP_NONE)
		{
			s2bRunContactOpT<SOLVER>(contactOp, a, t - li.nJ);
		}
	}
}

// L1 warm-up for the serial overflow walk: request (prefetch.global.L1) every line an op on this constraint may read
__device__ __forceinline__ void s2bPrefetchL1(const void* ptr)
{
	asm volatile("prefetch.global.L1 [%0];" ::"l"(ptr));
}

// ---- block-wide first-touch warm start (TGS_Soft bias sweep, colour 0; DESIGN.md §3.1 (d)) -----------------------------
// Nearly every body is first touched in colour 0, so in that step nearly every thread gathered two bodies after the wait:
// per body its head, its incidence entries and both 16-byte warm rows of every entry, about 220 KB per block from L2 in every
// sub-step. Instead, the bodies a block's share of colour 0 first-touches come from a table built with the schedule
// (ConstraintView::firstTable, solver.cu s2bFirstTable*Kernel), and what the launch does not change is kept in dynamic shared
// memory for the whole launch: incidence entries, flags, parameters and forces from the start, and the entries' anchors
// (warmAnchor, which a rebuild step's prepare pass writes) from the first colour-0 step on, behind its synchronisation. After the
// wait only the velocity and pose of every body and the impulse row of every entry come from L2, and one thread per body runs
// the unchanged gather, s2bIntegrateVelocityWarmHead: the same operations in the same order, hence the same bits as the
// per-thread gather, which a block whose copy is over budget keeps (both paths mix in one launch). That memory is otherwise
// only used by resident regions and the overflow staging, and neither runs with the first-touch warm start.
#define S2B_FT_SHARED_BYTES (144 * 1024)
// dynamic shared memory a launch of the persistent kernel may ask for
#define S2B_SOLVE_SHARED_MAX (S2B_FT_SHARED_BYTES > S2B_DYN_SHARED_BYTES ? S2B_FT_SHARED_BYTES : S2B_DYN_SHARED_BYTES)

struct S2bFirstTableShared
{
	float4* prm;
	float4* frc;
	int4* info;		 // body, flags, begin, end (entries of the block's copy)
	float4* anchors; // per entry: warmAnchor of its constraint and side
	int* entries;
};

__device__ __forceinline__ S2bFirstTableShared s2bFirstTableLayout(int slots, int entries)
{
	extern __shared__ __align__(16) unsigned char s2bFtShared[];
	S2bFirstTableShared L;
	L.prm = reinterpret_cast<float4*>(s2bFtShared);
	L.frc = L.prm + slots;
	L.info = reinterpret_cast<int4*>(L.frc + slots);
	L.anchors = reinterpret_cast<float4*>(L.info + slots);
	L.entries = reinterpret_cast<int*>(L.anchors + entries);
	return L;
}

// once per launch (every thread of the block): sFt[0] = the block's slots (-1: it gathers per thread), sFt[1] = its entries,
// sFt[2] = 0: the anchors are not staged yet
__device__ __forceinline__ void s2bFirstTableStage(const SolveArgs& a, int* sFt)
{
	const int* table = a.cc.firstTable;
	int4 hd = reinterpret_cast<const int4*>(table)[blockIdx.x];
	int slots = hd.y;
	int base = slots >= 0 ? table[hd.z] : 0;
	int entries = slots >= 0 ? table[hd.z + slots] - base : 0;
	if (threadIdx.x == 0)
	{
		sFt[0] = slots;
		sFt[1] = entries;
		sFt[2] = 0;
	}
	S2bFirstTableShared L = s2bFirstTableLayout(max(slots, 0), entries);
	for (int k = threadIdx.x; k < slots; k += blockDim.x)
	{
		int i = table[hd.x + k];
		L.prm[k] = a.bodies.prm[i];
		L.frc[k] = a.bodies.frc[i];
		L.info[k] = make_int4(i, (int)a.bodies.flags[i], table[hd.z + k] - base, table[hd.z + k + 1] - base);
	}
	for (int j = threadIdx.x; j < entries; j += blockDim.x)
	{
		L.entries[j] = table[hd.w + j];
	}
}

// after the synchronisation of the bias sweep's colour-0 step: s2IntegrateVelocities + the warm start of every body of the
// block's table (every thread of the block; ends with the block barrier the solves need)
__device__ __forceinline__ void s2bFirstTableGather(const SolveArgs& a, int* sFt)
{
	int slots = sFt[0], entries = sFt[1];
	S2bFirstTableShared L = s2bFirstTableLayout(slots, entries);
	if (sFt[2] == 0)
	{
		// (the first colour-0 step of the launch: prepare, if it ran, is behind the grid barrier just taken)
		for (int j = threadIdx.x; j < entries; j += blockDim.x)
		{
			int e = L.entries[j];
			L.anchors[j] = (e & S2B_INC_CONTACT) ? a.cc.warmAnchor[(size_t)(e >> 2) * 2 + ((e & S2B_INC_SIDE_B) ? 1 : 0)] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		}
		__syncthreads();
		if (threadIdx.x == 0)
		{
			sFt[2] = 1;
		}
	}
	for (int k = threadIdx.x; k < slots; k += blockDim.x)
	{
		int4 info = L.info[k];
		GatherHead hd;
		hd.f = (unsigned)info.y;
		hd.vel = a.bodies.vel[info.x];
		hd.prm = L.prm[k];
		hd.frc = L.frc[k];
		hd.pose = a.bodies.pose[info.x];
		hd.begin = info.z;
		hd.end = info.w;
		s2bIntegrateVelocityWarmHead<false>(a, info.x, a.ctx.h, hd, false, nullptr, L.entries, L.anchors);
	}
	__syncthreads();
}

// the TGS_Soft row of a contact constraint (what s2bLoadContactStream reads)
__device__ __forceinline__ void s2bTouchContactRow(const SolveArgs& a, int t)
{
	s2bPrefetchL1(a.cc.idx + t);
	s2bPrefetchL1(a.cc.nf + t);
	s2bPrefetchL1(a.cc.anchor[0] + t);
	s2bPrefetchL1(a.cc.pm[0] + t);
	s2bPrefetchL1(a.cc.lambda[0] + t);
	s2bPrefetchL1(a.cc.anchor[1] + t);
	s2bPrefetchL1(a.cc.pm[1] + t);
	s2bPrefetchL1(a.cc.lambda[1] + t);
}

// ---- resident regions (TGS_Soft) -------------------------------------------------------------------------------------
// sVel / sPose = the region's copy; body k of the region is body slot regBodies[bodyBegin + k] of the world.

// body passes of the TGS_Soft program on the region's copy
__device__ __forceinline__ void s2bResidentBodyPass(int bodyOp, const SolveArgs& a, const S2bLaunchInfo& li, float4* sVel, float4* sPose)
{
	int nb = li.bodyEnd - li.bodyBegin;
	for (int k = threadIdx.x; k < nb; k += blockDim.x)
	{
		int i = a.regBodies[li.bodyBegin + k];
		if (bodyOp == BOP_INTEGRATE_VELOCITIES_WARM)
		{
			GatherHead hd;
			hd.f = a.bodies.flags[i];
			hd.prm = a.bodies.prm[i];
			hd.frc = a.bodies.frc[i];
			hd.begin = a.incStart[i];
			hd.end = a.incStart[i + 1];
			hd.vel = sVel[k];
			hd.pose = sPose[k];
			s2bIntegrateVelocityWarmHead<false>(a, i, a.ctx.h, hd, false, sVel + k);
		}
		else if (bodyOp == BOP_INTEGRATE_POSITIONS)
		{
			// s2IntegratePositions (reference src/solve_common.c:47-68)
			unsigned f = a.bodies.flags[i];
			if ((f & S2B_BODY_VALID) != 0 && S2B_BODY_TYPE(f) != S2B_BODY_STATIC)
			{
				float4 vel = sVel[k];
				float4 pose = sPose[k];
				s2Vec2 dp = s2MulAdd(V2(pose.x, pose.y), a.ctx.h, V2(vel.x, vel.y));
				s2Rot q = s2IntegrateRot(R2(pose.z, pose.w), a.ctx.h * vel.z);
				sPose[k] = make_float4(dp.x, dp.y, q.s, q.c);
			}
		}
		else if (bodyOp == BOP_FINALIZE_POSITIONS)
		{
			// s2FinalizePositions (reference src/solve_common.c:70-91) + the copy goes home
			unsigned f = a.bodies.flags[i];
			if ((f & S2B_BODY_VALID) != 0 && S2B_BODY_TYPE(f) != S2B_BODY_STATIC)
			{
				float4 pos = a.bodies.pos[i];
				float4 pose = sPose[k];
				s2Vec2 pn = s2Add(V2(pos.x, pos.y), V2(pose.x, pose.y));
				a.bodies.pos[i] = make_float4(pn.x, pn.y, pos.z, pos.w);
				a.bodies.pose[i] = make_float4(0.0f, 0.0f, pose.z, pose.w);
				a.bodies.vel[i] = sVel[k];
			}
		}
	}
}

// one Gauss-Seidel sweep over the region's constraints, colour by colour, on the region's copy
template <int SOLVER>
__device__ __forceinline__ void s2bResidentSweep(int contactOp, const SolveArgs& a, float4* sVel, float4* sPose, const S2bLaunchInfo& li,
												 const int* sRegC)
{
	bool store = contactOp == COP_TGS_SOFT_RELAX_STORE;
	bool bias = contactOp == COP_TGS_SOFT_BIAS;
	bool writeWarm = bias ? a.ctx.extraIterations == 0 : true;
	bool first = true;
	for (int c = 0; c < li.primary; ++c)
	{
		int cBegin = sRegC[c];
		int nc = sRegC[c + 1] - cBegin;
		if (nc == 0)
		{
			continue; // uniform within the block
		}
		int t = threadIdx.x;
		if (t < nc)
		{
			s2bTouchContactRow(a, cBegin + t);
		}
		if (first == false)
		{
			__syncthreads();
		}
		first = false;
		for (; t < nc; t += blockDim.x)
		{
			if (t + (int)blockDim.x < nc)
			{
				s2bTouchContactRow(a, cBegin + t + blockDim.x);
			}
			ContactStream cs = s2bLoadContactStream(a, cBegin + t, store);
			s2bSolveContactTgsSoftStream<true>(a, cBegin + t, cs, a.ctx.inv_h, bias, writeWarm, store, a.bodies.vel, a.bodies.pose, sVel, sPose);
		}
	}
}

__device__ __forceinline__ void s2bTouchBody(const SolveArgs& a, int i)
{
	s2bPrefetchL1(a.bodies.vel + i);
	s2bPrefetchL1(a.bodies.pose + i);
	s2bPrefetchL1(a.bodies.pos + i);
	if (a.bodies.aux0 != nullptr)
	{
		s2bPrefetchL1(a.bodies.aux0 + i);
	}
}

__device__ __forceinline__ void s2bTouchContact(const SolveArgs& a, int t, bool bodies = true)
{
	int2 idx = a.cc.idx[t];
	s2bPrefetchL1(a.cc.nf + t);
	s2bPrefetchL1(a.cc.src + t);
#pragma unroll
	for (int j = 0; j < 2; ++j)
	{
		s2bPrefetchL1(a.cc.anchor[j] + t);
		s2bPrefetchL1(a.cc.pm[j] + t);
		s2bPrefetchL1(a.cc.lambda[j] + t);
		if (a.cc.r0[j] != nullptr)
		{
			s2bPrefetchL1(a.cc.r0[j] + t);
		}
		if (a.cc.sep[j] != nullptr)
		{
			s2bPrefetchL1(a.cc.sep[j] + t);
		}
		if (a.cc.fanchor[j] != nullptr)
		{
			s2bPrefetchL1(a.cc.fanchor[j] + t);
			s2bPrefetchL1(a.cc.tsep[j] + t);
		}
	}
	if (bodies)
	{
		s2bTouchBody(a, idx.x);
		s2bTouchBody(a, idx.y & S2B_CF_INDEX_MASK);
	}
}

__device__ __forceinline__ void s2bTouchJoint(const SolveArgs& a, int t, bool bodies = true)
{
	int4 head = a.jc.head[t];
	s2bPrefetchL1(a.jc.anchor + t);
	s2bPrefetchL1(a.jc.mass + t);
	s2bPrefetchL1(a.jc.d0ax + t);
	s2bPrefetchL1(a.jc.lim + t);
	s2bPrefetchL1(a.jc.motor + t);
	s2bPrefetchL1(a.jc.coef + t);
	s2bPrefetchL1(a.jc.pivot + t);
	s2bPrefetchL1(a.jc.imp + t);
	s2bPrefetchL1(a.jc.limp + t);
	if (bodies)
	{
		if (head.y >= 0)
		{
			s2bTouchBody(a, head.y);
		}
		s2bTouchBody(a, head.z);
	}
}

// One Gauss-Seidel sweep: the interior constraints of this block's region colour by colour (block barriers), then the
// device-wide groups (cut colours / wavefront levels, a grid barrier before each), then the serial overflow group.
template <int SOLVER>
__device__ __forceinline__ void s2bGroupPass(int jointOp, int contactOp, const SolveArgs& a, const PassPtrs& p, const S2bLaunchInfo& li,
											 S2bSync& sync, const int* sRegJ, const int* sRegC, const int* sGroupJ, const int* sGroupC, int* sNbr,
											 int* sFt)
{
	int traceCode = (PASS_GROUP << 8) | contactOp;
	if (li.regions && li.primary > 0)
	{
		// (every block passes through here, also one whose region holds no interior constraint: `pending` stays grid-uniform)
		s2bSyncBeforeLocal(a, sync);
		bool first = true;
		for (int c = 0; c < li.primary; ++c)
		{
			int jBegin = sRegJ[c], cBegin = sRegC[c];
			int nj = jointOp != JOP_NONE ? sRegJ[c + 1] - jBegin : 0;
			int nc = contactOp != COP_NONE ? sRegC[c + 1] - cBegin : 0;
			if (nj + nc == 0)
			{
				continue; // uniform within the block
			}
			if (SOLVER == 7 && (contactOp == COP_TGS_SOFT_BIAS || contactOp == COP_TGS_SOFT_RELAX || contactOp == COP_TGS_SOFT_RELAX_STORE))
			{
				// The headline op, region-local: a thread's rows are private to it, so the row of its first constraint of this
				// colour is requested (prefetch into L1: no registers held) BEFORE the block barrier that ends the previous
				// colour, and the row of its next constraint while the current one is being solved: what stays on the dependent
				// chain of a round is the two bodies, the arithmetic and the stores. (Holding the next row in registers instead
				// pushed the kernel over 128 registers.)
				bool store = contactOp == COP_TGS_SOFT_RELAX_STORE;
				bool bias = contactOp == COP_TGS_SOFT_BIAS;
				bool writeWarm = bias ? a.ctx.extraIterations == 0 : true;
				int t = threadIdx.x;
				if (t < nc)
				{
					s2bTouchContactRow(a, cBegin + t);
				}
				if (first == false)
				{
					__syncthreads();
				}
				first = false;
				for (int tj = threadIdx.x; tj < nj; tj += blockDim.x)
				{
					s2bRunJointOpT<SOLVER>(jointOp, a, jBegin + tj, p);
				}
				for (; t < nc; t += blockDim.x)
				{
					if (t + (int)blockDim.x < nc)
					{
						s2bTouchContactRow(a, cBegin + t + blockDim.x);
					}
					s2bSolveContactTgsSoft(a, cBegin + t, a.ctx.inv_h, bias, writeWarm, store);
				}
				continue;
			}
			if (first == false)
			{
				__syncthreads();
			}
			first = false;
			for (int t = threadIdx.x; t < nj + nc; t += blockDim.x)
			{
				if (t < nj)
				{
					s2bRunJointOpT<SOLVER>(jointOp, a, jBegin + t, p);
				}
				else
				{
					s2bRunContactOpT<SOLVER>(contactOp, a, cBegin + (t - nj));
				}
			}
		}
		sync.pending = S2B_PENDING_LOCAL;
		sync.code = traceCode;
	}

	for (int g = 0; g < li.groups; ++g)
	{
		int jBegin, cBegin, jEnd, cEnd;
		if (sGroupJ != nullptr)
		{
			jBegin = sGroupJ[g], jEnd = sGroupJ[g + 1], cBegin = sGroupC[g], cEnd = sGroupC[g + 1];
		}
		else
		{
			jBegin = a.jGroupOff[g], jEnd = a.jGroupOff[g + 1], cBegin = a.cGroupOff[g], cEnd = a.cGroupOff[g + 1];
		}
		if ((jointOp != JOP_NONE ? jEnd - jBegin : 0) + (contactOp != COP_NONE ? cEnd - cBegin : 0) == 0)
		{
			continue; // uniform: every thread reads the same table
		}
		// this block's share of the group's items u (joints, then contacts), whatever the pass's ops: the mapping the neighbour
		// tables were built from
		int njAll = jEnd - jBegin;
		int n = njAll + cEnd - cBegin;
		int share = s2bGroupShare(n, gridDim.x);
		int uEnd = min(n, ((int)blockIdx.x + 1) * share);
		int u = (int)blockIdx.x * share + threadIdx.x;
		if (SOLVER == 7 && (contactOp == COP_TGS_SOFT_BIAS || contactOp == COP_TGS_SOFT_RELAX || contactOp == COP_TGS_SOFT_RELAX_STORE) &&
			(jointOp == JOP_NONE || njAll == 0))
		{
			// The headline op. Nothing in a thread's constraint row is written by another thread (the impulses by this very
			// thread, one sweep ago), so the row is fetched BEFORE the barrier: what remains after it is the dependent part
			// proper — the two bodies, the arithmetic, the stores (one L2 round trip less per device-wide step).
			bool mine = u >= njAll && u < uEnd;
			bool store = contactOp == COP_TGS_SOFT_RELAX_STORE;
			bool bias = contactOp == COP_TGS_SOFT_BIAS;
			bool fold = bias && li.foldPositions;
			// first-touch warm start: the marked bodies of a row are gathered right before its solve (warm_gather.cuh)
			int firstMarks = bias && li.firstTouch ? S2B_TOUCH_FIRST_A | S2B_TOUCH_FIRST_B : 0;
			// ... or, in colour 0, by the whole block from its first-touch table (block-uniform)
			bool blockWarm = firstMarks != 0 && g == 0 && sFt[0] >= 0;
			int t = cBegin + u - njAll;
			ContactStream cs;
			if (mine && blockWarm == false)
			{
				cs = s2bLoadContactStream(a, t, store);
				cs.last = fold ? a.cc.lastTouch[t] : 0;
				if (cs.last & firstMarks & S2B_TOUCH_FIRST_A)
				{
					s2bFirstTouchPrefetch(a, cs.idx.x);
				}
				if (cs.last & firstMarks & S2B_TOUCH_FIRST_B)
				{
					s2bFirstTouchPrefetch(a, cs.idx.y & S2B_CF_INDEX_MASK);
				}
			}
			if (sync.pending == S2B_PENDING_NEIGHBOURS)
			{
				s2bNeighbourWait(a, sync, sNbr);
			}
			else
			{
				s2bSyncBeforeGlobal(a, sync);
			}
			bool writeWarm = bias ? a.ctx.extraIterations == 0 : true;
			if (blockWarm)
			{
				// (the row is read after the gathers rather than held in registers through them)
				s2bFirstTableGather(a, sFt);
				if (mine)
				{
					cs = s2bLoadContactStream(a, t, store);
					cs.last = a.cc.lastTouch[t];
				}
				firstMarks = 0;
			}
			if (mine)
			{
				if (cs.last & firstMarks)
				{
					// (the row is fetched again after the gather instead of being held through it: holding it spilled. The
					// solve's body loads wait for the fetched indices, one L2 round trip more on a marked row)
					int last = cs.last;
					s2bFirstTouchWarm(a, cs.idx, last);
					cs = s2bLoadContactStream(a, t, store);
					cs.last = last;
				}
				s2bSolveContactTgsSoftStream(a, t, cs, a.ctx.inv_h, bias, writeWarm, store);
			}
			for (u += blockDim.x; u < uEnd; u += blockDim.x)
			{
				t = cBegin + u - njAll;
				if (u >= njAll)
				{
					int last = fold ? a.cc.lastTouch[t] : 0;
					if (last & firstMarks)
					{
						s2bFirstTouchWarm(a, a.cc.idx[t], last);
					}
					ContactStream more = s2bLoadContactStream(a, t, store);
					more.last = last;
					s2bSolveContactTgsSoftStream(a, t, more, a.ctx.inv_h, bias, writeWarm, store);
				}
			}
		}
		else
		{
			if (sync.pending == S2B_PENDING_NEIGHBOURS)
			{
				s2bNeighbourWait(a, sync, sNbr);
			}
			else
			{
				s2bSyncBeforeGlobal(a, sync);
			}
			for (; u < uEnd; u += blockDim.x)
			{
				if (u < njAll)
				{
					if (jointOp != JOP_NONE)
					{
						s2bRunJointOpT<SOLVER>(jointOp, a, jBegin + u, p);
					}
				}
				else if (contactOp != COP_NONE)
				{
					s2bRunContactOpT<SOLVER>(contactOp, a, cBegin + (u - njAll));
				}
			}
		}
		if (li.neighbours)
		{
			s2bPublishEpoch(a, sync, sNbr);
			sync.code = traceCode | 0x4000;
		}
		else
		{
			sync.pending = S2B_PENDING_GLOBAL;
			sync.code = traceCode | 0x8000;
		}
	}
	int ovC = contactOp != COP_NONE ? li.ovC : 0;
	int ovJ = jointOp != JOP_NONE ? li.ovJ : 0;
	if (ovC + ovJ > 0)
	{
		// The overflow group (constraints of bodies with more neighbours than there are colours — a container wall touching
		// hundreds of boxes) is inherently sequential: one thread walks it. What can be parallel is the memory: the rest of
		// block 0 first pulls every line that thread is going to touch into this SM's L1, so the walk pays L1 latency per
		// item instead of several dependent L2 round trips.
		s2bSyncBeforeGlobal(a, sync);
		if (blockIdx.x == 0)
		{
			int jBegin = a.jGroupOff[S2B_MAX_COLORS], cBegin = a.cGroupOff[S2B_MAX_COLORS];
			int nBodies = a.ovBodies != nullptr ? a.ovBodies[0] : 0;
			bool staged = a.ovBodies != nullptr && nBodies <= S2B_OV_MAX_BODIES && li.ovC <= S2B_OV_MAX_CONTACTS && li.ovJ <= S2B_OV_MAX_JOINTS;
			extern __shared__ __align__(16) unsigned char s2bOvShared[];
			float4* sVel = reinterpret_cast<float4*>(s2bOvShared);
			float4* sPose = sVel + S2B_OV_MAX_BODIES;
			float4* sAux = sPose + S2B_OV_MAX_BODIES;
			int2* sIdx = reinterpret_cast<int2*>(sAux + S2B_OV_MAX_BODIES);
			int4* sHead = reinterpret_cast<int4*>(sIdx + S2B_OV_MAX_CONTACTS);
			if (staged)
			{
				for (int k = threadIdx.x; k < nBodies; k += blockDim.x)
				{
					int body = a.ovBodies[1 + k];
					sVel[k] = a.bodies.vel[body];
					sPose[k] = a.bodies.pose[body];
					if (a.bodies.aux0 != nullptr)
					{
						sAux[k] = a.bodies.aux0[body];
					}
				}
				// (the rows are re-mapped for all of the group's contacts / joints, whichever of the two this pass solves: cheap)
				for (int k = threadIdx.x; k < li.ovC; k += blockDim.x)
				{
					int2 idx = a.cc.idx[cBegin + k];
					int ib = idx.y & S2B_CF_INDEX_MASK;
					sIdx[k] = make_int2(a.ovBodySlot[idx.x], a.ovBodySlot[ib] | (idx.y & ~S2B_CF_INDEX_MASK));
				}
				for (int k = threadIdx.x; k < li.ovJ; k += blockDim.x)
				{
					int4 head = a.jc.head[jBegin + k];
					sHead[k] = make_int4(head.x, head.y >= 0 ? a.ovBodySlot[head.y] : head.y, a.ovBodySlot[head.z], head.w);
				}
			}
			// the rest of block 0 pulls every stream line the walk is going to touch into this SM's L1 (the bodies
			// themselves sit in shared memory)
			for (int t = threadIdx.x; t < ovJ + ovC; t += blockDim.x)
			{
				if (t < ovJ)
				{
					s2bTouchJoint(a, jBegin + t, staged == false);
				}
				else
				{
					s2bTouchContact(a, cBegin + (t - ovJ), staged == false);
				}
			}
			__syncthreads();
			if (threadIdx.x == 0)
			{
				if (staged)
				{
					SolveArgs b = a;
					b.bodies.vel = sVel;
					b.bodies.pose = sPose;
					b.bodies.aux0 = a.bodies.aux0 != nullptr ? sAux : nullptr;
					b.cc.idx = sIdx - cBegin;
					b.jc.head = sHead - jBegin;
					for (int t = 0; t < ovJ; ++t)
					{
						s2bRunJointOpT<SOLVER>(jointOp, b, jBegin + t, p);
					}
					for (int t = 0; t < ovC; ++t)
					{
						s2bRunContactOpT<SOLVER>(contactOp, b, cBegin + t);
					}
				}
				else
				{
					for (int t = 0; t < ovJ; ++t)
					{
						s2bRunJointOpT<SOLVER>(jointOp, a, jBegin + t, p);
					}
					for (int t = 0; t < ovC; ++t)
					{
						s2bRunContactOpT<SOLVER>(contactOp, a, cBegin + t);
					}
				}
			}
			if (staged)
			{
				__syncthreads();
				for (int k = threadIdx.x; k < nBodies; k += blockDim.x)
				{
					int body = a.ovBodies[1 + k];
					a.bodies.vel[body] = sVel[k];
					a.bodies.pose[body] = sPose[k];
					if (a.bodies.aux0 != nullptr)
					{
						a.bodies.aux0[body] = sAux[k];
					}
				}
			}
		}
		sync.pending = S2B_PENDING_GLOBAL;
		sync.code = traceCode | 0xC000;
	}
}

// ---- ticketed ("dataflow") Gauss-Seidel pass ------------------------------------------------------------------
// A grid barrier after every colour costs its bare latency plus the tail of the slowest block, ten times per pass; on a 100 k-body
// scene that is most of the solver's time. What a constraint really has to wait for is only the previous constraint that
// touched each of its two bodies. Every movable body therefore carries a TICKET = number of incident constraints executed
// on it so far in this launch; the k-th item of a body's (solve-ordered) incidence list of d items runs in pass m when the
// ticket reads m * d + k, and sets it to m * d + k + 1 when done (release / acquire at GPU scope). The passes keep the
// stream order (group-major), so the outcome is bit-identical to the barrier version — the colouring now only decides how
// much runs concurrently — and the whole Gauss-Seidel sweep needs no grid barrier at all.
// Progress: every thread walks its items in stream order, an item only waits for items earlier in that order, and all
// blocks of a cooperative launch are resident, so the earliest unfinished item can always run. The work sits INSIDE the
// polling loop so that a lane that is ready never waits at a reconvergence point for a lane that is still polling.
// (Experimental, measured slower than barriers; runs without regions: all groups are device-wide.)

#define S2B_FLOW_SPIN_LIMIT (1 << 22)

__device__ __forceinline__ int s2bLoadAcquire(const int* p)
{
	int v;
	asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
	return v;
}

__device__ __forceinline__ void s2bStoreRelaxed(int* p, int v)
{
	asm volatile("st.relaxed.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

template <int SOLVER, bool JOINT>
__device__ __forceinline__ void s2bFlowItem(int op, const SolveArgs& a, const PassPtrs& p, int t, int passIndex)
{
	int ia, ib;
	int2 fa, fb;
	if (JOINT)
	{
		int4 head = a.jc.head[t];
		ia = head.y;
		ib = head.z;
		fa = a.jFlowA[t];
		fb = a.jFlowB[t];
	}
	else
	{
		int2 idx = a.cc.idx[t];
		ia = idx.x;
		ib = idx.y & S2B_CF_INDEX_MASK;
		fa = a.cFlowA[t];
		fb = a.cFlowB[t];
	}
	int needA = passIndex * fa.y + fa.x, needB = passIndex * fb.y + fb.x;
	bool done = false;
	int spins = 0;
	while (done == false)
	{
		bool ready = true;
		if (fa.x >= 0)
		{
			ready = s2bLoadAcquire(a.bodyTicket + ia) == needA;
		}
		if (ready && fb.x >= 0)
		{
			ready = s2bLoadAcquire(a.bodyTicket + ib) == needB;
		}
		if (ready)
		{
			if (JOINT)
			{
				s2bRunJointOpT<SOLVER>(op, a, t, p);
			}
			else
			{
				s2bRunContactOpT<SOLVER>(op, a, t);
			}
			__threadfence();
			if (fa.x >= 0)
			{
				s2bStoreRelaxed(a.bodyTicket + ia, needA + 1);
			}
			if (fb.x >= 0)
			{
				s2bStoreRelaxed(a.bodyTicket + ib, needB + 1);
			}
			done = true;
		}
		else if (a.flowSleepNs > 0)
		{
			__nanosleep(a.flowSleepNs);
		}
		if (done == false && (++spins > S2B_FLOW_SPIN_LIMIT || ((spins & 1023) == 0 && *(volatile int*)a.flowError != 0)))
		{
			// never expected; bail out of the whole launch quickly instead of hanging the device
			a.flowError[0] = 1;
			done = true;
		}
	}
}

// joints and contacts of every group in stream order, no barrier; a pass with an op of only one kind still walks the other
// kind (op NONE) to keep the tickets of its bodies moving
template <int SOLVER>
__device__ __forceinline__ void s2bFlowPass(int jointOp, int contactOp, const SolveArgs& a, const PassPtrs& p, const S2bLaunchInfo& li,
											int passIndex)
{
	int stride = gridDim.x * blockDim.x;
	int tid = blockIdx.x * blockDim.x + threadIdx.x;
	for (int g = 0; g <= li.groups; ++g)
	{
		bool overflow = g == li.groups;
		if (overflow && li.ovC + li.ovJ == 0)
		{
			break;
		}
		int table = overflow ? S2B_MAX_COLORS : g;
		int jBegin = a.jGroupOff[table], cBegin = a.cGroupOff[table];
		int nj = overflow ? li.ovJ : a.jGroupOff[g + 1] - jBegin;
		int nc = overflow ? li.ovC : a.cGroupOff[g + 1] - cBegin;
		for (int t = tid; t < nj; t += stride)
		{
			s2bFlowItem<SOLVER, true>(jointOp, a, p, jBegin + t, passIndex);
		}
		for (int t = tid; t < nc; t += stride)
		{
			s2bFlowItem<SOLVER, false>(contactOp, a, p, cBegin + t, passIndex);
		}
	}
}

// ---- the kernel --------------------------------------------------------------------------------------------------

// The whole solver stage of one step: the variant's program from prepare to store, one launch.
// The restitution instantiation runs on the variant's grid (one block per SM), so it is told that one resident block per SM
// is enough: left to itself ptxas keeps it at 64 registers (two blocks per SM) and spills.
template <int SOLVER> __global__ void __launch_bounds__(S2B_BLOCK, SOLVER == S2B_RESTITUTION_PROGRAM ? 1 : 0) s2bPersistentSolveT(SolveArgs a, PassPtrs p, Program prog)
{
	__shared__ int sRegJ[S2B_REG_STRIDE], sRegC[S2B_REG_STRIDE];
	__shared__ int sGroupJ[S2B_MAX_COLORS + 2], sGroupC[S2B_MAX_COLORS + 2];
	__shared__ int sNbr[S2B_NSYNC_STRIDE + 1];
	__shared__ int sFt[3]; // the block's first-touch table in dynamic shared memory: slots (-1: none), entries, anchors staged

	S2bSync sync;
	sync.base = *((volatile unsigned*)(a.barrier + 32));
	sync.arrivals = 0;
	if (threadIdx.x == 0)
	{
		sNbr[S2B_NBR_EPOCH] = (int)*((volatile unsigned*)(a.barrier + S2B_EPOCH_BASE_WORD));
	}
	sync.pending = S2B_PENDING_NONE;
	sync.code = 0;
	s2bTrace(a, 0xFFFF);

	S2bLaunchInfo li;
	li.nJ = a.counts[CNT_JOINTS];
	li.nC = a.counts[CNT_CONTACTS];
	li.primary = a.counts[CNT_PRIMARY];
	li.groups = a.counts[CNT_GROUPS];
	li.ovJ = a.counts[CNT_OVERFLOW_J];
	li.ovC = a.counts[CNT_OVERFLOW_C];
	li.regions = a.regions > 0 && a.counts[CNT_REGIONS_ON] != 0;
	li.hubs = (li.regions && a.heavyBodies != nullptr) ? a.heavyBodies[0] : 0;
	li.neighbours = a.nsyncNbr != nullptr && a.counts[CNT_NSYNC] == (int)gridDim.x && li.regions == false && li.ovC + li.ovJ == 0 &&
					a.bodyTicket == nullptr;
	if (li.neighbours)
	{
		for (int k = threadIdx.x; k < S2B_NSYNC_STRIDE; k += blockDim.x)
		{
			sNbr[k] = a.nsyncNbr[blockIdx.x * S2B_NSYNC_STRIDE + k];
		}
	}
	// s2IntegratePositions folded into the TGS_Soft bias sweep: only in the plain colour schedule of a scene without joints,
	// hub bodies or an overflow group (every movable body with a constraint then has a CONTACT as its last toucher, and
	// every bias step runs through the branch below that looks at the marks); all of it is grid-uniform
	li.foldPositions = SOLVER == 7 && a.cc.lastTouch != nullptr && li.regions == false && li.nJ == 0 && li.ovC + li.ovJ == 0 &&
					   (a.heavyBodies == nullptr || a.heavyBodies[0] == 0) && a.bodyTicket == nullptr && li.nC > 0;
	// the warm-start gather folded into the same sweep, at each body's first constraint: wherever positions are folded, unless a
	// constraint reads a kinematic body. Such a body has no incidence list (s2bItemEndpoints) and only the warm-start pass
	// integrates its pose every sub-step (alsoPosition), so that pass stays. (A program with the fold always warm-starts:
	// lastTouch is only handed over with the gather on.)
	li.firstTouch = li.foldPositions && a.counts[CNT_KINEMATIC_ITEMS] == 0;
	li.resident = SOLVER == 7 && li.regions && a.bodyLocal != nullptr && a.counts[CNT_RESIDENT] != 0 && a.bodyTicket == nullptr;
	if (threadIdx.x == 0)
	{
		sFt[0] = -1;
	}
	if (SOLVER == 7 && li.firstTouch && a.cc.firstTable != nullptr && a.counts[CNT_FIRST_TABLE] == (int)gridDim.x)
	{
		s2bFirstTableStage(a, sFt);
	}
	li.bodyBegin = li.bodyEnd = 0;
	if (li.regions)
	{
		// (the grid has exactly `regions` blocks)
		li.bodyBegin = a.regBodyStart[blockIdx.x];
		li.bodyEnd = a.regBodyStart[blockIdx.x + 1];
		for (int c = threadIdx.x; c < S2B_REG_STRIDE; c += blockDim.x)
		{
			sRegJ[c] = a.jRegOff[blockIdx.x * S2B_REG_STRIDE + c];
			sRegC[c] = a.cRegOff[blockIdx.x * S2B_REG_STRIDE + c];
		}
	}
	bool groupsInShared = li.groups <= S2B_MAX_COLORS;
	if (groupsInShared)
	{
		for (int c = threadIdx.x; c < S2B_MAX_COLORS + 2; c += blockDim.x)
		{
			sGroupJ[c] = a.jGroupOff[c];
			sGroupC[c] = a.cGroupOff[c];
		}
	}
	// resident regions: the block's copy of its bodies (nothing has changed them yet: prepare, the first pass, only reads)
	extern __shared__ __align__(16) unsigned char s2bDynShared[];
	float4* sVel = reinterpret_cast<float4*>(s2bDynShared);
	float4* sPose = sVel + S2B_RES_MAX_BODIES;
	if (li.resident)
	{
		for (int k = li.bodyBegin + threadIdx.x; k < li.bodyEnd; k += blockDim.x)
		{
			int i = a.regBodies[k];
			sVel[k - li.bodyBegin] = a.bodies.vel[i];
			sPose[k - li.bodyBegin] = a.bodies.pose[i];
		}
	}
	__syncthreads();

	bool flow = a.bodyTicket != nullptr;
	int flowPasses = 0;
	for (int s = 0; s < prog.segmentCount; ++s)
	{
		for (int r = 0; r < prog.repeat[s]; ++r)
		{
			for (int k = 0; k < prog.passCount[s]; ++k)
			{
				PassDesc pass = prog.passes[s][k];
				if (li.resident && pass.kind == PASS_GROUP)
				{
					// (a resident launch has no joints, no device-wide groups and no overflow group: the sweep is the region's own)
					s2bSyncBeforeLocal(a, sync);
					s2bResidentSweep<SOLVER>(pass.contactOp, a, sVel, sPose, li, sRegC);
					sync.pending = S2B_PENDING_LOCAL;
					sync.code = (PASS_GROUP << 8) | pass.contactOp;
				}
				else if (li.resident && pass.kind == PASS_BODY)
				{
					s2bSyncBeforeLocal(a, sync);
					s2bResidentBodyPass(pass.bodyOp, a, li, sVel, sPose);
					sync.pending = S2B_PENDING_LOCAL;
					sync.code = (PASS_BODY << 8) | pass.bodyOp;
				}
				else if (pass.kind == PASS_GROUP)
				{
					if (flow)
					{
						if (sync.pending != S2B_PENDING_FLOW)
						{
							s2bSyncBeforeGlobal(a, sync);
						}
						s2bFlowPass<SOLVER>(pass.jointOp, pass.contactOp, a, p, li, flowPasses);
						flowPasses += 1;
						sync.pending = S2B_PENDING_FLOW;
					}
					else
					{
						s2bGroupPass<SOLVER>(pass.jointOp, pass.contactOp, a, p, li, sync, sRegJ, sRegC, groupsInShared ? sGroupJ : nullptr,
											 groupsInShared ? sGroupC : nullptr, sNbr, sFt);
					}
				}
				else if (pass.kind == PASS_BODY && li.foldPositions && pass.bodyOp == BOP_INTEGRATE_POSITIONS)
				{
					// done by the bias sweep before it (and for bodies without constraints by the velocity pass, or by finalize)
				}
				else if (pass.kind == PASS_BODY && li.firstTouch && pass.bodyOp == BOP_INTEGRATE_VELOCITIES_WARM)
				{
					// done by the bias sweep after it (and for bodies without constraints by finalize): the previous sweep's last
					// colour step flows into the bias sweep's first one through a neighbour wait
				}
				else if (pass.kind == PASS_BODY)
				{
					int code = (PASS_BODY << 8) | pass.bodyOp;
					if (li.regions)
					{
						s2bSyncBeforeLocal(a, sync);
						s2bBodyPass<SOLVER>(pass.bodyOp, a, li);
						sync.pending = S2B_PENDING_LOCAL;
						sync.code = code;
					}
					else
					{
						s2bSyncBeforeGlobal(a, sync);
						s2bBodyPass<SOLVER>(pass.bodyOp, a, li);
						sync.pending = S2B_PENDING_GLOBAL;
						sync.code = code;
					}
				}
				else
				{
					int contactOp = pass.contactOp;
					if constexpr (s2bUsesContactOp(SOLVER, COP_PREPARE) || s2bUsesContactOp(SOLVER, COP_PREPARE_COLD))
					{
						if ((contactOp == COP_PREPARE || contactOp == COP_PREPARE_COLD) && a.counts[CNT_ROWS_READY] != 0)
						{
							// the narrow phase has written this step's contact rows (narrowphase.cu): prepare leaves the contacts
							// alone, and without joints the pass and its barrier go (grid-uniform: nothing writes the count while
							// the kernel runs)
							contactOp = COP_NONE;
						}
					}
					if ((pass.jointOp == JOP_NONE || li.nJ == 0) && (contactOp == COP_NONE || li.nC == 0))
					{
						// nothing to do for anybody (the counts are grid-uniform): no barrier either
					}
					else
					{
						s2bSyncBeforeGlobal(a, sync);
						s2bFlatPass<SOLVER>(pass.jointOp, contactOp, a, p, li);
						sync.pending = S2B_PENDING_GLOBAL;
						sync.code = (PASS_FLAT << 8) | contactOp;
					}
				}
			}
		}
	}
	// hand the arrival count and the epoch to the next launch. Every block has read both bases before block 0 gets here if a
	// grid barrier lies between; neighbour waits alone do not ensure that (blocks of another island may not have started), so a
	// launch without a grid barrier (the restitution pass) takes one here.
	if (li.neighbours && sync.arrivals == 0)
	{
		s2bGridBarrier(a, sync);
	}
	s2bTrace(a, sync.code);
	if (blockIdx.x == 0 && threadIdx.x == 0 && gridDim.x > 1)
	{
		a.barrier[32] = sync.base + sync.arrivals;
		a.barrier[S2B_EPOCH_BASE_WORD] = (unsigned)sNbr[S2B_NBR_EPOCH];
	}
}

// host-side handle of an instantiation (defined in persistent_*.cu)
void* s2bPersistentKernel(int solverType);
// the instantiation that runs the restitution pass (S2B_RESTITUTION_PROGRAM, persistent_r.cu)
void* s2bRestitutionKernel();
