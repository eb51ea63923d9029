// solver2d-b200 — device-side world: SoA columns, scratch arena, launch helpers. Internal to the CUDA library.
#pragma once

#include "s2b_device.h"
#include "solver2d/constants.h"
#include "solver2d/aabb.h"
#include "solver2d/math.h"

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#define S2B_CHECK(call)                                                                                                \
	do                                                                                                                 \
	{                                                                                                                  \
		cudaError_t err__ = (call);                                                                                    \
		if (err__ != cudaSuccess)                                                                                      \
		{                                                                                                              \
			fprintf(stderr, "solver2d-b200: CUDA error %s at %s:%d (%s) — no CPU fallback, aborting\n",                 \
					cudaGetErrorString(err__), __FILE__, __LINE__, #call);                                             \
			abort();                                                                                                   \
		}                                                                                                              \
	} while (0)

// ---- body flags (bflags column) -------------------------------------------------------------------------------
#define S2B_BODY_VALID 0x1u
#define S2B_BODY_TYPE(f) (((f) >> 1) & 0x3u)
// a body takes part in conflict detection / write-back only if it can move in the solver
#define S2B_BODY_STATIC 0u
#define S2B_BODY_KINEMATIC 1u
#define S2B_BODY_DYNAMIC 2u

// ---- contact info word (cInfo.x) ------------------------------------------------------------------------------
// bits 0-1 pointCount, bit 2 frictionPersisted, bit 3 persisted0, bit 4 persisted1
#define S2B_CI_COUNT(x) ((x) & 0x3)
#define S2B_CI_FRICTION_PERSISTED 0x4
#define S2B_CI_PERSISTED0 0x8
#define S2B_CI_PERSISTED1 0x10

// A growable device array. grow() keeps the old contents (device-to-device copy on the world's stream).
// bumped whenever any device array is re-allocated: a captured CUDA graph bakes device pointers in, so the solver's graph
// cache keys on this epoch
inline unsigned long long& s2bAllocEpoch()
{
	static unsigned long long epoch = 0;
	return epoch;
}

// Scope guard for code whose (re)allocations no captured graph refers to (broad-phase scratch, transfer staging, the L2
// flush buffer): the epoch is put back on exit so that those allocations do not force a re-capture of the solver graph.
struct S2bEpochFreeze
{
	unsigned long long saved;
	S2bEpochFreeze() : saved(s2bAllocEpoch())
	{
	}
	~S2bEpochFreeze()
	{
		s2bAllocEpoch() = saved;
	}
};

template <typename T> struct DevArray
{
	T* p = nullptr;
	size_t cap = 0;

	void reserve(size_t n, cudaStream_t stream, bool keep = true, bool zero = true)
	{
		if (n <= cap)
		{
			return;
		}
		size_t newCap = cap ? cap : 64;
		while (newCap < n)
		{
			newCap += newCap / 2 + 64;
		}
		T* q = nullptr;
		S2B_CHECK(cudaMalloc((void**)&q, newCap * sizeof(T)));
		if (zero)
		{
			S2B_CHECK(cudaMemsetAsync(q, 0, newCap * sizeof(T), stream));
		}
		if (p != nullptr)
		{
			if (keep && cap > 0)
			{
				S2B_CHECK(cudaMemcpyAsync(q, p, cap * sizeof(T), cudaMemcpyDeviceToDevice, stream));
			}
			// The old buffer came from cudaMalloc, so cudaFreeAsync would not order its release behind this stream: another world's
			// allocation could take it over while the copy above (or a kernel still queued here) reads it. Wait, then free.
			S2B_CHECK(cudaStreamSynchronize(stream));
			S2B_CHECK(cudaFree(p));
		}
		p = q;
		cap = newCap;
		s2bAllocEpoch() += 1;
	}

	void release()
	{
		if (p)
		{
			cudaFree(p);
		}
		p = nullptr;
		cap = 0;
	}
};

// per-contact persistent columns; two sets (ping-pong) so a broad-phase pass can re-sort into the other one
struct ContactColumns
{
	DevArray<unsigned long long> key; // lo shape << 32 | hi shape
	DevArray<int2> shapes;			  // (A, B) in manifold order
	DevArray<int2> bodies;			  // (A, B)
	DevArray<int4> info;			  // x: count/flags, y: id0 | id1 << 16, z: GJK cache (count | iA<<2.. ), w: cache metric bits
	DevArray<float4> nf;			  // normal.x normal.y friction restitution
	DevArray<int> color;			  // colour the constraint was last solved with (-1: none)
	DevArray<float4> anchor[2];		  // localAnchorA.xy localAnchorB.xy   (body-origin relative, body frame)
	DevArray<float4> impulse[2];	  // separation normalImpulse tangentImpulse 0
	DevArray<float4> fanchor[2];	  // frictionAnchorA.xy frictionAnchorB.xy   (sticky only)
	DevArray<float4> fnormal[2];	  // frictionNormalA.xy frictionNormalB.xy   (sticky only)

	void reserve(size_t n, cudaStream_t s, bool sticky, bool keep)
	{
		key.reserve(n, s, keep);
		shapes.reserve(n, s, keep);
		bodies.reserve(n, s, keep);
		info.reserve(n, s, keep);
		nf.reserve(n, s, keep);
		color.reserve(n, s, keep);
		for (int p = 0; p < 2; ++p)
		{
			anchor[p].reserve(n, s, keep);
			impulse[p].reserve(n, s, keep);
			if (sticky)
			{
				fanchor[p].reserve(n, s, keep);
				fnormal[p].reserve(n, s, keep);
			}
		}
	}

	void release()
	{
		key.release();
		shapes.release();
		bodies.release();
		info.release();
		nf.release();
		color.release();
		for (int p = 0; p < 2; ++p)
		{
			anchor[p].release();
			impulse[p].release();
			fanchor[p].release();
			fnormal[p].release();
		}
	}
};

// raw-pointer view of the contact columns handed to kernels
struct ContactView
{
	unsigned long long* key;
	int2* shapes;
	int2* bodies;
	int4* info;
	float4* nf;
	int* color;
	float4* anchor[2];
	float4* impulse[2];
	float4* fanchor[2];
	float4* fnormal[2];
};

inline ContactView makeView(ContactColumns& c)
{
	ContactView v;
	v.key = c.key.p;
	v.shapes = c.shapes.p;
	v.bodies = c.bodies.p;
	v.info = c.info.p;
	v.nf = c.nf.p;
	v.color = c.color.p;
	for (int p = 0; p < 2; ++p)
	{
		v.anchor[p] = c.anchor[p].p;
		v.impulse[p] = c.impulse[p].p;
		v.fanchor[p] = c.fanchor[p].p;
		v.fnormal[p] = c.fnormal[p].p;
	}
	return v;
}

// per-step contact-constraint columns in solve order (group-major). Which optional columns are live depends on the
// solver variant (DESIGN.md "constraint stream").
struct ConstraintView
{
	int2* idx;		  // bodyA, bodyB | flags in the two top bits of y (see S2B_CF_*)
	float4* nf;		  // normal.x normal.y friction invI_A
	float4* anchor[2]; // COM-relative local anchors: A.xy B.xy
	float4* pm[2];	  // adjustedSeparation normalMass tangentMass invI_B(point 0) / spare(point 1)
	float2* lambda[2]; // normalImpulse tangentImpulse (read-modify-write every pass)
	float4* r0[2];	  // prepare-time world anchors rA0.xy rB0.xy (fixed-anchor variants, XPBD)
	float* sep[2];	  // prepare-time separation (PGS family, NGS)
	int* src;		  // contact slot this constraint came from
	// warm-start gather (warm_gather.cuh): what one body needs from one incident constraint, in two 16-byte rows instead of
	// six scattered columns. warmP[t] = {P0.x, P0.y, P1.x, P1.y}, P = lambda_n * n + lambda_t * t per point, rewritten by
	// whichever pass last changes the impulses before the next gather (P1.x = NaN: one-point manifold);
	// warmAnchor[t * 2 + side] = {anchor0.xy, anchor1.xy} of that side, written by prepare (COM-relative local anchors;
	// prepare-time world anchors for SoftStep). Null when the variant does not gather.
	float4* warmP;
	float4* warmAnchor;
	// per constraint, the touch marks: bit 0 / bit 1 = this constraint is the LAST one of the solve order that touches its
	// body A / B, bit 2 / bit 3 = it is the FIRST one (S2B_TOUCH_*). The TGS_Soft bias sweep then integrates a last-touched
	// body's position itself (s2IntegratePositions folded into the sweep) and warm-starts a first-touched body's velocity
	// itself (the warm-start gather folded into the sweep), one device-wide body pass less each per sub-step (persistent.cuh).
	// Null: positions are integrated and velocities gathered by their own body passes.
	const int* lastTouch;
	// per block of the persistent kernel, the bodies its share of colour 0 first-touches, with their incidence entries
	// (persistent.cuh, S2B_FT_*); null: every first-touch gather runs in the thread of the body's row
	const int* firstTable;
	// sticky extras
	float4* fanchor[2]; // COM-relative local friction anchors A.xy B.xy
	float2* tsep[2];	// tangentSeparation, spare
};

// ConstraintView::lastTouch bits
#define S2B_TOUCH_LAST_A 1
#define S2B_TOUCH_LAST_B 2
#define S2B_TOUCH_FIRST_A 4
#define S2B_TOUCH_FIRST_B 8

#define S2B_CF_TWO_POINTS 0x40000000
#define S2B_CF_STATIC_SOFT 0x80000000u
#define S2B_CF_INDEX_MASK 0x3FFFFFFF
// resident regions (persistent.cuh): body indices of a row are positions in the region's shared-memory copy; an index with
// this bit set is a body slot in global memory instead (a body no constraint can move: read only)
#define S2B_RES_GLOBAL 0x20000000

// view of the body columns
struct BodyView
{
	float4* vel;  // v.x v.y w invMass
	float4* pose; // dp.x dp.y q.s q.c
	float4* pos;  // p.x p.y invI I      (centre of mass)
	float4* org;  // origin.x origin.y localCenter.x localCenter.y
	float4* frc;  // force.x force.y torque mass
	float4* prm;  // linearDamping angularDamping gravityScale invI
	float4* aux0; // Jacobi: dv.x dv.y dw 0 ; XPBD: dp0.x dp0.y q0.s q0.c
	float4* aux1; // XPBD: v0.x v0.y w0 0
	uint8_t* flags;
	int capacity;
};

// view of the shape columns
struct ShapeView
{
	int4* head;		 // flags(valid|type<<1|moved<<4), body, proxyKey, vertex count
	int4* filter;	 // categoryBits maskBits groupIndex 0
	float4* aabb;	 // tight + speculative
	float4* fat;	 // broad-phase box
	float2* fr;		 // friction, radius
	float2* verts;	 // [shape * 8 + i]
	float2* normals; // [shape * 8 + i]
	int capacity;
	float* restitution; // per shape
};

// per-joint columns (slot order)
struct JointView
{
	int4* head;		// flags, bodyA, bodyB, 0
	float4* anchors; // localOriginAnchorA.xy localOriginAnchorB.xy
	float4* lim;	// referenceAngle lowerAngle upperAngle 0
	float4* motor;	// maxMotorTorque motorSpeed hertz dampingRatio
	float4* target; // mouse target.xy, prismatic localAxisA.xy
	float4* imp;	// impulse.x impulse.y motorImpulse springImpulse
	float4* limp;	// lowerImpulse upperImpulse 0 0
	int* color;		// colour the joint was last solved with (-1: none)
	int capacity;
};

// per-step joint-constraint columns in solve order
struct JointConstraintView
{
	int4* head;		// flags(type, limit, motor, spring), bodyA, bodyB, source joint slot. The spring flag stays only on rows
					// whose spring acts (DESIGN.md §3.14); XPBD spring rows add S2B_JC_STATIC_A / _B.
	float4* anchor; // COM-relative local anchors A.xy B.xy
	float4* mass;	// invMassA invIA invMassB invIB
	float4* d0ax;	// centerDiff0.xy axialMass springImpulseScale
	float4* lim;	// referenceAngle lowerAngle upperAngle springMassScale (XPBD: spring dampingRatio)
	float4* motor;	// maxMotorTorque motorSpeed 0 0 (prismatic: maxMotorForce motorSpeed localAxisA.xy;
					// motor joint: maxTorque 0 maxForce correctionFactor)
	float4* coef;	// biasCoefficient massCoefficient impulseCoefficient springBias (XPBD: 2 pi hertz h)
	float4* pivot;	// pivotMass cx.x cx.y cy.x cy.y (mouse, non-fresh revolute)
	float4* imp;	// impulse.x impulse.y motorImpulse springImpulse (r/w)
	float4* limp;	// lowerImpulse upperImpulse 0 0              (r/w)
};

struct StageTimer
{
	cudaEvent_t ev[5];
	bool recorded = false;
};

struct s2bWorld
{
	int device = 0;
	int solverType = 0;
	cudaStream_t stream = nullptr;
	float2 gravity = {0.0f, -10.0f};
	int schedule = S2B_SCHEDULE_COLOR;
	int maxColors = 24;
	int persistent = 1;
	int useGraph = 1;		// replay the solver stage as a CUDA graph when nothing changed; s2b_set_graph / S2B_GRAPH=0 disable
	bool capturing = false;
	unsigned long long contactTableVersion = 0; // bumped whenever the contact table is replaced (pair pass commit, upload) // a stream capture of the solver stage is in progress
	// region-local schedule of the persistent kernel (persistent.cuh): 0 off, 1 when the cut set needs at most regionCutLimit
	// colours (decided on the device every time the schedule is built), 2 always; s2b_set_regions / S2B_REGIONS
	int useRegions = 1;
	int regionCutLimit = 3; // S2B_REGION_CUT_LIMIT
	int dataflow = 0;	// ticketed Gauss-Seidel passes in the persistent kernel (experimental, measured slower: DESIGN.md §3.1);
						// s2b_set_dataflow / S2B_DATAFLOW=1 enable it
	int restitution = 0;			   // s2b_set_restitution: end the solver stage with the restitution pass
	float restitutionThreshold = 1.0f; // approach speed (m/s) below which a contact does not bounce
	int continuous = 0;				   // s2b_set_continuous: sweep fast bodies against static shapes after the solver stage
	int gatherWarm = 1; // per-body warm-start gather (warm_gather.cuh); s2b_set_warm_gather / S2B_WARM_GATHER=0 disable it
	int smCount = 132;
	int coopSupported = 0;
	int colorGrid = 0;	// cooperative grid sizes, computed once
	int solveGrid = 0;
	int solveGridSolver = -1; // variant the grid was sized for (each variant is its own kernel)
	DevArray<int> schedDirty; // [0] != 0: the set of live constraints changed since the solve schedule was built (device flag)
	DevArray<unsigned> solveBarrier; // arrival counter of the persistent kernel's grid barrier (persistent.cuh)
	unsigned long long scheduleEpoch = 0; // bumped by every host-side change the solve schedule depends on (uploads, settings)

	// bodies
	int bodyCap = 0;
	DevArray<float4> bVel, bPose, bPos, bOrg, bFrc, bPrm, bAux0, bAux1;
	DevArray<uint8_t> bFlags;
	DevArray<float2> bExt; // minExtent maxExtent (continuous collision; kept out of BodyView, which the solver kernels take)
	// per body slot: the last uploaded row was valid, dynamic and a bullet (S2B_BODY_BULLET); the bullet pass runs only while
	// bulletCount > 0, so a world without bullets launches nothing for it
	std::vector<uint8_t> bulletSlot;
	int bulletCount = 0;

	// shapes
	int shapeCap = 0;
	DevArray<int4> sHead, sFilter;
	DevArray<float4> sAabb, sFat;
	DevArray<float2> sFr, sVerts, sNormals;
	DevArray<float> sRestitution;

	// joints
	int jointCap = 0;
	DevArray<int4> jHead;
	DevArray<float4> jAnchors, jLim, jMotor, jTarget, jImp, jLimp;
	DevArray<int> jColor;
	// breakForce breakTorque per joint slot (0 = no threshold). Kept out of JointView, which SolveArgs carries into every solver
	// kernel: only the scatter, the gather and the reaction pass read it
	DevArray<float2> jBreak;
	// per joint slot: the last uploaded row was valid and had a threshold; the reaction pass runs after finalize only while
	// breakCount > 0, so a world without thresholds launches nothing for it (DESIGN.md §3.13)
	std::vector<uint8_t> breakSlot;
	int breakCount = 0;
	float reactionRate = 0.0f; // 1 / the interval the last s2b_solve accumulated joint impulses over (s2MakeJointReaction)
	DevArray<int> dBroken;	   // [0] count, then the slots over a threshold (device order)
	int* hostBroken = nullptr; // pinned copy of dBroken, jointCap + 1 ints
	int hostBrokenCap = 0;
	cudaEvent_t brokenEvent = nullptr; // recorded behind the copy into hostBroken
	bool brokenPending = false;		   // the last finalize ran the pass: hostBroken is valid once brokenEvent has passed
	int jointsChecked = 0;			   // slots the last finalize's pass checked (0: it did not run)
	DevArray<unsigned long long> jointPairKeys; // every jointed body pair: blocks new contacts
	int jointPairCount = 0;
	DevArray<unsigned long long> jointDestroyKeys; // pairs whose existing contacts are removed
	int jointDestroyCount = 0;

	// pinned read-back buffer of s2b_sync_body_state
	float* hostState = nullptr;
	// bulk paths (s2b_add_forces, s2b_download_transforms)
	void* bulkHost[2] = {nullptr, nullptr};
	size_t bulkBytes[2] = {0, 0};
	cudaEvent_t bulkEvent[2] = {nullptr, nullptr};
	int bulkNext = 0, bulkCurrent = 0;
	DevArray<char> dBulk;
	float* hostXf = nullptr;
	size_t hostXfFloats = 0;
	DevArray<float4> dXf;
	size_t hostStateFloats = 0;
	DevArray<float4> dState;

	// contacts
	ContactColumns contacts[2];
	int cur = 0;		  // which column set is live
	int contactCount = 0; // host mirror (valid after a pair pass or upload)
	bool sticky = false;

	// broad phase
	bool pairsDirty = true; // host-side structural change
	unsigned long long uploadEpoch = 0; // bumped by every row upload: a pair search started before it is stale
	unsigned long long shapeEpoch = 0;	// bumped by every shape upload: a hierarchy refitted before it may miss static boxes
	int prefetchPairs = 1;	// start the pair search of the next step behind finalize (S2B_PREFETCH_PAIRS=0: off)
	int kempe = 1;		// empty a sparse top colour by Kempe chains after colouring (S2B_KEMPE=0 disables)
	int wholeIslandBodies = 1200; // regions: islands up to this size are never cut (S2B_WHOLE_ISLAND)
	int residentRegions = 1; // TGS_Soft: regions with nothing device-wide to solve keep their bodies in shared memory (S2B_RESIDENT=0 disables)
	int hubDegree = 48; // constraints of a body with more incident constraints go to the serial overflow group uncoloured (S2B_HUB_DEGREE, 0 = colour them)
	int fusePositions = 1; // TGS_Soft: s2IntegratePositions folded into the bias sweep (S2B_FUSE_POSITIONS=0 disables)
	int neighbourSync = 1; // device-wide colour steps wait for neighbouring blocks only, where the device finds that possible
						   // (persistent.cuh; S2B_NEIGHBOUR_SYNC=0 keeps a grid barrier before every colour step)
	int narrowphasePrepare = 1; // while the solve schedule stands, the narrow phase writes the contact rows and the solver's
								// prepare pass skips them (narrowphase.cu; S2B_NARROWPHASE_PREPARE=0 leaves it all to prepare)
	int blockWarm = 1;		// TGS_Soft: the bias sweep's colour-0 step warm-starts a block's first-touched bodies together, from a
							// table built with the schedule (persistent.cuh; S2B_BLOCK_WARM=0 keeps the gather per thread)
	int blockWarmBytes = 0; // shared-memory budget of one block's table; 0 = the kernel's dynamic shared memory (S2B_BLOCK_WARM_BYTES)
	int fusedRefit = 1; // finalize refits the pair search's hierarchy and collects its moved proxies when the search will
						// reuse the topology (broadphase.cu s2bFinalizeRefit; S2B_FINALIZE_REFIT=0: the search does both)
	int kempeGrid = 0;
	DevArray<int> dMovedFlag; // [0] = number of proxies moved in last finalize (device counter)
	int pairPassCount = 0;
	int finalizeRefits = 0; // pair passes whose refit and moved proxies came from finalize (s2bFinalizeRefit)
	int pairRetries = 0;	// pair searches run again because their candidate pairs overflowed the pair buffer
	int prefetchRetries = 0; // ... of which the overflowing search was the prefetched one
	int largeMovers = 0;	// BC_LARGE of the last committed pass (uncapped)
	int treeBuilds = 0;		// pair-search hierarchies built from scratch
	int pairBuffer = 0;		// initial candidate-pair capacity; 0 = 8 per shape slot + 1024 (S2B_PAIR_BUFFER)
	int treeHeight = 0;

	// solve-order hint (validation)
	std::vector<unsigned long long> orderHint;

	// scratch + bookkeeping for the solver stage live in solver_state.cuh (opaque here)
	struct SolverScratch* scratch = nullptr;
	struct BroadScratch* broad = nullptr;

	// pinned host mailbox for small device->host counters
	int* hostMail = nullptr; // pinned, 64 ints
	int* devMail = nullptr;	 // device, 64 ints

	int kernelLaunches = 0;
	// device-side work meter: [0] constraint-iterations, [1] solver stages run (bench metric, SURVEY §8d)
	DevArray<unsigned long long> dWork;
	// device time of the last persistent solver kernel (roofline probe)
	cudaEvent_t solveKernelStart = nullptr, solveKernelEnd = nullptr;
	bool solveKernelTimed = false;
	cudaEvent_t markEvents[2] = {nullptr, nullptr};
	cudaEvent_t movedEvent = nullptr; // recorded behind the D2H copy of the moved-proxy counter at the end of every step
	cudaEvent_t finalizedEvent = nullptr; // recorded behind finalize's kernels: the side stream's copies wait for it
	// transforms are read back on a stream of their own when finalize was the last thing to write them: the read-back then
	// runs beside whatever the world's stream has queued behind finalize (the pair search of the next step) instead of after it
	cudaStream_t copyStream = nullptr;
	unsigned long long xfSeq = 0, finalizeSeq = ~0ull; // bumped by everything that writes body transforms / at the last finalize
	int sideCopies = 1;								   // S2B_SIDE_COPIES=0: all read-backs on the world's stream
	StageTimer timer;
	float stageMs[4] = {0, 0, 0, 0};

	DevArray<char> l2Flush;
};

inline BodyView bodyView(s2bWorld* w)
{
	BodyView v;
	v.vel = w->bVel.p;
	v.pose = w->bPose.p;
	v.pos = w->bPos.p;
	v.org = w->bOrg.p;
	v.frc = w->bFrc.p;
	v.prm = w->bPrm.p;
	v.aux0 = w->bAux0.p;
	v.aux1 = w->bAux1.p;
	v.flags = w->bFlags.p;
	v.capacity = w->bodyCap;
	return v;
}

inline ShapeView shapeView(s2bWorld* w)
{
	ShapeView v;
	v.head = w->sHead.p;
	v.filter = w->sFilter.p;
	v.aabb = w->sAabb.p;
	v.fat = w->sFat.p;
	v.fr = w->sFr.p;
	v.verts = w->sVerts.p;
	v.normals = w->sNormals.p;
	v.capacity = w->shapeCap;
	v.restitution = w->sRestitution.p;
	return v;
}

inline JointView jointView(s2bWorld* w)
{
	JointView v;
	v.head = w->jHead.p;
	v.anchors = w->jAnchors.p;
	v.lim = w->jLim.p;
	v.motor = w->jMotor.p;
	v.target = w->jTarget.p;
	v.imp = w->jImp.p;
	v.limp = w->jLimp.p;
	v.color = w->jColor.p;
	v.capacity = w->jointCap;
	return v;
}

// mailbox slots
enum
{
	MAIL_MOVED = 0,
	MAIL_CONSTRAINTS = 1,
	MAIL_GROUPS = 2,
	MAIL_OVERFLOW = 3,
	MAIL_NEW_PAIRS = 4,
	MAIL_KEPT = 5,
	MAIL_JOINTS = 6,
	MAIL_UNCOLORED = 7,
	MAIL_PAIR_OVERFLOW = 8,
	MAIL_REGIONS_ON = 9, // CNT_REGIONS_ON of the last schedule built outside a graph with regions on trial (a hint, read a step later)
	MAIL_COUNT = 64
};

inline int gridFor(int n, int block)
{
	return (n + block - 1) / block;
}

#define S2B_LAUNCH(world, kernel, grid, block, smem, ...)                                                              \
	do                                                                                                                 \
	{                                                                                                                  \
		kernel<<<(grid), (block), (smem), (world)->stream>>>(__VA_ARGS__);                                             \
		(world)->kernelLaunches += 1;                                                                                  \
	} while (0)

// stage entry points implemented in the other translation units
void s2bBroadphaseUpdatePairs(s2bWorld* w);
void s2bPrefetchPairSearch(s2bWorld* w);
float s2bLastPairSearchMs(s2bWorld* w);
void s2bNarrowphaseUpdate(s2bWorld* w);
void s2bSolve(s2bWorld* w, int solverType, const s2bStepContext* ctx);
void s2bFinalize(s2bWorld* w);
void s2bFreeSolverScratch(s2bWorld* w);
void s2bFreeBroadScratch(s2bWorld* w);
// continuous collision (broadphase.cu, DESIGN.md §3.11): the start poses before the solver stage, the sweep and clamp after it
// the bits of 1.0f: a per-body time of impact of "none" (a fraction is non-negative, so its bits order like the float)
#define S2B_FRACTION_ONE 0x3F800000u
void s2bContinuousSnapshot(s2bWorld* w);
void s2bContinuousPass(s2bWorld* w);
// the bullet pass (broadphase.cu, DESIGN.md §3.12): inside finalize, after its kernels and before the moved counter's copy
void s2bBulletPass(s2bWorld* w);
// (finalize.cu) boxes and fat-box moves of the listed shapes whose body has a fraction below 1, for its clamped pose; with
// `movedLeaves`, a shape that escapes its fat box only now is appended to the moved proxies finalize collected
void s2bRefinalizeBulletShapes(s2bWorld* w, const int* list, const int* count, const unsigned* fraction, const int* shapeLeaf,
							   int* movedLeaves, int* movedLeafCount);
// (broadphase.cu) finalize's shapes, the refit and the moved proxies of the next pair search in one launch, when that search
// will reuse the hierarchy's topology; false: nothing launched, finalize runs s2bFinalizeShapes (DESIGN.md §3.3)
bool s2bFinalizeRefit(s2bWorld* w);
// (reactions.cu, DESIGN.md §3.13) the reaction pass at the end of finalize, when some joint has a threshold
void s2bJointBreakPass(s2bWorld* w, cudaStream_t copyStream);
// [0] continuousShapes [1] continuousHits [2] bulletShapes [3] bulletHits of the last step
void s2bContinuousCounters(s2bWorld* w, int out[4]);
