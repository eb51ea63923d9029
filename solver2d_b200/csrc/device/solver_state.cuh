// solver2d-b200 — per-step solver scratch (constraint streams, colouring, group tables) and the argument block
// every solver kernel receives by value.
#pragma once

#include "s2b_internal.cuh"

// threads per block of the solver kernels
#define S2B_BLOCK 512
// colours of the constraint graph: 0..S2B_MAX_COLORS-1, or the serial overflow group
#define S2B_MAX_COLORS 64
#define S2B_OVERFLOW_KEY 255

// soft-constraint coefficients (reference src/solve_common.c:264-271)
struct SoftCoef
{
	float bias, mass, impulse;
};

// device-resident counters of the current solve (written by the set-up kernels, read by every later kernel, so the
// host never has to synchronise to learn them)
enum
{
	CNT_CONTACTS = 0,  // contact constraints (manifolds with >= 1 point)
	CNT_JOINTS = 1,	   // live joints
	CNT_GROUPS = 2,	   // parallel groups (colours / wavefront levels), excluding the serial overflow group
	CNT_OVERFLOW_C = 3, // contact constraints in the overflow group
	CNT_OVERFLOW_J = 4, // joints in the overflow group
	CNT_REMAINING = 5, // colouring work counters (three rotating slots: 5, 6, 7)
	CNT_ROUNDS = 8,
	CNT_UNCOLOURED = 9, // blocks that saw an uncoloured item at the start of the colouring kernel
	CNT_PRIMARY = 10,	// region-local schedule: colours used by interior constraints (0 = no regions)
	CNT_COLORS = 11,	// colours of the constraint graph (what s2bCounters.groupCount reports under the colour schedule)
	CNT_OWNED = 12,		// bodies that belong to a region (valid, not a hub)
	CNT_CUT = 13,		// constraints in the cut set (straddle two regions or touch a hub body)
	CNT_CUT_COLORS = 14, // colours the cut set needed
	CNT_REGIONS_ON = 15, // 1: the solve order is region-major (persistent.cuh); 0: one device-wide group per colour
	CNT_MAX_REGION = 21, // bodies in the largest region
	CNT_RESIDENT = 22,	 // 1: every region runs out of shared memory (persistent.cuh, "resident regions"); decided by s2bFinishGroups
	CNT_CUT_ABORT = 20,	// the cut colouring gave up: it needs more colours than regions are worth
	CNT_BOUNDS = 16,	// 4 slots: order-preserving keys of max x, max -x, max y, max -y over the bodies' centres
	CNT_NSYNC = 23,		// grid the neighbour tables were built for: device-wide colour steps wait for neighbouring blocks only; 0 = off
	CNT_KINEMATIC_ITEMS = 24, // constraints with an endpoint no constraint moves but whose pose changes (kinematic, s2bItemEndpoints -2)
	CNT_ROWS_READY = 25, // 1: the narrow phase wrote this solve's contact rows, prepare leaves them (narrowphase.cu, s2bScheduleGate)
	CNT_FIRST_TABLE = 26, // grid the first-touch table (ConstraintView::firstTable) was built for; 0 = none or unusable
	CNT_FIRST_TABLE_BLOCKS = 27, // blocks whose copy of the table fits the budget (the others gather per thread)
	CNT_SIZE = 32
};

// ConstraintView::firstTable, one int array: [4 b, 4 b + 4) = block b's header {index of its first slot's body, slots (-1: over
// budget, the block gathers per thread), index of its first slot's entry offset, index of its first entry}; then per slot the body, then
// per slot + 1 the offset of the slot's entries (running sum), then the entries (incidence entries in list order)
#define S2B_FT_HEADER (4 * 512)
// shared memory of one slot (body, flags, parameters, forces, entry range) and of one entry (the entry and its side's anchors)
// of a block's copy (persistent.cuh, S2bFirstTableShared)
#define S2B_FT_SLOT_BYTES 48
#define S2B_FT_ENTRY_BYTES 20

// Device-wide group steps: block b runs items [b * share, (b + 1) * share) of a group of n items (its joints, then its
// contacts). Every block gets work and a warp's rows stay contiguous (coalesced column loads). The neighbour tables
// (solver.cu, s2bItemBlockKernel) are built from the same mapping.
__host__ __device__ __forceinline__ int s2bGroupShare(int n, int blocks)
{
	return ((n + blocks - 1) / blocks + 31) & ~31;
}

// neighbour-synchronised colour steps (persistent.cuh): per block, the number of its neighbours, then up to S2B_NSYNC_K ids
#define S2B_NSYNC_K 16
#define S2B_NSYNC_STRIDE (S2B_NSYNC_K + 1)
// distinct blocks one body's constraints may be spread over before the mode gives up (a hub)
#define S2B_NSYNC_BODY_BLOCKS 8
// SolveArgs::barrier layout: [64 + 32 b] = epoch of block b (one 128-byte line each), [33] = epoch at the next launch's start
#define S2B_EPOCH_BASE_WORD 33
#define S2B_EPOCH_WORD(b) (64 + 32 * (b))
#define S2B_BARRIER_WORDS S2B_EPOCH_WORD(512)

struct SolveArgs
{
	BodyView bodies;
	ContactView contacts;
	JointView joints;
	ConstraintView cc;
	JointConstraintView jc;
	const int* counts;	  // CNT_*
	const int* cGroupOff; // contact-constraint group offsets, CNT_GROUPS + 2 entries (last group = overflow)
	const int* jGroupOff; // joint-constraint group offsets, same shape
	const int* incStart;  // per body: range of its incidence list (warm_gather.cuh); null when the gather is not used
	const int* incList;	  // incidence entries sorted by solve order
	const int* heavyBodies; // [0] count, then body indices with more than S2B_HEAVY_DEGREE incident items (null = none split off)
	// region-local schedule of the persistent kernel (persistent.cuh); regions == 0: every group is device-wide
	int regions;			 // number of regions = blocks of the persistent kernel
	const int* regBodyStart; // regions + 1: range of each region in regBodies
	const int* regBodies;	 // body slots sorted by region (Hilbert order of their centres)
	const int* jRegOff;		 // regions x (S2B_MAX_COLORS + 1): joint-constraint stream offsets of (region, colour)
	const int* cRegOff;		 // same for contact constraints
	const int* bodyLocal;	 // per body: its position in its region's slice of regBodies (resident regions); null: not offered
	unsigned* barrier;		 // [0] monotonic arrival counter of the grid barrier, [32] its value at the start of the next launch;
							 // epochs of the neighbour-synchronised colour steps: S2B_EPOCH_WORD(b), S2B_EPOCH_BASE_WORD
	const int* nsyncNbr;	 // per block: S2B_NSYNC_STRIDE entries, neighbour count then neighbour blocks (used when CNT_NSYNC == grid)
	// serial overflow group on a shared-memory copy of its bodies (persistent.cuh): the distinct bodies its constraints touch
	const int* ovBodies;	 // [0] count, then body slots (null: walk in global memory)
	const int* ovBodySlot;	 // per body: position in that list, or -1
	// ticketed ("dataflow") Gauss-Seidel passes: null when the passes synchronise with grid barriers instead
	int* bodyTicket; // per body: incident-item executions completed in this launch
	union
	{
		struct
		{
			const int2 *cFlowA, *cFlowB; // per contact constraint and side: {ordinal in the body's incidence list, its degree} or -1
			const int2 *jFlowA, *jFlowB; // same per joint constraint
		};
		// The restitution pass (DESIGN.md §3.7) runs without tickets, so its inputs share these slots: SolveArgs, and with it
		// the parameter layout and stack frame of every variant's kernel, stays the size it is without restitution.
		struct
		{
			const float4* restVr;	// per contact slot, captured at the start of the stage: vr0 vr1 normalMass0 normalMass1
			const float4* restR[2]; // per contact slot: rA.xy rB.xy of point 0 / 1
			float restitutionThreshold;
		};
	};
	unsigned long long* trace; // diagnostic: block 0 stamps %globaltimer after every grid barrier (null = off)
	int traceCap;
	int flowSleepNs;			   // back-off between polls (0 = none)
	int* flowError;				   // set when a wait ran into its spin limit (a bug, never expected)
	s2bStepContext ctx;
	float2 gravity;
	SoftCoef softDynamic; // contact, both bodies movable
	SoftCoef softStatic;  // contact against a body with zero inverse mass (doubled hertz)
	SoftCoef softJoint;
	float contactHertz;
	float jointHertz;
	float xpbdInvH;
	int solverType;
	int sticky;
};

struct SolverScratch
{
	// set-up
	DevArray<int> counts;		  // CNT_SIZE
	DevArray<int> activeFlag;	  // per contact slot: manifold has points
	DevArray<int> activeSlots;	  // compacted contact slots, natural order
	DevArray<int> jointFlag;	  // per joint slot: live
	DevArray<int> jointSlots;	  // compacted joint slots, natural order
	DevArray<int2> itemBodies;	  // per item (joints first, then contacts): conflict endpoints or -1
	DevArray<int> degree;		  // per body
	DevArray<int> adjStart;		  // per body + 1
	DevArray<int> adjCursor;	  // per body
	DevArray<int> adj;			  // 2 * items
	DevArray<int> colorA, colorB; // per item: colour, tentative colour of the speculative rounds
	DevArray<int> colorC;		  // per item: colour inside the cut set
	DevArray<int> kempeState, kempeClaim, kempePath; // s2bKempeKernel: KS_* words, per-body claims, recorded chains
	DevArray<int> itemRegion;	  // per item: region it is interior to, or -1 (cut set)
	DevArray<unsigned short> sortKeyIn, sortKeyOut; // solve-order keys (region x colour | cut colour | overflow), see s2bMakeSortKeys
	// regions
	DevArray<unsigned long long> bodyKeyIn, bodyKeyOut; // (island, Hilbert position) keys of the bodies
	DevArray<int> bodyValIn, bodySorted;	  // body slots, unsorted / sorted by key
	DevArray<int> regBodies;				  // body slots grouped by region
	DevArray<int> islandParent;				  // union-find forest over the body slots
	DevArray<int> island;					  // per body: label of its island (smallest body slot in it)
	DevArray<int> islandSize, islandStart;	  // per label: bodies in the island, its first rank in the sorted order
	DevArray<int> regCount;					  // [0, 512): bodies per region; [512, 1024): fill cursors
	DevArray<int> bodyRegion;				  // per body: region or -1 (hub, invalid)
	DevArray<int> bodyLocal;				  // per body: position in its region's list (SolveArgs::bodyLocal)
	DevArray<int> regBodyStart;				  // regions + 1
	DevArray<int> cRegOff, jRegOff;			  // regions x (S2B_MAX_COLORS + 1)
	int regions = 0;						  // regions of the last schedule (0: none)
	DevArray<int> sortValIn, sortValOut;
	DevArray<int> cGroupOff, jGroupOff; // maxGroups + 2
	DevArray<int> cPerm;				// solve position -> natural contact-constraint index
	DevArray<int> jPerm;
	DevArray<char> cubTemp;
	DevArray<unsigned long long> itemVal, incWork; // warm-start gather: per-item sort value, per-body sort scratch
	DevArray<int> incList;
	DevArray<int> lastTouch; // ConstraintView::lastTouch
	DevArray<int> firstTable;		// ConstraintView::firstTable
	DevArray<int> ftRowSlot, ftDegree; // its build: per colour-0 row its first slot (running sum), per slot the body's degree
	DevArray<int> heavyBodies;
	DevArray<int> longBodies;			// [0] count, then bodies whose incidence list is sorted by a whole block
	DevArray<int> ovBodies, ovBodySlot; // bodies of the serial overflow group (SolveArgs::ovBodies)
	DevArray<int> itemBlock;			// per item: block that runs it in its device-wide colour step (-1: overflow group)
	DevArray<unsigned> nsyncBits;		// grid x words block adjacency bits, + 1 word: "the mode cannot be used"
	DevArray<int> nsyncNbr;				// SolveArgs::nsyncNbr
	DevArray<int2> flow;	  // cFlowA | cFlowB | jFlowA | jFlowB
	DevArray<int> bodyTicket; // + 1 int error flag at the end
	int flowErrorOffset = 0;
	DevArray<unsigned long long> trace; // [0] = number of stamps, then (code << 48 | ns) entries
	int traceCap = 0;
	int maxGroups = 0;

	// contact constraint columns
	DevArray<int2> idx;
	DevArray<float4> nf;
	DevArray<float4> anchor[2], pm[2], r0[2], fanchor[2];
	DevArray<float2> lambda[2], tsep[2];
	DevArray<float> sep[2];
	DevArray<int> src;
	DevArray<int> rowOf; // per contact slot: its row in the solve order (the inverse of src), -1: none; built with the schedule
	DevArray<float4> warmP, warmAnchor; // ConstraintView::warmP (1 per constraint), ::warmAnchor (2 per constraint)
	// restitution capture, per contact slot (SolveArgs::restVr / restR); allocated while restitution is enabled
	DevArray<float4> restVr, restR[2];

	// joint constraint columns
	DevArray<int4> jhead;
	DevArray<float4> janchor, jmass, jd0ax, jlim, jmotor, jcoef, jpivot, jimp, jlimp;

	// CUDA graph of the whole solver stage (set-up kernels + persistent kernel), replayed while nothing it depends on
	// changes: see s2bSolve
	cudaGraphExec_t graphExec = nullptr;
	std::vector<unsigned char> graphSig, graphCandidate;
	std::vector<unsigned char> scheduleSig; // signature the schedule buffers were last built for
	int graphLaunches = 0;
	bool graphDisabled = false;
	int graphReplays = 0, graphCaptures = 0;
	// regions on trial (useRegions == 1) and found useless (hub bodies, a cut set that needs too many colours): the rebuilds
	// of the next S2B_REGION_RETRY schedules do not build islands, Hilbert keys and the cut colouring only to drop them
	int regionSkip = 0;
	bool regionVerdictPending = false;
	int stepsSinceEager = 0; // solves since the last one that rebuilt the schedule outside the graph (how quiet the scene is)

	// argument block of the last solve (the per-colour kernel probe re-launches one of its passes)
	SolveArgs lastArgs;
	const int* lastJointSlots = nullptr;
	const int* lastJPerm = nullptr;
	bool lastArgsValid = false;
	// where the next step's narrow phase may write the contact rows (s2bNarrowphaseRows): those of the last solve that ran,
	// eager or a graph replay (then the ones the graph was captured with)
	struct RowTarget
	{
		SolveArgs args;
		int kind = -1; // prepare kind of the solve's program; -1: the solve cannot take rows from the narrow phase
		int cur = 0, contactCount = 0;			   // the contact table and allocations it was planned for
		unsigned long long tableVersion = 0, epoch = 0;
	};
	RowTarget rows, graphRows;

	// host mirrors (valid when the last solve synchronised: multi-launch and wavefront modes)
	int hostContacts = 0, hostJoints = 0, hostGroups = 0, hostOverflowC = 0, hostOverflowJ = 0;
	bool hostCountsValid = false;
	std::vector<int> hostCGroupOff, hostJGroupOff;
};

SolverScratch* s2bGetSolverScratch(s2bWorld* w);

// schedDirty words (s2b_internal.cuh): [0] rebuild wanted, [1..3] the Kempe pass's view of the recent past, [4] solves whose
// contact rows came from the narrow phase (s2bCounters::narrowphaseRowSteps); see s2bScheduleGate
#define S2B_SCHED_ROW_STEPS 4
#define S2B_SCHED_WORDS 8

// The prepare kind (PREPARE_SOFT / PREPARE_COLD) the narrow phase writes this step's contact rows with, into *args' columns
// at the rows *rowOf names; -1: it writes none. *rowsReady: where it says whether it did (counts[CNT_ROWS_READY], null before
// the first solve); s2bScheduleGate decides whether the solver then uses them.
int s2bNarrowphaseRows(s2bWorld* w, SolveArgs* args, const int** rowOf, int** rowsReady);
