// solver2d-b200 — stages 1+2 (and the destroy half of stage 3) of s2World_Step on the device.
//
// Replaces s2UpdateBroadPhasePairs / s2FindPairs / s2PairQueryCallback (reference src/broad_phase.c:166-367), the three
// incrementally-updated dynamic AABB trees (src/dynamic_tree.c) with their rebuild (broad_phase.c:381-385), the pair
// hash set (src/table.c) and the fat-AABB overlap test + s2DestroyContact of world.c:149-166.
//
// GPU-first design instead of a port of the pointer-chasing tree:
//   * a linear BVH (Morton order + Karras radix tree, collapsed into a tree of up to 8 children per node) over ALL proxies
//     is rebuilt from scratch, fully in parallel, every 17th pass or when the host created/destroyed something, and
//     refitted in the passes in between;
//   * one thread per *moved* proxy walks the BVH and applies the reference's pair rules (both-moved de-duplication by
//     proxy key, body-type rules of the three-tree query, existing pair, same body, filter, joint override, shape-type
//     table) — so the set of created contacts equals the reference's;
//   * existing contacts whose fat AABBs stopped overlapping are dropped, survivors and new pairs are merged by a radix
//     sort on the 64-bit shape-pair key and all contact columns are gathered into the other column set.
// The contact table is therefore always sorted by pair key: the device's natural (wavefront) constraint order.
#include "s2b_internal.cuh"

#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>

struct BroadScratch
{
	DevArray<int> validFlag;	   // per shape slot
	DevArray<int> leafShape;	   // compacted valid shapes
	DevArray<unsigned> mortonIn, mortonOut;
	DevArray<int> leafIn, leafOut; // sorted leaf -> index into leafShape
	DevArray<int> counters;		   // [0] leaf count [1] new pair count [2] kept count [3] bounds ready ...
	DevArray<int> boundsBits;	   // 4 ordered-int encoded floats: min.x min.y max.x max.y
	DevArray<int2> children;	   // binary internal nodes
	DevArray<int> parent;		   // all binary nodes (internal [0,n-1), leaves [n-1, 2n-1))
	// the wide hierarchy (s2bBuildWide): a wide node is kept at the index of the binary node it was collapsed from
	DevArray<float4> wideBox;	   // S2B_WIDE per wide node: the boxes of its children, adjacent
	DevArray<int> wideChild;	   // S2B_WIDE per wide node: wide node index, ~shape for a leaf, S2B_WIDE_EMPTY
	DevArray<int> wideCount;	   // children per wide node
	DevArray<int> wideSlot;		   // per binary node: slot (wide parent * S2B_WIDE + i) it occupies, -1 for the root
	DevArray<int> visit;		   // refit arrival counters (wide nodes); the last arriver resets its counter
	DevArray<float4> rootBox;	   // box of the whole scene
	DevArray<int> movedLeaves;	   // sorted-leaf indices of moved proxies
	DevArray<int> movedFlag;
	DevArray<int> largeShapes;	   // shapes of moved proxies with scene-sized boxes
	DevArray<unsigned long long> newKey;
	DevArray<int2> newShapes;
	DevArray<int> keepFlag, keepSlots;
	DevArray<unsigned long long> mergeKeyIn, mergeKeyOut;
	DevArray<int> mergeSrcIn, mergeSrcOut;
	DevArray<char> cubTemp;
	int newPairCap = 0;
	// the hierarchy of the last pass: while no shape was created, destroyed or re-uploaded its TOPOLOGY is reused and only
	// the boxes are refitted (boxes drift a little per step; a periodic rebuild keeps the tree tight)
	bool treeValid = false;
	int treeShapeCap = 0;
	int treeReuses = 0;
	// open-addressing hash set of the shape-pair keys of the current contact table ("does this pair already exist?")
	DevArray<unsigned long long> pairHash;
	unsigned long long hashMask = 0;
	unsigned long long hashVersion = ~0ull; // contact table version the set was built from
	// pair search started behind the previous step (s2bPrefetchPairSearch)
	bool prefetched = false;	   // a search is in flight / finished and not consumed yet
	bool lastPassRan = false;	   // the last pass found moved proxies (the scene is in motion)
	bool searchTimed = false;
	unsigned long long prefetchEpoch = 0, searchedVersion = 0;
	int searchedCount = 0;
	size_t prefetchTempBytes = 0;
	cudaEvent_t evSearch[2] = {nullptr, nullptr};
	cudaEvent_t searchDone = nullptr;
};

#define S2B_TREE_REUSE_LIMIT 16

static BroadScratch* getBroad(s2bWorld* w)
{
	if (w->broad == nullptr)
	{
		w->broad = new BroadScratch();
	}
	return w->broad;
}

void s2bFreeBroadScratch(s2bWorld* w)
{
	BroadScratch* b = w->broad;
	if (b == nullptr)
	{
		return;
	}
	b->validFlag.release();
	b->leafShape.release();
	b->mortonIn.release();
	b->mortonOut.release();
	b->leafIn.release();
	b->leafOut.release();
	b->counters.release();
	b->boundsBits.release();
	b->children.release();
	b->parent.release();
	b->wideBox.release();
	b->wideChild.release();
	b->wideCount.release();
	b->wideSlot.release();
	b->visit.release();
	b->rootBox.release();
	b->movedLeaves.release();
	b->movedFlag.release();
	b->newKey.release();
	b->newShapes.release();
	b->keepFlag.release();
	b->keepSlots.release();
	b->mergeKeyIn.release();
	b->mergeKeyOut.release();
	b->mergeSrcIn.release();
	b->mergeSrcOut.release();
	b->cubTemp.release();
	b->largeShapes.release();
	b->pairHash.release();
	for (int i = 0; i < 2; ++i)
	{
		if (b->evSearch[i] != nullptr)
		{
			cudaEventDestroy(b->evSearch[i]);
		}
	}
	if (b->searchDone != nullptr)
	{
		cudaEventDestroy(b->searchDone);
	}
	delete b;
	w->broad = nullptr;
}

enum
{
	// set when the hierarchy is built, kept while it is reused
	BC_LEAVES = 0,
	BC_HEIGHT = 1, // height of the binary hierarchy
	// cleared by every pass
	BC_NEW_PAIRS = 2,
	BC_KEPT = 3,
	BC_MOVED = 4,
	BC_LARGE = 5, // moved proxies handled by the leaf-side query
	BC_SIZE = 8
};

// The hierarchy the refit and the queries walk is WIDE: the binary radix tree collapsed so that a wide node stands for
// S2B_WIDE_LEVELS binary levels (up to S2B_WIDE children). A query visiting a wide node reads the boxes of all its
// children with one contiguous 8 x 16 B = 128 B access (one L2 line), and both walks climb a third of the levels.
#define S2B_WIDE_LEVELS 3
#define S2B_WIDE (1 << S2B_WIDE_LEVELS)
#define S2B_WIDE_EMPTY (-0x7FFFFFFF - 1) // unused child slot
// Depth bound of the radix tree: every internal node's keys share a longer common prefix than its parent's, and the
// prefix of the (31-bit Morton code, 32-bit position) keys is 1..63 bits, so internal nodes lie at binary depth 0..62.
// Wide nodes sit at binary depths 0, 3, ..., 60: at most 21 wide levels.
#define S2B_MAX_INTERNAL_DEPTH 62
#define S2B_MAX_WIDE_DEPTH (S2B_MAX_INTERNAL_DEPTH / S2B_WIDE_LEVELS)
// A query descends into one overlapping wide child and stacks the others: it stacks at most S2B_WIDE - 1 nodes of each
// depth 1..S2B_MAX_WIDE_DEPTH, and a stacked node is popped before anything of a smaller depth. The stack never holds more
// than that, so no node is ever dropped.
#define S2B_QUERY_STACK ((S2B_WIDE - 1) * S2B_MAX_WIDE_DEPTH)

// ---------------------------------------------------------------------------------------------------------------
// helpers
// ---------------------------------------------------------------------------------------------------------------

__device__ __forceinline__ int s2bFloatToOrdered(float f)
{
	int i = __float_as_int(f);
	return i >= 0 ? i : i ^ 0x7FFFFFFF;
}

__device__ __forceinline__ float s2bOrderedToFloat(int i)
{
	return __int_as_float(i >= 0 ? i : i ^ 0x7FFFFFFF);
}

__device__ __forceinline__ unsigned s2bExpandBits(unsigned v)
{
	// 16 bits -> every other bit of 32
	v &= 0xFFFFu;
	v = (v | (v << 8)) & 0x00FF00FFu;
	v = (v | (v << 4)) & 0x0F0F0F0Fu;
	v = (v | (v << 2)) & 0x33333333u;
	v = (v | (v << 1)) & 0x55555555u;
	return v;
}

__device__ __forceinline__ bool s2bBoxesOverlap(float4 a, float4 b)
{
	// s2AABB_Overlaps (reference include/solver2d/aabb.h:111-123): closed test
	float d1x = b.x - a.z, d1y = b.y - a.w;
	float d2x = a.x - b.z, d2y = a.y - b.w;
	if (d1x > 0.0f || d1y > 0.0f)
	{
		return false;
	}
	if (d2x > 0.0f || d2y > 0.0f)
	{
		return false;
	}
	return true;
}

// s2ShouldShapesCollide (reference src/contact.h:70-79)
__device__ __forceinline__ bool s2bShouldShapesCollide(int4 fa, int4 fb)
{
	if (fa.z == fb.z && fa.z != 0)
	{
		return fa.z > 0;
	}
	return ((unsigned)fa.y & (unsigned)fb.x) != 0 && ((unsigned)fa.x & (unsigned)fb.y) != 0;
}

// joints with collideConnected == false override collision (replaces the joint-list walk of s2ShouldBodiesCollide,
// reference src/body.c:386-417) — binary search in the sorted body-pair keys uploaded by the host
__device__ __forceinline__ bool s2bJointOverride(const unsigned long long* keys, int count, int bodyA, int bodyB)
{
	if (count == 0)
	{
		return false;
	}
	unsigned long long lo = (unsigned long long)(bodyA < bodyB ? bodyA : bodyB);
	unsigned long long hi = (unsigned long long)(bodyA < bodyB ? bodyB : bodyA);
	unsigned long long key = (lo << 32) | hi;
	int l = 0, r = count;
	while (l < r)
	{
		int m = (l + r) >> 1;
		if (keys[m] < key)
		{
			l = m + 1;
		}
		else
		{
			r = m;
		}
	}
	return l < count && keys[l] == key;
}

// pair-key hash set (replaces an 18-step binary search per candidate pair by one or two probes)
__device__ __forceinline__ unsigned long long s2bMix64(unsigned long long x)
{
	x ^= x >> 33;
	x *= 0xff51afd7ed558ccdull;
	x ^= x >> 33;
	x *= 0xc4ceb9fe1a85ec53ull;
	x ^= x >> 33;
	return x;
}

__global__ void s2bBuildPairHash(const unsigned long long* keys, int count, unsigned long long* table, unsigned long long mask)
{
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= count)
	{
		return;
	}
	unsigned long long key = keys[i];
	unsigned long long slot = s2bMix64(key) & mask;
	for (;;)
	{
		unsigned long long prev = atomicCAS(table + slot, ~0ull, key);
		if (prev == ~0ull || prev == key)
		{
			return;
		}
		slot = (slot + 1) & mask;
	}
}

__device__ __forceinline__ bool s2bPairInHash(const unsigned long long* table, unsigned long long mask, unsigned long long key)
{
	unsigned long long slot = s2bMix64(key) & mask;
	for (;;)
	{
		unsigned long long v = table[slot];
		if (v == key)
		{
			return true;
		}
		if (v == ~0ull)
		{
			return false;
		}
		slot = (slot + 1) & mask;
	}
}

__device__ __forceinline__ bool s2bKeyExists(const unsigned long long* keys, int count, unsigned long long key)
{
	int l = 0, r = count;
	while (l < r)
	{
		int m = (l + r) >> 1;
		if (keys[m] < key)
		{
			l = m + 1;
		}
		else
		{
			r = m;
		}
	}
	return l < count && keys[l] == key;
}

// manifold function table of the reference (src/contact.c:139-154): is (typeA, typeB) a primary pair, a flipped pair,
// or not collidable at all (segment vs segment)?
// returns 0 = none, 1 = primary, 2 = flip
__device__ __forceinline__ int s2bPairKind(int t1, int t2)
{
	// primary pairs: (circle,circle) (capsule,circle) (capsule,capsule) (polygon,circle) (polygon,capsule)
	// (polygon,polygon) (segment,circle) (segment,capsule) (segment,polygon)
	const int CAP = S2B_SHAPE_CAPSULE, CIR = S2B_SHAPE_CIRCLE, POL = S2B_SHAPE_POLYGON, SEG = S2B_SHAPE_SEGMENT;
	if (t1 == SEG && t2 == SEG)
	{
		return 0;
	}
	bool primary = (t1 == CIR && t2 == CIR) || (t1 == CAP && t2 == CIR) || (t1 == CAP && t2 == CAP) || (t1 == POL && t2 == CIR) ||
				   (t1 == POL && t2 == CAP) || (t1 == POL && t2 == POL) || (t1 == SEG && t2 != SEG);
	return primary ? 1 : 2;
}

// ---------------------------------------------------------------------------------------------------------------
// BVH build
// ---------------------------------------------------------------------------------------------------------------

__global__ void s2bFlagValidShapes(ShapeView s, int* validFlag)
{
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < s.capacity)
	{
		validFlag[i] = (s.head[i].x & S2B_ROW_VALID) ? 1 : 0;
	}
}

__global__ void s2bSceneBounds(ShapeView s, const int* leafShape, const int* counters, int* boundsBits)
{
	int n = counters[BC_LEAVES];
	int k = blockIdx.x * blockDim.x + threadIdx.x;
	float minx = 3.0e38f, miny = 3.0e38f, maxx = -3.0e38f, maxy = -3.0e38f;
	if (k < n)
	{
		float4 f = s.fat[leafShape[k]];
		float cx = 0.5f * (f.x + f.z), cy = 0.5f * (f.y + f.w);
		minx = maxx = cx;
		miny = maxy = cy;
	}
	for (int o = 16; o > 0; o >>= 1)
	{
		minx = fminf(minx, __shfl_xor_sync(0xFFFFFFFFu, minx, o));
		miny = fminf(miny, __shfl_xor_sync(0xFFFFFFFFu, miny, o));
		maxx = fmaxf(maxx, __shfl_xor_sync(0xFFFFFFFFu, maxx, o));
		maxy = fmaxf(maxy, __shfl_xor_sync(0xFFFFFFFFu, maxy, o));
	}
	if ((threadIdx.x & 31) == 0)
	{
		atomicMin(boundsBits + 0, s2bFloatToOrdered(minx));
		atomicMin(boundsBits + 1, s2bFloatToOrdered(miny));
		atomicMax(boundsBits + 2, s2bFloatToOrdered(maxx));
		atomicMax(boundsBits + 3, s2bFloatToOrdered(maxy));
	}
}

__global__ void s2bMortonCodes(ShapeView s, const int* leafShape, const int* counters, const int* boundsBits, unsigned* morton,
							   int* leafIndex, int capacity)
{
	int n = counters[BC_LEAVES];
	int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= capacity)
	{
		return;
	}
	if (k >= n)
	{
		morton[k] = 0xFFFFFFFFu; // padding sorts last
		leafIndex[k] = k;
		return;
	}
	float minx = s2bOrderedToFloat(boundsBits[0]), miny = s2bOrderedToFloat(boundsBits[1]);
	float maxx = s2bOrderedToFloat(boundsBits[2]), maxy = s2bOrderedToFloat(boundsBits[3]);
	float4 f = s.fat[leafShape[k]];
	float cx = 0.5f * (f.x + f.z), cy = 0.5f * (f.y + f.w);
	float ex = fmaxf(maxx - minx, 1.0e-6f), ey = fmaxf(maxy - miny, 1.0e-6f);
	float ux = fminf(fmaxf((cx - minx) / ex, 0.0f), 1.0f);
	float uy = fminf(fmaxf((cy - miny) / ey, 0.0f), 1.0f);
	unsigned qx = (unsigned)(ux * 32767.0f), qy = (unsigned)(uy * 32767.0f);
	morton[k] = (s2bExpandBits(qx) | (s2bExpandBits(qy) << 1)) & 0x7FFFFFFFu;
	leafIndex[k] = k;
}

// common-prefix length of sorted keys i and j; ties on the code are broken by the position (Karras 2012)
__device__ __forceinline__ int s2bDelta(const unsigned* codes, int n, int i, int j)
{
	if (j < 0 || j >= n)
	{
		return -1;
	}
	unsigned a = codes[i], b = codes[j];
	if (a == b)
	{
		return 32 + __clz((unsigned)i ^ (unsigned)j);
	}
	return __clz(a ^ b);
}

__global__ void s2bBuildRadixTree(const unsigned* codes, const int* counters, int2* children, int* parent)
{
	int n = counters[BC_LEAVES];
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n - 1)
	{
		return;
	}
	int d = (s2bDelta(codes, n, i, i + 1) - s2bDelta(codes, n, i, i - 1)) >= 0 ? 1 : -1;
	int deltaMin = s2bDelta(codes, n, i, i - d);
	int lmax = 2;
	while (s2bDelta(codes, n, i, i + lmax * d) > deltaMin)
	{
		lmax <<= 1;
	}
	int l = 0;
	for (int t = lmax >> 1; t >= 1; t >>= 1)
	{
		if (s2bDelta(codes, n, i, i + (l + t) * d) > deltaMin)
		{
			l += t;
		}
	}
	int j = i + l * d;
	int deltaNode = s2bDelta(codes, n, i, j);
	int s = 0;
	int t = l;
	do
	{
		t = (t + 1) >> 1;
		if (s2bDelta(codes, n, i, i + (s + t) * d) > deltaNode)
		{
			s += t;
		}
	} while (t > 1);
	int gamma = i + s * d + min(d, 0);
	int left = min(i, j) == gamma ? (n - 1) + gamma : gamma;
	int right = max(i, j) == gamma + 1 ? (n - 1) + gamma + 1 : gamma + 1;
	children[i] = make_int2(left, right);
	parent[left] = i;
	parent[right] = i;
	if (i == 0)
	{
		parent[0] = -1;
	}
}

// one child of wide node `wide`: the binary descendant `node`, `levels` binary levels further down at most. Binary nodes
// in between are expanded (left to right), so the children keep Morton order.
template <int levels>
__device__ __forceinline__ void s2bWideChildren(int wide, int node, int n, const int2* children, const int* leafShape, const int* sortedLeaf,
												int* wideChild, int* wideSlot, int& count)
{
	bool leaf = node >= n - 1;
	if constexpr (levels > 0)
	{
		if (leaf == false)
		{
			int2 ch = children[node];
			s2bWideChildren<levels - 1>(wide, ch.x, n, children, leafShape, sortedLeaf, wideChild, wideSlot, count);
			s2bWideChildren<levels - 1>(wide, ch.y, n, children, leafShape, sortedLeaf, wideChild, wideSlot, count);
			return;
		}
	}
	int slot = wide * S2B_WIDE + count;
	wideChild[slot] = leaf ? ~leafShape[sortedLeaf[node - (n - 1)]] : node;
	wideSlot[node] = slot;
	count += 1;
}

// Collapse the binary radix tree into the wide hierarchy, one thread per binary internal node. The binary nodes at a depth
// divisible by S2B_WIDE_LEVELS become wide nodes (kept at their binary index); their children are their descendants
// S2B_WIDE_LEVELS levels down, or the leaves met before. The binary height (deepest leaf) is taken here once per build:
// the refit no longer visits the binary tree.
__global__ void s2bBuildWide(const int* leafShape, const int* sortedLeaf, int* counters, const int2* children, const int* parent,
							 int* wideChild, int* wideCount, int* wideSlot)
{
	int n = counters[BC_LEAVES];
	int u = blockIdx.x * blockDim.x + threadIdx.x;
	if (u >= n - 1)
	{
		return;
	}
	int depth = 0;
	for (int p = parent[u]; p >= 0; p = parent[p])
	{
		depth += 1;
	}
	int2 ch = children[u];
	if (ch.x >= n - 1 || ch.y >= n - 1)
	{
		atomicMax(counters + BC_HEIGHT, depth + 1);
	}
	if (depth % S2B_WIDE_LEVELS != 0)
	{
		return;
	}
	int count = 0;
	s2bWideChildren<S2B_WIDE_LEVELS - 1>(u, ch.x, n, children, leafShape, sortedLeaf, wideChild, wideSlot, count);
	s2bWideChildren<S2B_WIDE_LEVELS - 1>(u, ch.y, n, children, leafShape, sortedLeaf, wideChild, wideSlot, count);
	wideCount[u] = count;
	for (int i = count; i < S2B_WIDE; ++i)
	{
		wideChild[u * S2B_WIDE + i] = S2B_WIDE_EMPTY;
	}
	if (u == 0)
	{
		wideSlot[0] = -1;
	}
}

// Boxes bottom-up: a leaf thread writes its fat box into its slot in the parent wide node and counts its arrival; the last
// child to arrive resets the counter for the next pass, unions the node's child boxes and carries that box one level up.
__global__ void s2bRefit(ShapeView s, const int* leafShape, const int* sortedLeaf, const int* counters, const int* wideCount,
						 const int* wideSlot, float4* wideBox, int* visit, float4* rootBox)
{
	int n = counters[BC_LEAVES];
	int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= n)
	{
		return;
	}
	float4 box = s.fat[leafShape[sortedLeaf[k]]];
	if (n == 1)
	{
		rootBox[0] = box;
		return;
	}
	int slot = wideSlot[(n - 1) + k];
	for (;;)
	{
		int p = slot / S2B_WIDE;
		int count = wideCount[p];
		wideBox[slot] = box;
		__threadfence();
		if (atomicAdd(visit + p, 1) != count - 1)
		{
			return; // a sibling arrives later and finishes this node
		}
		visit[p] = 0;
		// L2 reads: the siblings published their boxes before their atomicAdd (threadfence above), L1 may not have them
		const float4* b = wideBox + p * S2B_WIDE;
		box = __ldcg(b);
#pragma unroll
		for (int i = 1; i < S2B_WIDE; ++i)
		{
			if (i < count)
			{
				float4 c = __ldcg(b + i);
				box = make_float4(fminf(box.x, c.x), fminf(box.y, c.y), fmaxf(box.z, c.z), fmaxf(box.w, c.w));
			}
		}
		slot = wideSlot[p];
		if (slot < 0)
		{
			rootBox[0] = box;
			return;
		}
	}
}

// ---------------------------------------------------------------------------------------------------------------
// pair queries
// ---------------------------------------------------------------------------------------------------------------

// append `value` to list[] (length in *count) for every thread with take == true: one atomic per BLOCK, and the block's
// entries keep their thread order (every thread of the block has to call this)
__device__ __forceinline__ void s2bBlockAppend(bool take, int value, int* list, int* count)
{
	__shared__ int warpOffset[32];
	__shared__ int blockBase;
	unsigned takers = __ballot_sync(0xFFFFFFFFu, take);
	int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	if (lane == 0)
	{
		warpOffset[warp] = __popc(takers);
	}
	__syncthreads();
	if (threadIdx.x == 0)
	{
		int total = 0;
		int warps = (blockDim.x + 31) >> 5;
		for (int k = 0; k < warps; ++k)
		{
			int c = warpOffset[k];
			warpOffset[k] = total;
			total += c;
		}
		blockBase = total > 0 ? atomicAdd(count, total) : 0;
	}
	__syncthreads();
	if (take)
	{
		list[blockBase + warpOffset[warp] + __popc(takers & ((1u << lane) - 1u))] = value;
	}
}

// The queries of this pass: the sorted-leaf indices of the proxies that moved (BC_MOVED, movedLeaves) — neighbours in Morton
// order stay neighbours in the list, a warp's queries walk the same part of the tree — except up to S2B_MAX_LARGE_MOVERS
// proxies with LARGE boxes (a container wall spanning the scene overlaps thousands of leaves: one thread walking them all
// takes milliseconds), which go to largeShapes (BC_LARGE) and are tested the other way round: every leaf against that short
// list (s2bFindPairsLarge). One kernel, one atomic per block (round 1: flag array + split + cub select).
#define S2B_MAX_LARGE_MOVERS 64

__global__ void s2bCollectMovers(ShapeView s, const int* leafShape, const int* sortedLeaf, int* counters, const float4* rootBox, int* movedLeaves,
								 int* largeShapes)
{
	int n = counters[BC_LEAVES];
	int k = blockIdx.x * blockDim.x + threadIdx.x;
	bool moved = false;
	if (k < n)
	{
		int shape = leafShape[sortedLeaf[k]];
		moved = (s.head[shape].x & S2B_SHAPE_MOVED) != 0;
		if (moved && n >= 256)
		{
			float4 root = rootBox[0];
			float4 box = s.fat[shape];
			float area = (box.z - box.x) * (box.w - box.y);
			float sceneArea = (root.z - root.x) * (root.w - root.y);
			if (area * 256.0f > sceneArea)
			{
				int slot = atomicAdd(counters + BC_LARGE, 1);
				if (slot < S2B_MAX_LARGE_MOVERS)
				{
					largeShapes[slot] = shape;
					moved = false;
				}
			}
		}
	}
	s2bBlockAppend(moved, k, movedLeaves, counters + BC_MOVED);
}

// what the query of proxy Q does with an overlapping proxy `other` (reference s2PairQueryCallback, src/broad_phase.c:166-258)
struct PairQuery
{
	int shapeQ, bodyQ, keyQ;
	unsigned typeBodyQ;
	int4 headQ, filterQ;
};

__device__ __forceinline__ void s2bConsiderPair(const PairQuery& q, int other, const ShapeView& s, const BodyView& b, int* counters,
												 const unsigned long long* pairHash, unsigned long long hashMask,
												 const unsigned long long* jointKeys, int jointKeyCount, unsigned long long* newKey,
												 int2* newShapes, int newCap)
{
	int shapeQ = q.shapeQ;
	if (other == shapeQ)
	{
		return;
	}
	int4 headO = s.head[other];
	int bodyO = headO.y;
	int keyO = headO.z;
	unsigned typeBodyO = S2B_BODY_TYPE((unsigned)b.flags[bodyO]);
	// a kinematic proxy only queries the dynamic tree
	if (q.typeBodyQ == S2B_BODY_KINEMATIC && typeBodyO != S2B_BODY_DYNAMIC)
	{
		return;
	}
	// both proxies moved: the one with the smaller key reports the pair
	if ((headO.x & S2B_SHAPE_MOVED) && keyO > q.keyQ)
	{
		// ... unless the other one cannot see us in its own query
		bool otherSeesUs = !(typeBodyO == S2B_BODY_KINEMATIC && q.typeBodyQ != S2B_BODY_DYNAMIC) && typeBodyO != S2B_BODY_STATIC;
		if (otherSeesUs)
		{
			return;
		}
	}
	if (bodyO == q.bodyQ)
	{
		return;
	}
	unsigned long long lo = (unsigned long long)(other < shapeQ ? other : shapeQ);
	unsigned long long hi = (unsigned long long)(other < shapeQ ? shapeQ : other);
	unsigned long long pairKey = (lo << 32) | hi;
	// "this pair already has a contact" — unless one of the shapes was (re)created since the table was built: the table's
	// contact then belongs to the shape that used to live in that slot and is dropped by this very pass (s2bCollectKeptContacts),
	// so the pair has to be reported again (the reference removes the key from its pair set when the old shape is destroyed,
	// src/contact.c:231-292, and creates the contact on the next update)
	bool recreated = ((q.headQ.x | headO.x) & S2B_SHAPE_FRESH) != 0;
	if (recreated == false && s2bPairInHash(pairHash, hashMask, pairKey))
	{
		return;
	}
	int shapeA, shapeB;
	if (keyO < q.keyQ)
	{
		shapeA = other;
		shapeB = shapeQ;
	}
	else
	{
		shapeA = shapeQ;
		shapeB = other;
	}
	int4 filterO = s.filter[other];
	if (s2bShouldShapesCollide(shapeA == shapeQ ? q.filterQ : filterO, shapeA == shapeQ ? filterO : q.filterQ) == false)
	{
		return;
	}
	if (s2bJointOverride(jointKeys, jointKeyCount, q.bodyQ, bodyO))
	{
		return;
	}
	int typeA = ((shapeA == shapeQ ? q.headQ.x : headO.x) >> 1) & 0x7;
	int typeB = ((shapeA == shapeQ ? headO.x : q.headQ.x) >> 1) & 0x7;
	int kind = s2bPairKind(typeA, typeB);
	if (kind == 0)
	{
		return;
	}
	if (kind == 2)
	{
		int tmp = shapeA;
		shapeA = shapeB;
		shapeB = tmp;
	}
	int slot = atomicAdd(counters + BC_NEW_PAIRS, 1);
	if (slot < newCap)
	{
		newKey[slot] = pairKey;
		newShapes[slot] = make_int2(shapeA, shapeB);
	}
}

__device__ __forceinline__ bool s2bMakeQuery(PairQuery& q, int shapeQ, const ShapeView& s, const BodyView& b)
{
	q.shapeQ = shapeQ;
	q.headQ = s.head[shapeQ];
	q.filterQ = s.filter[shapeQ];
	q.bodyQ = q.headQ.y;
	q.keyQ = q.headQ.z;
	q.typeBodyQ = S2B_BODY_TYPE((unsigned)b.flags[q.bodyQ]);
	return q.typeBodyQ != S2B_BODY_STATIC; // static proxies never query (reference src/broad_phase.c:284-299)
}

#define S2B_QUERY_BATCH 16
#define S2B_QUERY_BLOCK 128

// moved proxies with ordinary boxes: one thread walks the wide hierarchy
__global__ void __launch_bounds__(S2B_QUERY_BLOCK) s2bFindPairs(ShapeView s, BodyView b, const int* leafShape, const int* sortedLeaf, int* counters,
								 const int* movedLeaves, const float4* wideBox, const int* wideChild,
								 const unsigned long long* pairHash, unsigned long long hashMask, const unsigned long long* jointKeys,
								 int jointKeyCount, unsigned long long* newKey, int2* newShapes, int newCap)
{
	// overlapping LEAVES are only collected during the walk and examined in batches afterwards: the walk (box tests) and the
	// pair rules (shape header, hash probe, filters) are two different instruction streams, and a warp whose lanes hit
	// leaves at different moments would otherwise execute both serially for every lane
	__shared__ int found[S2B_QUERY_BATCH][S2B_QUERY_BLOCK];
	int n = counters[BC_LEAVES];
	int movedCount = counters[BC_MOVED];
	int qi = blockIdx.x * blockDim.x + threadIdx.x;
	if (qi >= movedCount)
	{
		return;
	}
	int leaf = movedLeaves[qi];
	PairQuery q;
	if (s2bMakeQuery(q, leafShape[sortedLeaf[leaf]], s, b) == false || n == 1)
	{
		return;
	}
	float4 boxQ = s.fat[q.shapeQ];

	// depth-first: test a wide node's children's boxes (one contiguous read), descend into the first overlapping wide child
	// directly and stack the others, collect the overlapping leaves. The stack is sized from the depth bound of the build
	// (S2B_QUERY_STACK).
	int stack[S2B_QUERY_STACK];
	int sp = 0;
	int node = 0;
	int nFound = 0;
	while (node >= 0 || nFound > 0)
	{
		while (node >= 0 && nFound <= S2B_QUERY_BATCH - S2B_WIDE)
		{
			// all loads of the node first (boxes of unused slots included): one round trip per visited node
			const float4* boxes = wideBox + node * S2B_WIDE;
			const int4* refs = reinterpret_cast<const int4*>(wideChild + node * S2B_WIDE);
			int child[S2B_WIDE];
			float4 box[S2B_WIDE];
#pragma unroll
			for (int i = 0; i < S2B_WIDE / 4; ++i)
			{
				int4 r = refs[i];
				child[4 * i] = r.x;
				child[4 * i + 1] = r.y;
				child[4 * i + 2] = r.z;
				child[4 * i + 3] = r.w;
			}
#pragma unroll
			for (int i = 0; i < S2B_WIDE; ++i)
			{
				box[i] = boxes[i];
			}
			int next = -1;
#pragma unroll
			for (int i = 0; i < S2B_WIDE; ++i)
			{
				int c = child[i];
				if (c != S2B_WIDE_EMPTY && s2bBoxesOverlap(boxQ, box[i]))
				{
					if (c < 0)
					{
						found[nFound++][threadIdx.x] = ~c;
					}
					else if (next < 0)
					{
						next = c;
					}
					else
					{
						stack[sp++] = c;
					}
				}
			}
			node = next >= 0 ? next : (sp > 0 ? stack[--sp] : -1);
		}
		for (int k = 0; k < nFound; ++k)
		{
			s2bConsiderPair(q, found[k][threadIdx.x], s, b, counters, pairHash, hashMask, jointKeys, jointKeyCount, newKey, newShapes, newCap);
		}
		nFound = 0;
	}
}

// every leaf against the short list of large movers (s2bCollectMovers). Same rules, same pairs; the order new pairs are
// emitted in never matters (they are sorted).
__global__ void s2bFindPairsLarge(ShapeView s, BodyView b, const int* leafShape, int* counters, const int* largeShapes,
								  const unsigned long long* pairHash, unsigned long long hashMask, const unsigned long long* jointKeys,
								  int jointKeyCount, unsigned long long* newKey, int2* newShapes, int newCap)
{
	int n = counters[BC_LEAVES];
	int large = min(counters[BC_LARGE], S2B_MAX_LARGE_MOVERS);
	int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= n || large == 0)
	{
		return;
	}
	int other = leafShape[k];
	float4 boxO = s.fat[other];
	for (int i = 0; i < large; ++i)
	{
		int shapeQ = largeShapes[i];
		if (s2bBoxesOverlap(s.fat[shapeQ], boxO) == false)
		{
			continue;
		}
		PairQuery q;
		if (s2bMakeQuery(q, shapeQ, s, b))
		{
			s2bConsiderPair(q, other, s, b, counters, pairHash, hashMask, jointKeys, jointKeyCount, newKey, newShapes, newCap);
		}
	}
}

// survivors: both shapes alive and not re-created, fat AABBs still overlap (reference src/world.c:149-166), and no joint
// created since forbids the pair (reference src/joint.c:214-217)
// The survivors' slots are appended to keepSlots (BC_KEPT): their order does not matter, the merged table is sorted by pair key.
__global__ void s2bCollectKeptContacts(ContactView c, int contactCount, ShapeView s, const unsigned long long* jointKeys, int jointKeyCount,
									   int* keepSlots, int* counters)
{
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	bool keep = false;
	if (i < contactCount)
	{
		int2 sh = c.shapes[i];
		int4 ha = s.head[sh.x], hb = s.head[sh.y];
		bool alive = (ha.x & S2B_ROW_VALID) && (hb.x & S2B_ROW_VALID) && (ha.x & S2B_SHAPE_FRESH) == 0 && (hb.x & S2B_SHAPE_FRESH) == 0;
		keep = alive && s2bBoxesOverlap(s.fat[sh.x], s.fat[sh.y]) && s2bJointOverride(jointKeys, jointKeyCount, ha.y, hb.y) == false;
	}
	s2bBlockAppend(keep, i, keepSlots, counters + BC_KEPT);
}

// The sort key is the pair key squeezed to 2 x shapeBits bits (lo << shapeBits | hi) so the radix sort runs only over
// significant digits.
__device__ __forceinline__ unsigned long long s2bSqueezeKey(unsigned long long pairKey, int shapeBits)
{
	return ((pairKey >> 32) << shapeBits) | (pairKey & 0xFFFFFFFFull);
}

__global__ void s2bMergeKeys(const int* counters, const int* keepSlots, const unsigned long long* oldKeys,
							 const unsigned long long* newKey, unsigned long long* mergeKey, int* mergeSrc, int capacity, int shapeBits)
{
	int kept = counters[BC_KEPT], fresh = counters[BC_NEW_PAIRS];
	int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= capacity)
	{
		return;
	}
	if (t < kept)
	{
		mergeKey[t] = s2bSqueezeKey(oldKeys[keepSlots[t]], shapeBits);
		mergeSrc[t] = keepSlots[t]; // >= 0: old slot
	}
	else if (t < kept + fresh)
	{
		mergeKey[t] = s2bSqueezeKey(newKey[t - kept], shapeBits);
		mergeSrc[t] = -1 - (t - kept); // < 0: new pair index
	}
	else
	{
		mergeKey[t] = ~0ull;
		mergeSrc[t] = 0;
	}
}

// s2CreateContact for new pairs (reference src/contact.c:156-229: empty manifold, empty cache, mixed friction and restitution), plain
// copy for survivors
__global__ void s2bGatherContactsSorted(const int* counters, const unsigned long long* sortedKey, const int* sortedSrc, ContactView src,
										ContactView dst, const int2* newShapes, ShapeView s, int sticky, int shapeBits)
{
	int total = counters[BC_KEPT] + counters[BC_NEW_PAIRS];
	int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= total)
	{
		return;
	}
	int from = sortedSrc[t];
	unsigned long long squeezed = sortedKey[t];
	dst.key[t] = ((squeezed >> shapeBits) << 32) | (squeezed & ((1ull << shapeBits) - 1ull));
	if (from >= 0)
	{
		dst.shapes[t] = src.shapes[from];
		dst.bodies[t] = src.bodies[from];
		dst.info[t] = src.info[from];
		dst.nf[t] = src.nf[from];
		dst.color[t] = src.color[from];
		for (int p = 0; p < 2; ++p)
		{
			dst.anchor[p][t] = src.anchor[p][from];
			dst.impulse[p][t] = src.impulse[p][from];
			if (sticky)
			{
				dst.fanchor[p][t] = src.fanchor[p][from];
				dst.fnormal[p][t] = src.fnormal[p][from];
			}
		}
	}
	else
	{
		int2 sh = newShapes[-1 - from];
		dst.shapes[t] = sh;
		dst.bodies[t] = make_int2(s.head[sh.x].y, s.head[sh.y].y);
		dst.info[t] = make_int4(0, 0, 0, 0);
		// s2MixFriction (reference src/contact.c:42-45)
		float friction = sqrtf(s.fr[sh.x].x * s.fr[sh.y].x);
		// s2MixRestitution (reference src/contact.c:49-52)
		float restitution = S2_MAX(s.restitution[sh.x], s.restitution[sh.y]);
		dst.nf[t] = make_float4(0.0f, 0.0f, friction, restitution);
		dst.color[t] = -1;
		for (int p = 0; p < 2; ++p)
		{
			dst.anchor[p][t] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
			dst.impulse[p][t] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
			if (sticky)
			{
				dst.fanchor[p][t] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
				dst.fnormal[p][t] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
			}
		}
	}
}

__global__ void s2bClearMovedFlags(ShapeView s, int* movedCounter)
{
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < s.capacity)
	{
		int4 h = s.head[i];
		if (h.x & (S2B_SHAPE_MOVED | S2B_SHAPE_FRESH))
		{
			s.head[i] = make_int4(h.x & ~(S2B_SHAPE_MOVED | S2B_SHAPE_FRESH), h.y, h.z, h.w);
		}
	}
	if (i == 0)
	{
		movedCounter[0] = 0;
	}
}

// ---------------------------------------------------------------------------------------------------------------
// host driver
// ---------------------------------------------------------------------------------------------------------------

// mailbox slots of the pair pass (pinned host memory, written by asynchronous copies)
#define MAIL_BC_BASE 16

// scratch sizes of a pass (host only; the pass itself never allocates between its kernels)
static size_t bpReserve(s2bWorld* w, BroadScratch* B)
{
	cudaStream_t st = w->stream;
	int shapeCap = w->shapeCap;
	int oldCount = w->contactCount;
	size_t nS = (size_t)shapeCap;
	B->validFlag.reserve(nS, st, false);
	B->leafShape.reserve(nS, st, false);
	B->mortonIn.reserve(nS, st, false);
	B->mortonOut.reserve(nS, st, false);
	B->leafIn.reserve(nS, st, false);
	B->leafOut.reserve(nS, st, false);
	B->counters.reserve(BC_SIZE, st, false);
	B->boundsBits.reserve(4, st, false);
	B->children.reserve(nS, st, false);
	B->parent.reserve(2 * nS, st, false);
	B->wideBox.reserve(S2B_WIDE * nS, st, false, false);
	B->wideChild.reserve(S2B_WIDE * nS, st, false, false);
	B->wideCount.reserve(nS, st, false, false);
	B->wideSlot.reserve(2 * nS, st, false, false);
	B->visit.reserve(nS, st, false); // zeroed once here: from then on every refit leaves its counters at zero
	B->rootBox.reserve(1, st, false);
	B->movedLeaves.reserve(nS, st, false);
	B->movedFlag.reserve(nS, st, false);
	B->largeShapes.reserve(S2B_MAX_LARGE_MOVERS, st, false);
	B->keepFlag.reserve((size_t)std::max(oldCount, 1), st, false);
	B->keepSlots.reserve((size_t)std::max(oldCount, 1), st, false);
	if (B->newPairCap == 0)
	{
		B->newPairCap = 8 * shapeCap + 1024;
	}
	size_t need = 0, tempBytes = 0;
	cub::DeviceSelect::Flagged(nullptr, need, thrust::counting_iterator<int>(0), (int*)nullptr, (int*)nullptr, (int*)nullptr,
							   std::max(shapeCap, oldCount), st);
	tempBytes = std::max(tempBytes, need);
	cub::DeviceRadixSort::SortPairs(nullptr, need, (unsigned*)nullptr, (unsigned*)nullptr, (int*)nullptr, (int*)nullptr, shapeCap, 0,
									32, st);
	tempBytes = std::max(tempBytes, need);
	B->newKey.reserve((size_t)B->newPairCap, st, false);
	B->newShapes.reserve((size_t)B->newPairCap, st, false);
	B->cubTemp.reserve(tempBytes + 256, st, false, false);
	return tempBytes;
}

// First half of a pass, no host synchronisation: hierarchy (re-used or rebuilt) and refit, pair-key hash of the current
// table, queries from the moved proxies -> candidate pairs (newKey / newShapes), survivors of the current table (keepSlots),
// and the counters of all that copied to the pinned mailbox.
static void bpSearch(s2bWorld* w, BroadScratch* B)
{
	cudaStream_t st = w->stream;
	int shapeCap = w->shapeCap;
	int oldCount = w->contactCount;
	ShapeView sv = shapeView(w);
	BodyView bv = bodyView(w);
	ContactColumns& cur = w->contacts[w->cur];
	int newCap = B->newPairCap;

	bool reuseTree = B->treeValid && w->pairsDirty == false && B->treeShapeCap == shapeCap && B->treeReuses < S2B_TREE_REUSE_LIMIT;
	if (reuseTree)
	{
		// keep BC_LEAVES and BC_HEIGHT of the build; clear the per-pass counters
		S2B_CHECK(cudaMemsetAsync(B->counters.p + BC_NEW_PAIRS, 0, sizeof(int) * (BC_SIZE - BC_NEW_PAIRS), st));
		B->treeReuses += 1;
	}
	else
	{
		S2B_CHECK(cudaMemsetAsync(B->counters.p, 0, sizeof(int) * BC_SIZE, st));

		// ---- leaves ----
		S2B_LAUNCH(w, s2bFlagValidShapes, gridFor(shapeCap, 256), 256, 0, sv, B->validFlag.p);
		size_t tb = B->cubTemp.cap;
		cub::DeviceSelect::Flagged(B->cubTemp.p, tb, thrust::counting_iterator<int>(0), B->validFlag.p, B->leafShape.p,
								   B->counters.p + BC_LEAVES, shapeCap, st);
		w->kernelLaunches += 2;

		// ---- Morton order ----
		int initBounds[4] = {0x7F7FFFFF, 0x7F7FFFFF, (int)0x80800000, (int)0x80800000};
		// ordered encoding: +FLT_MAX -> 0x7F7FFFFF, -FLT_MAX -> 0xFF7FFFFF ^ 0x7FFFFFFF = 0x80800000
		S2B_CHECK(cudaMemcpyAsync(B->boundsBits.p, initBounds, sizeof(initBounds), cudaMemcpyHostToDevice, st));
		S2B_LAUNCH(w, s2bSceneBounds, gridFor(shapeCap, 256), 256, 0, sv, B->leafShape.p, B->counters.p, B->boundsBits.p);
		S2B_LAUNCH(w, s2bMortonCodes, gridFor(shapeCap, 256), 256, 0, sv, B->leafShape.p, B->counters.p, B->boundsBits.p,
				   B->mortonIn.p, B->leafIn.p, shapeCap);
		tb = B->cubTemp.cap;
		cub::DeviceRadixSort::SortPairs(B->cubTemp.p, tb, B->mortonIn.p, B->mortonOut.p, B->leafIn.p, B->leafOut.p, shapeCap, 0, 32, st);
		w->kernelLaunches += 5;

		// ---- hierarchy ----
		S2B_LAUNCH(w, s2bBuildRadixTree, gridFor(shapeCap, 256), 256, 0, B->mortonOut.p, B->counters.p, B->children.p, B->parent.p);
		S2B_LAUNCH(w, s2bBuildWide, gridFor(shapeCap, 256), 256, 0, B->leafShape.p, B->leafOut.p, B->counters.p, B->children.p,
				   B->parent.p, B->wideChild.p, B->wideCount.p, B->wideSlot.p);
		B->treeValid = true;
		B->treeShapeCap = shapeCap;
		B->treeReuses = 0;
	}

	// ---- refit ----
	S2B_LAUNCH(w, s2bRefit, gridFor(shapeCap, 256), 256, 0, sv, B->leafShape.p, B->leafOut.p, B->counters.p, B->wideCount.p,
			   B->wideSlot.p, B->wideBox.p, B->visit.p, B->rootBox.p);

	// ---- pair-key hash set of the current contact table (rebuilt only when the table changed) ----
	if (B->hashVersion != w->contactTableVersion || B->pairHash.p == nullptr)
	{
		unsigned long long size = 1024;
		while (size < 2ull * (unsigned long long)std::max(oldCount, 1))
		{
			size <<= 1;
		}
		B->pairHash.reserve((size_t)size, st, false, false);
		B->hashMask = size - 1;
		S2B_CHECK(cudaMemsetAsync(B->pairHash.p, 0xFF, sizeof(unsigned long long) * (size_t)size, st));
		if (oldCount > 0)
		{
			S2B_LAUNCH(w, s2bBuildPairHash, gridFor(oldCount, 256), 256, 0, cur.key.p, oldCount, B->pairHash.p, B->hashMask);
		}
		B->hashVersion = w->contactTableVersion;
	}

	// ---- queries from moved proxies ----
	S2B_LAUNCH(w, s2bCollectMovers, gridFor(shapeCap, 256), 256, 0, sv, B->leafShape.p, B->leafOut.p, B->counters.p, B->rootBox.p,
			   B->movedLeaves.p, B->largeShapes.p);
	S2B_LAUNCH(w, s2bFindPairs, gridFor(shapeCap, S2B_QUERY_BLOCK), S2B_QUERY_BLOCK, 0, sv, bv, B->leafShape.p, B->leafOut.p,
			   B->counters.p, B->movedLeaves.p, B->wideBox.p, B->wideChild.p, B->pairHash.p, B->hashMask, w->jointPairKeys.p,
			   w->jointPairCount, B->newKey.p, B->newShapes.p, newCap);
	S2B_LAUNCH(w, s2bFindPairsLarge, gridFor(shapeCap, 256), 256, 0, sv, bv, B->leafShape.p, B->counters.p, B->largeShapes.p,
			   B->pairHash.p, B->hashMask, w->jointPairKeys.p, w->jointPairCount, B->newKey.p, B->newShapes.p, newCap);

	// ---- survivors ----
	if (oldCount > 0)
	{
		S2B_LAUNCH(w, s2bCollectKeptContacts, gridFor(oldCount, 256), 256, 0, makeView(cur), oldCount, sv, w->jointDestroyKeys.p,
				   w->jointDestroyCount, B->keepSlots.p, B->counters.p);
	}
	S2B_CHECK(cudaMemcpyAsync(w->hostMail + MAIL_BC_BASE, B->counters.p, sizeof(int) * BC_SIZE, cudaMemcpyDeviceToHost, st));
	B->searchedCount = oldCount;
	B->searchedVersion = w->contactTableVersion;
}

// Second half: the host knows how many candidate pairs and survivors the search found. Merge them into the other column
// set (or leave the table as it is), clear the MOVED / FRESH flags.
static void bpCommit(s2bWorld* w, BroadScratch* B, int fresh, int kept, size_t tempBytes)
{
	cudaStream_t st = w->stream;
	int shapeCap = w->shapeCap;
	int oldCount = w->contactCount;
	ShapeView sv = shapeView(w);
	ContactColumns& cur = w->contacts[w->cur];
	ContactColumns& nxt = w->contacts[w->cur ^ 1];
	int total = kept + fresh;
	if (fresh == 0 && kept == oldCount)
	{
		// the moved proxies still overlap exactly the shapes they overlapped before: the contact table stands as it is
		// (the usual outcome on a slowly settling pile)
	}
	else
	{
		nxt.reserve((size_t)std::max(total, 1), st, w->sticky, false);
		if (total > 0)
		{
			size_t need = 0;
			B->mergeKeyIn.reserve((size_t)total, st, false);
			B->mergeKeyOut.reserve((size_t)total, st, false);
			B->mergeSrcIn.reserve((size_t)total, st, false);
			B->mergeSrcOut.reserve((size_t)total, st, false);
			cub::DeviceRadixSort::SortPairs(nullptr, need, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr,
											(int*)nullptr, total, 0, 64, st);
			B->cubTemp.reserve(std::max(tempBytes, need) + 256, st, false, false);
			int shapeBits = 1;
			while ((1 << shapeBits) < shapeCap && shapeBits < 31)
			{
				shapeBits += 1;
			}
			S2B_LAUNCH(w, s2bMergeKeys, gridFor(total, 256), 256, 0, B->counters.p, B->keepSlots.p, cur.key.p, B->newKey.p,
					   B->mergeKeyIn.p, B->mergeSrcIn.p, total, shapeBits);
			size_t tb = B->cubTemp.cap;
			cub::DeviceRadixSort::SortPairs(B->cubTemp.p, tb, B->mergeKeyIn.p, B->mergeKeyOut.p, B->mergeSrcIn.p, B->mergeSrcOut.p,
											total, 0, 2 * shapeBits, st);
			w->kernelLaunches += 9;
			S2B_LAUNCH(w, s2bGatherContactsSorted, gridFor(total, 128), 128, 0, B->counters.p, B->mergeKeyOut.p, B->mergeSrcOut.p,
					   makeView(cur), makeView(nxt), B->newShapes.p, sv, w->sticky ? 1 : 0, shapeBits);
		}
		w->cur ^= 1;
		w->contactCount = total;
		w->contactTableVersion += 1;
		// size what the NEXT pass needs for this table now, while a re-allocation is already being paid for: the survivor
		// flags and the pair-key hash set (built lazily by that pass)
		B->keepFlag.reserve((size_t)std::max(total, 1), st, false);
		B->keepSlots.reserve((size_t)std::max(total, 1), st, false);
		{
			unsigned long long size = 1024;
			while (size < 2ull * (unsigned long long)std::max(total, 1))
			{
				size <<= 1;
			}
			B->pairHash.reserve((size_t)size, st, false, false);
		}
	}
	S2B_LAUNCH(w, s2bClearMovedFlags, gridFor(shapeCap, 256), 256, 0, sv, w->dMovedFlag.p);
	w->hostMail[MAIL_MOVED] = 0;
	w->pairsDirty = false;
	w->pairPassCount += 1;
}

// Start the pair search of the NEXT step behind this one (called after finalize): its inputs — fat AABBs, MOVED flags, the
// contact table — are final once finalize has run, and its counters then reach the host together with the end of the step,
// which the caller waits for anyway before it reads results. The next s2b_update_pairs picks the result up without having to
// stop in the middle of the pass (DESIGN.md §3.3). Anything the host uploads in between invalidates the search (uploadEpoch).
void s2bPrefetchPairSearch(s2bWorld* w)
{
	S2bEpochFreeze freeze;
	BroadScratch* B = getBroad(w);
	B->prefetched = false;
	// only scenes in motion: on a settled scene nothing is enqueued and the next pass is skipped from the moved counter alone
	if (w->prefetchPairs == 0 || w->shapeCap == 0 || B->lastPassRan == false || w->pairsDirty)
	{
		return;
	}
	if (B->evSearch[0] == nullptr)
	{
		S2B_CHECK(cudaEventCreate(&B->evSearch[0]));
		S2B_CHECK(cudaEventCreate(&B->evSearch[1]));
		S2B_CHECK(cudaEventCreateWithFlags(&B->searchDone, cudaEventDisableTiming));
	}
	B->prefetchTempBytes = bpReserve(w, B);
	S2B_CHECK(cudaEventRecord(B->evSearch[0], w->stream));
	bpSearch(w, B);
	S2B_CHECK(cudaEventRecord(B->evSearch[1], w->stream));
	S2B_CHECK(cudaEventRecord(B->searchDone, w->stream));
	B->prefetched = true;
	B->prefetchEpoch = w->uploadEpoch;
	B->searchTimed = true;
}

float s2bLastPairSearchMs(s2bWorld* w)
{
	BroadScratch* B = w->broad;
	if (B == nullptr || B->searchTimed == false)
	{
		return 0.0f;
	}
	float ms = 0.0f;
	if (cudaEventQuery(B->evSearch[1]) == cudaSuccess)
	{
		cudaEventElapsedTime(&ms, B->evSearch[0], B->evSearch[1]);
	}
	return ms;
}

void s2bBroadphaseUpdatePairs(s2bWorld* w)
{
	// scratch of this pass is not referenced by the solver's graph; a REPLACED contact table is, and shows up in the graph
	// signature through w->cur / w->contactCount / w->contactTableVersion
	S2bEpochFreeze freeze;
	cudaStream_t st = w->stream;
	BroadScratch* B = getBroad(w);
	w->dMovedFlag.reserve(4, st, true);

	// ---- the search was started behind the previous step: its counters are (about to be) in the mailbox ----
	if (B->prefetched)
	{
		B->prefetched = false;
		bool valid = w->pairsDirty == false && B->prefetchEpoch == w->uploadEpoch && B->searchedVersion == w->contactTableVersion &&
					 B->searchedCount == w->contactCount && w->prefetchPairs == 1; // (2: search but never use the result — debugging)
		if (valid)
		{
			S2B_CHECK(cudaEventSynchronize(B->searchDone));
			S2B_CHECK(cudaEventRecord(w->timer.ev[0], st));
			const int* hc = w->hostMail + MAIL_BC_BASE;
			int fresh = hc[BC_NEW_PAIRS], kept = hc[BC_KEPT];
			if (fresh <= B->newPairCap)
			{
				w->treeHeight = hc[BC_HEIGHT];
				B->lastPassRan = hc[BC_MOVED] > 0 || hc[BC_LARGE] > 0;
				bpCommit(w, B, fresh, kept, B->prefetchTempBytes);
				return;
			}
			B->newPairCap = fresh + fresh / 2 + 1024; // rare: redo the pass below with a larger pair buffer
		}
		// (something was uploaded since: the search is stale — e.g. new shapes — and is redone)
	}

	// Did anything move in the last finalize? The counter was copied to the pinned mailbox at the end of the previous
	// step; wait for that copy (normally long done) and read it.
	bool run = w->pairsDirty;
	if (run == false)
	{
		// (wait for THAT copy only — not for whatever the caller has enqueued since: force uploads, row scatters — so that the
		// kernels of this step can be queued behind them without the host idling)
		if (w->movedEvent != nullptr)
		{
			S2B_CHECK(cudaEventSynchronize(w->movedEvent));
		}
		else
		{
			S2B_CHECK(cudaStreamSynchronize(st));
		}
		run = w->hostMail[MAIL_MOVED] > 0;
	}
	S2B_CHECK(cudaEventRecord(w->timer.ev[0], st));
	B->lastPassRan = run && w->shapeCap > 0;
	if (run == false || w->shapeCap == 0)
	{
		return;
	}

	for (int attempt = 0; attempt < 4; ++attempt)
	{
		size_t tempBytes = bpReserve(w, B);
		bpSearch(w, B);
		// the new table size has to be known on the host (column reservation): one small synchronising read-back, paid only
		// when the search could not be started behind the previous step (first steps, after uploads, settled scenes)
		S2B_CHECK(cudaStreamSynchronize(st));
		const int* hc = w->hostMail + MAIL_BC_BASE;
		int fresh = hc[BC_NEW_PAIRS], kept = hc[BC_KEPT];
		if (fresh > B->newPairCap)
		{
			B->newPairCap = fresh + fresh / 2 + 1024;
			continue; // rare: redo the pass with a larger pair buffer
		}
		w->treeHeight = hc[BC_HEIGHT];
		bpCommit(w, B, fresh, kept, tempBytes);
		break;
	}
}
