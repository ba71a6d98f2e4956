// k nearest neighbours (include/mgs_rasterizer.h, mgs_knn): for each query the k nearest reference points by fp32 squared
// distance, sorted by (d2, index), without host reads.
//
// Stages (knn_run below):
//   grid     the points' bounding box (field_bbox_kernel) and a cubic grid of 2^21 fine cells along its longest axis; every
//            finite point gets the 63-bit Morton code of its fine cell (non-finite points ~0), and a stable radix sort by
//            code leaves the points of any cell of any level L (2^L fine cells a side) contiguous, in ascending index;
//   level    one pass over the sorted codes histograms, per adjacent pair, the finest level at which the two fall in one
//            cell (the top set bit of their XOR / 3); so the occupied cells at every level are counted at once, and one
//            thread picks the start level L0 whose occupied cells hold about max(k, 8) points on average.  A surface
//            cloud fills few cells of its box, so a resolution from N alone would leave hundreds of points per cell;
//   queries  sorted by code the same way (the sorted points themselves when queries is NULL), cut into runs of one L0 cell
//            and into warp items of at most 32 (field_ranges / warp_count / items kernels over the run ids);
//   search   one warp per item, lane = query, its sorted top-k in registers.  The warp visits a growing box of fine cells:
//            first its L0 cell, then a shell of one cell around the box at the current level, coarsening the level by one
//            whenever the box is wider than four cells, so that far neighbours (outliers) are reached in a logarithmic
//            number of steps.  A shell's cells are looked up lane-parallel by binary search of their code range; cells
//            inside the visited box are skipped, points of partly visited cells are skipped by their fine coordinates.
//            The points of each cell are staged through shared memory with cp.async.  A lane is done when its list holds
//            k entries and its k-th d2 lies below the squared distance from the query to the unvisited part of the grid
//            (the box's faces that do not reach the grid's edge, in fine units less a margin of two for the rounding of
//            the binning, and a relative 1e-5 for that of d2), or when the box covers the whole grid.
#include <algorithm>
#include <map>
#include <mutex>
#include <tuple>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include "../../include/mgs_rasterizer.h"
#include "mgs_common.cuh"
#include "mgs_kernels.h"

namespace mgs {

constexpr int KNN_BITS = 21;                          // fine cells per axis: 2^21, three axes in a 63-bit Morton code
constexpr int KNN_LEVELS = KNN_BITS + 1;              // level L: cells of 2^L fine cells a side, L = 0 .. 21
constexpr unsigned long long KNN_NONE = ~0ull;       // code of a non-finite point or query
constexpr uint32_t KNN_EMPTY = 0xffffffffu;          // index of an empty slot
constexpr int KNN_WARPS = 4;                          // warps per search CTA
static_assert(KNN_MAX_K == 32, "the largest list bucket is 32");

struct KnnGrid {
	float lo[3];    // corner of the points' bounding box
	float inv;      // fine cells per unit length (0 when the box is a point)
	int gmax[3];    // the last fine cell holding points along each axis
	int level;      // start level L0
	int nvalid;     // finite points
};

struct KnnArgs {
	int k, self;
	const KnnGrid* grid;
	const float* queries;               // [Q,3] (the points when self)
	const float4* pts;                  // [N] the points in code order, {x, y, z, index bits}
	const unsigned long long* codes;    // [N] their codes, ascending
	const uint32_t* qorder;             // [Q] query ids in code order
	const uint4* items;                 // warp items {first, end (in qorder), run, 0}
	const int* nitems;
	long long* out_index;               // [Q,k]
	float* out_dist2;                   // [Q,k]
};

// ---- Morton codes of 21-bit cell coordinates ----
__device__ __forceinline__ unsigned long long spread3(uint32_t v)
{
	unsigned long long x = v & 0x1fffffu;
	x = (x | x << 32) & 0x1f00000000ffffull;
	x = (x | x << 16) & 0x1f0000ff0000ffull;
	x = (x | x << 8) & 0x100f00f00f00f00full;
	x = (x | x << 4) & 0x10c30c30c30c30c3ull;
	x = (x | x << 2) & 0x1249249249249249ull;
	return x;
}
__device__ __forceinline__ uint32_t compact3(unsigned long long x)
{
	x &= 0x1249249249249249ull;
	x = (x ^ (x >> 2)) & 0x10c30c30c30c30c3ull;
	x = (x ^ (x >> 4)) & 0x100f00f00f00f00full;
	x = (x ^ (x >> 8)) & 0x1f0000ff0000ffull;
	x = (x ^ (x >> 16)) & 0x1f00000000ffffull;
	x = (x ^ (x >> 32)) & 0x1fffffull;
	return (uint32_t)x;
}
__device__ __forceinline__ unsigned long long morton3(uint32_t x, uint32_t y, uint32_t z)
{
	return spread3(x) | spread3(y) << 1 | spread3(z) << 2;
}

// fine position of coordinate x along axis k (unclamped) and its cell, clamped to the grid
__device__ __forceinline__ float fine_pos(float x, const KnnGrid& g, int k) { return (x - g.lo[k]) * g.inv; }
__device__ __forceinline__ int fine_cell(float u, int gmax)
{
	const float t = floorf(u);
	return t <= 0.f ? 0 : (t >= (float)gmax ? gmax : (int)t);
}

// one thread: the grid over the box of field_bbox_kernel
__global__ void knn_grid_kernel(const uint32_t* __restrict__ box, KnnGrid* __restrict__ grid)
{
	KnnGrid g{};
	if (box[0] <= box[3]) {
		float emax = 0.f;
#pragma unroll
		for (int k = 0; k < 3; k++) {
			g.lo[k] = funkey(box[k]);
			emax = fmaxf(emax, funkey(box[3 + k]) - g.lo[k]);
		}
		const float inv = (float)(1 << KNN_BITS) / emax;
		g.inv = (emax > 0.f && isfinite(inv)) ? inv : 0.f;
#pragma unroll
		for (int k = 0; k < 3; k++) g.gmax[k] = fine_cell(fine_pos(funkey(box[3 + k]), g, k), (1 << KNN_BITS) - 1);
	}
	*grid = g;
}

__global__ void __launch_bounds__(256) knn_code_kernel(int n, const float* __restrict__ p, const KnnGrid* __restrict__ grid,
	unsigned long long* __restrict__ codes, uint32_t* __restrict__ iota)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const KnnGrid g = *grid;
	const float x = p[3 * i], y = p[3 * i + 1], z = p[3 * i + 2];
	unsigned long long c = KNN_NONE;
	if (isfinite(x) && isfinite(y) && isfinite(z))
		c = morton3(fine_cell(fine_pos(x, g, 0), g.gmax[0]), fine_cell(fine_pos(y, g, 1), g.gmax[1]), fine_cell(fine_pos(z, g, 2), g.gmax[2]));
	codes[i] = c;
	iota[i] = (uint32_t)i;
}

// the points in code order as {x, y, z, index}; hist[l] += adjacent finite pairs whose cells first merge at level l + 1
// (they share the level-L cell for L > l), *nvalid += finite points
__global__ void __launch_bounds__(256) knn_pack_kernel(int N, const float* __restrict__ p, const unsigned long long* __restrict__ codes,
	const uint32_t* __restrict__ order, float4* __restrict__ pts, uint32_t* __restrict__ hist, uint32_t* __restrict__ nvalid)
{
	__shared__ uint32_t s_hist[KNN_LEVELS];
	__shared__ uint32_t s_valid;
	if (threadIdx.x < KNN_LEVELS) s_hist[threadIdx.x] = 0;
	if (threadIdx.x == 0) s_valid = 0;
	__syncthreads();
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < N) {
		const uint32_t id = order[i];
		pts[i] = make_float4(p[3 * id], p[3 * id + 1], p[3 * id + 2], __uint_as_float(id));
		const unsigned long long c = codes[i];
		if (c != KNN_NONE) {
			atomicAdd(&s_valid, 1u);
			const unsigned long long x = i > 0 ? c ^ codes[i - 1] : 0ull;
			if (x != 0ull) atomicAdd(&s_hist[(63 - __clzll((long long)x)) / 3], 1u);
		}
	}
	__syncthreads();
	if (threadIdx.x < KNN_LEVELS && s_hist[threadIdx.x]) atomicAdd(hist + threadIdx.x, s_hist[threadIdx.x]);
	if (threadIdx.x == 0 && s_valid) atomicAdd(nvalid, s_valid);
}

// one thread: occupied cells at level L = 1 + sum_{l >= L} hist[l]; L0 is the level whose mean occupancy is nearest to
// target (in ratio) among the two around the first level that reaches it
__global__ void knn_level_kernel(int k, const uint32_t* __restrict__ hist, const uint32_t* __restrict__ nvalid, KnnGrid* __restrict__ grid)
{
	const double n = (double)*nvalid, target = (double)max(k, 8);
	double occ[KNN_LEVELS];
	double run = 1.0;
	for (int L = KNN_LEVELS - 1; L >= 0; L--) { run += hist[L]; occ[L] = run; }
	int L0 = KNN_LEVELS - 1;
	for (int L = 0; L < KNN_LEVELS; L++)
		if (n >= target * occ[L]) { L0 = L; break; }
	if (L0 > 0 && target * target * occ[L0 - 1] * occ[L0] < n * n) L0--;  // mean(L0 - 1) is nearer to target than mean(L0)
	grid->level = L0;
	grid->nvalid = (int)*nvalid;
}

// flags[i] = 1 where sorted query i starts a new L0 cell (0 for the first)
__global__ void __launch_bounds__(256) knn_run_flags_kernel(int Q, const unsigned long long* __restrict__ qcodes,
	const KnnGrid* __restrict__ grid, uint32_t* __restrict__ flags)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= Q) return;
	const int sh = 3 * grid->level;
	flags[i] = (i > 0 && (qcodes[i] >> sh) != (qcodes[i - 1] >> sh)) ? 1u : 0u;
}

__device__ __forceinline__ bool knn_less(float d, uint32_t i, float e, uint32_t j) { return d < e || (d == e && i < j); }

// (dc, ic) into the sorted list, the last entry falling off
template <int K>
__device__ __forceinline__ void knn_insert(float (&d)[K], uint32_t (&id)[K], float dc, uint32_t ic)
{
#pragma unroll
	for (int j = K - 1; j > 0; j--) {
		if (knn_less(dc, ic, d[j - 1], id[j - 1])) { d[j] = d[j - 1]; id[j] = id[j - 1]; }
		else if (knn_less(dc, ic, d[j], id[j])) { d[j] = dc; id[j] = ic; }
	}
	if (knn_less(dc, ic, d[0], id[0])) { d[0] = dc; id[0] = ic; }
}

// first position in codes[0, n) with codes[pos] >= key
__device__ __forceinline__ int lower_bound64(const unsigned long long* codes, int n, unsigned long long key)
{
	int lo = 0, hi = n;
	while (lo < hi) {
		const int mid = (lo + hi) >> 1;
		if (__ldg(codes + mid) < key) lo = mid + 1; else hi = mid;
	}
	return lo;
}

template <int K>
__global__ void __launch_bounds__(32 * KNN_WARPS) knn_search_kernel(KnnArgs a)
{
	__shared__ __align__(16) float4 s_pt[KNN_WARPS][32];
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const int item = blockIdx.x * KNN_WARPS + warp;
	if (item >= *a.nitems) return;
	float4* const stage = s_pt[warp];
	const KnnGrid g = *a.grid;
	const uint4 it = a.items[item];
	const bool has = lane < (int)(it.y - it.x);
	const uint32_t qid = has ? a.qorder[it.x + lane] : 0u;
	float q[3] = { 0.f, 0.f, 0.f };
	if (has) { q[0] = a.queries[3 * qid]; q[1] = a.queries[3 * qid + 1]; q[2] = a.queries[3 * qid + 2]; }
	const bool valid = has && g.nvalid > 0 && isfinite(q[0]) && isfinite(q[1]) && isfinite(q[2]);
	// the list: slots K - k .. K - 1 hold the k best, the K - k slots in front of them -inf, which no candidate displaces; so
	// the k-th entry is always slot K - 1
	float d[K];
	uint32_t id[K];
#pragma unroll
	for (int j = 0; j < K; j++) { d[j] = j < K - a.k ? -INFINITY : INFINITY; id[j] = KNN_EMPTY; }
	float u[3];
	int b0[3], b1[3];      // the warp's fine cells: min and max over its valid lanes
#pragma unroll
	for (int k = 0; k < 3; k++) {
		u[k] = fine_pos(q[k], g, k);
		const int c = fine_cell(u[k], g.gmax[k]);
		b0[k] = valid ? c : INT_MAX;
		b1[k] = valid ? c : -1;
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) {
			b0[k] = min(b0[k], __shfl_xor_sync(0xffffffffu, b0[k], o));
			b1[k] = max(b1[k], __shfl_xor_sync(0xffffffffu, b1[k], o));
		}
	}
	bool done = !valid;
	int L = g.level;
	int v0[3] = { 0, 0, 0 }, v1[3] = { -1, -1, -1 };  // the visited fine box (empty)
	bool first = true;
	while (!__all_sync(0xffffffffu, done)) {
		// ---- the next box: the warp's L0 cells, then one more cell of level L2 on every side ----
		const int wide = max(max((v1[0] - v0[0]) >> L, (v1[1] - v0[1]) >> L), (v1[2] - v0[2]) >> L) + 1;
		const int L2 = (!first && wide > 4 && L < KNN_BITS) ? L + 1 : L;
		int n0[3], n1[3], cl[3], cn[3];
#pragma unroll
		for (int k = 0; k < 3; k++) {
			const int lo = first ? (b0[k] >> L2) : (v0[k] >> L2) - 1;
			const int hi = first ? (b1[k] >> L2) : (v1[k] >> L2) + 1;
			cl[k] = max(lo, 0);
			cn[k] = min(hi, g.gmax[k] >> L2) - cl[k] + 1;
			n0[k] = cl[k] << L2;
			n1[k] = min(((cl[k] + cn[k]) << L2) - 1, g.gmax[k]);
		}
		const int total = cn[0] * cn[1] * cn[2];
		for (int base = 0; base < total; base += 32) {
			// ---- lane t: cell base + t of the box, its code range unless the visited box holds it ----
			const int t = base + lane;
			int f0[3], f1[3];
			bool inside = !first, overlap = !first;
			{
				const int c[3] = { cl[0] + t % cn[0], cl[1] + (t / cn[0]) % cn[1], cl[2] + t / (cn[0] * cn[1]) };
#pragma unroll
				for (int k = 0; k < 3; k++) {
					f0[k] = c[k] << L2;
					f1[k] = min(f0[k] + (1 << L2) - 1, g.gmax[k]);
					inside = inside && f0[k] >= v0[k] && f1[k] <= v1[k];
					overlap = overlap && f0[k] <= v1[k] && f1[k] >= v0[k];
				}
			}
			int ra = 0, rb = 0;
			if (t < total && !inside) {
				const unsigned long long m = morton3(f0[0] >> L2, f0[1] >> L2, f0[2] >> L2);
				ra = lower_bound64(a.codes, g.nvalid, m << (3 * L2));
				rb = ra + lower_bound64(a.codes + ra, g.nvalid - ra, (m + 1) << (3 * L2));
			}
			uint32_t todo = __ballot_sync(0xffffffffu, rb > ra);
			while (todo) {
				const int src = __ffs(todo) - 1;
				todo &= todo - 1;
				const int ca = __shfl_sync(0xffffffffu, ra, src), cb = __shfl_sync(0xffffffffu, rb, src);
				const bool part = __shfl_sync(0xffffffffu, (int)overlap, src) != 0;
				for (int p0 = ca; p0 < cb; p0 += 32) {
					const int cnt = min(32, cb - p0);
					if (lane < cnt) cp_async16(stage + lane, a.pts + p0 + lane);
					cp_async_commit();
					// points of a partly visited cell that lie in the visited box were seen before
					bool seen = false;
					if (part && lane < cnt) {
						const unsigned long long c = __ldg(a.codes + p0 + lane);
						const int x = (int)compact3(c), y = (int)compact3(c >> 1), z = (int)compact3(c >> 2);
						seen = x >= v0[0] && x <= v1[0] && y >= v0[1] && y <= v1[1] && z >= v0[2] && z <= v1[2];
					}
					const uint32_t skip = __ballot_sync(0xffffffffu, seen);
					cp_async_wait<0>();
					__syncwarp();
					if (!done) {
						for (int j = 0; j < cnt; j++) {
							if ((skip >> j) & 1u) continue;
							const float4 p = stage[j];
							const uint32_t pid = __float_as_uint(p.w);
							const float dx = q[0] - p.x, dy = q[1] - p.y, dz = q[2] - p.z;
							const float dd = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
							if (!knn_less(dd, pid, d[K - 1], id[K - 1]) || (a.self && pid == qid)) continue;
							knn_insert<K>(d, id, dd, pid);
						}
					}
					__syncwarp();  // the stage is rewritten by the next chunk
				}
			}
		}
#pragma unroll
		for (int k = 0; k < 3; k++) { v0[k] = n0[k]; v1[k] = n1[k]; }
		L = L2;
		first = false;
		if (!done) {
			// distance from the query to the unvisited fine cells, in fine units: faces that reach the grid's edge bound nothing
			float lb = INFINITY;
#pragma unroll
			for (int k = 0; k < 3; k++) {
				if (v0[k] > 0) lb = fminf(lb, u[k] - (float)v0[k] - 2.f);
				if (v1[k] < g.gmax[k]) lb = fminf(lb, (float)(v1[k] + 1) - u[k] - 2.f);
			}
			if (lb == INFINITY) done = true;
			else {
				const float w = fmaxf(lb, 0.f) / g.inv;
				done = id[K - 1] != KNN_EMPTY && d[K - 1] < w * w * (1.f - 1e-5f);
			}
		}
	}
	if (has) {
		long long* oi = a.out_index + (size_t)qid * a.k;
		float* od = a.out_dist2 + (size_t)qid * a.k;
#pragma unroll
		for (int j = 0; j < K; j++) {
			const int o = j - (K - a.k);
			if (o >= 0) {
				oi[o] = id[j] == KNN_EMPTY ? -1ll : (long long)id[j];
				od[o] = id[j] == KNN_EMPTY ? INFINITY : d[j];
			}
		}
	}
}

// N = 0: every slot padded
__global__ void __launch_bounds__(256) knn_pad_kernel(size_t n, long long* __restrict__ out_index, float* __restrict__ out_dist2)
{
	const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	out_index[i] = -1;
	out_dist2[i] = INFINITY;
}

// ---------------------------------------------------------------------------------------------------------------- host
#define KNN_TRY(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return e_; } while (0)

static int knn_items(int Q) { return Q + (Q + 31) / 32; }  // runs of one cell cut into warps of at most 32

// CUB's scratch size on the current device for (N, Q).  Cached, because the size queries look up device attributes and a
// steady-state call (or its capture in a CUDA graph) should not repeat them; the cache is emptied when it reaches
// KNN_CACHE entries, so callers whose N varies from call to call do not grow it without bound.
constexpr size_t KNN_CACHE = 256;
static cudaError_t knn_temp_bytes(int N, int Q, size_t* bytes)
{
	static std::mutex mu;
	static std::map<std::tuple<int, int, int>, size_t> cache;
	int dev = 0;
	KNN_TRY(cudaGetDevice(&dev));
	std::lock_guard<std::mutex> lk(mu);
	const auto key = std::make_tuple(dev, N, Q);
	const auto it = cache.find(key);
	if (it != cache.end()) { *bytes = it->second; return cudaSuccess; }
	size_t a = 0, b = 0;
	KNN_TRY(cub::DeviceRadixSort::SortPairs(nullptr, a, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
		(const uint32_t*)nullptr, (uint32_t*)nullptr, std::max(N, Q), 0, 64));
	KNN_TRY(cub::DeviceScan::InclusiveSum(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, Q));
	if (cache.size() >= KNN_CACHE) cache.clear();
	*bytes = cache[key] = std::max(a, b);
	return cudaSuccess;
}

template <typename T>
static void carve(char*& chunk, T*& ptr, size_t count)
{
	const size_t offset = (reinterpret_cast<uintptr_t>(chunk) + 127) & ~(uintptr_t)127;
	ptr = reinterpret_cast<T*>(offset);
	chunk = reinterpret_cast<char*>(ptr + count);
}

struct KnnState {
	KnnGrid* grid; int* nitems; uint32_t* box; uint32_t* hist; uint32_t* nvalid;
	unsigned long long* codes; unsigned long long* codes_sorted; uint32_t* iota; uint32_t* order; float4* pts;
	unsigned long long* qcodes; unsigned long long* qcodes_sorted; uint32_t* qiota; uint32_t* qorder;
	uint32_t* flags; uint32_t* run; uint2* qrange; uint32_t* wcnt; uint32_t* woff; uint4* items;
	char* temp; size_t temp_bytes;
	static KnnState at(char* chunk, int N, int Q, size_t temp_bytes)
	{
		KnnState s;
		carve(chunk, s.grid, 1);
		carve(chunk, s.nitems, 1);
		carve(chunk, s.box, 8);
		carve(chunk, s.hist, KNN_LEVELS + 1);  // hist, then nvalid: one memset
		s.nvalid = s.hist + KNN_LEVELS;
		carve(chunk, s.codes, N);
		carve(chunk, s.codes_sorted, N);
		carve(chunk, s.iota, N);
		carve(chunk, s.order, N);
		carve(chunk, s.pts, N);
		carve(chunk, s.qcodes, Q);
		carve(chunk, s.qcodes_sorted, Q);
		carve(chunk, s.qiota, Q);
		carve(chunk, s.qorder, Q);
		carve(chunk, s.flags, Q);
		carve(chunk, s.run, Q);
		carve(chunk, s.qrange, Q);
		carve(chunk, s.wcnt, Q);
		carve(chunk, s.woff, Q);
		carve(chunk, s.items, knn_items(Q));
		s.temp_bytes = temp_bytes;
		carve(chunk, s.temp, s.temp_bytes);
		return s;
	}
};

cudaError_t knn_state_bytes(int N, int Q, size_t* bytes)
{
	size_t tb = 0;
	KNN_TRY(knn_temp_bytes(N, Q, &tb));
	const KnnState s = KnnState::at(nullptr, N, Q, tb);
	*bytes = (size_t)(s.temp + s.temp_bytes - (char*)nullptr) + 128;
	return cudaSuccess;
}

template <int K>
static void launch_search(const KnnArgs& a, int Q, cudaStream_t st)
{
	knn_search_kernel<K><<<ceil_div(knn_items(Q), KNN_WARPS), 32 * KNN_WARPS, 0, st>>>(a);
}

cudaError_t knn_run(char* state, int N, int Q, int k, const float* points, const float* queries, long long* out_index,
	float* out_dist2, cudaStream_t st)
{
	if (Q == 0) return cudaSuccess;
	if (N == 0) {
		const size_t n = (size_t)Q * k;
		knn_pad_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, out_index, out_dist2);
		return cudaGetLastError();
	}
	size_t temp_bytes = 0;
	KNN_TRY(knn_temp_bytes(N, Q, &temp_bytes));
	const KnnState s = KnnState::at(state, N, Q, temp_bytes);
	const bool self = queries == nullptr;
	// ---- the grid over the points, the points in code order, the start level ----
	KNN_TRY(cudaMemsetAsync(s.box, 0xff, 3 * sizeof(uint32_t), st));
	KNN_TRY(cudaMemsetAsync(s.box + 3, 0, 3 * sizeof(uint32_t), st));
	KNN_TRY(cudaMemsetAsync(s.hist, 0, (KNN_LEVELS + 1) * sizeof(uint32_t), st));
	field_bbox_kernel<<<ceil_div(N, 256), 256, 0, st>>>(N, points, s.box);
	knn_grid_kernel<<<1, 1, 0, st>>>(s.box, s.grid);
	knn_code_kernel<<<ceil_div(N, 256), 256, 0, st>>>(N, points, s.grid, s.codes, s.iota);
	size_t tb = s.temp_bytes;
	KNN_TRY(cub::DeviceRadixSort::SortPairs(s.temp, tb, s.codes, s.codes_sorted, s.iota, s.order, N, 0, 64, st));
	knn_pack_kernel<<<ceil_div(N, 256), 256, 0, st>>>(N, points, s.codes_sorted, s.order, s.pts, s.hist, s.nvalid);
	knn_level_kernel<<<1, 1, 0, st>>>(k, s.hist, s.nvalid, s.grid);
	// ---- the queries in code order, cut into runs of one start-level cell and warp items ----
	const unsigned long long* qcodes = s.codes_sorted;
	const uint32_t* qorder = s.order;
	if (!self) {
		knn_code_kernel<<<ceil_div(Q, 256), 256, 0, st>>>(Q, queries, s.grid, s.qcodes, s.qiota);
		tb = s.temp_bytes;
		KNN_TRY(cub::DeviceRadixSort::SortPairs(s.temp, tb, s.qcodes, s.qcodes_sorted, s.qiota, s.qorder, Q, 0, 64, st));
		qcodes = s.qcodes_sorted;
		qorder = s.qorder;
	}
	knn_run_flags_kernel<<<ceil_div(Q, 256), 256, 0, st>>>(Q, qcodes, s.grid, s.flags);
	tb = s.temp_bytes;
	KNN_TRY(cub::DeviceScan::InclusiveSum(s.temp, tb, s.flags, s.run, Q, st));
	KNN_TRY(cudaMemsetAsync(s.qrange, 0, (size_t)Q * sizeof(uint2), st));
	field_ranges_kernel<<<ceil_div(Q, 256), 256, 0, st>>>(Q, s.run, s.qrange);
	field_warp_count_kernel<<<ceil_div(Q, 256), 256, 0, st>>>(Q, s.qrange, s.wcnt);
	tb = s.temp_bytes;
	KNN_TRY(cub::DeviceScan::InclusiveSum(s.temp, tb, s.wcnt, s.woff, Q, st));
	field_items_kernel<<<ceil_div(Q, 256), 256, 0, st>>>(Q, s.qrange, s.wcnt, s.woff, s.items, s.nitems);
	// ---- the search ----
	KnnArgs a{};
	a.k = k; a.self = self; a.grid = s.grid; a.queries = self ? points : queries;
	a.pts = s.pts; a.codes = s.codes_sorted; a.qorder = qorder; a.items = s.items; a.nitems = s.nitems;
	a.out_index = out_index; a.out_dist2 = out_dist2;
	if (k <= 4) launch_search<4>(a, Q, st);
	else if (k <= 8) launch_search<8>(a, Q, st);
	else if (k <= 16) launch_search<16>(a, Q, st);
	else launch_search<32>(a, Q, st);
	return cudaGetLastError();
}

}  // namespace mgs
