// Farthest-point sampling (include/mgs_rasterizer.h, mgs_fps): for each of B clouds, n picks, each the unpicked finite point
// farthest (fp32 squared distance, fixed order, no FMA) from the picks before it, ties to the lower index.
//
// One thread-block cluster of C CTAs per cloud; CTA r of the cluster holds the points i = j C T + r T + tid (thread tid,
// j = 0 .. K - 1), so a ragged cloud's points spread over every CTA.  Each point's d (squared distance to the nearest pick)
// is -1 once it is picked or when it is not available (non-finite, or at or beyond the cloud's length).  Per pick:
//   update   every thread lowers the d of its points against the last pick and marks that pick taken;
//   key      each point's 64-bit key (bits(d) + 1) << 32 | ~i (0 for d < 0): for d >= 0 the float bits rise with d, so the
//            largest key is the largest d, and among equal d the lowest index;
//   argmax   warp shuffles, then warp 0 over the warp maxima in shared memory, which writes the CTA's {key, x, y, z} into
//            the slot of the pick's parity; one cluster.sync(), after which every warp reads the C slots of the cluster
//            through distributed shared memory and takes the same maximum.  A CTA overwrites slot t & 1 at pick t + 2, and
//            every reader of pick t passes the barrier of pick t + 1 before it can get there; so one cluster barrier per pick
//            suffices, and a last one keeps each CTA's slots alive until the others have read them.
// Clusters never wait on each other: a batch larger than the GPU runs in waves, without a grid-wide barrier.
//
// Tiers, chosen on the host from P alone (fps_plan):
//   registers  fps_kernel<K>: 512 threads x K points per thread x C CTAs, the coordinates and d in registers: K = 4 with
//              C = 1 .. 8 up to 16,384 points, then K = 16 with C = 4, 8, 16 up to 131,072;
//   streaming  fps_stream_kernel: clouds above the largest register tier keep a packed {x, y, z, d} copy in the state
//              buffer (16 bytes a point, L2-resident at c3 size) and re-read it every pick.
#include <cooperative_groups.h>
#include <algorithm>
#include <map>
#include <mutex>
#include "../../include/mgs_rasterizer.h"
#include "mgs_common.cuh"
#include "mgs_kernels.h"

namespace cg = cooperative_groups;

namespace mgs {

constexpr int FPS_THREADS = 512;          // threads per CTA
constexpr int FPS_STREAM_BATCH = 8;       // points a streaming thread loads before it uses them
constexpr int FPS_MAX_CLUSTER = 16;

struct __align__(8) FpsSlot {
	unsigned long long key;
	float x, y, z;
};

struct FpsArgs {
	int P, n;
	const float* points;        // [B,P,3]
	const long long* lengths;   // [B] or NULL
	const long long* start;     // [B] or NULL
	float4* state;              // [B,P] {x, y, z, d} (streaming tier)
	long long* out_index;       // [B,n]
	float* out_dist2;           // [B,n]
};

// the fp32 squared distance of the definition: ((dx dx) + (dy dy)) + dz dz, every operation rounded, never contracted
__device__ __forceinline__ float fps_d2(float x, float y, float z, float sx, float sy, float sz)
{
	const float dx = __fsub_rn(x, sx), dy = __fsub_rn(y, sy), dz = __fsub_rn(z, sz);
	return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ unsigned long long fps_key(float d, int i)
{
	return d >= 0.f ? ((unsigned long long)(__float_as_uint(d) + 1u) << 32) | (uint32_t)~(uint32_t)i : 0ull;
}

// the lane's {key, x, y, z} with the largest key of the warp (keys > 0 are distinct), in every lane
__device__ __forceinline__ FpsSlot fps_warp_max(FpsSlot s)
{
	unsigned long long m = s.key;
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
		const unsigned long long v = __shfl_xor_sync(0xffffffffu, m, o);
		m = v > m ? v : m;
	}
	const int src = __ffs(__ballot_sync(0xffffffffu, s.key == m)) - 1;
	return FpsSlot{ m, __shfl_sync(0xffffffffu, s.x, src), __shfl_sync(0xffffffffu, s.y, src), __shfl_sync(0xffffffffu, s.z, src) };
}

// the cluster's largest {key, x, y, z} from each thread's own candidate, in every thread of the cluster (see the top)
template <int T>
__device__ __forceinline__ FpsSlot fps_argmax(const cg::cluster_group& cluster, FpsSlot mine, FpsSlot* s_warp,
	FpsSlot (&s_cta)[2], int parity)
{
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const FpsSlot w = fps_warp_max(mine);
	if (lane == 0) s_warp[warp] = w;
	__syncthreads();
	if (warp == 0) {
		const FpsSlot c = fps_warp_max(lane < T / 32 ? s_warp[lane] : FpsSlot{ 0ull, 0.f, 0.f, 0.f });
		if (lane == 0) s_cta[parity] = c;
	}
	cluster.sync();
	const int C = (int)cluster.num_blocks();
	FpsSlot r{ 0ull, 0.f, 0.f, 0.f };
	if (lane < C) r = *cluster.map_shared_rank(&s_cta[parity], lane);
	return fps_warp_max(r);
}

// the cloud's length, and pick 0 {index, x, y, z} when start names an available point (else key ~0: pick 0 is the argmax)
__device__ __forceinline__ int fps_length(const FpsArgs& a, int b)
{
	const long long L = a.lengths ? a.lengths[b] : (long long)a.P;
	return (int)(L < 0 ? 0 : (L > a.P ? a.P : L));
}
__device__ __forceinline__ bool fps_available(const float* p) { return isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]); }
__device__ __forceinline__ FpsSlot fps_start(const FpsArgs& a, int b, int L)
{
	const long long s = a.start ? a.start[b] : -1;
	if (s >= 0 && s < L) {
		const float* p = a.points + ((size_t)b * a.P + s) * 3;
		if (fps_available(p)) return FpsSlot{ (unsigned long long)s, p[0], p[1], p[2] };
	}
	return FpsSlot{ ~0ull, 0.f, 0.f, 0.f };
}

// rank 0, thread t: the rest of the row from pick t on is padding
__device__ __forceinline__ void fps_pad(const FpsArgs& a, int b, int t, int T)
{
	for (int k = t + (int)threadIdx.x; k < a.n; k += T) {
		a.out_index[(size_t)b * a.n + k] = -1;
		a.out_dist2[(size_t)b * a.n + k] = INFINITY;
	}
}

// The pick loop both tiers share.  update(sidx, sx, sy, sz, first) lowers the thread's d against pick sidx (nothing when
// first) and returns its best {key, x, y, z}.
template <int T, typename Update>
__device__ __forceinline__ void fps_loop(const FpsArgs& a, int b, int L, FpsSlot* s_warp, FpsSlot (&s_cta)[2], Update update)
{
	const cg::cluster_group cluster = cg::this_cluster();
	const bool writer = cluster.block_rank() == 0 && threadIdx.x == 0;
	FpsSlot pick = fps_start(a, b, L);
	int sidx = -1;
	for (int t = 0; t < a.n; t++) {
		float dist;
		if (t == 0 && pick.key != ~0ull) {
			sidx = (int)pick.key;
			dist = INFINITY;
		} else {
			const FpsSlot mine = update(sidx, pick.x, pick.y, pick.z, t == 0);
			pick = fps_argmax<T>(cluster, mine, s_warp, s_cta, t & 1);
			if (pick.key == 0ull) {
				if (cluster.block_rank() == 0) fps_pad(a, b, t, T);
				break;
			}
			sidx = (int)~(uint32_t)pick.key;
			dist = __uint_as_float((uint32_t)(pick.key >> 32) - 1u);
		}
		if (writer) {
			a.out_index[(size_t)b * a.n + t] = sidx;
			a.out_dist2[(size_t)b * a.n + t] = dist;
		}
	}
	cluster.sync();  // the other CTAs may still read this CTA's slots
}

template <int K>
__global__ void __launch_bounds__(FPS_THREADS, 1) fps_kernel(FpsArgs a)
{
	__shared__ FpsSlot s_warp[FPS_THREADS / 32];
	__shared__ FpsSlot s_cta[2];
	const cg::cluster_group cluster = cg::this_cluster();
	const int C = (int)cluster.num_blocks();
	const int b = blockIdx.x / C;
	const int first = (int)cluster.block_rank() * FPS_THREADS + threadIdx.x, stride = C * FPS_THREADS;
	const int L = fps_length(a, b);
	float px[K], py[K], pz[K], d[K];
#pragma unroll
	for (int j = 0; j < K; j++) {
		const int i = first + j * stride;
		px[j] = py[j] = pz[j] = 0.f;
		d[j] = -1.f;
		if (i < L) {
			const float* p = a.points + ((size_t)b * a.P + i) * 3;
			if (fps_available(p)) { px[j] = p[0]; py[j] = p[1]; pz[j] = p[2]; d[j] = INFINITY; }
		}
	}
	fps_loop<FPS_THREADS>(a, b, L, s_warp, s_cta, [&](int sidx, float sx, float sy, float sz, bool first_pick) {
		// the slot j that holds the last pick, if this thread holds it; j and the running best are compile-time selects, so
		// no per-point index lives in a register.  Within a thread the index rises with j, so a strictly larger d wins.
		const int r = sidx - first;
		const int sj = !first_pick && r >= 0 && r % stride == 0 ? r / stride : -1;
		float bd = -1.f, bx = 0.f, by = 0.f, bz = 0.f;
		int bj = 0;
#pragma unroll
		for (int j = 0; j < K; j++) {
			if (!first_pick) d[j] = j == sj ? -1.f : fminf(d[j], fps_d2(px[j], py[j], pz[j], sx, sy, sz));
			if (d[j] > bd) { bd = d[j]; bj = j; bx = px[j]; by = py[j]; bz = pz[j]; }
		}
		return FpsSlot{ fps_key(bd, first + bj * stride), bx, by, bz };
	});
}

__global__ void __launch_bounds__(FPS_THREADS, 1) fps_stream_kernel(FpsArgs a)
{
	__shared__ FpsSlot s_warp[FPS_THREADS / 32];
	__shared__ FpsSlot s_cta[2];
	const cg::cluster_group cluster = cg::this_cluster();
	const int C = (int)cluster.num_blocks();
	const int b = blockIdx.x / C;
	const int first = (int)cluster.block_rank() * FPS_THREADS + threadIdx.x, stride = C * FPS_THREADS;
	const int L = fps_length(a, b);
	float4* const st = a.state + (size_t)b * a.P;
	for (int i = first; i < L; i += stride) {
		const float* p = a.points + ((size_t)b * a.P + i) * 3;
		st[i] = fps_available(p) ? make_float4(p[0], p[1], p[2], INFINITY) : make_float4(0.f, 0.f, 0.f, -1.f);
	}
	// each thread re-reads only the entries it wrote: no barrier is needed before the loop
	fps_loop<FPS_THREADS>(a, b, L, s_warp, s_cta, [&](int sidx, float sx, float sy, float sz, bool first_pick) {
		FpsSlot best{ 0ull, 0.f, 0.f, 0.f };
		for (int i0 = first; i0 < L; i0 += FPS_STREAM_BATCH * stride) {
			float4 q[FPS_STREAM_BATCH];
#pragma unroll
			for (int u = 0; u < FPS_STREAM_BATCH; u++) {
				const int i = i0 + u * stride;
				q[u] = i < L ? st[i] : make_float4(0.f, 0.f, 0.f, -1.f);
			}
#pragma unroll
			for (int u = 0; u < FPS_STREAM_BATCH; u++) {
				const int i = i0 + u * stride;
				float dd = q[u].w;
				if (!first_pick && dd >= 0.f) {
					dd = i == sidx ? -1.f : fminf(dd, fps_d2(q[u].x, q[u].y, q[u].z, sx, sy, sz));
					if (dd != q[u].w) st[i].w = dd;
				}
				const unsigned long long key = fps_key(dd, i);
				if (key > best.key) best = FpsSlot{ key, q[u].x, q[u].y, q[u].z };
			}
		}
		return best;
	});
}

// ---------------------------------------------------------------------------------------------------------------- host
struct FpsPlan {
	int K;  // points per thread of the register tier, 0 for the streaming tier
	int C;  // CTAs per cluster
};

// The largest cluster a kernel can run on the current device (16 needs the non-portable attribute, and a GPU whose GPCs
// cannot hold 16 such CTAs reports 0 active clusters for it).  Cached per device and kernel: a steady-state call, or its
// capture in a CUDA graph, does not repeat the queries.
static cudaError_t fps_max_cluster(const void* fn, int threads, int* max_c)
{
	static std::mutex mu;
	static std::map<std::pair<int, const void*>, int> cache;
	int dev = 0;
	cudaError_t e = cudaGetDevice(&dev);
	if (e != cudaSuccess) return e;
	std::lock_guard<std::mutex> lk(mu);
	const auto key = std::make_pair(dev, fn);
	const auto it = cache.find(key);
	if (it != cache.end()) { *max_c = it->second; return cudaSuccess; }
	e = cudaFuncSetAttribute(fn, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
	if (e != cudaSuccess) return e;
	int c = FPS_MAX_CLUSTER;
	for (; c > 1; c >>= 1) {
		cudaLaunchConfig_t cfg = {};
		cudaLaunchAttribute attr[1];
		attr[0].id = cudaLaunchAttributeClusterDimension;
		attr[0].val.clusterDim.x = c; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
		cfg.gridDim = dim3(c); cfg.blockDim = dim3(threads); cfg.attrs = attr; cfg.numAttrs = 1;
		int clusters = 0;
		e = cudaOccupancyMaxActiveClusters(&clusters, fn, &cfg);
		if (e != cudaSuccess) return e;
		if (clusters > 0) break;
	}
	*max_c = cache[key] = c;
	return cudaSuccess;
}

// 4 points per thread in the smallest cluster of up to 8 CTAs that holds P points, else 16 points per thread in the smallest
// cluster that does, else streaming.  On an H100 a pick of 16 CTAs x 4 points costs more than one of 8 CTAs x 16 points
// (DESIGN.md section 5): the cluster barrier, not the points, sets the pace.
static FpsPlan fps_plan(int P, int max_c4, int max_c16)
{
	for (int K : { 4, 16 }) {
		const int max_c = K == 4 ? std::min(max_c4, 8) : max_c16;
		for (int C = 1; C <= max_c; C *= 2)
			if ((long long)C * FPS_THREADS * K >= P) return FpsPlan{ K, C };
	}
	return FpsPlan{ 0, 0 };
}

size_t fps_state_bytes(int B, int P) { return (size_t)B * (size_t)P * sizeof(float4) + 256; }

template <typename... Args>
static cudaError_t fps_launch(void (*fn)(Args...), int B, int C, int threads, cudaStream_t st, const FpsArgs& a)
{
	cudaLaunchConfig_t cfg = {};
	cudaLaunchAttribute attr[1];
	attr[0].id = cudaLaunchAttributeClusterDimension;
	attr[0].val.clusterDim.x = C; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
	cfg.gridDim = dim3((unsigned)B * (unsigned)C);
	cfg.blockDim = dim3(threads);
	cfg.stream = st;
	cfg.attrs = attr;
	cfg.numAttrs = 1;
	return cudaLaunchKernelEx(&cfg, fn, a);
}

cudaError_t fps_run(void* state, int B, int P, int n, const float* points, const long long* lengths, const long long* start,
	long long* out_index, float* out_dist2, cudaStream_t st)
{
	if (B == 0 || n == 0) return cudaSuccess;
	int c4 = 0, c16 = 0, cs = 0;
	cudaError_t e = fps_max_cluster((const void*)fps_kernel<4>, FPS_THREADS, &c4);
	if (e == cudaSuccess) e = fps_max_cluster((const void*)fps_kernel<16>, FPS_THREADS, &c16);
	if (e != cudaSuccess) return e;
	const FpsPlan plan = fps_plan(P, c4, c16);
	FpsArgs a{ P, n, points, lengths, start, reinterpret_cast<float4*>((reinterpret_cast<uintptr_t>(state) + 255) & ~(uintptr_t)255),
		out_index, out_dist2 };
	if (plan.K == 4) return fps_launch(fps_kernel<4>, B, plan.C, FPS_THREADS, st, a);
	if (plan.K == 16) return fps_launch(fps_kernel<16>, B, plan.C, FPS_THREADS, st, a);
	e = fps_max_cluster((const void*)fps_stream_kernel, FPS_THREADS, &cs);
	if (e != cudaSuccess) return e;
	return fps_launch(fps_stream_kernel, B, cs, FPS_THREADS, st, a);
}

}  // namespace mgs
