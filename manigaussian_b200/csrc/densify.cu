// Default density control (include/mgs_rasterizer.h, mgs_densify_stats / mgs_densify_count / mgs_densify_emit; 3DGS's
// adaptive density control as gsplat's DefaultStrategy runs it).
//
// Statistics, every step: one thread per Gaussian walks the views of a launch in order (up to DENSIFY_VIEW_CHUNK views,
// whose sizes travel by value), with every operation rounded to fp32 and no FMA; no atomics, nothing read back.
//
// Refinement, two calls:
//   count    classify: one thread per Gaussian writes its flags (original kept, clone kept, children kept) and adds
//            its clone and split decisions to the totals with warp-aggregated integer atomics;
//            scan: CUB's inclusive int4 sum of the three flags;
//            totals: one thread writes {n_new, cloned, split, pruned}, which the caller reads back to size the outputs;
//   emit     one thread per (Gaussian, tensor) writes the Gaussian's rows at its exclusive offsets in the four output
//            segments [kept originals | kept clones | kept first children | kept second children]; the means and
//            log-scale blocks compute the children, the means block writes `source`; then one thread advances the offset.
// The tensors travel by value in one __grid_constant__ struct, as mcmc.cu's do.
#include <cub/device/device_scan.cuh>
#include <cub/iterator/transform_input_iterator.cuh>
#include <map>
#include <mutex>
#include "../../include/mgs_rasterizer.h"
#include "mgs_common.cuh"
#include "mgs_kernels.h"
#include "philox.cuh"

namespace mgs {

constexpr int DENSIFY_THREADS = 256;
constexpr int DENSIFY_MAX_TENSORS = 4 + MGS_MCMC_MAX_ROWS + MGS_MCMC_MAX_MOMENTS;
constexpr uint32_t DENSIFY_TAG_CHILD = 2;  // counter word 3: child b draws at tag 2 + b; mcmc.cu owns tags 0 and 1
constexpr double DENSIFY_LOG_1_6 = 0.47000362924573558;  // log(1.6): a child's scale is its parent's / 1.6
constexpr uint32_t F_KEEP = 1u, F_CLONE = 2u, F_CHILD = 4u;

// ---------------------------------------------------------------------------------------------------------------- statistics
__global__ void __launch_bounds__(DENSIFY_THREADS) densify_stats_kernel(int P, const float* __restrict__ grad,
	const int* __restrict__ radii, const __grid_constant__ DensifyViews views, float scale_host, const float* __restrict__ scale,
	float* __restrict__ grad2d, int* __restrict__ count, float* __restrict__ radius)
{
	const int i = blockIdx.x * DENSIFY_THREADS + threadIdx.x;
	if (i >= P) return;
	const float sc = scale ? __ldg(scale) : scale_host;
	float g = grad2d[i], r = radius[i];
	int c = count[i];
	for (int v = 0; v < views.V; v++) {
		const size_t vi = (size_t)v * P + i;
		const int rv = radii[vi];
		if (rv <= 0) continue;
		const float gx = grad[3 * vi], gy = grad[3 * vi + 1];
		const float n = __fsqrt_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)));
		g = __fadd_rn(g, __fmul_rn(n, sc));
		c += 1;
		r = fmaxf(r, __fdiv_rn((float)rv, views.size[v]));
	}
	grad2d[i] = g;
	count[i] = c;
	radius[i] = r;
}

cudaError_t densify_stats(int V, int P, const float* viewspace_grad, const int* radii, const int* sizes, float scale,
	const float* scale_device, float* grad2d, int* count, float* radius, cudaStream_t st)
{
	if (P == 0) return cudaSuccess;
	for (int v0 = 0; v0 < V; v0 += DENSIFY_VIEW_CHUNK) {
		DensifyViews views{};
		views.V = std::min(V - v0, DENSIFY_VIEW_CHUNK);
		for (int u = 0; u < views.V; u++) views.size[u] = (float)sizes[v0 + u];
		densify_stats_kernel<<<ceil_div(P, DENSIFY_THREADS), DENSIFY_THREADS, 0, st>>>(P, viewspace_grad + (size_t)v0 * P * 3,
			radii + (size_t)v0 * P, views, scale, scale_device, grad2d, count, radius);
	}
	return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------- count
struct DensifyRule {
	float grad_threshold, t_small, grow_scale2d, t_opa, t_big, prune_scale2d;
	int prune_too_big;
	__device__ __forceinline__ bool pruned(float x, float L, float r) const
	{
		return x < t_opa || (prune_too_big && (L > t_big || r > prune_scale2d));
	}
};

// fmaxf ignores a NaN operand
__device__ __forceinline__ float densify_largest(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
__device__ __forceinline__ float densify_child_scale(float ls) { return (float)((double)ls - DENSIFY_LOG_1_6); }

__global__ void __launch_bounds__(DENSIFY_THREADS) densify_classify_kernel(int P, const float* __restrict__ log_scales,
	const float* __restrict__ x, const float* __restrict__ grad2d, const int* __restrict__ count, const float* __restrict__ radius,
	const DensifyRule rule, uint8_t* __restrict__ flags, long long* __restrict__ out_counts)
{
	const int i = blockIdx.x * DENSIFY_THREADS + threadIdx.x;
	bool clone = false, split = false;
	if (i < P) {
		const float* ls = log_scales + 3 * (size_t)i;
		const float l0 = ls[0], l1 = ls[1], l2 = ls[2];
		const float L = densify_largest(l0, l1, l2);
		const float Lc = densify_largest(densify_child_scale(l0), densify_child_scale(l1), densify_child_scale(l2));
		const float r = radius[i], xi = x[i];
		const bool high = __fdiv_rn(grad2d[i], (float)max(count[i], 1)) > rule.grad_threshold;
		const bool small = L <= rule.t_small;
		clone = high && small;
		split = (high && !small) || r > rule.grow_scale2d;
		const bool gone = rule.pruned(xi, L, r);
		uint32_t f = 0;
		if (!split && !gone) f |= F_KEEP;
		if (clone && !gone) f |= F_CLONE;
		if (split && !rule.pruned(xi, Lc, r)) f |= F_CHILD;
		flags[i] = (uint8_t)f;
	}
	const unsigned bc = __ballot_sync(0xffffffffu, clone), bs = __ballot_sync(0xffffffffu, split);
	const int lane = threadIdx.x & 31;
	if (bc && lane == __ffs(bc) - 1) atomicAdd((unsigned long long*)(out_counts + 1), (unsigned long long)__popc(bc));
	if (bs && lane == __ffs(bs) - 1) atomicAdd((unsigned long long*)(out_counts + 2), (unsigned long long)__popc(bs));
}

struct DensifyFlagCounts {
	__device__ __forceinline__ int4 operator()(uint8_t f) const
	{
		return make_int4(f & F_KEEP, (f & F_CLONE) >> 1, (f & F_CHILD) >> 2, 0);
	}
};
struct DensifySum {
	__device__ __forceinline__ int4 operator()(const int4& a, const int4& b) const
	{
		return make_int4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
	}
};
using DensifyFlagIt = cub::TransformInputIterator<int4, DensifyFlagCounts, const uint8_t*>;

__global__ void densify_totals_kernel(int P, const int4* __restrict__ scan, long long* __restrict__ out_counts)
{
	const int4 t = scan[P - 1];
	const long long n_new = (long long)t.x + t.y + 2 * (long long)t.z;
	out_counts[0] = n_new;
	out_counts[3] = (long long)P + out_counts[1] + out_counts[2] - n_new;
}

#define DENSIFY_TRY(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return e_; } while (0)

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// CUB's scan scratch for P items on the current device, cached as mcmc.cu caches its own
static cudaError_t densify_temp_bytes(int P, size_t* bytes)
{
	static std::mutex mu;
	static std::map<std::pair<int, int>, size_t> cache;
	int dev = 0;
	DENSIFY_TRY(cudaGetDevice(&dev));
	std::lock_guard<std::mutex> lk(mu);
	const auto key = std::make_pair(dev, P);
	const auto it = cache.find(key);
	if (it != cache.end()) { *bytes = it->second; return cudaSuccess; }
	size_t b = 0;
	DENSIFY_TRY(cub::DeviceScan::InclusiveScan(nullptr, b, DensifyFlagIt(nullptr, DensifyFlagCounts{}), (int4*)nullptr,
		DensifySum{}, std::max(P, 1)));
	if (cache.size() >= 256) cache.clear();
	*bytes = cache[key] = b;
	return cudaSuccess;
}

cudaError_t densify_state_bytes(int P, size_t* bytes)
{
	size_t tb = 0;
	DENSIFY_TRY(densify_temp_bytes(P, &tb));
	*bytes = align256((size_t)P) + align256((size_t)P * sizeof(int4)) + tb + 256;
	return cudaSuccess;
}

struct DensifyStateView {
	uint8_t* flags;
	int4* scan;
	void* temp;
};

static DensifyStateView densify_carve(void* state, int P)
{
	char* p = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(state) + 255) & ~(uintptr_t)255);
	DensifyStateView s;
	s.flags = reinterpret_cast<uint8_t*>(p); p += align256((size_t)P);
	s.scan = reinterpret_cast<int4*>(p); p += align256((size_t)P * sizeof(int4));
	s.temp = p;
	return s;
}

cudaError_t densify_count(void* state, int P, const float* log_scales, const float* opacity_logit, const float* grad2d,
	const int* count, const float* radius, double scene_scale, float grad_threshold, double grow_scale3d, float grow_scale2d,
	double prune_opacity, double prune_scale3d, float prune_scale2d, int prune_too_big, long long* out_counts, cudaStream_t st)
{
	DENSIFY_TRY(cudaMemsetAsync(out_counts, 0, 4 * sizeof(long long), st));
	if (P == 0) return cudaSuccess;
	DensifyRule rule;
	rule.grad_threshold = grad_threshold;
	rule.t_small = (float)log(grow_scale3d * scene_scale);
	rule.grow_scale2d = grow_scale2d;
	rule.t_opa = (float)log(prune_opacity / (1.0 - prune_opacity));
	rule.t_big = (float)log(prune_scale3d * scene_scale);
	rule.prune_scale2d = prune_scale2d;
	rule.prune_too_big = prune_too_big ? 1 : 0;
	const DensifyStateView s = densify_carve(state, P);
	densify_classify_kernel<<<ceil_div(P, DENSIFY_THREADS), DENSIFY_THREADS, 0, st>>>(P, log_scales, opacity_logit, grad2d, count,
		radius, rule, s.flags, out_counts);
	DENSIFY_TRY(cudaGetLastError());
	size_t tb = 0;
	DENSIFY_TRY(densify_temp_bytes(P, &tb));
	DENSIFY_TRY(cub::DeviceScan::InclusiveScan(s.temp, tb, DensifyFlagIt(s.flags, DensifyFlagCounts{}), s.scan, DensifySum{}, P, st));
	densify_totals_kernel<<<1, 1, 0, st>>>(P, s.scan, out_counts);
	return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------- emit
struct DensifyTensors {
	int n_copy;                          // tensors [0, n_copy) are copied to every output row, [n_copy, n) are moments
	int n;
	const float* src[DENSIFY_MAX_TENSORS];
	float* dst[DENSIFY_MAX_TENSORS];
	int width[DENSIFY_MAX_TENSORS];      // floats per row
};

__device__ __forceinline__ void densify_copy_row(const float* __restrict__ s, float* __restrict__ d, int w, bool vec)
{
	if (vec) {
		for (int k = 0; k < w; k += 4) *reinterpret_cast<float4*>(d + k) = *reinterpret_cast<const float4*>(s + k);
	} else {
		for (int k = 0; k < w; k++) d[k] = s[k];
	}
}

__device__ __forceinline__ void densify_zero_row(float* __restrict__ d, int w, bool vec)
{
	if (vec) {
		for (int k = 0; k < w; k += 4) *reinterpret_cast<float4*>(d + k) = make_float4(0.f, 0.f, 0.f, 0.f);
	} else {
		for (int k = 0; k < w; k++) d[k] = 0.f;
	}
}

// child b's mean: mu + R(q^) diag(exp(ls)) z, q^ = q / max(|q|, 1e-12), z from slot i at tag 2 + b
__device__ __forceinline__ void densify_child_mean(const float* mu, const float* q, const float* ls, const long long* rng,
	uint32_t i, uint32_t b, float* out)
{
	float z[3];
	philox_normals(philox_draw(rng, i, DENSIFY_TAG_CHILD + b), z[0], z[1], z[2]);
	const float inv = 1.f / fmaxf(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), 1e-12f);
	const float r = q[0] * inv, x = q[1] * inv, y = q[2] * inv, w = q[3] * inv;
	const float R[3][3] = {
		{ 1.f - 2.f * (y * y + w * w), 2.f * (x * y - r * w), 2.f * (x * w + r * y) },
		{ 2.f * (x * y + r * w), 1.f - 2.f * (x * x + w * w), 2.f * (y * w - r * x) },
		{ 2.f * (x * w - r * y), 2.f * (y * w + r * x), 1.f - 2.f * (x * x + y * y) } };
	const float d[3] = { expf(ls[0]) * z[0], expf(ls[1]) * z[1], expf(ls[2]) * z[2] };
#pragma unroll
	for (int k = 0; k < 3; k++) out[k] = mu[k] + (R[k][0] * d[0] + R[k][1] * d[1] + R[k][2] * d[2]);
}

__global__ void __launch_bounds__(DENSIFY_THREADS) densify_emit_kernel(int P, const uint8_t* __restrict__ flags,
	const int4* __restrict__ scan, const long long* __restrict__ rng, long long* __restrict__ source,
	const __grid_constant__ DensifyTensors a)
{
	const int i = blockIdx.x * DENSIFY_THREADS + threadIdx.x;
	if (i >= P) return;
	const uint32_t f = flags[i];
	if (!f) return;
	const int4 tot = scan[P - 1], s = scan[i];
	const size_t o_keep = (size_t)(s.x - (int)(f & F_KEEP));
	const size_t o_clone = (size_t)tot.x + (s.y - (int)((f & F_CLONE) >> 1));
	const size_t o_child0 = (size_t)tot.x + tot.y + (s.z - (int)((f & F_CHILD) >> 2));
	const size_t o_child1 = o_child0 + tot.z;
	const int k = blockIdx.y;
	const int w = a.width[k];
	const float* src = a.src[k] + (size_t)i * w;
	float* const dst = a.dst[k];
	const bool vec = (w & 3) == 0 && ((reinterpret_cast<uintptr_t>(a.src[k]) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0;
	if (k >= a.n_copy) {  // a moment: the kept original's row, zero for every new row
		if (f & F_KEEP) densify_copy_row(src, dst + o_keep * w, w, vec);
		if (f & F_CLONE) densify_zero_row(dst + o_clone * w, w, vec);
		if (f & F_CHILD) { densify_zero_row(dst + o_child0 * w, w, vec); densify_zero_row(dst + o_child1 * w, w, vec); }
		return;
	}
	if (f & F_KEEP) densify_copy_row(src, dst + o_keep * w, w, vec);
	if (f & F_CLONE) densify_copy_row(src, dst + o_clone * w, w, vec);
	if (k == 0) {
		if (f & F_KEEP) source[o_keep] = i;
		if (f & F_CLONE) source[o_clone] = i;
		if (f & F_CHILD) { source[o_child0] = i; source[o_child1] = i; }
	}
	if (!(f & F_CHILD)) return;
	if (k == 0) {
		const float* q = a.src[1] + 4 * (size_t)i;
		const float* ls = a.src[2] + 3 * (size_t)i;
		densify_child_mean(src, q, ls, rng, (uint32_t)i, 0, dst + o_child0 * 3);
		densify_child_mean(src, q, ls, rng, (uint32_t)i, 1, dst + o_child1 * 3);
	} else if (k == 2) {
#pragma unroll
		for (int q = 0; q < 3; q++) {
			const float c = densify_child_scale(src[q]);
			dst[o_child0 * 3 + q] = c;
			dst[o_child1 * 3 + q] = c;
		}
	} else {
		densify_copy_row(src, dst + o_child0 * w, w, vec);
		densify_copy_row(src, dst + o_child1 * w, w, vec);
	}
}

__global__ void densify_advance_kernel(long long* rng) { rng[1] += 1; }

cudaError_t densify_emit(void* state, int P, const float* means, const float* quats, const float* log_scales,
	const float* opacity_logit, int num_rows, const float* const* rows, const int* row_widths, int num_moments,
	const float* const* moments, const int* moment_widths, float* new_means, float* new_quats, float* new_log_scales,
	float* new_opacity_logit, float* const* new_rows, float* const* new_moments, long long* rng, long long* out_source,
	cudaStream_t st)
{
	DensifyTensors a{};
	const float* base[4] = { means, quats, log_scales, opacity_logit };
	float* new_base[4] = { new_means, new_quats, new_log_scales, new_opacity_logit };
	const int base_w[4] = { 3, 4, 3, 1 };
	for (int k = 0; k < 4; k++) { a.src[a.n] = base[k]; a.dst[a.n] = new_base[k]; a.width[a.n++] = base_w[k]; }
	for (int k = 0; k < num_rows; k++) { a.src[a.n] = rows[k]; a.dst[a.n] = new_rows[k]; a.width[a.n++] = row_widths[k]; }
	a.n_copy = a.n;
	for (int k = 0; k < num_moments; k++) { a.src[a.n] = moments[k]; a.dst[a.n] = new_moments[k]; a.width[a.n++] = moment_widths[k]; }
	if (P > 0) {
		const DensifyStateView s = densify_carve(state, P);
		densify_emit_kernel<<<dim3(ceil_div(P, DENSIFY_THREADS), a.n), DENSIFY_THREADS, 0, st>>>(P, s.flags, s.scan, rng, out_source, a);
		DENSIFY_TRY(cudaGetLastError());
	}
	densify_advance_kernel<<<1, 1, 0, st>>>(rng);  // after every reader of the offset
	return cudaGetLastError();
}

}  // namespace mgs
