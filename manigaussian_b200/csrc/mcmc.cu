// MCMC density control (include/mgs_rasterizer.h, mgs_mcmc_relocate / mgs_mcmc_perturb; 3DGS as Markov chain Monte Carlo,
// Kheradmand et al. 2024, as gsplat's MCMCStrategy runs it).
//
// Relocation, a chain of launches on the caller's stream, nothing read back:
//   scan     CUB's inclusive uint64 sum of the weights w_i = floor(2^24 sigmoid_f64(x_i)) (0 where dead), computed on the
//            fly by a transform iterator: S [P_old];
//   draw     one thread per slot j: the dead test, u = mulhi64(r64_j, T), src_j = min{i : S_i > u} by binary search,
//            atomicAdd into m[src_j], a warp-aggregated atomicAdd into the destination count;
//   source   one thread per slot i < P_old with m_i > 0: the fp64 opacity and scale of the definition, written into the
//            source's own row, its moments zeroed; thread 0 advances the generator's offset (every reader has finished);
//   copy     blockIdx.y picks one tensor: params and extra rows are copied from src_j to j, moments zeroed at j.
// The tensors travel by value in one __grid_constant__ struct, so a captured graph holds no device pointer table.
//
// Perturbation: one thread per Gaussian, then a one-thread launch that advances the offset.
#include <cub/device/device_scan.cuh>
#include <cub/iterator/transform_input_iterator.cuh>
#include <map>
#include <mutex>
#include "../../include/mgs_rasterizer.h"
#include "mgs_common.cuh"
#include "mgs_kernels.h"
#include "philox.cuh"

namespace mgs {

constexpr int MCMC_THREADS = 256;
constexpr int MCMC_MAX_TENSORS = 4 + MGS_MCMC_MAX_ROWS + MGS_MCMC_MAX_MOMENTS;
constexpr int MCMC_N_MAX = 51;            // gsplat's clamp of n = m + 1
constexpr uint32_t MCMC_TAG_RELOCATE = 0;  // counter word 3: relocation and perturbation never share a draw
constexpr uint32_t MCMC_TAG_PERTURB = 1;

// ---------------------------------------------------------------------------------------------------------------- relocation
struct McmcTensors {
	int n_copy;                          // tensors [0, n_copy) are copied, [n_copy, n) zeroed
	int n;
	float* ptr[MCMC_MAX_TENSORS];
	int width[MCMC_MAX_TENSORS];         // floats per row
};

struct McmcWeight {
	float t;
	__device__ __forceinline__ unsigned long long operator()(float x) const
	{
		// NaN is not <= t, so it counts as alive, with weight 0: never a source, never a destination
		if (!(x > t)) return 0ull;
		const double o = 1.0 / (1.0 + exp(-(double)x));
		return (unsigned long long)floor(o * 16777216.0);
	}
};
using McmcWeightIt = cub::TransformInputIterator<unsigned long long, McmcWeight, const float*>;

__device__ __forceinline__ bool mcmc_dest(int j, int P_old, const float* x, float t)
{
	return j >= P_old || x[j] <= t;
}

__global__ void __launch_bounds__(MCMC_THREADS) mcmc_draw_kernel(int P_old, int P, float t, const float* __restrict__ x,
	const unsigned long long* __restrict__ S, const long long* __restrict__ rng, uint32_t* __restrict__ m,
	long long* __restrict__ source, long long* __restrict__ relocated)
{
	const int j = blockIdx.x * MCMC_THREADS + threadIdx.x;
	long long src = -1;
	const unsigned long long T = P_old > 0 ? S[P_old - 1] : 0ull;
	if (j < P && T > 0 && mcmc_dest(j, P_old, x, t)) {
		const uint4 w = philox_draw(rng, (uint32_t)j, MCMC_TAG_RELOCATE);
		const unsigned long long u = __umul64hi(((unsigned long long)w.y << 32) | w.x, T);  // u < T
		int lo = 0, hi = P_old - 1;  // S[hi] = T > u
		while (lo < hi) {
			const int mid = (lo + hi) >> 1;
			if (S[mid] > u) hi = mid; else lo = mid + 1;
		}
		src = lo;
		atomicAdd(m + lo, 1u);
	}
	const unsigned b = __ballot_sync(0xffffffffu, src >= 0);
	if (b && (threadIdx.x & 31) == __ffs(b) - 1) atomicAdd((unsigned long long*)relocated, (unsigned long long)__popc(b));
	if (j < P) source[j] = src;
}

__device__ __forceinline__ void mcmc_zero_row(float* p, int w, size_t i)
{
	float* r = p + i * w;
	if ((w & 3) == 0 && (reinterpret_cast<uintptr_t>(p) & 15) == 0) {
		for (int k = 0; k < w; k += 4) *reinterpret_cast<float4*>(r + k) = make_float4(0.f, 0.f, 0.f, 0.f);
	} else {
		for (int k = 0; k < w; k++) r[k] = 0.f;
	}
}

// o' = -expm1(log1p(-o) / n);  s' / s = o / sum_{j=1..n} C(n,j) (-1)^(j-1) o'^j / sqrt(j)  (all fp64)
__device__ __forceinline__ double mcmc_scale_ratio(double o, int n, double* o_new)
{
	const double a = -expm1(log1p(-o) / n);
	double c = 1.0, p = 1.0, den = 0.0;
	for (int j = 1; j <= n; j++) {
		c = c * (n - j + 1) / j;  // C(n, j), exact: every intermediate is an integer below 2^53
		p *= a;
		const double term = c * p / sqrt((double)j);
		den += (j & 1) ? term : -term;
	}
	*o_new = a;
	return o / den;
}

__global__ void __launch_bounds__(MCMC_THREADS) mcmc_source_kernel(int P_old, double min_opacity, float* __restrict__ x,
	float* __restrict__ log_scales, const uint32_t* __restrict__ m, long long* __restrict__ rng, const __grid_constant__ McmcTensors a)
{
	const int i = blockIdx.x * MCMC_THREADS + threadIdx.x;
	if (i == 0) rng[1] += 1;  // the draw launch, the only reader of the offset, has finished
	if (i >= P_old || m[i] == 0) return;
	const int n = min((int)m[i] + 1, MCMC_N_MAX);
	const double o = 1.0 / (1.0 + exp(-(double)x[i]));
	double on;
	const double ratio = mcmc_scale_ratio(o, n, &on);
	on = fmin(fmax(on, min_opacity), 1.0 - 1.0 / 8388608.0);
	x[i] = (float)log(on / (1.0 - on));
#pragma unroll
	for (int k = 0; k < 3; k++) log_scales[3 * (size_t)i + k] = (float)log(exp((double)log_scales[3 * (size_t)i + k]) * ratio);
	for (int k = a.n_copy; k < a.n; k++) mcmc_zero_row(a.ptr[k], a.width[k], (size_t)i);
}

__global__ void __launch_bounds__(MCMC_THREADS) mcmc_copy_kernel(int P, const long long* __restrict__ source,
	const __grid_constant__ McmcTensors a)
{
	const int j = blockIdx.x * MCMC_THREADS + threadIdx.x;
	if (j >= P) return;
	const long long s = source[j];
	if (s < 0) return;
	const int k = blockIdx.y;
	float* const p = a.ptr[k];
	const int w = a.width[k];
	if (k >= a.n_copy) { mcmc_zero_row(p, w, (size_t)j); return; }
	const float* src = p + (size_t)s * w;
	float* dst = p + (size_t)j * w;
	if ((w & 3) == 0 && (reinterpret_cast<uintptr_t>(p) & 15) == 0) {
		for (int q = 0; q < w; q += 4) *reinterpret_cast<float4*>(dst + q) = *reinterpret_cast<const float4*>(src + q);
	} else {
		for (int q = 0; q < w; q++) dst[q] = src[q];
	}
}

// ---------------------------------------------------------------------------------------------------------------- host
#define MCMC_TRY(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return e_; } while (0)

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// CUB's scan scratch for P items on the current device, cached like knn_temp_bytes (a steady-state call, or its capture
// in a CUDA graph, does not repeat the size query); emptied at 256 entries, since P grows over a fit
static cudaError_t mcmc_temp_bytes(int P, size_t* bytes)
{
	static std::mutex mu;
	static std::map<std::pair<int, int>, size_t> cache;
	int dev = 0;
	MCMC_TRY(cudaGetDevice(&dev));
	std::lock_guard<std::mutex> lk(mu);
	const auto key = std::make_pair(dev, P);
	const auto it = cache.find(key);
	if (it != cache.end()) { *bytes = it->second; return cudaSuccess; }
	size_t b = 0;
	MCMC_TRY(cub::DeviceScan::InclusiveSum(nullptr, b, McmcWeightIt(nullptr, McmcWeight{ 0.f }), (unsigned long long*)nullptr,
		std::max(P, 1)));
	if (cache.size() >= 256) cache.clear();
	*bytes = cache[key] = b;
	return cudaSuccess;
}

cudaError_t mcmc_state_bytes(int P, size_t* bytes)
{
	size_t tb = 0;
	MCMC_TRY(mcmc_temp_bytes(P, &tb));
	*bytes = align256((size_t)P * sizeof(unsigned long long)) + align256((size_t)P * sizeof(uint32_t)) + tb + 256;
	return cudaSuccess;
}

cudaError_t mcmc_relocate(void* state, int P_old, int P, float min_opacity, float* means, float* quats, float* log_scales,
	float* opacity_logit, int num_rows, float* const* rows, const int* row_widths, int num_moments, float* const* moments,
	const int* moment_widths, long long* rng, long long* out_source, long long* out_relocated, cudaStream_t st)
{
	const double mo = (double)min_opacity;
	const float t = (float)log(mo / (1.0 - mo));
	McmcTensors a{};
	float* base[4] = { means, quats, log_scales, opacity_logit };
	const int base_w[4] = { 3, 4, 3, 1 };
	for (int k = 0; k < 4; k++) { a.ptr[a.n] = base[k]; a.width[a.n++] = base_w[k]; }
	for (int k = 0; k < num_rows; k++) { a.ptr[a.n] = rows[k]; a.width[a.n++] = row_widths[k]; }
	a.n_copy = a.n;
	for (int k = 0; k < num_moments; k++) { a.ptr[a.n] = moments[k]; a.width[a.n++] = moment_widths[k]; }

	char* p = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(state) + 255) & ~(uintptr_t)255);
	unsigned long long* S = reinterpret_cast<unsigned long long*>(p); p += align256((size_t)P_old * sizeof(unsigned long long));
	uint32_t* m = reinterpret_cast<uint32_t*>(p); p += align256((size_t)P_old * sizeof(uint32_t));
	MCMC_TRY(cudaMemsetAsync(out_relocated, 0, sizeof(long long), st));
	if (P_old > 0) {
		size_t tb = 0;
		MCMC_TRY(mcmc_temp_bytes(P_old, &tb));
		MCMC_TRY(cub::DeviceScan::InclusiveSum(p, tb, McmcWeightIt(opacity_logit, McmcWeight{ t }), S, P_old, st));
		MCMC_TRY(cudaMemsetAsync(m, 0, (size_t)P_old * sizeof(uint32_t), st));
	}
	if (P > 0)
		mcmc_draw_kernel<<<ceil_div(P, MCMC_THREADS), MCMC_THREADS, 0, st>>>(P_old, P, t, opacity_logit, S, rng, m, out_source,
			out_relocated);
	mcmc_source_kernel<<<std::max(ceil_div(P_old, MCMC_THREADS), 1), MCMC_THREADS, 0, st>>>(P_old, mo, opacity_logit, log_scales,
		m, rng, a);
	MCMC_TRY(cudaGetLastError());
	if (P > 0) mcmc_copy_kernel<<<dim3(ceil_div(P, MCMC_THREADS), a.n), MCMC_THREADS, 0, st>>>(P, out_source, a);
	return cudaGetLastError();
}

__global__ void __launch_bounds__(MCMC_THREADS) mcmc_perturb_kernel(int P, float* __restrict__ means, const float4* __restrict__ quats,
	const float* __restrict__ log_scales, const float* __restrict__ x, const float* __restrict__ scale, const long long* __restrict__ rng)
{
	const int i = blockIdx.x * MCMC_THREADS + threadIdx.x;
	if (i >= P) return;
	float z0, z1, z2;
	philox_normals(philox_draw(rng, (uint32_t)i, MCMC_TAG_PERTURB), z0, z1, z2);

	float4 q = quats[i];
	const float inv = 1.f / fmaxf(sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w), 1e-12f);
	const float qn[4] = { q.x * inv, q.y * inv, q.z * inv, q.w * inv };
	const float s[3] = { expf(log_scales[3 * (size_t)i]), expf(log_scales[3 * (size_t)i + 1]), expf(log_scales[3 * (size_t)i + 2]) };
	float c[6];
	cov3d_from_scale_rot(s, 1.f, qn, c);
	const float o = 1.f / (1.f + expf(-x[i]));
	const float g = 1.f / (1.f + expf(-100.f * ((1.f - o) - 0.995f))) * __ldg(scale);
	float* mu = means + 3 * (size_t)i;
	mu[0] += (c[0] * z0 + c[1] * z1 + c[2] * z2) * g;
	mu[1] += (c[1] * z0 + c[3] * z1 + c[4] * z2) * g;
	mu[2] += (c[2] * z0 + c[4] * z1 + c[5] * z2) * g;
}

__global__ void mcmc_advance_kernel(long long* rng) { rng[1] += 1; }

cudaError_t mcmc_perturb(int P, float* means, const float* quats, const float* log_scales, const float* opacity_logit,
	const float* scale, long long* rng, cudaStream_t st)
{
	if (P > 0)
		mcmc_perturb_kernel<<<ceil_div(P, MCMC_THREADS), MCMC_THREADS, 0, st>>>(P, means, reinterpret_cast<const float4*>(quats),
			log_scales, opacity_logit, scale, rng);
	mcmc_advance_kernel<<<1, 1, 0, st>>>(rng);
	return cudaGetLastError();
}

}  // namespace mgs
