// Camera rays: the ray of each pixel of a view through the inverse of the projection's map of a mean (include/mgs_rasterizer.h,
// mgs_camera_rays; camera.cuh: camera_ray and camera_ray_bwd, beside screen_mean).  Both directions run one thread per (view,
// pixel) with the view in blockIdx.y.  The backward recomputes each ray rather than storing it, and sums its camera terms over
// the warp by shuffles in a fixed order, then over the CTA's warps in warp order, into one row per CTA, as
// vis_points_bwd_kernel does; camera_grad_reduce_kernel finishes the sums.
#include "camera.cuh"

namespace mgs {

__device__ __forceinline__ void ray_pixel(const RaysArgs& a, size_t q, int i, float& u, float& v)
{
	if (a.pixels) { u = a.pixels[2 * q]; v = a.pixels[2 * q + 1]; }
	else { u = (float)(i % a.grid_w); v = (float)(i / a.grid_w); }
}

__global__ void __launch_bounds__(RAYS_THREADS) rays_fwd_kernel(RaysArgs a)
{
	const int i = blockIdx.x * RAYS_THREADS + threadIdx.x;
	if (i >= a.N) return;
	const size_t q = (size_t)blockIdx.y * a.N + i;
	float u, v, o[3], d[3];
	ray_pixel(a, q, i, u, v);
	const bool ok = camera_ray(a.cam[blockIdx.y], u, v, o, d);
	const float nan = __int_as_float(0x7fffffff);
#pragma unroll
	for (int k = 0; k < 3; k++) {
		a.origin[3 * q + k] = ok ? o[k] : nan;
		a.direction[3 * q + k] = ok ? d[k] : nan;
	}
	a.valid[q] = ok ? 1 : 0;
}

template <bool CAM>
__global__ void __launch_bounds__(RAYS_THREADS) rays_bwd_kernel(RaysArgs a)
{
	const int i = blockIdx.x * RAYS_THREADS + threadIdx.x;
	const int w = blockIdx.y;
	const bool in = i < a.N;
	const size_t q = (size_t)w * a.N + (in ? i : 0);
	__shared__ float cam_sm[CAM ? RAYS_THREADS / 32 * CAM_ALL_TERMS : 1];
	float cg[CAM ? CAM_ALL_TERMS : 1];
	float go[3] = { 0.f, 0.f, 0.f }, gd[3] = { 0.f, 0.f, 0.f }, gu = 0.f, gv = 0.f;
	if (in) {
#pragma unroll
		for (int k = 0; k < 3; k++) {
			if (a.dL_dorigin) go[k] = a.dL_dorigin[3 * q + k];
			if (a.dL_ddirection) gd[k] = a.dL_ddirection[3 * q + k];
		}
		float u, v;
		ray_pixel(a, q, i, u, v);
		// an invalid ray's outputs are NaN constants: its cotangents are ignored, and it writes zeros
		camera_ray_bwd<CAM>(a.cam[w], u, v, go, gd, gu, gv, cg);
		if (a.dL_dpixels) { a.dL_dpixels[2 * q] = gu; a.dL_dpixels[2 * q + 1] = gv; }
	} else if constexpr (CAM) {
#pragma unroll
		for (int k = 0; k < CAM_ALL_TERMS; k++) cg[k] = 0.f;
	}
	if constexpr (CAM) {
		float* rows = a.cam_rows[w];
		if (!rows) return;  // uniform over the CTA
		const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
		for (int k = 0; k < CAM_ALL_TERMS; k++) {
			float s = cg[k];
#pragma unroll
			for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
			if (lane == 0) cam_sm[warp * CAM_ALL_TERMS + k] = s;
		}
		__syncthreads();
		float* intr = a.intr_rows[w];
		for (int k = threadIdx.x; k < CAM_ALL_TERMS; k += RAYS_THREADS) {
			float s = 0.f;
			for (int u2 = 0; u2 < RAYS_THREADS / 32; u2++) s += cam_sm[u2 * CAM_ALL_TERMS + k];
			if (k < CAM_TERMS) rows[(size_t)blockIdx.x * CAM_TERMS + k] = s;
			else if (intr) intr[(size_t)blockIdx.x * CAM_INTR_TERMS + k - CAM_TERMS] = s;
		}
	}
}

void launch_rays_fwd(const RaysArgs& a, cudaStream_t s)
{
	if (a.N <= 0 || a.V <= 0) return;
	rays_fwd_kernel<<<dim3(ceil_div(a.N, RAYS_THREADS), a.V), RAYS_THREADS, 0, s>>>(a);
}

void launch_rays_bwd(const RaysArgs& a, cudaStream_t s)
{
	if (a.N <= 0 || a.V <= 0) return;
	bool cam = false;
	for (int v = 0; v < a.V; v++) cam |= a.cam_rows[v] != nullptr;
	const dim3 grid(ceil_div(a.N, RAYS_THREADS), a.V);
	if (cam) rays_bwd_kernel<true><<<grid, RAYS_THREADS, 0, s>>>(a);
	else rays_bwd_kernel<false><<<grid, RAYS_THREADS, 0, s>>>(a);
}

}  // namespace mgs
