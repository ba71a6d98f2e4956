// Per-Gaussian optical flow between a cloud and its paired next-frame means (include/mgs_rasterizer.h, flow plane): the
// screen displacement delta_i = m'_i - m_i of Gaussian i in one view, m its screen mean and m' the same map applied to its
// next-frame mean, in pixels, 0 where the next mean fails the projection's cull.  The forward writes the quad
// {dx, dy, 0, 0} into the view's quad slot, where the normal plane keeps its quads, so the NRM instantiations of the blend
// carry it in columns 4..7 of the {r,g,b,depth} tile unchanged.  The backward takes the blend's quad gradients gn and
// chains them through both ends: -gn into the screen-mean slots of the blend-stage records, which the per-Gaussian chain
// rule then carries to means3D, the camera and the field of view, and (dm'/dmu')^T gn into dL/d(next means), plus the
// camera terms of m' where a view renders m' with its own camera.
//
// Kernels of their own rather than modes of the projection kernels: those compile to pinned instruction sequences (tile ids
// and sort keys depend on them, DESIGN.md section 4).  Both ends come from one device function, so a next mean equal to the
// current one under the view's own camera gives delta = 0 bit for bit.
#include "camera.cuh"

namespace mgs {

__global__ void __launch_bounds__(256) flow_fwd_kernel(FlowFwdArgs a)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= a.P) return;
	float dx = 0.f, dy = 0.f;
	if (a.radii[i] > 0) {
		const V3 p = { a.means3D[3 * (size_t)i], a.means3D[3 * (size_t)i + 1], a.means3D[3 * (size_t)i + 2] };
		const V3 q = { a.next_means3D[3 * (size_t)i], a.next_means3D[3 * (size_t)i + 1], a.next_means3D[3 * (size_t)i + 2] };
		float mx, my, nx, ny;
		screen_mean(a.cur, p, mx, my);  // passes: the projection kept the Gaussian
		if (screen_mean(a.next, q, nx, ny)) { dx = nx - mx; dy = ny - my; }
	}
	a.quad[i] = make_float4(dx, dy, 0.f, 0.f);
}

// CAM: the launch writes camera rows.  One thread per Gaussian over the launch's views in order; per view the camera terms are
// summed over the warp by shuffles in a fixed order, then over the CTA's 4 warps in warp order: deterministic rows.
template <bool CAM>
__global__ void __launch_bounds__(FLOW_BWD_THREADS) flow_bwd_kernel(FlowBwdArgs a)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	const bool in = i < a.P;
	const int id = in ? i : 0;
	__shared__ float cam_sm[CAM ? FLOW_BWD_THREADS / 32 * CAM_ALL_TERMS : 1];
	// a cloud without next means (no view of it has flow) still writes its views' camera rows, as zeros
	const float* nm = a.next_means3D;
	const float p[3] = { nm ? nm[3 * (size_t)id] : 0.f, nm ? nm[3 * (size_t)id + 1] : 0.f, nm ? nm[3 * (size_t)id + 2] : 0.f };
	float gp[3] = { 0.f, 0.f, 0.f };
	for (int v = 0; v < a.V; v++) {
		const FlowBwdView& w = a.view[v];
		float cg[CAM ? CAM_ALL_TERMS : 1];
		if constexpr (CAM) {
#pragma unroll
			for (int k = 0; k < CAM_ALL_TERMS; k++) cg[k] = 0.f;
		}
		if (in && w.gn && w.radii[id] > 0) {
			// an invalid pair's delta is 0 whatever m and m' are: it receives nothing through either end
			const V3 q = { p[0], p[1], p[2] };
			float nx, ny;
			if (screen_mean(w.cam, q, nx, ny)) {
				const float4 g = w.gn[id];
				// m path: -g onto the blend's screen-mean gradient, in its convention (ndc: pixels times W / 2, H / 2)
				float* gb = w.gb + (size_t)id * GB_STRIDE;
				gb[0] -= g.x * (0.5f * w.cam.W);
				gb[1] -= g.y * (0.5f * w.cam.H);
				// m' path
				flow_mean_bwd<CAM>(w.cam, p, g.x, g.y, gp, cg);
				if constexpr (CAM) {
					// a next pose is a constant of the loss: its view's camera takes the m path only
#pragma unroll
					for (int k = 0; k < CAM_ALL_TERMS; k++) cg[k] = w.own_camera ? cg[k] : 0.f;
				}
			}
		}
		if constexpr (CAM) {
			if (w.cam_rows) {
				const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
				for (int k = 0; k < CAM_ALL_TERMS; k++) {
					float s = cg[k];
#pragma unroll
					for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
					if (lane == 0) cam_sm[warp * CAM_ALL_TERMS + k] = s;
				}
				__syncthreads();
				for (int k = threadIdx.x; k < CAM_ALL_TERMS; k += blockDim.x) {
					float s = 0.f;
					for (int u = 0; u < FLOW_BWD_THREADS / 32; u++) s += cam_sm[u * CAM_ALL_TERMS + k];
					if (k < CAM_TERMS) w.cam_rows[(size_t)blockIdx.x * CAM_TERMS + k] = s;
					else if (w.intr_rows) w.intr_rows[(size_t)blockIdx.x * CAM_INTR_TERMS + k - CAM_TERMS] = s;
				}
				__syncthreads();
			}
		}
	}
	if (!in || !a.dL_dnext_means3D) return;
	float* o = a.dL_dnext_means3D + 3 * (size_t)i;
#pragma unroll
	for (int k = 0; k < 3; k++) o[k] = a.accumulate ? o[k] + gp[k] : gp[k];
}

void launch_flow_fwd(const FlowFwdArgs& a, cudaStream_t s)
{
	if (a.P > 0) flow_fwd_kernel<<<ceil_div(a.P, 256), 256, 0, s>>>(a);
}

void launch_flow_bwd(const FlowBwdArgs& a, cudaStream_t s)
{
	if (a.P <= 0 || a.V <= 0) return;
	bool cam = false;
	for (int v = 0; v < a.V; v++) cam |= a.view[v].cam_rows != nullptr;
	const int grid = ceil_div(a.P, FLOW_BWD_THREADS);
	if (cam) flow_bwd_kernel<true><<<grid, FLOW_BWD_THREADS, 0, s>>>(a);
	else flow_bwd_kernel<false><<<grid, FLOW_BWD_THREADS, 0, s>>>(a);
}

}  // namespace mgs
