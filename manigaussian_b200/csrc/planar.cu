// Per-Gaussian planar-depth quads (include/mgs_rasterizer.h, planar depth): the depth of Gaussian i along the ray of pixel p
// is z + a (px - mu_x) + b (py - mu_y), the regression of t.z on the dilated screen position, with (a, b) = k Q,
// k = e3^T Sigma_c J^T the covariance of depth with screen position and Q the conic the blend evaluates.  The quad
// {a, b, e = -(a mu_x + b mu_y), 0} fills columns 4..7 of the {r,g,b,depth} tile, so the blend's depth is
// col3 + px col4 + py col5 + col6.  Its backward is part of the per-Gaussian chain rule (project_bwd.cu, PLN).
//
// A kernel of its own rather than a mode of the projection kernels: those compile to pinned instruction sequences (tile ids
// and sort keys depend on them, DESIGN.md section 4).  It reads the projection's record (mean, conic) and rebuilds t, J and
// Sigma_c as the projection forms them.
#include "mgs_common.cuh"
#include "mgs_kernels.h"

namespace mgs {

__global__ void __launch_bounds__(256) planar_fwd_kernel(PlanarFwdArgs a)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= a.P) return;
	if (a.radii[i] <= 0) { a.quad[i] = make_float4(0.f, 0.f, 0.f, 0.f); return; }
	const float* vm = a.viewmatrix;  // Rv[r][c] = vm[4 c + r]
	float Rv[3][3];
#pragma unroll
	for (int r = 0; r < 3; r++)
#pragma unroll
		for (int c = 0; c < 3; c++) Rv[r][c] = vm[4 * c + r];
	const float* p = a.means3D + 3 * (size_t)i;
	const float tx = Rv[0][0] * p[0] + Rv[0][1] * p[1] + Rv[0][2] * p[2] + vm[12];
	const float ty = Rv[1][0] * p[0] + Rv[1][1] * p[1] + Rv[1][2] * p[2] + vm[13];
	const float tz = Rv[2][0] * p[0] + Rv[2][1] * p[1] + Rv[2][2] * p[2] + vm[14];
	const float tanx = a.tan_fov ? a.tan_fov[0] : a.tan_fovx, tany = a.tan_fov ? a.tan_fov[1] : a.tan_fovy;
	const float fx = a.W / (2.0f * tanx), fy = a.H / (2.0f * tany);
	// J (2x3, pixels), as project.cu's cov2d_terms forms it for the view's model
	float J[2][3];
	if (a.model == 1) {
		J[0][0] = fx; J[0][1] = 0.f; J[0][2] = 0.f;
		J[1][0] = 0.f; J[1][1] = fy; J[1][2] = 0.f;
	} else if (a.model == 2) {
		const FisheyeRadial fr = fisheye_radial<false>(tx, ty, tz, a.fe_k);
		const float cxy = fr.c * tx * ty;
		J[0][0] = fx * (fr.a + fr.c * tx * tx); J[0][1] = fx * cxy; J[0][2] = -fx * tx * fr.g;
		J[1][0] = fy * cxy; J[1][1] = fy * (fr.a + fr.c * ty * ty); J[1][2] = -fy * ty * fr.g;
	} else if (a.model == 3) {
		const float iz = 1.0f / tz, x = tx * iz, y = ty * iz;
		const DistTerms ds = distortion_terms<false>(x, y, a.dc_k);
		J[0][0] = fx * ds.d00 * iz; J[0][1] = fx * ds.d01 * iz; J[0][2] = -fx * (ds.d00 * x + ds.d01 * y) * iz;
		J[1][0] = fy * ds.d01 * iz; J[1][1] = fy * ds.d11 * iz; J[1][2] = -fy * (ds.d01 * x + ds.d11 * y) * iz;
	} else {
		// the pinhole Jacobian at the frustum-clamped t.xy
		const float limx = 1.3f * tanx, limy = 1.3f * tany;
		const float cx = fminf(limx, fmaxf(-limx, tx / tz)) * tz, cy = fminf(limy, fmaxf(-limy, ty / tz)) * tz;
		const float iz = 1.0f / tz;
		J[0][0] = fx * iz; J[0][1] = 0.f; J[0][2] = -fx * cx * iz * iz;
		J[1][0] = 0.f; J[1][1] = fy * iz; J[1][2] = -fy * cy * iz * iz;
	}
	const float* c6 = a.cov3D + 6 * (size_t)i;
	const float S[3][3] = { { c6[0], c6[1], c6[2] }, { c6[1], c6[3], c6[4] }, { c6[2], c6[4], c6[5] } };
	// k_j = Rv2^T S m_j with m_j = row j of M = J Rv: the covariance of t.z with screen coordinate j
	float sr[3];  // S Rv2
#pragma unroll
	for (int r = 0; r < 3; r++) sr[r] = S[r][0] * Rv[2][0] + S[r][1] * Rv[2][1] + S[r][2] * Rv[2][2];
	float k[2];
#pragma unroll
	for (int j = 0; j < 2; j++) {
		float m[3];
#pragma unroll
		for (int c = 0; c < 3; c++) m[c] = J[j][0] * Rv[0][c] + J[j][1] * Rv[1][c] + J[j][2] * Rv[2][c];
		k[j] = m[0] * sr[0] + m[1] * sr[1] + m[2] * sr[2];
	}
	const float4 q = a.conic_opacity[i];
	const float2 mu = a.means2D[i];
	const float pa = k[0] * q.x + k[1] * q.y, pb = k[0] * q.y + k[1] * q.z;
	a.quad[i] = make_float4(pa, pb, -(pa * mu.x + pb * mu.y), 0.f);
}

void launch_planar_fwd(const PlanarFwdArgs& a, cudaStream_t s)
{
	if (a.P > 0) planar_fwd_kernel<<<ceil_div(a.P, 256), 256, 0, s>>>(a);
}

}  // namespace mgs
