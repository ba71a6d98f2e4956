// Per-Gaussian planar-depth quads (include/mgs_rasterizer.h, planar depth): the depth of Gaussian i along the ray of pixel p
// is z + a (px - mu_x) + b (py - mu_y), the regression of t.z on the dilated screen position, with (a, b) = k Q,
// k = e3^T Sigma_c J^T the covariance of depth with screen position and Q the conic the blend evaluates.  The quad
// {a, b, e = -(a mu_x + b mu_y), 0} fills columns 4..7 of the {r,g,b,depth} tile, so the blend's depth is
// col3 + px col4 + py col5 + col6.  Its backward is part of the per-Gaussian chain rule (project_bwd.cu, PLN).
//
// A kernel of its own rather than a mode of the projection kernels: those compile to pinned instruction sequences (tile ids
// and sort keys depend on them, DESIGN.md section 4).  It reads the projection's record (mean, conic) and rebuilds t, J and
// Sigma_c as the projection forms them.
#include "camera.cuh"

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
	const ViewFov f = view_fov(a);
	const float tanx = f.tanx, tany = f.tany, fx = f.fx, fy = f.fy;
	// J (2x3, pixels), as project.cu's cov2d_terms forms it for the view's model
	float J[2][3];
	if (a.lens.model == MODEL_ORTHO) {
		ortho_jacobian(fx, fy, J);
	} else if (a.lens.model == MODEL_FISHEYE) {
		fisheye_jacobian(fisheye_radial<false>(tx, ty, tz, a.lens.fe_k), tx, ty, fx, fy, J);
	} else if (a.lens.model == MODEL_DISTORTED) {
		const float iz = 1.0f / tz, x = tx * iz, y = ty * iz;
		distorted_jacobian(distortion_terms<false>(x, y, a.lens.dc_k), x, y, iz, fx, fy, J);
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
