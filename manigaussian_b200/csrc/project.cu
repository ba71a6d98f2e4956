// Per-Gaussian stages: 3D->2D projection (forward) and the frustum test (the chain-rule backward lives in project_bwd.cu).
//
// Replaces, behind the C-ABI in include/mgs_rasterizer.h:
//   forward  : FORWARD::preprocess / preprocessCUDA    (DGR/cuda_rasterizer/forward.cu:156-257)
//   visible  : checkFrustum (rasterizer_impl.cu:54-66)
// The forward's expressions keep the reference's shapes (left-to-right sums of products, double-precision ndc2pix): tile
// ids and sort keys must agree bit for bit, which requires nvcc to contract the same FMAs.
#include "camera.cuh"

namespace mgs {

// SH constants (values as published with 3DGS; reference auxiliary.h:22-39)
__device__ const float kSH_C0 = 0.28209479177387814f;
__device__ const float kSH_C1 = 0.4886025119029199f;
__device__ const float kSH_C2[] = { 1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
	-1.0925484305920792f, 0.5462742152960396f };
__device__ const float kSH_C3[] = { -0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
	0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f, -0.5900435899266435f };

struct Cov2DTerms {
	V3 t;
	float txtz, tytz;
	M3 T, Vrk, W;
};
// Shared by the forward (forward.cu:75-107) and the backward recomputation (backward.cu:163-196).  The orthographic, fisheye
// and distorted Jacobians are camera.cuh's, at the unclamped t; only the pinhole one clamps t to the frustum.
template <int MODEL = MODEL_PINHOLE>
__device__ __forceinline__ Cov2DTerms cov2d_terms(const V3& mean, float fx, float fy, float tanx, float tany,
	const float* cov3D, const float* vm, const FisheyeRadial* fr = nullptr, const DistTerms* ds = nullptr)
{
	Cov2DTerms o;
	V3 t = xform4x3(mean, vm);
	M3 J;
	float txtz = 0.f, tytz = 0.f;
	if constexpr (MODEL != MODEL_PINHOLE) {
		float j[2][3];
		if constexpr (MODEL == MODEL_ORTHO) {
			ortho_jacobian(fx, fy, j);
		} else if constexpr (MODEL == MODEL_FISHEYE) {
			fisheye_jacobian(*fr, t.x, t.y, fx, fy, j);
		} else {
			const float iz = 1.0f / t.z;
			distorted_jacobian(*ds, t.x * iz, t.y * iz, iz, fx, fy, j);
		}
		J = m3(j[0][0], j[0][1], j[0][2], j[1][0], j[1][1], j[1][2], 0.f, 0.f, 0.f);
	} else {
		const float limx = 1.3f * tanx;
		const float limy = 1.3f * tany;
		txtz = t.x / t.z;
		tytz = t.y / t.z;
		t.x = min(limx, max(-limx, txtz)) * t.z;
		t.y = min(limy, max(-limy, tytz)) * t.z;
		J = m3(
			fx / t.z, 0.0f, -(fx * t.x) / (t.z * t.z),
			0.0f, fy / t.z, -(fy * t.y) / (t.z * t.z),
			0.f, 0.f, 0.f);
	}
	o.W = m3(vm[0], vm[4], vm[8], vm[1], vm[5], vm[9], vm[2], vm[6], vm[10]);
	o.T = mul(o.W, J);
	o.Vrk = m3(cov3D[0], cov3D[1], cov3D[2], cov3D[1], cov3D[3], cov3D[4], cov3D[2], cov3D[4], cov3D[5]);
	o.t = t; o.txtz = txtz; o.tytz = tytz;
	return o;
}

// SH -> RGB with the +0.5 offset and clamp-at-zero mask; forward.cu:21-72
__device__ __forceinline__ void sh_to_rgb(int idx, int deg, int max_coeffs, const float* means, const float* campos,
	const float* shs, uint8_t* clamped_bits, float out[3])
{
	float dx = means[3 * idx] - campos[0], dy = means[3 * idx + 1] - campos[1], dz = means[3 * idx + 2] - campos[2];
	float len = sqrtf(dx * dx + dy * dy + dz * dz);
	float x = dx / len, y = dy / len, z = dz / len;
	const float* sh = shs + (size_t)idx * max_coeffs * 3;
	uint8_t bits = 0;
#pragma unroll
	for (int c = 0; c < 3; c++) {
#define SHK(k) sh[3 * (k) + c]
		float result = kSH_C0 * SHK(0);
		if (deg > 0) {
			result = result - kSH_C1 * y * SHK(1) + kSH_C1 * z * SHK(2) - kSH_C1 * x * SHK(3);
			if (deg > 1) {
				float xx = x * x, yy = y * y, zz = z * z;
				float xy = x * y, yz = y * z, xz = x * z;
				result = result +
					kSH_C2[0] * xy * SHK(4) +
					kSH_C2[1] * yz * SHK(5) +
					kSH_C2[2] * (2.0f * zz - xx - yy) * SHK(6) +
					kSH_C2[3] * xz * SHK(7) +
					kSH_C2[4] * (xx - yy) * SHK(8);
				if (deg > 2) {
					result = result +
						kSH_C3[0] * y * (3.0f * xx - yy) * SHK(9) +
						kSH_C3[1] * xy * z * SHK(10) +
						kSH_C3[2] * y * (4.0f * zz - xx - yy) * SHK(11) +
						kSH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * SHK(12) +
						kSH_C3[4] * x * (4.0f * zz - xx - yy) * SHK(13) +
						kSH_C3[5] * z * (xx - yy) * SHK(14) +
						kSH_C3[6] * x * (xx - 3.0f * yy) * SHK(15);
				}
			}
		}
#undef SHK
		result += 0.5f;
		if (result < 0) bits |= (uint8_t)(1u << c);
		out[c] = max(result, 0.0f);
	}
	clamped_bits[idx] = bits;
}

// AA: the anti-aliased mode (Mip-Splatting's 2D filter, DESIGN.md section 4): the opacity is scaled by
// s = sqrt(max(2.5e-5, det(Sigma) / det(Sigma + 0.3 I))), so that the dilated splat carries the energy of the undilated one.
// Only conic_opacity.w and the extent's opacity change; the conic, radius, tiles and keys are those of AA = false.
// FOV: the field of view is read from the device ({tan_fovx, tan_fovy} at a.tan_fov) and the focal lengths are formed here
// with the host's float expression, so equal values give the host path's results bit for bit.
// MODEL_ORTHO: an orthographic view (include/mgs_rasterizer.h, mgs_render_options.ortho): tan_fov holds the view volume's half
// extents, fx = W / (2 tan_fovx) is in pixels per unit, and J does not depend on t.  The screen mean still goes through the
// caller's projmatrix (w = 1 for an orthographic matrix), and everything after the covariance is the perspective path's.
// MODEL_FISHEYE: a Kannala-Brandt view (mgs_render_options.fisheye): projmatrix is not read; the screen mean is
// (fx a t.x + cx, fy a t.y + cy), J the map's Jacobian (fisheye.cuh), and a mean with theta > theta_max is culled like one
// behind the near plane.  Everything after the covariance is the perspective path's.
// MODEL_DISTORTED: an OpenCV distorted-pinhole view (mgs_render_options.distortion): projmatrix is not read; the screen mean
// is (fx xd + cx, fy yd + cy), J = diag(fx, fy) Dd (d(x, y) / dt) (distortion.cuh), and a mean past the first fold
// (r2 > r2_max) or on a local fold (det Dd <= 0) is culled like one behind the near plane.
template <bool AA, bool FOV, int MODEL>
__global__ void __launch_bounds__(256) project_fwd_kernel(ProjectFwdArgs a)
{
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= a.P) return;

	// defaults for a culled Gaussian (forward.cu:191-192); everything the later stages read is defined
	int out_radius = 0;
	uint32_t out_tiles = 0;
	a.radii[idx] = 0;
	a.tiles_touched[idx] = 0;
	a.iota[idx] = (uint32_t)idx;
	a.depths[idx] = __uint_as_float(0x7f800000u);  // +inf: culled Gaussians sort behind every visible one

	V3 p_orig = { a.means3D[3 * idx], a.means3D[3 * idx + 1], a.means3D[3 * idx + 2] };
	float p_proj_x = 0.f, p_proj_y = 0.f;
	if constexpr (MODEL != MODEL_FISHEYE && MODEL != MODEL_DISTORTED) {
		float4 p_hom = xform4x4(p_orig, a.projmatrix);
		float p_w = 1.0f / (p_hom.w + 0.0000001f);
		p_proj_x = p_hom.x * p_w; p_proj_y = p_hom.y * p_w;
	}
	V3 p_view = xform4x3(p_orig, a.viewmatrix);
	if (p_view.z <= NEAR_Z) return;  // near cull only (auxiliary.h:154)
	FisheyeRadial fr{};
	if constexpr (MODEL == MODEL_FISHEYE) {
		fr = fisheye_radial<false>(p_view.x, p_view.y, p_view.z, a.lens.fe_k);
		if (fisheye_culled(fr, a.lens.theta_max)) return;
	}
	DistTerms ds{};
	if constexpr (MODEL == MODEL_DISTORTED) {
		const float iz = 1.0f / p_view.z;
		ds = distortion_terms<false>(p_view.x * iz, p_view.y * iz, a.lens.dc_k);
		if (distorted_culled(ds, a.lens.r2_max)) return;
	}

	const float* cov3D;
	if (a.cov3D_precomp != nullptr) {
		cov3D = a.cov3D_precomp + (size_t)idx * 6;
	} else {
		cov3d_from_scale_rot(a.scales + 3 * (size_t)idx, a.scale_modifier, a.rotations + 4 * (size_t)idx, a.cov3D + (size_t)idx * 6);
		cov3D = a.cov3D + (size_t)idx * 6;
	}

	float tanx = a.tan_fovx, tany = a.tan_fovy, fx = a.focal_x, fy = a.focal_y;
	if constexpr (FOV) {
		tanx = a.tan_fov[0]; tany = a.tan_fov[1];
		fx = focal_length(a.W, tanx); fy = focal_length(a.H, tany);
	}
	Cov2DTerms ct = cov2d_terms<MODEL>(p_orig, fx, fy, tanx, tany, cov3D, a.viewmatrix, &fr, &ds);
	M3 cov = mul(mul(transpose(ct.T), transpose(ct.Vrk)), ct.T);
	float det0 = 0.f;  // det of the screen-space covariance before the low-pass (AA only)
	if (AA) det0 = fmaf(-cov.m[0][1], cov.m[0][1], cov.m[0][0] * cov.m[1][1]);  // explicit fma: rounding independent of contraction
	cov.m[0][0] += 0.3f;  // low-pass (forward.cu:111-112)
	cov.m[1][1] += 0.3f;
	const float cx = cov.m[0][0], cy = cov.m[0][1], cz = cov.m[1][1];

	float det = (cx * cz - cy * cy);
	if (det == 0.0f) return;
	float det_inv = 1.f / det;
	float conic_x = cz * det_inv, conic_y = -cy * det_inv, conic_z = cx * det_inv;

	float mid = 0.5f * (cx + cz);
	float lambda1 = mid + sqrtf(max(0.1f, mid * mid - det));
	float lambda2 = mid - sqrtf(max(0.1f, mid * mid - det));
	float my_radius = ceilf(3.f * sqrtf(max(lambda1, lambda2)));
	float2 pm;
	if constexpr (MODEL == MODEL_FISHEYE) {
		pm = fisheye_mean(a.lens, fr, p_view.x, p_view.y, fx, fy);
	} else if constexpr (MODEL == MODEL_DISTORTED) {
		pm = distorted_mean(a.lens, ds, fx, fy);
	} else {
		pm = make_float2(ndc2pix(p_proj_x, a.W), ndc2pix(p_proj_y, a.H));
	}
	const float px = pm.x, py = pm.y;
	uint2 rmin, rmax;
	tile_rect(px, py, (int)my_radius, rmin, rmax, a.grid_x, a.grid_y);
	if ((rmax.x - rmin.x) * (rmax.y - rmin.y) == 0) return;

	float c[3];
	if (a.colors_precomp == nullptr) {
		sh_to_rgb(idx, a.D, a.M, a.means3D, a.cam_pos, a.shs, a.clamped, c);
	} else {
		c[0] = a.colors_precomp[3 * idx]; c[1] = a.colors_precomp[3 * idx + 1]; c[2] = a.colors_precomp[3 * idx + 2];
	}
	a.rgbd[idx] = make_float4(c[0], c[1], c[2], p_view.z);  // blend channel quad 0 (depth rides as a channel)

	float opacity = a.opacities[idx];
	if (AA) opacity *= sqrtf(max(2.5e-5f, det0 / det));  // the blend sees o_eff = o s
	out_radius = (int)my_radius;
	out_tiles = (rmax.y - rmin.y) * (rmax.x - rmin.x);
	a.depths[idx] = p_view.z;
	a.radii[idx] = out_radius;
	a.means2D[idx] = make_float2(px, py);
	a.conic_opacity[idx] = make_float4(conic_x, conic_y, conic_z, opacity);
	a.tiles_touched[idx] = out_tiles;

	// Conservative footprint of {alpha >= 1/255}: 0.5 d^T Q d <= tau, tau = ln(255 * opacity).
	// Used only to skip whole 8x4 pixel blocks in the blend kernels; never changes a pixel's result.
	float hx = 1e30f, hy = 1e30f;
	const float o255 = 255.0f * opacity;
	if (!(o255 >= 0.999f)) {
		hx = hy = -1.0f;  // alpha = min(0.99, o*G) <= o < 1/255 everywhere: never contributes
	} else {
		const float tau = logf(o255) * 1.0005f + 1e-3f;
		const float ac = conic_x * conic_z;
		const float dq = ac - conic_y * conic_y;
		if (conic_x > 0.f && conic_z > 0.f && dq > 1e-3f * ac) {
			hx = sqrtf(2.0f * tau * conic_z / dq) * 1.001f + 0.01f;
			hy = sqrtf(2.0f * tau * conic_x / dq) * 1.001f + 0.01f;
		}
	}
	a.extent[idx] = make_float2(hx, hy);
}

__global__ void __launch_bounds__(256) mark_visible_kernel(int P, const float* means3D, const float* viewmatrix, uint8_t* present)
{
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= P) return;
	V3 p = { means3D[3 * idx], means3D[3 * idx + 1], means3D[3 * idx + 2] };
	present[idx] = xform4x3(p, viewmatrix).z > NEAR_Z;
}

template <int MODEL>
static void launch_project_fwd_model(const ProjectFwdArgs& a, int grid, cudaStream_t s)
{
	if (a.tan_fov) {
		if (a.antialias) project_fwd_kernel<true, true, MODEL><<<grid, 256, 0, s>>>(a);
		else project_fwd_kernel<false, true, MODEL><<<grid, 256, 0, s>>>(a);
	} else {
		if (a.antialias) project_fwd_kernel<true, false, MODEL><<<grid, 256, 0, s>>>(a);
		else project_fwd_kernel<false, false, MODEL><<<grid, 256, 0, s>>>(a);
	}
}

void launch_project_fwd(const ProjectFwdArgs& a, cudaStream_t s)
{
	if (a.P <= 0) return;
	const int grid = ceil_div(a.P, 256);
	switch (a.lens.model) {
	case MODEL_DISTORTED: launch_project_fwd_model<MODEL_DISTORTED>(a, grid, s); break;
	case MODEL_FISHEYE: launch_project_fwd_model<MODEL_FISHEYE>(a, grid, s); break;
	case MODEL_ORTHO: launch_project_fwd_model<MODEL_ORTHO>(a, grid, s); break;
	default: launch_project_fwd_model<MODEL_PINHOLE>(a, grid, s);
	}
}
void launch_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present, cudaStream_t s)
{
	if (P > 0) mark_visible_kernel<<<ceil_div(P, 256), 256, 0, s>>>(P, means3D, viewmatrix, present);
}

}  // namespace mgs
