// The device maths of a view's camera model (Lens, mgs_kernels.h) that more than one kernel forms: the focal lengths of a
// field of view, the fisheye and distorted screen mean with its cull, and the orthographic, fisheye and distorted Jacobians
// J = d(pixel) / dt (2x3), and the derivative of the screen mean (flow_mean_bwd).  Every kernel that projects (project.cu,
// planar.cu, project_bwd.cu, flow.cu, visibility.cu) takes them from here, so that all of them agree with the renderer bit for
// bit.  The pinhole Jacobian stays with each kernel: the forward's expressions are pinned to the reference's (tile ids and
// sort keys, DESIGN.md section 4), the others round differently.
#pragma once
#include "mgs_common.cuh"
#include "mgs_kernels.h"

namespace mgs {

// the focal length of an image side of n pixels with half-angle tangent tan_half, as the host forms focal_x / focal_y
__device__ __forceinline__ float focal_length(int n, float tan_half) { return n / (2.0f * tan_half); }

// the field of view of a view c (FlowCam, PlanarFwdArgs: members tan_fov, tan_fovx, tan_fovy, W, H), {tan_fovx, tan_fovy} at
// c.tan_fov (device) or the host values where it is NULL, and its focal lengths in pixels
struct ViewFov {
	float tanx, tany, fx, fy;
};
template <class Cam>
__device__ __forceinline__ ViewFov view_fov(const Cam& c)
{
	const float tanx = c.tan_fov ? c.tan_fov[0] : c.tan_fovx, tany = c.tan_fov ? c.tan_fov[1] : c.tan_fovy;
	return ViewFov{ tanx, tany, focal_length(c.W, tanx), focal_length(c.H, tany) };
}

// the culls of a mean: a fisheye view's past theta_max (the Lens's), a distorted view's past the first fold (r2 > r2_max) or
// on a local fold (det Dd <= 0); fr, ds the terms at the mean's unclamped t (fisheye.cuh, distortion.cuh)
__device__ __forceinline__ bool fisheye_culled(const FisheyeRadial& fr, float theta_max) { return fr.theta > theta_max; }
__device__ __forceinline__ bool distorted_culled(const DistTerms& ds, float r2_max)
{
	return ds.r2 > r2_max || fmaf(-ds.d01, ds.d01, ds.d00 * ds.d11) <= 0.f;
}

// the screen means in pixels: (fx a t.x + cx, fy a t.y + cy) and (fx xd + cx, fy yd + cy)
__device__ __forceinline__ float2 fisheye_mean(const Lens& l, const FisheyeRadial& fr, float tx, float ty, float fx, float fy)
{
	return make_float2(fx * fr.a * tx + l.cx, fy * fr.a * ty + l.cy);
}
__device__ __forceinline__ float2 distorted_mean(const Lens& l, const DistTerms& ds, float fx, float fy)
{
	return make_float2(fx * ds.xd + l.cx, fy * ds.yd + l.cy);
}

// J of an orthographic view: [[fx, 0, 0], [0, fy, 0]], fx, fy in pixels per view-space unit; no dependence on t
__device__ __forceinline__ void ortho_jacobian(float fx, float fy, float J[2][3])
{
	J[0][0] = fx; J[0][1] = 0.f; J[0][2] = 0.f;
	J[1][0] = 0.f; J[1][1] = fy; J[1][2] = 0.f;
}
// J of a fisheye view from the radial terms fr of the unclamped t (fisheye.cuh)
__device__ __forceinline__ void fisheye_jacobian(const FisheyeRadial& fr, float tx, float ty, float fx, float fy, float J[2][3])
{
	const float cxy = fr.c * tx * ty;
	J[0][0] = fx * (fr.a + fr.c * tx * tx); J[0][1] = fx * cxy; J[0][2] = -fx * tx * fr.g;
	J[1][0] = fy * cxy; J[1][1] = fy * (fr.a + fr.c * ty * ty); J[1][2] = -fy * ty * fr.g;
}
// J = diag(fx, fy) Dd [[1/z, 0, -x/z], [0, 1/z, -y/z]] of a distorted view, from the distortion terms ds at the unclamped
// (x, y) = t.xy / t.z, iz = 1 / t.z (distortion.cuh)
__device__ __forceinline__ void distorted_jacobian(const DistTerms& ds, float x, float y, float iz, float fx, float fy, float J[2][3])
{
	J[0][0] = fx * ds.d00 * iz; J[0][1] = fx * ds.d01 * iz; J[0][2] = -fx * (ds.d00 * x + ds.d01 * y) * iz;
	J[1][0] = fy * ds.d01 * iz; J[1][1] = fy * ds.d11 * iz; J[1][2] = -fy * (ds.d01 * x + ds.d11 * y) * iz;
}

// the view's screen mean (px, py) of p in pixels (the projection's expressions for the lens), and whether p passes the
// projection's cull of a mean.  The view-space depth t.z is xform4x3(p, c.viewmatrix).z, as here.
__device__ __forceinline__ bool screen_mean(const FlowCam& c, const V3& p, float& px, float& py)
{
	const V3 t = xform4x3(p, c.viewmatrix);
	if (c.lens.model == MODEL_PINHOLE || c.lens.model == MODEL_ORTHO) {
		const float4 h = xform4x4(p, c.projmatrix);
		const float w = 1.0f / (h.w + 0.0000001f);
		px = ndc2pix(h.x * w, c.W); py = ndc2pix(h.y * w, c.H);
		return t.z > NEAR_Z;
	}
	px = py = 0.f;
	if (t.z <= NEAR_Z) return false;
	const ViewFov f = view_fov(c);
	const float fx = f.fx, fy = f.fy;
	if (c.lens.model == MODEL_FISHEYE) {
		const FisheyeRadial fr = fisheye_radial<false>(t.x, t.y, t.z, c.lens.fe_k);
		if (fisheye_culled(fr, c.lens.theta_max)) return false;
		const float2 m = fisheye_mean(c.lens, fr, t.x, t.y, fx, fy);
		px = m.x; py = m.y;
		return true;
	}
	const float iz = 1.0f / t.z;
	const DistTerms ds = distortion_terms<false>(t.x * iz, t.y * iz, c.lens.dc_k);
	if (distorted_culled(ds, c.lens.r2_max)) return false;
	const float2 m = distorted_mean(c.lens, ds, fx, fy);
	px = m.x; py = m.y;
	return true;
}

// the derivative of screen_mean (the flow plane's m' chain, a query point's uv chain): g the pixel cotangent of the screen
// mean at p (valid), into dL/dp (added to gp) and, with cg, the camera terms of the view (CAM_ALL_TERMS, laid out as the
// per-Gaussian backward's rows: dL/dvm, dL/dpm, dL/dcampos, dL/dtan_fov; the terms of the model are written, the others left)
template <bool CAM>
__device__ __forceinline__ void flow_mean_bwd(const FlowCam& c, const float p[3], float gx, float gy, float gp[3], float* cg)
{
	const float* vm = c.viewmatrix;
	if (c.lens.model == MODEL_PINHOLE || c.lens.model == MODEL_ORTHO) {
		// ndc = (P p).xy / ((P p).w + 1e-7), pixel = ((ndc + 1) S - 1) / 2: the ndc cotangent is the pixel one times S / 2
		const float* pm = c.projmatrix;
		const float dx = gx * (0.5f * c.W), dy = gy * (0.5f * c.H);
		const float hx = pm[0] * p[0] + pm[4] * p[1] + pm[8] * p[2] + pm[12];
		const float hy = pm[1] * p[0] + pm[5] * p[1] + pm[9] * p[2] + pm[13];
		const float hw = pm[3] * p[0] + pm[7] * p[1] + pm[11] * p[2] + pm[15];
		const float iw = 1.0f / (hw + 0.0000001f);
		const float kx = hx * iw * iw, ky = hy * iw * iw;
#pragma unroll
		for (int k = 0; k < 3; k++) gp[k] += (pm[4 * k] * iw - pm[4 * k + 3] * kx) * dx + (pm[4 * k + 1] * iw - pm[4 * k + 3] * ky) * dy;
		if constexpr (CAM) {
			const float ax = dx * iw, ay = dy * iw, aw = -(dx * kx + dy * ky);
			const float ph[4] = { p[0], p[1], p[2], 1.f };
#pragma unroll
			for (int k = 0; k < 4; k++) { cg[12 + 3 * k] = ax * ph[k]; cg[13 + 3 * k] = ay * ph[k]; cg[14 + 3 * k] = aw * ph[k]; }
		}
		return;
	}
	const float tx = vm[0] * p[0] + vm[4] * p[1] + vm[8] * p[2] + vm[12];
	const float ty = vm[1] * p[0] + vm[5] * p[1] + vm[9] * p[2] + vm[13];
	const float tz = vm[2] * p[0] + vm[6] * p[1] + vm[10] * p[2] + vm[14];
	const ViewFov f = view_fov(c);
	const float tanx = f.tanx, tany = f.tany, fx = f.fx, fy = f.fy;
	float dt[3], ftx, fty;  // dL/dt; (u - cx, v - cy) for the field of view
	if (c.lens.model == MODEL_FISHEYE) {
		// J = [[fx (a + c x^2), fx c x y, -fx x g], [fy c x y, fy (a + c y^2), -fy y g]] (fisheye.cuh)
		const FisheyeRadial fr = fisheye_radial<false>(tx, ty, tz, c.lens.fe_k);
		const float ex = fx * gx, ey = fy * gy, cxy = fr.c * tx * ty;
		dt[0] = ex * (fr.a + fr.c * tx * tx) + ey * cxy;
		dt[1] = ex * cxy + ey * (fr.a + fr.c * ty * ty);
		dt[2] = -(ex * tx + ey * ty) * fr.g;
		ftx = fx * fr.a * tx; fty = fy * fr.a * ty;
	} else {
		// (u, v) = F (xd, yd) + c, d(xd, yd) / d(x, y) = Dd (symmetric), (x, y) = t.xy / t.z
		const float iz = 1.0f / tz, x = tx * iz, y = ty * iz;
		const DistTerms ds = distortion_terms<false>(x, y, c.lens.dc_k);
		const float ex = fx * gx, ey = fy * gy;
		const float qx = ds.d00 * ex + ds.d01 * ey, qy = ds.d01 * ex + ds.d11 * ey;
		dt[0] = qx * iz; dt[1] = qy * iz; dt[2] = -(qx * x + qy * y) * iz;
		ftx = fx * ds.xd; fty = fy * ds.yd;
	}
#pragma unroll
	for (int k = 0; k < 3; k++) gp[k] += vm[4 * k] * dt[0] + vm[4 * k + 1] * dt[1] + vm[4 * k + 2] * dt[2];
	if constexpr (CAM) {
		// t = Rv p + tv: dL/dRv[r][k] = dt[r] p[k] at 3k + r, dL/dtv = dt at 9 + r; fx = W / (2 tan_fovx) scales u - cx
#pragma unroll
		for (int k = 0; k < 3; k++) { cg[3 * k] = dt[0] * p[k]; cg[3 * k + 1] = dt[1] * p[k]; cg[3 * k + 2] = dt[2] * p[k]; }
		cg[9] = dt[0]; cg[10] = dt[1]; cg[11] = dt[2];
		cg[27] = -gx * ftx / tanx; cg[28] = -gy * fty / tany;
	}
}

}  // namespace mgs
