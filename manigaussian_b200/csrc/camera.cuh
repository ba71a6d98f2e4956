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

// ---- the inverse maps (include/mgs_rasterizer.h, mgs_camera_rays): the ray p(z) = o + z d of pixel (u, v), z = t.z ----
// Pinhole and orthographic views solve screen_mean's two projection rows and view-matrix row 2 as the 3x3 system A p = b + z
// e3; fisheye and distorted views invert their lens map at t.z = 1 into (X, Y) and take t = z (X, Y, 1).

constexpr int FISHEYE_RAY_ITERS = 16;  // safeguarded Newton steps on theta rho(theta) = theta_d
constexpr int DIST_RAY_ITERS = 20;     // Newton steps on distort(x, y) = (xd, yd)
// a distorted ray is valid only if |distort(x, y) - (xd, yd)| <= DIST_RAY_TOL (1 + |(xd, yd)|): fp32 evaluates distort at
// |x| <~ 2 to a few ulps (2.4e-7 each at 2), so a converged iterate passes and one stuck on a fold or past it does not
constexpr float DIST_RAY_TOL = 1e-6f;

// A = [P0 - nx P3; P1 - ny P3; V2] (the first three columns), b = (nx (P3.w + 1e-7) - P0.w, ny (P3.w + 1e-7) - P1.w, -V2.w),
// Pk / Vk the rows of projmatrix / viewmatrix, (nx, ny) the ndc of the pixel (ndc2pix's inverse)
struct PinholeRay {
	float A[3][3], b[3], nx, ny;
};
__device__ __forceinline__ PinholeRay pinhole_ray_system(const FlowCam& c, float u, float v)
{
	const float* pm = c.projmatrix;
	const float* vm = c.viewmatrix;
	PinholeRay s;
	s.nx = (2.0f * u + 1.0f) / c.W - 1.0f;
	s.ny = (2.0f * v + 1.0f) / c.H - 1.0f;
#pragma unroll
	for (int k = 0; k < 3; k++) {
		s.A[0][k] = pm[4 * k] - s.nx * pm[4 * k + 3];
		s.A[1][k] = pm[4 * k + 1] - s.ny * pm[4 * k + 3];
		s.A[2][k] = vm[4 * k + 2];
	}
	const float w = pm[15] + 0.0000001f;
	s.b[0] = s.nx * w - pm[12];
	s.b[1] = s.ny * w - pm[13];
	s.b[2] = -vm[14];
	return s;
}
// the columns of A^-1: ci[k] = (a_{k+1} x a_{k+2}) / det; false where A is singular
__device__ __forceinline__ bool inverse3(const float A[3][3], float ci[3][3])
{
#pragma unroll
	for (int k = 0; k < 3; k++) {
		const float* a = A[(k + 1) % 3];
		const float* b = A[(k + 2) % 3];
		ci[k][0] = a[1] * b[2] - a[2] * b[1];
		ci[k][1] = a[2] * b[0] - a[0] * b[2];
		ci[k][2] = a[0] * b[1] - a[1] * b[0];
	}
	const float det = A[0][0] * ci[0][0] + A[0][1] * ci[0][1] + A[0][2] * ci[0][2];
	if (!(det != 0.f) || !isfinite(det)) return false;
	const float id = 1.0f / det;
#pragma unroll
	for (int k = 0; k < 3; k++) { ci[k][0] *= id; ci[k][1] *= id; ci[k][2] *= id; }
	return true;
}

// theta_d = theta rho(theta) and D1 = d theta_d / d theta
__device__ __forceinline__ void fisheye_theta_d(const FisheyeK& k, float th, float& td, float& d1)
{
	const float t2 = th * th;
	td = th * (1.0f + t2 * (k.k1 + t2 * (k.k2 + t2 * (k.k3 + t2 * k.k4))));
	d1 = 1.0f + t2 * (3.0f * k.k1 + t2 * (5.0f * k.k2 + t2 * (7.0f * k.k3 + t2 * (9.0f * k.k4))));
}
// fisheye: (X, Y) = s (xd, yd), s = tan(theta) / theta_d, theta in [0, theta_max] the root of theta rho(theta) = theta_d =
// |(xd, yd)| (monotone there: cameras.fisheye_theta_max), by Newton steps kept inside the sign bracket (bisection where a
// step leaves it).  s = (tan(theta) / theta) / rho(theta), with tan(theta) / theta from its series below theta^2 = 1/64, so
// the axis pixel is (0, 0) with finite derivatives.  Valid iff theta_d <= theta_max rho(theta_max) and s is finite, >= 0.
__device__ __forceinline__ bool fisheye_unmap(const Lens& l, float xd, float yd, float& X, float& Y)
{
	const FisheyeK& k = l.fe_k;
	const float tdd = sqrtf(xd * xd + yd * yd);
	float tdm, d1;
	fisheye_theta_d(k, l.theta_max, tdm, d1);
	X = Y = 0.f;
	if (!(tdd <= tdm)) return false;
	float lo = 0.f, hi = l.theta_max, th = fminf(tdd, l.theta_max);
	for (int i = 0; i < FISHEYE_RAY_ITERS; i++) {
		float f, df;
		fisheye_theta_d(k, th, f, df);
		f -= tdd;
		if (f == 0.f) break;
		if (f > 0.f) hi = th; else lo = th;
		float nt = th - f / df;
		if (!(nt > lo && nt < hi)) nt = 0.5f * (lo + hi);
		if (nt == th) break;
		th = nt;
	}
	const float t2 = th * th;
	const float rho = 1.0f + t2 * (k.k1 + t2 * (k.k2 + t2 * (k.k3 + t2 * k.k4)));
	const float tq = t2 < FISHEYE_SERIES_E2 ? 1.0f + t2 * (1.0f / 3.0f + t2 * (2.0f / 15.0f + t2 * (17.0f / 315.0f))) : tanf(th) / th;
	const float s = tq / rho;
	X = s * xd; Y = s * yd;
	return isfinite(s) && s >= 0.f;
}
// distorted: Newton on distort(x, y) = (xd, yd) from (xd, yd) with Dd, at most DIST_RAY_ITERS steps; ds the terms at the
// returned (x, y).  Valid iff the iterate passes the projection's cull (distorted_culled) and its residual DIST_RAY_TOL.
__device__ __forceinline__ bool distorted_unmap(const Lens& l, float xd, float yd, float& x, float& y, DistTerms& ds)
{
	const float tol = DIST_RAY_TOL * (1.0f + sqrtf(xd * xd + yd * yd));
	x = xd; y = yd;
	float e2;
	for (int i = 0;; i++) {
		ds = distortion_terms<false>(x, y, l.dc_k);
		const float ex = xd - ds.xd, ey = yd - ds.yd;
		e2 = ex * ex + ey * ey;
		const float det = fmaf(-ds.d01, ds.d01, ds.d00 * ds.d11);
		if (i == DIST_RAY_ITERS || !(det > 0.f) || e2 <= 0.0625f * tol * tol) break;
		const float id = 1.0f / det;
		x += (ds.d11 * ex - ds.d01 * ey) * id;
		y += (ds.d00 * ey - ds.d01 * ex) * id;
	}
	return !distorted_culled(ds, l.r2_max) && e2 <= tol * tol;
}

// Rv[r][k] = vm[4k + r].  The lens rays invert it rather than transpose it: the same for a rigid pose, and exact for a learnable
// pose an optimizer has moved off the rotations, so that the ray still projects back to its pixel at its depth.
__device__ __forceinline__ void view_rotation(const float* vm, float R[3][3])
{
#pragma unroll
	for (int r = 0; r < 3; r++)
#pragma unroll
		for (int k = 0; k < 3; k++) R[r][k] = vm[4 * k + r];
}

// the ray of pixel (u, v) in view c: origin o and direction d in world space (d's view-space z component 1), and whether
// it is valid (the pixel is the image of points the projection keeps)
__device__ __forceinline__ bool camera_ray(const FlowCam& c, float u, float v, float o[3], float d[3])
{
	const float* vm = c.viewmatrix;
	if (c.lens.model == MODEL_PINHOLE || c.lens.model == MODEL_ORTHO) {
		const PinholeRay s = pinhole_ray_system(c, u, v);
		float ci[3][3];
		const bool ok = inverse3(s.A, ci);
#pragma unroll
		for (int k = 0; k < 3; k++) {
			o[k] = ci[0][k] * s.b[0] + ci[1][k] * s.b[1] + ci[2][k] * s.b[2];
			d[k] = ci[2][k];
		}
		return ok;
	}
	const ViewFov f = view_fov(c);
	const float xd = (u - c.lens.cx) / f.fx, yd = (v - c.lens.cy) / f.fy;
	float X, Y;
	bool ok;
	if (c.lens.model == MODEL_FISHEYE) {
		ok = fisheye_unmap(c.lens, xd, yd, X, Y);
	} else {
		DistTerms ds;
		ok = distorted_unmap(c.lens, xd, yd, X, Y, ds);
	}
	// p = Rv^-1 (t - tv): o = -Rv^-1 tv, d = Rv^-1 (X, Y, 1)
	float R[3][3], ci[3][3];
	view_rotation(vm, R);
	ok = inverse3(R, ci) && ok;
#pragma unroll
	for (int k = 0; k < 3; k++) {
		o[k] = -(ci[0][k] * vm[12] + ci[1][k] * vm[13] + ci[2][k] * vm[14]);
		d[k] = ci[0][k] * X + ci[1][k] * Y + ci[2][k];
	}
	return ok;
}

// the derivative of camera_ray by implicit differentiation: go, gd the cotangents of o and d, into (gu, gv) and, with CAM,
// the camera terms of the view (CAM_ALL_TERMS, the rows of flow_mean_bwd: dL/dvm, dL/dpm, dL/dcampos = 0, dL/dtan_fov;
// every term written).  Returns camera_ray's validity; an invalid ray has (gu, gv) = 0 and no camera terms.
template <bool CAM>
__device__ __forceinline__ bool camera_ray_bwd(const FlowCam& c, float u, float v, const float go[3], const float gd[3], float& gu,
	float& gv, float* cg)
{
	const float* vm = c.viewmatrix;
	gu = gv = 0.f;
	if constexpr (CAM) {
#pragma unroll
		for (int k = 0; k < CAM_ALL_TERMS; k++) cg[k] = 0.f;
	}
	if (c.lens.model == MODEL_PINHOLE || c.lens.model == MODEL_ORTHO) {
		// o = A^-1 b, d = A^-1 e3: with lo = A^-T go, ld = A^-T gd, dL/dA = -(lo o^T + ld d^T) and dL/db = lo
		const PinholeRay s = pinhole_ray_system(c, u, v);
		float ci[3][3];
		if (!inverse3(s.A, ci)) return false;
		float o[3], d[3], lo[3], ld[3];
#pragma unroll
		for (int k = 0; k < 3; k++) {
			o[k] = ci[0][k] * s.b[0] + ci[1][k] * s.b[1] + ci[2][k] * s.b[2];
			d[k] = ci[2][k];
			lo[k] = ci[k][0] * go[0] + ci[k][1] * go[1] + ci[k][2] * go[2];
			ld[k] = ci[k][0] * gd[0] + ci[k][1] * gd[1] + ci[k][2] * gd[2];
		}
		float GA[3][3];
#pragma unroll
		for (int r = 0; r < 3; r++)
#pragma unroll
			for (int k = 0; k < 3; k++) GA[r][k] = -(lo[r] * o[k] + ld[r] * d[k]);
		const float* pm = c.projmatrix;
		const float w = pm[15] + 0.0000001f;
		// A[0][k] = pm[4k] - nx pm[4k + 3], b[0] = nx w - pm[12]; likewise row 1 with ny; ndc = (2 pixel + 1) / S - 1
		float gnx = lo[0] * w, gny = lo[1] * w;
#pragma unroll
		for (int k = 0; k < 3; k++) { gnx -= GA[0][k] * pm[4 * k + 3]; gny -= GA[1][k] * pm[4 * k + 3]; }
		gu = gnx * (2.0f / c.W);
		gv = gny * (2.0f / c.H);
		if constexpr (CAM) {
#pragma unroll
			for (int k = 0; k < 3; k++) {
				cg[3 * k + 2] = GA[2][k];                                   // vm[4k + 2]
				cg[12 + 3 * k] = GA[0][k];                                  // pm[4k]
				cg[13 + 3 * k] = GA[1][k];                                  // pm[4k + 1]
				cg[14 + 3 * k] = -(s.nx * GA[0][k] + s.ny * GA[1][k]);      // pm[4k + 3]
			}
			cg[11] = -lo[2];                                                // vm[14]
			cg[21] = -lo[0]; cg[22] = -lo[1]; cg[23] = s.nx * lo[0] + s.ny * lo[1];  // pm[12], pm[13], pm[15]
		}
		return true;
	}
	const ViewFov f = view_fov(c);
	const float xd = (u - c.lens.cx) / f.fx, yd = (v - c.lens.cy) / f.fy;
	float X, Y, m00, m01, m11;  // M = d(xd, yd) / d(X, Y), symmetric
	if (c.lens.model == MODEL_FISHEYE) {
		if (!fisheye_unmap(c.lens, xd, yd, X, Y)) return false;
		// at t = (X, Y, 1): (xd, yd) = a (X, Y), M = J / f of fisheye_jacobian (series near the axis)
		const FisheyeRadial fr = fisheye_radial<false>(X, Y, 1.0f, c.lens.fe_k);
		m00 = fr.a + fr.c * X * X; m01 = fr.c * X * Y; m11 = fr.a + fr.c * Y * Y;
	} else {
		DistTerms ds;
		if (!distorted_unmap(c.lens, xd, yd, X, Y, ds)) return false;
		m00 = ds.d00; m01 = ds.d01; m11 = ds.d11;
	}
	// o = Rv^-1 b, d = Rv^-1 w with b = -tv, w = (X, Y, 1): lo = Rv^-T go, ld = Rv^-T gd, dL/dRv = -(lo o^T + ld d^T),
	// dL/dtv = -lo, dL/d(X, Y) = ld.xy; (X, Y) solves (xd, yd)(X, Y) = ((u - cx) / fx, (v - cy) / fy)
	float R[3][3], ci[3][3];
	view_rotation(vm, R);
	if (!inverse3(R, ci)) return false;
	float o[3], d[3], lo[3], ld[3];
#pragma unroll
	for (int k = 0; k < 3; k++) {
		o[k] = -(ci[0][k] * vm[12] + ci[1][k] * vm[13] + ci[2][k] * vm[14]);
		d[k] = ci[0][k] * X + ci[1][k] * Y + ci[2][k];
		lo[k] = ci[k][0] * go[0] + ci[k][1] * go[1] + ci[k][2] * go[2];
		ld[k] = ci[k][0] * gd[0] + ci[k][1] * gd[1] + ci[k][2] * gd[2];
	}
	const float gX = ld[0], gY = ld[1];
	const float id = 1.0f / fmaf(-m01, m01, m00 * m11);
	const float lx = (m11 * gX - m01 * gY) * id, ly = (m00 * gY - m01 * gX) * id;  // M^-1 (gX, gY) = dL/d(xd, yd)
	gu = lx / f.fx;
	gv = ly / f.fy;
	if constexpr (CAM) {
		// dL/dRv[r][k] at 3k + r, dL/dtv[r] at 9 + r; xd = (u - cx) 2 tan_fovx / W
#pragma unroll
		for (int k = 0; k < 3; k++)
#pragma unroll
			for (int r = 0; r < 3; r++) cg[3 * k + r] = -(lo[r] * o[k] + ld[r] * d[k]);
#pragma unroll
		for (int r = 0; r < 3; r++) cg[9 + r] = -lo[r];
		cg[27] = lx * xd / f.tanx;
		cg[28] = ly * yd / f.tany;
	}
	return true;
}

}  // namespace mgs
