// Backward of the per-Gaussian projection for ALL views of a step in one launch.
//
// Replaces BACKWARD::preprocess = computeCov2DCUDA + preprocessCUDA (DGR/cuda_rasterizer/backward.cu:144-274, :346-396,
// with the SH and covariance helpers :20-139, :278-341) and the ten zero-fills of rasterize_points.cu:167-184.
// Same mathematics and the same conventions where the reference departs from the textbook derivative (SURVEY.md
// 8(c) traps: the x/y frustum clamp masks d/dt.x, d/dt.y but is a constant in d/dt.z; the quaternion is used
// un-normalised; dL/dscale carries no factor for scale_modifier; dL/dconic.y arrives halved), but written from the
// matrix calculus of the forward, not from the reference's expressions:
//
//   t = Rv p + tv,  M = J(t) Rv  (2x3),  S' = M S M^T + 0.3 I = [[a,b],[b,c]],  Q = S'^-1  (the conic the blend saw)
//   dL/dS' = H = -w adj(S') G adj(S'),   G = blend-stage dL/dQ,  w = 1 / (det^2 + 1e-7)
//   dL/dS  = M^T H M                     (summed over the views BEFORE the chain to scale / rotation: S is per Gaussian)
//   dL/dM  = 2 H M S,   dL/dJ = dL/dM Rv^T,   dL/dt from the four non-constant entries of J,   dL/dp = Rv^T dL/dt
//   S = L L^T, L = R(q) diag(s):   dL/dL = 2 (dL/dS) L,   dL/ds_j = <R_j, (dL/dL)_j>,   dL/dR = (dL/dL) diag(s)
//
// One thread owns one Gaussian and loops over the V views: per view it reads that view's 48-byte blend-stage record,
// radius and clamp bits; the Gaussian's own inputs are read once, every output row is written once, and the sum over
// views happens in registers -- no atomics, no zero-fill pass, no per-view gradient tensors.  The multi-view callers
// (rasterize_views_backward_raw, render_views) write straight into the packed buffer that is the all-reduce message.
// project_bwd_clouds_kernel runs the same body for several clouds in one launch (mgs_backward_clouds, DESIGN.md section 4).
#include "mgs_common.cuh"
#include "mgs_kernels.h"

namespace mgs {

namespace {

struct Sh16 {
	float c0, c1, c2[5], c3[7];
};
// real SH constants as published with 3DGS (reference auxiliary.h:22-39)
__device__ const Sh16 kSh = { 0.28209479177387814f, 0.4886025119029199f,
	{ 1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f, -1.0925484305920792f, 0.5462742152960396f },
	{ -0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f, 0.3731763325901154f, -0.4570457994644658f,
	  1.445305721320277f, -0.5900435899266435f } };

__device__ __forceinline__ float dot3(const float* u, const float* v) { return u[0] * v[0] + u[1] * v[1] + u[2] * v[2]; }

}  // namespace

// NSH = floats of SH gradient kept in registers (3 (deg + 1)^2 for the largest degree the instantiation serves): the
// kernel is latency bound (dependent loads per view, ~1000 instructions per Gaussian), so registers = occupancy = speed;
// degree <= 1 (ManiGaussian's setting) runs at 5 blocks per SM instead of 3.
#ifndef MGS_PBWD_MINB
#define MGS_PBWD_MINB 5
#endif
// The chain rule of Gaussian idx over the views a.view[0 .. a.V).  Args: ProjectBwdViewsArgs, or CloudBwd (one cloud of a
// multi-cloud launch) -- the same member names.
//
// AA (anti-aliased mode): the blend saw o_eff = o s, s = sqrt(max(2.5e-5, r)), r = d0 / d1, d0 = det(S' - 0.3 I), d1 = det S'.
// The record's opacity gradient g is dL/do_eff, so dL/do = sum_v s_v g_v, and where r > 2.5e-5 the view's dL/dS' gains
// g o ds = g o_eff (grad d0 / d0 - grad d1 / d1) / 2 (s^2 = r there): no raw opacity and no square root beyond s itself.
// o_eff is read back from the view's conic_opacity.w; s is recomputed from S'.
template <int NSH, bool AA, class Args>
__device__ __forceinline__ void project_bwd_gaussian(const Args& a, const int idx)
{
	const float p[3] = { a.means3D[3 * idx], a.means3D[3 * idx + 1], a.means3D[3 * idx + 2] };

	// ---- the Gaussian's own covariance: S = L L^T, L = R(q) diag(mod * s), or the caller's ----
	// (only S, q and s live across the view loop; R(q) is rebuilt for the chain to scale / rotation at the end)
	float se[3] = { 0.f, 0.f, 0.f }, q4[4] = { 0.f, 0.f, 0.f, 0.f };
	float S[3][3];
	const bool from_sr = a.scales != nullptr;
	auto rotation = [&](float R[3][3]) {
		const float r = q4[0], x = q4[1], y = q4[2], z = q4[3];
		R[0][0] = 1.f - 2.f * (y * y + z * z); R[0][1] = 2.f * (x * y - r * z); R[0][2] = 2.f * (x * z + r * y);
		R[1][0] = 2.f * (x * y + r * z); R[1][1] = 1.f - 2.f * (x * x + z * z); R[1][2] = 2.f * (y * z - r * x);
		R[2][0] = 2.f * (x * z - r * y); R[2][1] = 2.f * (y * z + r * x); R[2][2] = 1.f - 2.f * (x * x + y * y);
	};
	if (from_sr) {
		const float4 qv = *reinterpret_cast<const float4*>(a.rotations + 4 * (size_t)idx);
		q4[0] = qv.x; q4[1] = qv.y; q4[2] = qv.z; q4[3] = qv.w;
		float R[3][3];
		rotation(R);
#pragma unroll
		for (int j = 0; j < 3; j++) se[j] = a.scale_modifier * a.scales[3 * (size_t)idx + j];
#pragma unroll
		for (int i = 0; i < 3; i++)
#pragma unroll
			for (int j = i; j < 3; j++)
				S[i][j] = S[j][i] = R[i][0] * se[0] * se[0] * R[j][0] + R[i][1] * se[1] * se[1] * R[j][1] + R[i][2] * se[2] * se[2] * R[j][2];
	} else {
		const float* c = a.cov3D_precomp + 6 * (size_t)idx;
		S[0][0] = c[0]; S[0][1] = S[1][0] = c[1]; S[0][2] = S[2][0] = c[2];
		S[1][1] = c[3]; S[1][2] = S[2][1] = c[4]; S[2][2] = c[5];
	}

	// ---- sums over the views ----
	float gp[3] = { 0.f, 0.f, 0.f };                       // dL/dp
	float D[6] = { 0.f, 0.f, 0.f, 0.f, 0.f, 0.f };         // dL/dS, entries 00 01 02 11 12 22 of the symmetric matrix
	float gop = 0.f, gcol[3] = { 0.f, 0.f, 0.f }, gm2[2] = { 0.f, 0.f };
	float gsh[NSH];
#pragma unroll
	for (int i = 0; i < NSH; i++) gsh[i] = 0.f;
	const float* sh = a.shs ? a.shs + (size_t)idx * a.M * 3 : nullptr;
	const int deg = min(a.D, NSH >= 48 ? 3 : NSH >= 27 ? 2 : 1);

	for (int v = 0; v < a.V; v++) {
		const ProjectBwdView& w = a.view[v];
		// the view's record is loaded before the radius is known (the scratch row of an invisible Gaussian is zero-filled
		// memory, never unmapped): the four loads of a view overlap instead of queueing behind the radius
		const float4* gb = reinterpret_cast<const float4*>(w.gb + (size_t)idx * GB_STRIDE);
		const float4 g0 = gb[0], g1 = gb[1], g2 = gb[2];
		const uint8_t cl = sh ? w.clamped[idx] : (uint8_t)0;
		const float o_eff = AA ? a.conic_opacity[v][idx].w : 0.f;
		const bool live = w.radii[idx] > 0;
		float dm[2] = { 0.f, 0.f };
		if (live) {
			dm[0] = g0.x; dm[1] = g0.y;
			const float gA = g0.z, gB = g0.w, gC = g1.x;        // dL/dconic (xx, xy halved, yy)
			const float dcol[3] = { g1.z, g1.w, g2.x };
			const float ddepth = g2.y;
			if (!AA) gop += g1.y;
			gcol[0] += dcol[0]; gcol[1] += dcol[1]; gcol[2] += dcol[2];
			if (a.dL_dconic && v == 0) {
				float* o = a.dL_dconic + 4 * (size_t)idx;
				o[0] = gA; o[1] = gB; o[2] = 0.f; o[3] = gC;
			}
			const float* vm = w.viewmatrix;  // Rv[r][c] = vm[4 c + r]
			float Rv[3][3];
#pragma unroll
			for (int r = 0; r < 3; r++)
#pragma unroll
				for (int c = 0; c < 3; c++) Rv[r][c] = vm[4 * c + r];
			const float tx = dot3(Rv[0], p) + vm[12], ty = dot3(Rv[1], p) + vm[13], tz = dot3(Rv[2], p) + vm[14];
			const float limx = 1.3f * w.tan_fovx, limy = 1.3f * w.tan_fovy;
			const float ux = tx / tz, uy = ty / tz;
			const bool inx = !(ux < -limx || ux > limx), iny = !(uy < -limy || uy > limy);
			const float cx = fminf(limx, fmaxf(-limx, ux)) * tz, cy = fminf(limy, fmaxf(-limy, uy)) * tz;
			const float iz = 1.0f / tz, iz2 = iz * iz;
			const float fx = w.focal_x, fy = w.focal_y;
			// M = J Rv: row 0 = (fx / tz) Rv0 - (fx cx / tz^2) Rv2, row 1 likewise with y
			float m0[3], m1[3], u0[3], u1[3];
#pragma unroll
			for (int c = 0; c < 3; c++) {
				m0[c] = fx * iz * Rv[0][c] - fx * cx * iz2 * Rv[2][c];
				m1[c] = fy * iz * Rv[1][c] - fy * cy * iz2 * Rv[2][c];
			}
#pragma unroll
			for (int c = 0; c < 3; c++) { u0[c] = dot3(S[c], m0); u1[c] = dot3(S[c], m1); }  // S M^T (S symmetric)
			// a0, c0: the covariance before the low-pass, kept for AA (recovering them as ca - 0.3 would cancel to a relative
			// error of u 0.3 / c0 on exactly the thin splats the compensation acts on)
			const float a0 = dot3(m0, u0), c0 = dot3(m1, u1);
			const float ca = a0 + 0.3f, cb = dot3(m0, u1), cc = c0 + 0.3f;
			const float det = ca * cc - cb * cb;
			const float wgt = 1.0f / (det * det + 0.0000001f);
			// H = -w adj(S') G adj(S')
			const float e00 = cc * gA - cb * gB, e01 = cc * gB - cb * gC, e10 = ca * gB - cb * gA, e11 = ca * gC - cb * gB;
			float H00 = -wgt * (e00 * cc - e01 * cb), H01 = -wgt * (e01 * ca - e00 * cb), H11 = -wgt * (e11 * ca - e10 * cb);
			if (AA) {
				// opacity compensation: grad d0 = (c0, -2b, a0), grad d1 = (c, -2b, a) w.r.t. (a, b, c), b one variable;
				// H01 is the gradient w.r.t. ONE off-diagonal entry, so it takes half of the b term
				const float d0 = fmaf(-cb, cb, a0 * c0);  // as the forward's det0
				const float r = d0 / det;
				gop += sqrtf(fmaxf(2.5e-5f, r)) * g1.y;
				if (r > 2.5e-5f) {
					const float k = 0.5f * g1.y * o_eff, i0 = 1.0f / d0, i1 = 1.0f / det;
					H00 += k * (c0 * i0 - cc * i1);
					H11 += k * (a0 * i0 - ca * i1);
					H01 += k * cb * (i1 - i0);
				}
			}
			// dL/dS += M^T H M
			float h0[3], h1[3];
#pragma unroll
			for (int c = 0; c < 3; c++) { h0[c] = H00 * m0[c] + H01 * m1[c]; h1[c] = H01 * m0[c] + H11 * m1[c]; }
			D[0] += m0[0] * h0[0] + m1[0] * h1[0]; D[1] += m0[0] * h0[1] + m1[0] * h1[1]; D[2] += m0[0] * h0[2] + m1[0] * h1[2];
			D[3] += m0[1] * h0[1] + m1[1] * h1[1]; D[4] += m0[1] * h0[2] + m1[1] * h1[2]; D[5] += m0[2] * h0[2] + m1[2] * h1[2];
			// dL/dM = 2 H (M S), dL/dJ = dL/dM Rv^T (only J00, J02, J11, J12 move with t)
			float q0[3], q1[3];
#pragma unroll
			for (int c = 0; c < 3; c++) { q0[c] = 2.f * (H00 * u0[c] + H01 * u1[c]); q1[c] = 2.f * (H01 * u0[c] + H11 * u1[c]); }
			const float dJ00 = dot3(q0, Rv[0]), dJ02 = dot3(q0, Rv[2]), dJ11 = dot3(q1, Rv[1]), dJ12 = dot3(q1, Rv[2]);
			const float iz3 = iz2 * iz;
			float dt[3];
			dt[0] = inx ? -fx * iz2 * dJ02 : 0.f;
			dt[1] = iny ? -fy * iz2 * dJ12 : 0.f;
			dt[2] = -fx * iz2 * dJ00 - fy * iz2 * dJ11 + 2.f * fx * cx * iz3 * dJ02 + 2.f * fy * cy * iz3 * dJ12 + ddepth;  // depth = t.z
			// screen-space mean through the full projection: ndc = (P p).xy / ((P p).w + 1e-7)
			const float* pm = w.projmatrix;  // P[r][c] = pm[4 c + r]
			const float hx = pm[0] * p[0] + pm[4] * p[1] + pm[8] * p[2] + pm[12];
			const float hy = pm[1] * p[0] + pm[5] * p[1] + pm[9] * p[2] + pm[13];
			const float hw = pm[3] * p[0] + pm[7] * p[1] + pm[11] * p[2] + pm[15];
			const float iw = 1.0f / (hw + 0.0000001f);
			const float kx = hx * iw * iw, ky = hy * iw * iw;
#pragma unroll
			for (int c = 0; c < 3; c++) {
				gp[c] += Rv[0][c] * dt[0] + Rv[1][c] * dt[1] + Rv[2][c] * dt[2]
					+ (pm[4 * c] * iw - pm[4 * c + 3] * kx) * dm[0] + (pm[4 * c + 1] * iw - pm[4 * c + 3] * ky) * dm[1];
			}
			// colour -> SH coefficients, and through the view direction into the mean
			if (sh) {
				const float dRGB[3] = { (cl & 1) ? 0.f : dcol[0], (cl & 2) ? 0.f : dcol[1], (cl & 4) ? 0.f : dcol[2] };
				const float vx = p[0] - w.cam_pos[0], vy = p[1] - w.cam_pos[1], vz = p[2] - w.cam_pos[2];
				const float il = 1.0f / sqrtf(vx * vx + vy * vy + vz * vz);
				const float x = vx * il, y = vy * il, z = vz * il;
				float dd[3] = { 0.f, 0.f, 0.f };  // dL/d(direction)
				// coefficient k: basis value B and its gradient (bx, by, bz) w.r.t. the direction
				auto term = [&](int k, float B, float bx, float by, float bz) {
					const float s = sh[3 * k] * dRGB[0] + sh[3 * k + 1] * dRGB[1] + sh[3 * k + 2] * dRGB[2];
					if (3 * k + 2 < NSH) { gsh[3 * k] += B * dRGB[0]; gsh[3 * k + 1] += B * dRGB[1]; gsh[3 * k + 2] += B * dRGB[2]; }
					dd[0] += bx * s; dd[1] += by * s; dd[2] += bz * s;
				};
				term(0, kSh.c0, 0.f, 0.f, 0.f);
				if (deg > 0) {
					term(1, -kSh.c1 * y, 0.f, -kSh.c1, 0.f);
					term(2, kSh.c1 * z, 0.f, 0.f, kSh.c1);
					term(3, -kSh.c1 * x, -kSh.c1, 0.f, 0.f);
				}
				if (NSH >= 27 && deg > 1) {
					const float xx = x * x, yy = y * y, zz = z * z;
					term(4, kSh.c2[0] * x * y, kSh.c2[0] * y, kSh.c2[0] * x, 0.f);
					term(5, kSh.c2[1] * y * z, 0.f, kSh.c2[1] * z, kSh.c2[1] * y);
					term(6, kSh.c2[2] * (2.f * zz - xx - yy), -2.f * kSh.c2[2] * x, -2.f * kSh.c2[2] * y, 4.f * kSh.c2[2] * z);
					term(7, kSh.c2[3] * x * z, kSh.c2[3] * z, 0.f, kSh.c2[3] * x);
					term(8, kSh.c2[4] * (xx - yy), 2.f * kSh.c2[4] * x, -2.f * kSh.c2[4] * y, 0.f);
					if (NSH >= 48 && deg > 2) {
						term(9, kSh.c3[0] * y * (3.f * xx - yy), kSh.c3[0] * 6.f * x * y, kSh.c3[0] * 3.f * (xx - yy), 0.f);
						term(10, kSh.c3[1] * x * y * z, kSh.c3[1] * y * z, kSh.c3[1] * x * z, kSh.c3[1] * x * y);
						term(11, kSh.c3[2] * y * (4.f * zz - xx - yy), kSh.c3[2] * -2.f * x * y, kSh.c3[2] * (4.f * zz - xx - 3.f * yy), kSh.c3[2] * 8.f * y * z);
						term(12, kSh.c3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy), kSh.c3[3] * -6.f * x * z, kSh.c3[3] * -6.f * y * z, kSh.c3[3] * (6.f * zz - 3.f * xx - 3.f * yy));
						term(13, kSh.c3[4] * x * (4.f * zz - xx - yy), kSh.c3[4] * (4.f * zz - 3.f * xx - yy), kSh.c3[4] * -2.f * x * y, kSh.c3[4] * 8.f * x * z);
						term(14, kSh.c3[5] * z * (xx - yy), kSh.c3[5] * 2.f * x * z, kSh.c3[5] * -2.f * y * z, kSh.c3[5] * (xx - yy));
						term(15, kSh.c3[6] * x * (xx - 3.f * yy), kSh.c3[6] * 3.f * (xx - yy), kSh.c3[6] * -6.f * x * y, 0.f);
					}
				}
				// through the normalisation: d dir / d v = (I - dir dir^T) / |v|
				const float along = x * dd[0] + y * dd[1] + z * dd[2];
				gp[0] += (dd[0] - x * along) * il; gp[1] += (dd[1] - y * along) * il; gp[2] += (dd[2] - z * along) * il;
			}
		} else if (a.dL_dconic && v == 0) {  // culled: the row is still written (the reference's zero-fill)
			float* o = a.dL_dconic + 4 * (size_t)idx;
			o[0] = 0.f; o[1] = 0.f; o[2] = 0.f; o[3] = 0.f;
		}
		// this view's screen-space gradient row (the reference's dL_dmeans2D, [P,3] with z = 0)
		if (a.shared_mean2D) { gm2[0] += dm[0]; gm2[1] += dm[1]; }
		else if (w.dL_dmean2D) {
			float* o = w.dL_dmean2D + 3 * (size_t)idx;
			o[0] = dm[0]; o[1] = dm[1]; o[2] = 0.f;
		}
	}

	// ---- covariance -> scale and quaternion (once, on the sum over views) ----
	float dscale[3] = { 0.f, 0.f, 0.f }, drot[4] = { 0.f, 0.f, 0.f, 0.f };
	if (from_sr) {
		const float Dm[3][3] = { { D[0], D[1], D[2] }, { D[1], D[3], D[4] }, { D[2], D[4], D[5] } };
		float R[3][3];
		rotation(R);
		float A[3][3];  // dL/dR = (2 D L) diag(s),  L = R diag(s)
#pragma unroll
		for (int j = 0; j < 3; j++) {
			float gl[3];
#pragma unroll
			for (int i = 0; i < 3; i++) gl[i] = 2.f * se[j] * (Dm[i][0] * R[0][j] + Dm[i][1] * R[1][j] + Dm[i][2] * R[2][j]);
			dscale[j] = R[0][j] * gl[0] + R[1][j] * gl[1] + R[2][j] * gl[2];
#pragma unroll
			for (int i = 0; i < 3; i++) A[i][j] = gl[i] * se[j];
		}
		const float r = q4[0], x = q4[1], y = q4[2], z = q4[3];
		drot[0] = 2.f * (z * (A[1][0] - A[0][1]) + y * (A[0][2] - A[2][0]) + x * (A[2][1] - A[1][2]));
		drot[1] = 2.f * (y * (A[0][1] + A[1][0]) + z * (A[0][2] + A[2][0]) + r * (A[2][1] - A[1][2])) - 4.f * x * (A[1][1] + A[2][2]);
		drot[2] = 2.f * (x * (A[0][1] + A[1][0]) + r * (A[0][2] - A[2][0]) + z * (A[1][2] + A[2][1])) - 4.f * y * (A[0][0] + A[2][2]);
		drot[3] = 2.f * (r * (A[1][0] - A[0][1]) + x * (A[0][2] + A[2][0]) + y * (A[1][2] + A[2][1])) - 4.f * z * (A[0][0] + A[1][1]);
	}

	// ---- outputs: every row written once (or added to the caller's running sum) ----
	const bool acc = a.accumulate != 0;
	auto put = [acc](float* o, float v) { *o = acc ? *o + v : v; };
	if (a.shared_mean2D && a.view[0].dL_dmean2D) {
		float* o = a.view[0].dL_dmean2D + 3 * (size_t)idx;
		put(o, gm2[0]); put(o + 1, gm2[1]); if (!acc) o[2] = 0.f;
	}
#pragma unroll
	for (int c = 0; c < 3; c++) put(a.dL_dmean3D + 3 * (size_t)idx + c, gp[c]);
	put(a.dL_dopacity + idx, gop);
	if (a.dL_dcolor) {
#pragma unroll
		for (int c = 0; c < 3; c++) put(a.dL_dcolor + 3 * (size_t)idx + c, gcol[c]);
	}
	if (a.dL_dcov3D) {
		float* o = a.dL_dcov3D + 6 * (size_t)idx;  // off-diagonal entries appear twice in the symmetric matrix
		put(o, D[0]); put(o + 1, 2.f * D[1]); put(o + 2, 2.f * D[2]); put(o + 3, D[3]); put(o + 4, 2.f * D[4]); put(o + 5, D[5]);
	}
	if (a.dL_dscale) {
#pragma unroll
		for (int c = 0; c < 3; c++) put(a.dL_dscale + 3 * (size_t)idx + c, dscale[c]);
	}
	if (a.dL_drot) {
#pragma unroll
		for (int c = 0; c < 4; c++) put(a.dL_drot + 4 * (size_t)idx + c, drot[c]);
	}
	if (a.dL_dsh) {
		float* o = a.dL_dsh + (size_t)idx * a.M * 3;
		const int used = sh ? 3 * (deg + 1) * (deg + 1) : 0;
#pragma unroll
		for (int i = 0; i < NSH; i++)
			if (i < 3 * a.M) put(o + i, i < used ? gsh[i] : 0.f);
		for (int i = NSH; i < 3 * a.M; i++) put(o + i, 0.f);  // coefficients above the active degree
	}
}

template <int NSH, int MIN_BLOCKS, bool AA>
__global__ void __launch_bounds__(128, MIN_BLOCKS) project_bwd_views_kernel(ProjectBwdViewsArgs a)
{
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= a.P) return;
	project_bwd_gaussian<NSH, AA>(a, idx);
}

namespace {
// one cloud of a ProjectBwdCloudsArgs launch under the member names project_bwd_gaussian reads; per-view screen-space
// gradients only, no dL_dconic
struct CloudBwd {
	int D, M, V;
	const float* means3D; const float* shs; const float* scales; const float* rotations; float scale_modifier;
	const float* cov3D_precomp;
	int accumulate;
	static constexpr int shared_mean2D = 0;
	float* dL_dmean3D; float* dL_dopacity; float* dL_dcolor; float* dL_dcov3D; float* dL_dsh; float* dL_dscale; float* dL_drot;
	static constexpr float* dL_dconic = nullptr;
	const ProjectBwdView* view;
	const float4* const* conic_opacity;  // AA only
};
}  // namespace

// several clouds in one launch: CTAs [cloud[c].block0, cloud[c + 1].block0) serve cloud c
template <int NSH, int MIN_BLOCKS, bool AA>
__global__ void __launch_bounds__(128, MIN_BLOCKS) project_bwd_clouds_kernel(ProjectBwdCloudsArgs a)
{
	int c = 0;
	while (c + 1 < a.B && (int)blockIdx.x >= a.cloud[c + 1].block0) c++;
	const ProjectBwdCloud& cl = a.cloud[c];
	const int idx = ((int)blockIdx.x - cl.block0) * blockDim.x + threadIdx.x;
	if (idx >= cl.P) return;
	const CloudBwd cb{ a.D, a.M, cl.V, cl.means3D, cl.shs, cl.scales, cl.rotations, a.scale_modifier, cl.cov3D_precomp, cl.accumulate,
		cl.dL_dmean3D, cl.dL_dopacity, cl.dL_dcolor, cl.dL_dcov3D, cl.dL_dsh, cl.dL_dscale, cl.dL_drot, a.view + cl.view0,
		AA ? a.conic_opacity + cl.view0 : nullptr };
	project_bwd_gaussian<NSH, AA>(cb, idx);
}

void launch_project_bwd_views(const ProjectBwdViewsArgs& a, cudaStream_t s)
{
	if (a.P <= 0 || a.V <= 0) return;
	const int grid = ceil_div(a.P, 128);
	const int deg = a.shs ? a.D : 0;
	if (a.antialias) {
		// 4 blocks per SM at degree <= 1: the compensation's registers do not fit the cap of 5 (96) without spilling
		if (deg <= 1) project_bwd_views_kernel<12, 4, true><<<grid, 128, 0, s>>>(a);
		else if (deg == 2) project_bwd_views_kernel<27, 4, true><<<grid, 128, 0, s>>>(a);
		else project_bwd_views_kernel<48, 3, true><<<grid, 128, 0, s>>>(a);
		return;
	}
	if (deg <= 1) project_bwd_views_kernel<12, MGS_PBWD_MINB, false><<<grid, 128, 0, s>>>(a);
	else if (deg == 2) project_bwd_views_kernel<27, 4, false><<<grid, 128, 0, s>>>(a);
	else project_bwd_views_kernel<48, 3, false><<<grid, 128, 0, s>>>(a);
}

void launch_project_bwd_clouds(ProjectBwdCloudsArgs a, cudaStream_t s)
{
	if (a.B <= 0) return;
	int grid = 0;
	bool sh = false;
	for (int c = 0; c < a.B; c++) {
		a.cloud[c].block0 = grid;
		grid += ceil_div(a.cloud[c].P, 128);
		sh |= a.cloud[c].shs != nullptr;
	}
	const int deg = sh ? a.D : 0;
	// 4 blocks per SM at degree <= 1: the register cap of 5 (96) spills here, and the launch is small where it matters most
	// (one CTA per 128 Gaussians of each cloud: 16k Gaussians fill one wave)
	if (a.antialias) {
		if (deg <= 1) project_bwd_clouds_kernel<12, 4, true><<<grid, 128, 0, s>>>(a);
		else if (deg == 2) project_bwd_clouds_kernel<27, 4, true><<<grid, 128, 0, s>>>(a);
		else project_bwd_clouds_kernel<48, 3, true><<<grid, 128, 0, s>>>(a);
		return;
	}
	if (deg <= 1) project_bwd_clouds_kernel<12, 4, false><<<grid, 128, 0, s>>>(a);
	else if (deg == 2) project_bwd_clouds_kernel<27, 4, false><<<grid, 128, 0, s>>>(a);
	else project_bwd_clouds_kernel<48, 3, false><<<grid, 128, 0, s>>>(a);
}

}  // namespace mgs
