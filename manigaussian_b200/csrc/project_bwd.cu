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
#include "camera.cuh"

#include <type_traits>

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

// one step of a warp's recursive halving over 2H values: lane pairs (l, l ^ H) add their halves, the lane with bit H set keeps
// the upper one in x[0 .. H).  Steps H = 16 .. 1 leave the warp's sum of x[l] on lane l.  The halves are picked with bit masks:
// a select between array elements would put x in local memory.
template <int H>
__device__ __forceinline__ void warp_halve(float* x, const int lane)
{
	const int up = (lane & H) ? -1 : 0;
#pragma unroll
	for (int k = 0; k < H; k++) {
		const int lo = __float_as_int(x[k]), hi = __float_as_int(x[k + H]);
		const float got = __shfl_xor_sync(0xffffffffu, __int_as_float((lo & up) | (hi & ~up)), H);
		x[k] = __int_as_float((hi & up) | (lo & ~up)) + got;
	}
}

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
//
// CAM (camera gradients, and the instantiation that reads a view's device field of view, a.intr[v].tan_fov, when set): per
// view, each thread forms the camera terms of its Gaussian (zeros where culled or past the end:
// `in` false), the warp sums them into cam_sm[(warp, view)][CAM_TERMS], and the kernel sums its warps after the loop.  A CAM
// thread therefore runs the whole view loop; it reads Gaussian 0 in place of a missing one and writes no per-Gaussian row.
//
// ORTHO (CAM only): bit v of a.ortho marks view v orthographic.  There J = [[fx, 0, 0], [0, fy, 0]] does not move with t, so
// M = J Rv has rows fx Rv0 and fy Rv1, dL/dt is the depth cotangent on t.z alone, the camera terms take J^T Q = (fx q0, fy q1, 0)
// and dL/dtan_fov = -(f / tan_fov) dJ00 (dJ11).  The bit is the same for every thread of the launch.
//
// FISH (ORTHO and CAM only): bit v of a.fisheye marks view v a Kannala-Brandt fisheye view with coefficients a.fe_k[v]
// (fisheye.cuh).  There the screen mean is the fisheye map of t in pixels, not of projmatrix: with (du, dv) = (dm0 / (W / 2),
// dm1 / (H / 2)) its cotangent (dm, the blend's dL/dmean2D, is w.r.t. ndc), dL/dt gains J^T (du, dv) and the
// projection-matrix terms are zero; all six entries of J move with t, dL/dt takes the contraction of dL/dJ with dJ/dt,
// the camera terms take the full J^T Q, and dL/dtan_fovx = -(du (u - cx) + sum_j dJ0j J0j) / tan_fovx (y likewise).
//
// DIST (FISH, ORTHO and CAM only): bit v of a.distorted marks view v an OpenCV distorted-pinhole view with coefficients
// a.dc_k[v] (distortion.cuh).  As for FISH, the screen mean (u, v) = (fx xd + cx, fy yd + cy) is in pixels and its cotangent is
// (du, dv); J = F Dd P with F = diag(fx, fy), P = d(x, y) / dt = [[1/z, 0, -x/z], [0, 1/z, -y/z]].  With G = F dL/dJ,
// dL/dJ : dJ/dt = (G P^T) : dDd/d(x, y) chained through P, plus (Dd G) : dP/dt (Dd is symmetric); J^T (du, dv) enters through
// the same chain.  The camera terms and dL/dtan_fov are the fisheye ones with u - cx = fx xd.
//
// PLN (DIST, FISH, ORTHO and CAM only): planar depth on the views with a.pl_g[v] set.  The blend's quad gradients of
// (a, b, e = -(a mu_x + b mu_y)) arrive with e's share folded in, {ga - mu_x ge, gb - mu_y ge, ge} = dL/d(a, b) and ge (formed
// relative to the mean in the blend, where its terms stay footprint-sized); through e, the screen mean's cotangent is
// -(a, b) ge in pixels, added to dm in its convention.  With (a, b) = k Q, k_j = Rv2^T S m_j (m_j row j of M = J Rv):
// dL/dQ = k^T dL/d(a, b) joins G, dk = dL/d(a, b) Q, and dk reaches S (sym(Rv2 n^T), n = dk_0 m_0 + dk_1 m_1), M (dL/dm_j +=
// dk_j S Rv2, so the existing chain carries it through J to t, the camera and the field of view) and the third row of Rv
// (dk_0 S m_0 + dk_1 S m_1).
template <int NSH, bool AA, bool CAM, bool ORTHO, bool FISH, bool DIST, bool PLN, class Args>
__device__ __forceinline__ void project_bwd_gaussian(const Args& a, const int idx_in, const bool in, float* cam_sm)
{
	const int idx = CAM && !in ? 0 : idx_in;
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
		const bool orv = ORTHO && ((a.ortho >> v) & 1u);  // view v is orthographic
		const bool fev = FISH && ((a.fisheye >> v) & 1u);  // view v is a fisheye view
		const bool dsv = DIST && ((a.distorted >> v) & 1u);  // view v is a distorted-pinhole view
		const float4* gb = reinterpret_cast<const float4*>(w.gb + (size_t)idx * GB_STRIDE);
		const float4 g0 = gb[0], g1 = gb[1], g2 = gb[2];
		const uint8_t cl = sh ? w.clamped[idx] : (uint8_t)0;
		const float o_eff = AA ? a.conic_opacity[v][idx].w : 0.f;
		const bool live = (!CAM || in) && w.radii[idx] > 0;
		float dm[2] = { 0.f, 0.f };
		float cg[32];  // CAM: this view's camera terms (CAM_TERMS used, padded to a warp)
#pragma unroll
		for (int k = 0; k < 32; k++) cg[k] = 0.f;
		if (live) {
			dm[0] = g0.x; dm[1] = g0.y;
			float gA = g0.z, gB = g0.w, gC = g1.x;              // dL/dconic (xx, xy halved, yy)
			bool plv = false;                                   // PLN: the view has planar depth
			float pga = 0.f, pgb = 0.f;                         // PLN: dL/d(a, b), e's share included
			if constexpr (PLN) {
				plv = a.pl_g[v] != nullptr;
				if (plv) {
					const float4 g = a.pl_g[v][idx], q = a.pl_q[v][idx];
					pga = g.x; pgb = g.y;  // the blend formed them relative to the mean (mgs_kernels.h, BlendArgs::planar)
					dm[0] -= q.x * g.z * (0.5f * a.intr[v].W); dm[1] -= q.y * g.z * (0.5f * a.intr[v].H);
				}
			}
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
			// CAM: the view's device field of view, when set; the focal lengths are then formed as the host forms focal_x / focal_y
			const float* dfov = nullptr;
			if constexpr (CAM) dfov = a.intr[v].tan_fov;
			const float tanx = dfov ? dfov[0] : w.tan_fovx, tany = dfov ? dfov[1] : w.tan_fovy;
			const float limx = 1.3f * tanx, limy = 1.3f * tany;
			const float ux = tx / tz, uy = ty / tz;
			const bool inx = !(ux < -limx || ux > limx), iny = !(uy < -limy || uy > limy);
			const float cx = fminf(limx, fmaxf(-limx, ux)) * tz, cy = fminf(limy, fmaxf(-limy, uy)) * tz;
			const float iz = 1.0f / tz, iz2 = iz * iz;
			const float fx = dfov ? focal_length(a.intr[v].W, tanx) : w.focal_x, fy = dfov ? focal_length(a.intr[v].H, tany) : w.focal_y;
			// M = J Rv: row 0 = (fx / tz) Rv0 - (fx cx / tz^2) Rv2, row 1 likewise with y
			float m0[3], m1[3], u0[3], u1[3];
			FisheyeRadial fr{};
			float J[2][3] = { { 0.f, 0.f, 0.f }, { 0.f, 0.f, 0.f } };  // FISH, DIST: J
			float du = 0.f, dv = 0.f;  // FISH, DIST: the cotangent of the pixel-space mean (u, v)
			DistTerms ds{};
			float nx = 0.f, ny = 0.f;  // DIST: the normalised coordinates t.xy / t.z
			if (dsv) {
				du = dm[0] / (0.5f * a.intr[v].W); dv = dm[1] / (0.5f * a.intr[v].H);
				nx = tx * iz; ny = ty * iz;
				ds = distortion_terms<true>(nx, ny, a.dc_k[v]);
				distorted_jacobian(ds, nx, ny, iz, fx, fy, J);
#pragma unroll
				for (int c = 0; c < 3; c++) {
					m0[c] = J[0][0] * Rv[0][c] + J[0][1] * Rv[1][c] + J[0][2] * Rv[2][c];
					m1[c] = J[1][0] * Rv[0][c] + J[1][1] * Rv[1][c] + J[1][2] * Rv[2][c];
				}
			} else if (fev) {
				// dm is the blend's dL/dmean2D, the gradient w.r.t. ndc = (2 u + 1) / W - 1 (the reference's convention: the
				// blend scales its pixel-space gradient by W / 2, H / 2); the fisheye mean is in pixels
				du = dm[0] / (0.5f * a.intr[v].W); dv = dm[1] / (0.5f * a.intr[v].H);
				fr = fisheye_radial<true>(tx, ty, tz, a.fe_k[v]);
				fisheye_jacobian(fr, tx, ty, fx, fy, J);
#pragma unroll
				for (int c = 0; c < 3; c++) {
					m0[c] = J[0][0] * Rv[0][c] + J[0][1] * Rv[1][c] + J[0][2] * Rv[2][c];
					m1[c] = J[1][0] * Rv[0][c] + J[1][1] * Rv[1][c] + J[1][2] * Rv[2][c];
				}
			} else if (orv) {
#pragma unroll
				for (int c = 0; c < 3; c++) { m0[c] = fx * Rv[0][c]; m1[c] = fy * Rv[1][c]; }
			} else {
#pragma unroll
				for (int c = 0; c < 3; c++) {
					m0[c] = fx * iz * Rv[0][c] - fx * cx * iz2 * Rv[2][c];
					m1[c] = fy * iz * Rv[1][c] - fy * cy * iz2 * Rv[2][c];
				}
			}
#pragma unroll
			for (int c = 0; c < 3; c++) { u0[c] = dot3(S[c], m0); u1[c] = dot3(S[c], m1); }  // S M^T (S symmetric)
			// a0, c0: the covariance before the low-pass, kept for AA (recovering them as ca - 0.3 would cancel to a relative
			// error of u 0.3 / c0 on exactly the thin splats the compensation acts on)
			const float a0 = dot3(m0, u0), c0 = dot3(m1, u1);
			const float ca = a0 + 0.3f, cb = dot3(m0, u1), cc = c0 + 0.3f;
			const float det = ca * cc - cb * cb;
			float dk0 = 0.f, dk1 = 0.f;  // PLN: dL/dk
			if constexpr (PLN) {
				if (plv) {
					const float k0 = dot3(Rv[2], u0), k1 = dot3(Rv[2], u1);
					const float idet = 1.0f / det, QA = cc * idet, QB = -cb * idet, QC = ca * idet;
					gA += k0 * pga; gC += k1 * pgb; gB += 0.5f * (k0 * pgb + k1 * pga);
					dk0 = pga * QA + pgb * QB; dk1 = pga * QB + pgb * QC;
					float n[3];
#pragma unroll
					for (int c = 0; c < 3; c++) n[c] = dk0 * m0[c] + dk1 * m1[c];
					const float* r2 = Rv[2];
					D[0] += r2[0] * n[0]; D[1] += 0.5f * (r2[0] * n[1] + n[0] * r2[1]); D[2] += 0.5f * (r2[0] * n[2] + n[0] * r2[2]);
					D[3] += r2[1] * n[1]; D[4] += 0.5f * (r2[1] * n[2] + n[1] * r2[2]); D[5] += r2[2] * n[2];
				}
			}
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
			if constexpr (PLN) {
				if (plv) {
#pragma unroll
					for (int c = 0; c < 3; c++) {
						const float sr = dot3(S[c], Rv[2]);
						q0[c] += dk0 * sr; q1[c] += dk1 * sr;
					}
				}
			}
			const float dJ00 = dot3(q0, Rv[0]), dJ02 = dot3(q0, Rv[2]), dJ11 = dot3(q1, Rv[1]), dJ12 = dot3(q1, Rv[2]);
			if constexpr (CAM) {
				// dL/dtan_fov: fx = W / (2 tan_fovx) moves J00 = fx / tz and J02 = -fx cx / tz^2 (dfx / dtan_fovx = -fx / tan_fovx),
				// and where the x clamp holds, cx = +-1.3 tan_fovx tz moves J02.  Likewise for y.
				if (dsv) {
					// u - cx = fx xd and every entry of J's first row scale with fx
					const float dJ01 = dot3(q0, Rv[1]), dJ10 = dot3(q1, Rv[0]);
					cg[27] = -(du * fx * ds.xd + dJ00 * J[0][0] + dJ01 * J[0][1] + dJ02 * J[0][2]) / tanx;
					cg[28] = -(dv * fy * ds.yd + dJ10 * J[1][0] + dJ11 * J[1][1] + dJ12 * J[1][2]) / tany;
				} else if (fev) {
					// u - cx = fx a t.x and every entry of J's first row scale with fx
					const float dJ01 = dot3(q0, Rv[1]), dJ10 = dot3(q1, Rv[0]);
					cg[27] = -(du * fx * fr.a * tx + dJ00 * J[0][0] + dJ01 * J[0][1] + dJ02 * J[0][2]) / tanx;
					cg[28] = -(dv * fy * fr.a * ty + dJ10 * J[1][0] + dJ11 * J[1][1] + dJ12 * J[1][2]) / tany;
				} else if (orv) {
					cg[27] = -(fx / tanx) * dJ00;
					cg[28] = -(fy / tany) * dJ11;
				} else {
					const float sx = ux > 0.f ? 1.3f : -1.3f, sy = uy > 0.f ? 1.3f : -1.3f;
					cg[27] = -(fx / tanx) * (dJ00 * iz - dJ02 * cx * iz2) - (inx ? 0.f : fx * dJ02 * sx * iz);
					cg[28] = -(fy / tany) * (dJ11 * iz - dJ12 * cy * iz2) - (iny ? 0.f : fy * dJ12 * sy * iz);
				}
			}
			const float iz3 = iz2 * iz;
			float dt[3];
			if (dsv) {
				// G = F dL/dJ; K = G P^T contracts with dDd/d(x, y), N = Dd G with dP/dt; (gx, gy) = dL/d(x, y), J^T (du, dv)
				// included through F Dd
				const float dJ01 = dot3(q0, Rv[1]), dJ10 = dot3(q1, Rv[0]);
				const float G00 = fx * dJ00, G01 = fx * dJ01, G02 = fx * dJ02, G10 = fy * dJ10, G11 = fy * dJ11, G12 = fy * dJ12;
				const float K00 = (G00 - nx * G02) * iz, Kx = (G01 - ny * G02 + G10 - nx * G12) * iz, K11 = (G11 - ny * G12) * iz;
				const float eu = fx * du, ev = fy * dv;
				const float gx = K00 * ds.hxxx + Kx * ds.hxxy + K11 * ds.hxyy + ds.d00 * eu + ds.d01 * ev;
				const float gy = K00 * ds.hxxy + Kx * ds.hxyy + K11 * ds.hyyy + ds.d01 * eu + ds.d11 * ev;
				const float N00 = ds.d00 * G00 + ds.d01 * G10, N02 = ds.d00 * G02 + ds.d01 * G12;
				const float N11 = ds.d01 * G01 + ds.d11 * G11, N12 = ds.d01 * G02 + ds.d11 * G12;
				dt[0] = (gx - N02 * iz) * iz;
				dt[1] = (gy - N12 * iz) * iz;
				dt[2] = (2.f * (N02 * nx + N12 * ny) - N00 - N11) * iz2 - (gx * nx + gy * ny) * iz + ddepth;
			} else if (fev) {
				// dL/dJ contracted with dJ/dt (fisheye.cuh: da/dx = c x, da/dz = -g, (dg/dr) / r = -cz), then J^T (du, dv)
				const float dJ01 = dot3(q0, Rv[1]), dJ10 = dot3(q1, Rv[0]);
				const float A = fx * dJ00, Bs = fx * dJ01 + fy * dJ10, Cc = fx * dJ02, Ee = fy * dJ11, Ff = fy * dJ12;
				const float cx2 = fr.c + fr.C1 * tx * tx, cy2 = fr.c + fr.C1 * ty * ty;
				dt[0] = A * tx * (2.f * fr.c + cx2) + Bs * ty * cx2 + Ee * tx * cy2 - Cc * (fr.g - fr.cz * tx * tx) + Ff * fr.cz * tx * ty;
				dt[1] = A * ty * cx2 + Bs * tx * cy2 + Ee * ty * (2.f * fr.c + cy2) + Cc * fr.cz * tx * ty - Ff * (fr.g - fr.cz * ty * ty);
				dt[2] = A * (fr.cz * tx * tx - fr.g) + Bs * fr.cz * tx * ty + Ee * (fr.cz * ty * ty - fr.g) - (Cc * tx + Ff * ty) * fr.gz
					+ ddepth;
				dt[0] += J[0][0] * du + J[1][0] * dv;
				dt[1] += J[0][1] * du + J[1][1] * dv;
				dt[2] += J[0][2] * du + J[1][2] * dv;
			} else if (orv) {
				dt[0] = 0.f; dt[1] = 0.f; dt[2] = ddepth;
			} else {
				dt[0] = inx ? -fx * iz2 * dJ02 : 0.f;
				dt[1] = iny ? -fy * iz2 * dJ12 : 0.f;
				dt[2] = -fx * iz2 * dJ00 - fy * iz2 * dJ11 + 2.f * fx * cx * iz3 * dJ02 + 2.f * fy * cy * iz3 * dJ12 + ddepth;  // depth = t.z
			}
			// screen-space mean through the full projection: ndc = (P p).xy / ((P p).w + 1e-7)
			const float* pm = w.projmatrix;  // P[r][c] = pm[4 c + r]
			const float hx = pm[0] * p[0] + pm[4] * p[1] + pm[8] * p[2] + pm[12];
			const float hy = pm[1] * p[0] + pm[5] * p[1] + pm[9] * p[2] + pm[13];
			const float hw = pm[3] * p[0] + pm[7] * p[1] + pm[11] * p[2] + pm[15];
			const float iw = 1.0f / (hw + 0.0000001f);
			const float kx = hx * iw * iw, ky = hy * iw * iw;
			const float dmp[2] = { fev || dsv ? 0.f : dm[0], fev || dsv ? 0.f : dm[1] };  // the mean's path through projmatrix
#pragma unroll
			for (int c = 0; c < 3; c++) {
				gp[c] += Rv[0][c] * dt[0] + Rv[1][c] * dt[1] + Rv[2][c] * dt[2]
					+ (pm[4 * c] * iw - pm[4 * c + 3] * kx) * dmp[0] + (pm[4 * c + 1] * iw - pm[4 * c + 3] * ky) * dmp[1];
			}
			if constexpr (CAM) {
				// t = Rv p + tv and M = J Rv with J held: dL/dRv = dt p^T + J^T dL/dM, dL/dtv = dt
				const bool full = fev || dsv;  // J has all six entries
				const float j00 = full ? J[0][0] : orv ? fx : fx * iz, j11 = full ? J[1][1] : orv ? fy : fy * iz;
				const float j02 = full ? J[0][2] : orv ? 0.f : -fx * cx * iz2, j12 = full ? J[1][2] : orv ? 0.f : -fy * cy * iz2;
#pragma unroll
				for (int c = 0; c < 3; c++) {
					cg[3 * c] = dt[0] * p[c] + j00 * q0[c];
					cg[3 * c + 1] = dt[1] * p[c] + j11 * q1[c];
					cg[3 * c + 2] = dt[2] * p[c] + j02 * q0[c] + j12 * q1[c];
					if (full) { cg[3 * c] += J[1][0] * q1[c]; cg[3 * c + 1] += J[0][1] * q0[c]; }
				}
				if constexpr (PLN) {
#pragma unroll
					for (int c = 0; c < 3; c++) cg[3 * c + 2] += dk0 * u0[c] + dk1 * u1[c];  // k through the third row of Rv
				}
				cg[9] = dt[0]; cg[10] = dt[1]; cg[11] = dt[2];
				// (hx, hy, hw) = P (p, 1): dL/dhx = dm0 iw, dL/dhy = dm1 iw, dL/dhw = -(dm0 kx + dm1 ky)
				const float ax = dmp[0] * iw, ay = dmp[1] * iw, aw = -(dmp[0] * kx + dmp[1] * ky);
				const float ph[4] = { p[0], p[1], p[2], 1.f };
#pragma unroll
				for (int c = 0; c < 4; c++) { cg[12 + 3 * c] = ax * ph[c]; cg[13 + 3 * c] = ay * ph[c]; cg[14 + 3 * c] = aw * ph[c]; }
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
				if constexpr (CAM) {  // v = p - campos: the same term with the opposite sign
					cg[24] = -(dd[0] - x * along) * il; cg[25] = -(dd[1] - y * along) * il; cg[26] = -(dd[2] - z * along) * il;
				}
			}
		} else if (a.dL_dconic && v == 0 && in) {  // culled: the row is still written (the reference's zero-fill)
			float* o = a.dL_dconic + 4 * (size_t)idx;
			o[0] = 0.f; o[1] = 0.f; o[2] = 0.f; o[3] = 0.f;
		}
		// this view's screen-space gradient row (the reference's dL_dmeans2D, [P,3] with z = 0)
		if (a.shared_mean2D) { gm2[0] += dm[0]; gm2[1] += dm[1]; }
		else if (w.dL_dmean2D && in) {
			float* o = w.dL_dmean2D + 3 * (size_t)idx;
			o[0] = dm[0]; o[1] = dm[1]; o[2] = 0.f;
		}
		if constexpr (CAM) {
			// recursive halving over the warp: 16 + 8 + 4 + 2 + 1 shuffles leave the sum of term `lane` on lane `lane`, in an
			// order fixed by the lane numbers
			const int lane = threadIdx.x & 31;
			warp_halve<16>(cg, lane); warp_halve<8>(cg, lane); warp_halve<4>(cg, lane); warp_halve<2>(cg, lane); warp_halve<1>(cg, lane);
			if (lane < CAM_ALL_TERMS) cam_sm[((threadIdx.x >> 5) * MAX_BWD_VIEWS + v) * CAM_ALL_TERMS + lane] = cg[0];
		}
	}
	if (CAM && !in) return;

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

// CAM: after the view loop, one barrier and a sum over the CTA's 4 warps in warp order; row `blk` of each view's camera rows
// (terms < CAM_TERMS) and of its focal-length rows (the rest)
__device__ __forceinline__ void cam_rows_out(const float* cam_sm, int V, float* const* rows, const ProjectBwdIntr* intr, int blk)
{
	__syncthreads();
	for (int j = threadIdx.x; j < V * CAM_ALL_TERMS; j += blockDim.x) {
		const int v = j / CAM_ALL_TERMS, k = j - v * CAM_ALL_TERMS;
		float s = 0.f;
#pragma unroll
		for (int w = 0; w < 4; w++) s += cam_sm[(w * MAX_BWD_VIEWS + v) * CAM_ALL_TERMS + k];
		if (k < CAM_TERMS) {
			if (rows[v]) rows[v][(size_t)blk * CAM_TERMS + k] = s;
		} else if (intr[v].rows) {
			intr[v].rows[(size_t)blk * CAM_INTR_TERMS + k - CAM_TERMS] = s;
		}
	}
}

// DIST, FISH, ORTHO, CAM, AA last in the template list: AA stays the last argument of every kernel name and CAM the one before
// it, as profiles and the coverage tests read them.  ORTHO is instantiated with CAM only, FISH with ORTHO and CAM only, DIST
// with FISH, ORTHO and CAM only.  The planar-depth backward (PLN) has kernels of its own names below.
template <int NSH, int MIN_BLOCKS, bool DIST, bool FISH, bool ORTHO, bool CAM, bool AA>
__global__ void __launch_bounds__(128, MIN_BLOCKS) project_bwd_views_kernel(ProjectBwdViewsArgs a)
{
	static_assert(CAM || !ORTHO, "the orthographic backward is a CAM instantiation");
	static_assert(ORTHO || !FISH, "the fisheye backward is an ORTHO instantiation");
	static_assert(FISH || !DIST, "the distorted backward is a FISH instantiation");
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if constexpr (CAM) {
		__shared__ float cam_sm[4 * MAX_BWD_VIEWS * CAM_ALL_TERMS];
		project_bwd_gaussian<NSH, AA, true, ORTHO, FISH, DIST, false>(a, idx, idx < a.P, cam_sm);
		cam_rows_out(cam_sm, a.V, a.cam_rows, a.intr, blockIdx.x);
	} else {
		if (idx >= a.P) return;
		project_bwd_gaussian<NSH, AA, false, false, false, false, false>(a, idx, true, nullptr);
	}
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
	const ProjectBwdIntr* intr;          // CAM only
	unsigned ortho;                      // ORTHO only: bit v, view v of the cloud is orthographic
	unsigned fisheye;                    // FISH only: bit v, view v of the cloud is a fisheye view
	const FisheyeK* fe_k;                // FISH only: per view of the cloud
	unsigned distorted;                  // DIST only: bit v, view v of the cloud is a distorted-pinhole view
	const DistK* dc_k;                   // DIST only: per view of the cloud
};
// PLN only: with each view's planar-depth arrays (a type of its own, so the other instantiations keep their code)
struct CloudBwdPln : CloudBwd {
	const float4* const* pl_g;
	const float4* const* pl_q;
	const float2* const* pl_mean;
};
// the parameter block a clouds launch passes: the larger one for the DIST kernels (mgs_kernels.h), the parent's otherwise
template <bool DIST>
using CloudsArgs = typename std::conditional<DIST, ProjectBwdCloudsDistArgs, ProjectBwdCloudsArgs>::type;
}  // namespace

// several clouds in one launch: CTAs [cloud[c].block0, cloud[c + 1].block0) serve cloud c.  Two overloads of one name: the
// parent's parameter block, and the DIST instantiations' larger one (mgs_kernels.h), which adds each view's coefficients.
template <int NSH, int MIN_BLOCKS, bool DIST, bool FISH, bool ORTHO, bool CAM, bool AA>
__global__ void __launch_bounds__(128, MIN_BLOCKS) project_bwd_clouds_kernel(ProjectBwdCloudsArgs a)
{
	static_assert(CAM || !ORTHO, "the orthographic backward is a CAM instantiation");
	static_assert(ORTHO || !FISH, "the fisheye backward is an ORTHO instantiation");
	static_assert(!DIST, "the distorted backward takes ProjectBwdCloudsDistArgs");
	int c = 0;
	while (c + 1 < a.B && (int)blockIdx.x >= a.cloud[c + 1].block0) c++;
	const ProjectBwdCloud& cl = a.cloud[c];
	const int idx = ((int)blockIdx.x - cl.block0) * blockDim.x + threadIdx.x;
	if (!CAM && idx >= cl.P) return;
	unsigned dmask = 0u;  // no distorted view
	const DistK* dk = nullptr;
	const CloudBwd cb{ a.D, a.M, cl.V, cl.means3D, cl.shs, cl.scales, cl.rotations, a.scale_modifier, cl.cov3D_precomp, cl.accumulate,
		cl.dL_dmean3D, cl.dL_dopacity, cl.dL_dcolor, cl.dL_dcov3D, cl.dL_dsh, cl.dL_dscale, cl.dL_drot, a.view + cl.view0,
		AA ? a.conic_opacity + cl.view0 : nullptr, CAM ? a.intr + cl.view0 : nullptr, ORTHO ? (unsigned)a.ortho >> cl.view0 : 0u,
		FISH ? (unsigned)a.fisheye >> cl.view0 : 0u, FISH ? a.fe_k + cl.view0 : nullptr, dmask, dk };
	if constexpr (CAM) {
		// the CTA serves one cloud: its rows belong to that cloud's views
		__shared__ float cam_sm[4 * MAX_BWD_VIEWS * CAM_ALL_TERMS];
		project_bwd_gaussian<NSH, AA, true, ORTHO, FISH, DIST, false>(cb, idx, idx < cl.P, cam_sm);
		cam_rows_out(cam_sm, cl.V, a.cam_rows + cl.view0, a.intr + cl.view0, (int)blockIdx.x - cl.block0);
	} else {
		project_bwd_gaussian<NSH, AA, false, false, false, false, false>(cb, idx, true, nullptr);
	}
}
template <int NSH, int MIN_BLOCKS, bool DIST, bool FISH, bool ORTHO, bool CAM, bool AA>
__global__ void __launch_bounds__(128, MIN_BLOCKS) project_bwd_clouds_kernel(ProjectBwdCloudsDistArgs a)
{
	static_assert(DIST && FISH && ORTHO && CAM, "the distorted backward is a FISH, ORTHO and CAM instantiation");
	int c = 0;
	while (c + 1 < a.B && (int)blockIdx.x >= a.cloud[c + 1].block0) c++;
	const ProjectBwdCloud& cl = a.cloud[c];
	const int idx = ((int)blockIdx.x - cl.block0) * blockDim.x + threadIdx.x;
	if (!CAM && idx >= cl.P) return;
	const CloudBwd cb{ a.D, a.M, cl.V, cl.means3D, cl.shs, cl.scales, cl.rotations, a.scale_modifier, cl.cov3D_precomp, cl.accumulate,
		cl.dL_dmean3D, cl.dL_dopacity, cl.dL_dcolor, cl.dL_dcov3D, cl.dL_dsh, cl.dL_dscale, cl.dL_drot, a.view + cl.view0,
		AA ? a.conic_opacity + cl.view0 : nullptr, CAM ? a.intr + cl.view0 : nullptr, ORTHO ? (unsigned)a.ortho >> cl.view0 : 0u,
		FISH ? (unsigned)a.fisheye >> cl.view0 : 0u, FISH ? a.fe_k + cl.view0 : nullptr, (unsigned)a.distorted >> cl.view0, a.dc_k + cl.view0 };
	if constexpr (CAM) {
		// the CTA serves one cloud: its rows belong to that cloud's views
		__shared__ float cam_sm[4 * MAX_BWD_VIEWS * CAM_ALL_TERMS];
		project_bwd_gaussian<NSH, AA, true, ORTHO, FISH, DIST, false>(cb, idx, idx < cl.P, cam_sm);
		cam_rows_out(cam_sm, cl.V, a.cam_rows + cl.view0, a.intr + cl.view0, (int)blockIdx.x - cl.block0);
	} else {
		project_bwd_gaussian<NSH, AA, false, false, false, false, false>(cb, idx, true, nullptr);
	}
}

// planar depth (PLN): the DIST, FISH, ORTHO and CAM body with the planar terms, for every model; kernels of their own names, so
// that the names of the kernels above stay as profiles and the coverage tests read them
template <int NSH, int MIN_BLOCKS, bool AA>
__global__ void __launch_bounds__(128, MIN_BLOCKS) project_bwd_views_planar_kernel(ProjectBwdViewsArgs a)
{
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	__shared__ float cam_sm[4 * MAX_BWD_VIEWS * CAM_ALL_TERMS];
	project_bwd_gaussian<NSH, AA, true, true, true, true, true>(a, idx, idx < a.P, cam_sm);
	cam_rows_out(cam_sm, a.V, a.cam_rows, a.intr, blockIdx.x);
}
template <int NSH, int MIN_BLOCKS, bool AA>
__global__ void __launch_bounds__(128, MIN_BLOCKS) project_bwd_clouds_planar_kernel(ProjectBwdCloudsDistArgs a)
{
	int c = 0;
	while (c + 1 < a.B && (int)blockIdx.x >= a.cloud[c + 1].block0) c++;
	const ProjectBwdCloud& cl = a.cloud[c];
	const int idx = ((int)blockIdx.x - cl.block0) * blockDim.x + threadIdx.x;
	const CloudBwdPln cp{ { a.D, a.M, cl.V, cl.means3D, cl.shs, cl.scales, cl.rotations, a.scale_modifier, cl.cov3D_precomp,
		cl.accumulate, cl.dL_dmean3D, cl.dL_dopacity, cl.dL_dcolor, cl.dL_dcov3D, cl.dL_dsh, cl.dL_dscale, cl.dL_drot, a.view + cl.view0,
		AA ? a.conic_opacity + cl.view0 : nullptr, a.intr + cl.view0, (unsigned)a.ortho >> cl.view0, (unsigned)a.fisheye >> cl.view0,
		a.fe_k + cl.view0, (unsigned)a.distorted >> cl.view0, a.dc_k + cl.view0 },
		a.pl_g + cl.view0, a.pl_q + cl.view0, a.pl_mean + cl.view0 };
	__shared__ float cam_sm[4 * MAX_BWD_VIEWS * CAM_ALL_TERMS];
	project_bwd_gaussian<NSH, AA, true, true, true, true, true>(cp, idx, idx < cl.P, cam_sm);
	cam_rows_out(cam_sm, cl.V, a.cam_rows + cl.view0, a.intr + cl.view0, (int)blockIdx.x - cl.block0);
}

// one CTA of CAM_REDUCE_THREADS per view.  Thread t first sums rows t, t + 256, ... of every column in row order, then a
// fixed tree over the 256 partials per column halves them 8 times: a fixed order, no serial chain over all rows.  Thread
// j < 37 then owns output float j: view matrix 0..15, projection matrix 16..31, camera centre 32..34, tan_fov 35..36.
constexpr int CAM_REDUCE_THREADS = 256;
__global__ void __launch_bounds__(CAM_REDUCE_THREADS) camera_grad_reduce_kernel(CamReduceArgs a)
{
	__shared__ float part[CAM_ALL_TERMS][CAM_REDUCE_THREADS];
	const CamReduceView& w = a.view[blockIdx.x];
	const int t = threadIdx.x;
	float acc[CAM_ALL_TERMS];
#pragma unroll
	for (int k = 0; k < CAM_ALL_TERMS; k++) acc[k] = 0.f;
	for (int r = t; r < w.nrows; r += CAM_REDUCE_THREADS) {
		const float* row = w.rows + (size_t)r * CAM_TERMS;
#pragma unroll
		for (int k = 0; k < CAM_TERMS; k++) acc[k] += row[k];
		if (w.intr_rows) {
#pragma unroll
			for (int k = 0; k < CAM_INTR_TERMS; k++) acc[CAM_TERMS + k] += w.intr_rows[(size_t)r * CAM_INTR_TERMS + k];
		}
	}
#pragma unroll
	for (int k = 0; k < CAM_ALL_TERMS; k++) part[k][t] = acc[k];
	__syncthreads();
	for (int h = CAM_REDUCE_THREADS / 2; h > 0; h >>= 1) {
		for (int j = t; j < CAM_ALL_TERMS * h; j += CAM_REDUCE_THREADS) {
			const int k = j / h, i = j - k * h;
			part[k][i] += part[k][i + h];
		}
		__syncthreads();
	}
	const int j = t;
	float* o = nullptr;
	int k = -1;  // the row column, or -1 for an entry the forward never reads
	if (j < 16) {
		o = w.dL_dviewmatrix ? w.dL_dviewmatrix + j : nullptr;
		if ((j & 3) != 3) k = 3 * (j >> 2) + (j & 3);
	} else if (j < 32) {
		const int i = j - 16, r = i & 3;
		o = w.dL_dprojmatrix ? w.dL_dprojmatrix + i : nullptr;
		if (r != 2) k = 12 + 3 * (i >> 2) + (r == 3 ? 2 : r);
	} else if (j < 35) {
		o = w.dL_dcampos ? w.dL_dcampos + (j - 32) : nullptr;
		k = 24 + (j - 32);
	} else if (j < 37) {
		o = w.dL_dtan_fov ? w.dL_dtan_fov + (j - 35) : nullptr;
		k = 27 + (j - 35);
	}
	if (!o) return;
	const float s = k >= 0 ? part[k][0] : 0.f;
	*o = a.accumulate ? *o + s : s;
}

void launch_camera_grad_reduce(const CamReduceArgs& a, cudaStream_t s)
{
	if (a.V > 0) camera_grad_reduce_kernel<<<a.V, CAM_REDUCE_THREADS, 0, s>>>(a);
}

// ORTHO, FISH and DIST run at the blocks per SM of their CAM sibling, except where a bound below says otherwise
template <bool CAM, bool ORTHO, bool FISH = false, bool DIST = false>
static void project_bwd_views(const ProjectBwdViewsArgs& a, int grid, int deg, cudaStream_t s)
{
	if (a.antialias) {
		// 4 blocks per SM at degree <= 1: the compensation's registers do not fit the cap of 5 (96) without spilling
		// CAM at degree 2: 3 blocks per SM, the camera and focal-length terms spill at the cap of 4 (128)
		// DIST: 3 blocks per SM at degree <= 1 and 2 at degree 3, where the distortion's second derivatives spill at the caps
		if (deg <= 1) project_bwd_views_kernel<12, DIST ? 3 : 4, DIST, FISH, ORTHO, CAM, true><<<grid, 128, 0, s>>>(a);
		else if (deg == 2) project_bwd_views_kernel<27, CAM ? 3 : 4, DIST, FISH, ORTHO, CAM, true><<<grid, 128, 0, s>>>(a);
		else project_bwd_views_kernel<48, DIST ? 2 : 3, DIST, FISH, ORTHO, CAM, true><<<grid, 128, 0, s>>>(a);
		return;
	}
	// CAM at degree <= 1: 4 blocks per SM, as for AA; the camera terms spill at the cap of 5 (96 registers)
	// FISH at degree 2: 3 blocks per SM, the fisheye second derivatives spill at the cap of 4 (128 registers)
	// DIST at degree <= 1: 3 blocks per SM, the distortion's second derivatives spill at the cap of 4 (128 registers)
	if (deg <= 1) project_bwd_views_kernel<12, DIST ? 3 : CAM ? 4 : MGS_PBWD_MINB, DIST, FISH, ORTHO, CAM, false><<<grid, 128, 0, s>>>(a);
	else if (deg == 2) project_bwd_views_kernel<27, FISH ? 3 : 4, DIST, FISH, ORTHO, CAM, false><<<grid, 128, 0, s>>>(a);
	else project_bwd_views_kernel<48, 3, DIST, FISH, ORTHO, CAM, false><<<grid, 128, 0, s>>>(a);
}

// the PLN kernels at the blocks per SM of the DIST ones, except at degree 3 without AA: 2, the planar terms spill at the cap of
// 3 (168 registers)
static void launch_planar_views(const ProjectBwdViewsArgs& a, int grid, int deg, cudaStream_t s)
{
	if (a.antialias) {
		if (deg <= 1) project_bwd_views_planar_kernel<12, 3, true><<<grid, 128, 0, s>>>(a);
		else if (deg == 2) project_bwd_views_planar_kernel<27, 3, true><<<grid, 128, 0, s>>>(a);
		else project_bwd_views_planar_kernel<48, 2, true><<<grid, 128, 0, s>>>(a);
	} else {
		if (deg <= 1) project_bwd_views_planar_kernel<12, 3, false><<<grid, 128, 0, s>>>(a);
		else if (deg == 2) project_bwd_views_planar_kernel<27, 3, false><<<grid, 128, 0, s>>>(a);
		else project_bwd_views_planar_kernel<48, 2, false><<<grid, 128, 0, s>>>(a);
	}
}
static void launch_planar_clouds(const ProjectBwdCloudsDistArgs& a, int grid, int deg, cudaStream_t s)
{
	if (a.antialias) {
		if (deg <= 1) project_bwd_clouds_planar_kernel<12, 3, true><<<grid, 128, 0, s>>>(a);
		else if (deg == 2) project_bwd_clouds_planar_kernel<27, 3, true><<<grid, 128, 0, s>>>(a);
		else project_bwd_clouds_planar_kernel<48, 2, true><<<grid, 128, 0, s>>>(a);
	} else {
		if (deg <= 1) project_bwd_clouds_planar_kernel<12, 3, false><<<grid, 128, 0, s>>>(a);
		else if (deg == 2) project_bwd_clouds_planar_kernel<27, 3, false><<<grid, 128, 0, s>>>(a);
		else project_bwd_clouds_planar_kernel<48, 2, false><<<grid, 128, 0, s>>>(a);
	}
}

static bool planar_any(const float4* const* pl_g, int V)
{
	for (int u = 0; u < V; u++)
		if (pl_g[u]) return true;
	return false;
}

void launch_project_bwd_views(const ProjectBwdViewsArgs& a, cudaStream_t s)
{
	if (a.P <= 0 || a.V <= 0) return;
	const int grid = ceil_div(a.P, 128);
	const int deg = a.shs ? a.D : 0;
	bool cam = false;  // camera rows, or a device field of view, which only the CAM instantiation reads
	for (int u = 0; u < a.V; u++) cam |= a.cam_rows[u] != nullptr || a.intr[u].tan_fov != nullptr;
	if (planar_any(a.pl_g, a.V)) launch_planar_views(a, grid, deg, s);  // planar depth: the PLN kernels, all four models
	else if (a.distorted) project_bwd_views<true, true, true, true>(a, grid, deg, s);  // a distorted view: DIST, all four models
	else if (a.fisheye) project_bwd_views<true, true, true>(a, grid, deg, s);  // a fisheye view: the FISH instantiation, all models
	else if (a.ortho) project_bwd_views<true, true>(a, grid, deg, s);  // an orthographic view: the ORTHO instantiation of CAM
	else if (cam) project_bwd_views<true, false>(a, grid, deg, s);
	else project_bwd_views<false, false>(a, grid, deg, s);
}

template <bool CAM, bool ORTHO, bool FISH = false, bool DIST = false>
static void launch_clouds(const CloudsArgs<DIST>& a, int grid, int deg, cudaStream_t s)
{
	// 4 blocks per SM at degree <= 1: the register cap of 5 (96) spills here, and the launch is small where it matters most
	// (one CTA per 128 Gaussians of each cloud: 16k Gaussians fill one wave)
	if (a.antialias) {
		if (deg <= 1) project_bwd_clouds_kernel<12, DIST ? 3 : 4, DIST, FISH, ORTHO, CAM, true><<<grid, 128, 0, s>>>(a);  // as in the views launcher
		else if (deg == 2) project_bwd_clouds_kernel<27, CAM ? 3 : 4, DIST, FISH, ORTHO, CAM, true><<<grid, 128, 0, s>>>(a);  // as in the views launcher
		else project_bwd_clouds_kernel<48, DIST ? 2 : 3, DIST, FISH, ORTHO, CAM, true><<<grid, 128, 0, s>>>(a);
		return;
	}
	if (deg <= 1) project_bwd_clouds_kernel<12, DIST ? 3 : 4, DIST, FISH, ORTHO, CAM, false><<<grid, 128, 0, s>>>(a);  // as in the views launcher
	else if (deg == 2) project_bwd_clouds_kernel<27, FISH ? 3 : 4, DIST, FISH, ORTHO, CAM, false><<<grid, 128, 0, s>>>(a);  // as in the views launcher
	else project_bwd_clouds_kernel<48, 3, DIST, FISH, ORTHO, CAM, false><<<grid, 128, 0, s>>>(a);
}

void launch_project_bwd_clouds(ProjectBwdCloudsDistArgs a, cudaStream_t s)
{
	if (a.B <= 0) return;
	int grid = 0, V = 0;
	bool sh = false;
	for (int c = 0; c < a.B; c++) {
		a.cloud[c].block0 = grid;
		grid += ceil_div(a.cloud[c].P, 128);
		sh |= a.cloud[c].shs != nullptr;
		V = a.cloud[c].view0 + a.cloud[c].V;
	}
	const int deg = sh ? a.D : 0;
	bool cam = false;
	for (int u = 0; u < V; u++) cam |= a.cam_rows[u] != nullptr || a.intr[u].tan_fov != nullptr;
	if (planar_any(a.pl_g, V)) {
		launch_planar_clouds(a, grid, deg, s);
		return;
	}
	if (a.distorted) {
		launch_clouds<true, true, true, true>(a, grid, deg, s);
		return;
	}
	const ProjectBwdCloudsArgs& b = a;  // the parent's parameter block
	if (b.fisheye) launch_clouds<true, true, true>(b, grid, deg, s);
	else if (b.ortho) launch_clouds<true, true>(b, grid, deg, s);
	else if (cam) launch_clouds<true, false>(b, grid, deg, s);
	else launch_clouds<false, false>(b, grid, deg, s);
}

}  // namespace mgs
