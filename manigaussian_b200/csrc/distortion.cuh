// OpenCV distorted-pinhole views (include/mgs_rasterizer.h, mgs_view_distortion): the map of the normalised coordinates
// (x, y) = (t.x / t.z, t.y / t.z) to the distorted ones (xd, yd), its Jacobian Dd = d(xd, yd) / d(x, y) and, on request,
// Dd's derivatives, shared by the forward (project.cu) and the backward (project_bwd.cu).
//
// With r2 = x^2 + y^2, R = N / Q, N = 1 + k1 r2 + k2 r2^2 + k3 r2^3, Q = 1 + k4 r2 + k5 r2^2 + k6 r2^3, and
// R1 = dR / dr2 = (N' - R Q') / Q, R2 = d^2R / dr2^2 = (N'' - 2 R1 Q' - R Q'') / Q:
//   xd = x R + 2 p1 x y + p2 (r2 + 2 x^2),   yd = y R + p1 (r2 + 2 y^2) + 2 p2 x y
//   Dd = [[R + 2 x^2 R1 + 2 p1 y + 6 p2 x, 2 x y R1 + 2 p1 x + 2 p2 y], [same, R + 2 y^2 R1 + 6 p1 y + 2 p2 x]]  (symmetric)
// Dd's derivatives have four distinct entries (the third derivatives of a map with symmetric Jacobian):
//   hxxx = dD00/dx,  hxxy = dD00/dy = dD01/dx,  hxyy = dD01/dy = dD11/dx,  hyyy = dD11/dy
// The map is a rational polynomial in x and y: no branch, no cancellation near the axis.
#pragma once

namespace mgs {

struct DistK {
	float k1, k2, p1, p2, k3, k4, k5, k6;  // OpenCV's order of the 8-coefficient D
};

struct DistTerms {
	float r2;
	float xd, yd;                    // the distorted normalised coordinates
	float d00, d01, d11;             // Dd (d10 = d01)
	float hxxx, hxxy, hxyy, hyyy;    // Dd's derivatives (SECOND only)
};

template <bool SECOND>
__device__ __forceinline__ DistTerms distortion_terms(float x, float y, const DistK& k)
{
	DistTerms o;
	const float xx = x * x, yy = y * y, xy = x * y, r2 = xx + yy;
	const float N = 1.0f + r2 * (k.k1 + r2 * (k.k2 + r2 * k.k3));
	const float Q = 1.0f + r2 * (k.k4 + r2 * (k.k5 + r2 * k.k6));
	const float N1 = k.k1 + r2 * (2.0f * k.k2 + r2 * (3.0f * k.k3));
	const float Q1 = k.k4 + r2 * (2.0f * k.k5 + r2 * (3.0f * k.k6));
	const float iQ = 1.0f / Q;
	const float R = N * iQ;
	const float R1 = (N1 - R * Q1) * iQ;
	o.r2 = r2;
	o.xd = x * R + 2.0f * k.p1 * xy + k.p2 * (r2 + 2.0f * xx);
	o.yd = y * R + k.p1 * (r2 + 2.0f * yy) + 2.0f * k.p2 * xy;
	o.d00 = R + 2.0f * xx * R1 + 2.0f * k.p1 * y + 6.0f * k.p2 * x;
	o.d01 = 2.0f * xy * R1 + 2.0f * k.p1 * x + 2.0f * k.p2 * y;
	o.d11 = R + 2.0f * yy * R1 + 6.0f * k.p1 * y + 2.0f * k.p2 * x;
	o.hxxx = o.hxxy = o.hxyy = o.hyyy = 0.f;
	if constexpr (SECOND) {
		const float N2 = 2.0f * k.k2 + 6.0f * k.k3 * r2, Q2 = 2.0f * k.k5 + 6.0f * k.k6 * r2;
		const float R2 = (N2 - 2.0f * R1 * Q1 - R * Q2) * iQ;
		o.hxxx = x * (6.0f * R1 + 4.0f * xx * R2) + 6.0f * k.p2;
		o.hxxy = y * (2.0f * R1 + 4.0f * xx * R2) + 2.0f * k.p1;
		o.hxyy = x * (2.0f * R1 + 4.0f * yy * R2) + 2.0f * k.p2;
		o.hyyy = y * (6.0f * R1 + 4.0f * yy * R2) + 6.0f * k.p1;
	}
	return o;
}

}  // namespace mgs
