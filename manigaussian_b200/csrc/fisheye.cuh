// Kannala-Brandt fisheye views (include/mgs_rasterizer.h, mgs_view_fisheye): the radial terms of the screen mean
// (u, v) = (fx a x + cx, fy a y + cy), a = theta_d / r, and of its Jacobian and second derivatives, shared by the forward
// (project.cu) and the backward (project_bwd.cu).
//
// With r = |(x, y)|, s = r^2 + z^2, theta = atan2(r, z), theta_d = theta rho(theta), D1 = d theta_d / d theta:
//   da/dx = c x, da/dy = c y, da/dz = -g,   c = (b - a) / r^2, b = D1 z / s,   g = D1 / s
//   J = [[fx (a + c x^2), fx c x y, -fx x g], [fy c x y, fy (a + c y^2), -fy y g]]
// The backward also needs C1 = (dc/dr) / r, cz = dc/dz, gz = dg/dz; (dg/dr) / r = -cz.
//
// c and C1 cancel catastrophically as r / z -> 0 (b - a = O(r^2 / z^3)): evaluated as written, their fp32 relative errors
// grow as u / e^2 and u / e^4 (e = r / z), and their share of dL/dt as u / e.  Below FISHEYE_SERIES_E2 (e < 1/8) they
// come from their Taylor series in e^2, truncated where the next term's share of dL/dt is O(e^7): the two errors meet
// near e = u^(1/8) = 0.125 (tests/fisheye_ref64.py bounds both branches; tests/test_fisheye_cpu.py checks continuity).
#pragma once

namespace mgs {

struct FisheyeK {
	float k1, k2, k3, k4;
};

constexpr float FISHEYE_SERIES_E2 = 1.0f / 64.0f;

struct FisheyeRadial {
	float theta;      // atan2(r, z)
	float a, c, g;    // the Jacobian's radial terms
	float C1, cz, gz; // second derivatives (SECOND only)
};

template <bool SECOND>
__device__ __forceinline__ FisheyeRadial fisheye_radial(float x, float y, float z, const FisheyeK& k)
{
	FisheyeRadial o;
	const float r2 = x * x + y * y, r = sqrtf(r2), s = r2 + z * z, is = 1.0f / s, iz = 1.0f / z;
	const float th = atan2f(r, z), t2 = th * th;
	const float rho = 1.0f + t2 * (k.k1 + t2 * (k.k2 + t2 * (k.k3 + t2 * k.k4)));                            // theta_d / theta
	const float D1 = 1.0f + t2 * (3.0f * k.k1 + t2 * (5.0f * k.k2 + t2 * (7.0f * k.k3 + t2 * (9.0f * k.k4)))); // d theta_d / d theta
	const float e2 = r2 * iz * iz;
	const bool series = e2 < FISHEYE_SERIES_E2;
	// q = theta / r; the series also covers r = 0, where q = 1 / z
	const float q = series ? iz * (1.0f + e2 * (-1.0f / 3.0f + e2 * (0.2f + e2 * (-1.0f / 7.0f)))) : th / r;
	o.theta = th;
	o.a = q * rho;
	o.g = D1 * is;
	// c z^3 = c0 + c1 e^2 + c2 e^4 + O(e^6)
	const float c0 = 2.0f * k.k1 - 2.0f / 3.0f;
	const float c1 = 4.0f * (k.k2 - k.k1) + 0.8f;
	const float c2 = 5.6f * k.k1 - 10.0f * k.k2 + 6.0f * k.k3 - 6.0f / 7.0f;
	const float iz3 = iz * iz * iz;
	o.c = series ? iz3 * (c0 + e2 * (c1 + e2 * c2)) : (D1 * z * is - o.a) / r2;
	o.C1 = o.cz = o.gz = 0.f;
	if constexpr (SECOND) {
		const float D2r = q * (6.0f * k.k1 + t2 * (20.0f * k.k2 + t2 * (42.0f * k.k3 + t2 * (72.0f * k.k4))));  // D2 / r
		const float is2 = is * is;
		o.C1 = series ? iz3 * iz * iz * (2.0f * c1 + 4.0f * c2 * e2) : ((D2r * z * z - 2.0f * z * D1) * is2 - 3.0f * o.c) / r2;
		o.cz = (2.0f * D1 - D2r * z) * is2;
		o.gz = -(D2r * r2 + 2.0f * z * D1) * is2;
	}
	return o;
}

}  // namespace mgs
