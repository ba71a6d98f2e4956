// Quaternion helpers shared by the dynamic-field kernels (neighbour_reg.cu, deform.cu).  Quaternions are (r, x, y, z), real
// part first, as the rasterizer reads them; qmul and qrot are INTEGRATION.md section 17's formulas, and the normalisation
// and its backward follow torch's F.normalize (norm clamped at 1e-12).
#pragma once
#include <cuda_runtime.h>

namespace mgs {

constexpr float QUAT_EPS = 1e-12f;  // F.normalize's clamp of the norm

struct Quat { float r, x, y, z; };

__device__ __forceinline__ Quat qmul(const Quat& a, const Quat& b)  // Hamilton product (r, x, y, z), as INTEGRATION.md's qmul
{
	return {a.r * b.r - a.x * b.x - a.y * b.y - a.z * b.z, a.r * b.x + a.x * b.r + a.y * b.z - a.z * b.y,
	        a.r * b.y - a.x * b.z + a.y * b.r + a.z * b.x, a.r * b.z + a.x * b.y - a.y * b.x + a.z * b.r};
}
__device__ __forceinline__ Quat conj(const Quat& a) { return {a.r, -a.x, -a.y, -a.z}; }
__device__ __forceinline__ float qnorm(const float4& v) { return sqrtf(v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w); }
__device__ __forceinline__ Quat normalized(const float4& v, float n)  // F.normalize: v / max(|v|, 1e-12)
{
	const float d = fmaxf(n, QUAT_EPS);
	return {v.x / d, v.y / d, v.z / d, v.w / d};
}
// the backward of F.normalize: dL/dv from dL/dq, q = v / max(n, eps); the norm's gradient only where the clamp is not active
__device__ __forceinline__ float4 normalize_bwd(const float4& v, float n, const Quat& q, const Quat& g)
{
	if (n >= QUAT_EPS) {
		const float qg = q.r * g.r + q.x * g.x + q.y * g.y + q.z * g.z;
		return make_float4((g.r - q.r * qg) / n, (g.x - q.x * qg) / n, (g.y - q.y * qg) / n, (g.z - q.z * qg) / n);
	}
	return make_float4(g.r / QUAT_EPS, g.x / QUAT_EPS, g.y / QUAT_EPS, g.z / QUAT_EPS);
}
// the rows of qrot(q) (not renormalised), each with w = 0
__device__ __forceinline__ void qrot_rows(const Quat& q, float4 (&R)[3])
{
	const float r = q.r, x = q.x, y = q.y, z = q.z;
	R[0] = make_float4(1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y), 0.f);
	R[1] = make_float4(2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x), 0.f);
	R[2] = make_float4(2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y), 0.f);
}
// dL/dq from dL/dR = G through R = qrot(q): dL/dq_c = sum_ab G_ab dR_ab/dq_c
__device__ __forceinline__ Quat qrot_bwd(const Quat& q, const float (&G)[3][3])
{
	const float r = q.r, x = q.x, y = q.y, z = q.z;
	const float gr = 2.f * (-z * G[0][1] + y * G[0][2] + z * G[1][0] - x * G[1][2] - y * G[2][0] + x * G[2][1]);
	const float gx = 2.f * (y * G[0][1] + z * G[0][2] + y * G[1][0] - 2.f * x * G[1][1] - r * G[1][2] + z * G[2][0]
	                        + r * G[2][1] - 2.f * x * G[2][2]);
	const float gy = 2.f * (-2.f * y * G[0][0] + x * G[0][1] + r * G[0][2] + x * G[1][0] + z * G[1][2] - r * G[2][0]
	                        + z * G[2][1] - 2.f * y * G[2][2]);
	const float gz = 2.f * (-2.f * z * G[0][0] - r * G[0][1] + x * G[0][2] + r * G[1][0] - 2.f * z * G[1][1] + y * G[1][2]
	                        + x * G[2][0] + y * G[2][1]);
	return {gr, gx, gy, gz};
}
// scalar accesses: a [P,4] tensor need not start on a 16-byte boundary (a slice of a larger one)
__device__ __forceinline__ float4 ld4(const float* p) { return make_float4(p[0], p[1], p[2], p[3]); }
__device__ __forceinline__ void st4(float* p, const float4& v) { p[0] = v.x; p[1] = v.y; p[2] = v.z; p[3] = v.w; }

}  // namespace mgs
