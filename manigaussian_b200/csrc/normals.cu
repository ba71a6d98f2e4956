// Per-Gaussian surface normals (include/mgs_rasterizer.h, mgs_view_normal): the shortest axis of each Gaussian in world
// space, turned to face the camera, as the quad {nx, ny, nz, 0} the blend kernels carry in columns 4..6 of the
// {r,g,b,depth} tile; and the chain from the blend stage's dL/dn back to the quaternions.
//
// Kernels of their own rather than a mode of the projection kernels: those compile to pinned instruction sequences (tile
// ids and sort keys depend on them, DESIGN.md section 4), and nothing here needs anything the projection computes.
#include "mgs_common.cuh"
#include "mgs_kernels.h"

namespace mgs {

// k = argmin_j scale[j], the lowest index on ties
__device__ __forceinline__ int shortest_axis(const float* s)
{
	int k = 0;
	if (s[1] < s[0]) k = 1;
	if (s[2] < s[k]) k = 2;
	return k;
}

// the unit quaternion q / |q| (r, x, y, z) and 1 / |q|
__device__ __forceinline__ float unit_quat(const float* rot, float (&q)[4])
{
	const float inv = rsqrtf(rot[0] * rot[0] + rot[1] * rot[1] + rot[2] * rot[2] + rot[3] * rot[3]);
#pragma unroll
	for (int i = 0; i < 4; i++) q[i] = rot[i] * inv;
	return inv;
}

// a = R(q) e_k for a unit q: the world-space direction of the axis that scale k stretches (Sigma a = s_k^2 a for the
// covariance cov3d_from_scale_rot builds, project.cu)
__device__ __forceinline__ V3 axis_of(const float (&q)[4], int k)
{
	const float r = q[0], x = q[1], y = q[2], z = q[3];
	if (k == 0) return V3{ 1.f - 2.f * (y * y + z * z), 2.f * (x * y + r * z), 2.f * (x * z - r * y) };
	if (k == 1) return V3{ 2.f * (x * y - r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z + r * x) };
	return V3{ 2.f * (x * z + r * y), 2.f * (y * z - r * x), 1.f - 2.f * (x * x + y * y) };
}

// +1 where the axis faces the camera (a . (campos - mean) >= 0), else -1
__device__ __forceinline__ float facing(const V3& a, const float* mean, const float* cam)
{
	const float d = a.x * (cam[0] - mean[0]) + a.y * (cam[1] - mean[1]) + a.z * (cam[2] - mean[2]);
	return d >= 0.f ? 1.f : -1.f;
}

__global__ void __launch_bounds__(256) normals_fwd_kernel(int P, const float* __restrict__ means3D, const float* __restrict__ scales,
	const float* __restrict__ rotations, const float* __restrict__ cam_pos, float4* __restrict__ nrm)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	float q[4];
	unit_quat(rotations + 4 * i, q);
	const V3 a = axis_of(q, shortest_axis(scales + 3 * i));
	const float s = facing(a, means3D + 3 * i, cam_pos);
	nrm[i] = make_float4(s * a.x, s * a.y, s * a.z, 0.f);
}

// dL/da = sum over the views of s_v gn_v (in view order, in registers: no atomics), then through column k of R(q^) and
// the normalisation q^ = q / |q| (Jacobian (I - q^ q^T) / |q|), ADDED to dL_drot: the per-Gaussian stage has written its
// own rotation gradient there by now.
__global__ void __launch_bounds__(256) normals_bwd_kernel(NormalsBwdArgs a)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= a.P) return;
	float q[4];
	const float inv = unit_quat(a.rotations + 4 * i, q);
	const int k = shortest_axis(a.scales + 3 * i);
	const V3 ax = axis_of(q, k);
	const float* mean = a.means3D + 3 * i;
	float gx = 0.f, gy = 0.f, gz = 0.f;
	for (int v = 0; v < a.V; v++) {
		const float4 g = reinterpret_cast<const float4*>(a.gn[v])[i];
		const float s = facing(ax, mean, a.cam_pos[v]);
		gx += s * g.x; gy += s * g.y; gz += s * g.z;
	}
	const float r = q[0], x = q[1], y = q[2], z = q[3];
	float d[4];  // dL/dq^
	if (k == 0) {
		d[0] = 2.f * (z * gy - y * gz);
		d[1] = 2.f * (y * gy + z * gz);
		d[2] = -4.f * y * gx + 2.f * (x * gy - r * gz);
		d[3] = -4.f * z * gx + 2.f * (r * gy + x * gz);
	} else if (k == 1) {
		d[0] = 2.f * (x * gz - z * gx);
		d[1] = -4.f * x * gy + 2.f * (y * gx + r * gz);
		d[2] = 2.f * (x * gx + z * gz);
		d[3] = -4.f * z * gy + 2.f * (y * gz - r * gx);
	} else {
		d[0] = 2.f * (y * gx - x * gy);
		d[1] = -4.f * x * gz + 2.f * (z * gx - r * gy);
		d[2] = -4.f * y * gz + 2.f * (r * gx + z * gy);
		d[3] = 2.f * (x * gx + y * gy);
	}
	const float qd = q[0] * d[0] + q[1] * d[1] + q[2] * d[2] + q[3] * d[3];
	float* out = a.dL_drot + 4 * (size_t)i;  // a caller's row need not be 16-byte aligned
#pragma unroll
	for (int c = 0; c < 4; c++) out[c] += (d[c] - q[c] * qd) * inv;
}

void launch_normals_fwd(int P, const float* means3D, const float* scales, const float* rotations, const float* cam_pos, float4* nrm,
	cudaStream_t s)
{
	if (P > 0) normals_fwd_kernel<<<ceil_div(P, 256), 256, 0, s>>>(P, means3D, scales, rotations, cam_pos, nrm);
}

void launch_normals_bwd(const NormalsBwdArgs& a, cudaStream_t s)
{
	if (a.P > 0 && a.V > 0) normals_bwd_kernel<<<ceil_div(a.P, 256), 256, 0, s>>>(a);
}

}  // namespace mgs
