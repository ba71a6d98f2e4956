// Shared definitions for the sm_90a Gaussian-splatting rasterizer kernels.
//
// Numerical contract: SURVEY.md Appendix A (restating DGR/cuda_rasterizer/{forward,backward}.cu,
// auxiliary.h, rasterizer_impl.cu of the reference).  Nothing here is copied from the reference;
// the per-Gaussian arithmetic is written so that nvcc's FMA contraction sees the same expression
// shapes as in the reference (left-to-right sums of products), which is what makes tile ids and
// sort keys bit-exact (checked on the GPU against oracle/_ref by tests/test_parity_gpu.py::test_vs_compiled_reference and tests/test_baseline_sizes_gpu.py).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace mgs {

constexpr int TILE_X = 16;          // reference config.h:17 (fixed: tile ids must match bit-exactly)
constexpr int TILE_Y = 16;          // reference config.h:18
constexpr int TILE_PIX = TILE_X * TILE_Y;
constexpr int WARP_BX = 8;          // a warp owns an 8x4 pixel block of its tile
constexpr int WARP_BY = 4;
constexpr float NEAR_Z = 0.2f;      // auxiliary.h:154
constexpr float ALPHA_MIN = 1.0f / 255.0f;  // forward.cu:354
constexpr float ALPHA_MAX = 0.99f;          // forward.cu:353
constexpr float T_STOP = 0.0001f;           // forward.cu:357

// Per-instance record, written in (tile, depth) order by the binning stage; a blend warp gathers the records of its
// block's work list by tile-list position (two 16-byte pieces each).  32 bytes.
struct __align__(16) InstRec {
	float x, y;        // pixel-space mean (geom means2D)
	float ca, cb;      // conic.x, conic.y
	float cc, op;      // conic.z, opacity
	uint32_t blocks;   // bit s: the alpha >= 1/255 footprint can reach 8x4 pixel block s of the instance's tile
	                   // (s = 2 * (y / 4) + x / 8).  Conservative; selects the block lists, never changes a pixel.
	uint32_t id;       // Gaussian index (== point_list entry)
};
static_assert(sizeof(InstRec) == 32, "InstRec must be 32 bytes");

// Blend-stage gradient record per Gaussian (atomically accumulated, then consumed by project_bwd).
// 12 floats = 3 x red.global.add.v4.f32.
constexpr int GB_STRIDE = 12;  // {dmx, dmy, dca, dcb | dcc, dop, dr, dg | db, ddepth, 0, 0}

// ---- small column-major 3x3 helpers (same summation order as glm: a0*b0 + a1*b1 + a2*b2) ----
struct V3 { float x, y, z; };
struct M3 {
	float m[3][3];  // m[col][row]
};
__device__ __forceinline__ M3 m3(float x0, float y0, float z0, float x1, float y1, float z1, float x2, float y2, float z2)
{
	M3 r;
	r.m[0][0] = x0; r.m[0][1] = y0; r.m[0][2] = z0;
	r.m[1][0] = x1; r.m[1][1] = y1; r.m[1][2] = z1;
	r.m[2][0] = x2; r.m[2][1] = y2; r.m[2][2] = z2;
	return r;
}
__device__ __forceinline__ M3 mul(const M3& a, const M3& b)
{
	M3 r;
#pragma unroll
	for (int j = 0; j < 3; j++)
#pragma unroll
		for (int i = 0; i < 3; i++)
			r.m[j][i] = a.m[0][i] * b.m[j][0] + a.m[1][i] * b.m[j][1] + a.m[2][i] * b.m[j][2];
	return r;
}
__device__ __forceinline__ M3 transpose(const M3& a)
{
	M3 r;
#pragma unroll
	for (int j = 0; j < 3; j++)
#pragma unroll
		for (int i = 0; i < 3; i++)
			r.m[j][i] = a.m[i][j];
	return r;
}
// Sigma = (S R)^T (S R) from scale and (un-normalised) quaternion; forward.cu:119-153 (project.cu, mcmc.cu)
__device__ __forceinline__ void cov3d_from_scale_rot(const float* scale, float mod, const float* rot, float* cov3D)
{
	M3 S = m3(mod * scale[0], 0.f, 0.f, 0.f, mod * scale[1], 0.f, 0.f, 0.f, mod * scale[2]);
	float r = rot[0], x = rot[1], y = rot[2], z = rot[3];
	M3 R = m3(
		1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y),
		2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x),
		2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y));
	M3 Mx = mul(S, R);
	M3 Sigma = mul(transpose(Mx), Mx);
	cov3D[0] = Sigma.m[0][0]; cov3D[1] = Sigma.m[0][1]; cov3D[2] = Sigma.m[0][2];
	cov3D[3] = Sigma.m[1][1]; cov3D[4] = Sigma.m[1][2]; cov3D[5] = Sigma.m[2][2];
}
__device__ __forceinline__ float dot(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

__device__ __forceinline__ V3 xform4x3(const V3& p, const float* m)
{
	V3 t = {
		m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12],
		m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
		m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14] };
	return t;
}
__device__ __forceinline__ float4 xform4x4(const V3& p, const float* m)
{
	float4 t = {
		m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12],
		m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
		m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14],
		m[3] * p.x + m[7] * p.y + m[11] * p.z + m[15] };
	return t;
}
// ((v + 1) * S - 1) / 2 evaluated in double like the reference's literals force (auxiliary.h:41-44)
__device__ __forceinline__ float ndc2pix(float v, int S) { return ((v + 1.0) * S - 1.0) * 0.5; }

__device__ __forceinline__ void tile_rect(float px, float py, int max_radius, uint2& rmin, uint2& rmax, uint32_t gx, uint32_t gy)
{
	rmin.x = min(gx, (uint32_t)max(0, (int)((px - max_radius) / TILE_X)));
	rmin.y = min(gy, (uint32_t)max(0, (int)((py - max_radius) / TILE_Y)));
	rmax.x = min(gx, (uint32_t)max(0, (int)((px + max_radius + TILE_X - 1) / TILE_X)));
	rmax.y = min(gy, (uint32_t)max(0, (int)((py + max_radius + TILE_Y - 1) / TILE_Y)));
}

// ------------------------------- PTX wrappers (sm_90+) -------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// 128-bit vector reduction to global memory (sm_90+): one L2 atomic transaction for 4 floats.
// 16-byte asynchronous copy global -> shared with a PER-LANE address (SASS LDGSTS), tracked by per-thread commit groups
__device__ __forceinline__ void cp_async16(void* dst_smem, const void* src_gmem)
{
	asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d)
{
	asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void red_add(float* addr, float a)
{
	asm volatile("red.global.add.f32 [%0], %1;" ::"l"(addr), "f"(a) : "memory");
}
// bring the line holding p into L1 (no register, nothing to wait for)
__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
__device__ __forceinline__ float4 ldg_nc_v4(const float4* p)
{
	float4 r;
	asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
	return r;
}

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// order-preserving unsigned keys of floats: a bounding box as atomicMin / atomicMax of keys (field.cu, knn.cu)
__device__ __forceinline__ uint32_t fkey(float f)
{
	const uint32_t b = __float_as_uint(f);
	return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float funkey(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

}  // namespace mgs
