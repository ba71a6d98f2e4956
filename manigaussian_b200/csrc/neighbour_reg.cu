// The neighbour regularisers of the dynamic field (include/mgs_rasterizer.h, mgs_neighbour_reg): local rigidity, rotation
// similarity and isometry between a cloud and its deformed next frame over fixed neighbour lists, forward and backward,
// without host reads.
//
// Forward (neighbour_reg_forward):
//   prologue  one thread per Gaussian: rel_i = normalize(rot_next_i) (x) conj(normalize(rot_i)) and R_i = qrot(rel_i); the
//             record {xyz, xyz_next, rel} that a pair gathers from its neighbour (three 16-byte pieces) and R_i (three rows);
//   pairs     one warp per Gaussian i, lane s = slot s < k: the three weighted terms of the slot, summed over the warp by a
//             shuffle butterfly and over the CTA's warps in warp order into one partial triple per CTA;
//   reduce    one CTA sums the partials in a fixed order (in double) and divides by P k, so the losses are bitwise identical
//             from call to call.
// Backward (neighbour_reg_backward), with the state the forward left for the same inputs:
//   zero      the padded [P,4] xyz, xyz_next and rel gradient rows of the state;
//   pairs     the same layout: each slot's gradients for its neighbour j go out as one red.global.add.v4.f32 per row; those
//             for Gaussian i (including dL/dR_i, chained to dL/drel_i in each lane) are summed over the warp by shuffles and
//             go out from lane 0 as one reduction per row;
//   epilogue  one thread per Gaussian: dL/drel through the Hamilton product and both normalisations to rot and rot_next, and
//             the xyz / xyz_next rows copied out, each only when its gradient is requested.
#include "../../include/mgs_rasterizer.h"
#include "mgs_common.cuh"
#include "mgs_kernels.h"
#include "quat.cuh"

namespace mgs {

constexpr int NR_WARPS = 8;        // Gaussians (warps) per pair-kernel CTA
constexpr int NR_REDUCE = 256;     // threads of the final reduce

static_assert(NEIGHBOUR_REG_MAX_K == 32, "one lane per slot");

// The state: [P] gather records (3 x float4: {x, y, z, xn.x}, {xn.y, xn.z, rel.r, rel.x}, {rel.y, rel.z, 0, 0}), [P] R
// rows (3 x float4, w unused), the pair kernel's CTA partials [ceil(P / NR_WARPS)][3], and the backward's gradient rows
// [P] x 3 float4 (xyz, xyz_next, rel), each piece aligned to 256 bytes.
struct NrState {
	float4* rec;
	float4* rmat;
	float* partial;
	float4* gx;
	float4* gxn;
	float4* grel;
	size_t end;
	static size_t align(size_t b) { return (b + 255) & ~size_t(255); }
	static NrState at(char* base, int P)
	{
		NrState s;
		size_t o = 0;
		const size_t p = (size_t)P;
		s.rec = reinterpret_cast<float4*>(base + o);     o += align(p * 3 * sizeof(float4));
		s.rmat = reinterpret_cast<float4*>(base + o);    o += align(p * 3 * sizeof(float4));
		s.partial = reinterpret_cast<float*>(base + o);  o += align((size_t)ceil_div(P, NR_WARPS) * 3 * sizeof(float));
		s.gx = reinterpret_cast<float4*>(base + o);      // gx, gxn, grel contiguous: one memset zeroes all three
		s.gxn = s.gx + p;
		s.grel = s.gx + 2 * p;
		o += align(p * 3 * sizeof(float4));
		s.end = o;
		return s;
	}
};

size_t neighbour_reg_state_bytes(int P) { return NrState::at(nullptr, P).end + 256; }

static char* align_state(void* state) { return reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(state) + 255) & ~uintptr_t(255)); }

__device__ __forceinline__ Quat rel_of(const float* rot, const float* rot_next, int i)
{
	const float4 a = ld4(rot + 4 * (size_t)i), b = ld4(rot_next + 4 * (size_t)i);
	return qmul(normalized(b, qnorm(b)), conj(normalized(a, qnorm(a))));
}

__global__ void __launch_bounds__(256) nr_prologue_kernel(int P, const float* __restrict__ xyz, const float* __restrict__ rot,
	const float* __restrict__ xyz_next, const float* __restrict__ rot_next, float4* __restrict__ rec, float4* __restrict__ rmat)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	const Quat q = rel_of(rot, rot_next, i);
	const float* p = xyz + 3 * (size_t)i;
	const float* n = xyz_next + 3 * (size_t)i;
	rec[3 * i + 0] = make_float4(p[0], p[1], p[2], n[0]);
	rec[3 * i + 1] = make_float4(n[1], n[2], q.r, q.x);
	rec[3 * i + 2] = make_float4(q.y, q.z, 0.f, 0.f);
	float4 R[3];  // INTEGRATION.md's qrot, rel not renormalised
	qrot_rows(q, R);
	rmat[3 * i + 0] = R[0];
	rmat[3 * i + 1] = R[1];
	rmat[3 * i + 2] = R[2];
}

// One slot's geometry: the offsets o = xyz_j - xyz_i, o' = xyz_next_j - xyz_next_i, d = o' - R_i o and v = rel_j - rel_i.
struct NrPair {
	float o[3], on[3], d[3], v[4];
};
__device__ __forceinline__ NrPair nr_pair(const float4 (&ri)[3], const float4 (&rj)[3], const float4 (&R)[3])
{
	NrPair s;
	s.o[0] = rj[0].x - ri[0].x; s.o[1] = rj[0].y - ri[0].y; s.o[2] = rj[0].z - ri[0].z;
	s.on[0] = rj[0].w - ri[0].w; s.on[1] = rj[1].x - ri[1].x; s.on[2] = rj[1].y - ri[1].y;
	s.d[0] = s.on[0] - (R[0].x * s.o[0] + R[0].y * s.o[1] + R[0].z * s.o[2]);
	s.d[1] = s.on[1] - (R[1].x * s.o[0] + R[1].y * s.o[1] + R[1].z * s.o[2]);
	s.d[2] = s.on[2] - (R[2].x * s.o[0] + R[2].y * s.o[1] + R[2].z * s.o[2]);
	s.v[0] = rj[1].z - ri[1].z; s.v[1] = rj[1].w - ri[1].w; s.v[2] = rj[2].x - ri[2].x; s.v[3] = rj[2].y - ri[2].y;
	return s;
}
__device__ __forceinline__ float norm3(const float* a) { return sqrtf(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]); }

// The slot (i, lane) of warp i: j, w and whether it is valid (0 <= j < P); nothing else is read for an invalid slot.
__device__ __forceinline__ bool nr_slot(int P, int k, int i, int lane, const long long* index, const float* weight, int& j, float& w)
{
	if (lane >= k) return false;
	const size_t e = (size_t)i * k + lane;
	const long long jj = index[e];
	if (jj < 0 || jj >= P) return false;
	j = (int)jj;
	w = weight[e];
	return true;
}

__device__ __forceinline__ void load3(const float4* p, float4 (&r)[3])
{
	r[0] = ldg_nc_v4(p); r[1] = ldg_nc_v4(p + 1); r[2] = ldg_nc_v4(p + 2);
}

__global__ void __launch_bounds__(32 * NR_WARPS) nr_fwd_pairs_kernel(int P, int k, const long long* __restrict__ index,
	const float* __restrict__ weight, const float4* __restrict__ rec, const float4* __restrict__ rmat, float* __restrict__ partial)
{
	__shared__ float part[NR_WARPS][3];
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const int i = blockIdx.x * NR_WARPS + warp;
	float t[3] = {0.f, 0.f, 0.f};
	int j;
	float w;
	if (i < P && nr_slot(P, k, i, lane, index, weight, j, w)) {
		float4 ri[3], rj[3], R[3];
		load3(rec + 3 * i, ri);
		load3(rmat + 3 * i, R);
		load3(rec + 3 * (size_t)j, rj);
		const NrPair s = nr_pair(ri, rj, R);
		t[0] = w * norm3(s.d);
		t[1] = w * sqrtf(s.v[0] * s.v[0] + s.v[1] * s.v[1] + s.v[2] * s.v[2] + s.v[3] * s.v[3]);
		t[2] = w * fabsf(norm3(s.on) - norm3(s.o));
	}
#pragma unroll
	for (int m = 16; m > 0; m >>= 1)
#pragma unroll
		for (int c = 0; c < 3; c++) t[c] += __shfl_xor_sync(0xffffffffu, t[c], m);
	if (lane == 0) { part[warp][0] = t[0]; part[warp][1] = t[1]; part[warp][2] = t[2]; }
	__syncthreads();
	if (threadIdx.x < 3) {
		float acc = 0.f;
#pragma unroll
		for (int q = 0; q < NR_WARPS; q++) acc += part[q][threadIdx.x];
		partial[3 * blockIdx.x + threadIdx.x] = acc;
	}
}

__global__ void __launch_bounds__(NR_REDUCE) nr_reduce_kernel(int P, int k, int nparts, const float* __restrict__ partial,
	float* __restrict__ out)
{
	__shared__ double red[NR_REDUCE][3];
	double a[3] = {0.0, 0.0, 0.0};
	for (int c = threadIdx.x; c < nparts; c += NR_REDUCE)
#pragma unroll
		for (int q = 0; q < 3; q++) a[q] += partial[3 * c + q];
#pragma unroll
	for (int q = 0; q < 3; q++) red[threadIdx.x][q] = a[q];
	__syncthreads();
	for (int h = NR_REDUCE / 2; h > 0; h >>= 1) {
		if (threadIdx.x < h)
#pragma unroll
			for (int q = 0; q < 3; q++) red[threadIdx.x][q] += red[threadIdx.x + h][q];
		__syncthreads();
	}
	if (threadIdx.x < 3) out[threadIdx.x] = P > 0 ? (float)(red[0][threadIdx.x] / ((double)P * k)) : 0.f;
}

// Each lane's slot: the gradients for its neighbour j (scattered) and its share of Gaussian i's (summed over the warp).
// need: bit 0 the xyz rows, bit 1 the xyz_next rows, bit 2 the rel rows.
__global__ void __launch_bounds__(32 * NR_WARPS) nr_bwd_pairs_kernel(int P, int k, int need, const long long* __restrict__ index,
	const float* __restrict__ weight, const float4* __restrict__ rec, const float4* __restrict__ rmat,
	const float* __restrict__ dL_dloss, float4* __restrict__ gx, float4* __restrict__ gxn, float4* __restrict__ grel)
{
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const int i = blockIdx.x * NR_WARPS + warp;
	if (i >= P) return;  // whole warps: i is uniform over the warp
	// Gaussian i's share: dL/dxyz_i [0..2], dL/dxyz_next_i [3..5], dL/drel_i [6..9]
	float gi[10];
#pragma unroll
	for (int c = 0; c < 10; c++) gi[c] = 0.f;
	int j;
	float w;
	if (nr_slot(P, k, i, lane, index, weight, j, w)) {
		float4 ri[3], rj[3], R[3];
		load3(rec + 3 * i, ri);
		load3(rmat + 3 * i, R);
		load3(rec + 3 * (size_t)j, rj);
		const NrPair s = nr_pair(ri, rj, R);
		const float scale = 1.f / ((float)P * (float)k);
		const float cr = dL_dloss[0] * scale * w, ct = dL_dloss[1] * scale * w, ci = dL_dloss[2] * scale * w;
		// rigid: u = dL/dd; d/do' = u, d/do = -R^T u, d/dR = -u o^T
		const float nd = norm3(s.d);
		const float fu = nd > 0.f ? cr / nd : 0.f;
		const float u[3] = {fu * s.d[0], fu * s.d[1], fu * s.d[2]};
		// isometry: sg = dL/da, a = |o'| - |o|; d|o'|/do' = o'/|o'|, d|o|/do = o/|o| (0 at 0)
		const float non = norm3(s.on), no = norm3(s.o);
		const float iso = non - no;
		const float sg = iso > 0.f ? ci : (iso < 0.f ? -ci : 0.f);
		const float fn = non > 0.f ? sg / non : 0.f, fo = no > 0.f ? sg / no : 0.f;
		float dxn[3], dx[3];
		dxn[0] = u[0] + fn * s.on[0];
		dxn[1] = u[1] + fn * s.on[1];
		dxn[2] = u[2] + fn * s.on[2];
		dx[0] = -(R[0].x * u[0] + R[1].x * u[1] + R[2].x * u[2]) - fo * s.o[0];
		dx[1] = -(R[0].y * u[0] + R[1].y * u[1] + R[2].y * u[2]) - fo * s.o[1];
		dx[2] = -(R[0].z * u[0] + R[1].z * u[1] + R[2].z * u[2]) - fo * s.o[2];
		// rotation: e = dL/dv
		const float nv = sqrtf(s.v[0] * s.v[0] + s.v[1] * s.v[1] + s.v[2] * s.v[2] + s.v[3] * s.v[3]);
		const float fe = nv > 0.f ? ct / nv : 0.f;
		const float e[4] = {fe * s.v[0], fe * s.v[1], fe * s.v[2], fe * s.v[3]};
		if (need & 1) red_add_v4(reinterpret_cast<float*>(gx + j), dx[0], dx[1], dx[2], 0.f);
		if (need & 2) red_add_v4(reinterpret_cast<float*>(gxn + j), dxn[0], dxn[1], dxn[2], 0.f);
		if (need & 4) red_add_v4(reinterpret_cast<float*>(grel + j), e[0], e[1], e[2], e[3]);
		// dL/dR_i = -u o^T, chained to rel_i = (r, x, y, z) through qrot: dL/drel_c = sum_ab G_ab dR_ab/drel_c
		float G[3][3];
#pragma unroll
		for (int aa = 0; aa < 3; aa++)
#pragma unroll
			for (int b = 0; b < 3; b++) G[aa][b] = -u[aa] * s.o[b];
		const Quat gq = qrot_bwd({ri[1].z, ri[1].w, ri[2].x, ri[2].y}, G);
		gi[0] = -dx[0]; gi[1] = -dx[1]; gi[2] = -dx[2];
		gi[3] = -dxn[0]; gi[4] = -dxn[1]; gi[5] = -dxn[2];
		gi[6] = gq.r - e[0]; gi[7] = gq.x - e[1]; gi[8] = gq.y - e[2]; gi[9] = gq.z - e[3];
	}
#pragma unroll
	for (int m = 16; m > 0; m >>= 1)
#pragma unroll
		for (int c = 0; c < 10; c++) gi[c] += __shfl_xor_sync(0xffffffffu, gi[c], m);
	if (lane == 0) {
		if (need & 1) red_add_v4(reinterpret_cast<float*>(gx + i), gi[0], gi[1], gi[2], 0.f);
		if (need & 2) red_add_v4(reinterpret_cast<float*>(gxn + i), gi[3], gi[4], gi[5], 0.f);
		if (need & 4) red_add_v4(reinterpret_cast<float*>(grel + i), gi[6], gi[7], gi[8], gi[9]);
	}
}

__global__ void __launch_bounds__(256) nr_epilogue_kernel(int P, const float* __restrict__ rot, const float* __restrict__ rot_next,
	const float4* __restrict__ gx, const float4* __restrict__ gxn, const float4* __restrict__ grel, float* __restrict__ dL_dxyz,
	float* __restrict__ dL_drot, float* __restrict__ dL_dxyz_next, float* __restrict__ dL_drot_next)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	if (dL_dxyz) {
		const float4 g = gx[i];
		dL_dxyz[3 * (size_t)i] = g.x; dL_dxyz[3 * (size_t)i + 1] = g.y; dL_dxyz[3 * (size_t)i + 2] = g.z;
	}
	if (dL_dxyz_next) {
		const float4 g = gxn[i];
		dL_dxyz_next[3 * (size_t)i] = g.x; dL_dxyz_next[3 * (size_t)i + 1] = g.y; dL_dxyz_next[3 * (size_t)i + 2] = g.z;
	}
	if (!dL_drot && !dL_drot_next) return;
	// rel = qn (x) p with p = conj(q): dL/dqn = g (x) conj(p) = g (x) q, dL/dp = conj(qn) (x) g, dL/dq = conj(dL/dp)
	const float4 gv = grel[i];
	const Quat g = {gv.x, gv.y, gv.z, gv.w};
	const float4 a = ld4(rot + 4 * (size_t)i), b = ld4(rot_next + 4 * (size_t)i);
	const float na = qnorm(a), nb = qnorm(b);
	const Quat q = normalized(a, na), qn = normalized(b, nb);
	if (dL_drot_next) st4(dL_drot_next + 4 * (size_t)i, normalize_bwd(b, nb, qn, qmul(g, q)));
	if (dL_drot) st4(dL_drot + 4 * (size_t)i, normalize_bwd(a, na, q, conj(qmul(conj(qn), g))));
}

cudaError_t neighbour_reg_forward(void* state, int P, int k, const float* xyz, const float* rot, const float* xyz_next,
	const float* rot_next, const long long* index, const float* weight, float* out_loss, cudaStream_t st)
{
	const NrState s = NrState::at(align_state(state), P);
	const int nparts = ceil_div(P, NR_WARPS);
	if (P > 0) {
		nr_prologue_kernel<<<ceil_div(P, 256), 256, 0, st>>>(P, xyz, rot, xyz_next, rot_next, s.rec, s.rmat);
		nr_fwd_pairs_kernel<<<nparts, 32 * NR_WARPS, 0, st>>>(P, k, index, weight, s.rec, s.rmat, s.partial);
	}
	nr_reduce_kernel<<<1, NR_REDUCE, 0, st>>>(P, k, nparts, s.partial, out_loss);
	return cudaGetLastError();
}

cudaError_t neighbour_reg_backward(void* state, int P, int k, const float* rot, const float* rot_next, const long long* index,
	const float* weight, const float* dL_dloss, float* dL_dxyz, float* dL_drot, float* dL_dxyz_next, float* dL_drot_next,
	cudaStream_t st)
{
	const NrState s = NrState::at(align_state(state), P);
	const int need = (dL_dxyz ? 1 : 0) | (dL_dxyz_next ? 2 : 0) | ((dL_drot || dL_drot_next) ? 4 : 0);
	if (!need) return cudaSuccess;
	cudaError_t e = cudaMemsetAsync(s.gx, 0, (size_t)P * 3 * sizeof(float4), st);
	if (e != cudaSuccess) return e;
	nr_bwd_pairs_kernel<<<ceil_div(P, NR_WARPS), 32 * NR_WARPS, 0, st>>>(P, k, need, index, weight, s.rec, s.rmat, dL_dloss, s.gx,
	                                                                     s.gxn, s.grel);
	nr_epilogue_kernel<<<ceil_div(P, 256), 256, 0, st>>>(P, rot, rot_next, s.gx, s.gxn, s.grel, dL_dxyz, dL_drot, dL_dxyz_next,
	                                                     dL_drot_next);
	return cudaGetLastError();
}

}  // namespace mgs
