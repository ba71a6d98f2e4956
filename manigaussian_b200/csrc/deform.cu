// Deformation of a cloud by a sparse control graph (include/mgs_rasterizer.h, mgs_deform): each Gaussian blends the rigid
// motions of the nodes its index row names, forward and backward, without host reads.
//
// Forward (deform_forward):
//   node      one thread per node j: q^_j = normalize(node_rot_j), negated where its real part is below 0, R_j = qrot(q^_j)
//             and c_j = node_xyz_j + node_t_j - R_j node_xyz_j, written as the record {R_j row 0, c_j.x}, {row 1, c_j.y},
//             {row 2, c_j.z}, q^_j (four float4);
//   gaussian  L lanes per Gaussian, lane s taking slots s, s + L, ...: the weighted moves w (R_j x + c_j - x) and quaternion
//             offsets w (q^_j - e) of its slots, summed over the Gaussian's lanes by a shuffle butterfly; lane 0 writes xyz',
//             rot' = normalize(r) (x) rot and r into the state.  No atomics: the outputs are bitwise identical from call to call.
// Backward (deform_backward), with the state the forward left for the same inputs:
//   zero      the [N] x 4 float4 node accumulators;
//   gaussian  the same layout: dL/dweight of each slot, and dL/dxyz and dL/drot from lane 0, written directly (each Gaussian
//             owns its rows); each slot's 16 node terms {w g x^T | w g} and w dL/dr are summed over the lanes of the warp
//             that name the same node (__match_any_sync and a pointer-jumping sum), and one leader per node sends them as four
//             red.global.add.v4.f32;
//   node      one thread per node: the chain rule through c, qrot, the sign and F.normalize, written only where asked for.
#include "../../include/mgs_rasterizer.h"
#include "mgs_common.cuh"
#include "mgs_kernels.h"
#include "quat.cuh"

namespace mgs {

// Lanes per Gaussian: the power of two >= k, at most MGS_DEFORM_LANES; lane s takes slots s, s + L, ...  At most 4 was
// measured fastest at k = 8 (DESIGN.md section 4).
#ifndef MGS_DEFORM_LANES
#define MGS_DEFORM_LANES 4
#endif
static_assert(MGS_DEFORM_LANES >= 1 && MGS_DEFORM_LANES <= 32 && (MGS_DEFORM_LANES & (MGS_DEFORM_LANES - 1)) == 0,
              "lanes per Gaussian: a power of two, at most a warp");
static_assert(DEFORM_MAX_K == 32, "k fits one warp");

constexpr int DF_THREADS = 256;  // threads per CTA of every deform kernel

// The state: the node records [N] x 4 float4, the backward's node accumulators [N] x 4 float4 and each Gaussian's
// unnormalised blend r_i [P] float4, each piece aligned to 256 bytes.
struct DfState {
	float4* rec;
	float4* acc;
	float4* r;
	size_t end;
	static size_t align(size_t b) { return (b + 255) & ~size_t(255); }
	static DfState at(char* base, int P, int N)
	{
		DfState s;
		size_t o = 0;
		s.rec = reinterpret_cast<float4*>(base + o);  o += align((size_t)N * 4 * sizeof(float4));
		s.acc = reinterpret_cast<float4*>(base + o);  o += align((size_t)N * 4 * sizeof(float4));
		s.r = reinterpret_cast<float4*>(base + o);    o += align((size_t)P * sizeof(float4));
		s.end = o;
		return s;
	}
};

size_t deform_state_bytes(int P, int N) { return DfState::at(nullptr, P, N).end + 256; }

static char* align_state(void* state) { return reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(state) + 255) & ~uintptr_t(255)); }

static int lane_shift(int k)
{
	int s = 0;
	while ((1 << s) < k && (1 << s) < MGS_DEFORM_LANES) s++;
	return s;
}

// q^_j: F.normalize, then the sign that puts the real part at or above 0 (sgn = -1 where it was flipped)
__device__ __forceinline__ Quat node_quat(const float4& v, float n, float& sgn)
{
	const Quat q = normalized(v, n);
	sgn = q.r < 0.f ? -1.f : 1.f;
	return {sgn * q.r, sgn * q.x, sgn * q.y, sgn * q.z};
}

__global__ void __launch_bounds__(DF_THREADS) deform_node_fwd_kernel(int N, const float* __restrict__ node_xyz,
	const float* __restrict__ node_rot, const float* __restrict__ node_t, float4* __restrict__ rec)
{
	const int j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= N) return;
	const float4 v = ld4(node_rot + 4 * (size_t)j);
	float sgn;
	const Quat q = node_quat(v, qnorm(v), sgn);
	float4 R[3];
	qrot_rows(q, R);
	const float* p = node_xyz + 3 * (size_t)j;
	const float* t = node_t + 3 * (size_t)j;
	const float p0 = p[0], p1 = p[1], p2 = p[2];
	R[0].w = p0 + t[0] - (R[0].x * p0 + R[0].y * p1 + R[0].z * p2);
	R[1].w = p1 + t[1] - (R[1].x * p0 + R[1].y * p1 + R[1].z * p2);
	R[2].w = p2 + t[2] - (R[2].x * p0 + R[2].y * p1 + R[2].z * p2);
	rec[4 * (size_t)j + 0] = R[0];
	rec[4 * (size_t)j + 1] = R[1];
	rec[4 * (size_t)j + 2] = R[2];
	rec[4 * (size_t)j + 3] = make_float4(q.r, q.x, q.y, q.z);
}

// Slot s of Gaussian i: j and w when it is valid (0 <= j < N); nothing else is read for an invalid slot.
__device__ __forceinline__ bool df_slot(int N, int k, int i, int s, const long long* index, const float* weight, int& j, float& w)
{
	const size_t e = (size_t)i * k + s;
	const long long jj = index[e];
	if (jj < 0 || jj >= N) return false;
	j = (int)jj;
	w = weight[e];
	return true;
}

__device__ __forceinline__ void load_rec(const float4* rec, int j, float4 (&n)[4])
{
	const float4* p = rec + 4 * (size_t)j;
	n[0] = ldg_nc_v4(p); n[1] = ldg_nc_v4(p + 1); n[2] = ldg_nc_v4(p + 2); n[3] = ldg_nc_v4(p + 3);
}

// R_j x + c_j - x
__device__ __forceinline__ void node_move(const float4 (&n)[4], const float (&x)[3], float (&u)[3])
{
	u[0] = n[0].x * x[0] + n[0].y * x[1] + n[0].z * x[2] + n[0].w - x[0];
	u[1] = n[1].x * x[0] + n[1].y * x[1] + n[1].z * x[2] + n[1].w - x[1];
	u[2] = n[2].x * x[0] + n[2].y * x[1] + n[2].z * x[2] + n[2].w - x[2];
}

__global__ void __launch_bounds__(DF_THREADS) deform_fwd_kernel(int P, int N, int k, int lshift, const float* __restrict__ xyz,
	const float* __restrict__ rot, const long long* __restrict__ index, const float* __restrict__ weight,
	const float4* __restrict__ rec, float4* __restrict__ rstate, float* __restrict__ out_xyz, float* __restrict__ out_rot)
{
	const int L = 1 << lshift;
	const int sub = threadIdx.x & (L - 1);
	const int i = blockIdx.x * (DF_THREADS >> lshift) + (threadIdx.x >> lshift);
	const bool live = i < P;  // no early return: the butterfly below needs every lane of the warp
	float x[3] = {0.f, 0.f, 0.f};
	if (live) { x[0] = xyz[3 * (size_t)i]; x[1] = xyz[3 * (size_t)i + 1]; x[2] = xyz[3 * (size_t)i + 2]; }
	float a[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // sum w (R x + c - x) [0..2], sum w (q^ - e) [3..6]
	for (int s = sub; live && s < k; s += L) {
		int j;
		float w;
		if (!df_slot(N, k, i, s, index, weight, j, w)) continue;
		float4 n[4];
		load_rec(rec, j, n);
		float u[3];
		node_move(n, x, u);
		a[0] += w * u[0]; a[1] += w * u[1]; a[2] += w * u[2];
		a[3] += w * (n[3].x - 1.f); a[4] += w * n[3].y; a[5] += w * n[3].z; a[6] += w * n[3].w;
	}
	for (int m = L >> 1; m > 0; m >>= 1)
#pragma unroll
		for (int c = 0; c < 7; c++) a[c] += __shfl_xor_sync(0xffffffffu, a[c], m);
	if (!live || sub != 0) return;
	out_xyz[3 * (size_t)i] = x[0] + a[0];
	out_xyz[3 * (size_t)i + 1] = x[1] + a[1];
	out_xyz[3 * (size_t)i + 2] = x[2] + a[2];
	const float4 r = make_float4(1.f + a[3], a[4], a[5], a[6]);
	rstate[i] = r;
	const float4 p = ld4(rot + 4 * (size_t)i);
	const Quat o = qmul(normalized(r, qnorm(r)), {p.x, p.y, p.z, p.w});
	st4(out_rot + 4 * (size_t)i, make_float4(o.r, o.x, o.y, o.z));
}

// Sums v over the lanes of the warp with the same key and sends the sum to acc[4 key ..] from the lowest such lane (keys
// below 0 are never sent).  Every lane of the warp calls it.  Each lane links to the next lane of its group, and the sums
// follow the links by pointer jumping: ceil(log2(largest group)) rounds of 17 shuffles, none when every key is distinct.
__device__ __forceinline__ void reduce_to_nodes(int key, float (&v)[16], float4* acc)
{
	const unsigned lane = threadIdx.x & 31;
	const unsigned grp = __match_any_sync(0xffffffffu, key);
	const unsigned above = grp & ~((2u << lane) - 1u);
	int nxt = above ? __ffs(above) - 1 : -1;
	while (__any_sync(0xffffffffu, nxt >= 0)) {
		const int src = nxt >= 0 ? nxt : (int)lane;
#pragma unroll
		for (int c = 0; c < 16; c++) {
			const float o = __shfl_sync(0xffffffffu, v[c], src);
			if (nxt >= 0) v[c] += o;
		}
		nxt = __shfl_sync(0xffffffffu, nxt, src);
	}
	if (key >= 0 && (grp & ((1u << lane) - 1u)) == 0) {
		float* p = reinterpret_cast<float*>(acc + 4 * (size_t)key);
		red_add_v4(p, v[0], v[1], v[2], v[3]);
		red_add_v4(p + 4, v[4], v[5], v[6], v[7]);
		red_add_v4(p + 8, v[8], v[9], v[10], v[11]);
		red_add_v4(p + 12, v[12], v[13], v[14], v[15]);
	}
}

// g = dL/dxyz' and h = dL/drot' (either NULL: zero).  nodes: whether the node accumulators are wanted.
__global__ void __launch_bounds__(DF_THREADS) deform_bwd_kernel(int P, int N, int k, int lshift, int nodes,
	const float* __restrict__ xyz, const float* __restrict__ rot, const long long* __restrict__ index,
	const float* __restrict__ weight, const float4* __restrict__ rec, const float4* __restrict__ rstate,
	const float* __restrict__ g_xyz, const float* __restrict__ g_rot, float4* __restrict__ acc, float* __restrict__ dL_dxyz,
	float* __restrict__ dL_drot, float* __restrict__ dL_dweight)
{
	const int L = 1 << lshift;
	const int sub = threadIdx.x & (L - 1);
	const int i = blockIdx.x * (DF_THREADS >> lshift) + (threadIdx.x >> lshift);
	const bool live = i < P;  // no early return: the shuffles below need every lane of the warp
	float x[3] = {0.f, 0.f, 0.f}, g[3] = {0.f, 0.f, 0.f};
	Quat dr = {0.f, 0.f, 0.f, 0.f};
	if (live) {
		x[0] = xyz[3 * (size_t)i]; x[1] = xyz[3 * (size_t)i + 1]; x[2] = xyz[3 * (size_t)i + 2];
		if (g_xyz) { g[0] = g_xyz[3 * (size_t)i]; g[1] = g_xyz[3 * (size_t)i + 1]; g[2] = g_xyz[3 * (size_t)i + 2]; }
		if (g_rot) {
			// rot' = n (x) p: dL/dn = h (x) conj(p), dL/dp = conj(n) (x) h; dL/dr through F.normalize
			const float4 hv = ld4(g_rot + 4 * (size_t)i), pv = ld4(rot + 4 * (size_t)i), r = rstate[i];
			const Quat h = {hv.x, hv.y, hv.z, hv.w}, p = {pv.x, pv.y, pv.z, pv.w};
			const float nr = qnorm(r);
			const Quat n = normalized(r, nr);
			const float4 d = normalize_bwd(r, nr, n, qmul(h, conj(p)));
			dr = {d.x, d.y, d.z, d.w};
			if (dL_drot && sub == 0) {
				const Quat dp = qmul(conj(n), h);
				st4(dL_drot + 4 * (size_t)i, make_float4(dp.r, dp.x, dp.y, dp.z));
			}
		} else if (dL_drot && sub == 0) {
			st4(dL_drot + 4 * (size_t)i, make_float4(0.f, 0.f, 0.f, 0.f));
		}
	}
	float gx[3] = {0.f, 0.f, 0.f};  // sum w (R^T g - g)
	for (int s0 = 0; s0 < k; s0 += L) {  // the same trip count on every lane: reduce_to_nodes is warp-collective
		const int s = s0 + sub;
		int j = -1;
		float w = 0.f;
		const bool valid = live && s < k && df_slot(N, k, i, s, index, weight, j, w);
		float v[16];
#pragma unroll
		for (int c = 0; c < 16; c++) v[c] = 0.f;
		if (valid) {
			float4 n[4];
			load_rec(rec, j, n);
			float u[3];
			node_move(n, x, u);
			gx[0] += w * (n[0].x * g[0] + n[1].x * g[1] + n[2].x * g[2] - g[0]);
			gx[1] += w * (n[0].y * g[0] + n[1].y * g[1] + n[2].y * g[2] - g[1]);
			gx[2] += w * (n[0].z * g[0] + n[1].z * g[1] + n[2].z * g[2] - g[2]);
			if (dL_dweight)
				dL_dweight[(size_t)i * k + s] = g[0] * u[0] + g[1] * u[1] + g[2] * u[2] + dr.r * (n[3].x - 1.f) + dr.x * n[3].y
				                                + dr.y * n[3].z + dr.z * n[3].w;
			const float wg[3] = {w * g[0], w * g[1], w * g[2]};
#pragma unroll
			for (int aa = 0; aa < 3; aa++) {
				v[4 * aa + 0] = wg[aa] * x[0];
				v[4 * aa + 1] = wg[aa] * x[1];
				v[4 * aa + 2] = wg[aa] * x[2];
				v[4 * aa + 3] = wg[aa];
			}
			v[12] = w * dr.r; v[13] = w * dr.x; v[14] = w * dr.y; v[15] = w * dr.z;
		} else if (live && s < k && dL_dweight) {
			dL_dweight[(size_t)i * k + s] = 0.f;
		}
		if (nodes) reduce_to_nodes(valid ? j : -1 - (int)(threadIdx.x & 31), v, acc);
	}
	for (int m = L >> 1; m > 0; m >>= 1)
#pragma unroll
		for (int c = 0; c < 3; c++) gx[c] += __shfl_xor_sync(0xffffffffu, gx[c], m);
	if (live && sub == 0 && dL_dxyz) {
		dL_dxyz[3 * (size_t)i] = g[0] + gx[0];
		dL_dxyz[3 * (size_t)i + 1] = g[1] + gx[1];
		dL_dxyz[3 * (size_t)i + 2] = g[2] + gx[2];
	}
}

// dL/dnode_t = G_c, dL/dnode_xyz = G_c - R^T G_c, and dL/dR = G_R - G_c node_xyz^T with G_q chained to node_rot
__global__ void __launch_bounds__(DF_THREADS) deform_node_bwd_kernel(int N, const float* __restrict__ node_xyz,
	const float* __restrict__ node_rot, const float4* __restrict__ acc, float* __restrict__ dL_dnode_xyz,
	float* __restrict__ dL_dnode_rot, float* __restrict__ dL_dnode_t)
{
	const int j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= N) return;
	const float4 a0 = acc[4 * (size_t)j], a1 = acc[4 * (size_t)j + 1], a2 = acc[4 * (size_t)j + 2], a3 = acc[4 * (size_t)j + 3];
	const float gc[3] = {a0.w, a1.w, a2.w};
	if (dL_dnode_t) {
		dL_dnode_t[3 * (size_t)j] = gc[0]; dL_dnode_t[3 * (size_t)j + 1] = gc[1]; dL_dnode_t[3 * (size_t)j + 2] = gc[2];
	}
	if (!dL_dnode_xyz && !dL_dnode_rot) return;
	const float4 v = ld4(node_rot + 4 * (size_t)j);
	const float nv = qnorm(v);
	float sgn;
	const Quat q = node_quat(v, nv, sgn);
	float4 R[3];
	qrot_rows(q, R);
	if (dL_dnode_xyz) {
		dL_dnode_xyz[3 * (size_t)j] = gc[0] - (R[0].x * gc[0] + R[1].x * gc[1] + R[2].x * gc[2]);
		dL_dnode_xyz[3 * (size_t)j + 1] = gc[1] - (R[0].y * gc[0] + R[1].y * gc[1] + R[2].y * gc[2]);
		dL_dnode_xyz[3 * (size_t)j + 2] = gc[2] - (R[0].z * gc[0] + R[1].z * gc[1] + R[2].z * gc[2]);
	}
	if (!dL_dnode_rot) return;
	const float p[3] = {node_xyz[3 * (size_t)j], node_xyz[3 * (size_t)j + 1], node_xyz[3 * (size_t)j + 2]};
	const float4 gr[3] = {a0, a1, a2};
	float G[3][3];
#pragma unroll
	for (int aa = 0; aa < 3; aa++) {
		G[aa][0] = gr[aa].x - gc[aa] * p[0];
		G[aa][1] = gr[aa].y - gc[aa] * p[1];
		G[aa][2] = gr[aa].z - gc[aa] * p[2];
	}
	const Quat dq = qrot_bwd(q, G);
	// q^ = sgn normalize(v): the sign passes the gradient through
	const Quat dn = {sgn * (dq.r + a3.x), sgn * (dq.x + a3.y), sgn * (dq.y + a3.z), sgn * (dq.z + a3.w)};
	st4(dL_dnode_rot + 4 * (size_t)j, normalize_bwd(v, nv, normalized(v, nv), dn));
}

cudaError_t deform_forward(void* state, int P, int N, int k, const float* xyz, const float* rot, const float* node_xyz,
	const float* node_rot, const float* node_t, const long long* index, const float* weight, float* out_xyz, float* out_rot,
	cudaStream_t st)
{
	const DfState s = DfState::at(align_state(state), P, N);
	if (N > 0) deform_node_fwd_kernel<<<ceil_div(N, DF_THREADS), DF_THREADS, 0, st>>>(N, node_xyz, node_rot, node_t, s.rec);
	if (P > 0) {
		const int ls = lane_shift(k);
		deform_fwd_kernel<<<ceil_div(P, DF_THREADS >> ls), DF_THREADS, 0, st>>>(P, N, k, ls, xyz, rot, index, weight, s.rec, s.r,
		                                                                        out_xyz, out_rot);
	}
	return cudaGetLastError();
}

cudaError_t deform_backward(void* state, int P, int N, int k, const float* xyz, const float* rot, const float* node_xyz,
	const float* node_rot, const long long* index, const float* weight, const float* dL_dout_xyz, const float* dL_dout_rot,
	float* dL_dxyz, float* dL_drot, float* dL_dnode_xyz, float* dL_dnode_rot, float* dL_dnode_t, float* dL_dweight,
	cudaStream_t st)
{
	const DfState s = DfState::at(align_state(state), P, N);
	const bool nodes = N > 0 && (dL_dnode_xyz || dL_dnode_rot || dL_dnode_t);
	if (nodes) {
		cudaError_t e = cudaMemsetAsync(s.acc, 0, (size_t)N * 4 * sizeof(float4), st);
		if (e != cudaSuccess) return e;
	}
	if (P > 0 && (nodes || dL_dxyz || dL_drot || dL_dweight)) {
		const int ls = lane_shift(k);
		deform_bwd_kernel<<<ceil_div(P, DF_THREADS >> ls), DF_THREADS, 0, st>>>(P, N, k, ls, nodes ? 1 : 0, xyz, rot, index, weight,
		                                                                        s.rec, s.r, dL_dout_xyz, dL_dout_rot, s.acc,
		                                                                        dL_dxyz, dL_drot, dL_dweight);
	}
	if (nodes)
		deform_node_bwd_kernel<<<ceil_div(N, DF_THREADS), DF_THREADS, 0, st>>>(N, node_xyz, node_rot, s.acc, dL_dnode_xyz,
		                                                                       dL_dnode_rot, dL_dnode_t);
	return cudaGetLastError();
}

}  // namespace mgs
