// Field queries: the Gaussian field's density and features at arbitrary 3D points (include/mgs_rasterizer.h,
// mgs_field_query), forward and backward.  For Gaussian i with frame rows A_k = R_k(q^) / s_k (R_k row k of the
// rasterizer's rotation of the unit quaternion, so Sigma = sum_k s_k^2 R_k^T R_k) and a point x:
//   u_k = A_k . (x - mu),  m = |u|^2,  g = o exp(-m / 2) if g >= 1/255 else 0,
//   density(x) = sum_i g_i(x),   features(x)[c] = sum_i g_i(x) f_i[c].
//
// Stages (field_* launchers below, orchestrated by mgs_field_query in api.cu):
//   bbox / grid  the queries' bounding box (finite points only) and a uniform grid of at most nb_max bins over it, chosen on
//                the device: the smallest cubic cell whose per-axis counts multiply to <= nb_max;
//   prep         one thread per Gaussian: the frame rows, mean, opacity and cutoff as a 64-byte record, the support's
//                axis-aligned half-extent sqrt(2 ln(255 o) Sigma_kk) (with a small slack) and the number of bins it touches;
//   queries      per query its bin; a stable radix sort groups them by bin, and every bin's queries are cut into warp items
//                of at most 32;
//   pairs        a 64-bit scan of the per-Gaussian bin counts sizes the (bin, Gaussian) pairs (read back once by the host),
//                the emission in Gaussian order and a stable radix sort by bin leave each bin's Gaussians in ascending id;
//   forward      one warp per item and channel group: lane = query for the weights (the density is summed in the lane),
//                the feature contraction on the tensor cores (m16n8k8 TF32, 3xTF32 split, blend_mma.cuh);
//   backward     one warp per item, all channel groups: GEMM 1 (dL/dg = dD + dF . f_i) on the tensor cores, the per-pair
//                geometric terms in the lane that owns the query (dL/dx summed there, no atomics), their per-Gaussian sums
//                over the warp sent out with red.global.add.v4.f32, and the transposed contraction dL/df_i = sum_x g dF
//                with the lift's gemm2_step / red_feature_row; then one thread per Gaussian chains the record's
//                gradients to means, scales, the quaternion (through its normalisation) and the opacity.
// Binning is conservative: a pair whose AABB reaches a bin but whose support misses the bin's queries adds exact zeros, so
// the bin size changes nothing but the order of the tensor-core sums.
#include <algorithm>
#include <map>
#include <mutex>
#include <tuple>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/iterator/transform_input_iterator.cuh>
#include "../../include/mgs_rasterizer.h"
#include "blend_mma.cuh"
#include "mgs_kernels.h"

namespace mgs {

constexpr int FQ_CH = 32;      // Gaussians per chunk of a warp's bin list
constexpr int FQ_WS = 36;      // forward weight tile [query][Gaussian] row stride: A fragments hit 32 banks
constexpr int FQ_FS_FWD = 40;  // forward feature rows [Gaussian][channel]: B fragments (k = Gaussian) hit 32 banks
constexpr int FQ_FS_BWD = 36;  // backward feature rows: GEMM 1's B fragments (k = channel) hit 32 banks

// ---- bounding box of the finite queries, as order-preserving unsigned keys (fkey / funkey, mgs_common.cuh) ----
__global__ void __launch_bounds__(256) field_bbox_kernel(int Q, const float* __restrict__ pts, uint32_t* __restrict__ box)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	uint32_t lo[3] = { 0xffffffffu, 0xffffffffu, 0xffffffffu }, hi[3] = { 0u, 0u, 0u };
	if (i < Q) {
		const float x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
		if (isfinite(x) && isfinite(y) && isfinite(z)) {
			lo[0] = hi[0] = fkey(x); lo[1] = hi[1] = fkey(y); lo[2] = hi[2] = fkey(z);
		}
	}
#pragma unroll
	for (int k = 0; k < 3; k++) {
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) {
			lo[k] = min(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o));
			hi[k] = max(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o));
		}
	}
	if ((threadIdx.x & 31) == 0 && lo[0] <= hi[0]) {
#pragma unroll
		for (int k = 0; k < 3; k++) { atomicMin(box + k, lo[k]); atomicMax(box + 3 + k, hi[k]); }
	}
}

// one thread: the grid over the box (FieldGrid in the state header)
__global__ void field_grid_kernel(const uint32_t* __restrict__ box, int nb_max, FieldGrid* __restrict__ grid)
{
	FieldGrid g{};
	g.n[0] = g.n[1] = g.n[2] = 1;
	if (box[0] <= box[3]) {
		float e[3], emax = 0.f;
#pragma unroll
		for (int k = 0; k < 3; k++) {
			g.lo[k] = funkey(box[k]);
			e[k] = fmaxf(funkey(box[3 + k]) - g.lo[k], 0.f);
			emax = fmaxf(emax, e[k]);
		}
		if (emax > 0.f) {
			// the smallest cubic cell h with prod_k max(1, ceil(e_k / h)) <= nb_max
			auto bins = [&](float h) {
				double p = 1.0;
				for (int k = 0; k < 3; k++) p *= fmax(1.0, ceil((double)e[k] / h));
				return p;
			};
			float h_ok = emax, h_bad = emax / (float)nb_max * 0.5f;
			for (int it = 0; it < 48 && bins(h_bad) > nb_max; it++) {
				const float h = 0.5f * (h_ok + h_bad);
				if (bins(h) <= nb_max) h_ok = h; else h_bad = h;
			}
#pragma unroll
			for (int k = 0; k < 3; k++) {
				g.n[k] = e[k] > 0.f ? max(1, (int)ceil((double)e[k] / h_ok)) : 1;
				g.inv[k] = e[k] > 0.f ? (float)g.n[k] / e[k] : 0.f;
			}
		}
	}
	*grid = g;
}

__device__ __forceinline__ int bin_coord(float x, const FieldGrid& g, int k)
{
	const float t = floorf((x - g.lo[k]) * g.inv[k]);
	return t <= 0.f ? 0 : (t >= (float)(g.n[k] - 1) ? g.n[k] - 1 : (int)t);  // NaN -> 0
}

// row k of R(q) for a unit q = (r, x, y, z): the direction that scale k stretches (as normals.cu's axis_of)
__device__ __forceinline__ void frame_row(const float (&q)[4], int k, float (&a)[3])
{
	const float r = q[0], x = q[1], y = q[2], z = q[3];
	if (k == 0) { a[0] = 1.f - 2.f * (y * y + z * z); a[1] = 2.f * (x * y + r * z); a[2] = 2.f * (x * z - r * y); }
	else if (k == 1) { a[0] = 2.f * (x * y - r * z); a[1] = 1.f - 2.f * (x * x + z * z); a[2] = 2.f * (y * z + r * x); }
	else { a[0] = 2.f * (x * z + r * y); a[1] = 2.f * (y * z - r * x); a[2] = 1.f - 2.f * (x * x + y * y); }
}

// The record of Gaussian i (recs[4i .. 4i+3]): {A0, mu.x}, {A1, mu.y}, {A2, mu.z}, {o, 0, 0, 0}; ext[i] = {half-extent, 1}
// for a Gaussian with support, else zeros (it is in no bin list and gets zero gradients).  cnt[i] = bins its box touches.
__global__ void __launch_bounds__(256) field_prep_kernel(int P, const float* __restrict__ means, const float* __restrict__ scales,
	const float* __restrict__ rot, const float* __restrict__ opac, const FieldGrid* __restrict__ grid, float4* __restrict__ recs,
	float4* __restrict__ ext, uint32_t* __restrict__ cnt)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	const float o = opac[i];
	const float s[3] = { scales[3 * i], scales[3 * i + 1], scales[3 * i + 2] };
	const float mu[3] = { means[3 * i], means[3 * i + 1], means[3 * i + 2] };
	float q[4];
	const float inv = rsqrtf(rot[4 * i] * rot[4 * i] + rot[4 * i + 1] * rot[4 * i + 1] + rot[4 * i + 2] * rot[4 * i + 2] + rot[4 * i + 3] * rot[4 * i + 3]);
#pragma unroll
	for (int c = 0; c < 4; c++) q[c] = rot[4 * i + c] * inv;
	float A[3][3], sig[3] = { 0.f, 0.f, 0.f };
	bool ok = o > ALPHA_MIN && isfinite(o) && isfinite(inv);
#pragma unroll
	for (int k = 0; k < 3; k++) {
		ok = ok && s[k] > 0.f && isfinite(s[k]) && isfinite(mu[k]);
		frame_row(q, k, A[k]);
#pragma unroll
		for (int j = 0; j < 3; j++) {
			sig[j] += s[k] * s[k] * A[k][j] * A[k][j];  // Sigma_jj
			A[k][j] /= s[k];
			ok = ok && isfinite(A[k][j]);
		}
	}
	recs[4 * i] = make_float4(A[0][0], A[0][1], A[0][2], mu[0]);
	recs[4 * i + 1] = make_float4(A[1][0], A[1][1], A[1][2], mu[1]);
	recs[4 * i + 2] = make_float4(A[2][0], A[2][1], A[2][2], mu[2]);
	recs[4 * i + 3] = make_float4(o, 0.f, 0.f, 0.f);
	uint32_t n = 0;
	float r[3] = { 0.f, 0.f, 0.f };
	if (ok) {
		const FieldGrid g = *grid;
		// exact box of m <= 2 ln(255 o), widened for the fp32 rounding of g near the cutoff
		const float tau = 2.f * logf(255.f * o) * 1.001f + 1e-4f;
		n = 1;
		bool hit = true;
#pragma unroll
		for (int k = 0; k < 3; k++) {
			r[k] = sqrtf(tau * sig[k]) * 1.0001f + 1e-7f;
			if (g.inv[k] > 0.f) {
				hit = hit && mu[k] + r[k] >= g.lo[k] && mu[k] - r[k] <= g.lo[k] + (float)g.n[k] / g.inv[k];
				n *= (uint32_t)(bin_coord(mu[k] + r[k], g, k) - bin_coord(mu[k] - r[k], g, k) + 1);
			} else {
				hit = hit && mu[k] + r[k] >= g.lo[k] && mu[k] - r[k] <= g.lo[k];
			}
		}
		if (!hit) n = 0;
	}
	ext[i] = make_float4(r[0], r[1], r[2], ok ? 1.f : 0.f);
	cnt[i] = n;
}

__global__ void __launch_bounds__(256) field_emit_kernel(int P, const float4* __restrict__ recs, const float4* __restrict__ ext,
	const uint32_t* __restrict__ cnt, const unsigned long long* __restrict__ off, const FieldGrid* __restrict__ grid,
	uint32_t* __restrict__ keys, uint32_t* __restrict__ vals)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P || cnt[i] == 0) return;
	const FieldGrid g = *grid;
	const float4 e = ext[i];
	const float mu[3] = { recs[4 * i].w, recs[4 * i + 1].w, recs[4 * i + 2].w };
	const float r[3] = { e.x, e.y, e.z };
	int b0[3], b1[3];
#pragma unroll
	for (int k = 0; k < 3; k++) { b0[k] = bin_coord(mu[k] - r[k], g, k); b1[k] = bin_coord(mu[k] + r[k], g, k); }
	unsigned long long p = off[i] - cnt[i];
	for (int z = b0[2]; z <= b1[2]; z++)
		for (int y = b0[1]; y <= b1[1]; y++)
			for (int x = b0[0]; x <= b1[0]; x++, p++) {
				keys[p] = (uint32_t)(x + g.n[0] * (y + g.n[1] * z));
				vals[p] = (uint32_t)i;
			}
}

__global__ void __launch_bounds__(256) field_query_keys_kernel(int Q, const float* __restrict__ pts, const FieldGrid* __restrict__ grid,
	uint32_t* __restrict__ keys, uint32_t* __restrict__ iota)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= Q) return;
	const FieldGrid g = *grid;
	const int x = bin_coord(pts[3 * i], g, 0), y = bin_coord(pts[3 * i + 1], g, 1), z = bin_coord(pts[3 * i + 2], g, 2);
	keys[i] = (uint32_t)(x + g.n[0] * (y + g.n[1] * z));
	iota[i] = (uint32_t)i;
}

// range[key] = [first, last + 1) of each key's run in the sorted keys (ranges zeroed by the caller)
__global__ void __launch_bounds__(256) field_ranges_kernel(int n, const uint32_t* __restrict__ keys, uint2* __restrict__ range)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const uint32_t k = keys[i];
	if (i == 0 || keys[i - 1] != k) range[k].x = (uint32_t)i;
	if (i == n - 1 || keys[i + 1] != k) range[k].y = (uint32_t)(i + 1);
}

__global__ void __launch_bounds__(256) field_warp_count_kernel(int nb, const uint2* __restrict__ qrange, uint32_t* __restrict__ wcnt)
{
	const int b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b < nb) wcnt[b] = (qrange[b].y - qrange[b].x + 31) / 32;
}

// items[woff[b] - wcnt[b] + w] = {first query, end, bin} of warp w of bin b; the last bin writes the item count
__global__ void __launch_bounds__(256) field_items_kernel(int nb, const uint2* __restrict__ qrange, const uint32_t* __restrict__ wcnt,
	const uint32_t* __restrict__ woff, uint4* __restrict__ items, int* __restrict__ nitems)
{
	const int b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b >= nb) return;
	const uint2 r = qrange[b];
	uint32_t k = woff[b] - wcnt[b];
	for (uint32_t s = r.x; s < r.y; s += 32, k++) items[k] = make_uint4(s, min(s + 32u, r.y), (uint32_t)b, 0u);
	if (b == nb - 1) *nitems = (int)woff[b];
}

// ---- the warp's work: its queries and its bin's Gaussian list ----
struct WarpItem {
	int n;            // queries of the item (1..32)
	uint32_t qid;     // this lane's query (valid when lane < n)
	float x, y, z;    // its point
	uint32_t g0;      // first pair of the bin's list
	int count;        // Gaussians in the list
};

__device__ __forceinline__ WarpItem load_item(const FieldArgs& a, int item, int lane)
{
	WarpItem w;
	const uint4 it = a.items[item];
	w.n = (int)(it.y - it.x);
	w.qid = lane < w.n ? a.qorder[it.x + lane] : 0u;
	w.x = lane < w.n ? a.points[3 * w.qid] : 0.f;
	w.y = lane < w.n ? a.points[3 * w.qid + 1] : 0.f;
	w.z = lane < w.n ? a.points[3 * w.qid + 2] : 0.f;
	const uint2 r = a.gbin[it.z];
	w.g0 = r.x;
	w.count = (int)(r.y - r.x);
	return w;
}

// Gaussian j of the chunk at x: u, the exponential E = exp(-m / 2) and g (0 outside the support)
struct PairEval { float d[3], u[3], E, g; };
__device__ __forceinline__ PairEval eval_pair(const float4* rec, float x, float y, float z)
{
	PairEval p;
	const float4 r0 = rec[0], r1 = rec[1], r2 = rec[2], r3 = rec[3];
	p.d[0] = x - r0.w; p.d[1] = y - r1.w; p.d[2] = z - r2.w;
	p.u[0] = r0.x * p.d[0] + r0.y * p.d[1] + r0.z * p.d[2];
	p.u[1] = r1.x * p.d[0] + r1.y * p.d[1] + r1.z * p.d[2];
	p.u[2] = r2.x * p.d[0] + r2.y * p.d[1] + r2.z * p.d[2];
	p.E = expf(-0.5f * (p.u[0] * p.u[0] + p.u[1] * p.u[1] + p.u[2] * p.u[2]));
	const float g = r3.x * p.E;
	p.g = g >= ALPHA_MIN ? g : 0.f;
	return p;
}

// records of list entries k0 .. k0 + cnt - 1 into s_rec (lane j: entry j); returns this lane's Gaussian id
__device__ __forceinline__ uint32_t gather_records(const FieldArgs& a, const WarpItem& w, int k0, int cnt, float4* s_rec, int lane)
{
	uint32_t id = 0;
	if (lane < cnt) {
		id = a.pairs[w.g0 + k0 + lane];
#pragma unroll
		for (int t = 0; t < 4; t++) cp_async16(s_rec + 4 * lane + t, a.recs + 4 * (size_t)id + t);
	}
	return id;
}

// feature rows (channels c0 .. c0 + Cg - 1) of the chunk's Gaussians (the id of row j in lane j) into s_f [j][FS]: 16-byte
// cp.async pieces when the rows allow it (VEC), else coalesced scalar loads, one row per trip
template <bool VEC, int FS>
__device__ __forceinline__ void gather_features(const float* feat, int C, int c0, int Cg, int cnt, uint32_t id, float* s_f, int lane)
{
	if (VEC) {
		for (int trip = 0; 4 * trip < cnt; trip++) {
			const int j = 4 * trip + (lane >> 3), p = lane & 7;
			const uint32_t g = __shfl_sync(0xffffffffu, id, j);
			if (j < cnt && 4 * p < Cg) cp_async16(s_f + j * FS + 4 * p, feat + (size_t)g * C + c0 + 4 * p);
		}
	} else {
		for (int j = 0; j < cnt; j++) {
			const uint32_t g = __shfl_sync(0xffffffffu, id, j);
			if (lane < Cg) s_f[j * FS + lane] = __ldg(feat + (size_t)g * C + c0 + lane);
		}
	}
}

__device__ __forceinline__ size_t feat_index(const FieldArgs& a, uint32_t q, int c)
{
	return a.channel_first ? (size_t)c * a.Q + q : (size_t)q * a.C + c;
}

// NFT: 8-wide channel tiles of the group (0 = density only, 1, 2, 4); VEC: 16-byte feature pieces.  blockIdx.x = item,
// blockIdx.y = channel group of 32.
template <int NFT, bool VEC>
__global__ void __launch_bounds__(32, 16) field_fwd_kernel(FieldArgs a)
{
	constexpr int NF = NFT > 0 ? NFT : 1;
	__shared__ __align__(16) float4 s_rec[2][FQ_CH * 4];                   // records of the current and the next chunk
	__shared__ __align__(16) float s_f[2][NFT > 0 ? FQ_CH * FQ_FS_FWD : 4];  // their feature rows
	__shared__ __align__(16) float s_w[NFT > 0 ? 32 * FQ_WS : 4];            // weights [query][Gaussian]
	const int lane = threadIdx.x, gid = lane >> 2, tig = lane & 3;
	if ((int)blockIdx.x >= *a.nitems) return;
	const WarpItem w = load_item(a, blockIdx.x, lane);
	const int grp = blockIdx.y, c0 = 32 * grp, Cg = min(a.C - c0, 32);
	const bool has = lane < w.n;
	float dens = 0.f;
	float acc[2][NF][4];
#pragma unroll
	for (int mt = 0; mt < 2; mt++)
#pragma unroll
		for (int nt = 0; nt < NF; nt++)
#pragma unroll
			for (int e = 0; e < 4; e++) acc[mt][nt][e] = 0.f;
	if (NFT > 0) {
		// rows past a chunk's end meet zero weights: they must hold finite values
		for (int i = lane; i < 2 * FQ_CH * FQ_FS_FWD; i += 32) (&s_f[0][0])[i] = 0.f;
		__syncwarp();
	}
	const int cnt0 = min(w.count, FQ_CH);
	uint32_t id = gather_records(a, w, 0, cnt0, s_rec[0], lane);
	if (NFT > 0) gather_features<VEC, FQ_FS_FWD>(a.features, a.C, c0, Cg, cnt0, id, s_f[0], lane);
	cp_async_commit();
	for (int k0 = 0, buf = 0; k0 < w.count; k0 += FQ_CH, buf ^= 1) {
		const int cnt = min(w.count - k0, FQ_CH);
		cp_async_wait<0>();
		__syncwarp();
		// ---- the next chunk's records and rows travel while this one runs ----
		const int cnt1 = max(0, min(w.count - k0 - FQ_CH, FQ_CH));
		id = gather_records(a, w, k0 + FQ_CH, cnt1, s_rec[buf ^ 1], lane);
		if (NFT > 0) gather_features<VEC, FQ_FS_FWD>(a.features, a.C, c0, Cg, cnt1, id, s_f[buf ^ 1], lane);
		cp_async_commit();
		// ---- weights: lane = query ----
		bool any = false;
		for (int j = 0; j < cnt; j++) {
			const float g = has ? eval_pair(s_rec[buf] + 4 * j, w.x, w.y, w.z).g : 0.f;
			dens += g;
			any |= g != 0.f;
			if (NFT > 0) s_w[lane * FQ_WS + j] = g;
		}
		if (NFT > 0) {
			for (int j = cnt; j < FQ_CH; j++) s_w[lane * FQ_WS + j] = 0.f;
			__syncwarp();
			// ---- contract: acc[q][ch] += w[q][j] f[j][ch]   (M = queries, K = Gaussians, N = channels) ----
			if (__any_sync(0xffffffffu, any)) {
#pragma unroll
				for (int ks = 0; ks < FQ_CH / 8; ks++) {
					uint32_t ahi[2][4], alo[2][4];
#pragma unroll
					for (int mt = 0; mt < 2; mt++) {
						const float* wr = s_w + (16 * mt + gid) * FQ_WS + 8 * ks + tig;
						tf32_split(wr[0], ahi[mt][0], alo[mt][0]);
						tf32_split(wr[8 * FQ_WS], ahi[mt][1], alo[mt][1]);
						tf32_split(wr[4], ahi[mt][2], alo[mt][2]);
						tf32_split(wr[8 * FQ_WS + 4], ahi[mt][3], alo[mt][3]);
					}
					const float* fr = s_f[buf] + (8 * ks + tig) * FQ_FS_FWD + gid;
#pragma unroll
					for (int nt = 0; nt < NFT; nt++) {
						uint32_t bh0, bl0, bh1, bl1;
						tf32_split(fr[8 * nt], bh0, bl0);
						tf32_split(fr[4 * FQ_FS_FWD + 8 * nt], bh1, bl1);
#pragma unroll
						for (int mt = 0; mt < 2; mt++) mma_3xtf32(acc[mt][nt], ahi[mt], alo[mt], bh0, bh1, bl0, bl1);
					}
				}
			}
			__syncwarp();  // s_w and this chunk's rows are rewritten by the next chunks
		}
	}
	cp_async_wait<0>();  // no copy may be in flight when the CTA exits
	if (grp == 0 && has) a.density[w.qid] = dens;
	if (NFT > 0) {
		// D rows gid (h = 0) and gid + 8 (h = 1) of tile mt are queries 16 mt + gid + 8 h, columns 2 tig + e of tile nt channels
		// 8 nt + 2 tig + e
#pragma unroll
		for (int mt = 0; mt < 2; mt++) {
#pragma unroll
			for (int h = 0; h < 2; h++) {
				const int row = 16 * mt + gid + 8 * h;
				const uint32_t q = __shfl_sync(0xffffffffu, w.qid, row);
				if (row >= w.n) continue;
#pragma unroll
				for (int nt = 0; nt < NFT; nt++)
#pragma unroll
					for (int e = 0; e < 2; e++) {
						const int col = 8 * nt + 2 * tig + e;
						if (col < Cg) a.out_features[feat_index(a, q, c0 + col)] = acc[mt][nt][2 * h + e];
					}
			}
		}
	}
}

// Sum of v[0..15] over the warp's lanes, transposed: afterwards lane l holds the total of value (l >> 1) in v[0]
// (16 shuffles instead of 80)
__device__ __forceinline__ void warp_sum16(float (&v)[16], int lane)
{
#pragma unroll
	for (int s = 0; s < 4; s++) {
		const int n = 8 >> s, off = 16 >> s;
		const bool up = (lane & off) != 0;
#pragma unroll
		for (int i = 0; i < n; i++) {
			const float send = up ? v[i] : v[i + n];
			const float keep = up ? v[i + n] : v[i];
			v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
		}
	}
	v[0] += __shfl_xor_sync(0xffffffffu, v[0], 1);
}

// One warp per item, every channel group in the warp (dL/dg sums over all channels).  Per chunk of the bin's list:
//   pass A   lane = query: the weights into the lift's [pi][j >> 1][e][j & 1] tile, and per Gaussian the ballot of the
//            queries inside its support;
//   groups   per channel group: the dF rows of the warp's queries ([pi][ch][e], staged once without groups), GEMM 1
//            D1[q][j] += dF[q][:] . f_j[:] (tensor cores, M = queries, N = Gaussians, K = channels) and GEMM 2
//            dL/df_j += sum_q w[q][j] dF[q][:] (gemm2_step, flushed with red_feature_row as the lift does);
//   pass C   lane = query, per Gaussian with a pair in the warp: dL/dg = dD + D1, then dL/do, dL/dmu and dL/dA_k in the
//            lane, dL/dx summed in the lane; the per-Gaussian terms summed over the warp (warp_sum16) and sent out with
//            red.global.add.v4.f32 into ggeo, laid out as the record.
template <int NFT, bool VEC, bool GRP>
__global__ void __launch_bounds__(32, 12) field_bwd_kernel(FieldArgs a)
{
	constexpr int NF = NFT > 0 ? NFT : 1;
	constexpr int GS = 16 * (NF + 1);   // dF rows: stride per query pair, as the lift's map rows
	constexpr int XS = 2 * FQ_CH + 4;   // weight tile: stride per query pair, as the lift's
	__shared__ __align__(16) float4 s_rec[2][FQ_CH * 4];
	__shared__ __align__(16) float s_f[NFT > 0 ? FQ_CH * FQ_FS_BWD : 4];
	__shared__ __align__(16) float s_g[NFT > 0 ? 16 * GS : 4];
	__shared__ __align__(16) float s_w[NFT > 0 ? 16 * XS : 4];
	__shared__ __align__(16) float s_dg[NFT > 0 ? 32 * FQ_WS : 4];
	__shared__ __align__(16) float s_red[FQ_CH * 16];
	__shared__ uint32_t s_pm[FQ_CH];
	const int lane = threadIdx.x, gid = lane >> 2, tig = lane & 3;
	if ((int)blockIdx.x >= *a.nitems) return;
	const WarpItem w = load_item(a, blockIdx.x, lane);
	const bool has = lane < w.n;
	const bool need_geo = a.ggeo != nullptr, need_x = a.dL_dpoints != nullptr;
	const bool with_dF = NFT > 0 && a.dL_dfeatures != nullptr;
	const bool need_f = with_dF && a.dL_dfeat != nullptr;
	const bool gemm1 = with_dF && (need_geo || need_x);
	const int groups = GRP ? a.groups : 1;
	const float dD = (has && a.dL_ddensity) ? a.dL_ddensity[w.qid] : 0.f;
	float dx[3] = { 0.f, 0.f, 0.f };
	bool staged = false;
	if (NFT > 0) {
		for (int i = lane; i < FQ_CH * FQ_FS_BWD; i += 32) s_f[i] = 0.f;
		__syncwarp();
	}
	uint32_t id = gather_records(a, w, 0, min(w.count, FQ_CH), s_rec[0], lane);
	cp_async_commit();
	for (int k0 = 0, buf = 0; k0 < w.count; k0 += FQ_CH, buf ^= 1) {
		const int cnt = min(w.count - k0, FQ_CH);
		const float4* const rec = s_rec[buf];
		const uint32_t id_cur = id;
		cp_async_wait<0>();
		__syncwarp();
		id = gather_records(a, w, k0 + FQ_CH, max(0, min(w.count - k0 - FQ_CH, FQ_CH)), s_rec[buf ^ 1], lane);
		cp_async_commit();
		// ---- pass A ----
		uint32_t chunk_any = 0u;
		for (int j = 0; j < FQ_CH; j++) {
			const float g = (j < cnt && has) ? eval_pair(rec + 4 * j, w.x, w.y, w.z).g : 0.f;
			if (need_f) s_w[(lane >> 1) * XS + (j >> 1) * 4 + (lane & 1) * 2 + (j & 1)] = g;
			const uint32_t b = __ballot_sync(0xffffffffu, g != 0.f);
			if (lane == 0) s_pm[j] = b;
			chunk_any |= b;
		}
		__syncwarp();
		if (chunk_any == 0u) continue;
		// ---- channel groups: GEMM 1 into D1, GEMM 2 flushed per group ----
		float D1[2][4][4];
#pragma unroll
		for (int mt = 0; mt < 2; mt++)
#pragma unroll
			for (int nt = 0; nt < 4; nt++)
#pragma unroll
				for (int e = 0; e < 4; e++) D1[mt][nt][e] = 0.f;
		if (gemm1 || need_f) {
			for (int grp = 0; grp < groups; grp++) {
				const int c0 = 32 * grp, Cg = min(a.C - c0, 32);
				if (GRP || !staged) {
					// element (query 2 pi + e, channel ch) at [pi][ch][e]; absent queries and channels hold 0
					float* grow = s_g + (lane >> 1) * GS + (lane & 1);
#pragma unroll
					for (int c = 0; c < 8 * NF; c++)
						grow[2 * c] = (has && c < Cg) ? __ldg(a.dL_dfeatures + feat_index(a, w.qid, c0 + c)) : 0.f;
					staged = true;
				}
				if (gemm1) {
					gather_features<VEC, FQ_FS_BWD>(a.features, a.C, c0, Cg, cnt, id_cur, s_f, lane);
					cp_async_commit();
					cp_async_wait<0>();
				}
				__syncwarp();
				if (gemm1) {
#pragma unroll
					for (int ks = 0; ks < NF; ks++) {
						uint32_t ahi[2][4], alo[2][4];
#pragma unroll
						for (int mt = 0; mt < 2; mt++) {
							// A: (query 16 mt + gid (+8), channel 8 ks + tig (+4)); queries 2 pi + e of pair pi
							const float* r0 = s_g + (8 * mt + (gid >> 1)) * GS + 2 * (8 * ks + tig) + (gid & 1);
							tf32_split(r0[0], ahi[mt][0], alo[mt][0]);
							tf32_split(r0[4 * GS], ahi[mt][1], alo[mt][1]);
							tf32_split(r0[8], ahi[mt][2], alo[mt][2]);
							tf32_split(r0[4 * GS + 8], ahi[mt][3], alo[mt][3]);
						}
#pragma unroll
						for (int nt = 0; nt < 4; nt++) {
							// B: (channel 8 ks + tig (+4), Gaussian 8 nt + gid)
							const float* fr = s_f + (8 * nt + gid) * FQ_FS_BWD + 8 * ks + tig;
							uint32_t bh0, bl0, bh1, bl1;
							tf32_split(fr[0], bh0, bl0);
							tf32_split(fr[4], bh1, bl1);
#pragma unroll
							for (int mt = 0; mt < 2; mt++) mma_3xtf32(D1[mt][nt], ahi[mt], alo[mt], bh0, bh1, bl0, bl1);
						}
					}
				}
				if (need_f) {
					// dC[j][ch] = w[:][j] . dF[:][ch]   (M = Gaussians, K = queries, N = channels), as lift_kernel
					float dC[2][NF + 1][4];
#pragma unroll
					for (int mt = 0; mt < 2; mt++)
#pragma unroll
						for (int nt = 0; nt <= NF; nt++)
#pragma unroll
							for (int e = 0; e < 4; e++) dC[mt][nt][e] = 0.f;
#pragma unroll
					for (int kp = 0; kp < 4; kp++) {
						uint32_t ahi[2][4], alo[2][4];
#pragma unroll
						for (int mt = 0; mt < 2; mt++) {
							const float4 w4 = *reinterpret_cast<const float4*>(s_w + (4 * kp + tig) * XS + mt * 32 + gid * 4);
							tf32_split(w4.x, ahi[mt][0], alo[mt][0]); tf32_split(w4.y, ahi[mt][1], alo[mt][1]);
							tf32_split(w4.z, ahi[mt][2], alo[mt][2]); tf32_split(w4.w, ahi[mt][3], alo[mt][3]);
						}
						gemm2_step<NF, 2>(dC, ahi, alo, s_g + (4 * kp + tig) * GS, gid, false);
					}
#pragma unroll
					for (int mt = 0; mt < 2; mt++) {
#pragma unroll
						for (int h = 0; h < 2; h++) {
							const int j = 16 * mt + 2 * gid + h;
							const uint32_t gj = __shfl_sync(0xffffffffu, id_cur, j);
							if (j < cnt && s_pm[j] != 0u)
								red_feature_row<NF, VEC, GRP>(a.dL_dfeat + (size_t)gj * a.C + c0, dC[mt], h, tig, Cg);
						}
					}
				}
				__syncwarp();  // s_f and s_g are rewritten by the next group
			}
		}
		if (gemm1) {
			// D1 rows gid (+8) of tile mt are queries 16 mt + gid (+8), columns 2 tig + e of tile nt Gaussians 8 nt + 2 tig + e
#pragma unroll
			for (int mt = 0; mt < 2; mt++)
#pragma unroll
				for (int nt = 0; nt < 4; nt++)
#pragma unroll
					for (int i = 0; i < 4; i++) s_dg[(16 * mt + gid + 8 * (i >> 1)) * FQ_WS + 8 * nt + 2 * tig + (i & 1)] = D1[mt][nt][i];
			__syncwarp();
		}
		// ---- pass C ----
		if (need_geo || need_x) {
			for (int j = 0; j < cnt; j++) {
				const uint32_t b = s_pm[j];
				if (b == 0u) continue;
				float v[16];
#pragma unroll
				for (int i = 0; i < 16; i++) v[i] = 0.f;
				if ((b >> lane) & 1u) {
					const PairEval p = eval_pair(rec + 4 * j, w.x, w.y, w.z);
					const float dg = dD + (gemm1 ? s_dg[lane * FQ_WS + j] : 0.f);
					const float t = -dg * p.g;  // dL/dm times 2
					v[12] = dg * p.E;           // dL/do
					float vx = 0.f, vy = 0.f, vz = 0.f;
#pragma unroll
					for (int k = 0; k < 3; k++) {
						const float4 A = rec[4 * j + k];
						const float ck = t * p.u[k];  // dL/du_k
						v[4 * k] = ck * p.d[0]; v[4 * k + 1] = ck * p.d[1]; v[4 * k + 2] = ck * p.d[2];
						vx += ck * A.x; vy += ck * A.y; vz += ck * A.z;
					}
					dx[0] += vx; dx[1] += vy; dx[2] += vz;
					v[3] = -vx; v[7] = -vy; v[11] = -vz;
				}
				if (need_geo) {
					warp_sum16(v, lane);
					if ((lane & 1) == 0) s_red[j * 16 + (lane >> 1)] = v[0];
				}
			}
			if (need_geo) {
				__syncwarp();
				if (lane < cnt && s_pm[lane] != 0u) {
					const float4* r = reinterpret_cast<const float4*>(s_red + 16 * lane);
					float* dst = reinterpret_cast<float*>(a.ggeo + 4 * (size_t)id_cur);
#pragma unroll
					for (int t = 0; t < 4; t++) {
						const float4 x = r[t];
						red_add_v4(dst + 4 * t, x.x, x.y, x.z, x.w);
					}
				}
			}
		}
		__syncwarp();  // s_pm, s_w, s_red and s_dg are rewritten by the next chunk
	}
	cp_async_wait<0>();
	if (need_x && has) {
		float* o = a.dL_dpoints + 3 * (size_t)w.qid;
		o[0] = dx[0]; o[1] = dx[1]; o[2] = dx[2];
	}
}

// dL/dq^ of g . R_k(q^) (the normals backward's expressions, for every row k)
__device__ __forceinline__ void frame_row_bwd(const float (&q)[4], int k, float gx, float gy, float gz, float (&d)[4])
{
	const float r = q[0], x = q[1], y = q[2], z = q[3];
	if (k == 0) {
		d[0] += 2.f * (z * gy - y * gz);
		d[1] += 2.f * (y * gy + z * gz);
		d[2] += -4.f * y * gx + 2.f * (x * gy - r * gz);
		d[3] += -4.f * z * gx + 2.f * (r * gy + x * gz);
	} else if (k == 1) {
		d[0] += 2.f * (x * gz - z * gx);
		d[1] += -4.f * x * gy + 2.f * (y * gx + r * gz);
		d[2] += 2.f * (x * gx + z * gz);
		d[3] += -4.f * z * gy + 2.f * (y * gz - r * gx);
	} else {
		d[0] += 2.f * (y * gx - x * gy);
		d[1] += -4.f * x * gz + 2.f * (z * gx - r * gy);
		d[2] += -4.f * y * gz + 2.f * (r * gx + z * gy);
		d[3] += 2.f * (x * gx + y * gy);
	}
}

// one thread per Gaussian: ggeo {dA_k, dmu_k}_k, {do} -> means, scales (A_k = R_k / s_k), the quaternion through R and its
// normalisation, the opacity; zeros for a Gaussian without support.  Each output is optional.
__global__ void __launch_bounds__(256) field_bwd_gauss_kernel(FieldArgs a)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= a.P) return;
	const bool ok = a.ext[i].w != 0.f;
	const float4 G[4] = { a.ggeo[4 * i], a.ggeo[4 * i + 1], a.ggeo[4 * i + 2], a.ggeo[4 * i + 3] };
	if (a.dL_dmeans) {
		float* o = a.dL_dmeans + 3 * (size_t)i;
		o[0] = ok ? G[0].w : 0.f; o[1] = ok ? G[1].w : 0.f; o[2] = ok ? G[2].w : 0.f;
	}
	if (a.dL_dopac) a.dL_dopac[i] = ok ? G[3].x : 0.f;
	if (!a.dL_dscales && !a.dL_drot) return;
	float ds[3] = { 0.f, 0.f, 0.f }, dq[4] = { 0.f, 0.f, 0.f, 0.f };
	if (ok) {
		const float* rot = a.rotations + 4 * (size_t)i;
		const float inv = rsqrtf(rot[0] * rot[0] + rot[1] * rot[1] + rot[2] * rot[2] + rot[3] * rot[3]);
		float q[4], d[4] = { 0.f, 0.f, 0.f, 0.f };
#pragma unroll
		for (int c = 0; c < 4; c++) q[c] = rot[c] * inv;
#pragma unroll
		for (int k = 0; k < 3; k++) {
			const float s = a.scales[3 * (size_t)i + k];
			const float4 A = a.recs[4 * i + k];
			ds[k] = -(G[k].x * A.x + G[k].y * A.y + G[k].z * A.z) / s;
			frame_row_bwd(q, k, G[k].x / s, G[k].y / s, G[k].z / s, d);
		}
		const float qd = q[0] * d[0] + q[1] * d[1] + q[2] * d[2] + q[3] * d[3];
#pragma unroll
		for (int c = 0; c < 4; c++) dq[c] = (d[c] - q[c] * qd) * inv;
	}
	if (a.dL_dscales) {
		float* o = a.dL_dscales + 3 * (size_t)i;
		o[0] = ds[0]; o[1] = ds[1]; o[2] = ds[2];
	}
	if (a.dL_drot) {
		float* o = a.dL_drot + 4 * (size_t)i;
		o[0] = dq[0]; o[1] = dq[1]; o[2] = dq[2]; o[3] = dq[3];
	}
}

// ---------------------------------------------------------------------------------------------------------------- host
struct ToU64 {
	__host__ __device__ __forceinline__ unsigned long long operator()(const uint32_t& x) const { return x; }
};
using U64It = cub::TransformInputIterator<unsigned long long, ToU64, const uint32_t*>;

int field_bins(int Q) { return std::max(1, std::min((Q + 31) / 32, 1 << 21)); }
int field_items(int Q) { return (Q + 31) / 32 + std::min(field_bins(Q), Q); }
static int key_bits(int nb)
{
	int b = 1;
	while ((1 << b) < nb) b++;
	return b;
}

// CUB's scratch sizes for (Q, P), cached: the size queries look up device attributes
static size_t field_temp_bytes(int Q, int P)
{
	static std::mutex mu;
	static std::map<std::tuple<int, int, int>, size_t> cache;
	int dev = 0;
	cudaGetDevice(&dev);
	std::lock_guard<std::mutex> lk(mu);
	const auto key = std::make_tuple(dev, Q, P);
	const auto it = cache.find(key);
	if (it != cache.end()) return it->second;
	const int nb = field_bins(Q);
	size_t a = 0, b = 0, c = 0;
	cub::DeviceScan::InclusiveSum(nullptr, a, U64It(nullptr, ToU64{}), (unsigned long long*)nullptr, P);
	cub::DeviceRadixSort::SortPairs(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
		(uint32_t*)nullptr, Q, 0, key_bits(nb));
	cub::DeviceScan::InclusiveSum(nullptr, c, (const uint32_t*)nullptr, (uint32_t*)nullptr, nb);
	return cache[key] = std::max(a, std::max(b, c));
}

template <typename T>
static void carve(char*& chunk, T*& ptr, size_t count)
{
	const size_t offset = (reinterpret_cast<uintptr_t>(chunk) + 127) & ~(uintptr_t)127;
	ptr = reinterpret_cast<T*>(offset);
	chunk = reinterpret_cast<char*>(ptr + count);
}

// The query state: everything sized by Q, P and the bin count.  Its layout is a function of (Q, P) alone, so the backward
// finds every array again.
struct FieldState {
	FieldGrid* grid; int* nitems; uint32_t* box;
	float4* recs; float4* ext; uint32_t* gcnt; unsigned long long* goff;
	uint32_t* qkey; uint32_t* qkey_sorted; uint32_t* qiota; uint32_t* qorder;
	uint2* qrange; uint2* grange; uint32_t* wcnt; uint32_t* woff; uint4* items;
	float4* ggeo;
	char* temp; size_t temp_bytes;
	static FieldState at(char* chunk, int Q, int P)
	{
		FieldState s;
		const int nb = field_bins(Q);
		carve(chunk, s.grid, 1);
		carve(chunk, s.nitems, 1);
		carve(chunk, s.box, 8);
		carve(chunk, s.recs, 4 * (size_t)P);
		carve(chunk, s.ext, P);
		carve(chunk, s.gcnt, P);
		carve(chunk, s.goff, P);
		carve(chunk, s.qkey, Q);
		carve(chunk, s.qkey_sorted, Q);
		carve(chunk, s.qiota, Q);
		carve(chunk, s.qorder, Q);
		carve(chunk, s.qrange, nb);
		carve(chunk, s.grange, nb);
		carve(chunk, s.wcnt, nb);
		carve(chunk, s.woff, nb);
		carve(chunk, s.items, field_items(Q));
		carve(chunk, s.ggeo, 4 * (size_t)P);
		s.temp_bytes = field_temp_bytes(Q, P);
		carve(chunk, s.temp, s.temp_bytes);
		return s;
	}
};

size_t field_state_bytes(int Q, int P)
{
	const FieldState s = FieldState::at(nullptr, Q, P);
	return (size_t)(s.temp + s.temp_bytes - (char*)nullptr) + 128;
}

// The pair state: the sorted Gaussian ids first (the only array the backward reads), then the sort's inputs and scratch.
struct PairState {
	uint32_t* vals_sorted; uint32_t* vals; uint32_t* keys; uint32_t* keys_sorted; char* temp; size_t temp_bytes;
	static PairState at(char* chunk, size_t n, int nb)
	{
		PairState s;
		carve(chunk, s.vals_sorted, n);
		carve(chunk, s.vals, n);
		carve(chunk, s.keys, n);
		carve(chunk, s.keys_sorted, n);
		s.temp_bytes = 0;
		cub::DeviceRadixSort::SortPairs(nullptr, s.temp_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
			(uint32_t*)nullptr, (int)n, 0, key_bits(nb));
		carve(chunk, s.temp, s.temp_bytes);
		return s;
	}
};

size_t field_pair_state_bytes(long long n, int Q)
{
	const PairState s = PairState::at(nullptr, (size_t)n, field_bins(Q));
	return (size_t)(s.temp + s.temp_bytes - (char*)nullptr) + 128;
}

#define FQ_TRY(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return e_; } while (0)

cudaError_t field_front(char* state, int Q, int P, const float* points, const float* means, const float* scales, const float* rot,
	const float* opac, unsigned long long* host_pairs, cudaStream_t st)
{
	const FieldState s = FieldState::at(state, Q, P);
	const int nb = field_bins(Q);
	FQ_TRY(cudaMemsetAsync(s.box, 0xff, 3 * sizeof(uint32_t), st));
	FQ_TRY(cudaMemsetAsync(s.box + 3, 0, 3 * sizeof(uint32_t), st));
	field_bbox_kernel<<<ceil_div(Q, 256), 256, 0, st>>>(Q, points, s.box);
	field_grid_kernel<<<1, 1, 0, st>>>(s.box, nb, s.grid);
	field_prep_kernel<<<ceil_div(P, 256), 256, 0, st>>>(P, means, scales, rot, opac, s.grid, s.recs, s.ext, s.gcnt);
	size_t tb = s.temp_bytes;
	FQ_TRY(cub::DeviceScan::InclusiveSum(s.temp, tb, U64It(s.gcnt, ToU64{}), s.goff, P, st));
	FQ_TRY(cudaMemcpyAsync(host_pairs, s.goff + P - 1, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
	// the queries, grouped by bin, and the warp items over them (independent of the pair count)
	field_query_keys_kernel<<<ceil_div(Q, 256), 256, 0, st>>>(Q, points, s.grid, s.qkey, s.qiota);
	tb = s.temp_bytes;
	FQ_TRY(cub::DeviceRadixSort::SortPairs(s.temp, tb, s.qkey, s.qkey_sorted, s.qiota, s.qorder, Q, 0, key_bits(nb), st));
	FQ_TRY(cudaMemsetAsync(s.qrange, 0, nb * sizeof(uint2), st));
	field_ranges_kernel<<<ceil_div(Q, 256), 256, 0, st>>>(Q, s.qkey_sorted, s.qrange);
	field_warp_count_kernel<<<ceil_div(nb, 256), 256, 0, st>>>(nb, s.qrange, s.wcnt);
	tb = s.temp_bytes;
	FQ_TRY(cub::DeviceScan::InclusiveSum(s.temp, tb, s.wcnt, s.woff, nb, st));
	field_items_kernel<<<ceil_div(nb, 256), 256, 0, st>>>(nb, s.qrange, s.wcnt, s.woff, s.items, s.nitems);
	return cudaGetLastError();
}

cudaError_t field_pairs(char* state, char* pair_state, int Q, int P, long long npairs, cudaStream_t st)
{
	const FieldState s = FieldState::at(state, Q, P);
	const int nb = field_bins(Q);
	FQ_TRY(cudaMemsetAsync(s.grange, 0, nb * sizeof(uint2), st));
	if (npairs == 0) return cudaGetLastError();
	const PairState ps = PairState::at(pair_state, (size_t)npairs, nb);
	field_emit_kernel<<<ceil_div(P, 256), 256, 0, st>>>(P, s.recs, s.ext, s.gcnt, s.goff, s.grid, ps.keys, ps.vals);
	size_t tb = ps.temp_bytes;
	FQ_TRY(cub::DeviceRadixSort::SortPairs(ps.temp, tb, ps.keys, ps.keys_sorted, ps.vals, ps.vals_sorted, (int)npairs, 0, key_bits(nb), st));
	field_ranges_kernel<<<ceil_div((int)npairs, 256), 256, 0, st>>>((int)npairs, ps.keys_sorted, s.grange);
	return cudaGetLastError();
}

bool feature_rows_vectorizable(const float* feature, int F);

static void fill_args(FieldArgs& a, char* state, char* pair_state, int Q, int P, int C)
{
	const FieldState s = FieldState::at(state, Q, P);
	a.Q = Q; a.P = P; a.C = C; a.groups = C > 32 ? ceil_div(C, 32) : 1;
	a.recs = s.recs; a.ext = s.ext; a.pairs = reinterpret_cast<const uint32_t*>((reinterpret_cast<uintptr_t>(pair_state) + 127) & ~(uintptr_t)127);  // PairState::vals_sorted
	 a.gbin = s.grange;
	a.qorder = s.qorder; a.items = s.items; a.nitems = s.nitems; a.ggeo = nullptr;
}

template <int NFT>
static void launch_fwd_t(const FieldArgs& a, dim3 grid, cudaStream_t st)
{
	if (NFT > 0 && feature_rows_vectorizable(a.features, a.C)) field_fwd_kernel<NFT, true><<<grid, 32, 0, st>>>(a);
	else field_fwd_kernel<NFT, false><<<grid, 32, 0, st>>>(a);
}

cudaError_t field_forward(char* state, char* pair_state, int Q, int P, int C, const float* points, const float* features,
	int channel_first, float* density, float* out_features, cudaStream_t st)
{
	FieldArgs a{};
	fill_args(a, state, pair_state, Q, P, C);
	a.points = points; a.features = C > 0 ? features : nullptr; a.channel_first = channel_first;
	a.density = density; a.out_features = C > 0 ? out_features : nullptr;
	const dim3 grid(field_items(Q), a.groups);
	if (a.groups > 1) launch_fwd_t<4>(a, grid, st);
	else switch (nft_for(C)) {
		case 0: launch_fwd_t<0>(a, grid, st); break;
		case 1: launch_fwd_t<1>(a, grid, st); break;
		case 2: launch_fwd_t<2>(a, grid, st); break;
		default: launch_fwd_t<4>(a, grid, st); break;
	}
	return cudaGetLastError();
}

template <int NFT, bool GRP>
static void launch_bwd_t(const FieldArgs& a, cudaStream_t st)
{
	// red_feature_row's vector path: 16-byte aligned rows with C % 4 == 0 (and whole tiles without groups); the feature
	// gather's: the same for the input rows
	const bool vec = NFT == 0 || (feature_rows_vectorizable(a.features, a.C) && (GRP || a.C == 8 * NFT) &&
		(!a.dL_dfeat || feature_rows_vectorizable(a.dL_dfeat, a.C)));
	if (vec) field_bwd_kernel<NFT, true, GRP><<<field_items(a.Q), 32, 0, st>>>(a);
	else field_bwd_kernel<NFT, false, GRP><<<field_items(a.Q), 32, 0, st>>>(a);
}

cudaError_t field_backward(char* state, char* pair_state, int Q, int P, int C, const float* points, const float* features,
	const float* scales, const float* rotations, int channel_first, const float* dL_ddensity, const float* dL_dfeatures,
	float* dL_dpoints, float* dL_dmeans, float* dL_dscales, float* dL_drot, float* dL_dopac, float* dL_dfeat, cudaStream_t st)
{
	FieldArgs a{};
	fill_args(a, state, pair_state, Q, P, C);
	const FieldState s = FieldState::at(state, Q, P);
	a.points = points; a.features = C > 0 ? features : nullptr; a.channel_first = channel_first;
	a.scales = scales; a.rotations = rotations;
	a.dL_ddensity = dL_ddensity; a.dL_dfeatures = C > 0 ? dL_dfeatures : nullptr;
	a.dL_dpoints = dL_dpoints; a.dL_dmeans = dL_dmeans; a.dL_dscales = dL_dscales; a.dL_drot = dL_drot; a.dL_dopac = dL_dopac;
	a.dL_dfeat = C > 0 ? dL_dfeat : nullptr;
	const bool geo = dL_dmeans || dL_dscales || dL_drot || dL_dopac;
	if (geo) {
		a.ggeo = s.ggeo;
		FQ_TRY(cudaMemsetAsync(s.ggeo, 0, 4 * (size_t)P * sizeof(float4), st));
	}
	if (a.dL_dfeat) FQ_TRY(cudaMemsetAsync(a.dL_dfeat, 0, (size_t)P * C * sizeof(float), st));
	const bool any_in = dL_ddensity || a.dL_dfeatures;
	if (dL_dpoints && !any_in) FQ_TRY(cudaMemsetAsync(dL_dpoints, 0, (size_t)Q * 3 * sizeof(float), st));
	if (any_in && (geo || dL_dpoints || (a.dL_dfeat && a.dL_dfeatures))) {
		if (a.groups > 1) launch_bwd_t<4, true>(a, st);
		else switch (nft_for(C)) {
			case 0: launch_bwd_t<0, false>(a, st); break;
			case 1: launch_bwd_t<1, false>(a, st); break;
			case 2: launch_bwd_t<2, false>(a, st); break;
			default: launch_bwd_t<4, false>(a, st); break;
		}
	}
	if (geo) field_bwd_gauss_kernel<<<ceil_div(P, 256), 256, 0, st>>>(a);
	return cudaGetLastError();
}

}  // namespace mgs
