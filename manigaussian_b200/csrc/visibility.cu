// Point visibility: where query points land in a view and how much of the cloud lies in front of them
// (include/mgs_rasterizer.h, mgs_visibility_views).  For point x: (u, v) and d = t.z from screen_mean (camera.cuh: the projection's own map
// of a mean, every camera model), in_view, and T = prod (1 - alpha_i) over the instances of the 16x16 tile holding pixel
// (floor(u + 0.5), floor(v + 0.5)) in tile-list order with depth z_i < d, alpha_i at the continuous (u, v) with walk_alphas
// and the forward's T_STOP rule.  At a pixel centre with d behind the scene that is the pixel's final_T bit for bit.
//
// Decomposition, per view, behind the view's projection and binning (the forward's front end, unchanged):
//   points    one thread per point: uv, depth, in_view, T = 1, and the point's tile key (T_tiles for a point outside the view,
//             which sorts last);
//   group     a stable radix sort of (tile key, point id) on the tile bits, per-tile point ranges, and one CTA that scans the
//             per-tile warp counts ceil(n_t / 32) into item ends;
//   query     one warp per item, i.e. up to 32 points of one tile: each lane binary-searches its cut (the number of the tile's
//             instances with z_i < d; the list is in depth order, and the depth is read through point_list from the geometry
//             state's depths), then the warp walks the tile's records in chunks of 32, gathered with cp.async one chunk ahead
//             as the blends gather theirs, each lane over its own prefix, until every lane is past its cut or below T_STOP.
// The tile's full range is walked, not the 8x4 block lists: a block mask is exact at the block's pixel centres only, and the
// query positions are continuous.  A heavy tile (100^3 voxel centres put ~15k points into one tile of a 128^2 view) becomes
// hundreds of independent warps, so the time follows points x cut, not points per tile.
#include <cub/block/block_scan.cuh>
#include "blend_common.cuh"
#include "camera.cuh"

namespace mgs {

constexpr int VIS_CH = 32;             // records per chunk: one per lane
constexpr int VIS_WARPS = 4;           // warps per CTA of the query kernel
constexpr int VIS_SCAN_THREADS = 1024;

__global__ void __launch_bounds__(256) vis_points_kernel(VisArgs a)
{
	const int q = blockIdx.x * blockDim.x + threadIdx.x;
	if (q >= a.Q) return;
	const V3 p = { a.points[3 * (size_t)q], a.points[3 * (size_t)q + 1], a.points[3 * (size_t)q + 2] };
	float u, v;
	const bool ok = screen_mean(a.cam, p, u, v);
	float d = xform4x3(p, a.cam.viewmatrix).z;  // screen_mean's t.z
	const float nan = __int_as_float(0x7fffffff);
	if (!ok) u = v = d = nan;
	const bool in = ok && u >= -0.5f && u < a.W - 0.5f && v >= -0.5f && v < a.H - 0.5f;
	if (a.out_uv) { a.out_uv[2 * (size_t)q] = u; a.out_uv[2 * (size_t)q + 1] = v; }
	if (a.out_depth) a.out_depth[q] = d;
	if (a.out_in_view) a.out_in_view[q] = in ? 1 : 0;
	a.out_T[q] = 1.0f;
	uint32_t key = (uint32_t)a.num_tiles;
	if (in) {
		// u + 0.5 may round up to W at the last ulp below W - 0.5: the pixel stays the last column
		const int ix = min((int)floorf(u + 0.5f), a.W - 1), iy = min((int)floorf(v + 0.5f), a.H - 1);
		key = (uint32_t)((iy / TILE_Y) * a.grid_x + ix / TILE_X);
	}
	a.keys[q] = key;
	a.idx[q] = (uint32_t)q;
	a.pt[q] = make_float4(u, v, d, 0.f);
}

// per-tile ranges of the sorted points (qranges zeroed by the caller); points outside the view carry key num_tiles
__global__ void __launch_bounds__(256) vis_ranges_kernel(VisArgs a)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= a.Q) return;
	const uint32_t key = a.keys_sorted[i];
	if (key >= (uint32_t)a.num_tiles) return;
	if (i == 0 || a.keys_sorted[i - 1] != key) a.qranges[key].x = (uint32_t)i;
	if (i == a.Q - 1 || a.keys_sorted[i + 1] != key) a.qranges[key].y = (uint32_t)i + 1u;
}

// item_end[t] = sum over tiles s <= t of ceil(n_s / 32): warp w of the query works on the tile t with item_end[t - 1] <= w <
// item_end[t]
__global__ void __launch_bounds__(VIS_SCAN_THREADS) vis_items_kernel(VisArgs a)
{
	using Scan = cub::BlockScan<uint32_t, VIS_SCAN_THREADS>;
	__shared__ typename Scan::TempStorage tmp;
	__shared__ uint32_t carry;
	if (threadIdx.x == 0) carry = 0u;
	__syncthreads();
	for (int base = 0; base < a.num_tiles; base += VIS_SCAN_THREADS) {
		const int t = base + threadIdx.x;
		uint32_t n = 0;
		if (t < a.num_tiles) { const uint2 r = a.qranges[t]; n = (r.y - r.x + 31u) >> 5; }
		uint32_t incl, total;
		Scan(tmp).InclusiveSum(n, incl, total);
		const uint32_t c = carry;
		if (t < a.num_tiles) a.item_end[t] = c + incl;
		__syncthreads();
		if (threadIdx.x == 0) carry = c + total;
		__syncthreads();
	}
}

__global__ void __launch_bounds__(32 * VIS_WARPS) vis_query_kernel(VisArgs a)
{
	__shared__ __align__(16) float4 s_rec[VIS_WARPS][2][VIS_CH * 2];
	const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
	const uint32_t w = blockIdx.x * VIS_WARPS + wib;
	const int nt = a.num_tiles;
	if (w >= a.item_end[nt - 1]) return;
	// the item's tile: the first t with item_end[t] > w (warp-uniform)
	int lo = 0, hi = nt - 1;
	while (lo < hi) {
		const int mid = (lo + hi) >> 1;
		if (a.item_end[mid] > w) hi = mid; else lo = mid + 1;
	}
	const int tile = lo;
	const uint32_t first_item = tile ? a.item_end[tile - 1] : 0u;
	const uint2 qr = a.qranges[tile];
	const uint32_t p0 = qr.x + 32u * (w - first_item);
	const int n = (int)min(32u, qr.y - p0);
	const bool live = lane < n;
	const uint32_t q = live ? a.idx_sorted[p0 + lane] : 0u;
	const float4 pt = live ? a.pt[q] : make_float4(0.f, 0.f, 0.f, 0.f);
	// the cut: instances of the tile with depth < d form a prefix of its list (depth order); lower bound of d
	const uint2 range = a.ranges[tile];
	int cut = 0;
	if (live) {
		uint32_t l = range.x, h = range.y;
		while (l < h) {
			const uint32_t m = (l + h) >> 1;
			if (__ldg(a.depths + a.point_list[m]) < pt.z) l = m + 1; else h = m;
		}
		cut = (int)(l - range.x);
	}
	int maxcut = cut;
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) maxcut = max(maxcut, __shfl_xor_sync(0xffffffffu, maxcut, o));
	const InstRec* const recs = a.recs + range.x;
	float4 (*const buf2)[VIS_CH * 2] = s_rec[wib];
	// the forward's recurrence (blend_fwd_kernel): T runs over every evaluated pair, T_out is T after the last accepted one
	float T = 1.0f, T_out = 1.0f;
	if (lane < min(maxcut, VIS_CH)) gather_rec(buf2[0] + 2 * lane, recs + lane);
	cp_async_commit();
	for (int k0 = 0, buf = 0; k0 < maxcut; k0 += VIS_CH, buf ^= 1) {
		const float4* const s_q = buf2[buf];
		cp_async_wait<0>();
		__syncwarp();
		const int k1 = k0 + VIS_CH;
		if (lane < min(maxcut - k1, VIS_CH)) gather_rec(buf2[buf ^ 1] + 2 * lane, recs + k1 + lane);
		cp_async_commit();
		const int cnt = max(0, min(cut - k0, VIS_CH));  // this lane's pairs of the chunk
		const int nks = (min(maxcut - k0, VIS_CH) + 7) >> 3;
		for (int ks = 0; ks < nks; ks++) {
			if (__all_sync(0xffffffffu, 8 * ks >= cnt || T < T_STOP)) break;
			float al[8];
			walk_alphas(s_q + 16 * ks, pt.x, pt.y, ks, cnt, al);
#pragma unroll
			for (int u = 0; u < 8; u++) {
				const float test_T = T * (1 - al[u]);
				T_out = !(test_T < T_STOP) ? test_T : T_out;
				T = test_T;
			}
		}
		__syncwarp();  // the buffer is refilled two chunks on
		if (__all_sync(0xffffffffu, k1 >= cut || T < T_STOP)) break;
	}
	cp_async_wait<0>();  // no record copy may be in flight when the warp exits
	if (live) a.out_T[q] = T_out;
}

// ---- backward (include/mgs_rasterizer.h, mgs_visibility_views_backward) ----
//   query     the query kernel's grid, items, cut and cp.async chunk walk, with the same walk_alphas and recurrence, so every
//             lane replays its point's decisions bit for bit.  T_out, the forward's T, is read from out_T: for an accepted
//             pair dL/dalpha_i = -dL/dT T_out / (1 - alpha_i), with dL/dG = o dL/dalpha (no mask for the 0.99 clamp) and
//             dL/do = G dL/dalpha.  Per k-step the 8 records' six blend-stage terms are summed over the warp's lanes by
//             recursive halving (31 shuffles for 32 values), and one lane per record sends them to gb with a v4 and a v2
//             reduction: one global reduction per (warp item, record), none per (point, Gaussian).  dL/duv of each point
//             (dG/duv = -dG/dmu) stays in its lane and is stored once.
//   points    one thread per point over the call's views in order (vis_points_bwd_kernel).

// red.global.add of two floats (8-byte aligned)
__device__ __forceinline__ void red_add_v2(float* addr, float a, float b)
{
	asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

// recursive halving of x[0 .. 2H) over the warp: afterwards x[0 .. H) holds sums over lane pairs (l, l ^ H), the upper half
// on the lanes with bit H set.  After H = 16, 8, 4, 2, 1 lane l holds the warp's sum of value l in x[0], in a fixed order.
template <int H>
__device__ __forceinline__ void vis_halve(float* x, int lane)
{
	const bool up = (lane & H) != 0;
#pragma unroll
	for (int k = 0; k < H; k++) {
		const float send = up ? x[k] : x[k + H], keep = up ? x[k + H] : x[k];
		x[k] = keep + __shfl_xor_sync(0xffffffffu, send, H);
	}
}

__global__ void __launch_bounds__(32 * VIS_WARPS) vis_query_bwd_kernel(VisQueryBwdArgs b)
{
	const VisArgs& a = b.f;
	__shared__ __align__(16) float4 s_rec[VIS_WARPS][2][VIS_CH * 2];
	const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
	const uint32_t w = blockIdx.x * VIS_WARPS + wib;
	const int nt = a.num_tiles;
	if (w >= a.item_end[nt - 1]) return;
	int lo = 0, hi = nt - 1;
	while (lo < hi) {
		const int mid = (lo + hi) >> 1;
		if (a.item_end[mid] > w) hi = mid; else lo = mid + 1;
	}
	const int tile = lo;
	const uint32_t first_item = tile ? a.item_end[tile - 1] : 0u;
	const uint2 qr = a.qranges[tile];
	const uint32_t p0 = qr.x + 32u * (w - first_item);
	const int n = (int)min(32u, qr.y - p0);
	const bool live = lane < n;
	const uint32_t q = live ? a.idx_sorted[p0 + lane] : 0u;
	const float4 pt = live ? a.pt[q] : make_float4(0.f, 0.f, 0.f, 0.f);
	// dL/dalpha_i = s / (1 - alpha_i); a lane with s = 0 has nothing to send and walks nothing
	const float s = live ? -b.dL_dT[q] * a.out_T[q] : 0.f;
	const uint2 range = a.ranges[tile];
	int cut = 0;
	if (live && s != 0.f) {
		uint32_t l = range.x, h = range.y;
		while (l < h) {
			const uint32_t m = (l + h) >> 1;
			if (__ldg(a.depths + a.point_list[m]) < pt.z) l = m + 1; else h = m;
		}
		cut = (int)(l - range.x);
	}
	int maxcut = cut;
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) maxcut = max(maxcut, __shfl_xor_sync(0xffffffffu, maxcut, o));
	const InstRec* const recs = a.recs + range.x;
	float4 (*const buf2)[VIS_CH * 2] = s_rec[wib];
	const float half_W = 0.5f * a.W, half_H = 0.5f * a.H;
	float T = 1.0f, gu = 0.f, gv = 0.f;
	if (lane < min(maxcut, VIS_CH)) gather_rec(buf2[0] + 2 * lane, recs + lane);
	cp_async_commit();
	for (int k0 = 0, buf = 0; k0 < maxcut; k0 += VIS_CH, buf ^= 1) {
		const float4* const s_q = buf2[buf];
		cp_async_wait<0>();
		__syncwarp();
		const int k1 = k0 + VIS_CH;
		if (lane < min(maxcut - k1, VIS_CH)) gather_rec(buf2[buf ^ 1] + 2 * lane, recs + k1 + lane);
		cp_async_commit();
		const int cnt = max(0, min(cut - k0, VIS_CH));
		const int nrec = min(maxcut - k0, VIS_CH);  // records of the chunk in shared memory
		const int nks = (nrec + 7) >> 3;
		for (int ks = 0; ks < nks; ks++) {
			if (__all_sync(0xffffffffu, 8 * ks >= cnt || T < T_STOP)) break;
			float al[8];
			walk_alphas(s_q + 16 * ks, pt.x, pt.y, ks, cnt, al);
			// per record u: {dmx, dmy, dca, dcb} at 4 u and {dcc, dop} at 2 u, in the blend backward's units
			float ga[32], gc[16];
			bool any = false;
#pragma unroll
			for (int u = 0; u < 8; u++) {
				const float test_T = T * (1 - al[u]);
				const bool acc = al[u] > 0.f && !(test_T < T_STOP);  // the forward's accepted pairs
				T = test_T;
				float m = 0.f, gx = 0.f, gy = 0.f, dx = 0.f, dy = 0.f, dop = 0.f;
				if (acc) {
					const float4 p = s_q[16 * ks + 2 * u], r = s_q[16 * ks + 2 * u + 1];
					dx = p.x - pt.x; dy = p.y - pt.y;
					const float G = expf(-0.5f * (p.z * dx * dx + r.x * dy * dy) - p.w * dx * dy);
					dop = G * (s / (1.f - al[u]));  // dL/do
					m = r.y * dop;                  // dL/dpower
					gx = -(p.z * dx + p.w * dy);    // dpower/dmu
					gy = -(r.x * dy + p.w * dx);
					any = true;
				}
				gu -= m * gx; gv -= m * gy;
				ga[4 * u] = half_W * m * gx; ga[4 * u + 1] = half_H * m * gy;
				ga[4 * u + 2] = -0.5f * m * dx * dx; ga[4 * u + 3] = -0.5f * m * dx * dy;
				gc[2 * u] = -0.5f * m * dy * dy; gc[2 * u + 1] = dop;
			}
			if (!b.gb || !__any_sync(0xffffffffu, any)) continue;
			vis_halve<16>(ga, lane); vis_halve<8>(ga, lane); vis_halve<4>(ga, lane); vis_halve<2>(ga, lane); vis_halve<1>(ga, lane);
#pragma unroll
			for (int k = 0; k < 16; k++) gc[k] += __shfl_xor_sync(0xffffffffu, gc[k], 16);
			vis_halve<8>(gc, lane); vis_halve<4>(gc, lane); vis_halve<2>(gc, lane); vis_halve<1>(gc, lane);
			// lane 4 u + t holds term t of record u, lane 2 u + t (and 16 + 2 u + t) term 4 + t
			const float a1 = __shfl_down_sync(0xffffffffu, ga[0], 1), a2 = __shfl_down_sync(0xffffffffu, ga[0], 2);
			const float a3 = __shfl_down_sync(0xffffffffu, ga[0], 3), c1 = __shfl_down_sync(0xffffffffu, gc[0], 1);
			const int ua = lane >> 2, uc = (lane & 15) >> 1;
			if ((lane & 3) == 0 && 8 * ks + ua < nrec && (ga[0] != 0.f || a1 != 0.f || a2 != 0.f || a3 != 0.f))
				red_add_v4(b.gb + (size_t)rec_id(s_q[16 * ks + 2 * ua + 1]) * GB_STRIDE, ga[0], a1, a2, a3);
			if (lane < 16 && (lane & 1) == 0 && 8 * ks + uc < nrec && (gc[0] != 0.f || c1 != 0.f))
				red_add_v2(b.gb + (size_t)rec_id(s_q[16 * ks + 2 * uc + 1]) * GB_STRIDE + 4, gc[0], c1);
		}
		__syncwarp();  // the buffer is refilled two chunks on
		if (__all_sync(0xffffffffu, k1 >= cut || T < T_STOP)) break;
	}
	cp_async_wait<0>();  // no record copy may be in flight when the warp exits
	if (live && b.duv) { b.duv[2 * (size_t)q] = gu; b.duv[2 * (size_t)q + 1] = gv; }
}

// CAM: the launch writes camera rows, summed over the warp by shuffles in a fixed order, then over the CTA's warps in warp
// order, as flow_bwd_kernel's.  dL/dpoints sums the views in view order in registers.
template <bool CAM>
__global__ void __launch_bounds__(VIS_PTS_BWD_THREADS) vis_points_bwd_kernel(VisPointsBwdArgs a)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	const bool in = i < a.Q;
	const size_t q = in ? (size_t)i : 0;
	__shared__ float cam_sm[CAM ? VIS_PTS_BWD_THREADS / 32 * CAM_ALL_TERMS : 1];
	const float p[3] = { a.points[3 * q], a.points[3 * q + 1], a.points[3 * q + 2] };
	float gp[3] = { 0.f, 0.f, 0.f };
	for (int v = 0; v < a.V; v++) {
		const VisPointsBwdView& w = a.view[v];
		float cg[CAM ? CAM_ALL_TERMS : 1];
		if constexpr (CAM) {
#pragma unroll
			for (int k = 0; k < CAM_ALL_TERMS; k++) cg[k] = 0.f;
		}
		float u, vv;
		// where the cull fails uv and depth are NaN constants: their cotangents are ignored; a non-finite point (whose outputs
		// are NaN whatever the cull says) receives nothing either
		if (in && isfinite(p[0] + p[1] + p[2]) && screen_mean(w.cam, V3{ p[0], p[1], p[2] }, u, vv)) {
			float gx = 0.f, gy = 0.f;
			if (w.dL_duv) { gx = w.dL_duv[2 * q]; gy = w.dL_duv[2 * q + 1]; }
			if (w.duv) { gx += w.duv[2 * q]; gy += w.duv[2 * q + 1]; }
			flow_mean_bwd<CAM>(w.cam, p, gx, gy, gp, cg);
			if (w.dL_ddepth) {
				// d = t.z = vm[2] p0 + vm[6] p1 + vm[10] p2 + vm[14]
				const float gd = w.dL_ddepth[q];
				const float* vm = w.cam.viewmatrix;
#pragma unroll
				for (int k = 0; k < 3; k++) gp[k] += vm[4 * k + 2] * gd;
				if constexpr (CAM) {
#pragma unroll
					for (int k = 0; k < 3; k++) cg[3 * k + 2] += gd * p[k];
					cg[11] += gd;
				}
			}
		}
		if constexpr (CAM) {
			if (w.cam_rows) {
				const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
				for (int k = 0; k < CAM_ALL_TERMS; k++) {
					float s = cg[k];
#pragma unroll
					for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
					if (lane == 0) cam_sm[warp * CAM_ALL_TERMS + k] = s;
				}
				__syncthreads();
				for (int k = threadIdx.x; k < CAM_ALL_TERMS; k += blockDim.x) {
					float s = 0.f;
					for (int u2 = 0; u2 < VIS_PTS_BWD_THREADS / 32; u2++) s += cam_sm[u2 * CAM_ALL_TERMS + k];
					if (k < CAM_TERMS) w.cam_rows[(size_t)blockIdx.x * CAM_TERMS + k] = s;
					else if (w.intr_rows) w.intr_rows[(size_t)blockIdx.x * CAM_INTR_TERMS + k - CAM_TERMS] = s;
				}
				__syncthreads();
			}
		}
	}
	if (!in || !a.dL_dpoints) return;
	float* o = a.dL_dpoints + 3 * q;
#pragma unroll
	for (int k = 0; k < 3; k++) o[k] = a.accumulate ? o[k] + gp[k] : gp[k];
}

void launch_visibility_points(const VisArgs& a, cudaStream_t s)
{
	if (a.Q > 0) vis_points_kernel<<<ceil_div(a.Q, 256), 256, 0, s>>>(a);
}

void launch_visibility_group(const VisArgs& a, cudaStream_t s)
{
	if (a.Q <= 0) return;
	cudaMemsetAsync(a.qranges, 0, sizeof(uint2) * (size_t)a.num_tiles, s);
	vis_ranges_kernel<<<ceil_div(a.Q, 256), 256, 0, s>>>(a);
	vis_items_kernel<<<1, VIS_SCAN_THREADS, 0, s>>>(a);
}

void launch_visibility_query(const VisArgs& a, cudaStream_t s)
{
	if (a.Q <= 0) return;
	// at most one partial item per tile beside the full ones; warps past the item count return at once
	const int warps = ceil_div(a.Q, 32) + a.num_tiles;
	vis_query_kernel<<<ceil_div(warps, VIS_WARPS), 32 * VIS_WARPS, 0, s>>>(a);
}

void launch_visibility_query_bwd(const VisQueryBwdArgs& a, cudaStream_t s)
{
	if (a.f.Q <= 0) return;
	const int warps = ceil_div(a.f.Q, 32) + a.f.num_tiles;
	vis_query_bwd_kernel<<<ceil_div(warps, VIS_WARPS), 32 * VIS_WARPS, 0, s>>>(a);
}

void launch_visibility_points_bwd(const VisPointsBwdArgs& a, cudaStream_t s)
{
	if (a.Q <= 0 || a.V <= 0) return;
	bool cam = false;
	for (int v = 0; v < a.V; v++) cam |= a.view[v].cam_rows != nullptr;
	const int grid = ceil_div(a.Q, VIS_PTS_BWD_THREADS);
	if (cam) vis_points_bwd_kernel<true><<<grid, VIS_PTS_BWD_THREADS, 0, s>>>(a);
	else vis_points_bwd_kernel<false><<<grid, VIS_PTS_BWD_THREADS, 0, s>>>(a);
}

}  // namespace mgs
