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

}  // namespace mgs
