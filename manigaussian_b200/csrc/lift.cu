// Lift: per-Gaussian sums of a 2D map weighted by the forward blend's own weights (include/mgs_rasterizer.h, mgs_lift_views):
//   lifted[g][c] += sum_p w_pg map[c][p],   weight[g] += sum_p w_pg,   w_pg = alpha T of Gaussian g at pixel p.
// lifted is dL/dfeature of a feature render with cotangent `map`, without the backward's replay, S recurrence, moments or
// per-Gaussian chain rule: the forward's walk produces w, and the backward's GEMM 2 and feature flush are the transposed
// contraction and its per-Gaussian reduction.
//
// Design: one single-warp CTA per 8x4 pixel block and channel group, indexed as blend_fwd_kernel's (longest tile lists first,
// the group varying faster than the rank).  Per chunk of LIFT_CH block-list entries:
//   walk      lane = pixel: the forward's walk (the same record gather, walk_alphas and transmittance recurrence, the same
//             early exit once every pixel of the block has stopped), so w is bit for bit the weight blend_fwd blends with.
//             The weights go to the backward's wgt layout [pi][j >> 1][e][j & 1] (pixel 2 pi + e, entry j), not the
//             forward's [tig][gid][mt][e][h]: the transposed GEMM's A quads (M = entries, K = pixels) are then one LDS.128;
//   contract  L[j][ch] = sum_p w[j][p] map[p][ch] on the tensor cores (gemm2_step, m16n8k8 TF32 with the 3xTF32 split).  The
//             block's map rows are the same for every chunk: staged once per CTA in the backward's cotangent layout
//             [pi][ch][e].  Column 0 of the {r,g,b,depth} tile holds 1 (group 0), so the MMAs issued anyway yield weight;
//   flush     per entry that contributed to a pixel of the block (ballot of the walk): the feature row into lifted + id C + 32 g
//             with the backward's red.global.add.v4.f32 pattern (red_feature_row), group 0 also red_add(weight + id).
// Nothing of the view's state is written: no pixel masks, block_nwalk, final_T or n_contrib.
#include "../../include/mgs_rasterizer.h"
#include "blend_common.cuh"
#include "blend_mma.cuh"

namespace mgs {

#ifndef MGS_LIFT_MIN_CTAS
#define MGS_LIFT_MIN_CTAS 16
#endif
constexpr int LIFT_CH = 32;  // block-list entries per chunk: two 16-row M tiles, as the forward's FWD_CH

// NFT: 8-wide map-channel tiles of the group (0, 1, 2, 4); VEC: whole 16-byte pieces of lifted rows (red.v4); GRP: C > 32.
template <int NFT, bool VEC, bool GRP>
__global__ void __launch_bounds__(32, MGS_LIFT_MIN_CTAS) lift_kernel(LiftArgs a)
{
	constexpr int NT = NFT + 1;           // column tiles: NFT map tiles + {1, 0 x 7}
	constexpr int CHP = 8 * NT;           // padded channel count
	constexpr int RGBD = 8 * NFT;         // the constant column's tile
	constexpr int GS = 2 * CHP;           // s_g stride per pixel pair
	constexpr int XS = 2 * LIFT_CH + 4;   // s_w stride per pixel pair (+4: spreads the pairs over the banks)
	constexpr int MT = LIFT_CH / 16;      // 16-row tiles of entries
	__shared__ __align__(16) float4 s_rec[2][LIFT_CH * 2];  // records of the current and the next chunk
	__shared__ __align__(16) float s_w[16 * XS];            // blend weights [pi][j >> 1][e][j & 1]
	__shared__ __align__(16) float s_g[16 * GS];            // map rows of the block's pixels [pi][ch][e]
	__shared__ uint32_t s_pm[LIFT_CH];                      // per entry: the pixels of the block it contributed to

	const int lane = threadIdx.x;
	const int gid = lane >> 2, tig = lane & 3;
	const int sub = blockIdx.x & 7;
	const int grp = GRP ? (int)(blockIdx.x >> 3) % a.groups : 0;
	const int rank = GRP ? (int)(blockIdx.x >> 3) / a.groups : (int)(blockIdx.x >> 3);
	const int tile = a.tile_order ? (int)a.tile_order[rank] : rank;  // longest lists first
	const int tile_x = tile % a.grid_x, tile_y = tile / a.grid_x;
	const int bx0 = tile_x * TILE_X + (sub & 1) * WARP_BX;
	const int by0 = tile_y * TILE_Y + (sub >> 1) * WARP_BY;
	const int pxi = bx0 + (lane >> 2), pyi = by0 + (lane & 3);  // walk role: lane = pixel (x = lane >> 2, y = lane & 3)
	const bool inside = pxi < a.W && pyi < a.H;
	if (__all_sync(0xffffffffu, !inside)) return;  // block entirely outside the image
	const int count = (int)a.block_count[8 * tile + sub];
	if (count == 0) return;
	const float pfx = (float)pxi, pfy = (float)pyi;
	const size_t HW = (size_t)a.H * a.W;
	const size_t pix = inside ? (size_t)a.W * pyi + pxi : 0;
	const int C = a.C;
	const int c0 = 32 * grp;                   // first channel of the group
	const int Cg = GRP ? min(C - c0, 32) : C;  // channels of the group
	const bool first = grp == 0;               // group 0 also sums weight

	// ---- the block's map rows, once: element (pixel 2 pi + e, channel ch) at [pi][ch][e]; pixels outside the image hold 0
	// (their weights are 0 too: T starts at 0 there) ----
	{
		float* grow = s_g + (lane >> 1) * GS + (lane & 1);
#pragma unroll
		for (int c = 0; c < 8; c++) grow[2 * (RGBD + c)] = (c == 0 && first && inside) ? 1.f : 0.f;
#pragma unroll
		for (int i = 0; i < 8 * NFT; i++) grow[2 * i] = (inside && i < Cg) ? __ldg(a.map + (size_t)(c0 + i) * HW + pix) : 0.f;
	}

	const uint2 range = a.ranges[tile];
	const InstRec* const recs = a.recs + range.x;                                  // the tile's records, by 0-based list position
	const uint32_t* const lrow = a.block_list + sub * a.mask_stride + range.x;    // this block's work list
	float T = inside ? 1.0f : 0.0f;  // the forward's running product (blend_fwd_kernel)
	const int xofs = (lane >> 1) * XS + (lane & 1) * 2;  // this pixel's slot in the [pi][j >> 1][e][j & 1] tile

	uint32_t pos = lane < min(count, LIFT_CH) ? lrow[lane] : 0u;
	if (lane < min(count, LIFT_CH)) gather_rec(s_rec[0] + 2 * lane, recs + pos);
	cp_async_commit();
	pos = lane < min(count - LIFT_CH, LIFT_CH) ? lrow[LIFT_CH + lane] : 0u;
	for (int k0 = 0, buf = 0; k0 < count; k0 += LIFT_CH, buf ^= 1) {
		const int cnt = min(count - k0, LIFT_CH);
		const float4* const s_q = s_rec[buf];
		cp_async_wait<0>();  // this chunk's records
		__syncwarp();
		// ---- the next chunk's records travel while this chunk runs ----
		const int k1 = k0 + LIFT_CH;
		if (lane < min(count - k1, LIFT_CH)) gather_rec(s_rec[buf ^ 1] + 2 * lane, recs + pos);
		cp_async_commit();
		pos = lane < min(count - k1 - LIFT_CH, LIFT_CH) ? lrow[k1 + LIFT_CH + lane] : 0u;
		// ---- walk: the forward's, one k-step of 8 entries per trip ----
		const int nks = (cnt + 7) >> 3;
		int ks = 0;
		for (; ks < nks; ks++) {
			if (ks > 0 && __all_sync(0xffffffffu, T < T_STOP)) break;
			float al[8];
			walk_alphas(s_q + 16 * ks, pfx, pfy, ks, cnt, al);
#pragma unroll
			for (int u = 0; u < 8; u++) {
				const float alpha = al[u];
				const float test_T = T * (1 - alpha);
				const bool use = !(test_T < T_STOP);  // as blend_fwd_kernel: a skipped pair passes with zero weight
				s_w[xofs + 16 * ks + (u >> 1) * 4 + (u & 1)] = use ? alpha * T : 0.f;
				T = test_T;
				s_pm[8 * ks + u] = __ballot_sync(0xffffffffu, use && alpha != 0.f);
			}
		}
		// entries of the k-steps the walk did not reach (every pixel had stopped) contributed nothing: their rows of the
		// weight tile are stale, and the flush skips them
		const int nwalked = 8 * ks;
		__syncwarp();
		// ---- contract: L[j][ch] = w[j][:] . map[:][ch]   (M = entries, K = pixels, N = channels) ----
		float dC[MT][NT][4];
#pragma unroll
		for (int mt = 0; mt < MT; mt++)
#pragma unroll
			for (int nt = 0; nt < NT; nt++)
#pragma unroll
				for (int i = 0; i < 4; i++) dC[mt][nt][i] = 0.f;
#pragma unroll
		for (int kp = 0; kp < 4; kp++) {
			// A quads: pixel pair pi = 4 kp + tig, entries 16 mt + 2 gid (+1)
			uint32_t ahi[MT][4], alo[MT][4];
#pragma unroll
			for (int mt = 0; mt < MT; mt++) {
				const float4 w4 = *reinterpret_cast<const float4*>(s_w + (4 * kp + tig) * XS + mt * 32 + gid * 4);
				tf32_split(w4.x, ahi[mt][0], alo[mt][0]); tf32_split(w4.y, ahi[mt][1], alo[mt][1]);
				tf32_split(w4.z, ahi[mt][2], alo[mt][2]); tf32_split(w4.w, ahi[mt][3], alo[mt][3]);
			}
			gemm2_step<NFT, MT>(dC, ahi, alo, s_g + (4 * kp + tig) * GS, gid, first);
		}
		// ---- flush: D rows gid (h = 0) and gid + 8 (h = 1) of tile mt are entries 16 mt + 2 gid + h ----
#pragma unroll
		for (int mt = 0; mt < MT; mt++) {
#pragma unroll
			for (int h = 0; h < 2; h++) {
				const int j = 16 * mt + 2 * gid + h;
				if (j < nwalked && s_pm[j] != 0u) {
					const uint32_t id = rec_id(s_q[2 * j + 1]);
					if (NFT > 0) red_feature_row<NFT, VEC, GRP>(a.lifted + (size_t)id * C + c0, dC[mt], h, tig, Cg);
					if (first && tig == 0) red_add(a.weight + id, dC[mt][NFT][2 * h]);  // column 0 of the constant tile
				}
			}
		}
		__syncwarp();  // s_w and s_pm are rewritten by the next chunk
		if (__all_sync(0xffffffffu, T < T_STOP)) break;  // every pixel of the block is finished
	}
	cp_async_wait<0>();  // no record copy may be in flight when the CTA exits
}

int blend_groups(int F);
bool feature_rows_vectorizable(const float* feature, int F);

template <int NFT, bool GRP>
static void launch_lift_t(const LiftArgs& a, cudaStream_t s)
{
	const int grid = a.grid_x * a.grid_y * 8 * a.groups;
	// whole 16-byte pieces of the lifted rows: an exact tile width (or a group of 32 whose rows start 16-byte aligned when
	// C % 4 == 0), else the scalar reductions of the padded path, as in the blends
	const bool vec = (NFT == 0) || ((a.C == 8 * NFT || GRP) && feature_rows_vectorizable(a.lifted, a.C));
	if (vec) lift_kernel<NFT, true, GRP><<<grid, 32, 0, s>>>(a);
	else lift_kernel<NFT, false, GRP><<<grid, 32, 0, s>>>(a);
}

void launch_lift(const LiftArgs& a, cudaStream_t s)
{
	if (a.grid_x * a.grid_y == 0) return;
	if (a.groups > 1) { launch_lift_t<4, true>(a, s); return; }
	switch (nft_for(a.C)) {
	case 0: launch_lift_t<0, false>(a, s); break;
	case 1: launch_lift_t<1, false>(a, s); break;
	case 2: launch_lift_t<2, false>(a, s); break;
	default: launch_lift_t<4, false>(a, s); break;
	}
}

}  // namespace mgs
