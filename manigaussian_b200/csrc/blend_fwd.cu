// Forward blend: front-to-back alpha compositing of RGB + depth + F feature channels.
//
// Replaces FORWARD::render / renderCUDA<3,F> (DGR/cuda_rasterizer/forward.cu:262-398) behind the C-ABI.
// Same per-pixel semantics (power > 0 skip, alpha = min(0.99, o*exp(power)), alpha < 1/255 skip, stop
// when T*(1-alpha) < 1e-4, colour gets + T*bg, features/depth do not; final_T and n_contrib saved).
//
// Design (not the reference's; see blend_common.cuh for the decomposition):
//  * one single-warp CTA per 8x4 pixel block; the warp walks its block's work list (the instances whose per-Gaussian
//    alpha >= 1/255 footprint can reach the block, built by the binning stage) in chunks of FWD_CH, gathering each
//    chunk's records by list position with cp.async while the previous chunk runs;
//  * every chunk runs in two phases:
//      walk       lane = pixel, sequential over the chunk's survivors: the exact transmittance recurrence of the
//                 reference (same expf, same skip/stop tests, so final_T and n_contrib agree bit for bit); instead of
//                 36 channel FMAs per survivor (7 of 32 lanes active on the benchmark cloud) the lane only stores its
//                 blend weight w = alpha*T (0 when the pair does not contribute) into a [survivor][pixel] tile; one
//                 ballot per survivor records which pixels of the block it contributed to (pix_mask, per block-list
//                 entry), so the backward replays these decisions instead of re-deriving them;
//      contract   acc[pixel][channel] += W[pixel][survivor] * C[survivor][channel] on the tensor cores (mma.sync
//                 m16n8k8 TF32, 3xTF32 split for fp32 accuracy, blend_mma.cuh), accumulators in the D fragments;
//    the channel rows C of the chunk ({r,g,b,depth} quad + feature row, gathered by Gaussian id with 16-byte cp.async
//    pieces, SASS LDGSTS) travel while the walk runs;
//  * index assignment that lets every MMA operand arrive in place (an A fragment is four consecutive registers, and a
//    register move per fragment would cost more than the MMA saves): MMA row 16 mt + 8 h + gid is pixel (x = gid,
//    y = 2 mt + h) = lane 4 gid + y of the walk, and the weight tile is stored per k-step as [tig][gid][mt][e][h]
//    (survivor 8 ks + tig + 4 e), so {a0..a3} of one 16-pixel tile is ONE LDS.128 and the hi/lo split writes the second
//    quad; the B pair {b0, b1} (survivors g0, g1, feature 8 nt + gid) is two conflict-free scalar loads of the channel rows;
//    with x = gid the output planes are written as full 32-byte sectors straight from the D fragments.
#include "../../include/mgs_rasterizer.h"
#include "blend_common.cuh"
#include "blend_mma.cuh"
#include "loss_heads.cuh"

namespace mgs {

#ifndef MGS_FWD_CH
#define MGS_FWD_CH 32
#endif
#ifndef MGS_FWD_MIN_CTAS
#define MGS_FWD_MIN_CTAS 14
#endif
constexpr int FWD_CH = MGS_FWD_CH;        // block-list entries per tensor-core chunk (multiple of 8, <= 32)
static_assert(FWD_CH % 8 == 0 && FWD_CH <= 32, "forward chunk size");

// GRP: F > 32, channel groups (BlendArgs::groups); the F <= 32 instantiations carry none of the group arithmetic.
// DM: the depth / mask heads (BlendArgs::tgt_depth / tgt_mask); the instantiations without them keep their registers.
// MED: the median contributor (BlendArgs::median_id / out_median_depth); likewise.
// NRM: the normal plane (BlendArgs::nrm / out_normal): the per-Gaussian quad {nx, ny, nz, 0} fills columns 4..7 of the
// {r,g,b,depth} tile, zero padding otherwise, so the MMAs the kernel issues anyway blend it; likewise.
// PLN: planar depth (BlendArgs::planar): the quad {a, b, e, 0} fills the same columns, and the depth is col3 + px col4 +
// py col5 + col6 (also for the depth / mask heads); the median depth is its contributor's z + a px + b py + e; likewise.
template <int NFT, bool VEC, bool GRP, bool DM, bool MED, bool NRM, bool PLN>
__global__ void __launch_bounds__(32, MGS_FWD_MIN_CTAS) blend_fwd_kernel(BlendArgs a)
{
	using L = RowLayout<NFT>;
	constexpr int RS = L::RS;
	constexpr int NT = NFT + 1;  // column tiles: NFT feature tiles + the {r,g,b,depth} tile
	__shared__ __align__(16) float4 s_rec[2][FWD_CH * 2];  // records of the current and the next chunk: {x,y,ca,cb}, {cc,op,mask,id}
	__shared__ __align__(16) float s_rows[FWD_CH * RS];   // channel rows of the current chunk
	__shared__ __align__(16) float s_w[FWD_CH * 32];      // blend weights, per k-step [tig][gid][mt][e][h]: survivor 8 ks + tig + 4 e, pixel 4 gid + 2 mt + h
	__shared__ uint32_t s_pm[FWD_CH];                     // pixel masks of the chunk's entries, staged for one coalesced store

#ifdef MGS_CTA_LOG
	const unsigned long long t_start = cta_log_now();
#endif
	const int lane = threadIdx.x;
	const int gid = lane >> 2, tig = lane & 3;
	const int sub = blockIdx.x & 7;
	// channel group (BlendArgs::groups): the walk is deterministic, so every group's CTA derives the same weights w = alpha T
	const int grp = GRP ? (int)(blockIdx.x >> 3) % a.groups : 0;
	const int rank = GRP ? (int)(blockIdx.x >> 3) / a.groups : (int)(blockIdx.x >> 3);
	const int tile = a.tile_order ? (int)a.tile_order[rank] : rank;  // longest lists first
	const int tile_x = tile % a.grid_x, tile_y = tile / a.grid_x;
	const int bx0 = tile_x * TILE_X + (sub & 1) * WARP_BX;
	const int by0 = tile_y * TILE_Y + (sub >> 1) * WARP_BY;
	// walk role: lane = pixel (x = lane >> 2, y = lane & 3)
	const int pxi = bx0 + (lane >> 2), pyi = by0 + (lane & 3);
	const bool inside = pxi < a.W && pyi < a.H;
	if (__all_sync(0xffffffffu, !inside)) return;  // block entirely outside the image (ragged right/bottom tiles); the backward skips it too
	const float pfx = (float)pxi, pfy = (float)pyi;
	const int F = a.F;                 // feature row stride
	const int c0 = 32 * grp;           // first channel of the group
	const int Fg = GRP ? min(F - c0, 32) : F;  // channels of the group
	const bool first = grp == 0;       // group 0 also blends {r,g,b,depth} and writes the per-pixel state

	// rows beyond a short last chunk are multiplied by zero weights: they must hold finite numbers
	for (int i = lane; i < FWD_CH * RS / 4; i += 32) reinterpret_cast<float4*>(s_rows)[i] = make_float4(0.f, 0.f, 0.f, 0.f);

	const uint2 range = a.ranges[tile];
	const InstRec* const recs = a.recs + range.x;                                  // the tile's records, by 0-based list position
	const uint32_t* const lrow = a.block_list + sub * a.mask_stride + range.x;    // this block's work list
	uint32_t* const mrow = a.pix_mask + sub * a.mask_stride + range.x;            // pixel masks, by block-list entry
	const int count = (int)a.block_count[8 * tile + sub];
	// T is the running product of (1 - alpha) over every evaluated pair, the stopping pair included: the product only
	// shrinks, so once one test T (1 - alpha) < 1e-4 has failed every later one fails too and no "done" flag has to sit
	// in the recurrence (the reference stops looking at that point; here the later pairs get zero weight).  T_out is the
	// transmittance after the last accepted pair = the reference's final T.  Pixels outside the image start at 0.
	float T = inside ? 1.0f : 0.0f, T_out = 1.0f;
	uint32_t last = 0;  // 1-based block-list entry of this pixel's last contributor
	uint32_t med = 0;   // MED: 1-based block-list entry of its last contributor with incoming T > 0.5
	float acc[2][NT][4];
#pragma unroll
	for (int mt = 0; mt < 2; mt++)
#pragma unroll
		for (int nt = 0; nt < NT; nt++)
#pragma unroll
			for (int i = 0; i < 4; i++) acc[mt][nt][i] = 0.f;

	const int wofs = (lane >> 2) * 8 + ((lane >> 1) & 1) * 4 + (lane & 1);  // this pixel's slot in a [tig][gid][mt][e][h] weight tile

	// lane j < FWD_CH gathers record j of a chunk; the list positions of the chunk after next are loaded a chunk ahead
	uint32_t pos = lane < min(count, FWD_CH) ? lrow[lane] : 0u;
	if (lane < min(count, FWD_CH)) gather_rec(s_rec[0] + 2 * lane, recs + pos);
	cp_async_commit();
	pos = lane < min(count - FWD_CH, FWD_CH) ? lrow[FWD_CH + lane] : 0u;
	for (int k0 = 0, buf = 0; k0 < count; k0 += FWD_CH, buf ^= 1) {
		const int cnt = min(count - k0, FWD_CH);
		const float4* const s_q = s_rec[buf];
		cp_async_wait<0>();  // this chunk's records
		__syncwarp();
		// ---- start the gather of the chunk's channel rows (lands while the walk runs) ----
		if (VEC) {
			// lane r knows the Gaussian id of entry r; the feature rows are cut into 16-byte pieces and 32 / (2 NFT) rows
			// are copied per trip (lane = row-in-trip x piece), the id travelling by shuffle: 4 instructions per LDGSTS
			const uint32_t myid = lane < cnt ? __float_as_uint(s_q[2 * lane + 1].w) : 0u;
			if (NFT > 0) {
				constexpr int NPF = NFT > 0 ? 2 * NFT : 1, RPI = 32 / NPF;  // pieces per feature row, rows per trip
				const int sub = lane / NPF, q = lane % NPF;
#pragma unroll
				for (int it = 0; it < FWD_CH / RPI; it++) {
					const int r = it * RPI + sub;
					const uint32_t id = __shfl_sync(0xffffffffu, myid, r);
					// a remainder group (Fg < 32) copies its 4-channel pieces only: the rest of the row keeps the zeros of the clear
					const float* frow = a.feature + (GRP ? (size_t)id * F + c0 : (size_t)id * (8 * NFT));
					if (r < cnt && (!GRP || 4 * q < Fg)) cp_async16(s_rows + r * RS + 4 * q, reinterpret_cast<const float4*>(frow) + q);
				}
			}
			if (lane < cnt && first) cp_async16(s_rows + lane * RS + L::RGBD, a.rgbd + myid);
			if ((NRM || PLN) && lane < cnt && first) cp_async16(s_rows + lane * RS + L::RGBD + 4, a.nrm + myid);
		} else if (lane < cnt) {  // feature rows that are not whole 8-wide tiles (e.g. F = 3): plain loads, zero padded
			const uint32_t id = __float_as_uint(s_q[2 * lane + 1].w);
			float* row = s_rows + lane * RS;
			if (first) *reinterpret_cast<float4*>(row + L::RGBD) = a.rgbd[id];
			if ((NRM || PLN) && first) *reinterpret_cast<float4*>(row + L::RGBD + 4) = a.nrm[id];
			if (NFT > 0) {
				const float* f = a.feature + (size_t)id * F + c0;
#pragma unroll
				for (int i = 0; i < 8 * NFT; i++) row[i] = (i < Fg) ? __ldg(f + i) : 0.f;
			}
		}
		cp_async_commit();
		// ---- the next chunk's records travel while this chunk runs ----
		const int k1 = k0 + FWD_CH;
		if (lane < min(count - k1, FWD_CH)) gather_rec(s_rec[buf ^ 1] + 2 * lane, recs + pos);
		cp_async_commit();
		pos = lane < min(count - k1 - FWD_CH, FWD_CH) ? lrow[k1 + FWD_CH + lane] : 0u;
		// ---- walk: one k-step (8 entries) per trip, in two passes so that the eight footprint evaluations (independent:
		// LDS, 8 FP ops, expf) overlap in the pipeline and only the short transmittance recurrence is sequential.
		// Slots beyond cnt hold stale records and get zero weights. ----
		const int nks = (cnt + 7) >> 3;
		int ks = 0;
		for (; ks < nks; ks++) {
			if (ks > 0 && __all_sync(0xffffffffu, T < T_STOP)) break;
			const float4* q4 = s_q + 16 * ks;
			float* wrow = s_w + 256 * ks;
			float al[8];      // alpha of the pair, 0 where the pair is skipped (power > 0, alpha < 1/255, empty slot)
			walk_alphas(q4, pfx, pfy, ks, cnt, al);
#pragma unroll
			for (int u = 0; u < 8; u++) {
				const float alpha = al[u];
				const float test_T = T * (1 - alpha);
				const bool use = !(test_T < T_STOP);  // a skipped pair (alpha = 0) passes with zero weight and T unchanged
				wrow[(u & 3) * 64 + (u >> 2) * 2 + wofs] = use ? alpha * T : 0.f;
				T_out = use ? test_T : T_out;
				last = (use && alpha != 0.f) ? (uint32_t)(k0 + 8 * ks + u + 1) : last;
				if (MED) med = (use && alpha != 0.f && T > 0.5f) ? (uint32_t)(k0 + 8 * ks + u + 1) : med;
				T = test_T;
				s_pm[8 * ks + u] = __ballot_sync(0xffffffffu, use && alpha != 0.f);  // warp-uniform: every lane stores the same word
			}
		}
		const int nk = ks;  // k-steps to contract
		__syncwarp();
		// The backward reads the masks of the entries up to the block's last contributor, and every one of them is walked
		// here: a k-step is only skipped once every pixel has terminated.  So the array needs no clearing.
		if (first && lane < min(cnt, 8 * nk)) mrow[k0 + lane] = s_pm[lane];
		cp_async_wait<1>();  // the channel rows (the next chunk's records may still travel)
		__syncwarp();
		// ---- contract on the tensor cores ----
		for (int ks = 0; ks < nk; ks++) {
			const int g0 = 8 * ks + tig, g1 = g0 + 4;
			// {a0..a3} of pixel tile mt: weights of entries g0 (k = tig) and g1 (k = tig + 4) at pixels 4 gid + 2 mt + {0, 1}
			const float4 wa = *reinterpret_cast<const float4*>(s_w + ks * 256 + tig * 64 + gid * 8);
			const float4 wb = *reinterpret_cast<const float4*>(s_w + ks * 256 + tig * 64 + gid * 8 + 4);
			uint32_t ahi[2][4], alo[2][4];
			tf32_split(wa.x, ahi[0][0], alo[0][0]); tf32_split(wa.y, ahi[0][1], alo[0][1]);
			tf32_split(wa.z, ahi[0][2], alo[0][2]); tf32_split(wa.w, ahi[0][3], alo[0][3]);
			tf32_split(wb.x, ahi[1][0], alo[1][0]); tf32_split(wb.y, ahi[1][1], alo[1][1]);
			tf32_split(wb.z, ahi[1][2], alo[1][2]); tf32_split(wb.w, ahi[1][3], alo[1][3]);
			const float* row0 = s_rows + g0 * RS;
			const float* row1 = s_rows + g1 * RS;
			// B fragments {b0, b1} = column gid of tile nt for entries g0 and g1: scalar, conflict-free loads straight into
			// the operand pair (a 128-bit row load would need a register move per operand)
#pragma unroll
			for (int nt = 0; nt < NFT; nt++) {
				uint32_t bh0, bl0, bh1, bl1;
				tf32_split(row0[8 * nt + gid], bh0, bl0);
				tf32_split(row1[8 * nt + gid], bh1, bl1);
				mma_3xtf32(acc[0][nt], ahi[0], alo[0], bh0, bh1, bl0, bl1);
				mma_3xtf32(acc[1][nt], ahi[1], alo[1], bh0, bh1, bl0, bl1);
			}
			if (first) {
				const float c0 = (NRM || PLN || gid < 4) ? row0[L::RGBD + gid] : 0.f;
				const float c1 = (NRM || PLN || gid < 4) ? row1[L::RGBD + gid] : 0.f;
				uint32_t bh0, bl0, bh1, bl1;
				tf32_split(c0, bh0, bl0);
				tf32_split(c1, bh1, bl1);
				mma_3xtf32(acc[0][NFT], ahi[0], alo[0], bh0, bh1, bl0, bl1);
				mma_3xtf32(acc[1][NFT], ahi[1], alo[1], bh0, bh1, bl0, bl1);
			}
		}
		__syncwarp();  // s_w, s_rows and s_pm are rewritten by the next chunk
		if (__all_sync(0xffffffffu, T < T_STOP)) break;  // every pixel of the block is finished
	}
	cp_async_wait<0>();  // no record copy may be in flight when the CTA exits

	// ---- outputs ----
	const size_t HW = (size_t)a.H * a.W;
	if (inside) {
		T = T_out;
		if (first) {
			const size_t pix = (size_t)a.W * pyi + pxi;
			a.final_T[pix] = T;
			a.n_contrib[pix] = last ? lrow[last - 1] + 1u : 0u;  // 1-based tile-list position, as the reference counts
			if (a.out_alpha) a.out_alpha[pix] = 1.f - T;
			if (MED) {
				// the entry's tile-list position names the Gaussian; its depth is the value the depth channel blends
				const int id = med ? (int)a.point_list[range.x + lrow[med - 1]] : -1;
				a.median_id[pix] = id;
				if constexpr (PLN) {
					// the contributor's planar depth z + a px + b py + e at this pixel
					if (a.out_median_depth) {
						float md = 0.f;
						if (med) { const float4 q = a.nrm[id]; md = a.rgbd[id].w + q.x * pfx + q.y * pfy + q.z; }
						a.out_median_depth[pix] = md;
					}
				} else if (a.out_median_depth) a.out_median_depth[pix] = med ? a.rgbd[id].w : 0.f;
			}
		}
	}
	if (first) {
		uint32_t nwalk = last;
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) nwalk = max(nwalk, __shfl_xor_sync(0xffffffffu, nwalk, o));
		if (lane == 0) a.block_nwalk[8 * tile + sub] = nwalk;
	}
	s_w[lane] = T;
	__syncwarp();
	const int ox = bx0 + gid;  // fragment role: this thread holds pixels (x = gid, y = 0..3)
	const bool heads = first && a.tgt_color != nullptr;     // fused loss heads (loss_heads.cuh)
	const bool embed = heads && NFT > 0 && a.tgt_feature != nullptr && !GRP;
	const bool dmh = DM && heads;                           // depth / mask heads
	const float invN = 1.0f / (float)HW;
	float s_rgb = 0.f, s_cos = 0.f;                         // this thread's share of the two loss sums
	float s_dep = 0.f, s_n = 0.f, s_bce = 0.f;              // ... and of the depth / mask heads' sums
#pragma unroll
	for (int mt = 0; mt < 2; mt++) {
#pragma unroll
		for (int h = 0; h < 2; h++) {
			const int y = 2 * mt + h, oy = by0 + y;
			const bool in = ox < a.W && oy < a.H;
			const size_t pix = in ? (size_t)a.W * oy + ox : 0;
			const float Tp = s_w[4 * gid + y];
			if constexpr (PLN) {
				// the depth, column 3 on thread tig = 1, gains px col4 + py col5 + col6 from threads tig = 2 and 3 of the quad
				const int q0 = lane & ~3;
				const float c4 = __shfl_sync(0xffffffffu, acc[mt][NFT][2 * h], q0 | 2);
				const float c5 = __shfl_sync(0xffffffffu, acc[mt][NFT][2 * h + 1], q0 | 2);
				const float c6 = __shfl_sync(0xffffffffu, acc[mt][NFT][2 * h], q0 | 3);
				if (tig == 1) acc[mt][NFT][2 * h + 1] += (float)ox * c4 + (float)oy * c5 + c6;
			}
#pragma unroll
			for (int nt = 0; nt < NFT; nt++) {
#pragma unroll
				for (int e = 0; e < 2; e++) {
					const int f = 8 * nt + 2 * tig + e;
					if (in && f < Fg) a.out_feature[(size_t)(c0 + f) * HW + pix] = acc[mt][nt][2 * h + e];
				}
			}
			float col[2];
#pragma unroll
			for (int e = 0; e < 2; e++) {
				const int c = 2 * tig + e;  // column of the {r,g,b,depth} tile
				col[e] = acc[mt][NFT][2 * h + e] + (c < 3 ? Tp * a.bg[c] : 0.f);
				if (!first) continue;
				if (in && c < 3) a.out_color[(size_t)c * HW + pix] = col[e];
				else if (in && c == 3 && a.out_depth) a.out_depth[pix] = col[e];
				else if (NRM && in && c > 3 && c < 7) a.out_normal[(size_t)(c - 4) * HW + pix] = col[e];  // no background term
			}
			if (heads) {  // warp-uniform
#pragma unroll
				for (int e = 0; e < 2; e++) {
					const int c = 2 * tig + e;
					if (in && c < 3) {
						const float d = col[e] - a.tgt_color[(size_t)c * HW + pix];
						s_rgb += d * d;
						a.cot_color[(size_t)c * HW + pix] = (2.0f / 3.0f) * invN * d;
					}
				}
				// column 3 of the {r,g,b,depth} tile is col[1] of thread tig = 1: that thread evaluates both heads of the pixel,
				// with the same D and A = 1 - T as the depth and alpha planes
				if (dmh && tig == 1 && in) {
					const float A = 1.f - Tp;
					if (a.tgt_depth) {
						const DepthTerms dt = depth_terms(col[1], A, a.tgt_depth[pix]);
						s_dep += dt.err;
						s_n += dt.n;
						a.cot_depth[pix] = dt.cot_d;
						a.cot_alpha_depth[pix] = dt.cot_a;
					}
					if (a.tgt_mask) {
						const MaskTerms mk = mask_terms(A, a.tgt_mask[pix]);
						s_bce += mk.bce;
						a.cot_alpha_mask[pix] = mk.grad * invN;
					}
				}
				if (embed) {
					// this thread holds 2 NFT of the pixel's features; the other three threads of the quad hold the rest
					float tg[NFT > 0 ? NFT : 1][2];
					float xy = 0.f, xx = 0.f, yy = 0.f;
#pragma unroll
					for (int nt = 0; nt < NFT; nt++) {
#pragma unroll
						for (int e = 0; e < 2; e++) {
							const int f = 8 * nt + 2 * tig + e;
							const float x = acc[mt][nt][2 * h + e];
							const float g = (in && f < F) ? a.tgt_feature[(size_t)f * HW + pix] : 0.f;
							tg[nt][e] = g;
							xy += x * g; xx += x * x; yy += g * g;
						}
					}
#pragma unroll
					for (int o = 1; o <= 2; o <<= 1) {
						xy += __shfl_xor_sync(0xffffffffu, xy, o);
						xx += __shfl_xor_sync(0xffffffffu, xx, o);
						yy += __shfl_xor_sync(0xffffffffu, yy, o);
					}
					const CosTerms ct = cos_terms(xy, xx, yy);
					if (in && tig == 0) s_cos += ct.cos;
#pragma unroll
					for (int nt = 0; nt < NFT; nt++) {
#pragma unroll
						for (int e = 0; e < 2; e++) {
							const int f = 8 * nt + 2 * tig + e;
							if (in && f < F) a.cot_feature[(size_t)f * HW + pix] = -invN * cos_grad(ct, acc[mt][nt][2 * h + e], tg[nt][e]);
						}
					}
				}
			}
		}
	}
	if (heads) {
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) {
			s_rgb += __shfl_xor_sync(0xffffffffu, s_rgb, o);
			s_cos += __shfl_xor_sync(0xffffffffu, s_cos, o);
		}
		if (lane == 0) {
			red_add(a.loss_acc, s_rgb);
			if (embed) red_add(a.loss_acc + 1, s_cos);
		}
	}
	if (dmh) {
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) {
			s_dep += __shfl_xor_sync(0xffffffffu, s_dep, o);
			s_n += __shfl_xor_sync(0xffffffffu, s_n, o);
			s_bce += __shfl_xor_sync(0xffffffffu, s_bce, o);
		}
		if (lane == 0) {
			if (a.tgt_depth) { red_add(a.dm_acc, s_dep); red_add(a.dm_acc + 1, s_n); }  // n: exact in fp32 up to 2^24 pixels
			if (a.tgt_mask) red_add(a.dm_acc + 2, s_bce);
		}
	}
#ifdef MGS_CTA_LOG
	cta_log_put(a, t_start, 0u, (unsigned int)sub, (unsigned int)count);
#endif
}

// F > 32 runs in channel groups of 32 (BlendArgs::groups), each with the F = 32 instantiations
int blend_supported(int F) { return F >= 0 && F <= MGS_MAX_FEATURE_CHANNELS; }
int blend_groups(int F) { return F > 32 ? ceil_div(F, 32) : 1; }

// 128-bit feature copies need 16-byte aligned rows of a 16-byte multiple
bool feature_rows_vectorizable(const float* feature, int F)
{
	return F > 0 && (F & 3) == 0 && (reinterpret_cast<uintptr_t>(feature) & 15) == 0;
}

template <int NFT, bool GRP, bool DM, bool MED, bool NRM, bool PLN>
static void launch_fwd_t(const BlendArgs& a, cudaStream_t s)
{
	const int grid = a.grid_x * a.grid_y * 8 * a.groups;
	// the cp.async row gather copies whole 8-wide feature tiles: exact fits only; other widths take the padded path.  With
	// groups, a row slice starts at channel 32 g: 16-byte aligned whenever F % 4 == 0, and a remainder group copies whole
	// 4-channel pieces only.
	const bool vec = (NFT == 0) || ((a.F == 8 * NFT || GRP) && feature_rows_vectorizable(a.feature, a.F));
	if (vec) blend_fwd_kernel<NFT, true, GRP, DM, MED, NRM, PLN><<<grid, 32, 0, s>>>(a);
	else blend_fwd_kernel<NFT, false, GRP, DM, MED, NRM, PLN><<<grid, 32, 0, s>>>(a);
}

template <bool DM, bool MED, bool NRM, bool PLN = false>
static void launch_fwd_dm(const BlendArgs& a, cudaStream_t s)
{
	if (a.groups > 1) { launch_fwd_t<4, true, DM, MED, NRM, PLN>(a, s); return; }
	switch (nft_for(a.F)) {
	case 0: launch_fwd_t<0, false, DM, MED, NRM, PLN>(a, s); break;
	case 1: launch_fwd_t<1, false, DM, MED, NRM, PLN>(a, s); break;
	case 2: launch_fwd_t<2, false, DM, MED, NRM, PLN>(a, s); break;
	default: launch_fwd_t<4, false, DM, MED, NRM, PLN>(a, s); break;
	}
}

void launch_blend_fwd(const BlendArgs& a, cudaStream_t s)
{
	const bool dm = a.tgt_color && (a.tgt_depth || a.tgt_mask);
	if (a.planar) {  // never with the normal plane: both take columns 4..6 (the entry points refuse the pair)
		if (a.median_id) {
			if (dm) launch_fwd_dm<true, true, false, true>(a, s);
			else launch_fwd_dm<false, true, false, true>(a, s);
		} else if (dm) launch_fwd_dm<true, false, false, true>(a, s);
		else launch_fwd_dm<false, false, false, true>(a, s);
	} else if (a.nrm) {  // never with the depth / mask heads: the entry points refuse that pair, so it has no instantiation
		if (a.median_id) launch_fwd_dm<false, true, true>(a, s);
		else launch_fwd_dm<false, false, true>(a, s);
	} else if (a.median_id) {
		if (dm) launch_fwd_dm<true, true, false>(a, s);
		else launch_fwd_dm<false, true, false>(a, s);
	} else if (dm) launch_fwd_dm<true, false, false>(a, s);
	else launch_fwd_dm<false, false, false>(a, s);
}

}  // namespace mgs
