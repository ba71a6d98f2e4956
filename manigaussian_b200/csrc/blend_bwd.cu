// Backward blend: per-pixel back-to-front replay that emits per-Gaussian gradients.
//
// Replaces BACKWARD::render / renderCUDA<3,F> (DGR/cuda_rasterizer/backward.cu:399-593) behind the
// C-ABI.  Same mathematics (SURVEY.md A.4): walking a pixel's contributors back to front,
//   T_k     = T_{k+1} / (1 - a_k)                      (T recovered by division from final_T, :521)
//   dL/dc_k = a_k T_k g                                 (g = dL/dpixel, all channels)
//   dL/da_k = T_k (c_k . g) - (S_k + T_final (bg . g_rgb - h)) / (1 - a_k),   S_k = sum_{j behind k} a_j T_j (c_j . g)
//           (h = dL/dalpha of the optional alpha plane 1 - T_final, whose derivative T_final / (1 - a_k) has the background
//           term's form)
//   dL/dG   = o_k dL/da_k  (the 0.99 clamp is gradient-transparent, :574), then mean2D / conic / opacity.
// S_k is the scalar form of the reference's per-channel `accum_rec` recursion.
//
// Design.  The reference has every pixel-thread issue 9+F global float atomics per contributing pair (41 at F=32).
// Here the sums over the pixels of a warp's 8x4 block ARE matrix products, and they run on the tensor cores
// (mma.sync m16n8k8 TF32, 3xTF32 split, blend_mma.cuh).  A two-warp CTA replays its block's work list back to front
// from the block's last contributor (block_nwalk), reading the list entries together with the pixel masks the forward
// wrote for them (bit p: the pair contributed to pixel p); it queues the entries whose mask is non-zero -- an instance that
// reached no pixel of the block has no gradient there -- gathers the records of each chunk of BWD_CH queued survivors by
// list position (cp.async, the next chunk's while the current one runs) and carries the mask in the record; per chunk:
//   1. gather    the chunk's channel rows C[g][ch] by Gaussian id (cp.async, 16-byte pieces)
//   2. GEMM 1    Wd[g][p] = sum_ch C[g][ch] Gpx[p][ch]          (c_k . g for every survivor x pixel; Gpx = the block's
//                                                                cotangent rows, staged once per CTA)
//   3. walk      lane = pixel, sequential over the chunk: alpha, T_k, S_k exactly as above (the per-pixel carried
//                state is two registers); writes wgt[g][p] = a_k T_k and q[g][p] = dL/dG * G, zero for pairs that did
//                not contribute (pixel mask bit clear: the forward's decision, so no threshold test is repeated here)
//   4. GEMM 2    dC[g][ch] = sum_p wgt[g][p] Gpx[p][ch]          (dL/dcolour, dL/ddepth, dL/dfeature)
//   5. GEMM 3    M[g][m]   = sum_p q[g][p] Y[p][m],  Y[p] = {1, x, y, x^2, x y, y^2} of pixel p relative to the block:
//                the six moments from which lane = Gaussian assembles dL/dmean2D, dL/dconic, dL/dopacity
//                (sum_p q (u - x)^2 = u^2 M0 - 2 u Mx + Mxx with u = mean.x - block.x, ...; Y is exact in TF32)
//   6. flush     per (block, Gaussian): 3 red.global.add.v4.f32 of the 10 small gradients + the feature row as
//                red.v4 straight from the D fragments (column gid of feature tile nt is feature NFT*gid + nt, so a thread
//                holds 8 consecutive features of its four Gaussians; at F = 32 neighbouring lanes swap halves so that every
//                pair of reductions fills whole 32-byte sectors).
// Roles.  Only the walk is sequential (T and S carry from chunk to chunk), so it has a warp of its own: warp 0, the
// walker W, owns T, S and the background term and runs step 3.  Warp 1, the companion C, runs everything else: the queue,
// the gathers, GEMM 2/3 and the flush.  GEMM 1 goes to whichever warp would otherwise wait (W_GEMM1 in the kernel): with
// feature tiles C carries the larger share of a chunk, and GEMM 1 moves to W, which reads the cotangent rows it staged
// and writes Wd, which only its own walk reads; at small F the walk is the longer share, and C keeps GEMM 1.  The warps
// hand chunks to each other through a two-stage ring of {rows -> wgt, Wd -> q} tiles (records: three slots) with named
// barriers (protocol at the loop below), so that while W walks chunk i, C finishes chunk i - 1 and prepares chunk i + 1.
// Splitting the roles also splits the registers: 128 per thread give 8 CTAs (16 warps) per SM at F = 32, against 12
// single-warp CTAs at 157 registers when one warp did all of it.
// Channel groups (F > 32) keep that single-warp CTA (blend_bwd_groups_kernel): their launches are several waves deep,
// and there two-warp CTAs measured slower.
// Index assignment.  An MMA A operand is four consecutive registers, a B operand two; a register move per operand would
// cost more than the tensor cores save, so every shared-memory tile is laid out such that operands ARRIVE in place:
//   pixels      p = 2 pi + e  (pair pi = 0..15).  K-side (GEMM 2/3): k-step pi >> 2, slots tig = pi & 3 (e = 0) and
//               tig + 4 (e = 1).  M-side (GEMM 1): tile pi >> 3, rows gid = pi & 7 (e = 0) and gid + 8 (e = 1).
//   survivors   j.  M-side (GEMM 2/3): tile j >> 4, rows gid = (j & 15) >> 1 (even j) and gid + 8 (odd j).
//               N-side (GEMM 1): tile j >> 3, column j & 7.
//   channels    K-side (GEMM 1): step ch >> 3, slots tig = (ch & 7) >> 1 (even ch) and tig + 4 (odd ch).
//               N-side (GEMM 2): column gid of feature tile nt is feature NFT gid + nt; {r,g,b,depth} tile: column gid.
//   s_g  [pi][ch][e]              cotangents: GEMM 1's A quad {(e0,ch),(e1,ch),(e0,ch+1),(e1,ch+1)} is one LDS.128, GEMM 2's
//                                 B pairs {(e0,ch),(e1,ch)} for a thread's NFT consecutive channels are LDS.128s
//   s_rows [j][ch]                channel rows as gathered: GEMM 1's B pair {ch, ch+1} is one LDS.64
//   s_x, s_wgt [pi][j >> 1][e][j & 1]   GEMM 1's D fragment is one STS.128, GEMM 2/3's A quad one LDS.128; the walk
//                                 (lane = pixel) reads Wd and writes q in place
#include "blend_common.cuh"
#include "blend_mma.cuh"

namespace mgs {

#ifndef MGS_BWD_CH
#define MGS_BWD_CH 32
#endif
#ifndef MGS_BWD_MIN_CTAS
#define MGS_BWD_MIN_CTAS 8  // two-warp CTAs per SM: at most 128 registers per thread
#endif
// Timing-only switches of the two-warp kernel, never in the default build; their gradients are wrong by construction
// (tools/bwd_phases.py, DESIGN §4):
//   MGS_BWD_ABL_NO_FEATURE_RED  skip the feature-row reductions of the flush (dL/dfeature stays zero)
//   MGS_BWD_ABL_FIXED_ROW       gather the channel rows of Gaussian id & 4095 instead of id: 576 KB of rows that stay in
//                               L2, spread over its slices (one single row would make every CTA hammer one L2 line)
#ifdef MGS_BWD_ABL_FIXED_ROW
__device__ __forceinline__ uint32_t bwd_row_id(uint32_t id) { return id & 4095u; }
#else
__device__ __forceinline__ uint32_t bwd_row_id(uint32_t id) { return id; }
#endif
#ifdef MGS_BWD_ABL_NO_FEATURE_RED
constexpr bool BWD_FEATURE_RED = false;
#else
constexpr bool BWD_FEATURE_RED = true;
#endif
constexpr int BWD_CH = MGS_BWD_CH;        // survivors per chunk: 16 or 32 (whole 16-row MMA tiles)
constexpr int BWD_QCAP = 64;              // survivor queue (a ring): a chunk plus the survivors of one more 32-entry step
constexpr int BWD_MT = BWD_CH / 16;       // 16-row tiles of Gaussians
constexpr int BWD_NREC = 3;               // record slots: chunk i (walked), i - 1 (flushed), i + 1 (gathered)
static_assert(BWD_CH == 16 || BWD_CH == 32, "backward chunk size");
// named barriers of the hand-off (0 is __syncthreads'), one per signal and stage s = chunk & 1, 64 threads each:
// FULL + s  companion -> walker: records, cnt and channel rows (W_GEMM1) or Wd (otherwise) of the chunk are in place
//           (bar.arrive by C, bar.sync by W)
// DONE + s  walker -> companion: wgt and q of the chunk are written            (bar.arrive by W, bar.sync by C)
constexpr int BWD_BAR_FULL = 1, BWD_BAR_DONE = 3;

// Cotangents of the depth and mask heads (loss_heads.cuh) for one in-image pixel, folded into the depth cotangent g_depth and
// the alpha cotangent h of the walker's prologue.  The forward wrote the planes for unit upstream gradients; the depth head's
// scale g_depth / max(n, 1) needs the view's valid-pixel count n, which the forward's accumulator holds by now.
__device__ __forceinline__ void depth_mask_cotangents(const BlendArgs& a, size_t pix, float& g_depth, float& h)
{
	if (a.tgt_depth) {
		const float s_d = (a.dm_scale ? a.dm_scale[0] : 1.f) / fmaxf(a.dm_acc[1], 1.f);
		g_depth += s_d * a.cot_depth[pix];
		h += s_d * a.cot_alpha_depth[pix];
	}
	if (a.tgt_mask) h += (a.dm_scale ? a.dm_scale[1] : 1.f) * a.cot_alpha_mask[pix];
}

// PLN: the gathered quads {a, b, e, 0} of a chunk's cnt survivors (rows of stride rs from q4, records rec) get e_b =
// -(a (mu_x - bx0) + b (mu_y - by0)) in place of e, the offset of the planar depth relative to the block origin.  Lane j < cnt
// rewrites row j.
__device__ __forceinline__ void planar_block_offset(float* q4, int rs, const float4* rec, int cnt, int lane, float fbx0, float fby0)
{
	if (lane < cnt) {
		const float4 r0 = rec[2 * lane];
		float* q = q4 + lane * rs;
		q[2] = -fmaf(q[0], r0.x - fbx0, q[1] * (r0.y - fby0));
	}
}

// F <= 32 (one channel group); channel groups run blend_bwd_groups_kernel below.  DM: the depth / mask heads
// (BlendArgs::tgt_depth / tgt_mask); the instantiations without them keep their registers.  NRM: the normal plane
// (BlendArgs::nrm / dL_dnormal / gn): the quad {nx, ny, nz, 0} and its cotangent fill columns 4..7 of the {r,g,b,depth} tile,
// so GEMM 1 and GEMM 2 carry them as issued, and the flush adds dL/dn into gn; likewise.  PLN: planar depth
// (BlendArgs::planar): in block-local pixel coordinates (lx, ly) = (px - bx0, py - by0) the depth is z + a lx + b ly + e_b
// with e_b = -(a (mu_x - bx0) + b (mu_y - by0)); the quad {a, b, e_b, 0} fills the same columns (e_b replaces the gathered e
// once the rows are in) and the depth cotangent g enters them as {g lx, g ly, g, 0}, so dL/dalpha is that of the planar
// depth.  The flush adds {sum w g (px - mu_x), sum w g (py - mu_y), sum w g, 0} = {dn.x - u dn.z, dn.y - v dn.z, dn.z, 0}
// (u, v: the mean relative to the block) into gn: dL/d(a, b) with e's share included, and dL/de.  Every term is
// footprint-sized, whatever the pixel coordinates; likewise.
template <int NFT, bool VEC, bool DM, bool NRM, bool PLN>
__global__ void __launch_bounds__(64, MGS_BWD_MIN_CTAS) blend_bwd_kernel(BlendArgs a)
{
	constexpr int NT = NFT + 1;          // channel tiles of 8: NFT feature tiles + {r,g,b,depth, 4 x zero}
	constexpr int CHP = 8 * NT;          // padded channel count
	constexpr int RS = CHP;              // channel-row stride (floats): [8 NFT features | r g b depth | 0 0 0 0]
	constexpr int RGBD = 8 * NFT;
	constexpr int GS = 2 * CHP;          // s_g stride per pixel pair
	constexpr int XS = 2 * BWD_CH + 4;   // s_x / s_wgt stride per pixel pair (+4: spreads the pairs over the banks)
	constexpr int ROWS_FLOATS = (BWD_CH * RS > 16 * XS) ? BWD_CH * RS : 16 * XS;  // the rows buffer is reused for the wgt tile
	// GEMM 1 on the walker at F > 16 only: there the companion's GEMM 2 and feature flush make it the warp that bounds a
	// chunk (c3, F = 32: blend_bwd 6 % shorter); at F <= 16 the walk does, and GEMM 1 on the walker made blend_bwd longer
	// (c3 shape, F = 16 / 8 / 0: +4 / +2 / +9 %; DESIGN §4)
	constexpr bool W_GEMM1 = NFT == 4;
	__shared__ __align__(16) float4 s_rec[BWD_NREC][BWD_CH * 2];  // records by chunk mod 3: {x,y,ca,cb}, {cc,op,pixel mask,id}
	__shared__ uint2 s_qe[BWD_QCAP];                              // survivor queue, back to front: {list position, pixel mask}
	__shared__ __align__(16) float s_rows[2][ROWS_FLOATS];        // by stage: C[j][RS]; after GEMM 1: wgt tile
	__shared__ __align__(16) float s_x[2][16 * XS];               // by stage: Wd tile; the walk overwrites it with q in place; then per-Gaussian staging
	__shared__ __align__(16) float s_g[16 * GS];                  // cotangent rows of the block's pixels
	__shared__ int s_cnt[2];                                      // by stage: survivors of the chunk, 0 = end of the list

#ifdef MGS_CTA_LOG
	const unsigned long long t_start = cta_log_now();
#endif
	const int lane = threadIdx.x & 31;
	// warp 0 walks, warp 1 is the companion.  The warp index comes through a shuffle so that the compiler knows it is
	// warp-uniform: from threadIdx.x < 32 it assumes the roles may diverge inside a warp and wraps every shuffle, ballot
	// and __syncwarp of the two branches in a divergence-safe WARPSYNC ... ENDCOLLECTIVE sequence (3,424 SASS instructions
	// against 2,704 at F = 32)
	const bool walker = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0) == 0;
	const int gid = lane >> 2, tig = lane & 3;
	const int sub = blockIdx.x & 7;
	const int rank = (int)(blockIdx.x >> 3);
	const int tile = a.tile_order ? (int)a.tile_order[rank] : rank;  // longest lists first
	const int tile_x = tile % a.grid_x, tile_y = tile / a.grid_x;
	const int bx0 = tile_x * TILE_X + (sub & 1) * WARP_BX;
	const int by0 = tile_y * TILE_Y + (sub >> 1) * WARP_BY;
	const int pxi = bx0 + (lane >> 2), pyi = by0 + (lane & 3);  // walk role: lane = pixel (x = lane >> 2, y = lane & 3)
	const bool inside = pxi < a.W && pyi < a.H;
	// Both early exits are taken by the whole CTA before its first barrier: both warps see the same pixels and read the
	// same block_nwalk.
	if (__all_sync(0xffffffffu, !inside)) return;  // the forward skipped this block: it has no block_nwalk
	// only the entries up to the block's last contributor can have contributed to a pixel of the block
	const int nwalk = (int)a.block_nwalk[8 * tile + sub];
	if (nwalk == 0) return;  // nothing blended into this block
	const size_t HW = (size_t)a.H * a.W;
	const size_t pix = (size_t)a.W * pyi + pxi;
	const int F = a.F;                 // feature row stride

	// ---- per-pixel state and cotangent rows (walker); zero channel rows (companion: the padding columns stay finite) ----
	float T = 0.f, bgterm = 0.f;
	if (walker) {
		float g4[4] = { 0.f, 0.f, 0.f, 0.f };
		float h = 0.f;  // alpha cotangent: d alpha / d a_k = T_final / (1 - a_k), the background term's form, with -h for bg . g
		// upstream gradients of the fused loss heads (loss_heads.cuh): the cotangent planes were written for d loss = 1
		const float sc_color = a.cot_scale ? a.cot_scale[0] : 1.f, sc_feat = a.cot_scale ? a.cot_scale[1] : 1.f;
		if (inside) {
			T = a.final_T[pix];
#pragma unroll
			for (int ch = 0; ch < 3; ch++) g4[ch] = sc_color * a.dL_dcolor[ch * HW + pix];
			if (a.dL_ddepth) g4[3] = a.dL_ddepth[pix];
			if (a.dL_dalpha) h = a.dL_dalpha[pix];
			if (DM) depth_mask_cotangents(a, pix, g4[3], h);
		}
		bgterm = T * (a.bg[0] * g4[0] + a.bg[1] * g4[1] + a.bg[2] * g4[2] - h);
		float* grow = s_g + (lane >> 1) * GS + (lane & 1);  // element (pixel, ch) at [pi][ch][e]
#pragma unroll
		for (int c = 0; c < 4; c++) {
			grow[2 * (RGBD + c)] = g4[c];
			// NRM: the normal plane's cotangent in columns 4..6, unscaled (the plane has no background term either)
			grow[2 * (RGBD + 4 + c)] = (NRM && c < 3 && inside) ? a.dL_dnormal[c * HW + pix] : 0.f;
			if (PLN) grow[2 * (RGBD + 4 + c)] = c == 0 ? g4[3] * (float)(lane >> 2) : c == 1 ? g4[3] * (float)(lane & 3) : c == 2 ? g4[3] : 0.f;
		}
		if (NFT > 0) {
#pragma unroll
			for (int i = 0; i < 8 * NFT; i++)
				grow[2 * i] = (inside && i < F && a.dL_dfeature) ? sc_feat * a.dL_dfeature[(size_t)i * HW + pix] : 0.f;
		}
	} else {
		for (int i = lane; i < 2 * ROWS_FLOATS / 4; i += 32) reinterpret_cast<float4*>(&s_rows[0][0])[i] = make_float4(0.f, 0.f, 0.f, 0.f);
	}
	__syncthreads();  // s_g and the zeroed rows buffers are in place: the CTA's only barrier over both warps besides the hand-off

	// GEMM 1 of the chunk whose channel rows sit in s_rows, into s_xs
	auto gemm1 = [&](const float* s_rows, float* s_xs) {
		// ---- 2. GEMM 1: Wd[p][j] = Gpx[p][:] . C[j][:]   (M = pixels (2 tiles), N = survivors, K = channels) ----
		float wd[2][BWD_CH / 8][4];
#pragma unroll
		for (int mt = 0; mt < 2; mt++)
#pragma unroll
			for (int nt = 0; nt < BWD_CH / 8; nt++)
#pragma unroll
				for (int i = 0; i < 4; i++) wd[mt][nt][i] = 0.f;
#pragma unroll
		for (int ks = 0; ks < NT; ks++) {
			uint32_t ahi[2][4], alo[2][4];
#pragma unroll
			for (int mt = 0; mt < 2; mt++) {
				const float4 v = *reinterpret_cast<const float4*>(s_g + (8 * mt + gid) * GS + (8 * ks + 2 * tig) * 2);
				tf32_split(v.x, ahi[mt][0], alo[mt][0]); tf32_split(v.y, ahi[mt][1], alo[mt][1]);
				tf32_split(v.z, ahi[mt][2], alo[mt][2]); tf32_split(v.w, ahi[mt][3], alo[mt][3]);
			}
#pragma unroll
			for (int nt = 0; nt < BWD_CH / 8; nt++) {
				const float2 v = *reinterpret_cast<const float2*>(s_rows + (8 * nt + gid) * RS + 8 * ks + 2 * tig);
				uint32_t bh0, bl0, bh1, bl1;
				tf32_split(v.x, bh0, bl0);
				tf32_split(v.y, bh1, bl1);
				mma_3xtf32(wd[0][nt], ahi[0], alo[0], bh0, bh1, bl0, bl1);
				mma_3xtf32(wd[1][nt], ahi[1], alo[1], bh0, bh1, bl0, bl1);
			}
		}
		// D fragment (mt, nt): pixels (pi = 8 mt + gid, e = 0 | 1), survivors 8 nt + 2 tig (+1): one 16-byte store
#pragma unroll
		for (int mt = 0; mt < 2; mt++)
#pragma unroll
			for (int nt = 0; nt < BWD_CH / 8; nt++)
				*reinterpret_cast<float4*>(s_xs + (8 * mt + gid) * XS + (4 * nt + tig) * 4) =
					make_float4(wd[mt][nt][0], wd[mt][nt][1], wd[mt][nt][2], wd[mt][nt][3]);
	};

	// Two-stage ring.  While W walks chunk i in stage i & 1 (with W_GEMM1 after its GEMM 1 turned the stage's rows into Wd;
	// the walk turns Wd into q in place and overwrites the rows with wgt), C finishes chunk i - 1 (GEMM 2/3, flush) and
	// prepares chunk i + 1 (records, rows, without W_GEMM1 its GEMM 1), both in stage (i + 1) & 1.  Each signal is raised
	// once per use of its stage and consumed before it can be raised again: C raises FULL + s for chunk i + 2 only after it
	// consumed DONE + s of chunk i, which W raises after it consumed FULL + s of chunk i; W raises DONE + s for chunk i + 2
	// only after it consumed FULL + s of chunk i + 2, which C raises after it consumed DONE + s of chunk i.  Neither warp
	// blocks on anything else but its own cp.async groups, so the waits cannot form a cycle (DESIGN §4).  The end of the
	// list travels as a chunk with cnt = 0 through FULL, after which W stops and C finishes the last real chunk: both warps
	// run the same sequence of barrier operations.
	if (walker) {
#ifdef MGS_BWD_PHASES
		BwdPhaseClock ph;
		ph.start();
#endif
		const float pfx = (float)pxi, pfy = (float)pyi;
		float S = 0.f;  // sum over the contributors behind the current one of a_j T_j (c_j . g)
		const int xofs = (lane >> 1) * XS + (lane & 1) * 2;  // this pixel's slot in the [pi][j >> 1][e][j & 1] tiles
		int r = 0;  // record slot of chunk k
#pragma unroll 1
		for (int k = 0;; k++) {
			const int s = k & 1;
			named_bar_sync<BWD_BAR_FULL, 64>(s);
			BWD_PH_LAP(ph, BWD_PH_FULL_WAIT);
			const int cnt = s_cnt[s];
			if (cnt == 0) break;
			const float4* const s_q = s_rec[r];
			float* const s_wgt = s_rows[s];
			float* const s_xs = s_x[s];
			r = r == BWD_NREC - 1 ? 0 : r + 1;
			if (W_GEMM1) {
				gemm1(s_rows[s], s_xs);
				__syncwarp();  // every lane's Wd is stored and every row read: the walk reads Wd and overwrites the rows with wgt
				BWD_PH_LAP(ph, BWD_PH_GEMM1);
			}
			// ---- 3. walk, back to front (queue order): lane = pixel.  Per k-step of 8 survivors: first the eight footprint
			// evaluations (independent, they overlap in the pipeline), then the short sequential recurrence on T and S. ----
#pragma unroll 1
			for (int j0 = 0; j0 < BWD_CH; j0 += 8) {
				float al[8], opG[8], rinv[8];  // alpha, opacity * G, 1 / (1 - alpha); alpha = opG = 0, rinv = 1 for pairs that did not contribute
#pragma unroll
				for (int u = 0; u < 8; u++) {
					const int j = j0 + u;
					const float4 r0 = s_q[2 * j], r1 = s_q[2 * j + 1];
					const float dx = r0.x - pfx, dy = r0.y - pfy;
					const float op = r1.y;
					const float power = -0.5f * (r0.z * dx * dx + r1.x * dy * dy) - r0.w * dx * dy;
					const float G = __expf(power);  // ex2.approx-based (rel. error ~1e-6): the decision below is the forward's, not this
					const float alpha = min(ALPHA_MAX, op * G);
					// whether the pair contributed is the forward's own decision (pixel mask); slots past cnt hold stale entries
					const bool valid = (j < cnt) && ((__float_as_uint(r1.z) >> lane) & 1u);
					al[u] = valid ? alpha : 0.f;
					opG[u] = valid ? op * G : 0.f;
					rinv[u] = __fdividef(1.f, 1.f - al[u]);
				}
#pragma unroll
				for (int u = 0; u < 8; u++) {
					const int jofs = (j0 >> 1) * 4 + (u >> 1) * 4 + (u & 1);  // survivor j0 + u
					const float wdot = s_xs[xofs + jofs];
					const float Tk = T * rinv[u];                                 // transmittance in front of this Gaussian
					const float wgt = al[u] * Tk;                                 // d(pixel channel) / d(colour of this Gaussian)
					const float dL_dalpha = Tk * wdot - (S + bgterm) * rinv[u];
					s_wgt[xofs + jofs] = wgt;
					s_xs[xofs + jofs] = opG[u] * dL_dalpha;                       // q = dL/dG * G  (dL/dG = opacity * dL/dalpha)
					T = Tk;                                                       // unchanged where the pair is skipped (rinv = 1)
					S = fmaf(wgt, wdot, S);                                       // likewise (wgt = 0)
				}
			}
			__syncwarp();
			named_bar_arrive<BWD_BAR_DONE, 64>(s);
			BWD_PH_LAP(ph, BWD_PH_WALK);
		}
#ifdef MGS_BWD_PHASES
		ph.put(a.bwd_phases, BWD_PH_FULL_WAIT, BWD_PH_WALK, BWD_PH_W_TOTAL, false);
#endif
	} else {
#ifdef MGS_BWD_PHASES
		BwdPhaseClock ph;
		ph.start();
		ph.acc[BWD_PH_CTAS] = 1u;
#endif
		const float fbx0 = (float)bx0, fby0 = (float)by0;
		const float half_W = 0.5f * a.W, half_H = 0.5f * a.H;
		const InstRec* const recs = a.recs + a.ranges[tile].x;                                   // the tile's records, by 0-based list position
		const uint32_t* const lrow = a.block_list + sub * a.mask_stride + a.ranges[tile].x;     // this block's work list
		const uint32_t* const mrow = a.pix_mask + sub * a.mask_stride + a.ranges[tile].x;       // pixel masks, by block-list entry
		// GEMM 3's B operand: moments basis of the two pixels of k-slots (ks, tig) and (ks, tig + 4): p = 8 ks + 2 tig + e,
		// x = p >> 2, y = p & 3; column gid selects {1, x, y, x^2, x y, y^2, 0, 0}
		uint32_t ymom[4][2];
#pragma unroll
		for (int ks = 0; ks < 4; ks++) {
#pragma unroll
			for (int e = 0; e < 2; e++) {
				const int p = 8 * ks + 2 * tig + e;
				const float x = (float)(p >> 2), y = (float)(p & 3);
				const float v = gid == 0 ? 1.f : gid == 1 ? x : gid == 2 ? y : gid == 3 ? x * x : gid == 4 ? x * y : gid == 5 ? y * y : 0.f;
				ymom[ks][e] = __float_as_uint(v);
			}
		}

		// Queue the survivors among the unread entries [0, hi), back to front, 32 entries per step (lane l takes entry
		// hi - 1 - l; the step's list entries and masks were loaded a step ahead) until a chunk is queued, then start the
		// gather of the chunk's records into rec: lane j < cnt gathers survivor j and keeps its pixel mask in cpm.
		int hi = nwalk, qhead = 0, qcount = 0;
		uint32_t epos = 0, epm = 0, cpm = 0;
		if (hi - 1 - lane >= 0) { epos = lrow[hi - 1 - lane]; epm = mrow[hi - 1 - lane]; }
		auto next_chunk = [&](float4* rec) -> int {
			__syncwarp();  // the queue slots of the previous chunk have been read
			while (qcount < BWD_CH && hi > 0) {
				const bool hit = hi - 1 - lane >= 0 && epm != 0u;  // a survivor that reached no pixel of the block has no gradient
				const uint32_t pos = epos, pm = epm;
				hi -= 32;
				if (hi - 1 - lane >= 0) { epos = lrow[hi - 1 - lane]; epm = mrow[hi - 1 - lane]; }
				// a chunk often takes two steps, and then the second step's loads above are waited on at once: bring the
				// entries of the step after them into L1 now (the two lines' ends of the 32-entry window, lanes 0 and 31)
				if (lane == 0 || lane == 31) {
					const int j = hi - 33 - lane;
					if (j >= 0) { prefetch_l1(lrow + j); prefetch_l1(mrow + j); }
				}
				const uint32_t mask = __ballot_sync(0xffffffffu, hit);
				if (hit) s_qe[(qhead + qcount + __popc(mask & ((1u << lane) - 1u))) & (BWD_QCAP - 1)] = make_uint2(pos, pm);
				qcount += __popc(mask);
			}
			__syncwarp();
			const int cnt = min(qcount, BWD_CH);
			if (lane < cnt) {
				const uint2 e = s_qe[(qhead + lane) & (BWD_QCAP - 1)];
				cpm = e.y;
				gather_rec(rec + 2 * lane, recs + e.x);
			}
			cp_async_commit();
			qhead += cnt;
			qcount -= cnt;
			BWD_PH_LAP(ph, BWD_PH_QUEUE);
			return cnt;
		};

		// chunk of cnt (<= BWD_CH) survivors whose records sit in s_q: start the gather of its channel rows into s_rows
		auto gather_rows = [&](int cnt, const float4* s_q, float* s_rows) {
			// ---- 1. gather the channel rows ----
			if (VEC) {
				// lane r knows the Gaussian id of survivor r; 32 / (2 NFT) feature rows are copied per trip (lane = row x 16-byte
				// piece), the id travelling by shuffle
				const uint32_t myid = lane < cnt ? bwd_row_id(__float_as_uint(s_q[2 * lane + 1].w)) : 0u;
				if (NFT > 0) {
					constexpr int NPF = NFT > 0 ? 2 * NFT : 1, RPI = 32 / NPF;
					const int sub = lane / NPF, q = lane % NPF;
#pragma unroll
					for (int it = 0; it < BWD_CH / RPI; it++) {
						const int r = it * RPI + sub;
						const uint32_t id = __shfl_sync(0xffffffffu, myid, r);
						const float* frow = a.feature + (size_t)id * (8 * NFT);
						if (r < cnt) cp_async16(s_rows + r * RS + 4 * q, reinterpret_cast<const float4*>(frow) + q);
					}
				}
				if (lane < cnt) cp_async16(s_rows + lane * RS + RGBD, a.rgbd + myid);
				if ((NRM || PLN) && lane < cnt) cp_async16(s_rows + lane * RS + RGBD + 4, a.nrm + myid);
			} else if (lane < cnt) {
				const uint32_t id = bwd_row_id(__float_as_uint(s_q[2 * lane + 1].w));
				float* row = s_rows + lane * RS;
				*reinterpret_cast<float4*>(row + RGBD) = a.rgbd[id];
				if (NRM || PLN) *reinterpret_cast<float4*>(row + RGBD + 4) = a.nrm[id];
				if (NFT > 0) {
					const float* f = a.feature + (size_t)id * F;
#pragma unroll
					for (int i = 0; i < 8 * NFT; i++) row[i] = (i < F) ? __ldg(f + i) : 0.f;
				}
			}
			cp_async_commit();
			BWD_PH_LAP(ph, BWD_PH_ROW_ISSUE);
		};

		// walked chunk of cnt survivors (records s_q, wgt tile s_wgt, q tile s_xs): GEMM 2/3, then between() (the wgt tile
		// has been read), then the flush
		auto finish = [&](int cnt, const float4* s_q, const float* s_wgt, float* s_xs, auto between) {
			// ---- 4 + 5. GEMM 2: dC[g][ch] = wgt[g][:] . Gpx[:][ch];  GEMM 3: M[g][m] = q[g][:] . Y[:][m]   (K = pixels) ----
			float dC[BWD_MT][NT][4], mom[BWD_MT][4];
#pragma unroll
			for (int mt = 0; mt < BWD_MT; mt++) {
#pragma unroll
				for (int i = 0; i < 4; i++) mom[mt][i] = 0.f;
#pragma unroll
				for (int nt = 0; nt < NT; nt++)
#pragma unroll
					for (int i = 0; i < 4; i++) dC[mt][nt][i] = 0.f;
			}
#pragma unroll
			for (int ks = 0; ks < 4; ks++) {
				// A quads of q and wgt: pixel pair pi = 4 ks + tig, survivors 16 mt + 2 gid (+1).  GEMM 3 first, so that the q
				// fragments are dead before the wgt fragments are loaded (registers: at most 128 per thread)
#pragma unroll
				for (int mt = 0; mt < BWD_MT; mt++) {
					// GEMM 3: the basis is exact in TF32, only q is split
					const float4 q4 = *reinterpret_cast<const float4*>(s_xs + (4 * ks + tig) * XS + mt * 32 + gid * 4);
					uint32_t qhi[4], qlo[4];
					tf32_split(q4.x, qhi[0], qlo[0]); tf32_split(q4.y, qhi[1], qlo[1]);
					tf32_split(q4.z, qhi[2], qlo[2]); tf32_split(q4.w, qhi[3], qlo[3]);
					mma_tf32(mom[mt], qlo[0], qlo[1], qlo[2], qlo[3], ymom[ks][0], ymom[ks][1]);
					mma_tf32(mom[mt], qhi[0], qhi[1], qhi[2], qhi[3], ymom[ks][0], ymom[ks][1]);
				}
				uint32_t ahi[BWD_MT][4], alo[BWD_MT][4];
#pragma unroll
				for (int mt = 0; mt < BWD_MT; mt++) {
					const float4 w4 = *reinterpret_cast<const float4*>(s_wgt + (4 * ks + tig) * XS + mt * 32 + gid * 4);
					tf32_split(w4.x, ahi[mt][0], alo[mt][0]); tf32_split(w4.y, ahi[mt][1], alo[mt][1]);
					tf32_split(w4.z, ahi[mt][2], alo[mt][2]); tf32_split(w4.w, ahi[mt][3], alo[mt][3]);
				}
				// B pairs of GEMM 2: cotangents of the pair's two pixels, channels NFT gid .. NFT gid + NFT - 1, then {r,g,b,depth}[gid].
				// This is gemm2_step (blend_mma.cuh) spelled out: through the helper ptxas schedules the NFT = 4 normal-plane
				// instantiation differently (same instruction count, other order), and this kernel's SASS stays as measured.
				const float* gp = s_g + (4 * ks + tig) * GS;
				if (NFT > 0) {
					float f[2 * (NFT > 0 ? NFT : 1)];
					if (NFT == 4) {
						const float4 u0 = *reinterpret_cast<const float4*>(gp + 8 * gid), u1 = *reinterpret_cast<const float4*>(gp + 8 * gid + 4);
						f[0] = u0.x; f[1] = u0.y; f[2 % (2 * NFT)] = u0.z; f[3 % (2 * NFT)] = u0.w;
						f[4 % (2 * NFT)] = u1.x; f[5 % (2 * NFT)] = u1.y; f[6 % (2 * NFT)] = u1.z; f[7 % (2 * NFT)] = u1.w;
					} else if (NFT == 2) {
						const float4 u0 = *reinterpret_cast<const float4*>(gp + 4 * gid);
						f[0] = u0.x; f[1] = u0.y; f[2 % (2 * NFT)] = u0.z; f[3 % (2 * NFT)] = u0.w;
					} else {
						const float2 u0 = *reinterpret_cast<const float2*>(gp + 2 * gid);
						f[0] = u0.x; f[1] = u0.y;
					}
#pragma unroll
					for (int nt = 0; nt < NFT; nt++) {
						uint32_t bh0, bl0, bh1, bl1;
						tf32_split(f[2 * nt], bh0, bl0);
						tf32_split(f[2 * nt + 1], bh1, bl1);
#pragma unroll
						for (int mt = 0; mt < BWD_MT; mt++) mma_3xtf32(dC[mt][nt], ahi[mt], alo[mt], bh0, bh1, bl0, bl1);
					}
				}
				{
					const float2 c = *reinterpret_cast<const float2*>(gp + 2 * (RGBD + gid));  // columns 4..7 are the zero padding
					uint32_t bh0, bl0, bh1, bl1;
					tf32_split(c.x, bh0, bl0);
					tf32_split(c.y, bh1, bl1);
#pragma unroll
					for (int mt = 0; mt < BWD_MT; mt++) mma_3xtf32(dC[mt][NFT], ahi[mt], alo[mt], bh0, bh1, bl0, bl1);
				}
			}
			__syncwarp();  // every lane has read its q and wgt fragments: s_xs becomes the per-Gaussian staging area
			BWD_PH_LAP(ph, BWD_PH_GEMM23);
			between();
			// ---- 6. flush ----
			// feature gradients straight from the D fragments; moments and {r,g,b,depth} gradients to s_xs[g][0..9]
			float* s_m = s_xs;  // [g][12]
#pragma unroll
			for (int mt = 0; mt < BWD_MT; mt++) {
#pragma unroll
				for (int h = 0; h < 2; h++) {
					const int g = 16 * mt + 2 * gid + h;  // D rows gid (h = 0) and gid + 8 (h = 1)
					if (tig < 3) *reinterpret_cast<float2*>(s_m + g * 12 + 2 * tig) = make_float2(mom[mt][2 * h], mom[mt][2 * h + 1]);
					if (tig < 2) *reinterpret_cast<float2*>(s_m + g * 12 + 6 + 2 * tig) = make_float2(dC[mt][NFT][2 * h], dC[mt][NFT][2 * h + 1]);
					// columns 4..7 of the tile, {dnx, dny, dnz, 0}, behind the [BWD_CH][12] rows
					if ((NRM || PLN) && tig >= 2) *reinterpret_cast<float2*>(s_m + BWD_CH * 12 + g * 4 + 2 * (tig - 2)) = make_float2(dC[mt][NFT][2 * h], dC[mt][NFT][2 * h + 1]);
					// F = 32: lane tig holds features 8 tig .. 8 tig + 7 of row g, one 32-byte sector (lo = the first four, hi
					// = the last four).  Lanes tig and tig ^ 1 swap halves so that each red.v4 below pairs with its neighbour's
					// into one whole sector: lane 2u + e adds into 16 u + 4 e (sector 2u: its own lo and the odd lane's lo), then
					// 16 u + 8 + 4 e (sector 2u + 1: the even lane's hi and its own hi).  Same reductions, same values per
					// address, but each one's L2 sector is written whole instead of as two half-sector updates.
					float sa[4], sb[4];
					if (VEC && NFT == 4) {
#pragma unroll
						for (int nt = 0; nt < 4; nt++) {
							const float lo = dC[mt][nt % NT][2 * h], hi = dC[mt][nt % NT][2 * h + 1];
							const float rv = __shfl_xor_sync(0xffffffffu, (tig & 1) ? lo : hi, 1);
							sa[nt] = (tig & 1) ? rv : lo;
							sb[nt] = (tig & 1) ? hi : rv;
						}
					}
					if (BWD_FEATURE_RED && NFT > 0 && g < cnt && a.dL_dfeat) {
						const uint32_t id = __float_as_uint(s_q[2 * g + 1].w);
						float* df = a.dL_dfeat + (size_t)id * F;
						// column 2 tig + e of feature tile nt is feature NFT (2 tig + e) + nt
						if (VEC) {
							if (NFT == 4) {
								const int p16 = 16 * (tig >> 1) + 4 * (tig & 1);
								red_add_v4(df + p16, sa[0], sa[1], sa[2], sa[3]);
								red_add_v4(df + p16 + 8, sb[0], sb[1], sb[2], sb[3]);
							} else if (NFT == 2) {
								red_add_v4(df + 4 * tig, dC[mt][0][2 * h], dC[mt][1 % NT][2 * h], dC[mt][0][2 * h + 1], dC[mt][1 % NT][2 * h + 1]);
							} else {
								red_add(df + 2 * tig, dC[mt][0][2 * h]);
								red_add(df + 2 * tig + 1, dC[mt][0][2 * h + 1]);
							}
						} else {
#pragma unroll
							for (int nt = 0; nt < NFT; nt++) {
#pragma unroll
								for (int e = 0; e < 2; e++) {
									const int f = NFT * (2 * tig + e) + nt;
									if (f < F) red_add(df + f, dC[mt][nt][2 * h + e]);
								}
							}
						}
					}
				}
			}
			__syncwarp();
			if (lane < cnt) {
				const float4 r0 = s_q[2 * lane], r1 = s_q[2 * lane + 1];
				const float4 m0 = *reinterpret_cast<const float4*>(s_m + lane * 12);      // {M0, Mx, My, Mxx}
				const float4 m1 = *reinterpret_cast<const float4*>(s_m + lane * 12 + 4);  // {Mxy, Myy, dr, dg}
				const float2 m2 = *reinterpret_cast<const float2*>(s_m + lane * 12 + 8);  // {db, ddepth}
				const float u = r0.x - fbx0, v = r0.y - fby0;  // mean relative to the block origin: d = (u - x, v - y)
				const float ca = r0.z, cb = r0.w, cc = r1.x, op = r1.y;
				const float q_dx = u * m0.x - m0.y, q_dy = v * m0.x - m0.z;
				const float q_dxx = u * (u * m0.x - 2.f * m0.y) + m0.w;
				const float q_dxy = u * (v * m0.x - m0.z) - v * m0.y + m1.x;
				const float q_dyy = v * (v * m0.x - 2.f * m0.z) + m1.y;
				const float dmx = half_W * (-ca * q_dx - cb * q_dy);
				const float dmy = half_H * (-cc * q_dy - cb * q_dx);
				float* gb = a.gb + (size_t)__float_as_uint(r1.w) * GB_STRIDE;
				red_add_v4(gb, dmx, dmy, -0.5f * q_dxx, -0.5f * q_dxy);
				red_add_v4(gb + 4, -0.5f * q_dyy, __fdividef(m0.x, op), m1.z, m1.w);
				red_add_v4(gb + 8, m2.x, m2.y, 0.f, 0.f);  // {db, ddepth}
				if (NRM || PLN) {
					const float4 dn = *reinterpret_cast<const float4*>(s_m + BWD_CH * 12 + lane * 4);
					float* gn = a.gn + (size_t)__float_as_uint(r1.w) * 4;
					if (PLN) red_add_v4(gn, fmaf(-u, dn.z, dn.x), fmaf(-v, dn.z, dn.y), dn.z, 0.f);  // mean-relative
					else red_add_v4(gn, dn.x, dn.y, dn.z, 0.f);
				}
			}
			BWD_PH_LAP(ph, BWD_PH_FLUSH);
		};

		// Chunk k: its records arrive in record slot r and its channel rows in stage k & 1, and the chunk is handed to W as
		// soon as the rows are in.  Then C finishes chunk k - 1 in stage (k - 1) & 1, and as soon as GEMM 2 has read that
		// stage's wgt tile the rows of chunk k + 1 start travelling into it, during the flush.  Record slot r + 1 (mod 3) last
		// held chunk k - 2, flushed in the previous trip.
		int cnt = next_chunk(s_rec[0]), cnt_prev = 0;
		int r = 0, rp = BWD_NREC - 1;
		auto rows_of = [&](int c, float4* rec, float* rows) {  // the chunk's records are in flight: carry the masks, gather its rows
			if (c == 0) return;
			cp_async_wait<0>();
			if (lane < c) rec[2 * lane + 1].z = __uint_as_float(cpm);  // the block mask is spent: carry the pixel mask
			__syncwarp();
			BWD_PH_LAP(ph, BWD_PH_REC_WAIT);
			gather_rows(c, rec, rows);
		};
		rows_of(cnt, s_rec[0], s_rows[0]);
#pragma unroll 1
		for (int k = 0;; k++) {
			const int s = k & 1;
			const int rn = r == BWD_NREC - 1 ? 0 : r + 1;
			if (cnt > 0) {
				cp_async_wait<0>();  // this chunk's channel rows
				if (PLN) {  // the quad's offset relative to the block origin (see above)
					__syncwarp();
					planar_block_offset(s_rows[s] + RGBD + 4, RS, s_rec[r], cnt, lane, fbx0, fby0);
				}
				if (!W_GEMM1) {
					__syncwarp();
					BWD_PH_LAP(ph, BWD_PH_ROW_WAIT);
					gemm1(s_rows[s], s_x[s]);
				}
#ifdef MGS_BWD_PHASES
				ph.acc[BWD_PH_CHUNKS]++;
#endif
			}
			if (lane == 0) s_cnt[s] = cnt;
			__syncwarp();
			named_bar_arrive<BWD_BAR_FULL, 64>(s);
			BWD_PH_LAP(ph, W_GEMM1 ? BWD_PH_ROW_WAIT : BWD_PH_GEMM1);
			const int cnt_next = cnt > 0 ? next_chunk(s_rec[rn]) : 0;  // the next chunk's records travel while this one is finished
			// the scalar-row path loads synchronously, nothing would travel during the flush: it gathers after it (registers)
			auto next_rows = [&]() { rows_of(cnt_next, s_rec[rn], s_rows[s ^ 1]); };
			if (k > 0) {
				named_bar_sync<BWD_BAR_DONE, 64>(s ^ 1);
				BWD_PH_LAP(ph, BWD_PH_DONE_WAIT);
				finish(cnt_prev, s_rec[rp], s_rows[s ^ 1], s_x[s ^ 1], [&]() { if (VEC) next_rows(); });
			}
			if (!VEC || k == 0) next_rows();
			if (cnt == 0) break;
			cnt_prev = cnt;
			cnt = cnt_next;
			rp = r;
			r = rn;
		}
#ifdef MGS_BWD_PHASES
		ph.put(a.bwd_phases, BWD_PH_QUEUE, BWD_PH_FLUSH, BWD_PH_C_TOTAL, true);
#endif
	}
#ifdef MGS_CTA_LOG
	__syncthreads();  // the CTA ends with the companion's last flush, after the walker has left its loop
	cta_log_put(a, t_start, 1u, (unsigned int)sub, (unsigned int)nwalk);
#endif
}

// Channel groups (F > 32, BlendArgs::groups): the same replay with one warp per block doing every step, 12 CTAs per SM.
// At F = 64 and 128 the launch is several waves deep, and there the two-warp kernel measured slower on an H100.
template <bool VEC, bool DM, bool NRM, bool PLN>
__global__ void __launch_bounds__(32, 12) blend_bwd_groups_kernel(BlendArgs a)
{
	constexpr int NFT = 4;
	constexpr bool GRP = true;
	constexpr int NT = NFT + 1;          // channel tiles of 8: NFT feature tiles + {r,g,b,depth, 4 x zero}
	constexpr int CHP = 8 * NT;          // padded channel count
	constexpr int RS = CHP;              // channel-row stride (floats): [8 NFT features | r g b depth | 0 0 0 0]
	constexpr int RGBD = 8 * NFT;
	constexpr int GS = 2 * CHP;          // s_g stride per pixel pair
	constexpr int XS = 2 * BWD_CH + 4;   // s_x / s_wgt stride per pixel pair (+4: spreads the pairs over the banks)
	constexpr int ROWS_FLOATS = (BWD_CH * RS > 16 * XS) ? BWD_CH * RS : 16 * XS;  // the rows buffer is reused for the wgt tile
	__shared__ __align__(16) float4 s_rec[2][BWD_CH * 2];  // records of the current and the next chunk: {x,y,ca,cb}, {cc,op,pixel mask,id}
	__shared__ uint2 s_qe[BWD_QCAP];                       // survivor queue, back to front: {list position, pixel mask}
	__shared__ __align__(16) float s_rows[ROWS_FLOATS];    // C[j][RS]; after GEMM 1: wgt tile
	__shared__ __align__(16) float s_x[16 * XS];           // Wd tile; the walk overwrites it with q in place; then per-Gaussian staging
	__shared__ __align__(16) float s_g[16 * GS];           // cotangent rows of the block's pixels

#ifdef MGS_CTA_LOG
	const unsigned long long t_start = cta_log_now();
#endif
	const int lane = threadIdx.x;
	const int gid = lane >> 2, tig = lane & 3;
	const int sub = blockIdx.x & 7;
	// channel group (BlendArgs::groups): dL/dalpha is linear in c . g, so it splits over the groups.  Group g takes its own
	// (c . g)_g and S_g; only group 0 carries the {r,g,b,depth} cotangents and the background term.
	const int grp = GRP ? (int)(blockIdx.x >> 3) % a.groups : 0;
	const int rank = GRP ? (int)(blockIdx.x >> 3) / a.groups : (int)(blockIdx.x >> 3);
	const int tile = a.tile_order ? (int)a.tile_order[rank] : rank;  // longest lists first
	const int tile_x = tile % a.grid_x, tile_y = tile / a.grid_x;
	const int bx0 = tile_x * TILE_X + (sub & 1) * WARP_BX;
	const int by0 = tile_y * TILE_Y + (sub >> 1) * WARP_BY;
	const int pxi = bx0 + (lane >> 2), pyi = by0 + (lane & 3);  // walk role: lane = pixel (x = lane >> 2, y = lane & 3)
	const bool inside = pxi < a.W && pyi < a.H;
	if (__all_sync(0xffffffffu, !inside)) return;  // the forward skipped this block: it has no block_nwalk
	const float fbx0 = (float)bx0, fby0 = (float)by0;
	const size_t HW = (size_t)a.H * a.W;
	const size_t pix = (size_t)a.W * pyi + pxi;
	const int F = a.F;                 // feature row stride
	const int c0 = 32 * grp;           // first channel of the group
	const int Fg = GRP ? min(F - c0, 32) : F;  // channels of the group
	const bool first = grp == 0;

	// ---- per-pixel state and cotangent rows ----
	float T = 0.f, bgterm = 0.f;
	{
		float g4[4] = { 0.f, 0.f, 0.f, 0.f };  // zero in groups >= 1: no colour / depth gradient, no background term
		float h = 0.f;                         // alpha cotangent (group 0 only), enters the background term as in blend_bwd_kernel
		// upstream gradients of the fused loss heads (loss_heads.cuh): the cotangent planes were written for d loss = 1
		const float sc_color = a.cot_scale ? a.cot_scale[0] : 1.f, sc_feat = a.cot_scale ? a.cot_scale[1] : 1.f;
		if (inside) {
			T = a.final_T[pix];
			if (first) {
#pragma unroll
				for (int ch = 0; ch < 3; ch++) g4[ch] = sc_color * a.dL_dcolor[ch * HW + pix];
				if (a.dL_ddepth) g4[3] = a.dL_ddepth[pix];
				if (a.dL_dalpha) h = a.dL_dalpha[pix];
				if (DM) depth_mask_cotangents(a, pix, g4[3], h);
			}
		}
		bgterm = T * (a.bg[0] * g4[0] + a.bg[1] * g4[1] + a.bg[2] * g4[2] - h);
		float* grow = s_g + (lane >> 1) * GS + (lane & 1);  // element (pixel, ch) at [pi][ch][e]
#pragma unroll
		for (int c = 0; c < 4; c++) {
			grow[2 * (RGBD + c)] = g4[c];
			// NRM: the normal plane's cotangent in columns 4..6, unscaled (the plane has no background term either)
			grow[2 * (RGBD + 4 + c)] = (NRM && c < 3 && inside && first) ? a.dL_dnormal[c * HW + pix] : 0.f;
			// PLN: g4 is zero outside the image and in groups >= 1
			if (PLN) grow[2 * (RGBD + 4 + c)] = c == 0 ? g4[3] * (float)(lane >> 2) : c == 1 ? g4[3] * (float)(lane & 3) : c == 2 ? g4[3] : 0.f;
		}
		if (NFT > 0) {
#pragma unroll
			for (int i = 0; i < 8 * NFT; i++)
				grow[2 * i] = (inside && i < Fg && a.dL_dfeature) ? sc_feat * a.dL_dfeature[(size_t)(c0 + i) * HW + pix] : 0.f;
		}
	}
	// only the entries up to the block's last contributor can have contributed to a pixel of the block
	const int nwalk = (int)a.block_nwalk[8 * tile + sub];
	if (nwalk == 0) return;  // nothing blended into this block
	for (int i = lane; i < ROWS_FLOATS / 4; i += 32) reinterpret_cast<float4*>(s_rows)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
	__syncwarp();

	const uint2 range = a.ranges[tile];
	const InstRec* const recs = a.recs + range.x;                                   // the tile's records, by 0-based list position
	const uint32_t* const lrow = a.block_list + sub * a.mask_stride + range.x;     // this block's work list
	const uint32_t* const mrow = a.pix_mask + sub * a.mask_stride + range.x;       // pixel masks, by block-list entry
	const float pfx = (float)pxi, pfy = (float)pyi;
	float S = 0.f;  // sum over the contributors behind the current one of a_j T_j (c_j . g)
	const int xofs = (lane >> 1) * XS + (lane & 1) * 2;  // this pixel's slot in the [pi][j >> 1][e][j & 1] tiles
	// GEMM 3's B operand: moments basis of the two pixels of k-slots (ks, tig) and (ks, tig + 4): p = 8 ks + 2 tig + e,
	// x = p >> 2, y = p & 3; column gid selects {1, x, y, x^2, x y, y^2, 0, 0}
	uint32_t ymom[4][2];
#pragma unroll
	for (int ks = 0; ks < 4; ks++) {
#pragma unroll
		for (int e = 0; e < 2; e++) {
			const int p = 8 * ks + 2 * tig + e;
			const float x = (float)(p >> 2), y = (float)(p & 3);
			const float v = gid == 0 ? 1.f : gid == 1 ? x : gid == 2 ? y : gid == 3 ? x * x : gid == 4 ? x * y : gid == 5 ? y * y : 0.f;
			ymom[ks][e] = __float_as_uint(v);
		}
	}
	const float half_W = 0.5f * a.W, half_H = 0.5f * a.H;

	// Queue the survivors among the unread entries [0, hi), back to front, 32 entries per step (lane l takes entry
	// hi - 1 - l; the step's list entries and masks were loaded a step ahead) until a chunk is queued, then start the
	// gather of the chunk's records into s_rec[b]: lane j < cnt gathers survivor j and keeps its pixel mask in cpm.
	int hi = nwalk, qhead = 0, qcount = 0;
	uint32_t epos = 0, epm = 0, cpm = 0;
	if (hi - 1 - lane >= 0) { epos = lrow[hi - 1 - lane]; epm = mrow[hi - 1 - lane]; }
	auto next_chunk = [&](int b) -> int {
		__syncwarp();  // the queue slots of the previous chunk have been read
		while (qcount < BWD_CH && hi > 0) {
			const bool hit = hi - 1 - lane >= 0 && epm != 0u;  // a survivor that reached no pixel of the block has no gradient
			const uint32_t pos = epos, pm = epm;
			hi -= 32;
			if (hi - 1 - lane >= 0) { epos = lrow[hi - 1 - lane]; epm = mrow[hi - 1 - lane]; }
			const uint32_t mask = __ballot_sync(0xffffffffu, hit);
			if (hit) s_qe[(qhead + qcount + __popc(mask & ((1u << lane) - 1u))) & (BWD_QCAP - 1)] = make_uint2(pos, pm);
			qcount += __popc(mask);
		}
		__syncwarp();
		const int cnt = min(qcount, BWD_CH);
		if (lane < cnt) {
			const uint2 e = s_qe[(qhead + lane) & (BWD_QCAP - 1)];
			cpm = e.y;
			gather_rec(s_rec[b] + 2 * lane, recs + e.x);
		}
		cp_async_commit();
		qhead += cnt;
		qcount -= cnt;
		return cnt;
	};
	int cnt_next = next_chunk(0);
	const float4* s_q = nullptr;

	// run the cnt (<= BWD_CH) survivors whose records sit in s_rec[buf]
	auto process_chunk = [&](int cnt, int buf) {
		// ---- 1. gather the channel rows ----
		if (VEC) {
			// lane r knows the Gaussian id of survivor r; 32 / (2 NFT) feature rows are copied per trip (lane = row x 16-byte
			// piece), the id travelling by shuffle
			const uint32_t myid = lane < cnt ? __float_as_uint(s_q[2 * lane + 1].w) : 0u;
			if (NFT > 0) {
				constexpr int NPF = NFT > 0 ? 2 * NFT : 1, RPI = 32 / NPF;
				const int sub = lane / NPF, q = lane % NPF;
#pragma unroll
				for (int it = 0; it < BWD_CH / RPI; it++) {
					const int r = it * RPI + sub;
					const uint32_t id = __shfl_sync(0xffffffffu, myid, r);
					// a remainder group (Fg < 32) copies its 4-channel pieces only: the columns behind them hold finite leftovers
					// of the wgt tile, and their cotangents are zero
					const float* frow = a.feature + (GRP ? (size_t)id * F + c0 : (size_t)id * (8 * NFT));
					if (r < cnt && (!GRP || 4 * q < Fg)) cp_async16(s_rows + r * RS + 4 * q, reinterpret_cast<const float4*>(frow) + q);
				}
			}
			if (lane < cnt) cp_async16(s_rows + lane * RS + RGBD, a.rgbd + myid);
			if ((NRM || PLN) && first && lane < cnt) cp_async16(s_rows + lane * RS + RGBD + 4, a.nrm + myid);
		} else if (lane < cnt) {
			const uint32_t id = __float_as_uint(s_q[2 * lane + 1].w);
			float* row = s_rows + lane * RS;
			*reinterpret_cast<float4*>(row + RGBD) = a.rgbd[id];
			if ((NRM || PLN) && first) *reinterpret_cast<float4*>(row + RGBD + 4) = a.nrm[id];
			if (NFT > 0) {
				const float* f = a.feature + (size_t)id * F + c0;
#pragma unroll
				for (int i = 0; i < 8 * NFT; i++) row[i] = (i < Fg) ? __ldg(f + i) : 0.f;
			}
		}
		cp_async_commit();
		cnt_next = next_chunk(buf ^ 1);  // the next chunk's records travel while this chunk runs
		cp_async_wait<1>();              // the channel rows
		__syncwarp();
		if (PLN && first) {  // the quad's offset relative to the block origin (blend_bwd_kernel)
			planar_block_offset(s_rows + RGBD + 4, RS, s_q, cnt, lane, fbx0, fby0);
			__syncwarp();
		}
		// ---- 2. GEMM 1: Wd[p][j] = Gpx[p][:] . C[j][:]   (M = pixels (2 tiles), N = survivors, K = channels) ----
		{
			float wd[2][BWD_CH / 8][4];
#pragma unroll
			for (int mt = 0; mt < 2; mt++)
#pragma unroll
				for (int nt = 0; nt < BWD_CH / 8; nt++)
#pragma unroll
					for (int i = 0; i < 4; i++) wd[mt][nt][i] = 0.f;
#pragma unroll
			for (int ks = 0; ks < NT; ks++) {
				uint32_t ahi[2][4], alo[2][4];
#pragma unroll
				for (int mt = 0; mt < 2; mt++) {
					const float4 v = *reinterpret_cast<const float4*>(s_g + (8 * mt + gid) * GS + (8 * ks + 2 * tig) * 2);
					tf32_split(v.x, ahi[mt][0], alo[mt][0]); tf32_split(v.y, ahi[mt][1], alo[mt][1]);
					tf32_split(v.z, ahi[mt][2], alo[mt][2]); tf32_split(v.w, ahi[mt][3], alo[mt][3]);
				}
#pragma unroll
				for (int nt = 0; nt < BWD_CH / 8; nt++) {
					const float2 v = *reinterpret_cast<const float2*>(s_rows + (8 * nt + gid) * RS + 8 * ks + 2 * tig);
					uint32_t bh0, bl0, bh1, bl1;
					tf32_split(v.x, bh0, bl0);
					tf32_split(v.y, bh1, bl1);
					mma_3xtf32(wd[0][nt], ahi[0], alo[0], bh0, bh1, bl0, bl1);
					mma_3xtf32(wd[1][nt], ahi[1], alo[1], bh0, bh1, bl0, bl1);
				}
			}
			// D fragment (mt, nt): pixels (pi = 8 mt + gid, e = 0 | 1), survivors 8 nt + 2 tig (+1): one 16-byte store
#pragma unroll
			for (int mt = 0; mt < 2; mt++)
#pragma unroll
				for (int nt = 0; nt < BWD_CH / 8; nt++)
					*reinterpret_cast<float4*>(s_x + (8 * mt + gid) * XS + (4 * nt + tig) * 4) =
						make_float4(wd[mt][nt][0], wd[mt][nt][1], wd[mt][nt][2], wd[mt][nt][3]);
		}
		__syncwarp();  // Wd complete; the rows buffer is free for the wgt tile
		// ---- 3. walk, back to front (queue order): lane = pixel.  Per k-step of 8 survivors: first the eight footprint
		// evaluations (independent, they overlap in the pipeline), then the short sequential recurrence on T and S. ----
		float* s_wgt = s_rows;
#pragma unroll 1
		for (int j0 = 0; j0 < BWD_CH; j0 += 8) {
			float al[8], opG[8], rinv[8];  // alpha, opacity * G, 1 / (1 - alpha); alpha = opG = 0, rinv = 1 for pairs that did not contribute
#pragma unroll
			for (int u = 0; u < 8; u++) {
				const int j = j0 + u;
				const float4 r0 = s_q[2 * j], r1 = s_q[2 * j + 1];
				const float dx = r0.x - pfx, dy = r0.y - pfy;
				const float op = r1.y;
				const float power = -0.5f * (r0.z * dx * dx + r1.x * dy * dy) - r0.w * dx * dy;
				const float G = __expf(power);  // ex2.approx-based (rel. error ~1e-6): the decision below is the forward's, not this
				const float alpha = min(ALPHA_MAX, op * G);
				// whether the pair contributed is the forward's own decision (pixel mask); slots past cnt hold stale entries
				const bool valid = (j < cnt) && ((__float_as_uint(r1.z) >> lane) & 1u);
				al[u] = valid ? alpha : 0.f;
				opG[u] = valid ? op * G : 0.f;
				rinv[u] = __fdividef(1.f, 1.f - al[u]);
			}
#pragma unroll
			for (int u = 0; u < 8; u++) {
				const int jofs = (j0 >> 1) * 4 + (u >> 1) * 4 + (u & 1);  // survivor j0 + u
				const float wdot = s_x[xofs + jofs];
				const float Tk = T * rinv[u];                                 // transmittance in front of this Gaussian
				const float wgt = al[u] * Tk;                                 // d(pixel channel) / d(colour of this Gaussian)
				const float dL_dalpha = Tk * wdot - (S + bgterm) * rinv[u];
				s_wgt[xofs + jofs] = wgt;
				s_x[xofs + jofs] = opG[u] * dL_dalpha;                        // q = dL/dG * G  (dL/dG = opacity * dL/dalpha)
				T = Tk;                                                       // unchanged where the pair is skipped (rinv = 1)
				S = fmaf(wgt, wdot, S);                                       // likewise (wgt = 0)
			}
		}
		__syncwarp();
		// ---- 4 + 5. GEMM 2: dC[g][ch] = wgt[g][:] . Gpx[:][ch];  GEMM 3: M[g][m] = q[g][:] . Y[:][m]   (K = pixels) ----
		float dC[BWD_MT][NT][4], mom[BWD_MT][4];
#pragma unroll
		for (int mt = 0; mt < BWD_MT; mt++) {
#pragma unroll
			for (int i = 0; i < 4; i++) mom[mt][i] = 0.f;
#pragma unroll
			for (int nt = 0; nt < NT; nt++)
#pragma unroll
				for (int i = 0; i < 4; i++) dC[mt][nt][i] = 0.f;
		}
#pragma unroll
		for (int ks = 0; ks < 4; ks++) {
			// A quads of wgt and q: pixel pair pi = 4 ks + tig, survivors 16 mt + 2 gid (+1)
			uint32_t ahi[BWD_MT][4], alo[BWD_MT][4], qhi[BWD_MT][4], qlo[BWD_MT][4];
#pragma unroll
			for (int mt = 0; mt < BWD_MT; mt++) {
				const float4 w4 = *reinterpret_cast<const float4*>(s_wgt + (4 * ks + tig) * XS + mt * 32 + gid * 4);
				const float4 q4 = *reinterpret_cast<const float4*>(s_x + (4 * ks + tig) * XS + mt * 32 + gid * 4);
				tf32_split(w4.x, ahi[mt][0], alo[mt][0]); tf32_split(w4.y, ahi[mt][1], alo[mt][1]);
				tf32_split(w4.z, ahi[mt][2], alo[mt][2]); tf32_split(w4.w, ahi[mt][3], alo[mt][3]);
				tf32_split(q4.x, qhi[mt][0], qlo[mt][0]); tf32_split(q4.y, qhi[mt][1], qlo[mt][1]);
				tf32_split(q4.z, qhi[mt][2], qlo[mt][2]); tf32_split(q4.w, qhi[mt][3], qlo[mt][3]);
			}
			// B pairs of GEMM 2: cotangents of the pair's two pixels, channels NFT gid .. NFT gid + NFT - 1, then {r,g,b,depth}[gid]
			gemm2_step<NFT, BWD_MT>(dC, ahi, alo, s_g + (4 * ks + tig) * GS, gid);
			// GEMM 3: the basis is exact in TF32, only q is split
#pragma unroll
			for (int mt = 0; mt < BWD_MT; mt++) {
				mma_tf32(mom[mt], qlo[mt][0], qlo[mt][1], qlo[mt][2], qlo[mt][3], ymom[ks][0], ymom[ks][1]);
				mma_tf32(mom[mt], qhi[mt][0], qhi[mt][1], qhi[mt][2], qhi[mt][3], ymom[ks][0], ymom[ks][1]);
			}
		}
		__syncwarp();  // every lane has read its q fragments: s_x becomes the per-Gaussian staging area
		// ---- 6. flush ----
		// feature gradients straight from the D fragments; moments and {r,g,b,depth} gradients to s_x[g][0..9]
		float* s_m = s_x;  // [g][12]
#pragma unroll
		for (int mt = 0; mt < BWD_MT; mt++) {
#pragma unroll
			for (int h = 0; h < 2; h++) {
				const int g = 16 * mt + 2 * gid + h;  // D rows gid (h = 0) and gid + 8 (h = 1)
				if (tig < 3) *reinterpret_cast<float2*>(s_m + g * 12 + 2 * tig) = make_float2(mom[mt][2 * h], mom[mt][2 * h + 1]);
				if (tig < 2) *reinterpret_cast<float2*>(s_m + g * 12 + 6 + 2 * tig) = make_float2(dC[mt][NFT][2 * h], dC[mt][NFT][2 * h + 1]);
				// columns 4..7 of the tile, {dnx, dny, dnz, 0}, behind the [BWD_CH][12] rows
				if ((NRM || PLN) && tig >= 2) *reinterpret_cast<float2*>(s_m + BWD_CH * 12 + g * 4 + 2 * (tig - 2)) = make_float2(dC[mt][NFT][2 * h], dC[mt][NFT][2 * h + 1]);
				if (NFT > 0 && g < cnt && a.dL_dfeat) {
					const uint32_t id = __float_as_uint(s_q[2 * g + 1].w);
					red_feature_row<NFT, VEC, GRP>(a.dL_dfeat + (size_t)id * F + c0, dC[mt], h, tig, Fg);
				}
			}
		}
		__syncwarp();
		if (lane < cnt) {
			const float4 r0 = s_q[2 * lane], r1 = s_q[2 * lane + 1];
			const float4 m0 = *reinterpret_cast<const float4*>(s_m + lane * 12);      // {M0, Mx, My, Mxx}
			const float4 m1 = *reinterpret_cast<const float4*>(s_m + lane * 12 + 4);  // {Mxy, Myy, dr, dg}
			const float2 m2 = *reinterpret_cast<const float2*>(s_m + lane * 12 + 8);  // {db, ddepth}
			const float u = r0.x - fbx0, v = r0.y - fby0;  // mean relative to the block origin: d = (u - x, v - y)
			const float ca = r0.z, cb = r0.w, cc = r1.x, op = r1.y;
			const float q_dx = u * m0.x - m0.y, q_dy = v * m0.x - m0.z;
			const float q_dxx = u * (u * m0.x - 2.f * m0.y) + m0.w;
			const float q_dxy = u * (v * m0.x - m0.z) - v * m0.y + m1.x;
			const float q_dyy = v * (v * m0.x - 2.f * m0.z) + m1.y;
			const float dmx = half_W * (-ca * q_dx - cb * q_dy);
			const float dmy = half_H * (-cc * q_dy - cb * q_dx);
			float* gb = a.gb + (size_t)__float_as_uint(r1.w) * GB_STRIDE;
			red_add_v4(gb, dmx, dmy, -0.5f * q_dxx, -0.5f * q_dxy);
			red_add_v4(gb + 4, -0.5f * q_dyy, __fdividef(m0.x, op), m1.z, m1.w);
			if (first) red_add_v4(gb + 8, m2.x, m2.y, 0.f, 0.f);  // {db, ddepth}: zero in the other groups
			if ((NRM || PLN) && first) {
				const float4 dn = *reinterpret_cast<const float4*>(s_m + BWD_CH * 12 + lane * 4);
				float* gn = a.gn + (size_t)__float_as_uint(r1.w) * 4;
				if (PLN) red_add_v4(gn, fmaf(-u, dn.z, dn.x), fmaf(-v, dn.z, dn.y), dn.z, 0.f);  // mean-relative
				else red_add_v4(gn, dn.x, dn.y, dn.z, 0.f);
			}
		}
	};

	for (int buf = 0; cnt_next > 0; buf ^= 1) {
		const int cnt = cnt_next;
		cp_async_wait<0>();  // this chunk's records
		s_q = s_rec[buf];
		if (lane < cnt) s_rec[buf][2 * lane + 1].z = __uint_as_float(cpm);  // the block mask is spent: carry the pixel mask
		__syncwarp();
		process_chunk(cnt, buf);
	}
#ifdef MGS_CTA_LOG
	cta_log_put(a, t_start, 1u, (unsigned int)sub, (unsigned int)nwalk);
#endif
}

bool feature_rows_vectorizable(const float* feature, int F);

template <int NFT, bool DM, bool NRM, bool PLN>
static void launch_bwd_t(const BlendArgs& a, cudaStream_t s)
{
	const int grid = a.grid_x * a.grid_y * 8;
	const bool vec = (NFT == 0) || (a.F == 8 * NFT && feature_rows_vectorizable(a.feature, a.F) &&
		(reinterpret_cast<uintptr_t>(a.dL_dfeat) & 15) == 0);
	if (vec) blend_bwd_kernel<NFT, true, DM, NRM, PLN><<<grid, 64, 0, s>>>(a);
	else blend_bwd_kernel<NFT, false, DM, NRM, PLN><<<grid, 64, 0, s>>>(a);
}

template <bool DM, bool NRM, bool PLN = false>
static void launch_bwd_dm(const BlendArgs& a, cudaStream_t s)
{
	if (a.groups > 1) {
		const int grid = a.grid_x * a.grid_y * 8 * a.groups;
		const bool vec = feature_rows_vectorizable(a.feature, a.F) && (reinterpret_cast<uintptr_t>(a.dL_dfeat) & 15) == 0;
		if (vec) blend_bwd_groups_kernel<true, DM, NRM, PLN><<<grid, 32, 0, s>>>(a);
		else blend_bwd_groups_kernel<false, DM, NRM, PLN><<<grid, 32, 0, s>>>(a);
		return;
	}
	switch (nft_for(a.F)) {
	case 0: launch_bwd_t<0, DM, NRM, PLN>(a, s); break;
	case 1: launch_bwd_t<1, DM, NRM, PLN>(a, s); break;
	case 2: launch_bwd_t<2, DM, NRM, PLN>(a, s); break;
	default: launch_bwd_t<4, DM, NRM, PLN>(a, s); break;
	}
}

void launch_blend_bwd(const BlendArgs& a, cudaStream_t s)
{
	if (a.planar) {  // never with the normal plane (launch_blend_fwd)
		if (a.tgt_depth || a.tgt_mask) launch_bwd_dm<true, false, true>(a, s);
		else launch_bwd_dm<false, false, true>(a, s);
	} else if (a.nrm) launch_bwd_dm<false, true>(a, s);  // never with the depth / mask heads (launch_blend_fwd)
	else if (a.tgt_depth || a.tgt_mask) launch_bwd_dm<true, false>(a, s);
	else launch_bwd_dm<false, false>(a, s);
}

// The median depth is the view-space z of one Gaussian per pixel, chosen by a piecewise-constant rule: its cotangent goes to
// that Gaussian's depth slot of the blend-stage records and nowhere else.  One thread per pixel.  PLN (planar depth): the
// median depth is z + a (px - mu_x) + b (py - mu_y), so the cotangent also goes to the contributor's quad gradients gn, in
// gn's mean-relative form (blend_bwd_kernel).
template <bool PLN>
__global__ void median_depth_bwd_kernel(int N, const int* __restrict__ median_id, const float* __restrict__ dL_dmedian, float* gb, int W,
	float* gn, const float2* __restrict__ means2D)
{
	const int p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p >= N) return;
	const int id = median_id[p];
	const float g = dL_dmedian[p];
	if (id >= 0 && g != 0.f) red_add(gb + (size_t)id * GB_STRIDE + 9, g);
	if (PLN && id >= 0 && g != 0.f) {
		const int py = p / W, px = p - py * W;
		const float2 mu = means2D[id];
		red_add_v4(gn + (size_t)id * 4, g * ((float)px - mu.x), g * ((float)py - mu.y), g, 0.f);
	}
}

void launch_median_depth_bwd(int N, const int* median_id, const float* dL_dmedian, float* gb, cudaStream_t s, int W, float* gn,
	const float2* means2D)
{
	if (N <= 0) return;
	if (gn) median_depth_bwd_kernel<true><<<ceil_div(N, 256), 256, 0, s>>>(N, median_id, dL_dmedian, gb, W, gn, means2D);
	else median_depth_bwd_kernel<false><<<ceil_div(N, 256), 256, 0, s>>>(N, median_id, dL_dmedian, gb, W, gn, means2D);
}

}  // namespace mgs
