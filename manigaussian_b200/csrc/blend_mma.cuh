// Warp-level tensor-core helpers for the channel contractions of the blend kernels.
//
// The per-pixel channel accumulation of the forward blend, acc[px][ch] += w[px][g] * c[g][ch], and the two channel
// contractions of the backward blend are small dense GEMMs per 32-survivor chunk of a warp's 8x4 pixel block
// ([32 px x 32 g] x [32 g x 36 ch]).  Done with FFMA they are 70 % of both kernels' instructions at 7-10 of 32 lanes
// active (a splat covers ~7 of a block's 32 pixels); done with mma.sync.m16n8k8 TF32 they cost one instruction per
// 1024 multiply-adds regardless of which lanes contribute.  fp32 accuracy (the 1e-4 bar against the reference) is kept
// with the 3xTF32 split: x = hi + lo, hi = x truncated to TF32, lo = x - hi (exact in fp32);  a*b ~= a_lo*b_hi + a_hi*b_lo + a_hi*b_hi
// (the dropped lo*lo term is 2^-20 relative).  HMMA.1688.F32.TF32 issues from the tensor pipe, which runs beside the FP32
// pipes.
//
// Fragment layout of mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 (gid = lane >> 2, tig = lane & 3):
//   A (16x8):  a0 (gid, tig)   a1 (gid+8, tig)   a2 (gid, tig+4)   a3 (gid+8, tig+4)
//   B (8x8):   b0 (k = tig, n = gid)             b1 (k = tig+4, n = gid)
//   C/D(16x8): c0 (gid, 2 tig)  c1 (gid, 2 tig+1)  c2 (gid+8, 2 tig)  c3 (gid+8, 2 tig+1)
// Row/column/k indices are ours to assign to pixels, Gaussians and channels (the contraction does not care about their
// order as long as A and B agree), which the kernels use to make every fragment load a 128-bit shared-memory access.
#pragma once
#include <cstdint>
#include "mgs_common.cuh"

namespace mgs {

// x = hi + lo with hi = x truncated to TF32 (the tensor core ignores the low 13 mantissa bits of a .tf32 operand, so x's
// own bits serve as hi) and lo = x - hi, exact in fp32 and itself truncated by the tensor core: the split carries x to
// 2^-20 relative.  Two instructions per value (LOP3 + FADD); cvt.rna.tf32.f32 has no SASS form on sm_90a and expands to
// four (FSETP + IADD + LOP3 and a constant), and rounding instead of truncating hi would not buy accuracy.
__device__ __forceinline__ void tf32_split(float x, uint32_t& hi, uint32_t& lo)
{
	hi = __float_as_uint(x);
	lo = __float_as_uint(x - __uint_as_float(hi & 0xffffe000u));
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1)
{
	asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
		: "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
		: "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// d += A * B with both operands split (3 tensor instructions, small terms first)
__device__ __forceinline__ void mma_3xtf32(float (&d)[4], const uint32_t (&ahi)[4], const uint32_t (&alo)[4], uint32_t bhi0, uint32_t bhi1,
	uint32_t blo0, uint32_t blo1)
{
	mma_tf32(d, alo[0], alo[1], alo[2], alo[3], bhi0, bhi1);
	mma_tf32(d, ahi[0], ahi[1], ahi[2], ahi[3], blo0, blo1);
	mma_tf32(d, ahi[0], ahi[1], ahi[2], ahi[3], bhi0, bhi1);
}

// Channel-row layout in shared memory shared by both blend kernels: NFT = number of 8-wide feature column tiles
// (0, 1, 2 or 4 for F = 0, <= 8, <= 16, <= 32), row = [8*NFT features (zero padded) | r g b depth], row stride RS floats
// chosen so that the fragment loads below are bank-conflict free.
template <int NFT> struct RowLayout;
template <> struct RowLayout<0> { static constexpr int RS = 8,  RGBD = 0; };
template <> struct RowLayout<1> { static constexpr int RS = 24, RGBD = 8; };
template <> struct RowLayout<2> { static constexpr int RS = 24, RGBD = 16; };
template <> struct RowLayout<4> { static constexpr int RS = 40, RGBD = 32; };

__host__ __device__ inline int nft_for(int F) { return F <= 0 ? 0 : (F <= 8 ? 1 : (F <= 16 ? 2 : 4)); }

// The NFT feature values a thread needs from one channel row for column tiles 0..NFT-1: column n = gid of tile nt is
// feature NFT*gid + nt, so they are contiguous (one LDS.128 / .64 / .32).
template <int NFT>
__device__ __forceinline__ void load_feat(const float* row, int gid, float (&f)[4])
{
	if (NFT == 4) {
		const float4 v = *reinterpret_cast<const float4*>(row + 4 * gid);
		f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
	} else if (NFT == 2) {
		const float2 v = *reinterpret_cast<const float2*>(row + 2 * gid);
		f[0] = v.x; f[1] = v.y;
	} else if (NFT == 1) {
		f[0] = row[gid];
	}
}

// GEMM 2 of the backward blend for one k-step of pixels (blend_bwd.cu), dC[g][ch] += wgt[g][p] C[p][ch]: the A quads of MT
// 16-row Gaussian tiles, split, times the B pairs of the channel rows gp of pixel pair 4 ks + tig in the [pi][ch][e] layout
// (row stride 2 (8 NFT + 8): channels NFT gid .. NFT gid + NFT - 1 for feature tiles 0 .. NFT - 1, then {r,g,b,depth}[gid] for
// tile NFT, whose columns 4..7 are the zero padding or the normal quad).  rgbd = false skips tile NFT.  Shared by blend_bwd and
// lift_kernel (lift.cu), which runs the same contraction with the blend weights against a 2D map.
template <int NFT, int MT>
__device__ __forceinline__ void gemm2_step(float (&dC)[MT][NFT + 1][4], const uint32_t (&ahi)[MT][4], const uint32_t (&alo)[MT][4],
	const float* gp, int gid, bool rgbd = true)
{
	constexpr int RGBD = 8 * NFT;
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
			for (int mt = 0; mt < MT; mt++) mma_3xtf32(dC[mt][nt], ahi[mt], alo[mt], bh0, bh1, bl0, bl1);
		}
	}
	if (rgbd) {
		const float2 c = *reinterpret_cast<const float2*>(gp + 2 * (RGBD + gid));  // columns 4..7 are the zero padding
		uint32_t bh0, bl0, bh1, bl1;
		tf32_split(c.x, bh0, bl0);
		tf32_split(c.y, bh1, bl1);
#pragma unroll
		for (int mt = 0; mt < MT; mt++) mma_3xtf32(dC[mt][NFT], ahi[mt], alo[mt], bh0, bh1, bl0, bl1);
	}
}

// The feature row of GEMM 2's D row (h = 0: gid, 1: gid + 8) of one Gaussian tile d into df (the row's first channel of the
// group) with float reductions: column 2 tig + e of feature tile nt is feature NFT (2 tig + e) + nt, so with VEC (16-byte
// aligned rows, Fg % 4 == 0, and Fg = 8 NFT without GRP) a thread holds whole 4-channel pieces and adds them as
// red.global.add.v4.f32 (at NFT = 4 two per 32-byte sector); else scalar reductions of the channels below Fg.  Shared by
// blend_bwd_groups_kernel and lift_kernel.
template <int NFT, bool VEC, bool GRP>
__device__ __forceinline__ void red_feature_row(float* df, const float (&d)[NFT + 1][4], int h, int tig, int Fg)
{
	constexpr int NT = NFT + 1;
	if (VEC) {
		if (NFT == 4) {  // Fg % 4 == 0 here
			if (!GRP || 8 * tig < Fg)
				red_add_v4(df + 8 * tig, d[0][2 * h], d[1 % NT][2 * h], d[2 % NT][2 * h], d[3 % NT][2 * h]);
			if (!GRP || 8 * tig + 4 < Fg)
				red_add_v4(df + 8 * tig + 4, d[0][2 * h + 1], d[1 % NT][2 * h + 1], d[2 % NT][2 * h + 1], d[3 % NT][2 * h + 1]);
		} else if (NFT == 2) {
			red_add_v4(df + 4 * tig, d[0][2 * h], d[1 % NT][2 * h], d[0][2 * h + 1], d[1 % NT][2 * h + 1]);
		} else {
			red_add(df + 2 * tig, d[0][2 * h]);
			red_add(df + 2 * tig + 1, d[0][2 * h + 1]);
		}
	} else {
#pragma unroll
		for (int nt = 0; nt < NFT; nt++) {
#pragma unroll
			for (int e = 0; e < 2; e++) {
				const int f = NFT * (2 * tig + e) + nt;
				if (f < Fg) red_add(df + f, d[nt][2 * h + e]);
			}
		}
	}
}

}  // namespace mgs
