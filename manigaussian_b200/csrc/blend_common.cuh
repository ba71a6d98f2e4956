// Shared by the forward and backward blend kernels.
//
// Work decomposition: ONE CTA = one 8x4 pixel block of a 16x16 tile (tile ids / work lists stay the reference's 16x16
// tiles; eight CTAs per tile, 8 G with G channel groups of 32 features when F > 32, BlendArgs::groups).  The forward's CTA
// is one warp; the backward's is two cooperating warps (a walker and a companion, blend_bwd.cu), one warp for channel groups.  The binning stage gives
// every block its own work list: the tile-list positions of the instances whose footprint can reach the block
// (block_lists_kernel, binning.cu).  A warp reads its list coalesced and gathers the chunk's 32-byte records by position
// with 16-byte cp.async (SASS LDGSTS), the next chunk's while the current one runs.  The only barriers are the ones
// between the two warps of a backward CTA; CTAs of a heavy tile never wait for each other, finished CTAs free their SM
// slot immediately, and the hardware scheduler balances the 8*T*V small CTAs across the 132 SMs of an H100.
#pragma once
#include "mgs_common.cuh"
#include "mgs_kernels.h"

namespace mgs {

// {x, y, ca, cb} and {cc, op, block mask, id} views of a record
__device__ __forceinline__ uint32_t rec_id(const float4& r1) { return __float_as_uint(r1.w); }
// start the copy of record `rec` into dst[0..1] (two 16-byte pieces; completes with the thread's next cp.async group)
__device__ __forceinline__ void gather_rec(float4* dst, const InstRec* rec)
{
	cp_async16(dst, rec);
	cp_async16(dst + 1, reinterpret_cast<const float4*>(rec) + 1);
}

// The footprint evaluations of one k-step of the forward walk (lane = pixel at (pfx, pfy)): alpha of the pairs with the
// eight records q4[2 u], q4[2 u + 1] of k-step ks, 0 where the pair is skipped (power > 0, alpha < 1/255, or slot 8 ks + u
// at or past cnt).  Shared by blend_fwd_kernel and lift_kernel, so that the lift's weights are the forward's bit for bit.
__device__ __forceinline__ void walk_alphas(const float4* q4, float pfx, float pfy, int ks, int cnt, float (&al)[8])
{
#pragma unroll
	for (int u = 0; u < 8; u++) {
		const float4 p = q4[2 * u], q = q4[2 * u + 1];
		const float dx = p.x - pfx, dy = p.y - pfy;
		const float power = -0.5f * (p.z * dx * dx + q.x * dy * dy) - p.w * dx * dy;
		const float alpha = min(ALPHA_MAX, q.y * expf(power));
		const bool ok = (8 * ks + u < cnt) && !(power > 0.0f) && !(alpha < ALPHA_MIN);
		al[u] = ok ? alpha : 0.f;
	}
}

// Named barrier BASE + s (s = 0 | 1, warp-uniform) over N threads: bar.sync waits for the barrier, bar.arrive signals it
// without waiting.  The ids stay immediates: with an id held in a register ptxas reserves all 16 barriers of the CTA.
template <int BASE, int N>
__device__ __forceinline__ void named_bar_sync(int s)
{
	if (s == 0) asm volatile("bar.sync %0, %1;" ::"n"(BASE), "n"(N) : "memory");
	else asm volatile("bar.sync %0, %1;" ::"n"(BASE + 1), "n"(N) : "memory");
}
template <int BASE, int N>
__device__ __forceinline__ void named_bar_arrive(int s)
{
	if (s == 0) asm volatile("bar.arrive %0, %1;" ::"n"(BASE), "n"(N) : "memory");
	else asm volatile("bar.arrive %0, %1;" ::"n"(BASE + 1), "n"(N) : "memory");
}

#ifdef MGS_CTA_LOG
__device__ __forceinline__ unsigned long long cta_log_now()
{
	unsigned long long t;
	asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
	return t;
}
__device__ __forceinline__ void cta_log_put(const BlendArgs& a, unsigned long long t0, unsigned int kind, unsigned int sub, unsigned int len)
{
	if (a.cta_log == nullptr || threadIdx.x != 0) return;
	const unsigned long long t1 = cta_log_now();
	const unsigned int i = atomicAdd(a.cta_log_n, 1u);
	if (i >= a.cta_log_cap) return;
	unsigned int sm;
	asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
	unsigned long long* o = a.cta_log + 4 * (size_t)i;
	o[0] = t0; o[1] = t1;
	o[2] = (unsigned long long)(kind | (sub << 8)) | ((unsigned long long)len << 32);
	o[3] = (unsigned long long)sm | ((unsigned long long)blockIdx.x << 32);
}
#endif

#ifdef MGS_BWD_PHASES
// Measurement build only (tools/bwd_phases.py): where a two-warp backward CTA spends its cycles.  Each warp keeps one
// counter per phase (clock64() laps, lane 0's) and adds them into BlendArgs::bwd_phases when it leaves.
enum BwdPhase {
	// companion
	BWD_PH_QUEUE,      // queue the next chunk's survivors, start its record gather
	BWD_PH_REC_WAIT,   // wait for the next chunk's records
	BWD_PH_ROW_ISSUE,  // issue the next chunk's channel-row copies
	BWD_PH_ROW_WAIT,   // wait for this chunk's channel rows (and the FULL signal when the walker runs GEMM 1)
	BWD_PH_DONE_WAIT,  // wait for the walker to finish the previous chunk
	BWD_PH_GEMM23,     // GEMM 2/3 of the previous chunk
	BWD_PH_FLUSH,      // its reductions
	BWD_PH_C_TOTAL,    // the companion's whole loop
	// walker
	BWD_PH_FULL_WAIT,  // wait for the next chunk
	BWD_PH_GEMM1,      // its GEMM 1 (at small F the companion's, with the FULL signal: W_GEMM1 in blend_bwd.cu)
	BWD_PH_WALK,       // walk it
	BWD_PH_W_TOTAL,    // the walker's whole loop
	BWD_PH_CHUNKS,     // chunks (non-empty) handed over
	BWD_PH_CTAS,       // CTAs that reached the loop
	BWD_PH_COUNT
};
struct BwdPhaseClock {
	unsigned int acc[BWD_PH_COUNT];
	long long t, t0;
	__device__ __forceinline__ void start()
	{
#pragma unroll
		for (int i = 0; i < BWD_PH_COUNT; i++) acc[i] = 0u;
		t = t0 = clock64();
	}
	__device__ __forceinline__ void lap(int ph)
	{
		const long long n = clock64();
		acc[ph] += (unsigned int)(n - t);
		t = n;
	}
	// total: the phase that receives the whole loop; phases [first, last] are this warp's, and the lead (the companion)
	// also adds GEMM 1, which stays zero on the warp that does not run it
	__device__ __forceinline__ void put(unsigned long long* out, int first, int last, int total, bool lead)
	{
		acc[total] = (unsigned int)(clock64() - t0);
		if (out == nullptr || (threadIdx.x & 31) != 0) return;
#pragma unroll
		for (int i = 0; i < BWD_PH_COUNT; i++)
			if ((i >= first && i <= last) || i == total || (lead && (i == BWD_PH_GEMM1 || i == BWD_PH_CHUNKS || i == BWD_PH_CTAS)))
				atomicAdd(out + i, (unsigned long long)acc[i]);
	}
};
#define BWD_PH_LAP(ph, p) (ph).lap(p)
#else
#define BWD_PH_LAP(ph, p) do { } while (0)
#endif

}  // namespace mgs
