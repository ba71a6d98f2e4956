// Shared by the forward and backward blend kernels.
//
// Work decomposition: ONE WARP = ONE CTA = one 8x4 pixel block of a 16x16 tile (tile ids / work lists stay the
// reference's 16x16 tiles; eight single-warp CTAs per tile, 8 G with G channel groups of 32 features when F > 32,
// BlendArgs::groups).  The binning stage gives every block its own work list: the tile-list positions of the instances
// whose footprint can reach the block (block_lists_kernel, binning.cu).  A warp reads its list coalesced and gathers the
// chunk's 32-byte records by position with 16-byte cp.async (SASS LDGSTS), the next chunk's while the current one runs.
// No CTA-wide barrier exists anywhere: warps of a heavy tile never wait for each other, finished warps free their SM
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

}  // namespace mgs
