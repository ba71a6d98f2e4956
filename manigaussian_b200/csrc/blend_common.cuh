// Shared by the forward and backward blend kernels.
//
// Work decomposition: ONE WARP = ONE CTA = one 8x4 pixel block of a 16x16 tile (tile ids / work lists stay the
// reference's 16x16 tiles; eight single-warp CTAs share a tile's list, 8 G with G channel groups of 32 features when
// F > 32, BlendArgs::groups).  A warp streams the tile's sorted 32-byte
// instance records through its own RING-deep shared-memory ring with 1-D TMA bulk copies (SASS UBLKCP), one copy per
// batch of records tracked by an mbarrier, keeps the records whose footprint reaches its block (one bit per block in the
// record, set by the binning stage) and works on the survivors.  No CTA-wide barrier exists anywhere: warps of a heavy
// tile never wait for each other, finished warps free their SM slot immediately, and the hardware scheduler balances
// the 8*T*V small CTAs across the 132 SMs of an H100.
#pragma once
#include "mgs_common.cuh"
#include "mgs_kernels.h"

namespace mgs {

#ifndef MGS_RING
#define MGS_RING 2
#endif
// record batches in flight / resident per warp
constexpr int RING = MGS_RING;

// {x, y, ca, cb} and {cc, op, block mask, id} views of a record
__device__ __forceinline__ uint32_t rec_id(const float4& r1) { return __float_as_uint(r1.w); }
// can the record contribute to 8x4 block `sub` (0..7, row-major 2 x 4) of its tile?  Decided once per instance by the
// binning stage (exact ellipse-vs-block test of the alpha >= 1/255 footprint, binning.cu); conservative, never changes a pixel.
__device__ __forceinline__ bool rec_hits_block(const float4& r1, int sub) { return (__float_as_uint(r1.z) >> sub) & 1u; }

// Per-warp record ring of BATCH-record buffers.  All methods are called by the whole (converged) warp.
// MASKS: every batch also brings the 32-bit pixel masks of its records (msrc[i] belongs to src[i]) into a second ring
// under the same mbarrier.  The bulk copy covers the 16-byte-aligned span around them, so the mask array must be readable
// up to the next 16-byte boundary on either side.
template <int BATCH, bool MASKS = false>
struct WarpRecRingT {
	static constexpr int MSTRIDE = BATCH + 8;  // u32 per mask buffer: BATCH masks + up to 3 + 3 alignment words, 16-byte multiple
	InstRec* buf;        // RING * BATCH records
	uint64_t* bar;       // RING mbarriers (count 1)
	const InstRec* src;  // first record of the (sub)list this warp walks
	int total;           // number of records to walk
	bool reverse;        // walk from the back (backward pass): batch 0 is the LAST BATCH-aligned block
	uint32_t* mbuf;        // MASKS: RING * MSTRIDE words, 16-byte aligned
	const uint32_t* msrc;  // MASKS: pixel mask of the first record

	__device__ __forceinline__ int num_batches() const { return (total + BATCH - 1) / BATCH; }
	__device__ __forceinline__ int batch_lo(int k) const { return reverse ? BATCH * (num_batches() - 1 - k) : BATCH * k; }
	__device__ __forceinline__ int batch_n(int k) const { return min(BATCH, total - batch_lo(k)); }

	__device__ __forceinline__ void init(InstRec* b, uint64_t* bars, const InstRec* s, int n, bool rev,
		uint32_t* mb = nullptr, const uint32_t* ms = nullptr)
	{
		buf = b; bar = bars; src = s; total = n; reverse = rev; mbuf = mb; msrc = ms;
		if ((threadIdx.x & 31) == 0) {
#pragma unroll
			for (int i = 0; i < RING; i++) mbar_init(&bar[i], 1);
			mbar_fence_init();
		}
		__syncwarp();
	}
	// start the copy of batch k into buffer k % RING (the buffer's previous contents must be dead)
	__device__ __forceinline__ void issue(int k)
	{
		__syncwarp();
		if ((threadIdx.x & 31) == 0) {
			const int b = k % RING, n = batch_n(k);
			uint32_t bytes = (uint32_t)n * (uint32_t)sizeof(InstRec);
			uintptr_t m0 = 0, m1 = 0;
			if (MASKS) {
				const uintptr_t m = reinterpret_cast<uintptr_t>(msrc + batch_lo(k));
				m0 = m & ~(uintptr_t)15;
				m1 = (m + 4u * (uint32_t)n + 15u) & ~(uintptr_t)15;
				bytes += (uint32_t)(m1 - m0);
			}
			fence_proxy_async();
			mbar_arrive_expect_tx(&bar[b], bytes);
			bulk_g2s(buf + b * BATCH, src + batch_lo(k), (uint32_t)n * (uint32_t)sizeof(InstRec), &bar[b]);
			if (MASKS) bulk_g2s(mbuf + b * MSTRIDE, reinterpret_cast<const void*>(m0), (uint32_t)(m1 - m0), &bar[b]);
		}
	}
	// MASKS: the pixel masks of batch k's records (valid after wait(k), until the batch's buffer is reissued).  batch_lo is a
	// multiple of 4 masks, so every batch starts at the same offset within its 16-byte-aligned copy.
	__device__ __forceinline__ const uint32_t* masks(int k) const
	{
		static_assert(BATCH % 4 == 0, "mask batches must keep the 16-byte phase of msrc");
		return mbuf + (k % RING) * MSTRIDE + ((reinterpret_cast<uintptr_t>(msrc) & 15u) >> 2);
	}
	__device__ __forceinline__ const float4* wait(int k)
	{
		const int b = k % RING;
		mbar_wait(&bar[b], (uint32_t)((k / RING) & 1));
		return reinterpret_cast<const float4*>(buf + b * BATCH);
	}
	__device__ __forceinline__ const float4* buffer(int k) const { return reinterpret_cast<const float4*>(buf + (k % RING) * BATCH); }
};

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
