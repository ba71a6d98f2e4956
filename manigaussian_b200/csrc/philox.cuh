// Philox4x32-10 (Random123) and the Box-Muller normals that MCMC density control (mcmc.cu) and default density control
// (densify.cu) draw from.  The counter is {slot, offset lo, offset hi, tag} and the key {seed lo, seed hi}; each caller owns
// its tags (include/mgs_rasterizer.h), so no two calls share a draw.
#pragma once
#include <cstdint>

namespace mgs {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1)
{
#pragma unroll
	for (int r = 0; r < 10; r++) {
		if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
		const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
		const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
		c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
	}
	return c;
}

// the words of slot `slot` at the generator state rng = {seed, offset} (device int64 [2])
__device__ __forceinline__ uint4 philox_draw(const long long* rng, uint32_t slot, uint32_t tag)
{
	const unsigned long long seed = (unsigned long long)rng[0], off = (unsigned long long)rng[1];
	return philox4x32_10(make_uint4(slot, (uint32_t)off, (uint32_t)(off >> 32), tag), (uint32_t)seed, (uint32_t)(seed >> 32));
}

// Box-Muller in fp32: (w0, w1) give z0 and z1, (w2, w3) give z2
__device__ __forceinline__ void philox_normals(uint4 w, float& z0, float& z1, float& z2)
{
	const float r0 = sqrtf(-2.f * logf(((float)w.x + 1.f) * 2.3283064365386963e-10f));
	const float r1 = sqrtf(-2.f * logf(((float)w.z + 1.f) * 2.3283064365386963e-10f));
	float s0, c0, s1, c1;
	sincospif(2.f * ((float)w.y * 2.3283064365386963e-10f), &s0, &c0);
	sincospif(2.f * ((float)w.w * 2.3283064365386963e-10f), &s1, &c1);
	z0 = r0 * c0;
	z1 = r0 * s0;
	z2 = r1 * c1;
}

}  // namespace mgs
