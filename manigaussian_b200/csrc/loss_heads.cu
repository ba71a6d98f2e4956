// The fused loss heads (loss_heads.cuh) for images that already sit in memory: V views, planar [V,3,N] / [V,F,N], one launch.
// One thread per pixel; the channel planes are read and written coalesced (a warp = 32 consecutive pixels of one plane).
#include "loss_heads.cuh"
#include "mgs_kernels.h"

namespace mgs {

__global__ void __launch_bounds__(256) loss_heads_kernel(int V, int F, int N, const float* __restrict__ color,
	const float* __restrict__ feature, const float* __restrict__ tgt_color, const float* __restrict__ tgt_feature,
	float* __restrict__ cot_color, float* __restrict__ cot_feature, float* __restrict__ loss_acc)
{
	const int v = blockIdx.y;
	const int px = blockIdx.x * blockDim.x + threadIdx.x;
	const bool in = px < N;
	const float invN = 1.0f / (float)N;
	float s_rgb = 0.f, s_cos = 0.f;
	const bool emb = F > 0 && feature && tgt_feature;
	if (in) {
		if (color) {  // null: features only (the blend epilogue did the colour head; F > 32)
			const size_t cb = (size_t)v * 3 * N + px;
#pragma unroll
			for (int c = 0; c < 3; c++) {
				const float d = color[cb + (size_t)c * N] - tgt_color[cb + (size_t)c * N];
				s_rgb += d * d;
				cot_color[cb + (size_t)c * N] = (2.0f / 3.0f) * invN * d;
			}
		}
		if (emb) {
			const size_t fb = (size_t)v * F * N + px;
			float xy = 0.f, xx = 0.f, yy = 0.f;
			for (int f = 0; f < F; f++) {
				const float x = feature[fb + (size_t)f * N], g = tgt_feature[fb + (size_t)f * N];
				xy += x * g; xx += x * x; yy += g * g;
			}
			const CosTerms ct = cos_terms(xy, xx, yy);
			s_cos = ct.cos;
			for (int f = 0; f < F; f++)
				cot_feature[fb + (size_t)f * N] = -invN * cos_grad(ct, feature[fb + (size_t)f * N], tgt_feature[fb + (size_t)f * N]);
		}
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
		s_rgb += __shfl_xor_sync(0xffffffffu, s_rgb, o);
		s_cos += __shfl_xor_sync(0xffffffffu, s_cos, o);
	}
	if ((threadIdx.x & 31) == 0) {
		if (color) red_add(loss_acc + 2 * v, s_rgb);
		if (emb) red_add(loss_acc + 2 * v + 1, s_cos);
	}
}

void launch_loss_heads(int V, int F, int N, const float* color, const float* feature, const float* tgt_color, const float* tgt_feature,
	float* cot_color, float* cot_feature, float* loss_acc, cudaStream_t s)
{
	if (V <= 0 || N <= 0) return;
	dim3 grid(ceil_div(N, 256), V);
	loss_heads_kernel<<<grid, 256, 0, s>>>(V, F, N, color, feature, tgt_color, tgt_feature, cot_color, cot_feature, loss_acc);
}

}  // namespace mgs
