// L1 + SSIM photometric loss (DESIGN row f9): the objective 3DGS trains with, (1 - lambda) L1 + lambda (1 - SSIM), as the
// reference's loss module defines it (gaussian-splatting utils/loss_utils.py `l1_loss`, `ssim`/_ssim; ManiGaussian ships
// a copy in agents/manigaussian_bc/loss.py).  Per plane (one colour channel of one view), with G the 11x11 Gaussian window
// (sigma 1.5) and G(*) its zero-padded ("same", padding 5) convolution:
//   mu_x = G(*)x, mu_g = G(*)g, sxx = G(*)x^2 - mu_x^2, sgg = G(*)g^2 - mu_g^2, sxg = G(*)(xg) - mu_x mu_g
//   A = 2 mu_x mu_g + C1, B = 2 sxg + C2, C = mu_x^2 + mu_g^2 + C1, D = sxx + sgg + C2,  S = A B / (C D)
//   ssim = mean S,  l1 = mean |x - g|  (N = C H W entries per view)
// and the gradient with respect to x (the target is a constant):
//   dS/dmu_x = 2 mu_g (B - A) / (C D) - 2 mu_x S (1/C - 1/D),  dS/dE[x^2] = -S / D,  dS/dE[xg] = 2 A / (C D)
//   d ssim / dx = (G(*)dS/dmu_x + 2 x G(*)dS/dE[x^2] + g G(*)dS/dE[xg]) / N
// (the window is symmetric, so the adjoint of the zero-padded convolution is the same convolution of the partials, which
// are zero outside the image).
//
// Both kernels: one CTA per SS_TW x SS_TH output tile of one plane.  The tile plus a 5-pixel halo is staged in shared memory
// (reads outside the image are 0), a horizontal 11-tap pass writes the row sums of the tile's columns for every halo row,
// and a vertical 11-tap pass finishes each output pixel.  The forward writes the three partials of every pixel as unscaled
// planes; the backward convolves them and writes the complete colour cotangent.
#include "mgs_common.cuh"
#include "mgs_kernels.h"

namespace mgs {

constexpr int SS_R = 5;                                 // window radius (11 taps)
constexpr int SS_TW = 32, SS_TH = 16;                   // output tile: a warp per tile row, 8 warps x 2 rows
constexpr int SS_THREADS = 256;
constexpr int SS_IW = SS_TW + 2 * SS_R, SS_IH = SS_TH + 2 * SS_R;
constexpr float SSIM_C1 = 0.01f * 0.01f, SSIM_C2 = 0.03f * 0.03f;

// exp(-(i - 5)^2 / 4.5) normalised to sum 1 (computed in float64, rounded once)
__constant__ float c_gauss[2 * SS_R + 1] = { 1.028380084e-03f, 7.598758135e-03f, 3.600077213e-02f, 1.093606895e-01f,
	2.130055377e-01f, 2.660117249e-01f, 2.130055377e-01f, 1.093606895e-01f, 3.600077213e-02f, 7.598758135e-03f, 1.028380084e-03f };

// blockIdx.z = v * C + c: plane c of view v.  x, g: [V,C,H,W]; terms: [V,3,C,H,W] ({dS/dmu_x, dS/dE[x^2], dS/dE[xg]} per
// channel); acc + v * acc_stride receives {sum |x - g|, sum S} of the view.
__global__ void __launch_bounds__(SS_THREADS) ssim_fwd_kernel(int C, int H, int W, const float* __restrict__ x,
	const float* __restrict__ g, float* __restrict__ terms, float* __restrict__ acc, int acc_stride)
{
	__shared__ float sx[SS_IH][SS_IW], sg[SS_IH][SS_IW];
	__shared__ float hz[5][SS_IH][SS_TW];
	const int plane = blockIdx.z, v = plane / C, c = plane - v * C;
	const size_t HW = (size_t)H * W;
	const float* xp = x + (size_t)plane * HW;
	const float* gp = g + (size_t)plane * HW;
	const int x0 = blockIdx.x * SS_TW, y0 = blockIdx.y * SS_TH;
	const int tid = threadIdx.x;
	for (int i = tid; i < SS_IH * SS_IW; i += SS_THREADS) {
		const int r = i / SS_IW, q = i - r * SS_IW;
		const int py = y0 - SS_R + r, px = x0 - SS_R + q;
		const bool in = py >= 0 && py < H && px >= 0 && px < W;
		const size_t o = in ? (size_t)py * W + px : 0;
		sx[r][q] = in ? xp[o] : 0.f;
		sg[r][q] = in ? gp[o] : 0.f;
	}
	__syncthreads();
	for (int i = tid; i < SS_IH * SS_TW; i += SS_THREADS) {
		const int r = i / SS_TW, q = i - r * SS_TW;
		float a = 0.f, b = 0.f, aa = 0.f, bb = 0.f, ab = 0.f;
#pragma unroll
		for (int k = 0; k <= 2 * SS_R; k++) {
			const float w = c_gauss[k], xv = sx[r][q + k], gv = sg[r][q + k];
			a += w * xv; b += w * gv; aa += w * xv * xv; bb += w * gv * gv; ab += w * xv * gv;
		}
		hz[0][r][q] = a; hz[1][r][q] = b; hz[2][r][q] = aa; hz[3][r][q] = bb; hz[4][r][q] = ab;
	}
	__syncthreads();
	const int tx = tid & 31, ty = tid >> 5;
	const size_t CHW = (size_t)C * HW;
	float* tp = terms + (size_t)v * 3 * CHW + (size_t)c * HW;
	float s_l1 = 0.f, s_S = 0.f;
#pragma unroll
	for (int j = 0; j < SS_TH / 8; j++) {
		const int r = ty + 8 * j, py = y0 + r, px = x0 + tx;
		if (py >= H || px >= W) continue;
		float m[5] = { 0.f, 0.f, 0.f, 0.f, 0.f };
#pragma unroll
		for (int k = 0; k <= 2 * SS_R; k++) {
			const float w = c_gauss[k];
#pragma unroll
			for (int t = 0; t < 5; t++) m[t] += w * hz[t][r + k][tx];
		}
		const float mux = m[0], mug = m[1];
		const float sxx = m[2] - mux * mux, sgg = m[3] - mug * mug, sxg = m[4] - mux * mug;
		const float A = 2.f * mux * mug + SSIM_C1, B = 2.f * sxg + SSIM_C2;
		const float Cc = mux * mux + mug * mug + SSIM_C1, D = sxx + sgg + SSIM_C2;
		const float inv_cd = 1.f / (Cc * D);
		const float S = A * B * inv_cd;
		const size_t o = (size_t)py * W + px;
		tp[o] = 2.f * mug * (B - A) * inv_cd - 2.f * mux * S * (1.f / Cc - 1.f / D);
		tp[CHW + o] = -S / D;
		tp[2 * CHW + o] = 2.f * A * inv_cd;
		s_S += S;
		s_l1 += fabsf(sx[r + SS_R][tx + SS_R] - sg[r + SS_R][tx + SS_R]);
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
		s_l1 += __shfl_xor_sync(0xffffffffu, s_l1, o);
		s_S += __shfl_xor_sync(0xffffffffu, s_S, o);
	}
	if (tx == 0) {
		red_add(acc + (size_t)v * acc_stride, s_l1);
		red_add(acc + (size_t)v * acc_stride + 1, s_S);
	}
}

// cot_out = cot_in_scale[0] * cot_in + g_l1 sign(x - g) / N + g_ssim d ssim / dx, with {g_l1, g_ssim} = scale[2 v ..] (scale
// NULL: 1) and cot_in NULL: 0, cot_in_scale NULL: 1.  blend_slot (single view only): receives {1, cot_in_scale[1]} -- the
// colour / feature scales the blend backward then reads.
__global__ void __launch_bounds__(SS_THREADS) ssim_bwd_kernel(int C, int H, int W, const float* __restrict__ x,
	const float* __restrict__ g, const float* __restrict__ terms, const float* __restrict__ scale, const float* __restrict__ cot_in,
	const float* __restrict__ cot_in_scale, float* __restrict__ cot_out, float* __restrict__ blend_slot)
{
	__shared__ float st[3][SS_IH][SS_IW];
	__shared__ float hz[3][SS_IH][SS_TW];
	const int plane = blockIdx.z, v = plane / C, c = plane - v * C;
	const size_t HW = (size_t)H * W, CHW = (size_t)C * HW;
	const float* tp = terms + (size_t)v * 3 * CHW + (size_t)c * HW;
	const int x0 = blockIdx.x * SS_TW, y0 = blockIdx.y * SS_TH;
	const int tid = threadIdx.x;
	if (blend_slot && tid == 0 && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) {
		blend_slot[0] = 1.f;
		blend_slot[1] = cot_in_scale ? cot_in_scale[1] : 1.f;
	}
	for (int i = tid; i < SS_IH * SS_IW; i += SS_THREADS) {
		const int r = i / SS_IW, q = i - r * SS_IW;
		const int py = y0 - SS_R + r, px = x0 - SS_R + q;
		const bool in = py >= 0 && py < H && px >= 0 && px < W;
		const size_t o = in ? (size_t)py * W + px : 0;
#pragma unroll
		for (int t = 0; t < 3; t++) st[t][r][q] = in ? tp[t * CHW + o] : 0.f;
	}
	__syncthreads();
	for (int i = tid; i < SS_IH * SS_TW; i += SS_THREADS) {
		const int r = i / SS_TW, q = i - r * SS_TW;
		float a = 0.f, b = 0.f, e = 0.f;
#pragma unroll
		for (int k = 0; k <= 2 * SS_R; k++) {
			const float w = c_gauss[k];
			a += w * st[0][r][q + k]; b += w * st[1][r][q + k]; e += w * st[2][r][q + k];
		}
		hz[0][r][q] = a; hz[1][r][q] = b; hz[2][r][q] = e;
	}
	__syncthreads();
	const float inv_n = 1.f / (float)CHW;
	const float g_l1 = (scale ? scale[2 * v] : 1.f) * inv_n, g_ss = (scale ? scale[2 * v + 1] : 1.f) * inv_n;
	const float s_in = cot_in_scale ? cot_in_scale[0] : 1.f;
	const size_t base = (size_t)plane * HW;
	const int tx = tid & 31, ty = tid >> 5;
#pragma unroll
	for (int j = 0; j < SS_TH / 8; j++) {
		const int r = ty + 8 * j, py = y0 + r, px = x0 + tx;
		if (py >= H || px >= W) continue;
		float m0 = 0.f, m1 = 0.f, m2 = 0.f;
#pragma unroll
		for (int k = 0; k <= 2 * SS_R; k++) {
			const float w = c_gauss[k];
			m0 += w * hz[0][r + k][tx]; m1 += w * hz[1][r + k][tx]; m2 += w * hz[2][r + k][tx];
		}
		const size_t o = base + (size_t)py * W + px;
		const float xv = x[o], gv = g[o], d = xv - gv;
		const float sgn = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
		float val = g_l1 * sgn + g_ss * (m0 + 2.f * xv * m1 + gv * m2);
		if (cot_in) val += s_in * cot_in[o];
		cot_out[o] = val;
	}
}

static dim3 ssim_grid(int V, int C, int H, int W) { return dim3(ceil_div(W, SS_TW), ceil_div(H, SS_TH), V * C); }

void launch_ssim_fwd(int V, int C, int H, int W, const float* x, const float* g, float* terms, float* acc, int acc_stride, cudaStream_t s)
{
	if (V <= 0 || C <= 0 || H <= 0 || W <= 0) return;
	ssim_fwd_kernel<<<ssim_grid(V, C, H, W), SS_THREADS, 0, s>>>(C, H, W, x, g, terms, acc, acc_stride);
}

void launch_ssim_bwd(int V, int C, int H, int W, const float* x, const float* g, const float* terms, const float* scale,
	const float* cot_in, const float* cot_in_scale, float* cot_out, float* blend_slot, cudaStream_t s)
{
	if (V <= 0 || C <= 0 || H <= 0 || W <= 0) return;
	ssim_bwd_kernel<<<ssim_grid(V, C, H, W), SS_THREADS, 0, s>>>(C, H, W, x, g, terms, scale, cot_in, cot_in_scale, cot_out,
		blend_slot);
}

}  // namespace mgs
