// Loss heads of ManiGaussian's neural-rendering objective, fused next to the rasterizer (SURVEY.md 8(f) row f4).
//
// Replaces, for the images the forward blend has just produced, the PyTorch operator chains of
//   l2_loss(render, gt)       = mean((render - gt)^2)                          agents/manigaussian_bc/loss.py:12-13
//   cosine_loss(embed, gt)    = 1 - mean_px cos_sim(embed[px, :], gt[px, :])   loss.py:18-23 (F.cosine_similarity, eps 1e-8)
// as NeuralRenderer.forward applies them (neural_rendering.py:300-318), together with their backward: per pixel the
// kernel produces the two loss partial sums and the cotangent planes dL/d(render), dL/d(embed) the backward blend reads,
// so that no image-sized PyTorch kernel runs between the forward and the backward of a training step.
//   S_rgb = sum (x - g)^2        ->  loss_rgb   = S_rgb / (3 N),     d loss_rgb / dx_c   = 2 (x_c - g_c) / (3 N)
//   S_cos = sum_px cos_px        ->  loss_embed = 1 - S_cos / N,     d loss_embed / dx_f = -(1/N) d cos / dx_f
//   cos = x.y / (nx ny), nx = max(|x|, eps), ny = max(|y|, eps);  d cos / dx = y / (nx ny) - cos x / (|x| nx)   for |x| > 0
//   (ATen's cosine_similarity backward: continuous at |x| = eps, where |x| nx = |x|^2 above eps and |x| eps below; 0 at x = 0).
//   Norms whose square overflows fp32 (|x| >~ 1e19) are outside what these heads evaluate.
#pragma once
#include "mgs_common.cuh"

namespace mgs {

constexpr float COS_EPS = 1e-8f;  // F.cosine_similarity's default eps

struct CosTerms {
	float inv_nn;   // 1 / (max(|x|, eps) max(|y|, eps))
	float k;        // cos / (|x| max(|x|, eps)) where |x| > 0, else 0
	float cos;
};
__device__ __forceinline__ CosTerms cos_terms(float xy, float xx, float yy)
{
	const float nx = sqrtf(xx), ny = sqrtf(yy);
	CosTerms t;
	t.inv_nn = 1.0f / (fmaxf(nx, COS_EPS) * fmaxf(ny, COS_EPS));
	t.cos = xy * t.inv_nn;
	// above eps |x| max(|x|, eps) = |x|^2 = xx; below it the clamped norm is a constant, but |x| still carries x's direction
	t.k = nx > COS_EPS ? t.cos / xx : (nx > 0.f ? t.cos / (nx * COS_EPS) : 0.f);
	return t;
}
// d cos / dx_f
__device__ __forceinline__ float cos_grad(const CosTerms& t, float x, float y) { return y * t.inv_nn - t.k * x; }

// Depth and mask heads (DESIGN row f7; INTEGRATION.md §4), per pixel from the depth plane D and the alpha plane A = 1 - final_T:
//   depth  valid = (g > 0) && (A > 0.5), a constant;  d = D / A;  loss_depth = sum_valid |d - g| / n,  n = sum valid (0 if n = 0)
//          d |d - g| / dD = sign(d - g) / A,  d |d - g| / dA = -sign(d - g) d / A   (ATen's div backward: -grad (D / A) / A)
//   mask   a = clamp(A, EPS, 1 - EPS);  loss_mask = mean_px BCE(a, m) as F.binary_cross_entropy: logs clamped at -100,
//          d BCE / da = (a - m) / max(a (1 - a), 1e-12), passed to A only inside [EPS, 1 - EPS] (ATen's clamp backward)
// The cotangent planes are unscaled: the depth head's upstream scale g_depth / n is only known once every CTA has counted
// its pixels, so the backward applies it (and g_mask) on load.
constexpr float DEPTH_MIN_ALPHA = 0.5f;
constexpr float MASK_EPS = 1e-4f, MASK_EPS_HI = 0.9999f;  // the float32 values torch.clamp(A, 1e-4, 1 - 1e-4) uses

struct DepthTerms {
	float err;    // |d - g| where valid, else 0
	float n;      // 1 where valid, else 0
	float cot_d;  // d |d - g| / dD
	float cot_a;  // d |d - g| / dA
};
__device__ __forceinline__ DepthTerms depth_terms(float D, float A, float g)
{
	DepthTerms t;
	const bool valid = g > 0.f && A > DEPTH_MIN_ALPHA;
	const float d = valid ? D / A : 0.f;
	const float diff = d - g;
	const float s = diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f);
	t.err = valid ? fabsf(diff) : 0.f;
	t.n = valid ? 1.f : 0.f;
	t.cot_d = valid ? s / A : 0.f;
	t.cot_a = valid ? -s * (d / A) : 0.f;
	return t;
}

struct MaskTerms {
	float bce;   // BCE(clamp(A), m)
	float grad;  // d BCE / dA
};
__device__ __forceinline__ MaskTerms mask_terms(float A, float m)
{
	MaskTerms t;
	const float a = fminf(fmaxf(A, MASK_EPS), MASK_EPS_HI);
	const float la = fmaxf(logf(a), -100.f), l1a = fmaxf(log1pf(-a), -100.f);
	t.bce = (m - 1.f) * l1a - m * la;
	t.grad = (A >= MASK_EPS && A <= MASK_EPS_HI) ? (a - m) / fmaxf((1.f - a) * a, 1e-12f) : 0.f;
	return t;
}

}  // namespace mgs
