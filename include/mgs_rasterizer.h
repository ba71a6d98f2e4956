/*
 * mgs_rasterizer.h -- C ABI of the H100-native (sm_90a) differentiable Gaussian-splatting rasterizer.
 *
 * This is the drop-in boundary for ManiGaussian's rasterizer hot path.  Each entry point replaces one
 * static method of the reference's raw-pointer C++ API, CudaRasterizer::Rasterizer
 * (third_party/gaussian-splatting/submodules/diff-gaussian-rasterization/cuda_rasterizer/rasterizer.h:20-92,
 * implemented in rasterizer_impl.cu), which the reference's torch glue (rasterize_points.cu:36-247) and pybind
 * module (ext.cpp:14-18) wrap.  Plain C types only: device pointers, sizes, scalars, a CUDA stream handle
 * as void*, and C function pointers where the reference passes std::function<char*(size_t)> allocators.
 *
 * Conventions shared with the reference:
 *  - all arrays are fp32 device memory unless noted; a NULL pointer means "not provided"
 *    (reference: forward.cu:206,242; backward.cu:390,394);
 *  - viewmatrix / projmatrix are the 16-float row-vector (transposed) matrices read as m[4*col+row]
 *    (auxiliary.h:58-77); tan_fov* are tan(fov/2);
 *  - geom/binning/image state buffers are opaque bytes owned by the caller between forward and backward
 *    (rasterizer_impl.h:29-65); their internal layout is private to this library.
 * Differences (supersets) from the reference:
 *  - F, the number of feature channels, is a RUN-TIME argument (0..MGS_MAX_FEATURE_CHANNELS = 512) instead of the
 *    compile-time NUM_CHANNELS_language_feature (config.h:16); include_feature == (F > 0 && feature != NULL).
 *    F > 32 is blended in groups of 32 channels (each group walks the tile lists again, so the blend costs grow with
 *    ceil(F / 32));
 *  - an optional depth plane (out_depth / dL_dpix_depth) renders view-space z as one more blended channel;
 *  - an optional alpha plane (mgs_view_alpha, multi-view and multi-cloud calls) returns the accumulated opacity 1 - final_T;
 *  - an optional median-depth plane and per-pixel surface Gaussian id (mgs_view_median, the same calls);
 *  - an optional surface-normal plane (mgs_view_normal, the same calls);
 *  - work is enqueued on `stream` (the reference uses the legacy default stream);
 *  - outputs are fully overwritten: callers need not zero-initialise them.
 *
 * All functions return >= 0 on success and a negative MGS_ERR_* code on failure; mgs_last_error() returns a
 * thread-local description.  No handles; re-entrant like the reference.  The only process-wide state is a cache of
 * sort/scan scratch sizes and the opt-in stage timers of mgs_profile_*.
 */
#ifndef MGS_RASTERIZER_H
#define MGS_RASTERIZER_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MGS_ERR_INVALID_ARG (-1)
#define MGS_ERR_UNSUPPORTED (-2)
#define MGS_ERR_CUDA (-3)
#define MGS_ERR_ALLOC (-4)

#define MGS_MAX_FEATURE_CHANNELS 512

/* Allocator callback: return a device pointer to at least `bytes` bytes (any alignment >= 16; the library
 * re-aligns to 128), or NULL.  Replaces std::function<char*(size_t)> (rasterizer.h:32-34). */
typedef char* (*mgs_alloc_fn)(void* user, size_t bytes);

/* Library / ABI version (major*100 + minor). */
int mgs_abi_version(void);
const char* mgs_last_error(void);

/* Bytes the forward will request for the geometry (per-Gaussian) and image (per-pixel) state. */
size_t mgs_geometry_state_bytes(int P);
size_t mgs_image_state_bytes(int width, int height);
size_t mgs_binning_state_bytes(int num_rendered);

/*
 * Forward.  Replaces CudaRasterizer::Rasterizer::forward (rasterizer.h:31-60, rasterizer_impl.cu:198-355).
 * Returns num_rendered (R, the number of Gaussian/tile instances), which the caller passes to mgs_backward.
 *   D = active SH degree, M = SH coefficients per Gaussian (0 when shs == NULL), F = feature channels
 *   (0..MGS_MAX_FEATURE_CHANNELS; larger F returns MGS_ERR_UNSUPPORTED, as do mgs_backward and the multi-view calls).
 *   out_color [3,H,W], out_feature [F,H,W] (ignored when F == 0), out_depth [H,W] or NULL, radii int32 [P].
 * One stream synchronisation happens inside (R is read back to size the binning state), as in the reference
 * (rasterizer_impl.cu:284).
 */
int mgs_forward(
	mgs_alloc_fn geometry_alloc, void* geometry_user,
	mgs_alloc_fn binning_alloc, void* binning_user,
	mgs_alloc_fn image_alloc, void* image_user,
	int P, int D, int M, int F,
	const float* background,
	int width, int height,
	const float* means3D,
	const float* shs,
	const float* colors_precomp,
	const float* feature_precomp,
	const float* opacities,
	const float* scales,
	float scale_modifier,
	const float* rotations,
	const float* cov3D_precomp,
	const float* viewmatrix,
	const float* projmatrix,
	const float* cam_pos,
	float tan_fovx, float tan_fovy,
	int prefiltered,
	float* out_color,
	float* out_feature,
	float* out_depth,
	int* radii,
	int debug,
	void* stream);

/*
 * Instance count of one view (no reference counterpart).  mgs_forward_begin enqueues the per-Gaussian projection,
 * depth ordering and instance-offset scan of one view on `stream` -- the first half of mgs_forward -- and copies the
 * instance count to *host_num_rendered (pinned host memory recommended) asynchronously; the caller synchronises
 * `stream` before reading it.  Nothing is binned or blended.  The count sizes the binning state (binning_capacity) of
 * later mgs_forward_views calls.  P must be > 0.
 */
int mgs_forward_begin(
	mgs_alloc_fn geometry_alloc, void* geometry_user,
	mgs_alloc_fn image_alloc, void* image_user,
	int P, int D, int M,
	int width, int height,
	const float* means3D,
	const float* shs,
	const float* colors_precomp,
	const float* opacities,
	const float* scales,
	float scale_modifier,
	const float* rotations,
	const float* cov3D_precomp,
	const float* viewmatrix,
	const float* projmatrix,
	const float* cam_pos,
	float tan_fovx, float tan_fovy,
	int* radii,
	int* host_num_rendered,
	int debug,
	void* stream);

/*
 * Backward.  Replaces CudaRasterizer::Rasterizer::backward (rasterizer.h:62-91, rasterizer_impl.cu:359-463).
 *   dL_dpix [3,H,W], dL_dpix_F [F,H,W] or NULL, dL_dpix_depth [H,W] or NULL.
 *   Outputs (each fully written; NULL allowed for dL_dconic, dL_dcolor, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, each on
 *   its own: dL_dmean3D keeps the SH view-direction term without dL_dsh; dL_dscale / dL_drot are zeros without scales and rotations;
 *   dL_dconic, a single-view output, is written only with accumulate = 0, zeros for the Gaussians the view culled):
 *     dL_dmean2D [P,3], dL_dconic [P,4] (slots x,y,w like the reference's float4), dL_dopacity [P],
 *     dL_dcolor [P,3], dL_dfeature [P,F], dL_dmean3D [P,3], dL_dcov3D [P,6], dL_dsh [P,M,3],
 *     dL_dscale [P,3], dL_drot [P,4].
 *   blend_scratch: device scratch of mgs_backward_scratch_bytes(P) bytes (contents irrelevant on entry).
 *   accumulate: 0 = every output row is written exactly once (the reference's semantics after its zero-fill);
 *               1 = every output row is ADDED to what the caller's buffer holds (read-modify-write by the row's one
 *                   thread; dL_dfeature with L2 reductions).  Calls that share output buffers must be serialised by
 *                   the caller; for several views of one cloud use mgs_backward_views, which sums in registers.
 */
size_t mgs_backward_scratch_bytes(int P);
int mgs_backward(
	int P, int D, int M, int F, int R,
	const float* background,
	int width, int height,
	const float* means3D,
	const float* shs,
	const float* colors_precomp,
	const float* feature_precomp,
	const float* scales,
	float scale_modifier,
	const float* rotations,
	const float* cov3D_precomp,
	const float* viewmatrix,
	const float* projmatrix,
	const float* campos,
	float tan_fovx, float tan_fovy,
	const int* radii,
	char* geometry_state,
	char* binning_state,
	char* image_state,
	const float* dL_dpix,
	const float* dL_dpix_F,
	const float* dL_dpix_depth,
	float* dL_dmean2D,
	float* dL_dconic,
	float* dL_dopacity,
	float* dL_dcolor,
	float* dL_dfeature,
	float* dL_dmean3D,
	float* dL_dcov3D,
	float* dL_dsh,
	float* dL_dscale,
	float* dL_drot,
	char* blend_scratch,
	int accumulate,
	int debug,
	void* stream);

/*
 * Multi-view step (no reference counterpart: the reference renders one view per call, asserts batch size 1 in its
 * caller, agents/manigaussian_bc/neural_rendering.py:386, and blocks the host on every view's instance count,
 * rasterizer_impl.cu:284).  V views of ONE Gaussian cloud are enqueued by ONE call with NO host synchronisation:
 * the caller owns the three state buffers of every view and sizes the binning state for `binning_capacity` instances
 * (mgs_binning_state_bytes(capacity)) -- e.g. the previous step's count plus slack; the real count stays on the device.
 * If it exceeds the capacity, the instances beyond it (the farthest Gaussians: emission is in depth order) are dropped,
 * the image is still well defined and consistent with the backward, and status[1] is raised; status (2 ints, pinned host
 * memory recommended, may be NULL) receives {instance count, overflow flag} asynchronously on the view's stream.
 * Work of view v is enqueued on views[v].stream; every view stream first waits for what `join_stream` holds at the call,
 * and `join_stream` waits for every view stream before the call returns, so the caller needs no stream logic of its own
 * (a view whose stream IS join_stream is simply serialised).  Nothing in these calls allocates or blocks: a step built
 * from them can be captured in a CUDA graph.
 * mgs_forward_views and mgs_backward_views are the one-cloud form of mgs_forward_clouds and mgs_backward_clouds (below):
 * the same code runs them with view_offsets = {0, V}.  Only the views backward has `stages` and `shared_mean2D`, and its
 * per-Gaussian launches run their own kernel, built for more blocks per SM than the clouds kernel.
 * mgs_backward_views runs the blend backward of every view on its stream, joins, and runs ONE per-Gaussian chain-rule
 * kernel that sums over the views in registers: outputs are the SUMS over the V views (the packed buffer of the
 * multi-GPU all-reduce can be passed directly), except dL_dmean2D which each view owns ([P,3], shared_mean2D = 0) or
 * which is summed into views[0].dL_dmean2D (shared_mean2D = 1).  Output NULL-ability as in mgs_backward.
 * `stages` splits the call in two so that a multi-GPU caller can start the all-reduce of dL_dfeature -- more than half of
 * the message, final after the blend stage -- while the per-Gaussian stage computes the remaining fields.
 * Every optional input of these calls and of the multi-cloud calls (extra planes, loss heads, camera models, gradients of
 * the camera) is a field of one mgs_render_options record, declared below after the structs it points to; the sections
 * between here and there describe each field.  A NULL record turns every one of them off.
 */
typedef struct mgs_view {
	const float* viewmatrix;     /* device, 16 floats */
	const float* projmatrix;     /* device, 16 floats */
	const float* cam_pos;        /* device, 3 floats (NULL with precomputed colours) */
	const float* background;     /* device, 3 floats */
	float tan_fovx, tan_fovy;
	int width, height;
	char* geometry_state;        /* mgs_geometry_state_bytes(P) */
	char* binning_state;         /* mgs_binning_state_bytes(binning_capacity) */
	char* image_state;           /* mgs_image_state_bytes(width, height) */
	int binning_capacity;
	float* out_color;            /* forward outputs: [3,H,W], [F,H,W] or NULL, [H,W] or NULL, int32 [P] */
	float* out_feature;
	float* out_depth;
	int* radii;
	int* status;                 /* host-accessible, 2 ints, or NULL */
	const float* dL_dpix;        /* backward inputs: [3,H,W], [F,H,W] or NULL, [H,W] or NULL */
	const float* dL_dpix_F;
	const float* dL_dpix_depth;
	char* blend_scratch;         /* backward: mgs_backward_scratch_bytes(P) */
	float* dL_dmean2D;           /* backward output [P,3] or NULL */
	void* stream;
	/* Fused loss heads ("next" row f4; all NULL = off).  Forward: with target_color [3,H,W] the blend epilogue also produces
	 * the L2 colour head of agents/manigaussian_bc/neural_rendering.py:300-308 (loss.py:12-13) and, with target_feature
	 * [F,H,W], the cosine embedding head (:310-318, loss.py:18-23): loss_acc (device, 2 floats, zeroed by the call) receives
	 * {sum (render - target)^2, sum_px cos_sim(embed, target)} -- loss_rgb = loss_acc[0] / (3 H W), loss_embed =
	 * 1 - loss_acc[1] / (H W) -- and cot_color [3,H,W] / cot_feature [F,H,W] receive d loss_rgb / d render and
	 * d loss_embed / d embed.  With F > 32 a pixel's feature vector spans several channel groups, so the embedding head
	 * runs in one small kernel behind the blend on the view's stream instead (same outputs).  Backward: pass those planes
	 * as dL_dpix / dL_dpix_F; cot_scale (device, 2 floats, or NULL for 1) holds the upstream gradients of the two scalar
	 * losses and multiplies the planes on load. */
	const float* target_color;
	const float* target_feature;
	float* cot_color;
	float* cot_feature;
	float* loss_acc;
	const float* cot_scale;
} mgs_view;


/*
 * Several clouds in one step (no reference counterpart).  A ManiGaussian training step with the dynamic field renders two
 * clouds -- the current frame and the deformed next frame (agents/manigaussian_bc/neural_rendering.py:283, :324) -- and
 * 2 B clouds for B samples per GPU, which the reference cannot do at all (it asserts bs == 1, :386).  Cloud b renders
 * views[view_offsets[b] .. view_offsets[b + 1]); view_offsets (host, B + 1 ints) starts at 0 and strictly increases.
 * D, M, F and scale_modifier are shared by every cloud; a cloud with feature == NULL renders no features.  Every mgs_view
 * field means what it means for mgs_forward_views / mgs_backward_views (capacity, status, overflow, loss heads, streams);
 * dL_dmean2D is each view's own [P_b,3].
 * mgs_forward_clouds enqueues stage by stage across ALL views of all clouds (every projection, then every binning chain,
 * then every blend) between one fork from and one join into join_stream, so one cloud's short kernels never queue behind
 * another cloud's blends.  No host synchronisation: a step built from these calls can be captured in a CUDA graph.
 * mgs_backward_clouds runs the blend backward of every view on its stream, joins, then the per-Gaussian stage on
 * join_stream in launches of up to 16 views that pack whole clouds.  Each cloud's outputs are the sums over its views
 * (overwritten, or added to with accumulate = 1); NULL-ability as in mgs_backward, except:
 *   - dL_dfeature NULL on a cloud with features: its feature gradient is not computed, but the feature cotangents still
 *     reach its mean, conic and opacity gradients;
 *   - shs without dL_dsh is MGS_ERR_INVALID_ARG, checked before anything is enqueued (mgs_backward and mgs_backward_views
 *     accept it and keep the view-direction term of dL_dmean3D; this entry point keeps its stricter check).
 * Argument errors (B <= 0, bad view_offsets, P <= 0, missing pointers) return MGS_ERR_INVALID_ARG before anything is enqueued.
 */
typedef struct mgs_cloud {
	int P;
	const float *means3D, *shs, *colors_precomp, *feature, *opacities, *scales, *rotations, *cov3D_precomp;
	/* backward outputs of this cloud: [P,3], [P] (or [P,1]), [P,3], [P,F], [P,6], [P,M,3], [P,3], [P,4] */
	float *dL_dmean3D, *dL_dopacity, *dL_dcolor, *dL_dfeature, *dL_dcov3D, *dL_dsh, *dL_dscale, *dL_drot;
} mgs_cloud;


/*
 * Alpha plane (no reference counterpart): the pixel's accumulated opacity alpha = 1 - final_T, e.g. for a mask loss or for
 * the expected depth out_depth / alpha (out_depth has no background term and falls to 0 where nothing covers the pixel).
 * mgs_render_options.alpha: one mgs_view_alpha per view, or NULL for none.
 * Forward: out_alpha [H,W] is fully overwritten.  Backward: dL_dpix_alpha [H,W] adds T_final / (1 - a_k) * dL_dalpha to
 * every contributor's dL/da_k (cot_scale does not scale it); a pixel nothing blended into has no alpha gradient.
 * Either pointer may be NULL per view.  mgs_view and mgs_cloud keep their layouts: existing arrays of them stay valid.
 */
typedef struct mgs_view_alpha {
	float* out_alpha;            /* forward output [H,W] = 1 - final_T, or NULL */
	const float* dL_dpix_alpha;  /* backward input [H,W], or NULL */
} mgs_view_alpha;


/*
 * Depth and mask heads (no reference counterpart; INTEGRATION.md §4): two more loss heads beside the fused colour and
 * embedding heads of mgs_view, evaluated in the same forward-blend epilogue from the view's depth plane D and alpha plane
 * A = 1 - final_T, so that a step with depth or mask supervision keeps the fused path (no image-sized kernel between the
 * forward and the backward, no host synchronisation).  Per view, N = H*W:
 *   depth  valid = (target_depth > 0) && (A > 0.5), d = D / A, n = sum valid:  loss_depth = sum_valid |d - target_depth| / n
 *          (0 when n = 0);
 *   mask   loss_mask = mean_px BCE(clamp(A, 1e-4, 1 - 1e-4), target_mask) as torch.nn.functional.binary_cross_entropy.
 * mgs_render_options.depth_mask: one mgs_view_depth_mask per view, or NULL for none.  Pass the same array to the forward
 * and the backward.  A view whose two targets are NULL has no depth or mask head.
 * Forward: the heads need the colour head (the view's target_color).  loss_acc (device, 3 floats, zeroed by the call)
 * receives {sum_valid |d - g|, n, sum_px BCE}: loss_depth = loss_acc[0] / max(loss_acc[1], 1), loss_mask = loss_acc[2] / N.
 * With target_depth, cot_depth and cot_alpha_depth [H,W] receive the unscaled cotangents sign(d - g) / A and
 * -sign(d - g) d / A on valid pixels, 0 elsewhere; with target_mask, cot_alpha_mask [H,W] receives d loss_mask / dA.
 * Backward: the planes are read back with cot_scale (device, 2 floats {g_depth, g_mask}, or NULL for 1): the depth plane's
 * cotangent is g_depth / max(n, 1) * cot_depth, and the alpha cotangent g_depth / max(n, 1) * cot_alpha_depth +
 * g_mask * cot_alpha_mask, with n read from loss_acc on the device.  Argument errors (a target without its planes or
 * loss_acc, a target without the view's colour head in the forward) return MGS_ERR_INVALID_ARG before anything is enqueued.
 */
typedef struct mgs_view_depth_mask {
	const float* target_depth;     /* [H,W] or NULL */
	const float* target_mask;      /* [H,W] in [0,1], or NULL */
	float* cot_depth;              /* [H,W], with target_depth */
	float* cot_alpha_depth;        /* [H,W], with target_depth */
	float* cot_alpha_mask;         /* [H,W], with target_mask */
	float* loss_acc;               /* device, 3 floats */
	const float* cot_scale;        /* device, 2 floats, or NULL */
} mgs_view_depth_mask;


/*
 * Anti-aliased projection (Mip-Splatting's "2D filter"; the `antialiasing` setting of the 3DGS authors' current rasterizer,
 * gsplat's rasterize_mode="antialiased"; INTEGRATION.md §5).  The projection dilates every screen-space covariance by
 * 0.3 px^2 (Sigma' = Sigma + 0.3 I, as the reference does); with antialiasing = 1 it also scales the Gaussian's opacity by
 *   s = sqrt(max(2.5e-5, det Sigma / det Sigma'))
 * so that the dilated splat carries the energy of the undilated one: the blend sees o_eff = o s.  The conic, radius, screen
 * mean, depth, tiles, instance count and sort keys are those of antialiasing = 0, bit for bit.  The backward chains dL/do_eff
 * to dL/do and, through s, to the covariance (and so to means, scales, rotations or cov3D).
 * mgs_render_options.antialiasing: 0 or 1, for every view of the call.  Pass the same value to the forward and the backward: the backward reads o_eff back from the forward's geometry
 * state.  Any other value returns MGS_ERR_INVALID_ARG before anything is enqueued.
 */

/*
 * L1 + SSIM photometric loss (no reference counterpart in the rasterizer; the objective 3DGS trains with,
 * (1 - lambda) L1 + lambda (1 - SSIM), lambda = 0.2, from gaussian-splatting utils/loss_utils.py, copied into ManiGaussian's
 * agents/manigaussian_bc/loss.py).  For one view, x = out_color [3,H,W] (background included, not clamped), g = target_color
 * [3,H,W], N = 3 H W:
 *   loss_l1 = sum |x - g| / N;  its gradient is sign(x - g) / N with sign(0) = 0;
 *   ssim    = mean over the 3 H W entries of S, exactly the reference's _ssim with window 11 and size_average: every plane is
 *             convolved on its own, with zero padding 5, by the 11x11 Gaussian window of sigma 1.5 (1-D weights
 *             exp(-(i - 5)^2 / 4.5) normalised to sum 1, outer product); with G(*) that convolution, mu_x = G(*)x,
 *             mu_g = G(*)g, sxx = G(*)x^2 - mu_x^2, sgg = G(*)g^2 - mu_g^2, sxg = G(*)(xg) - mu_x mu_g, C1 = 0.01^2,
 *             C2 = 0.03^2: S = (2 mu_x mu_g + C1)(2 sxg + C2) / ((mu_x^2 + mu_g^2 + C1)(sxx + sgg + C2)).
 *             The result is SSIM itself, not 1 - SSIM.
 * Gradient with respect to x only (the target is a constant).  With A, B, C, D the four factors of S above:
 *   dS/dmu_x = 2 mu_g (B - A) / (C D) - 2 mu_x S (1/C - 1/D),  dS/dE[x^2] = -S / D,  dS/dE[xg] = 2 A / (C D),
 *   d ssim / dx = (G(*)dS/dmu_x + 2 x G(*)dS/dE[x^2] + g G(*)dS/dE[xg]) / N.
 * Images smaller than the window (down to 1x1) are valid.
 * mgs_render_options.ssim: one mgs_view_ssim per view, or NULL for none.  Every entry of a non-NULL array is an SSIM head.
 * Forward: behind the view's blend, on its stream, the head reads out_color and target_color, zeroes loss_acc and adds
 * {sum |x - g|, sum S} into loss_acc[0..1] (loss_l1 = loss_acc[0] / N, ssim = loss_acc[1] / N), and writes the unscaled
 * partials {dS/dmu_x, dS/dE[x^2], dS/dE[xg]} of every pixel into ssim_terms [3 partials x 3 channels, H, W].
 * Backward: before the view's blend backward, on its stream, the head writes the view's complete colour cotangent
 *   cot_color = s_rgb dL_dpix + g_l1 sign(x - g) / N + g_ssim d ssim / dx
 * with s_rgb = the view's cot_scale[0] (or 1) and {g_l1, g_ssim} = cot_scale of this struct (or 1); the blend backward then
 * reads cot_color with a colour scale of 1 and the view's feature scale unchanged (the head leaves both in loss_acc[2..3]).
 * The view's out_color and target_color must again point at the forward's image and target.  Argument errors (an entry on
 * a view without target_color, a missing ssim_terms, loss_acc or cot_color, or, in the backward, a missing out_color)
 * return MGS_ERR_INVALID_ARG before anything is enqueued.
 */
typedef struct mgs_view_ssim {
	float* ssim_terms;             /* [9,H,W]: written by the forward, read by the backward */
	float* loss_acc;               /* device, 4 floats: {sum |x - g|, sum S}, then the blend backward's two scales */
	const float* cot_scale;        /* device, 2 floats {g_l1, g_ssim}, or NULL for 1 */
	float* cot_color;              /* [3,H,W]: receives the combined colour cotangent in the backward */
} mgs_view_ssim;


/*
 * Camera gradients (no reference counterpart: the reference's backward returns None for the camera).
 * mgs_render_options.camera_grad, read by the backward calls only: one mgs_view_camera_grad per view, or NULL.  An entry asks for the gradients of its view
 * when any of its three outputs is non-NULL; each output is written (accumulate = 0) or added to (accumulate = 1) by the
 * per-Gaussian stage (stage 2), a NULL output is skipped.  An entry with an output but no scratch returns
 * MGS_ERR_INVALID_ARG before anything is enqueued.
 *
 * Definition.  With vm the view's viewmatrix (Rv[r][c] = vm[4c + r], tv[r] = vm[12 + r]), pm its projmatrix read the same
 * way, and, per Gaussian p of the view with radius > 0, the chain rule of the per-Gaussian backward:
 *   t = Rv p + tv; dt = dL/dt with the x/y frustum clamp masking d/dt.x, d/dt.y and the depth cotangent on t.z;
 *   Q = [q0; q1] = dL/dM = 2 H M S (H including the anti-aliased compensation), cx, cy the clamped t.x, t.y;
 *   dm = the screen-mean cotangent, (hx, hy, hw) = P (p, 1), iw = 1 / (hw + 1e-7), kx = hx iw^2, ky = hy iw^2;
 * the gradients are the sums over those Gaussians of
 *   dL/dvm[4c + r] = dt[r] p[c] + (J^T Q)[r][c]   (r, c < 3; J held at its value:
 *                    (J^T Q)[0] = fx / tz q0, (J^T Q)[1] = fy / tz q1, (J^T Q)[2] = -fx cx / tz^2 q0 - fy cy / tz^2 q1)
 *   dL/dvm[12 + r] = dt[r];  dL/dvm[3], [7], [11], [15] = 0 (the forward never reads them)
 *   dL/dpm[4c] = dm0 iw ph[c],  dL/dpm[4c + 1] = dm1 iw ph[c],  dL/dpm[4c + 3] = -(dm0 kx + dm1 ky) ph[c],  ph = (p, 1);
 *                    dL/dpm[4c + 2] = 0 (the forward does not use the clip-space z)
 *   dL/dcampos = -(dd - dir along) / |v|  (v = p - campos, the SH branch's direction gradient dd and along = dir . dd: the
 *                    view-direction term of dL/dmeans3D with the opposite sign; 0 without SHs).
 * The gradient of a 16-float array is the gradient with respect to those 16 floats, so as a torch [4,4] it is directly the
 * gradient of world_view_transform / full_proj_transform.  In these calls tan_fov, the focal lengths, the 1.3 tan_fov clamp
 * limit, the near-plane cull, the radii and the tiles are constants: a projmatrix built from a learnable focal length
 * receives only the screen-mean path.  mgs_render_options.intrinsics below adds the focal-length path through J and the
 * clamp limit.
 * The sums are deterministic: every CTA of the per-Gaussian kernel writes one row of 27 partial sums per view into the
 * entry's scratch in a fixed order, and a reduce kernel on join_stream sums each view's rows in a fixed tree.  A view's rows
 * all come from one launch of at most 16 views.
 */
typedef struct mgs_view_camera_grad {
	float* dL_dviewmatrix;   /* device, 16 floats, or NULL */
	float* dL_dprojmatrix;   /* device, 16 floats, or NULL */
	float* dL_dcampos;       /* device, 3 floats, or NULL (zeros without SHs) */
	float* scratch;          /* device, mgs_camera_grad_scratch_bytes(P) of the view's cloud */
} mgs_view_camera_grad;

size_t mgs_camera_grad_scratch_bytes(int P);

/*
 * Learnable intrinsics (no reference counterpart).  mgs_render_options.intrinsics: one mgs_view_intrinsics per view, or NULL;
 * without it the camera gradients keep the definition given above.
 *
 * Device field of view.  An entry's tan_fov, when set, points at the view's {tan_fovx, tan_fovy} in device memory, and the
 * projection forward and backward read it there in place of mgs_view.tan_fovx / tan_fovy: a value an optimizer step has just
 * written is used with no device->host read, and a captured CUDA graph reads the value at replay.  The kernels form
 * fx = W / (2 tan_fovx) and fy = H / (2 tan_fovy) with the same float expression as the host path (the build has no fast
 * math), so a device value equal to the host floats gives the host path's radii, sort keys, tiles and images bit for bit.
 * The backward then runs the camera-gradient instantiation of the per-Gaussian stage (with or without outputs).
 *
 * Focal-length gradient.  dL_dtan_fov, when set, receives {dL/dtan_fovx, dL/dtan_fovy} under the rules of the camera outputs
 * above: written (accumulate = 0) or added to (1) by stage 2, and it needs the view's mgs_view_camera_grad entry with scratch
 * (MGS_ERR_INVALID_ARG before anything is enqueued otherwise); its per-CTA partial sums are kept in the view's geometry
 * state, so mgs_camera_grad_scratch_bytes is unchanged and remains the only scratch size to provide.  Definition, with the quantities of the camera-gradient
 * definition above (Q = [q0; q1] = dL/dM including the anti-aliased compensation, cx, cy the clamped t.x, t.y, tz = t.z) and
 * dJ00 = q0 . Rv0, dJ02 = q0 . Rv2, dJ11 = q1 . Rv1, dJ12 = q1 . Rv2, the sum over the view's Gaussians with radius > 0 of
 *   dL/dtan_fovx = -(fx / tan_fovx) (dJ00 / tz - dJ02 cx / tz^2)          (J through fx = W / (2 tan_fovx))
 *                  - [|t.x / tz| > 1.3 tan_fovx] fx dJ02 (+-1.3) / tz      (the clamp cx = +-1.3 tan_fovx tz, sign of t.x / tz)
 * and likewise dL/dtan_fovy with fy, dJ11, dJ12, cy.  The near-plane cull, the radii, the tiles and the sort stay constants.
 * The projection-matrix path of the focal lengths and the principal point is dL/dprojmatrix above, to be chained by the
 * caller (for a projmatrix built from K).  With intrinsics on, the 27 other camera terms are those camera_grad alone writes.
 */
typedef struct mgs_view_intrinsics {
	const float* tan_fov;    /* device, 2 floats, or NULL: use mgs_view.tan_fovx / tan_fovy */
	float* dL_dtan_fov;      /* device, 2 floats, or NULL */
} mgs_view_intrinsics;


/*
 * Median depth and surface Gaussian (no reference counterpart; 2DGS's median_contributor).
 * mgs_render_options.median: one mgs_view_median per view, or NULL.
 *
 * Definition.  For pixel p, walk its contributors front to back with the forward blend's own decisions (the pairs whose
 * pixel-mask bit is set, "pixel_masks" of mgs_state_array) and its fp32 transmittance T before each pair:
 *   - the median contributor is the last contributor whose incoming T > 0.5.  T only decreases, so this is the contributor
 *     at which T first falls to 0.5 or below; where T never gets there it is the pixel's last contributor (mask such pixels
 *     with the alpha plane, e.g. alpha > 0.5);
 *   - median_id[p] = that Gaussian's index in its cloud, or -1 where the pixel has no contributor;
 *   - out_median_depth[p] = that Gaussian's view-space depth, bit for bit the value the depth channel blends for it, or 0
 *     where the pixel has no contributor.
 * Backward: dL/dz_i += sum over the pixels p with median_id[p] = i of dL_dpix_median_depth[p], z_i the view-space depth of
 * Gaussian i, which reaches means3D and the camera gradients through the projection's depth path.  The choice of the
 * contributor is piecewise constant: no gradient goes to opacity, conic, colour, features or means2D.  The sums use float
 * atomics, like the blend backward's.
 * Per view each pointer may be NULL; median_id must be set wherever out_median_depth (forward) or dL_dpix_median_depth
 * (backward) is, else MGS_ERR_INVALID_ARG before anything is enqueued.  The backward reads the median_id its forward wrote.
 */
typedef struct mgs_view_median {
	float* out_median_depth;              /* forward output [H,W], or NULL */
	int* median_id;                       /* forward output [H,W] int32; backward input */
	const float* dL_dpix_median_depth;    /* backward input [H,W], or NULL */
} mgs_view_median;


/*
 * Surface normals (no reference counterpart; the rend_normal plane of 2DGS / RaDe-GS / GaussianShader).
 * mgs_render_options.normal: one mgs_view_normal per view, or NULL.
 *
 * Definition.  Per Gaussian i and view v, from scales [P,3] and rotations [P,4] (r, x, y, z):
 *   - k = argmin_j scales[i][j], the lowest index on ties (scale_modifier does not change it);
 *   - q^ = q / |q| (normalised here: a normal is a unit vector even when the caller's quaternion is not), and
 *     a = R(q^) e_k, the WORLD-space direction of the axis that scale k stretches (Sigma a = s_k^2 a for the covariance the
 *     projection builds), R(q^) the rotation matrix of q^:
 *       e_0 -> (1 - 2(y^2 + z^2), 2(xy + rz), 2(xz - ry)),  e_1 -> (2(xy - rz), 1 - 2(x^2 + z^2), 2(yz + rx)),
 *       e_2 -> (2(xz + ry), 2(yz - rx), 1 - 2(x^2 + y^2));
 *   - s = +1 if a . (cam_pos_v - mean_i) >= 0, else -1, and n_{i,v} = s a: the normal faces the camera.
 * Plane: out_normal[c][p] = sum_k w_{p,k} n_{k,v}[c], c < 3, with the blend weights w = alpha T and the contributors of the
 * colour image.  No background term and no clamp, like depth and features.  The plane is NOT normalised: its length is about
 * alpha where one surface dominates; divide by the alpha plane or normalise.
 * Backward, given dL_dpix_normal [3,H,W]: the normal channels enter dL/dalpha (and through it opacity, conic, means2D) like
 * any other channel; dL/dn_{i,v} = sum_p w_{p,i} dL_dpix_normal[:, p]; dL/da_i = sum_v s_{i,v} dL/dn_{i,v} is chained through
 * R(q^) e_k and the normalisation ((I - q^ q^T) / |q|) and ADDED to dL_drot.  k and s are piecewise constant: scales, means3D
 * and the camera receive nothing from them, and as the plane is in world space the view matrix does not enter it.
 * State: a view with a normal plane needs a geometry_state of mgs_geometry_state_bytes_normal(P) bytes, and in the backward
 * a blend_scratch of mgs_backward_scratch_bytes_normal(P) bytes (the per-Gaussian quads and their gradients live behind the
 * other arrays; "geometry" / "nrm" of mgs_state_array).  Per view each pointer may be NULL.  MGS_ERR_INVALID_ARG, before
 * anything is enqueued: a plane or cotangent with cov3D_precomp (there is no rotation to take a normal from), without cam_pos,
 * or beside the depth / mask heads (mgs_view_depth_mask targets); a dL_dpix_normal without out_normal, the plane that view's
 * forward wrote (the backward reads the quads that forward stored).
 */
typedef struct mgs_view_normal {
	float* out_normal;              /* forward output [3,H,W], or NULL; names the forward's plane in the backward */
	const float* dL_dpix_normal;    /* backward input [3,H,W], or NULL */
} mgs_view_normal;

size_t mgs_geometry_state_bytes_normal(int P);
size_t mgs_backward_scratch_bytes_normal(int P);

/*
 * Orthographic views (no reference counterpart; gsplat's camera_model="ortho", the virtual views of RVT / RVT-2 and the
 * top-down colour and height maps of Transporter / CLIPort).  mgs_render_options.ortho
 * (and the `ortho` argument of mgs_lift_views, mgs_visibility_views and mgs_camera_rays): a host array of one int per view,
 * 0 for a perspective view and 1 for an orthographic one, or NULL for all perspective.  One call may mix both kinds, also among the views of one cloud; the backward sums them in one pass.
 * Definition, for an orthographic view, with t = Rv p + tv as for a pinhole view:
 *   - tan_fovx / tan_fovy (mgs_view, or mgs_view_intrinsics.tan_fov on the device) hold the half-width and half-height of
 *     the view volume in view-space units.  fx = W / (2 tan_fovx) and fy = H / (2 tan_fovy), the same float expressions as
 *     for a pinhole view, are then pixels per unit.
 *   - The Jacobian is J = [[fx, 0, 0], [0, fy, 0]], independent of t, with no frustum clamp.
 *   - Unchanged from the pinhole path: the near cull t.z > 0.2; the screen mean through the caller's projmatrix,
 *     ndc = (P p).xy / ((P p).w + 1e-7) (an orthographic matrix has w = 1); the depth t.z; the 0.3 px^2 dilation, the
 *     anti-aliased compensation, conic, radius, tiles, sort keys and everything after the projection.
 *   - The SH view direction and the normal plane's facing test use p - cam_pos as for a pinhole view (as gsplat does for
 *     every camera model), not the view's constant ray direction.
 *   - Backward: M = J Rv has rows fx Rv0 and fy Rv1; dL/dt is the depth cotangent on t.z alone.  Camera gradients take
 *     J^T dL/dM with rows (fx q0, fy q1, 0); dL/dtan_fovx = -(fx / tan_fovx) dL/dJ00 and dL/dtan_fovy = -(fy / tan_fovy) dL/dJ11,
 *     the gradient of a learnable half extent.
 * Argument errors: an ortho entry other than 0 or 1 returns MGS_ERR_INVALID_ARG before anything is enqueued.
 */

/*
 * Fisheye views (gsplat's camera_model="fisheye"; OpenCV's cv::fisheye model, Kannala-Brandt with four coefficients, all
 * k = 0 being the equidistant fisheye).  mgs_render_options.fisheye (and the `fisheye` argument of the lift, visibility and
 * ray calls): a host array of one mgs_view_fisheye per view, or NULL for none.  An entry with fisheye = 0 is ignored (the
 * view is perspective or, by its ortho flag, orthographic).  One call may mix all three models, also among the views of one cloud.
 * Definition, for a fisheye view, with t = Rv p + tv as for a pinhole view:
 *   - r = sqrt(t.x^2 + t.y^2), theta = atan2(r, t.z), theta_d = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6 + k4 theta^8).
 *   - Screen mean: u = fx theta_d t.x / r + cx, v = fy theta_d t.y / r + cy ((cx, cy) at r = 0).  (cx, cy) are in the blend's
 *     pixel coordinates, where pixel (i, j) has its centre at (i, j), as in OpenCV: calibrated values are used as they are,
 *     and a centred camera has cx = (W - 1) / 2.  projmatrix is not read (its gradient is zero); the argument checks are
 *     unchanged, so callers pass the pinhole matrix of the same K.
 *   - fx = W / (2 tan_fovx), fy = H / (2 tan_fovy), the same float expressions as for a pinhole view: tan_fovx holds
 *     W / (2 fx) with fx in pixels per radian.  mgs_view_intrinsics.tan_fov and dL_dtan_fov work unchanged; dL_dtan_fov is then
 *     the gradient of a learnable fisheye focal length.
 *   - Jacobian of (u, v) w.r.t. t, with a = theta_d / r, rho' = d theta_d / d theta = 1 + 3 k1 theta^2 + 5 k2 theta^4 +
 *     7 k3 theta^6 + 9 k4 theta^8, s = r^2 + t.z^2, b = rho' t.z / s and c = (b - a) / r^2:
 *         J = [[fx (a + c x^2), fx c x y, -fx x rho' / s], [fy c x y, fy (a + c y^2), -fy y rho' / s]]   (x, y = t.x, t.y)
 *     As r -> 0, a -> 1 / t.z and c -> (2 k1 - 2/3) / t.z^3.  Below r / t.z = 1/8 the kernels take a and c (and c's
 *     derivatives) from their series in (r / t.z)^2, where the expression above cancels in fp32.  No frustum clamp.
 *   - Cull: the near cull t.z > 0.2, and a Gaussian whose mean has theta > theta_max is culled the same way (radius 0).
 *   - Depth is t.z (sort key and depth plane); the SH view direction and the normal plane's facing test use p - cam_pos.
 *     Every stage after the projection is unchanged.  The covariance is the EWA linearisation J Sigma J^T at the mean, as in
 *     gsplat: large splats near the rim of a wide view are approximated by it, a property of the model.
 *   - Backward: the blend's dL/dmean2D (dm) is, for every view, the gradient w.r.t. ndc = (2 u + 1) / W - 1 (the reference's
 *     convention), so the pixel-space mean (u, v) has the cotangent (du, dv) = (dm0 / (W / 2), dm1 / (H / 2)).  M = J Rv;
 *     dL/dt = J^T (du, dv) + (dL/dJ = dL/dM Rv^T contracted with dJ/dt, all six entries) + the depth cotangent on t.z.
 *     Camera gradients: dL/dRv = dt p^T + J^T dL/dM, dL/dtv = dt, dL/dprojmatrix = 0, dL/dcampos as for a pinhole view (SH),
 *     dL/dtan_fovx = -(du (u - cx) + sum_j dJ0j J0j) / tan_fovx and likewise for y.  The principal point,
 *     the coefficients and theta_max receive no gradient.
 * Argument errors, MGS_ERR_INVALID_ARG before anything is enqueued: a fisheye flag other than 0 or 1; a view that is both
 * orthographic and fisheye; a non-finite cx, cy, k1..k4 or theta_max; theta_max outside (0, pi/2].
 */
typedef struct mgs_view_fisheye {
	int fisheye;                    /* 1: a fisheye view; 0: the entry is ignored */
	float cx, cy;                   /* principal point in pixels (pixel centres at integers) */
	float k1, k2, k3, k4;           /* Kannala-Brandt coefficients */
	float theta_max;                /* cull: theta of the mean above it, in (0, pi/2] */
} mgs_view_fisheye;

/*
 * Distorted-pinhole views (OpenCV's cv::projectPoints with the 8-coefficient D = (k1, k2, p1, p2, k3, k4, k5, k6);
 * COLMAP's OPENCV / FULL_OPENCV).  mgs_render_options.distortion (and the `distortion` argument of the lift, visibility and
 * ray calls): a host array of one mgs_view_distortion per view, or NULL for none.  An entry with distorted = 0 is ignored
 * (the view's model is then given by its ortho flag and fisheye entry).  One call may mix all four models, also among the views of one cloud.
 * Definition, for a distorted view, with t = Rv p + tv as for every view:
 *   - x = t.x / t.z, y = t.y / t.z, r2 = x^2 + y^2,
 *     R = (1 + k1 r2 + k2 r2^2 + k3 r2^3) / (1 + k4 r2 + k5 r2^2 + k6 r2^3),
 *     xd = x R + 2 p1 x y + p2 (r2 + 2 x^2),   yd = y R + p1 (r2 + 2 y^2) + 2 p2 x y.
 *   - Screen mean: u = fx xd + cx, v = fy yd + cy.  (cx, cy) are in the blend's pixel coordinates, where pixel (i, j) has its
 *     centre at (i, j), as in OpenCV and as for fisheye views.  projmatrix is not read (its gradient is zero).
 *   - fx = W / (2 tan_fovx), fy = H / (2 tan_fovy), as for every view: tan_fovx holds W / (2 fx).  mgs_view_intrinsics.tan_fov
 *     and dL_dtan_fov work unchanged; dL_dtan_fov is then the gradient of a learnable focal length.
 *   - Jacobian of (u, v) w.r.t. t, exact at the mean: J = diag(fx, fy) Dd [[1/t.z, 0, -x/t.z], [0, 1/t.z, -y/t.z]], with
 *     Dd = d(xd, yd) / d(x, y) = [[R + 2 x^2 R' + 2 p1 y + 6 p2 x, 2 x y R' + 2 p1 x + 2 p2 y],
 *                                 [2 x y R' + 2 p1 x + 2 p2 y, R + 2 y^2 R' + 6 p1 y + 2 p2 x]],  R' = dR / dr2.  No frustum clamp.
 *   - Cull, like a mean behind the near plane (radius 0): r2 > r_max^2 (past the first fold of the radial map, where far-off
 *     points fold back into the image), or det Dd <= 0 (a local fold, which the tangential terms can add).  Every kept
 *     Gaussian then has a finite EWA conic.
 *   - Depth is t.z (sort key and depth plane); the SH view direction and the normal plane's facing test use p - cam_pos.
 *     Every stage after the projection is unchanged.
 *   - Backward: (du, dv) = (dm0 / (W / 2), dm1 / (H / 2)) is the pixel-space mean's cotangent (dm, the blend's dL/dmean2D,
 *     is w.r.t. ndc, as for fisheye views).  M = J Rv; dL/dt = J^T (du, dv) + (dL/dJ = dL/dM Rv^T contracted with dJ/dt, which
 *     takes Dd's derivatives) + the depth cotangent on t.z.  Camera gradients: dL/dRv = dt p^T + J^T dL/dM, dL/dtv = dt,
 *     dL/dprojmatrix = 0, dL/dcampos as for a pinhole view (SH), dL/dtan_fovx = -(du (u - cx) + sum_j dJ0j J0j) / tan_fovx and
 *     likewise for y.  The principal point, the coefficients and r_max receive no gradient.
 * Argument errors, MGS_ERR_INVALID_ARG before anything is enqueued: a flag other than 0 or 1; a distorted view that is also
 * orthographic or fisheye; a non-finite cx, cy or coefficient; r_max <= 0 or NaN (r_max = +inf is allowed).
 */
typedef struct mgs_view_distortion {
	int distorted;                  /* 1: a distorted-pinhole view; 0: the entry is ignored */
	float cx, cy;                   /* principal point in pixels (pixel centres at integers) */
	float k1, k2, p1, p2, k3, k4, k5, k6;  /* OpenCV's D, in its order; 4 or 5 coefficients: the rest 0 */
	float r_max;                    /* cull: sqrt(x^2 + y^2) of the mean above it, > 0 or +inf */
} mgs_view_distortion;

/*
 * Planar depth.  mgs_render_options.planar_depth: 0 or 1, for every view of the call, like antialiasing.  Without it each Gaussian
 * paints its centre depth z = t.z over its whole footprint; with it, Gaussian i's depth at pixel p is its depth along the
 * pixel's ray, affine in the pixel offset (RaDe-GS, PGSR).  Definition, for Gaussian i in view v, with t = Rv p + tv:
 *   - Sigma_c = Rv S Rv^T, S the world-space covariance (from scales and rotations, or cov3D_precomp);
 *   - J the 2x3 screen Jacobian the projection uses for the view's model, in pixels (pinhole with its 1.3 tan_fov clamp,
 *     orthographic, fisheye or distorted), Q the blend's conic, the inverse of J Sigma_c J^T + 0.3 I (also in AA mode);
 *   - k = e3^T Sigma_c J^T, the covariance of depth with screen position, and (a, b) = k Q, the regression of t.z on the
 *     dilated screen position;
 *   - d_i(p) = z + a (px - mu_x) + b (py - mu_y), mu the blend's screen mean in pixels, pixel (i, j) centred at (i, j).
 * The depth plane is sum_i w_i d_i(p) (w the blend weights), and so are what is derived from it: the expected-depth L1 head
 * (mgs_view_depth_mask.target_depth), depth / alpha, and the median depth, which becomes d_i(p) of the pixel's median
 * contributor.  Colour, features, alpha, radii, tiles, sort keys and median_id do not change.  The blend carries the
 * per-Gaussian quad {a, b, e = -(a mu_x + b mu_y), 0} in columns 4..7 of its {r,g,b,depth} tile, so the depth is
 * col3 + px col4 + py col5 + col6; the quads live where the normal plane's do, so the geometry state must be sized by
 * mgs_geometry_state_bytes_normal and the backward scratch by mgs_backward_scratch_bytes_normal.
 * Backward: the depth cotangent g (including the depth head's) enters the blend as the column cotangents (g, g px, g py, g),
 * which makes dL/dalpha that of the planar depth; the blend returns dL/d(a, b, e) per Gaussian and view (formed relative to
 * each Gaussian's screen mean, so its precision does not depend on the pixel coordinates), and the per-Gaussian
 * stage chains them through e to mu (added to dL/dmean2D in its convention), through Q (added to the conic's gradient) and
 * through k to Sigma_c, J and the third row of Rv, and from there to means3D, scales, rotations (or cov3D), the camera
 * gradients and dL_dtan_fov for all four models.  The median depth's cotangent reaches z, a, b and mu of its contributor.
 * dL_dconic (single-view calls) stays the blend's conic gradient.
 * Argument errors, MGS_ERR_INVALID_ARG before anything is enqueued: planar_depth other than 0 or 1; planar_depth together
 * with a normal plane in the same call (both need columns 4..6 of the tile; a fourth column tile for both is left for later).
 */

/*
 * Optical flow.  mgs_render_options.flow: one mgs_view_flow per view, or NULL; mgs_render_options.flow_next: one
 * mgs_cloud_flow per cloud (one for a views call), or NULL.  The flow plane relates a cloud to its deformed next frame: for
 * one view v of a cloud with means mu_i and paired next-frame means mu'_i (flow_next[b].means3D [P,3], the same P, paired
 * by index):
 *   - m_i is Gaussian i's screen mean in pixels, as the projection forms it: through projmatrix and ndc2pix for pinhole and
 *     orthographic views, the lens map for fisheye and distorted views;
 *   - m'_i is the same map applied to mu'_i, with the view's own camera, or with the view's next-frame pose when one is given
 *     (next_viewmatrix / next_projmatrix, e.g. a wrist camera that moved with the gripper).  The model, intrinsics (a device
 *     tan_fov included), principal point, coefficients and image size are always the view's own;
 *   - valid_i holds when mu'_i passes the cull the projection applies to a mean of that model: view-space z > NEAR_Z, and for
 *     fisheye views theta <= theta_max, for distorted views r2 <= r2_max and det Dd > 0;
 *   - delta_i = valid_i ? m'_i - m_i : 0, in pixels (m' has no frustum clamp: it is a mean, not the Jacobian);
 *   - flow[c][p] = sum_i w_{p,i} delta_i[c], c = 0 (x, to the right) and 1 (y, down), w = alpha T the weights the colour
 *     image blends with.  There is no background term and no normalisation: flow / alpha is the expected flow.
 * Both ends come from one device function, so delta_i is 0 bit for bit when mu'_i == mu_i and no next pose is given.  The
 * per-Gaussian quads {dx, dy, 0, 0} live where the normal plane's do (columns 4..7 of the blend's {r,g,b,depth} tile): the
 * geometry state must be sized by mgs_geometry_state_bytes_normal and the backward scratch by mgs_backward_scratch_bytes_normal.
 * Backward, for a cotangent g [2,H,W] (channel 2 of dL_dpix_flow is ignored): the channels enter dL/dalpha like any other
 * channel (opacity, conic and means2D of the current frame, with the anti-aliased compensation where it is on); with
 * gd_i = sum_p w_{p,i} g[:, p], -gd_i joins view v's dL/dmean2D in the blend's convention (pixels times W / 2, H / 2), from
 * where the per-Gaussian stage carries it to means3D, the camera gradients and dL_dtan_fov; (dm'/dmu')^T gd_i, summed over
 * the cloud's views, is flow_next[b].dL_dmeans3D (written, or added with accumulate = 1; NULL skips it), and where the view has no next pose
 * (dm'/dcamera)^T gd_i joins its dL_dviewmatrix, dL_dprojmatrix and dL_dtan_fov.  Invalid pairs receive nothing through delta.
 * Flow needs no rotations (cov3D_precomp works), and adds no host synchronisation.
 * Argument errors, MGS_ERR_INVALID_ARG before anything is enqueued: flow beside a normal plane or planar_depth (they share the
 * tile's columns 4..7), or beside the depth / mask heads of the same view; out_flow without next means (the cloud's
 * mgs_cloud_flow.means3D); dL_dpix_flow without out_flow, the plane that view's forward wrote; only one of
 * next_viewmatrix and next_projmatrix.
 */
typedef struct mgs_view_flow {
	const float* next_viewmatrix;   /* [16] the next frame's pose, or NULL for the view's own */
	const float* next_projmatrix;   /* [16], NULL exactly when next_viewmatrix is */
	float* out_flow;                /* forward output [3,H,W] (channel 2 written as 0), or NULL; names the forward's plane in the backward */
	const float* dL_dpix_flow;      /* backward input [3,H,W] (channel 2 ignored), or NULL */
} mgs_view_flow;
/* one per cloud of a clouds call: the cloud's next-frame means [P,3] (or NULL) and their gradient [P,3] (or NULL) */
typedef struct mgs_cloud_flow {
	const float* means3D;
	float* dL_dmeans3D;
} mgs_cloud_flow;

/*
 * The optional inputs of mgs_forward_views, mgs_backward_views, mgs_forward_clouds and mgs_backward_clouds, each described in
 * its section above.  Per-view arrays have V entries (views calls) or view_offsets[B] entries (clouds calls); NULL turns the
 * input off.  A NULL record means the same as a record with every field zero.  The forward ignores the backward-only fields
 * (camera_grad, flow_next[.].dL_dmeans3D and the gradient fields of the per-view structs), as it does those of mgs_view.
 * A new optional per-view input becomes a field of this record; a change of its layout changes mgs_abi_version().
 */
typedef struct mgs_render_options {
	/* per-view arrays: V entries (views calls) or view_offsets[B] entries (clouds calls), or NULL for none */
	const mgs_view_alpha* alpha;
	const mgs_view_depth_mask* depth_mask;
	const mgs_view_ssim* ssim;
	const mgs_view_camera_grad* camera_grad;   /* read by the backward only */
	const mgs_view_intrinsics* intrinsics;
	const mgs_view_median* median;
	const mgs_view_normal* normal;
	const int* ortho;
	const mgs_view_fisheye* fisheye;
	const mgs_view_distortion* distortion;
	const mgs_view_flow* flow;
	/* next-frame means of the flow planes: 1 entry for a views call, B for a clouds call, or NULL */
	const mgs_cloud_flow* flow_next;
	int antialiasing;                          /* 0 or 1 */
	int planar_depth;                          /* 0 or 1 */
} mgs_render_options;

int mgs_forward_views(
	int V, const mgs_view* views, const mgs_render_options* options,
	int P, int D, int M, int F,
	const float* means3D,
	const float* shs,
	const float* colors_precomp,
	const float* feature_precomp,
	const float* opacities,
	const float* scales,
	float scale_modifier,
	const float* rotations,
	const float* cov3D_precomp,
	int prefiltered,
	int debug,
	void* join_stream);
int mgs_backward_views(
	int V, const mgs_view* views, const mgs_render_options* options,
	int P, int D, int M, int F,
	const float* means3D,
	const float* shs,
	const float* colors_precomp,
	const float* feature_precomp,
	const float* scales,
	float scale_modifier,
	const float* rotations,
	const float* cov3D_precomp,
	float* dL_dmean3D,
	float* dL_dopacity,
	float* dL_dcolor,
	float* dL_dfeature,
	float* dL_dcov3D,
	float* dL_dsh,
	float* dL_dscale,
	float* dL_drot,
	int shared_mean2D,
	int accumulate,
	int stages,            /* 1: blend stage of every view (dL_dfeature is final afterwards), 2: the per-Gaussian stage, 3: both */
	int debug,
	void* join_stream);
int mgs_forward_clouds(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_render_options* options, int D, int M, int F, float scale_modifier, int prefiltered, int debug, void* join_stream);
int mgs_backward_clouds(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_render_options* options, int D, int M, int F, float scale_modifier, int accumulate, int debug, void* join_stream);

/*
 * Lifting 2D maps onto the Gaussians (no reference counterpart; the lift of Gaussian Grouping, SAGA, Feature Splatting and
 * LUDVIG).  Given one map per view, mgs_lift_views computes per Gaussian g
 *   lifted[g][c] = sum_v sum_p w_vpg map_v[c][p],     weight[g] = sum_v sum_p w_vpg,
 * so lifted / weight is the Gaussian's blend-weighted average of the maps and weight alone its visibility over the views.
 * Definition.  For each view the contributors and weights are the forward blend's own: the same expf, the same skip tests
 * (power > 0, alpha < 1/255), the same 0.99 clamp, the same T (1 - alpha) < 1e-4 stop, and T the running product, so
 * w_vpg is bit for bit the weight with which the colour image of that view blends Gaussian g into pixel p (alpha with the
 * compensated opacity o_eff when antialiasing = 1).  There is no background term; pixels outside the image do not count.
 * lifted is dL/dfeature of a feature render (normalize_feature off) with cotangent map_v, without the backward's geometry.
 *   - map_v (mgs_view_lift.map) is [C,H,W] fp32, planar like the feature images; C in [0, MGS_MAX_FEATURE_CHANNELS] is the
 *     same for every view; with C = 0 only weight is computed and lift may be NULL.
 *   - out_lifted [P,C] (NULL allowed with C = 0) and out_weight [P] are zero-filled by the call on join_stream, then every
 *     view of the call is summed into them (float atomics: the order of the sums is not fixed).
 *   - Per view: viewmatrix, projmatrix, cam_pos (with SHs), radii (written, as by the forward), the three state buffers
 *     (sized as for mgs_forward_views) and binning_capacity, status and stream are used; background and every image,
 *     backward and loss-head field are ignored.  The view's state afterwards holds its projection and binning; the blend
 *     state (final_T, n_contrib, pixel masks, block_nwalk) is not written, so it cannot serve a backward.
 *   - shs or colors_precomp must be given as in mgs_forward_views, and are never read for the lift: the projection stage
 *     is the forward's own.  intr (NULL, or one mgs_view_intrinsics per view) gives device fields of view; its dL_dtan_fov
 *     is not used.  The outputs are not differentiable.
 * Argument errors return, with mgs_last_error set and before anything is enqueued: MGS_ERR_UNSUPPORTED for C outside
 * [0, MGS_MAX_FEATURE_CHANNELS]; MGS_ERR_INVALID_ARG for V <= 0, P <= 0, a NULL map while C > 0, a NULL output, a view
 * without its state buffers, matrices or radii, and the Gaussian-argument errors of mgs_forward_views.
 */
typedef struct mgs_view_lift {
	const float* map;               /* [C,H,W] fp32, or NULL with C = 0 */
} mgs_view_lift;

int mgs_lift_views(
	int V, const mgs_view* views, const mgs_view_lift* lift, int antialiasing, const mgs_view_intrinsics* intr, const int* ortho,
	const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion,
	int P, int D, int M, int C,
	const float* means3D, const float* shs, const float* colors_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* out_lifted, float* out_weight, int debug, void* join_stream);

/*
 * Field queries (no reference counterpart): the cloud's density and features at Q arbitrary 3D points, with no camera.
 * Definition, for Gaussian i (mean mu, scales s, quaternion q, opacity o, feature row f) and a point x, with q^ = q / |q| and
 * R(q^) the rasterizer's rotation (Sigma = R^T S^2 R for a unit quaternion):
 *   m_i(x) = | S^-1 R(q^) (x - mu) |^2   (evaluated in the Gaussian's own frame, never through an inverted Sigma),
 *   g_i(x) = o exp(-m_i(x) / 2) if that is >= 1/255, else 0   (the blend's alpha threshold, without its 0.99 clamp),
 *   density(x) = sum_i g_i(x),     features(x)[c] = sum_i g_i(x) f[c],   C = 0 .. MGS_MAX_FEATURE_CHANNELS.
 * The support of Gaussian i is the ellipsoid m <= 2 ln(255 o); a Gaussian with o <= 1/255, a scale <= 0 or a non-finite mean,
 * scale, quaternion or opacity contributes nothing and gets zero gradients.  A non-finite point gets density 0.  Features
 * are used as given (they must be finite: they enter tensor-core sums with zero weights).
 *   - points [Q,3], means3D [P,3], scales [P,3], rotations [P,4], opacities [P], features [P,C] (NULL with C = 0).
 *   - out_density [Q]; out_features [Q,C], or [C,Q] with channel_first = 1 (a channel-first voxel grid without a copy);
 *     both fully written.
 * Method: a uniform grid of bins over the points' bounding box (its size is internal and picked from Q and the box; it
 * changes nothing but the order of fp32 sums), per-bin lists of the Gaussians whose support box reaches the bin in
 * ascending id, and one warp per 32 points of a bin with the feature contraction on the tensor cores (3xTF32).  The state
 * is requested through the two allocators: the query state (sized by Q and P) first, then, after the one stream
 * synchronisation of the call (the pair count is read back to size the bin lists exactly, so no pair is dropped), the
 * pair state.  Returns the (bin, Gaussian) pair count (MGS_ERR_UNSUPPORTED above 2^31 - 1).  Not capturable in a CUDA graph.
 * Backward: mgs_field_query_backward takes both state buffers as the forward left them (it allocates and reads back
 * nothing), the same points, scales, rotations, features and channel_first, and the cotangents dL_ddensity [Q] and
 * dL_dout_features (laid out as out_features), each NULL for zero.  It writes, each output optional (NULL skips it and the
 * work only it needs): dL_dpoints [Q,3], dL_dmeans3D [P,3], dL_dscales [P,3], dL_drotations [P,4] (through the
 * normalisation of q), dL_dopacities [P] and dL_dfeature [P,C].  The cutoff is held fixed, as the blend holds its thresholds.
 * Argument errors return, with mgs_last_error set and before anything is enqueued: MGS_ERR_UNSUPPORTED for C outside
 * [0, MGS_MAX_FEATURE_CHANNELS]; MGS_ERR_INVALID_ARG for Q <= 0, P <= 0, a NULL allocator, input or required output, and
 * channel_first other than 0 or 1.
 */
int mgs_field_query(
	mgs_alloc_fn state_alloc, void* state_user,
	mgs_alloc_fn pair_alloc, void* pair_user,
	int Q, int P, int C,
	const float* points,
	const float* means3D,
	const float* scales,
	const float* rotations,
	const float* opacities,
	const float* features,
	int channel_first,
	float* out_density,
	float* out_features,
	int debug,
	void* stream);
int mgs_field_query_backward(
	const char* state, const char* pair_state,
	int Q, int P, int C,
	const float* points,
	const float* scales,
	const float* rotations,
	const float* features,
	int channel_first,
	const float* dL_ddensity,
	const float* dL_dout_features,
	float* dL_dpoints,
	float* dL_dmeans3D,
	float* dL_dscales,
	float* dL_drotations,
	float* dL_dopacities,
	float* dL_dfeature,
	int debug,
	void* stream);

/*
 * Point visibility (no reference counterpart): where Q 3D points land in each view, and how much of the cloud lies between
 * the camera and each point, with the blend's own tile lists, depth order, thresholds and early stop.  For view v and a
 * point x, with the expressions the projection and the forward blend already use:
 *   - Projection: (u, v) is the screen position of x under the view's model (pinhole and orthographic through projmatrix and
 *     ndc2pix, fisheye and distorted views through their lens maps: the map the projection applies to a Gaussian's mean,
 *     the same device function as the flow plane's m), d = t.z its view-space depth.  Pixel centres are at integers.
 *   - in_view: x passes that map's cull (t.z > NEAR_Z; fisheye theta <= theta_max; distorted r2 <= r_max^2 and det Dd > 0)
 *     and -0.5 <= u < W - 0.5, -0.5 <= v < H - 0.5.
 *   - Candidates: the instances of the 16x16 tile holding pixel (floor(u + 0.5), floor(v + 0.5)), in the tile list's order
 *     (depth, then the stable sort's order), restricted to instances with depth z_i < d (strict): a prefix of the list.
 *   - transmittance: T = prod (1 - alpha_i) over the candidates, alpha_i at the continuous (u, v) with the forward's
 *     expression min(0.99, o exp(power)) (o the compensated opacity with antialiasing = 1), a candidate skipped where
 *     power > 0 or alpha < 1/255, accumulated in list order with the forward's stop: the factor that would take T below 1e-4
 *     is not applied, and the product ends there.
 *   - Outside the view (in_view false) T = 1.  uv and depth are written wherever the cull passes, NaN where it fails.
 * Hence at a pixel centre with d behind every Gaussian, T is that pixel's final_T bit for bit (the 8x4 block lists drop only
 * pairs with alpha < 1/255 at every pixel centre of the block, which contribute nothing); a point in front of every Gaussian
 * has T = 1; along a ray T does not increase with d.  mgs_visibility_views_backward below differentiates them.
 * Arguments are those of mgs_lift_views with the map arguments replaced by the points and the outputs:
 *   - points [Q,3]; out_uv [V,Q,2], out_depth [V,Q], out_in_view [V,Q] (uint8 0/1), each NULL to skip it; out_T [V,Q].
 *   - Per view: viewmatrix, projmatrix, cam_pos (with SHs), radii (written, as by the forward), the three state buffers
 *     (sized as for mgs_forward_views), binning_capacity, status and stream as for the lift, and blend_scratch, the point
 *     scratch of mgs_visibility_scratch_bytes(Q, width, height) bytes (contents irrelevant on entry).  Every other field is
 *     ignored (dL_dmean2D carries the backward's scratch).  The view's state afterwards holds its projection and binning;
 *     the blend state is not written.
 *   - Nothing allocates or blocks: a call can be captured in a CUDA graph.  Q = 0 returns 0 and enqueues nothing.
 * Argument errors return, with mgs_last_error set and before anything is enqueued, MGS_ERR_INVALID_ARG for: V <= 0, Q < 0,
 * points NULL with Q > 0, out_T NULL, a view without its state buffers, blend_scratch, matrices or radii, the camera-model
 * errors of the distortion section, and the Gaussian-argument errors of mgs_lift_views.
 */
size_t mgs_visibility_scratch_bytes(int Q, int width, int height);
int mgs_visibility_views(
	int V, const mgs_view* views, int antialiasing, const mgs_view_intrinsics* intr, const int* ortho,
	const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion,
	int P, int D, int M, int Q, const float* points,
	const float* means3D, const float* shs, const float* colors_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* out_uv, float* out_depth, uint8_t* out_in_view, float* out_T, int debug, void* join_stream);

/*
 * Point visibility backward (no reference counterpart): the chain of cotangents dL_dT, dL_duv and dL_ddepth of the outputs of
 * mgs_visibility_views into the points, the cloud and the cameras.  With uv, d, in_view and T those outputs for view v and
 * point x:
 *   - Transmittance, where in_view only.  A, the accepted candidates, are the candidates in tile-list order with power <= 0
 *     and alpha >= 1/255 before the factor that would take T below 1e-4.  dT/dalpha_i = -T / (1 - alpha_i) for i in A, 0
 *     for every other instance, with alpha_i = min(0.99, o_i G_i(uv)).  As in the blend backward, dL/dG = o dL/dalpha with
 *     no mask for the 0.99 clamp and dL/do = G dL/dalpha (o the compensated opacity with antialiasing = 1).  The tile, the
 *     candidate set, the depth cut, the 1/255 cut and the stop are constants: d receives nothing through T.  Through G_i(uv)
 *     T reaches the Gaussian's screen mean, conic and opacity, and uv, with dG/duv = -dG/dmean.
 *   - uv and depth, where the view's cull passes: uv through the projection's map of a mean, d = t.z through row 2 of the
 *     view matrix, to the point and the view's camera.  Where the cull fails (uv and depth NaN) their cotangents are ignored.
 *   - Outputs, each NULL to skip it and fully written otherwise (sums over the V views): dL_dpoints [Q,3]; dL_dmean3D [P,3],
 *     dL_dopacity [P], dL_dscale [P,3], dL_drot [P,4] (zeros without scales and rotations) and dL_dcov3D [P,6] (with
 *     cov3D_precomp) through the per-Gaussian chain of the render's backward; per view through `cam` (one
 *     mgs_view_camera_grad per view, or NULL; its scratch field is ignored) dL_dviewmatrix, dL_dprojmatrix and dL_dcampos
 *     (0: no SHs), and through intr (as mgs_render_options.intrinsics) dL_dtan_fov with a device field of view.  A camera's gradient
 *     sums the Gaussian path and the point path, with the definitions of the camera-gradient and intrinsics sections.
 *   - Arguments: those of mgs_visibility_views, unchanged since that call (its views' state buffers and point scratch in
 *     blend_scratch are read as it left them), with its outputs replaced by out_T [V,Q] (its T; needed with dL_dT), the
 *     cotangents dL_dT [V,Q], dL_duv [V,Q,2] and dL_ddepth [V,Q] (each nullable), the outputs and `cam`.  Each view also
 *     carries its backward scratch of mgs_visibility_backward_scratch_bytes(P, Q) bytes (contents irrelevant on entry) in
 *     mgs_view.dL_dmean2D, cast; mgs_visibility_views ignores that field.
 *   - The per-Gaussian chain runs when a cloud or camera output is asked for, the point chain when dL_dpoints or a camera
 *     output is.  The blend-stage rows of the Gaussians are summed with float reductions, so their last bits may vary from
 *     call to call, as the render backward's; dL_dpoints and the point path's camera sums are deterministic (each point sums
 *     its views in order; the camera rows are fixed-order partial sums).
 *   - Nothing allocates, blocks or reads back to the host: a call can be captured in a CUDA graph.  Q = 0 returns 0 and
 *     enqueues nothing.
 * Argument errors return, with mgs_last_error set and before anything is enqueued, MGS_ERR_INVALID_ARG for those of
 * mgs_visibility_views (out_T only with dL_dT), a view without its backward scratch, and dL_dcov3D without cov3D_precomp.
 */
size_t mgs_visibility_backward_scratch_bytes(int P, int Q);
int mgs_visibility_views_backward(
	int V, const mgs_view* views, int antialiasing, const mgs_view_intrinsics* intr, const int* ortho,
	const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion,
	int P, int D, int M, int Q, const float* points,
	const float* means3D, const float* shs, const float* colors_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	const float* out_T, const float* dL_dT, const float* dL_duv, const float* dL_ddepth,
	float* dL_dpoints, float* dL_dmean3D, float* dL_dopacity, float* dL_dscale, float* dL_drot, float* dL_dcov3D,
	const mgs_view_camera_grad* cam, int debug, void* join_stream);

/*
 * Camera rays (no reference counterpart): the inverse of the map the projection applies to a mean (screen_mean, as in point
 * visibility), from a pixel to the world points it is the image of.  For view v and pixel position (u, v) (pixel centres at
 * integers), the ray is the set of points p whose screen position is (u, v); each is labelled by its view-space depth z = t.z,
 * the quantity the depth plane holds, and for every camera model that set is the line
 *   p(z) = origin + z direction,   direction's view-space z component exactly 1 (not unit length),
 * so origin + depth direction unprojects a z-depth image, or the renderer's own depth / alpha.
 *   - Pinhole and orthographic: with (nx, ny) = ((2u + 1) / W - 1, (2v + 1) / H - 1) (ndc2pix's inverse) and Pk, Vk the rows
 *     of projmatrix and viewmatrix, the rows (P0 - nx P3) (p, 1) = nx 1e-7, (P1 - ny P3) (p, 1) = ny 1e-7 and V2 (p, 1) = z:
 *     a 3x3 system A p = b + z e3, so origin = A^-1 b and direction = A^-1 e3.  An off-centre principal point baked into
 *     projmatrix and the orthographic origin that moves with the pixel are covered.  Valid where det A is finite and non-zero.
 *   - Fisheye: (xd, yd) = ((u - cx) / fx, (v - cy) / fy), theta_d = |(xd, yd)|, theta in [0, theta_max] the root of
 *     theta rho(theta) = theta_d (safeguarded Newton, FISHEYE_RAY_ITERS = 16 steps at most; monotone there by
 *     cameras.fisheye_theta_max), t = z (tan theta xd / theta_d, tan theta yd / theta_d, 1), p = Rv^T (t - tv).  The axis pixel
 *     takes tan(theta) / theta from its series.  Valid iff theta_d <= theta_max rho(theta_max) (and tan theta finite, >= 0).
 *   - Distorted pinhole: Newton's method with Dd on distort(x, y) = (xd, yd) from (xd, yd), DIST_RAY_ITERS = 20 steps at
 *     most; t = z (x, y, 1).  Valid iff the iterate passes the projection's cull (r2 <= r_max^2, det Dd > 0) and
 *     |distort(x, y) - (xd, yd)| <= 1e-6 (1 + |(xd, yd)|): fp32 evaluates distort at |x| <~ 2 to a few ulps of 2.4e-7, so a
 *     converged iterate passes it; at fx = 500 px the bound is 5e-4 px.
 *   - fx = W / (2 tan_fovx), fy = H / (2 tan_fovy) (or the device field of view, as for the projection).
 *   - For a valid ray and z > NEAR_Z, p(z) passes the model's cull and projects back to (u, v) up to fp32 rounding.  An invalid
 *     ray (the pixel is not the image of points the projection keeps, or is not finite) has origin and direction NaN.
 * Arguments: views, intr, ortho, fisheye and distortion as mgs_visibility_views takes them; of each view only viewmatrix,
 * projmatrix (both required), tan_fovx, tan_fovy, width and height are read.  pixels [V,Q,2], or NULL for every pixel centre
 * of the W x H grid, ray i at (i % W, i / W): then Q must equal width * height of every view.  Outputs out_origin [V,Q,3],
 * out_direction [V,Q,3] and out_valid [V,Q] (uint8 0/1), all required with Q > 0.  One stream for every view.
 * Backward, by implicit differentiation of those maps (the 3x3 solve, the inverse of the fisheye forward Jacobian, Dd^-1): the
 * forward's inputs unchanged, the cotangents dL_dorigin and dL_ddirection ([V,Q,3], each NULL for zero), and the outputs
 * dL_dpixels [V,Q,2] (NULL to skip; needs pixels) and, per view through `cam` (one mgs_view_camera_grad per view, or NULL),
 * dL_dviewmatrix, dL_dprojmatrix (pinhole and orthographic only) and dL_dcampos (always 0), and through intr dL_dtan_fov
 * (fisheye and distorted views: fx enters no pinhole or orthographic term, as in screen_mean).  A view with a camera output
 * needs its entry's scratch of mgs_camera_rays_scratch_bytes(Q) bytes.  The principal point, the coefficients, theta_max,
 * r_max and NEAR_Z are constants, valid has no gradient, and an invalid ray's cotangents are ignored (its pixel gradient is
 * 0).  Every output is written.  The camera sums are fixed-order partial sums (one row per CTA of RAYS_THREADS rays, summed
 * by the camera-gradient reduce): the backward is deterministic.
 * Nothing allocates, blocks or reads back to the host: both calls can be captured in a CUDA graph.  Q = 0 returns 0 and
 * enqueues nothing (no output is written).
 * Argument errors return, with mgs_last_error set and before anything is enqueued, MGS_ERR_INVALID_ARG for: V <= 0 or views
 * NULL, the camera-model errors of the distortion section, Q < 0, a view without its matrices or with a size <= 0, pixels NULL
 * with Q != width * height of a view, a NULL output (forward, Q > 0), dL_dpixels without pixels, and a camera output without
 * its entry's scratch.
 */
size_t mgs_camera_rays_scratch_bytes(int Q);
int mgs_camera_rays(int V, const mgs_view* views, const mgs_view_intrinsics* intr, const int* ortho,
	const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion, int Q, const float* pixels,
	float* out_origin, float* out_direction, uint8_t* out_valid, int debug, void* stream);
int mgs_camera_rays_backward(int V, const mgs_view* views, const mgs_view_intrinsics* intr, const int* ortho,
	const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion, int Q, const float* pixels,
	const float* dL_dorigin, const float* dL_ddirection, float* dL_dpixels, const mgs_view_camera_grad* cam, int debug,
	void* stream);

/*
 * k nearest neighbours (no reference counterpart; simple-knn's distCUDA2 is the mean of the first three d2 of each point):
 * for each of Q queries, its k nearest of N reference points by the fp32 squared distance
 *   d2 = (qx - px)^2 + (qy - py)^2 + (qz - pz)^2,
 * the exact k-nearest set for those distances (there is no approximate mode).
 *   - queries [Q,3], or NULL: the points themselves (Q must equal N), and then query i never returns index i (a duplicate
 *     of point i at distance 0 is returned).
 *   - Order: each query's results ascend by (d2, index), so ties go to the lower index; the results are deterministic.
 *   - A point with a non-finite coordinate is never a neighbour; a non-finite query has every slot padded.  Where fewer
 *     than k neighbours exist, the remaining slots are index -1, d2 = +inf.
 *   - out_index [Q,k] (long long: usable as a torch index without a conversion), out_dist2 [Q,k], both fully written.
 *   - state: mgs_knn_state_bytes(N, Q) bytes of device memory on the device current at the call (contents irrelevant on
 *     entry); the size depends on the device, so query it with the same device current as mgs_knn.  0 means CUDA's size
 *     query failed (mgs_last_error says why).
 *   - k is 1 .. 32 (larger k returns MGS_ERR_UNSUPPORTED).  Q = 0 returns 0 and enqueues nothing; N = 0 pads every slot.
 * Method: a grid over the points' bounding box whose resolution is chosen on the device from the occupied cells, the points
 * and queries sorted by cell, and one warp per 32 queries of a cell searching shells of cells until the distance to the
 * unvisited cells exceeds each query's k-th d2.  Nothing allocates, blocks or reads back to the host: a call can be
 * captured in a CUDA graph.
 * Argument errors return, with mgs_last_error set and before anything is enqueued: MGS_ERR_UNSUPPORTED for k > 32;
 * MGS_ERR_INVALID_ARG for k < 1, N < 0, Q < 0, queries NULL with Q != N (Q > 0), and a NULL state, points (N > 0) or
 * output (Q > 0).
 */
size_t mgs_knn_state_bytes(int N, int Q);
int mgs_knn(void* state, int N, int Q, int k, const float* points, const float* queries, long long* out_index, float* out_dist2,
	int debug, void* stream);

/*
 * Neighbour regularisers of a dynamic field (Dynamic 3D Gaussians, Luiten et al.; no reference counterpart): local rigidity,
 * rotation similarity and isometry between a cloud (xyz [P,3], rot [P,4]) and its deformed next frame (xyz_next [P,3],
 * rot_next [P,4]) over fixed neighbour lists index [P,k] (as mgs_knn returns them) with constant weights weight [P,k]
 * (callers pass exp(-lambda dist2) from the same mgs_knn call).  Quaternions are (r, x, y, z), real part first.  Per Gaussian i:
 *   q_i = rot_i / max(|rot_i|, 1e-12),  qn_i = rot_next_i / max(|rot_next_i|, 1e-12)            (F.normalize)
 *   rel_i = qn_i (x) conj(q_i)                                                                    (Hamilton product)
 *   R_i = qrot(rel_i)   (INTEGRATION.md section 17's formula; rel is not renormalised)
 * Per slot (i, s) with j = index[i,s], w = weight[i,s]: the slot is valid iff 0 <= j < P (padding -1 and out-of-range
 * indices are skipped before anything is read; j = i gives zero offsets); o = xyz_j - xyz_i, o' = xyz_next_j - xyz_next_i;
 *   rigid    = 1/(P k) sum_valid w |o' - R_i o|
 *   rotation = 1/(P k) sum_valid w |rel_j - rel_i|
 *   isometry = 1/(P k) sum_valid w | |o'| - |o| |
 * written to out_loss[0..2] (device memory).  P = 0 writes three zeros.  The losses are bitwise identical from call to call.
 * Backward: dL_dloss [3] in device memory (never read by the host); gradients, each NULL to skip it and fully written
 * otherwise, to xyz [P,3], rot [P,4], xyz_next [P,3] and rot_next [P,4], none to weight or index.  Conventions as torch:
 * d|v|/dv = v/|v| and 0 at v = 0; d|a|/da = sign(a), 0 at 0; below the 1e-12 clamp the normalisation's gradient is that
 * of x / 1e-12.  The backward's float atomics make its last bits depend on the order of the reductions.
 *   - state: mgs_neighbour_reg_state_bytes(P, k) bytes of device memory, any alignment; the backward reads what the forward
 *     with the same inputs left there (the offsets and rel of every Gaussian), so it takes the forward's arguments unchanged.
 *   - k is 1 .. 32 (larger k returns MGS_ERR_UNSUPPORTED).
 * Nothing allocates, blocks or reads back to the host: both calls can be captured in a CUDA graph.
 * Argument errors return, with mgs_last_error set and before anything is enqueued: MGS_ERR_UNSUPPORTED for k > 32;
 * MGS_ERR_INVALID_ARG for k < 1, P < 0, and a NULL state, out_loss / dL_dloss, or input (P > 0).
 */
size_t mgs_neighbour_reg_state_bytes(int P, int k);
int mgs_neighbour_reg(void* state, int P, int k, const float* xyz, const float* rot, const float* xyz_next,
	const float* rot_next, const long long* index, const float* weight, float* out_loss, int debug, void* stream);
int mgs_neighbour_reg_backward(void* state, int P, int k, const float* xyz, const float* rot, const float* xyz_next,
	const float* rot_next, const long long* index, const float* weight, const float* dL_dloss, float* dL_dxyz, float* dL_drot,
	float* dL_dxyz_next, float* dL_drot_next, int debug, void* stream);

/*
 * Deformation by a sparse control graph (embedded deformation, Sumner et al.; SC-GS; no reference counterpart): a cloud
 * (xyz [P,3], rot [P,4]) moved by N control nodes (node_xyz [N,3], node_rot [N,4], node_t [N,3]), each Gaussian blending
 * the rigid motions of the nodes its row of index [P,k] names (as mgs_knn returns it for the nodes, queried at xyz) with
 * weights weight [P,k], used exactly as given (not normalised).  Quaternions are (r, x, y, z), real part first.  Per node j:
 *   q^_j = node_rot_j / max(|node_rot_j|, 1e-12), negated where its real part is below 0 (kept at exactly 0)
 *   R_j = qrot(q^_j)   (INTEGRATION.md section 17's formula),   c_j = node_xyz_j + node_t_j - R_j node_xyz_j
 * so node j moves a point x to R_j x + c_j, a rotation about the node followed by its translation.  Per Gaussian i, summed
 * over its valid slots s (0 <= j = index[i,s] < N; padding -1 and out-of-range indices are skipped before anything is read),
 * w = weight[i,s] and e = (1, 0, 0, 0):
 *   out_xyz_i = xyz_i + sum_s w (R_j xyz_i + c_j - xyz_i)
 *   r_i = e + sum_s w (q^_j - e),   out_rot_i = normalize(r_i) (x) rot_i     (Hamilton product; rot_i used as given)
 * Weight missing from 1 goes to the identity motion: a row without a valid slot, or with zero weights, is copied unchanged.
 * The outputs are bitwise identical from call to call.
 * Backward: dL_dout_xyz [P,3] and dL_dout_rot [P,4] (each NULL: zero); gradients, each NULL to skip it and fully written
 * otherwise, to xyz [P,3], rot [P,4], node_xyz [N,3], node_rot [N,4], node_t [N,3] and weight [P,k] (0 in invalid slots).
 * Conventions as torch: below the 1e-12 clamp the normalisation's gradient is that of x / 1e-12, and the sign of q^_j passes
 * the gradient through.  The node gradients are float atomics: their last bits depend on the order of the reductions.
 *   - state: mgs_deform_state_bytes(P, N, k) bytes of device memory, any alignment (k does not change it); the backward
 *     reads what the forward with the same inputs left there (the node records and each r_i), so it takes the forward's
 *     arguments unchanged.
 *   - k is 1 .. 32 (larger k returns MGS_ERR_UNSUPPORTED).  P = 0 or N = 0 is allowed.
 * Nothing allocates, blocks or reads back to the host: both calls can be captured in a CUDA graph.
 * Argument errors return, with mgs_last_error set and before anything is enqueued: MGS_ERR_UNSUPPORTED for k > 32;
 * MGS_ERR_INVALID_ARG for k < 1, P < 0, N < 0, a NULL state, a NULL xyz, rot, index or weight (P > 0), a NULL node_xyz,
 * node_rot or node_t (N > 0), and a NULL out_xyz or out_rot of the forward (P > 0).
 */
size_t mgs_deform_state_bytes(int P, int N, int k);
int mgs_deform(void* state, int P, int N, int k, const float* xyz, const float* rot, const float* node_xyz, const float* node_rot,
	const float* node_t, const long long* index, const float* weight, float* out_xyz, float* out_rot, int debug, void* stream);
int mgs_deform_backward(void* state, int P, int N, int k, const float* xyz, const float* rot, const float* node_xyz,
	const float* node_rot, const float* node_t, const long long* index, const float* weight, const float* dL_dout_xyz,
	const float* dL_dout_rot, float* dL_dxyz, float* dL_drot, float* dL_dnode_xyz, float* dL_dnode_rot, float* dL_dnode_t,
	float* dL_dweight, int debug, void* stream);

/*
 * Farthest-point sampling (no reference counterpart; SC-GS control nodes, point-cloud policy inputs): n picks from each of
 * B clouds points [B,P,3].  Cloud b is points[b, :L_b] with L_b = lengths[b] clamped to 0 .. P (P when lengths is NULL).
 *   - Only points with three finite coordinates can be picked.  Each starts with d_i = +inf.
 *   - Pick 0 is start[b] when start is given and start[b] is a finite point in 0 .. L_b - 1; otherwise the lowest-index
 *     finite point (which the argmax rule below gives when every d is +inf).
 *   - After each pick s, every unpicked finite point i takes d_i = min(d_i, D(i, s)), and s is never picked again.  D is
 *     the fp32 squared distance in a fixed order with every operation rounded to float32 and no FMA contraction:
 *       dx = x_i - x_s, dy = y_i - y_s, dz = z_i - z_s,   D = ((dx*dx) + (dy*dy)) + (dz*dz)
 *   - Pick t >= 1 is the unpicked finite point with the largest d; ties go to the lower index.
 *   - out_index [B,n] is each pick as an index into its cloud; out_dist2 [B,n] is its d at the time of the pick, the squared
 *     distance to the nearest earlier pick (out_dist2[b,0] = +inf).  Where fewer than n finite points exist, the rest of
 *     the row is index -1, d2 = +inf.  So the picks of a row are distinct, out_dist2[b,1:] never increases along the valid
 *     picks, and duplicate points are picked at d2 = 0 in ascending index once every distinct position is taken.
 *   - The outputs are bitwise identical from call to call.
 *   - lengths [B] and start [B] (each NULL to omit) are in device memory and never read by the host.
 *   - state: mgs_fps_state_bytes(B, P) bytes of device memory (contents irrelevant on entry).
 *   - B = 0 or n = 0 returns 0 and enqueues nothing; P = 0 pads every slot.
 * Method: one thread-block cluster per cloud, its CTAs holding the cloud's points and their d in registers (clouds above
 * 131,072 points stream a packed copy kept in the state), one cluster-wide argmax through distributed shared memory per
 * pick.  Nothing allocates, blocks or reads back to the host: a call can be captured in a CUDA graph.
 * Argument errors return, with mgs_last_error set and before anything is enqueued: MGS_ERR_INVALID_ARG for B, P or n < 0,
 * and for a NULL state, out_index or out_dist2 (B > 0 and n > 0) or points (also P > 0).
 */
size_t mgs_fps_state_bytes(int B, int P);
int mgs_fps(void* state, int B, int P, int n, const float* points, const long long* lengths, const long long* start,
	long long* out_index, float* out_dist2, int debug, void* stream);

/*
 * TSDF fusion (no reference counterpart; KinectFusion's and Open3D's rule with unit weights, no bitwise parity with Open3D
 * claimed): V depth images fused into a truncated signed-distance volume over the [X,Y,Z] grid of bounds (host double[6],
 * x0 y0 z0 x1 y1 z1).  Voxel (i, j, k) sits at voxel_centres' point: per axis lo + (i + 1/2) ((hi - lo) / n) evaluated in
 * double (no FMA), rounded once to float.  For each voxel centre x, over the views v = 0 .. V-1 in order:
 *   1. (px, py) and z = t.z from the projection's map of a mean (screen_mean, as in point visibility), with its cull
 *      (NEAR_Z, a fisheye's theta_max, a distorted lens's r_max and fold); a culled view is skipped;
 *   2. the pixel is (i, j) = (floor(px + 0.5), floor(py + 0.5)), pixel centres at integers; a view is skipped unless
 *      (px, py) lies in [-0.5, W - 0.5) x [-0.5, H - 0.5) (point visibility's bounds; i and j are clamped to W - 1, H - 1);
 *   3. d = depth[v, j, i]; a view is skipped where d is not finite or d <= 0 (no return);
 *   4. s = d - z; a view is skipped where s < -trunc (the voxel is occluded);
 *   5. f = min(1, s / trunc), tsdf <- (tsdf w + f) / (w + 1), for each channel c <- (c w + color[v, :, j, i]) / (w + 1),
 *      then w <- w + 1, every operation rounded to float32 in this order (no FMA).
 * Arguments: views, intr, ortho, fisheye and distortion as mgs_camera_rays takes them (of each view viewmatrix, projmatrix,
 * tan_fovx, tan_fovy, width and height are read; every view has the same width W and height H).  depth [V,H,W] view-space z;
 * color [V,C,H,W] or NULL with C = 0, C in 0 .. 32; trunc > 0 in world units.  tsdf [X,Y,Z], weight [X,Y,Z] and
 * color_volume [C,X,Y,Z] (NULL with C = 0) are read and updated in place: a fresh volume holds tsdf 1, weight 0, colour 0.
 *   - The result is bitwise repeatable, one call over V views is bitwise equal to successive calls over any split of the
 *     same views in order, and a voxel no view updates is left bitwise unchanged (it is not written).
 *   - Views run in launches of up to 64, each reading and writing the volume once.
 * Nothing allocates, blocks or reads back to the host: a call can be captured in a CUDA graph.  Not differentiable.
 * Argument errors return, with mgs_last_error set and before anything is enqueued, MGS_ERR_INVALID_ARG for: V <= 0 or views
 * NULL, the camera-model errors of the distortion section, a view without its matrices or with a size <= 0, views of
 * different sizes, X, Y or Z <= 0, trunc <= 0 or not finite, C outside 0 .. 32, bounds NULL, not finite or not increasing,
 * and a NULL depth, tsdf or weight, or color or color_volume with C > 0.
 */
int mgs_tsdf_fuse(int V, const mgs_view* views, const mgs_view_intrinsics* intr, const int* ortho,
	const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion, const float* depth, int C, const float* color,
	const double* bounds, int X, int Y, int Z, float trunc, float* tsdf, float* weight, float* color_volume, int debug,
	void* stream);

/*
 * Marching cubes (no reference counterpart): the level surface of values [X,Y,Z] (a TSDF at level 0, or a density) as an
 * indexed triangle mesh.  Grid point (i, j, k) sits at its voxel centre over bounds, as in mgs_tsdf_fuse.
 *   - A grid point is valid when its value is finite and, with weight [X,Y,Z] (NULL for none), its weight is > 0.  The
 *     cells are the (X-1)(Y-1)(Z-1) cubes of 8 neighbouring points; a cell with an invalid corner emits nothing.  Corner c
 *     of the cell with lower corner (i, j, k) is the point (i + (c & 1), j + ((c >> 1) & 1), k + ((c >> 2) & 1)), below when
 *     value < level; the case index has bit c set for a below corner (csrc/mc_table.cuh holds the table and its numbering).
 *   - Each crossed cell edge (exactly one endpoint below) that an emitted triangle uses gets exactly one vertex, shared by
 *     every cell around the edge: no vertex is duplicated or unused.  With a the edge's lower endpoint (first in x-major
 *     order) and b the other, t = (level - v_a) / (v_b - v_a) and p = c_a + t (c_b - c_a) per coordinate, each operation
 *     rounded to float32 (no FMA); colours (color [C,X,Y,Z], C in 0 .. 32) are interpolated with the same t.  Vertices are
 *     ordered by (a in x-major order, then the edge's axis x < y < z).
 *   - Faces follow the table's triangles, cells in x-major order.  Each normal (v1 - v0) x (v2 - v0) points toward
 *     increasing value.  An ambiguous face always cuts off its below corners, from both cells that share it, so a level
 *     set inside the valid region gives a closed mesh.  Zero-area triangles (a value exactly at the level) are kept.
 *   - The mesh is bitwise repeatable (no atomics).
 * Two calls: mgs_marching_cubes_count fills the state (mgs_marching_cubes_state_bytes(X, Y, Z) bytes of device memory,
 * contents irrelevant on entry: 18 bytes per grid point and CUB's scan space) and writes out_counts (device, 2 long long)
 * = {vertex count Nv, face count Nf}; the caller reads them back and sizes out_vertices [Nv,3], out_faces [Nf,3] (long long)
 * and out_colors [Nv,C] (NULL with C = 0) for mgs_marching_cubes_emit, which takes the same state, values and level.
 * A grid with a side below 2 has no cell: both calls return 0 and enqueue nothing (out_counts is not written).
 * Argument errors return, with mgs_last_error set and before anything is enqueued, MGS_ERR_INVALID_ARG for: X, Y or Z < 0,
 * C outside 0 .. 32, bounds NULL, not finite or not increasing (emit), and a NULL state, values, out_counts, out_vertices or
 * out_faces, or color or out_colors with C > 0.
 */
size_t mgs_marching_cubes_state_bytes(int X, int Y, int Z);
int mgs_marching_cubes_count(void* state, int X, int Y, int Z, const float* values, const float* weight, float level,
	long long* out_counts, int debug, void* stream);
int mgs_marching_cubes_emit(void* state, int X, int Y, int Z, const float* values, float level, const double* bounds, int C,
	const float* color, float* out_vertices, long long* out_faces, float* out_colors, int debug, void* stream);

/*
 * MCMC density control (3DGS as Markov chain Monte Carlo, Kheradmand et al. 2024; gsplat's MCMCStrategy; no reference
 * counterpart).  Parameters are raw, in 3DGS's parameterisation, fp32, contiguous, on one device: means [P,3], quats [P,4]
 * (r, x, y, z; not necessarily unit), log_scales [P,3] (s = exp(log_scales)), opacity_logit [P] (o = sigmoid(x)).  Further
 * per-Gaussian rows (SH [P,K,3], features [P,F], ...) travel as host arrays rows[num_rows] of device pointers with
 * row_widths[num_rows] floats per Gaussian; optimizer moments (exp_avg, exp_avg_sq, max_exp_avg_sq of every parameter,
 * the four above included) likewise as moments[num_moments] with moment_widths.
 *
 * Random numbers: Philox4x32-10 (Random123) with key {seed lo, seed hi} and counter {slot, offset lo, offset hi, tag}, tag 0
 * for relocation and 1 for perturbation.  rng is device int64 [2] = {seed, offset}; each call reads it on the device and
 * then advances offset by one there, so a replayed CUDA graph draws fresh numbers and equals the same eager calls.  Of the
 * four output words w0..w3: a uniform 64-bit draw is r64 = w0 + 2^32 w1; normals are Box-Muller in fp32 with
 * u1 = (float(w) + 1) 2^-32 and u2 = float(w') 2^-32: z0 = sqrt(-2 ln u1) cos(2 pi u2) and z1 = ... sin(2 pi u2) from
 * (w0, w1), z2 = the cosine of (w2, w3).
 *
 * Relocation and growth, mgs_mcmc_relocate: rows [P_old, P) are newly appended rows.
 *   - t = fp32(logit(min_opacity)).  Gaussian i < P_old is dead iff x_i <= t.  The destinations are the dead slots and every
 *     slot in [P_old, P).
 *   - w_i = floor(2^24 sigmoid_f64(x_i)) for alive i, 0 otherwise (also for a NaN x_i, which is neither dead nor a source);
 *     S is their inclusive uint64 scan, T = S[P_old - 1].
 *   - Destination j draws r64_j (slot j), u = mulhi64(r64_j, T), and takes src_j = min{i : S_i > u}: integer-exact, so it
 *     does not depend on the scan's order.
 *   - m_i = the number of destinations that picked i; n_i = min(m_i + 1, 51) (gsplat's clamp).  A source (m_i > 0) gets, in
 *     fp64, o' = -expm1(log1p(-o) / n) and s' = s o / sum_{j=1..n} C(n,j) (-1)^(j-1) o'^j / sqrt(j) (gsplat's double sum
 *     collapsed by the hockey-stick identity); o' is then clamped to [min_opacity, 1 - 2^-23], and the source's x and
 *     log_scales become fp32(logit(o')) and fp32(log(s')).  The alternating sum loses about log10 of its largest term in
 *     digits: 3 at o = 1 - 5e-5 (x = 10) and n = 51, all of them as o -> 1.
 *   - Every destination becomes a copy of its source's new row: means, quats, log_scales, opacity_logit and every listed
 *     row.  Every listed moment row is zeroed at every source and every destination (gsplat zeroes only the sources, which
 *     leaves a copy with the dead Gaussian's stale moments).
 *   - out_relocated: device int64 [1], the number of destinations filled; out_source: device int64 [P], src_j or -1 where
 *     there is none, so callers can carry their own non-float state (labels, neighbour rows).
 *   - T = 0 (nothing alive) writes no row, and out_relocated is 0.
 *   - The result is bitwise repeatable (integer atomics count, and the per-source maths has no reduction), so the ranks of a
 *     view-parallel run stay identical without a broadcast.
 *   - state: mgs_mcmc_state_bytes(P_old) bytes of device memory on the device current at the call (contents irrelevant on
 *     entry: the weights' scan, the counts and CUB's scan space; 12 bytes per Gaussian and the scan space).  0 means CUDA's
 *     size query failed (mgs_last_error says why).
 * Method: CUB's scan over the weights, then one thread per slot (dead test, draw, binary search, count), one per source
 * (fp64 maths, moments), and one per (slot, tensor) for the copies; the tensors go to the kernels by value.
 * Argument errors return, with mgs_last_error set and before anything is enqueued, MGS_ERR_INVALID_ARG for: P_old < 0 or
 * P < P_old, min_opacity outside (0, 1), a NULL state, rng or out_relocated, a NULL out_source or parameter with P > 0,
 * num_rows outside 0 .. MGS_MCMC_MAX_ROWS or num_moments outside 0 .. MGS_MCMC_MAX_MOMENTS, a NULL pointer or width array
 * with a count > 0, a width <= 0, and a NULL row or moment pointer with P > 0.
 *
 * Position noise, mgs_mcmc_perturb: per Gaussian i, means_i += Sigma_i z_i g(o_i) scale with
 *   Sigma_i = R(q^) diag(s^2) R(q^)^T, q^ = q / max(|q|, 1e-12)   (the projection's covariance formula, fp32)
 *   z_i ~ N(0, I3) from slot i,   g(o) = 1 / (1 + exp(-100 ((1 - o) - 0.995))),
 * scale (device float [1]) = lr_means * noise_lr (gsplat: noise_lr = 5e5), read on the device so a captured graph follows
 * the learning-rate schedule.  Only means is written.  quats must be 16-byte aligned.  P = 0 only advances the offset.
 * Argument errors return, with mgs_last_error set and before anything is enqueued, MGS_ERR_INVALID_ARG for: P < 0, a NULL
 * rng, a NULL means, quats, log_scales, opacity_logit or scale with P > 0, and misaligned quats.
 * Neither call allocates, blocks or reads back to the host: both can be captured in a CUDA graph.  Not differentiable.
 */
#define MGS_MCMC_MAX_ROWS 16
#define MGS_MCMC_MAX_MOMENTS 64
size_t mgs_mcmc_state_bytes(int P);
int mgs_mcmc_relocate(void* state, int P_old, int P, float min_opacity, float* means, float* quats, float* log_scales,
	float* opacity_logit, int num_rows, float* const* rows, const int* row_widths, int num_moments, float* const* moments,
	const int* moment_widths, long long* rng, long long* out_source, long long* out_relocated, int debug, void* stream);
int mgs_mcmc_perturb(int P, float* means, const float* quats, const float* log_scales, const float* opacity_logit,
	const float* scale, long long* rng, int debug, void* stream);

/*
 * Default density control (3DGS's adaptive density control as gsplat's DefaultStrategy runs it; no reference counterpart).
 * Parameters, extra rows and moments as in the MCMC section above.
 *
 * Statistics, mgs_densify_stats: for each Gaussian i, over the views v = 0 .. V-1 in order, where radii[v,i] > 0:
 *   n = sqrt(gx gx + gy gy) with (gx, gy) the first two components of viewspace_grad[v,i];
 *   grad2d_i += n scale;   count_i += 1;   radius_i = max(radius_i, float(radii[v,i]) / float(sizes[v]))
 * every operation rounded to fp32 without FMA, so the result is bitwise equal to a float32 restatement.
 *   - viewspace_grad [V,P,3] fp32 (each view's screen-space mean gradient, the reference's viewspace_points.grad);
 *     radii [V,P] int32; sizes host int[V], each view's max(W, H) > 0; grad2d [P] fp32, count [P] int32 and radius [P]
 *     fp32 are read and updated in place (zero for fresh statistics).
 *   - scale: scale_device (device float [1]) when not NULL, else the host value scale.  A loss averaged over V views has
 *     per-view gradients 1/V as large; scale = V undoes that, as gsplat's n_cameras factor does.
 *   - One thread per Gaussian, no atomics: bitwise repeatable.  Views run in launches of up to 64.  V = 0 or P = 0
 *     enqueues nothing.
 * Argument errors return, with mgs_last_error set and before anything is enqueued, MGS_ERR_INVALID_ARG for: V or P < 0,
 * a NULL viewspace_grad, radii, sizes, grad2d, count or radius with V, P > 0, a size <= 0, and a scale that is not finite
 * with a NULL scale_device.
 *
 * Refinement, mgs_densify_count then mgs_densify_emit (gsplat's duplicate, then split, then prune).  The thresholds move
 * into the log / logit domain once, in fp64, rounded to fp32:
 *   t_opa = fp32(logit(prune_opacity)),  t_small = fp32(log(grow_scale3d scene_scale)),  t_big = fp32(log(prune_scale3d scene_scale)).
 * Per Gaussian i, with L_i = fmaxf(fmaxf(ls0, ls1), ls2) its largest log scale (a NaN operand is ignored) and r_i = radius_i:
 *   - high_i = grad2d_i / max(count_i, 1) > grad_threshold (fp32 division);  small_i = L_i <= t_small;
 *   - clone_i = high_i && small_i;  split_i = (high_i && !small_i) || r_i > grow_scale2d (a Gaussian can be both);
 *   - a row with logit x, largest log scale L and radius r is pruned when
 *     x < t_opa || (prune_too_big && (L > t_big || r > prune_scale2d));
 *   - the kept original: present when !split_i and not pruned; all its rows and moment rows are copied;
 *   - the clone: present when clone_i and the original's row is not pruned; its rows are copied, its moments zero;
 *   - the children b = 0, 1 of a split i, present when not pruned by their own L (their logit and radius are the parent's):
 *     log scales fp32((double)ls - log(1.6)) per axis; means mu + R(q^) diag(exp(ls)) z_{i,b} in fp32 with the parent's
 *     log scales ls and q^ = q / max(|q|, 1e-12); quats, opacity and every extra row copied; moments zero.
 *   - z_{i,b}: the normals z0, z1, z2 of the MCMC section's Box-Muller from Philox counter {i, offset lo, offset hi, 2 + b}.
 *   - Output order (gsplat's concatenation): [kept originals] ++ [kept clones] ++ [kept first children] ++ [kept second
 *     children], each segment in ascending i.
 * grow_scale2d and prune_scale2d take INFINITY to turn their test off (gsplat's None).
 * mgs_densify_count classifies, scans the three per-Gaussian flags (original kept, clone kept, children kept) with CUB and
 * writes out_counts (device int64 [4]) = {n_new, cloned, split, pruned}: cloned and split count clone_i and split_i, and
 * n_new = P + cloned + split - pruned.  state: mgs_densify_state_bytes(P) bytes of device memory (17 bytes per Gaussian
 * and CUB's scan space; contents irrelevant on entry; 0 means CUDA's size query failed).  The caller reads out_counts back
 * (the one host read of a refinement), allocates the n_new-row tensors and calls mgs_densify_emit with the same state, P
 * and old tensors; the new tensors have n_new rows of the same widths (new_rows[k] and new_moments[k] beside rows[k] and
 * moments[k]).  emit writes every new row and out_source (device int64 [n_new], each row's parent i), reads rng = {seed,
 * offset} (device int64 [2]) on the device and advances the offset by one there.  Both calls are bitwise repeatable
 * (integer atomics count; the scan and the rows have no float reduction).  P = 0 writes zero totals; n_new = 0 writes
 * no row.  Argument errors return, with mgs_last_error set and before anything is enqueued, MGS_ERR_INVALID_ARG for:
 *   count: P < 0, a NULL state or out_counts, a NULL input with P > 0, scene_scale, grow_scale3d or prune_scale3d not
 *     finite and > 0, prune_opacity outside (0, 1), and a NaN grad_threshold, grow_scale2d or prune_scale2d;
 *   emit: P or n_new < 0, n_new > 0 with P = 0, a NULL state or rng, a NULL old parameter with P > 0, a NULL new parameter
 *     or out_source with n_new > 0, the row-list errors of mgs_mcmc_relocate (at most MGS_MCMC_MAX_ROWS rows and
 *     MGS_MCMC_MAX_MOMENTS moments), and a NULL new_rows / new_moments array or entry with n_new > 0.
 * Not differentiable.
 */
int mgs_densify_stats(int V, int P, const float* viewspace_grad, const int* radii, const int* sizes, float scale,
	const float* scale_device, float* grad2d, int* count, float* radius, int debug, void* stream);
size_t mgs_densify_state_bytes(int P);
int mgs_densify_count(void* state, int P, const float* log_scales, const float* opacity_logit, const float* grad2d,
	const int* count, const float* radius, double scene_scale, float grad_threshold, double grow_scale3d, float grow_scale2d,
	double prune_opacity, double prune_scale3d, float prune_scale2d, int prune_too_big, long long* out_counts, int debug,
	void* stream);
int mgs_densify_emit(void* state, int P, int n_new, const float* means, const float* quats, const float* log_scales,
	const float* opacity_logit, int num_rows, const float* const* rows, const int* row_widths, int num_moments,
	const float* const* moments, const int* moment_widths, float* new_means, float* new_quats, float* new_log_scales,
	float* new_opacity_logit, float* const* new_rows, float* const* new_moments, long long* rng, long long* out_source, int debug,
	void* stream);

/* The same two loss heads for V images that already sit in device memory (planar color [V,3,N], feature [V,F,N] or NULL,
 * N = H*W): loss_acc [V,2] (zeroed by the call) and the cotangent planes as above, one launch. */
int mgs_loss_heads(int V, int F, int N, const float* color, const float* feature, const float* target_color,
	const float* target_feature, float* cot_color, float* cot_feature, float* loss_acc, void* stream);

/* L1 + SSIM (definitions above) for V images of C planes each that already sit in device memory, x and g [V,C,H,W]; any
 * C >= 1 works (every plane is independent; N = C H W per image) with V C <= 65535.  mgs_ssim writes ssim_terms
 * [V,3,C,H,W] and loss_acc [V,2] = {sum |x - g|, sum S} (zeroed by the call).  mgs_ssim_backward writes cot_out [V,C,H,W] =
 * cot_in + scale[v,0] sign(x - g) / N + scale[v,1] d ssim / dx, with scale [V,2] (device; NULL for 1) and cot_in [V,C,H,W]
 * (NULL for 0); x, g and ssim_terms must be those of the forward. */
int mgs_ssim(int V, int C, int H, int W, const float* x, const float* g, float* ssim_terms, float* loss_acc, void* stream);
int mgs_ssim_backward(int V, int C, int H, int W, const float* x, const float* g, const float* ssim_terms, const float* scale,
	const float* cot_in, float* cot_out, void* stream);

/* Frustum test.  Replaces CudaRasterizer::Rasterizer::markVisible (rasterizer.h:24-29, rasterizer_impl.cu:141-153).
 * present: uint8 [P], 1 where view-space z > 0.2. */
int mgs_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
	uint8_t* present, void* stream);

/*
 * View-independent per-Gaussian pre-ops, one fused kernel per direction ("next" row f2 of the scope table).
 * Replaces the elementwise PyTorch chain ManiGaussian applies to the rasterizer's inputs once per step:
 *   means  = means + d_means                                   (agents/manigaussian_bc/models_embed.py:248, :299)
 *   rot    = normalize(rot + d_rot), x / max(||x||, 1e-12)      (models_embed.py:250, :301)
 *   scales = min(exp(scales + d_scales), scale_max)            (models_embed.py:245-246; scale_mode 1; 0 = identity)
 *   opac   = sigmoid(opac)                                     (models_embed.py:252; opacity_mode 1; 0 = identity)
 *   feat   = feat / (||feat|| + 1e-12)                         (agents/manigaussian_bc/gaussian_renderer/__init__.py:66-68)
 * Every d_* offset is optional (NULL); every output is optional (NULL skips the field).  Outputs must not alias inputs.
 * F is unrestricted here (>= 0).  mgs_activate_backward takes dL/d(activated arrays) -- typically the sums over all
 * views that mgs_backward accumulated -- recomputes the forward from the raw inputs and writes dL/d(raw) and, where
 * asked, the same values as dL/d(offset).  NULL g_* skips a field; NULL outputs are not written.
 */
int mgs_activate(int P, int F,
	const float* means, const float* d_means, const float* rot, const float* d_rot,
	const float* scales, const float* d_scales, const float* opac, const float* feature,
	int scale_mode, float scale_max, int opacity_mode, int rot_normalize, int feature_normalize,
	float* out_means, float* out_rot, float* out_scales, float* out_opac, float* out_feature,
	void* stream);
int mgs_activate_backward(int P, int F,
	const float* means, const float* d_means, const float* rot, const float* d_rot,
	const float* scales, const float* d_scales, const float* opac, const float* feature,
	int scale_mode, float scale_max, int opacity_mode, int rot_normalize, int feature_normalize,
	const float* g_means, const float* g_rot, const float* g_scales, const float* g_opac, const float* g_feature,
	float* dL_dmeans, float* dL_dd_means, float* dL_drot, float* dL_dd_rot,
	float* dL_dscales, float* dL_dd_scales, float* dL_dopac, float* dL_dfeature,
	void* stream);

/*
 * Test/diagnostic access to the opaque state (used by the parity tests to compare stage by stage with the
 * reference's GeometryState / BinningState / ImageState, rasterizer_impl.h:29-65).  Each call writes the
 * device address of the named array inside the given state buffer; names:
 *   geometry: "depths" f32[P], "means2D" f32[2P], "cov3D" f32[6P], "conic_opacity" f32[4P], "rgbd" f32[4P] {r,g,b,depth},
 *             "tiles_touched" u32[P], "point_offsets" u32[P] (inclusive sum in depth order), "depth_order" u32[P],
 *             "clamped" u8[P] (3 bits), "extent" f32[2P]
 *   binning : "point_list" u32[R] (== the reference's point_list), "tile_ids" u32[R] (== high word of the reference's
 *             sorted keys; the low word is the depth bits of point_list[i]), "point_list_unsorted" u32[R],
 *             "tile_ids_unsorted" u32[R], "records" 32-byte records [R], "block_bits" u8[R] (bit s = the instance can
 *             reach 8x4 block s of its tile, s = 2 * (y / 4) + x / 8), "block_lists" u32[8][S] with S = (R + 11) & ~3
 *             (row s, entries range.x .. range.x + block_count - 1 of a tile: the 0-based tile-list positions of the
 *             instances with bit s set, in list order), "pixel_masks" u32[8][S] (same rows and slots, per block-list
 *             entry: bit x * 4 + y = the instance contributed to pixel (x, y) of the block; written by the forward blend
 *             only where the backward reads it, other words are undefined)
 *   image   : "final_T" f32[N], "n_contrib" u32[N], "ranges" u32[2T], "tile_order" u32[T] (tiles by descending list length,
 *             ties by tile id: the launch order of the blend CTAs; no reference counterpart), "block_count" u32[8T]
 *             (entries of block s's list of tile t at 8 t + s), "block_nwalk" u32[8T] (block-list entries up to and
 *             including the block's last contributor, written by the forward blend for blocks with a pixel in the image)
 *   scratch : a view's blend_scratch after a backward, P_or_R_or_width = P: "gb" f32[P][12], the blend-stage record of each
 *             Gaussian {dL/dmean2D x, y, dL/dconic a, b | c, dL/dopacity, dL/dcolour r, g | b, dL/ddepth, 0, 0} (dL/dmean2D
 *             with the 0.5 W / 0.5 H factors, dL/dconic b the half-weight off-diagonal term), "gn" f32[P][4] (scratch sized
 *             by mgs_backward_scratch_bytes_normal only: the normal plane's dL/dn {x, y, z, 0}, or planar depth's quad
 *             gradient, or flow's)
 *   visibility_backward : one view's backward scratch of mgs_visibility_views_backward (its dL_dmean2D) after the call,
 *             P_or_R_or_width = P, height = Q: "gb" f32[P][12] (the blend-stage records as in scratch, slots 0..5 written
 *             where the call asks for a cloud or camera gradient), "duv" f32[Q][2] (each point's dL/duv through T, written
 *             where it asks for a point or camera gradient)
 * Returns 0, or MGS_ERR_INVALID_ARG for an unknown name.
 */
int mgs_state_array(const char* which_state, const char* name, char* state, int P_or_R_or_width, int height,
	void** out_ptr);

/*
 * Measurement hooks (no reference counterpart; the reference's own timing code is commented out,
 * forward.cu:416,433-437): when enabled, every stage launch is bracketed by CUDA events on the caller's
 * stream.  mgs_profile_read sums the per-stage durations (ms) and launch counts recorded since the last
 * read into arrays of mgs_profile_num_stages() entries and clears the record.
 */
int mgs_profile_enable(int on);
int mgs_profile_num_stages(void);
const char* mgs_profile_stage_name(int i);
int mgs_profile_read(float* total_ms, int* counts);

#ifdef __cplusplus
}
#endif
#endif /* MGS_RASTERIZER_H */
