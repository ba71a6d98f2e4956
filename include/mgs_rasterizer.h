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
 * mgs_backward_views runs the blend backward of every view on its stream, joins, and runs ONE per-Gaussian chain-rule
 * kernel that sums over the views in registers: outputs are the SUMS over the V views (the packed buffer of the
 * multi-GPU all-reduce can be passed directly), except dL_dmean2D which each view owns ([P,3], shared_mean2D = 0) or
 * which is summed into views[0].dL_dmean2D (shared_mean2D = 1).  Output NULL-ability as in mgs_backward.
 * `stages` splits the call in two so that a multi-GPU caller can start the all-reduce of dL_dfeature -- more than half of
 * the message, final after the blend stage -- while the per-Gaussian stage computes the remaining fields.
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

int mgs_forward_views(
	int V, const mgs_view* views,
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
	int V, const mgs_view* views,
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

int mgs_forward_clouds(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	int D, int M, int F, float scale_modifier, int prefiltered, int debug, void* join_stream);
int mgs_backward_clouds(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	int D, int M, int F, float scale_modifier, int accumulate, int debug, void* join_stream);

/*
 * Alpha plane (no reference counterpart): the pixel's accumulated opacity alpha = 1 - final_T, e.g. for a mask loss or for
 * the expected depth out_depth / alpha (out_depth has no background term and falls to 0 where nothing covers the pixel).
 * The four calls below are the multi-view and multi-cloud calls above with one more argument, `alpha`: one mgs_view_alpha
 * per view (V entries, or view_offsets[B] for clouds), or NULL for none; the calls above are these with alpha == NULL.
 * Forward: out_alpha [H,W] is fully overwritten.  Backward: dL_dpix_alpha [H,W] adds T_final / (1 - a_k) * dL_dalpha to
 * every contributor's dL/da_k (cot_scale does not scale it); a pixel nothing blended into has no alpha gradient.
 * Either pointer may be NULL per view.  mgs_view and mgs_cloud keep their layouts: existing arrays of them stay valid.
 */
typedef struct mgs_view_alpha {
	float* out_alpha;            /* forward output [H,W] = 1 - final_T, or NULL */
	const float* dL_dpix_alpha;  /* backward input [H,W], or NULL */
} mgs_view_alpha;

int mgs_forward_views_alpha(
	int V, const mgs_view* views, const mgs_view_alpha* alpha,
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
int mgs_backward_views_alpha(
	int V, const mgs_view* views, const mgs_view_alpha* alpha,
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
	int stages,
	int debug,
	void* join_stream);
int mgs_forward_clouds_alpha(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, int D, int M, int F, float scale_modifier, int prefiltered, int debug, void* join_stream);
int mgs_backward_clouds_alpha(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, int D, int M, int F, float scale_modifier, int accumulate, int debug, void* join_stream);

/*
 * Depth and mask heads (no reference counterpart; INTEGRATION.md §4): two more loss heads beside the fused colour and
 * embedding heads of mgs_view, evaluated in the same forward-blend epilogue from the view's depth plane D and alpha plane
 * A = 1 - final_T, so that a step with depth or mask supervision keeps the fused path (no image-sized kernel between the
 * forward and the backward, no host synchronisation).  Per view, N = H*W:
 *   depth  valid = (target_depth > 0) && (A > 0.5), d = D / A, n = sum valid:  loss_depth = sum_valid |d - target_depth| / n
 *          (0 when n = 0);
 *   mask   loss_mask = mean_px BCE(clamp(A, 1e-4, 1 - 1e-4), target_mask) as torch.nn.functional.binary_cross_entropy.
 * The calls below are the _alpha calls with one more argument, `depth_mask`: one mgs_view_depth_mask per view (V entries,
 * or view_offsets[B] for clouds), or NULL for none; the _alpha calls are these with depth_mask == NULL.  Pass the same
 * array to the forward and the backward.  A view whose two targets are NULL has no depth or mask head.
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

int mgs_forward_views_depth_mask(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask,
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
int mgs_backward_views_depth_mask(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask,
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
	int stages,
	int debug,
	void* join_stream);
int mgs_forward_clouds_depth_mask(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int D, int M, int F, float scale_modifier, int prefiltered,
	int debug, void* join_stream);
int mgs_backward_clouds_depth_mask(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int D, int M, int F, float scale_modifier, int accumulate,
	int debug, void* join_stream);

/*
 * Anti-aliased projection (Mip-Splatting's "2D filter"; the `antialiasing` setting of the 3DGS authors' current rasterizer,
 * gsplat's rasterize_mode="antialiased"; INTEGRATION.md §5).  The projection dilates every screen-space covariance by
 * 0.3 px^2 (Sigma' = Sigma + 0.3 I, as the reference does); with antialiasing = 1 it also scales the Gaussian's opacity by
 *   s = sqrt(max(2.5e-5, det Sigma / det Sigma'))
 * so that the dilated splat carries the energy of the undilated one: the blend sees o_eff = o s.  The conic, radius, screen
 * mean, depth, tiles, instance count and sort keys are those of antialiasing = 0, bit for bit.  The backward chains dL/do_eff
 * to dL/do and, through s, to the covariance (and so to means, scales, rotations or cov3D).
 * The calls below are the _depth_mask calls with one more argument, `antialiasing` (0 or 1); the _depth_mask calls are these
 * with 0.  Pass the same value to the forward and the backward: the backward reads o_eff back from the forward's geometry
 * state.  Any other value returns MGS_ERR_INVALID_ARG before anything is enqueued.
 */
int mgs_forward_views_aa(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
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
int mgs_backward_views_aa(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
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
	int stages,
	int debug,
	void* join_stream);
int mgs_forward_clouds_aa(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, int D, int M, int F, float scale_modifier,
	int prefiltered, int debug, void* join_stream);
int mgs_backward_clouds_aa(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, int D, int M, int F, float scale_modifier,
	int accumulate, int debug, void* join_stream);

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
 * The calls below are the _aa calls with one more argument, `ssim`: one mgs_view_ssim per view (V entries, or view_offsets[B]
 * for clouds), or NULL for none; the _aa calls are these with ssim == NULL.  Every entry of a non-NULL array is an SSIM head.
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

int mgs_forward_views_ssim(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim,
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
int mgs_backward_views_ssim(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim,
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
	int stages,
	int debug,
	void* join_stream);
int mgs_forward_clouds_ssim(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim, int D, int M,
	int F, float scale_modifier, int prefiltered, int debug, void* join_stream);
int mgs_backward_clouds_ssim(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim, int D, int M,
	int F, float scale_modifier, int accumulate, int debug, void* join_stream);

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
