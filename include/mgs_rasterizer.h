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
 *   Outputs (each fully written; NULL allowed for dL_dconic, dL_dcolor, dL_dcov3D, dL_dsh, dL_dscale, dL_drot):
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

/* The same two loss heads for V images that already sit in device memory (planar color [V,3,N], feature [V,F,N] or NULL,
 * N = H*W): loss_acc [V,2] (zeroed by the call) and the cotangent planes as above, one launch. */
int mgs_loss_heads(int V, int F, int N, const float* color, const float* feature, const float* target_color,
	const float* target_feature, float* cot_color, float* cot_feature, float* loss_acc, void* stream);

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
