// Internal launch interface between the C-ABI (api.cu) and the kernels.  Plain structs of raw pointers.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

#include "distortion.cuh"
#include "fisheye.cuh"

namespace mgs {

struct InstRec;

// A view's camera model, beside its pose and field of view (include/mgs_rasterizer.h: the ortho flags, mgs_view_fisheye and
// mgs_view_distortion).  Pinhole and orthographic views take their screen mean through the projection matrix (an
// orthographic view's tan_fov holds its half extents); fisheye (Kannala-Brandt, fisheye.cuh) and distorted-pinhole (OpenCV,
// distortion.cuh) views form it from (cx, cy) and their coefficients without it, and cull a mean past theta_max or r2_max.
// camera.cuh holds the device maths of each model.
constexpr int MODEL_PINHOLE = 0, MODEL_ORTHO = 1, MODEL_FISHEYE = 2, MODEL_DISTORTED = 3;
struct Lens {
	int model;                   // MODEL_*
	float cx, cy;                // fisheye or distorted principal point
	float theta_max;             // fisheye cull
	float r2_max;                // distorted cull: r_max^2
	FisheyeK fe_k;
	DistK dc_k;
};

struct ProjectFwdArgs {
	int P, D, M;
	const float* means3D;
	const float* scales;
	float scale_modifier;
	const float* rotations;
	const float* opacities;
	const float* shs;
	const float* cov3D_precomp;
	const float* colors_precomp;
	const float* viewmatrix;
	const float* projmatrix;
	const float* cam_pos;
	int W, H;
	float tan_fovx, tan_fovy, focal_x, focal_y;
	uint32_t grid_x, grid_y;
	// outputs
	int* radii;
	float2* means2D;
	float* depths;
	float* cov3D;
	float4* rgbd;  // {r, g, b, view-space depth} per Gaussian: the first quad of the blend channel row
	float4* conic_opacity;
	float2* extent;
	uint8_t* clamped;  // 3 bits per Gaussian
	uint32_t* tiles_touched;
	uint32_t* iota;    // identity permutation (values of the depth sort)
	// device {tan_fovx, tan_fovy}, or NULL: tan_fov* and focal_* above.  Non-NULL picks the instantiation that reads it and
	// forms the focal lengths as the host does (W / (2 tan_fovx)).
	const float* tan_fov;
	int antialias;     // 1: opacity compensation for the 0.3 px^2 low-pass (picks the AA instantiation)
	// the view's camera model (picks the MODEL instantiation).  It starts 4 bytes past an 8-byte boundary, as in FlowCam: the
	// pairs the kernel reads together ((cx, cy) and the coefficients) then sit on 8-byte boundaries, and are loaded as such.
	Lens lens;
};

// project_bwd.cu: per-Gaussian chain rule for up to MAX_BWD_VIEWS views in one launch
constexpr int MAX_BWD_VIEWS = 16;
struct ProjectBwdView {
	const int* radii;          // [P] of this view
	const float* gb;           // [P, GB_STRIDE] blend-stage gradients of this view
	const uint8_t* clamped;    // [P] SH clamp bits of this view (nullable without SHs)
	const float* viewmatrix;
	const float* projmatrix;
	const float* cam_pos;
	float* dL_dmean2D;         // [P,3] of this view (nullable); with shared_mean2D only view 0's is used and receives the sum
	float tan_fovx, tan_fovy, focal_x, focal_y;
};
// a view's device field of view: {tan_fovx, tan_fovy} read in the kernel, or NULL for the ProjectBwdView's host values; W, H
// the image size the focal lengths are formed from (fx = W / (2 tan_fovx), as on the host); rows: the view's focal-length
// rows [CTAs of the launch][CAM_INTR_TERMS] (in its geometry state), or NULL
struct ProjectBwdIntr {
	const float* tan_fov;
	int W, H;
	float* rows;
};
struct ProjectBwdViewsArgs {
	int P, D, M, V;
	const float* means3D;
	const float* shs;            // nullable (precomputed colours)
	const float* scales;         // nullable (precomputed covariance)
	const float* rotations;
	float scale_modifier;
	const float* cov3D_precomp;  // used when scales is null
	int accumulate;              // 0: every output row is written; 1: added to what the row holds (caller serialises writers)
	int shared_mean2D;
	float* dL_dmean3D;  // [P,3]
	float* dL_dopacity; // [P]
	float* dL_dcolor;   // [P,3] nullable
	float* dL_dcov3D;   // [P,6] nullable
	float* dL_dsh;      // [P,M,3] nullable
	float* dL_dscale;   // [P,3] nullable
	float* dL_drot;     // [P,4] nullable
	float* dL_dconic;   // [P,4] nullable; view 0 only (single-view callers)
	ProjectBwdView view[MAX_BWD_VIEWS];
	// anti-aliased mode only (the launcher picks the instantiation): view u's conic_opacity [P] from its geometry state, whose
	// .w is the compensated opacity o_eff the blend saw.  Kept out of ProjectBwdView and behind every other member so that the
	// AA = false kernels read their parameters at the same offsets and strides as before the mode existed.
	int antialias;
	const float4* conic_opacity[MAX_BWD_VIEWS];
	// camera gradients (the launcher picks the CAM instantiation when any is set): view u's rows [CTAs of the launch][CAM_TERMS],
	// one per CTA, or NULL.  Behind every other member for the same reason as conic_opacity.
	float* cam_rows[MAX_BWD_VIEWS];
	// device fields of view (the CAM instantiation reads them; the launcher picks it when any is set): behind cam_rows
	ProjectBwdIntr intr[MAX_BWD_VIEWS];
	// bit u: view u is orthographic.  Only the ORTHO instantiations (of CAM) read it; the launcher picks them when any bit is
	// set.  Behind intr for the same reason as conic_opacity.
	uint16_t ortho;
	// bit u: view u is a fisheye view with coefficients fe_k[u].  Only the FISHEYE instantiations (of ORTHO and CAM: they serve
	// all three models) read them; the launcher picks them when any bit is set.  Behind ortho for the same reason.
	uint16_t fisheye;
	FisheyeK fe_k[MAX_BWD_VIEWS];
	// bit u: view u is a distorted-pinhole view with coefficients dc_k[u].  Only the DIST instantiations (of FISH, ORTHO and
	// CAM: they serve all four models) read them; the launcher picks them when any bit is set.  Behind fe_k for the same reason.
	uint16_t distorted;
	DistK dc_k[MAX_BWD_VIEWS];
	// planar depth: view u's blend-stage quad gradients pl_g [P] ({dL/da, dL/db, dL/de, 0}), its forward quads pl_q [P]
	// ({a, b, e, 0}, planar.cu) and its screen means pl_mean [P] (pixels), or NULL where the view has none.  Only the planar
	// kernels (project_bwd_{views,clouds}_planar_kernel: the DIST body, all four models) read them; the launcher picks them when
	// any is set.  Behind dc_k for the same reason as conic_opacity.
	const float4* pl_g[MAX_BWD_VIEWS];
	const float4* pl_q[MAX_BWD_VIEWS];
	const float2* pl_mean[MAX_BWD_VIEWS];
};
// the 27 camera terms one CTA writes per view into its camera rows: dL/dvm[4c + r] at 3c + r (c < 4, r < 3), dL/dpm[4c + {0, 1,
// 3}] at 12 + 3c + {0, 1, 2}, dL/dcampos at 24 + i.  The other 8 of the 35 outputs are constants of the forward.  The kernel
// forms CAM_ALL_TERMS: terms 27 + i, dL/dtan_fov, go to the view's focal-length rows (ProjectBwdIntr::rows), so the camera
// rows keep their width and mgs_camera_grad_scratch_bytes its value.
constexpr int CAM_TERMS = 27;
constexpr int CAM_INTR_TERMS = 2;
constexpr int CAM_ALL_TERMS = CAM_TERMS + CAM_INTR_TERMS;
// the same chain rule for several clouds in one launch: cloud c sums views view[view0 .. view0 + V) of the launch
// (every cloud has a view, so MAX_BWD_VIEWS clouds at most); dL_dmean2D per view only, no dL_dconic
struct ProjectBwdCloud {
	int P, V, view0;
	int block0;                  // first CTA of the cloud, set by the launcher
	const float* means3D;
	const float* shs;            // nullable (precomputed colours)
	const float* scales;         // nullable (precomputed covariance)
	const float* rotations;
	const float* cov3D_precomp;  // used when scales is null
	int accumulate;
	float* dL_dmean3D; float* dL_dopacity; float* dL_dcolor; float* dL_dcov3D; float* dL_dsh; float* dL_dscale; float* dL_drot;
};
struct ProjectBwdCloudsArgs {
	int D, M, B;  // SH degree and coefficients of every cloud, B clouds
	float scale_modifier;
	ProjectBwdCloud cloud[MAX_BWD_VIEWS];
	ProjectBwdView view[MAX_BWD_VIEWS];
	int antialias;                                 // as in ProjectBwdViewsArgs
	const float4* conic_opacity[MAX_BWD_VIEWS];    // per view of the launch, AA only
	float* cam_rows[MAX_BWD_VIEWS];                // per view of the launch: [CTAs of its cloud][CAM_TERMS], or NULL
	ProjectBwdIntr intr[MAX_BWD_VIEWS];            // per view of the launch, as in ProjectBwdViewsArgs
	uint16_t ortho;                                // bit u: view u of the launch is orthographic, as in ProjectBwdViewsArgs
	uint16_t fisheye;                              // bit u: view u of the launch is a fisheye view, as in ProjectBwdViewsArgs
	FisheyeK fe_k[MAX_BWD_VIEWS];                  // per view of the launch, as in ProjectBwdViewsArgs
};
// the clouds launch with distorted-pinhole views: the DIST instantiations take this larger block (CUDA 12.1+ on Volta and
// later accept kernel parameters up to 32,764 bytes), so every other clouds kernel keeps its parameter block under 4 KB
struct ProjectBwdCloudsDistArgs : ProjectBwdCloudsArgs {
	uint16_t distorted;                            // bit u: view u of the launch is a distorted-pinhole view
	DistK dc_k[MAX_BWD_VIEWS];                     // per view of the launch, as in ProjectBwdViewsArgs
	const float4* pl_g[MAX_BWD_VIEWS];             // per view of the launch, as in ProjectBwdViewsArgs (PLN only)
	const float4* pl_q[MAX_BWD_VIEWS];
	const float2* pl_mean[MAX_BWD_VIEWS];
};
static_assert(MAX_BWD_VIEWS <= 16, "the orthographic, fisheye and distorted view masks have 16 bits");
static_assert(sizeof(ProjectBwdViewsArgs) <= 4096, "kernel parameters are limited to 4 KB");
static_assert(sizeof(ProjectBwdCloudsArgs) <= 4096, "kernel parameters are limited to 4 KB");
static_assert(sizeof(ProjectBwdCloudsDistArgs) <= 32764, "large kernel parameters are limited to 32,764 bytes");
// the second half of the camera gradients: view u's rows summed in row order into its 35 outputs (each nullable), written
// (accumulate = 0) or added (1)
struct CamReduceView {
	const float* rows;
	int nrows;
	float* dL_dviewmatrix;  // 16
	float* dL_dprojmatrix;  // 16
	float* dL_dcampos;      // 3
	const float* intr_rows; // [nrows][CAM_INTR_TERMS] focal-length rows, or NULL
	float* dL_dtan_fov;     // 2
};
struct CamReduceArgs {
	int V, accumulate;
	CamReduceView view[MAX_BWD_VIEWS];
};
inline size_t camera_rows_bytes(int P) { return (size_t)((P + 127) / 128) * CAM_TERMS * sizeof(float); }
inline size_t camera_intr_rows(int P) { return (size_t)((P + 127) / 128) * CAM_INTR_TERMS; }  // floats, in the geometry state

struct BlendArgs {
	int W, H;
	int grid_x, grid_y;
	int F;                       // user feature channels (0 = none): also the row stride of feature / dL_dfeat
	// Channel groups: G = ceil(F / 32) (1 when F <= 32); group g blends channels [32 g, min(F, 32 g + 32)).  Every group
	// walks the same tile list; CTA index = (tile rank, group, 8x4 block), the group varying faster than the rank.
	int groups;
	const uint2* ranges;         // [T]
	const uint32_t* tile_order;  // [T] launch order of the tiles (tile rank i works on tile tile_order[i]); null = identity
	const uint32_t* point_list;  // [R] sorted Gaussian ids
	const InstRec* recs;         // [R] sorted packed records
	const uint32_t* block_list;  // [8][mask_stride] per 8x4 block of the tile: 0-based list positions of the instances that can reach it
	const uint32_t* block_count; // [8T] entries of each block's list
	const float4* rgbd;          // [P] {r,g,b,depth}
	const float* feature;        // [P,F] or null
	const float* bg;             // [3]
	int want_depth;
	// forward outputs / backward inputs
	float* final_T;              // [N]
	uint32_t* n_contrib;         // [N]
	uint32_t* pix_mask;          // [8][mask_stride] per block-list entry: bit p = the pair contributed to pixel p of the block
	size_t mask_stride;          // a multiple of 4: every row starts 16-byte aligned
	uint32_t* block_nwalk;       // [8T] block-list entries up to and including the block's last contributor
	float* out_color;            // [3,H,W]
	float* out_feature;          // [F,H,W]
	float* out_depth;            // [H,W] nullable
	float* out_alpha;            // [H,W] nullable: accumulated opacity 1 - final_T
	// backward only
	const float* dL_dcolor;      // [3,H,W]
	const float* dL_dfeature;    // [F,H,W] nullable
	const float* dL_ddepth;      // [H,W] nullable
	const float* dL_dalpha;      // [H,W] nullable: cotangent of out_alpha, enters the background term only
	float* gb;                   // [P,GB_STRIDE] (zeroed by caller)
	float* dL_dfeat;             // [P,F] (zeroed by caller) nullable
	// fused loss heads (loss_heads.cuh), all nullable.  Forward: with tgt_color the epilogue also writes the cotangent planes
	// cot_color [3,H,W] (and, with tgt_feature, cot_feature [F,H,W]) and adds {sum (x-g)^2, sum_px cos} into loss_acc[0..1].
	// tgt_feature only with groups == 1: the cosine needs a pixel's whole feature vector, which one CTA then holds.
	// Backward: cot_scale[0..1] (device) multiply the colour / feature cotangent planes on load (the upstream gradients of
	// the two scalar losses).
	const float* tgt_color;
	const float* tgt_feature;
	float* cot_color;
	float* cot_feature;
	float* loss_acc;
	const float* cot_scale;
	// depth and mask heads (loss_heads.cuh), with the colour head only, all nullable.  Forward: tgt_depth [H,W] writes cot_depth and
	// cot_alpha_depth, tgt_mask [H,W] writes cot_alpha_mask (all [H,W], unscaled), and {sum |d - g|, n, sum BCE} are added into
	// dm_acc[0..2].  Backward: with tgt_depth the depth cotangent is dm_scale[0] / max(dm_acc[1], 1) * cot_depth and the alpha
	// cotangent gains the same scale times cot_alpha_depth; with tgt_mask it gains dm_scale[1] * cot_alpha_mask (dm_scale NULL: 1).
	const float* tgt_depth;
	const float* tgt_mask;
	float* cot_depth;
	float* cot_alpha_depth;
	float* cot_alpha_mask;
	float* dm_acc;
	const float* dm_scale;
	// median depth (forward, nullable; the launcher picks the MED instantiation when median_id is set): median_id [H,W]
	// receives the id of the pixel's median contributor, the last one whose incoming T > 0.5 (-1 without a contributor), and
	// out_median_depth [H,W] (nullable) its view-space depth rgbd[id].w (0 without).  Behind every other member, so that the
	// blend kernels without it read their parameters at the same offsets as before.
	int* median_id;
	float* out_median_depth;
	// normal plane (nullable; the launchers pick the NRM instantiations when nrm is set): nrm [P] is the view's per-Gaussian
	// quad {nx, ny, nz, 0} (normals.cu), blended in columns 4..6 of the {r,g,b,depth} tile.  Forward: out_normal [3,H,W].
	// Backward: dL_dnormal [3,H,W] is its cotangent, and gn [P,4] (zeroed by the caller) receives dL/dn.  Behind
	// out_median_depth for the same reason.
	const float4* nrm;
	float* out_normal;
	const float* dL_dnormal;
	float* gn;
	// planar depth (the launchers pick the PLN instantiations when set): nrm holds the view's planar quads {a, b, e, 0}
	// (planar.cu) instead, and the depth plane, the depth / mask heads and the median depth take each Gaussian's depth
	// z + a px + b py + e at pixel (px, py).  Backward: gn receives {dL/da, dL/db, dL/de, 0} with e's share folded into dL/da
	// and dL/db (e = -(a mu_x + b mu_y)): {sum w g (px - mu_x), sum w g (py - mu_y), sum w g, 0}, formed in block-local
	// coordinates so that no term grows with the pixel coordinates.  Behind gn for the same reason.
	int planar;
#ifdef MGS_CTA_LOG
	// measurement build only (tools/cta_timeline.py): every blend CTA appends {t0, t1 (globaltimer ns), kind | sub << 8, entries of
	// the block's list (forward) or replayed (backward), SM id, block id} -- the timeline of the blend CTAs across kernels and streams
	unsigned long long* cta_log; unsigned int* cta_log_n; unsigned int cta_log_cap;
#endif
#ifdef MGS_BWD_PHASES
	// measurement build only (tools/bwd_phases.py): the two-warp backward adds its clock64() cycles per phase and its chunk
	// count into bwd_phases[BWD_PH_COUNT] (blend_common.cuh)
	unsigned long long* bwd_phases;
#endif
};
// loss_heads.cu: the same heads for images that already sit in memory (planar [3,H,W] / [F,H,W], V views in one launch).
// color == null: features only -- the embedding head alone, into loss_acc[2 v + 1] (the colour head ran elsewhere).
void launch_loss_heads(int V, int F, int N, const float* color, const float* feature, const float* tgt_color, const float* tgt_feature,
	float* cot_color, float* cot_feature, float* loss_acc, cudaStream_t s);

// ssim.cu: L1 + SSIM of V views of C planes each (x, g [V,C,H,W]).  Forward: terms [V,3,C,H,W] receives the unscaled
// partials of S, acc + v * acc_stride the sums {|x - g|, S} (added).  Backward: cot_out [V,C,H,W] = cot_in_scale[0] * cot_in
// + scale[2v] d l1 / dx + scale[2v+1] d ssim / dx (scale, cot_in, cot_in_scale nullable); blend_slot (nullable, V = 1)
// receives {1, cot_in_scale[1]}.
void launch_ssim_fwd(int V, int C, int H, int W, const float* x, const float* g, float* terms, float* acc, int acc_stride, cudaStream_t s);
void launch_ssim_bwd(int V, int C, int H, int W, const float* x, const float* g, const float* terms, const float* scale,
	const float* cot_in, const float* cot_in_scale, float* cot_out, float* blend_slot, cudaStream_t s);

// activate.cu: view-independent per-Gaussian pre-ops (activations, deformation offsets, feature normalisation)
struct ActivateArgs {
	int P, F;
	const float* means;     // [P,3]
	const float* d_means;   // [P,3] offset added before use, nullable
	const float* rot;       // [P,4]
	const float* d_rot;     // [P,4] nullable
	const float* scales;    // [P,3]
	const float* d_scales;  // [P,3] nullable
	const float* opac;      // [P]
	const float* feature;   // [P,F] nullable
	int scale_mode;         // 0 identity, 1 min(exp(x), scale_max)
	float scale_max;
	int opacity_mode;       // 0 identity, 1 sigmoid
	int rot_normalize;      // x / max(||x||, 1e-12)
	int feature_normalize;  // x / (||x|| + 1e-12)
	// forward outputs (a null output skips that field)
	float *o_means, *o_rot, *o_scales, *o_opac, *o_feature;
	// backward inputs: gradients w.r.t. the activated arrays (a null input skips that field)
	const float *g_means, *g_rot, *g_scales, *g_opac, *g_feature;
	// backward outputs: gradients w.r.t. the raw arrays and (same values) the offsets; each nullable
	float *dL_means, *dL_dmeans, *dL_rot, *dL_drot, *dL_scales, *dL_dscales, *dL_opac, *dL_feature;
	// filled by the launcher
	int small_blocks, feature_group, feature_group4, feature_vec4;
};
void launch_activate_fwd(ActivateArgs a, cudaStream_t s);
void launch_activate_bwd(ActivateArgs a, cudaStream_t s);

void launch_project_fwd(const ProjectFwdArgs& a, cudaStream_t s);
void launch_project_bwd_views(const ProjectBwdViewsArgs& a, cudaStream_t s);
void launch_project_bwd_clouds(ProjectBwdCloudsDistArgs a, cudaStream_t s);
void launch_camera_grad_reduce(const CamReduceArgs& a, cudaStream_t s);
void launch_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present, cudaStream_t s);

// binning.cu
size_t scan_temp_bytes(int P);
size_t depth_sort_temp_bytes(int P);
size_t tile_sort_temp_bytes(int R);
void launch_depth_sort(void* temp, size_t temp_bytes, const uint32_t* depth_bits, uint32_t* depth_bits_sorted,
	const uint32_t* iota, uint32_t* order, int P, cudaStream_t s);
void launch_scan_sorted(void* temp, size_t temp_bytes, const uint32_t* order, const uint32_t* tiles_touched, uint32_t* offsets,
	int P, cudaStream_t s);
// capacity: size of the instance arrays; instances beyond it are dropped and *overflow (device, nullable) is set
void launch_emit_tiles(int P, const uint32_t* order, const float2* means2D, const uint32_t* offsets, const int* radii,
	uint32_t grid_x, uint32_t grid_y, uint32_t* tile_keys, uint32_t* values, uint32_t capacity, int* status, cudaStream_t s);
// instance slots [R, capacity) get the last tile id and an invalid Gaussian id: a stable sort of all `capacity` slots
// leaves them behind the R real instances (R = offsets[P-1] on the device)
void launch_fill_tail(const uint32_t* offsets, int P, uint32_t capacity, uint32_t last_tile, uint32_t* tile_keys, uint32_t* values, cudaStream_t s);
void launch_tile_sort(void* temp, size_t temp_bytes, const uint32_t* keys_in, uint32_t* keys_out,
	const uint32_t* vals_in, uint32_t* vals_out, int R, int end_bit, cudaStream_t s);
void launch_tile_order(const uint2* ranges, int num_tiles, uint32_t* order, cudaStream_t s);
// the instance count is read on the device from *R_dev (clamped to `capacity`), the grid covers `capacity`
void launch_ranges_and_pack(const uint32_t* R_dev, int capacity, int num_tiles, int grid_x, const uint32_t* tile_keys, const uint32_t* point_list,
	const float2* means2D, const float4* conic_opacity, const float2* extent, uint2* ranges, InstRec* recs, uint8_t* block_bits,
	uint32_t* tile_order, cudaStream_t s);
// per (tile, 8x4 block): the 0-based tile-list positions of the instances whose block bit is set, in list order, into row s
// of block_list ([8][stride], entries at range.x + k), and their number into block_count[8 tile + s]
void launch_block_lists(const uint2* ranges, int num_tiles, const uint8_t* block_bits, uint32_t* block_list, size_t stride,
	uint32_t* block_count, cudaStream_t s);

// blend_fwd.cu / blend_bwd.cu
int blend_supported(int F);
int blend_groups(int F);  // channel groups of 32 (BlendArgs::groups)
void launch_blend_fwd(const BlendArgs& a, cudaStream_t s);
void launch_blend_bwd(const BlendArgs& a, cudaStream_t s);
// the median depth's backward: gb[median_id[p] * GB_STRIDE + 9] += dL_dmedian[p] for every pixel p with median_id[p] >= 0;
// with gn (planar depth, W the image width, means2D the view's screen means) also gn[median_id[p]] += dL_dmedian[p]
// {px - mu_x, py - mu_y, 1, 0} (gn's mean-relative form, BlendArgs::planar)
void launch_median_depth_bwd(int N, const int* median_id, const float* dL_dmedian, float* gb, cudaStream_t s, int W = 0,
	float* gn = nullptr, const float2* means2D = nullptr);

// lift.cu: lifted[id][c] += sum_p w_p,id map[c][p] and weight[id] += sum_p w_p,id over one view's pixels, w = alpha T the
// forward blend's weights (include/mgs_rasterizer.h, mgs_lift_views).  The tile grid, lists and records are the view's, as
// in BlendArgs; nothing of the view's state is written.
struct LiftArgs {
	int W, H;
	int grid_x, grid_y;
	int C;                       // map channels (0 = weights only): also the row stride of lifted
	int groups;                  // channel groups of 32 (blend_groups(C)), indexed as in BlendArgs
	const uint2* ranges;         // [T]
	const uint32_t* tile_order;  // [T] or null
	const InstRec* recs;         // [R]
	const uint32_t* block_list;  // [8][mask_stride]
	const uint32_t* block_count; // [8T]
	size_t mask_stride;
	const float* map;            // [C,H,W] or null (C = 0)
	float* lifted;               // [P,C] (zeroed by the caller) or null (C = 0)
	float* weight;               // [P] (zeroed by the caller)
};
void launch_lift(const LiftArgs& a, cudaStream_t s);

// normals.cu: nrm[i] = {s a, 0}, a the world-space direction of Gaussian i's shortest axis (unit, from the normalised
// quaternion), s = +-1 so that it faces cam_pos
void launch_normals_fwd(int P, const float* means3D, const float* scales, const float* rotations, const float* cam_pos, float4* nrm,
	cudaStream_t s);
// dL_drot[i] += the chain of sum_v s_{i,v} gn[v][i] through the axis and the quaternion's normalisation, for the V views of
// one launch (gn[v]: view v's [P,4] blend-stage normal gradients, cam_pos[v] its camera centre)
struct NormalsBwdArgs {
	int P, V;
	const float* means3D;
	const float* scales;
	const float* rotations;
	float* dL_drot;  // [P,4]
	const float* gn[MAX_BWD_VIEWS];
	const float* cam_pos[MAX_BWD_VIEWS];
};
void launch_normals_bwd(const NormalsBwdArgs& a, cudaStream_t s);

// planar.cu: quad[i] = {a, b, e, 0} of Gaussian i in one view (include/mgs_rasterizer.h, planar depth): (a, b) = k Q with
// k = e3^T Sigma_c J^T and Q the conic of the projection's record, e = -(a mu_x + b mu_y); zeros where radii[i] == 0
struct PlanarFwdArgs {
	int P;
	const float* means3D;
	const float* cov3D;          // [P,6] world-space covariance: the caller's, or the projection's own
	const float* viewmatrix;
	int W, H;
	float tan_fovx, tan_fovy;    // host field of view (tan_fov NULL)
	const float* tan_fov;        // device {tan_fovx, tan_fovy}, or NULL
	Lens lens;
	const int* radii;
	const float2* means2D;
	const float4* conic_opacity;
	float4* quad;
};
void launch_planar_fwd(const PlanarFwdArgs& a, cudaStream_t s);

// field.cu: density and features of the Gaussian field at 3D points (include/mgs_rasterizer.h, mgs_field_query).  The query
// state (field_state_bytes) holds the grid, the records, the grouped queries and the warp items; the pair state
// (field_pair_state_bytes of the pair count field_front returns) the bin lists.  The backward reads both as the forward left
// them.
struct FieldGrid {
	float lo[3];   // corner of the queries' bounding box
	float inv[3];  // bins per unit length along each axis (0 on an axis of zero extent)
	int n[3];      // bins along each axis
};
struct FieldArgs {
	int Q, P, C, groups, channel_first;
	const float* points;          // [Q,3]
	const float* features;        // [P,C] or null
	const float* scales;          // [P,3] (backward)
	const float* rotations;       // [P,4] (backward)
	const float4* recs;           // [P][4] records {A_k, mu_k}_k, {o, 0, 0, 0}
	const float4* ext;            // [P] support half-extent, w = 1 for a Gaussian with support
	const uint32_t* pairs;        // Gaussian ids sorted by bin, ascending within a bin
	const uint2* gbin;            // [bins] range of each bin's Gaussians in pairs
	const uint32_t* qorder;       // query ids sorted by bin
	const uint4* items;           // warp items {first, end (in qorder), bin, 0}
	const int* nitems;            // item count
	float* density;               // [Q]
	float* out_features;          // [Q,C] or [C,Q] (channel_first)
	const float* dL_ddensity;     // [Q] or null
	const float* dL_dfeatures;    // as out_features, or null
	float* dL_dpoints;            // [Q,3] or null
	float4* ggeo;                 // [P][4] per-Gaussian record gradients (zeroed), or null
	float* dL_dfeat;              // [P,C] (zeroed) or null
	float* dL_dmeans; float* dL_dscales; float* dL_drot; float* dL_dopac;  // each [P,k] or null
};
int field_bins(int Q);
size_t field_state_bytes(int Q, int P);
size_t field_pair_state_bytes(long long npairs, int Q);
// enqueues the grid, the records, the query grouping and the scan of the per-Gaussian bin counts, and copies the pair count
// to *host_pairs (the caller synchronises before reading it)
cudaError_t field_front(char* state, int Q, int P, const float* points, const float* means, const float* scales, const float* rot,
	const float* opac, unsigned long long* host_pairs, cudaStream_t st);
cudaError_t field_pairs(char* state, char* pair_state, int Q, int P, long long npairs, cudaStream_t st);
cudaError_t field_forward(char* state, char* pair_state, int Q, int P, int C, const float* points, const float* features,
	int channel_first, float* density, float* out_features, cudaStream_t st);
cudaError_t field_backward(char* state, char* pair_state, int Q, int P, int C, const float* points, const float* features,
	const float* scales, const float* rotations, int channel_first, const float* dL_ddensity, const float* dL_dfeatures,
	float* dL_dpoints, float* dL_dmeans, float* dL_dscales, float* dL_drot, float* dL_dopac, float* dL_dfeat, cudaStream_t st);
// the field's front-end kernels that knn.cu runs as well (launched with 256 threads per CTA):
//   field_bbox_kernel       box[0..2] = min, box[3..5] = max of the finite points' fkey (box preset to ~0 / 0);
//   field_ranges_kernel     range[key] = [first, last + 1) of each run of equal sorted keys (range zeroed by the caller);
//   field_warp_count_kernel wcnt[b] = warps of 32 over range b;
//   field_items_kernel      items[woff[b] - wcnt[b] + w] = {first, end, b, 0} of warp w of range b (woff the inclusive scan
//                           of wcnt), *nitems = woff[nb - 1].
__global__ void __launch_bounds__(256) field_bbox_kernel(int Q, const float* __restrict__ pts, uint32_t* __restrict__ box);
__global__ void __launch_bounds__(256) field_ranges_kernel(int n, const uint32_t* __restrict__ keys, uint2* __restrict__ range);
__global__ void __launch_bounds__(256) field_warp_count_kernel(int nb, const uint2* __restrict__ qrange, uint32_t* __restrict__ wcnt);
__global__ void __launch_bounds__(256) field_items_kernel(int nb, const uint2* __restrict__ qrange, const uint32_t* __restrict__ wcnt,
	const uint32_t* __restrict__ woff, uint4* __restrict__ items, int* __restrict__ nitems);

// knn.cu: the k nearest of N points to each of Q queries (include/mgs_rasterizer.h, mgs_knn); queries NULL: the points
// themselves, each without its own index.  The state (knn_state_bytes) holds the grid, the sorted points and queries and the
// warp items; nothing is read back to the host.  Both functions size the state for the current device.
constexpr int KNN_MAX_K = 32;
cudaError_t knn_state_bytes(int N, int Q, size_t* bytes);
cudaError_t knn_run(char* state, int N, int Q, int k, const float* points, const float* queries, long long* out_index,
	float* out_dist2, cudaStream_t st);

// flow.cu: the flow plane's per-Gaussian quads {dx, dy, 0, 0} (include/mgs_rasterizer.h, flow plane) and their backward.
// FlowCam: the map of one end of a view's flow, the view's pose, field of view and image size with its lens.
struct FlowCam {
	const float* viewmatrix;
	const float* projmatrix;     // pinhole and orthographic only
	const float* tan_fov;        // device {tan_fovx, tan_fovy}, or NULL for the host values
	float tan_fovx, tan_fovy;
	int W, H;
	Lens lens;
};
struct FlowFwdArgs {
	int P;
	const float* means3D;
	const float* next_means3D;
	FlowCam cur, next;           // the view's camera, and the one its next-frame means are projected with
	const int* radii;
	float4* quad;
};
void launch_flow_fwd(const FlowFwdArgs& a, cudaStream_t s);
// the backward runs behind the blend backward and ahead of the per-Gaussian stage, on the same stream, for up to
// MAX_BWD_VIEWS views of one cloud; CTAs of FLOW_BWD_THREADS, so its camera rows have the per-Gaussian stage's row count
constexpr int FLOW_BWD_THREADS = 128;
struct FlowBwdView {
	FlowCam cam;                 // the camera of the view's next-frame means
	int own_camera;              // 1: cam is the view's own camera (no next pose), whose gradients take the m' terms
	const int* radii;
	const float4* gn;            // [P] blend-stage quad gradients, or NULL (the view has no flow cotangent)
	float* gb;                   // [P, GB_STRIDE] blend-stage records: the screen-mean slots receive -gn
	float* cam_rows;             // [CTAs][CAM_TERMS] camera rows, or NULL
	float* intr_rows;            // [CTAs][CAM_INTR_TERMS] focal-length rows, or NULL
};
struct FlowBwdArgs {
	int P, V;
	const float* next_means3D;
	float* dL_dnext_means3D;     // [P,3] or NULL
	int accumulate;
	FlowBwdView view[MAX_BWD_VIEWS];
};
static_assert(sizeof(FlowBwdArgs) <= 4096, "kernel parameters are limited to 4 KB");
void launch_flow_bwd(const FlowBwdArgs& a, cudaStream_t s);

// visibility.cu: screen position, depth, in_view and transmittance of Q points in one view (include/mgs_rasterizer.h,
// mgs_visibility_views), behind the view's projection and binning.  The points' tile keys are sorted between the points and
// the group launches (launch_tile_sort over keys / idx into keys_sorted / idx_sorted).
struct VisArgs {
	int Q, W, H, grid_x, num_tiles;
	FlowCam cam;                 // the view's own camera
	const float* points;         // [Q,3]
	float* out_uv;               // [Q,2] or NULL
	float* out_depth;            // [Q] or NULL
	uint8_t* out_in_view;        // [Q] or NULL
	float* out_T;                // [Q]
	// scratch
	float4* pt;                  // [Q] {u, v, d, 0}
	uint32_t* keys;              // [Q] tile of each point, num_tiles outside the view
	uint32_t* idx;               // [Q] point ids
	const uint32_t* keys_sorted; // [Q]
	const uint32_t* idx_sorted;  // [Q]
	uint2* qranges;              // [num_tiles] range of each tile's points in the sorted order
	uint32_t* item_end;          // [num_tiles] inclusive scan of the per-tile warp counts
	// the view's projection and binning
	const uint2* ranges;
	const uint32_t* point_list;
	const float* depths;
	const InstRec* recs;
};
void launch_visibility_points(const VisArgs& a, cudaStream_t s);
void launch_visibility_group(const VisArgs& a, cudaStream_t s);
void launch_visibility_query(const VisArgs& a, cudaStream_t s);
// the backward (include/mgs_rasterizer.h, mgs_visibility_views_backward).  The query backward replays one view's query over
// the forward's point scratch (f, with f.out_T the forward's T): per accepted pair the cotangent dL_dT[q] of the point's T goes
// into the Gaussian's blend-stage record (gb, zeroed by the caller, or NULL) and into dL/duv of the point (duv [Q,2], zeroed
// by the caller, or NULL).
struct VisQueryBwdArgs {
	VisArgs f;
	const float* dL_dT;          // [Q]
	float* gb;                   // [P, GB_STRIDE] or NULL
	float* duv;                  // [Q,2] or NULL
};
void launch_visibility_query_bwd(const VisQueryBwdArgs& a, cudaStream_t s);
// the point chain: one thread per point over the launch's views in order, uv's cotangent (dL_duv plus the T path's duv) through
// screen_mean's derivative and depth's through row 2 of the view matrix, where the view's cull passes; camera rows as the
// flow backward's.  CTAs of VIS_PTS_BWD_THREADS.
constexpr int VIS_PTS_BWD_THREADS = 128;
struct VisPointsBwdView {
	FlowCam cam;
	const float* dL_duv;         // [Q,2] or NULL
	const float* dL_ddepth;      // [Q] or NULL
	const float* duv;            // [Q,2] the T path's uv cotangent, or NULL
	float* cam_rows;             // [CTAs][CAM_TERMS] or NULL
	float* intr_rows;            // [CTAs][CAM_INTR_TERMS] or NULL
};
struct VisPointsBwdArgs {
	int Q, V;
	const float* points;
	float* dL_dpoints;           // [Q,3] or NULL
	int accumulate;              // 0: dL_dpoints written, 1: added to
	VisPointsBwdView view[MAX_BWD_VIEWS];
};
static_assert(sizeof(VisPointsBwdArgs) <= 4096, "kernel parameters are limited to 4 KB");
void launch_visibility_points_bwd(const VisPointsBwdArgs& a, cudaStream_t s);

// rays.cu: the ray of each pixel of up to MAX_BWD_VIEWS views per launch (include/mgs_rasterizer.h, mgs_camera_rays), one
// thread per (view, pixel): blockIdx.y is the view of the launch, CTAs of RAYS_THREADS pixels.  Every pointer is that of the
// launch's first view; view u's rays start at u N.
constexpr int RAYS_THREADS = 128;
struct RaysArgs {
	int V, N;                    // views of the launch, rays per view
	int grid_w;                  // pixels NULL: ray i is pixel centre (i % grid_w, i / grid_w)
	const float* pixels;         // [V,N,2] or NULL
	float* origin;               // forward: [V,N,3]
	float* direction;            // forward: [V,N,3]
	uint8_t* valid;              // forward: [V,N]
	const float* dL_dorigin;     // backward: [V,N,3] or NULL
	const float* dL_ddirection;  // backward: [V,N,3] or NULL
	float* dL_dpixels;           // backward: [V,N,2] or NULL
	float* cam_rows[MAX_BWD_VIEWS];   // backward: view u's [CTAs][CAM_TERMS] or NULL (the launcher picks CAM when any is set)
	float* intr_rows[MAX_BWD_VIEWS];  // backward: view u's [CTAs][CAM_INTR_TERMS] or NULL
	FlowCam cam[MAX_BWD_VIEWS];
};
static_assert(sizeof(RaysArgs) <= 4096, "kernel parameters are limited to 4 KB");
void launch_rays_fwd(const RaysArgs& a, cudaStream_t s);
void launch_rays_bwd(const RaysArgs& a, cudaStream_t s);

// neighbour_reg.cu: the dynamic field's local-rigidity, rotation-similarity and isometry terms over [P,k] neighbour lists
// (include/mgs_rasterizer.h, mgs_neighbour_reg).  The state (neighbour_reg_state_bytes, any alignment) holds the per-Gaussian
// records and R_i the forward writes, its CTA partials and the backward's gradient rows; the backward reads the records of
// the forward with the same inputs.  Nothing is read back to the host.
constexpr int NEIGHBOUR_REG_MAX_K = 32;
size_t neighbour_reg_state_bytes(int P);
cudaError_t neighbour_reg_forward(void* state, int P, int k, const float* xyz, const float* rot, const float* xyz_next,
	const float* rot_next, const long long* index, const float* weight, float* out_loss, cudaStream_t st);
cudaError_t neighbour_reg_backward(void* state, int P, int k, const float* rot, const float* rot_next, const long long* index,
	const float* weight, const float* dL_dloss, float* dL_dxyz, float* dL_drot, float* dL_dxyz_next, float* dL_drot_next,
	cudaStream_t st);

}  // namespace mgs
