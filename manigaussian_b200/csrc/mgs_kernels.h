// Internal launch interface between the C-ABI (api.cu) and the kernels.  Plain structs of raw pointers.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace mgs {

struct InstRec;

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
};

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
	// backward only
	const float* dL_dcolor;      // [3,H,W]
	const float* dL_dfeature;    // [F,H,W] nullable
	const float* dL_ddepth;      // [H,W] nullable
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

}  // namespace mgs
