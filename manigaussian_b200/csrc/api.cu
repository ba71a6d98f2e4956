// C-ABI entry points (include/mgs_rasterizer.h): orchestration of the per-view forward and backward.
//
// Replaces CudaRasterizer::Rasterizer::{forward,backward,markVisible}
// (DGR/cuda_rasterizer/rasterizer_impl.cu:198-355, :359-463, :141-153).  Stage order and the meaning of
// every argument follow the reference; the state-buffer layout, kernels and stream handling are ours.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>
#include "../../include/mgs_rasterizer.h"
#include "mgs_common.cuh"
#include "mgs_kernels.h"

namespace mgs {

static thread_local std::string g_err;
#define MGS_STR_(x) #x
#define MGS_STR(x) MGS_STR_(x)
static const char* const bad_width_msg = "feature channel count must be in [0, " MGS_STR(MGS_MAX_FEATURE_CHANNELS) "]";

static int fail(int code, const std::string& msg)
{
	g_err = msg;
	return code;
}

#define MGS_CUDA(call)                                                                                   \
	do {                                                                                                 \
		cudaError_t e_ = (call);                                                                         \
		if (e_ != cudaSuccess)                                                                           \
			return fail(MGS_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_));               \
	} while (0)

// after each stage: launch errors always, execution errors when debug (the reference's CHECK_CUDA, auxiliary.h:166-173)
static const bool g_trace = getenv("MGS_TRACE") != nullptr;  // diagnostic: name every stage on stderr as it is enqueued
#define MGS_STAGE(name)                                                                                  \
	do {                                                                                                 \
		if (g_trace) { fprintf(stderr, "[mgs] stage %s enqueued\n", name); fflush(stderr); }            \
		cudaError_t e_ = cudaGetLastError();                                                             \
		if (e_ == cudaSuccess && debug) e_ = cudaStreamSynchronize(st);                                  \
		if (e_ != cudaSuccess)                                                                           \
			return fail(MGS_ERR_CUDA, std::string("stage ") + name + ": " + cudaGetErrorString(e_));     \
	} while (0)

// ---- optional per-stage CUDA-event timing (bench.py's roofline leg); off by default, zero cost when off ----
enum Stage { ST_PROJECT_FWD = 0, ST_DEPTH_SORT, ST_SCAN, ST_EMIT, ST_SORT, ST_RANGES_PACK, ST_BLOCK_LISTS, ST_BLEND_FWD, ST_BLEND_BWD, ST_PROJECT_BWD, ST_ACTIVATE_FWD, ST_ACTIVATE_BWD, ST_SSIM_FWD, ST_SSIM_BWD, ST_COUNT };
struct StageEvt { int stage; cudaEvent_t a, b; };
static std::mutex g_prof_mu;
static bool g_prof_on = false;
static std::vector<StageEvt> g_prof_evts;
struct StageTimer {
	cudaStream_t st; bool on; StageEvt e;
	StageTimer(int stage, cudaStream_t s) : st(s), on(g_prof_on)
	{
		if (!on) return;
		e.stage = stage;
		cudaEventCreate(&e.a); cudaEventCreate(&e.b);
		cudaEventRecord(e.a, st);
	}
	~StageTimer()
	{
		if (!on) return;
		cudaEventRecord(e.b, st);
		std::lock_guard<std::mutex> lk(g_prof_mu);
		g_prof_evts.push_back(e);
	}
};

// MGS_TILE_ORDER=0 launches the blend CTAs in tile order instead of longest-list-first (A/B switch for measurements)
static bool use_tile_order()
{
	static const bool on = [] { const char* e = getenv("MGS_TILE_ORDER"); return !(e && e[0] == '0'); }();
	return on;
}

#ifdef MGS_CTA_LOG
static unsigned long long* g_cta_log = nullptr;
static unsigned int* g_cta_log_n = nullptr;
static unsigned int g_cta_log_cap = 0;
extern "C" int mgs_debug_set_cta_log(void* log, void* counter, unsigned int cap)
{
	g_cta_log = static_cast<unsigned long long*>(log); g_cta_log_n = static_cast<unsigned int*>(counter); g_cta_log_cap = cap;
	return 0;
}
#define MGS_CTA_LOG_ARGS(ba) do { (ba).cta_log = g_cta_log; (ba).cta_log_n = g_cta_log_n; (ba).cta_log_cap = g_cta_log_cap; } while (0)
#else
#define MGS_CTA_LOG_ARGS(ba) do { } while (0)
#endif
#ifdef MGS_BWD_PHASES
static unsigned long long* g_bwd_phases = nullptr;
extern "C" int mgs_debug_set_bwd_phases(void* acc)
{
	g_bwd_phases = static_cast<unsigned long long*>(acc);
	return 0;
}
#define MGS_BWD_PHASES_ARGS(ba) do { (ba).bwd_phases = g_bwd_phases; } while (0)
#else
#define MGS_BWD_PHASES_ARGS(ba) do { } while (0)
#endif

template <typename T>
static void obtain(char*& chunk, T*& ptr, size_t count, size_t alignment = 128)
{
	size_t offset = (reinterpret_cast<uintptr_t>(chunk) + alignment - 1) & ~(alignment - 1);
	ptr = reinterpret_cast<T*>(offset);
	chunk = reinterpret_cast<char*>(ptr + count);
}

// CUB temp-storage sizes depend on the item count and the device; the queries are not free (device attribute lookups), so
// cache them.  Sizes are taken for the item count rounded up to the next multiple of 1/8 of its power of two (monotone in
// n, few distinct keys, at most 12.5 % above the exact need).
static size_t cached_temp_bytes(int which, int n)
{
	static std::mutex mu;
	static std::map<std::tuple<int, int, int>, size_t> cache;
	int p2 = 1024;
	while (p2 < n && p2 < (1 << 30)) p2 <<= 1;
	const int q = std::max(128, p2 >> 3);
	const int nb = (int)std::min<long long>(((long long)std::max(n, 1) + q - 1) / q * q, (long long)p2);
	int dev = 0;
	cudaGetDevice(&dev);
	std::lock_guard<std::mutex> lk(mu);
	auto key = std::make_tuple(dev, which, nb);
	auto it = cache.find(key);
	if (it != cache.end()) return it->second;
	const size_t bytes = which == 0 ? std::max(scan_temp_bytes(nb), depth_sort_temp_bytes(nb)) : tile_sort_temp_bytes(nb);
	cache[key] = bytes;
	return bytes;
}

struct GeomState {
	float* depths; uint8_t* clamped; float2* means2D; float* cov3D; float4* conic_opacity; float4* rgbd;
	float2* extent; uint32_t* tiles_touched; uint32_t* point_offsets; uint32_t* iota; uint32_t* order; uint32_t* depth_sorted;
	char* temp; size_t temp_bytes;
	float* cam_intr;  // the backward's focal-length rows of this view (mgs_view_intrinsics.dL_dtan_fov), CAM_INTR_TERMS per CTA
	static GeomState carve(char*& chunk, size_t P)
	{
		GeomState g;
		obtain(chunk, g.depths, P);
		obtain(chunk, g.clamped, P);
		obtain(chunk, g.means2D, P);
		obtain(chunk, g.cov3D, P * 6);
		obtain(chunk, g.conic_opacity, P);
		obtain(chunk, g.rgbd, P);
		obtain(chunk, g.extent, P);
		obtain(chunk, g.tiles_touched, P);
		obtain(chunk, g.point_offsets, P);  // inclusive sum of tiles_touched in DEPTH order
		obtain(chunk, g.iota, P);
		obtain(chunk, g.order, P);          // Gaussian ids sorted by depth bits (stable)
		obtain(chunk, g.depth_sorted, P);
		g.temp_bytes = cached_temp_bytes(0, (int)P);
		obtain(chunk, g.temp, g.temp_bytes);
		obtain(chunk, g.cam_intr, camera_intr_rows((int)P));
		return g;
	}
};
struct ImageState {
	float* final_T; uint32_t* n_contrib; uint2* ranges; int* status; uint32_t* tile_order; uint32_t* block_count; uint32_t* block_nwalk;
	static ImageState carve(char*& chunk, size_t N, size_t T)
	{
		ImageState s;
		obtain(chunk, s.final_T, N);
		obtain(chunk, s.n_contrib, N);
		obtain(chunk, s.ranges, T);
		obtain(chunk, s.status, 4);  // {instance count, overflow flag}, written by the instance emission
		obtain(chunk, s.tile_order, T);
		obtain(chunk, s.block_count, 8 * T);  // entries of each 8x4 block's work list, written by block_lists
		obtain(chunk, s.block_nwalk, 8 * T);  // entries the backward replays, written by the forward blend
		return s;
	}
};
struct BinState {
	uint32_t* point_list; uint32_t* point_list_unsorted; uint32_t* tile_keys; uint32_t* tile_keys_unsorted; InstRec* recs;
	uint32_t* pix_mask; size_t mask_stride; uint32_t* block_list; uint8_t* block_bits;
	char* sort_temp; size_t sort_bytes;
	static BinState carve(char*& chunk, size_t R)
	{
		BinState b;
		const size_t Rp = R + 8;
		obtain(chunk, b.point_list, Rp);           // Gaussian ids in (tile, depth) order == the reference's point_list
		obtain(chunk, b.point_list_unsorted, Rp);  // ... in depth order, before the stable per-tile pass
		obtain(chunk, b.tile_keys, Rp);            // tile id of every sorted instance (high word of the reference's keys)
		obtain(chunk, b.tile_keys_unsorted, Rp);
		obtain(chunk, b.recs, Rp);
		// per-pixel contribution masks, [block of the tile][block-list entry]: written by the forward blend, read by the
		// backward.  Never cleared: the forward writes the mask of every entry the backward reads (blend_fwd.cu).
		b.mask_stride = (Rp + 3) & ~(size_t)3;
		obtain(chunk, b.pix_mask, 8 * b.mask_stride);
		// per-block work lists, same rows and slots as the masks: a block's list is a subset of its tile's
		obtain(chunk, b.block_list, 8 * b.mask_stride);
		obtain(chunk, b.block_bits, Rp + 8);       // the records' block masks, one byte per instance; block_lists reads whole 16-byte chunks
		b.sort_bytes = cached_temp_bytes(1, (int)R);
		obtain(chunk, b.sort_temp, b.sort_bytes);
		return b;
	}
};
template <typename F>
static size_t required(F carve)
{
	char* p = nullptr;
	carve(p);
	return reinterpret_cast<size_t>(p) + 128;
}
static size_t num_tiles(int W, int H) { return (size_t)ceil_div(W, TILE_X) * ceil_div(H, TILE_Y); }

// next-highest bit of the MSB (number of bits needed for tile ids); same result as the reference's
// getHigherMsb (rasterizer_impl.cu:35-50) for n >= 1
static int higher_msb(uint32_t n)
{
	int bits = 0;
	while (bits < 32 && (n >> bits)) bits++;
	return bits;
}

// launch view u of a per-Gaussian backward (ProjectBwdViewsArgs or ProjectBwdCloudsDistArgs) with lens l: bit u of its
// model's mask and, for a fisheye or distorted view, its coefficients
template <class Args>
static void bwd_lens(Args& a, int u, const Lens& l)
{
	const uint16_t bit = (uint16_t)(1u << u);
	if (l.model == MODEL_ORTHO) a.ortho |= bit;
	if (l.model == MODEL_FISHEYE) { a.fisheye |= bit; a.fe_k[u] = l.fe_k; }
	if (l.model == MODEL_DISTORTED) { a.distorted |= bit; a.dc_k[u] = l.dc_k; }
}

}  // namespace mgs

using namespace mgs;

extern "C" {

int mgs_abi_version(void) { return 300; }
const char* mgs_last_error(void) { return g_err.c_str(); }

size_t mgs_geometry_state_bytes(int P) { return required([&](char*& p) { GeomState::carve(p, (size_t)P); }); }
size_t mgs_image_state_bytes(int width, int height)
{
	return required([&](char*& p) { ImageState::carve(p, (size_t)width * height, num_tiles(width, height)); });
}
size_t mgs_binning_state_bytes(int R) { return required([&](char*& p) { BinState::carve(p, (size_t)R); }); }
size_t mgs_backward_scratch_bytes(int P) { return (size_t)P * GB_STRIDE * sizeof(float) + 128; }
size_t mgs_camera_grad_scratch_bytes(int P) { return P > 0 ? camera_rows_bytes(P) : 0; }
// with the normal plane: the per-Gaussian quads nrm [P] behind the geometry state, the gradients gn [P,4] behind the scratch
size_t mgs_geometry_state_bytes_normal(int P)
{
	return required([&](char*& p) { GeomState::carve(p, (size_t)P); float4* nrm; obtain(p, nrm, (size_t)P); });
}
size_t mgs_backward_scratch_bytes_normal(int P) { return mgs_backward_scratch_bytes(P) + (size_t)P * 4 * sizeof(float) + 128; }


// ---------------------------------------------------------------------------------------------------------------------
// Per-view stages.  The multi-view entry points run them for V views of ONE Gaussian cloud with no host synchronisation
// anywhere; the single-view entry points run them for one view.
// ---------------------------------------------------------------------------------------------------------------------
namespace mgs {
// fork/join events between the caller's stream and the per-view streams (created once, reused; never destroyed)
struct EventPool {
	std::mutex mu;
	std::vector<cudaEvent_t> free_;
	cudaEvent_t get()
	{
		{
			std::lock_guard<std::mutex> lk(mu);
			if (!free_.empty()) { cudaEvent_t e = free_.back(); free_.pop_back(); return e; }
		}
		cudaEvent_t e = nullptr;
		cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
		return e;
	}
	void put(cudaEvent_t e) { std::lock_guard<std::mutex> lk(mu); free_.push_back(e); }
};
static EventPool g_events;

// every view stream waits for what the join stream has enqueued so far
static int fork_streams(int V, const mgs_view* views, cudaStream_t join)
{
	bool need = false;
	for (int v = 0; v < V; v++) need |= reinterpret_cast<cudaStream_t>(views[v].stream) != join;
	if (!need) return 0;
	cudaEvent_t e = g_events.get();
	MGS_CUDA(cudaEventRecord(e, join));
	for (int v = 0; v < V; v++) {
		cudaStream_t st = reinterpret_cast<cudaStream_t>(views[v].stream);
		if (st != join) MGS_CUDA(cudaStreamWaitEvent(st, e, 0));
	}
	g_events.put(e);  // recorded and waited on: safe to re-record later (waits captured the earlier record)
	return 0;
}
// every view stream waits for what every OTHER view stream has enqueued so far
static int cross_wait_streams(int V, const mgs_view* views)
{
	std::vector<cudaStream_t> uniq;
	for (int v = 0; v < V; v++) {
		cudaStream_t st = reinterpret_cast<cudaStream_t>(views[v].stream);
		bool seen = false;
		for (cudaStream_t u : uniq) seen |= u == st;
		if (!seen) uniq.push_back(st);
	}
	if (uniq.size() < 2) return 0;
	std::vector<cudaEvent_t> ev(uniq.size());
	for (size_t i = 0; i < uniq.size(); i++) {
		ev[i] = g_events.get();
		MGS_CUDA(cudaEventRecord(ev[i], uniq[i]));
	}
	for (size_t i = 0; i < uniq.size(); i++)
		for (size_t j = 0; j < uniq.size(); j++)
			if (i != j) MGS_CUDA(cudaStreamWaitEvent(uniq[i], ev[j], 0));
	for (cudaEvent_t e : ev) g_events.put(e);
	return 0;
}
static bool barrier_before_blend()
{
	static const bool on = [] { const char* e = getenv("MGS_BLEND_BARRIER"); return e && e[0] == '1'; }();
	return on;
}
// the join stream waits for every view stream
static int join_streams(int V, const mgs_view* views, cudaStream_t join)
{
	for (int v = 0; v < V; v++) {
		cudaStream_t st = reinterpret_cast<cudaStream_t>(views[v].stream);
		if (st == join) continue;
		bool seen = false;
		for (int u = 0; u < v; u++) seen |= views[u].stream == views[v].stream;
		if (seen) continue;
		cudaEvent_t e = g_events.get();
		MGS_CUDA(cudaEventRecord(e, st));
		MGS_CUDA(cudaStreamWaitEvent(join, e, 0));
		g_events.put(e);
	}
	return 0;
}

// per-Gaussian inputs shared by every view of one cloud
struct Cloud {
	int P, D, M, F;
	const float* means3D; const float* shs; const float* colors_precomp; const float* feature; const float* opacities;
	const float* scales; float scale_modifier; const float* rotations; const float* cov3D_precomp;
	int antialias;  // 1: the anti-aliased projection (opacity compensation); 0 where an initialiser leaves it out
	int planar;     // 1: planar depth (include/mgs_rasterizer.h, mgs_forward_views_planar); 0 where an initialiser leaves it out
};

// a view's tile grid and its state buffers, carved (pointers into a buffer the view does not provide are never used)
struct ViewState {
	int gx, gy;
	size_t T;
	GeomState geom; ImageState img; BinState bin;
	float* gb;  // blend-stage gradients of the backward, [P, GB_STRIDE] in blend_scratch
	// normal plane only (buffers sized by the _normal queries): the per-Gaussian quads behind the geometry state, and the
	// blend-stage normal gradients [P,4] behind gb
	float4* nrm;
	float* gn;
};
// the blend-stage records in a view's blend_scratch: gb [P, GB_STRIDE], then (buffers sized by the _normal queries) gn [P,4]
static void carve_scratch(char* sc, int P, float*& gb, float*& gn)
{
	obtain(sc, gb, (size_t)P * GB_STRIDE);
	obtain(sc, gn, (size_t)P * 4);
}
static ViewState carve_view(const mgs_view& w, int P)
{
	ViewState s;
	s.gx = ceil_div(w.width, TILE_X);
	s.gy = ceil_div(w.height, TILE_Y);
	s.T = (size_t)s.gx * s.gy;
	char* g = w.geometry_state; char* i = w.image_state; char* b = w.binning_state; char* sc = w.blend_scratch;
	s.geom = GeomState::carve(g, (size_t)P);
	s.img = ImageState::carve(i, (size_t)w.width * w.height, s.T);
	s.bin = BinState::carve(b, (size_t)w.binning_capacity);
	obtain(g, s.nrm, (size_t)P);
	carve_scratch(sc, P, s.gb, s.gn);
	return s;
}

// the view's device {tan_fovx, tan_fovy} (intr: one entry per view, or NULL), or NULL for mgs_view.tan_fovx / tan_fovy
static const float* device_fov(const mgs_view_intrinsics* intr, int v) { return intr ? intr[v].tan_fov : nullptr; }

// the views' camera models into lens[0 .. V) (ortho: one flag per view, or NULL; fisheye, distortion: one entry per view, or
// NULL, an entry whose flag is 0 ignored).  Each model is checked over every view before the next, so a call with several
// faults reports the same one whatever the views' order.
static int view_lenses(const int* ortho, const mgs_view_fisheye* fe, const mgs_view_distortion* dc, int V, std::vector<Lens>& lens)
{
	lens.assign(V, Lens{});
	for (int v = 0; ortho && v < V; v++) {
		if (ortho[v] != 0 && ortho[v] != 1) return fail(MGS_ERR_INVALID_ARG, "ortho: every entry must be 0 (perspective) or 1 (orthographic)");
		if (ortho[v]) lens[v].model = MODEL_ORTHO;
	}
	for (int v = 0; fe && v < V; v++) {
		const mgs_view_fisheye& f = fe[v];
		if (f.fisheye != 0 && f.fisheye != 1) return fail(MGS_ERR_INVALID_ARG, "fisheye: every flag must be 0 or 1");
		if (!f.fisheye) continue;
		if (lens[v].model == MODEL_ORTHO) return fail(MGS_ERR_INVALID_ARG, "fisheye: a view cannot be both orthographic and fisheye");
		const float x[7] = { f.cx, f.cy, f.k1, f.k2, f.k3, f.k4, f.theta_max };
		for (float xi : x)
			if (!std::isfinite(xi)) return fail(MGS_ERR_INVALID_ARG, "fisheye: cx, cy, k1..k4 and theta_max must be finite");
		if (!(f.theta_max > 0.f && f.theta_max <= 1.57079637f))  // (0, pi/2], pi/2 rounded to float
			return fail(MGS_ERR_INVALID_ARG, "fisheye: theta_max must lie in (0, pi/2]");
		Lens& l = lens[v];
		l.model = MODEL_FISHEYE;
		l.cx = f.cx; l.cy = f.cy; l.theta_max = f.theta_max; l.fe_k = FisheyeK{ f.k1, f.k2, f.k3, f.k4 };
	}
	for (int v = 0; dc && v < V; v++) {
		const mgs_view_distortion& d = dc[v];
		if (d.distorted != 0 && d.distorted != 1) return fail(MGS_ERR_INVALID_ARG, "distortion: every flag must be 0 or 1");
		if (!d.distorted) continue;
		if (lens[v].model != MODEL_PINHOLE)
			return fail(MGS_ERR_INVALID_ARG, "distortion: a distorted view cannot also be orthographic or fisheye");
		const float x[10] = { d.cx, d.cy, d.k1, d.k2, d.p1, d.p2, d.k3, d.k4, d.k5, d.k6 };
		for (float xi : x)
			if (!std::isfinite(xi)) return fail(MGS_ERR_INVALID_ARG, "distortion: cx, cy and the coefficients must be finite");
		if (!(d.r_max > 0.f)) return fail(MGS_ERR_INVALID_ARG, "distortion: r_max must be > 0 (+inf for no fold)");
		Lens& l = lens[v];
		l.model = MODEL_DISTORTED;
		l.cx = d.cx; l.cy = d.cy; l.r2_max = d.r_max * d.r_max;  // +inf stays +inf
		l.dc_k = DistK{ d.k1, d.k2, d.p1, d.p2, d.k3, d.k4, d.k5, d.k6 };
	}
	return 0;
}

// per-Gaussian projection, depth order and instance offsets; the instance count ends up in geom.point_offsets[P - 1].
// tan_fov: the view's device field of view, or NULL; lens: its camera model
static int enqueue_project(const Cloud& c, const mgs_view& w, const float* tan_fov, const Lens& lens, int debug)
{
	cudaStream_t st = reinterpret_cast<cudaStream_t>(w.stream);
	const ViewState s = carve_view(w, c.P);
	const GeomState& geom = s.geom;
	ProjectFwdArgs pa{};
	pa.P = c.P; pa.D = c.D; pa.M = c.M;
	pa.means3D = c.means3D; pa.scales = c.scales; pa.scale_modifier = c.scale_modifier; pa.rotations = c.rotations;
	pa.opacities = c.opacities; pa.shs = c.shs; pa.cov3D_precomp = c.cov3D_precomp; pa.colors_precomp = c.colors_precomp;
	pa.viewmatrix = w.viewmatrix; pa.projmatrix = w.projmatrix; pa.cam_pos = w.cam_pos;
	pa.W = w.width; pa.H = w.height; pa.tan_fovx = w.tan_fovx; pa.tan_fovy = w.tan_fovy;
	pa.focal_x = w.width / (2.0f * w.tan_fovx); pa.focal_y = w.height / (2.0f * w.tan_fovy);  // rasterizer_impl.cu:225-226
	pa.grid_x = s.gx; pa.grid_y = s.gy;
	pa.radii = w.radii; pa.means2D = geom.means2D; pa.depths = geom.depths; pa.cov3D = geom.cov3D; pa.rgbd = geom.rgbd;
	pa.conic_opacity = geom.conic_opacity; pa.extent = geom.extent; pa.clamped = geom.clamped; pa.tiles_touched = geom.tiles_touched;
	pa.iota = geom.iota;
	pa.antialias = c.antialias;
	pa.tan_fov = tan_fov;
	pa.lens = lens;
	{ StageTimer t_(ST_PROJECT_FWD, st); launch_project_fwd(pa, st); }
	MGS_STAGE("project_fwd");
	if (c.planar) {
		// the view's planar-depth quads, where the normal plane keeps its quads (the _normal size queries)
		PlanarFwdArgs la{};
		la.P = c.P; la.means3D = c.means3D; la.cov3D = c.cov3D_precomp ? c.cov3D_precomp : geom.cov3D; la.viewmatrix = w.viewmatrix;
		la.W = w.width; la.H = w.height; la.tan_fovx = w.tan_fovx; la.tan_fovy = w.tan_fovy; la.tan_fov = tan_fov; la.lens = lens;
		la.radii = w.radii; la.means2D = geom.means2D; la.conic_opacity = geom.conic_opacity; la.quad = s.nrm;
		launch_planar_fwd(la, st);
		MGS_STAGE("planar_fwd");
	}

	// Gaussians in depth order (stable: ascending id among equal depth bits; culled ones carry +inf and emit nothing)
	{
		StageTimer t_(ST_DEPTH_SORT, st);
		launch_depth_sort(geom.temp, geom.temp_bytes, reinterpret_cast<const uint32_t*>(geom.depths), geom.depth_sorted, geom.iota,
			geom.order, c.P, st);
	}
	MGS_STAGE("depth_sort");
	{ StageTimer t_(ST_SCAN, st); launch_scan_sorted(geom.temp, geom.temp_bytes, geom.order, geom.tiles_touched, geom.point_offsets, c.P, st); }
	MGS_STAGE("scan");
	return 0;
}

// instance emission, per-tile order, ranges and records into the view's binning_capacity slots.  The kernels read the
// instance count on the device and clamp it to the capacity; w.status, when set, receives {count, overflow flag}.
// exact_capacity: the caller read the count back and sized the capacity to it, so no slot is left over.
static int enqueue_binning(const Cloud& c, const mgs_view& w, bool exact_capacity, int debug)
{
	cudaStream_t st = reinterpret_cast<cudaStream_t>(w.stream);
	const int P = c.P;
	const ViewState s = carve_view(w, P);
	const GeomState& geom = s.geom;
	const BinState& bin = s.bin;
	const uint32_t cap = (uint32_t)w.binning_capacity;
	{
		StageTimer t_(ST_EMIT, st);
		launch_emit_tiles(P, geom.order, geom.means2D, geom.point_offsets, w.radii, s.gx, s.gy, bin.tile_keys_unsorted, bin.point_list_unsorted,
			cap, s.img.status, st);
		// the slots behind the R real instances sort to the very end: last tile id, ids never read
		if (!exact_capacity)
			launch_fill_tail(geom.point_offsets, P, cap, (uint32_t)(s.T - 1), bin.tile_keys_unsorted, bin.point_list_unsorted, st);
	}
	MGS_STAGE("emit_tiles");
	if (cap > 0) {
		// stable pass(es) over the tile-id bits only: instances already arrive in depth order
		const int bit = s.T > 1 ? higher_msb((uint32_t)(s.T - 1)) : 1;
		StageTimer t_(ST_SORT, st);
		launch_tile_sort(bin.sort_temp, bin.sort_bytes, bin.tile_keys_unsorted, bin.tile_keys, bin.point_list_unsorted, bin.point_list,
			(int)cap, bit, st);
		MGS_STAGE("tile_sort");
	}
	{
		StageTimer t_(ST_RANGES_PACK, st);
		launch_ranges_and_pack(geom.point_offsets + P - 1, (int)cap, (int)s.T, s.gx, bin.tile_keys, bin.point_list, geom.means2D,
			geom.conic_opacity, geom.extent, s.img.ranges, bin.recs, bin.block_bits, s.img.tile_order, st);
	}
	MGS_STAGE("ranges_pack");
	{
		StageTimer t_(ST_BLOCK_LISTS, st);
		launch_block_lists(s.img.ranges, (int)s.T, bin.block_bits, bin.block_list, bin.mask_stride, s.img.block_count, st);
	}
	MGS_STAGE("block_lists");
	if (w.status) MGS_CUDA(cudaMemcpyAsync(w.status, s.img.status, 2 * sizeof(int), cudaMemcpyDefault, st));
	return 0;
}

// the BlendArgs fields the forward and the backward blend share
static BlendArgs blend_args(const ViewState& s, const mgs_view& w, int F, const float* feature)
{
	BlendArgs ba{};
	ba.W = w.width; ba.H = w.height; ba.grid_x = s.gx; ba.grid_y = s.gy; ba.F = F; ba.groups = blend_groups(F);
	ba.ranges = s.img.ranges; ba.tile_order = use_tile_order() ? s.img.tile_order : nullptr; ba.point_list = s.bin.point_list; ba.recs = s.bin.recs;
	ba.rgbd = s.geom.rgbd; ba.feature = F > 0 ? feature : nullptr; ba.bg = w.background;
	ba.block_list = s.bin.block_list; ba.block_count = s.img.block_count; ba.block_nwalk = s.img.block_nwalk;
	ba.final_T = s.img.final_T; ba.n_contrib = s.img.n_contrib; ba.pix_mask = s.bin.pix_mask; ba.mask_stride = s.bin.mask_stride;
	MGS_CTA_LOG_ARGS(ba);
	MGS_BWD_PHASES_ARGS(ba);
	return ba;
}

// the depth / mask heads of one view: a target needs its planes and the accumulator, and (forward) the colour head
static int check_depth_mask(const mgs_view& w, const mgs_view_depth_mask* dm, bool forward)
{
	if (!dm || (!dm->target_depth && !dm->target_mask)) return 0;
	if (forward && !w.target_color) return fail(MGS_ERR_INVALID_ARG, "view: the depth / mask heads need the colour head (target_color)");
	if (!dm->loss_acc) return fail(MGS_ERR_INVALID_ARG, "view: the depth / mask heads need loss_acc");
	if (dm->target_depth && (!dm->cot_depth || !dm->cot_alpha_depth))
		return fail(MGS_ERR_INVALID_ARG, "view: target_depth needs cot_depth and cot_alpha_depth");
	if (dm->target_mask && !dm->cot_alpha_mask) return fail(MGS_ERR_INVALID_ARG, "view: target_mask needs cot_alpha_mask");
	return 0;
}

// the BlendArgs fields of the depth / mask heads (dm nullable; checked by check_depth_mask)
static void depth_mask_args(BlendArgs& ba, const mgs_view_depth_mask* dm)
{
	if (!dm || (!dm->target_depth && !dm->target_mask)) return;
	ba.tgt_depth = dm->target_depth; ba.tgt_mask = dm->target_mask;
	ba.cot_depth = dm->cot_depth; ba.cot_alpha_depth = dm->cot_alpha_depth; ba.cot_alpha_mask = dm->cot_alpha_mask;
	ba.dm_acc = dm->loss_acc; ba.dm_scale = dm->cot_scale;
}

// the median plane of one view (m nullable): a median-depth output or cotangent needs the id plane
static int check_median(const mgs_view_median* m)
{
	if (m && !m->median_id && (m->out_median_depth || m->dL_dpix_median_depth))
		return fail(MGS_ERR_INVALID_ARG, "view: out_median_depth and dL_dpix_median_depth need median_id (in its mgs_view_median)");
	return 0;
}

// the normal plane of one view (n nullable): it needs scales and rotations to take the axis from, the camera centre to face,
// and has no instantiation beside the depth / mask heads; a cotangent needs the plane its forward wrote
static int check_normal(const mgs_view& w, const mgs_view_normal* n, const float* scales, const float* rotations,
	const float* cov3D_precomp, const mgs_view_depth_mask* dm)
{
	if (!n || (!n->out_normal && !n->dL_dpix_normal)) return 0;
	if (cov3D_precomp || !scales || !rotations)
		return fail(MGS_ERR_INVALID_ARG, "view: the normal plane needs scales and rotations (a precomputed covariance has no axis to take)");
	if (!n->out_normal) return fail(MGS_ERR_INVALID_ARG, "view: dL_dpix_normal needs out_normal, the plane its forward wrote");
	if (!w.cam_pos) return fail(MGS_ERR_INVALID_ARG, "view: the normal plane needs cam_pos");
	if (dm && (dm->target_depth || dm->target_mask))
		return fail(MGS_ERR_INVALID_ARG, "view: the normal plane cannot be combined with the depth / mask heads");
	return 0;
}

// the view's per-Gaussian normal quads, behind its projection on its stream (nm nullable)
static int enqueue_normals_fwd(const Cloud& c, const mgs_view& w, const mgs_view_normal* nm, int debug)
{
	if (!nm || !nm->out_normal) return 0;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(w.stream);
	launch_normals_fwd(c.P, c.means3D, c.scales, c.rotations, w.cam_pos, carve_view(w, c.P).nrm, st);
	MGS_STAGE("normals_fwd");
	return 0;
}

// forward blend, with the fused loss heads when the view has a target; out_alpha (nullable) receives 1 - final_T; dm
// (nullable): the view's depth / mask heads; med (nullable): its median plane (checked by check_median); nm (nullable): its
// normal plane (checked by check_normal)
static int enqueue_blend_fwd(const Cloud& c, const mgs_view& w, float* out_alpha, const mgs_view_depth_mask* dm,
	const mgs_view_median* med, const mgs_view_normal* nm, int debug)
{
	cudaStream_t st = reinterpret_cast<cudaStream_t>(w.stream);
	const int F = (c.F > 0 && c.feature && w.out_feature) ? c.F : 0;
	const ViewState vs = carve_view(w, c.P);
	BlendArgs ba = blend_args(vs, w, F, c.feature);
	if (nm && nm->out_normal) { ba.nrm = vs.nrm; ba.out_normal = nm->out_normal; }
	if (c.planar) { ba.nrm = vs.nrm; ba.planar = 1; }
	ba.want_depth = w.out_depth != nullptr;
	ba.out_color = w.out_color; ba.out_feature = w.out_feature; ba.out_depth = w.out_depth; ba.out_alpha = out_alpha;
	if (med && med->median_id) { ba.median_id = med->median_id; ba.out_median_depth = med->out_median_depth; }
	// the cosine embedding head needs a pixel's whole feature vector: in the blend epilogue when one CTA holds it (F <= 32),
	// else in a features-only pass of the loss-heads kernel over the planes the blend just wrote
	const bool embed = w.target_color && w.target_feature && F > 0;
	const bool embed_after = embed && ba.groups > 1;
	if (w.target_color) {
		if (!w.cot_color || !w.loss_acc || (embed && !w.cot_feature))
			return fail(MGS_ERR_INVALID_ARG, "view: loss heads need cot_color, loss_acc (and cot_feature with target_feature)");
		ba.tgt_color = w.target_color; ba.tgt_feature = (embed && !embed_after) ? w.target_feature : nullptr;
		ba.cot_color = w.cot_color; ba.cot_feature = w.cot_feature; ba.loss_acc = w.loss_acc;
		MGS_CUDA(cudaMemsetAsync(w.loss_acc, 0, 2 * sizeof(float), st));
		depth_mask_args(ba, dm);
		if (ba.dm_acc) MGS_CUDA(cudaMemsetAsync(ba.dm_acc, 0, 3 * sizeof(float), st));
	}
	{
		StageTimer t_(ST_BLEND_FWD, st);
		launch_blend_fwd(ba, st);
		if (embed_after)
			launch_loss_heads(1, F, w.width * w.height, nullptr, w.out_feature, nullptr, w.target_feature, nullptr, w.cot_feature,
				w.loss_acc, st);
	}
	MGS_STAGE("blend_fwd");
	return 0;
}

// the SSIM head of one view (s nullable): it reads the view's image and target, and needs its planes and accumulator
static int check_ssim(const mgs_view& w, const mgs_view_ssim* s, bool forward)
{
	if (!s) return 0;
	if (!w.target_color) return fail(MGS_ERR_INVALID_ARG, "view: the SSIM head needs the colour target (target_color)");
	if (!s->ssim_terms || !s->loss_acc || !s->cot_color) return fail(MGS_ERR_INVALID_ARG, "view: the SSIM head needs ssim_terms, loss_acc and cot_color");
	if (!forward && !w.out_color) return fail(MGS_ERR_INVALID_ARG, "view: the SSIM backward needs out_color (the forward's image)");
	return 0;
}

// L1 + SSIM of one view's finished image, behind its blend on its stream (s nullable)
static int enqueue_ssim_fwd(const mgs_view& w, const mgs_view_ssim* s, int debug)
{
	if (!s) return 0;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(w.stream);
	MGS_CUDA(cudaMemsetAsync(s->loss_acc, 0, 4 * sizeof(float), st));
	{ StageTimer t_(ST_SSIM_FWD, st); launch_ssim_fwd(1, 3, w.height, w.width, w.out_color, w.target_color, s->ssim_terms, s->loss_acc, 2, st); }
	MGS_STAGE("ssim_fwd");
	return 0;
}

// the view's complete colour cotangent, before its blend backward on its stream (s nullable).  w becomes the view the
// blend backward sees: that plane as dL_dpix, and the scales {1, the view's feature scale} the kernel leaves in loss_acc[2..3]
static int enqueue_ssim_bwd(mgs_view& w, const mgs_view_ssim* s, int debug)
{
	if (!s) return 0;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(w.stream);
	{
		StageTimer t_(ST_SSIM_BWD, st);
		launch_ssim_bwd(1, 3, w.height, w.width, w.out_color, w.target_color, s->ssim_terms, s->cot_scale, w.dL_dpix, w.cot_scale,
			s->cot_color, s->loss_acc + 2, st);
	}
	MGS_STAGE("ssim_bwd");
	w.dL_dpix = s->cot_color;
	w.cot_scale = s->loss_acc + 2;
	return 0;
}

// blend backward of one view on its stream: the view's blend-stage records, and the feature gradients summed with 128-bit
// reductions straight into dL_dfeature.  dL_dfeature NULL with c.F > 0: the feature cotangents still reach the mean, conic
// and opacity gradients; only the feature rows are not reduced.  dL_dalpha (nullable): cotangent of the alpha plane; dm
// (nullable): the view's depth / mask heads, whose cotangent planes the walker's prologue folds in; med (nullable): its
// median plane, whose cotangent goes to the median contributors' depth slots; nm (nullable): its normal plane, whose
// cotangent is blended back into the view's gn.
static int enqueue_blend_bwd(const Cloud& c, const mgs_view& w, float* dL_dfeature, const float* dL_dalpha, const mgs_view_depth_mask* dm,
	const mgs_view_median* med, const mgs_view_normal* nm, int debug)
{
	cudaStream_t st = reinterpret_cast<cudaStream_t>(w.stream);
	const int F = c.F;
	const ViewState s = carve_view(w, c.P);
	MGS_CUDA(cudaMemsetAsync(s.gb, 0, (size_t)c.P * GB_STRIDE * sizeof(float), st));
	if (c.planar) MGS_CUDA(cudaMemsetAsync(s.gn, 0, (size_t)c.P * 4 * sizeof(float), st));
	if (med && med->dL_dpix_median_depth) {
		launch_median_depth_bwd(w.width * w.height, med->median_id, med->dL_dpix_median_depth, s.gb, st, w.width,
			c.planar ? s.gn : nullptr, s.geom.means2D);
		MGS_STAGE("median_depth_bwd");
	}
	BlendArgs ba = blend_args(s, w, F, c.feature);
	ba.dL_dcolor = w.dL_dpix; ba.dL_dfeature = F > 0 ? w.dL_dpix_F : nullptr; ba.dL_ddepth = w.dL_dpix_depth; ba.dL_dalpha = dL_dalpha;
	ba.gb = s.gb; ba.dL_dfeat = F > 0 ? dL_dfeature : nullptr;
	ba.cot_scale = w.cot_scale;
	if (nm && nm->dL_dpix_normal) {
		MGS_CUDA(cudaMemsetAsync(s.gn, 0, (size_t)c.P * 4 * sizeof(float), st));
		ba.nrm = s.nrm; ba.dL_dnormal = nm->dL_dpix_normal; ba.gn = s.gn;
	}
	if (c.planar) { ba.nrm = s.nrm; ba.gn = s.gn; ba.planar = 1; }
	depth_mask_args(ba, dm);
	ba.want_depth = w.dL_dpix_depth != nullptr || ba.tgt_depth != nullptr;  // the depth head's cotangent reaches the view-space z
	if (w.binning_capacity > 0) {
		{ StageTimer t_(ST_BLEND_BWD, st); launch_blend_bwd(ba, st); }
		MGS_STAGE("blend_bwd");
	}
	return 0;
}

// the per-Gaussian stage's view of one view: its blend-stage records, clamp bits and camera
static ProjectBwdView bwd_view(const mgs_view& w, int P, float* dL_dmean2D)
{
	const ViewState s = carve_view(w, P);
	ProjectBwdView pv;
	pv.radii = w.radii; pv.gb = s.gb; pv.clamped = s.geom.clamped; pv.viewmatrix = w.viewmatrix; pv.projmatrix = w.projmatrix;
	pv.cam_pos = w.cam_pos; pv.dL_dmean2D = dL_dmean2D;
	pv.tan_fovx = w.tan_fovx; pv.tan_fovy = w.tan_fovy;
	pv.focal_x = w.width / (2.0f * w.tan_fovx); pv.focal_y = w.height / (2.0f * w.tan_fovy);
	return pv;
}
// the per-Gaussian stage's planar-depth arrays of one view: its quad gradients, quads and screen means
static void planar_view(const Cloud& c, const mgs_view& w, const float4*& g, const float4*& q, const float2*& mean)
{
	if (!c.planar) return;
	const ViewState s = carve_view(w, c.P);
	g = reinterpret_cast<const float4*>(s.gn); q = s.nrm; mean = s.geom.means2D;
}

// camera gradients of view v (cam, intr: one entry per view, or NULL): the view asks for them when its camera entry or its
// intrinsics entry has an output; the rows live in the camera entry's scratch
static float* tan_fov_grad(const mgs_view_intrinsics* intr, int v) { return intr ? intr[v].dL_dtan_fov : nullptr; }
static bool camera_on(const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, int v)
{
	return (cam && (cam[v].dL_dviewmatrix || cam[v].dL_dprojmatrix || cam[v].dL_dcampos)) || tan_fov_grad(intr, v);
}
static int check_camera(const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, int V)
{
	for (int v = 0; v < V; v++)
		if (camera_on(cam, intr, v) && !(cam && cam[v].scratch))
			return fail(MGS_ERR_INVALID_ARG, "camera gradients: an entry with an output needs scratch (in its mgs_view_camera_grad)");
	return 0;
}
// the view's rows pointer and device field of view for its per-Gaussian launch, and its entry in that launch's reduce
static void camera_view(const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, const mgs_view& w, int v, int P, float*& rows,
	ProjectBwdIntr& ki, CamReduceArgs& cr)
{
	float* dtf = tan_fov_grad(intr, v);
	ki = ProjectBwdIntr{ device_fov(intr, v), w.width, w.height, dtf ? carve_view(w, P).geom.cam_intr : nullptr };
	if (!camera_on(cam, intr, v)) return;
	const mgs_view_camera_grad& e = cam[v];
	rows = e.scratch;
	cr.view[cr.V++] = CamReduceView{ e.scratch, (P + 127) / 128, e.dL_dviewmatrix, e.dL_dprojmatrix, e.dL_dcampos, ki.rows, dtf };
}

// the normal planes' share of dL_drot for views [v0, v0 + n) of one cloud (n <= MAX_BWD_VIEWS), behind the per-Gaussian
// launch that wrote dL_drot, on the same stream: the views with a normal cotangent, in view order
static int enqueue_normals_bwd(const Cloud& c, const mgs_view* views, const mgs_view_normal* nm, int v0, int n, float* dL_drot, int debug,
	cudaStream_t st)
{
	if (!nm || !dL_drot) return 0;
	NormalsBwdArgs na{};
	na.P = c.P; na.means3D = c.means3D; na.scales = c.scales; na.rotations = c.rotations; na.dL_drot = dL_drot;
	for (int v = v0; v < v0 + n; v++) {
		if (!nm[v].dL_dpix_normal) continue;
		na.gn[na.V] = carve_view(views[v], c.P).gn;
		na.cam_pos[na.V++] = views[v].cam_pos;
	}
	if (na.V == 0) return 0;
	launch_normals_bwd(na, st);
	MGS_STAGE("normals_bwd");
	return 0;
}

// the flow plane (include/mgs_rasterizer.h, mgs_forward_views_flow) of views [v0, v1) of one cloud: fl NULL or one entry per
// view of the call, next_means the cloud's next-frame means; it takes the normal plane's tile columns and quad slot
static bool flow_on(const mgs_view_flow* fl, int v) { return fl && (fl[v].out_flow || fl[v].dL_dpix_flow); }
// the whole call: flow never beside planar depth or a normal plane (they share the tile's columns 4..7); V views
static int check_flow_call(const mgs_view_flow* fl, int V, int planar_depth, const mgs_view_normal* normal)
{
	bool any = false;
	for (int v = 0; v < V; v++) any |= flow_on(fl, v);
	if (!any) return 0;
	if (planar_depth) return fail(MGS_ERR_INVALID_ARG, "flow cannot be combined with planar_depth (both take columns 4..7 of the tile)");
	for (int v = 0; v < V && normal; v++)
		if (normal[v].out_normal || normal[v].dL_dpix_normal)
			return fail(MGS_ERR_INVALID_ARG, "flow cannot be combined with a normal plane (both take columns 4..7 of the tile)");
	return 0;
}
// views [v0, v1) of one cloud with next-frame means next_means (or NULL); dm: one entry per view of the call, or NULL
static int check_flow(const mgs_view_flow* fl, const float* next_means, int v0, int v1, const mgs_view_depth_mask* dm)
{
	for (int v = v0; v < v1; v++) {
		if (!flow_on(fl, v)) continue;
		const mgs_view_flow& f = fl[v];
		if (dm && (dm[v].target_depth || dm[v].target_mask))
			return fail(MGS_ERR_INVALID_ARG, "view: the flow plane cannot be combined with the depth / mask heads");
		if (!f.out_flow) return fail(MGS_ERR_INVALID_ARG, "view: dL_dpix_flow needs out_flow, the plane its forward wrote");
		if (!next_means) return fail(MGS_ERR_INVALID_ARG, "view: out_flow needs the cloud's next-frame means");
		if (!f.next_viewmatrix != !f.next_projmatrix)
			return fail(MGS_ERR_INVALID_ARG, "view: next_viewmatrix and next_projmatrix are given together or not at all");
	}
	return 0;
}
// the blend's view of a flow plane: the normal plane's arguments (V entries), or `normal` itself when no view has flow
static const mgs_view_normal* flow_blend_planes(const mgs_view_flow* fl, int V, const mgs_view_normal* normal,
	std::vector<mgs_view_normal>& keep)
{
	bool any = false;
	for (int v = 0; v < V; v++) any |= flow_on(fl, v);
	if (!any) return normal;
	keep.assign(V, mgs_view_normal{ nullptr, nullptr });
	for (int v = 0; v < V; v++)
		if (flow_on(fl, v)) keep[v] = mgs_view_normal{ fl[v].out_flow, fl[v].dL_dpix_flow };
	return keep.data();
}
// view w's camera with the pose (vm, pm): its field of view, image size and lens
static FlowCam flow_cam(const mgs_view& w, const float* tan_fov, const Lens& lens, const float* vm, const float* pm)
{
	return FlowCam{ vm, pm, tan_fov, w.tan_fovx, w.tan_fovy, w.width, w.height, lens };
}
static const float* next_vm(const mgs_view_flow& f, const mgs_view& w) { return f.next_viewmatrix ? f.next_viewmatrix : w.viewmatrix; }
static const float* next_pm(const mgs_view_flow& f, const mgs_view& w) { return f.next_viewmatrix ? f.next_projmatrix : w.projmatrix; }

// the view's flow quads {dx, dy, 0, 0}, behind its projection on its stream (fl nullable), in the normal plane's quad slot
static int enqueue_flow_fwd(const Cloud& c, const mgs_view& w, const mgs_view_flow* fl, const float* next_means, const float* tan_fov,
	const Lens& lens, int debug)
{
	if (!fl || !fl->out_flow) return 0;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(w.stream);
	FlowFwdArgs a{};
	a.P = c.P; a.means3D = c.means3D; a.next_means3D = next_means;
	a.cur = flow_cam(w, tan_fov, lens, w.viewmatrix, w.projmatrix);
	a.next = flow_cam(w, tan_fov, lens, next_vm(*fl, w), next_pm(*fl, w));
	a.radii = w.radii; a.quad = carve_view(w, c.P).nrm;
	launch_flow_fwd(a, st);
	MGS_STAGE("flow_fwd");
	return 0;
}

// the flow planes' backward for views [v0, v0 + n) of one cloud (n <= MAX_BWD_VIEWS), on `st` behind the blend backward and
// ahead of the per-Gaussian launch that holds those views: the m path into each view's blend-stage records, the m' path into
// dL_dnext (written, or added with `accumulate`), and the m' camera terms into the views' camera rows, which one reduce sums
// into the camera outputs with `accumulate` (the per-Gaussian stage's reduce then adds to them).  Returns whether it enqueued
// that reduce.
static int enqueue_flow_bwd(const Cloud& c, const mgs_view* views, const mgs_view_flow* fl, const float* next_means, float* dL_dnext,
	const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, const Lens* lens, int v0, int n, int accumulate_next,
	int accumulate_cam, int debug, cudaStream_t st, bool& reduced)
{
	reduced = false;
	FlowBwdArgs a{};
	a.P = c.P; a.V = n; a.next_means3D = next_means; a.dL_dnext_means3D = dL_dnext; a.accumulate = accumulate_next;
	CamReduceArgs cr{};
	cr.accumulate = accumulate_cam;
	for (int u = 0; u < n; u++) {
		const int v = v0 + u;
		const mgs_view& w = views[v];
		FlowBwdView& b = a.view[u];
		const ViewState s = carve_view(w, c.P);
		const float* tf = device_fov(intr, v);
		b.radii = w.radii; b.gb = s.gb;
		if (flow_on(fl, v) && fl[v].dL_dpix_flow) {
			b.gn = reinterpret_cast<const float4*>(s.gn);
			b.cam = flow_cam(w, tf, lens[v], next_vm(fl[v], w), next_pm(fl[v], w));
			b.own_camera = fl[v].next_viewmatrix ? 0 : 1;
		}
		ProjectBwdIntr ki{};
		camera_view(cam, intr, w, v, c.P, b.cam_rows, ki, cr);
		b.intr_rows = ki.rows;
	}
	launch_flow_bwd(a, st);
	if (cr.V > 0) { launch_camera_grad_reduce(cr, st); reduced = true; }
	MGS_STAGE("flow_bwd");
	return 0;
}

// stages bit 0: the blend backward of every view on its stream, then the join; bit 1: the per-Gaussian chain rule on
// `join`, one launch per MAX_BWD_VIEWS views summed in registers.  dL_dconic (or NULL) is written only by a launch that
// does not accumulate, i.e. the first one when `accumulate` is 0: single-view callers only.  alpha, dm, ssim: V entries or NULL;
// lens: V entries.
static int backward_views(int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* dm,
	const mgs_view_ssim* ssim, const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, const mgs_view_median* med,
	const mgs_view_normal* nm, const Lens* lens, const Cloud& c, float* dL_dmean3D,
	float* dL_dopacity, float* dL_dcolor, float* dL_dfeature, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dconic, int shared_mean2D,
	int accumulate, int stages, int debug, cudaStream_t join, const mgs_view_flow* fl = nullptr, const float* flow_means3D = nullptr,
	float* dL_dflow = nullptr)
{
	const int P = c.P, F = c.F;
	std::vector<mgs_view_normal> flow_planes;
	const mgs_view_normal* blend_nm = flow_blend_planes(fl, V, nm, flow_planes);  // a flow plane rides in the normal plane's columns
	bool flow_bwd = false;  // a view has a flow cotangent
	for (int v = 0; v < V; v++) flow_bwd |= flow_on(fl, v) && fl[v].dL_dpix_flow;
	if (stages & 1) {
		if (F > 0 && !accumulate) MGS_CUDA(cudaMemsetAsync(dL_dfeature, 0, (size_t)P * F * sizeof(float), join));
		int rc = fork_streams(V, views, join);
		if (rc < 0) return rc;
		for (int v = 0; v < V; v++) {
			mgs_view w = views[v];
			rc = enqueue_ssim_bwd(w, ssim ? ssim + v : nullptr, debug);
			if (rc == 0)
				rc = enqueue_blend_bwd(c, w, dL_dfeature, alpha ? alpha[v].dL_dpix_alpha : nullptr, dm ? dm + v : nullptr,
					med ? med + v : nullptr, blend_nm ? blend_nm + v : nullptr, debug);
			if (rc < 0) return rc;
		}
		rc = join_streams(V, views, join);
		if (rc < 0) return rc;
	}  // blend stage: dL_dfeature is final here -- a caller may start exchanging it while the per-Gaussian stage runs
	if (!(stages & 2)) return 0;
	// the chain to scale / rotation runs when either gradient is asked for; without scales (cov3D_precomp) the rows
	// asked for are written as zeros.  shs are read whether or not dL_dsh is asked for: they carry the view-direction
	// term of dL_dmean3D.
	const bool have_sr = c.scales && c.rotations && (dL_dscale || dL_drot);
	for (int v0 = 0; v0 < V; v0 += MAX_BWD_VIEWS) {
		cudaStream_t st = join;
		ProjectBwdViewsArgs pb{};
		pb.P = P; pb.D = c.D; pb.M = c.M; pb.V = std::min(V - v0, (int)MAX_BWD_VIEWS);
		pb.means3D = c.means3D; pb.shs = c.shs;
		pb.scales = have_sr ? c.scales : nullptr; pb.rotations = c.rotations; pb.scale_modifier = c.scale_modifier;
		pb.cov3D_precomp = c.cov3D_precomp;
		if (!have_sr && !c.cov3D_precomp) {
			// gradients w.r.t. scale/rotation not requested: the forward's own covariance (any view's copy) serves
			pb.cov3D_precomp = carve_view(views[0], P).geom.cov3D;
		}
		pb.accumulate = (accumulate || v0 > 0) ? 1 : 0;
		pb.shared_mean2D = shared_mean2D;
		pb.dL_dmean3D = dL_dmean3D; pb.dL_dopacity = dL_dopacity; pb.dL_dcolor = dL_dcolor; pb.dL_dcov3D = dL_dcov3D;
		pb.dL_dsh = dL_dsh; pb.dL_dscale = dL_dscale; pb.dL_drot = dL_drot;
		pb.dL_dconic = pb.accumulate ? nullptr : dL_dconic;
		for (int u = 0; u < pb.V; u++)
			pb.view[u] = bwd_view(views[v0 + u], P, shared_mean2D ? views[0].dL_dmean2D : views[v0 + u].dL_dmean2D);
		pb.antialias = c.antialias;
		for (int u = 0; u < pb.V && c.antialias; u++) pb.conic_opacity[u] = carve_view(views[v0 + u], P).geom.conic_opacity;
		bool flow_reduced = false;  // the flow's camera terms already hold the camera outputs
		if (flow_bwd) {
			const int rc = enqueue_flow_bwd(c, views, fl, flow_means3D, dL_dflow, cam, intr, lens, v0, pb.V,
				(accumulate || v0 > 0) ? 1 : 0, accumulate ? 1 : 0, debug, st, flow_reduced);
			if (rc < 0) return rc;
		}
		CamReduceArgs cr{};
		cr.accumulate = (accumulate || flow_reduced) ? 1 : 0;
		for (int u = 0; u < pb.V; u++) camera_view(cam, intr, views[v0 + u], v0 + u, P, pb.cam_rows[u], pb.intr[u], cr);
		for (int u = 0; u < pb.V; u++) bwd_lens(pb, u, lens[v0 + u]);
		for (int u = 0; u < pb.V; u++) planar_view(c, views[v0 + u], pb.pl_g[u], pb.pl_q[u], pb.pl_mean[u]);
		// the camera reduce is timed with the launch it completes: the stage list ends with the SSIM stages
		{ StageTimer t_(ST_PROJECT_BWD, st); launch_project_bwd_views(pb, st); if (cr.V > 0) launch_camera_grad_reduce(cr, st); }
		MGS_STAGE("project_bwd");
		const int rc = enqueue_normals_bwd(c, views, nm, v0, pb.V, dL_drot, debug, st);
		if (rc < 0) return rc;
	}
	return 0;
}

// first half of a single-view forward (P > 0): checks the projection inputs, allocates the geometry and image state,
// enqueues the projection stage and copies the instance count to *host_count asynchronously on the view's stream
static int project_single_view(const Cloud& c, mgs_view& w, mgs_alloc_fn geometry_alloc, void* geometry_user, mgs_alloc_fn image_alloc,
	void* image_user, int* host_count, int debug)
{
	if (!c.means3D || !c.opacities || !w.viewmatrix || !w.projmatrix || !w.radii)
		return fail(MGS_ERR_INVALID_ARG, "means3D/opacities/viewmatrix/projmatrix/radii are required");
	if (!c.colors_precomp && !c.shs) return fail(MGS_ERR_INVALID_ARG, "provide SHs or precomputed colours");
	if (!c.colors_precomp && !w.cam_pos) return fail(MGS_ERR_INVALID_ARG, "cam_pos is required with SHs");
	if (!c.cov3D_precomp && (!c.scales || !c.rotations)) return fail(MGS_ERR_INVALID_ARG, "provide scales+rotations or a precomputed 3D covariance");
	w.geometry_state = geometry_alloc(geometry_user, mgs_geometry_state_bytes(c.P));
	w.image_state = image_alloc(image_user, mgs_image_state_bytes(w.width, w.height));
	if (!w.geometry_state || !w.image_state) return fail(MGS_ERR_ALLOC, "state allocation failed");
	int rc = enqueue_project(c, w, nullptr, Lens{}, debug);
	if (rc < 0) return rc;
	MGS_CUDA(cudaMemcpyAsync(host_count, carve_view(w, c.P).geom.point_offsets + c.P - 1, sizeof(int), cudaMemcpyDeviceToHost,
		reinterpret_cast<cudaStream_t>(w.stream)));
	return 0;
}

static int check_fwd_view(const mgs_view& w, bool need_cam_pos)
{
	if (!w.viewmatrix || !w.projmatrix || !w.background || !w.geometry_state || !w.binning_state || !w.image_state || !w.out_color || !w.radii)
		return fail(MGS_ERR_INVALID_ARG, "view: matrices, background, the three state buffers, out_color and radii are required");
	if (need_cam_pos && !w.cam_pos) return fail(MGS_ERR_INVALID_ARG, "view: cam_pos is required with SHs");
	if (w.width <= 0 || w.height <= 0 || w.binning_capacity < 0) return fail(MGS_ERR_INVALID_ARG, "view: bad size or capacity");
	return 0;
}

static int check_bwd_view(const mgs_view& w, bool need_dpix_F)
{
	if (!w.viewmatrix || !w.projmatrix || !w.background || !w.geometry_state || !w.binning_state || !w.image_state || !w.radii ||
		!w.dL_dpix || !w.blend_scratch)
		return fail(MGS_ERR_INVALID_ARG, "view: matrices, background, state buffers, radii, dL_dpix and blend_scratch are required");
	if (need_dpix_F && !w.dL_dpix_F) return fail(MGS_ERR_INVALID_ARG, "view: dL_dpix_F is required with features");
	return 0;
}

// the checks the multi-cloud forward and backward share: B, the view ranges and every cloud's size
static int check_clouds(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views)
{
	if (B <= 0 || !clouds || !view_offsets || !views) return fail(MGS_ERR_INVALID_ARG, "need at least one cloud, view_offsets and views");
	if (view_offsets[0] != 0) return fail(MGS_ERR_INVALID_ARG, "view_offsets must start at 0");
	for (int b = 0; b < B; b++) {
		if (view_offsets[b + 1] <= view_offsets[b])
			return fail(MGS_ERR_INVALID_ARG, "view_offsets must be strictly increasing: every cloud needs at least one view");
		if (clouds[b].P <= 0) return fail(MGS_ERR_INVALID_ARG, "cloud: P must be > 0");
	}
	return 0;
}

static Cloud cloud_of(const mgs_cloud& k, int D, int M, int F, float scale_modifier, int antialias, int planar = 0)
{
	return Cloud{ k.P, D, M, k.feature ? F : 0, k.means3D, k.shs, k.colors_precomp, k.feature, k.opacities, k.scales, scale_modifier,
		k.rotations, k.cov3D_precomp, antialias, planar };
}

static int check_antialias(int antialiasing)
{
	if (antialiasing != 0 && antialiasing != 1) return fail(MGS_ERR_INVALID_ARG, "antialiasing must be 0 or 1");
	return 0;
}

// planar depth: a flag, and never beside a normal plane (both take columns 4..6 of the blend's {r,g,b,depth} tile); normal: V
// entries or NULL
static int check_planar(int planar_depth, const mgs_view_normal* normal, int V)
{
	if (planar_depth != 0 && planar_depth != 1) return fail(MGS_ERR_INVALID_ARG, "planar_depth must be 0 or 1");
	for (int v = 0; planar_depth && normal && v < V; v++)
		if (normal[v].out_normal || normal[v].dL_dpix_normal)
			return fail(MGS_ERR_INVALID_ARG, "planar_depth cannot be combined with a normal plane in the same call");
	return 0;
}


}  // namespace mgs

int mgs_forward(
	mgs_alloc_fn geometry_alloc, void* geometry_user,
	mgs_alloc_fn binning_alloc, void* binning_user,
	mgs_alloc_fn image_alloc, void* image_user,
	int P, int D, int M, int F,
	const float* background, int width, int height,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations,
	const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix, const float* cam_pos,
	float tan_fovx, float tan_fovy, int prefiltered,
	float* out_color, float* out_feature, float* out_depth, int* radii, int debug, void* stream)
{
	(void)prefiltered;  // the reference only uses it to trap on inconsistent input (auxiliary.h:156-160)
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	if (!geometry_alloc || !binning_alloc || !image_alloc) return fail(MGS_ERR_INVALID_ARG, "allocator callbacks are required");
	if (P < 0 || width <= 0 || height <= 0) return fail(MGS_ERR_INVALID_ARG, "bad P/width/height");
	if (!out_color || !background) return fail(MGS_ERR_INVALID_ARG, "out_color/background are required");
	if (F < 0 || F > MGS_MAX_FEATURE_CHANNELS || !blend_supported(F))
		return fail(MGS_ERR_UNSUPPORTED, bad_width_msg);
	if (F > 0 && (!feature_precomp || !out_feature)) F = 0;  // include_feature == false
	const size_t N = (size_t)width * height;
	if (P == 0) {
		// reference: outputs keep their zero fill when there are no Gaussians (rasterize_points.cu:70-92)
		MGS_CUDA(cudaMemsetAsync(out_color, 0, 3 * N * sizeof(float), st));
		if (F > 0) MGS_CUDA(cudaMemsetAsync(out_feature, 0, (size_t)F * N * sizeof(float), st));
		if (out_depth) MGS_CUDA(cudaMemsetAsync(out_depth, 0, N * sizeof(float), st));
		return 0;
	}
	const Cloud c{ P, D, M, F, means3D, shs, colors_precomp, feature_precomp, opacities, scales, scale_modifier, rotations, cov3D_precomp };
	mgs_view w{};
	w.viewmatrix = viewmatrix; w.projmatrix = projmatrix; w.cam_pos = cam_pos; w.background = background;
	w.tan_fovx = tan_fovx; w.tan_fovy = tan_fovy; w.width = width; w.height = height;
	w.out_color = out_color; w.out_feature = out_feature; w.out_depth = out_depth; w.radii = radii; w.stream = stream;
	int num_rendered = 0;
	int rc = project_single_view(c, w, geometry_alloc, geometry_user, image_alloc, image_user, &num_rendered, debug);
	if (rc < 0) return rc;
	MGS_CUDA(cudaStreamSynchronize(st));  // the one host sync of the forward, as in the reference (rasterizer_impl.cu:284)
	if (num_rendered < 0) return fail(MGS_ERR_UNSUPPORTED, "more than 2^31-1 tile instances");
	// binning state for exactly the R instances: nothing is dropped, and the kernels cover the same R slots as the count
	w.binning_state = binning_alloc(binning_user, mgs_binning_state_bytes(num_rendered));
	if (!w.binning_state) return fail(MGS_ERR_ALLOC, "binning state allocation failed");
	w.binning_capacity = num_rendered;
	rc = enqueue_binning(c, w, true, debug);
	if (rc < 0) return rc;
	rc = enqueue_blend_fwd(c, w, nullptr, nullptr, nullptr, nullptr, debug);
	return rc < 0 ? rc : num_rendered;
}

int mgs_forward_begin(
	mgs_alloc_fn geometry_alloc, void* geometry_user, mgs_alloc_fn image_alloc, void* image_user,
	int P, int D, int M, int width, int height,
	const float* means3D, const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
	float scale_modifier, const float* rotations, const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
	const float* cam_pos, float tan_fovx, float tan_fovy, int* radii, int* host_num_rendered, int debug, void* stream)
{
	if (P <= 0 || width <= 0 || height <= 0) return fail(MGS_ERR_INVALID_ARG, "bad P/width/height (P must be > 0)");
	if (!geometry_alloc || !image_alloc || !host_num_rendered) return fail(MGS_ERR_INVALID_ARG, "allocators and host_num_rendered are required");
	const Cloud c{ P, D, M, 0, means3D, shs, colors_precomp, nullptr, opacities, scales, scale_modifier, rotations, cov3D_precomp };
	mgs_view w{};
	w.viewmatrix = viewmatrix; w.projmatrix = projmatrix; w.cam_pos = cam_pos;
	w.tan_fovx = tan_fovx; w.tan_fovy = tan_fovy; w.width = width; w.height = height; w.radii = radii; w.stream = stream;
	return project_single_view(c, w, geometry_alloc, geometry_user, image_alloc, image_user, host_num_rendered, debug);
}

int mgs_backward(
	int P, int D, int M, int F, int R,
	const float* background, int width, int height,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx, float tan_fovy,
	const int* radii, char* geometry_state, char* binning_state, char* image_state,
	const float* dL_dpix, const float* dL_dpix_F, const float* dL_dpix_depth,
	float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_dfeature,
	float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
	char* blend_scratch, int accumulate, int debug, void* stream)
{
	if (P < 0 || width <= 0 || height <= 0 || R < 0) return fail(MGS_ERR_INVALID_ARG, "bad P/R/width/height");
	if (P == 0) return 0;
	if (F < 0 || F > MGS_MAX_FEATURE_CHANNELS) return fail(MGS_ERR_UNSUPPORTED, bad_width_msg);
	if (F > 0 && (!feature_precomp || !dL_dpix_F || !dL_dfeature)) F = 0;
	if (!geometry_state || !binning_state || !image_state || !blend_scratch)
		return fail(MGS_ERR_INVALID_ARG, "state buffers and scratch are required");
	if (!dL_dpix || !dL_dmean2D || !dL_dopacity || !dL_dmean3D || !means3D || !radii || !background)
		return fail(MGS_ERR_INVALID_ARG, "required pointer is NULL");
	const Cloud c{ P, D, M, F, means3D, shs, colors_precomp, feature_precomp, nullptr, scales, scale_modifier, rotations, cov3D_precomp };
	mgs_view w{};
	w.viewmatrix = viewmatrix; w.projmatrix = projmatrix; w.cam_pos = campos; w.background = background;
	w.tan_fovx = tan_fovx; w.tan_fovy = tan_fovy; w.width = width; w.height = height;
	w.geometry_state = geometry_state; w.binning_state = binning_state; w.image_state = image_state; w.binning_capacity = R;
	w.radii = const_cast<int*>(radii);  // read only by the backward
	w.dL_dpix = dL_dpix; w.dL_dpix_F = dL_dpix_F; w.dL_dpix_depth = dL_dpix_depth;
	w.blend_scratch = blend_scratch; w.dL_dmean2D = dL_dmean2D; w.stream = stream;
	const Lens pinhole{};
	return backward_views(1, &w, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, &pinhole, c, dL_dmean3D, dL_dopacity, dL_dcolor, dL_dfeature, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, dL_dconic,
		1, accumulate, 3, debug, reinterpret_cast<cudaStream_t>(stream));
}

int mgs_forward_views(
	int V, const mgs_view* views,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_views_alpha(V, views, nullptr, P, D, M, F, means3D, shs, colors_precomp, feature_precomp, opacities, scales,
		scale_modifier, rotations, cov3D_precomp, prefiltered, debug, join_stream);
}

int mgs_forward_views_alpha(
	int V, const mgs_view* views, const mgs_view_alpha* alpha,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_views_depth_mask(V, views, alpha, nullptr, P, D, M, F, means3D, shs, colors_precomp, feature_precomp, opacities,
		scales, scale_modifier, rotations, cov3D_precomp, prefiltered, debug, join_stream);
}

int mgs_forward_views_depth_mask(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_views_aa(V, views, alpha, depth_mask, 0, P, D, M, F, means3D, shs, colors_precomp, feature_precomp, opacities,
		scales, scale_modifier, rotations, cov3D_precomp, prefiltered, debug, join_stream);
}

int mgs_forward_views_aa(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_views_ssim(V, views, alpha, depth_mask, antialiasing, nullptr, P, D, M, F, means3D, shs, colors_precomp,
		feature_precomp, opacities, scales, scale_modifier, rotations, cov3D_precomp, prefiltered, debug, join_stream);
}

int mgs_forward_views_ssim(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_views_intr(V, views, alpha, depth_mask, antialiasing, ssim, nullptr, P, D, M, F, means3D, shs, colors_precomp,
		feature_precomp, opacities, scales, scale_modifier, rotations, cov3D_precomp, prefiltered, debug, join_stream);
}

int mgs_forward_views_intr(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim, const mgs_view_intrinsics* intr,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_views_median(V, views, alpha, depth_mask, antialiasing, ssim, intr, nullptr, P, D, M, F, means3D, shs,
		colors_precomp, feature_precomp, opacities, scales, scale_modifier, rotations, cov3D_precomp, prefiltered, debug, join_stream);
}

int mgs_forward_views_median(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim, const mgs_view_intrinsics* intr, const mgs_view_median* median,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_views_normal(V, views, alpha, depth_mask, antialiasing, ssim, intr, median, nullptr, P, D, M, F, means3D, shs,
		colors_precomp, feature_precomp, opacities, scales, scale_modifier, rotations, cov3D_precomp, prefiltered, debug, join_stream);
}

int mgs_forward_views_normal(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim, const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_views_ortho(V, views, alpha, depth_mask, antialiasing, ssim, intr, median, normal, nullptr, P, D, M, F, means3D,
		shs, colors_precomp, feature_precomp, opacities, scales, scale_modifier, rotations, cov3D_precomp, prefiltered, debug, join_stream);
}

int mgs_forward_views_ortho(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim, const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal,
	const int* ortho,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_views_fisheye(V, views, alpha, depth_mask, antialiasing, ssim, intr, median, normal, ortho, nullptr, P, D, M, F,
		means3D, shs, colors_precomp, feature_precomp, opacities, scales, scale_modifier, rotations, cov3D_precomp, prefiltered, debug,
		join_stream);
}

int mgs_forward_views_fisheye(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim, const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal,
	const int* ortho, const mgs_view_fisheye* fisheye,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_views_distorted(V, views, alpha, depth_mask, antialiasing, ssim, intr, median, normal, ortho, fisheye,
		nullptr, P, D, M, F, means3D, shs, colors_precomp, feature_precomp, opacities, scales, scale_modifier, rotations,
		cov3D_precomp, prefiltered, debug, join_stream);
}

int mgs_forward_views_distorted(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim, const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal,
	const int* ortho, const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_views_planar(V, views, alpha, depth_mask, antialiasing, ssim, intr, median, normal, ortho, fisheye,
		distortion, 0, P, D, M, F, means3D, shs, colors_precomp, feature_precomp, opacities, scales, scale_modifier, rotations,
		cov3D_precomp, prefiltered, debug, join_stream);
}

int mgs_forward_views_planar(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim, const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal,
	const int* ortho, const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion, int planar_depth,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_views_flow(V, views, alpha, depth_mask, antialiasing, ssim, intr, median, normal, ortho, fisheye, distortion,
		planar_depth, nullptr, nullptr, P, D, M, F, means3D, shs, colors_precomp, feature_precomp, opacities, scales, scale_modifier,
		rotations, cov3D_precomp, prefiltered, debug, join_stream);
}

int mgs_forward_views_flow(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim, const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal,
	const int* ortho, const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion, int planar_depth,
	const mgs_view_flow* flow, const float* flow_means3D,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	int prefiltered, int debug, void* join_stream)
{
	(void)prefiltered;
	if (check_antialias(antialiasing) < 0) return MGS_ERR_INVALID_ARG;
	if (V <= 0 || !views) return fail(MGS_ERR_INVALID_ARG, "need at least one view");
	if (check_planar(planar_depth, normal, V) < 0) return MGS_ERR_INVALID_ARG;
	if (check_flow_call(flow, V, planar_depth, normal) < 0 || check_flow(flow, flow_means3D, 0, V, depth_mask) < 0)
		return MGS_ERR_INVALID_ARG;
	std::vector<Lens> lens;
	if (view_lenses(ortho, fisheye, distortion, V, lens) < 0) return MGS_ERR_INVALID_ARG;
	if (P <= 0) return fail(MGS_ERR_INVALID_ARG, "P must be > 0");
	if (!means3D || !opacities) return fail(MGS_ERR_INVALID_ARG, "means3D/opacities are required");
	if (!colors_precomp && !shs) return fail(MGS_ERR_INVALID_ARG, "provide SHs or precomputed colours");
	if (!cov3D_precomp && (!scales || !rotations)) return fail(MGS_ERR_INVALID_ARG, "provide scales+rotations or a precomputed 3D covariance");
	if (F < 0 || F > MGS_MAX_FEATURE_CHANNELS || !blend_supported(F)) return fail(MGS_ERR_UNSUPPORTED, bad_width_msg);
	for (int v = 0; v < V; v++) {
		int rc = check_fwd_view(views[v], !colors_precomp);
		if (rc == 0) rc = check_depth_mask(views[v], depth_mask ? depth_mask + v : nullptr, true);
		if (rc == 0) rc = check_ssim(views[v], ssim ? ssim + v : nullptr, true);
		if (rc == 0) rc = check_median(median ? median + v : nullptr);
		if (rc == 0) rc = check_normal(views[v], normal ? normal + v : nullptr, scales, rotations, cov3D_precomp, depth_mask ? depth_mask + v : nullptr);
		if (rc < 0) return rc;
	}
	const Cloud c{ P, D, M, F, means3D, shs, colors_precomp, feature_precomp, opacities, scales, scale_modifier, rotations, cov3D_precomp,
		antialiasing, planar_depth };
	std::vector<mgs_view_normal> flow_planes;
	const mgs_view_normal* blend_nm = flow_blend_planes(flow, V, normal, flow_planes);
	cudaStream_t join = reinterpret_cast<cudaStream_t>(join_stream);
	int rc = fork_streams(V, views, join);
	if (rc < 0) return rc;
	// stage by stage across the views: the short per-Gaussian and binning kernels of every view are enqueued before any
	// view's long blend kernel, so no view's chain queues behind another view's blend
	for (int phase = 0; phase < 3; phase++) {
		// MGS_BLEND_BARRIER=1: all blends start together, after the binning chain of EVERY view.  A blend launch is one
		// wave of small CTAs that takes every shared-memory slot of the GPU, and the short binning kernels of the
		// other views crawl behind it (CTA timeline, tools/cta_timeline.py: blends 0 and 1 each run alone, 790 us for the
		// four forward blends of the bench step; started together 590 us) -- but four binning chains side by side take
		// 0.38 ms instead of 0.22 ms for the first alone, and the step time comes out the same (2.21 ms either way,
		// DESIGN.md section 7), so the default keeps the dependency-free schedule.
		if (phase == 2 && barrier_before_blend()) {
			rc = cross_wait_streams(V, views);
			if (rc < 0) return rc;
		}
		for (int v = 0; v < V; v++) {
			rc = phase == 0 ? enqueue_project(c, views[v], device_fov(intr, v), lens[v], debug)
				: phase == 1 ? enqueue_binning(c, views[v], false, debug)
				: enqueue_blend_fwd(c, views[v], alpha ? alpha[v].out_alpha : nullptr, depth_mask ? depth_mask + v : nullptr,
					median ? median + v : nullptr, blend_nm ? blend_nm + v : nullptr, debug);
			if (rc == 0 && phase == 0) rc = enqueue_normals_fwd(c, views[v], normal ? normal + v : nullptr, debug);
			if (rc == 0 && phase == 0)
				rc = enqueue_flow_fwd(c, views[v], flow ? flow + v : nullptr, flow_means3D, device_fov(intr, v), lens[v], debug);
			if (rc == 0 && phase == 2) rc = enqueue_ssim_fwd(views[v], ssim ? ssim + v : nullptr, debug);
			if (rc < 0) return rc;
		}
	}
	return join_streams(V, views, join);
}

int mgs_lift_views(
	int V, const mgs_view* views, const mgs_view_lift* lift, int antialiasing, const mgs_view_intrinsics* intr,
	int P, int D, int M, int C,
	const float* means3D, const float* shs, const float* colors_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* out_lifted, float* out_weight, int debug, void* join_stream)
{
	return mgs_lift_views_ortho(V, views, lift, antialiasing, intr, nullptr, P, D, M, C, means3D, shs, colors_precomp, opacities, scales,
		scale_modifier, rotations, cov3D_precomp, out_lifted, out_weight, debug, join_stream);
}

int mgs_lift_views_ortho(
	int V, const mgs_view* views, const mgs_view_lift* lift, int antialiasing, const mgs_view_intrinsics* intr, const int* ortho,
	int P, int D, int M, int C,
	const float* means3D, const float* shs, const float* colors_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* out_lifted, float* out_weight, int debug, void* join_stream)
{
	return mgs_lift_views_fisheye(V, views, lift, antialiasing, intr, ortho, nullptr, P, D, M, C, means3D, shs, colors_precomp, opacities,
		scales, scale_modifier, rotations, cov3D_precomp, out_lifted, out_weight, debug, join_stream);
}

int mgs_lift_views_fisheye(
	int V, const mgs_view* views, const mgs_view_lift* lift, int antialiasing, const mgs_view_intrinsics* intr, const int* ortho,
	const mgs_view_fisheye* fisheye,
	int P, int D, int M, int C,
	const float* means3D, const float* shs, const float* colors_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* out_lifted, float* out_weight, int debug, void* join_stream)
{
	return mgs_lift_views_distorted(V, views, lift, antialiasing, intr, ortho, fisheye, nullptr, P, D, M, C, means3D, shs,
		colors_precomp, opacities, scales, scale_modifier, rotations, cov3D_precomp, out_lifted, out_weight, debug, join_stream);
}

int mgs_lift_views_distorted(
	int V, const mgs_view* views, const mgs_view_lift* lift, int antialiasing, const mgs_view_intrinsics* intr, const int* ortho,
	const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion,
	int P, int D, int M, int C,
	const float* means3D, const float* shs, const float* colors_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* out_lifted, float* out_weight, int debug, void* join_stream)
{
	if (check_antialias(antialiasing) < 0) return MGS_ERR_INVALID_ARG;
	if (V <= 0 || !views) return fail(MGS_ERR_INVALID_ARG, "need at least one view");
	std::vector<Lens> lens;
	if (view_lenses(ortho, fisheye, distortion, V, lens) < 0) return MGS_ERR_INVALID_ARG;
	if (C < 0 || C > MGS_MAX_FEATURE_CHANNELS) return fail(MGS_ERR_UNSUPPORTED, "map channel count must be in [0, " MGS_STR(MGS_MAX_FEATURE_CHANNELS) "]");
	if (P <= 0) return fail(MGS_ERR_INVALID_ARG, "P must be > 0");
	if (!means3D || !opacities) return fail(MGS_ERR_INVALID_ARG, "means3D/opacities are required");
	if (!colors_precomp && !shs) return fail(MGS_ERR_INVALID_ARG, "provide SHs or precomputed colours (never read: they keep the projection the forward's)");
	if (!cov3D_precomp && (!scales || !rotations)) return fail(MGS_ERR_INVALID_ARG, "provide scales+rotations or a precomputed 3D covariance");
	if (!out_weight || (C > 0 && !out_lifted)) return fail(MGS_ERR_INVALID_ARG, "out_weight (and out_lifted with C > 0) are required");
	if (C > 0 && !lift) return fail(MGS_ERR_INVALID_ARG, "C > 0 needs one mgs_view_lift per view");
	for (int v = 0; v < V; v++) {
		const mgs_view& w = views[v];
		if (!w.geometry_state || !w.binning_state || !w.image_state)
			return fail(MGS_ERR_INVALID_ARG, "view: the three state buffers are required");
		if (!w.viewmatrix || !w.projmatrix || !w.radii) return fail(MGS_ERR_INVALID_ARG, "view: matrices and radii are required");
		if (shs && !colors_precomp && !w.cam_pos) return fail(MGS_ERR_INVALID_ARG, "view: cam_pos is required with SHs");
		if (w.width <= 0 || w.height <= 0 || w.binning_capacity < 0) return fail(MGS_ERR_INVALID_ARG, "view: bad size or capacity");
		if (C > 0 && !lift[v].map) return fail(MGS_ERR_INVALID_ARG, "view: map is required with C > 0");
	}
	const Cloud c{ P, D, M, 0, means3D, shs, colors_precomp, nullptr, opacities, scales, scale_modifier, rotations, cov3D_precomp,
		antialiasing };
	cudaStream_t join = reinterpret_cast<cudaStream_t>(join_stream);
	// every view adds into the same outputs: zero them before any view stream starts
	MGS_CUDA(cudaMemsetAsync(out_weight, 0, (size_t)P * sizeof(float), join));
	if (C > 0) MGS_CUDA(cudaMemsetAsync(out_lifted, 0, (size_t)P * C * sizeof(float), join));
	int rc = fork_streams(V, views, join);
	if (rc < 0) return rc;
	// stage by stage across the views, as mgs_forward_views_normal: the lift takes the forward blend's place
	for (int phase = 0; phase < 3; phase++) {
		for (int v = 0; v < V; v++) {
			const mgs_view& w = views[v];
			if (phase == 0) rc = enqueue_project(c, w, device_fov(intr, v), lens[v], debug);
			else if (phase == 1) rc = enqueue_binning(c, w, false, debug);
			else {
				cudaStream_t st = reinterpret_cast<cudaStream_t>(w.stream);
				const ViewState s = carve_view(w, P);
				LiftArgs la{};
				la.W = w.width; la.H = w.height; la.grid_x = s.gx; la.grid_y = s.gy; la.C = C; la.groups = blend_groups(C);
				la.ranges = s.img.ranges; la.tile_order = use_tile_order() ? s.img.tile_order : nullptr; la.recs = s.bin.recs;
				la.block_list = s.bin.block_list; la.block_count = s.img.block_count; la.mask_stride = s.bin.mask_stride;
				la.map = C > 0 ? lift[v].map : nullptr; la.lifted = C > 0 ? out_lifted : nullptr; la.weight = out_weight;
				{ StageTimer t_(ST_BLEND_FWD, st); launch_lift(la, st); }
				MGS_STAGE("lift");
			}
			if (rc < 0) return rc;
		}
	}
	return join_streams(V, views, join);
}

}  // extern "C"

namespace mgs {
// the point scratch of one view of mgs_visibility_views, carved from its blend_scratch
struct VisScratch {
	float4* pt; uint32_t* keys; uint32_t* keys_sorted; uint32_t* idx; uint32_t* idx_sorted; uint2* qranges; uint32_t* item_end;
	char* sort_temp; size_t sort_bytes;
	static VisScratch carve(char*& chunk, size_t Q, size_t T)
	{
		VisScratch s;
		obtain(chunk, s.pt, Q);
		obtain(chunk, s.keys, Q);
		obtain(chunk, s.keys_sorted, Q);
		obtain(chunk, s.idx, Q);
		obtain(chunk, s.idx_sorted, Q);
		obtain(chunk, s.qranges, T);
		obtain(chunk, s.item_end, T);
		s.sort_bytes = cached_temp_bytes(1, (int)Q);
		obtain(chunk, s.sort_temp, s.sort_bytes);
		return s;
	}
};
// the query arguments of one view of mgs_visibility_views over its state s and point scratch x (outputs left NULL)
static VisArgs vis_args(const mgs_view& w, const ViewState& s, const VisScratch& x, const FlowCam& cam, int Q, const float* points)
{
	VisArgs a{};
	a.Q = Q; a.W = w.width; a.H = w.height; a.grid_x = s.gx; a.num_tiles = (int)s.T;
	a.cam = cam;
	a.points = points;
	a.pt = x.pt; a.keys = x.keys; a.idx = x.idx; a.keys_sorted = x.keys_sorted; a.idx_sorted = x.idx_sorted;
	a.qranges = x.qranges; a.item_end = x.item_end;
	a.ranges = s.img.ranges; a.point_list = s.bin.point_list; a.depths = s.geom.depths; a.recs = s.bin.recs;
	return a;
}
// the backward scratch of one view of mgs_visibility_views_backward, carved from its dL_dmean2D: the blend-stage rows gb, the
// T path's uv cotangents, the point path's camera and focal-length rows (one per VIS_PTS_BWD_THREADS points), the Gaussian
// path's camera rows, and the two cloud outputs the per-Gaussian chain always writes, for a call that asks only for cameras
struct VisBwdScratch {
	float* gb; float* duv; float* pt_rows; float* pt_intr; float* g_rows; float* mean3D; float* opacity;
	static VisBwdScratch carve(char*& chunk, size_t P, size_t Q)
	{
		VisBwdScratch s;
		const size_t qb = (Q + VIS_PTS_BWD_THREADS - 1) / VIS_PTS_BWD_THREADS;
		obtain(chunk, s.gb, P * GB_STRIDE);
		obtain(chunk, s.duv, 2 * Q);
		obtain(chunk, s.pt_rows, qb * CAM_TERMS);
		obtain(chunk, s.pt_intr, qb * CAM_INTR_TERMS);
		obtain(chunk, s.g_rows, camera_rows_bytes((int)P) / sizeof(float));
		obtain(chunk, s.mean3D, 3 * P);
		obtain(chunk, s.opacity, P);
		return s;
	}
};
}  // namespace mgs

extern "C" {

size_t mgs_visibility_scratch_bytes(int Q, int width, int height)
{
	return required([&](char*& p) { VisScratch::carve(p, (size_t)std::max(Q, 0), num_tiles(width, height)); });
}

int mgs_visibility_views(
	int V, const mgs_view* views, int antialiasing, const mgs_view_intrinsics* intr, const int* ortho,
	const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion,
	int P, int D, int M, int Q, const float* points,
	const float* means3D, const float* shs, const float* colors_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* out_uv, float* out_depth, uint8_t* out_in_view, float* out_T, int debug, void* join_stream)
{
	if (check_antialias(antialiasing) < 0) return MGS_ERR_INVALID_ARG;
	if (V <= 0 || !views) return fail(MGS_ERR_INVALID_ARG, "need at least one view");
	std::vector<Lens> lens;
	if (view_lenses(ortho, fisheye, distortion, V, lens) < 0) return MGS_ERR_INVALID_ARG;
	if (Q < 0) return fail(MGS_ERR_INVALID_ARG, "Q must be >= 0");
	if (Q > 0 && !points) return fail(MGS_ERR_INVALID_ARG, "points are required with Q > 0");
	if (P <= 0) return fail(MGS_ERR_INVALID_ARG, "P must be > 0");
	if (!means3D || !opacities) return fail(MGS_ERR_INVALID_ARG, "means3D/opacities are required");
	if (!colors_precomp && !shs) return fail(MGS_ERR_INVALID_ARG, "provide SHs or precomputed colours (never read: they keep the projection the forward's)");
	if (!cov3D_precomp && (!scales || !rotations)) return fail(MGS_ERR_INVALID_ARG, "provide scales+rotations or a precomputed 3D covariance");
	if (!out_T) return fail(MGS_ERR_INVALID_ARG, "out_T is required");
	for (int v = 0; v < V; v++) {
		const mgs_view& w = views[v];
		if (!w.geometry_state || !w.binning_state || !w.image_state)
			return fail(MGS_ERR_INVALID_ARG, "view: the three state buffers are required");
		if (!w.blend_scratch) return fail(MGS_ERR_INVALID_ARG, "view: blend_scratch (mgs_visibility_scratch_bytes) is required");
		if (!w.viewmatrix || !w.projmatrix || !w.radii) return fail(MGS_ERR_INVALID_ARG, "view: matrices and radii are required");
		if (shs && !colors_precomp && !w.cam_pos) return fail(MGS_ERR_INVALID_ARG, "view: cam_pos is required with SHs");
		if (w.width <= 0 || w.height <= 0 || w.binning_capacity < 0) return fail(MGS_ERR_INVALID_ARG, "view: bad size or capacity");
	}
	if (Q == 0) return 0;
	const Cloud c{ P, D, M, 0, means3D, shs, colors_precomp, nullptr, opacities, scales, scale_modifier, rotations, cov3D_precomp,
		antialiasing };
	cudaStream_t join = reinterpret_cast<cudaStream_t>(join_stream);
	int rc = fork_streams(V, views, join);
	if (rc < 0) return rc;
	// stage by stage across the views, as the lift: the point passes take the blend's place
	for (int phase = 0; phase < 3; phase++) {
		for (int v = 0; v < V; v++) {
			const mgs_view& w = views[v];
			if (phase == 0) rc = enqueue_project(c, w, device_fov(intr, v), lens[v], debug);
			else if (phase == 1) rc = enqueue_binning(c, w, false, debug);
			else {
				cudaStream_t st = reinterpret_cast<cudaStream_t>(w.stream);
				const ViewState s = carve_view(w, P);
				char* sc = w.blend_scratch;
				const VisScratch x = VisScratch::carve(sc, (size_t)Q, s.T);
				const size_t o = (size_t)v * Q;
				VisArgs a = vis_args(w, s, x, flow_cam(w, device_fov(intr, v), lens[v], w.viewmatrix, w.projmatrix), Q, points);
				a.out_uv = out_uv ? out_uv + 2 * o : nullptr; a.out_depth = out_depth ? out_depth + o : nullptr;
				a.out_in_view = out_in_view ? out_in_view + o : nullptr; a.out_T = out_T + o;
				launch_visibility_points(a, st);
				MGS_STAGE("visibility_points");
				// tile ids up to num_tiles (the key of a point outside the view): stable, so a tile's points stay in id order
				launch_tile_sort(x.sort_temp, x.sort_bytes, x.keys, x.keys_sorted, x.idx, x.idx_sorted, Q, higher_msb((uint32_t)s.T), st);
				MGS_STAGE("visibility_sort");
				launch_visibility_group(a, st);
				MGS_STAGE("visibility_group");
				launch_visibility_query(a, st);
				MGS_STAGE("visibility_query");
			}
			if (rc < 0) return rc;
		}
	}
	return join_streams(V, views, join);
}

size_t mgs_visibility_backward_scratch_bytes(int P, int Q)
{
	return required([&](char*& p) { VisBwdScratch::carve(p, (size_t)std::max(P, 0), (size_t)std::max(Q, 0)); });
}

int mgs_visibility_views_backward(
	int V, const mgs_view* views, int antialiasing, const mgs_view_intrinsics* intr, const int* ortho,
	const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion,
	int P, int D, int M, int Q, const float* points,
	const float* means3D, const float* shs, const float* colors_precomp,
	const float* opacities, const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	const float* out_T, const float* dL_dT, const float* dL_duv, const float* dL_ddepth,
	float* dL_dpoints, float* dL_dmean3D, float* dL_dopacity, float* dL_dscale, float* dL_drot, float* dL_dcov3D,
	const mgs_view_camera_grad* cam, int debug, void* join_stream)
{
	if (check_antialias(antialiasing) < 0) return MGS_ERR_INVALID_ARG;
	if (V <= 0 || !views) return fail(MGS_ERR_INVALID_ARG, "need at least one view");
	std::vector<Lens> lens;
	if (view_lenses(ortho, fisheye, distortion, V, lens) < 0) return MGS_ERR_INVALID_ARG;
	if (Q < 0) return fail(MGS_ERR_INVALID_ARG, "Q must be >= 0");
	if (Q > 0 && !points) return fail(MGS_ERR_INVALID_ARG, "points are required with Q > 0");
	if (P <= 0) return fail(MGS_ERR_INVALID_ARG, "P must be > 0");
	if (!means3D || !opacities) return fail(MGS_ERR_INVALID_ARG, "means3D/opacities are required");
	if (!colors_precomp && !shs) return fail(MGS_ERR_INVALID_ARG, "provide SHs or precomputed colours (never read: they keep the projection the forward's)");
	if (!cov3D_precomp && (!scales || !rotations)) return fail(MGS_ERR_INVALID_ARG, "provide scales+rotations or a precomputed 3D covariance");
	if (dL_dT && !out_T) return fail(MGS_ERR_INVALID_ARG, "dL_dT needs out_T, the transmittance the forward wrote");
	if (dL_dcov3D && !cov3D_precomp) return fail(MGS_ERR_INVALID_ARG, "dL_dcov3D needs cov3D_precomp");
	for (int v = 0; v < V; v++) {
		const mgs_view& w = views[v];
		if (!w.geometry_state || !w.binning_state || !w.image_state)
			return fail(MGS_ERR_INVALID_ARG, "view: the three state buffers are required");
		if (!w.blend_scratch) return fail(MGS_ERR_INVALID_ARG, "view: blend_scratch (mgs_visibility_scratch_bytes) is required");
		if (!w.dL_dmean2D)
			return fail(MGS_ERR_INVALID_ARG, "view: dL_dmean2D must carry the backward scratch (mgs_visibility_backward_scratch_bytes)");
		if (!w.viewmatrix || !w.projmatrix || !w.radii) return fail(MGS_ERR_INVALID_ARG, "view: matrices and radii are required");
		if (shs && !colors_precomp && !w.cam_pos) return fail(MGS_ERR_INVALID_ARG, "view: cam_pos is required with SHs");
		if (w.width <= 0 || w.height <= 0 || w.binning_capacity < 0) return fail(MGS_ERR_INVALID_ARG, "view: bad size or capacity");
	}
	if (Q == 0) return 0;
	const Cloud c{ P, D, M, 0, means3D, shs, colors_precomp, nullptr, opacities, scales, scale_modifier, rotations, cov3D_precomp,
		antialiasing };
	bool any_cam = false;
	for (int v = 0; v < V; v++) any_cam |= camera_on(cam, intr, v);
	const bool gauss = dL_dmean3D || dL_dopacity || dL_dscale || dL_drot || dL_dcov3D || any_cam;  // the per-Gaussian chain
	const bool chain = dL_dpoints || any_cam;                                                      // the point chain
	const bool tpath = dL_dT && (gauss || chain);
	cudaStream_t join = reinterpret_cast<cudaStream_t>(join_stream);
	// the views' scratch, carved once
	std::vector<VisBwdScratch> ys(V);
	for (int v = 0; v < V; v++) {
		char* bc = reinterpret_cast<char*>(views[v].dL_dmean2D);
		ys[v] = VisBwdScratch::carve(bc, (size_t)P, (size_t)Q);
	}
	// per view on its stream: the T path's replay into gb and duv
	int rc = fork_streams(V, views, join);
	if (rc < 0) return rc;
	for (int v = 0; v < V; v++) {
		const mgs_view& w = views[v];
		cudaStream_t st = reinterpret_cast<cudaStream_t>(w.stream);
		const VisBwdScratch& y = ys[v];
		if (gauss) MGS_CUDA(cudaMemsetAsync(y.gb, 0, (size_t)P * GB_STRIDE * sizeof(float), st));
		if (!tpath) continue;
		if (chain) MGS_CUDA(cudaMemsetAsync(y.duv, 0, 2 * (size_t)Q * sizeof(float), st));
		const ViewState s = carve_view(w, P);
		char* sc = w.blend_scratch;
		const VisScratch x = VisScratch::carve(sc, (size_t)Q, s.T);
		VisQueryBwdArgs b{};
		b.f = vis_args(w, s, x, flow_cam(w, device_fov(intr, v), lens[v], w.viewmatrix, w.projmatrix), Q, points);
		b.f.out_T = const_cast<float*>(out_T + (size_t)v * Q);  // read only
		b.dL_dT = dL_dT + (size_t)v * Q;
		b.gb = gauss ? y.gb : nullptr;
		b.duv = chain ? y.duv : nullptr;
		launch_visibility_query_bwd(b, st);
		MGS_STAGE("visibility_query_bwd");
	}
	rc = join_streams(V, views, join);
	if (rc < 0) return rc;
	cudaStream_t st = join;
	// the point chain on the join stream, MAX_BWD_VIEWS views per launch; its camera sums are written, the Gaussian path's added
	for (int v0 = 0; chain && v0 < V; v0 += MAX_BWD_VIEWS) {
		VisPointsBwdArgs pa{};
		pa.Q = Q; pa.V = std::min(V - v0, (int)MAX_BWD_VIEWS); pa.points = points; pa.dL_dpoints = dL_dpoints; pa.accumulate = v0 > 0;
		CamReduceArgs cr{};
		for (int u = 0; u < pa.V; u++) {
			const int v = v0 + u;
			const mgs_view& w = views[v];
			VisPointsBwdView& pv = pa.view[u];
			pv.cam = flow_cam(w, device_fov(intr, v), lens[v], w.viewmatrix, w.projmatrix);
			pv.dL_duv = dL_duv ? dL_duv + 2 * (size_t)v * Q : nullptr;
			pv.dL_ddepth = dL_ddepth ? dL_ddepth + (size_t)v * Q : nullptr;
			pv.duv = tpath ? ys[v].duv : nullptr;
			if (!camera_on(cam, intr, v)) continue;
			float* dtf = tan_fov_grad(intr, v);
			pv.cam_rows = ys[v].pt_rows;
			pv.intr_rows = dtf ? ys[v].pt_intr : nullptr;
			const mgs_view_camera_grad* e = cam ? cam + v : nullptr;
			cr.view[cr.V++] = CamReduceView{ pv.cam_rows, ceil_div(Q, VIS_PTS_BWD_THREADS), e ? e->dL_dviewmatrix : nullptr,
				e ? e->dL_dprojmatrix : nullptr, e ? e->dL_dcampos : nullptr, pv.intr_rows, dtf };
		}
		launch_visibility_points_bwd(pa, st);
		if (cr.V > 0) launch_camera_grad_reduce(cr, st);
		MGS_STAGE("visibility_points_bwd");
	}
	if (!gauss) return 0;
	// the per-Gaussian chain of the render's backward (backward_views' stage 2) over the views' gb
	const bool have_sr = c.scales && c.rotations && (dL_dscale || dL_drot);
	for (int v0 = 0; v0 < V; v0 += MAX_BWD_VIEWS) {
		ProjectBwdViewsArgs pb{};
		pb.P = P; pb.D = c.D; pb.M = c.M; pb.V = std::min(V - v0, (int)MAX_BWD_VIEWS);
		pb.means3D = c.means3D; pb.shs = c.shs;
		pb.scales = have_sr ? c.scales : nullptr; pb.rotations = c.rotations; pb.scale_modifier = c.scale_modifier;
		pb.cov3D_precomp = c.cov3D_precomp;
		if (!have_sr && !c.cov3D_precomp) pb.cov3D_precomp = carve_view(views[0], P).geom.cov3D;
		pb.accumulate = v0 > 0;
		// with camera outputs only, the two rows the chain always writes go to view 0's scratch
		pb.dL_dmean3D = dL_dmean3D ? dL_dmean3D : ys[0].mean3D;
		pb.dL_dopacity = dL_dopacity ? dL_dopacity : ys[0].opacity;
		pb.dL_dcov3D = dL_dcov3D; pb.dL_dscale = dL_dscale; pb.dL_drot = dL_drot;
		pb.antialias = c.antialias;
		CamReduceArgs cr{};
		cr.accumulate = 1;  // the point chain wrote every camera output
		for (int u = 0; u < pb.V; u++) {
			const int v = v0 + u;
			const mgs_view& w = views[v];
			const ViewState s = carve_view(w, P);
			pb.view[u] = bwd_view(w, P, nullptr);
			pb.view[u].gb = ys[v].gb;
			if (c.antialias) pb.conic_opacity[u] = s.geom.conic_opacity;
			float* dtf = tan_fov_grad(intr, v);
			pb.intr[u] = ProjectBwdIntr{ device_fov(intr, v), w.width, w.height, dtf ? s.geom.cam_intr : nullptr };
			bwd_lens(pb, u, lens[v]);
			if (!camera_on(cam, intr, v)) continue;
			pb.cam_rows[u] = ys[v].g_rows;
			const mgs_view_camera_grad* e = cam ? cam + v : nullptr;
			cr.view[cr.V++] = CamReduceView{ ys[v].g_rows, (P + 127) / 128, e ? e->dL_dviewmatrix : nullptr,
				e ? e->dL_dprojmatrix : nullptr, e ? e->dL_dcampos : nullptr, pb.intr[u].rows, dtf };
		}
		{ StageTimer t_(ST_PROJECT_BWD, st); launch_project_bwd_views(pb, st); if (cr.V > 0) launch_camera_grad_reduce(cr, st); }
		MGS_STAGE("visibility_project_bwd");
	}
	return 0;
}

}  // extern "C"

namespace mgs {
// the argument checks shared by mgs_camera_rays and its backward; the views' camera models into lens
static int check_rays(int V, const mgs_view* views, const int* ortho, const mgs_view_fisheye* fisheye,
	const mgs_view_distortion* distortion, int Q, const float* pixels, std::vector<Lens>& lens)
{
	if (V <= 0 || !views) return fail(MGS_ERR_INVALID_ARG, "need at least one view");
	if (view_lenses(ortho, fisheye, distortion, V, lens) < 0) return MGS_ERR_INVALID_ARG;
	if (Q < 0) return fail(MGS_ERR_INVALID_ARG, "Q must be >= 0");
	for (int v = 0; v < V; v++) {
		const mgs_view& w = views[v];
		if (!w.viewmatrix || !w.projmatrix) return fail(MGS_ERR_INVALID_ARG, "view: matrices are required");
		if (w.width <= 0 || w.height <= 0) return fail(MGS_ERR_INVALID_ARG, "view: bad size");
		if (!pixels && Q > 0 && (long long)w.width * w.height != Q)
			return fail(MGS_ERR_INVALID_ARG, "pixels NULL (every pixel centre): Q must equal width * height of every view");
	}
	return 0;
}
// the launch over views [v0, v0 + MAX_BWD_VIEWS) of a call with Q rays per view (outputs and cotangents left NULL)
static RaysArgs rays_args(const mgs_view* views, const mgs_view_intrinsics* intr, const std::vector<Lens>& lens, int v0, int V,
	int Q, const float* pixels)
{
	RaysArgs a{};
	a.V = std::min(V - v0, (int)MAX_BWD_VIEWS);
	a.N = Q;
	a.grid_w = views[v0].width;
	a.pixels = pixels ? pixels + 2 * (size_t)v0 * Q : nullptr;
	for (int u = 0; u < a.V; u++) {
		const mgs_view& w = views[v0 + u];
		a.cam[u] = flow_cam(w, device_fov(intr, v0 + u), lens[v0 + u], w.viewmatrix, w.projmatrix);
	}
	return a;
}
}  // namespace mgs

extern "C" {

size_t mgs_camera_rays_scratch_bytes(int Q)
{
	return (size_t)ceil_div(std::max(Q, 0), RAYS_THREADS) * (CAM_TERMS + CAM_INTR_TERMS) * sizeof(float);
}

int mgs_camera_rays(int V, const mgs_view* views, const mgs_view_intrinsics* intr, const int* ortho,
	const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion, int Q, const float* pixels,
	float* out_origin, float* out_direction, uint8_t* out_valid, int debug, void* stream)
{
	std::vector<Lens> lens;
	if (check_rays(V, views, ortho, fisheye, distortion, Q, pixels, lens) < 0) return MGS_ERR_INVALID_ARG;
	if (Q == 0) return 0;
	if (!out_origin || !out_direction || !out_valid)
		return fail(MGS_ERR_INVALID_ARG, "out_origin, out_direction and out_valid are required");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	for (int v0 = 0; v0 < V; v0 += MAX_BWD_VIEWS) {
		RaysArgs a = rays_args(views, intr, lens, v0, V, Q, pixels);
		const size_t o = (size_t)v0 * Q;
		a.origin = out_origin + 3 * o; a.direction = out_direction + 3 * o; a.valid = out_valid + o;
		launch_rays_fwd(a, st);
		MGS_STAGE("camera_rays");
	}
	return 0;
}

int mgs_camera_rays_backward(int V, const mgs_view* views, const mgs_view_intrinsics* intr, const int* ortho,
	const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion, int Q, const float* pixels,
	const float* dL_dorigin, const float* dL_ddirection, float* dL_dpixels, const mgs_view_camera_grad* cam, int debug,
	void* stream)
{
	std::vector<Lens> lens;
	if (check_rays(V, views, ortho, fisheye, distortion, Q, pixels, lens) < 0) return MGS_ERR_INVALID_ARG;
	if (dL_dpixels && !pixels) return fail(MGS_ERR_INVALID_ARG, "dL_dpixels needs pixels (the grid's pixel centres are constants)");
	if (check_camera(cam, intr, V) < 0) return MGS_ERR_INVALID_ARG;
	if (Q == 0) return 0;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const int nrows = ceil_div(Q, RAYS_THREADS);
	for (int v0 = 0; v0 < V; v0 += MAX_BWD_VIEWS) {
		RaysArgs a = rays_args(views, intr, lens, v0, V, Q, pixels);
		const size_t o = (size_t)v0 * Q;
		a.dL_dorigin = dL_dorigin ? dL_dorigin + 3 * o : nullptr;
		a.dL_ddirection = dL_ddirection ? dL_ddirection + 3 * o : nullptr;
		a.dL_dpixels = dL_dpixels ? dL_dpixels + 2 * o : nullptr;
		CamReduceArgs cr{};
		for (int u = 0; u < a.V; u++) {
			const int v = v0 + u;
			if (!camera_on(cam, intr, v)) continue;
			float* dtf = tan_fov_grad(intr, v);
			a.cam_rows[u] = cam[v].scratch;
			a.intr_rows[u] = dtf ? cam[v].scratch + (size_t)nrows * CAM_TERMS : nullptr;
			cr.view[cr.V++] = CamReduceView{ a.cam_rows[u], nrows, cam[v].dL_dviewmatrix, cam[v].dL_dprojmatrix, cam[v].dL_dcampos,
				a.intr_rows[u], dtf };
		}
		if (!a.dL_dpixels && cr.V == 0) continue;
		launch_rays_bwd(a, st);
		if (cr.V > 0) launch_camera_grad_reduce(cr, st);
		MGS_STAGE("camera_rays_backward");
	}
	return 0;
}

int mgs_backward_views(
	int V, const mgs_view* views,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* dL_dmean3D, float* dL_dopacity, float* dL_dcolor, float* dL_dfeature, float* dL_dcov3D, float* dL_dsh,
	float* dL_dscale, float* dL_drot, int shared_mean2D, int accumulate, int stages, int debug, void* join_stream)
{
	return mgs_backward_views_alpha(V, views, nullptr, P, D, M, F, means3D, shs, colors_precomp, feature_precomp, scales, scale_modifier,
		rotations, cov3D_precomp, dL_dmean3D, dL_dopacity, dL_dcolor, dL_dfeature, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, shared_mean2D,
		accumulate, stages, debug, join_stream);
}

int mgs_backward_views_alpha(
	int V, const mgs_view* views, const mgs_view_alpha* alpha,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* dL_dmean3D, float* dL_dopacity, float* dL_dcolor, float* dL_dfeature, float* dL_dcov3D, float* dL_dsh,
	float* dL_dscale, float* dL_drot, int shared_mean2D, int accumulate, int stages, int debug, void* join_stream)
{
	return mgs_backward_views_depth_mask(V, views, alpha, nullptr, P, D, M, F, means3D, shs, colors_precomp, feature_precomp, scales,
		scale_modifier, rotations, cov3D_precomp, dL_dmean3D, dL_dopacity, dL_dcolor, dL_dfeature, dL_dcov3D, dL_dsh, dL_dscale, dL_drot,
		shared_mean2D, accumulate, stages, debug, join_stream);
}

int mgs_backward_views_depth_mask(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* dL_dmean3D, float* dL_dopacity, float* dL_dcolor, float* dL_dfeature, float* dL_dcov3D, float* dL_dsh,
	float* dL_dscale, float* dL_drot, int shared_mean2D, int accumulate, int stages, int debug, void* join_stream)
{
	return mgs_backward_views_aa(V, views, alpha, depth_mask, 0, P, D, M, F, means3D, shs, colors_precomp, feature_precomp, scales,
		scale_modifier, rotations, cov3D_precomp, dL_dmean3D, dL_dopacity, dL_dcolor, dL_dfeature, dL_dcov3D, dL_dsh, dL_dscale, dL_drot,
		shared_mean2D, accumulate, stages, debug, join_stream);
}

int mgs_backward_views_aa(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* dL_dmean3D, float* dL_dopacity, float* dL_dcolor, float* dL_dfeature, float* dL_dcov3D, float* dL_dsh,
	float* dL_dscale, float* dL_drot, int shared_mean2D, int accumulate, int stages, int debug, void* join_stream)
{
	return mgs_backward_views_ssim(V, views, alpha, depth_mask, antialiasing, nullptr, P, D, M, F, means3D, shs, colors_precomp,
		feature_precomp, scales, scale_modifier, rotations, cov3D_precomp, dL_dmean3D, dL_dopacity, dL_dcolor, dL_dfeature, dL_dcov3D,
		dL_dsh, dL_dscale, dL_drot, shared_mean2D, accumulate, stages, debug, join_stream);
}

int mgs_backward_views_ssim(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* dL_dmean3D, float* dL_dopacity, float* dL_dcolor, float* dL_dfeature, float* dL_dcov3D, float* dL_dsh,
	float* dL_dscale, float* dL_drot, int shared_mean2D, int accumulate, int stages, int debug, void* join_stream)
{
	return mgs_backward_views_cam(V, views, alpha, depth_mask, antialiasing, ssim, nullptr, P, D, M, F, means3D, shs, colors_precomp,
		feature_precomp, scales, scale_modifier, rotations, cov3D_precomp, dL_dmean3D, dL_dopacity, dL_dcolor, dL_dfeature, dL_dcov3D,
		dL_dsh, dL_dscale, dL_drot, shared_mean2D, accumulate, stages, debug, join_stream);
}

int mgs_backward_views_cam(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim, const mgs_view_camera_grad* cam,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* dL_dmean3D, float* dL_dopacity, float* dL_dcolor, float* dL_dfeature, float* dL_dcov3D, float* dL_dsh,
	float* dL_dscale, float* dL_drot, int shared_mean2D, int accumulate, int stages, int debug, void* join_stream)
{
	return mgs_backward_views_intr(V, views, alpha, depth_mask, antialiasing, ssim, cam, nullptr, P, D, M, F, means3D, shs,
		colors_precomp, feature_precomp, scales, scale_modifier, rotations, cov3D_precomp, dL_dmean3D, dL_dopacity, dL_dcolor,
		dL_dfeature, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, shared_mean2D, accumulate, stages, debug, join_stream);
}

int mgs_backward_views_intr(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim, const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* dL_dmean3D, float* dL_dopacity, float* dL_dcolor, float* dL_dfeature, float* dL_dcov3D, float* dL_dsh,
	float* dL_dscale, float* dL_drot, int shared_mean2D, int accumulate, int stages, int debug, void* join_stream)
{
	return mgs_backward_views_median(V, views, alpha, depth_mask, antialiasing, ssim, cam, intr, nullptr, P, D, M, F, means3D, shs,
		colors_precomp, feature_precomp, scales, scale_modifier, rotations, cov3D_precomp, dL_dmean3D, dL_dopacity, dL_dcolor,
		dL_dfeature, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, shared_mean2D, accumulate, stages, debug, join_stream);
}

int mgs_backward_views_median(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim, const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, const mgs_view_median* median,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* dL_dmean3D, float* dL_dopacity, float* dL_dcolor, float* dL_dfeature, float* dL_dcov3D, float* dL_dsh,
	float* dL_dscale, float* dL_drot, int shared_mean2D, int accumulate, int stages, int debug, void* join_stream)
{
	return mgs_backward_views_normal(V, views, alpha, depth_mask, antialiasing, ssim, cam, intr, median, nullptr, P, D, M, F, means3D,
		shs, colors_precomp, feature_precomp, scales, scale_modifier, rotations, cov3D_precomp, dL_dmean3D, dL_dopacity, dL_dcolor,
		dL_dfeature, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, shared_mean2D, accumulate, stages, debug, join_stream);
}

int mgs_backward_views_normal(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim, const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, const mgs_view_median* median,
	const mgs_view_normal* normal,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* dL_dmean3D, float* dL_dopacity, float* dL_dcolor, float* dL_dfeature, float* dL_dcov3D, float* dL_dsh,
	float* dL_dscale, float* dL_drot, int shared_mean2D, int accumulate, int stages, int debug, void* join_stream)
{
	return mgs_backward_views_ortho(V, views, alpha, depth_mask, antialiasing, ssim, cam, intr, median, normal, nullptr, P, D, M, F,
		means3D, shs, colors_precomp, feature_precomp, scales, scale_modifier, rotations, cov3D_precomp, dL_dmean3D, dL_dopacity,
		dL_dcolor, dL_dfeature, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, shared_mean2D, accumulate, stages, debug, join_stream);
}

int mgs_backward_views_ortho(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim, const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, const mgs_view_median* median,
	const mgs_view_normal* normal, const int* ortho,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* dL_dmean3D, float* dL_dopacity, float* dL_dcolor, float* dL_dfeature, float* dL_dcov3D, float* dL_dsh,
	float* dL_dscale, float* dL_drot, int shared_mean2D, int accumulate, int stages, int debug, void* join_stream)
{
	return mgs_backward_views_fisheye(V, views, alpha, depth_mask, antialiasing, ssim, cam, intr, median, normal, ortho, nullptr, P, D,
		M, F, means3D, shs, colors_precomp, feature_precomp, scales, scale_modifier, rotations, cov3D_precomp, dL_dmean3D, dL_dopacity,
		dL_dcolor, dL_dfeature, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, shared_mean2D, accumulate, stages, debug, join_stream);
}

int mgs_backward_views_fisheye(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim, const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, const mgs_view_median* median,
	const mgs_view_normal* normal, const int* ortho, const mgs_view_fisheye* fisheye,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* dL_dmean3D, float* dL_dopacity, float* dL_dcolor, float* dL_dfeature, float* dL_dcov3D, float* dL_dsh,
	float* dL_dscale, float* dL_drot, int shared_mean2D, int accumulate, int stages, int debug, void* join_stream)
{
	return mgs_backward_views_distorted(V, views, alpha, depth_mask, antialiasing, ssim, cam, intr, median, normal, ortho,
		fisheye, nullptr, P, D, M, F, means3D, shs, colors_precomp, feature_precomp, scales, scale_modifier, rotations, cov3D_precomp,
		dL_dmean3D, dL_dopacity, dL_dcolor, dL_dfeature, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, shared_mean2D, accumulate, stages,
		debug, join_stream);
}

int mgs_backward_views_distorted(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim, const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, const mgs_view_median* median,
	const mgs_view_normal* normal, const int* ortho, const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* dL_dmean3D, float* dL_dopacity, float* dL_dcolor, float* dL_dfeature, float* dL_dcov3D, float* dL_dsh,
	float* dL_dscale, float* dL_drot, int shared_mean2D, int accumulate, int stages, int debug, void* join_stream)
{
	return mgs_backward_views_planar(V, views, alpha, depth_mask, antialiasing, ssim, cam, intr, median, normal, ortho, fisheye,
		distortion, 0, P, D, M, F, means3D, shs, colors_precomp, feature_precomp, scales, scale_modifier, rotations, cov3D_precomp,
		dL_dmean3D, dL_dopacity, dL_dcolor, dL_dfeature, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, shared_mean2D, accumulate, stages,
		debug, join_stream);
}

int mgs_backward_views_planar(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim, const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, const mgs_view_median* median,
	const mgs_view_normal* normal, const int* ortho, const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion,
	int planar_depth,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* dL_dmean3D, float* dL_dopacity, float* dL_dcolor, float* dL_dfeature, float* dL_dcov3D, float* dL_dsh,
	float* dL_dscale, float* dL_drot, int shared_mean2D, int accumulate, int stages, int debug, void* join_stream)
{
	return mgs_backward_views_flow(V, views, alpha, depth_mask, antialiasing, ssim, cam, intr, median, normal, ortho, fisheye,
		distortion, planar_depth, nullptr, nullptr, nullptr, P, D, M, F, means3D, shs, colors_precomp, feature_precomp, scales,
		scale_modifier, rotations, cov3D_precomp, dL_dmean3D, dL_dopacity, dL_dcolor, dL_dfeature, dL_dcov3D, dL_dsh, dL_dscale,
		dL_drot, shared_mean2D, accumulate, stages, debug, join_stream);
}

int mgs_backward_views_flow(
	int V, const mgs_view* views, const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing,
	const mgs_view_ssim* ssim, const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, const mgs_view_median* median,
	const mgs_view_normal* normal, const int* ortho, const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion,
	int planar_depth, const mgs_view_flow* flow, const float* flow_means3D, float* dL_dflow_means3D,
	int P, int D, int M, int F,
	const float* means3D, const float* shs, const float* colors_precomp, const float* feature_precomp,
	const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp,
	float* dL_dmean3D, float* dL_dopacity, float* dL_dcolor, float* dL_dfeature, float* dL_dcov3D, float* dL_dsh,
	float* dL_dscale, float* dL_drot, int shared_mean2D, int accumulate, int stages, int debug, void* join_stream)
{
	if (check_antialias(antialiasing) < 0) return MGS_ERR_INVALID_ARG;
	if (V > 0 && views && check_planar(planar_depth, normal, V) < 0) return MGS_ERR_INVALID_ARG;
	if (V > 0 && views && (check_flow_call(flow, V, planar_depth, normal) < 0 || check_flow(flow, flow_means3D, 0, V, depth_mask) < 0))
		return MGS_ERR_INVALID_ARG;
	if (!(stages & 3)) return fail(MGS_ERR_INVALID_ARG, "stages must name the blend stage (1), the per-Gaussian stage (2) or both (3)");
	if (V <= 0 || !views) return fail(MGS_ERR_INVALID_ARG, "need at least one view");
	std::vector<Lens> lens;
	if (view_lenses(ortho, fisheye, distortion, V, lens) < 0) return MGS_ERR_INVALID_ARG;
	if (P <= 0) return fail(MGS_ERR_INVALID_ARG, "P must be > 0");
	if (!means3D || !dL_dmean3D || !dL_dopacity) return fail(MGS_ERR_INVALID_ARG, "means3D, dL_dmean3D and dL_dopacity are required");
	if (F < 0 || F > MGS_MAX_FEATURE_CHANNELS) return fail(MGS_ERR_UNSUPPORTED, bad_width_msg);
	if (F > 0 && (!feature_precomp || !dL_dfeature)) F = 0;
	for (int v = 0; v < V; v++) {
		int rc = check_bwd_view(views[v], F > 0);
		if (rc == 0) rc = check_depth_mask(views[v], depth_mask ? depth_mask + v : nullptr, false);
		if (rc == 0) rc = check_ssim(views[v], ssim ? ssim + v : nullptr, false);
		if (rc == 0) rc = check_median(median ? median + v : nullptr);
		if (rc == 0) rc = check_normal(views[v], normal ? normal + v : nullptr, scales, rotations, cov3D_precomp, depth_mask ? depth_mask + v : nullptr);
		if (rc < 0) return rc;
	}
	if (check_camera(cam, intr, V) < 0) return MGS_ERR_INVALID_ARG;
	const Cloud c{ P, D, M, F, means3D, shs, colors_precomp, feature_precomp, nullptr, scales, scale_modifier, rotations, cov3D_precomp,
		antialiasing, planar_depth };
	return backward_views(V, views, alpha, depth_mask, ssim, cam, intr, median, normal, lens.data(), c, dL_dmean3D, dL_dopacity, dL_dcolor, dL_dfeature, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, nullptr,
		shared_mean2D, accumulate, stages, debug, reinterpret_cast<cudaStream_t>(join_stream), flow, flow_means3D, dL_dflow_means3D);
}

int mgs_forward_clouds(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views, int D, int M, int F,
	float scale_modifier, int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_clouds_alpha(B, clouds, view_offsets, views, nullptr, D, M, F, scale_modifier, prefiltered, debug, join_stream);
}

int mgs_forward_clouds_alpha(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views, const mgs_view_alpha* alpha,
	int D, int M, int F, float scale_modifier, int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_clouds_depth_mask(B, clouds, view_offsets, views, alpha, nullptr, D, M, F, scale_modifier, prefiltered, debug,
		join_stream);
}

int mgs_forward_clouds_depth_mask(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int D, int M, int F, float scale_modifier, int prefiltered,
	int debug, void* join_stream)
{
	return mgs_forward_clouds_aa(B, clouds, view_offsets, views, alpha, depth_mask, 0, D, M, F, scale_modifier, prefiltered, debug,
		join_stream);
}

int mgs_forward_clouds_aa(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, int D, int M, int F, float scale_modifier,
	int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_clouds_ssim(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, nullptr, D, M, F, scale_modifier,
		prefiltered, debug, join_stream);
}

int mgs_forward_clouds_ssim(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim, int D, int M,
	int F, float scale_modifier, int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_clouds_intr(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, ssim, nullptr, D, M, F,
		scale_modifier, prefiltered, debug, join_stream);
}

int mgs_forward_clouds_intr(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim,
	const mgs_view_intrinsics* intr, int D, int M, int F, float scale_modifier, int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_clouds_median(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, ssim, intr, nullptr, D, M, F,
		scale_modifier, prefiltered, debug, join_stream);
}

int mgs_forward_clouds_median(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim,
	const mgs_view_intrinsics* intr, const mgs_view_median* median, int D, int M, int F, float scale_modifier, int prefiltered,
	int debug, void* join_stream)
{
	return mgs_forward_clouds_normal(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, ssim, intr, median, nullptr, D, M,
		F, scale_modifier, prefiltered, debug, join_stream);
}

int mgs_forward_clouds_normal(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim,
	const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal, int D, int M, int F,
	float scale_modifier, int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_clouds_ortho(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, ssim, intr, median, normal, nullptr,
		D, M, F, scale_modifier, prefiltered, debug, join_stream);
}

int mgs_forward_clouds_ortho(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim,
	const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal, const int* ortho, int D, int M,
	int F, float scale_modifier, int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_clouds_fisheye(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, ssim, intr, median, normal, ortho,
		nullptr, D, M, F, scale_modifier, prefiltered, debug, join_stream);
}

int mgs_forward_clouds_fisheye(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim,
	const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal, const int* ortho,
	const mgs_view_fisheye* fisheye, int D, int M, int F, float scale_modifier, int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_clouds_distorted(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, ssim, intr, median,
		normal, ortho, fisheye, nullptr, D, M, F, scale_modifier, prefiltered, debug, join_stream);
}

int mgs_forward_clouds_distorted(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim,
	const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal, const int* ortho,
	const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion, int D, int M, int F, float scale_modifier, int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_clouds_planar(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, ssim, intr, median, normal, ortho,
		fisheye, distortion, 0, D, M, F, scale_modifier, prefiltered, debug, join_stream);
}

int mgs_forward_clouds_planar(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim,
	const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal, const int* ortho,
	const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion, int planar_depth, int D, int M, int F, float scale_modifier, int prefiltered, int debug, void* join_stream)
{
	return mgs_forward_clouds_flow(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, ssim, intr, median, normal, ortho,
		fisheye, distortion, planar_depth, nullptr, nullptr, D, M, F, scale_modifier, prefiltered, debug, join_stream);
}

// the next-frame means of cloud b (flow_clouds: B entries or NULL)
static const float* cloud_next(const mgs_cloud_flow* fc, int b) { return fc ? fc[b].means3D : nullptr; }

int mgs_forward_clouds_flow(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim,
	const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal, const int* ortho,
	const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion, int planar_depth, const mgs_view_flow* flow,
	const mgs_cloud_flow* flow_clouds, int D, int M, int F, float scale_modifier, int prefiltered, int debug, void* join_stream)
{
	(void)prefiltered;
	if (check_antialias(antialiasing) < 0) return MGS_ERR_INVALID_ARG;
	int rc = check_clouds(B, clouds, view_offsets, views);
	if (rc < 0) return rc;
	std::vector<Lens> lens;
	if (view_lenses(ortho, fisheye, distortion, view_offsets[B], lens) < 0) return MGS_ERR_INVALID_ARG;
	if (check_planar(planar_depth, normal, view_offsets[B]) < 0) return MGS_ERR_INVALID_ARG;
	if (check_flow_call(flow, view_offsets[B], planar_depth, normal) < 0) return MGS_ERR_INVALID_ARG;
	for (int b = 0; b < B; b++)
		if (check_flow(flow, cloud_next(flow_clouds, b), view_offsets[b], view_offsets[b + 1], depth_mask) < 0) return MGS_ERR_INVALID_ARG;
	if (F < 0 || F > MGS_MAX_FEATURE_CHANNELS || !blend_supported(F)) return fail(MGS_ERR_UNSUPPORTED, bad_width_msg);
	for (int b = 0; b < B; b++) {
		const mgs_cloud& k = clouds[b];
		if (!k.means3D || !k.opacities) return fail(MGS_ERR_INVALID_ARG, "cloud: means3D/opacities are required");
		if (!k.colors_precomp && !k.shs) return fail(MGS_ERR_INVALID_ARG, "cloud: provide SHs or precomputed colours");
		if (!k.cov3D_precomp && (!k.scales || !k.rotations))
			return fail(MGS_ERR_INVALID_ARG, "cloud: provide scales+rotations or a precomputed 3D covariance");
		for (int v = view_offsets[b]; v < view_offsets[b + 1]; v++) {
			rc = check_fwd_view(views[v], !k.colors_precomp);
			if (rc == 0) rc = check_depth_mask(views[v], depth_mask ? depth_mask + v : nullptr, true);
			if (rc == 0) rc = check_ssim(views[v], ssim ? ssim + v : nullptr, true);
			if (rc == 0) rc = check_median(median ? median + v : nullptr);
			if (rc == 0)
				rc = check_normal(views[v], normal ? normal + v : nullptr, k.scales, k.rotations, k.cov3D_precomp,
					depth_mask ? depth_mask + v : nullptr);
			if (rc < 0) return rc;
		}
	}
	const int V = view_offsets[B];
	std::vector<mgs_view_normal> flow_planes;
	const mgs_view_normal* blend_nm = flow_blend_planes(flow, V, normal, flow_planes);
	cudaStream_t join = reinterpret_cast<cudaStream_t>(join_stream);
	rc = fork_streams(V, views, join);
	if (rc < 0) return rc;
	// stage by stage across the views of every cloud, as in mgs_forward_views
	for (int phase = 0; phase < 3; phase++) {
		for (int b = 0; b < B; b++) {
			const Cloud c = cloud_of(clouds[b], D, M, F, scale_modifier, antialiasing, planar_depth);
			for (int v = view_offsets[b]; v < view_offsets[b + 1]; v++) {
				rc = phase == 0 ? enqueue_project(c, views[v], device_fov(intr, v), lens[v], debug)
					: phase == 1 ? enqueue_binning(c, views[v], false, debug)
					: enqueue_blend_fwd(c, views[v], alpha ? alpha[v].out_alpha : nullptr, depth_mask ? depth_mask + v : nullptr,
						median ? median + v : nullptr, blend_nm ? blend_nm + v : nullptr, debug);
				if (rc == 0 && phase == 0) rc = enqueue_normals_fwd(c, views[v], normal ? normal + v : nullptr, debug);
				if (rc == 0 && phase == 0)
					rc = enqueue_flow_fwd(c, views[v], flow ? flow + v : nullptr, cloud_next(flow_clouds, b), device_fov(intr, v), lens[v], debug);
				if (rc == 0 && phase == 2) rc = enqueue_ssim_fwd(views[v], ssim ? ssim + v : nullptr, debug);
				if (rc < 0) return rc;
			}
		}
	}
	return join_streams(V, views, join);
}

int mgs_backward_clouds(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views, int D, int M, int F,
	float scale_modifier, int accumulate, int debug, void* join_stream)
{
	return mgs_backward_clouds_alpha(B, clouds, view_offsets, views, nullptr, D, M, F, scale_modifier, accumulate, debug, join_stream);
}

int mgs_backward_clouds_alpha(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views, const mgs_view_alpha* alpha,
	int D, int M, int F, float scale_modifier, int accumulate, int debug, void* join_stream)
{
	return mgs_backward_clouds_depth_mask(B, clouds, view_offsets, views, alpha, nullptr, D, M, F, scale_modifier, accumulate, debug,
		join_stream);
}

int mgs_backward_clouds_depth_mask(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int D, int M, int F, float scale_modifier, int accumulate,
	int debug, void* join_stream)
{
	return mgs_backward_clouds_aa(B, clouds, view_offsets, views, alpha, depth_mask, 0, D, M, F, scale_modifier, accumulate, debug,
		join_stream);
}

int mgs_backward_clouds_aa(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, int D, int M, int F, float scale_modifier,
	int accumulate, int debug, void* join_stream)
{
	return mgs_backward_clouds_ssim(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, nullptr, D, M, F, scale_modifier,
		accumulate, debug, join_stream);
}

int mgs_backward_clouds_ssim(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim, int D, int M,
	int F, float scale_modifier, int accumulate, int debug, void* join_stream)
{
	return mgs_backward_clouds_cam(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, ssim, nullptr, D, M, F,
		scale_modifier, accumulate, debug, join_stream);
}

int mgs_backward_clouds_cam(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim,
	const mgs_view_camera_grad* cam, int D, int M, int F, float scale_modifier, int accumulate, int debug, void* join_stream)
{
	return mgs_backward_clouds_intr(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, ssim, cam, nullptr, D, M, F,
		scale_modifier, accumulate, debug, join_stream);
}

int mgs_backward_clouds_intr(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim,
	const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, int D, int M, int F, float scale_modifier, int accumulate,
	int debug, void* join_stream)
{
	return mgs_backward_clouds_median(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, ssim, cam, intr, nullptr, D, M,
		F, scale_modifier, accumulate, debug, join_stream);
}

int mgs_backward_clouds_median(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim,
	const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, const mgs_view_median* median, int D, int M, int F,
	float scale_modifier, int accumulate, int debug, void* join_stream)
{
	return mgs_backward_clouds_normal(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, ssim, cam, intr, median, nullptr,
		D, M, F, scale_modifier, accumulate, debug, join_stream);
}

int mgs_backward_clouds_normal(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim,
	const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal,
	int D, int M, int F, float scale_modifier, int accumulate, int debug, void* join_stream)
{
	return mgs_backward_clouds_ortho(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, ssim, cam, intr, median, normal,
		nullptr, D, M, F, scale_modifier, accumulate, debug, join_stream);
}

int mgs_backward_clouds_ortho(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim,
	const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal,
	const int* ortho, int D, int M, int F, float scale_modifier, int accumulate, int debug, void* join_stream)
{
	return mgs_backward_clouds_fisheye(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, ssim, cam, intr, median, normal,
		ortho, nullptr, D, M, F, scale_modifier, accumulate, debug, join_stream);
}

int mgs_backward_clouds_fisheye(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim,
	const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal,
	const int* ortho, const mgs_view_fisheye* fisheye, int D, int M, int F, float scale_modifier, int accumulate, int debug,
	void* join_stream)
{
	return mgs_backward_clouds_distorted(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, ssim, cam, intr, median,
		normal, ortho, fisheye, nullptr, D, M, F, scale_modifier, accumulate, debug, join_stream);
}

int mgs_backward_clouds_distorted(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim,
	const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal,
	const int* ortho, const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion, int D, int M, int F, float scale_modifier, int accumulate, int debug,
	void* join_stream)
{
	return mgs_backward_clouds_planar(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, ssim, cam, intr, median, normal,
		ortho, fisheye, distortion, 0, D, M, F, scale_modifier, accumulate, debug, join_stream);
}

int mgs_backward_clouds_planar(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim,
	const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal,
	const int* ortho, const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion, int planar_depth, int D, int M, int F, float scale_modifier, int accumulate, int debug,
	void* join_stream)
{
	return mgs_backward_clouds_flow(B, clouds, view_offsets, views, alpha, depth_mask, antialiasing, ssim, cam, intr, median, normal,
		ortho, fisheye, distortion, planar_depth, nullptr, nullptr, D, M, F, scale_modifier, accumulate, debug, join_stream);
}

int mgs_backward_clouds_flow(int B, const mgs_cloud* clouds, const int* view_offsets, const mgs_view* views,
	const mgs_view_alpha* alpha, const mgs_view_depth_mask* depth_mask, int antialiasing, const mgs_view_ssim* ssim,
	const mgs_view_camera_grad* cam, const mgs_view_intrinsics* intr, const mgs_view_median* median, const mgs_view_normal* normal,
	const int* ortho, const mgs_view_fisheye* fisheye, const mgs_view_distortion* distortion, int planar_depth,
	const mgs_view_flow* flow, const mgs_cloud_flow* flow_clouds, int D, int M, int F,
	float scale_modifier, int accumulate, int debug, void* join_stream)
{
	if (check_antialias(antialiasing) < 0) return MGS_ERR_INVALID_ARG;
	int rc = check_clouds(B, clouds, view_offsets, views);
	if (rc < 0) return rc;
	std::vector<Lens> lens;
	if (view_lenses(ortho, fisheye, distortion, view_offsets[B], lens) < 0) return MGS_ERR_INVALID_ARG;
	if (check_planar(planar_depth, normal, view_offsets[B]) < 0) return MGS_ERR_INVALID_ARG;
	if (check_flow_call(flow, view_offsets[B], planar_depth, normal) < 0) return MGS_ERR_INVALID_ARG;
	for (int b = 0; b < B; b++)
		if (check_flow(flow, cloud_next(flow_clouds, b), view_offsets[b], view_offsets[b + 1], depth_mask) < 0) return MGS_ERR_INVALID_ARG;
	if (F < 0 || F > MGS_MAX_FEATURE_CHANNELS) return fail(MGS_ERR_UNSUPPORTED, bad_width_msg);
	for (int b = 0; b < B; b++) {
		const mgs_cloud& k = clouds[b];
		if (!k.means3D || !k.dL_dmean3D || !k.dL_dopacity)
			return fail(MGS_ERR_INVALID_ARG, "cloud: means3D, dL_dmean3D and dL_dopacity are required");
		if (k.shs && !k.dL_dsh)
			return fail(MGS_ERR_INVALID_ARG, "cloud: dL_dsh is required with SHs (it carries the view-direction term of dL_dmean3D)");
		for (int v = view_offsets[b]; v < view_offsets[b + 1]; v++) {
			rc = check_bwd_view(views[v], F > 0 && k.feature);
			if (rc == 0) rc = check_depth_mask(views[v], depth_mask ? depth_mask + v : nullptr, false);
			if (rc == 0) rc = check_ssim(views[v], ssim ? ssim + v : nullptr, false);
			if (rc == 0) rc = check_median(median ? median + v : nullptr);
			if (rc == 0)
				rc = check_normal(views[v], normal ? normal + v : nullptr, k.scales, k.rotations, k.cov3D_precomp,
					depth_mask ? depth_mask + v : nullptr);
			if (rc < 0) return rc;
		}
	}
	const int V = view_offsets[B];
	if (check_camera(cam, intr, V) < 0) return MGS_ERR_INVALID_ARG;
	cudaStream_t join = reinterpret_cast<cudaStream_t>(join_stream);
	for (int b = 0; b < B; b++) {
		const mgs_cloud& k = clouds[b];
		if (F > 0 && k.feature && k.dL_dfeature && !accumulate)
			MGS_CUDA(cudaMemsetAsync(k.dL_dfeature, 0, (size_t)k.P * F * sizeof(float), join));
	}
	std::vector<mgs_view_normal> flow_planes;
	const mgs_view_normal* blend_nm = flow_blend_planes(flow, V, normal, flow_planes);
	rc = fork_streams(V, views, join);
	if (rc < 0) return rc;
	for (int b = 0; b < B; b++) {
		const Cloud c = cloud_of(clouds[b], D, M, F, scale_modifier, antialiasing, planar_depth);
		for (int v = view_offsets[b]; v < view_offsets[b + 1]; v++) {
			mgs_view w = views[v];
			rc = enqueue_ssim_bwd(w, ssim ? ssim + v : nullptr, debug);
			if (rc == 0)
				rc = enqueue_blend_bwd(c, w, clouds[b].dL_dfeature, alpha ? alpha[v].dL_dpix_alpha : nullptr,
					depth_mask ? depth_mask + v : nullptr, median ? median + v : nullptr, blend_nm ? blend_nm + v : nullptr, debug);
			if (rc < 0) return rc;
		}
	}
	rc = join_streams(V, views, join);
	if (rc < 0) return rc;

	// per-Gaussian stage on `join`: launches of at most MAX_BWD_VIEWS views that pack whole clouds; a cloud with more views
	// spans launches, and its later launches add to what the earlier ones wrote
	const cudaStream_t st = join;
	// the flow planes' backward first, one launch per cloud and MAX_BWD_VIEWS of its views: it adds to the blend-stage records
	// the per-Gaussian stage reads, and its camera reduce writes the camera outputs the per-Gaussian stage's reduce adds to
	bool flow_bwd = false, flow_reduced = false;
	for (int v = 0; v < V; v++) flow_bwd |= flow_on(flow, v) && flow[v].dL_dpix_flow;
	for (int b = 0; b < B && flow_bwd; b++) {
		const Cloud c = cloud_of(clouds[b], D, M, F, scale_modifier, antialiasing);
		for (int v0 = view_offsets[b]; v0 < view_offsets[b + 1]; v0 += MAX_BWD_VIEWS) {
			bool red = false;
			rc = enqueue_flow_bwd(c, views, flow, cloud_next(flow_clouds, b), flow_clouds ? flow_clouds[b].dL_dmeans3D : nullptr, cam, intr,
				lens.data(), v0, std::min(view_offsets[b + 1] - v0, (int)MAX_BWD_VIEWS),
				(accumulate || v0 > view_offsets[b]) ? 1 : 0, accumulate ? 1 : 0, debug, st, red);
			if (rc < 0) return rc;
			flow_reduced |= red;
		}
	}
	// a view's camera rows are summed by the reduce behind the one launch that holds the view
	ProjectBwdCloudsDistArgs pb{};
	pb.D = D; pb.M = M; pb.scale_modifier = scale_modifier; pb.antialias = antialiasing;
	CamReduceArgs cr{};
	cr.accumulate = (accumulate || flow_reduced) ? 1 : 0;
	int nv = 0;  // views in pb
	auto flush = [&]() -> int {
		if (pb.B == 0) return 0;
		{ StageTimer t_(ST_PROJECT_BWD, st); launch_project_bwd_clouds(pb, st); if (cr.V > 0) launch_camera_grad_reduce(cr, st); }
		MGS_STAGE("project_bwd");
		pb.B = 0; nv = 0; cr.V = 0; pb.ortho = 0; pb.fisheye = 0; pb.distorted = 0;
		for (float*& r : pb.cam_rows) r = nullptr;
		for (ProjectBwdIntr& ki : pb.intr) ki = ProjectBwdIntr{};
		for (int u = 0; u < MAX_BWD_VIEWS; u++) { pb.pl_g[u] = nullptr; pb.pl_q[u] = nullptr; pb.pl_mean[u] = nullptr; }
		return 0;
	};
	for (int b = 0; b < B; b++) {
		const mgs_cloud& k = clouds[b];
		const bool have_sr = k.scales && k.rotations && (k.dL_dscale || k.dL_drot);  // as in backward_views
		for (int v0 = view_offsets[b]; v0 < view_offsets[b + 1]; v0 += MAX_BWD_VIEWS) {
			const int n = std::min(view_offsets[b + 1] - v0, (int)MAX_BWD_VIEWS);
			if (nv + n > MAX_BWD_VIEWS) {
				rc = flush();
				if (rc < 0) return rc;
			}
			ProjectBwdCloud& pc = pb.cloud[pb.B++];
			pc.P = k.P; pc.V = n; pc.view0 = nv;
			pc.means3D = k.means3D; pc.shs = k.shs; pc.scales = have_sr ? k.scales : nullptr; pc.rotations = k.rotations;
			// gradients w.r.t. scale/rotation not requested: the forward's own covariance (any view's copy) serves
			pc.cov3D_precomp = (have_sr || k.cov3D_precomp) ? k.cov3D_precomp : carve_view(views[view_offsets[b]], k.P).geom.cov3D;
			pc.accumulate = (accumulate || v0 > view_offsets[b]) ? 1 : 0;
			pc.dL_dmean3D = k.dL_dmean3D; pc.dL_dopacity = k.dL_dopacity; pc.dL_dcolor = k.dL_dcolor; pc.dL_dcov3D = k.dL_dcov3D;
			pc.dL_dsh = k.dL_dsh; pc.dL_dscale = k.dL_dscale; pc.dL_drot = k.dL_drot;
			for (int u = 0; u < n; u++) {
				pb.view[nv + u] = bwd_view(views[v0 + u], k.P, views[v0 + u].dL_dmean2D);
				pb.conic_opacity[nv + u] = antialiasing ? carve_view(views[v0 + u], k.P).geom.conic_opacity : nullptr;
				camera_view(cam, intr, views[v0 + u], v0 + u, k.P, pb.cam_rows[nv + u], pb.intr[nv + u], cr);
				bwd_lens(pb, nv + u, lens[v0 + u]);
				planar_view(cloud_of(k, D, M, F, scale_modifier, antialiasing, planar_depth), views[v0 + u], pb.pl_g[nv + u], pb.pl_q[nv + u],
					pb.pl_mean[nv + u]);
			}
			nv += n;
		}
	}
	rc = flush();
	if (rc < 0) return rc;
	// the normal planes' share of every cloud's dL_drot, behind the launches that wrote it: one launch per cloud and
	// MAX_BWD_VIEWS of its views
	for (int b = 0; b < B && normal; b++) {
		const Cloud c = cloud_of(clouds[b], D, M, F, scale_modifier, antialiasing);
		for (int v0 = view_offsets[b]; v0 < view_offsets[b + 1]; v0 += MAX_BWD_VIEWS) {
			rc = enqueue_normals_bwd(c, views, normal, v0, std::min(view_offsets[b + 1] - v0, (int)MAX_BWD_VIEWS), clouds[b].dL_drot,
				debug, st);
			if (rc < 0) return rc;
		}
	}
	return 0;
}

int mgs_loss_heads(int V, int F, int N, const float* color, const float* feature, const float* target_color,
	const float* target_feature, float* cot_color, float* cot_feature, float* loss_acc, void* stream)
{
	if (V <= 0 || N <= 0 || F < 0) return fail(MGS_ERR_INVALID_ARG, "bad V/N/F");
	if (!color || !target_color || !cot_color || !loss_acc) return fail(MGS_ERR_INVALID_ARG, "color, target_color, cot_color and loss_acc are required");
	const bool emb = F > 0 && feature && target_feature;
	if (emb && !cot_feature) return fail(MGS_ERR_INVALID_ARG, "cot_feature is required with features");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	MGS_CUDA(cudaMemsetAsync(loss_acc, 0, (size_t)V * 2 * sizeof(float), st));
	launch_loss_heads(V, emb ? F : 0, N, color, emb ? feature : nullptr, target_color, emb ? target_feature : nullptr, cot_color, cot_feature,
		loss_acc, st);
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess) return fail(MGS_ERR_CUDA, std::string("loss_heads: ") + cudaGetErrorString(e));
	return 0;
}

static int check_ssim_planes(int V, int C, int H, int W)
{
	if (V <= 0 || C <= 0 || H <= 0 || W <= 0) return fail(MGS_ERR_INVALID_ARG, "bad V/C/H/W");
	if ((long long)V * C > 65535) return fail(MGS_ERR_INVALID_ARG, "V * C must be at most 65535");
	return 0;
}

int mgs_ssim(int V, int C, int H, int W, const float* x, const float* g, float* ssim_terms, float* loss_acc, void* stream)
{
	if (check_ssim_planes(V, C, H, W) < 0) return MGS_ERR_INVALID_ARG;
	if (!x || !g || !ssim_terms || !loss_acc) return fail(MGS_ERR_INVALID_ARG, "x, g, ssim_terms and loss_acc are required");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	MGS_CUDA(cudaMemsetAsync(loss_acc, 0, (size_t)V * 2 * sizeof(float), st));
	{ StageTimer t_(ST_SSIM_FWD, st); launch_ssim_fwd(V, C, H, W, x, g, ssim_terms, loss_acc, 2, st); }
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess) return fail(MGS_ERR_CUDA, std::string("ssim: ") + cudaGetErrorString(e));
	return 0;
}

int mgs_ssim_backward(int V, int C, int H, int W, const float* x, const float* g, const float* ssim_terms, const float* scale,
	const float* cot_in, float* cot_out, void* stream)
{
	if (check_ssim_planes(V, C, H, W) < 0) return MGS_ERR_INVALID_ARG;
	if (!x || !g || !ssim_terms || !cot_out) return fail(MGS_ERR_INVALID_ARG, "x, g, ssim_terms and cot_out are required");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	{ StageTimer t_(ST_SSIM_BWD, st); launch_ssim_bwd(V, C, H, W, x, g, ssim_terms, scale, cot_in, nullptr, cot_out, nullptr, st); }
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess) return fail(MGS_ERR_CUDA, std::string("ssim_backward: ") + cudaGetErrorString(e));
	return 0;
}

int mgs_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix, uint8_t* present, void* stream)
{
	(void)projmatrix;
	if (P < 0) return fail(MGS_ERR_INVALID_ARG, "bad P");
	if (P == 0) return 0;
	if (!means3D || !viewmatrix || !present) return fail(MGS_ERR_INVALID_ARG, "required pointer is NULL");
	launch_mark_visible(P, means3D, viewmatrix, present, reinterpret_cast<cudaStream_t>(stream));
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess) return fail(MGS_ERR_CUDA, cudaGetErrorString(e));
	return 0;
}

static int activate_common(ActivateArgs& a, int P, int F, const float* means, const float* d_means, const float* rot, const float* d_rot,
	const float* scales, const float* d_scales, const float* opac, const float* feature,
	int scale_mode, float scale_max, int opacity_mode, int rot_normalize, int feature_normalize)
{
	if (P < 0 || F < 0) return fail(MGS_ERR_INVALID_ARG, "bad P or F");
	if (scale_mode < 0 || scale_mode > 1 || opacity_mode < 0 || opacity_mode > 1) return fail(MGS_ERR_INVALID_ARG, "unknown activation mode");
	memset(&a, 0, sizeof(a));
	a.P = P; a.F = F;
	a.means = means; a.d_means = d_means; a.rot = rot; a.d_rot = d_rot; a.scales = scales; a.d_scales = d_scales;
	a.opac = opac; a.feature = F > 0 ? feature : nullptr;
	a.scale_mode = scale_mode; a.scale_max = scale_max; a.opacity_mode = opacity_mode;
	a.rot_normalize = rot_normalize != 0; a.feature_normalize = feature_normalize != 0;
	return 0;
}

int mgs_activate(int P, int F,
	const float* means, const float* d_means, const float* rot, const float* d_rot,
	const float* scales, const float* d_scales, const float* opac, const float* feature,
	int scale_mode, float scale_max, int opacity_mode, int rot_normalize, int feature_normalize,
	float* out_means, float* out_rot, float* out_scales, float* out_opac, float* out_feature,
	void* stream)
{
	ActivateArgs a;
	int rc = activate_common(a, P, F, means, d_means, rot, d_rot, scales, d_scales, opac, feature,
		scale_mode, scale_max, opacity_mode, rot_normalize, feature_normalize);
	if (rc) return rc;
	if (P == 0) return 0;
	if ((out_means && !means) || (out_rot && !rot) || (out_scales && !scales) || (out_opac && !opac) || (out_feature && F > 0 && !feature))
		return fail(MGS_ERR_INVALID_ARG, "an output was requested for an input that is NULL");
	a.o_means = out_means; a.o_rot = out_rot; a.o_scales = out_scales; a.o_opac = out_opac; a.o_feature = F > 0 ? out_feature : nullptr;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	{ StageTimer t_(ST_ACTIVATE_FWD, st); launch_activate_fwd(a, st); }
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess) return fail(MGS_ERR_CUDA, std::string("activate: ") + cudaGetErrorString(e));
	return 0;
}

int mgs_activate_backward(int P, int F,
	const float* means, const float* d_means, const float* rot, const float* d_rot,
	const float* scales, const float* d_scales, const float* opac, const float* feature,
	int scale_mode, float scale_max, int opacity_mode, int rot_normalize, int feature_normalize,
	const float* g_means, const float* g_rot, const float* g_scales, const float* g_opac, const float* g_feature,
	float* dL_dmeans, float* dL_dd_means, float* dL_drot, float* dL_dd_rot,
	float* dL_dscales, float* dL_dd_scales, float* dL_dopac, float* dL_dfeature,
	void* stream)
{
	ActivateArgs a;
	int rc = activate_common(a, P, F, means, d_means, rot, d_rot, scales, d_scales, opac, feature,
		scale_mode, scale_max, opacity_mode, rot_normalize, feature_normalize);
	if (rc) return rc;
	if (P == 0) return 0;
	if ((g_rot && !rot) || (g_scales && scale_mode == 1 && !scales) || (g_opac && opacity_mode == 1 && !opac) || (g_feature && F > 0 && !feature))
		return fail(MGS_ERR_INVALID_ARG, "a gradient was given for an input that is NULL");
	a.g_means = g_means; a.g_rot = g_rot; a.g_scales = g_scales; a.g_opac = g_opac; a.g_feature = F > 0 ? g_feature : nullptr;
	a.dL_means = dL_dmeans; a.dL_dmeans = dL_dd_means; a.dL_rot = dL_drot; a.dL_drot = dL_dd_rot;
	a.dL_scales = dL_dscales; a.dL_dscales = dL_dd_scales; a.dL_opac = dL_dopac; a.dL_feature = F > 0 ? dL_dfeature : nullptr;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	{ StageTimer t_(ST_ACTIVATE_BWD, st); launch_activate_bwd(a, st); }
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess) return fail(MGS_ERR_CUDA, std::string("activate_backward: ") + cudaGetErrorString(e));
	return 0;
}

int mgs_profile_enable(int on)
{
	std::lock_guard<std::mutex> lk(g_prof_mu);
	g_prof_on = on != 0;
	return 0;
}

// Sums the recorded stage durations (ms) and launch counts since the last call, then clears them.
// total_ms / counts: arrays of mgs_profile_num_stages() entries.  Synchronises on the recorded events.
int mgs_profile_num_stages(void) { return ST_COUNT; }
const char* mgs_profile_stage_name(int i)
{
	static const char* names[ST_COUNT] = { "project_fwd", "depth_sort", "scan", "emit_tiles", "tile_sort", "ranges_pack", "block_lists", "blend_fwd", "blend_bwd", "project_bwd", "activate_fwd", "activate_bwd", "ssim_fwd", "ssim_bwd" };
	return (i >= 0 && i < ST_COUNT) ? names[i] : "";
}
int mgs_profile_read(float* total_ms, int* counts)
{
	std::lock_guard<std::mutex> lk(g_prof_mu);
	for (int i = 0; i < ST_COUNT; i++) { total_ms[i] = 0.f; counts[i] = 0; }
	for (auto& e : g_prof_evts) {
		float ms = 0.f;
		cudaEventSynchronize(e.b);
		if (cudaEventElapsedTime(&ms, e.a, e.b) == cudaSuccess) { total_ms[e.stage] += ms; counts[e.stage]++; }
		cudaEventDestroy(e.a); cudaEventDestroy(e.b);
	}
	g_prof_evts.clear();
	return 0;
}

int mgs_state_array(const char* which_state, const char* name, char* state, int a0, int a1, void** out_ptr)
{
	if (!which_state || !name || !state || !out_ptr) return fail(MGS_ERR_INVALID_ARG, "NULL argument");
	const std::string w(which_state), n(name);
	void* p = nullptr;
	if (w == "geometry") {
		GeomState g = GeomState::carve(state, (size_t)a0);
		if (n == "depths") p = g.depths; else if (n == "means2D") p = g.means2D; else if (n == "cov3D") p = g.cov3D;
		else if (n == "conic_opacity") p = g.conic_opacity; else if (n == "rgbd") p = g.rgbd;
		else if (n == "tiles_touched") p = g.tiles_touched; else if (n == "point_offsets") p = g.point_offsets;
		else if (n == "depth_order") p = g.order;
		else if (n == "clamped") p = g.clamped; else if (n == "extent") p = g.extent;
		else if (n == "nrm") { float4* q; obtain(state, q, (size_t)a0); p = q; }  // a state sized by mgs_geometry_state_bytes_normal
	} else if (w == "binning") {
		BinState b = BinState::carve(state, (size_t)a0);
		if (n == "point_list") p = b.point_list; else if (n == "tile_ids") p = b.tile_keys;
		else if (n == "point_list_unsorted") p = b.point_list_unsorted; else if (n == "tile_ids_unsorted") p = b.tile_keys_unsorted;
		else if (n == "records") p = b.recs; else if (n == "pixel_masks") p = b.pix_mask;
		else if (n == "block_lists") p = b.block_list; else if (n == "block_bits") p = b.block_bits;
	} else if (w == "image") {
		ImageState s = ImageState::carve(state, (size_t)a0 * a1, num_tiles(a0, a1));
		if (n == "final_T") p = s.final_T; else if (n == "n_contrib") p = s.n_contrib; else if (n == "ranges") p = s.ranges;
		else if (n == "tile_order") p = s.tile_order; else if (n == "block_count") p = s.block_count;
		else if (n == "block_nwalk") p = s.block_nwalk;
	} else if (w == "scratch") {
		float* gb; float* gn;
		carve_scratch(state, a0, gb, gn);
		if (n == "gb") p = gb; else if (n == "gn") p = gn;
	}
	if (!p) return fail(MGS_ERR_INVALID_ARG, "unknown state array " + w + "/" + n);
	*out_ptr = p;
	return 0;
}

}  // extern "C"

int mgs_field_query(
	mgs_alloc_fn state_alloc, void* state_user, mgs_alloc_fn pair_alloc, void* pair_user,
	int Q, int P, int C,
	const float* points, const float* means3D, const float* scales, const float* rotations, const float* opacities,
	const float* features, int channel_first, float* out_density, float* out_features, int debug, void* stream)
{
	using namespace mgs;
	if (C < 0 || C > MGS_MAX_FEATURE_CHANNELS) return fail(MGS_ERR_UNSUPPORTED, bad_width_msg);
	if (Q <= 0 || P <= 0) return fail(MGS_ERR_INVALID_ARG, "Q and P must be > 0");
	if (!state_alloc || !pair_alloc) return fail(MGS_ERR_INVALID_ARG, "allocator callbacks are required");
	if (!points || !means3D || !scales || !rotations || !opacities || !out_density)
		return fail(MGS_ERR_INVALID_ARG, "points, means3D, scales, rotations, opacities and out_density are required");
	if (C > 0 && (!features || !out_features)) return fail(MGS_ERR_INVALID_ARG, "features and out_features are required with C > 0");
	if (channel_first != 0 && channel_first != 1) return fail(MGS_ERR_INVALID_ARG, "channel_first must be 0 or 1");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	char* state = state_alloc(state_user, field_state_bytes(Q, P));
	if (!state) return fail(MGS_ERR_ALLOC, "query state allocation failed");
	unsigned long long npairs = 0;
	MGS_CUDA(field_front(state, Q, P, points, means3D, scales, rotations, opacities, &npairs, st));
	MGS_STAGE("field_front");
	MGS_CUDA(cudaStreamSynchronize(st));  // the one host read of the query: the pair count sizes the bin lists
	if (npairs > 0x7fffffffull) return fail(MGS_ERR_UNSUPPORTED, "more than 2^31-1 (bin, Gaussian) pairs");
	char* pairs = pair_alloc(pair_user, field_pair_state_bytes((long long)npairs, Q));
	if (!pairs) return fail(MGS_ERR_ALLOC, "pair state allocation failed");
	MGS_CUDA(field_pairs(state, pairs, Q, P, (long long)npairs, st));
	MGS_STAGE("field_pairs");
	MGS_CUDA(field_forward(state, pairs, Q, P, C, points, features, channel_first, out_density, out_features, st));
	MGS_STAGE("field_forward");
	return (int)npairs;
}

int mgs_field_query_backward(
	const char* state, const char* pair_state, int Q, int P, int C,
	const float* points, const float* scales, const float* rotations, const float* features, int channel_first,
	const float* dL_ddensity, const float* dL_dout_features,
	float* dL_dpoints, float* dL_dmeans3D, float* dL_dscales, float* dL_drotations, float* dL_dopacities, float* dL_dfeature,
	int debug, void* stream)
{
	using namespace mgs;
	if (C < 0 || C > MGS_MAX_FEATURE_CHANNELS) return fail(MGS_ERR_UNSUPPORTED, bad_width_msg);
	if (Q <= 0 || P <= 0) return fail(MGS_ERR_INVALID_ARG, "Q and P must be > 0");
	if (!state || !pair_state || !points || !scales || !rotations)
		return fail(MGS_ERR_INVALID_ARG, "state, pair_state, points, scales and rotations are required");
	if (C > 0 && dL_dout_features && !features) return fail(MGS_ERR_INVALID_ARG, "features are required with dL_dout_features");
	if (channel_first != 0 && channel_first != 1) return fail(MGS_ERR_INVALID_ARG, "channel_first must be 0 or 1");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	MGS_CUDA(field_backward(const_cast<char*>(state), const_cast<char*>(pair_state), Q, P, C, points, features, scales, rotations,
		channel_first, dL_ddensity, dL_dout_features, dL_dpoints, dL_dmeans3D, dL_dscales, dL_drotations, dL_dopacities, dL_dfeature, st));
	MGS_STAGE("field_backward");
	return 0;
}

size_t mgs_knn_state_bytes(int N, int Q)
{
	size_t bytes = 0;
	const cudaError_t e = mgs::knn_state_bytes(std::max(N, 0), std::max(Q, 0), &bytes);
	if (e != cudaSuccess) {
		mgs::fail(MGS_ERR_CUDA, std::string("mgs_knn_state_bytes: ") + cudaGetErrorString(e));
		return 0;
	}
	return bytes;
}

int mgs_knn(void* state, int N, int Q, int k, const float* points, const float* queries, long long* out_index, float* out_dist2,
	int debug, void* stream)
{
	using namespace mgs;
	if (k > KNN_MAX_K) return fail(MGS_ERR_UNSUPPORTED, "k must be at most 32");
	if (k < 1) return fail(MGS_ERR_INVALID_ARG, "k must be >= 1");
	if (N < 0 || Q < 0) return fail(MGS_ERR_INVALID_ARG, "N and Q must be >= 0");
	if (Q == 0) return 0;
	if (!queries && Q != N) return fail(MGS_ERR_INVALID_ARG, "without queries the points are the queries: Q must equal N");
	if (!state || !out_index || !out_dist2) return fail(MGS_ERR_INVALID_ARG, "state, out_index and out_dist2 are required");
	if (N > 0 && !points) return fail(MGS_ERR_INVALID_ARG, "points are required with N > 0");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	MGS_CUDA(knn_run(static_cast<char*>(state), N, Q, k, points, queries, out_index, out_dist2, st));
	MGS_STAGE("knn");
	return 0;
}

size_t mgs_neighbour_reg_state_bytes(int P, int /*k*/)
{
	return mgs::neighbour_reg_state_bytes(std::max(P, 0));
}

// the argument checks both directions share (include/mgs_rasterizer.h, mgs_neighbour_reg)
static int neighbour_reg_args(const char* where, void* state, int P, int k, const float* xyz, const float* rot,
	const float* xyz_next, const float* rot_next, const long long* index, const float* weight, const void* loss)
{
	using namespace mgs;
	const std::string w(where);
	if (k > NEIGHBOUR_REG_MAX_K) return fail(MGS_ERR_UNSUPPORTED, w + ": k must be at most 32");
	if (k < 1) return fail(MGS_ERR_INVALID_ARG, w + ": k must be >= 1");
	if (P < 0) return fail(MGS_ERR_INVALID_ARG, w + ": P must be >= 0");
	if (!state || !loss) return fail(MGS_ERR_INVALID_ARG, w + ": state and the [3] loss buffer are required");
	if (P > 0 && (!xyz || !rot || !xyz_next || !rot_next || !index || !weight))
		return fail(MGS_ERR_INVALID_ARG, w + ": xyz, rot, xyz_next, rot_next, index and weight are required with P > 0");
	return 0;
}

int mgs_neighbour_reg(void* state, int P, int k, const float* xyz, const float* rot, const float* xyz_next,
	const float* rot_next, const long long* index, const float* weight, float* out_loss, int debug, void* stream)
{
	using namespace mgs;
	if (int r = neighbour_reg_args("mgs_neighbour_reg", state, P, k, xyz, rot, xyz_next, rot_next, index, weight, out_loss))
		return r;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	MGS_CUDA(neighbour_reg_forward(state, P, k, xyz, rot, xyz_next, rot_next, index, weight, out_loss, st));
	MGS_STAGE("neighbour_reg");
	return 0;
}

int mgs_neighbour_reg_backward(void* state, int P, int k, const float* xyz, const float* rot, const float* xyz_next,
	const float* rot_next, const long long* index, const float* weight, const float* dL_dloss, float* dL_dxyz, float* dL_drot,
	float* dL_dxyz_next, float* dL_drot_next, int debug, void* stream)
{
	using namespace mgs;
	if (int r = neighbour_reg_args("mgs_neighbour_reg_backward", state, P, k, xyz, rot, xyz_next, rot_next, index, weight,
	                               dL_dloss))
		return r;
	if (P == 0) return 0;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	MGS_CUDA(neighbour_reg_backward(state, P, k, rot, rot_next, index, weight, dL_dloss, dL_dxyz, dL_drot, dL_dxyz_next,
	                                dL_drot_next, st));
	MGS_STAGE("neighbour_reg_bwd");
	return 0;
}
