// TSDF fusion (include/mgs_rasterizer.h, mgs_tsdf_fuse): depth images of V views into a truncated signed-distance volume.
//
// One thread per voxel, z fastest, so that the volume's loads and stores coalesce.  A launch takes a chunk of up to
// TSDF_CHUNK views: its CTAs first copy each view's matrices, field of view and lens into shared memory, then every thread
// keeps its voxel's tsdf, weight and colour in registers across the chunk's views in order, and writes them back once, and
// only where a view updated them.  The per-view map and cull are screen_mean's (camera.cuh), the projection's own, so a
// voxel lands on the pixel a Gaussian at its centre would.  Every update is written with _rn intrinsics: nothing is
// contracted into an FMA, and the result does not depend on how the views are split into calls.
#include "camera.cuh"

namespace mgs {

constexpr int TSDF_THREADS = 256;

// a chunk view as staged in shared memory: the matrices copied, the field of view resolved (device or host value)
struct TsdfSmView {
	float vm[16], pm[16];
	float tanx, tany;
	int W, H;
	Lens lens;
};

template <int CB>
__global__ void __launch_bounds__(TSDF_THREADS) tsdf_fuse_kernel(const TsdfArgs a)
{
	__shared__ TsdfSmView sv[TSDF_CHUNK];
	for (int q = threadIdx.x; q < a.V * 32; q += TSDF_THREADS) {
		const int u = q >> 5, e = q & 31;
		if (e < 16) sv[u].vm[e] = a.cam[u].viewmatrix[e];
		else sv[u].pm[e - 16] = a.cam[u].projmatrix[e - 16];
		if (e == 0) {
			const ViewFov f = view_fov(a.cam[u]);
			sv[u].tanx = f.tanx; sv[u].tany = f.tany;
			sv[u].W = a.cam[u].W; sv[u].H = a.cam[u].H;
			sv[u].lens = a.cam[u].lens;
		}
	}
	__syncthreads();
	const size_t N = (size_t)a.X * a.Y * a.Z;
	const size_t n = (size_t)blockIdx.x * TSDF_THREADS + threadIdx.x;
	if (n >= N) return;
	const int k = (int)(n % a.Z), j = (int)((n / a.Z) % a.Y), i = (int)(n / ((size_t)a.Y * a.Z));
	// voxel_centres' point: lo + (i + 1/2) step in double, rounded once to float
	const V3 p = { (float)__dadd_rn(a.lo[0], __dmul_rn(__dadd_rn((double)i, 0.5), a.step[0])),
	               (float)__dadd_rn(a.lo[1], __dmul_rn(__dadd_rn((double)j, 0.5), a.step[1])),
	               (float)__dadd_rn(a.lo[2], __dmul_rn(__dadd_rn((double)k, 0.5), a.step[2])) };
	float ts = a.tsdf[n], w = a.weight[n];
	float col[CB > 0 ? CB : 1];
#pragma unroll
	for (int c = 0; c < CB; c++)
		if (c < a.C) col[c] = a.color_volume[(size_t)c * N + n];
	bool touched = false;
	const size_t plane = (size_t)a.H * a.W;
	for (int u = 0; u < a.V; u++) {
		const TsdfSmView& s = sv[u];
		const FlowCam cam{ s.vm, s.pm, nullptr, s.tanx, s.tany, s.W, s.H, s.lens };
		float px, py;
		if (!screen_mean(cam, p, px, py)) continue;
		const float z = xform4x3(p, s.vm).z;  // screen_mean's t.z
		if (!(px >= -0.5f && px < a.W - 0.5f && py >= -0.5f && py < a.H - 0.5f)) continue;
		// px + 0.5 may round up to W at the last ulp below W - 0.5: the pixel stays the last column (as point_visibility)
		const int pi = min((int)floorf(px + 0.5f), a.W - 1), pj = min((int)floorf(py + 0.5f), a.H - 1);
		const size_t pix = (size_t)pj * a.W + pi;
		const float d = __ldg(a.depth + (size_t)u * plane + pix);
		if (!isfinite(d) || !(d > 0.f)) continue;
		const float sd = __fsub_rn(d, z);
		if (sd < -a.trunc) continue;
		const float f = fminf(1.0f, __fdiv_rn(sd, a.trunc));
		const float w1 = __fadd_rn(w, 1.0f);
		ts = __fdiv_rn(__fadd_rn(__fmul_rn(ts, w), f), w1);
#pragma unroll
		for (int c = 0; c < CB; c++)
			if (c < a.C) {
				const float x = __ldg(a.color + ((size_t)u * a.C + c) * plane + pix);
				col[c] = __fdiv_rn(__fadd_rn(__fmul_rn(col[c], w), x), w1);
			}
		w = w1;
		touched = true;
	}
	if (!touched) return;  // a voxel no view updates keeps its bits
	a.tsdf[n] = ts;
	a.weight[n] = w;
#pragma unroll
	for (int c = 0; c < CB; c++)
		if (c < a.C) a.color_volume[(size_t)c * N + n] = col[c];
}

void launch_tsdf_fuse(const TsdfArgs& a, cudaStream_t s)
{
	const size_t N = (size_t)a.X * a.Y * a.Z;
	if (a.V <= 0 || N == 0) return;
	const unsigned grid = (unsigned)((N + TSDF_THREADS - 1) / TSDF_THREADS);
	if (a.C == 0) tsdf_fuse_kernel<0><<<grid, TSDF_THREADS, 0, s>>>(a);
	else if (a.C <= 4) tsdf_fuse_kernel<4><<<grid, TSDF_THREADS, 0, s>>>(a);
	else if (a.C <= 8) tsdf_fuse_kernel<8><<<grid, TSDF_THREADS, 0, s>>>(a);
	else if (a.C <= 16) tsdf_fuse_kernel<16><<<grid, TSDF_THREADS, 0, s>>>(a);
	else tsdf_fuse_kernel<32><<<grid, TSDF_THREADS, 0, s>>>(a);
}

}  // namespace mgs
