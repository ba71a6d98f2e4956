// Tile binning: produces, per 16x16 tile, the list of Gaussian instances in (depth, Gaussian id) order -- the SAME
// order as the reference's 64-bit (tile << 32 | depth) radix sort (rasterizer_impl.cu:70-111 duplicateWithKeys,
// :303-311 SortPairs, :116-138 identifyTileRanges), obtained with a fraction of its memory traffic:
//
//   reference : emit R (u64 key, u32 id) pairs, LSD-sort 32+ceil(log2 T) bits  -> 5-6 passes over 12-byte pairs of R
//   here      : 1. sort the P Gaussians once by their 32-bit depth bits (stable, ids ascending among equal depths)
//               2. scan tiles_touched in that order, emit (tile id, Gaussian id) per instance in that order
//               3. ONE stable 8-bit pass (two above 256 tiles) over 8-byte pairs of R by tile id
//   Stability of both sorts makes the result identical to sorting by (tile, depth bits) with ties in ascending
//   Gaussian id -- exactly what the reference's stable sort of row-major emitted keys yields.  The test-suite
//   reconstructs the reference's 64-bit keys from (tile, depth bits of the id) and compares bit for bit.
//
// The device-wide scan and radix passes are the CUDA toolkit's CUB primitives (a library call, as in the
// reference; BASELINE.json's north_star asks for "cub-style radix sort").  The emit and ranges+pack kernels are
// hand-written; the latter also gathers the per-instance 32-byte blend record into tile order and decides which 8x4
// pixel blocks of its tile each instance can reach, and block_lists turns that into one work list per block, so a blend
// warp gathers only the records that can reach its pixels.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/iterator/transform_input_iterator.cuh>
#include "mgs_common.cuh"
#include "mgs_kernels.h"

namespace mgs {

struct GatherTiles {
	const uint32_t* tiles_touched;
	__host__ __device__ __forceinline__ uint32_t operator()(const uint32_t& idx) const { return tiles_touched[idx]; }
};
using GatherIt = cub::TransformInputIterator<uint32_t, GatherTiles, const uint32_t*>;

size_t depth_sort_temp_bytes(int P)
{
	size_t bytes = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
		(const uint32_t*)nullptr, (uint32_t*)nullptr, P);
	return bytes;
}

size_t scan_temp_bytes(int P)
{
	size_t bytes = 0;
	GatherIt it(nullptr, GatherTiles{ nullptr });
	cub::DeviceScan::InclusiveSum(nullptr, bytes, it, (uint32_t*)nullptr, P);
	return bytes;
}

size_t tile_sort_temp_bytes(int R)
{
	size_t bytes = 0;
	cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
		(const uint32_t*)nullptr, (uint32_t*)nullptr, R);
	return bytes;
}

// depth bits of visible Gaussians are positive floats (z > 0.2), so their unsigned order is their numeric order;
// culled Gaussians carry +inf and sort last
void launch_depth_sort(void* temp, size_t temp_bytes, const uint32_t* depth_bits, uint32_t* depth_bits_sorted,
	const uint32_t* iota, uint32_t* order, int P, cudaStream_t s)
{
	cub::DeviceRadixSort::SortPairs(temp, temp_bytes, depth_bits, depth_bits_sorted, iota, order, P, 0, 32, s);
}

// inclusive sum of tiles_touched taken in depth order
void launch_scan_sorted(void* temp, size_t temp_bytes, const uint32_t* order, const uint32_t* tiles_touched, uint32_t* offsets,
	int P, cudaStream_t s)
{
	GatherIt it(order, GatherTiles{ tiles_touched });
	cub::DeviceScan::InclusiveSum(temp, temp_bytes, it, offsets, P, s);
}

// One thread per Gaussian in depth order; emits its tile rect row-major (y outer, x inner).  The instance arrays hold
// `capacity` slots: when the caller sized them without knowing the instance count (no host read-back), instances
// beyond the capacity -- the farthest Gaussians, emission is in depth order -- are dropped and status[1] is raised.
__global__ void __launch_bounds__(256) emit_tiles_kernel(int P, const uint32_t* __restrict__ order,
	const float2* __restrict__ means2D, const uint32_t* __restrict__ offsets, const int* __restrict__ radii,
	uint32_t grid_x, uint32_t grid_y, uint32_t* __restrict__ tile_keys, uint32_t* __restrict__ values, uint32_t capacity,
	int* __restrict__ status)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	if (i == P - 1 && status) {
		const uint32_t R = offsets[P - 1];
		status[0] = (int)R;
		status[1] = R > capacity ? 1 : 0;
	}
	const uint32_t g = order[i];
	const int radius = radii[g];
	if (radius <= 0) return;
	uint32_t off = (i == 0) ? 0 : offsets[i - 1];
	const float2 xy = means2D[g];
	uint2 rmin, rmax;
	tile_rect(xy.x, xy.y, radius, rmin, rmax, grid_x, grid_y);
	for (uint32_t y = rmin.y; y < rmax.y; y++) {
		for (uint32_t x = rmin.x; x < rmax.x; x++) {
			if (off < capacity) {
				tile_keys[off] = y * grid_x + x;
				values[off] = g;
			}
			off++;
		}
	}
}

void launch_emit_tiles(int P, const uint32_t* order, const float2* means2D, const uint32_t* offsets, const int* radii,
	uint32_t grid_x, uint32_t grid_y, uint32_t* tile_keys, uint32_t* values, uint32_t capacity, int* status, cudaStream_t s)
{
	if (P > 0) emit_tiles_kernel<<<ceil_div(P, 256), 256, 0, s>>>(P, order, means2D, offsets, radii, grid_x, grid_y, tile_keys, values, capacity, status);
}

__global__ void __launch_bounds__(256) fill_tail_kernel(const uint32_t* __restrict__ offsets, int P, uint32_t capacity, uint32_t last_tile,
	uint32_t* __restrict__ tile_keys, uint32_t* __restrict__ values)
{
	const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= capacity || idx < offsets[P - 1]) return;
	tile_keys[idx] = last_tile;
	values[idx] = 0xffffffffu;
}

void launch_fill_tail(const uint32_t* offsets, int P, uint32_t capacity, uint32_t last_tile, uint32_t* tile_keys, uint32_t* values, cudaStream_t s)
{
	if (capacity > 0) fill_tail_kernel<<<ceil_div((int)capacity, 256), 256, 0, s>>>(offsets, P, capacity, last_tile, tile_keys, values);
}

void launch_tile_sort(void* temp, size_t temp_bytes, const uint32_t* keys_in, uint32_t* keys_out,
	const uint32_t* vals_in, uint32_t* vals_out, int R, int end_bit, cudaStream_t s)
{
	cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys_in, keys_out, vals_in, vals_out, R, 0, end_bit, s);
}

// Which of the eight 8x4 pixel blocks of tile (tx, ty) can the footprint {alpha >= 1/255} of a Gaussian reach?
// alpha = min(0.99, o exp(-q/2)), q(d) = ca dx^2 + 2 cb dx dy + cc dy^2, d = mean - pixel: the pair can contribute iff
// q(d) <= 2 ln(255 o) =: 2 tau.  Per block the minimum of q over the rectangle of its pixel centres is compared with
// 2 tau (exact up to the slack folded into tau): 0 if the mean lies inside, else the smallest of the four edge minima
// (a convex quadratic restricted to a segment).  ext = the axis-aligned half-extent from the projection kernel
// (-1: never contributes, 1e30: conic degenerate, do not cull), used as the cheap first test.
__device__ __forceinline__ uint32_t block_mask(float gx, float gy, float ca, float cb, float cc, float op, float2 ext, int tx, int ty)
{
	if (ext.x < 0.f) return 0u;
	if (ext.x > 1e29f) return 0xffu;
	const float tau2 = 2.0f * (logf(255.0f * op) * 1.0005f + 1e-3f);  // same slack as the extent (project.cu)
	const float icc = 1.0f / cc, ica = 1.0f / ca;                      // ca, cc > 0 whenever ext is finite
	uint32_t mask = 0;
#pragma unroll
	for (int s = 0; s < 8; s++) {
		const float x0 = (float)(tx * TILE_X + (s & 1) * WARP_BX), x1 = x0 + (float)(WARP_BX - 1);
		const float y0 = (float)(ty * TILE_Y + (s >> 1) * WARP_BY), y1 = y0 + (float)(WARP_BY - 1);
		if (!((gx + ext.x >= x0) && (gx - ext.x <= x1) && (gy + ext.y >= y0) && (gy - ext.y <= y1))) continue;
		// d ranges over [dxl, dxh] x [dyl, dyh]
		const float dxl = gx - x1, dxh = gx - x0, dyl = gy - y1, dyh = gy - y0;
		float qmin = 0.f;
		if (!(dxl <= 0.f && dxh >= 0.f && dyl <= 0.f && dyh >= 0.f)) {
			qmin = 3.0e38f;
#pragma unroll
			for (int e = 0; e < 2; e++) {
				const float X = e ? dxh : dxl;
				const float dy = fminf(fmaxf(-cb * X * icc, dyl), dyh);
				qmin = fminf(qmin, ca * X * X + 2.0f * cb * X * dy + cc * dy * dy);
				const float Y = e ? dyh : dyl;
				const float dx = fminf(fmaxf(-cb * Y * ica, dxl), dxh);
				qmin = fminf(qmin, ca * dx * dx + 2.0f * cb * dx * Y + cc * Y * Y);
			}
		}
		if (qmin <= tau2 * 1.0001f + 1e-4f) mask |= 1u << s;
	}
	return mask;
}

// One thread per sorted instance: tile boundary detection + gather of the 32-byte blend record; the block mask also goes
// to the compact block_bits array that block_lists_kernel reads.
__global__ void __launch_bounds__(256) ranges_pack_kernel(const uint32_t* __restrict__ R_dev, int capacity, int grid_x,
	const uint32_t* __restrict__ tile_keys,
	const uint32_t* __restrict__ point_list, const float2* __restrict__ means2D,
	const float4* __restrict__ conic_opacity, const float2* __restrict__ extent,
	uint2* __restrict__ ranges, InstRec* __restrict__ recs, uint8_t* __restrict__ block_bits)
{
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	const int R = (int)min(*R_dev, (uint32_t)capacity);
	if (idx >= R) return;
	const uint32_t currtile = tile_keys[idx];
	if (idx == 0) {
		ranges[currtile].x = 0;
	} else {
		const uint32_t prevtile = tile_keys[idx - 1];
		if (currtile != prevtile) {
			ranges[prevtile].y = idx;
			ranges[currtile].x = idx;
		}
	}
	if (idx == R - 1) ranges[currtile].y = R;

	const uint32_t g = point_list[idx];
	const float2 xy = means2D[g];
	const float4 co = conic_opacity[g];
	const float2 ex = extent[g];
	const uint32_t mask = block_mask(xy.x, xy.y, co.x, co.y, co.z, co.w, ex, (int)(currtile % (uint32_t)grid_x), (int)(currtile / (uint32_t)grid_x));
	float4* dst = reinterpret_cast<float4*>(recs + idx);
	dst[0] = make_float4(xy.x, xy.y, co.x, co.y);
	dst[1] = make_float4(co.z, co.w, __uint_as_float(mask), __uint_as_float(g));
	block_bits[idx] = (uint8_t)mask;
}

// Per-block work lists: one CTA per tile, warp s compacts, in list order, the 0-based tile-list positions of the
// instances whose block bit s is set into row s of block_list (at range.x + k, so a row never outgrows the tile's slots)
// and writes their number to block_count[8 tile + s].  The blend warp of block s then touches only the records that can
// reach its pixels.  block_bits is read 16 bytes per lane from the 16-byte-aligned chunk at or below range.x (the array is
// padded for the last one); the loop is a chain of dependent loads, so each lane takes as many instances as one load gives.
__global__ void __launch_bounds__(256) block_lists_kernel(const uint2* __restrict__ ranges, const uint8_t* __restrict__ block_bits,
	uint32_t* __restrict__ block_list, size_t stride, uint32_t* __restrict__ block_count)
{
	const int tile = blockIdx.x;
	const int s = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const uint2 range = ranges[tile];
	uint32_t* const row = block_list + s * stride + range.x;
	const uint4* const chunks = reinterpret_cast<const uint4*>(block_bits);
	uint32_t n = 0;
	uint32_t c = (range.x >> 4) + lane;
	uint4 v = 16 * c < range.y ? chunks[c] : make_uint4(0u, 0u, 0u, 0u);
	for (uint32_t base = range.x & ~15u; base < range.y; base += 512) {
		const uint4 cur = v;
		const uint32_t p0 = 16 * c;
		c += 32;
		if (16 * c < range.y) v = chunks[c];  // the next step's bytes are in flight while this step is compacted
		const uint32_t w[4] = { cur.x, cur.y, cur.z, cur.w };
		uint32_t m = 0;  // bit b: instance p0 + b is in the tile and has block bit s
#pragma unroll
		for (int b = 0; b < 16; b++) {
			const uint32_t p = p0 + b;
			if (p >= range.x && p < range.y && ((w[b >> 2] >> (8 * (b & 3) + s)) & 1u)) m |= 1u << b;
		}
		// list order is lane-major: an inclusive scan of the per-lane counts places each lane's entries
		const uint32_t cnt = __popc(m);
		uint32_t incl = cnt;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) {
			const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
			if (lane >= o) incl += t;
		}
		uint32_t k = n + incl - cnt;
		for (; m; m &= m - 1u) row[k++] = p0 + (uint32_t)(__ffs(m) - 1) - range.x;
		n += __shfl_sync(0xffffffffu, incl, 31);
	}
	if (lane == 0) block_count[8 * tile + s] = n;
}

// Launch order of the blend CTAs: tiles by descending list length (rank by counting, ties by tile id).  The blend grids
// are about one wave of small CTAs (one or two warps per 8x4 block) whose run time follows the list length; starting the long ones first leaves
// the short ones for the tail of the wave (and of the last view's kernel in a multi-view step).
__global__ void __launch_bounds__(256) tile_order_kernel(const uint2* __restrict__ ranges, int T, uint32_t* __restrict__ order)
{
	__shared__ uint32_t s_len[256];
	const int t = blockIdx.x * blockDim.x + threadIdx.x;
	uint32_t mine = 0;
	if (t < T) { const uint2 r = ranges[t]; mine = r.y - r.x; }
	uint32_t rank = 0;
	for (int base = 0; base < T; base += 256) {
		const int u = base + threadIdx.x;
		uint32_t len = 0;
		if (u < T) { const uint2 r = ranges[u]; len = r.y - r.x; }
		__syncthreads();
		s_len[threadIdx.x] = len;
		__syncthreads();
		const int m = min(256, T - base);
		for (int i = 0; i < m; i++) {
			const uint32_t l = s_len[i];
			rank += (l > mine || (l == mine && base + i < t)) ? 1u : 0u;
		}
	}
	if (t < T) order[rank] = (uint32_t)t;
}

void launch_tile_order(const uint2* ranges, int num_tiles, uint32_t* order, cudaStream_t s)
{
	if (num_tiles > 0) tile_order_kernel<<<ceil_div(num_tiles, 256), 256, 0, s>>>(ranges, num_tiles, order);
}

void launch_ranges_and_pack(const uint32_t* R_dev, int capacity, int num_tiles, int grid_x, const uint32_t* tile_keys,
	const uint32_t* point_list, const float2* means2D, const float4* conic_opacity, const float2* extent, uint2* ranges, InstRec* recs,
	uint8_t* block_bits, uint32_t* tile_order, cudaStream_t s)
{
	cudaMemsetAsync(ranges, 0, sizeof(uint2) * (size_t)num_tiles, s);
	if (capacity > 0) ranges_pack_kernel<<<ceil_div(capacity, 256), 256, 0, s>>>(R_dev, capacity, grid_x, tile_keys, point_list, means2D, conic_opacity, extent, ranges, recs, block_bits);
	if (tile_order) launch_tile_order(ranges, num_tiles, tile_order, s);
}

void launch_block_lists(const uint2* ranges, int num_tiles, const uint8_t* block_bits, uint32_t* block_list, size_t stride,
	uint32_t* block_count, cudaStream_t s)
{
	if (num_tiles > 0) block_lists_kernel<<<num_tiles, 256, 0, s>>>(ranges, block_bits, block_list, stride, block_count);
}

}  // namespace mgs
