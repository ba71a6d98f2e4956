// Marching cubes (include/mgs_rasterizer.h, mgs_marching_cubes_count / _emit): the level surface of an [X,Y,Z] grid as an
// indexed triangle mesh, with the case table of mc_table.cuh.  No atomics: every output slot comes from a scan, so the
// mesh is bitwise repeatable.  One thread per grid point n = (i Y + j) Z + k throughout, z fastest.
//   cells   the case byte of the cell whose lower corner is n (0 where a corner is invalid or n has no cell);
//   edges   the 3 edge-used bits of n's own +x, +y, +z edges, from the edge masks of the <= 4 cells around each;
//   scans   inclusive 64-bit sums of the points' vertex counts (popcount of the bits) and of the cells' triangle counts;
//           the last entries are the two totals;
//   emit    each point writes its vertices (ids in (point, axis) order), each cell its triangles; a triangle finds an
//           edge's vertex as its owner point's first id plus the popcount of the owner's lower-axis bits.
#include <cub/device/device_scan.cuh>
#include <cub/iterator/transform_input_iterator.cuh>
#include "mgs_common.cuh"
#include "mgs_kernels.h"
#include "mc_table.cuh"

namespace mgs {

constexpr int MC_THREADS = 256;

struct McState {
	uint8_t* cases;        // [N]
	uint8_t* bits;         // [N]
	long long* voff;       // [N] inclusive sum of the vertex counts
	long long* foff;       // [N] inclusive sum of the triangle counts
	void* temp;
	size_t temp_bytes;
};

struct VertexCount {
	__device__ long long operator()(uint8_t b) const { return __popc(b); }
};
struct TriangleCount {
	__device__ long long operator()(uint8_t c) const { return MC_TRI_COUNT[c]; }
};
using VertexIt = cub::TransformInputIterator<long long, VertexCount, const uint8_t*>;
using TriangleIt = cub::TransformInputIterator<long long, TriangleCount, const uint8_t*>;

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

static size_t scan_temp_bytes(size_t N)
{
	size_t a = 0, b = 0;
	cub::DeviceScan::InclusiveSum(nullptr, a, VertexIt(nullptr, VertexCount{}), (long long*)nullptr, (int)N);
	cub::DeviceScan::InclusiveSum(nullptr, b, TriangleIt(nullptr, TriangleCount{}), (long long*)nullptr, (int)N);
	return std::max(a, b);
}

static McState carve(void* state, size_t N)
{
	char* p = static_cast<char*>(state);
	McState s;
	s.cases = reinterpret_cast<uint8_t*>(p); p += align256(N);
	s.bits = reinterpret_cast<uint8_t*>(p); p += align256(N);
	s.voff = reinterpret_cast<long long*>(p); p += align256(N * sizeof(long long));
	s.foff = reinterpret_cast<long long*>(p); p += align256(N * sizeof(long long));
	s.temp = p;
	s.temp_bytes = scan_temp_bytes(N);
	return s;
}

size_t mc_state_bytes(int X, int Y, int Z)
{
	const size_t N = (size_t)X * Y * Z;
	return 2 * align256(N) + 2 * align256(N * sizeof(long long)) + scan_temp_bytes(N);
}

__device__ __forceinline__ bool mc_valid(const float* values, const float* weight, size_t n)
{
	return isfinite(values[n]) && (!weight || weight[n] > 0.f);
}

__global__ void __launch_bounds__(MC_THREADS) mc_cells_kernel(int X, int Y, int Z, const float* __restrict__ values,
	const float* __restrict__ weight, float level, uint8_t* __restrict__ cases)
{
	const size_t N = (size_t)X * Y * Z;
	const size_t n = (size_t)blockIdx.x * MC_THREADS + threadIdx.x;
	if (n >= N) return;
	const int k = (int)(n % Z), j = (int)((n / Z) % Y), i = (int)(n / ((size_t)Y * Z));
	uint32_t c = 0;
	if (i < X - 1 && j < Y - 1 && k < Z - 1) {
		bool ok = true;
#pragma unroll
		for (int q = 0; q < 8; q++) {
			const size_t m = n + (size_t)(q & 1) * Y * Z + (size_t)((q >> 1) & 1) * Z + ((q >> 2) & 1);
			ok = ok && mc_valid(values, weight, m);
			c |= (values[m] < level ? 1u : 0u) << q;
		}
		if (!ok) c = 0;
	}
	cases[n] = (uint8_t)c;
}

__global__ void __launch_bounds__(MC_THREADS) mc_edges_kernel(int X, int Y, int Z, const uint8_t* __restrict__ cases,
	uint8_t* __restrict__ bits)
{
	const size_t N = (size_t)X * Y * Z;
	const size_t n = (size_t)blockIdx.x * MC_THREADS + threadIdx.x;
	if (n >= N) return;
	const int idx[3] = { (int)(n / ((size_t)Y * Z)), (int)((n / Z) % Y), (int)(n % Z) };
	const int dim[3] = { X, Y, Z };
	const size_t stride[3] = { (size_t)Y * Z, (size_t)Z, 1 };
	uint32_t out = 0;
#pragma unroll
	for (int a = 0; a < 3; a++) {
		if (idx[a] + 1 >= dim[a]) continue;
		const int u = a == 0 ? 1 : 0, v = a == 2 ? 1 : 2;  // the other two axes, the lower first
		uint32_t used = 0;
#pragma unroll
		for (int s = 0; s < 4; s++) {
			// the cell whose lower corner is n - (s & 1) e_u - (s >> 1) e_v holds this edge as its edge 4 a + s
			const int ou = s & 1, ov = s >> 1;
			if (idx[u] - ou < 0 || idx[u] - ou >= dim[u] - 1 || idx[v] - ov < 0 || idx[v] - ov >= dim[v] - 1) continue;
			const uint8_t c = cases[n - ou * stride[u] - ov * stride[v]];
			used |= (MC_EDGE_MASK[c] >> (4 * a + s)) & 1u;
		}
		out |= used << a;
	}
	bits[n] = (uint8_t)out;
}

__global__ void mc_totals_kernel(size_t N, const long long* voff, const long long* foff, long long* out)
{
	out[0] = voff[N - 1];
	out[1] = foff[N - 1];
}

__global__ void __launch_bounds__(MC_THREADS) mc_vertices_kernel(int X, int Y, int Z, const float* __restrict__ values, float level,
	McState s, double lo0, double lo1, double lo2, double st0, double st1, double st2, int C, const float* __restrict__ color,
	float* __restrict__ out_vertices, float* __restrict__ out_colors)
{
	const size_t N = (size_t)X * Y * Z;
	const size_t n = (size_t)blockIdx.x * MC_THREADS + threadIdx.x;
	if (n >= N) return;
	const uint32_t b = s.bits[n];
	if (!b) return;
	const int idx[3] = { (int)(n / ((size_t)Y * Z)), (int)((n / Z) % Y), (int)(n % Z) };
	const size_t stride[3] = { (size_t)Y * Z, (size_t)Z, 1 };
	const double lo[3] = { lo0, lo1, lo2 }, st[3] = { st0, st1, st2 };
	float ca[3], cb[3];
#pragma unroll
	for (int q = 0; q < 3; q++) {
		ca[q] = (float)__dadd_rn(lo[q], __dmul_rn(__dadd_rn((double)idx[q], 0.5), st[q]));
		cb[q] = (float)__dadd_rn(lo[q], __dmul_rn(__dadd_rn((double)(idx[q] + 1), 0.5), st[q]));
	}
	long long id = s.voff[n] - __popc(b);
	const float va = values[n];
#pragma unroll
	for (int a = 0; a < 3; a++) {
		if (!((b >> a) & 1u)) continue;
		const size_t m = n + stride[a];
		const float t = __fdiv_rn(__fsub_rn(level, va), __fsub_rn(values[m], va));
#pragma unroll
		for (int q = 0; q < 3; q++) {
			const float e = q == a ? cb[q] : ca[q];
			out_vertices[3 * id + q] = __fadd_rn(ca[q], __fmul_rn(t, __fsub_rn(e, ca[q])));
		}
		for (int c = 0; c < C; c++) {
			const float qa = color[(size_t)c * N + n], qb = color[(size_t)c * N + m];
			out_colors[id * C + c] = __fadd_rn(qa, __fmul_rn(t, __fsub_rn(qb, qa)));
		}
		id++;
	}
}

__global__ void __launch_bounds__(MC_THREADS) mc_faces_kernel(int X, int Y, int Z, McState s, long long* __restrict__ out_faces)
{
	const size_t N = (size_t)X * Y * Z;
	const size_t n = (size_t)blockIdx.x * MC_THREADS + threadIdx.x;
	if (n >= N) return;
	const uint8_t c = s.cases[n];
	const int nt = MC_TRI_COUNT[c];
	if (!nt) return;
	long long f = s.foff[n] - nt;
	const size_t sYZ = (size_t)Y * Z;
	for (int t = 0; t < nt; t++, f++) {
#pragma unroll
		for (int q = 0; q < 3; q++) {
			const int e = MC_TRIS[c][3 * t + q];
			const int a = e >> 2, sb = e & 3;
			// the strides of the edge's other two axes, the lower first (mc_table.cuh's numbering)
			const size_t su = a == 0 ? (size_t)Z : sYZ, sv = a == 2 ? (size_t)Z : 1;
			const size_t owner = n + (sb & 1) * su + (sb >> 1) * sv;
			const uint32_t ob = s.bits[owner];
			out_faces[3 * f + q] = s.voff[owner] - __popc(ob) + __popc(ob & ((1u << a) - 1u));
		}
	}
}

cudaError_t mc_count(void* state, int X, int Y, int Z, const float* values, const float* weight, float level, long long* out_counts,
	cudaStream_t st)
{
	const size_t N = (size_t)X * Y * Z;
	McState s = carve(state, N);
	const unsigned grid = (unsigned)((N + MC_THREADS - 1) / MC_THREADS);
	mc_cells_kernel<<<grid, MC_THREADS, 0, st>>>(X, Y, Z, values, weight, level, s.cases);
	mc_edges_kernel<<<grid, MC_THREADS, 0, st>>>(X, Y, Z, s.cases, s.bits);
	cudaError_t e = cub::DeviceScan::InclusiveSum(s.temp, s.temp_bytes, VertexIt(s.bits, VertexCount{}), s.voff, (int)N, st);
	if (e != cudaSuccess) return e;
	e = cub::DeviceScan::InclusiveSum(s.temp, s.temp_bytes, TriangleIt(s.cases, TriangleCount{}), s.foff, (int)N, st);
	if (e != cudaSuccess) return e;
	mc_totals_kernel<<<1, 1, 0, st>>>(N, s.voff, s.foff, out_counts);
	return cudaGetLastError();
}

cudaError_t mc_emit(void* state, int X, int Y, int Z, const float* values, float level, const double lo[3], const double step[3],
	int C, const float* color, float* out_vertices, long long* out_faces, float* out_colors, cudaStream_t st)
{
	const size_t N = (size_t)X * Y * Z;
	McState s = carve(state, N);
	const unsigned grid = (unsigned)((N + MC_THREADS - 1) / MC_THREADS);
	mc_vertices_kernel<<<grid, MC_THREADS, 0, st>>>(X, Y, Z, values, level, s, lo[0], lo[1], lo[2], step[0], step[1], step[2], C,
		color, out_vertices, out_colors);
	mc_faces_kernel<<<grid, MC_THREADS, 0, st>>>(X, Y, Z, s, out_faces);
	return cudaGetLastError();
}

}  // namespace mgs
