// Micro-benchmark: issue rate / latency of the legacy warp-level tensor path (mma.sync TF32 m16n8k8, BF16 m16n8k16)
// against FFMA, to size the 3xTF32 channel contraction of the blend kernels.  nvcc -arch=sm_90a -O3 -o mma_rate mma_rate.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2])
{
	asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
	             : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
	             : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2])
{
	asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
	             : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
	             : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// ILP independent accumulator tiles per warp; mode 0 tf32, 1 bf16, 2 ffma (32 FMAs per "op" to compare per-instruction)
template <int MODE, int ILP>
__global__ void k(float* out, long long* cyc, int iters, uint32_t seed)
{
	const long long c0 = clock64();
	float d[ILP][4];
	uint32_t a[4], b[2];
	for (int i = 0; i < 4; i++) a[i] = seed * (threadIdx.x + i + 1);
	for (int i = 0; i < 2; i++) b[i] = seed * (threadIdx.x + 7 + i);
	for (int j = 0; j < ILP; j++) for (int i = 0; i < 4; i++) d[j][i] = (float)j;
	float fa = __uint_as_float(0x3f800000u | (a[0] & 0xffff)), fb = 1e-3f;
	for (int it = 0; it < iters; it++) {
#pragma unroll
		for (int j = 0; j < ILP; j++) {
			if (MODE == 0) mma_tf32(d[j], a, b);
			else if (MODE == 1) mma_bf16(d[j], a, b);
			else {
#pragma unroll
				for (int i = 0; i < 4; i++) d[j][i] = fmaf(d[j][i], fa, fb);
			}
		}
	}
	float s = 0.f;
	for (int j = 0; j < ILP; j++) for (int i = 0; i < 4; i++) s += d[j][i];
	out[blockIdx.x * blockDim.x + threadIdx.x] = s;
	if (blockIdx.x == 0 && threadIdx.x == 0) *cyc = clock64() - c0;  // SM cycles of the timed loop, whatever the clock
}

template <int MODE, int ILP>
void run(const char* name, int warps_per_sm, int nsm, float* out, long long* cyc)
{
	const int iters = 4096;
	// one CTA per SM slot: warps_per_sm warps in ONE CTA per SM
	dim3 grid(nsm), block(32 * warps_per_sm);
	cudaEvent_t e0, e1;
	cudaEventCreate(&e0); cudaEventCreate(&e1);
	k<MODE, ILP><<<grid, block>>>(out, cyc, 16, 3u);
	cudaDeviceSynchronize();
	cudaEventRecord(e0);
	k<MODE, ILP><<<grid, block>>>(out, cyc, iters, 3u);
	cudaEventRecord(e1);
	cudaDeviceSynchronize();
	float ms = 0.f;
	cudaEventElapsedTime(&ms, e0, e1);
	const double ops = (double)nsm * warps_per_sm * iters * ILP * (MODE == 2 ? 4 : 1);  // warp-level instructions
	const double per_sm_per_us = ops / nsm / (ms * 1e3);
	// FMAs per instruction: tf32 m16n8k8 = 1024, bf16 m16n8k16 = 2048, ffma = 32
	const double fma = MODE == 0 ? 1024 : (MODE == 1 ? 2048 : 32);
	long long c = 0;
	cudaMemcpy(&c, cyc, sizeof(c), cudaMemcpyDeviceToHost);
	// issue interval in SM cycles per warp instruction and scheduler (4 schedulers per SM), and the clock it implies
	const double per_sched = (double)iters * ILP * (MODE == 2 ? 4 : 1) * (warps_per_sm < 4 ? 1 : warps_per_sm / 4);
	printf("%-6s ilp %d warps/SM %2d: %.3f ms  %.1f warp-instr/us/SM  %.1f FMA/ns/SM  chip %.1f TFMA/s  %.2f cycles/instr/scheduler"
	       "  (%.0f MHz)\n", name, ILP, warps_per_sm, ms, per_sm_per_us, per_sm_per_us * fma / 1e3, per_sm_per_us * fma * nsm / 1e6,
	       c / per_sched, c / (ms * 1e3));
}

int main()
{
	cudaDeviceProp p;
	cudaGetDeviceProperties(&p, 0);
	const int nsm = p.multiProcessorCount;
	printf("%s, %d SMs, %d MHz\n", p.name, nsm, p.clockRate / 1000);
	float* out;
	cudaMalloc(&out, sizeof(float) * nsm * 1024);
	long long* cyc;
	cudaMalloc(&cyc, sizeof(long long));
	for (int w : {1, 4, 8, 16}) {
		if (w == 1) { run<0, 1>("tf32", w, nsm, out, cyc); run<1, 1>("bf16", w, nsm, out, cyc); run<2, 1>("ffma", w, nsm, out, cyc); }
		run<0, 4>("tf32", w, nsm, out, cyc);
		run<1, 4>("bf16", w, nsm, out, cyc);
		run<2, 4>("ffma", w, nsm, out, cyc);
		run<0, 8>("tf32", w, nsm, out, cyc);
	}
	printf("cuda status: %s\n", cudaGetErrorString(cudaGetLastError()));
	return 0;
}
