// Microbenchmark: throughput of red.global.add.noftz f16x2 reductions of 4 / 8 / 16 bytes at random addresses of a table
// (the access pattern of the hash-grid gradient scatter), as a function of the number of SMs that issue them and of the
// table's footprint -- a table that stays in L2 against one that does not.
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o red_bench red_bench.cu ; run on an H100.
//   red_bench            32 MB table, sweep over CTAs, widths and locality
//   red_bench MB [MB..]  one 132-CTA row per width for each table footprint in MB (e.g. red_bench 2 8 26 52)
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

template <int V>
__global__ void red_kernel(uint32_t* __restrict__ table, uint32_t n, uint32_t iters, uint32_t addend, uint32_t locality) {
	uint32_t s = (threadIdx.x + blockIdx.x * blockDim.x) * 2654435761u + 12345u;
#pragma unroll 4
	for (uint32_t i = 0; i < iters; ++i) {
		s = s * 1664525u + 1013904223u;
		uint32_t idx = __umulhi(s, n);  // uniform in [0, n)
		if (locality) idx = (idx & ~1023u) | ((threadIdx.x * 4 + (i & 3)) & 1023u);  // lanes of a warp fall into the same 128-byte lines
		if (V == 1) asm volatile("red.relaxed.gpu.global.add.noftz.f16x2 [%0], %1;" ::"l"(table + idx), "r"(addend) : "memory");
		if (V == 2) asm volatile("red.relaxed.gpu.global.add.noftz.v2.f16x2 [%0], {%1, %2};" ::"l"(table + (idx & ~1u)), "r"(addend), "r"(addend) : "memory");
		if (V == 4) asm volatile("red.relaxed.gpu.global.add.noftz.v4.f16x2 [%0], {%1, %2, %3, %4};" ::"l"(table + (idx & ~3u)), "r"(addend), "r"(addend), "r"(addend), "r"(addend) : "memory");
	}
}

template <int V>
static void run(uint32_t* table, uint32_t n, int ctas, int threads, uint32_t locality, float ghz) {
	const uint32_t iters = 2048;
	cudaEvent_t a, b;
	cudaEventCreate(&a);
	cudaEventCreate(&b);
	red_kernel<V><<<ctas, threads>>>(table, n, 64, 0, locality);
	cudaEventRecord(a);
	red_kernel<V><<<ctas, threads>>>(table, n, iters, 0, locality);
	cudaEventRecord(b);
	cudaEventSynchronize(b);
	float ms;
	cudaEventElapsedTime(&ms, a, b);
	const double lanes = (double)ctas * threads * iters;
	printf("{\"table_mb\": %.1f, \"bytes\": %d, \"ctas\": %d, \"threads\": %d, \"local\": %u, \"ms\": %.4f, \"Glanes_s\": %.2f, \"lanes_per_clk_per_cta\": %.3f}\n", n * 4.0 / (1 << 20), V * 4,
	       ctas, threads, locality, ms, lanes / ms * 1e-6, lanes / (ms * 1e-3) / (ghz * 1e9) / ctas);
}

int main(int argc, char** argv) {
	uint32_t* table;
	const uint32_t n_max = 64u << 18;  // 64 MB of f16x2 entries
	cudaMalloc(&table, (size_t)n_max * 4);
	cudaMemset(table, 0, (size_t)n_max * 4);
	int khz = 0;
	cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
	const float ghz = khz * 1e-6f;
	printf("{\"clock_ghz\": %.3f}\n", ghz);
	if (argc > 1) {
		for (int a = 1; a < argc; ++a) {
			const uint32_t n = (uint32_t)(atof(argv[a]) * (1 << 18));
			if (n < 1024 || n > n_max) return 2;
			run<1>(table, n, 132, 512, 0, ghz);
			run<2>(table, n, 132, 512, 0, ghz);
			run<4>(table, n, 132, 512, 0, ghz);
		}
		return cudaDeviceSynchronize() != cudaSuccess;
	}
	const uint32_t n = 1u << 23;  // 32 MB
	for (uint32_t local = 0; local < 2; ++local) {
		for (int ctas : {8, 33, 66, 132}) {  // up to one CTA per SM of an H100
			run<1>(table, n, ctas, 512, local, ghz);
			run<2>(table, n, ctas, 512, local, ghz);
			run<4>(table, n, ctas, 512, local, ghz);
		}
	}
	run<2>(table, n, 132, 1024, 0, ghz);
	run<2>(table, n, 264, 512, 0, ghz);
	return cudaDeviceSynchronize() != cudaSuccess;
}
