// Microbenchmark: throughput of random-address fp16x2 table gathers (the access pattern of the hash-grid corner-pair gather),
// counted per corner PAIR, for the load shapes a pair can take, with and without L1 allocation (ld.global.nc.L1::no_allocate):
//   4B        one 4-byte load per pair (the rate of single requests)
//   2x4B      two 4-byte loads to unrelated entries (a pair whose entries do not share a slot)
//   8B        one 8-byte load of an aligned slot (a merged pair)
//   2x4B_slot two 4-byte loads to the two halves of one aligned 8-byte slot (a pair that shares a slot, fetched unmerged)
// and a mixed row per shape: half the warps gather from one table while the other half issue 4-byte f16x2 reductions into a
// second table of the same size, as the training kernel's memory warps do.
// Every thread keeps 16 pairs in flight (the fused training kernel keeps three levels of 4 (2-D) or 8 (3-D) pairs in flight).
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o gather_bench gather_bench.cu ; run on an H100.
//   gather_bench [MB]    table footprint in MB (default 26, the headline configuration's fp16 table), 132 CTAs x 512 threads
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

enum : int { SHAPE_4B = 0, SHAPE_2X4B = 1, SHAPE_8B = 2, SHAPE_2X4B_SLOT = 3 };
static const char* shape_name[] = {"4B", "2x4B", "8B", "2x4B_slot"};
constexpr int PAIRS = 16;

template <bool NA>
__device__ __forceinline__ uint32_t ld32(const uint32_t* p) {
	uint32_t v;
	if (NA) asm volatile("ld.global.nc.L1::no_allocate.b32 %0, [%1];" : "=r"(v) : "l"(p));
	else asm volatile("ld.global.nc.b32 %0, [%1];" : "=r"(v) : "l"(p));
	return v;
}
template <bool NA>
__device__ __forceinline__ void ld64(const uint32_t* p, uint32_t& a, uint32_t& b) {
	if (NA) asm volatile("ld.global.nc.L1::no_allocate.v2.b32 {%0, %1}, [%2];" : "=r"(a), "=r"(b) : "l"(p));
	else asm volatile("ld.global.nc.v2.b32 {%0, %1}, [%2];" : "=r"(a), "=r"(b) : "l"(p));
}

// `mixed`: odd warps reduce into `red_table` instead of gathering (each of them issues PAIRS 4-byte reductions per iteration).
template <int SHAPE, bool NA>
__global__ void gather_kernel(const uint32_t* __restrict__ table, uint32_t* __restrict__ red_table, uint32_t n, uint32_t iters, uint32_t mixed, uint32_t* __restrict__ sink) {
	uint32_t s = (threadIdx.x + blockIdx.x * blockDim.x) * 2654435761u + 12345u;
	uint32_t acc = 0;
	const bool reducer = mixed && ((threadIdx.x >> 5) & 1u);
	for (uint32_t i = 0; i < iters; ++i) {
		uint32_t idx[PAIRS], idx2[PAIRS];
#pragma unroll
		for (int k = 0; k < PAIRS; ++k) {
			s = s * 1664525u + 1013904223u;
			idx[k] = __umulhi(s, n);  // uniform in [0, n)
			if (SHAPE == SHAPE_2X4B) {
				s = s * 1664525u + 1013904223u;
				idx2[k] = __umulhi(s, n);
			}
		}
		if (reducer) {
#pragma unroll
			for (int k = 0; k < PAIRS; ++k) asm volatile("red.relaxed.gpu.global.add.noftz.f16x2 [%0], %1;" ::"l"(red_table + idx[k]), "r"(0u) : "memory");
			continue;
		}
		// all loads of the iteration are issued before any value is used
		uint32_t v0[PAIRS], v1[PAIRS];
#pragma unroll
		for (int k = 0; k < PAIRS; ++k) {
			if (SHAPE == SHAPE_4B) v0[k] = ld32<NA>(table + idx[k]), v1[k] = 0;
			if (SHAPE == SHAPE_2X4B) v0[k] = ld32<NA>(table + idx[k]), v1[k] = ld32<NA>(table + idx2[k]);
			if (SHAPE == SHAPE_8B) ld64<NA>(table + (idx[k] & ~1u), v0[k], v1[k]);
			if (SHAPE == SHAPE_2X4B_SLOT) v0[k] = ld32<NA>(table + (idx[k] & ~1u)), v1[k] = ld32<NA>(table + (idx[k] | 1u));
		}
#pragma unroll
		for (int k = 0; k < PAIRS; ++k) acc ^= v0[k] + v1[k];
	}
	if (acc == 0x9e3779b9u) *sink = acc;  // keeps the loads live; the table is zero, so this never stores
}

template <int SHAPE, bool NA>
static void run(const uint32_t* table, uint32_t* red_table, uint32_t n, uint32_t mixed, uint32_t* sink) {
	const int ctas = 132, threads = 512;
	const uint32_t iters = 256;
	cudaEvent_t a, b;
	cudaEventCreate(&a);
	cudaEventCreate(&b);
	gather_kernel<SHAPE, NA><<<ctas, threads>>>(table, red_table, n, 8, mixed, sink);
	cudaEventRecord(a);
	gather_kernel<SHAPE, NA><<<ctas, threads>>>(table, red_table, n, iters, mixed, sink);
	cudaEventRecord(b);
	cudaEventSynchronize(b);
	float ms;
	cudaEventElapsedTime(&ms, a, b);
	// in a mixed run half the threads gather and half reduce, each issuing PAIRS operations per iteration
	const double per_role = (double)ctas * threads * iters * PAIRS / (mixed ? 2 : 1);
	printf("{\"table_mb\": %.1f, \"shape\": \"%s\", \"no_allocate\": %d, \"mixed\": %u, \"ms\": %.4f, \"Gpairs_s\": %.2f, \"Greds_s\": %.2f}\n", n * 4.0 / (1 << 20), shape_name[SHAPE], NA ? 1 : 0,
	       mixed, ms, per_role / ms * 1e-6, mixed ? per_role / ms * 1e-6 : 0.0);
	cudaEventDestroy(a);
	cudaEventDestroy(b);
}

template <int SHAPE>
static void run_shape(const uint32_t* table, uint32_t* red_table, uint32_t n, uint32_t* sink) {
	run<SHAPE, false>(table, red_table, n, 0, sink);
	run<SHAPE, true>(table, red_table, n, 0, sink);
	run<SHAPE, true>(table, red_table, n, 1, sink);
}

int main(int argc, char** argv) {
	const double mb = argc > 1 ? atof(argv[1]) : 26.0;
	const uint32_t n = (uint32_t)(mb * (1 << 18));
	if (n < 1024 || n > (64u << 18)) return 2;
	uint32_t *table, *red_table, *sink;
	cudaMalloc(&table, (size_t)n * 4);
	cudaMalloc(&red_table, (size_t)n * 4);
	cudaMalloc(&sink, 4);
	cudaMemset(table, 0, (size_t)n * 4);
	cudaMemset(red_table, 0, (size_t)n * 4);
	int khz = 0;
	cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
	printf("{\"clock_ghz\": %.3f}\n", khz * 1e-6);
	run_shape<SHAPE_4B>(table, red_table, n, sink);
	run_shape<SHAPE_2X4B>(table, red_table, n, sink);
	run_shape<SHAPE_8B>(table, red_table, n, sink);
	run_shape<SHAPE_2X4B_SLOT>(table, red_table, n, sink);
	return cudaDeviceSynchronize() != cudaSuccess;
}
