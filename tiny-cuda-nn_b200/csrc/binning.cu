// binning.cu -- per-step spatial binning of the batch (counting sort by the (y, z) column of each sample).
//
// Why: the multiresolution gather / scatter is bound by the number of distinct 32-byte sectors the memory system has to
// serve. Both the dense index (x + y*res + z*res^2, common_device.h:866-871) and the coherent-prime hash (x*1 ^ y*p1 ^ z*p2,
// common_device.h:787-791) are CONTIGUOUS IN X for a fixed (y, z) cell. If the 32 samples of a warp share a (y, z) column, their
// corner entries on the coarse and middle levels fall into a handful of 128-byte lines (and repeat across warps, so they hit
// in L1) instead of 32 different ones. Gradients and the loss are sums over samples, so processing the batch in a different
// order changes nothing but the (already unordered) accumulation order; per-sample outputs are written through `perm`.
//
// The reference has no counterpart (it consumes the batch in the caller's order); this is a scheduling step of this library.
#include "binning.h"

namespace tcnnb {

namespace {

__device__ __forceinline__ uint32_t part1by1(uint32_t v) {  // spread the low 8 bits: abcdefgh -> 0a0b0c0d0e0f0g0h
	v &= 0xFFu;
	v = (v | (v << 4)) & 0x0F0Fu;
	v = (v | (v << 2)) & 0x3333u;
	v = (v | (v << 1)) & 0x5555u;
	return v;
}

template <uint32_t D>
__device__ __forceinline__ uint32_t bin_key(const float* __restrict__ pos, uint32_t i, uint32_t log2_r) {
	const uint32_t R = 1u << log2_r;
	if (D == 2) {
		const float y = pos[(size_t)i * 2 + 1];
		return min(R - 1u, (uint32_t)max(0, (int)(y * (float)R)));
	}
	const float y = pos[(size_t)i * D + 1], z = pos[(size_t)i * D + 2];
	const uint32_t yc = min(R - 1u, (uint32_t)max(0, (int)(y * (float)R)));
	const uint32_t zc = min(R - 1u, (uint32_t)max(0, (int)(z * (float)R)));
	// Morton order of the columns keeps consecutive bins (= consecutive tiles) spatially adjacent
	return part1by1(yc) | (part1by1(zc) << 1);
}

template <uint32_t D>
__global__ void bin_count_kernel(uint32_t n, const float* __restrict__ pos, uint32_t log2_r, uint32_t* __restrict__ keys, uint32_t* __restrict__ hist, uint4* __restrict__ zero_ptr, uint32_t zero_n16, float* __restrict__ zero_scalar) {
	const uint32_t i = threadIdx.x + blockIdx.x * blockDim.x;
	pdl_wait();
	pdl_launch_dependents();
	// This kernel waits on atomic round trips and leaves the memory pipes idle: the step's gradient zeroing (GradientMode::Overwrite,
	// grid.h:865-867) rides along here instead of being a separate 26 MB memset launch in front of the fused kernel.
	for (uint32_t j = i; j < zero_n16; j += gridDim.x * blockDim.x) zero_ptr[j] = make_uint4(0u, 0u, 0u, 0u);
	if (i == 0 && zero_scalar) *zero_scalar = 0.0f;
	if (i >= n) return;
	const uint32_t k = bin_key<D>(pos, i, log2_r);
	// the value returned by the counting atomic is this sample's rank inside its bin: the scatter pass needs no atomics
	const uint32_t rank = atomicAdd(hist + k, 1u);
	reinterpret_cast<uint2*>(keys)[i] = make_uint2(k, rank);
}

// Exclusive scan of `n_bins` counters by one block of 1024 threads: cursor[b] = first output slot of bin b.
// The counters are staged through shared memory with coalesced accesses (all loads of a thread are independent), each
// thread scans a contiguous run of the staged copy, and the 1024 run totals are combined with shuffles.
// The counters are re-armed to zero for the next step, so no memset is needed per step.
constexpr uint32_t SCAN_CHUNK = 16384;  // bins staged per pass (66 KB of shared memory incl. padding)
// one padding word every 32: thread t's contiguous run (stride 16 words) then falls into distinct banks across a warp
__device__ __forceinline__ uint32_t scan_pad(uint32_t i) { return i + (i >> 5); }
constexpr uint32_t SCAN_SMEM_WORDS = SCAN_CHUNK + SCAN_CHUNK / 32;

__global__ void __launch_bounds__(1024) bin_scan_kernel(uint32_t n_bins, uint32_t* __restrict__ hist, uint32_t* __restrict__ cursor) {
	extern __shared__ uint32_t staged[];
	__shared__ uint32_t warp_sums[32];
	__shared__ uint32_t carry;
	pdl_wait();
	pdl_launch_dependents();
	if (threadIdx.x == 0) carry = 0;
	for (uint32_t base = 0; base < n_bins; base += SCAN_CHUNK) {
		const uint32_t n = min(SCAN_CHUNK, n_bins - base);
		{
			// all 16 loads of a thread in flight at once (a rolled loop would pay one memory latency per iteration)
			uint32_t v[SCAN_CHUNK / 1024];
#pragma unroll
			for (uint32_t j = 0; j < SCAN_CHUNK / 1024; ++j) {
				const uint32_t i = threadIdx.x + j * 1024;
				v[j] = i < n ? hist[base + i] : 0u;
			}
#pragma unroll
			for (uint32_t j = 0; j < SCAN_CHUNK / 1024; ++j) {
				const uint32_t i = threadIdx.x + j * 1024;
				if (i < n) {
					staged[scan_pad(i)] = v[j];
					hist[base + i] = 0;
				}
			}
		}
		__syncthreads();
		const uint32_t per = (n + 1023u) / 1024u;
		const uint32_t begin = min(n, threadIdx.x * per), end = min(n, begin + per);
		uint32_t total = 0;
		for (uint32_t i = begin; i < end; ++i) total += staged[scan_pad(i)];
		uint32_t incl = total;
#pragma unroll
		for (uint32_t o = 1; o < 32; o <<= 1) {
			const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, o);
			if ((threadIdx.x & 31u) >= o) incl += t;
		}
		if ((threadIdx.x & 31u) == 31u) warp_sums[threadIdx.x >> 5] = incl;
		__syncthreads();
		if (threadIdx.x < 32) {
			uint32_t w = warp_sums[threadIdx.x];
#pragma unroll
			for (uint32_t o = 1; o < 32; o <<= 1) {
				const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, w, o);
				if (threadIdx.x >= o) w += t;
			}
			warp_sums[threadIdx.x] = w;
		}
		__syncthreads();
		const uint32_t c = carry;
		uint32_t run = c + ((threadIdx.x >> 5) ? warp_sums[(threadIdx.x >> 5) - 1] : 0u) + incl - total;
		for (uint32_t i = begin; i < end; ++i) {
			const uint32_t v = staged[scan_pad(i)];
			staged[scan_pad(i)] = run;
			run += v;
		}
		__syncthreads();
		for (uint32_t i = threadIdx.x; i < n; i += 1024) cursor[base + i] = staged[scan_pad(i)];
		if (threadIdx.x == 1023) carry = c + warp_sums[31];
		__syncthreads();
	}
}

// perm[first slot of the sample's bin + its rank inside the bin] = sample. Only the permutation is materialised: the fused
// kernel fetches positions / targets through it (one extra 12-byte read per sample, against ~100 table sectors per sample).
__global__ void bin_scatter_kernel(uint32_t n, const uint32_t* __restrict__ keys, const uint32_t* __restrict__ cursor, uint32_t* __restrict__ perm) {
	const uint32_t i = threadIdx.x + blockIdx.x * blockDim.x;
	pdl_wait();
	pdl_launch_dependents();
	if (i >= n) return;
	const uint2 kr = reinterpret_cast<const uint2*>(keys)[i];
	perm[__ldg(cursor + kr.x) + kr.y] = i;
}

}  // namespace

uint32_t binning_log2_resolution(uint32_t n_samples, uint32_t n_pos_dims) {
	// aim at ~16 samples per bin: n_bins = n / 16 = R^(D-1)
	uint32_t log2_bins = 0;
	while ((1ull << (log2_bins + 1)) * 16ull <= n_samples) ++log2_bins;
	uint32_t log2_r = n_pos_dims == 2 ? log2_bins : log2_bins / 2;
	if (n_pos_dims != 2 && log2_r > 8) log2_r = 8;  // part1by1 interleaves 8 bits per axis
	if (log2_r > 16) log2_r = 16;
	return log2_r;
}

uint32_t binning_n_bins(uint32_t log2_r, uint32_t n_pos_dims) { return n_pos_dims == 2 ? (1u << log2_r) : (1u << (2 * log2_r)); }

cudaError_t launch_binning(cudaStream_t stream, uint32_t n_pos_dims, uint32_t n, const float* pos, uint32_t log2_r, uint32_t* keys, uint32_t* hist, uint32_t* perm, void* zero_ptr, size_t zero_bytes, float* zero_scalar) {
	if (((uintptr_t)zero_ptr | zero_bytes) & 15u) return cudaErrorMisalignedAddress;
	const uint32_t zero_n16 = (uint32_t)(zero_bytes / 16);
	const uint32_t n_bins = binning_n_bins(log2_r, n_pos_dims);
	uint32_t* cursor = hist + n_bins;  // hist: [n_bins counters (zero between calls) | n_bins cursors]
	const uint32_t blocks = (n + 255) / 256;
	// per launch: the attribute is per device / context, and a process may build models on several GPUs
	cudaError_t err = cudaFuncSetAttribute(bin_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(SCAN_SMEM_WORDS * sizeof(uint32_t)));
	if (err != cudaSuccess) return err;
	if (n_pos_dims == 2) {
		err = launch_pdl(bin_count_kernel<2>, blocks, 256, 0, stream, n, pos, log2_r, keys, hist, (uint4*)zero_ptr, zero_n16, zero_scalar);
	} else if (n_pos_dims == 3) {
		err = launch_pdl(bin_count_kernel<3>, blocks, 256, 0, stream, n, pos, log2_r, keys, hist, (uint4*)zero_ptr, zero_n16, zero_scalar);
	} else {
		return cudaErrorInvalidValue;
	}
	if (err != cudaSuccess) return err;
	err = launch_pdl(bin_scan_kernel, 1, 1024, SCAN_SMEM_WORDS * sizeof(uint32_t), stream, n_bins, hist, cursor);
	if (err != cudaSuccess) return err;
	return launch_pdl(bin_scatter_kernel, blocks, 256, 0, stream, n, (const uint32_t*)keys, (const uint32_t*)cursor, perm);
}

}  // namespace tcnnb
