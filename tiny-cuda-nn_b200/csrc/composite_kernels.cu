// composite_kernels.cu -- Sum / Product reductions of a Composite encoding (encodings/composite.h:47-133) and the sum of overlapping
// nested input gradients. Pure streaming kernels: one thread per (sample, V columns), 16-byte accesses (V = 8) when the widths, row
// strides and pointers allow, else one column per thread. The arithmetic is the reference's, operation for operation: fp32
// accumulators in nested order, one rounding to fp16 at the end.
#include "composite_kernels.h"

namespace tcnnb {

namespace {

template <uint32_t V>
struct alignas(2 * V) HalfVec {
	__half h[V];
};

template <bool PRODUCT, uint32_t V>
__global__ void reduce_forward_kernel(uint32_t n, uint32_t K, uint32_t width, const __half* __restrict__ nested, __half* __restrict__ out, uint32_t row_stride) {
	const uint32_t chunks = width / V;
	const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= (size_t)n * chunks) return;
	const size_t i = t / chunks;
	const uint32_t c = (uint32_t)(t - i * chunks) * V;
	const __half* __restrict__ src = nested + i * K * width + c;
	float acc[V];
#pragma unroll
	for (uint32_t v = 0; v < V; ++v) acc[v] = PRODUCT ? 1.0f : 0.0f;
	for (uint32_t k = 0; k < K; ++k) {
		const HalfVec<V> x = *reinterpret_cast<const HalfVec<V>*>(src + (size_t)k * width);
#pragma unroll
		for (uint32_t v = 0; v < V; ++v) {
			if (PRODUCT) acc[v] *= __half2float(x.h[v]);
			else acc[v] += __half2float(x.h[v]);
		}
	}
	HalfVec<V> y;
#pragma unroll
	for (uint32_t v = 0; v < V; ++v) y.h[v] = __float2half_rn(acc[v]);
	*reinterpret_cast<HalfVec<V>*>(out + i * row_stride + c) = y;
}

// composite.h:106-133: the reference's quadratic loop (no division by the own factor, so zeros are exact)
template <uint32_t V>
__global__ void reduce_product_backward_kernel(uint32_t n, uint32_t K, uint32_t width, const __half* __restrict__ dL_dy, uint32_t row_stride, const __half* __restrict__ nested,
                                               __half* __restrict__ dL_dnested) {
	const uint32_t chunks = width / V;
	const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= (size_t)n * chunks) return;
	const size_t i = t / chunks;
	const uint32_t c = (uint32_t)(t - i * chunks) * V;
	const __half* __restrict__ src = nested + i * K * width + c;
	const HalfVec<V> dy = *reinterpret_cast<const HalfVec<V>*>(dL_dy + i * row_stride + c);
	for (uint32_t k = 0; k < K; ++k) {
		float r[V];
#pragma unroll
		for (uint32_t v = 0; v < V; ++v) r[v] = __half2float(dy.h[v]);
		for (uint32_t l = 0; l + 1 < K; ++l) {
			const HalfVec<V> x = *reinterpret_cast<const HalfVec<V>*>(src + (size_t)(l < k ? l : l + 1) * width);
#pragma unroll
			for (uint32_t v = 0; v < V; ++v) r[v] *= __half2float(x.h[v]);
		}
		HalfVec<V> y;
#pragma unroll
		for (uint32_t v = 0; v < V; ++v) y.h[v] = __float2half_rn(r[v]);
		*reinterpret_cast<HalfVec<V>*>(dL_dnested + i * K * width + (size_t)k * width + c) = y;
	}
}

__global__ void sum_input_gradients_kernel(const FeatureSegments segs, uint32_t n, uint32_t n_in, const float* __restrict__ slabs, float* __restrict__ dL_dx) {
	const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	const size_t total = (size_t)n * n_in;
	if (t >= total) return;
	const uint32_t d = (uint32_t)(t % n_in);
	float acc = 0.0f;
	for (uint32_t k = 0; k < segs.n; ++k) {
		const FeatureSegment& sg = segs.s[k];
		if (sg.type != FEAT_EMPTY && d >= sg.in_begin && d < sg.in_begin + sg.n_in) acc += slabs[(size_t)k * total + t];
	}
	dL_dx[t] = acc;
}

inline bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

inline uint32_t n_blocks(size_t threads) { return (uint32_t)((threads + 255) / 256); }

}  // namespace

cudaError_t launch_reduce_forward(cudaStream_t stream, bool product, uint32_t K, uint32_t width, uint32_t n, const __half* nested, __half* out, uint32_t row_stride) {
	if (n == 0 || width == 0) return cudaSuccess;
	if (K == 0 || K > MAX_FEATURE_SEGMENTS || !nested || !out) return cudaErrorInvalidValue;
	const bool vec = width % 8 == 0 && row_stride % 8 == 0 && aligned16(nested) && aligned16(out);
	const size_t threads = (size_t)n * (vec ? width / 8 : width);
	if (vec && product) reduce_forward_kernel<true, 8><<<n_blocks(threads), 256, 0, stream>>>(n, K, width, nested, out, row_stride);
	else if (vec) reduce_forward_kernel<false, 8><<<n_blocks(threads), 256, 0, stream>>>(n, K, width, nested, out, row_stride);
	else if (product) reduce_forward_kernel<true, 1><<<n_blocks(threads), 256, 0, stream>>>(n, K, width, nested, out, row_stride);
	else reduce_forward_kernel<false, 1><<<n_blocks(threads), 256, 0, stream>>>(n, K, width, nested, out, row_stride);
	return cudaGetLastError();
}

cudaError_t launch_reduce_product_backward(cudaStream_t stream, uint32_t K, uint32_t width, uint32_t n, const __half* dL_dy, uint32_t row_stride, const __half* nested,
                                           __half* dL_dnested) {
	if (n == 0 || width == 0) return cudaSuccess;
	if (K == 0 || K > MAX_FEATURE_SEGMENTS || !dL_dy || !nested || !dL_dnested) return cudaErrorInvalidValue;
	const bool vec = width % 8 == 0 && row_stride % 8 == 0 && aligned16(dL_dy) && aligned16(nested) && aligned16(dL_dnested);
	const size_t threads = (size_t)n * (vec ? width / 8 : width);
	if (vec) reduce_product_backward_kernel<8><<<n_blocks(threads), 256, 0, stream>>>(n, K, width, dL_dy, row_stride, nested, dL_dnested);
	else reduce_product_backward_kernel<1><<<n_blocks(threads), 256, 0, stream>>>(n, K, width, dL_dy, row_stride, nested, dL_dnested);
	return cudaGetLastError();
}

cudaError_t launch_sum_input_gradients(cudaStream_t stream, const FeatureSegments& segs, uint32_t n, uint32_t n_in, const float* slabs, float* dL_dx) {
	if (n == 0 || n_in == 0) return cudaSuccess;
	if (segs.n > MAX_FEATURE_SEGMENTS || !slabs || !dL_dx) return cudaErrorInvalidValue;
	sum_input_gradients_kernel<<<n_blocks((size_t)n * n_in), 256, 0, stream>>>(segs, n, n_in, slabs, dL_dx);
	return cudaGetLastError();
}

}  // namespace tcnnb
