// composite_kernels.h -- the reductions of a Composite encoding (encodings/composite.h:47-133) and the sum of the input gradients of
// nested encodings whose input ranges overlap (composite_kernels.cu).
#pragma once
#include "feature_encodings.h"

namespace tcnnb {

// out rows [n][row_stride] (first `width` columns) = Sum / Product over k of nested rows [n][K * width] (slab k at column k * width):
// an fp32 accumulator that starts at 0 / 1 takes the K fp16 values in order k = 0 .. K-1 and is rounded to fp16 once.
cudaError_t launch_reduce_forward(cudaStream_t stream, bool product, uint32_t K, uint32_t width, uint32_t n, const __half* nested, __half* out, uint32_t row_stride);
// dL_dnested rows [n][K * width] = Product backward: slab k = fp16(float(dL_dy) * prod_{l != k} nested_l), multiplied in ascending l in
// fp32. dL_dy rows [n][row_stride] (first `width` columns).
cudaError_t launch_reduce_product_backward(cudaStream_t stream, uint32_t K, uint32_t width, uint32_t n, const __half* dL_dy, uint32_t row_stride, const __half* nested,
                                           __half* dL_dnested);
// dL_dx rows [n][n_in] (OVERWRITTEN, every column) = sum over the non-Empty segments k that read a column, in segment order, of
// slabs[k] rows [n][n_in]; 0 where no segment reads it.
cudaError_t launch_sum_input_gradients(cudaStream_t stream, const FeatureSegments& segs, uint32_t n, uint32_t n_in, const float* slabs, float* dL_dx);

}  // namespace tcnnb
