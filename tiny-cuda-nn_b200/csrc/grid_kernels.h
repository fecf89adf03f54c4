// grid_kernels.h -- launch interface of the stand-alone multiresolution-grid kernels (grid_kernels.cu): the encoding on its own
// (tcnn::cpp::create_encoding, cpp_api.h:124) and the input-position gradient of the module tier.
#pragma once
#include "common.cuh"

namespace tcnnb {

struct GridKernelArgs {
	uint32_t n_pos_dims;             // 2, 3, 4
	uint32_t n_features_per_level;   // 1, 2, 4, 8
	uint32_t n_levels;
	uint32_t interpolation;          // InterpolationType
	float max_level;                 // fraction of the levels that is active, as GridEncoding::set_max_level (grid.h:69-92); 1 = all
	const LevelInfo* levels_dev;     // [n_levels] in device memory
	uint32_t n_elements;
	const float* positions;          // rows [n][pos_stride] fp32, the grid's D coordinates first (a Composite passes a column offset)
	uint32_t pos_stride;             // floats per row of positions AND of dL_dx (>= D)
	uint32_t row_stride;             // fp16 elements per row of encoded / dL_dy (>= n_levels * F + pad_cols)
	uint32_t pad_cols;               // forward: columns behind the features that are zeroed (the grid's own alignment padding)
	// backward only (optional, see plan_grid_scatter): the coarse levels scatter into one of n_replicas private copies
	__half* replica_scratch;         // [n_replicas][replica_entries * F] fp16, ZERO on entry (left zero on exit)
	uint32_t n_replicas;             // 0 / 1 = off
	uint32_t replica_entries;        // levels with offset + size <= replica_entries are replicated
};

// Coarse levels receive thousands of reductions per table entry (2^18 samples x 4 corners over the 289 vertices of a 16 x 16 level:
// 3 600 each) and reductions to ONE address complete one after the other in L2, so that level alone sets the kernel's duration.
// Those levels scatter into n_replicas private copies (chosen by block index) that a small kernel sums into the gradient table.
// Sums of the same addends in a different order: the reference's own accumulation order is unspecified (atomics).
struct GridScatterPlan {
	uint32_t n_replicas = 1;
	uint32_t replica_entries = 0;
	size_t scratch_halfs = 0;  // n_replicas * replica_entries * F
};
GridScatterPlan plan_grid_scatter(const LevelInfo* levels_host, uint32_t n_levels, uint32_t n_features_per_level, uint32_t n_pos_dims, uint32_t n_elements);

// encoded [n][row_stride] fp16 (row = sample; columns level * F + f; the pad_cols columns behind them are zeroed)        grid.h:49-169
cudaError_t launch_grid_forward(cudaStream_t stream, const GridKernelArgs& a, const __half* table, __half* encoded);
// grad_table (fp16, n_params, accumulated INTO: the caller zeroes it) += scatter of dL_dy [n][row_stride] fp16       grid.h:215-320
// F == 1 accumulates in `tmp_fp32` (n_params floats, zeroed by the caller) and casts at the end, as the reference (grid.h:858-894).
cudaError_t launch_grid_backward(cudaStream_t stream, const GridKernelArgs& a, const __half* dL_dy, __half* grad_table, float* tmp_fp32, uint32_t n_params);
// dL_dx [n][pos_stride] fp32 (first D columns) = sum over features of dL_dy * d(encoded)/d(position)                                           grid.h:170-212,322-350
cudaError_t launch_grid_input_gradient(cudaStream_t stream, const GridKernelArgs& a, const __half* table, const __half* dL_dy, float* dL_dx);
// Second-order derivatives (grid_bwd_bwd.cu; grid.h:351-655,910-1042) from dL_ddLdx [n][pos_stride] fp32 (first D columns) and
// dL_dy [n][row_stride] fp16; each of the three results is computed when its pointer is non-null:
//   grad_table (fp16, n_params, accumulated INTO: the caller zeroes it; F == 1 accumulates in `tmp_fp32`, zeroed by the caller, and casts)
//   dL_ddLdy [n][row_stride] fp16 (OVERWRITTEN, pad_cols behind the features zeroed)
//   dL_dx [n][pos_stride] fp32 (first D columns, OVERWRITTEN)
// One launch (plus the cast when F == 1). Replicated scatter (replica_scratch) is not used.
cudaError_t launch_grid_backward_backward_input(cudaStream_t stream, const GridKernelArgs& a, const __half* table, const __half* dL_dy, const float* dL_ddLdx,
                                                __half* grad_table, float* tmp_fp32, uint32_t n_params, __half* dL_ddLdy, float* dL_dx);

}  // namespace tcnnb
