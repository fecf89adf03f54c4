// grid_kernels.cu -- the multiresolution grid encoding on its own: forward, parameter-gradient scatter, input-position gradient.
//
// These are the kernels behind tcnn::cpp::create_encoding (cpp_api.h:124, src/cpp_api.cu:165-174) and behind the module tier's
// dL/d(input); the training / inference hot path does NOT use them (there the gather and the scatter are fused into the MLP
// kernel, fused_ws.cu). They cover the reference's whole grid configuration space -- n_features_per_level 1 / 2 / 4 / 8, 2 to 4
// input dimensions, Hash / Dense / Tiled, Nearest / Linear / Smoothstep, max_level -- with the same arithmetic:
//   kernel_grid                 grid.h:49-212   one thread per (sample, level); fp32 weights, fp16 fma chain in corner order
//   kernel_grid_backward        grid.h:215-320  addend = (half)weight * dL_dy (fp16 multiply), atomics in the gradient precision
//                                               (fp16 pairs; fp32 scratch + cast when F == 1, grid.h:858-894)
//   dy_dx + kernel_grid_backward_input  grid.h:170-212,322-350  summed over features in feature order, fp32
// Index arithmetic is shared with the fused kernel (grid_device.cuh) and bit-exact with the reference.
// HBM/L2-bound scattered 2..16-byte accesses. Thread <-> (sample, level) with the level fastest (the reference runs one block row per
// level to keep a level's table hot in a small L2, grid.h:769-771; the whole table of the benchmarked configuration nearly fits the H100's 50 MB L2, and level-fastest makes the
// feature-row accesses whole sectors).
#include "grid_kernels.h"

#include "grid_device.cuh"

namespace tcnnb {

namespace {

template <uint32_t F>
struct Entry {
	__half v[F];
};

template <uint32_t F>
__device__ __forceinline__ Entry<F> load_entry(const __half* __restrict__ p) {
	Entry<F> e;
	if (F == 1) {
		e.v[0] = __ldg(p);
	} else if (F == 2) {
		*reinterpret_cast<uint32_t*>(e.v) = __ldg(reinterpret_cast<const uint32_t*>(p));
	} else if (F == 4) {
		*reinterpret_cast<uint2*>(e.v) = __ldg(reinterpret_cast<const uint2*>(p));
	} else {
		*reinterpret_cast<uint4*>(e.v) = __ldg(reinterpret_cast<const uint4*>(p));
	}
	return e;
}

template <uint32_t F>
__device__ __forceinline__ void store_entry(__half* p, const Entry<F>& e) {
	if (F == 1) {
		p[0] = e.v[0];
	} else if (F == 2) {
		*reinterpret_cast<uint32_t*>(p) = *reinterpret_cast<const uint32_t*>(e.v);
	} else if (F == 4) {
		*reinterpret_cast<uint2*>(p) = *reinterpret_cast<const uint2*>(e.v);
	} else {
		*reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(e.v);
	}
}

// one reduction per corner: f16x2, v2.f16x2 or v4.f16x2 (an entry of F fp16 is F * 2 bytes and aligned to that)
template <uint32_t F>
__device__ __forceinline__ void red_entry(__half* p, const Entry<F>& e) {
	const uint32_t* w = reinterpret_cast<const uint32_t*>(e.v);
	if (F == 2) {
		asm volatile("red.relaxed.gpu.global.add.noftz.f16x2 [%0], %1;" ::"l"(p), "r"(w[0]) : "memory");
	} else if (F == 4) {
		asm volatile("red.relaxed.gpu.global.add.noftz.v2.f16x2 [%0], {%1, %2};" ::"l"(p), "r"(w[0]), "r"(w[1]) : "memory");
	} else if (F == 8) {
		asm volatile("red.relaxed.gpu.global.add.noftz.v4.f16x2 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3]) : "memory");
	}
}

template <uint32_t D>
__device__ __forceinline__ void load_position(const float* __restrict__ positions, uint32_t stride, uint32_t i, float (&x)[D]) {
#pragma unroll
	for (uint32_t d = 0; d < D; ++d) x[d] = __ldg(positions + (size_t)i * stride + d);
}

__device__ __forceinline__ float active_levels(const GridKernelArgs& a) {
	// max_level = (max_level * num_grid_features) / N_FEATURES_PER_LEVEL (grid.h:69-73)
	return (a.max_level * (float)(a.n_levels * a.n_features_per_level)) / (float)a.n_features_per_level;
}

template <uint32_t D, uint32_t F>
__global__ void grid_forward_kernel(const GridKernelArgs a, const __half* __restrict__ table, __half* __restrict__ encoded) {
	// thread <-> (sample, level), LEVEL fastest: the lanes of a warp write (read, in the backward kernel) consecutive columns of a
	// few rows -- whole 32-byte sectors -- instead of one column of 32 different rows
	const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	const uint32_t i = (uint32_t)(t / a.n_levels);
	if (i >= a.n_elements) return;
	const uint32_t level = (uint32_t)(t - (uint64_t)i * a.n_levels);
	__half* row = encoded + (size_t)i * a.row_stride;
	if (level == 0) {  // padding columns are zero (grid.h:757-766)
		for (uint32_t c = a.n_levels * F; c < a.n_levels * F + a.pad_cols; ++c) row[c] = __float2half_rn(0.0f);
	}
	Entry<F> result;
#pragma unroll
	for (uint32_t f = 0; f < F; ++f) result.v[f] = __float2half_rn(0.0f);
	if ((float)level >= active_levels(a) + 1e-3f) {
		store_entry<F>(row + level * F, result);
		return;
	}
	const LevelInfo lv = a.levels_dev[level];
	const __half* __restrict__ ltab = table + (size_t)lv.offset * F;
	float x[D];
	load_position<D>(a.positions, a.pos_stride, i, x);
	if (a.interpolation == INTERP_NEAREST) {
		CellPos<D> cp;
		pos_fract<D>(x, lv.scale, INTERP_LINEAR, cp);
		result = load_entry<F>(ltab + (size_t)corner_index<D>(lv, cp.cell) * F);
	} else {
		LevelCorners<D> lc;
		level_corners<D>(lv, x, a.interpolation, lc);
		Entry<F> vals[1u << D];
#pragma unroll
		for (uint32_t c = 0; c < (1u << D); ++c) vals[c] = load_entry<F>(ltab + (size_t)lc.idx[c] * F);
#pragma unroll
		for (uint32_t c = 0; c < (1u << D); ++c) {
			const __half w = __float2half_rn(lc.w[c]);
#pragma unroll
			for (uint32_t f = 0; f < F; ++f) result.v[f] = __hfma(w, vals[c].v[f], result.v[f]);  // fma((T)weight, val, result), grid.h:162
		}
	}
	store_entry<F>(row + level * F, result);
}

template <uint32_t D, uint32_t F>
__global__ void grid_backward_kernel(const GridKernelArgs a, const __half* __restrict__ dL_dy, __half* __restrict__ grad_table, float* __restrict__ grad_fp32) {
	const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	const uint32_t i = (uint32_t)(t / a.n_levels);
	if (i >= a.n_elements) return;
	const uint32_t level = (uint32_t)(t - (uint64_t)i * a.n_levels);
	if ((float)level > active_levels(a) + 1e-3f) return;  // grid.h:242 (strict, unlike the forward's >=)
	const LevelInfo lv = a.levels_dev[level];
	float x[D];
	load_position<D>(a.positions, a.pos_stride, i, x);
	const Entry<F> grad = load_entry<F>(dL_dy + (size_t)i * a.row_stride + level * F);
	// coarse levels: one of n_replicas private copies of the level (see plan_grid_scatter)
	__half* const target = (F > 1 && a.n_replicas > 1 && lv.offset + lv.size <= a.replica_entries) ? a.replica_scratch + (size_t)(blockIdx.x % a.n_replicas) * a.replica_entries * F : grad_table;
	auto add = [&](uint32_t idx, float weight) {
		const size_t at = ((size_t)lv.offset + idx) * F;
		if (F == 1) {
			atomicAdd(grad_fp32 + at, weight * __half2float(grad.v[0]));  // grad_t == float when F == 1 (grid.h:858-863)
		} else {
			Entry<F> e;
			const __half w = __float2half_rn(weight);
#pragma unroll
			for (uint32_t f = 0; f < F; ++f) e.v[f] = __hmul(w, grad.v[f]);  // (GRAD_T)weight * grad, grid.h:252-255
			red_entry<F>(target + at, e);
		}
	};
	if (a.interpolation == INTERP_NEAREST) {
		CellPos<D> cp;
		pos_fract<D>(x, lv.scale, INTERP_LINEAR, cp);
		add(corner_index<D>(lv, cp.cell), 1.0f);
		return;
	}
	LevelCorners<D> lc;
	level_corners<D>(lv, x, a.interpolation, lc);
#pragma unroll
	for (uint32_t c = 0; c < (1u << D); ++c) add(lc.idx[c], lc.w[c]);
}

// grad_table[word] = sum over the replicas (fp32), replicas re-armed to zero. One thread per f16x2 word of the replicated levels.
__global__ void replica_reduce_kernel(uint32_t n_words, uint32_t n_replicas, uint32_t* __restrict__ scratch, uint32_t* __restrict__ grad_table) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_words) return;
	float lo = 0.0f, hi = 0.0f;
	for (uint32_t r = 0; r < n_replicas; ++r) {
		const uint32_t w = scratch[(size_t)r * n_words + i];
		if (w) {
			const float2 v = __half22float2(*reinterpret_cast<const __half2*>(&w));
			lo += v.x;
			hi += v.y;
			scratch[(size_t)r * n_words + i] = 0u;
		}
	}
	const __half2 out = __floats2half2_rn(lo, hi);
	grad_table[i] = *reinterpret_cast<const uint32_t*>(&out);
}

__global__ void cast_grad_kernel(uint32_t n, const float* __restrict__ in, __half* __restrict__ out) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) out[i] = __float2half_rn(in[i]);
}

template <uint32_t D, uint32_t F>
__global__ void grid_input_gradient_kernel(const GridKernelArgs a, const __half* __restrict__ table, const __half* __restrict__ dL_dy, float* __restrict__ dL_dx) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= a.n_elements) return;
	float x[D], result[D];
	load_position<D>(a.positions, a.pos_stride, i, x);
#pragma unroll
	for (uint32_t d = 0; d < D; ++d) result[d] = 0.0f;
	const float n_active = active_levels(a);
	if (a.interpolation != INTERP_NEAREST) {  // Nearest: dy_dx is zero (grid.h:120-133)
		for (uint32_t level = 0; level < a.n_levels; ++level) {
			if ((float)level >= n_active + 1e-3f) break;  // dy_dx of the masked levels is zero (grid.h:84-89)
			const LevelInfo lv = a.levels_dev[level];
			const __half* __restrict__ ltab = table + (size_t)lv.offset * F;
			LevelCorners<D> lc;
			level_corners<D>(lv, x, a.interpolation, lc);
			// pos_derivative (common_device.h:1031-1043): 1 for Linear, smoothstep'(t) = 6 t (1 - t) on the RAW fractional position
			float deriv[D];
#pragma unroll
			for (uint32_t d = 0; d < D; ++d) {
				float pr = __fmaf_rn(lv.scale, x[d], 0.5f);
				pr -= floorf(pr);
				deriv[d] = a.interpolation == INTERP_SMOOTHSTEP ? 6.0f * pr * (1.0f - pr) : 1.0f;
			}
			Entry<F> vals[1u << D];
#pragma unroll
			for (uint32_t c = 0; c < (1u << D); ++c) vals[c] = load_entry<F>(ltab + (size_t)lc.idx[c] * F);
			float grads[F][D];
#pragma unroll
			for (uint32_t f = 0; f < F; ++f)
#pragma unroll
				for (uint32_t d = 0; d < D; ++d) grads[f][d] = 0.0f;
#pragma unroll
			for (uint32_t gd = 0; gd < D; ++gd) {
#pragma unroll
				for (uint32_t idx = 0; idx < (1u << (D - 1)); ++idx) {
					// weight = scale * product over the OTHER dimensions, in dimension order (grid.h:180-195)
					float weight = lv.scale;
					uint32_t corner = 0;
#pragma unroll
					for (uint32_t nd = 0; nd < D - 1; ++nd) {
						const uint32_t dim = nd >= gd ? nd + 1 : nd;
						if ((idx & (1u << nd)) == 0) {
							weight *= 1.0f - lc.frac[dim];
						} else {
							weight *= lc.frac[dim];
							corner |= 1u << dim;
						}
					}
					const Entry<F>& left = vals[corner];
					const Entry<F>& right = vals[corner | (1u << gd)];
#pragma unroll
					for (uint32_t f = 0; f < F; ++f) grads[f][gd] += weight * (__half2float(right.v[f]) - __half2float(left.v[f])) * deriv[gd];
				}
			}
			const Entry<F> dy = load_entry<F>(dL_dy + (size_t)i * a.row_stride + level * F);
#pragma unroll
			for (uint32_t f = 0; f < F; ++f) {
				const float dyf = __half2float(dy.v[f]);
#pragma unroll
				for (uint32_t d = 0; d < D; ++d) result[d] += dyf * grads[f][d];  // kernel_grid_backward_input, grid.h:336-345
			}
		}
	}
#pragma unroll
	for (uint32_t d = 0; d < D; ++d) dL_dx[(size_t)i * a.pos_stride + d] = result[d];
}

bool args_ok(const GridKernelArgs& a) {
	const uint32_t F = a.n_features_per_level;
	return a.pos_stride >= a.n_pos_dims && a.n_levels * F + a.pad_cols <= a.row_stride && a.n_pos_dims >= 2 && a.n_pos_dims <= 4 && (F == 1 || F == 2 || F == 4 || F == 8) && a.n_levels > 0 && a.row_stride >= a.n_levels * F && a.row_stride % F == 0 &&
	       a.levels_dev && a.positions;
}

// dispatch on (D, F): 12 instantiations of each kernel
template <typename Fn>
cudaError_t dispatch(const GridKernelArgs& a, Fn&& fn) {
#define TCNNB_DF(DD, FF) \
	if (a.n_pos_dims == DD && a.n_features_per_level == FF) return fn(std::integral_constant<uint32_t, DD>{}, std::integral_constant<uint32_t, FF>{});
	TCNNB_DF(2, 1) TCNNB_DF(2, 2) TCNNB_DF(2, 4) TCNNB_DF(2, 8)
	TCNNB_DF(3, 1) TCNNB_DF(3, 2) TCNNB_DF(3, 4) TCNNB_DF(3, 8)
	TCNNB_DF(4, 1) TCNNB_DF(4, 2) TCNNB_DF(4, 4) TCNNB_DF(4, 8)
#undef TCNNB_DF
	return cudaErrorInvalidValue;
}

}  // namespace

cudaError_t launch_grid_forward(cudaStream_t stream, const GridKernelArgs& a, const __half* table, __half* encoded) {
	if (!args_ok(a) || !table || !encoded) return cudaErrorInvalidValue;
	if (a.n_elements == 0) return cudaSuccess;
	const uint64_t n_threads = (uint64_t)a.n_elements * a.n_levels;
	if ((n_threads + 255) / 256 > 0x7FFFFFFFull) return cudaErrorInvalidValue;
	const dim3 grid((uint32_t)((n_threads + 255) / 256));
	return dispatch(a, [&](auto d, auto f) {
		grid_forward_kernel<decltype(d)::value, decltype(f)::value><<<grid, 256, 0, stream>>>(a, table, encoded);
		return cudaGetLastError();
	});
}

cudaError_t launch_grid_backward(cudaStream_t stream, const GridKernelArgs& a, const __half* dL_dy, __half* grad_table, float* tmp_fp32, uint32_t n_params) {
	if (!args_ok(a) || !dL_dy || !grad_table) return cudaErrorInvalidValue;
	if (a.n_features_per_level == 1 && !tmp_fp32) return cudaErrorInvalidValue;
	if (a.n_elements == 0) return cudaSuccess;
	const uint64_t n_threads = (uint64_t)a.n_elements * a.n_levels;
	if ((n_threads + 255) / 256 > 0x7FFFFFFFull) return cudaErrorInvalidValue;
	const dim3 grid((uint32_t)((n_threads + 255) / 256));
	cudaError_t err = dispatch(a, [&](auto d, auto f) {
		grid_backward_kernel<decltype(d)::value, decltype(f)::value><<<grid, 256, 0, stream>>>(a, dL_dy, grad_table, tmp_fp32);
		return cudaGetLastError();
	});
	if (err != cudaSuccess) return err;
	if (a.n_features_per_level > 1 && a.n_replicas > 1 && a.replica_entries) {
		if (!a.replica_scratch) return cudaErrorInvalidValue;
		const uint32_t n_words = a.replica_entries * a.n_features_per_level / 2;
		replica_reduce_kernel<<<(n_words + 255) / 256, 256, 0, stream>>>(n_words, a.n_replicas, reinterpret_cast<uint32_t*>(a.replica_scratch), reinterpret_cast<uint32_t*>(grad_table));
		err = cudaGetLastError();
	}
	if (a.n_features_per_level == 1) {
		cast_grad_kernel<<<(n_params + 255) / 256, 256, 0, stream>>>(n_params, tmp_fp32, grad_table);
		err = cudaGetLastError();
	}
	return err;
}

GridScatterPlan plan_grid_scatter(const LevelInfo* levels, uint32_t n_levels, uint32_t F, uint32_t D, uint32_t n_elements) {
	GridScatterPlan plan;
	if (F < 2 || n_levels == 0 || n_elements < 16384) return plan;
	const double corners = (double)n_elements * (double)(1u << D);
	// replicate the levels whose entries receive more than ~64 reductions each, with enough copies to bring the coarsest one there
	uint32_t entries = 0;
	for (uint32_t l = 0; l < n_levels; ++l) {
		if (levels[l].offset != entries || corners / (double)levels[l].size <= 64.0) break;
		entries += levels[l].size;
	}
	if (entries == 0) return plan;
	uint32_t r = 1;
	while (r < 64 && corners / (double)levels[0].size / (double)r > 128.0) r *= 2;
	while (r > 1 && (size_t)r * entries * F * sizeof(__half) > ((size_t)64 << 20)) r /= 2;
	if (r < 2) return plan;
	plan.n_replicas = r;
	plan.replica_entries = entries;
	plan.scratch_halfs = (size_t)r * entries * F;
	return plan;
}

cudaError_t launch_grid_input_gradient(cudaStream_t stream, const GridKernelArgs& a, const __half* table, const __half* dL_dy, float* dL_dx) {
	if (!args_ok(a) || !table || !dL_dy || !dL_dx) return cudaErrorInvalidValue;
	if (a.n_elements == 0) return cudaSuccess;
	return dispatch(a, [&](auto d, auto f) {
		grid_input_gradient_kernel<decltype(d)::value, decltype(f)::value><<<(a.n_elements + 127) / 128, 128, 0, stream>>>(a, table, dL_dy, dL_dx);
		return cudaGetLastError();
	});
}

}  // namespace tcnnb
