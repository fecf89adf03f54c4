// grid_bwd_bwd.cu -- second-order derivatives of the multiresolution grid encoding (GridEncoding::backward_backward_input,
// grid.h:910-1042): what a loss on dL/d(position) -- the eikonal term of a signed-distance field -- sends back through the encoding.
//
// Inputs per sample: the position x, u = dL/d(encoded) (the gradient the first backward pass contracted with), v = dL/d(dL/dx).
// With y_{l,f}(x) = sum_c w_c(t(x)) theta_{l,c,f}, t_d = S(p_d) (S = identity or smoothstep of the raw fractional position p_d) and
// dL/dx_d = sum_{l,f} u_{l,f} dy_{l,f}/dx_d, the three results are
//   dL_dparams     theta_{l,c,f}  += u_{l,f} * sum_d v_d scale_l S'(p_d) dw_c/dt_d          kernel_grid_backward_input_backward_grid    grid.h:351-455
//   dL_ddLdoutput  (l, f)          = sum_d v_d dy_{l,f}/dx_d                                  kernel_grid_backward_input_backward_dLdoutput grid.h:625-655
//   dL_dinput      e              += sum_{l,f} u_{l,f} sum_d v_d d2y_{l,f}/dx_d dx_e           kernel_grid_backward_input_backward_input   grid.h:457-623
// where the Hessian has off-diagonal terms scale^2 S'(p_d) S'(p_e) d2w/dt_d dt_e and (Smoothstep only) diagonal terms
// scale^2 S''(p_d) dw/dt_d; S' = 6 p (1 - p) and S'' = 6 - 12 p on the RAW p (common_device.h:980-990, as grid_input_gradient_kernel).
//
// The reference runs three kernels (one thread per sample, feature pair and level) that each gather the corners again. Here ONE
// thread per sample walks all levels; each level's 2^D corner entries are gathered once and give all three results:
//   W_c = sum_d (scale S'(p_d) v_d) dw_c/dt_d        is the parameter-gradient weight of corner c, and dL_ddLdoutput_f = sum_c W_c theta_{c,f};
//   theta_u[c] = sum_f u_f theta_{c,f}               contracts the features once, and the Hessian terms are sums over the corners of theta_u.
// Compile-time flags drop the parts whose outputs were not asked for: dL_dparams alone reads no table entries, and the Hessian is
// only evaluated for dL_dinput. The parameter-gradient addend of a corner is (half)W_c * u (the fp16 multiply of the first-order
// scatter, grid.h:252-255; the reference adds the D per-dimension terms of W_c one by one) with one red.f16x2 / v2 / v4 per corner;
// F == 1 accumulates in fp32 and is cast afterwards, as the reference does (grid.h:858-894).
#include "grid_kernels.h"

#include "grid_device.cuh"
#include "misc_kernels.h"

namespace tcnnb {

namespace {

// d w_c / d t_d for corner c: the weight with the factor of dimension d replaced by its derivative, -1 (bit d clear) or +1.
template <uint32_t D>
__device__ __forceinline__ float dweight(const float (&t)[D], uint32_t c, uint32_t d) {
	float w = (c >> d) & 1u ? 1.0f : -1.0f;
#pragma unroll
	for (uint32_t k = 0; k < D; ++k) {
		if (k != d) w *= (c >> k) & 1u ? t[k] : 1.0f - t[k];
	}
	return w;
}

// d2 w_c / d t_d d t_e for d != e (the weight is linear in every t_d, so the diagonal is zero).
template <uint32_t D>
__device__ __forceinline__ float ddweight(const float (&t)[D], uint32_t c, uint32_t d, uint32_t e) {
	float w = (((c >> d) ^ (c >> e)) & 1u) ? -1.0f : 1.0f;
#pragma unroll
	for (uint32_t k = 0; k < D; ++k) {
		if (k != d && k != e) w *= (c >> k) & 1u ? t[k] : 1.0f - t[k];
	}
	return w;
}

template <uint32_t D, uint32_t F, bool PARAMS, bool DOUT, bool DIN>
__global__ void __launch_bounds__(128) grid_bwd_bwd_kernel(const GridKernelArgs a, const __half* __restrict__ table, const __half* __restrict__ dL_dy,
                                                          const float* __restrict__ dL_ddLdx, __half* __restrict__ grad_table, float* __restrict__ grad_fp32,
                                                          __half* __restrict__ dL_ddLdy, float* __restrict__ dL_dx) {
	constexpr uint32_t NC = 1u << D;
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= a.n_elements) return;
	float x[D], v[D], result[D];
	load_position<D>(a.positions, a.pos_stride, i, x);
	load_position<D>(dL_ddLdx, a.pos_stride, i, v);
#pragma unroll
	for (uint32_t d = 0; d < D; ++d) result[d] = 0.0f;
	const float n_active = grid_active_levels(a.max_level, a.n_levels, F);
	const __half* __restrict__ u_row = dL_dy + (size_t)i * a.row_stride;
	__half* const out_row = DOUT ? dL_ddLdy + (size_t)i * a.row_stride : nullptr;
	Entry<F> zero;
#pragma unroll
	for (uint32_t f = 0; f < F; ++f) zero.v[f] = __float2half_rn(0.0f);

	for (uint32_t level = 0; level < a.n_levels; ++level) {
		// Nearest: every derivative of the encoding w.r.t. the position is zero (grid.h:420-423, 522-525); masked levels contribute nothing
		if (a.interpolation == INTERP_NEAREST || (float)level >= n_active + 1e-3f) {
			if (DOUT) store_entry<F>(out_row + level * F, zero);
			continue;
		}
		const LevelInfo lv = a.levels_dev[level];
		LevelCorners<D> lc;
		level_corners<D>(lv, x, a.interpolation, lc);
		Entry<F> vals[NC];
		if (DOUT || DIN) {
			const __half* __restrict__ ltab = table + (size_t)lv.offset * F;
#pragma unroll
			for (uint32_t c = 0; c < NC; ++c) vals[c] = load_entry<F>(ltab + (size_t)lc.idx[c] * F);
		}
		Entry<F> u;
		if (PARAMS || DIN) u = load_entry<F>(u_row + level * F);
		// S'(p) and S''(p) on the raw fractional position (pos_fract with smoothstep_derivative / smoothstep_2nd_derivative)
		float d1[D], d2[D], g[D];
#pragma unroll
		for (uint32_t d = 0; d < D; ++d) {
			float pr = __fmaf_rn(lv.scale, x[d], 0.5f);
			pr -= floorf(pr);
			const bool smooth = a.interpolation == INTERP_SMOOTHSTEP;
			d1[d] = smooth ? 6.0f * pr * (1.0f - pr) : 1.0f;
			d2[d] = smooth ? 6.0f - 12.0f * pr : 0.0f;
			g[d] = lv.scale * v[d] * d1[d];  // grad_in = scale * dL_ddLdx * pos_derivative (grid.h:428)
		}
		if (PARAMS || DOUT) {
			float W[NC];
#pragma unroll
			for (uint32_t c = 0; c < NC; ++c) {
				W[c] = 0.0f;
#pragma unroll
				for (uint32_t d = 0; d < D; ++d) W[c] += g[d] * dweight<D>(lc.frac, c, d);
			}
			if (PARAMS) {
				const size_t base = (size_t)lv.offset * F;
#pragma unroll
				for (uint32_t c = 0; c < NC; ++c) {
					const size_t at = base + (size_t)lc.idx[c] * F;
					if (F == 1) {
						atomicAdd(grad_fp32 + at, W[c] * __half2float(u.v[0]));
					} else {
						Entry<F> e;
						const __half w = __float2half_rn(W[c]);
#pragma unroll
						for (uint32_t f = 0; f < F; ++f) e.v[f] = __hmul(w, u.v[f]);
						red_entry<F>(grad_table + at, e);
					}
				}
			}
			if (DOUT) {
				Entry<F> out;
#pragma unroll
				for (uint32_t f = 0; f < F; ++f) {
					float s = 0.0f;
#pragma unroll
					for (uint32_t c = 0; c < NC; ++c) s += W[c] * __half2float(vals[c].v[f]);
					out.v[f] = __float2half_rn(s);
				}
				store_entry<F>(out_row + level * F, out);
			}
		}
		if (DIN) {
			float tu[NC];
#pragma unroll
			for (uint32_t c = 0; c < NC; ++c) {
				tu[c] = 0.0f;
#pragma unroll
				for (uint32_t f = 0; f < F; ++f) tu[c] += __half2float(u.v[f]) * __half2float(vals[c].v[f]);
			}
			const float s2 = lv.scale * lv.scale;
#pragma unroll
			for (uint32_t e = 0; e < D; ++e) {
				float acc = 0.0f;
				if (a.interpolation == INTERP_SMOOTHSTEP) {  // diagonal of the Hessian: zero for Linear
					float g1 = 0.0f;
#pragma unroll
					for (uint32_t c = 0; c < NC; ++c) g1 += dweight<D>(lc.frac, c, e) * tu[c];
					acc += v[e] * d2[e] * g1;
				}
#pragma unroll
				for (uint32_t d = 0; d < D; ++d) {
					if (d == e) continue;
					float h = 0.0f;
#pragma unroll
					for (uint32_t c = 0; c < NC; ++c) h += ddweight<D>(lc.frac, c, d, e) * tu[c];
					acc += v[d] * d1[d] * d1[e] * h;
				}
				result[e] += s2 * acc;
			}
		}
	}
	if (DOUT) {
		for (uint32_t c = a.n_levels * F; c < a.n_levels * F + a.pad_cols; ++c) out_row[c] = __float2half_rn(0.0f);
	}
	if (DIN) {
#pragma unroll
		for (uint32_t d = 0; d < D; ++d) dL_dx[(size_t)i * a.pos_stride + d] = result[d];
	}
}

template <uint32_t D, uint32_t F>
cudaError_t launch_df(cudaStream_t stream, const GridKernelArgs& a, bool params, bool dout, bool din, const __half* table, const __half* dL_dy, const float* dL_ddLdx,
                      __half* grad_table, float* grad_fp32, __half* dL_ddLdy, float* dL_dx) {
	const dim3 grid((a.n_elements + 127) / 128), block(128);
#define TCNNB_BB(P, O, I)                                                                                                               \
	if (params == P && dout == O && din == I) {                                                                                         \
		grid_bwd_bwd_kernel<D, F, P, O, I><<<grid, block, 0, stream>>>(a, table, dL_dy, dL_ddLdx, grad_table, grad_fp32, dL_ddLdy, dL_dx); \
		return cudaGetLastError();                                                                                                      \
	}
	TCNNB_BB(true, false, false) TCNNB_BB(false, true, false) TCNNB_BB(true, true, false) TCNNB_BB(false, false, true)
	TCNNB_BB(true, false, true) TCNNB_BB(false, true, true) TCNNB_BB(true, true, true)
#undef TCNNB_BB
	return cudaSuccess;  // nothing asked for
}

}  // namespace

cudaError_t launch_grid_backward_backward_input(cudaStream_t stream, const GridKernelArgs& a, const __half* table, const __half* dL_dy, const float* dL_ddLdx,
                                                __half* grad_table, float* tmp_fp32, uint32_t n_params, __half* dL_ddLdy, float* dL_dx) {
	const uint32_t D = a.n_pos_dims, F = a.n_features_per_level;
	if (a.pos_stride < D || D < 2 || D > 4 || !(F == 1 || F == 2 || F == 4 || F == 8) || a.n_levels == 0 || a.row_stride < a.n_levels * F + a.pad_cols ||
	    a.row_stride % F != 0 || !a.levels_dev || !a.positions || !dL_ddLdx)
		return cudaErrorInvalidValue;
	// Nearest: the parameter gradient is zero (the caller has zeroed it), nothing is scattered
	const bool params = grad_table && a.interpolation != INTERP_NEAREST;
	const bool dout = dL_ddLdy != nullptr, din = dL_dx != nullptr;
	if ((params || din) && !dL_dy) return cudaErrorInvalidValue;
	if ((dout || din) && !table) return cudaErrorInvalidValue;
	if (params && F == 1 && !tmp_fp32) return cudaErrorInvalidValue;
	if (a.n_elements == 0) return cudaSuccess;
	float* const grad_fp32 = params && F == 1 ? tmp_fp32 : nullptr;
	cudaError_t err = cudaErrorInvalidValue;
#define TCNNB_DF(DD, FF) \
	if (D == DD && F == FF) err = launch_df<DD, FF>(stream, a, params, dout, din, table, dL_dy, dL_ddLdx, grad_table, grad_fp32, dL_ddLdy, dL_dx);
	TCNNB_DF(2, 1) TCNNB_DF(2, 2) TCNNB_DF(2, 4) TCNNB_DF(2, 8)
	TCNNB_DF(3, 1) TCNNB_DF(3, 2) TCNNB_DF(3, 4) TCNNB_DF(3, 8)
	TCNNB_DF(4, 1) TCNNB_DF(4, 2) TCNNB_DF(4, 4) TCNNB_DF(4, 8)
#undef TCNNB_DF
	if (err != cudaSuccess) return err;
	if (params && F == 1) err = launch_cast_params(stream, n_params, tmp_fp32, grad_table);
	return err;
}

}  // namespace tcnnb
