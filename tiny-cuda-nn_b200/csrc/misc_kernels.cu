// misc_kernels.cu -- the streaming kernels around the fused step: parameter initialisation (pcg32 jump-ahead fill),
// fp32 -> fp16 parameter cast, per-level scale evaluation, and the Adam step.
//
// Compiled with --use_fast_math like the reference (CMakeLists.txt:288-290) so that exp2f / powf / sqrtf / '/' lower
// to the same approximate instructions as in the reference's kernels.
#include "common.cuh"
#include "misc_kernels.h"

#include "fused_common.cuh"

#include <algorithm>

namespace tcnnb {

// ------------------------------------------------------------------------------------------------------------------
// pcg32 (PCG-XSH-RR 64/32, O'Neill) on the device: next_uint / next_float / advance as specified in
// dependencies/pcg32/pcg32.h:62-69,103-112,145-166.
// ------------------------------------------------------------------------------------------------------------------
namespace {

constexpr uint64_t PCG32_MULT = 0x5851f42d4c957f2dULL;

__device__ __forceinline__ uint32_t pcg_next_uint(Pcg32& r) {
	const uint64_t old = r.state;
	r.state = old * PCG32_MULT + r.inc;
	const uint32_t xorshifted = (uint32_t)(((old >> 18u) ^ old) >> 27u);
	const uint32_t rot = (uint32_t)(old >> 59u);
	return (xorshifted >> rot) | (xorshifted << ((~rot + 1u) & 31));
}

__device__ __forceinline__ float pcg_next_float(Pcg32& r) {
	return __uint_as_float((pcg_next_uint(r) >> 9) | 0x3f800000u) - 1.0f;
}

__device__ __forceinline__ void pcg_advance(Pcg32& r, uint64_t delta) {
	uint64_t cur_mult = PCG32_MULT, cur_plus = r.inc, acc_mult = 1u, acc_plus = 0u;
	while (delta > 0) {
		if (delta & 1) {
			acc_mult *= cur_mult;
			acc_plus = acc_plus * cur_mult + cur_plus;
		}
		cur_plus = (cur_mult + 1) * cur_plus;
		cur_mult *= cur_mult;
		delta /= 2;
	}
	r.state = acc_mult * r.state + acc_plus;
}

// generate_random_kernel (random.h:40-53): thread i jumps ahead 4i draws and writes elements i, i+n_thr, i+2n_thr, i+3n_thr.
__global__ void random_uniform_kernel(uint64_t n_elements, Pcg32 rng, float* __restrict__ out, float lower, float upper) {
	const uint64_t i = threadIdx.x + (uint64_t)blockIdx.x * blockDim.x;
	const uint64_t n_threads = (uint64_t)blockDim.x * gridDim.x;
	pcg_advance(rng, i * 4);
#pragma unroll
	for (uint64_t j = 0; j < 4; ++j) {
		const uint64_t idx = i + n_threads * j;
		if (idx >= n_elements) return;
		out[idx] = pcg_next_float(rng) * (upper - lower) + lower;  // contracted to one FMA, as in random.h:69
	}
}

// The same for T = __half (random.h:40-69 with T = __half): the draw is rounded to half, then scaled and shifted in half arithmetic.
__global__ void random_uniform_half_kernel(uint64_t n_elements, Pcg32 rng, __half* __restrict__ out, __half lower, __half upper) {
	const uint64_t i = threadIdx.x + (uint64_t)blockIdx.x * blockDim.x;
	const uint64_t n_threads = (uint64_t)blockDim.x * gridDim.x;
	pcg_advance(rng, i * 4);
#pragma unroll
	for (uint64_t j = 0; j < 4; ++j) {
		const uint64_t idx = i + n_threads * j;
		if (idx >= n_elements) return;
		out[idx] = __float2half(pcg_next_float(rng)) * (upper - lower) + lower;
	}
}

// dst [cols][rows] = src [rows][cols]^T through a padded 32 x 32 shared-memory tile: both the loads and the stores are coalesced.
// Column tiles on grid.x; row tiles on grid.y and a stride loop over it, so any number of rows fits the grid.
template <typename T>
__global__ void transpose_kernel(uint32_t rows, uint32_t cols, const T* __restrict__ src, T* __restrict__ dst) {
	__shared__ T tile[32][33];
	const uint32_t c0 = blockIdx.x * 32;
	for (uint64_t r0 = (uint64_t)blockIdx.y * 32; r0 < rows; r0 += (uint64_t)gridDim.y * 32) {
		for (uint32_t k = threadIdx.y; k < 32; k += blockDim.y) {
			const uint64_t r = r0 + k;
			const uint32_t c = c0 + threadIdx.x;
			if (r < rows && c < cols) tile[k][threadIdx.x] = src[r * cols + c];
		}
		__syncthreads();
		for (uint32_t k = threadIdx.y; k < 32; k += blockDim.y) {
			const uint32_t c = c0 + k;
			const uint64_t r = r0 + threadIdx.x;
			if (r < rows && c < cols) dst[(uint64_t)c * rows + r] = tile[threadIdx.x][k];
		}
		__syncthreads();
	}
}

__global__ void cast_params_kernel(uint64_t n, const float* __restrict__ in, __half* __restrict__ out) {
	const uint64_t i = threadIdx.x + (uint64_t)blockIdx.x * blockDim.x;
	if (i < n) out[i] = (__half)in[i];
}

// grid_scale evaluated on the device exactly as the reference's kernels do (common_device.h:886-891 called from
// grid.h:97 with log2_per_level_scale = std::log2(per_level_scale) computed on the host, grid.h:782).
__global__ void level_scales_kernel(uint32_t n_levels, float log2_per_level_scale, uint32_t base_resolution, float* __restrict__ scales) {
	const uint32_t level = threadIdx.x;
	if (level < n_levels) {
		scales[level] = exp2f(level * log2_per_level_scale) * base_resolution - 1.0f;
	}
}

// ------------------------------------------------------------------------------------------------------------------
// Adam (optimizers/adam.h:48-129). One thread per parameter, same expression order as the reference.
// Differences in data flow only:
//   * matrix (MLP) weight gradients arrive as fp32 sums in dw_accum (written by the fused kernel with red.add.f32);
//     they are rounded to fp16 here -- which is what the reference's gradient buffer holds -- stored to `gradients`
//     for API visibility, and the accumulator is re-armed to zero for the next step.
//   * optimizer state streams use evict-first loads/stores so that the fp16 table + gradient table stay L2 resident.
// ------------------------------------------------------------------------------------------------------------------
// One Adam update, shared by every Adam kernel. Returns false if the parameter is skipped. `Step` is the per-parameter counter:
// uint32_t, or uint16_t saturating at 65535 -- exact when adam_u16_steps_exact() holds, because from t = 65535 on the bias
// correction below is exactly 1 for every larger t.
template <typename Step>
__device__ __forceinline__ bool adam_update(const AdamParams& a, const bool is_matrix, const float loss_scale, const __half grad_h,
                                            float& weight_fp, float& first_moment, float& second_moment, Step& step) {
	float gradient = (float)grad_h / loss_scale;
	if (!is_matrix) {
		if (!a.optimize_non_matrix_params || (gradient == 0 && a.skip_zero_grad_non_matrix_params)) return false;
	} else {
		if (!a.optimize_matrix_params) return false;
	}
	if (is_matrix) {
		gradient += a.l2_reg * weight_fp;
	} else {
		gradient += a.non_matrix_l2_reg * weight_fp;
	}
	if (a.gradient_clipping_magnitude != 0.0f) {
		gradient = copysignf(fminf(fabsf(gradient), a.gradient_clipping_magnitude), gradient);
	}
	const float gradient_sq = gradient * gradient;
	first_moment = a.beta1 * first_moment + (1 - a.beta1) * gradient;
	second_moment = a.beta2 * second_moment + (1 - a.beta2) * gradient_sq;
	float learning_rate = a.learning_rate;
	if (!is_matrix) learning_rate *= a.non_matrix_learning_rate_factor;
	if constexpr (sizeof(Step) == 2) {
		step = step == 0xFFFFu ? step : (Step)(step + 1);
	} else {
		++step;
	}
	const uint32_t current_step = step;
	learning_rate *= sqrtf(1 - powf(a.beta2, (float)current_step)) / (1 - powf(a.beta1, (float)current_step));
	const float effective_learning_rate = fminf(fmaxf(learning_rate / (sqrtf(second_moment) + a.epsilon), a.lower_lr_bound), a.upper_lr_bound);
	const float decayed_weight = (1 - a.relative_decay * learning_rate) * weight_fp - copysignf(a.absolute_decay * learning_rate, weight_fp);
	float new_weight = decayed_weight - effective_learning_rate * first_moment;
	if (a.clipping_magnitude != 0.0f) {
		new_weight = fminf(fmaxf(new_weight, -a.clipping_magnitude), a.clipping_magnitude);
	}
	weight_fp = new_weight;
	return true;
}

// One parameter per thread: the tail / unaligned path (caller-provided arrays that are not 16-byte aligned, lengths that are not a
// multiple of eight); same update as the 8-wide kernel.
template <typename Step>
__global__ void adam_step_kernel(const AdamParams a, const uint32_t n_elements, const uint32_t n_matrix_weights, const float loss_scale,
                                 float* __restrict__ weights_full_precision, __half* __restrict__ weights, __half* __restrict__ gradients,
                                 float* __restrict__ dw_accum, float* __restrict__ first_moments, float* __restrict__ second_moments,
                                 Step* __restrict__ param_steps) {
	pdl_wait();  // no early pdl_launch_dependents(): a long bandwidth-bound kernel should not share its SMs with parked CTAs
	const uint32_t i = threadIdx.x + blockIdx.x * blockDim.x;
	if (i >= n_elements) return;
	__half grad_h;
	if (i < n_matrix_weights && dw_accum != nullptr) {
		grad_h = (__half)dw_accum[i];
		dw_accum[i] = 0.0f;
		gradients[i] = grad_h;
	} else {
		grad_h = gradients[i];
	}
	float w = __ldcs(weights_full_precision + i), m = __ldcs(first_moments + i), v = __ldcs(second_moments + i);
	Step st = __ldcs(param_steps + i);
	if (!adam_update(a, i < n_matrix_weights, loss_scale, grad_h, w, m, v, st)) return;
	__stcs(weights_full_precision + i, w);
	__stcs(first_moments + i, m);
	__stcs(second_moments + i, v);
	__stcs(param_steps + i, st);
	weights[i] = (__half)w;
}

// 8 parameters per thread, every access 128 bits wide: two float4 of each fp32 stream, one uint4 of fp16 params / gradients, and
// one (uint16_t) or two (uint32_t) uint4 of step counters. Groups whose eight gradients are all zero (untouched hash-table entries)
// write nothing back.
template <typename Step>
__global__ void __launch_bounds__(256) adam_step_vec8_kernel(const AdamParams a, const uint32_t n_groups, const uint32_t n_matrix_weights, const float loss_scale,
                                      float4* __restrict__ weights_full_precision, uint4* __restrict__ weights, uint4* __restrict__ gradients,
                                      float4* __restrict__ dw_accum, float4* __restrict__ first_moments, float4* __restrict__ second_moments,
                                      uint4* __restrict__ param_steps) {
	constexpr uint32_t S = sizeof(Step) / 2;  // uint4 chunks of step counters per group
	pdl_wait();
	const uint32_t gidx = threadIdx.x + blockIdx.x * blockDim.x;
	if (gidx >= n_groups) return;
	const uint32_t i0 = gidx * 8;

	// Issue every load of this group up front (independent 128-bit streams); the zero-gradient early-out below only
	// saves the write-back -- untouched groups are ~2 % of a step, memory-level parallelism matters more.
	const bool from_accum = i0 + 7 < n_matrix_weights && dw_accum != nullptr;
	const uint4 raw = from_accum ? make_uint4(0, 0, 0, 0) : gradients[gidx];
	const float4 wa = __ldcs(weights_full_precision + 2 * gidx), wb = __ldcs(weights_full_precision + 2 * gidx + 1);
	const float4 ma = __ldcs(first_moments + 2 * gidx), mb = __ldcs(first_moments + 2 * gidx + 1);
	const float4 va = __ldcs(second_moments + 2 * gidx), vb = __ldcs(second_moments + 2 * gidx + 1);
	union {
		uint4 q[S];
		Step s[8];
	} st;
#pragma unroll
	for (uint32_t k = 0; k < S; ++k) st.q[k] = __ldcs(param_steps + S * gidx + k);

	union {
		uint4 q;
		__half h[8];
	} g;
	if (from_accum) {
		const float4 acc0 = dw_accum[2 * gidx], acc1 = dw_accum[2 * gidx + 1];
		dw_accum[2 * gidx] = make_float4(0.f, 0.f, 0.f, 0.f);
		dw_accum[2 * gidx + 1] = make_float4(0.f, 0.f, 0.f, 0.f);
		g.h[0] = (__half)acc0.x; g.h[1] = (__half)acc0.y; g.h[2] = (__half)acc0.z; g.h[3] = (__half)acc0.w;
		g.h[4] = (__half)acc1.x; g.h[5] = (__half)acc1.y; g.h[6] = (__half)acc1.z; g.h[7] = (__half)acc1.w;
		gradients[gidx] = g.q;
	} else {
		g.q = raw;
		if (i0 >= n_matrix_weights && a.skip_zero_grad_non_matrix_params && ((raw.x | raw.y | raw.z | raw.w) & 0x7FFF7FFFu) == 0) return;  // all eight are +-0
	}

	float w[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w}, m[8] = {ma.x, ma.y, ma.z, ma.w, mb.x, mb.y, mb.z, mb.w}, v[8] = {va.x, va.y, va.z, va.w, vb.x, vb.y, vb.z, vb.w};
	bool any = false;
#pragma unroll
	for (uint32_t k = 0; k < 8; ++k) {
		any |= adam_update(a, i0 + k < n_matrix_weights, loss_scale, g.h[k], w[k], m[k], v[k], st.s[k]);
	}
	if (!any) return;
	__stcs(weights_full_precision + 2 * gidx, make_float4(w[0], w[1], w[2], w[3]));
	__stcs(weights_full_precision + 2 * gidx + 1, make_float4(w[4], w[5], w[6], w[7]));
	__stcs(first_moments + 2 * gidx, make_float4(m[0], m[1], m[2], m[3]));
	__stcs(first_moments + 2 * gidx + 1, make_float4(m[4], m[5], m[6], m[7]));
	__stcs(second_moments + 2 * gidx, make_float4(v[0], v[1], v[2], v[3]));
	__stcs(second_moments + 2 * gidx + 1, make_float4(v[4], v[5], v[6], v[7]));
#pragma unroll
	for (uint32_t k = 0; k < S; ++k) __stcs(param_steps + S * gidx + k, st.q[k]);
	union {
		uint4 q;
		__half h[8];
	} h;
#pragma unroll
	for (uint32_t k = 0; k < 8; ++k) h.h[k] = (__half)w[k];
	weights[gidx] = h.q;
}

// One thread: whether 1 - powf(beta, t) is exactly 1.0f for both betas at t = 65535 and at the largest 32-bit count, with the
// device's own (fast-math) powf. powf(beta, t) is monotone in t, so every t in between gives the same bias correction, 1.
__global__ void adam_u16_steps_exact_kernel(float beta1, float beta2, uint32_t* out) {
	bool exact = true;
	for (const float t : {65535.0f, 4294967295.0f}) exact = exact && 1 - powf(beta1, t) == 1.0f && 1 - powf(beta2, t) == 1.0f;
	*out = exact;
}

__global__ void widen_steps_kernel(uint64_t n, const uint16_t* __restrict__ in, uint32_t* __restrict__ out) {
	const uint64_t i = threadIdx.x + (uint64_t)blockIdx.x * blockDim.x;
	if (i < n) out[i] = in[i];
}

__global__ void narrow_steps_kernel(uint64_t n, const uint32_t* __restrict__ in, uint16_t* __restrict__ out) {
	const uint64_t i = threadIdx.x + (uint64_t)blockIdx.x * blockDim.x;
	if (i < n) out[i] = (uint16_t)min(in[i], 0xFFFFu);
}

__global__ void mlp_grad_finalize_kernel(uint32_t n, float* __restrict__ dw_accum, __half* __restrict__ gradients) {
	pdl_wait();
	pdl_launch_dependents();
	const uint32_t i = threadIdx.x + blockIdx.x * blockDim.x;
	if (i < n) {
		gradients[i] = (__half)dw_accum[i];
		dw_accum[i] = 0.0f;
	}
}

// Adds `value` of every thread of the block (256 threads) onto *sum with ONE atomic per block (a per-warp atomic on a single word
// serialises the whole kernel). Every thread of the block must call it.
__device__ __forceinline__ void block_sum_add(float value, float* sum) {
	__shared__ float warp_sums[8];
#pragma unroll
	for (uint32_t o = 16; o > 0; o >>= 1) value += __shfl_xor_sync(0xFFFFFFFFu, value, o);
	if ((threadIdx.x & 31u) == 0) warp_sums[threadIdx.x >> 5] = value;
	__syncthreads();
	if (threadIdx.x == 0 && sum) {
		float total = 0.0f;
		for (uint32_t w = 0; w < blockDim.x / 32; ++w) total += warp_sums[w];
		if (total != 0.0f) atomicAdd(sum, total);
	}
}

// ---- loss on its own (general, unfused training path; Trainer::forward): prediction rows [batch][stride] fp16 + targets [batch][n_out]
// fp32 -> dL/d(output) rows (x loss_scale, through the output activation's transfer, padding columns zero), per-element values
// [batch][values_stride] (columns from n_out on zero), sum. Same expressions as the fused kernel's output epilogue (fused_common.cuh
// loss_element).
__global__ void loss_kernel(uint32_t loss_type, uint32_t out_act, uint32_t batch, uint32_t n_out, uint32_t stride, float loss_scale, float n_total, const __half* __restrict__ prediction,
                            const float* __restrict__ targets, const float* __restrict__ data_pdf, __half* __restrict__ dL_dy, float* __restrict__ loss_values,
                            uint32_t values_stride, float* __restrict__ loss_sum) {
	pdl_wait();
	pdl_launch_dependents();
	// one thread per (sample, group of 8 output columns): 16-byte loads / stores of the fp16 rows
	const uint32_t groups = stride / 8;
	const uint32_t i = threadIdx.x + blockIdx.x * blockDim.x;
	float value_sum = 0.0f;
	if (i < batch * groups) {
		const uint32_t sample = i / groups, q0 = (i % groups) * 8;
		const uint4 raw = *reinterpret_cast<const uint4*>(prediction + (size_t)sample * stride + q0);
		const __half* y = reinterpret_cast<const __half*>(&raw);
		__half dy[8];
		const float luminance = loss_type == LOSS_RELATIVE_L2_LUMINANCE ? fused::row_luminance(prediction + (size_t)sample * stride, n_out) : 0.0f;
#pragma unroll
		for (uint32_t k = 0; k < 8; ++k) {
			const uint32_t q = q0 + k;
			float gq = 0.0f, value = 0.0f;
			if (q < n_out) {
				float grad;
				const size_t t = (size_t)sample * n_out + q;
				if (data_pdf) fused::loss_element_pdf(loss_type, __half2float(y[k]), targets[t], data_pdf[t], n_total, luminance, value, grad);
				else fused::loss_element(loss_type, __half2float(y[k]), targets[t], n_total, luminance, value, grad);
				gq = loss_scale * grad / n_total;
				value_sum += value;
			}
			if (loss_values && q < values_stride) loss_values[(size_t)sample * values_stride + q] = value;
			dy[k] = fused::act_bwd_h(out_act, __float2half_rn(gq), y[k]);
		}
		if (dL_dy) *reinterpret_cast<uint4*>(dL_dy + (size_t)sample * stride + q0) = *reinterpret_cast<const uint4*>(dy);
	}
	block_sum_add(value_sum, loss_sum);
}

// reduce_sum (reduce_sum.h:132-146): grid-stride partial sums, one atomic per block onto *sum (zeroed by the launcher)
__global__ void reduce_sum_kernel(uint64_t n, const float* __restrict__ values, float* __restrict__ sum) {
	float v = 0.0f;
	for (uint64_t i = threadIdx.x + (uint64_t)blockIdx.x * blockDim.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) v += values[i];
	block_sum_add(v, sum);
}

// dL/d(output) of a caller (Network::backward, fully_fused_mlp.cu:755-762) through the output activation's transfer.
__global__ void activation_backward_output_kernel(uint32_t act, uint64_t n, const __half* __restrict__ grad, const __half* __restrict__ fwd, __half* __restrict__ out) {
	pdl_wait();
	pdl_launch_dependents();
	const uint64_t i = threadIdx.x + (uint64_t)blockIdx.x * blockDim.x;
	if (i < n) out[i] = fused::act_bwd_h(act, grad[i], fwd[i]);
}

// optimizers/ema.h:46-75: debiased exponential moving average of the working weights; `tmp` (fp32 copy of the average) when the
// wrapper runs in full precision.
__global__ void ema_step_kernel(uint32_t n, float decay, float debias_old, float debias_new, const __half* __restrict__ weights, __half* __restrict__ weights_ema, float* __restrict__ tmp) {
	pdl_wait();
	pdl_launch_dependents();
	const uint32_t i = threadIdx.x + blockIdx.x * blockDim.x;
	if (i >= n) return;
	const float prev = tmp ? tmp[i] : __half2float(weights_ema[i]);
	const float filtered = (prev * decay * debias_old + __half2float(weights[i]) * (1.0f - decay)) * debias_new;
	if (tmp) tmp[i] = filtered;
	weights_ema[i] = __float2half_rn(filtered);
}

// ------------------------------------------------------------------------------------------------------------------
// Data parallelism over peer memory. See misc_kernels.h for the protocol.
// ------------------------------------------------------------------------------------------------------------------
__global__ void dp_barrier_kernel(const DpPeers peers, const uint32_t epoch) {
	const uint32_t t = threadIdx.x;
	if (t >= peers.world) return;
	__threadfence_system();  // this rank's earlier writes (gradients, published weights) before the signal
	asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(peers.flags[t] + peers.rank), "r"(epoch) : "memory");
	const uint32_t* mine = peers.flags[peers.rank] + t;
	const long long t0 = clock64();
	for (;;) {
		uint32_t seen;
		asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(seen) : "l"(mine) : "memory");
		if ((int32_t)(seen - epoch) >= 0) break;
		if (clock64() - t0 > 40000000000LL) __trap();  // ~20 s: a peer died; fail loudly instead of hanging the GPU
	}
}

template <bool MULTICAST, typename Step>
__global__ void __launch_bounds__(256) adam_step_dp_kernel(const AdamParams a, const DpPeers peers, const uint64_t first, const uint32_t n_groups, const uint32_t n_matrix_weights,
                                                            const uint64_t n_params, const float loss_scale, float* __restrict__ weights_full_precision,
                                                            float* __restrict__ first_moments, float* __restrict__ second_moments, Step* __restrict__ param_steps) {
	constexpr uint32_t S = sizeof(Step) / 2;  // uint4 chunks of step counters per group of 8
	const uint32_t gidx = threadIdx.x + blockIdx.x * blockDim.x;
	if (gidx >= n_groups) return;
	const uint64_t i0 = first + (uint64_t)gidx * 8;
	if (i0 >= n_params) return;  // padding of the parameter vector: never touched

	// ---- the reduced gradient of 8 consecutive parameters: one 16-byte access per rank, or one in-switch reduction
	uint32_t gw[4];
	if (MULTICAST) {
		asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0, %1, %2, %3}, [%4];" : "=r"(gw[0]), "=r"(gw[1]), "=r"(gw[2]), "=r"(gw[3]) : "l"(peers.grads_mc + i0) : "memory");
	} else {
		float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
		for (uint32_t r = 0; r < peers.world; ++r) {
			uint32_t w[4];
			asm volatile("ld.relaxed.sys.global.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "l"(peers.grads[r] + i0) : "memory");
#pragma unroll
			for (uint32_t k = 0; k < 4; ++k) {
				const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[k]));
				acc[2 * k] += f.x;
				acc[2 * k + 1] += f.y;
			}
		}
#pragma unroll
		for (uint32_t k = 0; k < 4; ++k) {
			const __half2 h = __floats2half2_rn(acc[2 * k], acc[2 * k + 1]);
			gw[k] = *reinterpret_cast<const uint32_t*>(&h);
		}
	}
	// the reduced gradient stays in the local gradient buffer (what trainer->param_gradients() shows for the owned slice)
	*reinterpret_cast<uint4*>(peers.grads[peers.rank] + i0) = make_uint4(gw[0], gw[1], gw[2], gw[3]);
	if (i0 >= n_matrix_weights && a.skip_zero_grad_non_matrix_params && ((gw[0] | gw[1] | gw[2] | gw[3]) & 0x7FFF7FFFu) == 0) return;  // untouched entries (adam.h:79-82)

	const float4* w4p = reinterpret_cast<const float4*>(weights_full_precision + i0);
	const float4* m4p = reinterpret_cast<const float4*>(first_moments + i0);
	const float4* v4p = reinterpret_cast<const float4*>(second_moments + i0);
	uint4* const s4p = reinterpret_cast<uint4*>(param_steps + i0);
	const float4 wa = __ldcs(w4p), wb = __ldcs(w4p + 1), ma = __ldcs(m4p), mb = __ldcs(m4p + 1), va = __ldcs(v4p), vb = __ldcs(v4p + 1);
	union {
		uint4 q[S];
		Step s[8];
	} st;
#pragma unroll
	for (uint32_t k = 0; k < S; ++k) st.q[k] = __ldcs(s4p + k);
	float w[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w}, m[8] = {ma.x, ma.y, ma.z, ma.w, mb.x, mb.y, mb.z, mb.w}, v[8] = {va.x, va.y, va.z, va.w, vb.x, vb.y, vb.z, vb.w};
	const __half* g = reinterpret_cast<const __half*>(gw);
	bool any = false;
#pragma unroll
	for (uint32_t k = 0; k < 8; ++k) any |= adam_update(a, i0 + k < n_matrix_weights, loss_scale, g[k], w[k], m[k], v[k], st.s[k]);
	if (!any) return;
	float4* w4o = reinterpret_cast<float4*>(weights_full_precision + i0);
	float4* m4o = reinterpret_cast<float4*>(first_moments + i0);
	float4* v4o = reinterpret_cast<float4*>(second_moments + i0);
	__stcs(w4o, make_float4(w[0], w[1], w[2], w[3]));
	__stcs(w4o + 1, make_float4(w[4], w[5], w[6], w[7]));
	__stcs(m4o, make_float4(m[0], m[1], m[2], m[3]));
	__stcs(m4o + 1, make_float4(m[4], m[5], m[6], m[7]));
	__stcs(v4o, make_float4(v[0], v[1], v[2], v[3]));
	__stcs(v4o + 1, make_float4(v[4], v[5], v[6], v[7]));
#pragma unroll
	for (uint32_t k = 0; k < S; ++k) __stcs(s4p + k, st.q[k]);
	// ---- publish the working-precision weights to every replica
	uint32_t hw[4];
#pragma unroll
	for (uint32_t k = 0; k < 4; ++k) {
		const __half2 h = __floats2half2_rn(w[2 * k], w[2 * k + 1]);
		hw[k] = *reinterpret_cast<const uint32_t*>(&h);
	}
	if (MULTICAST) {
		asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(peers.params_mc + i0), "r"(hw[0]), "r"(hw[1]), "r"(hw[2]), "r"(hw[3]) : "memory");
	} else {
		for (uint32_t r = 0; r < peers.world; ++r) {
			asm volatile("st.relaxed.sys.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(peers.params[r] + i0), "r"(hw[0]), "r"(hw[1]), "r"(hw[2]), "r"(hw[3]) : "memory");
		}
	}
}

}  // namespace

static inline uint32_t blocks_for(uint64_t n, uint32_t threads) { return (uint32_t)((n + threads - 1) / threads); }

cudaError_t launch_random_uniform(cudaStream_t stream, Pcg32 rng, uint64_t n_elements, float* out, float lower, float upper) {
	if (n_elements == 0) return cudaSuccess;
	const uint64_t n_threads = (n_elements + 3) / 4;
	random_uniform_kernel<<<blocks_for(n_threads, 128), 128, 0, stream>>>(n_elements, rng, out, lower, upper);
	return cudaGetLastError();
}

cudaError_t launch_random_uniform_half(cudaStream_t stream, Pcg32 rng, uint64_t n_elements, __half* out, __half lower, __half upper) {
	if (n_elements == 0) return cudaSuccess;
	const uint64_t n_threads = (n_elements + 3) / 4;
	random_uniform_half_kernel<<<blocks_for(n_threads, 128), 128, 0, stream>>>(n_elements, rng, out, lower, upper);
	return cudaGetLastError();
}

cudaError_t launch_transpose(cudaStream_t stream, uint32_t rows, uint32_t cols, uint32_t element_bytes, const void* src, void* dst) {
	if (rows == 0 || cols == 0) return cudaSuccess;
	const dim3 grid{(cols + 31) / 32, std::min((rows + 31) / 32, 65535u)}, block{32, 8};
	if (element_bytes == 2) transpose_kernel<uint16_t><<<grid, block, 0, stream>>>(rows, cols, (const uint16_t*)src, (uint16_t*)dst);
	else if (element_bytes == 4) transpose_kernel<uint32_t><<<grid, block, 0, stream>>>(rows, cols, (const uint32_t*)src, (uint32_t*)dst);
	else return cudaErrorInvalidValue;
	return cudaGetLastError();
}

cudaError_t launch_cast_params(cudaStream_t stream, uint64_t n, const float* in, __half* out) {
	if (n == 0) return cudaSuccess;
	cast_params_kernel<<<blocks_for(n, 256), 256, 0, stream>>>(n, in, out);
	return cudaGetLastError();
}

cudaError_t launch_level_scales(cudaStream_t stream, uint32_t n_levels, float log2_per_level_scale, uint32_t base_resolution, float* scales_dev) {
	level_scales_kernel<<<1, 128, 0, stream>>>(n_levels, log2_per_level_scale, base_resolution, scales_dev);
	return cudaGetLastError();
}

template <typename Step>
cudaError_t launch_adam_step(cudaStream_t stream, const AdamParams& a, uint32_t n_elements, uint32_t n_matrix_weights, float loss_scale,
                             float* weights_full_precision, __half* weights, __half* gradients, float* dw_accum, float* first_moments,
                             float* second_moments, Step* param_steps) {
	if (n_elements == 0) return cudaSuccess;
	auto aligned = [](const void* p, size_t a) { return ((uintptr_t)p % a) == 0; };
	// A skipped lane of a partially updated group is written back with its loaded (unchanged) value, which is only
	// equivalent to "not touched" if the weights' fp16 copy equals (half)fp32 master -- true for trainer-owned buffers.
	const bool vec_ok = n_elements % 8 == 0 && n_matrix_weights % 8 == 0 && aligned(weights_full_precision, 16) && aligned(weights, 16) && aligned(gradients, 16) &&
	                    aligned(first_moments, 16) && aligned(second_moments, 16) && aligned(param_steps, 16) && (dw_accum == nullptr || aligned(dw_accum, 16));
	if (vec_ok) {
		const uint32_t n_groups = n_elements / 8;
		return launch_pdl(adam_step_vec8_kernel<Step>, blocks_for(n_groups, 256), 256, 0, stream, a, n_groups, n_matrix_weights, loss_scale, (float4*)weights_full_precision,
		                  (uint4*)weights, (uint4*)gradients, (float4*)dw_accum, (float4*)first_moments, (float4*)second_moments, (uint4*)param_steps);
	} else {
		return launch_pdl(adam_step_kernel<Step>, blocks_for(n_elements, 256), 256, 0, stream, a, n_elements, n_matrix_weights, loss_scale, weights_full_precision, weights,
		                  gradients, dw_accum, first_moments, second_moments, param_steps);
	}
}
template cudaError_t launch_adam_step<uint16_t>(cudaStream_t, const AdamParams&, uint32_t, uint32_t, float, float*, __half*, __half*, float*, float*, float*, uint16_t*);
template cudaError_t launch_adam_step<uint32_t>(cudaStream_t, const AdamParams&, uint32_t, uint32_t, float, float*, __half*, __half*, float*, float*, float*, uint32_t*);

cudaError_t adam_u16_steps_exact(const AdamParams& a, bool* exact) {
	uint32_t* flag = nullptr;
	cudaError_t err = cudaMalloc(&flag, sizeof(uint32_t));
	if (err != cudaSuccess) return err;
	adam_u16_steps_exact_kernel<<<1, 1>>>(a.beta1, a.beta2, flag);
	uint32_t value = 0;
	err = cudaMemcpy(&value, flag, sizeof(uint32_t), cudaMemcpyDeviceToHost);
	cudaFree(flag);
	*exact = value != 0;
	return err;
}

cudaError_t launch_widen_steps(cudaStream_t stream, uint64_t n, const uint16_t* in, uint32_t* out) {
	if (n == 0) return cudaSuccess;
	widen_steps_kernel<<<blocks_for(n, 256), 256, 0, stream>>>(n, in, out);
	return cudaGetLastError();
}

cudaError_t launch_narrow_steps(cudaStream_t stream, uint64_t n, const uint32_t* in, uint16_t* out) {
	if (n == 0) return cudaSuccess;
	narrow_steps_kernel<<<blocks_for(n, 256), 256, 0, stream>>>(n, in, out);
	return cudaGetLastError();
}

cudaError_t launch_mlp_grad_finalize(cudaStream_t stream, uint32_t n, float* dw_accum, __half* gradients) {
	if (n == 0) return cudaSuccess;
	return launch_pdl(mlp_grad_finalize_kernel, blocks_for(n, 256), 256, 0, stream, n, dw_accum, gradients);
}

cudaError_t launch_loss(cudaStream_t stream, uint32_t loss_type, uint32_t output_activation, uint32_t batch, uint32_t n_out, uint32_t stride, float loss_scale, uint32_t n_total,
                        const __half* prediction, const float* targets, const float* data_pdf, __half* dL_dy, float* loss_values, uint32_t values_stride, float* loss_sum) {
	if ((uint64_t)batch * stride >= (1ull << 32) || stride % 8 != 0 || values_stride < n_out || values_stride > stride) return cudaErrorInvalidValue;
	return launch_pdl(loss_kernel, blocks_for(batch * (stride / 8), 256), 256, 0, stream, loss_type, output_activation, batch, n_out, stride, loss_scale, (float)n_total, prediction, targets,
	                  data_pdf, dL_dy, loss_values, values_stride, loss_sum);
}

cudaError_t launch_reduce_sum(cudaStream_t stream, uint64_t n, const float* values, float* sum) {
	cudaError_t e = cudaMemsetAsync(sum, 0, sizeof(float), stream);
	if (e != cudaSuccess || n == 0) return e;
	reduce_sum_kernel<<<(uint32_t)std::min<uint64_t>((n + 255) / 256, 1024), 256, 0, stream>>>(n, values, sum);
	return cudaGetLastError();
}

cudaError_t launch_activation_backward_output(cudaStream_t stream, uint32_t activation, uint64_t n, const __half* grad, const __half* forward_output, __half* out) {
	if (n == 0) return cudaSuccess;
	return launch_pdl(activation_backward_output_kernel, (uint32_t)((n + 255) / 256), 256, 0, stream, activation, n, grad, forward_output, out);
}

cudaError_t launch_ema_step(cudaStream_t stream, uint32_t n, float decay, float debias_old, float debias_new, const __half* weights, __half* weights_ema, float* tmp) {
	if (n == 0) return cudaSuccess;
	return launch_pdl(ema_step_kernel, blocks_for(n, 256), 256, 0, stream, n, decay, debias_old, debias_new, weights, weights_ema, tmp);
}

cudaError_t launch_dp_barrier(cudaStream_t stream, const DpPeers& peers, uint32_t epoch) {
	if (peers.world < 1 || peers.world > DP_MAX_RANKS) return cudaErrorInvalidValue;
	dp_barrier_kernel<<<1, 32, 0, stream>>>(peers, epoch);
	return cudaGetLastError();
}

template <typename Step>
cudaError_t launch_adam_step_dp(cudaStream_t stream, const AdamParams& a, const DpPeers& peers, uint64_t first, uint64_t count, uint32_t n_matrix_weights, uint64_t n_params,
                                float loss_scale, float* weights_full_precision, float* first_moments, float* second_moments, Step* param_steps) {
	if (count == 0) return cudaSuccess;
	if (first % 8 != 0 || count % 8 != 0 || n_params % 8 != 0 || n_matrix_weights % 8 != 0) return cudaErrorInvalidValue;
	const uint32_t n_groups = (uint32_t)(count / 8);
	if (peers.grads_mc && peers.params_mc) {
		adam_step_dp_kernel<true, Step><<<blocks_for(n_groups, 256), 256, 0, stream>>>(a, peers, first, n_groups, n_matrix_weights, n_params, loss_scale, weights_full_precision, first_moments,
		                                                                                second_moments, param_steps);
	} else {
		adam_step_dp_kernel<false, Step><<<blocks_for(n_groups, 256), 256, 0, stream>>>(a, peers, first, n_groups, n_matrix_weights, n_params, loss_scale, weights_full_precision, first_moments,
		                                                                                 second_moments, param_steps);
	}
	return cudaGetLastError();
}
template cudaError_t launch_adam_step_dp<uint16_t>(cudaStream_t, const AdamParams&, const DpPeers&, uint64_t, uint64_t, uint32_t, uint64_t, float, float*, float*, float*, uint16_t*);
template cudaError_t launch_adam_step_dp<uint32_t>(cudaStream_t, const AdamParams&, const DpPeers&, uint64_t, uint64_t, uint32_t, uint64_t, float, float*, float*, float*, uint32_t*);

}  // namespace tcnnb
