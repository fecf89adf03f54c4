// fused_common.cuh -- device helpers shared by the wgmma kernels (fused_ws.cu, mlp_fused.cu).
#pragma once
#include "common.cuh"
#include "ptx.cuh"

namespace tcnnb {
namespace fused {

using namespace ptx;

constexpr uint32_t TILE_BYTES = TILE_M * 128;  // [128][64] fp16
constexpr uint32_t WIDTH = 64;

// Byte offset of 16-byte chunk `c` (0..7) of row `r` inside a SWIZZLE_128B tile.
__device__ __forceinline__ uint32_t sw128(uint32_t r, uint32_t c) {
	return r * 128u + ((c ^ (r & 7u)) << 4);
}

__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
	asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

__device__ __forceinline__ void ld_shared_v4(uint32_t addr, uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d) {
	asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"(addr) : "memory");
}

__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
	__half2 h = __floats2half2_rn(lo, hi);
	return *reinterpret_cast<uint32_t*>(&h);
}

__device__ __forceinline__ uint32_t relu_pack(uint32_t lo_bits, uint32_t hi_bits) {
	// fp32 accumulator -> fp16 (rn) -> ReLU in fp16, as warp_activation<__half> does (common_device.h:115-121).
	__half2 h = __floats2half2_rn(__uint_as_float(lo_bits), __uint_as_float(hi_bits));
	h = __hmax2(h, __float2half2_rn(0.0f));
	return *reinterpret_cast<uint32_t*>(&h);
}

// gradient (fp32 acc -> fp16) * (forward > 0), warp_activation_backward ReLU (common_device.h:363-368).
__device__ __forceinline__ uint32_t relu_bwd_pack(uint32_t lo_bits, uint32_t hi_bits, uint32_t fwd_bits) {
	__half2 g = __floats2half2_rn(__uint_as_float(lo_bits), __uint_as_float(hi_bits));
	const __half2 f = *reinterpret_cast<const __half2*>(&fwd_bits);
	const __half2 mask = __hgt2(f, __float2half2_rn(0.0f));  // 1.0 / 0.0
	g = __hmul2(g, mask);
	return *reinterpret_cast<uint32_t*>(&g);
}

// ---- generic activations, evaluated like the reference's warp_activation<__half> / warp_activation_backward<__half>
// (common_device.h:110-215, 354-420): on the fp16-rounded value, transcendental math in fp32, result rounded to fp16.
__device__ __forceinline__ __half act_fwd_h(uint32_t act, __half x) {
	const float xf = __half2float(x);
	switch (act) {
		case ACT_RELU: return __hmax(x, __float2half_rn(0.0f));
		case ACT_LEAKY_RELU: return __hmul(x, __float2half_rn(__hgt(x, __float2half_rn(0.0f)) ? 1.0f : 0.01f));
		case ACT_EXPONENTIAL: return __float2half_rn(expf(xf));
		case ACT_SIGMOID: return __float2half_rn(1.0f / (1.0f + expf(-xf)));
		case ACT_SQUAREPLUS: { const float v = xf * 10.0f; return __float2half_rn(0.5f * (v + sqrtf(v * v + 4)) / 10.0f); }
		case ACT_SOFTPLUS: return __float2half_rn(logf(expf(xf * 10.0f) + 1.0f) / 10.0f);
		case ACT_TANH: return __float2half_rn(tanhf(xf));
		default: return x;  // None
	}
}

// grad * f'(.) expressed through the stored FORWARD (post-activation) value, all products in fp16 like the reference.
__device__ __forceinline__ __half act_bwd_h(uint32_t act, __half grad, __half fwd) {
	const float f = __half2float(fwd);
	switch (act) {
		case ACT_RELU: return __hmul(grad, __float2half_rn(__hgt(fwd, __float2half_rn(0.0f)) ? 1.0f : 0.0f));
		case ACT_LEAKY_RELU: return __hmul(grad, __float2half_rn(__hgt(fwd, __float2half_rn(0.0f)) ? 1.0f : 0.01f));
		case ACT_EXPONENTIAL: return __hmul(grad, fwd);
		case ACT_SIGMOID: return __hmul(grad, __hmul(fwd, __float2half_rn(1.0f - f)));
		case ACT_SQUAREPLUS: { const float y = f * 10.0f; return __hmul(grad, __float2half_rn(y * y / (y * y + 1))); }
		case ACT_SOFTPLUS: return __hmul(grad, __float2half_rn(1.0f - expf(-f * 10.0f)));
		case ACT_TANH: return __hmul(grad, __float2half_rn(1.0f - f * f));
		default: return grad;  // None
	}
}

__device__ __forceinline__ uint32_t act_pack(uint32_t act, uint32_t lo_bits, uint32_t hi_bits) {
	if (act == ACT_RELU) return relu_pack(lo_bits, hi_bits);  // packed fast path
	const __half2 x = __floats2half2_rn(__uint_as_float(lo_bits), __uint_as_float(hi_bits));
	const __half2 y = __halves2half2(act_fwd_h(act, __low2half(x)), act_fwd_h(act, __high2half(x)));
	return *reinterpret_cast<const uint32_t*>(&y);
}

__device__ __forceinline__ uint32_t act_bwd_pack(uint32_t act, uint32_t lo_bits, uint32_t hi_bits, uint32_t fwd_bits) {
	if (act == ACT_RELU) return relu_bwd_pack(lo_bits, hi_bits, fwd_bits);
	const __half2 g = __floats2half2_rn(__uint_as_float(lo_bits), __uint_as_float(hi_bits));
	const __half2 f = *reinterpret_cast<const __half2*>(&fwd_bits);
	const __half2 y = __halves2half2(act_bwd_h(act, __low2half(g), __low2half(f)), act_bwd_h(act, __high2half(g), __high2half(f)));
	return *reinterpret_cast<const uint32_t*>(&y);
}

// One element of the loss (src/loss.cu:57-66; losses/l2.h:56-74, relative_l2.h:56-75, relative_l2_luminance.h:40-86, l1.h:68-73,
// relative_l1.h:71-76, mape.h:72-77, smape.h:72-77, cross_entropy.h:40-76, variance_is.h:40-77; data_pdf == 1): `value` is already
// divided by n_total = loss-batch size x output dims, `grad` is d(value)/d(pred) x n_total. `luminance`: of the row's predictions
// (RelativeL2Luminance only, see row_luminance).
__device__ __forceinline__ void loss_element(uint32_t loss_type, float pred, float target, float n_total, float luminance, float& value, float& grad) {
	const float diff = pred - target;
	if (loss_type == LOSS_RELATIVE_L2 || loss_type == LOSS_RELATIVE_L2_LUMINANCE) {
		const float base = loss_type == LOSS_RELATIVE_L2 ? pred : luminance;
		const float psq = base * base + 0.01f;
		value = diff * diff / psq / n_total;
		grad = 2.0f * diff / psq;
	} else if (loss_type == LOSS_L2) {
		value = diff * diff / n_total;
		grad = 2.0f * diff;
	} else if (loss_type == LOSS_L1) {
		value = fabsf(diff) / n_total;
		grad = copysignf(1.0f, diff);
	} else if (loss_type == LOSS_CROSS_ENTROPY) {
		const float factor = -target / n_total;
		value = factor * logf(pred);
		grad = factor / pred * n_total;
	} else if (loss_type == LOSS_VARIANCE_IS) {
		const float factor = target * target / n_total;
		value = factor / pred - factor;
		grad = -factor / (pred * pred) * n_total;
	} else {  // RelativeL1 / Mape / Smape
		const float denom = loss_type == LOSS_RELATIVE_L1 ? fabsf(pred) : (loss_type == LOSS_MAPE ? fabsf(target) : 0.5f * (fabsf(target) + fabsf(pred)));
		const float scale = 1.0f / (denom + 1e-2f);
		value = fabsf(diff) * scale / n_total;
		grad = copysignf(scale, diff);
	}
}

// 0.299 r + 0.587 g + 0.114 b of a row of predictions; with 6 or more outputs, channels 3..5 are added to 0..2 first
// (relative_l2_luminance.h:69-77). `row`: the first 6 predictions of the sample.
__device__ __forceinline__ float row_luminance(const __half* row, uint32_t dims) {
	float r = __half2float(row[0]), g = __half2float(row[1]), b = __half2float(row[2]);
	if (dims >= 6) {
		r += __half2float(row[3]);
		g += __half2float(row[4]);
		b += __half2float(row[5]);
	}
	return 0.299f * r + 0.587f * g + 0.114f * b;
}

struct SmemSync {
	// dynamic shared memory, 1024-byte aligned:
	//   [ enc_0 | enc_1 | h_0 .. h_{NH-1} | dy | (park) | W_0 .. W_{NH-1} | W_out ] then barriers
	uint32_t enc, h0, dy, park, w0, w_out, bar, tmem_slot, levels;
};


}  // namespace fused
}  // namespace tcnnb
