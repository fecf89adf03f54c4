// misc_kernels.h -- launch interface of misc_kernels.cu.
#pragma once
#include "common.cuh"

namespace tcnnb {

// Hyper-parameters of optimizers/adam.h:221-303 with the reference's defaults (adam.h:337-355).
struct AdamParams {
	float learning_rate = 1e-3f;
	float beta1 = 0.9f;
	float beta2 = 0.999f;
	float epsilon = 1e-8f;
	float l2_reg = 1e-8f;
	float relative_decay = 0.0f;
	float absolute_decay = 0.0f;
	float clipping_magnitude = 0.0f;
	float gradient_clipping_magnitude = 0.0f;
	float non_matrix_learning_rate_factor = 1.0f;
	float non_matrix_l2_reg = 0.0f;
	float lower_lr_bound = 0.0f;          // AdaBound bounds, recomputed per step on the host (adam.h:161-168)
	float upper_lr_bound = 3.402823466e+38f;
	int adabound = 0;
	int optimize_matrix_params = 1;
	int optimize_non_matrix_params = 1;
	int skip_zero_grad_non_matrix_params = 1;
};

cudaError_t launch_random_uniform(cudaStream_t stream, Pcg32 rng, uint64_t n_elements, float* out, float lower, float upper);
// generate_random_uniform<__half> (random.h:40-69 with T = __half): the same stream as the float fill, rounded to half before the affine map.
cudaError_t launch_random_uniform_half(cudaStream_t stream, Pcg32 rng, uint64_t n_elements, __half* out, __half lower, __half upper);
// dst [cols][rows] = src [rows][cols]^T for 2- or 4-byte elements (row-major <-> column-major matrices of the C++ object tier).
cudaError_t launch_transpose(cudaStream_t stream, uint32_t rows, uint32_t cols, uint32_t element_bytes, const void* src, void* dst);
cudaError_t launch_cast_params(cudaStream_t stream, uint64_t n, const float* in, __half* out);
cudaError_t launch_level_scales(cudaStream_t stream, uint32_t n_levels, float log2_per_level_scale, uint32_t base_resolution, float* scales_dev);
// Adam's per-parameter step counters are uint32_t, or uint16_t saturating at 65535 when adam_u16_steps_exact() says that this gives
// bit-identical updates (Step = uint16_t or uint32_t).
template <typename Step>
cudaError_t launch_adam_step(cudaStream_t stream, const AdamParams& a, uint32_t n_elements, uint32_t n_matrix_weights, float loss_scale,
                             float* weights_full_precision, __half* weights, __half* gradients, float* dw_accum, float* first_moments,
                             float* second_moments, Step* param_steps);
// Whether Adam's bias correction sqrtf(1 - powf(beta2, t)) / (1 - powf(beta1, t)), evaluated on the device, is exactly 1 for every
// t >= 65535: then a counter that stops at 65535 updates exactly like one that keeps counting. Synchronous (one-thread probe).
cudaError_t adam_u16_steps_exact(const AdamParams& a, bool* exact);
// uint16_t <-> uint32_t copies of the step counters (narrowing saturates at 65535).
cudaError_t launch_widen_steps(cudaStream_t stream, uint64_t n, const uint16_t* in, uint32_t* out);
cudaError_t launch_narrow_steps(cudaStream_t stream, uint64_t n, const uint32_t* in, uint16_t* out);
cudaError_t launch_mlp_grad_finalize(cudaStream_t stream, uint32_t n, float* dw_accum, __half* gradients);

// General (unfused) training path and Trainer::forward: loss + dL/d(output) from fp16 prediction rows [batch][stride]; data_pdf ([batch][n_out],
// divides the loss as in losses/*.h), dL_dy, loss_values ([batch][values_stride], n_out <= values_stride <= stride, columns from n_out on
// zero) and loss_sum may be null.
cudaError_t launch_loss(cudaStream_t stream, uint32_t loss_type, uint32_t output_activation, uint32_t batch, uint32_t n_out, uint32_t stride, float loss_scale, uint32_t n_total,
                        const __half* prediction, const float* targets, const float* data_pdf, __half* dL_dy, float* loss_values, uint32_t values_stride, float* loss_sum);
// *sum = the fp32 sum of values[0, n) (reduce_sum.h:132-146), stream-ordered.
cudaError_t launch_reduce_sum(cudaStream_t stream, uint64_t n, const float* values, float* sum);
// out = grad * f'(.) of the output activation, expressed through the forward output (element-wise, fp16).
cudaError_t launch_activation_backward_output(cudaStream_t stream, uint32_t activation, uint64_t n, const __half* grad, const __half* forward_output, __half* out);

// Ema wrapper (optimizers/ema.h:46-75): weights_ema = (weights_ema * decay * debias_old + weights * (1 - decay)) * debias_new; tmp optional (fp32 average)
cudaError_t launch_ema_step(cudaStream_t stream, uint32_t n, float decay, float debias_old, float debias_new, const __half* weights, __half* weights_ema, float* tmp);

// ---- data parallelism over peer memory (NVLink / NVSwitch): one-pass "reduce + Adam + publish" on this rank's slice ----------------
// Every rank holds [fp16 params | fp16 gradients | flags] at the SAME offsets of a symmetric allocation that all peers have
// mapped (rendezvous by the host framework). peers.* are this rank's views of every rank's copy; *_mc are the NVLS multicast
// views of the same regions (null when the fabric has no multicast: the kernels then loop over the peer pointers).
constexpr uint32_t DP_MAX_RANKS = 8;
struct DpPeers {
	uint32_t world, rank;
	__half* params[DP_MAX_RANKS];
	__half* grads[DP_MAX_RANKS];
	uint32_t* flags[DP_MAX_RANKS];  // [DP_MAX_RANKS] monotonic epoch counters per rank: flags[r][q] = last barrier rank q has reached, as seen by rank r
	__half* params_mc;
	__half* grads_mc;
};
// Cross-GPU barrier on `stream`: everything enqueued before it on every rank's stream is complete and visible to all ranks before
// anything enqueued after it starts. `epoch` must increase by one per call, identically on all ranks.
cudaError_t launch_dp_barrier(cudaStream_t stream, const DpPeers& peers, uint32_t epoch);
// Adam over the parameters [first, first + count) (multiples of 8) of the padded vector: the gradient of a parameter is the SUM over
// ranks of grads[r][i] (multimem.ld_reduce in the switch, or peer loads), evaluated once by the slice's owner; the updated fp16
// weight is published into every rank's params (multimem.st, or peer stores); the reduced gradient is left in the local gradient
// buffer. State arrays (fp32 master, moments, steps) are local and indexed by the global parameter index.
template <typename Step>
cudaError_t launch_adam_step_dp(cudaStream_t stream, const AdamParams& a, const DpPeers& peers, uint64_t first, uint64_t count, uint32_t n_matrix_weights, uint64_t n_params,
                                float loss_scale, float* weights_full_precision, float* first_moments, float* second_moments, Step* param_steps);

}  // namespace tcnnb
