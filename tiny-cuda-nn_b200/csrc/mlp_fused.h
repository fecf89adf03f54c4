// mlp_fused.h -- launch interface of the stand-alone FullyFusedMLP forward kernel (mlp_fused.cu).
#pragma once
#include "common.cuh"

namespace tcnnb {

// What the kernel reads from its parameter block (mlp_fused.cu, MlpKernelParams); the launch interface is MlpForwardParams below.
struct MlpChainParams {
	// network (fully_fused_mlp.cu:635-672): W_0 [width][in_width], (n_hidden_layers - 1) x [width][width], W_out [out_width][width],
	// row-major fp16, contiguous in this order
	uint32_t width;              // 16 / 32 / 64 / 128 / 256
	uint32_t in_width;           // multiple of 16, <= max(width, 64) ... see mlp_forward_supported()
	uint32_t out_width;          // PADDED output width: multiple of 16, <= MLP_MAX_OUTPUT_WIDTH (wider than `width`: the WIDE kernels)
	uint32_t n_hidden_layers;    // >= 1
	uint32_t activation;         // hidden activation (Activation enum)
	uint32_t output_activation;
	const __half* weights;
	// batch
	uint32_t batch_size;         // multiple of 128
	// input: exactly one of the two
	const __half* input_fp16;    // [batch][in_width] fp16 (Network<T>::inference_mixed_precision, column-major in_width x batch)
	const float* input_fp32;     // [batch][n_input_dims] fp32 through the Identity encoding (encodings/identity.h:46-67):
	uint32_t n_input_dims;       //   feature j < n_input_dims = (half)x_j, features n_input_dims .. in_width-1 = 1 (padding with ones)
	// output: either / both may be null
	__half* output_fp16;         // [batch][out_width]
	float* output_fp32;          // [batch][n_output_dims] (network->inference: trimmed + cast, object.h:214-282)
	uint32_t n_output_dims;
	// optional: post-activation hidden layers [n_hidden_layers][batch][width] fp16 (forward pass kept for a backward pass)
	__half* hidden_out;
	// backward chain (Network<T>::backward's dgrad half, fully_fused_mlp.cu:733-800): with `backward` set,
	//   input_fp16  = dL/d(output) [batch][out_width], already multiplied by the output activation's derivative,
	//   hidden_in   = the forward pass's `hidden_out` (Sine / SiLU: its `hidden_pre_out`),
	//   hidden_out  = g_l = dL/d(pre-activation of hidden layer l) [n_hidden_layers][batch][width] (may be null),
	//   output_fp16 = dL/d(input) [batch][in_width] (may be null: the last step of the chain is then skipped).
	uint32_t backward;
	const __half* hidden_in;
	// profiling only (tcnnb_network_debug_clocks): clock64 stamps [cta][consumer warpgroup (5 slots)][64 events][8], null in production
	long long* dbg_clock;
};

struct MlpForwardParams : MlpChainParams {
	// Sine / SiLU hidden activation only (activation_needs_preact): the fp16 PRE-activation rows z_l [n_hidden_layers][batch][width],
	// required with hidden_out (the backward chain reads them as its `hidden_in`); hidden_out = act(hidden_pre_out) bit for bit.
	// Kept out of MlpChainParams so that the parameter block of the other activations' kernels keeps its layout.
	__half* hidden_pre_out;
};

// Widest padded network output the stand-alone kernels run. An output wider than n_neurons is computed in chunks of n_neurons rows of
// the output matrix (the WIDE kernels).
constexpr uint32_t MLP_MAX_OUTPUT_WIDTH = 1024;

// Maximum number of weight matrices that stay resident in shared memory for a width (more layers stream through a ring).
uint32_t mlp_forward_resident_layers(uint32_t width);
bool mlp_forward_supported(const MlpForwardParams& p, const char** why);
cudaError_t launch_mlp_forward(const MlpForwardParams& p, uint32_t n_sms, cudaStream_t stream);

// ---- weight gradients of the stand-alone network (mlp_wgrad.cu) ------------------------------------------------------------
struct MlpWgradParams {
	uint32_t width, in_width, out_width, n_hidden_layers;
	uint32_t batch_size;          // multiple of 128
	const __half* input;          // [batch][in_width]                   the network input of the forward pass
	const __half* hidden;         // [n_hidden_layers][batch][width]     forward activations (mlp forward `hidden_out`)
	const __half* grad_hidden;    // [n_hidden_layers][batch][width]     g_l (backward chain `hidden_out`)
	const __half* grad_output;    // [batch][out_width]                  dL/d(output) through the output activation's transfer
	float* dw_accum;              // fp32 sums in parameter order, ADDED into (red.global.add.f32): the caller zeroes them
};
// dW_l += g_l^T . h_{l-1} for every weight matrix (the reference's split-k GEMMs, fully_fused_mlp.cu:802-866).
bool mlp_wgrad_supported(const MlpWgradParams& p, const char** why);
cudaError_t launch_mlp_wgrad(const MlpWgradParams& p, uint32_t n_sms, cudaStream_t stream, uint32_t* n_launches = nullptr);


// ---- the whole backward pass of the stand-alone network: [output activation backward] -> dgrad chain -> weight gradients ------
struct MlpBackwardArgs {
	uint32_t width, in_width, out_width, n_hidden_layers, activation, output_activation;
	const __half* weights;
	uint32_t batch_size;
	const __half* input;          // [batch][in_width] forward input (weight gradients of the first matrix); may be null if dw_accum is
	const __half* hidden;         // [n_hidden_layers][batch][width] forward activations
	const __half* hidden_pre;     // [n_hidden_layers][batch][width] forward pre-activations; Sine / SiLU only (activation_needs_preact)
	const __half* output;         // [batch][out_width] forward output; only read when output_activation != None
	const __half* dL_doutput;     // [batch][out_width]
	__half* grad_hidden;          // scratch [n_hidden_layers][batch][width]
	__half* grad_output;          // scratch [batch][out_width]; only written when output_activation != None
	__half* dL_dinput;            // [batch][in_width] or null
	float* dw_accum;              // fp32 sums, added into; null = no weight gradients
};
cudaError_t launch_mlp_backward(const MlpBackwardArgs& a, uint32_t n_sms, cudaStream_t stream, uint32_t* n_launches);
bool mlp_backward_supported(const MlpBackwardArgs& a, const char** why);

}  // namespace tcnnb
