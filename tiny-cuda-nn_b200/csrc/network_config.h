// network_config.h -- host-side description of the MLP behind every tier (model.cu: trainer / module tiers; network.cu: the
// stand-alone network tier): the "network" JSON with the reference's keys, defaults and error texts (src/network.cu:51-141), the
// parameter layout and the xavier initialisation (fully_fused_mlp.cu:635-672, 868-892), and the runner of the stand-alone network
// kernels that the network tier and the general path share.
#pragma once
#include "common.cuh"
#include "host_common.h"
#include "json_mini.h"
#include "mlp_fused.h"

#include <cmath>
#include <string>
#include <utility>
#include <vector>

namespace tcnnb {

struct MlpConfig {
	std::string otype = "FullyFusedMLP";
	uint32_t in_width = 0;
	uint32_t width = 128;
	uint32_t n_hidden_layers = 5;
	uint32_t out_width = 0;
	uint32_t padded_out_width = 0;
	uint32_t activation = ACT_RELU;
	uint32_t output_activation = ACT_NONE;
	uint32_t n_params = 0;
};

// `in_width`: the (padded) width of the encoding in front of the network; `n_out`: the unpadded output width.
inline MlpConfig parse_network(const json::Value& net, uint32_t in_width, uint32_t n_out) {
	MlpConfig c;
	c.otype = net.value("otype", "MLP");  // src/network.cu:52-54
	const bool fully_fused = ieq(c.otype, "FullyFusedMLP") || ieq(c.otype, "MegakernelMLP");
	const bool cutlass = ieq(c.otype, "MLP") || ieq(c.otype, "CutlassMLP");
	if (!fully_fused && !cutlass) throw std::runtime_error("Invalid network type: " + c.otype);
	c.width = (uint32_t)net.value("n_neurons", 128.0);
	c.n_hidden_layers = (uint32_t)net.value("n_hidden_layers", 5.0);
	c.activation = parse_activation(net.value("activation", "ReLU"));
	c.output_activation = parse_activation(net.value("output_activation", "None"));
	// Both otypes run on the same wgmma kernels (there is no separate non-fused network in this library), so both take the fused
	// kernel's widths, and CutlassMLP also 256 (the width of SIREN and neural-SDF networks); the reference's CutlassMLP accepts any
	// multiple of 8.
	if (!(c.width == 16 || c.width == 32 || c.width == 64 || c.width == 128 || (cutlass && c.width == 256))) {
		const std::string msg = "FullyFusedMLP only supports 16, 32, 64, and 128 neurons, but got " + std::to_string(c.width) + ". Use CutlassMLP instead if this is a requirement.";
		throw std::runtime_error(cutlass ? msg + " (tcnn_b200's CutlassMLP runs these widths and 256.)" : msg);
	}
	if (c.n_hidden_layers < 1) throw std::runtime_error("FullyFusedMLP requires at least 1 hidden layer (3 layers in total).");
	// Sine and SiLU need stored pre-activations: FullyFusedMLP rejects them (fully_fused_mlp.cu:689-699); CutlassMLP keeps them
	// (cutlass_mlp.cu:53, 162-209) as the hidden activation. As output activation they have no derivative in the reference
	// (warp_activation_backward leaves the gradient unwritten, common_device.h:375-390), so both otypes reject them there.
	if (fully_fused && activation_needs_preact(c.activation)) throw std::runtime_error("Unsupported activation.");
	if (activation_needs_preact(c.output_activation)) {
		throw std::runtime_error("Unsupported activation. Sine / SiLU are not supported as output_activation: they have no output-activation derivative (CutlassMLP accepts them as the hidden activation).");
	}
	c.in_width = in_width;
	c.out_width = n_out;
	c.padded_out_width = next_multiple(n_out, 16u);
	c.n_params = c.width * c.in_width + (c.n_hidden_layers - 1) * c.width * c.width + c.padded_out_width * c.width;
	return c;
}

// Xavier uniform per matrix on the host, sequential draws from `rng` (fully_fused_mlp.cu:868-892, gpu_matrix.h:292-306). A Sine
// network takes the SIREN initialisation instead (cutlass_mlp.cu:362-371): bound scale * 30 / fan_in for the first matrix
// (initialize_siren_uniform_first, gpu_matrix.h:360-377), scale * sqrt(6 / fan_in) for the others, the output matrix included
// (initialize_siren_uniform, gpu_matrix.h:343-358); same draw order and expression per element.
// `dst`: DEVICE fp32 array of c.n_params elements.
inline void init_mlp_params(const MlpConfig& c, HostPcg32& rng, float* dst, float scale) {
	std::vector<float> w(c.n_params);
	std::vector<std::pair<uint32_t, uint32_t>> mats;  // (rows = fan_out, cols = fan_in)
	mats.emplace_back(c.width, c.in_width);
	for (uint32_t i = 0; i + 1 < c.n_hidden_layers; ++i) mats.emplace_back(c.width, c.width);
	mats.emplace_back(c.padded_out_width, c.width);
	size_t pos = 0;
	for (size_t m = 0; m < mats.size(); ++m) {
		const auto& rc = mats[m];
		float bound = scale;
		if (c.activation != ACT_SINE) bound *= std::sqrt(6.0f / (float)(rc.second + rc.first));
		else if (m == 0) bound *= 30.0f / (float)rc.second;
		else bound *= std::sqrt(6.0f / (float)rc.second);
		for (size_t i = 0; i < (size_t)rc.first * rc.second; ++i) w[pos++] = rng.next_float() * 2.0f * bound - bound;
	}
	TCNNB_CUDA_CHECK(cudaMemcpy(dst, w.data(), sizeof(float) * w.size(), cudaMemcpyHostToDevice));
}

// ---- runner of the stand-alone network kernels (mlp_fused.cu / mlp_wgrad.cu), defined in network.cu. The activations a forward pass
// keeps for the backward pass are `hidden` [n_forward_activations][batch][width]: the post-activations of every hidden layer, and for
// Sine / SiLU the pre-activations after them (CutlassMLP::num_forward_activations(), cutlass_mlp.cu:162-209).
inline uint32_t n_forward_activations(const MlpConfig& c) { return activation_needs_preact(c.activation) ? 2 * c.n_hidden_layers : c.n_hidden_layers; }

// Whether the kernels cover this network's shape (they have their own limits, e.g. dL/d(input) wider than the layers): nullptr, else
// the reason they do not. `input_gradient`: the backward pass has to produce dL/d(input).
const char* mlp_unsupported(const MlpConfig& c, bool input_gradient);

// Forward-pass arguments for `batch` rows; with `hidden`, the pass keeps its activations there. The caller sets input and output.
MlpForwardParams mlp_forward_params(const MlpConfig& c, const __half* weights, uint32_t batch, __half* hidden = nullptr);
// Throws the kernel's reason if it does not cover `p`, else launches it (adds to g_kernel_launches).
void run_mlp_forward(const MlpForwardParams& p, int n_sms, cudaStream_t stream);

// Scratch of a tier that runs backward passes, grown on demand and reused.
struct MlpScratch {
	DeviceBuffer<__half> hidden;       // activations kept by a forward pass (hidden_rows)
	DeviceBuffer<__half> grad_hidden;  // g_l = dL/d(pre-activation of hidden layer l), for the weight gradients
	DeviceBuffer<__half> grad_output;  // dL/d(output) through the output activation
	// tests only (tcnnb_network_debug_grad_hidden): when set, the backward pass writes g_l here instead of `grad_hidden`, with or
	// without weight gradients -- [n_hidden_layers][batch][width] fp16, owned by the caller
	__half* grad_hidden_tap = nullptr;
	__half* hidden_rows(const MlpConfig& c, uint32_t batch);
};

// Network<T>::backward (fully_fused_mlp.cu:733-866) from a forward pass's input, `hidden` and output: dL/d(input) (fp16 rows) into
// `dL_dinput` and the weight gradients ADDED into the fp32 sums `dw_accum`; either may be null. `apply_output_activation`: dL_doutput
// has yet to pass the output activation's derivative. Throws the kernels' reason if they do not cover the call, else launches them
// (adds to g_kernel_launches).
void run_mlp_backward(const MlpConfig& c, MlpScratch& s, int n_sms, cudaStream_t stream, uint32_t batch, const __half* weights, const __half* input, const __half* hidden,
                      const __half* output, const __half* dL_doutput, bool apply_output_activation, __half* dL_dinput, float* dw_accum);

}  // namespace tcnnb
