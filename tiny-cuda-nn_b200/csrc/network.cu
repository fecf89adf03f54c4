// network.cu -- the stand-alone network tier of the C ABI (include/tcnn_b200.h, tcnnb_network_*), and the runner of the stand-alone
// network kernels that this tier and the general path of model.cu share (network_config.h).
//
// Mirrors, for FullyFusedMLP on its own,
//   src/network.cu:51-141         create_network<T>(json): "otype", "n_neurons", "n_hidden_layers", "activation", "output_activation"
//   fully_fused_mlp.cu:635-672    parameter layout: W_0 [width][in], (n_hidden - 1) x [width][width], W_out [padded_out][width]
//   fully_fused_mlp.cu:868-892    initialize_params: xavier uniform per matrix, one pcg32 stream (gpu_matrix.h:292-306); SIREN for a
//                                 Sine CutlassMLP (cutlass_mlp.cu:362-371)
//   cutlass_mlp.cu:162-209        Sine / SiLU (CutlassMLP): the forward pass keeps pre- and post-activations, num_forward_activations()
//                                 = 2 x n_hidden_layers (tcnnb_network_n_forward_activations)
//   object.h:214-282 / network.h  inference_mixed_precision (fp16 in, fp16 out) and inference (fp32 in, fp32 out)
//   src/cpp_api.cu:160-162        cpp::create_network = the network behind an Identity encoding (encodings/identity.h:46-67)
// Parameters are CALLER-owned fp16 device arrays, as in the module tier. No fallback: an unsupported shape is an error.
#include "../../include/tcnn_b200.h"

#include "encoding_plan.h"
#include "host_common.h"
#include "json_mini.h"
#include "misc_kernels.h"
#include "mlp_fused.h"
#include "network_config.h"

#include <memory>

namespace tcnnb {

// ---- the runner (network_config.h) --------------------------------------------------------------------------------------------
const char* mlp_unsupported(const MlpConfig& c, bool input_gradient) {
	MlpBackwardArgs probe{};
	probe.width = c.width;
	probe.in_width = c.in_width;
	probe.out_width = c.padded_out_width;
	probe.n_hidden_layers = c.n_hidden_layers;
	probe.batch_size = 256;
	probe.dL_dinput = input_gradient ? (__half*)16 : nullptr;
	const char* why_not = nullptr;
	return mlp_backward_supported(probe, &why_not) ? nullptr : why_not;
}

// The pre-activation half of a `hidden` buffer (Sine / SiLU), else null.
template <typename T>
static T* hidden_pre_of(const MlpConfig& c, T* hidden, uint32_t batch) {
	return (hidden && activation_needs_preact(c.activation)) ? hidden + (size_t)c.n_hidden_layers * batch * c.width : nullptr;
}

MlpForwardParams mlp_forward_params(const MlpConfig& c, const __half* weights, uint32_t batch, __half* hidden) {
	MlpForwardParams p{};
	p.width = c.width;
	p.in_width = c.in_width;
	p.out_width = c.padded_out_width;
	p.n_hidden_layers = c.n_hidden_layers;
	p.activation = c.activation;
	p.output_activation = c.output_activation;
	p.weights = weights;
	p.batch_size = batch;
	p.n_output_dims = c.out_width;
	p.hidden_out = hidden;
	p.hidden_pre_out = hidden_pre_of(c, hidden, batch);
	return p;
}

void run_mlp_forward(const MlpForwardParams& p, int n_sms, cudaStream_t stream) {
	const char* why = nullptr;
	if (!mlp_forward_supported(p, &why)) throw std::runtime_error(why);
	TCNNB_CUDA_CHECK(launch_mlp_forward(p, (uint32_t)n_sms, stream));
	++g_kernel_launches;
}

__half* MlpScratch::hidden_rows(const MlpConfig& c, uint32_t batch) {
	grow(hidden, (size_t)n_forward_activations(c) * batch * c.width);
	return hidden.ptr;
}

void run_mlp_backward(const MlpConfig& c, MlpScratch& s, int n_sms, cudaStream_t stream, uint32_t batch, const __half* weights, const __half* input, const __half* hidden,
                      const __half* output, const __half* dL_doutput, bool apply_output_activation, __half* dL_dinput, float* dw_accum) {
	MlpBackwardArgs a{};
	a.width = c.width;
	a.in_width = c.in_width;
	a.out_width = c.padded_out_width;
	a.n_hidden_layers = c.n_hidden_layers;
	a.activation = c.activation;
	a.output_activation = apply_output_activation ? c.output_activation : (uint32_t)ACT_NONE;
	a.weights = weights;
	a.batch_size = batch;
	a.input = input;
	a.hidden = hidden;
	a.hidden_pre = hidden_pre_of(c, hidden, batch);
	a.output = output;
	a.dL_doutput = dL_doutput;
	a.dL_dinput = dL_dinput;
	if (s.grad_hidden_tap) {
		a.grad_hidden = s.grad_hidden_tap;
	} else if (dw_accum) {
		grow(s.grad_hidden, (size_t)c.n_hidden_layers * batch * c.width);
		a.grad_hidden = s.grad_hidden.ptr;
	}
	a.dw_accum = dw_accum;
	if (a.output_activation != ACT_NONE) {
		grow(s.grad_output, (size_t)batch * c.padded_out_width);
		a.grad_output = s.grad_output.ptr;
	}
	const char* why = nullptr;
	if (!mlp_backward_supported(a, &why)) throw std::runtime_error(why);
	uint32_t launches = 0;
	TCNNB_CUDA_CHECK(launch_mlp_backward(a, (uint32_t)n_sms, stream, &launches));
	g_kernel_launches += launches;
}

// ---- the network tier ---------------------------------------------------------------------------------------------------------
struct Network {
	uint32_t n_input_dims = 0;   // cfg.in_width rounds it up to 16 (the Identity encoding pads with ones)
	MlpConfig cfg;
	EncodingPlan identity;       // the Identity encoding in front of the network (module_backward), identity.width == cfg.in_width
	int n_sms = 132;
	long long* dbg_clock = nullptr;  // profiling only (tcnnb_network_debug_clocks)
	MlpScratch scratch;
	// module_backward (fp32 inputs): the Identity-encoded input rows, the recomputed output and dL/d(encoded input); fp32 weight-
	// gradient sums of the backward pass
	DeviceBuffer<__half> enc_input, output, grad_input;
	DeviceBuffer<float> dw_accum;
};

static void build_network(Network& n, uint32_t n_in, uint32_t n_out, const json::Value& net) {
	n.n_sms = require_sm90();
	n.cfg = parse_network(net, next_multiple(n_in, 16u), n_out);
	if (n_in == 0 || n_out == 0) throw std::runtime_error("network: n_input_dims and n_output_dims must be positive.");
	n.n_input_dims = n_in;
	build_encoding_plan(n.identity, n_in, json::parse("{\"otype\": \"Identity\"}"), 16);
	if (const char* why = mlp_unsupported(n.cfg, false)) throw std::runtime_error(why);
}

static void check_args(uint32_t batch, const void* params) {
	check_batch(batch);
	if (!params) throw std::runtime_error("network: params is null.");
	if ((uintptr_t)params % 16 != 0) throw std::runtime_error("network: params must be 16-byte aligned.");
}

static MlpForwardParams make_params(const Network& n, uint32_t batch, const void* params, __half* hidden = nullptr) {
	check_args(batch, params);
	MlpForwardParams p = mlp_forward_params(n.cfg, (const __half*)params, batch, hidden);
	p.n_input_dims = n.n_input_dims;
	p.dbg_clock = n.dbg_clock;
	return p;
}

// Network<T>::backward (fully_fused_mlp.cu:733-866): dL/d(input) (fp16 rows, optional) and dL/d(params) (fp16, OVERWRITTEN, optional)
// from the forward pass's input, activations and output.
static void network_backward(Network& n, cudaStream_t stream, uint32_t batch, const __half* input, const __half* output, const __half* hidden, const __half* dL_doutput,
                             const void* params, __half* dL_dinput, __half* dL_dparams) {
	if (!dL_dinput && !dL_dparams) return;
	check_args(batch, params);
	if (!input || !hidden || !dL_doutput) throw std::runtime_error("network: backward needs the forward pass's input and hidden activations and dL_doutput.");
	if (n.cfg.output_activation != ACT_NONE && !output) throw std::runtime_error("network: backward through an output activation needs the forward pass's output.");
	if (dL_dparams && n.dw_accum.n != n.cfg.n_params) {
		n.dw_accum.resize(n.cfg.n_params);
		n.dw_accum.zero(stream);  // launch_mlp_grad_finalize re-zeroes it after every use
	}
	run_mlp_backward(n.cfg, n.scratch, n.n_sms, stream, batch, (const __half*)params, input, hidden, output, dL_doutput, true, dL_dinput, dL_dparams ? n.dw_accum.ptr : nullptr);
	if (dL_dparams) {
		TCNNB_CUDA_CHECK(launch_mlp_grad_finalize(stream, (uint32_t)n.cfg.n_params, n.dw_accum.ptr, dL_dparams));
		++g_kernel_launches;
	}
}

}  // namespace tcnnb

using namespace tcnnb;

struct tcnnb_network {
	Network impl;
};

extern "C" {

int tcnnb_network_create(uint32_t n_input_dims, uint32_t n_output_dims, const char* network_json, tcnnb_network** out) {
	TCNNB_API_BEGIN
	if (!out) throw std::runtime_error("tcnnb_network_create: out is null");
	*out = nullptr;
	auto n = std::make_unique<tcnnb_network>();
	build_network(n->impl, n_input_dims, n_output_dims, json::parse(network_json ? network_json : "{}"));
	*out = n.release();
	TCNNB_API_END
}

void tcnnb_network_destroy(tcnnb_network* n) { delete n; }
uint64_t tcnnb_network_n_params(const tcnnb_network* n) { return n->impl.cfg.n_params; }
uint32_t tcnnb_network_input_width(const tcnnb_network* n) { return n->impl.cfg.in_width; }
uint32_t tcnnb_network_padded_output_width(const tcnnb_network* n) { return n->impl.cfg.padded_out_width; }
uint32_t tcnnb_network_width(const tcnnb_network* n) { return n->impl.cfg.width; }
uint32_t tcnnb_network_n_hidden_layers(const tcnnb_network* n) { return n->impl.cfg.n_hidden_layers; }
uint32_t tcnnb_network_n_forward_activations(const tcnnb_network* n) { return n_forward_activations(n->impl.cfg); }

int tcnnb_network_debug_clocks(tcnnb_network* n, void* clocks_dev) {
	TCNNB_API_BEGIN
	n->impl.dbg_clock = (long long*)clocks_dev;
	TCNNB_API_END
}

int tcnnb_network_debug_grad_hidden(tcnnb_network* n, void* grad_hidden_dev) {
	TCNNB_API_BEGIN
	if ((uintptr_t)grad_hidden_dev % 16 != 0) throw std::runtime_error("network: grad_hidden must be 16-byte aligned.");
	n->impl.scratch.grad_hidden_tap = (__half*)grad_hidden_dev;
	TCNNB_API_END
}

int tcnnb_network_initialize_params(tcnnb_network* n, uint64_t seed, float* params_full_precision_dev, float scale) {
	TCNNB_API_BEGIN
	if (!params_full_precision_dev) throw std::runtime_error("network: params_full_precision is null.");
	HostPcg32 rng{seed};
	init_mlp_params(n->impl.cfg, rng, params_full_precision_dev, scale);
	TCNNB_API_END
}

int tcnnb_network_inference_mixed_precision(tcnnb_network* n, tcnnb_stream stream, uint32_t n_elements, const void* input_dev, void* output_dev, const void* params_dev) {
	TCNNB_API_BEGIN
	const Network& net = n->impl;
	if (net.n_input_dims != net.cfg.in_width) {
		throw std::runtime_error("network: fp16 inputs need n_input_dims to be a multiple of 16 (got " + std::to_string(net.n_input_dims) + "); use tcnnb_network_inference (Identity encoding pads the input).");
	}
	if (!input_dev || !output_dev) throw std::runtime_error("network: input / output is null.");
	if (((uintptr_t)input_dev | (uintptr_t)output_dev) % 16 != 0) throw std::runtime_error("network: input / output must be 16-byte aligned.");
	MlpForwardParams p = make_params(net, n_elements, params_dev);
	p.input_fp16 = (const __half*)input_dev;
	p.output_fp16 = (__half*)output_dev;
	run_mlp_forward(p, net.n_sms, (cudaStream_t)stream);
	TCNNB_API_END
}

int tcnnb_network_forward(tcnnb_network* n, tcnnb_stream stream, uint32_t n_elements, const void* input_dev, void* output_dev, void* hidden_dev, const void* params_dev) {
	TCNNB_API_BEGIN
	const Network& net = n->impl;
	if (net.n_input_dims != net.cfg.in_width) throw std::runtime_error("network: fp16 inputs need n_input_dims to be a multiple of 16.");
	if (!input_dev) throw std::runtime_error("network: input is null.");
	if (((uintptr_t)input_dev | (uintptr_t)output_dev | (uintptr_t)hidden_dev) % 16 != 0) throw std::runtime_error("network: input / output / hidden must be 16-byte aligned.");
	MlpForwardParams p = make_params(net, n_elements, params_dev, (__half*)hidden_dev);
	p.input_fp16 = (const __half*)input_dev;
	p.output_fp16 = (__half*)output_dev;
	run_mlp_forward(p, net.n_sms, (cudaStream_t)stream);
	TCNNB_API_END
}

int tcnnb_network_backward(tcnnb_network* n, tcnnb_stream stream, uint32_t n_elements, const void* input_dev, const void* output_dev, const void* hidden_dev, const void* dL_doutput_dev,
                           const void* params_dev, void* dL_dinput_dev, void* dL_dparams_dev) {
	TCNNB_API_BEGIN
	Network& net = n->impl;
	if (net.n_input_dims != net.cfg.in_width) throw std::runtime_error("network: fp16 inputs need n_input_dims to be a multiple of 16.");
	if (((uintptr_t)input_dev | (uintptr_t)output_dev | (uintptr_t)hidden_dev | (uintptr_t)dL_doutput_dev | (uintptr_t)dL_dinput_dev | (uintptr_t)dL_dparams_dev) % 16 != 0) {
		throw std::runtime_error("network: all arrays must be 16-byte aligned.");
	}
	network_backward(net, (cudaStream_t)stream, n_elements, (const __half*)input_dev, (const __half*)output_dev, (const __half*)hidden_dev, (const __half*)dL_doutput_dev, params_dev,
	                 (__half*)dL_dinput_dev, (__half*)dL_dparams_dev);
	TCNNB_API_END
}

// cpp::Module::backward of cpp::create_network (src/cpp_api.cu:104-125 with the Identity encoding in front): fp32 inputs; nothing is
// kept from the forward call -- the activations are recomputed here (one more forward pass, no context to hold between the calls).
int tcnnb_network_module_backward(tcnnb_network* n, tcnnb_stream stream_, uint32_t n_elements, float* dL_dinput_dev, const void* dL_doutput_dev, void* dL_dparams_dev, const float* input_dev,
                                  const void* params_dev) {
	TCNNB_API_BEGIN
	Network& net = n->impl;
	cudaStream_t stream = (cudaStream_t)stream_;
	if (!dL_dinput_dev && !dL_dparams_dev) return 0;
	if (!input_dev || !dL_doutput_dev) throw std::runtime_error("network: input / dL_doutput is null.");
	if (((uintptr_t)dL_doutput_dev | (uintptr_t)dL_dparams_dev) % 16 != 0) throw std::runtime_error("network: dL_doutput / dL_dparams must be 16-byte aligned.");
	check_args(n_elements, params_dev);  // before any scratch is sized by n_elements
	MlpForwardParams p = make_params(net, n_elements, params_dev, net.scratch.hidden_rows(net.cfg, n_elements));
	grow(net.enc_input, (size_t)n_elements * net.cfg.in_width);
	grow(net.output, (size_t)n_elements * net.cfg.padded_out_width);
	plan_forward(net.identity, stream, n_elements, input_dev, nullptr, net.enc_input.ptr, net.cfg.in_width, 1.0f);
	p.input_fp16 = net.enc_input.ptr;
	p.output_fp16 = net.output.ptr;
	run_mlp_forward(p, net.n_sms, stream);
	__half* dL_denc = nullptr;
	if (dL_dinput_dev) {
		grow(net.grad_input, (size_t)n_elements * net.cfg.in_width);
		dL_denc = net.grad_input.ptr;
	}
	network_backward(net, stream, n_elements, net.enc_input.ptr, net.output.ptr, p.hidden_out, (const __half*)dL_doutput_dev, params_dev, dL_denc, (__half*)dL_dparams_dev);
	if (dL_dinput_dev) plan_input_gradient(net.identity, stream, n_elements, input_dev, nullptr, dL_denc, net.cfg.in_width, dL_dinput_dev, 1.0f);
	TCNNB_API_END
}

int tcnnb_network_module_inference(tcnnb_network* n, tcnnb_stream stream, uint32_t n_elements, const float* input_dev, void* output_dev, const void* params_dev) {
	TCNNB_API_BEGIN
	const Network& net = n->impl;
	if (!input_dev || !output_dev) throw std::runtime_error("network: input / output is null.");
	if ((uintptr_t)output_dev % 16 != 0) throw std::runtime_error("network: output must be 16-byte aligned.");
	MlpForwardParams p = make_params(net, n_elements, params_dev);
	p.input_fp32 = input_dev;
	p.output_fp16 = (__half*)output_dev;
	run_mlp_forward(p, net.n_sms, (cudaStream_t)stream);
	TCNNB_API_END
}

int tcnnb_network_inference_half_input(tcnnb_network* n, tcnnb_stream stream, uint32_t n_elements, const void* input_dev, float* output_dev, const void* params_dev) {
	TCNNB_API_BEGIN
	const Network& net = n->impl;
	if (net.n_input_dims != net.cfg.in_width) throw std::runtime_error("network: fp16 inputs need n_input_dims to be a multiple of 16.");
	if (!input_dev || !output_dev) throw std::runtime_error("network: input / output is null.");
	if ((uintptr_t)input_dev % 16 != 0) throw std::runtime_error("network: input must be 16-byte aligned.");
	MlpForwardParams p = make_params(net, n_elements, params_dev);
	p.input_fp16 = (const __half*)input_dev;
	p.output_fp32 = output_dev;
	run_mlp_forward(p, net.n_sms, (cudaStream_t)stream);
	TCNNB_API_END
}

int tcnnb_network_inference(tcnnb_network* n, tcnnb_stream stream, uint32_t n_elements, const float* input_dev, float* output_dev, const void* params_dev) {
	TCNNB_API_BEGIN
	const Network& net = n->impl;
	if (!input_dev || !output_dev) throw std::runtime_error("network: input / output is null.");
	MlpForwardParams p = make_params(net, n_elements, params_dev);
	p.input_fp32 = input_dev;
	p.output_fp32 = output_dev;
	run_mlp_forward(p, net.n_sms, (cudaStream_t)stream);
	TCNNB_API_END
}

}  // extern "C"
