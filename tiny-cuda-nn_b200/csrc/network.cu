// network.cu -- the stand-alone network tier of the C ABI (include/tcnn_b200.h, tcnnb_network_*).
//
// Mirrors, for FullyFusedMLP on its own,
//   src/network.cu:51-141         create_network<T>(json): "otype", "n_neurons", "n_hidden_layers", "activation", "output_activation"
//   fully_fused_mlp.cu:635-672    parameter layout: W_0 [width][in], (n_hidden - 1) x [width][width], W_out [padded_out][width]
//   fully_fused_mlp.cu:868-892    initialize_params: xavier uniform per matrix, one pcg32 stream (gpu_matrix.h:292-306)
//   object.h:214-282 / network.h  inference_mixed_precision (fp16 in, fp16 out) and inference (fp32 in, fp32 out)
//   src/cpp_api.cu:160-162        cpp::create_network = the network behind an Identity encoding (encodings/identity.h:46-67)
// Parameters are CALLER-owned fp16 device arrays, as in the module tier. No fallback: an unsupported shape is an error.
#include "../../include/tcnn_b200.h"

#include "host_common.h"
#include "json_mini.h"
#include "misc_kernels.h"
#include "mlp_fused.h"

#include <cmath>
#include <memory>
#include <vector>

namespace tcnnb {

struct Network {
	uint32_t n_input_dims = 0, n_output_dims = 0;
	uint32_t in_width = 0;       // n_input_dims rounded up to 16 (Identity encoding pads with ones)
	uint32_t width = 128, n_hidden_layers = 5;
	uint32_t padded_out_width = 0;
	uint32_t activation = ACT_RELU, output_activation = ACT_NONE;
	uint64_t n_params = 0;
	int n_sms = 132;
	long long* dbg_clock = nullptr;  // profiling only (tcnnb_network_debug_clocks)
	std::string otype, hyperparams_json;
	// scratch of the backward pass (grown on demand, reused): g_l rows, dL/d(output) through the output activation, fp32 weight-gradient
	// sums, and -- module tier, fp32 inputs -- the Identity-encoded input rows, the recomputed activations and dL/d(encoded input)
	DeviceBuffer<__half> grad_hidden, grad_output, enc_input, hidden, output, grad_input;
	DeviceBuffer<float> dw_accum;
};

static void build_network(Network& n, uint32_t n_in, uint32_t n_out, const json::Value& net) {
	int device = 0;
	TCNNB_CUDA_CHECK(cudaGetDevice(&device));
	cudaDeviceProp prop;
	TCNNB_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
	if (prop.major != 9) throw std::runtime_error("tcnn_b200 requires an sm_90-class GPU (H100); found compute capability " + std::to_string(prop.major) + "." + std::to_string(prop.minor));
	n.n_sms = prop.multiProcessorCount;
	n.otype = net.value("otype", "MLP");  // src/network.cu:52-54
	const bool fully_fused = ieq(n.otype, "FullyFusedMLP") || ieq(n.otype, "MegakernelMLP");
	const bool cutlass = ieq(n.otype, "MLP") || ieq(n.otype, "CutlassMLP");
	if (!fully_fused && !cutlass) throw std::runtime_error("Invalid network type: " + n.otype);
	n.width = (uint32_t)net.value("n_neurons", 128.0);
	n.n_hidden_layers = (uint32_t)net.value("n_hidden_layers", 5.0);
	n.activation = parse_activation(net.value("activation", "ReLU"));
	n.output_activation = parse_activation(net.value("output_activation", "None"));
	// Both otypes run on the same wgmma kernel (there is no separate non-fused path in this library), so both take the fused
	// kernel's widths; the reference's CutlassMLP accepts any multiple of 8.
	if (!(n.width == 16 || n.width == 32 || n.width == 64 || n.width == 128)) {
		throw std::runtime_error("FullyFusedMLP only supports 16, 32, 64, and 128 neurons, but got " + std::to_string(n.width) + ". Use CutlassMLP instead if this is a requirement.");
	}
	if (n.n_hidden_layers < 1) throw std::runtime_error("FullyFusedMLP requires at least 1 hidden layer (3 layers in total).");
	for (uint32_t act : {n.activation, n.output_activation}) {
		if (act == ACT_SINE || act == ACT_SILU) throw std::runtime_error("Unsupported activation.");  // fully_fused_mlp.cu:689-699
	}
	if (n_in == 0 || n_out == 0) throw std::runtime_error("network: n_input_dims and n_output_dims must be positive.");
	n.n_input_dims = n_in;
	n.n_output_dims = n_out;
	n.in_width = next_multiple(n_in, 16u);
	n.padded_out_width = next_multiple(n_out, 16u);
	n.n_params = (uint64_t)n.width * n.in_width + (uint64_t)(n.n_hidden_layers - 1) * n.width * n.width + (uint64_t)n.padded_out_width * n.width;
	MlpForwardParams probe{};
	probe.width = n.width;
	probe.in_width = n.in_width;
	probe.out_width = n.padded_out_width;
	probe.n_hidden_layers = n.n_hidden_layers;
	probe.batch_size = 256;
	probe.input_fp16 = (const __half*)16;
	const char* why = nullptr;
	if (!mlp_forward_supported(probe, &why)) throw std::runtime_error(why);
}

static MlpForwardParams make_params(const Network& n, uint32_t batch, const void* params) {
	if (batch == 0 || batch % BATCH_GRANULARITY != 0) {
		throw std::runtime_error("batch size " + std::to_string(batch) + " must be a non-zero multiple of " + std::to_string(BATCH_GRANULARITY));
	}
	if (!params) throw std::runtime_error("network: params is null.");
	if ((uintptr_t)params % 16 != 0) throw std::runtime_error("network: params must be 16-byte aligned.");
	MlpForwardParams p{};
	p.width = n.width;
	p.in_width = n.in_width;
	p.out_width = n.padded_out_width;
	p.n_hidden_layers = n.n_hidden_layers;
	p.activation = n.activation;
	p.output_activation = n.output_activation;
	p.weights = (const __half*)params;
	p.batch_size = batch;
	p.n_input_dims = n.n_input_dims;
	p.n_output_dims = n.n_output_dims;
	p.dbg_clock = n.dbg_clock;
	return p;
}

static void launch(const Network& n, const MlpForwardParams& p, cudaStream_t stream) {
	const char* why = nullptr;
	if (!mlp_forward_supported(p, &why)) throw std::runtime_error(why);
	TCNNB_CUDA_CHECK(launch_mlp_forward(p, (uint32_t)n.n_sms, stream));
	++g_kernel_launches;
}

template <typename T>
static void grow(DeviceBuffer<T>& b, size_t n) {
	if (b.n < n) b.resize(n);
}

// Network<T>::backward (fully_fused_mlp.cu:733-866): dL/d(input) (fp16 rows, optional) and dL/d(params) (fp16, OVERWRITTEN, optional)
// from the forward pass's input, activations and output.
static void network_backward(Network& n, cudaStream_t stream, uint32_t batch, const __half* input, const __half* output, const __half* hidden, const __half* dL_doutput,
                             const void* params, __half* dL_dinput, __half* dL_dparams) {
	if (!dL_dinput && !dL_dparams) return;
	MlpForwardParams probe = make_params(n, batch, params);  // validates batch / params
	(void)probe;
	if (!input || !hidden || !dL_doutput) throw std::runtime_error("network: backward needs the forward pass's input and hidden activations and dL_doutput.");
	if (n.output_activation != ACT_NONE && !output) throw std::runtime_error("network: backward through an output activation needs the forward pass's output.");
	MlpBackwardArgs a{};
	a.width = n.width;
	a.in_width = n.in_width;
	a.out_width = n.padded_out_width;
	a.n_hidden_layers = n.n_hidden_layers;
	a.activation = n.activation;
	a.output_activation = n.output_activation;
	a.weights = (const __half*)params;
	a.batch_size = batch;
	a.input = input;
	a.hidden = hidden;
	a.output = output;
	a.dL_doutput = dL_doutput;
	a.dL_dinput = dL_dinput;
	if (dL_dparams) {
		grow(n.grad_hidden, (size_t)n.n_hidden_layers * batch * n.width);
		a.grad_hidden = n.grad_hidden.ptr;
		if (n.dw_accum.n != n.n_params) {
			n.dw_accum.resize(n.n_params);
			n.dw_accum.zero(stream);  // launch_mlp_grad_finalize re-zeroes it after every use
		}
		a.dw_accum = n.dw_accum.ptr;
	}
	if (n.output_activation != ACT_NONE) {
		grow(n.grad_output, (size_t)batch * n.padded_out_width);
		a.grad_output = n.grad_output.ptr;
	}
	const char* why = nullptr;
	if (!mlp_backward_supported(a, &why)) throw std::runtime_error(why);
	uint32_t launches = 0;
	TCNNB_CUDA_CHECK(launch_mlp_backward(a, (uint32_t)n.n_sms, stream, &launches));
	if (dL_dparams) {
		TCNNB_CUDA_CHECK(launch_mlp_grad_finalize(stream, (uint32_t)n.n_params, n.dw_accum.ptr, dL_dparams));
		++launches;
	}
	g_kernel_launches += launches;
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
uint64_t tcnnb_network_n_params(const tcnnb_network* n) { return n->impl.n_params; }
uint32_t tcnnb_network_input_width(const tcnnb_network* n) { return n->impl.in_width; }
uint32_t tcnnb_network_padded_output_width(const tcnnb_network* n) { return n->impl.padded_out_width; }
uint32_t tcnnb_network_width(const tcnnb_network* n) { return n->impl.width; }
uint32_t tcnnb_network_n_hidden_layers(const tcnnb_network* n) { return n->impl.n_hidden_layers; }

int tcnnb_network_debug_clocks(tcnnb_network* n, void* clocks_dev) {
	TCNNB_API_BEGIN
	n->impl.dbg_clock = (long long*)clocks_dev;
	TCNNB_API_END
}

int tcnnb_network_initialize_params(tcnnb_network* n, uint64_t seed, float* params_full_precision_dev, float scale) {
	TCNNB_API_BEGIN
	if (!params_full_precision_dev) throw std::runtime_error("network: params_full_precision is null.");
	const Network& net = n->impl;
	HostPcg32 rng{seed};
	std::vector<float> w(net.n_params);
	std::vector<std::pair<uint32_t, uint32_t>> mats;  // (rows = fan_out, cols = fan_in), fully_fused_mlp.cu:868-892
	mats.emplace_back(net.width, net.in_width);
	for (uint32_t i = 0; i + 1 < net.n_hidden_layers; ++i) mats.emplace_back(net.width, net.width);
	mats.emplace_back(net.padded_out_width, net.width);
	size_t pos = 0;
	for (auto& rc : mats) {
		const float bound = scale * std::sqrt(6.0f / (float)(rc.second + rc.first));
		for (size_t i = 0; i < (size_t)rc.first * rc.second; ++i) w[pos++] = rng.next_float() * 2.0f * bound - bound;
	}
	TCNNB_CUDA_CHECK(cudaMemcpy(params_full_precision_dev, w.data(), sizeof(float) * w.size(), cudaMemcpyHostToDevice));
	TCNNB_API_END
}

int tcnnb_network_inference_mixed_precision(tcnnb_network* n, tcnnb_stream stream, uint32_t n_elements, const void* input_dev, void* output_dev, const void* params_dev) {
	TCNNB_API_BEGIN
	const Network& net = n->impl;
	if (net.n_input_dims != net.in_width) {
		throw std::runtime_error("network: fp16 inputs need n_input_dims to be a multiple of 16 (got " + std::to_string(net.n_input_dims) + "); use tcnnb_network_inference (Identity encoding pads the input).");
	}
	if (!input_dev || !output_dev) throw std::runtime_error("network: input / output is null.");
	if (((uintptr_t)input_dev | (uintptr_t)output_dev) % 16 != 0) throw std::runtime_error("network: input / output must be 16-byte aligned.");
	MlpForwardParams p = make_params(net, n_elements, params_dev);
	p.input_fp16 = (const __half*)input_dev;
	p.output_fp16 = (__half*)output_dev;
	launch(net, p, (cudaStream_t)stream);
	TCNNB_API_END
}

int tcnnb_network_forward(tcnnb_network* n, tcnnb_stream stream, uint32_t n_elements, const void* input_dev, void* output_dev, void* hidden_dev, const void* params_dev) {
	TCNNB_API_BEGIN
	const Network& net = n->impl;
	if (net.n_input_dims != net.in_width) throw std::runtime_error("network: fp16 inputs need n_input_dims to be a multiple of 16.");
	if (!input_dev) throw std::runtime_error("network: input is null.");
	if (((uintptr_t)input_dev | (uintptr_t)output_dev | (uintptr_t)hidden_dev) % 16 != 0) throw std::runtime_error("network: input / output / hidden must be 16-byte aligned.");
	MlpForwardParams p = make_params(net, n_elements, params_dev);
	p.input_fp16 = (const __half*)input_dev;
	p.output_fp16 = (__half*)output_dev;
	p.hidden_out = (__half*)hidden_dev;
	launch(net, p, (cudaStream_t)stream);
	TCNNB_API_END
}

int tcnnb_network_backward(tcnnb_network* n, tcnnb_stream stream, uint32_t n_elements, const void* input_dev, const void* output_dev, const void* hidden_dev, const void* dL_doutput_dev,
                           const void* params_dev, void* dL_dinput_dev, void* dL_dparams_dev) {
	TCNNB_API_BEGIN
	Network& net = n->impl;
	if (net.n_input_dims != net.in_width) throw std::runtime_error("network: fp16 inputs need n_input_dims to be a multiple of 16.");
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
	MlpForwardParams p = make_params(net, n_elements, params_dev);
	grow(net.enc_input, (size_t)n_elements * net.in_width);
	grow(net.hidden, (size_t)net.n_hidden_layers * n_elements * net.width);
	grow(net.output, (size_t)n_elements * net.padded_out_width);
	TCNNB_CUDA_CHECK(launch_identity_encode(stream, n_elements, net.n_input_dims, net.in_width, 1.0f, 0.0f, input_dev, net.enc_input.ptr));
	++g_kernel_launches;
	p.input_fp16 = net.enc_input.ptr;
	p.output_fp16 = net.output.ptr;
	p.hidden_out = net.hidden.ptr;
	launch(net, p, stream);
	__half* dL_denc = nullptr;
	if (dL_dinput_dev) {
		grow(net.grad_input, (size_t)n_elements * net.in_width);
		dL_denc = net.grad_input.ptr;
	}
	network_backward(net, stream, n_elements, net.enc_input.ptr, net.output.ptr, net.hidden.ptr, (const __half*)dL_doutput_dev, params_dev, dL_denc, (__half*)dL_dparams_dev);
	if (dL_dinput_dev) {
		TCNNB_CUDA_CHECK(launch_identity_backward(stream, n_elements, net.n_input_dims, net.in_width, 1.0f, dL_denc, dL_dinput_dev));
		++g_kernel_launches;
	}
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
	launch(net, p, (cudaStream_t)stream);
	TCNNB_API_END
}

int tcnnb_network_inference(tcnnb_network* n, tcnnb_stream stream, uint32_t n_elements, const float* input_dev, float* output_dev, const void* params_dev) {
	TCNNB_API_BEGIN
	const Network& net = n->impl;
	if (!input_dev || !output_dev) throw std::runtime_error("network: input / output is null.");
	MlpForwardParams p = make_params(net, n_elements, params_dev);
	p.input_fp32 = input_dev;
	p.output_fp32 = output_dev;
	launch(net, p, (cudaStream_t)stream);
	TCNNB_API_END
}

}  // extern "C"
