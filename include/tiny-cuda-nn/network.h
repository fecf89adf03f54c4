/* tiny-cuda-nn/network.h -- Network<T, PARAMS_T> and create_network<T>(json) (reference: network.h:40-60, src/network.cu:51-141), over the
 * network tier of libtcnn_b200 (tcnnb_network_*): FullyFusedMLP and CutlassMLP / MLP on the sm_90a MLP kernels. The JSON carries
 * "n_input_dims" and "n_output_dims" besides the network's own keys. Inputs are fp16 rows of n_input_dims features, a multiple of 16. */
#pragma once
#include <vector>

#include "object.h"

namespace tcnn {

template <typename T, typename PARAMS_T = T>
class Network : public DifferentiableObject<T, PARAMS_T, PARAMS_T> {
public:
	virtual ~Network() {}
	virtual uint32_t width(uint32_t layer) const = 0;
	virtual uint32_t num_forward_activations() const = 0;
};

namespace detail {

/* create_network<__half>: the object over one tcnnb_network handle. Parameters are the caller's (or the Trainer's): W_0, the hidden
 * matrices and W_out, row-major, as in fully_fused_mlp.cu:635-672. */
class NetworkObject : public Network<__half> {
public:
	explicit NetworkObject(const json& config) : m_config(config) {
		if (!config.contains("n_input_dims") || !config.contains("n_output_dims")) throw std::runtime_error{"create_network: the JSON needs n_input_dims and n_output_dims"};
		m_n_in = config["n_input_dims"].get<uint32_t>();
		m_n_out = config["n_output_dims"].get<uint32_t>();
		json network = config;
		network.erase("n_input_dims");
		network.erase("n_output_dims");
		TCNNB_CHECK_THROW(tcnnb_network_create(m_n_in, m_n_out, network.dump().c_str(), &m_h));
	}
	~NetworkObject() override { tcnnb_network_destroy(m_h); }
	NetworkObject(const NetworkObject&) = delete;
	NetworkObject& operator=(const NetworkObject&) = delete;

	void inference_mixed_precision_impl(cudaStream_t stream, const GPUMatrixDynamic<__half>& input, GPUMatrixDynamic<__half>& output, bool use_inference_params = true) override {
		const __half* in = cm_data(stream, input, m_in_scratch);
		__half* out = cm_target(output, m_out_scratch);
		TCNNB_CHECK_THROW(tcnnb_network_inference_mixed_precision(m_h, (tcnnb_stream)stream, input.n(), in, out, weights(use_inference_params)));
		finish_cm(stream, output, m_out_scratch);
	}
	void inference_impl(cudaStream_t stream, const GPUMatrixDynamic<__half>& input, GPUMatrixDynamic<float>& output, bool use_inference_params) override {
		const __half* in = cm_data(stream, input, m_in_scratch);
		float* out = cm_target(output, m_out_scratch_f32);
		TCNNB_CHECK_THROW(tcnnb_network_inference_half_input(m_h, (tcnnb_stream)stream, input.n(), in, out, weights(use_inference_params)));
		finish_cm(stream, output, m_out_scratch_f32);
	}

	/* the post- (and for Sine / SiLU pre-) activations of the hidden layers, what tcnnb_network_backward reads */
	struct ForwardContext : public Context {
		GPUMemory<__half> hidden;
	};
	std::unique_ptr<Context> forward_impl(cudaStream_t stream, const GPUMatrixDynamic<__half>& input, GPUMatrixDynamic<__half>* output = nullptr, bool use_inference_params = false,
	                                      bool = false) override {
		auto ctx = std::make_unique<ForwardContext>();
		ctx->hidden.resize((size_t)num_forward_activations() * input.n() * tcnnb_network_width(m_h));
		const __half* in = cm_data(stream, input, m_in_scratch);
		__half* out = output ? cm_target(*output, m_out_scratch) : nullptr;
		TCNNB_CHECK_THROW(tcnnb_network_forward(m_h, (tcnnb_stream)stream, input.n(), in, out, ctx->hidden.data(), weights(use_inference_params)));
		if (output) finish_cm(stream, *output, m_out_scratch);
		return ctx;
	}

	void backward_impl(cudaStream_t stream, const Context& ctx, const GPUMatrixDynamic<__half>& input, const GPUMatrixDynamic<__half>& output, const GPUMatrixDynamic<__half>& dL_doutput,
	                   GPUMatrixDynamic<__half>* dL_dinput = nullptr, bool use_inference_params = false, GradientMode param_gradients_mode = GradientMode::Overwrite) override {
		const auto* fwd = dynamic_cast<const ForwardContext*>(&ctx);
		if (!fwd) throw std::runtime_error{"Network::backward: the context was not made by this network's forward()"};
		if (param_gradients_mode == GradientMode::Accumulate) throw std::runtime_error{"Network::backward: GradientMode::Accumulate is not built for a network object; the Trainer accumulates"};
		const __half* in = cm_data(stream, input, m_in_scratch);
		const __half* out = cm_data(stream, output, m_out_scratch);
		const __half* dy = cm_data(stream, dL_doutput, m_dy_scratch);
		__half* dx = dL_dinput ? cm_target(*dL_dinput, m_dx_scratch) : nullptr;
		__half* dparams = param_gradients_mode == GradientMode::Overwrite ? this->gradients() : nullptr;
		TCNNB_CHECK_THROW(tcnnb_network_backward(m_h, (tcnnb_stream)stream, input.n(), in, out, fwd->hidden.data(), dy, weights(use_inference_params), dx, dparams));
		if (dL_dinput) finish_cm(stream, *dL_dinput, m_dx_scratch);
	}

	/* fully_fused_mlp.cu:868-892 from pcg32{seed}. The reference draws from the caller's generator; this seeds it from the generator's
	 * next number, so a Trainer's own initialisation (the reference's stream, bit for bit) goes through the trainer handle instead. */
	void initialize_params(pcg32& rnd, float* params_full_precision, float scale = 1) override {
		TCNNB_CHECK_THROW(tcnnb_network_initialize_params(m_h, rnd.next_uint(), params_full_precision, scale));
	}
	size_t n_params() const override { return tcnnb_network_n_params(m_h); }

	uint32_t input_width() const override { return m_n_in; }
	uint32_t padded_output_width() const override { return tcnnb_network_padded_output_width(m_h); }
	uint32_t output_width() const override { return m_n_out; }
	uint32_t required_input_alignment() const override { return 16; }
	uint32_t width(uint32_t layer) const override { return layer == 0 ? tcnnb_network_input_width(m_h) : tcnnb_network_width(m_h); }
	uint32_t num_forward_activations() const override { return tcnnb_network_n_forward_activations(m_h); }

	json hyperparams() const override { return m_config; }
	std::string name() const override { return m_config.value("otype", std::string{"FullyFusedMLP"}); }

private:
	const __half* weights(bool use_inference_params) const { return use_inference_params ? this->inference_params() : this->params(); }

	tcnnb_network* m_h = nullptr;
	uint32_t m_n_in = 0, m_n_out = 0;
	json m_config;
	GPUMemory<__half> m_in_scratch, m_out_scratch, m_dy_scratch, m_dx_scratch;
	GPUMemory<float> m_out_scratch_f32;
};

}  // namespace detail

/* src/network.cu:51-141 */
template <typename T>
Network<T, T>* create_network(const json& network) {
	static_assert(sizeof(T) == 2, "tcnn_b200 mirrors the half-precision build of the reference: create_network<T> is built for T = __half");
	return new detail::NetworkObject{network};
}

}  // namespace tcnn

#include "config.h"
