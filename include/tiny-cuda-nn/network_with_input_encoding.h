/* tiny-cuda-nn/network_with_input_encoding.h -- NetworkWithInputEncoding<T> (reference: network_with_input_encoding.h:42-160): an encoding
 * followed by a network, fp32 inputs, fp16 outputs. However it is built -- from two JSON blobs or from an Encoding and a Network object
 * -- it is the configuration {"encoding", "network"} of libtcnn_b200, so a Trainer over it runs the same kernels (the fused training
 * kernel wherever the configuration allows) as create_from_config of the same JSON.
 *
 * Two handles sit behind it, each made when first needed: the trainer-tier model (tcnnb_create_from_config) that inference() runs on
 * -- the Trainer's, once one exists (trainer.h:69-87: the trainer owns the parameters and the network reads them), else one of its own
 * with the default seed -- and a module-tier handle (tcnnb_module_*) for the DifferentiableObject calls on caller-owned parameters. */
#pragma once
#include "encoding.h"
#include "network.h"

namespace tcnn {

namespace detail {
struct ModelHandle {
	tcnnb_model* m = nullptr;
	ModelHandle(uint32_t n_in, uint32_t n_out, const json& config, uint32_t seed) { TCNNB_CHECK_THROW(tcnnb_create_from_config(n_in, n_out, config.dump().c_str(), seed, &m)); }
	/* a trainer over a network alone (tcnnb_create_network_trainer): fp16 input rows */
	struct NetworkTrainer {};
	ModelHandle(NetworkTrainer, uint32_t n_in, uint32_t n_out, const json& config, uint32_t seed) {
		TCNNB_CHECK_THROW(tcnnb_create_network_trainer(n_in, n_out, config.dump().c_str(), seed, &m));
	}
	ModelHandle(const ModelHandle&) = delete;
	ModelHandle& operator=(const ModelHandle&) = delete;
	~ModelHandle() { tcnnb_destroy(m); }
};

/* a network's own keys: create_network's JSON without the widths it also carries */
inline json network_keys(json network) {
	network.erase("n_input_dims");
	network.erase("n_output_dims");
	return network;
}
}  // namespace detail

template <typename T>
class NetworkWithInputEncoding : public Network<float, T> {
public:
	/* network_with_input_encoding.h:55 */
	NetworkWithInputEncoding(uint32_t n_dims_to_encode, uint32_t n_output_dims, const json& encoding, const json& network)
	: m_n_in{n_dims_to_encode}, m_n_out{n_output_dims}, m_encoding(encoding), m_network(network) {}
	/* network_with_input_encoding.h:44: the two objects' configurations. The network reads the encoding's output padded to 16, so its
	 * input width must be that padded width. The objects keep their identity: set_params() hands each its part of the parameters
	 * ([network | encoding], network_with_input_encoding.h:115-130), as the reference does. */
	NetworkWithInputEncoding(std::shared_ptr<Encoding<T>> encoding, std::shared_ptr<Network<T>> network)
	: m_n_in{encoding->input_width()}, m_n_out{network->output_width()}, m_encoding(encoding->hyperparams()), m_network(detail::network_keys(network->hyperparams())),
	  m_encoding_obj{encoding}, m_network_obj{network} {
		if (network->input_width() != next_multiple(encoding->padded_output_width(), 16u)) {
			throw std::runtime_error{"NetworkWithInputEncoding: the network takes " + std::to_string(network->input_width()) + " inputs, the encoding gives " +
			                         std::to_string(encoding->padded_output_width()) + " features (padded to " + std::to_string(next_multiple(encoding->padded_output_width(), 16u)) + ")"};
		}
	}
	/* network_with_input_encoding.h:46-53 */
	NetworkWithInputEncoding(std::shared_ptr<Encoding<T>> encoding, uint32_t n_output_dims, const json& network)
	: m_n_in{encoding->input_width()}, m_n_out{n_output_dims}, m_encoding(encoding->hyperparams()), m_network(network), m_encoding_obj{encoding} {}

	void set_params_impl(T* params, T* inference_params, T* gradients) override {
		if (!m_encoding_obj) return;  /* built from JSON: no component objects */
		const size_t n_net = m_network_obj ? m_network_obj->n_params() : n_params() - m_encoding_obj->n_params();
		if (m_network_obj) {
			if (n_net + m_encoding_obj->n_params() != n_params()) throw std::runtime_error{"NetworkWithInputEncoding: the objects' parameter counts do not add up"};
			m_network_obj->set_params(params, inference_params, gradients);
		}
		auto offset = [n_net](T* p) { return p ? p + n_net : nullptr; };
		m_encoding_obj->set_params(offset(params), offset(inference_params), offset(gradients));
	}
	~NetworkWithInputEncoding() override { if (m_module) tcnnb_destroy(m_module); }

	/* object.h:214-282 on the trainer's inference parameters: input n_in x B (column-major = sample-contiguous), output n_out x B fp32 */
	void inference(cudaStream_t stream, const GPUMatrixDynamic<float>& input, GPUMatrixDynamic<float>& output) {
		if (input.m() != m_n_in || output.m() != m_n_out || input.n() != output.n()) throw std::runtime_error{"inference: matrix shapes do not match the network"};
		if (input.layout() != CM || output.layout() != CM) throw std::runtime_error{"inference: column-major (sample-contiguous) matrices only"};
		TCNNB_CHECK_THROW(tcnnb_inference(model(), (tcnnb_stream)stream, input.n(), input.data(), output.data()));
	}
	void inference(const GPUMatrixDynamic<float>& input, GPUMatrixDynamic<float>& output) { inference(nullptr, input, output); }

	/* DifferentiableObject, on the parameters set_params() handed over (the Trainer's, once one exists) */
	void inference_impl(cudaStream_t stream, const GPUMatrixDynamic<float>& input, GPUMatrixDynamic<float>& output, bool use_inference_params) override {
		if (!m_model || !use_inference_params || this->inference_params() != tcnnb_params_inference(m_model->m)) {
			throw std::runtime_error{"NetworkWithInputEncoding::inference with fp32 outputs runs on its trainer's inference parameters; inference_mixed_precision takes any"};
		}
		inference(stream, input, output);
	}
	void inference_mixed_precision_impl(cudaStream_t stream, const GPUMatrixDynamic<float>& input, GPUMatrixDynamic<T>& output, bool use_inference_params = true) override {
		const float* in = detail::cm_data(stream, input, m_in_scratch);
		T* out = detail::cm_target(output, m_out_scratch);
		TCNNB_CHECK_THROW(tcnnb_module_inference(module(), (tcnnb_stream)stream, input.n(), in, out, weights(use_inference_params)));
		detail::finish_cm(stream, output, m_out_scratch);
	}
	std::unique_ptr<Context> forward_impl(cudaStream_t stream, const GPUMatrixDynamic<float>& input, GPUMatrixDynamic<T>* output = nullptr, bool use_inference_params = false,
	                                      bool prepare_input_gradients = false) override {
		if (output) {
			const float* in = detail::cm_data(stream, input, m_in_scratch);
			T* out = detail::cm_target(*output, m_out_scratch);
			TCNNB_CHECK_THROW(tcnnb_module_forward(module(), (tcnnb_stream)stream, input.n(), in, out, weights(use_inference_params), prepare_input_gradients ? 1 : 0));
			detail::finish_cm(stream, *output, m_out_scratch);
		}
		return std::make_unique<Context>();  /* backward recomputes the forward pass */
	}
	void backward_impl(cudaStream_t stream, const Context&, const GPUMatrixDynamic<float>& input, const GPUMatrixDynamic<T>& output, const GPUMatrixDynamic<T>& dL_doutput,
	                   GPUMatrixDynamic<float>* dL_dinput = nullptr, bool use_inference_params = false, GradientMode param_gradients_mode = GradientMode::Overwrite) override {
		if (param_gradients_mode == GradientMode::Accumulate) throw std::runtime_error{"NetworkWithInputEncoding::backward: GradientMode::Accumulate is not built for the object; the Trainer accumulates"};
		const float* in = detail::cm_data(stream, input, m_in_scratch);
		const T* dy = detail::cm_data(stream, dL_doutput, m_out_scratch);
		float* dx = dL_dinput ? detail::cm_target(*dL_dinput, m_dx_scratch) : nullptr;
		T* dparams = param_gradients_mode == GradientMode::Overwrite ? this->gradients() : nullptr;
		TCNNB_CHECK_THROW(tcnnb_module_backward(module(), (tcnnb_stream)stream, input.n(), dx, dy, dparams, in, nullptr, weights(use_inference_params)));
		if (dL_dinput) detail::finish_cm(stream, *dL_dinput, m_dx_scratch);
	}
	/* network_with_input_encoding.h:124-130 from pcg32{seed}, seeded from the caller's generator (see NetworkObject::initialize_params) */
	void initialize_params(pcg32& rnd, float* params_full_precision, float scale = 1) override {
		TCNNB_CHECK_THROW(tcnnb_module_initialize_params(module(), rnd.next_uint(), params_full_precision, scale));
	}

	size_t n_params() const override { return tcnnb_n_params(const_cast<NetworkWithInputEncoding*>(this)->model()); }
	uint32_t input_width() const override { return m_n_in; }
	uint32_t output_width() const override { return m_n_out; }
	uint32_t padded_output_width() const override { return tcnnb_padded_output_width(const_cast<NetworkWithInputEncoding*>(this)->model()); }
	uint32_t width(uint32_t layer) const override { return layer == 0 ? tcnnb_encoded_width(const_cast<NetworkWithInputEncoding*>(this)->model()) : m_network.value("n_neurons", 128u); }
	uint32_t num_forward_activations() const override { return m_network.value("n_hidden_layers", 5u); }
	json hyperparams() const override { return json::parse(tcnnb_hyperparams(const_cast<NetworkWithInputEncoding*>(this)->model())); }
	std::string name() const override { return "NetworkWithInputEncoding"; }

	const json& encoding_opts() const { return m_encoding; }
	const json& network_opts() const { return m_network; }
	/* used by Trainer: share the trainer's model */
	void attach(std::shared_ptr<detail::ModelHandle> h) { m_model = std::move(h); }
	tcnnb_model* model() {
		if (!m_model) m_model = std::make_shared<detail::ModelHandle>(m_n_in, m_n_out, json{{"encoding", m_encoding}, {"network", m_network}}, 1337u);
		return m_model->m;
	}

private:
	const T* weights(bool use_inference_params) const { return use_inference_params ? this->inference_params() : this->params(); }
	tcnnb_model* module() {
		if (!m_module) TCNNB_CHECK_THROW(tcnnb_module_create(m_n_in, m_n_out, m_encoding.dump().c_str(), m_network.dump().c_str(), &m_module));
		return m_module;
	}

	uint32_t m_n_in, m_n_out;
	json m_encoding, m_network;
	std::shared_ptr<detail::ModelHandle> m_model;
	std::shared_ptr<Encoding<T>> m_encoding_obj;  /* the objects it was composed from, if any */
	std::shared_ptr<Network<T>> m_network_obj;
	tcnnb_model* m_module = nullptr;
	GPUMemory<float> m_in_scratch, m_dx_scratch;
	GPUMemory<T> m_out_scratch;
};

}  // namespace tcnn

#include "config.h"
