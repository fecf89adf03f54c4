/* tiny-cuda-nn/config.h -- create_from_config, TrainableModel, Trainer, NetworkWithInputEncoding, Loss, Optimizer with the
 * signatures applications use (reference: config.h:46-63, trainer.h:51-161,254-482, network_with_input_encoding.h:49-160,
 * loss.h:60-75, optimizer.h:46-90), implemented over the C ABI of libtcnn_b200.
 *
 * The JSON type is nlohmann::json, as in the reference (`tcnn::json`); it comes from the application's include path
 * (<json/json.hpp> in a tiny-cuda-nn checkout, <nlohmann/json.hpp> elsewhere).
 *
 * Object model. The reference builds loss, optimizer and network separately and ties them together in the Trainer; the C ABI
 * has ONE handle per trainable model. So Loss / Optimizer / NetworkWithInputEncoding here are light objects that carry their JSON
 * options, and the Trainer constructor creates the tcnnb_model from the combined configuration and attaches it to the network, so
 * that network->inference() afterwards runs on the trainer's parameters -- the reference's behaviour (trainer.h:69-87: the
 * trainer owns the parameter buffer and hands pointers into it to the model). A network that is used for inference before any
 * trainer exists gets a model of its own with the default seed. */
#pragma once
#if __has_include(<json/json.hpp>)
#include <json/json.hpp>
#else
#include <nlohmann/json.hpp>
#endif

#include <cctype>
#include <memory>
#include <string>
#include <vector>

#include "common.h"
#include "gpu_matrix.h"
#include "gpu_memory.h"
#include "object.h"
#include "random.h"

namespace tcnn {

using json = nlohmann::json;

namespace detail {
struct ModelHandle {
	tcnnb_model* m = nullptr;
	ModelHandle(uint32_t n_in, uint32_t n_out, const json& config, uint32_t seed) { TCNNB_CHECK_THROW(tcnnb_create_from_config(n_in, n_out, config.dump().c_str(), seed, &m)); }
	ModelHandle(const ModelHandle&) = delete;
	ModelHandle& operator=(const ModelHandle&) = delete;
	~ModelHandle() { tcnnb_destroy(m); }
};
}  // namespace detail

template <typename T>
class Loss {
public:
	explicit Loss(const json& opts) : m_opts(opts) {}  /* parentheses: brace-initialising a json from a json makes an array */
	const json& hyperparams() const { return m_opts; }
private:
	json m_opts;
};

template <typename T>
class Optimizer {
public:
	explicit Optimizer(const json& opts) : m_opts(opts) {}
	const json& hyperparams() const { return m_opts; }
private:
	json m_opts;
};

template <typename T>
Loss<T>* create_loss(const json& opts) { return new Loss<T>{opts}; }           /* src/loss.cu:82-90 */
template <typename T>
Optimizer<T>* create_optimizer(const json& opts) { return new Optimizer<T>{opts}; } /* src/optimizer.cu:50-80 */

template <typename T>
class NetworkWithInputEncoding {
public:
	/* network_with_input_encoding.h:49-55 */
	NetworkWithInputEncoding(uint32_t n_dims_to_encode, uint32_t n_output_dims, const json& encoding, const json& network)
	: m_n_in{n_dims_to_encode}, m_n_out{n_output_dims}, m_encoding(encoding), m_network(network) {}

	/* object.h:214-282: input n_in x B (column-major = sample-contiguous), output n_out x B fp32 */
	void inference(cudaStream_t stream, const GPUMatrixDynamic<float>& input, GPUMatrixDynamic<float>& output) {
		if (input.m() != m_n_in || output.m() != m_n_out || input.n() != output.n()) throw std::runtime_error{"inference: matrix shapes do not match the network"};
		if (input.layout() != CM || output.layout() != CM) throw std::runtime_error{"inference: column-major (sample-contiguous) matrices only"};
		TCNNB_CHECK_THROW(tcnnb_inference(model(), (tcnnb_stream)stream, input.n(), input.data(), output.data()));
	}
	void inference(const GPUMatrixDynamic<float>& input, GPUMatrixDynamic<float>& output) { inference(nullptr, input, output); }

	size_t n_params() const { return tcnnb_n_params(const_cast<NetworkWithInputEncoding*>(this)->model()); }
	uint32_t input_width() const { return m_n_in; }
	uint32_t output_width() const { return m_n_out; }
	uint32_t padded_output_width() const { return tcnnb_padded_output_width(const_cast<NetworkWithInputEncoding*>(this)->model()); }
	json hyperparams() const { return json::parse(tcnnb_hyperparams(const_cast<NetworkWithInputEncoding*>(this)->model())); }
	void set_jit_fusion(bool) {}            /* accepted and ignored: the fused kernel is always on */
	bool jit_fusion() const { return false; }

	const json& encoding_opts() const { return m_encoding; }
	const json& network_opts() const { return m_network; }
	/* used by Trainer: share the trainer's model */
	void attach(std::shared_ptr<detail::ModelHandle> h) { m_model = std::move(h); }
	tcnnb_model* model() {
		if (!m_model) m_model = std::make_shared<detail::ModelHandle>(m_n_in, m_n_out, json{{"encoding", m_encoding}, {"network", m_network}}, 1337u);
		return m_model->m;
	}

private:
	uint32_t m_n_in, m_n_out;
	json m_encoding, m_network;
	std::shared_ptr<detail::ModelHandle> m_model;
};

template <typename T, typename PARAMS_T, typename COMPUTE_T = PARAMS_T>
class Trainer {
public:
	/* trainer.h:89-95. Filled by forward(): output, dL_doutput and L are padded_output_width x batch, column-major (sample-contiguous);
	 * L holds the loss per element (padding rows 0; zero with external_dL_dy) and dL_doutput the loss gradient x loss scale, or views the
	 * caller's external_dL_dy.
	 * perturbed_output stays empty (perturbation_sigma is not built) and model_ctx is empty: backward recomputes the forward pass.
	 * A context of training_step() is empty; its loss is kept by the model. */
	struct ForwardContext : public Context {
		GPUMatrix<COMPUTE_T> perturbed_output;
		GPUMatrix<COMPUTE_T> output;
		GPUMatrix<COMPUTE_T> dL_doutput;
		GPUMatrix<float> L;
		std::unique_ptr<Context> model_ctx;
	};

	/* trainer.h:51-58 */
	Trainer(std::shared_ptr<NetworkWithInputEncoding<COMPUTE_T>> model, std::shared_ptr<Optimizer<PARAMS_T>> optimizer, std::shared_ptr<Loss<COMPUTE_T>> loss, uint32_t seed = 1337)
	: m_model{std::move(model)}, m_optimizer{std::move(optimizer)}, m_loss{std::move(loss)} {
		const json config = {{"loss", m_loss->hyperparams()}, {"optimizer", m_optimizer->hyperparams()}, {"encoding", m_model->encoding_opts()}, {"network", m_model->network_opts()}};
		m_handle = std::make_shared<detail::ModelHandle>(m_model->input_width(), m_model->output_width(), config, seed);
		m_model->attach(m_handle);
	}

	/* trainer.h:254-357. Matrices are n_dims x batch, column-major: input, target, data_pdf and dL_dinput fp32, external_dL_dy
	 * COMPUTE_T (fp16) padded_output_width x batch and already multiplied by the loss scale. With external_dL_dy the loss is not
	 * evaluated (target and data_pdf are not read) and loss() returns 0. */
	std::unique_ptr<ForwardContext> training_step(cudaStream_t stream, const GPUMatrixDynamic<T>& input, const GPUMatrixDynamic<float>& target, const GPUMatrixDynamic<float>* data_pdf = nullptr,
	                                       bool run_optimizer = true, GPUMatrixDynamic<T>* dL_dinput = nullptr, bool use_inference_params = false,
	                                       GradientMode param_gradients_mode = GradientMode::Overwrite, const GPUMatrixDynamic<COMPUTE_T>* external_dL_dy = nullptr) {
		if (!data_pdf && !dL_dinput && !use_inference_params && param_gradients_mode == GradientMode::Overwrite && !external_dL_dy) {
			if (input.n() != target.n()) throw std::runtime_error{"training_step: input and target batch sizes differ"};
			if (input.layout() != CM || target.layout() != CM) throw std::runtime_error{"training_step: column-major (sample-contiguous) matrices only"};
			TCNNB_CHECK_THROW(tcnnb_training_step(m_handle->m, (tcnnb_stream)stream, input.n(), input.data(), target.data(), run_optimizer ? 1 : 0));
			return std::make_unique<ForwardContext>();
		}
		const uint32_t batch_size = input.n();
		if (input.layout() != CM) throw std::runtime_error{"training_step: column-major (sample-contiguous) matrices only"};
		if (external_dL_dy) {  /* trainer.h:127-131 */
			CHECK_THROW(external_dL_dy->m() == m_model->padded_output_width());
			CHECK_THROW(external_dL_dy->n() == batch_size);
			if (external_dL_dy->layout() != CM) throw std::runtime_error{"training_step: column-major (sample-contiguous) matrices only"};
		} else {  /* trainer.h:133-138, losses/relative_l2.h:93-96 */
			CHECK_THROW(input.n() == target.n());
			CHECK_THROW(m_model->output_width() == target.m());
			const uint32_t dims = target.m();
			CHECK_THROW(!data_pdf || data_pdf->m() == dims);
			CHECK_THROW(!data_pdf || data_pdf->n() == batch_size);
			if (target.layout() != CM || (data_pdf && data_pdf->layout() != CM)) throw std::runtime_error{"training_step: column-major (sample-contiguous) matrices only"};
		}
		if (dL_dinput) {
			CHECK_THROW(dL_dinput->m() == m_model->input_width());
			CHECK_THROW(dL_dinput->n() == batch_size);
			if (dL_dinput->layout() != CM) throw std::runtime_error{"training_step: column-major (sample-contiguous) matrices only"};
		}
		TCNNB_CHECK_THROW(tcnnb_training_step_ex(m_handle->m, (tcnnb_stream)stream, batch_size, input.data(), external_dL_dy ? nullptr : target.data(),
		                                         external_dL_dy || !data_pdf ? nullptr : data_pdf->data(), run_optimizer ? 1 : 0, dL_dinput ? dL_dinput->data() : nullptr,
		                                         use_inference_params ? 1 : 0, (int)param_gradients_mode, external_dL_dy ? external_dL_dy->data() : nullptr));
		return std::make_unique<ForwardContext>();
	}
	std::unique_ptr<ForwardContext> training_step(const GPUMatrixDynamic<T>& input, const GPUMatrixDynamic<float>& target, const GPUMatrixDynamic<float>* data_pdf = nullptr,
	                                       bool run_optimizer = true, GPUMatrixDynamic<T>* dL_dinput = nullptr, bool use_inference_params = false,
	                                       GradientMode param_gradients_mode = GradientMode::Overwrite, const GPUMatrixDynamic<COMPUTE_T>* external_dL_dy = nullptr) {
		return training_step(nullptr, input, target, data_pdf, run_optimizer, dL_dinput, use_inference_params, param_gradients_mode, external_dL_dy);
	}

	/* trainer.h:97-145: the predictions, and unless external_dL_dy is given the loss values and loss gradient, of one batch. The loss
	 * scale is the trainer's own (default_loss_scale, 128). With external_dL_dy, ctx->dL_doutput is a view of the caller's matrix: what the
	 * caller writes there before backward() is what backward() propagates. */
	std::unique_ptr<ForwardContext> forward(cudaStream_t stream, const float loss_scale, const GPUMatrixDynamic<T>& input, const GPUMatrix<float>& target,
	                                        const GPUMatrix<float>* data_pdf = nullptr, bool use_inference_params = false, bool prepare_input_gradients = false,
	                                        const GPUMatrix<COMPUTE_T>* external_dL_dy = nullptr) {
		const uint32_t batch_size = input.n(), padded = m_model->padded_output_width();
		if (loss_scale != tcnnb_default_loss_scale()) throw std::runtime_error{"forward: the trainer's loss scale is default_loss_scale (128)"};
		if (input.layout() != CM) throw std::runtime_error{"forward: column-major (sample-contiguous) matrices only"};
		auto ctx = std::make_unique<ForwardContext>();
		ctx->output = GPUMatrix<COMPUTE_T>{padded, batch_size};
		ctx->model_ctx = std::make_unique<Context>();
		ctx->L = GPUMatrix<float>{padded, batch_size};
		if (external_dL_dy) {  /* trainer.h:127-131 */
			CHECK_THROW(external_dL_dy->m() == padded);
			CHECK_THROW(external_dL_dy->n() == batch_size);
			ctx->dL_doutput = GPUMatrix<COMPUTE_T>{external_dL_dy->data(), padded, batch_size};
			ctx->L.memset_async(stream, 0);  /* no loss is evaluated: loss(ctx) is 0, as for training_step with external_dL_dy */
		} else {  /* trainer.h:133-138 */
			CHECK_THROW(input.n() == target.n());
			CHECK_THROW(m_model->output_width() == target.m());
			CHECK_THROW(!data_pdf || (data_pdf->m() == target.m() && data_pdf->n() == batch_size));
			ctx->dL_doutput = GPUMatrix<COMPUTE_T>{padded, batch_size};
		}
		TCNNB_CHECK_THROW(tcnnb_forward(m_handle->m, (tcnnb_stream)stream, batch_size, input.data(), external_dL_dy ? nullptr : target.data(),
		                                external_dL_dy || !data_pdf ? nullptr : data_pdf->data(), use_inference_params ? 1 : 0, prepare_input_gradients ? 1 : 0,
		                                external_dL_dy ? external_dL_dy->data() : nullptr, ctx->output.data(), ctx->L.data(), external_dL_dy ? nullptr : ctx->dL_doutput.data()));
		return ctx;
	}
	std::unique_ptr<ForwardContext> forward(const float loss_scale, const GPUMatrixDynamic<T>& input, const GPUMatrix<float>& target, const GPUMatrix<float>* data_pdf = nullptr,
	                                        bool use_inference_params = false, bool prepare_input_gradients = false, const GPUMatrix<COMPUTE_T>* external_dL_dy = nullptr) {
		return forward(nullptr, loss_scale, input, target, data_pdf, use_inference_params, prepare_input_gradients, external_dL_dy);
	}

	/* trainer.h:147-153: back-propagates ctx.dL_doutput into the gradient buffer (GradientMode as in training_step); no optimizer step */
	void backward(cudaStream_t stream, const ForwardContext& ctx, const GPUMatrixDynamic<T>& input, GPUMatrixDynamic<T>* dL_dinput = nullptr, bool use_inference_params = false,
	              GradientMode param_gradients_mode = GradientMode::Overwrite) {
		const uint32_t batch_size = input.n();
		if (input.layout() != CM) throw std::runtime_error{"backward: column-major (sample-contiguous) matrices only"};
		CHECK_THROW(ctx.dL_doutput.m() == m_model->padded_output_width());
		CHECK_THROW(ctx.dL_doutput.n() == batch_size);
		if (dL_dinput) {
			CHECK_THROW(dL_dinput->m() == m_model->input_width());
			CHECK_THROW(dL_dinput->n() == batch_size);
			if (dL_dinput->layout() != CM) throw std::runtime_error{"backward: column-major (sample-contiguous) matrices only"};
		}
		TCNNB_CHECK_THROW(tcnnb_backward(m_handle->m, (tcnnb_stream)stream, batch_size, input.data(), ctx.output.data(), ctx.dL_doutput.data(), dL_dinput ? dL_dinput->data() : nullptr,
		                                 use_inference_params ? 1 : 0, (int)param_gradients_mode));
	}
	void backward(const ForwardContext& ctx, const GPUMatrixDynamic<T>& input, GPUMatrixDynamic<T>* dL_dinput = nullptr, bool use_inference_params = false,
	              GradientMode param_gradients_mode = GradientMode::Overwrite) {
		backward(nullptr, ctx, input, dL_dinput, use_inference_params, param_gradients_mode);
	}

	void optimizer_step(cudaStream_t stream, float /*loss_scale*/) { TCNNB_CHECK_THROW(tcnnb_optimizer_step(m_handle->m, (tcnnb_stream)stream)); } /* trainer.h:155-157 */

	/* trainer.h:372-378: the sum of ctx.L for a context of forward(); for a context of training_step(), the sum of the per-element
	 * losses of the last step. Device -> host, synchronises the stream. */
	float loss(cudaStream_t stream, const ForwardContext& ctx) const {
		float v = 0;
		if (ctx.L.data()) TCNNB_CHECK_THROW(tcnnb_reduce_sum((tcnnb_stream)stream, ctx.L.data(), ctx.L.n_elements(), &v));
		else TCNNB_CHECK_THROW(tcnnb_loss(m_handle->m, (tcnnb_stream)stream, &v));
		return v;
	}
	float loss(const ForwardContext& ctx) const { return loss(nullptr, ctx); }

	/* trainer.h:442-482 + optimizers/adam.h:303-325: the reference's snapshot schema (nlohmann binary values; instant-ngp stores it as
	 * msgpack): {"n_params", "params_type": "__half", "params_binary", "optimizer": {"current_step", "base_learning_rate",
	 * "first_moments_binary", "second_moments_binary", "param_steps_binary"}}. Under ExponentialDecay the Adam state is nested as in
	 * optimizers/exponential_decay.h:136-148: "optimizer": {"nested": {Adam's keys, with base_learning_rate the DECAYED rate},
	 * "learning_rate": the undecayed base rate, "learning_rate_factor"}. Snapshots written by tiny-cuda-nn load here and vice versa. */
	json serialize(bool serialize_optimizer = false) {
		const size_t n = n_params();
		auto blob = [](const void* dev, size_t bytes) {
			json::binary_t b;
			b.resize(bytes);
			CUDA_CHECK_THROW(cudaMemcpy(b.data(), dev, bytes, cudaMemcpyDeviceToHost));
			return b;
		};
		CUDA_CHECK_THROW(cudaDeviceSynchronize());
		json data;
		data["n_params"] = n;
		data["params_type"] = "__half";
		data["params_binary"] = blob(tcnnb_params(m_handle->m), n * sizeof(__half));
		if (serialize_optimizer) {
			float *m1 = nullptr, *m2 = nullptr, lr = 0;
			uint32_t *steps = nullptr, cur = 0;
			TCNNB_CHECK_THROW(tcnnb_optimizer_state(m_handle->m, &m1, &m2, &steps, &cur, &lr));
			const bool decay = exponential_decay();
			const float factor = tcnnb_learning_rate_factor(m_handle->m);
			json opt;
			opt["current_step"] = cur;
			opt["base_learning_rate"] = decay ? lr * factor : lr;  /* the nested Adam runs at the decayed rate (exponential_decay.h:69) */
			opt["first_moments_binary"] = blob(m1, n * sizeof(float));
			opt["second_moments_binary"] = blob(m2, n * sizeof(float));
			opt["param_steps_binary"] = blob(steps, n * sizeof(uint32_t));
			if (decay) {
				data["optimizer"] = {{"nested", opt}, {"learning_rate", lr}, {"learning_rate_factor", factor}};
			} else {
				data["optimizer"] = opt;
			}
		}
		return data;
	}

	void deserialize(const json& data) {
		auto bytes_of = [](const json& j) -> std::vector<uint8_t> {
			if (j.is_binary()) return j.get_binary();
			if (j.is_object()) {  /* the textual form of a binary value, gpu_memory_json.h:58-67 */
				std::vector<uint8_t> out;
				for (const auto& v : j.at("bytes")) out.push_back((uint8_t)v.get<unsigned>());
				return out;
			}
			throw std::runtime_error{"Invalid json type: must be either binary or object"};
		};
		const size_t n = n_params();
		const std::string type = data.value("params_type", std::string{"__half"});
		const std::vector<uint8_t> p = bytes_of(data.at("params_binary"));
		if (type == "float") {
			if (p.size() != n * sizeof(float)) throw std::runtime_error{"Can't set fp params because buffer has the wrong size."};
			TCNNB_CHECK_THROW(tcnnb_set_params_full_precision(m_handle->m, (const float*)p.data(), n, 0));
		} else if (type == "__half") {
			if (p.size() != n * sizeof(__half)) throw std::runtime_error{"Can't set params because buffer has the wrong size."};
			TCNNB_CHECK_THROW(tcnnb_set_params(m_handle->m, p.data(), n, 0));
		} else {
			throw std::runtime_error{"Trainer: snapshot parameters must be of type float of __half"};
		}
		if (data.contains("optimizer")) {
			/* ExponentialDecay's schema nests the Adam state; a flat one (the wrapper's factor then follows from the step count) loads too */
			const bool nested = exponential_decay() && data["optimizer"].contains("nested");
			const json& opt = nested ? data["optimizer"]["nested"] : data["optimizer"];
			float *m1 = nullptr, *m2 = nullptr;
			uint32_t* steps = nullptr;
			TCNNB_CHECK_THROW(tcnnb_optimizer_state(m_handle->m, &m1, &m2, &steps, nullptr, nullptr));
			const std::vector<uint8_t> a = bytes_of(opt.at("first_moments_binary")), b = bytes_of(opt.at("second_moments_binary"));
			if (a.size() != n * sizeof(float) || b.size() != n * sizeof(float)) throw std::runtime_error{"Trainer: optimizer snapshot has the wrong size."};
			CUDA_CHECK_THROW(cudaMemcpy(m1, a.data(), a.size(), cudaMemcpyHostToDevice));
			CUDA_CHECK_THROW(cudaMemcpy(m2, b.data(), b.size(), cudaMemcpyHostToDevice));
			if (opt.contains("param_steps_binary")) {
				const std::vector<uint8_t> c = bytes_of(opt["param_steps_binary"]);
				if (c.size() != n * sizeof(uint32_t)) throw std::runtime_error{"Trainer: optimizer snapshot has the wrong size."};
				CUDA_CHECK_THROW(cudaMemcpy(steps, c.data(), c.size(), cudaMemcpyHostToDevice));
			} else {
				CUDA_CHECK_THROW(cudaMemset(steps, 0, n * sizeof(uint32_t)));
			}
			const float base_lr = nested ? data["optimizer"].at("learning_rate").get<float>() : opt.at("base_learning_rate").get<float>();
			TCNNB_CHECK_THROW(tcnnb_set_optimizer_progress(m_handle->m, opt.at("current_step").get<uint32_t>(), base_lr));
			if (nested && data["optimizer"].contains("learning_rate_factor")) {
				TCNNB_CHECK_THROW(tcnnb_set_learning_rate_factor(m_handle->m, data["optimizer"]["learning_rate_factor"].get<float>()));
			}
		}
		CUDA_CHECK_THROW(cudaDeviceSynchronize());
	}

	float* params_full_precision() const { return tcnnb_params_full_precision(m_handle->m); }
	PARAMS_T* params() const { return (PARAMS_T*)tcnnb_params(m_handle->m); }
	PARAMS_T* param_gradients() const { return (PARAMS_T*)tcnnb_param_gradients(m_handle->m); }
	size_t n_params() const { return tcnnb_n_params(m_handle->m); }
	std::shared_ptr<NetworkWithInputEncoding<COMPUTE_T>> model() const { return m_model; }
	tcnnb_model* handle() const { return m_handle->m; }

private:
	/* whether the optimizer is Adam inside ExponentialDecay (src/optimizer.cu compares names case-insensitively) */
	bool exponential_decay() const {
		std::string name = m_optimizer->hyperparams().value("otype", std::string{"Adam"});
		for (char& c : name) c = (char)std::tolower((unsigned char)c);
		return name == "exponentialdecay";
	}

	std::shared_ptr<NetworkWithInputEncoding<COMPUTE_T>> m_model;
	std::shared_ptr<Optimizer<PARAMS_T>> m_optimizer;
	std::shared_ptr<Loss<COMPUTE_T>> m_loss;
	std::shared_ptr<detail::ModelHandle> m_handle;
};

/* config.h:46-63 */
struct TrainableModel {
	std::shared_ptr<Loss<network_precision_t>> loss;
	std::shared_ptr<Optimizer<network_precision_t>> optimizer;
	std::shared_ptr<NetworkWithInputEncoding<network_precision_t>> network;
	std::shared_ptr<Trainer<float, network_precision_t, network_precision_t>> trainer;
};

inline TrainableModel create_from_config(uint32_t n_input_dims, uint32_t n_output_dims, json config) {
	const json loss_opts = config.value("loss", json::object()), optimizer_opts = config.value("optimizer", json::object());
	const json network_opts = config.value("network", json::object()), encoding_opts = config.value("encoding", json::object());
	std::shared_ptr<Loss<network_precision_t>> loss{create_loss<network_precision_t>(loss_opts)};
	std::shared_ptr<Optimizer<network_precision_t>> optimizer{create_optimizer<network_precision_t>(optimizer_opts)};
	auto network = std::make_shared<NetworkWithInputEncoding<network_precision_t>>(n_input_dims, n_output_dims, encoding_opts, network_opts);
	auto trainer = std::make_shared<Trainer<float, network_precision_t, network_precision_t>>(network, optimizer, loss);
	return {loss, optimizer, network, trainer};
}

}  // namespace tcnn
