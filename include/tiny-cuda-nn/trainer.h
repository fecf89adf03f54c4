/* tiny-cuda-nn/trainer.h -- Trainer<T, PARAMS_T, COMPUTE_T> with the signatures applications use (reference: trainer.h:51-161,254-482),
 * implemented over the trainer tier of libtcnn_b200. The loss and the optimizer are light objects that carry their JSON options; the
 * Trainer makes ONE tcnnb_model handle of the model, loss and optimizer together. Inputs and targets may be row- or column-major. */
#pragma once
#include <random>
#include <vector>

#include "loss.h"
#include "network_with_input_encoding.h"
#include "optimizer.h"

namespace tcnn {

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

	using Model = DifferentiableObject<T, PARAMS_T, COMPUTE_T>;

	/* trainer.h:51-87. The trainer owns the parameters and hands pointers into them to the model (set_params), so that the model's own
	 * calls afterwards run on the trained weights. Parameters are initialised from pcg32{seed_seq{seed}} as in the reference.
	 *   NetworkWithInputEncoding (from JSON or from two objects): the create_from_config model of {"loss", "optimizer", "encoding", "network"}.
	 *   Network<__half> of create_network: a trainer over the network alone (tcnnb_create_network_trainer), fp16 inputs.
	 *   Encoding: parameters only; training an encoding alone is not built. */
	Trainer(std::shared_ptr<Model> model, std::shared_ptr<Optimizer<PARAMS_T>> optimizer, std::shared_ptr<Loss<COMPUTE_T>> loss, uint32_t seed = 1337)
	: m_model{std::move(model)}, m_optimizer{std::move(optimizer)}, m_loss{std::move(loss)} {
		const json loss_opts = m_loss->hyperparams(), optimizer_opts = m_optimizer->hyperparams();
		if (auto* nwie = dynamic_cast<NetworkWithInputEncoding<COMPUTE_T>*>(m_model.get())) {
			const json config = {{"loss", loss_opts}, {"optimizer", optimizer_opts}, {"encoding", nwie->encoding_opts()}, {"network", nwie->network_opts()}};
			m_handle = std::make_shared<detail::ModelHandle>(m_model->input_width(), m_model->output_width(), config, seed);
			nwie->attach(m_handle);
		} else if (dynamic_cast<detail::NetworkObject*>(m_model.get())) {
			const json config = {{"loss", loss_opts}, {"optimizer", optimizer_opts}, {"network", detail::network_keys(m_model->hyperparams())}};
			m_handle = std::make_shared<detail::ModelHandle>(detail::ModelHandle::NetworkTrainer{}, m_model->input_width(), m_model->output_width(), config, seed);
		} else if (auto* encoding = dynamic_cast<detail::EncodingObject*>(m_model.get())) {
			initialize_encoding_params(*encoding, seed);
			return;
		} else {
			throw std::runtime_error{"Trainer: " + m_model->name() + " is not a model tcnn_b200 trains (NetworkWithInputEncoding, create_network, create_encoding)"};
		}
		m_model->set_params((PARAMS_T*)tcnnb_params(h()), (PARAMS_T*)tcnnb_params_inference(h()), (PARAMS_T*)tcnnb_param_gradients(h()));
	}

	/* trainer.h:254-357. Matrices are n_dims x batch, column-major: input, target, data_pdf and dL_dinput fp32, external_dL_dy
	 * COMPUTE_T (fp16) padded_output_width x batch and already multiplied by the loss scale. With external_dL_dy the loss is not
	 * evaluated (target and data_pdf are not read) and loss() returns 0. */
	std::unique_ptr<ForwardContext> training_step(cudaStream_t stream, const GPUMatrixDynamic<T>& input, const GPUMatrixDynamic<float>& target, const GPUMatrixDynamic<float>* data_pdf = nullptr,
	                                       bool run_optimizer = true, GPUMatrixDynamic<T>* dL_dinput = nullptr, bool use_inference_params = false,
	                                       GradientMode param_gradients_mode = GradientMode::Overwrite, const GPUMatrixDynamic<COMPUTE_T>* external_dL_dy = nullptr) {
		const float* in = (const float*)detail::cm_data(stream, input, m_input_scratch);
		if (!data_pdf && !dL_dinput && !use_inference_params && param_gradients_mode == GradientMode::Overwrite && !external_dL_dy) {
			if (input.n() != target.n()) throw std::runtime_error{"training_step: input and target batch sizes differ"};
			TCNNB_CHECK_THROW(tcnnb_training_step(h(), (tcnnb_stream)stream, input.n(), in, detail::cm_data(stream, target, m_target_scratch), run_optimizer ? 1 : 0));
			return std::make_unique<ForwardContext>();
		}
		const uint32_t batch_size = input.n();
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
			if (data_pdf && data_pdf->layout() != CM) throw std::runtime_error{"training_step: column-major (sample-contiguous) data_pdf only"};
		}
		if (dL_dinput) {
			CHECK_THROW(dL_dinput->m() == m_model->input_width());
			CHECK_THROW(dL_dinput->n() == batch_size);
			if (dL_dinput->layout() != CM) throw std::runtime_error{"training_step: column-major (sample-contiguous) matrices only"};
		}
		TCNNB_CHECK_THROW(tcnnb_training_step_ex(h(), (tcnnb_stream)stream, batch_size, in, external_dL_dy ? nullptr : detail::cm_data(stream, target, m_target_scratch),
		                                         external_dL_dy || !data_pdf ? nullptr : data_pdf->data(), run_optimizer ? 1 : 0, dL_dinput ? (float*)dL_dinput->data() : nullptr,
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
		const float* in = (const float*)detail::cm_data(stream, input, m_input_scratch);
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
		TCNNB_CHECK_THROW(tcnnb_forward(h(), (tcnnb_stream)stream, batch_size, in, external_dL_dy ? nullptr : detail::cm_data(stream, target, m_target_scratch),
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
		const float* in = (const float*)detail::cm_data(stream, input, m_input_scratch);
		CHECK_THROW(ctx.dL_doutput.m() == m_model->padded_output_width());
		CHECK_THROW(ctx.dL_doutput.n() == batch_size);
		if (dL_dinput) {
			CHECK_THROW(dL_dinput->m() == m_model->input_width());
			CHECK_THROW(dL_dinput->n() == batch_size);
			if (dL_dinput->layout() != CM) throw std::runtime_error{"backward: column-major (sample-contiguous) matrices only"};
		}
		TCNNB_CHECK_THROW(tcnnb_backward(h(), (tcnnb_stream)stream, batch_size, in, ctx.output.data(), ctx.dL_doutput.data(), dL_dinput ? (float*)dL_dinput->data() : nullptr,
		                                 use_inference_params ? 1 : 0, (int)param_gradients_mode));
	}
	void backward(const ForwardContext& ctx, const GPUMatrixDynamic<T>& input, GPUMatrixDynamic<T>* dL_dinput = nullptr, bool use_inference_params = false,
	              GradientMode param_gradients_mode = GradientMode::Overwrite) {
		backward(nullptr, ctx, input, dL_dinput, use_inference_params, param_gradients_mode);
	}

	void optimizer_step(cudaStream_t stream, float /*loss_scale*/) { TCNNB_CHECK_THROW(tcnnb_optimizer_step(h(), (tcnnb_stream)stream)); } /* trainer.h:155-157 */

	/* trainer.h:372-378: the sum of ctx.L for a context of forward(); for a context of training_step(), the sum of the per-element
	 * losses of the last step. Device -> host, synchronises the stream. */
	float loss(cudaStream_t stream, const ForwardContext& ctx) const {
		float v = 0;
		if (ctx.L.data()) TCNNB_CHECK_THROW(tcnnb_reduce_sum((tcnnb_stream)stream, ctx.L.data(), ctx.L.n_elements(), &v));
		else TCNNB_CHECK_THROW(tcnnb_loss(h(), (tcnnb_stream)stream, &v));
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
		data["params_binary"] = blob(tcnnb_params(h()), n * sizeof(__half));
		if (serialize_optimizer) {
			float *m1 = nullptr, *m2 = nullptr, lr = 0;
			uint32_t *steps = nullptr, cur = 0;
			TCNNB_CHECK_THROW(tcnnb_optimizer_state(h(), &m1, &m2, &steps, &cur, &lr));
			const bool decay = exponential_decay();
			const float factor = tcnnb_learning_rate_factor(h());
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
			TCNNB_CHECK_THROW(tcnnb_set_params_full_precision(h(), (const float*)p.data(), n, 0));
		} else if (type == "__half") {
			if (p.size() != n * sizeof(__half)) throw std::runtime_error{"Can't set params because buffer has the wrong size."};
			TCNNB_CHECK_THROW(tcnnb_set_params(h(), p.data(), n, 0));
		} else {
			throw std::runtime_error{"Trainer: snapshot parameters must be of type float of __half"};
		}
		if (data.contains("optimizer")) {
			/* ExponentialDecay's schema nests the Adam state; a flat one (the wrapper's factor then follows from the step count) loads too */
			const bool nested = exponential_decay() && data["optimizer"].contains("nested");
			const json& opt = nested ? data["optimizer"]["nested"] : data["optimizer"];
			float *m1 = nullptr, *m2 = nullptr;
			uint32_t* steps = nullptr;
			TCNNB_CHECK_THROW(tcnnb_optimizer_state(h(), &m1, &m2, &steps, nullptr, nullptr));
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
			TCNNB_CHECK_THROW(tcnnb_set_optimizer_progress(h(), opt.at("current_step").get<uint32_t>(), base_lr));
			if (nested && data["optimizer"].contains("learning_rate_factor")) {
				TCNNB_CHECK_THROW(tcnnb_set_learning_rate_factor(h(), data["optimizer"]["learning_rate_factor"].get<float>()));
			}
		}
		CUDA_CHECK_THROW(cudaDeviceSynchronize());
	}

	float* params_full_precision() const { return m_handle ? tcnnb_params_full_precision(h()) : m_encoding_params_fp32.data(); }
	PARAMS_T* params() const { return m_handle ? (PARAMS_T*)tcnnb_params(h()) : m_encoding_params.data(); }
	PARAMS_T* param_gradients() const { return m_handle ? (PARAMS_T*)tcnnb_param_gradients(h()) : m_encoding_params.data() + m_model->n_params(); }
	size_t n_params() const { return m_handle ? tcnnb_n_params(h()) : m_model->n_params(); }
	std::shared_ptr<Model> model() const { return m_model; }
	tcnnb_model* handle() const { return h(); }

private:
	tcnnb_model* h() const {
		if (!m_handle) throw std::runtime_error{"Trainer: training an Encoding on its own is not built; train it inside a NetworkWithInputEncoding"};
		return m_handle->m;
	}

	/* trainer.h:69-87 for an Encoding: [fp32 master | fp16 params | fp16 gradients] owned here, initialised like the encoding tier's */
	void initialize_encoding_params(detail::EncodingObject& encoding, uint32_t seed) {
		const size_t n = m_model->n_params();
		std::seed_seq seq{seed};
		std::vector<uint32_t> seeds(2);
		seq.generate(seeds.begin(), seeds.end());
		m_encoding_params_fp32.resize(n);
		m_encoding_params.resize(2 * n);
		m_encoding_params.memset(0);
		if (n) {
			encoding.initialize_params_from_seed(seeds.front(), m_encoding_params_fp32.data());
			std::vector<float> host(n);
			m_encoding_params_fp32.copy_to_host(host);
			std::vector<PARAMS_T> half(2 * n);
			for (size_t i = 0; i < n; ++i) half[i] = (PARAMS_T)host[i];
			m_encoding_params.copy_from_host(half);
		}
		m_model->set_params(m_encoding_params.data(), m_encoding_params.data(), m_encoding_params.data() + n);
	}

	/* whether the optimizer is Adam inside ExponentialDecay (src/optimizer.cu compares names case-insensitively) */
	bool exponential_decay() const {
		std::string name = m_optimizer->hyperparams().value("otype", std::string{"Adam"});
		for (char& c : name) c = (char)std::tolower((unsigned char)c);
		return name == "exponentialdecay";
	}

	std::shared_ptr<Model> m_model;
	std::shared_ptr<Optimizer<PARAMS_T>> m_optimizer;
	std::shared_ptr<Loss<COMPUTE_T>> m_loss;
	std::shared_ptr<detail::ModelHandle> m_handle;  /* null for an Encoding */
	GPUMemory<float> m_encoding_params_fp32;
	GPUMemory<PARAMS_T> m_encoding_params;
	/* column-major copies of row-major inputs and targets */
	GPUMemory<T> m_input_scratch;
	GPUMemory<float> m_target_scratch;
};

}  // namespace tcnn

#include "config.h"
