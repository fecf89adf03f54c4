/* tiny-cuda-nn/encoding.h -- Encoding<T> and create_encoding<T>(n_dims, json) (reference: encoding.h:39-90, src/encoding.cu:60-150), over the
 * encoding tier of libtcnn_b200 (tcnnb_encoding_*). fp32 inputs in [0, 1], fp16 outputs of the encoding's own width (no padding). An
 * encoding is trained inside a NetworkWithInputEncoding; training one alone is not built. */
#pragma once
#include "object.h"

namespace tcnn {

template <typename T>
class Encoding : public DifferentiableObject<float, T, T> {
public:
	virtual ~Encoding() {}
	/* the output is never padded here: the width a network reads is padded by the NetworkWithInputEncoding */
	virtual void set_padded_output_width(uint32_t padded_output_width) {
		if (padded_output_width != this->output_width()) throw std::runtime_error{"tcnn_b200: encodings on their own are not padded"};
	}
	virtual uint32_t required_output_alignment() const { return 1; }
	virtual MatrixLayout preferred_output_layout() const { return CM; }
};

namespace detail {

class EncodingObject : public Encoding<__half> {
public:
	EncodingObject(uint32_t n_dims_to_encode, const json& config) : m_config(config) {
		TCNNB_CHECK_THROW(tcnnb_encoding_create(n_dims_to_encode, config.dump().c_str(), &m_h));
	}
	~EncodingObject() override { tcnnb_encoding_destroy(m_h); }
	EncodingObject(const EncodingObject&) = delete;
	EncodingObject& operator=(const EncodingObject&) = delete;

	void inference_mixed_precision_impl(cudaStream_t stream, const GPUMatrixDynamic<float>& input, GPUMatrixDynamic<__half>& output, bool use_inference_params = true) override {
		const float* in = cm_data(stream, input, m_in_scratch);
		__half* out = cm_target(output, m_out_scratch);
		TCNNB_CHECK_THROW(tcnnb_encoding_forward(m_h, (tcnnb_stream)stream, input.n(), in, out, weights(use_inference_params)));
		finish_cm(stream, output, m_out_scratch);
	}
	void inference_impl(cudaStream_t, const GPUMatrixDynamic<float>&, GPUMatrixDynamic<float>&, bool) override {
		throw std::runtime_error{"tcnn_b200: Encoding::inference with fp32 outputs is not built; inference_mixed_precision gives the fp16 features"};
	}
	std::unique_ptr<Context> forward_impl(cudaStream_t stream, const GPUMatrixDynamic<float>& input, GPUMatrixDynamic<__half>* output = nullptr, bool use_inference_params = false,
	                                      bool = false) override {
		if (output) inference_mixed_precision_impl(stream, input, *output, use_inference_params);
		return std::make_unique<Context>();  /* nothing to keep: backward recomputes from the input */
	}
	void backward_impl(cudaStream_t stream, const Context&, const GPUMatrixDynamic<float>& input, const GPUMatrixDynamic<__half>&, const GPUMatrixDynamic<__half>& dL_doutput,
	                   GPUMatrixDynamic<float>* dL_dinput = nullptr, bool use_inference_params = false, GradientMode param_gradients_mode = GradientMode::Overwrite) override {
		if (param_gradients_mode == GradientMode::Accumulate) throw std::runtime_error{"Encoding::backward: GradientMode::Accumulate is not built for an encoding object"};
		const float* in = cm_data(stream, input, m_in_scratch);
		const __half* dy = cm_data(stream, dL_doutput, m_out_scratch);
		float* dx = dL_dinput ? cm_target(*dL_dinput, m_dx_scratch) : nullptr;
		__half* dparams = param_gradients_mode == GradientMode::Overwrite && n_params() ? this->gradients() : nullptr;
		TCNNB_CHECK_THROW(tcnnb_encoding_backward(m_h, (tcnnb_stream)stream, input.n(), dx, dy, dparams, in, weights(use_inference_params)));
		if (dL_dinput) finish_cm(stream, *dL_dinput, m_dx_scratch);
	}
	/* grid.h:910-1042, column-major matrices */
	void backward_backward_input_impl(cudaStream_t stream, const Context&, const GPUMatrixDynamic<float>& input, const GPUMatrixDynamic<float>& dL_ddLdinput,
	                                  const GPUMatrixDynamic<__half>& dL_doutput, GPUMatrixDynamic<__half>* dL_ddLdoutput = nullptr, GPUMatrixDynamic<float>* dL_dinput = nullptr,
	                                  bool use_inference_params = false, GradientMode param_gradients_mode = GradientMode::Overwrite) override {
		if (input.layout() != CM || dL_ddLdinput.layout() != CM || dL_doutput.layout() != CM || (dL_ddLdoutput && dL_ddLdoutput->layout() != CM) || (dL_dinput && dL_dinput->layout() != CM)) {
			throw std::runtime_error{"Encoding::backward_backward_input: column-major (sample-contiguous) matrices only"};
		}
		if (param_gradients_mode == GradientMode::Accumulate) throw std::runtime_error{"Encoding::backward_backward_input: GradientMode::Accumulate is not built for an encoding object"};
		__half* dparams = param_gradients_mode == GradientMode::Overwrite && n_params() ? this->gradients() : nullptr;
		TCNNB_CHECK_THROW(tcnnb_encoding_backward_backward_input(m_h, (tcnnb_stream)stream, input.n(), dL_ddLdinput.data(), input.data(), dL_doutput.data(), dparams,
		                                                         dL_ddLdoutput ? dL_ddLdoutput->data() : nullptr, dL_dinput ? dL_dinput->data() : nullptr, weights(use_inference_params)));
	}

	/* grid.h:1076-1079 from pcg32{seed}, seeded from the caller's generator (see NetworkObject::initialize_params) */
	void initialize_params(pcg32& rnd, float* params_full_precision, float scale = 1) override {
		TCNNB_CHECK_THROW(tcnnb_encoding_initialize_params(m_h, rnd.next_uint(), params_full_precision, scale));
	}
	/* the same from pcg32{seed}: what a Trainer's initialisation draws (trainer.h:51-87) */
	void initialize_params_from_seed(uint64_t seed, float* params_full_precision, float scale = 1) {
		TCNNB_CHECK_THROW(tcnnb_encoding_initialize_params(m_h, seed, params_full_precision, scale));
	}
	size_t n_params() const override { return tcnnb_encoding_n_params(m_h); }

	uint32_t input_width() const override { return tcnnb_encoding_n_input_dims(m_h); }
	uint32_t padded_output_width() const override { return tcnnb_encoding_n_output_dims(m_h); }
	uint32_t output_width() const override { return tcnnb_encoding_n_output_dims(m_h); }

	json hyperparams() const override { return m_config; }
	std::string name() const override { return m_config.value("otype", std::string{"OneBlob"}); }

private:
	const __half* weights(bool use_inference_params) const { return use_inference_params ? this->inference_params() : this->params(); }

	tcnnb_encoding* m_h = nullptr;
	json m_config;
	GPUMemory<float> m_in_scratch, m_dx_scratch;
	GPUMemory<__half> m_out_scratch;
};

}  // namespace detail

/* src/encoding.cu:132-150. The half-precision build only, as in tcnn::cpp::create_encoding. */
template <typename T>
Encoding<T>* create_encoding(uint32_t n_dims_to_encode, const json& encoding, uint32_t /*alignment*/ = 8) {
	static_assert(sizeof(T) == 2, "tcnn_b200 mirrors the half-precision build of the reference: create_encoding with Precision::Fp32 is not built");
	return new detail::EncodingObject{n_dims_to_encode, encoding};
}

}  // namespace tcnn

#include "config.h"
