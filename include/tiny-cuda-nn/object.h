/* tiny-cuda-nn/object.h -- the object model applications compose (reference: object.h:46-730): ParametricObject and
 * DifferentiableObject<T, PARAMS_T, COMPUTE_T> with the reference's public methods. Parameters are caller-owned device pointers handed
 * over with set_params() (a Trainer does this, trainer.h:69-87). Matrices of either layout are accepted; row-major ones pass through one
 * transpose kernel of libtcnn_b200 on the way in and out. */
#pragma once
#if __has_include(<json/json.hpp>)
#include <json/json.hpp>
#else
#include <nlohmann/json.hpp>
#endif

#include <functional>
#include <memory>
#include <string>

#include "common.h"
#include "gpu_matrix.h"
#include "random.h"

namespace tcnn {

using json = nlohmann::json;

/* object.h:116-120 */
enum class GradientMode {
	Ignore,
	Overwrite,
	Accumulate,
};

#ifndef TCNN_B200_CONTEXT_DEFINED  /* cpp_api.h defines the same type */
#define TCNN_B200_CONTEXT_DEFINED
struct Context { /* cpp_api.h:39-47: what a forward pass hands to its backward pass */
	Context() = default;
	virtual ~Context() {}
	Context(const Context&) = delete;
	Context& operator=(const Context&) = delete;
	Context(Context&&) = delete;
	Context& operator=(Context&&) = delete;
};
#endif

/* common.h:243 */
template <typename T>
constexpr float default_loss_scale() { return sizeof(T) == 2 ? LOSS_SCALE : 1.0f; }

/* common_host.h: log callbacks and the run-time compiler's directories. Nothing here logs and nothing is compiled at run time. */
enum class LogSeverity { Info, Debug, Warning, Error, Success };
inline void set_log_callback(const std::function<void(LogSeverity, const std::string&)>&) {}
inline void rtc_set_cache_dir(const std::string&) {}
inline void rtc_set_include_dir(const std::string&) {}

namespace detail {
/* Device pointer to `m` in column-major (sample-contiguous) layout: the matrix itself, or its transpose in `scratch`. */
template <typename X>
const X* cm_data(cudaStream_t stream, const GPUMatrixDynamic<X>& m, GPUMemory<X>& scratch) {
	if (m.layout() == CM) return m.data();
	scratch.enlarge(m.n_elements());
	TCNNB_CHECK_THROW(tcnnb_transpose((tcnnb_stream)stream, m.m(), m.n(), sizeof(X), m.data(), scratch.data()));
	return scratch.data();
}
/* Where a result for `m` is written in column-major layout; finish_cm() moves it into `m` when `m` is row-major. */
template <typename X>
X* cm_target(GPUMatrixDynamic<X>& m, GPUMemory<X>& scratch) {
	if (m.layout() == CM) return m.data();
	scratch.enlarge(m.n_elements());
	return scratch.data();
}
template <typename X>
void finish_cm(cudaStream_t stream, GPUMatrixDynamic<X>& m, const GPUMemory<X>& scratch) {
	if (m.layout() != CM) TCNNB_CHECK_THROW(tcnnb_transpose((tcnnb_stream)stream, m.n(), m.m(), sizeof(X), scratch.data(), m.data()));
}
}  // namespace detail

/* object.h:46-52 */
class Object {
public:
	virtual ~Object() {}
	virtual json hyperparams() const = 0;
	virtual std::string name() const = 0;
};

/* object.h:64-105 */
template <typename PARAMS_T>
class ParametricObject : public Object {
public:
	virtual ~ParametricObject() {}
	virtual void set_params_impl(PARAMS_T* params, PARAMS_T* inference_params, PARAMS_T* gradients) {}
	void set_params(PARAMS_T* params, PARAMS_T* inference_params, PARAMS_T* gradients) {
		m_params = params;
		m_inference_params = inference_params;
		m_gradients = gradients;
		set_params_impl(params, inference_params, gradients);
	}
	/* Fills the device array params_full_precision [n_params()] from `rnd` and advances it as the reference does. */
	virtual void initialize_params(pcg32& rnd, float* params_full_precision, float scale = 1) = 0;
	virtual size_t n_params() const = 0;
	PARAMS_T* params() const { return m_params; }
	PARAMS_T* inference_params() const { return m_inference_params; }
	PARAMS_T* gradients() const { return m_gradients; }

private:
	PARAMS_T* m_params = nullptr;
	PARAMS_T* m_inference_params = nullptr;
	PARAMS_T* m_gradients = nullptr;
};

/* object.h:154-730. Shapes: input input_width() x batch, output padded_output_width() x batch (inference: output_width() x batch, fp32),
 * batch a multiple of BATCH_SIZE_GRANULARITY. forward() keeps what backward() needs in the returned Context. */
template <typename T, typename PARAMS_T, typename COMPUTE_T = T>
class DifferentiableObject : public ParametricObject<PARAMS_T> {
public:
	virtual ~DifferentiableObject() {}

	virtual void inference_mixed_precision_impl(cudaStream_t stream, const GPUMatrixDynamic<T>& input, GPUMatrixDynamic<COMPUTE_T>& output, bool use_inference_params = true) = 0;
	void inference_mixed_precision(cudaStream_t stream, const GPUMatrixDynamic<T>& input, GPUMatrixDynamic<COMPUTE_T>& output, bool use_inference_params = true) {
		check_io(input.m(), input.n(), output.m(), output.n(), padded_output_width());
		check_params(use_inference_params);
		inference_mixed_precision_impl(stream, input, output, use_inference_params);
	}
	void inference_mixed_precision(const GPUMatrixDynamic<T>& input, GPUMatrixDynamic<COMPUTE_T>& output, bool use_inference_params = true) {
		inference_mixed_precision(nullptr, input, output, use_inference_params);
	}

	/* object.h:214-282: the mixed-precision result, trimmed to output_width() and cast to fp32 */
	virtual void inference_impl(cudaStream_t stream, const GPUMatrixDynamic<T>& input, GPUMatrixDynamic<float>& output, bool use_inference_params) = 0;
	void inference(cudaStream_t stream, const GPUMatrixDynamic<T>& input, GPUMatrixDynamic<float>& output, bool use_inference_params = true) {
		check_io(input.m(), input.n(), output.m(), output.n(), output_width());
		check_params(use_inference_params);
		inference_impl(stream, input, output, use_inference_params);
	}
	void inference(const GPUMatrixDynamic<T>& input, GPUMatrixDynamic<float>& output, bool use_inference_params = true) { inference(nullptr, input, output, use_inference_params); }

	virtual std::unique_ptr<Context> forward_impl(cudaStream_t stream, const GPUMatrixDynamic<T>& input, GPUMatrixDynamic<COMPUTE_T>* output = nullptr, bool use_inference_params = false,
	                                              bool prepare_input_gradients = false) = 0;
	std::unique_ptr<Context> forward(cudaStream_t stream, const GPUMatrixDynamic<T>& input, GPUMatrixDynamic<COMPUTE_T>* output = nullptr, bool use_inference_params = false,
	                                 bool prepare_input_gradients = false) {
		if (output) check_io(input.m(), input.n(), output->m(), output->n(), padded_output_width());
		else check_io(input.m(), input.n(), padded_output_width(), input.n(), padded_output_width());
		check_params(use_inference_params);
		return forward_impl(stream, input, output, use_inference_params, prepare_input_gradients);
	}
	std::unique_ptr<Context> forward(const GPUMatrixDynamic<T>& input, GPUMatrixDynamic<COMPUTE_T>* output = nullptr, bool use_inference_params = false, bool prepare_input_gradients = false) {
		return forward(nullptr, input, output, use_inference_params, prepare_input_gradients);
	}

	/* dL_dinput (optional) is overwritten; the parameter gradients go to gradients() according to param_gradients_mode */
	virtual void backward_impl(cudaStream_t stream, const Context& ctx, const GPUMatrixDynamic<T>& input, const GPUMatrixDynamic<COMPUTE_T>& output, const GPUMatrixDynamic<COMPUTE_T>& dL_doutput,
	                           GPUMatrixDynamic<T>* dL_dinput = nullptr, bool use_inference_params = false, GradientMode param_gradients_mode = GradientMode::Overwrite) = 0;
	void backward(cudaStream_t stream, const Context& ctx, const GPUMatrixDynamic<T>& input, const GPUMatrixDynamic<COMPUTE_T>& output, const GPUMatrixDynamic<COMPUTE_T>& dL_doutput,
	              GPUMatrixDynamic<T>* dL_dinput = nullptr, bool use_inference_params = false, GradientMode param_gradients_mode = GradientMode::Overwrite) {
		check_io(input.m(), input.n(), output.m(), output.n(), padded_output_width());
		CHECK_THROW(dL_doutput.m() == padded_output_width() && dL_doutput.n() == input.n());
		CHECK_THROW(!dL_dinput || (dL_dinput->m() == input_width() && dL_dinput->n() == input.n()));
		check_params(use_inference_params);
		if (param_gradients_mode != GradientMode::Ignore && this->n_params() > 0) CHECK_THROW(this->gradients() != nullptr);
		backward_impl(stream, ctx, input, output, dL_doutput, dL_dinput, use_inference_params, param_gradients_mode);
	}
	void backward(const Context& ctx, const GPUMatrixDynamic<T>& input, const GPUMatrixDynamic<COMPUTE_T>& output, const GPUMatrixDynamic<COMPUTE_T>& dL_doutput,
	              GPUMatrixDynamic<T>* dL_dinput = nullptr, bool use_inference_params = false, GradientMode param_gradients_mode = GradientMode::Overwrite) {
		backward(nullptr, ctx, input, output, dL_doutput, dL_dinput, use_inference_params, param_gradients_mode);
	}

	/* object.h:468-560: second-order derivatives. Built for the grid encodings of create_encoding; every other object throws. */
	virtual void backward_backward_input_impl(cudaStream_t stream, const Context& ctx, const GPUMatrixDynamic<T>& input, const GPUMatrixDynamic<T>& dL_ddLdinput,
	                                          const GPUMatrixDynamic<COMPUTE_T>& dL_doutput, GPUMatrixDynamic<COMPUTE_T>* dL_ddLdoutput = nullptr, GPUMatrixDynamic<T>* dL_dinput = nullptr,
	                                          bool use_inference_params = false, GradientMode param_gradients_mode = GradientMode::Overwrite) {
		throw std::runtime_error{"tcnn_b200: second-order derivatives (backward_backward_input) of " + this->name() + " are not built"};
	}
	void backward_backward_input(cudaStream_t stream, const Context& ctx, const GPUMatrixDynamic<T>& input, const GPUMatrixDynamic<T>& dL_ddLdinput, const GPUMatrixDynamic<COMPUTE_T>& dL_doutput,
	                             GPUMatrixDynamic<COMPUTE_T>* dL_ddLdoutput = nullptr, GPUMatrixDynamic<T>* dL_dinput = nullptr, bool use_inference_params = false,
	                             GradientMode param_gradients_mode = GradientMode::Overwrite) {
		check_params(use_inference_params);
		backward_backward_input_impl(stream, ctx, input, dL_ddLdinput, dL_doutput, dL_ddLdoutput, dL_dinput, use_inference_params, param_gradients_mode);
	}
	void backward_backward_input(const Context& ctx, const GPUMatrixDynamic<T>& input, const GPUMatrixDynamic<T>& dL_ddLdinput, const GPUMatrixDynamic<COMPUTE_T>& dL_doutput,
	                             GPUMatrixDynamic<COMPUTE_T>* dL_ddLdoutput = nullptr, GPUMatrixDynamic<T>* dL_dinput = nullptr, bool use_inference_params = false,
	                             GradientMode param_gradients_mode = GradientMode::Overwrite) {
		backward_backward_input(nullptr, ctx, input, dL_ddLdinput, dL_doutput, dL_ddLdoutput, dL_dinput, use_inference_params, param_gradients_mode);
	}

	virtual uint32_t input_width() const = 0;
	virtual uint32_t padded_output_width() const = 0;
	virtual uint32_t output_width() const = 0;
	virtual uint32_t required_input_alignment() const { return 1; }

	/* accepted and ignored: there is no run-time compilation, the built kernels always run (supports_jit_fusion() is false) */
	bool jit_fusion() const { return false; }
	void set_jit_fusion(bool) {}

protected:
	void check_params(bool use_inference_params) const {
		if (this->n_params() == 0) return;
		if ((use_inference_params ? this->inference_params() : this->params()) == nullptr) {
			throw std::runtime_error{this->name() + ": parameters are not set (set_params, or construct a Trainer over the object)"};
		}
	}

private:
	void check_io(uint32_t in_m, uint32_t in_n, uint32_t out_m, uint32_t out_n, uint32_t want_out_m) const {
		CHECK_THROW(in_m == input_width());
		CHECK_THROW(out_m == want_out_m);
		CHECK_THROW(in_n % BATCH_SIZE_GRANULARITY == 0);
		CHECK_THROW(in_n == out_n);
	}
};

}  // namespace tcnn

#include "config.h"
