/* tiny-cuda-nn/cpp_api.h -- the type-erased tier `tcnn::cpp` (reference: include/tiny-cuda-nn/cpp_api.h:39-125, src/cpp_api.cu:39-174):
 * the interface the PyTorch extension binds (bindings/torch/tinycudann/bindings.cpp:77-343). Same names, signatures and conventions
 * -- the reference's bindings.cpp compiles against this header unchanged -- implemented header-only over the C ABI of libtcnn_b200
 * (tcnnb_module_* / tcnnb_network_* / tcnnb_encoding_*).
 *
 * Conventions (src/cpp_api.cu:71-158): input fp32 [n][n_input_dims]; output / dL_doutput in output_precision() (fp16)
 * [n][n_output_dims()] with n_output_dims() the PADDED width; params / dL_dparams caller-owned arrays of n_params() elements in
 * param_precision() (fp16); gradients are OVERWRITTEN; a null result pointer means "do not compute"; factories return owning raw
 * pointers. Differences, by design: forward() keeps no activations (backward recomputes the forward pass inside the fused kernel),
 * so the returned Context only marks "a forward pass was made"; jit fusion does not exist (the fused kernel is the product).
 * backward_backward_input is built where the reference builds it, for the grid encodings of create_encoding (recomputed from the
 * input and the parameters, no forward context needed); every other encoding reports "<name> does not support double backward."
 * and the network modules throw. */
#pragma once
#if __has_include(<json/json.hpp>)
#include <json/json.hpp>
#else
#include <nlohmann/json.hpp>
#endif

#include <cuda_runtime.h>

#include <functional>
#include <memory>
#include <stdexcept>
#include <string>

#include "../tcnn_b200.h"

namespace tcnn {
#ifndef TCNN_B200_CONTEXT_DEFINED
#define TCNN_B200_CONTEXT_DEFINED
struct Context { /* cpp_api.h:39-47 */
	Context() = default;
	virtual ~Context() {}
	Context(const Context&) = delete;
	Context& operator=(const Context&) = delete;
	Context(Context&&) = delete;
	Context& operator=(Context&&) = delete;
};
#endif
}  // namespace tcnn

namespace tcnn { namespace cpp {

enum class LogSeverity { Info, Debug, Warning, Error, Success };

using json = nlohmann::json;

#define TCNNB_CPP_CHECK(x)                                             \
	do {                                                               \
		if ((x) != 0) throw std::runtime_error{tcnnb_last_error()};     \
	} while (0)

inline uint32_t batch_size_granularity() { return tcnnb_batch_size_granularity(); }
inline int cuda_device() { return tcnnb_cuda_device(); }
inline void set_cuda_device(int device) { TCNNB_CPP_CHECK(tcnnb_set_cuda_device(device)); }
inline void free_temporary_memory() {}  /* no arenas: nothing is allocated per call */
inline bool has_networks() { return true; }

enum class Precision { Fp32, Fp16 };

inline float default_loss_scale(Precision p) { return p == Precision::Fp16 ? tcnnb_default_loss_scale() : 1.0f; }
inline Precision preferred_precision() { return Precision::Fp16; }
inline bool supports_jit_fusion(int = -1) { return false; }
inline void rtc_set_cache_dir(const std::string&) {}
inline void rtc_set_include_dir(const std::string&) {}
inline void set_log_callback(const std::function<void(LogSeverity, const std::string&)>&) {}

struct Context {
	std::unique_ptr<tcnn::Context> ctx;
};

class Module {
public:
	Module(Precision param_precision, Precision output_precision) : m_param_precision{param_precision}, m_output_precision{output_precision} {}
	virtual ~Module() {}

	virtual void inference(cudaStream_t stream, uint32_t n_elements, const float* input, void* output, void* params) = 0;
	virtual Context forward(cudaStream_t stream, uint32_t n_elements, const float* input, void* output, void* params, bool prepare_input_gradients) = 0;
	virtual void backward(cudaStream_t stream, const Context& ctx, uint32_t n_elements, float* dL_dinput, const void* dL_doutput, void* dL_dparams, const float* input, const void* output, const void* params) = 0;
	virtual void backward_backward_input(cudaStream_t stream, const Context& ctx, uint32_t n_elements, const float* dL_ddLdinput, const float* input, const void* dL_doutput, void* dL_dparams, void* dL_ddLdoutput, float* dL_dinput, const void* params) = 0;

	virtual uint32_t n_input_dims() const = 0;
	virtual uint32_t n_output_dims() const = 0;
	Precision output_precision() const { return m_output_precision; }

	virtual size_t n_params() const = 0;
	Precision param_precision() const { return m_param_precision; }

	virtual void initialize_params(size_t seed, float* params_full_precision, float scale = 1.0f) = 0;

	virtual json hyperparams() const = 0;
	virtual std::string name() const = 0;

	virtual bool jit_fusion() const = 0;
	virtual void set_jit_fusion(bool val) = 0;

private:
	Precision m_param_precision;
	Precision m_output_precision;
};

namespace detail {

inline Context made_forward_pass() {
	Context c;
	c.ctx = std::make_unique<tcnn::Context>();
	return c;
}

/* create_network_with_input_encoding: src/cpp_api.cu:71-158 over tcnnb_module_* */
class NetworkWithInputEncodingModule : public Module {
public:
	NetworkWithInputEncodingModule(uint32_t n_input_dims, uint32_t n_output_dims, const json& encoding, const json& network) : Module{Precision::Fp16, Precision::Fp16} {
		TCNNB_CPP_CHECK(tcnnb_module_create(n_input_dims, n_output_dims, encoding.dump().c_str(), network.dump().c_str(), &m_h));
	}
	~NetworkWithInputEncodingModule() override { tcnnb_destroy(m_h); }
	void inference(cudaStream_t stream, uint32_t n, const float* input, void* output, void* params) override {
		TCNNB_CPP_CHECK(tcnnb_module_inference(m_h, (tcnnb_stream)stream, n, input, output, params));
	}
	Context forward(cudaStream_t stream, uint32_t n, const float* input, void* output, void* params, bool prepare_input_gradients) override {
		TCNNB_CPP_CHECK(tcnnb_module_forward(m_h, (tcnnb_stream)stream, n, input, output, params, prepare_input_gradients ? 1 : 0));
		return made_forward_pass();
	}
	void backward(cudaStream_t stream, const Context&, uint32_t n, float* dL_dinput, const void* dL_doutput, void* dL_dparams, const float* input, const void* output, const void* params) override {
		TCNNB_CPP_CHECK(tcnnb_module_backward(m_h, (tcnnb_stream)stream, n, dL_dinput, dL_doutput, dL_dparams, input, output, params));
	}
	void backward_backward_input(cudaStream_t, const Context&, uint32_t, const float*, const float*, const void*, void*, void*, float*, const void*) override {
		throw std::runtime_error{"tcnn_b200: second-order derivatives (backward_backward_input) are outside the built path"};
	}
	uint32_t n_input_dims() const override { return tcnnb_n_input_dims(m_h); }
	uint32_t n_output_dims() const override { return tcnnb_padded_output_width(m_h); } /* the PADDED width, src/cpp_api.cu:137 */
	size_t n_params() const override { return tcnnb_n_params(m_h); }
	void initialize_params(size_t seed, float* params_full_precision, float scale = 1.0f) override { TCNNB_CPP_CHECK(tcnnb_module_initialize_params(m_h, seed, params_full_precision, scale)); }
	json hyperparams() const override { return json::parse(tcnnb_hyperparams(m_h)); }
	std::string name() const override { return "NetworkWithInputEncoding"; }
	bool jit_fusion() const override { return false; }
	void set_jit_fusion(bool) override {}

private:
	tcnnb_model* m_h = nullptr;
};

/* create_network: src/cpp_api.cu:160-162 (the network behind an Identity encoding) over tcnnb_network_* */
class NetworkModule : public Module {
public:
	NetworkModule(uint32_t n_input_dims, uint32_t n_output_dims, const json& network) : Module{Precision::Fp16, Precision::Fp16}, m_n_in{n_input_dims}, m_config(network) {
		TCNNB_CPP_CHECK(tcnnb_network_create(n_input_dims, n_output_dims, network.dump().c_str(), &m_h));
	}
	~NetworkModule() override { tcnnb_network_destroy(m_h); }
	void inference(cudaStream_t stream, uint32_t n, const float* input, void* output, void* params) override {
		TCNNB_CPP_CHECK(tcnnb_network_module_inference(m_h, (tcnnb_stream)stream, n, input, output, params));
	}
	Context forward(cudaStream_t stream, uint32_t n, const float* input, void* output, void* params, bool) override {
		inference(stream, n, input, output, params);
		return made_forward_pass();
	}
	void backward(cudaStream_t stream, const Context&, uint32_t n, float* dL_dinput, const void* dL_doutput, void* dL_dparams, const float* input, const void*, const void* params) override {
		TCNNB_CPP_CHECK(tcnnb_network_module_backward(m_h, (tcnnb_stream)stream, n, dL_dinput, dL_doutput, dL_dparams, input, params));
	}
	void backward_backward_input(cudaStream_t, const Context&, uint32_t, const float*, const float*, const void*, void*, void*, float*, const void*) override {
		throw std::runtime_error{"tcnn_b200: second-order derivatives (backward_backward_input) are outside the built path"};
	}
	uint32_t n_input_dims() const override { return m_n_in; }
	uint32_t n_output_dims() const override { return tcnnb_network_padded_output_width(m_h); }
	size_t n_params() const override { return tcnnb_network_n_params(m_h); }
	void initialize_params(size_t seed, float* params_full_precision, float scale = 1.0f) override { TCNNB_CPP_CHECK(tcnnb_network_initialize_params(m_h, seed, params_full_precision, scale)); }
	json hyperparams() const override { return {{"encoding", {{"otype", "Identity"}}}, {"network", m_config}}; }
	std::string name() const override { return "NetworkWithInputEncoding"; }
	bool jit_fusion() const override { return false; }
	void set_jit_fusion(bool) override {}

private:
	tcnnb_network* m_h = nullptr;
	uint32_t m_n_in;
	json m_config;
};

/* create_encoding: src/cpp_api.cu:165-174 over tcnnb_encoding_* */
class EncodingModule : public Module {
public:
	EncodingModule(uint32_t n_input_dims, const json& encoding) : Module{Precision::Fp16, Precision::Fp16}, m_config(encoding) {
		TCNNB_CPP_CHECK(tcnnb_encoding_create(n_input_dims, encoding.dump().c_str(), &m_h));
	}
	~EncodingModule() override { tcnnb_encoding_destroy(m_h); }
	void inference(cudaStream_t stream, uint32_t n, const float* input, void* output, void* params) override {
		TCNNB_CPP_CHECK(tcnnb_encoding_forward(m_h, (tcnnb_stream)stream, n, input, output, params));
	}
	Context forward(cudaStream_t stream, uint32_t n, const float* input, void* output, void* params, bool) override {
		inference(stream, n, input, output, params);
		return made_forward_pass();
	}
	void backward(cudaStream_t stream, const Context&, uint32_t n, float* dL_dinput, const void* dL_doutput, void* dL_dparams, const float* input, const void*, const void* params) override {
		TCNNB_CPP_CHECK(tcnnb_encoding_backward(m_h, (tcnnb_stream)stream, n, dL_dinput, dL_doutput, dL_dparams, input, params));
	}
	void backward_backward_input(cudaStream_t stream, const Context&, uint32_t n, const float* dL_ddLdinput, const float* input, const void* dL_doutput, void* dL_dparams, void* dL_ddLdoutput,
	                             float* dL_dinput, const void* params) override {
		TCNNB_CPP_CHECK(tcnnb_encoding_backward_backward_input(m_h, (tcnnb_stream)stream, n, dL_ddLdinput, input, dL_doutput, dL_dparams, dL_ddLdoutput, dL_dinput, params));
	}
	uint32_t n_input_dims() const override { return tcnnb_encoding_n_input_dims(m_h); }
	uint32_t n_output_dims() const override { return tcnnb_encoding_n_output_dims(m_h); }
	size_t n_params() const override { return tcnnb_encoding_n_params(m_h); }
	void initialize_params(size_t seed, float* params_full_precision, float scale = 1.0f) override { TCNNB_CPP_CHECK(tcnnb_encoding_initialize_params(m_h, seed, params_full_precision, scale)); }
	json hyperparams() const override { return m_config; }
	std::string name() const override { return "GridEncoding"; }
	bool jit_fusion() const override { return false; }
	void set_jit_fusion(bool) override {}

private:
	tcnnb_encoding* m_h = nullptr;
	json m_config;
};

}  // namespace detail

/* Owning raw pointers: the caller deletes (bindings.cpp:267,271-282 wrap them in unique_ptr). */
inline Module* create_network_with_input_encoding(uint32_t n_input_dims, uint32_t n_output_dims, const json& encoding, const json& network) {
	return new detail::NetworkWithInputEncodingModule{n_input_dims, n_output_dims, encoding, network};
}
inline Module* create_network(uint32_t n_input_dims, uint32_t n_output_dims, const json& network) { return new detail::NetworkModule{n_input_dims, n_output_dims, network}; }
inline Module* create_encoding(uint32_t n_input_dims, const json& encoding, Precision requested_precision) {
	if (requested_precision == Precision::Fp32) throw std::runtime_error{"tcnn_b200 mirrors the half-precision build of the reference: create_encoding with Precision::Fp32 is not built"};
	return new detail::EncodingModule{n_input_dims, encoding};
}

}}  // namespace tcnn::cpp
