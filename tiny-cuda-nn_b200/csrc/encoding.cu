// encoding.cu -- the stand-alone encoding tier of the C ABI (include/tcnn_b200.h, tcnnb_encoding_*).
//
// Mirrors tcnn::cpp::create_encoding (cpp_api.h:124, src/cpp_api.cu:165-174: a DifferentiableObject<__half> around
// create_encoding<__half>(n_input_dims, json, alignment 0)), i.e. what the PyTorch extension's tcnn.Encoding binds
// (bindings.cpp:284-343), for "Grid" / "HashGrid" / "TiledGrid" / "DenseGrid", "Identity", "Frequency", "TriangleWave", "OneBlob",
// "SphericalHarmonics", "Empty", "Composite" of those with the Concatenation / Sum / Product reductions and "NRC" / "OneBlobFrequency"
// (src/encoding.cu:60-120):
//   forward / inference   fp32 inputs [n][n_input_dims] -> fp16 features [n][n_output_dims]
//   backward              dL_dparams (fp16, OVERWRITTEN; grids only) and / or dL_dinput fp32 from dL_doutput
//   backward_backward_input  second-order derivatives of a single grid (grid.h:910-1042, grid_bwd_bwd.cu); every other
//                         encoding throws "<name> does not support double backward." as the reference (object.h:468-482)
//   initialize_params     grids: U(-1e-4, 1e-4) * scale from pcg32{seed}, nested encodings one after the other (grid.h:1076-1079)
// The configuration is resolved into a segment table (encoding_plan.h); grids run grid_kernels.cu, everything else
// feature_encodings.cu. Parameters are CALLER-owned. Only the fp16 build of the reference is mirrored (Precision::Fp32 is rejected).
#include "../../include/tcnn_b200.h"

#include "encoding_plan.h"
#include "grid_config.h"
#include "grid_kernels.h"
#include "host_common.h"
#include "json_mini.h"

#include <memory>
#include <vector>

namespace tcnnb {

struct Encoding {
	EncodingPlan plan;
	float max_level = 1.0f;
	uint32_t max_align = 2;             // strictest pointer alignment the kernels need for feature rows / parameters (bytes)
};

static void build_encoding(Encoding& e, uint32_t n_input_dims, const json::Value& cfg) {
	require_sm90();
	build_encoding_plan(e.plan, n_input_dims, cfg, 0);
	for (auto& g : e.plan.grids) {
		e.max_align = std::max(e.max_align, 2 * g->cfg.n_features_per_level);
		// feature rows are read / written with one vector access per level: every row has to start on that boundary
		if (e.plan.width % g->cfg.n_features_per_level != 0) throw std::runtime_error("tcnn_b200: the total width of this Composite encoding must be a multiple of the grid's n_features_per_level");
	}
}

static void check_ptr(const void* p, const char* what, size_t align) {
	if (!p) throw std::runtime_error(std::string("encoding: ") + what + " is null.");
	if ((uintptr_t)p % align != 0) throw std::runtime_error(std::string("encoding: ") + what + " must be " + std::to_string(align) + "-byte aligned.");
}

}  // namespace tcnnb

using namespace tcnnb;

struct tcnnb_encoding {
	Encoding impl;
};

extern "C" {

int tcnnb_encoding_create(uint32_t n_input_dims, const char* encoding_json, tcnnb_encoding** out) {
	TCNNB_API_BEGIN
	if (!out) throw std::runtime_error("tcnnb_encoding_create: out is null");
	*out = nullptr;
	auto e = std::make_unique<tcnnb_encoding>();
	build_encoding(e->impl, n_input_dims, json::parse(encoding_json ? encoding_json : "{}"));
	*out = e.release();
	TCNNB_API_END
}

void tcnnb_encoding_destroy(tcnnb_encoding* e) { delete e; }
uint64_t tcnnb_encoding_n_params(const tcnnb_encoding* e) { return e->impl.plan.n_params; }
uint32_t tcnnb_encoding_n_input_dims(const tcnnb_encoding* e) { return e->impl.plan.n_in; }
uint32_t tcnnb_encoding_n_output_dims(const tcnnb_encoding* e) { return e->impl.plan.width; }

// Level table of the (first) grid of the encoding; n_levels = 0 when there is none.
int tcnnb_encoding_grid_levels(const tcnnb_encoding* e, uint32_t* n_levels, uint32_t* offsets, float* scales, uint32_t* resolutions) {
	TCNNB_API_BEGIN
	const EncodingPlan& plan = e->impl.plan;
	write_level_table(plan.grids.empty() ? nullptr : &plan.grids.front()->cfg, n_levels, offsets, scales, resolutions);
	TCNNB_API_END
}

int tcnnb_encoding_set_max_level(tcnnb_encoding* e, float max_level) {
	TCNNB_API_BEGIN
	e->impl.max_level = max_level;  // GridEncoding::set_max_level: fraction of the levels that is active
	TCNNB_API_END
}

int tcnnb_encoding_initialize_params(tcnnb_encoding* e, uint64_t seed, float* params_full_precision_dev, float scale) {
	TCNNB_API_BEGIN
	if (e->impl.plan.n_params == 0) return 0;
	if (!params_full_precision_dev) throw std::runtime_error("encoding: params_full_precision is null.");
	HostPcg32 rng{seed};
	init_plan_params(e->impl.plan, rng, params_full_precision_dev, scale);
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	TCNNB_API_END
}

int tcnnb_encoding_forward(tcnnb_encoding* e, tcnnb_stream stream, uint32_t n_elements, const float* input_dev, void* output_dev, const void* params_dev) {
	TCNNB_API_BEGIN
	Encoding& enc = e->impl;
	check_batch(n_elements);
	check_ptr(input_dev, "input", 4);
	check_ptr(output_dev, "output", enc.max_align);
	if (enc.plan.n_params) check_ptr(params_dev, "params", enc.max_align);
	plan_forward(enc.plan, (cudaStream_t)stream, n_elements, input_dev, (const __half*)params_dev, (__half*)output_dev, enc.plan.width, enc.max_level);
	TCNNB_API_END
}

int tcnnb_encoding_backward(tcnnb_encoding* e, tcnnb_stream stream, uint32_t n_elements, float* dL_dinput_dev, const void* dL_doutput_dev, void* dL_dparams_dev, const float* input_dev,
                            const void* params_dev) {
	TCNNB_API_BEGIN
	Encoding& enc = e->impl;
	EncodingPlan& plan = enc.plan;
	check_batch(n_elements);
	check_ptr(input_dev, "input", 4);
	check_ptr(dL_doutput_dev, "dL_doutput", enc.max_align);
	if (dL_dparams_dev && plan.n_params) check_ptr(dL_dparams_dev, "dL_dparams", enc.max_align);
	// a Product recomputes the nested outputs from (input, params): nothing of an earlier forward call is read
	if ((dL_dinput_dev || (dL_dparams_dev && plan.reduction == REDUCE_PRODUCT)) && !plan.grids.empty()) check_ptr(params_dev, "params", enc.max_align);
	// GradientMode::Overwrite (src/cpp_api.cu:115)
	plan_backward(plan, (cudaStream_t)stream, n_elements, input_dev, (const __half*)params_dev, (const __half*)dL_doutput_dev, plan.width, (__half*)dL_dparams_dev, dL_dinput_dev,
	              enc.max_level);
	TCNNB_API_END
}

int tcnnb_encoding_backward_backward_input(tcnnb_encoding* e, tcnnb_stream stream, uint32_t n_elements, const float* dL_ddLdinput_dev, const float* input_dev,
                                           const void* dL_doutput_dev, void* dL_dparams_dev, void* dL_ddLdoutput_dev, float* dL_dinput_dev, const void* params_dev) {
	TCNNB_API_BEGIN
	Encoding& enc = e->impl;
	EncodingPlan& plan = enc.plan;
	check_batch(n_elements);
	check_ptr(input_dev, "input", 4);
	check_ptr(dL_ddLdinput_dev, "dL_ddLdinput", 4);
	if (dL_dparams_dev || dL_dinput_dev) check_ptr(dL_doutput_dev, "dL_doutput", enc.max_align);
	if (dL_dparams_dev && plan.n_params) check_ptr(dL_dparams_dev, "dL_dparams", enc.max_align);
	if (dL_ddLdoutput_dev) check_ptr(dL_ddLdoutput_dev, "dL_ddLdoutput", enc.max_align);
	if (dL_dinput_dev) check_ptr(dL_dinput_dev, "dL_dinput", 4);
	if ((dL_ddLdoutput_dev || dL_dinput_dev) && plan.n_params) check_ptr(params_dev, "params", enc.max_align);
	plan_backward_backward_input(plan, (cudaStream_t)stream, n_elements, input_dev, (const __half*)params_dev, (const __half*)dL_doutput_dev, plan.width, dL_ddLdinput_dev,
	                             (__half*)dL_dparams_dev, (__half*)dL_ddLdoutput_dev, dL_dinput_dev, enc.max_level);
	TCNNB_API_END
}

}  // extern "C"
