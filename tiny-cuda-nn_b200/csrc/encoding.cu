// encoding.cu -- the stand-alone encoding tier of the C ABI (include/tcnn_b200.h, tcnnb_encoding_*).
//
// Mirrors tcnn::cpp::create_encoding (cpp_api.h:124, src/cpp_api.cu:165-174: a DifferentiableObject<__half> around
// create_encoding<__half>(n_input_dims, json, alignment 0)), i.e. what the PyTorch extension's tcnn.Encoding binds
// (bindings.cpp:284-343), for "Grid" / "HashGrid" / "TiledGrid" / "DenseGrid", "Identity", "Frequency", "TriangleWave", "OneBlob",
// "SphericalHarmonics" and "Composite" of those (src/encoding.cu:60-120):
//   forward / inference   fp32 inputs [n][n_input_dims] -> fp16 features [n][n_output_dims]
//   backward              dL_dparams (fp16, OVERWRITTEN; grids only) and / or dL_dinput fp32 from dL_doutput
//   initialize_params     grids: U(-1e-4, 1e-4) * scale from pcg32{seed}, nested encodings one after the other (grid.h:1076-1079)
// The configuration is resolved into a segment table (encoding_plan.h); grids run grid_kernels.cu, everything else
// feature_encodings.cu. Parameters are CALLER-owned. Only the fp16 build of the reference is mirrored (Precision::Fp32 is rejected).
#include "../../include/tcnn_b200.h"

#include "encoding_plan.h"
#include "grid_config.h"
#include "grid_kernels.h"
#include "host_common.h"
#include "json_mini.h"
#include "misc_kernels.h"

#include <memory>
#include <vector>

namespace tcnnb {

struct Encoding {
	EncodingPlan plan;
	DeviceBuffer<float> scratch;        // level scales; fp32 gradient accumulator when F == 1
	DeviceBuffer<__half> replicas;      // private copies of the coarse levels' gradients (grid_kernels.h plan_grid_scatter)
	float max_level = 1.0f;
	std::string hyperparams_json;
	uint32_t max_align = 2;             // strictest pointer alignment the kernels need for feature rows / parameters (bytes)
};

static void build_encoding(Encoding& e, uint32_t n_input_dims, const json::Value& cfg) {
	int device = 0;
	TCNNB_CUDA_CHECK(cudaGetDevice(&device));
	cudaDeviceProp prop;
	TCNNB_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
	if (prop.major != 9) throw std::runtime_error("tcnn_b200 requires an sm_90-class GPU (H100); found compute capability " + std::to_string(prop.major) + "." + std::to_string(prop.minor));
	e.scratch.resize(128);
	build_encoding_plan(e.plan, n_input_dims, cfg, 0, e.scratch.ptr);
	for (auto& g : e.plan.grids) {
		e.max_align = std::max(e.max_align, 2 * g->cfg.n_features_per_level);
		// feature rows are read / written with one vector access per level: every row has to start on that boundary
		if (e.plan.width % g->cfg.n_features_per_level != 0) throw std::runtime_error("tcnn_b200: the total width of this Composite encoding must be a multiple of the grid's n_features_per_level");
	}
}

static void check_n(uint32_t n) {
	if (n == 0 || n % BATCH_GRANULARITY != 0) throw std::runtime_error("batch size " + std::to_string(n) + " must be a non-zero multiple of " + std::to_string(BATCH_GRANULARITY));
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
	if (e->impl.plan.grids.empty()) {
		if (n_levels) *n_levels = 0;
		if (offsets) offsets[0] = 0;
		return 0;
	}
	const GridConfig& g = e->impl.plan.grids.front()->cfg;
	if (n_levels) *n_levels = g.n_levels;
	for (uint32_t l = 0; l < g.n_levels; ++l) {
		if (offsets) offsets[l] = g.offsets[l];
		if (scales) scales[l] = g.scales[l];
		if (resolutions) resolutions[l] = (uint32_t)ceilf(g.scales[l]) + 1;
	}
	if (offsets) offsets[g.n_levels] = g.offsets[g.n_levels];
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
	for (auto& g : e->impl.plan.grids) {
		TCNNB_CUDA_CHECK(launch_random_uniform(nullptr, rng.device(), g->cfg.n_params, params_full_precision_dev + g->param_offset, -1e-4f * scale, 1e-4f * scale));
		++g_kernel_launches;
		rng.advance(g->cfg.n_params);
	}
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	TCNNB_API_END
}

int tcnnb_encoding_forward(tcnnb_encoding* e, tcnnb_stream stream, uint32_t n_elements, const float* input_dev, void* output_dev, const void* params_dev) {
	TCNNB_API_BEGIN
	Encoding& enc = e->impl;
	const EncodingPlan& plan = enc.plan;
	check_n(n_elements);
	check_ptr(input_dev, "input", 4);
	check_ptr(output_dev, "output", enc.max_align);
	if (plan.n_params) check_ptr(params_dev, "params", enc.max_align);
	cudaStream_t s = (cudaStream_t)stream;
	if (plan.has_plain_features()) {
		TCNNB_CUDA_CHECK(launch_feature_forward(s, plan.segs, n_elements, input_dev, plan.n_in, (__half*)output_dev, plan.width));
		++g_kernel_launches;
	}
	for (auto& g : plan.grids) {
		const FeatureSegment& sg = plan.segs.s[g->segment];
		GridKernelArgs a = plan_grid_args(*g, n_elements, input_dev + sg.in_begin, plan.n_in, plan.width, enc.max_level);
		a.pad_cols = sg.n_pad;
		TCNNB_CUDA_CHECK(launch_grid_forward(s, a, (const __half*)params_dev + g->param_offset, (__half*)output_dev + sg.out_begin));
		++g_kernel_launches;
	}
	TCNNB_API_END
}

int tcnnb_encoding_backward(tcnnb_encoding* e, tcnnb_stream stream, uint32_t n_elements, float* dL_dinput_dev, const void* dL_doutput_dev, void* dL_dparams_dev, const float* input_dev,
                            const void* params_dev) {
	TCNNB_API_BEGIN
	Encoding& enc = e->impl;
	const EncodingPlan& plan = enc.plan;
	check_n(n_elements);
	check_ptr(input_dev, "input", 4);
	check_ptr(dL_doutput_dev, "dL_doutput", enc.max_align);
	cudaStream_t s = (cudaStream_t)stream;
	const __half* dy = (const __half*)dL_doutput_dev;
	if (dL_dparams_dev && plan.n_params) {  // GradientMode::Overwrite (src/cpp_api.cu:115)
		check_ptr(dL_dparams_dev, "dL_dparams", enc.max_align);
		TCNNB_CUDA_CHECK(cudaMemsetAsync(dL_dparams_dev, 0, sizeof(__half) * plan.n_params, s));
		for (auto& g : plan.grids) {
			const FeatureSegment& sg = plan.segs.s[g->segment];
			const uint32_t F = g->cfg.n_features_per_level;
			GridKernelArgs a = plan_grid_args(*g, n_elements, input_dev + sg.in_begin, plan.n_in, plan.width, enc.max_level);
			if (enc.max_level >= 1.0f) {  // contended coarse levels scatter into private copies
				const GridScatterPlan sp = plan_grid_scatter(g->levels.data(), g->cfg.n_levels, F, g->cfg.n_pos_dims, n_elements);
				if (sp.n_replicas > 1) {
					if (enc.replicas.n < sp.scratch_halfs) {
						enc.replicas.resize(sp.scratch_halfs);
						enc.replicas.zero(s);
					}
					a.replica_scratch = enc.replicas.ptr;
					a.n_replicas = sp.n_replicas;
					a.replica_entries = sp.replica_entries;
				}
			}
			float* tmp = nullptr;
			if (F == 1) {
				enc.scratch.resize(std::max<size_t>(enc.scratch.n, g->cfg.n_params));
				tmp = enc.scratch.ptr;
				TCNNB_CUDA_CHECK(cudaMemsetAsync(tmp, 0, sizeof(float) * g->cfg.n_params, s));
			}
			TCNNB_CUDA_CHECK(launch_grid_backward(s, a, dy + sg.out_begin, (__half*)dL_dparams_dev + g->param_offset, tmp, g->cfg.n_params));
			g_kernel_launches += F == 1 ? 2 : 1;
		}
	}
	if (dL_dinput_dev) {
		if (plan.composite) TCNNB_CUDA_CHECK(cudaMemsetAsync(dL_dinput_dev, 0, sizeof(float) * (size_t)n_elements * plan.n_in, s));
		if (plan.has_plain_features()) {
			TCNNB_CUDA_CHECK(launch_feature_input_gradient(s, plan.segs, n_elements, input_dev, plan.n_in, dy, plan.width, dL_dinput_dev));
			++g_kernel_launches;
		}
		for (auto& g : plan.grids) {
			const FeatureSegment& sg = plan.segs.s[g->segment];
			check_ptr(params_dev, "params", enc.max_align);
			const GridKernelArgs a = plan_grid_args(*g, n_elements, input_dev + sg.in_begin, plan.n_in, plan.width, enc.max_level);
			TCNNB_CUDA_CHECK(launch_grid_input_gradient(s, a, (const __half*)params_dev + g->param_offset, dy + sg.out_begin, dL_dinput_dev + sg.in_begin));
			++g_kernel_launches;
		}
	}
	TCNNB_API_END
}

}  // extern "C"
