// encoding_plan.h -- an encoding configuration (src/encoding.cu:60-150) resolved into a table of segments: which input dimensions each
// (nested) encoding reads, which output columns it writes, how it is padded, where its parameters live. Shared by the general path of
// the model (model.cu) and the encoding tier (encoding.cu), which both run it with the plan operations below (encoding_plan.cu).
//
// Composite (encodings/composite.h:135-215): "nested" array, each entry with "n_dims_to_encode" (one entry may leave it out and takes
// the remaining dimensions); outputs are concatenated; every nested encoding but the last is padded so that the NEXT one starts at a
// multiple of its required alignment (grids: n_features_per_level, everything else 1), the last one takes the padding up to the
// alignment the consumer asks for (16 in front of a network). Padding columns hold ONE (zero behind a grid); SphericalHarmonics puts its
// padding IN FRONT of its coefficients (spherical_harmonics.h:56-60). Parameters of nested encodings are concatenated in order.
//
// "reduction" (composite.h:47-133, 189-211; matched case-insensitively): Concatenation, or Sum / Product of the nested outputs. Under
// a reduction every nested encoding is padded to the same width w (the lcm a of the nested alignments, then lcm(a, consumer alignment)),
// each with its own padding values, and the segment table describes the UNREDUCED rows [n][K w] (segment k at column k w) that the
// nested encodings fill in the plan's scratch; a reduce kernel (composite_kernels.cu) then sums / multiplies the K slabs column by
// column in fp32, in nested order. "dims_to_encode_begin" (composite.h:147-186) sets the input offset of a nested encoding that also
// has "n_dims_to_encode"; ranges may overlap and come in any order, and the input gradients of overlapping ranges are SUMMED (the
// reference overwrites them from concurrent streams, so its value there is order-dependent). Empty (encodings/empty.h): no output
// columns, ONE in its padding columns, zero input gradient. "NRC" / "OneBlobFrequency" (src/encoding.cu:93-115) expands to
// Composite{TriangleWave on 3 dims, OneBlob on 5 dims, Identity on the rest}.
// Not built: nested Composite, stochastic_interpolation.
#pragma once
#include "feature_encodings.h"
#include "grid_config.h"
#include "grid_kernels.h"
#include "host_common.h"
#include "json_mini.h"

#include <memory>
#include <numeric>
#include <vector>

namespace tcnnb {

enum Reduction : uint32_t { REDUCE_CONCATENATION = 0, REDUCE_SUM = 1, REDUCE_PRODUCT = 2 };

struct EncodingPlan {
	struct Grid {
		GridConfig cfg;
		uint32_t segment = 0;       // index into segs
		size_t param_offset = 0;    // first parameter of this grid inside the encoding's parameter vector
		std::vector<LevelInfo> levels;
		DeviceBuffer<LevelInfo> levels_dev;
	};
	uint32_t n_in = 0;
	uint32_t width = 0;             // padded output width
	uint32_t n_features = 0;        // output width without the final alignment padding
	size_t n_params = 0;
	bool composite = false;
	uint32_t reduction = REDUCE_CONCATENATION;  // Sum / Product: every segment is `width` columns wide, segment k at column k * width
	bool overlap = false;           // two nested encodings read one input dimension: their input gradients are summed
	bool zero_dx = false;           // some input dimensions may have no reader: dL/dx is zeroed before the segments write theirs
	FeatureSegments segs{};
	std::vector<std::unique_ptr<Grid>> grids;
	// scratch of the table-gradient scatter (plan_param_gradients), grown on demand
	DeviceBuffer<float> grad_fp32;     // n_features_per_level == 1: fp32 scatter target (grid.h:858-894)
	DeviceBuffer<__half> replicas;     // private copies of the coarse levels' gradients (grid_kernels.h plan_grid_scatter); zero between uses
	// scratch of the reductions and of overlapping input ranges, grown on demand
	DeviceBuffer<__half> nested_out;   // Sum / Product: the nested encodings' outputs, rows [n][segs.n * width]
	DeviceBuffer<__half> dL_dnested;   // Product: dL/d(nested outputs), same rows
	DeviceBuffer<float> dx_slabs;      // overlapping ranges: each segment's input gradient, [segs.n][n][n_in]
	bool reduced() const { return reduction != REDUCE_CONCATENATION; }
	bool has_plain_features() const {
		for (uint32_t i = 0; i < segs.n; ++i) if (segs.s[i].type != FEAT_GRID) return true;
		return false;
	}
};

namespace plan_detail {

inline bool is_grid_otype(const std::string& lower) { return lower == "grid" || lower == "hashgrid" || lower == "tiledgrid" || lower == "densegrid"; }

// One nested (or top-level) encoding over `n_dims` input dimensions -> segment (out_begin / n_pad filled in by the caller).
inline void add_segment(EncodingPlan& plan, uint32_t in_begin, uint32_t n_dims, const json::Value& e) {
	if (plan.segs.n >= MAX_FEATURE_SEGMENTS) throw std::runtime_error("tcnn_b200: a Composite encoding may nest at most 8 encodings");
	const std::string otype = e.value("otype", "OneBlob");  // src/encoding.cu:133
	const std::string lower = to_lower(otype);
	FeatureSegment sg{};
	sg.in_begin = in_begin;
	sg.n_in = n_dims;
	sg.scale = 1.0f;
	if (is_grid_otype(lower)) {
		auto g = std::make_unique<EncodingPlan::Grid>();
		g->cfg = parse_grid(n_dims, e);
		if (g->cfg.stochastic_interpolation) throw std::runtime_error("tcnn_b200: stochastic_interpolation is not built");
		g->segment = plan.segs.n;
		sg.type = FEAT_GRID;
		sg.n_out = g->cfg.n_levels * g->cfg.n_features_per_level;
		sg.param = g->cfg.n_features_per_level;
		plan.grids.push_back(std::move(g));
	} else if (lower == "identity") {
		sg.type = FEAT_IDENTITY;
		sg.n_out = n_dims;
		sg.scale = (float)e.value("scale", 1.0);
		sg.offset = (float)e.value("offset", 0.0);
	} else if (lower == "frequency") {
		sg.type = FEAT_FREQUENCY;
		sg.param = (uint32_t)e.value("n_frequencies", 12.0);
		sg.n_out = n_dims * sg.param * 2;
	} else if (lower == "trianglewave") {
		sg.type = FEAT_TRIANGLE_WAVE;
		sg.param = (uint32_t)e.value("n_frequencies", 12.0);
		sg.n_out = n_dims * sg.param;
	} else if (lower == "oneblob") {
		const uint32_t n_bins = (uint32_t)e.value("n_bins", 16.0);
		if (n_bins == 0 || (n_bins & (n_bins - 1)) != 0) throw std::runtime_error("Number of bins must be a power of 2");  // oneblob.h:170-172
		sg.type = FEAT_ONEBLOB;
		uint32_t log2_bins = 0;
		while ((1u << log2_bins) < n_bins) ++log2_bins;
		sg.param = log2_bins;
		sg.n_out = n_dims * n_bins;
	} else if (lower == "sphericalharmonics") {
		sg.type = FEAT_SPHERICAL_HARMONICS;
		sg.param = (uint32_t)e.value("degree", 4.0);
		if (n_dims != 3) throw std::runtime_error("Can only encode 3D directions in spherical harmonics.");  // spherical_harmonics.h:109-111
		if (sg.param == 0) throw std::runtime_error("Spherical harmonics must have positive degree.");
		if (sg.param > 8) throw std::runtime_error("Spherical harmonics are only implemented up to degree 8.");
		sg.n_out = sg.param * sg.param;
	} else if (lower == "empty") {
		sg.type = FEAT_EMPTY;
		sg.n_out = 0;
	} else if (lower == "composite" || lower == "oneblobfrequency" || lower == "nrc") {
		throw std::runtime_error("Encoding '" + otype + "' nested inside a Composite is not built in tcnn_b200");
	} else {
		throw std::runtime_error("Encoding '" + otype + "' not found");
	}
	plan.segs.s[plan.segs.n++] = sg;
}

inline uint32_t required_alignment(const EncodingPlan& plan, uint32_t seg) { return plan.segs.s[seg].type == FEAT_GRID ? plan.segs.s[seg].param : 1u; }

// Concatenation: output columns and padding of each segment
inline void layout_concatenation(EncodingPlan& plan, uint32_t alignment) {
	uint32_t so_far = 0;
	for (uint32_t i = 0; i < plan.segs.n; ++i) {
		FeatureSegment& sg = plan.segs.s[i];
		sg.out_begin = so_far;
		uint32_t padded = sg.n_out;
		if (i + 1 < plan.segs.n) {
			const uint32_t a = required_alignment(plan, i + 1);
			padded = next_multiple(so_far + sg.n_out, a) - so_far;
		} else {
			plan.n_features = so_far + sg.n_out;
			uint32_t a = alignment ? alignment : 1u;
			// lcm(alignment, own requirement): both are powers of two here
			const uint32_t own = required_alignment(plan, i);
			while (a % own != 0) a *= 2;
			padded = next_multiple(so_far + sg.n_out, a) - so_far;
		}
		sg.n_pad = padded - sg.n_out;
		so_far += padded;
	}
	plan.width = so_far;
	if (plan.width == 0 && alignment) {  // nothing but Empty: a network still reads `alignment` columns (of ones, empty.h:76-88)
		plan.segs.s[plan.segs.n - 1].n_pad = alignment;
		plan.width = alignment;
	}
}

}  // namespace plan_detail

// `alignment`: what the consumer needs the padded width to be a multiple of (16 in front of a network, 1 for cpp::create_encoding).
inline void build_encoding_plan(EncodingPlan& plan, uint32_t n_in, const json::Value& cfg, uint32_t alignment) {
	using namespace plan_detail;
	plan.n_in = n_in;
	const std::string lower = to_lower(cfg.value("otype", "OneBlob"));
	json::Value nrc;
	const json::Value* ccfg = &cfg;
	if (lower == "nrc" || lower == "oneblobfrequency") {  // src/encoding.cu:93-115
		const uint32_t n_frequencies = (uint32_t)cfg.value("n_frequencies", 12.0), n_bins = (uint32_t)cfg.value("n_bins", 4.0);
		nrc = json::parse("{\"otype\": \"Composite\", \"nested\": [{\"n_dims_to_encode\": 3, \"otype\": \"TriangleWave\", \"n_frequencies\": " + std::to_string(n_frequencies) +
		                  "}, {\"n_dims_to_encode\": 5, \"otype\": \"OneBlob\", \"n_bins\": " + std::to_string(n_bins) + "}, {\"otype\": \"Identity\"}]}");
		ccfg = &nrc;
	}
	if (lower == "composite" || ccfg == &nrc) {
		plan.composite = true;
		const json::Value* nested = ccfg->find("nested");
		if (!nested || nested->type != json::Value::Array) throw std::runtime_error("Must provide an array of nested encodings to CompositeEncoding.");
		const std::string reduction = ccfg->value("reduction", "Concatenation");  // common_host.cu:181-191
		const std::string red = to_lower(reduction);
		if (red == "sum") plan.reduction = REDUCE_SUM;
		else if (red == "product") plan.reduction = REDUCE_PRODUCT;
		else if (red != "concatenation") throw std::runtime_error("Invalid reduction type: " + reduction);
		uint32_t total = 0;
		uint32_t n_unspecified = 0;
		bool any_begin = false;  // then the total is not checked, and every nested encoding must give its n_dims_to_encode (composite.h:147-178)
		for (auto& e : nested->arr) {
			if (e.contains("n_dims_to_encode")) total += (uint32_t)e.value("n_dims_to_encode", 0.0);
			else ++n_unspecified;
			any_begin = any_begin || e.contains("dims_to_encode_begin");
		}
		if (!any_begin && total > n_in) throw std::runtime_error("CompositeEncoding: nested encodings must not encode more dims " + std::to_string(total) + " than composite " + std::to_string(n_in));
		if (n_unspecified > (any_begin ? 0u : 1u)) throw std::runtime_error("CompositeEncoding: may only leave 'n_dims_to_encode' unspecified for a single nested encoding");
		uint32_t offset = 0;
		for (auto& e : nested->arr) {
			const uint32_t dims = e.contains("n_dims_to_encode") ? (uint32_t)e.value("n_dims_to_encode", 0.0) : n_in - total;
			if (e.contains("n_dims_to_encode") && e.contains("dims_to_encode_begin")) offset = (uint32_t)e.value("dims_to_encode_begin", 0.0);
			// the reference reads past the input rows here; an explicit error instead
			if ((uint64_t)offset + dims > n_in)
				throw std::runtime_error("CompositeEncoding: nested encoding reads input dims [" + std::to_string(offset) + ", " + std::to_string(offset + dims) + ") of a composite over " +
				                         std::to_string(n_in));
			if (dims > 0) add_segment(plan, offset, dims, e);
			offset += dims;
		}
		if (plan.segs.n == 0) throw std::runtime_error("tcnn_b200: Composite encoding without any nested encoding");
	} else {
		add_segment(plan, 0, n_in, cfg);
	}
	// which input dimensions are read, and by how many nested encodings
	std::vector<uint32_t> readers(n_in, 0);
	for (uint32_t i = 0; i < plan.segs.n; ++i) {
		const FeatureSegment& sg = plan.segs.s[i];
		if (sg.type == FEAT_EMPTY) plan.zero_dx = true;
		else for (uint32_t d = sg.in_begin; d < sg.in_begin + sg.n_in; ++d) plan.overlap = plan.overlap || ++readers[d] > 1;
	}
	plan.zero_dx = plan.zero_dx || plan.composite;
	if (plan.reduced()) {
		// composite.h:199-211: every nested encoding padded to a multiple of the lcm of their alignments; those widths must agree; the
		// consumer's alignment then re-pads all of them (encoding.h:70-72)
		uint32_t a = 1;
		for (uint32_t i = 0; i < plan.segs.n; ++i) a = std::lcm(a, required_alignment(plan, i));
		const uint32_t w = next_multiple(plan.segs.s[0].n_out, a);
		for (uint32_t i = 1; i < plan.segs.n; ++i) {
			if (next_multiple(plan.segs.s[i].n_out, a) != w) {
				std::string widths;
				for (uint32_t j = 0; j < plan.segs.n; ++j) widths += (j ? ", " : "") + std::to_string(next_multiple(plan.segs.s[j].n_out, a));
				throw std::runtime_error(std::string("CompositeEncoding: the nested encodings of a ") + (plan.reduction == REDUCE_SUM ? "Sum" : "Product") + " reduction must have equal output widths, got " + widths);
			}
		}
		plan.n_features = w;
		plan.width = next_multiple(w, std::lcm(alignment ? alignment : 1u, a));
		if (plan.width == 0) plan.width = alignment;  // nothing but Empty: a network still reads `alignment` columns (of ones)
		for (uint32_t i = 0; i < plan.segs.n; ++i) {
			plan.segs.s[i].out_begin = i * plan.width;
			plan.segs.s[i].n_pad = plan.width - plan.segs.s[i].n_out;
		}
	} else {
		layout_concatenation(plan, alignment);
	}
	// grids: parameters, device-evaluated level scales, level tables
	size_t param_offset = 0;
	for (auto& g : plan.grids) {
		g->param_offset = param_offset;
		param_offset += g->cfg.n_params;
		g->cfg.padded_width = g->cfg.n_levels * g->cfg.n_features_per_level;
		evaluate_level_scales(g->cfg);
		g->levels.resize(g->cfg.n_levels);
		for (uint32_t l = 0; l < g->cfg.n_levels; ++l) g->levels[l] = make_level_info(g->cfg, l);
		g->levels_dev.resize(g->levels.size());
		TCNNB_CUDA_CHECK(cudaMemcpy(g->levels_dev.ptr, g->levels.data(), sizeof(LevelInfo) * g->levels.size(), cudaMemcpyHostToDevice));
	}
	plan.n_params = param_offset;
}


// Kernel arguments of grid `g` of the plan for rows of `n` samples: positions rows [n][x_stride], feature rows [n][row_stride]
// (pointers already advanced to the grid's own input / output columns by the caller).
inline GridKernelArgs plan_grid_args(const EncodingPlan::Grid& g, uint32_t n, const float* x_cols, uint32_t x_stride, uint32_t row_stride, float max_level = 1.0f) {
	GridKernelArgs a{};
	a.n_pos_dims = g.cfg.n_pos_dims;
	a.n_features_per_level = g.cfg.n_features_per_level;
	a.n_levels = g.cfg.n_levels;
	a.interpolation = g.cfg.interpolation;
	a.max_level = max_level;
	a.levels_dev = g.levels_dev.ptr;
	a.n_elements = n;
	a.positions = x_cols;
	a.pos_stride = x_stride;
	a.row_stride = row_stride;
	return a;
}

// ---- running a plan (encoding_plan.cu). Positions are rows [n][plan.n_in] fp32; encoded features and dL/d(encoded) are fp16 rows
// [n][row_stride] whose first plan.width columns belong to the plan; `params` / `dL_dparams` hold the plan's own n_params entries.
// `max_level`: fraction of the grid levels that is active (GridEncoding::set_max_level); 1 = all. Each adds the kernels it
// launches to g_kernel_launches.

// encoded = features of the n samples (padding columns included). Sum / Product: the nested encodings fill plan.nested_out, then the
// reduce kernel writes `encoded`.
void plan_forward(EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const __half* params, __half* encoded, uint32_t row_stride, float max_level);
// Backward pass of the plan from dL/d(encoded); each non-null result is OVERWRITTEN:
//   dL_dparams (GradientMode::Overwrite) = the grids' table gradients. Contended coarse levels scatter into private copies when
//   max_level >= 1.
//   dL_dx [n][plan.n_in] fp32 = dL/d(encoded) contracted with d(encoded)/d(position), summed over the nested encodings that read a
//   dimension, zero where none does.
// Sum hands every nested encoding dL/d(encoded) itself. Product needs the nested outputs: they are recomputed from (x, params) unless
// `nested_out_ready` says that plan.nested_out holds them already (the plan_forward of the same samples and parameters just ran on
// this stream, as in one training step), then its backward kernel writes dL/d(nested) to plan.dL_dnested.
void plan_backward(EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const __half* params, const __half* dL_dencoded, uint32_t row_stride, __half* dL_dparams,
                   float* dL_dx, float max_level, bool nested_out_ready = false);
// plan_backward for one of the two results
void plan_param_gradients(EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const __half* params, const __half* dL_dencoded, uint32_t row_stride,
                          __half* dL_dparams, float max_level);
void plan_input_gradient(EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const __half* params, const __half* dL_dencoded, uint32_t row_stride,
                         float* dL_dx, float max_level);
// Second-order derivatives of a plan that is ONE grid (GridEncoding::backward_backward_input; anything else throws "... does not
// support double backward", object.h:468-482) from dL_ddLdinput [n][plan.n_in] fp32 and dL_doutput [n][row_stride] fp16. Each
// non-null result is OVERWRITTEN: dL_dparams fp16 [n_params], dL_ddLdoutput fp16 [n][row_stride], dL_dinput fp32 [n][plan.n_in].
void plan_backward_backward_input(EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const __half* params, const __half* dL_doutput,
                                  uint32_t row_stride, const float* dL_ddLdinput, __half* dL_dparams, __half* dL_ddLdoutput, float* dL_dinput, float max_level);
// Grid tables U(-1e-4, 1e-4) * scale from `rng`, nested grids one after the other (grid.h:1076-1079, composite.h initialize_params).
// `dst`: DEVICE fp32 array of plan.n_params elements.
void init_plan_params(const EncodingPlan& plan, HostPcg32& rng, float* dst, float scale);

}  // namespace tcnnb
