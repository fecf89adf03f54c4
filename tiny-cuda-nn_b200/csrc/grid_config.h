// grid_config.h -- host-side description of the multiresolution grid encoding, shared by the trainer / module tiers (model.cu) and
// the stand-alone encoding tier (encoding.cu): JSON parsing with the reference's keys, defaults and error texts
// (grid.h:1726-1851, src/encoding.cu:69-75,132-150), level sizing (grid.h:692-737) and the per-level lookup descriptors the
// kernels consume (grid_index's dense / hash decision, common_device.h:847-884).
#pragma once
#include "common.cuh"
#include "host_common.h"
#include "json_mini.h"
#include "misc_kernels.h"

#include <cmath>
#include <limits>
#include <string>
#include <vector>

namespace tcnnb {

// ------------------------------------------------------------------------------------------------------------------
struct GridConfig {
	uint32_t n_pos_dims = 3;
	uint32_t n_levels = 16;
	uint32_t n_features_per_level = 2;
	uint32_t log2_hashmap_size = 19;
	uint32_t base_resolution = 16;
	float per_level_scale = 2.0f;
	uint32_t grid_type = GRID_HASH;
	uint32_t interpolation = INTERP_LINEAR;
	bool stochastic_interpolation = false;
	bool fixed_point_pos = false;
	std::string otype = "HashGrid";
	// derived
	std::vector<uint32_t> offsets;      // n_levels + 1, in entries
	std::vector<uint32_t> resolutions;  // from the host evaluation (sizing, grid.h:701)
	std::vector<float> scales;          // device evaluation (lookup)
	uint32_t n_params = 0;
	uint32_t padded_width = 0;
};

// grid.h:1726-1851
inline GridConfig parse_grid(uint32_t n_dims_to_encode, const json::Value& e) {
	GridConfig g;
	g.otype = e.value("otype", "OneBlob");  // src/encoding.cu:133 default
	const std::string lower = to_lower(g.otype);
	if (!(lower == "grid" || lower == "hashgrid" || lower == "tiledgrid" || lower == "densegrid")) {
		static const char* known[] = {"composite", "empty", "frequency", "identity", "oneblob", "sphericalharmonics", "trianglewave", "oneblobfrequency", "nrc"};
		for (auto k : known) {
			if (lower == k) throw std::runtime_error("Encoding '" + g.otype + "' is outside the tcnn_b200 hot path (only Grid/HashGrid/DenseGrid/TiledGrid are built)");
		}
		throw std::runtime_error("Encoding '" + g.otype + "' not found");
	}
	const std::string hash = e.value("hash", "CoherentPrime");
	if (!ieq(hash, "CoherentPrime")) {
		static const char* other[] = {"Prime", "ReversedPrime", "Rng", "BaseConvert"};
		for (auto k : other) if (ieq(hash, k)) throw std::runtime_error(std::string("GridEncoding: compiled without ") + k + " hash support.");
		throw std::runtime_error("Invalid hash type: " + hash);
	}
	g.n_features_per_level = (uint32_t)e.value("n_features_per_level", 2.0);
	if (!(g.n_features_per_level == 1 || g.n_features_per_level == 2 || g.n_features_per_level == 4 || g.n_features_per_level == 8)) {
		throw std::runtime_error("GridEncoding: n_features_per_level must be 1, 2, 4, or 8.");
	}
	g.log2_hashmap_size = (uint32_t)e.value("log2_hashmap_size", 19.0);
	const std::string default_type = lower == "tiledgrid" ? "Tiled" : (lower == "densegrid" ? "Dense" : "Hash");
	uint32_t n_features;
	if (e.contains("n_features") || e.contains("n_grid_features")) {
		n_features = (uint32_t)(e.contains("n_features") ? e.value("n_features", 0.0) : e.value("n_grid_features", 0.0));
		if (e.contains("n_levels")) {
			throw std::runtime_error("GridEncoding: may not specify n_features and n_levels simultaneously (one determines the other)");
		}
	} else {
		n_features = g.n_features_per_level * (uint32_t)e.value("n_levels", 16.0);
	}
	if (n_features % g.n_features_per_level != 0) {
		throw std::runtime_error("GridEncoding: n_features=" + std::to_string(n_features) + " must be a multiple of N_FEATURES_PER_LEVEL=" + std::to_string(g.n_features_per_level));
	}
	g.n_levels = n_features / g.n_features_per_level;
	const std::string type = e.value("type", default_type);
	if (ieq(type, "Hash")) g.grid_type = GRID_HASH;
	else if (ieq(type, "Dense")) g.grid_type = GRID_DENSE;
	else if (ieq(type, "Tiled") || ieq(type, "Tile")) g.grid_type = GRID_TILED;
	else throw std::runtime_error("Invalid grid type: " + type);
	g.base_resolution = (uint32_t)e.value("base_resolution", 16.0);
	g.fixed_point_pos = e.value("fixed_point_pos", false);
	const float default_scale = g.grid_type == GRID_DENSE ? std::exp(std::log(256.0f / (float)g.base_resolution) / (g.n_levels - 1)) : 2.0f;
	g.per_level_scale = (float)e.value("per_level_scale", (double)default_scale);
	g.stochastic_interpolation = e.value("stochastic_interpolation", false);
	const std::string interp = e.value("interpolation", "Linear");
	if (ieq(interp, "Nearest")) g.interpolation = INTERP_NEAREST;
	else if (ieq(interp, "Linear")) g.interpolation = INTERP_LINEAR;
	else if (ieq(interp, "Smoothstep")) g.interpolation = INTERP_SMOOTHSTEP;
	else throw std::runtime_error("Invalid interpolation type: " + interp);
	if (n_dims_to_encode < 2 || n_dims_to_encode > 4) throw std::runtime_error("GridEncoding: number of input dims must be 2 or 3.");
	g.n_pos_dims = n_dims_to_encode;
	if (g.n_levels > 128) throw std::runtime_error("GridEncoding: m_n_levels=" + std::to_string(g.n_levels) + " must be at most MAX_N_LEVELS=128");

	// Level sizing, grid.h:692-737 (host evaluation of grid_scale / grid_resolution).
	const float log2_scale = std::log2(g.per_level_scale);
	uint32_t offset = 0;
	g.offsets.resize(g.n_levels + 1);
	g.resolutions.resize(g.n_levels);
	for (uint32_t i = 0; i < g.n_levels; ++i) {
		const float scale = exp2f(i * log2_scale) * g.base_resolution - 1.0f;
		const uint32_t resolution = (uint32_t)ceilf(scale) + 1;
		g.resolutions[i] = resolution;
		const uint32_t max_params = std::numeric_limits<uint32_t>::max() / 2;
		uint32_t params_in_level = std::pow((float)resolution, (float)g.n_pos_dims) > (float)max_params ? max_params : powi(resolution, g.n_pos_dims);
		params_in_level = next_multiple(params_in_level, 8u);
		if (g.grid_type == GRID_TILED) params_in_level = std::min(params_in_level, powi(g.base_resolution, g.n_pos_dims));
		else if (g.grid_type == GRID_HASH) params_in_level = std::min(params_in_level, 1u << g.log2_hashmap_size);
		g.offsets[i] = offset;
		offset += params_in_level;
	}
	g.offsets[g.n_levels] = offset;
	g.n_params = offset * g.n_features_per_level;
	return g;
}


// Per-level scales evaluated on the DEVICE like the reference's kernels (common_device.h:886-891; fast-math ex2.approx + fma), so
// that cell selection matches them bit for bit.
inline void evaluate_level_scales(GridConfig& g) {
	DeviceBuffer<float> scales_dev;
	scales_dev.resize(g.n_levels);
	g.scales.resize(g.n_levels);
	TCNNB_CUDA_CHECK(launch_level_scales(nullptr, g.n_levels, std::log2(g.per_level_scale), g.base_resolution, scales_dev.ptr));
	++g_kernel_launches;
	TCNNB_CUDA_CHECK(cudaMemcpy(g.scales.data(), scales_dev.ptr, sizeof(float) * g.n_levels, cudaMemcpyDeviceToHost));
}

// The level table as the C ABI exports it (ParamsOffsetTable, multi_level_interface.h:84-88): n_levels, n_levels + 1 offsets,
// and per level the scale and resolution. `g` == nullptr: no grid (n_levels = 0, offsets = {0}). Every output is optional.
inline void write_level_table(const GridConfig* g, uint32_t* n_levels, uint32_t* offsets, float* scales, uint32_t* resolutions) {
	const uint32_t n = g ? g->n_levels : 0;
	if (n_levels) *n_levels = n;
	for (uint32_t l = 0; l < n; ++l) {
		if (offsets) offsets[l] = g->offsets[l];
		if (scales) scales[l] = g->scales[l];
		if (resolutions) resolutions[l] = (uint32_t)ceilf(g->scales[l]) + 1;
	}
	if (offsets) offsets[n] = g ? g->offsets[n] : 0;
}

// LevelInfo of level l (needs g.scales).
inline LevelInfo make_level_info(const GridConfig& g, uint32_t l) {
	static const uint32_t MAX_BASES[] = {0x0, 0xFFFFFFFF, 0xFFFF, 0x659, 0xFF, 0x54, 0x28, 0x17, 0xF, 0xB, 0x9};
	LevelInfo lv{};
	lv.offset = g.offsets[l];
	lv.size = g.offsets[l + 1] - g.offsets[l];
	lv.scale = g.scales[l];
	lv.resolution = (uint32_t)ceilf(lv.scale) + 1;  // grid_resolution(scale) as the kernels evaluate it (grid.h:98)
	// grid_index (common_device.h:847-884)
	uint32_t stride = 1;
	const bool dense_ok = lv.resolution <= MAX_BASES[g.n_pos_dims];
	if (dense_ok) {
		for (uint32_t d = 0; d < g.n_pos_dims; ++d) stride *= lv.resolution;
	} else {
		stride = 0xFFFFFFFFu;
	}
	if (g.grid_type == GRID_HASH && lv.size < stride) lv.use_hash = 1;
	else lv.use_hash = dense_ok ? 0 : 2;
	lv.pow2_mask = (lv.size & (lv.size - 1)) == 0 ? lv.size - 1 : 0;
	lv.wide_ok = (lv.offset % 4u) == 0 ? 1 : 0;
	// dense index <= res * (res^D - 1) / (res - 1) < 2 * res^D: a conditional subtract is an exact modulo when size >= res^D
	lv.small_mod = (lv.use_hash == 0 && stride != 0xFFFFFFFFu && lv.size >= stride && lv.resolution >= 2) ? 1 : 0;
	return lv;
}

}  // namespace tcnnb
