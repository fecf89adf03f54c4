// oracle_cpu.cpp -- CPU restatement of the reference hot path (HashGrid + FullyFusedMLP training step).
//
// TEST INFRASTRUCTURE ONLY -- see oracle_cpu.h. Not a product path; nothing under tiny-cuda-nn_b200/
// may call this. The restatement follows the reference's algorithm function by function; each block
// cites the file:line (relative to /root/reference) it follows. fp16 arithmetic is emulated with
// _Float16 (IEEE binary16, round-to-nearest-even) so that the encoding and every fp16 rounding point of
// the reference are reproduced exactly; only accumulation ORDER (atomics, split-K) is not modelled and is
// replaced by exact (double) sums.
//
// Pinning: tests/test_oracle_golden.py checks this file against tests/golden/* (vectors dumped from the
// reference itself, compiled from its sources and run on the GPU by tests/golden/make_golden.sh) and
// against the reference's own known-answer test tests/test_grid.cu:54-71.
#include "oracle_cpu.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <random>
#include <vector>

#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

typedef _Float16 half_t;

inline half_t bits_to_half(uint16_t b) { half_t h; std::memcpy(&h, &b, 2); return h; }
inline uint16_t half_to_bits(half_t h) { uint16_t b; std::memcpy(&b, &h, 2); return b; }
inline float h2f(uint16_t b) { return (float)bits_to_half(b); }
inline uint16_t f2h(float f) { return half_to_bits((half_t)f); }
inline uint16_t d2h(double d) { return half_to_bits((half_t)d); }

// __hfma2 per component (vec.h:372-378): one rounding of a*b+c to binary16.
inline half_t hfma(half_t a, half_t b, half_t c) { return (half_t)((double)a * (double)b + (double)c); }
// __hmul2 per component.
inline half_t hmul(half_t a, half_t b) { return (half_t)((double)a * (double)b); }

inline uint32_t next_multiple(uint32_t v, uint32_t d) { return ((v + d - 1) / d) * d; }
inline uint32_t powi(uint32_t base, uint32_t e) { uint32_t r = 1; for (uint32_t i = 0; i < e; ++i) r *= base; return r; }  // common_host.h:361-368

const uint64_t PCG32_MULT = 0x5851f42d4c957f2dULL;

// common_device.h:886-895
inline float grid_scale(uint32_t level, float log2_per_level_scale, uint32_t base_resolution) {
	return exp2f(level * log2_per_level_scale) * base_resolution - 1.0f;
}
inline uint32_t grid_resolution(float scale) { return (uint32_t)ceilf(scale) + 1; }

// common_device.h:787-791 (coherent_prime_hash) + :847-884 (grid_index)
inline uint32_t grid_index(uint32_t D, uint32_t grid_type, uint32_t hashmap_size, uint32_t resolution, const uint32_t* pos_grid) {
	static const uint32_t MAX_BASES[] = {0x0, 0xFFFFFFFF, 0xFFFF, 0x659, 0xFF, 0x54, 0x28, 0x17, 0xF, 0xB, 0x9};
	static const uint32_t factors[7] = {1u, 2654435761u, 805459861u, 3674653429u, 2097192037u, 1434869437u, 2165219737u};
	uint32_t stride = 1;
	uint32_t index = 0;
	if (resolution <= MAX_BASES[D]) {
		for (uint32_t dim = 0; dim < D; ++dim) {
			index += pos_grid[dim] * stride;
			stride *= resolution;
		}
	} else {
		stride = 0xFFFFFFFF;
	}
	if (grid_type == ORC_GRID_HASH && hashmap_size < stride) {
		index = 0;
		for (uint32_t dim = 0; dim < D; ++dim) {
			index ^= pos_grid[dim] * factors[dim];
		}
	}
	return index % hashmap_size;
}

inline float smoothstep(float x) { return x * x * (3.0f - 2.0f * x); }  // common_device.h smoothstep

// common_device.h:1031-1043 pos_fract
inline void pos_fract(float input, float scale, uint32_t interpolation, float* pos, uint32_t* pos_grid) {
	float p = fmaf(scale, input, 0.5f);
	float tmp = floorf(p);
	*pos_grid = (uint32_t)(int)tmp;
	p -= tmp;
	*pos = interpolation == ORC_INTERP_SMOOTHSTEP ? smoothstep(p) : p;
}

// common_device.h:110-350 activations, evaluated like warp_activation<__half>: on the fp16 value.
inline half_t activation_fwd(uint32_t act, half_t x) {
	switch (act) {
		case ORC_ACT_RELU: return x > (half_t)0.0f ? x : (half_t)0.0f;
		case ORC_ACT_LEAKY_RELU: return hmul(x, (half_t)(x > (half_t)0.0f ? 1.0f : 0.01f));
		case ORC_ACT_EXPONENTIAL: return (half_t)expf((float)x);
		case ORC_ACT_SIGMOID: return (half_t)(1.0f / (1.0f + expf(-(float)x)));
		case ORC_ACT_SQUAREPLUS: { float v = (float)x * 10.0f; return (half_t)(0.5f * (v + sqrtf(v * v + 4)) / 10.0f); }
		case ORC_ACT_SOFTPLUS: return (half_t)(logf(expf((float)x * 10.0f) + 1.0f) / 10.0f);
		case ORC_ACT_TANH: return (half_t)tanhf((float)x);
		case ORC_ACT_NONE: default: return x;
	}
}

// warp_activation_backward (common_device.h:363-440): gradient * f'(.) using the stored FORWARD (post-activation) value.
inline half_t activation_bwd(uint32_t act, half_t grad, half_t fwd) {
	switch (act) {
		case ORC_ACT_RELU: return hmul(grad, (half_t)(fwd > (half_t)0.0f ? 1.0f : 0.0f));
		case ORC_ACT_LEAKY_RELU: return hmul(grad, (half_t)(fwd > (half_t)0.0f ? 1.0f : 0.01f));
		case ORC_ACT_EXPONENTIAL: return hmul(grad, fwd);
		case ORC_ACT_SIGMOID: return hmul(grad, hmul(fwd, (half_t)(1.0f - (float)fwd)));  // frag * (T)(fwd * (T)(1 - fwd)), common_device.h:392-396
		case ORC_ACT_SQUAREPLUS: { float y = (float)fwd * 10.0f; float y2 = y * y; return hmul(grad, (half_t)(y2 / (y2 + 1))); }
		case ORC_ACT_SOFTPLUS: return hmul(grad, (half_t)(1.0f - expf(-(float)fwd * 10.0f)));
		case ORC_ACT_TANH: return hmul(grad, (half_t)(1.0f - (float)fwd * (float)fwd));
		case ORC_ACT_NONE: default: return grad;
	}
}

// One output neuron of act(W.x): products of fp16 values are exact in double; the accumulator model
// selects where the running sum is rounded (see ORC_ACCUM_* in oracle_cpu.h).
inline half_t dot_accum(int accum_mode, const uint16_t* w, const half_t* x, uint32_t n) {
	if (accum_mode == ORC_ACCUM_FP16_K16) {
		half_t acc = (half_t)0.0f;
		for (uint32_t k0 = 0; k0 < n; k0 += 16) {
			double s = (double)acc;
			for (uint32_t k = k0; k < std::min(n, k0 + 16); ++k) s += (double)bits_to_half(w[k]) * (double)x[k];
			acc = (half_t)s;
		}
		return acc;
	}
	double s = 0.0;
	for (uint32_t k = 0; k < n; ++k) s += (double)bits_to_half(w[k]) * (double)x[k];
	return (half_t)(float)s;  // fp32 accumulator, then one rounding to fp16
}

}  // namespace

extern "C" {

int orc_num_threads(void) {
#ifdef _OPENMP
	return omp_get_max_threads();
#else
	return 1;
#endif
}

// ---------------------------------------------------------------------------------------------
// pcg32 -- restated from the published PCG-XSH-RR 64/32 algorithm (O'Neill) as used by
// dependencies/pcg32/pcg32.h:53-69 (seed/next_uint), :103-112 (next_float), :145-166 (advance).
// ---------------------------------------------------------------------------------------------
uint32_t orc_pcg32_next_uint(orc_pcg32_t* rng) {
	const uint64_t old = rng->state;
	rng->state = old * PCG32_MULT + rng->inc;
	const uint32_t xorshifted = (uint32_t)(((old >> 18u) ^ old) >> 27u);
	const uint32_t rot = (uint32_t)(old >> 59u);
	return (xorshifted >> rot) | (xorshifted << ((~rot + 1u) & 31));
}

void orc_pcg32_seed(orc_pcg32_t* rng, uint64_t initstate, uint64_t initseq) {
	rng->state = 0;
	rng->inc = (initseq << 1u) | 1u;
	orc_pcg32_next_uint(rng);
	rng->state += initstate;
	orc_pcg32_next_uint(rng);
}

float orc_pcg32_next_float(orc_pcg32_t* rng) {
	const uint32_t u = (orc_pcg32_next_uint(rng) >> 9) | 0x3f800000u;
	float f;
	std::memcpy(&f, &u, 4);
	return f - 1.0f;
}

void orc_pcg32_advance(orc_pcg32_t* rng, int64_t delta_) {
	uint64_t cur_mult = PCG32_MULT, cur_plus = rng->inc, acc_mult = 1u, acc_plus = 0u;
	uint64_t delta = (uint64_t)delta_;
	while (delta > 0) {
		if (delta & 1) {
			acc_mult *= cur_mult;
			acc_plus = acc_plus * cur_mult + cur_plus;
		}
		cur_plus = (cur_mult + 1) * cur_plus;
		cur_mult *= cur_mult;
		delta /= 2;
	}
	rng->state = acc_mult * rng->state + acc_plus;
}

// trainer.h:51-58
void orc_trainer_rng(uint32_t seed, orc_pcg32_t* rng) {
	std::seed_seq seq{seed};
	std::vector<uint32_t> seeds(2);
	seq.generate(seeds.begin(), seeds.end());
	orc_pcg32_seed(rng, seeds.front(), 1);
}

// random.h:40-69 -- N_TO_GENERATE = 4, 128 threads per block (common_host.h N_THREADS_LINEAR).
void orc_generate_random_uniform(orc_pcg32_t* rng, uint64_t n_elements, float* out, float lower, float upper) {
	const uint64_t n_threads_needed = (n_elements + 3) / 4;
	const uint64_t n_blocks = (n_threads_needed + 127) / 128;
	const uint64_t n_threads = n_blocks * 128;
	const float range = upper - lower;
#pragma omp parallel for schedule(static)
	for (int64_t i = 0; i < (int64_t)n_threads; ++i) {
		orc_pcg32_t local = *rng;
		orc_pcg32_advance(&local, i * 4);
		for (uint64_t j = 0; j < 4; ++j) {
			const uint64_t idx = (uint64_t)i + n_threads * j;
			if (idx >= n_elements) break;
			// `val * (upper - lower) + lower` is contracted to an FMA by nvcc (random.h:69).
			out[idx] = fmaf(orc_pcg32_next_float(&local), range, lower);
		}
	}
	orc_pcg32_advance(rng, (int64_t)n_elements);
}

// ---------------------------------------------------------------------------------------------
// Sizing
// ---------------------------------------------------------------------------------------------
// grid.h:692-737
int orc_grid_setup(orc_grid_t* g) {
	if (g->n_levels == 0 || g->n_levels > ORC_MAX_LEVELS) return -1;
	if (g->n_pos_dims < 1 || g->n_pos_dims > 4) return -1;
	uint32_t offset = 0;
	const float log2_scale = std::log2(g->per_level_scale);
	for (uint32_t i = 0; i < g->n_levels; ++i) {
		const float scale = grid_scale(i, log2_scale, g->base_resolution);
		const uint32_t resolution = grid_resolution(scale);
		g->scales[i] = scale;
		g->resolutions[i] = resolution;
		const uint32_t max_params = std::numeric_limits<uint32_t>::max() / 2;
		uint32_t params_in_level = std::pow((float)resolution, (float)g->n_pos_dims) > (float)max_params ? max_params : powi(resolution, g->n_pos_dims);
		params_in_level = next_multiple(params_in_level, 8u);
		if (g->grid_type == ORC_GRID_DENSE) {
		} else if (g->grid_type == ORC_GRID_TILED) {
			params_in_level = std::min(params_in_level, powi(g->base_resolution, g->n_pos_dims));
		} else if (g->grid_type == ORC_GRID_HASH) {
			params_in_level = std::min(params_in_level, (1u << g->log2_hashmap_size));
		} else {
			return -1;
		}
		g->offsets[i] = offset;
		offset += params_in_level;
	}
	g->offsets[g->n_levels] = offset;
	g->n_params = offset * g->n_features_per_level;
	if (g->padded_width < g->n_levels * g->n_features_per_level) {
		g->padded_width = next_multiple(g->n_levels * g->n_features_per_level, 16u);
	}
	return 0;
}

// fully_fused_mlp.cu:635-672
int orc_mlp_setup(orc_mlp_t* m) {
	if (m->n_hidden_layers < 1) return -1;
	m->padded_out_width = next_multiple(m->out_width, 16u);
	m->n_params = m->width * m->in_width + (m->n_hidden_layers - 1) * m->width * m->width + m->padded_out_width * m->width;
	return 0;
}

// ---------------------------------------------------------------------------------------------
// Parameter initialisation
// ---------------------------------------------------------------------------------------------
void orc_initialize_params(const orc_grid_t* g, const orc_mlp_t* m, orc_pcg32_t* rng, float* params) {
	// fully_fused_mlp.cu:868-892 + gpu_matrix.h:292-306: xavier uniform on the host, sequential draws, row-major [out][in].
	std::vector<std::pair<uint32_t, uint32_t>> mats;  // (rows = fan_out, cols = fan_in)
	mats.emplace_back(m->width, m->in_width);
	for (uint32_t i = 0; i + 1 < m->n_hidden_layers; ++i) mats.emplace_back(m->width, m->width);
	mats.emplace_back(m->padded_out_width, m->width);
	float* p = params;
	for (auto& rc : mats) {
		const float scale = 1.0f * std::sqrt(6.0f / (float)(rc.second + rc.first));
		const size_t n = (size_t)rc.first * rc.second;
		for (size_t i = 0; i < n; ++i) {
			p[i] = orc_pcg32_next_float(rng) * 2.0f * scale - scale;
		}
		p += n;
	}
	// grid.h:1076-1079: generate_random_uniform(rnd, n_params, ptr, -1e-4f * scale, 1e-4f * scale), scale = 1.
	if (g && g->n_params > 0) {
		orc_generate_random_uniform(rng, g->n_params, p, -1e-4f, 1e-4f);
	}
}

void orc_cast_to_half(uint64_t n, const float* in, uint16_t* out) {
#pragma omp parallel for schedule(static)
	for (int64_t i = 0; i < (int64_t)n; ++i) out[i] = f2h(in[i]);
}

void orc_cast_from_half(uint64_t n, const uint16_t* in, float* out) {
#pragma omp parallel for schedule(static)
	for (int64_t i = 0; i < (int64_t)n; ++i) out[i] = h2f(in[i]);
}

// ---------------------------------------------------------------------------------------------
// Grid encoding
// ---------------------------------------------------------------------------------------------
// kernel_grid (grid.h:49-212): per (sample, level): pos_fract, 2^D corners in idx order, weight in fp32,
// result = __hfma2((half)w, grid[index], result); SoA store out[i + (level*F+f)*B]. Pad rows zeroed (grid.h:759-766).
void orc_grid_forward(const orc_grid_t* g, uint32_t B, const float* positions, const uint16_t* grid, uint16_t* out, uint32_t* indices) {
	const uint32_t D = g->n_pos_dims, F = g->n_features_per_level, L = g->n_levels;
	const uint32_t n_corners = 1u << D;
	for (uint32_t r = L * F; r < g->padded_width; ++r) {
		std::memset(out + (size_t)r * B, 0, sizeof(uint16_t) * B);
	}
#pragma omp parallel for schedule(static)
	for (int64_t ii = 0; ii < (int64_t)B; ++ii) {
		const uint32_t i = (uint32_t)ii;
		for (uint32_t level = 0; level < L; ++level) {
			const uint16_t* level_grid = grid + (size_t)g->offsets[level] * F;
			const uint32_t hashmap_size = g->offsets[level + 1] - g->offsets[level];
			const float scale = g->scales[level];
			const uint32_t resolution = grid_resolution(scale);
			float pos[4];
			uint32_t pos_grid[4];
			for (uint32_t d = 0; d < D; ++d) pos_fract(positions[(size_t)i * D + d], scale, g->interpolation, &pos[d], &pos_grid[d]);

			half_t result[8];
			for (uint32_t f = 0; f < F; ++f) result[f] = (half_t)0.0f;

			if (g->interpolation == ORC_INTERP_NEAREST) {
				const uint32_t index = grid_index(D, g->grid_type, hashmap_size, resolution, pos_grid);
				if (indices) indices[((size_t)i * L + level) * n_corners] = index;
				for (uint32_t f = 0; f < F; ++f) result[f] = bits_to_half(level_grid[(size_t)index * F + f]);
			} else {
				for (uint32_t idx = 0; idx < n_corners; ++idx) {
					float weight = 1;
					uint32_t local[4];
					for (uint32_t d = 0; d < D; ++d) {
						if ((idx & (1u << d)) == 0) {
							weight *= 1 - pos[d];
							local[d] = pos_grid[d];
						} else {
							weight *= pos[d];
							local[d] = pos_grid[d] + 1;
						}
					}
					const uint32_t index = grid_index(D, g->grid_type, hashmap_size, resolution, local);
					if (indices) indices[((size_t)i * L + level) * n_corners + idx] = index;
					const half_t w = (half_t)weight;
					for (uint32_t f = 0; f < F; ++f) {
						result[f] = hfma(w, bits_to_half(level_grid[(size_t)index * F + f]), result[f]);
					}
				}
			}
			for (uint32_t f = 0; f < F; ++f) out[i + (size_t)(level * F + f) * B] = half_to_bits(result[f]);
		}
	}
}

// Input gradient of the grid encoding, for the module tier's dL_dinput (next row of SURVEY.md section 8f; the CUDA side does
// not compute it yet): kernel_grid's `dy_dx` branch (grid.h:171-210) followed by kernel_grid_backward_input (grid.h:322-350).
// Per level and feature, dy/dx_d = sum over the 2^(D-1) corners of the other dimensions of
//   scale * prod_other(w) * ((float)val(x_d + 1) - (float)val(x_d)) * pos_derivative_d
// in fp32 in the reference's loop order; then dL/dx_d = sum_k dL/dy_k * dy_k/dx_d over the encoded features k in order.
// pos_derivative is 1 for Linear and 6 p (1 - p) for Smoothstep (common_device.h:980-982, 1017-1029).
void orc_grid_input_gradient(const orc_grid_t* g, uint32_t B, const float* positions, const uint16_t* grid, const uint16_t* dL_denc, float* dL_dx) {
	const uint32_t D = g->n_pos_dims, F = g->n_features_per_level, L = g->n_levels;
#pragma omp parallel for schedule(static)
	for (int64_t ii = 0; ii < (int64_t)B; ++ii) {
		const uint32_t i = (uint32_t)ii;
		float result[4] = {0, 0, 0, 0};
		for (uint32_t level = 0; level < L; ++level) {
			const uint16_t* level_grid = grid + (size_t)g->offsets[level] * F;
			const uint32_t hashmap_size = g->offsets[level + 1] - g->offsets[level];
			const float scale = g->scales[level];
			const uint32_t resolution = grid_resolution(scale);
			float pos[4], pos_derivative[4];
			uint32_t pos_grid[4];
			for (uint32_t d = 0; d < D; ++d) {
				float p = fmaf(scale, positions[(size_t)i * D + d], 0.5f);
				const float tmp = floorf(p);
				pos_grid[d] = (uint32_t)(int)tmp;
				p -= tmp;
				pos_derivative[d] = g->interpolation == ORC_INTERP_SMOOTHSTEP ? 6 * p * (1.0f - p) : 1.0f;  // smoothstep_derivative, common_device.h:980-982
				pos[d] = g->interpolation == ORC_INTERP_SMOOTHSTEP ? smoothstep(p) : p;
			}
			float grads[8][4] = {};
			if (g->interpolation != ORC_INTERP_NEAREST) {  // Nearest: dy_dx stays zero (grid.h:120-133 returns before the gradient branch)
				for (uint32_t grad_dim = 0; grad_dim < D; ++grad_dim) {
					for (uint32_t idx = 0; idx < (1u << (D - 1)); ++idx) {
						float weight = scale;
						uint32_t local[4];
						for (uint32_t non_grad_dim = 0; non_grad_dim + 1 < D; ++non_grad_dim) {
							const uint32_t dim = non_grad_dim >= grad_dim ? non_grad_dim + 1 : non_grad_dim;
							if ((idx & (1u << non_grad_dim)) == 0) {
								weight *= 1 - pos[dim];
								local[dim] = pos_grid[dim];
							} else {
								weight *= pos[dim];
								local[dim] = pos_grid[dim] + 1;
							}
						}
						local[grad_dim] = pos_grid[grad_dim];
						const uint32_t left = grid_index(D, g->grid_type, hashmap_size, resolution, local);
						local[grad_dim] = pos_grid[grad_dim] + 1;
						const uint32_t right = grid_index(D, g->grid_type, hashmap_size, resolution, local);
						for (uint32_t f = 0; f < F; ++f) {
							grads[f][grad_dim] += weight * (h2f(level_grid[(size_t)right * F + f]) - h2f(level_grid[(size_t)left * F + f])) * pos_derivative[grad_dim];
						}
					}
				}
			}
			for (uint32_t f = 0; f < F; ++f) {
				const float dL_dy_local = h2f(dL_denc[i + (size_t)(level * F + f) * B]);
				for (uint32_t d = 0; d < D; ++d) result[d] += dL_dy_local * grads[f][d];
			}
		}
		for (uint32_t d = 0; d < D; ++d) dL_dx[(size_t)i * D + d] = result[d];
	}
}

// kernel_grid_backward (grid.h:215-320): addend = (half)w * dL_dy (fp16 multiply), accumulated per entry.
void orc_grid_backward(const orc_grid_t* g, uint32_t B, const float* positions, const uint16_t* dL_denc, double* grad_sum) {
	const uint32_t D = g->n_pos_dims, F = g->n_features_per_level, L = g->n_levels;
	const uint32_t n_corners = 1u << D;
	std::memset(grad_sum, 0, sizeof(double) * g->n_params);
	// One level is owned by one thread -> no write conflicts, deterministic.
#pragma omp parallel for schedule(dynamic, 1)
	for (int64_t lvl = 0; lvl < (int64_t)L; ++lvl) {
		const uint32_t level = (uint32_t)lvl;
		double* level_grad = grad_sum + (size_t)g->offsets[level] * F;
		const uint32_t hashmap_size = g->offsets[level + 1] - g->offsets[level];
		const float scale = g->scales[level];
		const uint32_t resolution = grid_resolution(scale);
		for (uint32_t i = 0; i < B; ++i) {
			float pos[4];
			uint32_t pos_grid[4];
			for (uint32_t d = 0; d < D; ++d) pos_fract(positions[(size_t)i * D + d], scale, g->interpolation, &pos[d], &pos_grid[d]);
			half_t grad[8];
			for (uint32_t f = 0; f < F; ++f) grad[f] = bits_to_half(dL_denc[i + (size_t)(level * F + f) * B]);
			if (g->interpolation == ORC_INTERP_NEAREST) {
				const uint32_t index = grid_index(D, g->grid_type, hashmap_size, resolution, pos_grid);
				for (uint32_t f = 0; f < F; ++f) level_grad[(size_t)index * F + f] += (double)grad[f];
				continue;
			}
			for (uint32_t idx = 0; idx < n_corners; ++idx) {
				float weight = 1;
				uint32_t local[4];
				for (uint32_t d = 0; d < D; ++d) {
					if ((idx & (1u << d)) == 0) {
						weight *= 1 - pos[d];
						local[d] = pos_grid[d];
					} else {
						weight *= pos[d];
						local[d] = pos_grid[d] + 1;
					}
				}
				const uint32_t index = grid_index(D, g->grid_type, hashmap_size, resolution, local);
				const half_t w = (half_t)weight;
				for (uint32_t f = 0; f < F; ++f) level_grad[(size_t)index * F + f] += (double)hmul(w, grad[f]);
			}
		}
	}
}

// ---------------------------------------------------------------------------------------------
// MLP
// ---------------------------------------------------------------------------------------------
void orc_mlp_forward(const orc_mlp_t* m, uint32_t B, int accum_mode, const uint16_t* weights, const uint16_t* input_soa, uint16_t* hidden, uint16_t* output) {
	const uint32_t W = m->width, IN = m->in_width, OUT = m->padded_out_width, NH = m->n_hidden_layers;
#pragma omp parallel for schedule(static)
	for (int64_t ii = 0; ii < (int64_t)B; ++ii) {
		const uint32_t i = (uint32_t)ii;
		std::vector<half_t> a(std::max(IN, W)), b(std::max(W, OUT));
		for (uint32_t k = 0; k < IN; ++k) a[k] = bits_to_half(input_soa[i + (size_t)k * B]);
		const uint16_t* w = weights;
		uint32_t n_in = IN;
		for (uint32_t l = 0; l < NH; ++l) {
			// threadblock_input_layer_forward_dynamic / threadblock_layer (fully_fused_mlp.cu:315-419, 47-129)
			for (uint32_t o = 0; o < W; ++o) {
				b[o] = activation_fwd(m->activation, dot_accum(accum_mode, w + (size_t)o * n_in, a.data(), n_in));
			}
			if (hidden) {
				for (uint32_t o = 0; o < W; ++o) hidden[((size_t)l * B + i) * W + o] = half_to_bits(b[o]);
			}
			w += (size_t)W * n_in;
			n_in = W;
			std::copy(b.begin(), b.begin() + W, a.begin());
		}
		// threadblock_last_layer_forward (fully_fused_mlp.cu:421-476)
		for (uint32_t o = 0; o < OUT; ++o) {
			output[(size_t)i * OUT + o] = half_to_bits(activation_fwd(m->output_activation, dot_accum(accum_mode, w + (size_t)o * W, a.data(), W)));
		}
	}
}

void orc_mlp_backward(const orc_mlp_t* m, uint32_t B, int accum_mode, const uint16_t* weights, const uint16_t* input_soa, const uint16_t* hidden, const uint16_t* dL_dout, double* dW, uint16_t* dL_din_soa) {
	const uint32_t W = m->width, IN = m->in_width, OUT = m->padded_out_width, NH = m->n_hidden_layers;
	std::memset(dW, 0, sizeof(double) * m->n_params);
	// Offsets of each weight matrix.
	std::vector<size_t> w_off(NH + 1);
	w_off[0] = 0;
	w_off[1] = (size_t)W * IN;
	for (uint32_t l = 2; l <= NH; ++l) w_off[l] = w_off[l - 1] + (size_t)W * W;

	const int n_thr = orc_num_threads();
	std::vector<std::vector<double>> dW_part(n_thr, std::vector<double>(m->n_params, 0.0));

#pragma omp parallel for schedule(static)
	for (int64_t ii = 0; ii < (int64_t)B; ++ii) {
		const uint32_t i = (uint32_t)ii;
#ifdef _OPENMP
		double* dWp = dW_part[omp_get_thread_num()].data();
#else
		double* dWp = dW_part[0].data();
#endif
		std::vector<half_t> g(std::max(OUT, W)), gn(std::max(W, IN));
		// NOTE: the output activation's transfer is applied by the caller before this function (fully_fused_mlp.cu:758-762).
		for (uint32_t o = 0; o < OUT; ++o) g[o] = bits_to_half(dL_dout[(size_t)i * OUT + o]);

		// Output layer weight gradient: dW_out = dL_dout . h_last^T (fully_fused_mlp.cu:784-787)
		{
			const uint16_t* h_last = hidden + ((size_t)(NH - 1) * B + i) * W;
			double* d = dWp + w_off[NH];
			for (uint32_t o = 0; o < OUT; ++o) {
				const double go = (double)g[o];
				if (go == 0.0) continue;
				for (uint32_t k = 0; k < W; ++k) d[(size_t)o * W + k] += go * (double)bits_to_half(h_last[k]);
			}
		}
		// Backprop through last layer (fully_fused_mlp.cu:192-240): g_h = (W_out^T . dL_dout) * act'(h_last)
		{
			const uint16_t* w = weights + w_off[NH];
			const uint16_t* h_last = hidden + ((size_t)(NH - 1) * B + i) * W;
			for (uint32_t k = 0; k < W; ++k) {
				// transposed weights: column k of W_out
				half_t acc;
				if (accum_mode == ORC_ACCUM_FP16_K16) {
					double s = 0;
					for (uint32_t o = 0; o < OUT; ++o) s += (double)bits_to_half(w[(size_t)o * W + k]) * (double)g[o];
					acc = (half_t)s;  // OUT == 16 -> one k-block
				} else {
					double s = 0;
					for (uint32_t o = 0; o < OUT; ++o) s += (double)bits_to_half(w[(size_t)o * W + k]) * (double)g[o];
					acc = (half_t)(float)s;
				}
				gn[k] = activation_bwd(m->activation, acc, bits_to_half(h_last[k]));
			}
			std::copy(gn.begin(), gn.begin() + W, g.begin());
		}
		// Hidden layers, from the last hidden matmul down to the first (fully_fused_mlp.cu:248-250, :815-830)
		for (uint32_t l = NH - 1; l >= 1; --l) {
			const uint16_t* h_prev = hidden + ((size_t)(l - 1) * B + i) * W;
			double* d = dWp + w_off[l];
			for (uint32_t o = 0; o < W; ++o) {
				const double go = (double)g[o];
				if (go == 0.0) continue;
				for (uint32_t k = 0; k < W; ++k) d[(size_t)o * W + k] += go * (double)bits_to_half(h_prev[k]);
			}
			const uint16_t* w = weights + w_off[l];
			for (uint32_t k = 0; k < W; ++k) {
				half_t acc;
				if (accum_mode == ORC_ACCUM_FP16_K16) {
					half_t a16 = (half_t)0.0f;
					for (uint32_t o0 = 0; o0 < W; o0 += 16) {
						double s = (double)a16;
						for (uint32_t o = o0; o < std::min(W, o0 + 16); ++o) s += (double)bits_to_half(w[(size_t)o * W + k]) * (double)g[o];
						a16 = (half_t)s;
					}
					acc = a16;
				} else {
					double s = 0;
					for (uint32_t o = 0; o < W; ++o) s += (double)bits_to_half(w[(size_t)o * W + k]) * (double)g[o];
					acc = (half_t)(float)s;
				}
				gn[k] = activation_bwd(m->activation, acc, bits_to_half(h_prev[k]));
			}
			std::copy(gn.begin(), gn.begin() + W, g.begin());
		}
		// First layer: dW_0 = g_0 . input^T (fully_fused_mlp.cu:827-830), dL_dinput = W_0^T . g_0 (:833-836)
		{
			double* d = dWp + w_off[0];
			for (uint32_t o = 0; o < W; ++o) {
				const double go = (double)g[o];
				if (go == 0.0) continue;
				for (uint32_t k = 0; k < IN; ++k) d[(size_t)o * IN + k] += go * (double)bits_to_half(input_soa[i + (size_t)k * B]);
			}
			if (dL_din_soa) {
				const uint16_t* w = weights + w_off[0];
				for (uint32_t k = 0; k < IN; ++k) {
					half_t acc;
					if (accum_mode == ORC_ACCUM_FP16_K16) {
						half_t a16 = (half_t)0.0f;
						for (uint32_t o0 = 0; o0 < W; o0 += 16) {
							double s = (double)a16;
							for (uint32_t o = o0; o < std::min(W, o0 + 16); ++o) s += (double)bits_to_half(w[(size_t)o * IN + k]) * (double)g[o];
							a16 = (half_t)s;
						}
						acc = a16;
					} else {
						double s = 0;
						for (uint32_t o = 0; o < W; ++o) s += (double)bits_to_half(w[(size_t)o * IN + k]) * (double)g[o];
						acc = (half_t)(float)s;
					}
					dL_din_soa[i + (size_t)k * B] = half_to_bits(acc);
				}
			}
		}
	}
	for (int t = 0; t < n_thr; ++t) {
		for (size_t j = 0; j < m->n_params; ++j) dW[j] += dW_part[t][j];
	}
}

// ---------------------------------------------------------------------------------------------
// Loss
// ---------------------------------------------------------------------------------------------
static void loss_impl(int loss_type, uint32_t B, uint32_t stride, uint32_t dims, float loss_scale, uint32_t n_total, const uint16_t* prediction, const float* target, float* values, uint16_t* grads);

void orc_loss(int loss_type, uint32_t B, uint32_t stride, uint32_t dims, float loss_scale, const uint16_t* prediction, const float* target, float* values, uint16_t* grads) {
	loss_impl(loss_type, B, stride, dims, loss_scale, B * stride / stride * dims, prediction, target, values, grads);
}

// n_total is the normalisation count (relative_l2.h:62); a data-parallel shard passes the GLOBAL batch * dims.
void orc_loss_n(int loss_type, uint32_t B, uint32_t stride, uint32_t dims, float loss_scale, uint32_t n_total, const uint16_t* prediction, const float* target, float* values, uint16_t* grads) {
	loss_impl(loss_type, B, stride, dims, loss_scale, n_total, prediction, target, values, grads);
}

static void loss_impl(int loss_type, uint32_t B, uint32_t stride, uint32_t dims, float loss_scale, uint32_t n_total, const uint16_t* prediction, const float* target, float* values, uint16_t* grads) {
	const uint32_t n_elements = B * stride;
#pragma omp parallel for schedule(static)
	for (int64_t ii = 0; ii < (int64_t)n_elements; ++ii) {
		const uint32_t i = (uint32_t)ii;
		const uint32_t intra = i % stride, inter = i / stride;
		if (intra >= dims) {
			if (values) values[i] = 0;
			grads[i] = 0;
			continue;
		}
		const uint32_t target_idx = inter * dims + intra;
		const float pred = h2f(prediction[i]);
		const float difference = pred - target[target_idx];
		float value, gradient;
		if (loss_type == ORC_LOSS_RELATIVE_L2_LUMINANCE) {
			// losses/relative_l2_luminance.h:66-86: the row's luminance (channels 3..5 folded onto 0..2 when there are 6+ outputs)
			float r = h2f(prediction[i - intra + 0]), g = h2f(prediction[i - intra + 1]), b = h2f(prediction[i - intra + 2]);
			if (dims >= 6) {
				r += h2f(prediction[i - intra + 3]);
				g += h2f(prediction[i - intra + 4]);
				b += h2f(prediction[i - intra + 5]);
			}
			const float luminance = 0.299f * r + 0.587f * g + 0.114f * b;
			const float psq = luminance * luminance + 0.01f;
			value = difference * difference / psq / 1.0f / n_total;
			gradient = 2 * difference / psq / 1.0f;
		} else if (loss_type == ORC_LOSS_CROSS_ENTROPY) {
			// losses/cross_entropy.h:66-75 (the factor already carries 1 / n_total: undone for the common scaling below)
			const float factor = -target[target_idx] / 1.0f / n_total;
			value = factor * logf(pred);
			gradient = factor / pred * n_total;
		} else if (loss_type == ORC_LOSS_VARIANCE_IS) {
			// losses/variance_is.h:66-76
			const float tgt = target[target_idx];
			const float factor = tgt * tgt / 1.0f / n_total;
			value = factor / pred - factor / 1.0f;
			gradient = -factor / (pred * pred) * n_total;
		} else if (loss_type == ORC_LOSS_RELATIVE_L2) {
			// losses/relative_l2.h:64-75
			const float psq = pred * pred + 0.01f;
			value = difference * difference / psq / 1.0f / n_total;
			gradient = 2 * difference / psq / 1.0f;
		} else if (loss_type == ORC_LOSS_L1) {
			// losses/l1.h:68-73
			value = fabsf(difference) / 1.0f / n_total;
			gradient = copysignf(1.0f / 1.0f, difference);
		} else if (loss_type == ORC_LOSS_RELATIVE_L1 || loss_type == ORC_LOSS_MAPE || loss_type == ORC_LOSS_SMAPE) {
			// losses/relative_l1.h:71-76, mape.h:72-77, smape.h:72-77: |d| * scale, the scale relative to prediction / target / their mean
			const float tgt = target[target_idx];
			const float denom = loss_type == ORC_LOSS_RELATIVE_L1 ? fabsf(pred) : (loss_type == ORC_LOSS_MAPE ? fabsf(tgt) : 0.5f * (fabsf(tgt) + fabsf(pred)));
			const float scale = 1.0f / (denom + 1e-2f) / 1.0f;
			value = fabsf(difference) * scale / n_total;
			gradient = copysignf(scale, difference);
		} else {
			// losses/l2.h:64-74
			value = difference * difference / 1.0f / n_total;
			gradient = 2 * difference / 1.0f;
		}
		if (values) values[i] = value;
		grads[i] = f2h(loss_scale * gradient / n_total);
	}
}

// ---------------------------------------------------------------------------------------------
// Adam (optimizers/adam.h:48-129)
// ---------------------------------------------------------------------------------------------
void orc_adam_step(const orc_adam_t* a, uint64_t n, uint64_t n_matrix, float loss_scale, float* weights_fp32, uint16_t* weights_fp16, const uint16_t* grads_fp16, float* m1, float* m2, uint32_t* steps) {
	const float lower_lr_bound = 0;
	const float upper_lr_bound = std::numeric_limits<float>::max();
#pragma omp parallel for schedule(static)
	for (int64_t ii = 0; ii < (int64_t)n; ++ii) {
		const uint64_t i = (uint64_t)ii;
		float gradient = h2f(grads_fp16[i]) / loss_scale;
		if (i >= n_matrix) {
			if (!a->optimize_non_matrix_params || (gradient == 0 && a->skip_zero_grad_non_matrix_params)) continue;
		} else {
			if (!a->optimize_matrix_params) continue;
		}
		const float weight_fp = weights_fp32[i];
		if (i < n_matrix) gradient += a->l2_reg * weight_fp;
		else gradient += a->non_matrix_l2_reg * weight_fp;
		if (a->gradient_clipping_magnitude != 0.0f) {
			gradient = copysignf(std::min(fabsf(gradient), a->gradient_clipping_magnitude), gradient);
		}
		const float gradient_sq = gradient * gradient;
		const float first_moment = m1[i] = a->beta1 * m1[i] + (1 - a->beta1) * gradient;
		const float second_moment = m2[i] = a->beta2 * m2[i] + (1 - a->beta2) * gradient_sq;
		float learning_rate = a->learning_rate;
		if (i >= n_matrix) learning_rate *= a->non_matrix_learning_rate_factor;
		const uint32_t current_step = ++steps[i];
		learning_rate *= sqrtf(1 - powf(a->beta2, (float)current_step)) / (1 - powf(a->beta1, (float)current_step));
		const float effective_learning_rate = fminf(fmaxf(learning_rate / (sqrtf(second_moment) + a->epsilon), lower_lr_bound), upper_lr_bound);
		// weight_decay (common_device.h:1045-1048)
		const float rel = a->relative_decay * learning_rate, abs_ = a->absolute_decay * learning_rate;
		const float decayed_weight = (1 - rel) * weight_fp - copysignf(abs_, weight_fp);
		float new_weight = decayed_weight - effective_learning_rate * first_moment;
		if (a->clipping_magnitude != 0.0f) {
			new_weight = std::min(std::max(new_weight, -a->clipping_magnitude), a->clipping_magnitude);
		}
		weights_fp32[i] = new_weight;
		weights_fp16[i] = f2h(new_weight);
	}
}

// ---------------------------------------------------------------------------------------------
// Whole step (trainer.h:254-357, non-JIT order of operations §3.2)
// ---------------------------------------------------------------------------------------------
double orc_training_step(const orc_model_t* model, uint32_t B, const float* positions, const float* targets, float* params_fp32, uint16_t* params_fp16, uint16_t* grads_fp16, float* m1, float* m2, uint32_t* steps, int run_optimizer, float* loss_values) {
	return orc_training_step_shard(model, B, B, positions, targets, params_fp32, params_fp16, grads_fp16, nullptr, m1, m2, steps, run_optimizer, loss_values);
}

// One rank's shard of a global batch (new: the reference has no multi-GPU path). The loss is normalised over the global
// batch so that summing the shards' gradients reproduces the single-process gradients. If grad_sums is non-null it
// receives the exact (double) gradient sums of this shard: ranks add those and round once, like the device's fp32 path.
double orc_training_step_shard(const orc_model_t* model, uint32_t B, uint32_t B_global, const float* positions, const float* targets, float* params_fp32, uint16_t* params_fp16, uint16_t* grads_fp16, double* grad_sums, float* m1, float* m2, uint32_t* steps, int run_optimizer, float* loss_values) {
	const orc_grid_t* g = model->grid;
	const orc_mlp_t* m = model->mlp;
	const size_t n_mlp = m->n_params, n_grid = g->n_params, n = n_mlp + n_grid;
	const uint32_t OUT = m->padded_out_width;

	std::vector<uint16_t> enc((size_t)g->padded_width * B), hidden((size_t)m->n_hidden_layers * B * m->width), out((size_t)B * OUT);
	orc_grid_forward(g, B, positions, params_fp16 + n_mlp, enc.data(), nullptr);
	orc_mlp_forward(m, B, model->accum_mode, params_fp16, enc.data(), hidden.data(), out.data());

	std::vector<float> L((size_t)B * OUT);
	std::vector<uint16_t> dL_dy((size_t)B * OUT);
	orc_loss_n(model->loss_type, B, OUT, m->out_width, model->loss_scale, B_global * m->out_width, out.data(), targets, L.data(), dL_dy.data());
	double loss_sum = 0;
	for (size_t i = 0; i < L.size(); ++i) loss_sum += L[i];
	if (loss_values) {
		for (uint32_t i = 0; i < B; ++i)
			for (uint32_t j = 0; j < m->out_width; ++j) loss_values[(size_t)i * m->out_width + j] = L[(size_t)i * OUT + j];
	}

	// Transfer of the output activation happens ahead of the backward kernel, from the forward OUTPUT values
	// (fully_fused_mlp.cu:758-762, activation_backward_output_gpu -> warp_activation_backward, common_device.h:354-420).
	if (m->output_activation != ORC_ACT_NONE) {
		for (size_t i = 0; i < dL_dy.size(); ++i) dL_dy[i] = half_to_bits(activation_bwd(m->output_activation, bits_to_half(dL_dy[i]), bits_to_half(out[i])));
	}

	std::vector<double> dW(n_mlp), dG(n_grid);
	std::vector<uint16_t> d_enc((size_t)g->padded_width * B);
	orc_mlp_backward(m, B, model->accum_mode, params_fp16, enc.data(), hidden.data(), dL_dy.data(), dW.data(), d_enc.data());
	orc_grid_backward(g, B, positions, d_enc.data(), dG.data());
	for (size_t i = 0; i < n_mlp; ++i) grads_fp16[i] = d2h(dW[i]);
	for (size_t i = 0; i < n_grid; ++i) grads_fp16[n_mlp + i] = d2h(dG[i]);
	if (grad_sums) {
		for (size_t i = 0; i < n_mlp; ++i) grad_sums[i] = dW[i];
		for (size_t i = 0; i < n_grid; ++i) grad_sums[n_mlp + i] = dG[i];
	}

	if (run_optimizer) {
		orc_adam_step(model->adam, n, n_mlp, model->loss_scale, params_fp32, params_fp16, grads_fp16, m1, m2, steps);
	}
	return loss_sum;
}

void orc_inference(const orc_model_t* model, uint32_t B, const float* positions, const uint16_t* params_fp16, float* out) {
	const orc_grid_t* g = model->grid;
	const orc_mlp_t* m = model->mlp;
	std::vector<uint16_t> enc((size_t)g->padded_width * B), o16((size_t)B * m->padded_out_width);
	orc_grid_forward(g, B, positions, params_fp16 + m->n_params, enc.data(), nullptr);
	orc_mlp_forward(m, B, model->accum_mode, params_fp16, enc.data(), nullptr, o16.data());
	for (uint32_t i = 0; i < B; ++i)
		for (uint32_t j = 0; j < m->out_width; ++j) out[(size_t)i * m->out_width + j] = h2f(o16[(size_t)i * m->padded_out_width + j]);
}

}  // extern "C"
