// grid_bwd_bwd_oracle.cpp -- CPU restatement, in double, of the reference's second-order derivatives of the grid encoding
// (GridEncodingTemplated::backward_backward_input_impl, include/tiny-cuda-nn/encodings/grid.h:910-1042). TEST INFRASTRUCTURE ONLY:
// loaded by tests/grid_bwd_bwd_oracle.py; the product (tiny-cuda-nn_b200/) never links it. It uses the grid description of
// oracle/oracle_cpu.h (orc_grid_t, filled by orc_grid_setup) so that both restatements index the same tables.
//
// Integer arithmetic (cells, indices) follows the reference bit for bit; the real arithmetic is done in double, so the device's
// fp16 / fp32 results are compared against exact values. Positions are converted to the fractional cell position in fp32 exactly
// as pos_fract does (common_device.h:1031-1043), so that every sample lands in the same cell as on the device.
#include "../../oracle/oracle_cpu.h"

#include <cmath>
#include <cstring>
#include <vector>

namespace {

inline float h2f(uint16_t b) {
	_Float16 h;
	std::memcpy(&h, &b, 2);
	return (float)h;
}

// common_device.h:886-895 (grid_resolution) and :787-791 + :847-884 (coherent_prime_hash, grid_index)
inline uint32_t grid_resolution(float scale) { return (uint32_t)ceilf(scale) + 1; }
inline uint32_t grid_index(uint32_t D, uint32_t grid_type, uint32_t hashmap_size, uint32_t resolution, const uint32_t* pos_grid) {
	static const uint32_t MAX_BASES[] = {0x0, 0xFFFFFFFF, 0xFFFF, 0x659, 0xFF};
	static const uint32_t factors[4] = {1u, 2654435761u, 805459861u, 3674653429u};
	uint32_t stride = 1, index = 0;
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
		for (uint32_t dim = 0; dim < D; ++dim) index ^= pos_grid[dim] * factors[dim];
	}
	return index % hashmap_size;
}

// pos_fract with the interpolation's derivatives (common_device.h:970-1043): the cell and the raw fractional position in fp32,
// then t = S(p), S'(p), S''(p) in double (identity: 1, 0; smoothstep: 3p^2 - 2p^3, 6p(1-p), 6 - 12p).
struct Pos {
	uint32_t grid[4];
	double t[4], d1[4], d2[4];
};
inline Pos pos_fract(uint32_t D, const float* x, float scale, uint32_t interpolation) {
	Pos r;
	for (uint32_t d = 0; d < D; ++d) {
		float p = fmaf(scale, x[d], 0.5f);
		const float tmp = floorf(p);
		r.grid[d] = (uint32_t)(int)tmp;
		const double pd = (double)(p - tmp);
		const bool smooth = interpolation == ORC_INTERP_SMOOTHSTEP;
		r.t[d] = smooth ? pd * pd * (3.0 - 2.0 * pd) : pd;
		r.d1[d] = smooth ? 6.0 * pd * (1.0 - pd) : 1.0;
		r.d2[d] = smooth ? 6.0 - 12.0 * pd : 0.0;
	}
	return r;
}

}  // namespace

extern "C" {

// positions [B][D] fp32; grid fp16 bits [n_params]; dL_denc SoA [padded_width][B] fp16 bits (u); dL_ddLdx [B][D] fp32 (v).
// max_level: fraction of the levels that is active (grid.h:69-92; level l takes part while l < max_level * L + 1e-3).
// Outputs (each may be NULL): dL_dparams double [n_params]; dL_ddLdoutput double [B][L * F]; dL_dinput double [B][D].
void orc_grid_backward_backward_input(const orc_grid_t* g, uint32_t B, const float* positions, const uint16_t* grid, const uint16_t* dL_denc, const float* dL_ddLdx,
                                      float max_level, double* dL_dparams, double* dL_ddLdoutput, double* dL_dinput) {
	const uint32_t D = g->n_pos_dims, F = g->n_features_per_level, L = g->n_levels;
	const float n_active = (max_level * (float)(L * F)) / (float)F;
	const bool linear_or_smooth = g->interpolation != ORC_INTERP_NEAREST;  // Nearest: all three are zero (grid.h:420-423, 522-525; dy_dx grid.h:120-133)
	if (dL_dparams) std::memset(dL_dparams, 0, sizeof(double) * g->n_params);
	if (dL_ddLdoutput) std::memset(dL_ddLdoutput, 0, sizeof(double) * (size_t)B * L * F);
	if (dL_dinput) std::memset(dL_dinput, 0, sizeof(double) * (size_t)B * D);
	if (!linear_or_smooth) return;
	for (uint32_t level = 0; level < L; ++level) {
		if ((float)level >= n_active + 1e-3f) break;
		const uint32_t hashmap_size = g->offsets[level + 1] - g->offsets[level];
		const float scale = g->scales[level];
		const uint32_t resolution = grid_resolution(scale);
		const uint16_t* level_grid = grid + (size_t)g->offsets[level] * F;
		for (uint32_t i = 0; i < B; ++i) {
			const float* x = positions + (size_t)i * D;
			const float* v = dL_ddLdx + (size_t)i * D;
			const Pos p = pos_fract(D, x, scale, g->interpolation);
			double u[8];
			for (uint32_t f = 0; f < F; ++f) u[f] = h2f(dL_denc[i + (size_t)(level * F + f) * B]);
			// corner `idx` along the other dimensions of `grad_dim`: index of its left / right corner and the product of the other weights
			auto corner_pair = [&](uint32_t grad_dim, uint32_t idx, uint32_t& left, uint32_t& right) {
				double weight = 1.0;
				uint32_t local[4];
				for (uint32_t non_grad_dim = 0; non_grad_dim + 1 < D; ++non_grad_dim) {
					const uint32_t dim = non_grad_dim >= grad_dim ? non_grad_dim + 1 : non_grad_dim;
					if ((idx & (1u << non_grad_dim)) == 0) {
						weight *= 1.0 - p.t[dim];
						local[dim] = p.grid[dim];
					} else {
						weight *= p.t[dim];
						local[dim] = p.grid[dim] + 1;
					}
				}
				local[grad_dim] = p.grid[grad_dim];
				left = grid_index(D, g->grid_type, hashmap_size, resolution, local);
				local[grad_dim] = p.grid[grad_dim] + 1;
				right = grid_index(D, g->grid_type, hashmap_size, resolution, local);
				return weight;
			};
			// kernel_grid_backward_input_backward_grid (grid.h:425-454): +-scale * v_d * S'(p_d) * (other weights) * u into left / right
			if (dL_dparams) {
				double* level_grad = dL_dparams + (size_t)g->offsets[level] * F;
				for (uint32_t grad_dim = 0; grad_dim < D; ++grad_dim) {
					const double grad_in = (double)scale * v[grad_dim] * p.d1[grad_dim];
					for (uint32_t idx = 0; idx < (1u << (D - 1)); ++idx) {
						uint32_t left, right;
						const double weight = grad_in * corner_pair(grad_dim, idx, left, right);
						for (uint32_t f = 0; f < F; ++f) {
							level_grad[(size_t)left * F + f] -= weight * u[f];
							level_grad[(size_t)right * F + f] += weight * u[f];
						}
					}
				}
			}
			// kernel_grid's dy_dx (grid.h:171-210) contracted with v: kernel_grid_backward_input_backward_dLdoutput (grid.h:625-655)
			if (dL_ddLdoutput) {
				for (uint32_t f = 0; f < F; ++f) {
					double result = 0.0;
					for (uint32_t grad_dim = 0; grad_dim < D; ++grad_dim) {
						double dy_dx = 0.0;
						for (uint32_t idx = 0; idx < (1u << (D - 1)); ++idx) {
							uint32_t left, right;
							const double weight = corner_pair(grad_dim, idx, left, right);
							dy_dx += (double)scale * weight * ((double)h2f(level_grid[(size_t)right * F + f]) - (double)h2f(level_grid[(size_t)left * F + f])) * p.d1[grad_dim];
						}
						result += dy_dx * v[grad_dim];
					}
					dL_ddLdoutput[(size_t)i * L * F + level * F + f] = result;
				}
			}
			// kernel_grid_backward_input_backward_input (grid.h:527-622)
			if (dL_dinput) {
				auto calc = [&](const uint32_t* local, double weight) {
					const uint32_t index = grid_index(D, g->grid_type, hashmap_size, resolution, local);
					double s = 0.0;
					for (uint32_t f = 0; f < F; ++f) s += (double)h2f(level_grid[(size_t)index * F + f]) * u[f] * weight;
					return s;
				};
				for (uint32_t grad_dim = 0; grad_dim < D; ++grad_dim) {
					double grad_out = 0.0;
					for (uint32_t idx = 0; idx < (1u << (D - 1)); ++idx) {
						uint32_t local[4];
						// diagonal of the Hessian, d(dy/dx_d)/dx_d: Smoothstep only (Linear's S'' is zero)
						if (g->interpolation == ORC_INTERP_SMOOTHSTEP) {
							double w = (double)scale * scale * v[grad_dim] * p.d2[grad_dim];
							for (uint32_t non_grad_dim = 0; non_grad_dim + 1 < D; ++non_grad_dim) {
								const uint32_t dim = non_grad_dim >= grad_dim ? non_grad_dim + 1 : non_grad_dim;
								if ((idx & (1u << non_grad_dim)) == 0) {
									w *= 1.0 - p.t[dim];
									local[dim] = p.grid[dim];
								} else {
									w *= p.t[dim];
									local[dim] = p.grid[dim] + 1;
								}
							}
							local[grad_dim] = p.grid[grad_dim];
							grad_out += calc(local, -w);
							local[grad_dim] = p.grid[grad_dim] + 1;
							grad_out += calc(local, w);
						}
						// the other entries of the Hessian, d(dy/dx_o)/dx_d for o != d
						for (uint32_t other = 0; other + 1 < D; ++other) {
							const uint32_t real_other = other >= grad_dim ? other + 1 : other;
							double w = (double)scale * scale * v[real_other] * p.d1[real_other] * p.d1[grad_dim];
							for (uint32_t non_grad_dim = 0; non_grad_dim + 1 < D; ++non_grad_dim) {
								const uint32_t dim = non_grad_dim >= real_other ? non_grad_dim + 1 : non_grad_dim;
								if ((idx & (1u << non_grad_dim)) == 0) {
									w *= dim != grad_dim ? 1.0 - p.t[dim] : -1.0;
									local[dim] = p.grid[dim];
								} else {
									if (dim != grad_dim) w *= p.t[dim];
									local[dim] = p.grid[dim] + 1;
								}
							}
							local[real_other] = p.grid[real_other];
							grad_out += calc(local, -w);
							local[real_other] = p.grid[real_other] + 1;
							grad_out += calc(local, w);
						}
					}
					dL_dinput[(size_t)i * D + grad_dim] += grad_out;
				}
			}
		}
	}
}

}  // extern "C"
