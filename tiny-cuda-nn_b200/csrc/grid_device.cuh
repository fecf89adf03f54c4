// grid_device.cuh -- per-sample multiresolution grid arithmetic shared by the standalone encoding kernels and the
// fused training kernel. Integer results (cells, indices) are bit-exact with the reference:
//   pos_fract            common_device.h:1031-1043
//   grid_index           common_device.h:847-884 (dense stride accumulation, coherent-prime hash, modulo)
//   coherent_prime_hash  common_device.h:787-791
//   N-linear weights     grid.h:142-163 (fp32 products in corner order, bit d of the corner index <-> dim d)
#pragma once
#include "common.cuh"

namespace tcnnb {

enum : uint32_t { LEVEL_DENSE = 0, LEVEL_HASH = 1, LEVEL_DEGENERATE = 2 };

__device__ __forceinline__ float smoothstep_f(float x) { return x * x * (3.0f - 2.0f * x); }

template <uint32_t D>
struct CellPos {
	uint32_t cell[D];
	float frac[D];
};

template <uint32_t D>
__device__ __forceinline__ void pos_fract(const float (&x)[D], float scale, uint32_t interpolation, CellPos<D>& out) {
#pragma unroll
	for (uint32_t d = 0; d < D; ++d) {
		float p = __fmaf_rn(scale, x[d], 0.5f);
		const float t = floorf(p);
		out.cell[d] = (uint32_t)(int)t;
		p -= t;
		out.frac[d] = interpolation == INTERP_SMOOTHSTEP ? smoothstep_f(p) : p;
	}
}

// index % size without a division wherever the level allows it (warp-uniform choice).
__device__ __forceinline__ uint32_t level_mod(const LevelInfo& lv, uint32_t index) {
	if (lv.pow2_mask) return index & lv.pow2_mask;
	if (lv.small_mod) {
		// in-range positions give index < 2 * size; positions outside [0,1) (wrap-around indexing) take the exact slow path
		index -= index >= lv.size ? lv.size : 0u;
		if (index >= lv.size) index %= lv.size;
		return index;
	}
	return index % lv.size;
}

// Entry index of one corner inside its level.
template <uint32_t D>
__device__ __forceinline__ uint32_t corner_index(const LevelInfo& lv, const uint32_t (&c)[D]) {
	uint32_t index = 0;
	if (lv.use_hash == LEVEL_HASH) {
		index = c[0];
		if (D > 1) index ^= c[1] * 2654435761u;
		if (D > 2) index ^= c[2] * 805459861u;
		if (D > 3) index ^= c[3] * 3674653429u;
	} else if (lv.use_hash == LEVEL_DENSE) {
		uint32_t stride = 1;
#pragma unroll
		for (uint32_t d = 0; d < D; ++d) {
			index += c[d] * stride;
			stride *= lv.resolution;
		}
	}
	return level_mod(lv, index);
}

// Corner `idx` of the cell: coordinates and fp32 interpolation weight, multiplied in dimension order like the reference.
template <uint32_t D>
__device__ __forceinline__ float corner(const CellPos<D>& p, uint32_t idx, uint32_t (&c)[D]) {
	float w = 1.0f;
#pragma unroll
	for (uint32_t d = 0; d < D; ++d) {
		if ((idx & (1u << d)) == 0) {
			w *= 1.0f - p.frac[d];
			c[d] = p.cell[d];
		} else {
			w *= p.frac[d];
			c[d] = p.cell[d] + 1;
		}
	}
	return w;
}

// The two corners of a cell that differ only in x (corner indices 2*pair and 2*pair+1): entry indices and weights.
// For a hashed level with a power-of-two table the coherent-prime hash multiplies x by 1, so for an even cell x the
// two entries are idx and idx^1, i.e. they share one aligned 8-byte slot; on dense levels they are idx and idx+1.
// `paired` tells the caller that one 64-bit access at (idx0 & ~1) covers both.
template <uint32_t D>
struct CornerPair {
	uint32_t idx0, idx1;
	float w0, w1;
	bool paired;
};

template <uint32_t D>
__device__ __forceinline__ CornerPair<D> corner_pair(const LevelInfo& lv, const CellPos<D>& p, uint32_t pair) {
	CornerPair<D> r;
	uint32_t c0[D], c1[D];
	r.w0 = corner<D>(p, 2 * pair, c0);
	r.w1 = corner<D>(p, 2 * pair + 1, c1);
	// Both corners share every coordinate but x: hash / stride contribution of dims 1.. is computed once.
	if (lv.use_hash == LEVEL_HASH) {
		uint32_t rest = 0;
		if (D > 1) rest ^= c0[1] * 2654435761u;
		if (D > 2) rest ^= c0[2] * 805459861u;
		if (D > 3) rest ^= c0[3] * 3674653429u;
		r.idx0 = level_mod(lv, c0[0] ^ rest);
		r.idx1 = level_mod(lv, c1[0] ^ rest);
	} else if (lv.use_hash == LEVEL_DENSE) {
		uint32_t rest = 0, stride = lv.resolution;
#pragma unroll
		for (uint32_t d = 1; d < D; ++d) {
			rest += c0[d] * stride;
			stride *= lv.resolution;
		}
		r.idx0 = level_mod(lv, c0[0] + rest);
		r.idx1 = level_mod(lv, c1[0] + rest);
	} else {
		r.idx0 = r.idx1 = 0;
	}
	r.paired = (r.idx0 ^ r.idx1) == 1u;
	return r;
}

// All 2^D corners of one cell at one level: interpolation weights in the reference's multiplication order
// (weight = 1 * t_x * t_y * t_z, grid.h:146-157), entry indices, and which x-pairs (corners 2k, 2k+1) share an aligned
// 8-byte slot. Contributions of the non-x dimensions to the hash / dense stride are computed once per value, not per corner.
template <uint32_t D>
struct LevelCorners {
	float frac[D];  // the (interpolation-mapped) fractional position the weights are built from
	float w[1u << D];
	uint32_t idx[1u << D];
	uint32_t paired;  // bit k: pair k is covered by one 64-bit access at (idx[2k] & ~1)
};

// weights: w[i] for corner bits (b0 = x, b1 = y, ...), built dimension by dimension -> ((t_x * t_y) * t_z)
template <uint32_t D>
__device__ __forceinline__ void corner_weights(const float (&frac)[D], float (&w)[1u << D]) {
	w[0] = 1.0f - frac[0];
	w[1] = frac[0];
#pragma unroll
	for (uint32_t d = 1; d < D; ++d) {
		const float hi = frac[d], lo = 1.0f - frac[d];
#pragma unroll
		for (uint32_t i = 0; i < (1u << d); ++i) {
			w[i + (1u << d)] = w[i] * hi;
			w[i] = w[i] * lo;
		}
	}
}

template <uint32_t D>
__device__ __forceinline__ void level_corners(const LevelInfo& lv, const float (&x)[D], uint32_t interpolation, LevelCorners<D>& out) {
	CellPos<D> cp;
	pos_fract<D>(x, lv.scale, interpolation, cp);
#pragma unroll
	for (uint32_t d = 0; d < D; ++d) out.frac[d] = cp.frac[d];
	corner_weights<D>(cp.frac, out.w);
	// indices: two straight-line paths selected by a warp-uniform test (all lanes of a warp work on the same level)
	uint32_t rest[1u << (D - 1)];
	rest[0] = 0;
	if (lv.use_hash == LEVEL_HASH && lv.pow2_mask != 0) {
		// hashed level, power-of-two table: index = (x ^ y*p1 ^ z*p2) & mask; the x-pair shares an aligned slot iff x is even
		constexpr uint32_t primes[4] = {1u, 2654435761u, 805459861u, 3674653429u};
#pragma unroll
		for (uint32_t d = 1; d < D; ++d) {
			const uint32_t h0 = cp.cell[d] * primes[d], h1 = h0 + primes[d];
#pragma unroll
			for (uint32_t i = 0; i < (1u << (d - 1)); ++i) {
				rest[i + (1u << (d - 1))] = rest[i] ^ h1;
				rest[i] = rest[i] ^ h0;
			}
		}
		const uint32_t x0 = cp.cell[0], x1 = cp.cell[0] + 1u;
#pragma unroll
		for (uint32_t k = 0; k < (1u << (D - 1)); ++k) {
			out.idx[2 * k] = (x0 ^ rest[k]) & lv.pow2_mask;
			out.idx[2 * k + 1] = (x1 ^ rest[k]) & lv.pow2_mask;
		}
		out.paired = (x0 & 1u) ? 0u : (1u << (1u << (D - 1))) - 1u;
		return;
	}
	if (lv.use_hash == LEVEL_HASH) {
		constexpr uint32_t primes[4] = {1u, 2654435761u, 805459861u, 3674653429u};
#pragma unroll
		for (uint32_t d = 1; d < D; ++d) {
			const uint32_t h0 = cp.cell[d] * primes[d], h1 = h0 + primes[d];
#pragma unroll
			for (uint32_t i = 0; i < (1u << (d - 1)); ++i) {
				rest[i + (1u << (d - 1))] = rest[i] ^ h1;
				rest[i] = rest[i] ^ h0;
			}
		}
#pragma unroll
		for (uint32_t k = 0; k < (1u << (D - 1)); ++k) {
			out.idx[2 * k] = (cp.cell[0] ^ rest[k]) % lv.size;
			out.idx[2 * k + 1] = ((cp.cell[0] + 1u) ^ rest[k]) % lv.size;
		}
	} else if (lv.use_hash == LEVEL_DENSE) {
		uint32_t stride = lv.resolution;
#pragma unroll
		for (uint32_t d = 1; d < D; ++d) {
			const uint32_t s0 = cp.cell[d] * stride, s1 = s0 + stride;
#pragma unroll
			for (uint32_t i = 0; i < (1u << (d - 1)); ++i) {
				rest[i + (1u << (d - 1))] = rest[i] + s1;
				rest[i] = rest[i] + s0;
			}
			stride *= lv.resolution;
		}
		bool slow = false;
#pragma unroll
		for (uint32_t k = 0; k < (1u << (D - 1)); ++k) {
			// in-range positions give index < 2 * size on a level that holds its full dense grid (small_mod)
			uint32_t i0 = cp.cell[0] + rest[k], i1 = i0 + 1u;
			i0 -= i0 >= lv.size ? lv.size : 0u;
			i1 -= i1 >= lv.size ? lv.size : 0u;
			slow |= i0 >= lv.size || i1 >= lv.size;
			out.idx[2 * k] = i0;
			out.idx[2 * k + 1] = i1;
		}
		if (slow || !lv.small_mod) {  // tiled grids, or positions outside [0,1): exact modulo (wrap-around indexing)
#pragma unroll
			for (uint32_t k = 0; k < (1u << D); ++k) out.idx[k] %= lv.size;
		}
	} else {
#pragma unroll
		for (uint32_t i = 0; i < (1u << D); ++i) out.idx[i] = 0;
	}
	out.paired = 0;
#pragma unroll
	for (uint32_t k = 0; k < (1u << (D - 1)); ++k) {
		if ((out.idx[2 * k] ^ out.idx[2 * k + 1]) == 1u) out.paired |= 1u << k;
	}
}

// max_level = (max_level * num_grid_features) / N_FEATURES_PER_LEVEL (grid.h:69-73). A level is active while
// level < grid_active_levels(...) + 1e-3: the forward pass and every derivative of it leave the other levels out.
__device__ __forceinline__ float grid_active_levels(float max_level, uint32_t n_levels, uint32_t n_features_per_level) {
	return (max_level * (float)(n_levels * n_features_per_level)) / (float)n_features_per_level;
}

// One table entry (the F features of one grid vertex), read and written with one access of F * 2 bytes.
template <uint32_t F>
struct Entry {
	__half v[F];
};

template <uint32_t F>
__device__ __forceinline__ Entry<F> load_entry(const __half* __restrict__ p) {
	Entry<F> e;
	if (F == 1) {
		e.v[0] = __ldg(p);
	} else if (F == 2) {
		*reinterpret_cast<uint32_t*>(e.v) = __ldg(reinterpret_cast<const uint32_t*>(p));
	} else if (F == 4) {
		*reinterpret_cast<uint2*>(e.v) = __ldg(reinterpret_cast<const uint2*>(p));
	} else {
		*reinterpret_cast<uint4*>(e.v) = __ldg(reinterpret_cast<const uint4*>(p));
	}
	return e;
}

template <uint32_t F>
__device__ __forceinline__ void store_entry(__half* p, const Entry<F>& e) {
	if (F == 1) {
		p[0] = e.v[0];
	} else if (F == 2) {
		*reinterpret_cast<uint32_t*>(p) = *reinterpret_cast<const uint32_t*>(e.v);
	} else if (F == 4) {
		*reinterpret_cast<uint2*>(p) = *reinterpret_cast<const uint2*>(e.v);
	} else {
		*reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(e.v);
	}
}

// one reduction per corner: f16x2, v2.f16x2 or v4.f16x2 (an entry of F fp16 is F * 2 bytes and aligned to that)
template <uint32_t F>
__device__ __forceinline__ void red_entry(__half* p, const Entry<F>& e) {
	const uint32_t* w = reinterpret_cast<const uint32_t*>(e.v);
	if (F == 2) {
		asm volatile("red.relaxed.gpu.global.add.noftz.f16x2 [%0], %1;" ::"l"(p), "r"(w[0]) : "memory");
	} else if (F == 4) {
		asm volatile("red.relaxed.gpu.global.add.noftz.v2.f16x2 [%0], {%1, %2};" ::"l"(p), "r"(w[0]), "r"(w[1]) : "memory");
	} else if (F == 8) {
		asm volatile("red.relaxed.gpu.global.add.noftz.v4.f16x2 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3]) : "memory");
	}
}

template <uint32_t D>
__device__ __forceinline__ void load_position(const float* __restrict__ positions, uint32_t stride, uint32_t i, float (&x)[D]) {
#pragma unroll
	for (uint32_t d = 0; d < D; ++d) x[d] = __ldg(positions + (size_t)i * stride + d);
}

// Gather the two fp16x2 entries of a corner pair: two independent 4-byte loads, or one 8-byte load (`merge`, below).
// Deliberately NO arithmetic on the loaded values here: callers
// keep several levels of loads in flight, and anything that touches a value -- an earlier version fetched the aligned 8-byte slot
// and SELECTED the two halves -- makes the warp wait for the loads it has just issued (that version ran at a depth of one
// level whatever the software pipeline said; scripts/ws_timeline.py: gather 10.2 -> see DESIGN.md section 3.1).
// `streaming` (warp-uniform): the loads do not allocate in L1. The training kernel uses it for the hashed levels, whose entries
// are spread at random over megabytes and are rarely met again by the same SM, so that the L1 (smaller in training: park and dy
// tiles) is left to the dense coarse levels that neighbouring samples of the binned batch share. Measured in DESIGN.md 5.1.
__device__ __forceinline__ uint32_t ld_table(const uint32_t* p, bool streaming) {
	uint32_t v;
	if (streaming) asm("ld.global.nc.L1::no_allocate.b32 %0, [%1];" : "=r"(v) : "l"(p));
	else v = __ldg(p);
	return v;
}
// `merge`: the pair shares an aligned 8-byte slot (`paired`) and the level base is 16-byte aligned (LevelInfo::wide_ok). The
// pair is then fetched with ONE 8-byte streaming load, which costs one L2 request instead of two (with L1 allocation the second
// 4-byte load hit the sector the first had just brought in, so merging saved nothing; measured in DESIGN.md 5.1). The words
// arrive in memory order, v0 = entry (idx0 & ~1): the return value is 1 when they are the other way round from corner order
// (idx0 odd -- the hash XORs the x bit with the other coordinates' bits), and the caller swaps them when it consumes them.
__device__ __forceinline__ uint32_t gather_pair_f16x2(const uint32_t* __restrict__ table, uint32_t idx0, uint32_t idx1, bool merge, bool streaming, uint32_t& v0, uint32_t& v1) {
	if (merge) {
		asm("ld.global.nc.L1::no_allocate.v2.b32 {%0, %1}, [%2];" : "=r"(v0), "=r"(v1) : "l"(table + (idx0 & ~1u)));
		return idx0 & 1u;
	}
	v0 = ld_table(table + idx0, streaming);
	v1 = ld_table(table + idx1, streaming);
	return 0u;
}

// Scatter-add two fp16x2 addends of a corner pair (red.global.add.noftz.f16x2 is what the reference's
// atomic_add_gmem(__half2) lowers to, vec.h:328-336). The L2 retires a fixed number of reduction OPERATIONS per second
// whatever their width (4, 8 and 16 bytes measure the same, scripts/experiments/red_bench.cu), so the pair goes out as ONE
// operation whenever both entries lie in one aligned 16-byte group: a 64-bit reduction if they share an aligned slot
// (x even), a 128-bit one with zero addends in the two other entries if they straddle the middle of a group (x % 4 == 1,
// dense or hashed: idx0 ^ idx1 == 3; adding +0 leaves the other entries unchanged). Otherwise two 32-bit reductions.
// (Sending the x-even case through the 128-bit form as well -- two shapes instead of three -- measured 2 % slower.)
// `wide_ok`: the level base is 16-byte aligned (LevelInfo::wide_ok), which the merged forms need; warp-uniform.
__device__ __forceinline__ void scatter_pair_f16x2(uint32_t* __restrict__ table, uint32_t idx0, uint32_t idx1, bool paired, bool wide_ok, uint32_t a0, uint32_t a1) {
	if (!wide_ok) {
		asm volatile("red.relaxed.gpu.global.add.noftz.f16x2 [%0], %1;" ::"l"(table + idx0), "r"(a0) : "memory");
		asm volatile("red.relaxed.gpu.global.add.noftz.f16x2 [%0], %1;" ::"l"(table + idx1), "r"(a1) : "memory");
	} else if (paired) {
		const bool odd = idx0 & 1u;
		const uint32_t lo = odd ? a1 : a0, hi = odd ? a0 : a1;
		asm volatile("red.relaxed.gpu.global.add.noftz.v2.f16x2 [%0], {%1, %2};" ::"l"(table + (idx0 & ~1u)), "r"(lo), "r"(hi) : "memory");
	} else if ((idx0 ^ idx1) == 3u) {
		const uint32_t p0 = idx0 & 3u;  // idx1 sits at p0 ^ 3
		const uint32_t v0 = p0 == 0u ? a0 : (p0 == 3u ? a1 : 0u);
		const uint32_t v1 = p0 == 1u ? a0 : (p0 == 2u ? a1 : 0u);
		const uint32_t v2 = p0 == 2u ? a0 : (p0 == 1u ? a1 : 0u);
		const uint32_t v3 = p0 == 3u ? a0 : (p0 == 0u ? a1 : 0u);
		asm volatile("red.relaxed.gpu.global.add.noftz.v4.f16x2 [%0], {%1, %2, %3, %4};" ::"l"(table + (idx0 & ~3u)), "r"(v0), "r"(v1), "r"(v2), "r"(v3) : "memory");
	} else {
		asm volatile("red.relaxed.gpu.global.add.noftz.f16x2 [%0], %1;" ::"l"(table + idx0), "r"(a0) : "memory");
		asm volatile("red.relaxed.gpu.global.add.noftz.f16x2 [%0], %1;" ::"l"(table + idx1), "r"(a1) : "memory");
	}
}

}  // namespace tcnnb
