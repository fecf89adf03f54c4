/* tiny-cuda-nn/random.h -- default_rng_t and generate_random_uniform (reference: random.h:40-69, common.h:262 `default_rng_t = pcg32`).
 * The generator is the published PCG-XSH-RR 64/32 (O'Neill 2014) with the stream constant the reference's pcg32 uses; the fill
 * runs on the device inside libtcnn_b200 with the reference's jump-ahead pattern (thread i draws 4 consecutive numbers after
 * advance(4 i)), so a given (seed, n) produces the same numbers as tiny-cuda-nn. */
#pragma once
#include "common.h"

namespace tcnn {

struct pcg32 {
	static constexpr uint64_t MULT = 0x5851f42d4c957f2dULL;
	uint64_t state, inc;

	pcg32(uint64_t initstate = 0x853c49e6748fea9bULL, uint64_t initseq = 1u) { seed(initstate, initseq); }
	void seed(uint64_t initstate, uint64_t initseq = 1u) {
		state = 0;
		inc = (initseq << 1u) | 1u;
		next_uint();
		state += initstate;
		next_uint();
	}
	uint32_t next_uint() {
		const uint64_t old = state;
		state = old * MULT + inc;
		const uint32_t xorshifted = (uint32_t)(((old >> 18u) ^ old) >> 27u);
		const uint32_t rot = (uint32_t)(old >> 59u);
		return (xorshifted >> rot) | (xorshifted << ((~rot + 1u) & 31u));
	}
	float next_float() {
		union { uint32_t u; float f; } x;
		x.u = (next_uint() >> 9) | 0x3f800000u;
		return x.f - 1.0f;
	}
	/* O(log delta) jump-ahead (Brown, "Random number generation with arbitrary strides") */
	void advance(uint64_t delta) {
		uint64_t cur_mult = MULT, cur_plus = inc, acc_mult = 1u, acc_plus = 0u;
		while (delta > 0) {
			if (delta & 1) {
				acc_mult *= cur_mult;
				acc_plus = acc_plus * cur_mult + cur_plus;
			}
			cur_plus = (cur_mult + 1) * cur_plus;
			cur_mult *= cur_mult;
			delta >>= 1;
		}
		state = acc_mult * state + acc_plus;
	}
};

using default_rng_t = pcg32;

/* random.h:56-69: fills `out` with n uniform numbers in [lower, upper) on `stream` and advances `rng` by n. T = float or __half (each
 * draw rounded to half, then scaled and shifted in half arithmetic, as the reference's kernel does for T = __half). */
template <typename T, typename RNG>
void generate_random_uniform(cudaStream_t stream, RNG& rng, size_t n_elements, T* out, const T lower = (T)0.0, const T upper = (T)1.0) {
	static_assert(sizeof(T) == sizeof(float) || sizeof(T) == sizeof(__half), "generate_random_uniform: float or __half only");
	if (sizeof(T) == sizeof(float)) {
		TCNNB_CHECK_THROW(tcnnb_generate_random_uniform((tcnnb_stream)stream, rng.state, rng.inc, (uint64_t)n_elements, (float*)out, (float)lower, (float)upper));
	} else {
		TCNNB_CHECK_THROW(tcnnb_generate_random_uniform_half((tcnnb_stream)stream, rng.state, rng.inc, (uint64_t)n_elements, out, (float)lower, (float)upper));
	}
	rng.advance(n_elements);
}

template <typename T, typename RNG>
void generate_random_uniform(RNG& rng, size_t n_elements, T* out, const T lower = (T)0.0, const T upper = (T)1.0) {
	generate_random_uniform(nullptr, rng, n_elements, out, lower, upper);
}

}  // namespace tcnn
