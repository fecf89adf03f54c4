// host_common.h -- host-side helpers shared by the C-ABI translation units (model.cu: trainer / module tiers; network.cu and
// encoding.cu: the stand-alone network and encoding tiers): error plumbing, device buffers, the device and batch checks, the host
// pcg32, name tables.
#pragma once
#include "common.cuh"

#include <algorithm>
#include <atomic>
#include <cstring>
#include <stdexcept>
#include <string>

namespace tcnnb {

extern std::atomic<uint64_t> g_kernel_launches;
extern thread_local std::string g_last_error;

#define TCNNB_CUDA_CHECK(x)                                                                                             \
	do {                                                                                                                  \
		cudaError_t _e = (x);                                                                                               \
		if (_e != cudaSuccess) throw std::runtime_error(std::string(#x " failed: ") + cudaGetErrorString(_e));              \
	} while (0)

inline std::string to_lower(std::string s) {
	std::transform(s.begin(), s.end(), s.begin(), [](unsigned char c) { return (char)std::tolower(c); });
	return s;
}
inline bool ieq(const std::string& a, const std::string& b) { return to_lower(a) == to_lower(b); }

inline uint32_t next_multiple(uint32_t v, uint32_t d) { return ((v + d - 1) / d) * d; }
inline uint32_t powi(uint32_t base, uint32_t e) { uint32_t r = 1; for (uint32_t i = 0; i < e; ++i) r *= base; return r; }

// ---- host pcg32 (same published algorithm as the device copy in misc_kernels.cu; pcg32.h:53-69,103-112,145-166)
struct HostPcg32 {
	uint64_t state, inc;
	static constexpr uint64_t MULT = 0x5851f42d4c957f2dULL;
	HostPcg32(uint64_t initstate, uint64_t initseq = 1) {
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
		return (xorshifted >> rot) | (xorshifted << ((~rot + 1u) & 31));
	}
	float next_float() {
		const uint32_t u = (next_uint() >> 9) | 0x3f800000u;
		float f;
		std::memcpy(&f, &u, 4);
		return f - 1.0f;
	}
	void advance(uint64_t delta) {
		uint64_t cur_mult = MULT, cur_plus = inc, acc_mult = 1u, acc_plus = 0u;
		while (delta > 0) {
			if (delta & 1) {
				acc_mult *= cur_mult;
				acc_plus = acc_plus * cur_mult + cur_plus;
			}
			cur_plus = (cur_mult + 1) * cur_plus;
			cur_mult *= cur_mult;
			delta /= 2;
		}
		state = acc_mult * state + acc_plus;
	}
	Pcg32 device() const { return Pcg32{state, inc}; }
};

template <typename T>
struct DeviceBuffer {
	T* ptr = nullptr;
	size_t n = 0;
	DeviceBuffer() {}
	DeviceBuffer(const DeviceBuffer&) = delete;
	DeviceBuffer& operator=(const DeviceBuffer&) = delete;
	~DeviceBuffer() { release(); }
	void release() {
		if (ptr) cudaFree(ptr);
		ptr = nullptr;
		n = 0;
	}
	void resize(size_t count) {
		if (count == n) return;
		release();
		if (count) TCNNB_CUDA_CHECK(cudaMalloc(&ptr, count * sizeof(T)));
		n = count;
	}
	void zero(cudaStream_t stream = nullptr) {
		if (n) TCNNB_CUDA_CHECK(cudaMemsetAsync(ptr, 0, n * sizeof(T), stream));
	}
};

template <typename T>
inline void grow(DeviceBuffer<T>& b, size_t n) {
	if (b.n < n) b.resize(n);
}

// The current device must be an sm_90-class GPU (the kernels are built for sm_90a only). Returns its SM count.
inline int require_sm90() {
	int device = 0;
	TCNNB_CUDA_CHECK(cudaGetDevice(&device));
	cudaDeviceProp prop;
	TCNNB_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
	if (prop.major != 9) throw std::runtime_error("tcnn_b200 requires an sm_90-class GPU (H100); found compute capability " + std::to_string(prop.major) + "." + std::to_string(prop.minor));
	return prop.multiProcessorCount;
}

inline void check_batch(uint32_t batch) {
	if (batch == 0 || batch % BATCH_GRANULARITY != 0) {
		// object.h:169: CHECK_THROW(input.n() % BATCH_SIZE_GRANULARITY == 0)
		throw std::runtime_error("batch size " + std::to_string(batch) + " must be a non-zero multiple of " + std::to_string(BATCH_GRANULARITY));
	}
}


inline uint32_t parse_activation(const std::string& name) {
	// src/common_host.cu:70-94
	static const std::pair<const char*, uint32_t> table[] = {
		{"None", ACT_NONE}, {"ReLU", ACT_RELU}, {"LeakyReLU", ACT_LEAKY_RELU}, {"SiLU", ACT_SILU}, {"Exponential", ACT_EXPONENTIAL},
		{"Sigmoid", ACT_SIGMOID}, {"Sine", ACT_SINE}, {"Squareplus", ACT_SQUAREPLUS}, {"Softplus", ACT_SOFTPLUS}, {"Tanh", ACT_TANH},
	};
	for (auto& kv : table) if (ieq(name, kv.first)) return kv.second;
	throw std::runtime_error("Invalid activation name: " + name);
}

inline const char* activation_name(uint32_t a) {
	switch (a) {
		case ACT_NONE: return "None";
		case ACT_RELU: return "ReLU";
		case ACT_LEAKY_RELU: return "LeakyReLU";
		case ACT_SILU: return "SiLU";
		case ACT_EXPONENTIAL: return "Exponential";
		case ACT_SIGMOID: return "Sigmoid";
		case ACT_SINE: return "Sine";
		case ACT_SQUAREPLUS: return "Squareplus";
		case ACT_SOFTPLUS: return "Softplus";
		case ACT_TANH: return "Tanh";
	}
	return "?";
}


}  // namespace tcnnb

#define TCNNB_API_BEGIN try {
#define TCNNB_API_END                         \
	return 0;                                   \
	}                                           \
	catch (const std::exception& e) {           \
		tcnnb::g_last_error = e.what();           \
		return 1;                                 \
	}                                           \
	catch (...) {                               \
		tcnnb::g_last_error = "unknown exception"; \
		return 1;                                 \
	}
