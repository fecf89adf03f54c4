/* tiny-cuda-nn/common.h -- source-compatibility shim over libtcnn_b200 (C ABI in ../tcnn_b200.h).
 *
 * These headers keep the NAMES a tiny-cuda-nn application uses on the HashGrid + FullyFusedMLP path
 * (reference: include/tiny-cuda-nn/common.h:96-260, common_host.h:71-110) and forward to the C ABI; they contain no kernels
 * and no arithmetic of their own. Anything outside that path is absent on purpose -- a program that needs it does not compile
 * instead of silently getting something else. Compile application code with nvcc (the reference is a CUDA library too). */
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <stdexcept>
#include <string>

#include "../tcnn_b200.h"

/* The reference's common_host.h:33 includes <fmt/format.h>, and its samples call fmt::format without including it themselves
 * (samples/mlp_learning_an_image.cu:291). fmt is the APPLICATION's dependency here, as nlohmann/json is: forwarded when present. */
#if __has_include(<fmt/format.h>)
#include <fmt/format.h>
#endif

namespace tcnn {

using network_precision_t = __half;                   /* common.h:121-126 (TCNN_HALF_PRECISION builds) */
static constexpr uint32_t BATCH_SIZE_GRANULARITY = 256; /* common.h:246 */
static constexpr float LOSS_SCALE = 128.0f;             /* common.h:243 (fp16 parameters) */
static constexpr uint32_t MIN_GPU_ARCH = 90;            /* this library is sm_90a-only */

enum class MatrixLayout { RowMajor = 0, SoA = 0, ColumnMajor = 1, AoS = 1 }; /* common.h:216-221 */
static constexpr MatrixLayout RM = MatrixLayout::RowMajor;
static constexpr MatrixLayout CM = MatrixLayout::ColumnMajor;

/* common_host.h:97-110 */
#define CUDA_CHECK_THROW(x)                                                                                               \
	do {                                                                                                                   \
		cudaError_t _result = (x);                                                                                         \
		if (_result != cudaSuccess) throw std::runtime_error{std::string(#x " failed: ") + cudaGetErrorString(_result)};   \
	} while (0)

/* common_host.h:71-72 */
#ifndef CHECK_THROW
#define TCNNB_STR_(x) #x
#define TCNNB_STR(x) TCNNB_STR_(x)
#define CHECK_THROW(x) \
	do { if (!(x)) throw std::runtime_error{__FILE__ ":" TCNNB_STR(__LINE__) " check failed: " #x}; } while (0)
#endif

#define TCNNB_CHECK_THROW(x)                                                                                              \
	do {                                                                                                                   \
		if ((x) != 0) throw std::runtime_error{tcnnb_last_error()};                                                        \
	} while (0)

template <typename T>
constexpr T div_round_up(T val, T divisor) { return (val + divisor - 1) / divisor; } /* common.h:250-253 */
template <typename T>
constexpr T next_multiple(T val, T divisor) { return div_round_up(val, divisor) * divisor; } /* common.h:255-258 */

static constexpr uint32_t N_THREADS_LINEAR = 128; /* common.h:247 */
static constexpr uint32_t n_threads_linear = N_THREADS_LINEAR; /* common.h:252 */
template <typename T>
constexpr uint32_t n_blocks_linear(T n_elements, uint32_t n_threads = N_THREADS_LINEAR) { return (uint32_t)div_round_up(n_elements, (T)n_threads); }

#ifdef __CUDACC__
/* common_host.h:259-273: launch `kernel(n_elements, args...)` over ceil(n / 128) blocks of 128 threads */
template <typename K, typename T, typename... Types>
inline void linear_kernel(K kernel, uint32_t shmem_size, cudaStream_t stream, T n_elements, Types... args) {
	if (n_elements <= 0) return;
	kernel<<<n_blocks_linear(n_elements), N_THREADS_LINEAR, shmem_size, stream>>>(n_elements, args...);
}
#endif

inline int cuda_device() { return tcnnb_cuda_device(); }                 /* common_host.cu:147-151 */
inline void set_cuda_device(int device) { tcnnb_set_cuda_device(device); }
inline uint32_t cuda_compute_capability(int = 0) { return 90; }
inline bool supports_jit_fusion(int = 0) { return false; } /* there is no run-time compilation here: the fused kernel is the product */
inline void free_all_gpu_memory_arenas() {}                 /* no arenas: nothing is allocated per step */

}  // namespace tcnn
