// common.cuh -- shared device/host declarations for the tcnn_b200 kernels.
#pragma once
#include <cstdlib>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace tcnnb {

constexpr uint32_t MAX_LEVELS = 32;            // levels handled by the by-value kernel argument (L*F <= 64 on the fused path)
constexpr uint32_t BATCH_GRANULARITY = 256;    // common.h:246 BATCH_SIZE_GRANULARITY
constexpr uint32_t TILE_M = 128;               // samples per MMA tile (two m64 wgmma products)

// Same numeric values as the reference enums (common.h:133-164).
enum Activation : uint32_t { ACT_RELU = 0, ACT_LEAKY_RELU = 1, ACT_SILU = 2, ACT_EXPONENTIAL = 3, ACT_SINE = 4, ACT_SIGMOID = 5, ACT_SQUAREPLUS = 6, ACT_SOFTPLUS = 7, ACT_TANH = 8, ACT_NONE = 9 };
enum GridType : uint32_t { GRID_HASH = 0, GRID_DENSE = 1, GRID_TILED = 2 };
enum InterpolationType : uint32_t { INTERP_NEAREST = 0, INTERP_LINEAR = 1, INTERP_SMOOTHSTEP = 2 };
enum LossType : uint32_t { LOSS_L2 = 0, LOSS_RELATIVE_L2 = 1, LOSS_L1 = 2, LOSS_RELATIVE_L1 = 3, LOSS_MAPE = 4, LOSS_SMAPE = 5, LOSS_RELATIVE_L2_LUMINANCE = 6, LOSS_CROSS_ENTROPY = 7, LOSS_VARIANCE_IS = 8 };

// One resolution level of the multiresolution grid, precomputed on the host from the reference's sizing rule
// (grid.h:692-737) with the per-level scale evaluated ON THE DEVICE by eval_level_scales() so that it carries the
// same bits as the reference's in-kernel grid_scale() (common_device.h:886-891, fast-math ex2.approx + fma).
struct LevelInfo {
	uint32_t offset;      // first entry of this level in the table (entries, not params)
	uint32_t size;        // number of entries ("hashmap_size", grid.h:92)
	float scale;          // grid_scale(level)
	uint32_t resolution;  // grid_resolution(scale)
	uint32_t use_hash;    // grid_type == Hash && size < dense stride (common_device.h:880)
	uint32_t pow2_mask;   // size - 1 if size is a power of two, else 0 (index % size == index & mask)
	uint32_t small_mod;   // 1 if every index this level can produce is < 2 * size (index % size == conditional subtract)
	uint32_t wide_ok;     // 1 if `offset` is a multiple of 4 entries: 8-/16-byte merged reductions relative to the level base are aligned
	                      // (Tiled grids with an odd base_resolution^D and log2_hashmap_size < 2 are not; they take 4-byte reductions)
};

struct GridMeta {
	uint32_t n_levels;
	uint32_t n_features;    // n_levels * F
	uint32_t padded_width;  // multiple of 16
	uint32_t interpolation;
	LevelInfo levels[MAX_LEVELS];
};

struct Pcg32 {
	uint64_t state, inc;
};


// ---- programmatic dependent launch (PDL). Every kernel of the training step is launched with programmatic stream
// serialization allowed: its CTAs may be scheduled -- and run their prologue -- while the kernel in front of it on the stream
// is still draining, and block in pdl_wait() until that kernel has completed and its writes are visible. pdl_wait() sits in
// front of the first global-memory access of each kernel, so the semantics are those of ordinary stream order; what is saved
// is the launch latency between the six kernels of a step. pdl_launch_dependents() tells the scheduler that the NEXT
// kernel's CTAs may start arriving (small kernels call it at once; the persistent fused kernel near its end).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
	cudaLaunchConfig_t cfg = {};
	cfg.gridDim = grid;
	cfg.blockDim = block;
	cfg.dynamicSmemBytes = smem;
	cfg.stream = stream;
	cudaLaunchAttribute attr[1];
	attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
#ifdef TCNNB_ENABLE_ABLATION  // profiling builds only: TCNNB_NO_PDL=1 = plain stream-ordered launches (A/B switch)
	static const int allowed = std::getenv("TCNNB_NO_PDL") ? 0 : 1;
#else
	const int allowed = 1;
#endif
	attr[0].val.programmaticStreamSerializationAllowed = allowed;
	cfg.attrs = attr;
	cfg.numAttrs = 1;
	return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

}  // namespace tcnnb
