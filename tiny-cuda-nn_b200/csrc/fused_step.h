// fused_step.h -- launch interface of the fused HashGrid + FullyFusedMLP kernel (fused_ws.cu).
#pragma once
#include "common.cuh"

namespace tcnnb {

// Ablation switches for profiling experiments (scripts/ablate.py); 0 in production. They skip memory operations only,
// so the results of an ablated launch are meaningless.
enum : uint32_t { ABLATE_GATHER = 1, ABLATE_SCATTER = 2, ABLATE_PAIRING = 4, ABLATE_GATHER_DENSE = 8, ABLATE_SCATTER_DENSE = 16, ABLATE_GATHER_HASH = 32, ABLATE_SCATTER_HASH = 64 };
// The switches are compiled in only with -DTCNNB_ENABLE_ABLATION (make ABLATION=1): in the production build they cost nothing.
#ifdef TCNNB_ENABLE_ABLATION
#define TCNNB_ABLATE(bit) (p.ablate & (bit))
#else
#define TCNNB_ABLATE(bit) false
#endif

struct FusedStepParams {
	uint32_t ablate;
	// model
	GridMeta grid;
	uint32_t width;                // hidden width 16 / 32 / 64 (narrower layers run as 64-wide tiles with zero-padded weights)
	uint32_t n_hidden_layers;      // 1..6
	uint32_t activation;           // hidden activation (Activation enum)
	uint32_t output_activation;    // applied to the network output before the loss
	uint32_t n_out;                // logical outputs (<= 16)
	uint32_t n_mlp_params;         // grid params start here in the parameter / gradient buffers
	uint32_t enc_identity;         // 1: Identity encoding instead of the grid (features = x * scale + offset, padding features = 1)
	float identity_scale, identity_offset;
	uint32_t loss_type;            // LossType
	float loss_scale;              // 128 for fp16 params (common.h:243)
	// batch
	uint32_t batch_size;           // samples processed by this launch (multiple of 256)
	uint32_t loss_batch_size;      // samples the loss is normalised over (== batch_size unless the batch is sharded over GPUs)
	const float* positions;        // [batch][D] fp32
	const float* targets;          // [batch][n_out] fp32 (training step only)
	const __half* ext_dy;          // [batch][16] fp16, module-tier backward: the caller's dL/d(output) replaces the loss (targets unused)
	const uint32_t* perm;          // optional spatial binning: tile row i processes the caller's sample perm[i] (positions/targets/outputs)
	// parameters: [MLP weights | grid table] fp16, and the matching fp16 gradient buffer (grid part accumulated with red.f16x2)
	const __half* params;
	__half* grads;
	float* dw_accum;               // fp32 [n_mlp_params] weight-gradient accumulator (red.add.f32), must be zero on entry
	float* loss_sum;               // fp32 scalar accumulator (may be null)
	float* loss_values;            // [batch][n_out] fp32 (may be null)
	__half* out_fp16;              // [batch][16] padded network output (may be null)
	float* out_fp32;               // [batch][n_out] (may be null)
	// debug taps (tests only; null in production): per-sample rows of every intermediate
	__half* dbg_enc;               // [batch][64]
	__half* dbg_hidden;            // [n_hidden][batch][64]
	__half* dbg_dy;                // [batch][16]
	__half* dbg_grad_hidden;       // [n_hidden][batch][64]
	__half* dbg_denc;              // [batch][64]
	long long* dbg_clock;          // ablation builds: [cta][role 3][tile 16][slot 16] clock64 stamps of the ws kernel's phases
};

// Shared memory of the fused kernel: encoded / hidden / dy tiles of 128 x 64 fp16 (an encoding of at most 32 features parks its
// gradients in the enc tiles, wider ones need two park tiles), the staged weights, and the barriers ...
__host__ __device__ inline uint32_t fused_ws_base_smem_bytes(uint32_t n_hidden_layers, uint32_t enc_width, bool train) {
	const uint32_t tiles = 2 + n_hidden_layers + (train ? (enc_width <= 32 ? 1 : 3) : 0);
	return tiles * TILE_M * 128 + n_hidden_layers * 64 * 128 + 16 * 128 + 128;
}
// ... and, in training, the CTA's fp32 weight-gradient sums ([64 x 64] per hidden-layer input matrix, [64 x 16] for the output
// matrix) when they fit beside it. Deeper networks add each tile's weight gradients to the global accumulator instead.
__host__ __device__ inline uint32_t fused_ws_dw_bytes(uint32_t n_hidden_layers) { return n_hidden_layers * 64 * 64 * 4 + 64 * 16 * 4; }
__host__ __device__ inline bool fused_ws_dw_in_smem(uint32_t n_hidden_layers, uint32_t enc_width) {
	return fused_ws_base_smem_bytes(n_hidden_layers, enc_width, true) + fused_ws_dw_bytes(n_hidden_layers) <= 227 * 1024;
}

// Warp-specialised kernel (fused_ws.cu): one 640-thread CTA per SM (n_ctas <= #SMs), training step and inference.
size_t fused_ws_smem_bytes(uint32_t n_hidden_layers, uint32_t enc_width, bool train);
cudaError_t launch_fused_ws(const FusedStepParams& p, uint32_t n_pos_dims, bool train, uint32_t n_ctas, cudaStream_t stream);

}  // namespace tcnnb
