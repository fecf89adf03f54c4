// mlp_wgrad.cu -- weight gradients of the stand-alone FullyFusedMLP: dW_l = g_l^T . h_{l-1}, summed over the batch.
//
// Replaces the reference's per-layer split-k CUTLASS GEMMs (fully_fused_mlp.cu:802-866: fc_multiply_split_k<LastLayerK / FullLayerK>
// on side streams). HBM-bound by construction -- 2 (in + 2 n_hidden width + out) bytes per sample against 2 width^2 flops per
// matrix and sample (64 flop/byte at 128 neurons, a quarter of the ridge) -- so the design goal is one pass over the operands:
//
//   * every CTA (one per SM) owns a contiguous range of 128-sample tiles and, for each tile and weight matrix, has TMA fetch the
//     two operand tiles [128 samples][width] (SWIZZLE_128B boxes of 64 columns; narrower matrices are zero-filled by the TMA unit)
//     into a ring of shared-memory stages;
//   * both operands are read MN-major by wgmma (the batch is the K dimension: 8 steps of 16 samples per tile), accumulating fp32 in
//     registers over all tiles of the CTA, one matrix after the other: M / 64 consumer warpgroups each own 64 rows of the
//     [width][fan-in] accumulator;
//   * at the end of a matrix each CTA adds its partial sums to the fp32 gradient accumulator with red.global.add.f32 (vectorised),
//     which the optimizer consumes directly (Adam reads fp32 sums for the matrix parameters) or launch_mlp_grad_finalize casts to fp16.
//
// Warp roles: warpgroups 0 .. M / 64 - 1 = MMA + flush, the last warp = TMA producer.
#include "mlp_fused.h"

#include "fused_common.cuh"
#include "misc_kernels.h"
#include "ptx.cuh"
#include "tma_host.h"

namespace tcnnb {

using namespace ptx;
using namespace fused;

namespace {

template <uint32_t W>
struct WgradCfg {
	static constexpr uint32_t M = W == 128 ? 128 : 64;          // rows of an accumulator (narrower layers are zero-padded by TMA)
	static constexpr uint32_t WGS = M / 64;                     // consumer warpgroups, 64 accumulator rows each
	static constexpr uint32_t KB = (W + 63) / 64;               // 64-column boxes per operand tile
	static constexpr uint32_t OPERAND_BYTES = KB * TILE_BYTES;
	static constexpr uint32_t STAGE_BYTES = 2 * OPERAND_BYTES;  // [A | B]
	static constexpr uint32_t STAGES = (200u * 1024u) / STAGE_BYTES < 8 ? (200u * 1024u) / STAGE_BYTES : 8;
	static constexpr uint32_t THREADS = WGS * 128 + 32;
};

struct WgradKernelParams {
	MlpWgradParams p;
};

}  // namespace

// WIDE = true: dL/d(output) is wider than an accumulator (out_width > NMAX, the widest fan-in). The output matrix then takes
// n_ob = ceil(out_width / NMAX) passes over the CTA's tiles, pass c accumulating dW_out rows NMAX c .. NMAX c + NMAX - 1 from
// dL/d(output) columns of the same range; every pass fetches h_{NH-1} again.
template <uint32_t W, bool WIDE>
__global__ void __launch_bounds__(WgradCfg<W>::THREADS, 1)
mlp_wgrad_kernel(const WgradKernelParams kp, const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_h, const __grid_constant__ CUtensorMap map_g,
                 const __grid_constant__ CUtensorMap map_go) {
	using C = WgradCfg<W>;
	const MlpWgradParams& p = kp.p;
	extern __shared__ __align__(1024) uint8_t smem_raw[];
	const uint32_t tid = threadIdx.x;
	const uint32_t warp = __shfl_sync(0xFFFFFFFFu, tid >> 5, 0);
	const uint32_t lane = tid & 31u;
	const uint32_t NH = p.n_hidden_layers;
	const uint32_t in_w = p.in_width, out_w = p.out_width;
	constexpr uint32_t NMAX = C::KB * 64;  // widest fan-in
	const uint32_t n_ob = WIDE ? (out_w + NMAX - 1) / NMAX : 1u;  // passes of the output matrix
	const uint32_t n_matrices = NH + n_ob;

	const uint32_t smem_base = smem_u32(smem_raw);
	if (smem_base & 1023u) __trap();
	const uint32_t s_bars = smem_base + C::STAGES * C::STAGE_BYTES;
	const uint32_t bar_full = s_bars;                    // [STAGES] TMA complete_tx
	const uint32_t bar_free = bar_full + 8 * C::STAGES;  // [STAGES] one arrival per consumer warp

	if (tid == 0) {
		for (uint32_t i = 0; i < C::STAGES; ++i) {
			mbar_init(bar_full + 8 * i, 1);
			mbar_init(bar_free + 8 * i, C::WGS * 4);
		}
		fence_mbar_init();
	}
	if (warp == C::WGS * 4 && lane == 0) {
		tma_prefetch_desc(&map_x);
		tma_prefetch_desc(&map_h);
		tma_prefetch_desc(&map_g);
		tma_prefetch_desc(&map_go);
	}
	__syncthreads();
	pdl_wait();

	const uint32_t n_tiles = p.batch_size / TILE_M;
	const uint32_t tile_begin = (uint32_t)((uint64_t)blockIdx.x * n_tiles / gridDim.x), tile_end = (uint32_t)((uint64_t)(blockIdx.x + 1) * n_tiles / gridDim.x);
	const uint32_t n_my = tile_end - tile_begin;
	const uint32_t n_items = n_my * n_matrices;  // (matrix, tile) pairs, tile fastest
	auto b_cols_of = [&](uint32_t mi) { return WIDE ? (mi == 0 ? in_w : (mi < NH ? W : min(NMAX, out_w - (mi - NH) * NMAX))) : (mi == 0 ? in_w : (mi == NH ? out_w : W)); };
	auto ob_of = [&](uint32_t mi) { return WIDE && mi > NH ? mi - NH : 0u; };  // pass of the output matrix

	if (warp == C::WGS * 4) {
		// =================================================================================== TMA producer
		if (lane == 0) {
			for (uint32_t it = 0; it < n_items; ++it) {
				const uint32_t mi = it / n_my, tile = tile_begin + it % n_my;
				const uint32_t stage = it % C::STAGES;
				if (it >= C::STAGES) mbar_wait(bar_free + 8 * stage, ((it / C::STAGES) - 1u) & 1u);
				const uint32_t a_dst = smem_base + stage * C::STAGE_BYTES, b_dst = a_dst + C::OPERAND_BYTES;
				const uint32_t full = bar_full + 8 * stage;
				const int32_t row = (int32_t)(tile * TILE_M);
				// matrix mi < NH: A = g_mi, B = h_{mi-1} (the network input for mi == 0);   output matrix: A = h_{NH-1}, B = dL/d(output)
				// (transposed product: the accumulator's 128 / 64 rows are the layer's neurons either way)
				const uint32_t b_boxes = (b_cols_of(mi) + 63) / 64;
				mbar_arrive_expect_tx(full, (C::KB + b_boxes) * TILE_BYTES);
				for (uint32_t b = 0; b < C::KB; ++b) {
					if (mi < NH) tma_load_2d(a_dst + b * TILE_BYTES, &map_g, full, (int32_t)(b * 64), (int32_t)(mi * p.batch_size) + row);
					else tma_load_2d(a_dst + b * TILE_BYTES, &map_h, full, (int32_t)(b * 64), (int32_t)((NH - 1) * p.batch_size) + row);
				}
				for (uint32_t b = 0; b < b_boxes; ++b) {
					if (mi == 0) tma_load_2d(b_dst + b * TILE_BYTES, &map_x, full, (int32_t)(b * 64), row);
					else if (mi < NH) tma_load_2d(b_dst + b * TILE_BYTES, &map_h, full, (int32_t)(b * 64), (int32_t)((mi - 1) * p.batch_size) + row);
					else tma_load_2d(b_dst + b * TILE_BYTES, &map_go, full, (int32_t)(b * 64 + ob_of(mi) * NMAX), row);
				}
			}
		}
	} else {
		// =================================================================================== consumer warpgroup h: accumulator rows 64 h ..
		const uint32_t h = warp / 4, wq = warp & 3u;
		const uint32_t fq = lane >> 2, ft = lane & 3u;
		float d[NMAX / 2];
		for (uint32_t it = 0; it < n_items; ++it) {
			const uint32_t mi = it / n_my;
			const bool first_tile = it % n_my == 0, last_tile = it % n_my == n_my - 1;
			const uint32_t stage = it % C::STAGES;
			const uint32_t n_cols = b_cols_of(mi);
			mbar_wait(bar_full + 8 * stage, (it / C::STAGES) & 1u);
			const uint32_t a_tile = smem_base + stage * C::STAGE_BYTES + h * TILE_BYTES, b_tile = smem_base + stage * C::STAGE_BYTES + C::OPERAND_BYTES;
			wgmma_fence();
#pragma unroll
			for (uint32_t kk = 0; kk < TILE_M / 16; ++kk) {
				// [128 K-rows][64 MN] boxes: 16 K-rows per step = 2 048 bytes; the next 64 MN elements are one box (TILE_BYTES) further
				const uint64_t a_desc = wgmma_desc_sw128(a_tile + kk * 2048u, TILE_BYTES, 1024u);
				const uint64_t b_desc = wgmma_desc_sw128(b_tile + kk * 2048u, TILE_BYTES, 1024u);
				const uint32_t acc = (!first_tile || kk > 0) ? 1u : 0u;
				if (NMAX == 128 && n_cols > 64) Wgmma<NMAX>::template ss<1, 1>(reinterpret_cast<float(&)[NMAX / 2]>(d), a_desc, b_desc, acc);
				else Wgmma<64>::template ss<1, 1>(reinterpret_cast<float(&)[32]>(d), a_desc, b_desc, acc);
			}
			wgmma_commit();
			wgmma_wait<0>();
			reg_fence(d);
			__syncwarp();
			if (lane == 0) mbar_arrive_plain(bar_free + 8 * stage);
			if (!last_tile) continue;
			// ---- flush: partial sums -> global fp32. d[4 i + q]: row m = 64 h + 16 wq + lane / 4 (+ 8 for q >= 2), column 8 i + 2 (lane % 4) + (q & 1)
			float* base = p.dw_accum + (mi == 0 ? 0 : (size_t)W * in_w + (size_t)((WIDE ? min(mi, NH) : mi) - 1) * W * W) + (size_t)ob_of(mi) * NMAX * W;
#pragma unroll
			for (uint32_t i = 0; i < NMAX / 8; ++i) {
				const uint32_t n = 8 * i + 2 * ft;
				if (n >= n_cols) continue;
#pragma unroll
				for (uint32_t hi = 0; hi < 2; ++hi) {
					const uint32_t m = h * 64 + wq * 16 + fq + hi * 8;
					if (m >= W) continue;
					const float v0 = d[4 * i + 2 * hi], v1 = d[4 * i + 2 * hi + 1];
					if (mi < NH) {
						red_add_v2_f32(base + (size_t)m * n_cols + n, v0, v1);  // W_mi[m][n ..]
					} else {
						red_add_f32(base + (size_t)n * W + m, v0);  // W_out[n][m]
						red_add_f32(base + (size_t)(n + 1) * W + m, v1);
					}
				}
			}
		}
	}

	pdl_launch_dependents();
}

// 256 neurons: an accumulator is [256][fan-in <= 256]. Four 64-row warpgroups at 128 fp32 registers each cannot be resident together
// (544 threads leave 120 registers each), so the rows are covered in two 128-row halves, one per CTA of a pair: CTA 2 c + q owns rows
// 128 q .. 128 q + 127 of every accumulator (two warpgroups x 64 rows x up to 256 columns) over pair c's tile range. Both CTAs of a
// pair fetch the same B tiles (h_{l-1}, the network input or dL/d(output)) in the same order at about the same time, so the second
// fetch is usually served by L2; the A tiles (g_l, or h_{NH-1} for the output matrix) are split between them.
struct Wgrad256 {
	static constexpr uint32_t W = 256;
	static constexpr uint32_t HALF = 128;
	static constexpr uint32_t WGS = 2;
	static constexpr uint32_t A_BOXES = HALF / 64;  // [128 samples][64 rows of the half]
	static constexpr uint32_t B_BOXES = W / 64;     // [128 samples][64 fan-in columns]
	static constexpr uint32_t STAGE_BYTES = (A_BOXES + B_BOXES) * TILE_BYTES;
	static constexpr uint32_t STAGES = 2;
	static constexpr uint32_t THREADS = WGS * 128 + 32;
};

// WIDE = true (out_width > 256): the output matrix takes n_ob = ceil(out_width / 256) passes, as in mlp_wgrad_kernel.
template <bool WIDE>
__device__ __forceinline__ void wgrad256_body(const WgradKernelParams& kp, const CUtensorMap& map_x, const CUtensorMap& map_h, const CUtensorMap& map_g, const CUtensorMap& map_go) {
	using C = Wgrad256;
	constexpr uint32_t W = C::W;
	const MlpWgradParams& p = kp.p;
	extern __shared__ __align__(1024) uint8_t smem_raw[];
	const uint32_t tid = threadIdx.x;
	const uint32_t warp = __shfl_sync(0xFFFFFFFFu, tid >> 5, 0);
	const uint32_t lane = tid & 31u;
	const uint32_t NH = p.n_hidden_layers;
	const uint32_t in_w = p.in_width, out_w = p.out_width;
	const uint32_t n_ob = WIDE ? (out_w + W - 1) / W : 1u;
	const uint32_t n_matrices = NH + n_ob;

	const uint32_t smem_base = smem_u32(smem_raw);
	if (smem_base & 1023u) __trap();
	const uint32_t bar_full = smem_base + C::STAGES * C::STAGE_BYTES;
	const uint32_t bar_free = bar_full + 8 * C::STAGES;

	if (tid == 0) {
		for (uint32_t i = 0; i < C::STAGES; ++i) {
			mbar_init(bar_full + 8 * i, 1);
			mbar_init(bar_free + 8 * i, C::WGS * 4);
		}
		fence_mbar_init();
	}
	if (warp == C::WGS * 4 && lane == 0) {
		tma_prefetch_desc(&map_x);
		tma_prefetch_desc(&map_h);
		tma_prefetch_desc(&map_g);
		tma_prefetch_desc(&map_go);
	}
	__syncthreads();
	pdl_wait();

	const uint32_t half = blockIdx.x & 1u, pair = blockIdx.x >> 1, n_pairs = gridDim.x >> 1;
	const uint32_t n_tiles = p.batch_size / TILE_M;
	const uint32_t tile_begin = (uint32_t)((uint64_t)pair * n_tiles / n_pairs), tile_end = (uint32_t)((uint64_t)(pair + 1) * n_tiles / n_pairs);
	const uint32_t n_my = tile_end - tile_begin;
	const uint32_t n_items = n_my * n_matrices;
	auto b_cols_of = [&](uint32_t mi) { return WIDE ? (mi == 0 ? in_w : (mi < NH ? W : min(W, out_w - (mi - NH) * W))) : (mi == 0 ? in_w : (mi == NH ? out_w : W)); };
	auto ob_of = [&](uint32_t mi) { return WIDE && mi > NH ? mi - NH : 0u; };

	if (warp == C::WGS * 4) {
		// =================================================================================== TMA producer
		if (lane == 0) {
			for (uint32_t it = 0; it < n_items; ++it) {
				const uint32_t mi = it / n_my, tile = tile_begin + it % n_my;
				const uint32_t stage = it % C::STAGES;
				if (it >= C::STAGES) mbar_wait(bar_free + 8 * stage, ((it / C::STAGES) - 1u) & 1u);
				const uint32_t a_dst = smem_base + stage * C::STAGE_BYTES, b_dst = a_dst + C::A_BOXES * TILE_BYTES;
				const uint32_t full = bar_full + 8 * stage;
				const int32_t row = (int32_t)(tile * TILE_M);
				const uint32_t b_boxes = (b_cols_of(mi) + 63) / 64;
				mbar_arrive_expect_tx(full, (C::A_BOXES + b_boxes) * TILE_BYTES);
				for (uint32_t b = 0; b < C::A_BOXES; ++b) {
					const int32_t col = (int32_t)(half * C::HALF + b * 64);
					if (mi < NH) tma_load_2d(a_dst + b * TILE_BYTES, &map_g, full, col, (int32_t)(mi * p.batch_size) + row);
					else tma_load_2d(a_dst + b * TILE_BYTES, &map_h, full, col, (int32_t)((NH - 1) * p.batch_size) + row);
				}
				for (uint32_t b = 0; b < b_boxes; ++b) {
					if (mi == 0) tma_load_2d(b_dst + b * TILE_BYTES, &map_x, full, (int32_t)(b * 64), row);
					else if (mi < NH) tma_load_2d(b_dst + b * TILE_BYTES, &map_h, full, (int32_t)(b * 64), (int32_t)((mi - 1) * p.batch_size) + row);
					else tma_load_2d(b_dst + b * TILE_BYTES, &map_go, full, (int32_t)(b * 64 + ob_of(mi) * W), row);
				}
			}
		}
	} else {
		// =================================================================================== consumer warpgroup h: rows 128 half + 64 h ..
		const uint32_t h = warp / 4, wq = warp & 3u;
		const uint32_t fq = lane >> 2, ft = lane & 3u;
		float d[W / 2];
		for (uint32_t it = 0; it < n_items; ++it) {
			const uint32_t mi = it / n_my;
			const bool first_tile = it % n_my == 0, last_tile = it % n_my == n_my - 1;
			const uint32_t stage = it % C::STAGES;
			const uint32_t n_cols = b_cols_of(mi);
			mbar_wait(bar_full + 8 * stage, (it / C::STAGES) & 1u);
			const uint32_t a_tile = smem_base + stage * C::STAGE_BYTES + h * TILE_BYTES, b_tile = smem_base + stage * C::STAGE_BYTES + C::A_BOXES * TILE_BYTES;
			wgmma_fence();
#pragma unroll
			for (uint32_t kk = 0; kk < TILE_M / 16; ++kk) {
				const uint64_t a_desc = wgmma_desc_sw128(a_tile + kk * 2048u, TILE_BYTES, 1024u);
				const uint64_t b_desc = wgmma_desc_sw128(b_tile + kk * 2048u, TILE_BYTES, 1024u);
				const uint32_t acc = (!first_tile || kk > 0) ? 1u : 0u;
				// N rounds n_cols up to 64 / 128 / 256: boxes past the loaded ones hold an earlier item's data (or nothing yet), and
				// the columns they feed (n >= n_cols) are dropped by the flush
				if (n_cols > 128) Wgmma<256>::ss<1, 1>(d, a_desc, b_desc, acc);
				else if (n_cols > 64) Wgmma<128>::ss<1, 1>(reinterpret_cast<float(&)[64]>(d), a_desc, b_desc, acc);
				else Wgmma<64>::ss<1, 1>(reinterpret_cast<float(&)[32]>(d), a_desc, b_desc, acc);
			}
			wgmma_commit();
			wgmma_wait<0>();
			reg_fence(d);
			__syncwarp();
			if (lane == 0) mbar_arrive_plain(bar_free + 8 * stage);
			if (!last_tile) continue;
			// ---- flush, as mlp_wgrad_kernel: d[4 i + q] = row m, column 8 i + 2 (lane % 4) + (q & 1)
			float* base = p.dw_accum + (mi == 0 ? 0 : (size_t)W * in_w + (size_t)((WIDE ? min(mi, NH) : mi) - 1) * W * W) + (size_t)ob_of(mi) * W * W;
#pragma unroll
			for (uint32_t i = 0; i < W / 8; ++i) {
				const uint32_t n = 8 * i + 2 * ft;
				if (n >= n_cols) continue;
#pragma unroll
				for (uint32_t hi = 0; hi < 2; ++hi) {
					const uint32_t m = half * C::HALF + h * 64 + wq * 16 + fq + hi * 8;
					const float v0 = d[4 * i + 2 * hi], v1 = d[4 * i + 2 * hi + 1];
					if (mi < NH) {
						red_add_v2_f32(base + (size_t)m * n_cols + n, v0, v1);
					} else {
						red_add_f32(base + (size_t)n * W + m, v0);
						red_add_f32(base + (size_t)(n + 1) * W + m, v1);
					}
				}
			}
		}
	}

	pdl_launch_dependents();
}

__global__ void __launch_bounds__(Wgrad256::THREADS, 1)
mlp_wgrad256_kernel(const WgradKernelParams kp, const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_h, const __grid_constant__ CUtensorMap map_g,
                    const __grid_constant__ CUtensorMap map_go) {
	wgrad256_body<false>(kp, map_x, map_h, map_g, map_go);
}

__global__ void __launch_bounds__(Wgrad256::THREADS, 1)
mlp_wgrad256_wide_kernel(const WgradKernelParams kp, const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_h, const __grid_constant__ CUtensorMap map_g,
                         const __grid_constant__ CUtensorMap map_go) {
	wgrad256_body<true>(kp, map_x, map_h, map_g, map_go);
}

namespace {

cudaError_t launch_wgrad256(const MlpWgradParams& p, uint32_t n_sms, cudaStream_t stream, uint32_t* n_launches) {
	using C = Wgrad256;
	const uint32_t NH = p.n_hidden_layers, B = p.batch_size;
	CUtensorMap mx, mh, mg, mgo;
	if (!make_fp16_matrix_map(&mx, p.input, B, p.in_width, TILE_M)) return cudaErrorInvalidValue;
	if (!make_fp16_matrix_map(&mh, p.hidden, (uint64_t)NH * B, C::W, TILE_M)) return cudaErrorInvalidValue;
	if (!make_fp16_matrix_map(&mg, p.grad_hidden, (uint64_t)NH * B, C::W, TILE_M)) return cudaErrorInvalidValue;
	if (!make_fp16_matrix_map(&mgo, p.grad_output, B, p.out_width, TILE_M)) return cudaErrorInvalidValue;
	const size_t smem = (size_t)C::STAGES * C::STAGE_BYTES + 8 * 2 * C::STAGES;
	auto kernel = p.out_width > C::W ? mlp_wgrad256_wide_kernel : mlp_wgrad256_kernel;
	cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
	if (err != cudaSuccess) return err;
	const uint32_t n_tiles = B / TILE_M, n_pairs = n_tiles < n_sms / 2 ? n_tiles : n_sms / 2;
	WgradKernelParams kp{};
	kp.p = p;
	err = launch_pdl(kernel, 2 * n_pairs, C::THREADS, smem, stream, kp, mx, mh, mg, mgo);
	if (err != cudaSuccess) return err;
	if (n_launches) ++*n_launches;
	return cudaSuccess;
}

template <uint32_t W, bool WIDE>
cudaError_t launch_wgrad_width(const MlpWgradParams& p, uint32_t n_sms, cudaStream_t stream, uint32_t* n_launches) {
	using C = WgradCfg<W>;
	const uint32_t NH = p.n_hidden_layers, B = p.batch_size;
	CUtensorMap mx, mh, mg, mgo;
	if (!make_fp16_matrix_map(&mx, p.input, B, p.in_width, TILE_M)) return cudaErrorInvalidValue;
	if (!make_fp16_matrix_map(&mh, p.hidden, (uint64_t)NH * B, W, TILE_M)) return cudaErrorInvalidValue;
	if (!make_fp16_matrix_map(&mg, p.grad_hidden, (uint64_t)NH * B, W, TILE_M)) return cudaErrorInvalidValue;
	if (!make_fp16_matrix_map(&mgo, p.grad_output, B, p.out_width, TILE_M)) return cudaErrorInvalidValue;
	auto kernel = mlp_wgrad_kernel<W, WIDE>;
	const size_t smem = (size_t)C::STAGES * C::STAGE_BYTES + 8 * 2 * C::STAGES;
	cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
	if (err != cudaSuccess) return err;
	const uint32_t n_tiles = B / TILE_M;
	WgradKernelParams kp{};
	kp.p = p;
	err = launch_pdl(kernel, n_tiles < n_sms ? n_tiles : n_sms, C::THREADS, smem, stream, kp, mx, mh, mg, mgo);
	if (err != cudaSuccess) return err;
	if (n_launches) ++*n_launches;
	return cudaSuccess;
}

// dL/d(output) wider than an accumulator (64 columns below 128 neurons, 128 at 128) takes the WIDE kernel
template <uint32_t W>
cudaError_t launch_wgrad_width(const MlpWgradParams& p, uint32_t n_sms, cudaStream_t stream, uint32_t* n_launches) {
	return p.out_width > WgradCfg<W>::KB * 64 ? launch_wgrad_width<W, true>(p, n_sms, stream, n_launches) : launch_wgrad_width<W, false>(p, n_sms, stream, n_launches);
}

}  // namespace

bool mlp_wgrad_supported(const MlpWgradParams& p, const char** why) {
	auto fail = [&](const char* msg) {
		if (why) *why = msg;
		return false;
	};
	if (!(p.width == 16 || p.width == 32 || p.width == 64 || p.width == 128 || p.width == 256)) return fail("FullyFusedMLP only supports 16, 32, 64, and 128 neurons");
	if (p.n_hidden_layers < 1) return fail("FullyFusedMLP requires at least 1 hidden layer (3 layers in total).");
	const uint32_t max_in = 64 * ((p.width + 63) / 64);
	if (p.in_width == 0 || p.in_width % 16 != 0 || p.in_width > max_in) return fail("tcnn_b200: network input width must be a multiple of 16 and at most 64 (128 / 256 for 128 / 256 neurons)");
	if (p.out_width == 0 || p.out_width % 16 != 0) return fail("tcnn_b200: padded network output width must be a multiple of 16 and at most n_neurons");
	if (p.out_width > MLP_MAX_OUTPUT_WIDTH) return fail("tcnn_b200: padded network output width must be at most 1024");
	if (p.batch_size == 0 || p.batch_size % TILE_M != 0) return fail("batch size must be a non-zero multiple of 256");
	if ((uint64_t)p.n_hidden_layers * p.batch_size >= (1ull << 31)) return fail("tcnn_b200: n_hidden_layers * batch_size must stay below 2^31 rows");
	return true;
}

cudaError_t launch_mlp_wgrad(const MlpWgradParams& p, uint32_t n_sms, cudaStream_t stream, uint32_t* n_launches) {
	if (!mlp_wgrad_supported(p, nullptr)) return cudaErrorInvalidValue;
	switch (p.width) {
		case 256: return launch_wgrad256(p, n_sms, stream, n_launches);
		case 128: return launch_wgrad_width<128>(p, n_sms, stream, n_launches);
		case 64: return launch_wgrad_width<64>(p, n_sms, stream, n_launches);
		case 32: return launch_wgrad_width<32>(p, n_sms, stream, n_launches);
		case 16: return launch_wgrad_width<16>(p, n_sms, stream, n_launches);
	}
	return cudaErrorInvalidValue;
}

static void split_backward(const MlpBackwardArgs& a, MlpForwardParams& d, MlpWgradParams& w) {
	d = MlpForwardParams{};
	d.width = a.width;
	d.in_width = a.in_width;
	d.out_width = a.out_width;
	d.n_hidden_layers = a.n_hidden_layers;
	d.activation = a.activation;
	d.output_activation = ACT_NONE;
	d.weights = a.weights;
	d.batch_size = a.batch_size;
	d.input_fp16 = a.output_activation == ACT_NONE ? a.dL_doutput : a.grad_output;
	d.output_fp16 = a.dL_dinput;
	d.hidden_out = a.grad_hidden;
	d.hidden_in = activation_needs_preact(a.activation) ? a.hidden_pre : a.hidden;  // Sine / SiLU: the derivative reads z
	d.backward = 1;
	w = MlpWgradParams{};
	w.width = a.width;
	w.in_width = a.in_width;
	w.out_width = a.out_width;
	w.n_hidden_layers = a.n_hidden_layers;
	w.batch_size = a.batch_size;
	w.input = a.input;
	w.hidden = a.hidden;
	w.grad_hidden = a.grad_hidden;
	w.grad_output = d.input_fp16;
	w.dw_accum = a.dw_accum;
}

bool mlp_backward_supported(const MlpBackwardArgs& a, const char** why) {
	MlpForwardParams d;
	MlpWgradParams w;
	split_backward(a, d, w);
	if (!d.input_fp16) d.input_fp16 = (const __half*)16;  // probing a shape: only null-ness matters
	if (!d.hidden_in) d.hidden_in = (const __half*)16;
	if (activation_needs_preact(a.activation) && a.hidden && !a.hidden_pre) {
		if (why) *why = "tcnn_b200: the backward pass of a Sine / SiLU network needs the forward pass's pre-activations (hidden_pre)";
		return false;
	}
	return mlp_forward_supported(d, why) && mlp_wgrad_supported(w, why);
}

cudaError_t launch_mlp_backward(const MlpBackwardArgs& a, uint32_t n_sms, cudaStream_t stream, uint32_t* n_launches) {
	MlpForwardParams d;
	MlpWgradParams w;
	split_backward(a, d, w);
	if (!d.hidden_in || (activation_needs_preact(a.activation) && a.dw_accum && !a.hidden)) return cudaErrorInvalidValue;
	uint32_t launches = 0;
	cudaError_t err = cudaSuccess;
	if (a.output_activation != ACT_NONE) {
		if (!a.output || !a.grad_output) return cudaErrorInvalidValue;
		err = launch_activation_backward_output(stream, a.output_activation, (uint64_t)a.batch_size * a.out_width, a.dL_doutput, a.output, a.grad_output);
		if (err != cudaSuccess) return err;
		++launches;
	}
	if (!a.grad_hidden && a.dw_accum) return cudaErrorInvalidValue;
	err = launch_mlp_forward(d, n_sms, stream);
	if (err != cudaSuccess) return err;
	++launches;
	if (a.dw_accum) {
		if (!a.input) return cudaErrorInvalidValue;
		err = launch_mlp_wgrad(w, n_sms, stream, &launches);
		if (err != cudaSuccess) return err;
	}
	if (n_launches) *n_launches += launches;
	return cudaSuccess;
}

}  // namespace tcnnb
