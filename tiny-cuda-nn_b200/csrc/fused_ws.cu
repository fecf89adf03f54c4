// fused_ws.cu -- the hot path in ONE warp-specialised kernel: HashGrid gather + N-linear blend -> FullyFusedMLP forward (wgmma)
// -> loss -> MLP backward (wgmma: dgrad and wgrad) -> hash-grid gradient scatter (f16x2 reductions); without its backward half
// it is the inference kernel.
//
// Replaces, for one training step, the reference's kernel_grid (grid.h:49), kernel_mlp_fused (fully_fused_mlp.cu:500),
// relative_l2_loss / l2_loss (losses/*.h:40), kernel_mlp_fused_backward (fully_fused_mlp.cu:151), the three CUTLASS split-K
// weight-gradient GEMMs and the dL/d(encoded) GEMM (fully_fused_mlp.cu:784-836) and kernel_grid_backward (grid.h:215). No
// activation ever leaves the SM: the only HBM/L2 traffic is positions, targets, the fp16 tables (gather), their fp16 gradient
// tables (red.f16x2) and 7 K fp32 weight-gradient partial sums per CTA.
//
// Data layout on chip: operand tiles are [128 rows][64 fp16] in the canonical SWIZZLE_128B layout; the SAME bytes are consumed as
// a K-major A operand by the forward / dgrad MMAs (M = samples, K = neurons) and as an MN-major operand by the wgrad MMAs
// (M/N = neurons, K = samples), so no transposes are ever materialised. Weights are staged once per CTA: W_l [out][in] row-major
// is the K-major B operand of the forward MMA and, read MN-major, the B operand of the dgrad MMA (W_l^T). Accumulators live in
// the MLP warpgroup's registers; the fp32 weight-gradient sums of all tiles of the CTA live in shared memory (when they fit, see
// fused_ws_dw_in_smem) and are flushed once with red.global.add.f32. The backward activations g_l overwrite h_l in place.
//
// Why warp-specialised: in a bulk-synchronous structure every MMA batch ends in a CTA-wide barrier, so the long and uneven
// latencies of the table gathers / gradient reductions that fill the wait slots end up on the critical path of the MLP chain.
// Here the two kinds of work never wait for each other inside a tile:
//
//   warps 0..3   "MLP group" (one warpgroup): issues the wgmma products and runs the epilogues of one 128-sample tile at a time,
//                tile after tile.
//   warps 4..19  "memory group": two sub-groups of 8 warps (256 threads = two threads per sample). Sub-group g owns the
//                tiles k = g, g+2, ... of this CTA: it gathers + blends tile k into enc[g], then scatters the parked
//                dL/d(enc) of its previous tile k-2, continuously, while the MLP group works on tile k-1.
//
// Hand-offs are mbarriers only:  enc_full[g]  (memory -> MLP: encoded tile ready)
//                                enc_free[g]  (MLP -> memory: the last wgmma that reads enc[g] has completed)
//                                park_full[g] (MLP -> memory: dL/d(enc) of the tile parked)
//                                park_free[g] (memory -> MLP: parked gradients consumed)
// One persistent CTA per SM, 640 threads (4 MLP warps + two memory sub-groups), grid = #SMs.
#include "common.cuh"
#include "fused_common.cuh"
#include "fused_step.h"
#include "grid_device.cuh"
#include "ptx.cuh"

namespace tcnnb {

// Phase timestamps for pipeline analysis (ablation builds only: make ABLATION=1; scripts/ws_timeline.py reads them).
#ifdef TCNNB_ENABLE_ABLATION
#define WS_STAMP(role, tile_idx, slot)                                                                                   \
	do {                                                                                                                \
		if (p.dbg_clock && (tile_idx) < 16u) p.dbg_clock[((blockIdx.x * 3u + (role)) * 16u + (tile_idx)) * 16u + (slot)] = clock64(); \
	} while (0)
#else
#define WS_STAMP(role, tile_idx, slot) \
	do {                               \
	} while (0)
#endif

using namespace ptx;
using namespace fused;

namespace {

// enc buffers per CTA (tile k uses buffer k % 2). Four -- so that a gather never waits for an earlier tile's backward pass -- was
// measured 1.6 % SLOWER: the 32 KB come out of the L1 that the table gathers live on.
constexpr uint32_t WS_ENC_BUFFERS = 2;
constexpr uint32_t WS_MLP_THREADS = 128;
constexpr uint32_t WS_SUB_THREADS = 256;
constexpr uint32_t SUBS = 2;  // memory sub-groups per CTA
constexpr uint32_t WS_THREADS = WS_MLP_THREADS + SUBS * WS_SUB_THREADS;  // 640
constexpr uint32_t WS_DW_BYTES = 64 * 64 * 4;  // fp32 weight-gradient sums of one hidden-layer input matrix

__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
	asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t n_threads) {
	asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n_threads) : "memory");
}

}  // namespace

// PDF: the loss divides by p.data_pdf (a flag of its own, so that the kernels without it carry no null check)
template <uint32_t D, uint32_t F, bool TRAIN, bool GENERIC_ACT, bool PDF>
__global__ void __launch_bounds__(WS_THREADS, 1) fused_ws_kernel(const FusedStepParams p) {
	// ReLU hidden / linear output (the reference's default and the benchmark configuration) fold to the packed fast path at compile time
	const uint32_t hid_act = GENERIC_ACT ? p.activation : (uint32_t)ACT_RELU;
	const uint32_t out_act = GENERIC_ACT ? p.output_activation : (uint32_t)ACT_NONE;
	static_assert(F == 2, "fused path: F == 2");
	extern __shared__ __align__(1024) uint8_t smem_raw[];
	const uint32_t tid = threadIdx.x;
	const uint32_t warp = __shfl_sync(0xFFFFFFFFu, tid >> 5, 0);  // broadcast: the compiler can treat it as warp-uniform
	const uint32_t NH = p.n_hidden_layers;
	const uint32_t in_w = p.grid.padded_width;

	// ---- shared memory: [ enc_0 .. enc_{NE-1} | h_0 .. h_{NH-1} | dy | park_0 | park_1 | W_0 .. W_{NH-1} | W_out ] barriers
	// The dynamic segment starts 1024-byte aligned (declared so above; there is no static shared memory in this kernel), so no
	// alignment slack is requested: the last kilobyte decides which shared-memory carve-out the SM uses, i.e. how much L1 is left.
	const uint32_t smem_base = smem_u32(smem_raw);
	if (smem_base & 1023u) __trap();
	const uint32_t s_enc = smem_base;
	constexpr uint32_t NE = WS_ENC_BUFFERS;  // tile k uses enc buffer k % NE
	const uint32_t s_h0 = s_enc + NE * TILE_BYTES;
	const uint32_t s_dy = s_h0 + NH * TILE_BYTES;
	const uint32_t s_park = s_dy + (TRAIN ? TILE_BYTES : 0);
	// The parked dL/d(enc) rows need enc_width columns; with an encoding of at most 32 features they fit the unused upper half
	// of the two enc tiles (tile k parks into enc[k & 1], NE == 2) and the kernel does without park tiles of its own -- 32 KB of
	// shared memory that the hardware hands to the L1 instead, which the table gathers make good use of.
	const bool park_in_enc = NE == 2 && in_w <= 32;
	const uint32_t s_w0 = s_park + (TRAIN && !park_in_enc ? 2 * TILE_BYTES : 0);
	// parked dL/d(enc) row `row`, 16-byte chunk `chunk` of buffer g: chunks 4..7 of enc[g], or park tiles of their own
	auto park_addr = [&](uint32_t g, uint32_t row, uint32_t chunk) {
		return park_in_enc ? s_enc + g * TILE_BYTES + sw128(row, 4u + chunk) : s_park + g * TILE_BYTES + sw128(row, chunk);
	};
	const uint32_t s_wout = s_w0 + NH * (WIDTH * 128);
	// fp32 weight-gradient sums of this CTA (training, when they fit: fused_ws_dw_in_smem): one [64 x 64] block per hidden-layer input
	// matrix W_0 .. W_{NH-1} and one [64 x 16] block for W_out, kept across all tiles. Stored in the accumulator fragment order of
	// the MLP warpgroup -- word (i * 128 + thread) * 4 + q holds d[4 i + q] of that thread -- so that every thread reloads and
	// stores only its own values.
	const bool dw_smem = TRAIN && fused_ws_dw_in_smem(NH, in_w);
	const uint32_t s_dw = s_wout + 16 * 128;
	const uint32_t s_bars = s_dw + (dw_smem ? fused_ws_dw_bytes(NH) : 0);  // 9 mbarriers
	const uint32_t bar_enc_full = s_bars + 8;    // [4]
	const uint32_t bar_enc_free = s_bars + 40;   // [4]
	const uint32_t bar_park_full = s_bars + 72;  // [2]
	const uint32_t bar_park_free = s_bars + 88;  // [2]

	if (tid == 0) {
		for (uint32_t e = 0; e < NE; ++e) {
			mbar_init(bar_enc_full + 8 * e, WS_SUB_THREADS / 32);   // one arrival per memory warp
			mbar_init(bar_enc_free + 8 * e, WS_MLP_THREADS / 32);   // one arrival per MLP warp once its last wgmma reading enc completed
		}
		for (uint32_t g = 0; g < 2; ++g) {
			mbar_init(bar_park_full + 8 * g, WS_MLP_THREADS / 32);  // one arrival per MLP warp
			mbar_init(bar_park_free + 8 * g, WS_SUB_THREADS / 32);
		}
		fence_mbar_init();
	}
	if (dw_smem) {
		for (uint32_t i = tid; i < fused_ws_dw_bytes(NH) / 16; i += WS_THREADS) st_shared_v4(s_dw + 16 * i, 0, 0, 0, 0);
	}

	pdl_wait();  // everything above touched only shared memory; from here on the previous kernel's writes are needed
	{
		// W_l [out][in] row-major -> 128-byte tile rows (K-major, SWIZZLE_128B). Rows / columns beyond the network's width
		// and the encoding's width are zero, which makes a 16- or 32-wide network an exact sub-problem of the 64-wide tiles.
		const __half* __restrict__ w = p.params;  // MLP weights come first in the parameter buffer
		const uint32_t NW = p.width;
		auto stage = [&](uint32_t tile, const __half* __restrict__ src, uint32_t rows, uint32_t cols, uint32_t tile_rows) {
			for (uint32_t i = tid; i < tile_rows * 8; i += WS_THREADS) {
				const uint32_t r = i >> 3, c = i & 7;
				uint4 v = make_uint4(0, 0, 0, 0);
				if (r < rows && c * 8 < cols) v = __ldg(reinterpret_cast<const uint4*>(src + r * cols + c * 8));
				st_shared_v4(tile + sw128(r, c), v.x, v.y, v.z, v.w);
			}
		};
		stage(s_w0, w, NW, in_w, WIDTH);
		w += NW * in_w;
		for (uint32_t l = 1; l < NH; ++l) {
			stage(s_w0 + l * (WIDTH * 128), w, NW, NW, WIDTH);
			w += NW * NW;
		}
		stage(s_wout, w, 16, NW, 16);
	}
	fence_proxy_async_smem();
	__syncthreads();

	const uint32_t n_tiles = p.batch_size / TILE_M;
	// Tiles of this CTA: a CONTIGUOUS range [cta_first, cta_end) of the (spatially binned) batch. With a round-robin assignment
	// (tile = blockIdx + k * gridDim) all CTAs work on neighbouring tiles at any moment, i.e. on the same few cells of the coarse
	// dense levels, and their reductions queue up on the same L2 addresses. Contiguous ranges put concurrent CTAs in different regions.
	const uint32_t cta_first = (uint32_t)(((uint64_t)blockIdx.x * n_tiles) / gridDim.x);
	const uint32_t cta_end = (uint32_t)(((uint64_t)(blockIdx.x + 1) * n_tiles) / gridDim.x);

	if (warp >= WS_MLP_THREADS / 32) {
		// =========================================================================================== memory group
		// 640 threads start with 96 registers each (the count ptxas reports for the kernel); the MLP warpgroup holds two 64-column
		// accumulator fragments and takes what the memory warps give up (512 x 80 + 128 x 160 = 640 x 96). ptxas allocates each
		// branch to its new limit: without the exchange the training variants spill several hundred bytes.
		asm volatile("setmaxnreg.dec.sync.aligned.u32 80;\n" ::: "memory");
		const uint32_t mt = tid - WS_MLP_THREADS;
		const uint32_t sub = mt / WS_SUB_THREADS;   // sub-group; with SUBS == 2 it owns the tiles (and buffers) of parity `sub`
		const uint32_t lt = mt % WS_SUB_THREADS;
		const uint32_t row = lt & 127u;
		const uint32_t hsel = lt >> 7;

		constexpr uint32_t LEVELS_PER_CHUNK = 8 / F;
		const uint32_t n_chunks = in_w / 8;
		const uint32_t level_begin = hsel * (n_chunks / 2) * LEVELS_PER_CHUNK;
		const uint32_t level_end = min(p.grid.n_levels, level_begin + (n_chunks / 2) * LEVELS_PER_CHUNK);
		const __half* __restrict__ table = p.params + p.n_mlp_params;
		__half* __restrict__ grad_table = p.grads + p.n_mlp_params;

		// The level descriptor is indexed by a warp-uniform loop counter: it is read straight from the kernel parameters
		// (constant bank, uniform registers) and costs the load/store unit nothing.
		auto load_level = [&](uint32_t level) -> const LevelInfo& { return p.grid.levels[level]; };

		float x_prev[D], x_cur[D];
		uint32_t os_cur = 0;
#pragma unroll
		for (uint32_t d = 0; d < D; ++d) x_prev[d] = x_cur[d] = 0.0f;

		auto scatter_prev = [&](uint32_t gp) {
#pragma unroll 1
			for (uint32_t level = level_begin; level < level_end; ++level) {
				const LevelInfo& lv = load_level(level);
				LevelCorners<D> lc;
				level_corners<D>(lv, x_prev, p.grid.interpolation, lc);
				uint32_t gbits;
				const uint32_t feat = level * F;
				asm volatile("ld.shared.b32 %0, [%1];" : "=r"(gbits) : "r"(park_addr(gp, row, feat >> 3) + (feat & 7u) * 2u));
				const __half2 grad = *reinterpret_cast<const __half2*>(&gbits);
				uint32_t* __restrict__ ltab = reinterpret_cast<uint32_t*>(grad_table + (size_t)lv.offset * F);
#pragma unroll
				for (uint32_t pr = 0; pr < (1u << (D - 1)); ++pr) {
					// (GRAD_T)weight * grad -> __hmul2, then atomic f16x2 add (grid.h:252-255, vec.h:328-336)
					const __half2 a0 = __hmul2(__float2half2_rn(lc.w[2 * pr]), grad);
					const __half2 a1 = __hmul2(__float2half2_rn(lc.w[2 * pr + 1]), grad);
					const bool paired = (lc.paired >> pr) & 1u;
					if (!(TCNNB_ABLATE(ABLATE_SCATTER)) && !(TCNNB_ABLATE(ABLATE_SCATTER_DENSE) && lv.use_hash == 0) && !(TCNNB_ABLATE(ABLATE_SCATTER_HASH) && lv.use_hash != 0)) {
						scatter_pair_f16x2(ltab, lc.idx[2 * pr], lc.idx[2 * pr + 1], paired && !(TCNNB_ABLATE(ABLATE_PAIRING)), lv.wide_ok != 0, *reinterpret_cast<const uint32_t*>(&a0), *reinterpret_cast<const uint32_t*>(&a1));
					}
				}
			}
		};

		auto sample_of = [&](uint32_t tile) {
			const uint32_t s = tile * TILE_M + row;
			return p.perm ? __ldg(p.perm + s) : s;
		};
		// tiles of this sub-group: k = sub, sub + 2, ... (SUBS == 2) or every tile of the CTA (SUBS == 1)
		const uint32_t k_first = SUBS == 2 ? sub : 0u, k_step = SUBS;
		const uint32_t tile_first = cta_first + k_first, tile_stride = k_step;
		uint32_t os_next = tile_first < cta_end ? sample_of(tile_first) : 0;
		uint32_t os_next2 = tile_first + tile_stride < cta_end ? sample_of(tile_first + tile_stride) : 0;
		float x_next[D];
#pragma unroll
		for (uint32_t d = 0; d < D; ++d) x_next[d] = tile_first < cta_end ? __ldg(p.positions + (size_t)os_next * D + d) : 0.0f;
		bool have_prev = false;
		uint32_t k_prev = 0;
		for (uint32_t k = k_first, tile = tile_first; tile < cta_end; k += k_step, tile += tile_stride) {
			const uint32_t e = k % NE, je = k / NE;  // enc buffer and its use count
			const uint32_t enc_tile = s_enc + e * TILE_BYTES;
			// ---- position of this thread's sample (fetched one tile ahead, its index two tiles ahead: no dependent global
			//      load latency in front of the gather)
			os_cur = os_next;
			os_next = os_next2;
#pragma unroll
			for (uint32_t d = 0; d < D; ++d) x_cur[d] = x_next[d];
			if (tile + tile_stride < cta_end) {
#pragma unroll
				for (uint32_t d = 0; d < D; ++d) x_next[d] = __ldg(p.positions + (size_t)os_next * D + d);
			}
			if (tile + 2 * tile_stride < cta_end) os_next2 = sample_of(tile + 2 * tile_stride);

			// ---- gather tile k into enc[k % NE] once the MMAs of tile k - NE have released it
			if (lt == 0) WS_STAMP(1 + sub, k, 0);
			if (je >= 1) mbar_wait(bar_enc_free + 8 * e, (je - 1) & 1u);
			if (lt == 0) WS_STAMP(1 + sub, k, 1);
			// zero this thread's half of the row (padding features are zero, grid.h:759-766). With park_in_enc the upper half of
			// the tile holds parked gradients instead: the forward MMA reads only the first in_w columns, and what the
			// weight-gradient MMA makes of the rest lands in accumulator columns that are never flushed.
			// With park_in_enc only this thread's chunks BELOW in_w are zeroed (the parked upper half must be left alone), and only
			// when the levels do not fill them (n_levels * F < in_w, e.g. 12 levels -> 24 features padded to 32): the L0 MMA and the
			// dW0 weight-gradient MMA read all in_w columns.
			if (!park_in_enc || p.grid.n_features < in_w) {
#pragma unroll
				for (uint32_t c = 0; c < 4; ++c) {
					if (c >= n_chunks / 2 && park_in_enc) break;
					const uint32_t chunk = c < n_chunks / 2 ? hsel * (n_chunks / 2) + c : n_chunks + hsel * ((8 - n_chunks) / 2) + (c - n_chunks / 2);
					st_shared_v4(enc_tile + sw128(row, chunk), 0, 0, 0, 0);
				}
			}
			if (p.enc_identity) {
				// Identity encoding (encodings/identity.h:46-67): feature j = (half)(x_j * scale + offset) for j < D, ONE for the padding
				// features up to the network's input width; this thread writes its half of the row's 16-byte chunks.
				for (uint32_t c = 0; c < n_chunks / 2; ++c) {
					const uint32_t chunk = hsel * (n_chunks / 2) + c;
					__half f[8];
#pragma unroll
					for (uint32_t i = 0; i < 8; ++i) {
						const uint32_t jf = chunk * 8 + i;
						float v = 1.0f;
#pragma unroll
						for (uint32_t d = 0; d < D; ++d) v = jf == d ? __fmaf_rn(x_cur[d], p.identity_scale, p.identity_offset) : v;
						f[i] = __float2half_rn(v);
					}
					const uint4 q = *reinterpret_cast<const uint4*>(f);
					st_shared_v4(enc_tile + sw128(row, chunk), q.x, q.y, q.z, q.w);
					if (p.dbg_enc) *reinterpret_cast<uint4*>(p.dbg_enc + (size_t)os_cur * 64 + chunk * 8) = q;
				}
			}
			{
				// Three levels in flight: the loads of levels l+1 and l+2 are issued before the values of level l are consumed.
				// What travels with the loads is the fractional position (D floats), not the 2^D weights: they are rebuilt at
				// consumption, which is what makes the third level fit the register budget.
				// issue() returns bit k set when pair k came back as one 8-byte slot with its words in the other order from corner
				// order (gather_pair_f16x2); the bits of the three levels in flight travel together in one word, `swaps`, NP bits a level.
				constexpr uint32_t NP = 1u << (D - 1);
				struct InFlight {
					uint32_t vals[1u << D];
					float frac[D];
				};
				auto issue = [&](uint32_t level, InFlight& f) -> uint32_t {
					const LevelInfo& lv = load_level(level);
					LevelCorners<D> lc;
					level_corners<D>(lv, x_cur, p.grid.interpolation, lc);
					const uint32_t* __restrict__ ltab = reinterpret_cast<const uint32_t*>(table + (size_t)lv.offset * F);
					// Training: the hashed levels' gathers do not allocate in L1 (headline step, H100 80GB HBM3 at 400 W: fused kernel
					// 0.518 -> 0.483 ms), and a pair that shares an aligned slot is fetched with one 8-byte load. Inference keeps them
					// in L1: streaming them there measured 0.168 -> 0.242 ms.
					const bool streaming = TRAIN && lv.use_hash == LEVEL_HASH;
					uint32_t swapped = 0;
#pragma unroll
					for (uint32_t pr = 0; pr < NP; ++pr) {
						const bool paired = (lc.paired >> pr) & 1u;
						if (TCNNB_ABLATE(ABLATE_GATHER) || (TCNNB_ABLATE(ABLATE_GATHER_DENSE) && lv.use_hash == 0) || (TCNNB_ABLATE(ABLATE_GATHER_HASH) && lv.use_hash != 0)) {
							f.vals[2 * pr] = lc.idx[2 * pr];
							f.vals[2 * pr + 1] = lc.idx[2 * pr + 1];
						} else {
							const bool merge = streaming && lv.wide_ok && paired && !(TCNNB_ABLATE(ABLATE_PAIRING));
							swapped |= gather_pair_f16x2(ltab, lc.idx[2 * pr], lc.idx[2 * pr + 1], merge, streaming, f.vals[2 * pr], f.vals[2 * pr + 1]) << pr;
						}
					}
#pragma unroll
					for (uint32_t d = 0; d < D; ++d) f.frac[d] = lc.frac[d];
					return swapped;
				};
				auto consume = [&](uint32_t level, const InFlight& f, uint32_t swapped) {
					float w[1u << D];
					corner_weights<D>(f.frac, w);
					__half2 result = __float2half2_rn(0.0f);
#pragma unroll
					for (uint32_t idx = 0; idx < (1u << D); ++idx) {
						const bool sw = (swapped >> (idx / 2)) & 1u;
						const uint32_t v = sw ? f.vals[idx ^ 1u] : f.vals[idx];
						// fma((T)weight, grid_val, result) with T = __half -> __hfma2 (grid.h:162, vec.h:372-378)
						result = __hfma2(__float2half2_rn(w[idx]), *reinterpret_cast<const __half2*>(&v), result);
					}
					const uint32_t feat = level * F;
					asm volatile("st.shared.b32 [%0], %1;" ::"r"(enc_tile + sw128(row, feat >> 3) + (feat & 7u) * 2u), "r"(*reinterpret_cast<uint32_t*>(&result)) : "memory");
					if (p.dbg_enc) *reinterpret_cast<uint32_t*>(p.dbg_enc + (size_t)os_cur * 64 + feat) = *reinterpret_cast<uint32_t*>(&result);
				};
				if (level_begin < level_end) {
					InFlight f0, f1, f2;
					uint32_t swaps = issue(level_begin, f0);
					if (level_begin + 1 < level_end) swaps |= issue(level_begin + 1, f1) << NP;
#pragma unroll 1
					for (uint32_t level = level_begin; level < level_end; ++level) {
						if (level + 2 < level_end) swaps |= issue(level + 2, f2) << (2 * NP);
						consume(level, f0, swaps);
						swaps >>= NP;
						f0 = f1;
						f1 = f2;
					}
				}
			}
			fence_proxy_async_smem();  // the tile is read by wgmma (async proxy)
			__syncwarp();
			if ((tid & 31u) == 0) mbar_arrive(bar_enc_full + 8 * e);
			if (lt == 0) WS_STAMP(1 + sub, k, 2);

			// ---- scatter the previous tile of this sub-group while the MLP group chews on the tiles in between
			if (TRAIN && have_prev) {
				const uint32_t gp = k_prev & 1u, jp = k_prev >> 1;
				mbar_wait(bar_park_full + 8 * gp, jp & 1u);
				if (lt == 0) WS_STAMP(1 + sub, k, 3);
				scatter_prev(gp);
				__syncwarp();
				if ((tid & 31u) == 0) mbar_arrive(bar_park_free + 8 * gp);
				if (lt == 0) WS_STAMP(1 + sub, k, 4);
			}
#pragma unroll
			for (uint32_t d = 0; d < D; ++d) x_prev[d] = x_cur[d];
			have_prev = true;
			k_prev = k;
		}
		pdl_launch_dependents();  // the optimizer's CTAs may start arriving (they block until this grid has completed)
		if (TRAIN && have_prev) {  // drain: the last tile of this sub-group
			const uint32_t gp = k_prev & 1u, jp = k_prev >> 1;
			mbar_wait(bar_park_full + 8 * gp, jp & 1u);
			scatter_prev(gp);
		}
	} else {
		// =========================================================================================== MLP group
		// One warpgroup. Every MMA covers the 128-row tile as two m64 halves; thread (warp w, lane) holds the accumulator fragment
		// rows mh * 64 + 16 w + lane / 4 (+ 8), columns 8 i + 2 (lane % 4) (+ 1) -- see Wgmma in ptx.cuh. The per-row work of the
		// output layer (loss, outputs) is done by thread `row` after the fragment has been staged in shared memory.
		asm volatile("setmaxnreg.inc.sync.aligned.u32 160;\n" ::: "memory");
		const uint32_t row = tid;  // 0..127
		const uint32_t fq = (tid & 31u) >> 2, ft = tid & 3u;
		float loss_acc = 0.0f;
		bool dw_started = false;
		auto frow = [&](uint32_t mh, uint32_t hi) { return mh * 64u + warp * 16u + fq + hi * 8u; };

		auto kmaj = [](uint32_t tile, uint32_t jj) { return wgmma_desc_sw128(tile + jj * 32u, 16u, 1024u); };
		auto mnmaj = [](uint32_t tile, uint32_t jj) { return wgmma_desc_sw128(tile + jj * 2048u, TILE_BYTES, 1024u); };
		auto stage_sync = [&]() {
			fence_proxy_async_smem();
			named_bar_sync(1, WS_MLP_THREADS);
		};
		// this warp's wgmma groups have completed: release an mbarrier that counts one arrival per MLP warp
		auto warp_arrive = [&](uint32_t bar) {
			__syncwarp();
			if ((tid & 31u) == 0) mbar_arrive(bar);
		};
		// acc[mh] = A[rows of half mh] . B over `ksteps` steps of 16: A K-major (128-row tile), B K-major (forward) or MN-major (dgrad)
		float acc[2][32];
		auto mma64 = [&](uint32_t a_tile, uint32_t b_tile, uint32_t ksteps, bool b_mn) {
			wgmma_fence();
#pragma unroll
			for (uint32_t mh = 0; mh < 2; ++mh) {
				for (uint32_t jj = 0; jj < ksteps; ++jj) {
					if (b_mn) Wgmma<64>::ss<0, 1>(acc[mh], kmaj(a_tile + mh * 8192u, jj), mnmaj(b_tile, jj), jj > 0);
					else Wgmma<64>::ss<0, 0>(acc[mh], kmaj(a_tile + mh * 8192u, jj), kmaj(b_tile, jj), jj > 0);
				}
			}
			wgmma_commit();
			wgmma_wait<0>();
			reg_fence(acc[0]);
			reg_fence(acc[1]);
		};
		// fragment words d[4 i .. 4 i + 3] of weight matrix l (l == NH: W_out) -> the global fp32 accumulator. d[4 i + q]: row
		// m = 16 w + lane / 4 (+ 8 for q >= 2), column n = 8 i + 2 (lane % 4) + (q & 1); the rows are the matrix's outputs, for W_out its inputs
		auto flush_dw = [&](uint32_t l, uint32_t i, const float* x) {
			const uint32_t n = 8 * i + 2 * ft;
#pragma unroll
			for (uint32_t hi = 0; hi < 2; ++hi) {
				const uint32_t m = warp * 16 + fq + hi * 8;
				const float v0 = x[2 * hi], v1 = x[2 * hi + 1];
				if (m >= p.width) continue;
				if (l == 0) {
					if (n < in_w) red_add_v2_f32(p.dw_accum + m * in_w + n, v0, v1);
				} else if (l < NH) {
					if (n < p.width) red_add_v2_f32(p.dw_accum + p.width * in_w + (l - 1) * p.width * p.width + m * p.width + n, v0, v1);
				} else {
					float* dst = p.dw_accum + p.width * in_w + (NH - 1) * p.width * p.width;  // W_out [16][width]
					red_add_f32(dst + n * p.width + m, v0);
					red_add_f32(dst + (n + 1) * p.width + m, v1);
				}
			}
		};
		// dW_l += A^T . B over the tile's 128 samples (both operands MN-major): N = 64, or 16 for W_out (l == NH). The fp32 sums
		// round-trip through s_dw, or go to the global accumulator after every tile.
		auto wgrad = [&](uint32_t l, uint32_t a_tile, uint32_t b_tile) {
			const uint32_t dw_addr = s_dw + l * WS_DW_BYTES;
			const uint32_t n_i = l == NH ? 2u : 8u;
			float d[32];
#pragma unroll
			for (uint32_t i = 0; i < 8; ++i) {
				uint32_t x = 0, y = 0, z = 0, w = 0;
				if (dw_smem && i < n_i) ld_shared_v4(dw_addr + (i * WS_MLP_THREADS + tid) * 16u, x, y, z, w);
				d[4 * i] = __uint_as_float(x), d[4 * i + 1] = __uint_as_float(y), d[4 * i + 2] = __uint_as_float(z), d[4 * i + 3] = __uint_as_float(w);
			}
			wgmma_fence();
			if (l == NH) {
#pragma unroll
				for (uint32_t jj = 0; jj < TILE_M / 16; ++jj) Wgmma<16>::ss<1, 1>(reinterpret_cast<float(&)[8]>(d[0]), mnmaj(a_tile, jj), mnmaj(b_tile, jj), 1);
			} else {
#pragma unroll
				for (uint32_t jj = 0; jj < TILE_M / 16; ++jj) Wgmma<64>::ss<1, 1>(d, mnmaj(a_tile, jj), mnmaj(b_tile, jj), 1);
			}
			wgmma_commit();
			wgmma_wait<0>();
			reg_fence(d);
#pragma unroll
			for (uint32_t i = 0; i < 8; ++i) {
				if (i >= n_i) continue;
				if (dw_smem) st_shared_v4(dw_addr + (i * WS_MLP_THREADS + tid) * 16u, __float_as_uint(d[4 * i]), __float_as_uint(d[4 * i + 1]), __float_as_uint(d[4 * i + 2]), __float_as_uint(d[4 * i + 3]));
				else flush_dw(l, i, d + 4 * i);
			}
		};

		const uint32_t n_batches = TRAIN ? 2 * NH + 2 : NH + 1;
		// The sample index (through the binning permutation) and the targets are global loads whose latency, under the memory
		// group's traffic, would otherwise sit in the middle of this group's dependent MMA / epilogue chain: the index is
		// fetched one tile ahead, the targets at the top of the tile (the loss needs them three MMA stages later).
		constexpr uint32_t N_TGT_PREFETCH = 4;
		auto sample_of = [&](uint32_t tile, uint32_t r) {
			const uint32_t s = tile * TILE_M + r;
			return p.perm ? __ldg(p.perm + s) : s;
		};
		uint32_t osample_next = cta_first < cta_end ? sample_of(cta_first, row) : 0;
		uint32_t k = 0;
		for (uint32_t tile = cta_first; tile < cta_end; ++tile, ++k) {
			const uint32_t g = k & 1u, j = k >> 1;
			const uint32_t e = k % NE, je = k / NE;
			const uint32_t enc_cur = s_enc + e * TILE_BYTES;
			const uint32_t osample = osample_next;
			float tgt[N_TGT_PREFETCH];
			uint4 edy_lo = make_uint4(0, 0, 0, 0), edy_hi = make_uint4(0, 0, 0, 0);
			if (TRAIN) {
				if (p.ext_dy) {  // module-tier backward: the caller's dL/d(output) row instead of targets
					edy_lo = __ldg(reinterpret_cast<const uint4*>(p.ext_dy + (size_t)osample * 16));
					edy_hi = __ldg(reinterpret_cast<const uint4*>(p.ext_dy + (size_t)osample * 16) + 1);
				} else {
#pragma unroll
					for (uint32_t q = 0; q < N_TGT_PREFETCH; ++q) tgt[q] = q < p.n_out ? __ldg(p.targets + (size_t)osample * p.n_out + q) : 0.0f;
				}
			}
			if (tile + 1 < cta_end) osample_next = sample_of(tile + 1, row);
			if (tid == 0) WS_STAMP(0, k, 0);
			mbar_wait(bar_enc_full + 8 * e, je & 1u);
			if (tid == 0) WS_STAMP(0, k, 1);

#pragma unroll 1
			for (uint32_t b = 0; b < n_batches; ++b) {
				if (tid == 0 && (b == 1 || b == NH + 1)) WS_STAMP(0, k, b == 1 ? 6 : 11);
				if (tid == 0 && (b == 2 || b == NH + 2)) WS_STAMP(0, k, b == 2 ? 10 : 15);
				stage_sync();
				if (tid == 0 && b == NH + 1) WS_STAMP(0, k, 2);
				if (tid == 0 && (b == 1 || b == NH + 1)) WS_STAMP(0, k, b == 1 ? 7 : 12);
				// ---- MMAs of batch b (the weight gradients first: the epilogue below overwrites h_{l-1} with g_{l-1} in place)
				if (b < NH) {
					mma64(b == 0 ? enc_cur : s_h0 + (b - 1) * TILE_BYTES, s_w0 + b * (WIDTH * 128), b == 0 ? in_w / 16 : WIDTH / 16, false);
					if (!TRAIN && b == 0) warp_arrive(bar_enc_free + 8 * e);  // inference: L0 is the only reader of enc
				} else if (b == NH) {
					wgmma_fence();
#pragma unroll
					for (uint32_t mh = 0; mh < 2; ++mh) {
						float(&a16)[8] = reinterpret_cast<float(&)[8]>(acc[mh][0]);
						for (uint32_t jj = 0; jj < WIDTH / 16; ++jj) Wgmma<16>::ss<0, 0>(a16, kmaj(s_h0 + (NH - 1) * TILE_BYTES + mh * 8192u, jj), kmaj(s_wout, jj), jj > 0);
					}
					wgmma_commit();
					wgmma_wait<0>();
					reg_fence(reinterpret_cast<float(&)[8]>(acc[0][0]));
					reg_fence(reinterpret_cast<float(&)[8]>(acc[1][0]));
				} else if (b <= 2 * NH) {
					const uint32_t l = 2 * NH + 1 - b;
					const uint32_t h_prev = s_h0 + (l - 1) * TILE_BYTES;
					if (l == NH) {
						wgrad(NH, h_prev, s_dy);
						mma64(s_dy, s_wout, 1, true);
					} else {
						const uint32_t g_tile = s_h0 + l * TILE_BYTES;
						wgrad(l, g_tile, h_prev);
						mma64(g_tile, s_w0 + l * (WIDTH * 128), WIDTH / 16, true);
					}
				} else {
					wgrad(0, s_h0, enc_cur);
					mma64(s_h0, s_w0, WIDTH / 16, true);
					warp_arrive(bar_enc_free + 8 * e);  // last reader of this enc buffer: release it to the memory group
				}
				// From the output layer on, the epilogue writes a tile that this batch's products have read: the staging tile of the
				// inference output (h_{NH-1}), h_{l-1} (dgrad overwrites it with g_{l-1} after the wgrad read it), the parked
				// dL/d(enc) rows in the enc tile (read by the dW_0 product). wgmma.wait_group covers only the calling warp's share of
				// a product, and every warp's share reads all 128 rows of an MN-major operand: the four warps meet here first.
				if (b >= NH) named_bar_sync(1, WS_MLP_THREADS);
				if (tid == 0 && (b == 1 || b == NH + 1)) WS_STAMP(0, k, b == 1 ? 9 : 14);

				// ---- epilogue of batch b on the accumulator fragment
				if (b < NH) {
					const uint32_t h_tile = s_h0 + b * TILE_BYTES;
#pragma unroll
					for (uint32_t mh = 0; mh < 2; ++mh) {
#pragma unroll
						for (uint32_t hi = 0; hi < 2; ++hi) {
							const uint32_t r = frow(mh, hi);
#pragma unroll
							for (uint32_t i = 0; i < 8; ++i) {
								const uint32_t v = act_pack(hid_act, __float_as_uint(acc[mh][4 * i + 2 * hi]), __float_as_uint(acc[mh][4 * i + 2 * hi + 1]));
								asm volatile("st.shared.b32 [%0], %1;" ::"r"(h_tile + sw128(r, i) + 4u * ft), "r"(v) : "memory");
								if (p.dbg_hidden) *reinterpret_cast<uint32_t*>(p.dbg_hidden + ((size_t)b * p.batch_size + sample_of(tile, r)) * 64 + 8 * i + 2 * ft) = v;
							}
						}
					}
				} else if (b == NH) {
					// the fp16-rounded outputs go through the row-major staging tile (dy in training, the last hidden layer's tile --
					// which the output MMA has finished reading -- in inference) to the thread that owns the row
					const uint32_t stg = TRAIN ? s_dy : s_h0 + (NH - 1) * TILE_BYTES;
#pragma unroll
					for (uint32_t mh = 0; mh < 2; ++mh) {
#pragma unroll
						for (uint32_t hi = 0; hi < 2; ++hi) {
#pragma unroll
							for (uint32_t i = 0; i < 2; ++i) {
								const uint32_t v = pack_half2(acc[mh][4 * i + 2 * hi], acc[mh][4 * i + 2 * hi + 1]);
								asm volatile("st.shared.b32 [%0], %1;" ::"r"(stg + sw128(frow(mh, hi), i) + 4u * ft), "r"(v) : "memory");
							}
						}
					}
					named_bar_sync(1, WS_MLP_THREADS);
					__half y16[16];
					{
						uint4 lo, hi;
						ld_shared_v4(stg + sw128(row, 0), lo.x, lo.y, lo.z, lo.w);
						ld_shared_v4(stg + sw128(row, 1), hi.x, hi.y, hi.z, hi.w);
						*reinterpret_cast<uint4*>(&y16[0]) = lo;
						*reinterpret_cast<uint4*>(&y16[8]) = hi;
					}
#pragma unroll
					for (uint32_t q = 0; q < 16; ++q) y16[q] = act_fwd_h(out_act, y16[q]);
					if (p.out_fp16) {
						uint4* dst = reinterpret_cast<uint4*>(p.out_fp16 + (size_t)osample * 16);
						dst[0] = *reinterpret_cast<uint4*>(&y16[0]);
						dst[1] = *reinterpret_cast<uint4*>(&y16[8]);
					}
					if (p.out_fp32) {
						for (uint32_t q = 0; q < p.n_out; ++q) p.out_fp32[(size_t)osample * p.n_out + q] = __half2float(y16[q]);
					}
					if (TRAIN) {
						// relative_l2_loss / l2_loss (losses/relative_l2.h:56-75, l2.h:56-74); pad lanes give 0.
						__half dy[16];
						const float n_total = (float)(p.loss_batch_size * p.n_out);
						const float luminance = p.loss_type == LOSS_RELATIVE_L2_LUMINANCE ? row_luminance(y16, p.n_out) : 0.0f;
						if (p.ext_dy) {
							// Module::backward (cpp_api.cu:115-124): dL/d(output) comes from the caller and, like the loss gradient below,
							// passes through the output activation's transfer (fully_fused_mlp.cu:758-762)
							*reinterpret_cast<uint4*>(&dy[0]) = edy_lo;
							*reinterpret_cast<uint4*>(&dy[8]) = edy_hi;
#pragma unroll
							for (uint32_t q = 0; q < 16; ++q) dy[q] = act_bwd_h(out_act, dy[q], y16[q]);
						} else
#pragma unroll
						for (uint32_t q = 0; q < 16; ++q) {
							float gq = 0.0f;
							if (q < p.n_out) {
								const float pred = __half2float(y16[q]);
								const float target = q < N_TGT_PREFETCH ? tgt[q] : __ldg(p.targets + (size_t)osample * p.n_out + q);
								float value, grad;
								if constexpr (PDF) loss_element_pdf(p.loss_type, pred, target, __ldg(p.data_pdf + (size_t)osample * p.n_out + q), n_total, luminance, value, grad);
								else loss_element(p.loss_type, pred, target, n_total, luminance, value, grad);
								gq = p.loss_scale * grad / n_total;
								loss_acc += value;
								if (p.loss_values) p.loss_values[(size_t)osample * p.n_out + q] = value;
							}
							// activation_backward_output (fully_fused_mlp.cu:755-759): dL/dy through the output activation, in fp16
						dy[q] = act_bwd_h(out_act, __float2half_rn(gq), y16[q]);
						}
						const uint4 lo = *reinterpret_cast<uint4*>(&dy[0]), hi = *reinterpret_cast<uint4*>(&dy[8]);
						st_shared_v4(s_dy + sw128(row, 0), lo.x, lo.y, lo.z, lo.w);
						st_shared_v4(s_dy + sw128(row, 1), hi.x, hi.y, hi.z, hi.w);
						if (p.dbg_dy) {
							uint4* dst = reinterpret_cast<uint4*>(p.dbg_dy + (size_t)osample * 16);
							dst[0] = lo;
							dst[1] = hi;
						}
					}
				} else if (b <= 2 * NH) {
					// g overwrites h in place: each thread rewrites the words of the fragment it has just read
					const uint32_t l = 2 * NH + 1 - b;
					const uint32_t h_tile = s_h0 + (l - 1) * TILE_BYTES;
#pragma unroll
					for (uint32_t mh = 0; mh < 2; ++mh) {
#pragma unroll
						for (uint32_t hi = 0; hi < 2; ++hi) {
							const uint32_t r = frow(mh, hi);
#pragma unroll
							for (uint32_t i = 0; i < 8; ++i) {
								const uint32_t addr = h_tile + sw128(r, i) + 4u * ft;
								uint32_t f;
								asm volatile("ld.shared.b32 %0, [%1];" : "=r"(f) : "r"(addr) : "memory");
								const uint32_t v = act_bwd_pack(hid_act, __float_as_uint(acc[mh][4 * i + 2 * hi]), __float_as_uint(acc[mh][4 * i + 2 * hi + 1]), f);
								asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
								if (p.dbg_grad_hidden) *reinterpret_cast<uint32_t*>(p.dbg_grad_hidden + ((size_t)(l - 1) * p.batch_size + sample_of(tile, r)) * 64 + 8 * i + 2 * ft) = v;
							}
						}
					}
				} else {
					// dL/d(encoded): round once to fp16 (fully_fused_mlp.cu:835) and park the row for the memory group
					dw_started = true;
					if (tid == 0) WS_STAMP(0, k, 3);
					if (j >= 1) mbar_wait(bar_park_free + 8 * g, (j - 1) & 1u);  // scatter of tile k-2 has consumed park[g]
					if (tid == 0) WS_STAMP(0, k, 4);
#pragma unroll
					for (uint32_t mh = 0; mh < 2; ++mh) {
#pragma unroll
						for (uint32_t hi = 0; hi < 2; ++hi) {
							const uint32_t r = frow(mh, hi);
#pragma unroll
							for (uint32_t i = 0; i < 8; ++i) {
								const uint32_t v = pack_half2(acc[mh][4 * i + 2 * hi], acc[mh][4 * i + 2 * hi + 1]);
								if (i * 8 < in_w) asm volatile("st.shared.b32 [%0], %1;" ::"r"(park_addr(g, r, i) + 4u * ft), "r"(v) : "memory");
								if (p.dbg_denc) *reinterpret_cast<uint32_t*>(p.dbg_denc + (size_t)sample_of(tile, r) * 64 + 8 * i + 2 * ft) = v;
							}
						}
					}
					warp_arrive(bar_park_full + 8 * g);
					if (tid == 0) WS_STAMP(0, k, 5);
				}
			}
		}

		pdl_launch_dependents();
		// ---- flush the weight-gradient sums and the loss
		if (TRAIN) {
			named_bar_sync(1, WS_MLP_THREADS);
			if (dw_smem && dw_started) {
				for (uint32_t l = 0; l <= NH; ++l) {
					for (uint32_t i = 0; i < (l == NH ? 2u : 8u); ++i) {
						uint32_t x[4];
						ld_shared_v4(s_dw + l * WS_DW_BYTES + (i * WS_MLP_THREADS + tid) * 16u, x[0], x[1], x[2], x[3]);
						const float v[4] = {__uint_as_float(x[0]), __uint_as_float(x[1]), __uint_as_float(x[2]), __uint_as_float(x[3])};
						flush_dw(l, i, v);
					}
				}
			}
#pragma unroll
			for (uint32_t o = 16; o > 0; o >>= 1) loss_acc += __shfl_xor_sync(0xFFFFFFFFu, loss_acc, o);
			if ((tid & 31u) == 0 && p.loss_sum) atomicAdd(p.loss_sum, loss_acc);
		}
	}
}

// ------------------------------------------------------------------------------------------------------------------
size_t fused_ws_smem_bytes(uint32_t n_hidden_layers, uint32_t enc_width, bool train) {
	return fused_ws_base_smem_bytes(n_hidden_layers, enc_width, train) + (train && fused_ws_dw_in_smem(n_hidden_layers, enc_width) ? fused_ws_dw_bytes(n_hidden_layers) : 0);
}

template <uint32_t D, bool TRAIN, bool GENERIC, bool PDF>
static cudaError_t launch_ws_impl(const FusedStepParams& p, uint32_t n_ctas, cudaStream_t stream) {
	auto kernel = fused_ws_kernel<D, 2, TRAIN, GENERIC, PDF>;
	const size_t smem = fused_ws_smem_bytes(p.n_hidden_layers, p.grid.padded_width, TRAIN);
	cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
	if (err != cudaSuccess) return err;
	// ask for the smallest shared-memory carve-out that holds the CTA (+1 KB the system reserves): the rest is L1
	const size_t per_sm = smem + 1024;
	err = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)(per_sm * 100 / (228 * 1024))  /* rounded DOWN: the driver still has to fit the kernel, so it takes the first configuration that does (rounding up skipped the 100 KB one) */);
	if (err != cudaSuccess) return err;
	return launch_pdl(kernel, n_ctas, WS_THREADS, smem, stream, p);
}

template <uint32_t D, bool TRAIN, bool PDF>
static cudaError_t launch_ws_act(const FusedStepParams& p, uint32_t n_ctas, cudaStream_t stream) {
	const bool generic = p.activation != ACT_RELU || p.output_activation != ACT_NONE;
	return generic ? launch_ws_impl<D, TRAIN, true, PDF>(p, n_ctas, stream) : launch_ws_impl<D, TRAIN, false, PDF>(p, n_ctas, stream);
}

// the pdf is read by the loss only: inference and steps on a caller's dL/d(output) run the kernels without it
template <uint32_t D, bool TRAIN>
static cudaError_t launch_ws_pdf(const FusedStepParams& p, uint32_t n_ctas, cudaStream_t stream) {
	if (TRAIN && p.data_pdf && !p.ext_dy) return launch_ws_act<D, TRAIN, TRAIN>(p, n_ctas, stream);
	return launch_ws_act<D, TRAIN, false>(p, n_ctas, stream);
}

cudaError_t launch_fused_ws(const FusedStepParams& p, uint32_t n_pos_dims, bool train, uint32_t n_ctas, cudaStream_t stream) {
	if (n_pos_dims == 3) return train ? launch_ws_pdf<3, true>(p, n_ctas, stream) : launch_ws_pdf<3, false>(p, n_ctas, stream);
	if (n_pos_dims == 2) return train ? launch_ws_pdf<2, true>(p, n_ctas, stream) : launch_ws_pdf<2, false>(p, n_ctas, stream);
	return cudaErrorInvalidValue;
}

}  // namespace tcnnb
