// mlp_fused.cu -- stand-alone FullyFusedMLP forward / inference on wgmma: the tensor-core-bound kernel of the general path.
//
// Replaces the reference's kernel_mlp_fused<WIDTH, ..., INFERENCE> (fully_fused_mlp.cu:499-557: threadblock_input_layer_forward_dynamic
// :315-419, threadblock_layer :47-129, threadblock_last_layer_forward :421-476) for Network<T>::inference_mixed_precision
// (benchmarks/mlp/bench_mlp_ours.cu:107-120) and, with the Identity encoding fused into the input load, for
// cpp::create_network / NetworkWithInputEncoding(Identity) (src/cpp_api.cu:160-162, encodings/identity.h:46-67).
//
// The reference keeps a 128-sample tile's activations in shared memory and re-reads the weights from L2 into registers for every
// layer of every block (HMMA.F16). Here, per persistent CTA (one per SM):
//
//   * weights are loaded ONCE with TMA (cp.async.bulk.tensor, SWIZZLE_128B boxes of 64 K-elements) into shared memory and stay
//     there as the K-major B operands of every tile; networks with more matrices than fit (128 wide: > 6) stream them through
//     the same stages as a ring (w_full / w_free mbarriers);
//   * activations NEVER touch shared memory: each consumer warpgroup owns a 64-sample unit of the batch; layer l accumulates
//     D = A_l . W_l^T in registers (fp32, wgmma m64nNk16), the warpgroup applies the activation in fp16 (as
//     warp_activation<__half>, common_device.h:110-215) and packs the result straight into the register fragment the next
//     layer's wgmma reads as its A operand (the accumulator and A fragments of wgmma share the row / column assignment);
//   * WGS consumer warpgroups work on independent units, so that one warpgroup's epilogue overlaps another's MMAs.
//
// Warp roles: warpgroups 0 .. WGS-1 = consumers (one 64-sample unit at a time); the last warp = TMA producer (weights).
// mbarriers:  w_full[stage] (TMA complete_tx), w_free[stage] (one arrival per consumer warp: ring mode only)
//
// Numerics: fp16 operands, fp32 accumulation, ONE rounding to fp16 per layer (the reference accumulates in fp16 inside HMMA;
// tolerance statement in DESIGN.md section 4).
#include "mlp_fused.h"

#include "fused_common.cuh"
#include "ptx.cuh"

#include "tma_host.h"

namespace tcnnb {

using namespace ptx;
using namespace fused;

namespace {

constexpr uint32_t MLPF_MAX_STAGES = 32;
constexpr uint32_t UNIT_M = 64;  // samples per consumer warpgroup and MMA

template <uint32_t W>
struct MlpCfg {
	static constexpr uint32_t WGS = W == 128 ? 2 : 4;          // consumer warpgroups
	static constexpr uint32_t THREADS = WGS * 128 + 32;        // + the TMA producer warp
	static constexpr uint32_t ACC_N = W < 32 ? 32 : W;         // accumulator columns: the widest product of the chain (dL/d(input) of
	                                                           // a 16-wide network is up to 32 wide)
	static constexpr uint32_t KMAX = W == 128 ? 128 : 64;      // widest K (the network input may be wider than the layers)
	static constexpr uint32_t KBLOCKS = (W + 63) / 64;         // 64-element K blocks of a weight stage
	static constexpr uint32_t KBLOCK_BYTES = W * 128;          // [W rows][64 fp16], SWIZZLE_128B
	static constexpr uint32_t STAGE_BYTES = KBLOCKS * KBLOCK_BYTES < 2048 ? 2048 : KBLOCKS * KBLOCK_BYTES;
};

struct MlpKernelParams {
	MlpChainParams p;
	uint32_t n_stages;  // == n_steps when all matrices are resident
	uint32_t resident;
	uint32_t n_steps;   // MMAs chained per unit: n_hidden_layers + 1 (the backward chain without dL/d(input): n_hidden_layers)
	__half* hidden_pre_out;  // MlpForwardParams::hidden_pre_out (PRE kernels only)
};

}  // namespace

// The forward output rows of the WIDE kernels. In the accumulator fragment lane (fq, ft) of a warp holds, for every i, columns
// 8 i + 2 ft and 8 i + 2 ft + 1 of row fq: stored as they are, a warp store writes 16 bytes in each of 8 rows. Four consecutive i
// (v0 .. v3, packed half2) are transposed across the lane's quad instead, so that lane ft ends up with the 8 columns of i = 4 j + ft
// and stores them as one 16-byte vector: a quad then writes 64 contiguous bytes of its row.
__device__ __forceinline__ uint4 quad_transpose(uint32_t v0, uint32_t v1, uint32_t v2, uint32_t v3, uint32_t lane) {
	const uint32_t ft = lane & 3u;
	uint32_t o0 = 0, o1 = 0, o2 = 0, o3 = 0;
#pragma unroll
	for (uint32_t r = 0; r < 4; ++r) {
		// round r: lane d reads lane s = d - r of its quad, which sends its v_{s + r} = v_d: columns 2 s, 2 s + 1 of d's 8
		const uint32_t k = (ft + r) & 3u, src = (ft - r) & 3u;
		const uint32_t got = __shfl_sync(0xFFFFFFFFu, k == 0 ? v0 : (k == 1 ? v1 : (k == 2 ? v2 : v3)), (lane & ~3u) | src);
		o0 = src == 0 ? got : o0;
		o1 = src == 1 ? got : o1;
		o2 = src == 2 ? got : o2;
		o3 = src == 3 ? got : o3;
	}
	return make_uint4(o0, o1, o2, o3);
}

// Phase stamps (tcnnb_network_debug_clocks, profiling only): [cta][role = consumer warpgroup 0..3, 4 unused][event = round * n_steps +
// step, < 64][field: 0 = waiting for the weights, 1 = weights ready, 2 = product complete, 3 = epilogue done], written by the first
// thread of the warpgroup.
#define MLPF_STAMP(role, event, field)                                                                                               \
	do {                                                                                                                             \
		if (p.dbg_clock && (event) < 64u) p.dbg_clock[(((size_t)blockIdx.x * 5u + (role)) * 64u + (event)) * 8u + (field)] = clock64(); \
	} while (0)

// The chain of one 64-sample unit in one consumer warpgroup. Thread (warp w of the group, lane) owns rows r0 = 16 w + lane / 4 and
// r0 + 8 of the unit, and the column pairs 8 i + 2 (lane % 4) of every accumulator / A fragment (ptx.cuh, Wgmma).
//
// BWD = true is the same machine run backwards (threadblock_layer<..., BACKWARD>, fully_fused_mlp.cu:47-129,151-259): the operand that
// enters is dL/d(output) (already through the output activation's transfer), step j multiplies by matrix NH - j read MN-major
// -- the SAME bytes TMA delivered, W^T without a transposed copy --, the hidden epilogue multiplies by the activation's derivative
// (from the forward pass's post-activation values in `hidden_in`) and writes g_l to `hidden_out` (for the weight-gradient kernel,
// mlp_wgrad.cu), and what leaves is dL/d(input).
//
// PRE = true (with GENERIC_ACT): the hidden activation is Sine or SiLU, whose derivative needs the PRE-activation z (the reference's
// CutlassMLP keeps both buffers for them, cutlass_mlp.cu:162-209, 266-304). Forward: the hidden epilogue rounds z to fp16, stores it
// to `hidden_pre_out` (when given) and applies the activation to that fp16 z. Backward: `hidden_in` holds the forward pass's z, and
// the epilogue multiplies by act'(z).
//
// WIDE = true: the padded output is wider than the layers (out_width > W). The output matrix then takes n_oc = ceil(out_width / W)
// steps of W of its rows each, every one a weight stage like a hidden matrix ([W rows][64 K] boxes, the last one zero-filled by TMA
// past out_width). Forward, the chunks all multiply the same A fragment -- the last hidden layer, which no epilogue overwrites any
// more -- and each writes its W output columns. Backward, the chunks are the K-blocks of the first product: each loads its W columns
// of dL/d(output) into the A fragment (after the previous chunk's wgmma has completed) and accumulates; only the last runs the
// epilogue.
template <uint32_t W, bool GENERIC_ACT, bool BWD, bool PRE, bool WIDE>
__global__ void __launch_bounds__(MlpCfg<W>::THREADS, 1)
mlp_forward_kernel(const MlpKernelParams kp, const __grid_constant__ CUtensorMap map_w0, const __grid_constant__ CUtensorMap map_wh, const __grid_constant__ CUtensorMap map_wo) {
	using C = MlpCfg<W>;
	static_assert(!PRE || GENERIC_ACT, "the pre-activation path is a generic-activation kernel");
	const MlpChainParams& p = kp.p;
	const uint32_t hid_act = GENERIC_ACT ? p.activation : (uint32_t)ACT_RELU;
	const uint32_t out_act = BWD ? (uint32_t)ACT_NONE : (GENERIC_ACT ? p.output_activation : (uint32_t)ACT_NONE);
	extern __shared__ __align__(1024) uint8_t smem_raw[];
	const uint32_t tid = threadIdx.x;
	const uint32_t warp = __shfl_sync(0xFFFFFFFFu, tid >> 5, 0);
	const uint32_t lane = tid & 31u;
	const uint32_t NH = p.n_hidden_layers, n_layers = kp.n_steps;
	const uint32_t in_w = p.in_width, out_w = p.out_width;
	const uint32_t first_w = BWD ? out_w : in_w;  // width of the rows that enter the chain ...
	const uint32_t last_w = BWD ? in_w : out_w;   // ... and of the rows that leave it
	const uint32_t n_stages = kp.n_stages;
	const bool resident = kp.resident != 0;
	const uint32_t n_oc = WIDE ? (out_w + W - 1) / W : 1u;  // steps of the output matrix
	// step of the unit -> layer of the chain (as counted without WIDE) and chunk of the output matrix
	auto chain_layer = [&](uint32_t step, uint32_t& oc) -> uint32_t {
		oc = 0;
		if (!WIDE) return step;
		if (BWD) {
			if (step < n_oc) oc = step;
			return step < n_oc ? 0u : step - n_oc + 1;
		}
		if (step >= NH) oc = step - NH;
		return step < NH ? step : NH;
	};

	const uint32_t smem_base = smem_u32(smem_raw);
	if (smem_base & 1023u) __trap();
	const uint32_t s_stage0 = smem_base;
	const uint32_t s_bars = s_stage0 + n_stages * C::STAGE_BYTES;
	const uint32_t bar_w_full = s_bars;                            // [MLPF_MAX_STAGES]
	const uint32_t bar_w_free = bar_w_full + 8 * MLPF_MAX_STAGES;  // [MLPF_MAX_STAGES]

	if (tid == 0) {
		for (uint32_t i = 0; i < n_stages; ++i) {
			mbar_init(bar_w_full + 8 * i, 1);
			mbar_init(bar_w_free + 8 * i, C::WGS * 4);
		}
		fence_mbar_init();
	}
	if (warp == C::WGS * 4 && lane == 0) {
		tma_prefetch_desc(&map_w0);
		tma_prefetch_desc(&map_wh);
		tma_prefetch_desc(&map_wo);
	}
	__syncthreads();
	pdl_wait();  // from here on global memory written by the previous kernel on the stream is read

	const uint32_t n_units = p.batch_size / UNIT_M;
	// units of this CTA: blockIdx.x + j * gridDim.x, j = 0 .. n_my - 1; round r gives unit j = r * WGS + s to consumer warpgroup s
	const uint32_t n_my = blockIdx.x < n_units ? (n_units - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
	const uint32_t n_rounds = (n_my + C::WGS - 1) / C::WGS;

	if (warp == C::WGS * 4) {
		// =============================================================================== TMA producer: weight matrices -> stages
		if (lane == 0) {
			const uint32_t n_loads = resident ? n_layers : n_rounds * n_layers;
			for (uint32_t g = 0; g < (n_my ? n_loads : 0u); ++g) {
				const uint32_t step = resident ? g : g % n_layers;
				uint32_t oc;
				const uint32_t lc = chain_layer(step, oc);
				const uint32_t l = BWD ? NH - lc : lc;  // matrix of this step
				const uint32_t stage = resident ? g : g % n_stages;
				if (!resident && g >= n_stages) mbar_wait(bar_w_free + 8 * stage, ((g / n_stages) - 1u) & 1u);
				const uint32_t dst = s_stage0 + stage * C::STAGE_BYTES;
				const uint32_t full = bar_w_full + 8 * stage;
				if (l == 0) {
					const uint32_t kb = (in_w + 63) / 64;
					mbar_arrive_expect_tx(full, kb * W * 128);
					for (uint32_t b = 0; b < kb; ++b) tma_load_2d(dst + b * C::KBLOCK_BYTES, &map_w0, full, (int32_t)(b * 64), 0);
				} else if (l < NH) {
					mbar_arrive_expect_tx(full, C::KBLOCKS * W * 128);
					for (uint32_t b = 0; b < C::KBLOCKS; ++b) tma_load_2d(dst + b * C::KBLOCK_BYTES, &map_wh, full, (int32_t)(b * 64), (int32_t)((l - 1) * W));
				} else {
					mbar_arrive_expect_tx(full, C::KBLOCKS * (WIDE ? W : out_w) * 128);
					for (uint32_t b = 0; b < C::KBLOCKS; ++b) tma_load_2d(dst + b * C::KBLOCK_BYTES, &map_wo, full, (int32_t)(b * 64), (int32_t)(oc * W));
				}
			}
		}
	} else {
		// =============================================================================== consumer warpgroup s
		const uint32_t s = warp / 4, wq = warp & 3u;
		const uint32_t fq = lane >> 2, ft = lane & 3u;
		const uint32_t r0 = wq * 16 + fq;  // rows r0 and r0 + 8 of the unit
		const bool stamp = wq == 0 && lane == 0;
		// In ring mode every consumer walks every round, also past its last unit: it then only releases the weight stages.
		const uint32_t my_rounds = resident ? (n_my > s ? (n_my - s + C::WGS - 1) / C::WGS : 0) : n_rounds;
		uint32_t a[C::KMAX / 16][4];      // A fragment of the next product: k-step kk, registers as in Wgmma::rs
		float acc[C::ACC_N / 2];
		for (uint32_t r = 0; r < my_rounds; ++r) {
			const uint32_t j = r * C::WGS + s;
			const bool real = j < n_my;
			const size_t row0 = (size_t)(blockIdx.x + j * gridDim.x) * UNIT_M;
			if (real) {
				// ---- the rows that enter the chain -> A fragment
#pragma unroll
				for (uint32_t kk = 0; kk < C::KMAX / 16; ++kk) {
#pragma unroll
					for (uint32_t q = 0; q < 4; ++q) {
						const size_t rr = row0 + r0 + (q & 1u) * 8;
						const uint32_t c = kk * 16 + (q >> 1) * 8 + 2 * ft;
						uint32_t v = 0;
						if (c < first_w) {
							if (p.input_fp16) {
								v = __ldg(reinterpret_cast<const uint32_t*>(p.input_fp16 + rr * first_w + c));
							} else {
								// Identity encoding (identity.h:46-67): the first n_input_dims features are the inputs, the padding features are ONE
								const float* src = p.input_fp32 + rr * p.n_input_dims;
								const float lo = c < p.n_input_dims ? __ldg(src + c) : 1.0f;
								const float hi = c + 1 < p.n_input_dims ? __ldg(src + c + 1) : 1.0f;
								v = pack_half2(lo, hi);
							}
						}
						a[kk][q] = v;
					}
				}
			}
			for (uint32_t step = 0; step < n_layers; ++step) {
				const uint32_t g = r * n_layers + step;
				const uint32_t stage = resident ? step : g % n_stages;
				uint32_t oc;
				const uint32_t l = chain_layer(step, oc);
				const bool k_chunk = WIDE && BWD && l == 0;  // one of the K-blocks of the first backward product
				if (stamp) MLPF_STAMP(s, g, 0);
				mbar_wait(bar_w_full + 8 * stage, resident ? 0u : (g / n_stages) & 1u);
				if (stamp) MLPF_STAMP(s, g, 1);
				if (!real) {
					__syncwarp();
					if (lane == 0) mbar_arrive_plain(bar_w_free + 8 * stage);
					continue;
				}
				if (k_chunk && oc > 0) {
					// dL/d(output) columns oc W .. oc W + W - 1 -> k-steps 0 .. W / 16 - 1 of the A fragment (the previous chunk's wgmma is complete)
#pragma unroll
					for (uint32_t kk = 0; kk < W / 16; ++kk) {
#pragma unroll
						for (uint32_t q = 0; q < 4; ++q) {
							const size_t rr = row0 + r0 + (q & 1u) * 8;
							const uint32_t c = oc * W + kk * 16 + (q >> 1) * 8 + 2 * ft;
							a[kk][q] = c < first_w ? __ldg(reinterpret_cast<const uint32_t*>(p.input_fp16 + rr * first_w + c)) : 0u;
						}
					}
				}
				// backward: the forward pass's activations (PRE: pre-activations) of the layer this step lands on (hidden layer NH - 1 - l),
				// fetched before the MMA so that the loads travel while it runs
				uint32_t fwd[BWD ? W / 4 : 1];
				if (BWD && l < NH && (!k_chunk || oc + 1 == n_oc)) {
					const __half* hsrc = p.hidden_in + ((size_t)(NH - 1 - l) * p.batch_size + row0 + r0) * W + 2 * ft;
#pragma unroll
					for (uint32_t i = 0; i < W / 8; ++i) {
						fwd[2 * i] = __ldg(reinterpret_cast<const uint32_t*>(hsrc + 8 * i));
						fwd[2 * i + 1] = __ldg(reinterpret_cast<const uint32_t*>(hsrc + 8 * W + 8 * i));
					}
				}
				// ---- D = A . B: forward: the stage holds [N rows][64 K] boxes, K-major; backward: the same boxes are [K rows][64 N],
				// MN-major (16 K-rows = 2 048 bytes per step, the next 64 N-columns one box further)
				const uint32_t b_smem = s_stage0 + stage * C::STAGE_BYTES;
				const uint32_t ksteps = (l == 0 ? (k_chunk ? W : first_w) : W) / 16;
				// every product is N = W wide except dL/d(input) of a 16-wide network, which may be 32 wide
				const bool wide = C::ACC_N != W && BWD && l == NH;
				wgmma_fence();
#pragma unroll
				for (uint32_t kk = 0; kk < C::KMAX / 16; ++kk) {
					if (kk < ksteps) {
						const uint64_t b_desc = BWD ? wgmma_desc_sw128(b_smem + kk * 2048u, C::KBLOCK_BYTES, 1024u)
						                            : wgmma_desc_sw128(b_smem + (kk >> 2) * C::KBLOCK_BYTES + (kk & 3u) * 32u, 16u, 1024u);
						if (wide) Wgmma<C::ACC_N>::template rs<BWD ? 1 : 0>(acc, a[kk], b_desc, kk > 0);
						else Wgmma<W>::template rs<BWD ? 1 : 0>(reinterpret_cast<float(&)[W / 2]>(acc), a[kk], b_desc, kk > 0 || (k_chunk && oc > 0));
					}
				}
				wgmma_commit();
				wgmma_wait<0>();
				reg_fence(acc);
				if (stamp) MLPF_STAMP(s, g, 2);
				if (!resident) {
					__syncwarp();
					if (lane == 0) mbar_arrive_plain(bar_w_free + 8 * stage);
				}
				if (k_chunk && oc + 1 < n_oc) continue;  // more K-blocks to accumulate
				if (l < NH) {
					// hidden layer: fp32 accumulator -> (derivative of the) activation in fp16 -> the next product's A fragment; the rows
					// also go to global memory when the caller keeps them (forward activations / backward g_l)
					__half* keep = p.hidden_out ? p.hidden_out + ((size_t)(BWD ? NH - 1 - l : l) * p.batch_size + row0 + r0) * W + 2 * ft : nullptr;
					__half* keep_pre = (PRE && !BWD && kp.hidden_pre_out) ? kp.hidden_pre_out + ((size_t)l * p.batch_size + row0 + r0) * W + 2 * ft : nullptr;
#pragma unroll
					for (uint32_t i = 0; i < W / 8; ++i) {
#pragma unroll
						for (uint32_t hi = 0; hi < 2; ++hi) {
							const uint32_t lo_bits = __float_as_uint(acc[4 * i + 2 * hi]), hi_bits = __float_as_uint(acc[4 * i + 2 * hi + 1]);
							uint32_t v;
							if (PRE && BWD) {
								v = act_bwd_pre_pack(hid_act, lo_bits, hi_bits, fwd[(2 * i + hi) % (BWD ? W / 4 : 1)]);
							} else if (PRE) {
								const uint32_t z = pack_half2(__uint_as_float(lo_bits), __uint_as_float(hi_bits));
								if (keep_pre) *reinterpret_cast<uint32_t*>(keep_pre + hi * 8 * W + 8 * i) = z;
								v = act_pre_pack(hid_act, z);
							} else {
								v = BWD ? act_bwd_pack(hid_act, lo_bits, hi_bits, fwd[(2 * i + hi) % (BWD ? W / 4 : 1)]) : act_pack(hid_act, lo_bits, hi_bits);
							}
							a[i / 2][(i & 1u) * 2 + hi] = v;
							if (keep) *reinterpret_cast<uint32_t*>(keep + hi * 8 * W + 8 * i) = v;
						}
					}
				} else {
					// output layer: activation, then fp16 rows (and / or trimmed fp32 rows) to global memory
					constexpr bool VEC16 = WIDE && !BWD && W >= 32;  // fp16 rows as 16-byte vectors (quad_transpose)
					if (VEC16 && p.output_fp16) {
#pragma unroll
						for (uint32_t j = 0; j < W / 32; ++j) {
#pragma unroll
							for (uint32_t hi = 0; hi < 2; ++hi) {
								uint32_t v[4];
#pragma unroll
								for (uint32_t k = 0; k < 4; ++k) {
									const uint32_t i = 4 * j + k;
									const __half2 y = __halves2half2(act_fwd_h(out_act, __float2half_rn(acc[4 * i + 2 * hi])), act_fwd_h(out_act, __float2half_rn(acc[4 * i + 2 * hi + 1])));
									v[k] = *reinterpret_cast<const uint32_t*>(&y);
								}
								const uint4 q = quad_transpose(v[0], v[1], v[2], v[3], lane);
								const uint32_t c = oc * W + 8 * (4 * j + ft);
								if (c < last_w) *reinterpret_cast<uint4*>(p.output_fp16 + (row0 + r0 + hi * 8) * last_w + c) = q;
							}
						}
					}
#pragma unroll
					for (uint32_t i = 0; i < (WIDE && !BWD ? W : C::ACC_N) / 8; ++i) {  // a forward chunk is W wide
						const uint32_t c = oc * W + 8 * i + 2 * ft;
						if (c >= last_w) continue;
#pragma unroll
						for (uint32_t hi = 0; hi < 2; ++hi) {
							const size_t rr = row0 + r0 + hi * 8;
							const __half2 y = __halves2half2(act_fwd_h(out_act, __float2half_rn(acc[4 * i + 2 * hi])), act_fwd_h(out_act, __float2half_rn(acc[4 * i + 2 * hi + 1])));
							if (p.output_fp16 && !VEC16) *reinterpret_cast<__half2*>(p.output_fp16 + rr * last_w + c) = y;
							if (p.output_fp32) {
								if (c < p.n_output_dims) p.output_fp32[rr * p.n_output_dims + c] = __low2float(y);
								if (c + 1 < p.n_output_dims) p.output_fp32[rr * p.n_output_dims + c + 1] = __high2float(y);
							}
						}
					}
				}
				if (stamp) MLPF_STAMP(s, g, 3);
			}
		}
	}

	pdl_launch_dependents();
}

// 256 neurons (CutlassMLP): the same machine, with every product split into two N = 128 halves. Unsplit, a thread would hold the
// K = 256 A fragment (64 registers), an N = 256 accumulator (128) and, backward, the prefetched forward rows (64) -- 256 registers before
// addresses, more than a thread can have. Split:
//   * half 0's epilogue packs into `a_lo`, a separate 32-register half of the next A fragment (half 1's MMAs still read all of `a`);
//     half 1's epilogue writes k-steps 8 .. 15 of `a` once its MMAs are complete, then `a_lo` moves into k-steps 0 .. 7;
//   * backward, the forward pass's rows are fetched per half (32 registers);
//   * every half is a weight stage of its own, 64 KB: forward [128 rows][256 K] (four K-major [128][64] boxes), backward two
//     MN-major [256 K rows][64 N] boxes. Three stages form a ring (a matrix is 128 KB: none stays resident);
//   * a last product at most 128 wide (the network output forward, dL/d(input) backward) is one half.
// mlp_forward256_wide_kernel (out_width > 256): forward, the output matrix takes n_oc = ceil(out_width / 256) steps of 256 rows (two halves each; a
// last chunk at most 128 wide is one half). Backward, the first product accumulates over n_oc K-blocks of 256 rows inside each half:
// half h walks its K-blocks (a stage each, [256 K rows][64 N] boxes), loading each block's dL/d(output) columns into `a` first. The
// blocks are loaded once per half, because an accumulator holds only one half.
// It is a kernel of its own so that the code of the kernel above stays as it was for every narrower output.
struct Mlp256 {
	static constexpr uint32_t W = 256;
	static constexpr uint32_t HALF = 128;
	// ONE consumer warpgroup: the SM's register file is four 16 384-register quarters, and a warp lives in one of them; with two
	// consumer warpgroups and the producer warp one quarter holds three warps, which caps every thread at 168 registers -- less than
	// a 256-wide chain needs without spills. Four consumer warps and the producer warp leave up to 255.
	static constexpr uint32_t WGS = 1;
	static constexpr uint32_t THREADS = WGS * 128 + 32;
	static constexpr uint32_t STAGE_BYTES = 65536;
	static constexpr uint32_t STAGES = 3;
	static constexpr uint32_t FWD_BOX_BYTES = HALF * 128;  // [128 rows][64 K]
	static constexpr uint32_t BWD_BOX_BYTES = W * 128;     // [256 K rows][64 N]
};

template <bool GENERIC_ACT, bool BWD, bool PRE>
__global__ void __launch_bounds__(Mlp256::THREADS, 1)
mlp_forward256_kernel(const MlpKernelParams kp, const __grid_constant__ CUtensorMap map_w0, const __grid_constant__ CUtensorMap map_wh, const __grid_constant__ CUtensorMap map_wo) {
	using C = Mlp256;
	constexpr uint32_t W = C::W;
	static_assert(!PRE || GENERIC_ACT, "the pre-activation path is a generic-activation kernel");
	const MlpChainParams& p = kp.p;
	const uint32_t hid_act = GENERIC_ACT ? p.activation : (uint32_t)ACT_RELU;
	const uint32_t out_act = BWD ? (uint32_t)ACT_NONE : (GENERIC_ACT ? p.output_activation : (uint32_t)ACT_NONE);
	extern __shared__ __align__(1024) uint8_t smem_raw[];
	const uint32_t tid = threadIdx.x;
	const uint32_t warp = __shfl_sync(0xFFFFFFFFu, tid >> 5, 0);
	const uint32_t lane = tid & 31u;
	const uint32_t NH = p.n_hidden_layers, n_layers = kp.n_steps;
	const uint32_t in_w = p.in_width, out_w = p.out_width;
	const uint32_t first_w = BWD ? out_w : in_w;
	const uint32_t last_w = BWD ? in_w : out_w;
	// Every step walks two half-stages. A last product at most 128 wide (the network output forward, dL/d(input) backward) needs
	// only half 0: half 1's stage then carries no load and no MMA (its barrier is only arrived at), so that the wgmma code has no
	// data-dependent branch around it.
	auto one_half = [&](uint32_t l) { return l == NH && last_w <= C::HALF; };

	const uint32_t smem_base = smem_u32(smem_raw);
	if (smem_base & 1023u) __trap();
	const uint32_t s_stage0 = smem_base;
	const uint32_t bar_w_full = s_stage0 + C::STAGES * C::STAGE_BYTES;
	const uint32_t bar_w_free = bar_w_full + 8 * MLPF_MAX_STAGES;

	if (tid == 0) {
		for (uint32_t i = 0; i < C::STAGES; ++i) {
			mbar_init(bar_w_full + 8 * i, 1);
			mbar_init(bar_w_free + 8 * i, C::WGS * 4);
		}
		fence_mbar_init();
	}
	if (warp == C::WGS * 4 && lane == 0) {
		tma_prefetch_desc(&map_w0);
		tma_prefetch_desc(&map_wh);
		tma_prefetch_desc(&map_wo);
	}
	__syncthreads();
	pdl_wait();

	const uint32_t n_units = p.batch_size / UNIT_M;
	const uint32_t n_my = blockIdx.x < n_units ? (n_units - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
	const uint32_t n_rounds = (n_my + C::WGS - 1) / C::WGS;

	if (warp == C::WGS * 4) {
		// =============================================================================== TMA producer: half-matrices -> the stage ring
		if (lane == 0) {
			uint32_t g = 0;
			for (uint32_t r = 0; r < (n_my ? n_rounds : 0u); ++r) {
				for (uint32_t step = 0; step < n_layers; ++step) {
					const uint32_t l = BWD ? NH - step : step;  // matrix of this step
					const CUtensorMap* map = l == 0 ? &map_w0 : (l < NH ? &map_wh : &map_wo);
					const int32_t row = l == 0 || l == NH ? 0 : (int32_t)((l - 1) * W);
					for (uint32_t h = 0; h < 2; ++h, ++g) {
						const uint32_t stage = g % C::STAGES;
						if (g >= C::STAGES) mbar_wait(bar_w_free + 8 * stage, ((g / C::STAGES) - 1u) & 1u);
						const uint32_t dst = s_stage0 + stage * C::STAGE_BYTES;
						const uint32_t full = bar_w_full + 8 * stage;
						if (h == 1 && one_half(step)) {
							mbar_arrive_plain(full);
						} else if (BWD) {
							// K = the matrix's rows (all of them, one box), N = its columns 128 h ..: two 64-column boxes
							mbar_arrive_expect_tx(full, 2 * C::BWD_BOX_BYTES);
							for (uint32_t b = 0; b < 2; ++b) tma_load_2d(dst + b * C::BWD_BOX_BYTES, map, full, (int32_t)((2 * h + b) * 64), row);
						} else {
							// N = the matrix's rows 128 h .., K = its columns: one [128][64] box per 64 K-columns
							const uint32_t kb = l == 0 ? (in_w + 63) / 64 : 4u;
							mbar_arrive_expect_tx(full, kb * C::FWD_BOX_BYTES);
							for (uint32_t b = 0; b < kb; ++b) tma_load_2d(dst + b * C::FWD_BOX_BYTES, map, full, (int32_t)(b * 64), row + (int32_t)(h * C::HALF));
						}
					}
				}
			}
		}
	} else {
		// =============================================================================== consumer warpgroup s
		const uint32_t s = warp / 4, wq = warp & 3u;
		const uint32_t fq = lane >> 2, ft = lane & 3u;
		const uint32_t r0 = wq * 16 + fq;
		const bool stamp = wq == 0 && lane == 0;
		uint32_t a[W / 16][4];          // A fragment of the next product
		uint32_t a_lo[W / 32][4];       // half 0's epilogue: k-steps 0 .. 7 of the product after next
		float acc[C::HALF / 2];
		uint32_t g = 0;
		for (uint32_t r = 0; r < n_rounds; ++r) {
			const uint32_t j = r * C::WGS + s;
			const bool real = j < n_my;
			const size_t row0 = (size_t)(blockIdx.x + j * gridDim.x) * UNIT_M;
			if (real) {
#pragma unroll
				for (uint32_t kk = 0; kk < W / 16; ++kk) {
#pragma unroll
					for (uint32_t q = 0; q < 4; ++q) {
						const size_t rr = row0 + r0 + (q & 1u) * 8;
						const uint32_t c = kk * 16 + (q >> 1) * 8 + 2 * ft;
						uint32_t v = 0;
						if (c < first_w) {
							if (p.input_fp16) {
								v = __ldg(reinterpret_cast<const uint32_t*>(p.input_fp16 + rr * first_w + c));
							} else {
								const float* src = p.input_fp32 + rr * p.n_input_dims;
								const float lo = c < p.n_input_dims ? __ldg(src + c) : 1.0f;
								const float hi = c + 1 < p.n_input_dims ? __ldg(src + c + 1) : 1.0f;
								v = pack_half2(lo, hi);
							}
						}
						a[kk][q] = v;
					}
				}
			}
			for (uint32_t l = 0; l < n_layers; ++l) {
				const uint32_t ksteps = (l == 0 ? first_w : W) / 16;
				const bool skip_half1 = one_half(l);
#pragma unroll
				for (uint32_t h = 0; h < 2; ++h) {
					const uint32_t stage = g % C::STAGES;
					if (stamp) MLPF_STAMP(s, g, 0);
					mbar_wait(bar_w_full + 8 * stage, (g / C::STAGES) & 1u);
					if (stamp) MLPF_STAMP(s, g, 1);
					++g;
					if (!real) {
						__syncwarp();
						if (lane == 0) mbar_arrive_plain(bar_w_free + 8 * stage);
						continue;
					}
					uint32_t fwd[BWD ? C::HALF / 4 : 1];
					if (BWD && l < NH) {
						const __half* hsrc = p.hidden_in + ((size_t)(NH - 1 - l) * p.batch_size + row0 + r0) * W + h * C::HALF + 2 * ft;
#pragma unroll
						for (uint32_t i = 0; i < C::HALF / 8; ++i) {
							fwd[(2 * i) % (BWD ? C::HALF / 4 : 1)] = __ldg(reinterpret_cast<const uint32_t*>(hsrc + 8 * i));
							fwd[(2 * i + 1) % (BWD ? C::HALF / 4 : 1)] = __ldg(reinterpret_cast<const uint32_t*>(hsrc + 8 * W + 8 * i));
						}
					}
					const uint32_t b_smem = s_stage0 + stage * C::STAGE_BYTES;
					wgmma_fence();
#pragma unroll
					for (uint32_t kk = 0; kk < W / 16; ++kk) {
						if (kk < ksteps && !(h == 1 && skip_half1)) {
							const uint64_t b_desc = BWD ? wgmma_desc_sw128(b_smem + kk * 2048u, C::BWD_BOX_BYTES, 1024u)
							                            : wgmma_desc_sw128(b_smem + (kk >> 2) * C::FWD_BOX_BYTES + (kk & 3u) * 32u, 16u, 1024u);
							Wgmma<C::HALF>::template rs<BWD ? 1 : 0>(acc, a[kk], b_desc, kk > 0);
						}
					}
					wgmma_commit();
					wgmma_wait<0>();
					reg_fence(acc);
					if (stamp) MLPF_STAMP(s, g - 1, 2);
					__syncwarp();
					if (lane == 0) mbar_arrive_plain(bar_w_free + 8 * stage);
					if (l < NH) {
						const size_t krow = ((size_t)(BWD ? NH - 1 - l : l) * p.batch_size + row0 + r0) * W + h * C::HALF + 2 * ft;
						__half* keep = p.hidden_out ? p.hidden_out + krow : nullptr;
						__half* keep_pre = (PRE && !BWD && kp.hidden_pre_out) ? kp.hidden_pre_out + krow : nullptr;
#pragma unroll
						for (uint32_t i = 0; i < C::HALF / 8; ++i) {
#pragma unroll
							for (uint32_t hi = 0; hi < 2; ++hi) {
								const uint32_t lo_bits = __float_as_uint(acc[4 * i + 2 * hi]), hi_bits = __float_as_uint(acc[4 * i + 2 * hi + 1]);
								uint32_t v;
								if (PRE && BWD) {
									v = act_bwd_pre_pack(hid_act, lo_bits, hi_bits, fwd[(2 * i + hi) % (BWD ? C::HALF / 4 : 1)]);
								} else if (PRE) {
									const uint32_t z = pack_half2(__uint_as_float(lo_bits), __uint_as_float(hi_bits));
									if (keep_pre) *reinterpret_cast<uint32_t*>(keep_pre + hi * 8 * W + 8 * i) = z;
									v = act_pre_pack(hid_act, z);
								} else {
									v = BWD ? act_bwd_pack(hid_act, lo_bits, hi_bits, fwd[(2 * i + hi) % (BWD ? C::HALF / 4 : 1)]) : act_pack(hid_act, lo_bits, hi_bits);
								}
								if (h == 0) a_lo[i / 2][(i & 1u) * 2 + hi] = v;
								else a[W / 32 + i / 2][(i & 1u) * 2 + hi] = v;
								if (keep) *reinterpret_cast<uint32_t*>(keep + hi * 8 * W + 8 * i) = v;
							}
						}
					} else {
#pragma unroll
						for (uint32_t i = 0; i < C::HALF / 8; ++i) {
							const uint32_t c = h * C::HALF + 8 * i + 2 * ft;
							if (c >= last_w) continue;
#pragma unroll
							for (uint32_t hi = 0; hi < 2; ++hi) {
								const size_t rr = row0 + r0 + hi * 8;
								const __half2 y = __halves2half2(act_fwd_h(out_act, __float2half_rn(acc[4 * i + 2 * hi])), act_fwd_h(out_act, __float2half_rn(acc[4 * i + 2 * hi + 1])));
								if (p.output_fp16) *reinterpret_cast<__half2*>(p.output_fp16 + rr * last_w + c) = y;
								if (p.output_fp32) {
									if (c < p.n_output_dims) p.output_fp32[rr * p.n_output_dims + c] = __low2float(y);
									if (c + 1 < p.n_output_dims) p.output_fp32[rr * p.n_output_dims + c + 1] = __high2float(y);
								}
							}
						}
					}
					if (stamp) MLPF_STAMP(s, g - 1, 3);
				}
				if (l < NH) {
#pragma unroll
					for (uint32_t kk = 0; kk < W / 32; ++kk) {
#pragma unroll
						for (uint32_t q = 0; q < 4; ++q) a[kk][q] = a_lo[kk][q];
					}
				}
			}
		}
	}

	pdl_launch_dependents();
}

template <bool GENERIC_ACT, bool BWD, bool PRE>
__global__ void __launch_bounds__(Mlp256::THREADS, 1)
mlp_forward256_wide_kernel(const MlpKernelParams kp, const __grid_constant__ CUtensorMap map_w0, const __grid_constant__ CUtensorMap map_wh, const __grid_constant__ CUtensorMap map_wo) {
	using C = Mlp256;
	constexpr uint32_t W = C::W;
	static_assert(!PRE || GENERIC_ACT, "the pre-activation path is a generic-activation kernel");
	const MlpChainParams& p = kp.p;
	const uint32_t hid_act = GENERIC_ACT ? p.activation : (uint32_t)ACT_RELU;
	const uint32_t out_act = BWD ? (uint32_t)ACT_NONE : (GENERIC_ACT ? p.output_activation : (uint32_t)ACT_NONE);
	extern __shared__ __align__(1024) uint8_t smem_raw[];
	const uint32_t tid = threadIdx.x;
	const uint32_t warp = __shfl_sync(0xFFFFFFFFu, tid >> 5, 0);
	const uint32_t lane = tid & 31u;
	const uint32_t NH = p.n_hidden_layers, n_layers = kp.n_steps;
	const uint32_t in_w = p.in_width, out_w = p.out_width;
	const uint32_t first_w = BWD ? out_w : in_w;
	const uint32_t last_w = BWD ? in_w : out_w;
	// Every step walks two half-stages. A last product at most 128 wide (the network output forward, dL/d(input) backward) needs
	// only half 0: half 1's stage then carries no load and no MMA (its barrier is only arrived at), so that the wgmma code has no
	// data-dependent branch around it.
	auto one_half = [&](uint32_t l, uint32_t oc) { return l == NH && last_w - oc * W <= C::HALF; };
	const uint32_t n_oc = (out_w + W - 1) / W;
	// step of the unit -> layer of the chain (as counted by mlp_forward256_kernel) and, forward, the chunk of the output matrix
	auto chain_layer = [&](uint32_t step, uint32_t& oc) -> uint32_t {
		oc = (!BWD && step >= NH) ? step - NH : 0u;
		return (!BWD && step >= NH) ? NH : step;
	};

	const uint32_t smem_base = smem_u32(smem_raw);
	if (smem_base & 1023u) __trap();
	const uint32_t s_stage0 = smem_base;
	const uint32_t bar_w_full = s_stage0 + C::STAGES * C::STAGE_BYTES;
	const uint32_t bar_w_free = bar_w_full + 8 * MLPF_MAX_STAGES;

	if (tid == 0) {
		for (uint32_t i = 0; i < C::STAGES; ++i) {
			mbar_init(bar_w_full + 8 * i, 1);
			mbar_init(bar_w_free + 8 * i, C::WGS * 4);
		}
		fence_mbar_init();
	}
	if (warp == C::WGS * 4 && lane == 0) {
		tma_prefetch_desc(&map_w0);
		tma_prefetch_desc(&map_wh);
		tma_prefetch_desc(&map_wo);
	}
	__syncthreads();
	pdl_wait();

	const uint32_t n_units = p.batch_size / UNIT_M;
	const uint32_t n_my = blockIdx.x < n_units ? (n_units - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
	const uint32_t n_rounds = (n_my + C::WGS - 1) / C::WGS;

	if (warp == C::WGS * 4) {
		// =============================================================================== TMA producer: half-matrices -> the stage ring
		if (lane == 0) {
			uint32_t g = 0;
			for (uint32_t r = 0; r < (n_my ? n_rounds : 0u); ++r) {
				for (uint32_t step = 0; step < n_layers; ++step) {
					// the output matrix: forward one step per 256 rows (row block oc); backward n_oc K-blocks per half inside step 0
					uint32_t oc;
					const uint32_t lc = chain_layer(step, oc);
					const uint32_t l = BWD ? NH - lc : lc;
					const CUtensorMap* map = l == 0 ? &map_w0 : (l < NH ? &map_wh : &map_wo);
					const int32_t row = l == 0 || l == NH ? (int32_t)(oc * W) : (int32_t)((l - 1) * W);
					const uint32_t n_k = BWD && lc == 0 ? n_oc : 1u;
					for (uint32_t h = 0; h < 2; ++h) {
						for (uint32_t kc = 0; kc < n_k; ++kc, ++g) {
							const uint32_t stage = g % C::STAGES;
							if (g >= C::STAGES) mbar_wait(bar_w_free + 8 * stage, ((g / C::STAGES) - 1u) & 1u);
							const uint32_t dst = s_stage0 + stage * C::STAGE_BYTES;
							const uint32_t full = bar_w_full + 8 * stage;
							if (h == 1 && one_half(lc, oc)) {
								mbar_arrive_plain(full);
							} else if (BWD) {
								mbar_arrive_expect_tx(full, 2 * C::BWD_BOX_BYTES);
								for (uint32_t b = 0; b < 2; ++b) tma_load_2d(dst + b * C::BWD_BOX_BYTES, map, full, (int32_t)((2 * h + b) * 64), row + (int32_t)(kc * W));
							} else {
								const uint32_t kb = l == 0 ? (in_w + 63) / 64 : 4u;
								mbar_arrive_expect_tx(full, kb * C::FWD_BOX_BYTES);
								for (uint32_t b = 0; b < kb; ++b) tma_load_2d(dst + b * C::FWD_BOX_BYTES, map, full, (int32_t)(b * 64), row + (int32_t)(h * C::HALF));
							}
						}
					}
				}
			}
		}
	} else {
		// =============================================================================== consumer warpgroup s
		const uint32_t s = warp / 4, wq = warp & 3u;
		const uint32_t fq = lane >> 2, ft = lane & 3u;
		const uint32_t r0 = wq * 16 + fq;
		const bool stamp = wq == 0 && lane == 0;
		uint32_t a[W / 16][4];          // A fragment of the next product
		uint32_t a_lo[W / 32][4];       // half 0's epilogue: k-steps 0 .. 7 of the product after next
		float acc[C::HALF / 2];
		// backward: dL/d(output) columns 256 kc .. 256 kc + 255 -> the A fragment (the previous block's wgmma is complete)
		auto load_block = [&](size_t row0, uint32_t kc) {
#pragma unroll
			for (uint32_t kk = 0; kk < W / 16; ++kk) {
#pragma unroll
				for (uint32_t q = 0; q < 4; ++q) {
					const size_t rr = row0 + r0 + (q & 1u) * 8;
					const uint32_t c = kc * W + kk * 16 + (q >> 1) * 8 + 2 * ft;
					a[kk][q] = c < first_w ? __ldg(reinterpret_cast<const uint32_t*>(p.input_fp16 + rr * first_w + c)) : 0u;
				}
			}
		};
		uint32_t g = 0;
		for (uint32_t r = 0; r < n_rounds; ++r) {
			const uint32_t j = r * C::WGS + s;
			const bool real = j < n_my;
			const size_t row0 = (size_t)(blockIdx.x + j * gridDim.x) * UNIT_M;
			if (real) {
#pragma unroll
				for (uint32_t kk = 0; kk < W / 16; ++kk) {
#pragma unroll
					for (uint32_t q = 0; q < 4; ++q) {
						const size_t rr = row0 + r0 + (q & 1u) * 8;
						const uint32_t c = kk * 16 + (q >> 1) * 8 + 2 * ft;
						uint32_t v = 0;
						if (c < first_w) {
							if (p.input_fp16) {
								v = __ldg(reinterpret_cast<const uint32_t*>(p.input_fp16 + rr * first_w + c));
							} else {
								const float* src = p.input_fp32 + rr * p.n_input_dims;
								const float lo = c < p.n_input_dims ? __ldg(src + c) : 1.0f;
								const float hi = c + 1 < p.n_input_dims ? __ldg(src + c + 1) : 1.0f;
								v = pack_half2(lo, hi);
							}
						}
						a[kk][q] = v;
					}
				}
			}
			for (uint32_t step = 0; step < n_layers; ++step) {
				uint32_t oc;
				const uint32_t l = chain_layer(step, oc);
				const bool k_chunks = BWD && l == 0;  // the first backward product in K-blocks
				const uint32_t ksteps = (l == 0 ? (k_chunks ? W : first_w) : W) / 16;
				const bool skip_half1 = one_half(l, oc);
#pragma unroll
				for (uint32_t h = 0; h < 2; ++h) {
					const uint32_t stage = g % C::STAGES;
					if (stamp) MLPF_STAMP(s, g, 0);
					mbar_wait(bar_w_full + 8 * stage, (g / C::STAGES) & 1u);
					if (stamp) MLPF_STAMP(s, g, 1);
					++g;
					if (!real) {
						__syncwarp();
						if (lane == 0) mbar_arrive_plain(bar_w_free + 8 * stage);
						if (k_chunks) {
							for (uint32_t kc = 1; kc < n_oc; ++kc, ++g) {
								mbar_wait(bar_w_full + 8 * (g % C::STAGES), (g / C::STAGES) & 1u);
								__syncwarp();
								if (lane == 0) mbar_arrive_plain(bar_w_free + 8 * (g % C::STAGES));
							}
						}
						continue;
					}
					if (k_chunks && h == 1) load_block(row0, 0);  // half 0 reads block 0 from the round's first load
					uint32_t fwd[BWD ? C::HALF / 4 : 1];
					if (BWD && l < NH) {
						const __half* hsrc = p.hidden_in + ((size_t)(NH - 1 - l) * p.batch_size + row0 + r0) * W + h * C::HALF + 2 * ft;
#pragma unroll
						for (uint32_t i = 0; i < C::HALF / 8; ++i) {
							fwd[(2 * i) % (BWD ? C::HALF / 4 : 1)] = __ldg(reinterpret_cast<const uint32_t*>(hsrc + 8 * i));
							fwd[(2 * i + 1) % (BWD ? C::HALF / 4 : 1)] = __ldg(reinterpret_cast<const uint32_t*>(hsrc + 8 * W + 8 * i));
						}
					}
					const uint32_t b_smem = s_stage0 + stage * C::STAGE_BYTES;
					wgmma_fence();
#pragma unroll
					for (uint32_t kk = 0; kk < W / 16; ++kk) {
						if (kk < ksteps && !(h == 1 && skip_half1)) {
							const uint64_t b_desc = BWD ? wgmma_desc_sw128(b_smem + kk * 2048u, C::BWD_BOX_BYTES, 1024u)
							                            : wgmma_desc_sw128(b_smem + (kk >> 2) * C::FWD_BOX_BYTES + (kk & 3u) * 32u, 16u, 1024u);
							Wgmma<C::HALF>::template rs<BWD ? 1 : 0>(acc, a[kk], b_desc, kk > 0);
						}
					}
					wgmma_commit();
					wgmma_wait<0>();
					reg_fence(acc);
					if (stamp) MLPF_STAMP(s, g - 1, 2);
					__syncwarp();
					if (lane == 0) mbar_arrive_plain(bar_w_free + 8 * stage);
					if (k_chunks) {
						// the output matrix's further K-blocks, accumulated into the same half
						for (uint32_t kc = 1; kc < n_oc; ++kc, ++g) {
							const uint32_t st = g % C::STAGES;
							mbar_wait(bar_w_full + 8 * st, (g / C::STAGES) & 1u);
							load_block(row0, kc);
							const uint32_t bs = s_stage0 + st * C::STAGE_BYTES;
							wgmma_fence();
#pragma unroll
							for (uint32_t kk = 0; kk < W / 16; ++kk) Wgmma<C::HALF>::template rs<1>(acc, a[kk], wgmma_desc_sw128(bs + kk * 2048u, C::BWD_BOX_BYTES, 1024u), 1u);
							wgmma_commit();
							wgmma_wait<0>();
							reg_fence(acc);
							__syncwarp();
							if (lane == 0) mbar_arrive_plain(bar_w_free + 8 * st);
						}
					}
					if (l < NH) {
						const size_t krow = ((size_t)(BWD ? NH - 1 - l : l) * p.batch_size + row0 + r0) * W + h * C::HALF + 2 * ft;
						__half* keep = p.hidden_out ? p.hidden_out + krow : nullptr;
						__half* keep_pre = (PRE && !BWD && kp.hidden_pre_out) ? kp.hidden_pre_out + krow : nullptr;
#pragma unroll
						for (uint32_t i = 0; i < C::HALF / 8; ++i) {
#pragma unroll
							for (uint32_t hi = 0; hi < 2; ++hi) {
								const uint32_t lo_bits = __float_as_uint(acc[4 * i + 2 * hi]), hi_bits = __float_as_uint(acc[4 * i + 2 * hi + 1]);
								uint32_t v;
								if (PRE && BWD) {
									v = act_bwd_pre_pack(hid_act, lo_bits, hi_bits, fwd[(2 * i + hi) % (BWD ? C::HALF / 4 : 1)]);
								} else if (PRE) {
									const uint32_t z = pack_half2(__uint_as_float(lo_bits), __uint_as_float(hi_bits));
									if (keep_pre) *reinterpret_cast<uint32_t*>(keep_pre + hi * 8 * W + 8 * i) = z;
									v = act_pre_pack(hid_act, z);
								} else {
									v = BWD ? act_bwd_pack(hid_act, lo_bits, hi_bits, fwd[(2 * i + hi) % (BWD ? C::HALF / 4 : 1)]) : act_pack(hid_act, lo_bits, hi_bits);
								}
								if (h == 0) a_lo[i / 2][(i & 1u) * 2 + hi] = v;
								else a[W / 32 + i / 2][(i & 1u) * 2 + hi] = v;
								if (keep) *reinterpret_cast<uint32_t*>(keep + hi * 8 * W + 8 * i) = v;
							}
						}
					} else {
#pragma unroll
						for (uint32_t i = 0; i < C::HALF / 8; ++i) {
							const uint32_t c = oc * W + h * C::HALF + 8 * i + 2 * ft;
							if (c >= last_w) continue;
#pragma unroll
							for (uint32_t hi = 0; hi < 2; ++hi) {
								const size_t rr = row0 + r0 + hi * 8;
								const __half2 y = __halves2half2(act_fwd_h(out_act, __float2half_rn(acc[4 * i + 2 * hi])), act_fwd_h(out_act, __float2half_rn(acc[4 * i + 2 * hi + 1])));
								if (p.output_fp16) *reinterpret_cast<__half2*>(p.output_fp16 + rr * last_w + c) = y;
								if (p.output_fp32) {
									if (c < p.n_output_dims) p.output_fp32[rr * p.n_output_dims + c] = __low2float(y);
									if (c + 1 < p.n_output_dims) p.output_fp32[rr * p.n_output_dims + c + 1] = __high2float(y);
								}
							}
						}
					}
					if (stamp) MLPF_STAMP(s, g - 1, 3);
				}
				if (l < NH) {
#pragma unroll
					for (uint32_t kk = 0; kk < W / 32; ++kk) {
#pragma unroll
						for (uint32_t q = 0; q < 4; ++q) a[kk][q] = a_lo[kk][q];
					}
				}
			}
		}
	}

	pdl_launch_dependents();
}

// ------------------------------------------------------------------------------------------------------------------ host side
namespace {

template <uint32_t W>
uint32_t max_stages() {
	return (uint32_t)((227u * 1024u - 1024u) / MlpCfg<W>::STAGE_BYTES) < MLPF_MAX_STAGES ? (uint32_t)((227u * 1024u - 1024u) / MlpCfg<W>::STAGE_BYTES) : MLPF_MAX_STAGES;
}

template <uint32_t W, bool GENERIC, bool BWD, bool PRE, bool WIDE>
cudaError_t launch_impl(const MlpForwardParams& p, uint32_t n_sms, cudaStream_t stream) {
	using C = MlpCfg<W>;
	const uint32_t n_oc = WIDE ? (p.out_width + W - 1) / W : 1;  // steps of the output matrix
	const uint32_t n_layers = p.n_hidden_layers + ((BWD && !p.output_fp16) ? 0 : 1) + n_oc - 1;  // steps of the chain
	MlpKernelParams kp{};
	kp.p = p;
	kp.n_steps = n_layers;
	kp.hidden_pre_out = p.hidden_pre_out;
	kp.resident = n_layers <= max_stages<W>() ? 1 : 0;
	kp.n_stages = kp.resident ? n_layers : max_stages<W>();
	CUtensorMap m0, mh, mo;
	const __half* w = p.weights;
	if (!make_fp16_matrix_map(&m0, w, W, p.in_width, W)) return cudaErrorInvalidValue;
	w += (size_t)W * p.in_width;
	if (p.n_hidden_layers > 1) {
		if (!make_fp16_matrix_map(&mh, w, (p.n_hidden_layers - 1) * W, W, W)) return cudaErrorInvalidValue;
	} else {
		mh = m0;  // never used
	}
	w += (size_t)(p.n_hidden_layers - 1) * W * W;
	if (!make_fp16_matrix_map(&mo, w, p.out_width, W, WIDE ? W : p.out_width)) return cudaErrorInvalidValue;
	auto kernel = mlp_forward_kernel<W, GENERIC, BWD, PRE, WIDE>;
	const size_t smem = (size_t)kp.n_stages * C::STAGE_BYTES + 8 * 2 * MLPF_MAX_STAGES;
	cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
	if (err != cudaSuccess) return err;
	const uint32_t n_groups = (p.batch_size / UNIT_M + C::WGS - 1) / C::WGS;  // CTAs that have a unit for every consumer warpgroup
	return launch_pdl(kernel, n_groups < n_sms ? n_groups : n_sms, C::THREADS, smem, stream, kp, m0, mh, mo);
}

template <uint32_t W, bool WIDE>
cudaError_t launch_width(const MlpForwardParams& p, uint32_t n_sms, cudaStream_t stream) {
	if (activation_needs_preact(p.activation)) return p.backward ? launch_impl<W, true, true, true, WIDE>(p, n_sms, stream) : launch_impl<W, true, false, true, WIDE>(p, n_sms, stream);
	if (p.backward) return p.activation != ACT_RELU ? launch_impl<W, true, true, false, WIDE>(p, n_sms, stream) : launch_impl<W, false, true, false, WIDE>(p, n_sms, stream);
	const bool generic = p.activation != ACT_RELU || p.output_activation != ACT_NONE;
	return generic ? launch_impl<W, true, false, false, WIDE>(p, n_sms, stream) : launch_impl<W, false, false, false, WIDE>(p, n_sms, stream);
}

// A padded output wider than the layers takes the WIDE kernels; every other shape the kernels it always ran.
template <uint32_t W>
cudaError_t launch_width(const MlpForwardParams& p, uint32_t n_sms, cudaStream_t stream) {
	return p.out_width > W ? launch_width<W, true>(p, n_sms, stream) : launch_width<W, false>(p, n_sms, stream);
}

template <bool GENERIC, bool BWD, bool PRE, bool WIDE>
cudaError_t launch_impl256(const MlpForwardParams& p, uint32_t n_sms, cudaStream_t stream) {
	using C = Mlp256;
	// forward, the output matrix takes one step per 256 rows; backward, its K-blocks are walked inside the first step
	const uint32_t n_oc = (WIDE && !BWD) ? (p.out_width + C::W - 1) / C::W : 1;
	const uint32_t n_layers = p.n_hidden_layers + ((BWD && !p.output_fp16) ? 0 : 1) + n_oc - 1;
	MlpKernelParams kp{};
	kp.p = p;
	kp.n_steps = n_layers;
	kp.hidden_pre_out = p.hidden_pre_out;
	kp.resident = 0;
	kp.n_stages = C::STAGES;
	// forward: [128 rows][64 K] boxes (half a matrix's rows); backward: [256 rows][64 N] boxes (all of a matrix's rows = its K)
	const uint32_t box_rows = BWD ? C::W : C::HALF;
	CUtensorMap m0, mh, mo;
	const __half* w = p.weights;
	if (!make_fp16_matrix_map(&m0, w, C::W, p.in_width, box_rows)) return cudaErrorInvalidValue;
	w += (size_t)C::W * p.in_width;
	if (p.n_hidden_layers > 1) {
		if (!make_fp16_matrix_map(&mh, w, (p.n_hidden_layers - 1) * C::W, C::W, box_rows)) return cudaErrorInvalidValue;
	} else {
		mh = m0;  // never used
	}
	w += (size_t)(p.n_hidden_layers - 1) * C::W * C::W;
	if (!make_fp16_matrix_map(&mo, w, p.out_width, C::W, box_rows)) return cudaErrorInvalidValue;
	auto kernel = WIDE ? mlp_forward256_wide_kernel<GENERIC, BWD, PRE> : mlp_forward256_kernel<GENERIC, BWD, PRE>;
	const size_t smem = (size_t)C::STAGES * C::STAGE_BYTES + 8 * 2 * MLPF_MAX_STAGES;
	cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
	if (err != cudaSuccess) return err;
	const uint32_t n_groups = (p.batch_size / UNIT_M + C::WGS - 1) / C::WGS;
	return launch_pdl(kernel, n_groups < n_sms ? n_groups : n_sms, C::THREADS, smem, stream, kp, m0, mh, mo);
}

template <bool WIDE>
cudaError_t launch_width256(const MlpForwardParams& p, uint32_t n_sms, cudaStream_t stream) {
	if (activation_needs_preact(p.activation)) return p.backward ? launch_impl256<true, true, true, WIDE>(p, n_sms, stream) : launch_impl256<true, false, true, WIDE>(p, n_sms, stream);
	if (p.backward) return p.activation != ACT_RELU ? launch_impl256<true, true, false, WIDE>(p, n_sms, stream) : launch_impl256<false, true, false, WIDE>(p, n_sms, stream);
	const bool generic = p.activation != ACT_RELU || p.output_activation != ACT_NONE;
	return generic ? launch_impl256<true, false, false, WIDE>(p, n_sms, stream) : launch_impl256<false, false, false, WIDE>(p, n_sms, stream);
}

}  // namespace

uint32_t mlp_forward_resident_layers(uint32_t width) {
	switch (width) {
		case 256: return 0;  // a 256 x 256 matrix is 128 KB: every matrix streams through the ring of half-matrix stages
		case 128: return max_stages<128>();
		case 64: return max_stages<64>();
		case 32: return max_stages<32>();
		default: return max_stages<16>();
	}
}

bool mlp_forward_supported(const MlpForwardParams& p, const char** why) {
	auto fail = [&](const char* msg) {
		if (why) *why = msg;
		return false;
	};
	if (!(p.width == 16 || p.width == 32 || p.width == 64 || p.width == 128 || p.width == 256)) return fail("FullyFusedMLP only supports 16, 32, 64, and 128 neurons");
	if (p.n_hidden_layers < 1) return fail("FullyFusedMLP requires at least 1 hidden layer (3 layers in total).");
	if (p.n_hidden_layers + 1 > 64) return fail("tcnn_b200: the stand-alone MLP kernel covers up to 63 hidden layers");
	const uint32_t max_in = 64 * ((p.width + 63) / 64);
	if (p.in_width == 0 || p.in_width % 16 != 0 || p.in_width > max_in) return fail("tcnn_b200: network input width must be a multiple of 16 and at most 64 (128 / 256 for 128 / 256 neurons)");
	if (p.out_width == 0 || p.out_width % 16 != 0) return fail("tcnn_b200: padded network output width must be a multiple of 16 and at most n_neurons");
	if (p.out_width > MLP_MAX_OUTPUT_WIDTH) return fail("tcnn_b200: padded network output width must be at most 1024");
	if (p.batch_size == 0 || p.batch_size % TILE_M != 0) return fail("batch size must be a non-zero multiple of 256");
	if ((p.input_fp16 != nullptr) == (p.input_fp32 != nullptr)) return fail("tcnn_b200: exactly one network input must be given");
	if (p.backward) {
		if (!p.input_fp16 || !p.hidden_in || p.output_fp32) return fail("tcnn_b200: the backward chain needs dL/d(output) and the forward activations in fp16");
		if (p.output_fp16 && p.in_width > (p.width < 32 ? 32u : p.width)) return fail("tcnn_b200: dL/d(input) of the stand-alone network covers inputs up to max(n_neurons, 32) wide");
	}
	if (activation_needs_preact(p.output_activation)) return fail("tcnn_b200: Sine / SiLU are hidden activations only; as output activation they have no derivative (warp_activation_backward)");
	if (activation_needs_preact(p.activation)) {
		if (!p.backward && p.hidden_out && !p.hidden_pre_out) return fail("tcnn_b200: Sine / SiLU keep the pre-activations for the backward pass: hidden_pre_out must be given with hidden_out");
	} else if (p.hidden_pre_out) {
		return fail("tcnn_b200: hidden_pre_out is only written for Sine / SiLU hidden activations");
	}
	if (p.input_fp32 && (p.n_input_dims == 0 || p.n_input_dims > p.in_width)) return fail("tcnn_b200: Identity encoding wider than the network input");
	return true;
}

cudaError_t launch_mlp_forward(const MlpForwardParams& p, uint32_t n_sms, cudaStream_t stream) {
	if (!mlp_forward_supported(p, nullptr)) return cudaErrorInvalidValue;
	switch (p.width) {
		case 256: return p.out_width > 256 ? launch_width256<true>(p, n_sms, stream) : launch_width256<false>(p, n_sms, stream);
		case 128: return launch_width<128>(p, n_sms, stream);
		case 64: return launch_width<64>(p, n_sms, stream);
		case 32: return launch_width<32>(p, n_sms, stream);
		case 16: return launch_width<16>(p, n_sms, stream);
	}
	return cudaErrorInvalidValue;
}

}  // namespace tcnnb
