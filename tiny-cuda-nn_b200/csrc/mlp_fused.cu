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
	MlpForwardParams p;
	uint32_t n_stages;  // == n_steps when all matrices are resident
	uint32_t resident;
	uint32_t n_steps;   // MMAs chained per unit: n_hidden_layers + 1 (the backward chain without dL/d(input): n_hidden_layers)
};

}  // namespace

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
template <uint32_t W, bool GENERIC_ACT, bool BWD>
__global__ void __launch_bounds__(MlpCfg<W>::THREADS, 1)
mlp_forward_kernel(const MlpKernelParams kp, const __grid_constant__ CUtensorMap map_w0, const __grid_constant__ CUtensorMap map_wh, const __grid_constant__ CUtensorMap map_wo) {
	using C = MlpCfg<W>;
	const MlpForwardParams& p = kp.p;
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
				const uint32_t l = BWD ? NH - step : step;  // matrix of this step
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
					mbar_arrive_expect_tx(full, C::KBLOCKS * out_w * 128);
					for (uint32_t b = 0; b < C::KBLOCKS; ++b) tma_load_2d(dst + b * C::KBLOCK_BYTES, &map_wo, full, (int32_t)(b * 64), 0);
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
			for (uint32_t l = 0; l < n_layers; ++l) {
				const uint32_t g = r * n_layers + l;
				const uint32_t stage = resident ? l : g % n_stages;
				if (stamp) MLPF_STAMP(s, g, 0);
				mbar_wait(bar_w_full + 8 * stage, resident ? 0u : (g / n_stages) & 1u);
				if (stamp) MLPF_STAMP(s, g, 1);
				if (!real) {
					__syncwarp();
					if (lane == 0) mbar_arrive_plain(bar_w_free + 8 * stage);
					continue;
				}
				// backward: the forward pass's activations of the layer this step lands on (hidden layer NH - 1 - l), fetched before
				// the MMA so that the loads travel while it runs
				uint32_t fwd[BWD ? W / 4 : 1];
				if (BWD && l < NH) {
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
				const uint32_t ksteps = (l == 0 ? first_w : W) / 16;
				// every product is N = W wide except dL/d(input) of a 16-wide network, which may be 32 wide
				const bool wide = C::ACC_N != W && BWD && l == NH;
				wgmma_fence();
#pragma unroll
				for (uint32_t kk = 0; kk < C::KMAX / 16; ++kk) {
					if (kk < ksteps) {
						const uint64_t b_desc = BWD ? wgmma_desc_sw128(b_smem + kk * 2048u, C::KBLOCK_BYTES, 1024u)
						                            : wgmma_desc_sw128(b_smem + (kk >> 2) * C::KBLOCK_BYTES + (kk & 3u) * 32u, 16u, 1024u);
						if (wide) Wgmma<C::ACC_N>::template rs<BWD ? 1 : 0>(acc, a[kk], b_desc, kk > 0);
						else Wgmma<W>::template rs<BWD ? 1 : 0>(reinterpret_cast<float(&)[W / 2]>(acc), a[kk], b_desc, kk > 0);
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
				if (l < NH) {
					// hidden layer: fp32 accumulator -> (derivative of the) activation in fp16 -> the next product's A fragment; the rows
					// also go to global memory when the caller keeps them (forward activations / backward g_l)
					__half* keep = p.hidden_out ? p.hidden_out + ((size_t)(BWD ? NH - 1 - l : l) * p.batch_size + row0 + r0) * W + 2 * ft : nullptr;
#pragma unroll
					for (uint32_t i = 0; i < W / 8; ++i) {
#pragma unroll
						for (uint32_t hi = 0; hi < 2; ++hi) {
							const uint32_t lo_bits = __float_as_uint(acc[4 * i + 2 * hi]), hi_bits = __float_as_uint(acc[4 * i + 2 * hi + 1]);
							const uint32_t v = BWD ? act_bwd_pack(hid_act, lo_bits, hi_bits, fwd[(2 * i + hi) % (BWD ? W / 4 : 1)]) : act_pack(hid_act, lo_bits, hi_bits);
							a[i / 2][(i & 1u) * 2 + hi] = v;
							if (keep) *reinterpret_cast<uint32_t*>(keep + hi * 8 * W + 8 * i) = v;
						}
					}
				} else {
					// output layer: activation, then fp16 rows (and / or trimmed fp32 rows) to global memory
#pragma unroll
					for (uint32_t i = 0; i < C::ACC_N / 8; ++i) {
						const uint32_t c = 8 * i + 2 * ft;
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
				if (stamp) MLPF_STAMP(s, g, 3);
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

template <uint32_t W, bool GENERIC, bool BWD>
cudaError_t launch_impl(const MlpForwardParams& p, uint32_t n_sms, cudaStream_t stream) {
	using C = MlpCfg<W>;
	const uint32_t n_layers = p.n_hidden_layers + ((BWD && !p.output_fp16) ? 0 : 1);  // steps of the chain
	MlpKernelParams kp{};
	kp.p = p;
	kp.n_steps = n_layers;
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
	if (!make_fp16_matrix_map(&mo, w, p.out_width, W, p.out_width)) return cudaErrorInvalidValue;
	auto kernel = mlp_forward_kernel<W, GENERIC, BWD>;
	const size_t smem = (size_t)kp.n_stages * C::STAGE_BYTES + 8 * 2 * MLPF_MAX_STAGES;
	cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
	if (err != cudaSuccess) return err;
	const uint32_t n_groups = (p.batch_size / UNIT_M + C::WGS - 1) / C::WGS;  // CTAs that have a unit for every consumer warpgroup
	return launch_pdl(kernel, n_groups < n_sms ? n_groups : n_sms, C::THREADS, smem, stream, kp, m0, mh, mo);
}

template <uint32_t W>
cudaError_t launch_width(const MlpForwardParams& p, uint32_t n_sms, cudaStream_t stream) {
	if (p.backward) return p.activation != ACT_RELU ? launch_impl<W, true, true>(p, n_sms, stream) : launch_impl<W, false, true>(p, n_sms, stream);
	const bool generic = p.activation != ACT_RELU || p.output_activation != ACT_NONE;
	return generic ? launch_impl<W, true, false>(p, n_sms, stream) : launch_impl<W, false, false>(p, n_sms, stream);
}

}  // namespace

uint32_t mlp_forward_resident_layers(uint32_t width) {
	switch (width) {
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
	if (!(p.width == 16 || p.width == 32 || p.width == 64 || p.width == 128)) return fail("FullyFusedMLP only supports 16, 32, 64, and 128 neurons");
	if (p.n_hidden_layers < 1) return fail("FullyFusedMLP requires at least 1 hidden layer (3 layers in total).");
	if (p.n_hidden_layers + 1 > 64) return fail("tcnn_b200: the stand-alone MLP kernel covers up to 63 hidden layers");
	const uint32_t max_in = 64 * ((p.width + 63) / 64);
	if (p.in_width == 0 || p.in_width % 16 != 0 || p.in_width > max_in) return fail("tcnn_b200: network input width must be a multiple of 16 and at most 64 (128 for 128 neurons)");
	if (p.out_width == 0 || p.out_width % 16 != 0 || p.out_width > p.width) return fail("tcnn_b200: padded network output width must be a multiple of 16 and at most n_neurons");
	if (p.batch_size == 0 || p.batch_size % TILE_M != 0) return fail("batch size must be a non-zero multiple of 256");
	if ((p.input_fp16 != nullptr) == (p.input_fp32 != nullptr)) return fail("tcnn_b200: exactly one network input must be given");
	if (p.backward) {
		if (!p.input_fp16 || !p.hidden_in || p.output_fp32) return fail("tcnn_b200: the backward chain needs dL/d(output) and the forward activations in fp16");
		if (p.output_fp16 && p.in_width > (p.width < 32 ? 32u : p.width)) return fail("tcnn_b200: dL/d(input) of the stand-alone network covers inputs up to max(n_neurons, 32) wide");
	}
	if (p.input_fp32 && (p.n_input_dims == 0 || p.n_input_dims > p.in_width)) return fail("tcnn_b200: Identity encoding wider than the network input");
	return true;
}

cudaError_t launch_mlp_forward(const MlpForwardParams& p, uint32_t n_sms, cudaStream_t stream) {
	if (!mlp_forward_supported(p, nullptr)) return cudaErrorInvalidValue;
	switch (p.width) {
		case 128: return launch_width<128>(p, n_sms, stream);
		case 64: return launch_width<64>(p, n_sms, stream);
		case 32: return launch_width<32>(p, n_sms, stream);
		case 16: return launch_width<16>(p, n_sms, stream);
	}
	return cudaErrorInvalidValue;
}

}  // namespace tcnnb
