// model.cu -- host side of the hot path and the C ABI declared in include/tcnn_b200.h.
//
// Mirrors, for the HashGrid + FullyFusedMLP path only, what the reference spreads over
//   config.h:53-63              create_from_config
//   src/encoding.cu:132-150     create_encoding ("otype" dispatch, case-insensitive)  + grid.h:1726-1851 (grid JSON keys)
//   src/network.cu:51-141       select_network / create_network
//   src/loss.cu:82-90           create_loss
//   trainer.h:51-87,254-378     Trainer ctor / initialize_params / training_step / loss
//   network_with_input_encoding.h:115-150  parameter layout [MLP | grid]
// The optimizer (create_optimizer, src/optimizer.cu:50-80) is optimizer.cu's.
// There is deliberately no fallback: unsupported configurations raise the error the caller sees via tcnnb_last_error().
#include "../../include/tcnn_b200.h"

#include "binning.h"
#include "common.cuh"
#include "encoding_plan.h"
#include "fused_step.h"
#include "grid_config.h"
#include "grid_kernels.h"
#include "host_common.h"
#include "json_mini.h"
#include "misc_kernels.h"
#include "mlp_fused.h"
#include "network_config.h"
#include "optimizer.h"

#include <dlfcn.h>
#include <nccl.h>  // types and prototypes only: libnccl is resolved at run time (dlopen), single-GPU users never need it

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <random>
#include <stdexcept>
#include <string>
#include <vector>

namespace tcnnb {

std::atomic<uint64_t> g_kernel_launches{0};
thread_local std::string g_last_error;

// ------------------------------------------------------------------------------------------------ NCCL (data parallel)
// libnccl.so.2 is looked up when the first data-parallel call is made. In a PyTorch process this resolves to the copy
// torch has already loaded, so both use one NCCL; tcnn_b200 itself has no link-time dependency on it.
struct NcclApi {
	decltype(&ncclGetUniqueId) GetUniqueId = nullptr;
	decltype(&ncclCommInitRank) CommInitRank = nullptr;
	decltype(&ncclCommDestroy) CommDestroy = nullptr;
	decltype(&ncclAllReduce) AllReduce = nullptr;
	decltype(&ncclReduceScatter) ReduceScatter = nullptr;
	decltype(&ncclAllGather) AllGather = nullptr;
	decltype(&ncclGetErrorString) GetErrorString = nullptr;
};

static NcclApi& nccl_api() {
	static NcclApi api = [] {
		NcclApi a;
		void* lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
		if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
		if (!lib) throw std::runtime_error(std::string("data-parallel training needs NCCL: ") + dlerror());
		auto sym = [&](const char* name) {
			void* f = dlsym(lib, name);
			if (!f) throw std::runtime_error(std::string("libnccl lacks ") + name);
			return f;
		};
		a.GetUniqueId = (decltype(a.GetUniqueId))sym("ncclGetUniqueId");
		a.CommInitRank = (decltype(a.CommInitRank))sym("ncclCommInitRank");
		a.CommDestroy = (decltype(a.CommDestroy))sym("ncclCommDestroy");
		a.AllReduce = (decltype(a.AllReduce))sym("ncclAllReduce");
		a.ReduceScatter = (decltype(a.ReduceScatter))sym("ncclReduceScatter");
		a.AllGather = (decltype(a.AllGather))sym("ncclAllGather");
		a.GetErrorString = (decltype(a.GetErrorString))sym("ncclGetErrorString");
		return a;
	}();
	return api;
}

#define TCNNB_NCCL_CHECK(x)                                                                                             \
	do {                                                                                                                \
		ncclResult_t _r = (x);                                                                                          \
		if (_r != ncclSuccess) throw std::runtime_error(std::string(#x " failed: ") + nccl_api().GetErrorString(_r));   \
	} while (0)

// Two communicators: the gradient reduction runs on the caller's stream, the parameter all-gather on a side stream, and two
// collectives of ONE communicator may not be in flight concurrently.
struct DpState {
	ncclComm_t comm_grads = nullptr, comm_params = nullptr;
	int world = 1, rank = 0;
	bool shard_optimizer = true;
	bool masters_synced = true;
	cudaStream_t gather_stream = nullptr;
	cudaEvent_t ev_updated = nullptr, ev_gathered = nullptr;
	// peer-memory engine (tcnnb_dp_attach_symmetric): the working parameters and the gradient vector live in a symmetric allocation
	// every rank has mapped; reduce-scatter + Adam + all-gather become ONE kernel between two cross-GPU barriers
	bool fused = false;
	DpPeers peers{};
	uint32_t epoch = 0;
	~DpState() {
		if (comm_grads) nccl_api().CommDestroy(comm_grads);
		if (comm_params) nccl_api().CommDestroy(comm_params);
		if (gather_stream) cudaStreamDestroy(gather_stream);
		if (ev_updated) cudaEventDestroy(ev_updated);
		if (ev_gathered) cudaEventDestroy(ev_gathered);
	}
};

struct Model {
	uint32_t n_in = 0, n_out = 0;
	std::string enc_otype;  // the encoding's "otype" as the caller wrote it (hyperparams of encodings other than one grid / Identity)
	EncodingPlan plan;      // the encoding: segment table, grids, parameter count and padded width
	MlpConfig mlp;
	uint32_t loss_type = LOSS_RELATIVE_L2;
	std::string loss_name = "RelativeL2";
	std::unique_ptr<Optimizer> opt;  // a module handle's is never allocated
	float loss_scale = 128.0f;  // default_loss_scale<__half>() (common.h:243)
	int n_sms = 132;

	size_t n_params = 0;
	// trainer.h:489-503: one allocation [fp32 master | fp16 params | fp16 gradients]
	DeviceBuffer<char> params_buffer;
	size_t n_params_padded = 0;
	bool module_only = false;  // tcnnb_module: no trainer-owned parameters
	// tcnnb_create_network_trainer: a Network without an encoding. The inputs (and dL/d(input)) are the network's own fp16 rows
	// [batch][n_in], read and written in place by the stand-alone network kernels (general path).
	bool half_input = false;
	float* params_fp32 = nullptr;
	__half* params_fp16 = nullptr;
	__half* grads_fp16 = nullptr;
	DeviceBuffer<float> dw_accum;   // fp32 MLP weight-gradient accumulator
	DeviceBuffer<float> scalars;    // [0] = loss sum
	DeviceBuffer<long long> dbg_clock;  // TCNNB_CLOCKS=<file> in ablation builds: phase stamps of the last ws launch
	FusedStepParams fused{};                // the fused kernel's per-model arguments (configurations it runs); make_params adds the per-call ones
	DeviceBuffer<__half> denc_scratch;      // fused path, dL/d(input): dL/d(encoded) rows [n][64] handed from the fused kernel to the input-gradient kernel
	DeviceBuffer<__half> grads_scratch;     // GradientMode::Ignore (fused path): table gradients nobody reads; Accumulate (general path): this call's table gradients
	DeviceBuffer<float> dw_scratch;         // GradientMode::Ignore (fused path): network weight-gradient sums nobody reads
	bool mlp_grads_in_accum = false;
	// General (unfused) path: configurations the fused kernel does not cover -- 128 neurons, n_features_per_level in {1, 4, 8}, 4-D
	// inputs, Nearest interpolation, wider encodings / outputs -- run as encoding kernel -> stand-alone MLP kernels -> encoding backward
	// kernel, with the activations of one batch in HBM (the reference's own structure, object.h / network_with_input_encoding.h).
	bool general = false;
	bool force_general = false;  // tcnnb_debug_set("general", 1): run the general path although the fused kernel covers the configuration
	bool use_general() const { return general || force_general; }
	DeviceBuffer<__half> g_enc, g_out, g_dy, g_denc;
	MlpScratch g_mlp;

	// spatial binning scratch (binning.cu): sorted copies of the batch + permutation
	bool binning = true;  // tcnnb_debug_set("binning", 0) (tests: binned and unbinned steps must touch the same entries)
	cudaStream_t last_stream = nullptr;  // stream of the most recent step (tcnnb_param_gradients orders itself behind it)
	DeviceBuffer<uint32_t> bin_keys, bin_hist, bin_perm;

	// host staging for the *_host entry points
	float* pinned = nullptr;
	size_t pinned_floats = 0;
	DeviceBuffer<float> stage_in, stage_out;
	cudaStream_t own_stream = nullptr;   // compute stream of the *_host entry points
	cudaStream_t copy_stream = nullptr;  // host->device copies of the pipelined host step (overlap the previous step's kernels)
	// Pipelined host-buffer training step (tcnnb_training_step_host_submit / _wait): two slots, so that the copies of step i+1
	// travel while the kernels of step i run. Each slot owns device staging, pinned host staging (for pageable callers) and events.
	struct HostSlot {
		DeviceBuffer<float> in, target;
		float* pinned = nullptr;  // [pinned_floats]: inputs, targets; last element = the loss read back
		size_t pinned_floats = 0;
		cudaEvent_t ev_in = nullptr, ev_target = nullptr, ev_done = nullptr;
		uint64_t ticket = 0;
		bool busy = false;
	};
	HostSlot slots[2];
	uint64_t next_ticket = 1;
	const void* known_pinned[4] = {nullptr, nullptr, nullptr, nullptr};  // caller buffers already seen to be page-locked (skips the driver query)
	uint32_t known_pinned_next = 0;
	std::unique_ptr<DpState> dp;  // set by tcnnb_dp_init
	cudaEvent_t pending_params_event = nullptr;  // caller-owned: the next reader of the parameters waits for it (tcnnb_wait_before_compute)
	void wait_pending(cudaStream_t stream) {
		if (pending_params_event) {
			cudaStreamWaitEvent(stream, pending_params_event, 0);
			pending_params_event = nullptr;
		}
	}

	tcnnb_debug_taps taps{};
	std::string hyperparams_json;

	// optional per-kernel timing (bench.py roofline): events around the fused kernel and the Adam kernel of every step
	uint32_t ablate = 0;  // profiling experiments only (TCNNB_ABLATE env var)
	bool profiling = false;
	std::vector<cudaEvent_t> prof_events;  // quadruples: step start, after binning, after the backward pass, after Adam

	~Model() {
		if (pinned) cudaFreeHost(pinned);
		for (auto& sl : slots) {
			if (sl.pinned) cudaFreeHost(sl.pinned);
			if (sl.ev_in) cudaEventDestroy(sl.ev_in);
			if (sl.ev_target) cudaEventDestroy(sl.ev_target);
			if (sl.ev_done) cudaEventDestroy(sl.ev_done);
		}
		if (own_stream) cudaStreamDestroy(own_stream);
		if (copy_stream) cudaStreamDestroy(copy_stream);
		for (auto e : prof_events) cudaEventDestroy(e);
	}

	cudaEvent_t prof_mark(cudaStream_t stream) {
		cudaEvent_t e = nullptr;
		if (profiling && prof_events.size() < 4 * 8192) {
			if (cudaEventCreate(&e) == cudaSuccess) {
				cudaEventRecord(e, stream);
				prof_events.push_back(e);
			}
		}
		return e;
	}
};

// Whether the encoding is exactly one encoding of `type` (FEAT_GRID / FEAT_IDENTITY) over all inputs: the two encodings the fused
// kernel reads. A Composite that nests a single encoding is neither.
static bool single_encoding(const EncodingPlan& plan, uint32_t type) { return !plan.composite && plan.segs.n == 1 && plan.segs.s[0].type == type; }

// initialize_params(rnd, params_full_precision, scale) of NetworkWithInputEncoding (network_with_input_encoding.h:124-130):
// network weights first, then the grid table, one pcg32 stream. `dst` is a DEVICE fp32 array of n_params elements.
static void init_params(Model& m, HostPcg32& rng, float* dst, float scale) {
	init_mlp_params(m.mlp, rng, dst, scale);
	init_plan_params(m.plan, rng, dst + m.mlp.n_params, scale);  // nested encodings draw one after the other from the same stream
}

// Whether the stand-alone network kernels cover this network: nullptr, else the reason they do not. The encoding's backward pass
// needs dL/d(encoded) when it has parameters.
static const char* general_path_unsupported(const Model& m) { return mlp_unsupported(m.mlp, m.plan.n_params != 0); }

// Whether the fused kernel (fused_ws.cu) covers this configuration: nullptr, else the first of its limits that it does not meet.
static const char* fused_kernel_unsupported(const EncodingPlan& plan, const MlpConfig& mlp, uint32_t n_in) {
	const GridConfig* grid = single_encoding(plan, FEAT_GRID) ? &plan.grids[0]->cfg : nullptr;
	if (!grid && !single_encoding(plan, FEAT_IDENTITY)) return "an encoding other than one grid / Identity";
	if (activation_needs_preact(mlp.activation)) return "an activation that needs stored pre-activations (Sine / SiLU)";
	if (mlp.width > 64) return "n_neurons > 64";
	if (mlp.n_hidden_layers > 6) return "n_hidden_layers > 6";
	if (mlp.padded_out_width != 16) return "more than 16 outputs";
	if (grid && grid->n_features_per_level != 2) return "n_features_per_level != 2";
	if (n_in != 2 && n_in != 3) return "input dimensions other than 2 / 3";
	if (plan.width > 64 || (grid && grid->n_levels > MAX_LEVELS)) return "encoding wider than 64 features";
	if (fused_ws_smem_bytes(mlp.n_hidden_layers, plan.width, true) > 227 * 1024) return "shared-memory footprint of this depth / encoding width";
	if (grid && grid->interpolation == INTERP_NEAREST) return "Nearest interpolation";
	return nullptr;
}

static void build_model(Model& m, uint32_t n_in, uint32_t n_out, const json::Value& cfg, uint32_t seed, bool module_only = false, bool half_input = false) {
	m.n_sms = require_sm90();
#ifdef TCNNB_ENABLE_ABLATION  // profiling builds only (make ABLATION=1); the production library reads no environment switches
	if (const char* e = std::getenv("TCNNB_ABLATE")) m.ablate = (uint32_t)std::atoi(e);
	if (std::getenv("TCNNB_CLOCKS")) {
		m.dbg_clock.resize((size_t)2 * m.n_sms * 3 * 16 * 16);
		m.dbg_clock.zero();
	}
#endif
	m.n_in = n_in;
	m.n_out = n_out;

	// ---- loss (src/loss.cu:82-90)
	const json::Value& loss = cfg.sub("loss");
	m.loss_name = loss.value("otype", "RelativeL2");
	if (ieq(m.loss_name, "RelativeL2")) m.loss_type = LOSS_RELATIVE_L2;
	else if (ieq(m.loss_name, "L2")) m.loss_type = LOSS_L2;
	else if (ieq(m.loss_name, "L1")) m.loss_type = LOSS_L1;
	else if (ieq(m.loss_name, "RelativeL1")) m.loss_type = LOSS_RELATIVE_L1;
	else if (ieq(m.loss_name, "Mape")) m.loss_type = LOSS_MAPE;
	else if (ieq(m.loss_name, "Smape")) m.loss_type = LOSS_SMAPE;
	else if (ieq(m.loss_name, "RelativeL2Luminance")) {
		if (n_out < 3) throw std::runtime_error("tcnn_b200: RelativeL2Luminance needs at least 3 outputs (r, g, b)");
		m.loss_type = LOSS_RELATIVE_L2_LUMINANCE;
	} else if (ieq(m.loss_name, "CrossEntropy")) m.loss_type = LOSS_CROSS_ENTROPY;
	else if (ieq(m.loss_name, "Variance")) m.loss_type = LOSS_VARIANCE_IS;
	else throw std::runtime_error("Loss '" + m.loss_name + "' not found");

	// ---- optimizer (src/optimizer.cu:50-80, adam.h:221-303)
	m.opt = std::make_unique<Optimizer>(cfg.sub("optimizer"));

	// ---- encoding, padded to the network's alignment (network_with_input_encoding.h:47; FullyFusedMLP / CutlassMLP REQUIRED_ALIGNMENT,
	// src/network.cu:79-98). One grid or one Identity (encodings/identity.h:46-67: feature j = x_j * scale + offset, padding features
	// ONE) can run in the fused kernel; the plan runs every encoding on the general path and the module tier's dL/d(input).
	// A network trainer has no encoding: its plan is the parameter-free Identity of width n_in that is never run.
	m.half_input = half_input;
	if (half_input && (n_in == 0 || n_in % 16 != 0)) {
		throw std::runtime_error("network trainer: fp16 inputs need n_input_dims to be a positive multiple of 16 (got " + std::to_string(n_in) + ").");
	}
	const json::Value identity = json::parse("{\"otype\": \"Identity\"}");
	const json::Value& enc_cfg = half_input ? identity : cfg.sub("encoding");
	m.enc_otype = enc_cfg.value("otype", "OneBlob");
	build_encoding_plan(m.plan, n_in, enc_cfg, 16);

	// ---- network (src/network.cu:51-141)
	MlpConfig& mlp = m.mlp;
	mlp = parse_network(cfg.sub("network"), m.plan.width, n_out);

	// ---- which kernels run this configuration. The fused kernel covers the benchmarked family; everything else the stand-alone
	// kernels cover takes the general path; the rest fails loudly (no fallback to anything that is not a kernel of this library).
	if (const char* why = half_input ? "fp16 network inputs" : fused_kernel_unsupported(m.plan, mlp, n_in)) {
		m.general = true;
		if (const char* why_not = general_path_unsupported(m)) throw std::runtime_error(std::string(why_not) + " (general path of tcnn_b200; the fused kernel does not cover this configuration: " + why + ")");
	} else {
		FusedStepParams& p = m.fused;
		p.ablate = m.ablate;
		p.grid.padded_width = m.plan.width;
		if (single_encoding(m.plan, FEAT_GRID)) {
			const EncodingPlan::Grid& g = *m.plan.grids[0];
			p.grid.n_levels = g.cfg.n_levels;
			p.grid.n_features = g.cfg.n_levels * g.cfg.n_features_per_level;
			p.grid.interpolation = g.cfg.interpolation;
			std::copy(g.levels.begin(), g.levels.end(), p.grid.levels);
		} else {
			p.enc_identity = 1;
			p.identity_scale = m.plan.segs.s[0].scale;
			p.identity_offset = m.plan.segs.s[0].offset;
		}
		p.width = mlp.width;
		p.n_hidden_layers = mlp.n_hidden_layers;
		p.activation = mlp.activation;
		p.output_activation = mlp.output_activation;
		p.n_out = n_out;
		p.n_mlp_params = mlp.n_params;
		p.loss_type = m.loss_type;
		p.loss_scale = m.loss_scale;
		p.dbg_clock = m.dbg_clock.n ? m.dbg_clock.ptr : nullptr;
	}

	// ---- parameter buffers (trainer.h:69-87,489-503)
	m.n_params = (size_t)mlp.n_params + m.plan.n_params;
	// Same order as the reference's single allocation [fp32 master | working fp16 | fp16 gradients]; each region is padded to
	// a multiple of 512 parameters (never-touched zero entries) so that a data-parallel job can cut it into equal, 16-byte
	// aligned slices for any world size up to 64 (tcnn_b200/dp.py).
	m.n_params_padded = (m.n_params + 511) / 512 * 512;
	m.module_only = module_only;
	if (!module_only) {  // the module tier works on caller-owned parameter / gradient arrays and has no optimizer state
		m.params_buffer.resize(m.n_params_padded * (sizeof(float) + 2 * sizeof(__half)));
		m.params_buffer.zero();
		m.params_fp32 = (float*)m.params_buffer.ptr;
		m.params_fp16 = (__half*)(m.params_buffer.ptr + sizeof(float) * m.n_params_padded);
		m.grads_fp16 = (__half*)(m.params_buffer.ptr + sizeof(float) * m.n_params_padded + sizeof(__half) * m.n_params_padded);
	}
	m.dw_accum.resize(mlp.n_params);
	m.dw_accum.zero();
	m.scalars.resize(4);
	m.scalars.zero();

	if (!module_only) {
		// ---- initialisation: std::seed_seq{seed} -> pcg32{seeds[0]} (trainer.h:51-58)
		std::seed_seq seq{seed};
		std::vector<uint32_t> seeds(2);
		seq.generate(seeds.begin(), seeds.end());
		HostPcg32 rng{seeds.front()};
		init_params(m, rng, m.params_fp32, 1.0f);
		// fp32 -> fp16 (trainer.h:409-421)
		TCNNB_CUDA_CHECK(launch_cast_params(nullptr, m.n_params, m.params_fp32, m.params_fp16));
		++g_kernel_launches;
		m.opt->allocate(m.n_params, m.n_params_padded, m.params_fp16);
	}
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	TCNNB_CUDA_CHECK(cudaStreamCreateWithFlags(&m.own_stream, cudaStreamNonBlocking));
	TCNNB_CUDA_CHECK(cudaStreamCreateWithFlags(&m.copy_stream, cudaStreamNonBlocking));
	for (auto& sl : m.slots) {
		TCNNB_CUDA_CHECK(cudaEventCreateWithFlags(&sl.ev_in, cudaEventDisableTiming));
		TCNNB_CUDA_CHECK(cudaEventCreateWithFlags(&sl.ev_target, cudaEventDisableTiming));
		TCNNB_CUDA_CHECK(cudaEventCreateWithFlags(&sl.ev_done, cudaEventDisableTiming));
	}
}

static FusedStepParams make_params(const Model& m, uint32_t batch, uint32_t loss_batch, const float* x, const float* y, const __half* params) {
	FusedStepParams p = m.fused;
	p.batch_size = batch;
	p.loss_batch_size = loss_batch;
	p.positions = x;
	p.targets = y;
	p.params = params;
	p.grads = m.grads_fp16;
	p.dw_accum = m.dw_accum.ptr;
	p.loss_sum = m.scalars.ptr;
	p.loss_values = m.taps.loss_values;
	p.out_fp16 = (__half*)m.taps.output;
	p.dbg_enc = (__half*)m.taps.encoded;
	p.dbg_hidden = (__half*)m.taps.hidden;
	p.dbg_dy = (__half*)m.taps.dL_doutput;
	p.dbg_grad_hidden = (__half*)m.taps.grad_hidden;
	p.dbg_denc = (__half*)m.taps.dL_dencoded;
	return p;
}

// What the optimizer updates: the trainer's parameter and gradient buffers, the network's gradients from the fp32 sums while they are
// current.
static OptimizerArrays optimizer_arrays(const Model& m) {
	return {m.params_fp32, m.params_fp16, m.grads_fp16, m.mlp_grads_in_accum ? m.dw_accum.ptr : nullptr, m.mlp.n_params, m.loss_scale};
}

// The optimizer over the parameter ranges [begin, begin + count) (all parameters when n_ranges == 0). A step that covers the network
// weights consumes their fp32 sums.
static void optimizer_step(Model& m, cudaStream_t stream, uint32_t n_ranges = 0, const uint64_t* begins = nullptr, const uint64_t* counts = nullptr) {
	if (!m.opt->allocated()) throw std::runtime_error("this handle was created with tcnnb_module_create: it has no optimizer.");
	m.wait_pending(stream);
	if (m.opt->step(stream, optimizer_arrays(m), n_ranges, begins, counts)) m.mlp_grads_in_accum = false;
}

// ---- general path: encoding kernel -> stand-alone network kernel (mlp_fused.cu), activations optionally kept for the backward pass
// The network's input rows: the encoded batch, or a network trainer's own fp16 input.
static const __half* network_input(const Model& m, const float* x) { return m.half_input ? (const __half*)x : m.g_enc.ptr; }

// A network trainer's input and dL/d(input) rows go to the network kernels as they are: the same 16-byte alignment as the network tier.
static void check_half_rows(const Model& m, const float* x, const float* dL_dinput) {
	if (!m.half_input) return;
	if (!x) throw std::runtime_error("network trainer: input is null.");
	if (((uintptr_t)x | (uintptr_t)dL_dinput) % 16 != 0) throw std::runtime_error("network trainer: fp16 input / dL_dinput rows must be 16-byte aligned.");
}

static void general_forward(Model& m, cudaStream_t stream, uint32_t batch, const float* x, const __half* params, __half* out_fp16, float* out_fp32, bool keep_hidden) {
	const MlpConfig& mlp = m.mlp;
	if (!m.half_input) {
		grow(m.g_enc, (size_t)batch * mlp.in_width);
		plan_forward(m.plan, stream, batch, x, params + mlp.n_params, m.g_enc.ptr, mlp.in_width, 1.0f);
	}
	MlpForwardParams p = mlp_forward_params(mlp, params, batch, keep_hidden ? m.g_mlp.hidden_rows(mlp, batch) : nullptr);
	p.input_fp16 = network_input(m, x);  // (after the encoding's rows are grown: the pointer is read here)
	p.output_fp16 = out_fp16;
	p.output_fp32 = out_fp32;
	run_mlp_forward(p, m.n_sms, stream);
	m.last_stream = stream;
}

__global__ void half_to_float_kernel(uint64_t n, const __half* __restrict__ in, float* __restrict__ out) {
	const uint64_t i = threadIdx.x + (uint64_t)blockIdx.x * blockDim.x;
	if (i < n) out[i] = (float)in[i];
}

__global__ void half_accumulate_kernel(uint64_t n, const __half* __restrict__ in, __half* __restrict__ inout) {
	const uint64_t i = threadIdx.x + (uint64_t)blockIdx.x * blockDim.x;
	if (i < n) inout[i] = __hadd(inout[i], in[i]);
}

// tcnn::GradientMode (object.h:116-120)
enum GradientMode : int { GRADIENT_IGNORE = 0, GRADIENT_OVERWRITE = 1, GRADIENT_ACCUMULATE = 2 };

// One backward call of the trainer or module tier: Trainer::training_step with all of its arguments (trainer.h:254-357) or
// Module::backward (cpp_api.cu:104-125).
struct BackwardCall {
	uint32_t batch = 0, loss_batch = 0;  // loss_batch: what the loss is normalised over (the global batch of a data-parallel shard)
	const float* x = nullptr;
	const float* y = nullptr;             // targets (unused with dL_doutput)
	const float* data_pdf = nullptr;      // optional [batch][n_out]: the loss divides by it
	const __half* params = nullptr;       // the trainer's working or Ema weights, or the module caller's
	const __half* dL_doutput = nullptr;   // optional fp16 [batch][padded_out_width], already x loss scale: replaces the loss
	GradientMode mode = GRADIENT_OVERWRITE;
	__half* grads = nullptr;              // [n_params]: the trainer's gradient buffer or the module caller's dL_dparams
	float* dL_dinput = nullptr;           // optional fp32 [batch][n_in], overwritten
	bool finalize = false;                // round the fp32 network sums into `grads` (the module tier hands out fp16 gradients)
	bool run_optimizer = false;
	cudaEvent_t targets_ready = nullptr;  // optional: the first kernel waits for it; gradient zeroing and binning only need `x`
};

// fp32 network weight-gradient sums -> fp16 entries of `grads` (what the reference's gradient buffer holds); re-arms the accumulator
static void finalize_mlp_grads(Model& m, cudaStream_t stream, __half* grads) {
	if (m.mlp_grads_in_accum) {
		TCNNB_CUDA_CHECK(launch_mlp_grad_finalize(stream, m.mlp.n_params, m.dw_accum.ptr, grads));
		++g_kernel_launches;
		m.mlp_grads_in_accum = false;
	}
}

// The general path's backward pass: forward with the activations kept, the loss (or the caller's dL/d(output)), the network backward
// adding into `dw` and the encoding backward overwriting `table_grads` (either may be null) and dL_dinput.
static void general_backward(Model& m, cudaStream_t stream, const BackwardCall& c, float* dw, __half* table_grads) {
	const MlpConfig& mlp = m.mlp;
	grow(m.g_out, (size_t)c.batch * mlp.padded_out_width);
	__half* const out_rows = (m.taps.output && mlp.padded_out_width == 16) ? (__half*)m.taps.output : m.g_out.ptr;  // (the test tap is 16 columns wide)
	general_forward(m, stream, c.batch, c.x, c.params, out_rows, nullptr, true);

	// Module::backward: the caller's dL/d(output) still has to pass the output activation (fully_fused_mlp.cu:755-762). Trainer: the
	// loss kernel writes loss gradient x loss_scale, through the output activation, in one kernel.
	const __half* dL_doutput = c.dL_doutput;
	if (!dL_doutput) {
		grow(m.g_dy, (size_t)c.batch * mlp.padded_out_width);
		__half* const dy_rows = (m.taps.dL_doutput && mlp.padded_out_width == 16) ? (__half*)m.taps.dL_doutput : m.g_dy.ptr;
		TCNNB_CUDA_CHECK(launch_loss(stream, m.loss_type, mlp.output_activation, c.batch, m.n_out, mlp.padded_out_width, m.loss_scale, c.loss_batch * m.n_out, out_rows, c.y,
		                             c.data_pdf, dy_rows, m.taps.loss_values, m.n_out, m.scalars.ptr));
		++g_kernel_launches;
		dL_doutput = dy_rows;
	}
	if (m.half_input) {  // no encoding: the network writes dL/d(input) straight into the caller's fp16 rows
		run_mlp_backward(mlp, m.g_mlp, m.n_sms, stream, c.batch, c.params, network_input(m, c.x), m.g_mlp.hidden.ptr, out_rows, dL_doutput, c.dL_doutput != nullptr,
		                 (__half*)c.dL_dinput, dw);
		return;
	}
	const bool need_denc = table_grads || c.dL_dinput;
	if (need_denc) grow(m.g_denc, (size_t)c.batch * mlp.in_width);
	run_mlp_backward(mlp, m.g_mlp, m.n_sms, stream, c.batch, c.params, m.g_enc.ptr, m.g_mlp.hidden.ptr, out_rows, dL_doutput, c.dL_doutput != nullptr,
	                 need_denc ? m.g_denc.ptr : nullptr, dw);
	// (a Product reads the nested outputs general_forward just left in the plan's scratch)
	plan_backward(m.plan, stream, c.batch, c.x, c.params + mlp.n_params, m.g_denc.ptr, mlp.in_width, table_grads, c.dL_dinput, 1.0f, true);
}

// Runs one backward call on the fused kernel or the general path, then the optimizer when asked. Records one profile quadruple.
static void backward_step(Model& m, cudaStream_t stream, const BackwardCall& c) {
	check_half_rows(m, c.x, c.dL_dinput);
	const uint32_t batch = c.batch, n_mlp = m.mlp.n_params;
	const bool general = m.use_general();
	const bool overwrite = c.mode == GRADIENT_OVERWRITE;
	if (c.dL_dinput && !general) {
		// Nothing checks the fused kernel's dL/d(encoded) rows of an Identity encoding; the general path computes this gradient.
		if (single_encoding(m.plan, FEAT_IDENTITY)) {
			throw std::runtime_error("input gradients through an Identity encoding are not built for configurations the fused kernel runs; the general path (e.g. n_neurons > 64) computes them.");
		}
		// dL/d(input) (NetworkWithInputEncoding::backward -> GridEncoding::backward_impl, grid.h:896-921): the fused kernel hands out
		// the network's input gradient rows, the plan's grid kernel contracts them with d(encoded)/d(position).
		grow(m.denc_scratch, (size_t)batch * 64);
	}

	// Where the gradients go. Overwrite / Accumulate: the network's into the model's fp32 sums, the table's into `grads`; the general
	// path overwrites the table gradients it computes, so Accumulate sends them to scratch and adds that onto `grads` afterwards.
	// Ignore: the fused kernel still scatters, into scratch that is never zeroed and never read (trainer.h:338 hands the reference's a
	// null gradient buffer); the general path computes no parameter gradients.
	__half* grads = c.grads;
	float* dw = m.dw_accum.ptr;
	if (c.mode == GRADIENT_IGNORE && general) {
		grads = nullptr;
		dw = nullptr;
	} else if (c.mode == GRADIENT_IGNORE || (c.mode == GRADIENT_ACCUMULATE && general)) {
		m.grads_scratch.resize(m.n_params_padded);
		grads = m.grads_scratch.ptr;
		if (!general) {
			m.dw_scratch.resize(n_mlp);
			dw = m.dw_scratch.ptr;
		}
	}
	if (c.mode == GRADIENT_ACCUMULATE && !m.mlp_grads_in_accum && n_mlp) {
		// the network's gradients are the fp16 values in the buffer (tcnnb_param_gradients materialised them): the fp32 sums continue
		// from there
		half_to_float_kernel<<<(n_mlp + 255) / 256, 256, 0, stream>>>(n_mlp, c.grads, m.dw_accum.ptr);
		TCNNB_CUDA_CHECK(cudaGetLastError());
		++g_kernel_launches;
		m.mlp_grads_in_accum = true;
	}

	// Overwrite zeroes the fused kernel's grid gradient table (grid.h:865-867), and the loss accumulator is zeroed -- inside the binning
	// pass when there is one, else as memsets. (The general path overwrites its table gradients itself; a module handle reports no loss.)
	__half* const grid_grads = grads ? grads + n_mlp : nullptr;
	const size_t grid_grad_bytes = sizeof(__half) * m.plan.n_params;
	const bool bin = !general && m.binning && batch >= 16384 && single_encoding(m.plan, FEAT_GRID);  // spatial order only matters to the table gathers
	const bool zero_in_binning = overwrite && bin && (((uintptr_t)grid_grads | grid_grad_bytes) & 15u) == 0;
	if (general) {
		if (!m.module_only) TCNNB_CUDA_CHECK(cudaMemsetAsync(m.scalars.ptr, 0, sizeof(float), stream));
	} else if (!zero_in_binning) {
		if (overwrite) TCNNB_CUDA_CHECK(cudaMemsetAsync(grid_grads, 0, grid_grad_bytes, stream));
		TCNNB_CUDA_CHECK(cudaMemsetAsync(m.scalars.ptr, 0, sizeof(float), stream));
	}
	if (overwrite && m.mlp_grads_in_accum) {
		// a previous step left un-consumed weight gradients (run_optimizer == false twice in a row): Overwrite semantics
		TCNNB_CUDA_CHECK(cudaMemsetAsync(m.dw_accum.ptr, 0, sizeof(float) * n_mlp, stream));
		m.mlp_grads_in_accum = false;
	}

	m.prof_mark(stream);
	// Process the batch in (y, z)-column order: same sums, far fewer distinct memory sectors on the coarse levels (binning.cu).
	if (bin) {
		const uint32_t log2_r = binning_log2_resolution(batch, m.n_in);
		m.bin_keys.resize(std::max(m.bin_keys.n, 2 * (size_t)batch));
		m.bin_perm.resize(std::max(m.bin_perm.n, (size_t)batch));
		{
			const size_t need = 2 * (size_t)binning_n_bins(log2_r, m.n_in);
			if (m.bin_hist.n != need) {  // layout depends on n_bins: (re)allocate and zero the counters once
				m.bin_hist.resize(need);
				m.bin_hist.zero(stream);
			}
		}
		TCNNB_CUDA_CHECK(launch_binning(stream, m.n_in, batch, c.x, log2_r, m.bin_keys.ptr, m.bin_hist.ptr, m.bin_perm.ptr, zero_in_binning ? grid_grads : nullptr,
		                                zero_in_binning ? grid_grad_bytes : 0, zero_in_binning ? (float*)m.scalars.ptr : nullptr));
		g_kernel_launches += 3;
	}
	m.prof_mark(stream);
	if (c.targets_ready) TCNNB_CUDA_CHECK(cudaStreamWaitEvent(stream, c.targets_ready, 0));
	m.wait_pending(stream);  // e.g. the all-gather of the previous data-parallel step: binning above did not need the parameters
	if (general) {
		general_backward(m, stream, c, dw, m.plan.n_params ? grid_grads : nullptr);
		if (c.mode == GRADIENT_ACCUMULATE && m.plan.n_params) {
			half_accumulate_kernel<<<(uint32_t)((m.plan.n_params + 255) / 256), 256, 0, stream>>>(m.plan.n_params, grid_grads, c.grads + n_mlp);
			TCNNB_CUDA_CHECK(cudaGetLastError());
			++g_kernel_launches;
		}
	} else {
		FusedStepParams p = make_params(m, batch, c.loss_batch, c.x, c.y, c.params);
		p.grads = grads;
		p.dw_accum = dw;
		p.data_pdf = c.data_pdf;
		if (bin) p.perm = m.bin_perm.ptr;
		if (c.dL_dinput) p.dbg_denc = m.denc_scratch.ptr;
		if (c.dL_doutput) {
			p.ext_dy = c.dL_doutput;
			p.targets = nullptr;
			p.loss_sum = nullptr;
			p.loss_values = nullptr;
		}
		// one persistent 640-thread CTA per SM (fused_ws.cu)
		TCNNB_CUDA_CHECK(launch_fused_ws(p, m.n_in, true,std::min(batch / TILE_M, (uint32_t)m.n_sms), stream));
		++g_kernel_launches;
	}
	m.last_stream = stream;
	if (c.mode != GRADIENT_IGNORE) m.mlp_grads_in_accum = true;
	if (c.finalize) finalize_mlp_grads(m, stream, c.grads);
	if (c.dL_dinput && !general) plan_input_gradient(m.plan, stream, batch, c.x, c.params + n_mlp, m.denc_scratch.ptr, 64, c.dL_dinput, 1.0f);
	m.prof_mark(stream);
	// the optimizer comes last: the input gradient reads the parameters the step used
	if (c.run_optimizer) optimizer_step(m, stream);
	m.prof_mark(stream);
}

static void check_trainer(const Model& m) {
	if (m.module_only) throw std::runtime_error("this handle was created with tcnnb_module_create: use the tcnnb_module_* calls.");
}

// The host-buffer and data-parallel entry points stage and shard fp32 inputs.
static void check_float_input(const Model& m, const char* what) {
	if (m.half_input) throw std::runtime_error(std::string(what) + " takes fp32 inputs; a network trainer (tcnnb_create_network_trainer) trains on device fp16 rows.");
}

// The trainer's own step: Overwrite into its gradient buffer (tcnnb_training_step / _shard, the host-buffer pipeline, the data-parallel
// step).
static void training_step(Model& m, cudaStream_t stream, uint32_t batch, uint32_t loss_batch, const float* x, const float* y, bool run_optimizer, cudaEvent_t targets_ready = nullptr) {
	check_batch(batch);
	check_trainer(m);
	BackwardCall c;
	c.batch = batch;
	c.loss_batch = loss_batch;
	c.x = x;
	c.y = y;
	c.params = m.params_fp16;
	c.grads = m.grads_fp16;
	c.run_optimizer = run_optimizer;
	c.targets_ready = targets_ready;
	backward_step(m, stream, c);
}

// One data-parallel step, natively over NCCL (tcnn_b200/dp.py has the same logic over torch.distributed; SURVEY.md section 8e).
//   sharded optimizer: fwd+bwd on the shard -> fp16 gradient vector -> reduce-scatter: this rank's slice of the padded parameter
//   vector -> Adam on that slice -> all-gather of the updated fp16 slices on a side stream. The next step's binning pass
//   overlaps the all-gather; its fused kernel waits for it (pending_params_event).
//   replicated: all-reduce of the table gradients (fp16) and of the network accumulator (fp32), full Adam everywhere.
static void dp_training_step(Model& m, cudaStream_t stream, uint32_t shard_batch, uint32_t global_batch, const float* x, const float* y) {
	if (!m.dp) throw std::runtime_error("dp_training_step: call tcnnb_dp_init first.");
	DpState& d = *m.dp;
	NcclApi& n = nccl_api();
	training_step(m, stream, shard_batch, global_batch, x, y, false);
	if (d.world == 1) {
		optimizer_step(m, stream);
		return;
	}
	if (!d.shard_optimizer) {
		TCNNB_NCCL_CHECK(n.AllReduce(m.grads_fp16 + m.mlp.n_params, m.grads_fp16 + m.mlp.n_params, m.plan.n_params, ncclHalf, ncclSum, d.comm_grads, stream));
		TCNNB_NCCL_CHECK(n.AllReduce(m.dw_accum.ptr, m.dw_accum.ptr, m.mlp.n_params, ncclFloat, ncclSum, d.comm_grads, stream));
		optimizer_step(m, stream);
		return;
	}
	finalize_mlp_grads(m, stream, m.grads_fp16);
	const size_t chunk = m.n_params_padded / (size_t)d.world, lo = chunk * (size_t)d.rank;
	if (d.fused) {
		// Peer-memory engine: [barrier: every rank's gradient vector is complete] -> ONE kernel on this rank's slice that sums the
		// gradient over the ranks (in the switch with multimem.ld_reduce, else by peer loads), applies Adam and publishes the fp16
		// weights into every replica (multimem.st / peer stores) -> [barrier: all slices have landed everywhere; the gradient
		// vectors may be zeroed again]. No NCCL call on the step.
		TCNNB_CUDA_CHECK(launch_dp_barrier(stream, d.peers, ++d.epoch));
		m.opt->step_peers(stream, d.peers, lo, chunk, optimizer_arrays(m));
		TCNNB_CUDA_CHECK(launch_dp_barrier(stream, d.peers, ++d.epoch));
		g_kernel_launches += 2;
		d.masters_synced = false;
		return;
	}
	TCNNB_NCCL_CHECK(n.ReduceScatter(m.grads_fp16, m.grads_fp16 + lo, chunk, ncclHalf, ncclSum, d.comm_grads, stream));
	const uint64_t begin = lo, count = lo < m.n_params ? std::min<uint64_t>(chunk, m.n_params - lo) : 0;
	if (count) optimizer_step(m, stream, 1, &begin, &count);
	else m.opt->skip_step();  // a rank with no parameters in its slice still advances the step count and the decay schedule
	TCNNB_CUDA_CHECK(cudaEventRecord(d.ev_updated, stream));
	TCNNB_CUDA_CHECK(cudaStreamWaitEvent(d.gather_stream, d.ev_updated, 0));
	TCNNB_NCCL_CHECK(n.AllGather(m.params_fp16 + lo, m.params_fp16, chunk, ncclHalf, d.comm_params, d.gather_stream));
	TCNNB_CUDA_CHECK(cudaEventRecord(d.ev_gathered, d.gather_stream));
	m.pending_params_event = d.ev_gathered;
	d.masters_synced = false;
}

// Whether each rank holds the optimizer state of its own slice only (ZeRO-1).
static bool optimizer_state_sharded(const Model& m) { return m.dp && m.dp->world > 1 && m.dp->shard_optimizer; }

// Sum of the ranks' partial losses (each normalised over the global batch) -> the global loss, in place on every rank.
static void dp_reduce_loss(Model& m, cudaStream_t stream) {
	if (m.dp && m.dp->world > 1) {
		TCNNB_NCCL_CHECK(nccl_api().AllReduce(m.scalars.ptr, m.scalars.ptr, 1, ncclFloat, ncclSum, m.dp->comm_grads, stream));
	}
}

// Forward pass with `params`: fp16 rows [batch][padded_output_width] (the module tier, column-major padded x n in the reference's
// terms, cpp_api.cu:82-83) or fp32 [batch][n_out] (Network::inference, object.h:214-282). Nothing is saved for the backward pass --
// it recomputes the forward inside the fused kernel (the gather + three MMAs per tile are cheaper than writing and re-reading
// 2 x 64 x n fp16 activations, which is what the reference's context holds).
static void forward(Model& m, cudaStream_t stream, uint32_t batch, const float* x, const __half* params, __half* out_fp16, float* out_fp32) {
	check_half_rows(m, x, nullptr);
	m.wait_pending(stream);
	if (m.use_general()) {
		general_forward(m, stream, batch, x, params, out_fp16, out_fp32, false);
		return;
	}
	FusedStepParams p = make_params(m, batch, batch, x, nullptr, params);
	if (out_fp16) p.out_fp16 = out_fp16;  // (else the output tap, when a test set one)
	p.out_fp32 = out_fp32;
	p.loss_sum = nullptr;
	// the warp-specialised kernel without its backward half (measured 0.0885 ms vs 0.127 ms for the bulk-synchronous kernel it replaced)
	TCNNB_CUDA_CHECK(launch_fused_ws(p, m.n_in, false,std::min(batch / TILE_M, (uint32_t)m.n_sms), stream));
	++g_kernel_launches;
	m.last_stream = stream;
}

// ---- module tier (tcnn::cpp::Module for NetworkWithInputEncoding, cpp_api.cu:71-158): caller-owned parameters -------------
static void check_module_ptr(const void* ptr, const char* what) {
	if (!ptr) throw std::runtime_error(std::string("module: ") + what + " is null.");
	if ((uintptr_t)ptr % 16 != 0) throw std::runtime_error(std::string("module: ") + what + " must be 16-byte aligned.");
}

// backward: dL_dparams (fp16 [n_params], OVERWRITTEN -- GradientMode::Overwrite, cpp_api.cu:115; Ignore when it is null) from
// dL_doutput (fp16 [n][padded]).
static void module_backward(Model& m, cudaStream_t stream, uint32_t n, float* dL_dinput, const void* dL_doutput, void* dL_dparams, const float* x, const void* params) {
	if (!dL_dparams && !dL_dinput) return;  // nothing to compute
	check_module_ptr(params, "params");
	check_module_ptr(dL_doutput, "dL_doutput");
	check_batch(n);
	if (dL_dparams) check_module_ptr(dL_dparams, "dL_dparams");
	BackwardCall c;
	c.batch = c.loss_batch = n;
	c.x = x;
	c.params = (const __half*)params;
	c.dL_doutput = (const __half*)dL_doutput;
	c.mode = dL_dparams ? GRADIENT_OVERWRITE : GRADIENT_IGNORE;
	c.grads = (__half*)dL_dparams;
	c.dL_dinput = dL_dinput;
	c.finalize = dL_dparams != nullptr;
	backward_step(m, stream, c);
}

// Trainer::training_step with all of its arguments (trainer.h:254-357): the loss weighted by `data_pdf`, or the caller's `ext_dL_dy`
// (fp16 [batch][padded_output_width], already x loss scale) in place of the loss; the gradients overwrite, add onto or leave alone the
// trainer's buffer; `dL_dinput` (fp32 [batch][n_in]) is overwritten.
static void training_step_ex(Model& m, cudaStream_t stream, uint32_t batch, const float* x, const float* y, const float* data_pdf, bool run_optimizer, float* dL_dinput,
                             bool use_inference_params, int mode, const __half* ext_dL_dy) {
	check_trainer(m);
	if (m.dp) throw std::runtime_error("training_step_ex: data-parallel handles train with tcnnb_dp_training_step.");
	if (mode != GRADIENT_IGNORE && mode != GRADIENT_OVERWRITE && mode != GRADIENT_ACCUMULATE) {
		throw std::runtime_error("training_step_ex: param_gradients_mode must be 0 (Ignore), 1 (Overwrite) or 2 (Accumulate).");
	}
	if (!ext_dL_dy && !y) throw std::runtime_error("training_step: target is null and no external_dL_dy replaces the loss.");
	if (!x) throw std::runtime_error("training_step: input is null.");
	check_batch(batch);
	BackwardCall c;
	c.batch = c.loss_batch = batch;
	c.x = x;
	c.y = y;
	c.data_pdf = ext_dL_dy ? nullptr : data_pdf;  // the loss is not evaluated (trainer.h:127-131)
	c.params = use_inference_params ? m.opt->inference_params(m.params_fp16) : m.params_fp16;
	c.dL_doutput = ext_dL_dy;
	c.mode = (GradientMode)mode;
	c.grads = m.grads_fp16;
	c.dL_dinput = dL_dinput;
	c.run_optimizer = run_optimizer;
	backward_step(m, stream, c);
}

// Trainer::forward (trainer.h:97-139): the padded fp16 predictions of the inference launch, then -- unless the caller brings its own
// dL/d(output) -- the loss on them: per-element values and dL/d(output) x loss scale, both [batch][padded_output_width] with zero
// padding columns. The gradient is the loss's alone, as in the reference's context: the backward pass takes it through the output
// activation like an external_dL_dy. Nothing is kept for the backward pass, which recomputes the forward.
static void trainer_forward(Model& m, cudaStream_t stream, uint32_t batch, const float* x, const float* y, const float* data_pdf, bool use_inference_params, bool external_dL_dy,
                            __half* output, float* loss_values, __half* dL_doutput) {
	check_trainer(m);
	if (m.dp) throw std::runtime_error("forward: data-parallel handles train with tcnnb_dp_training_step.");
	if (!external_dL_dy && !y) throw std::runtime_error("forward: target is null and no external_dL_dy replaces the loss.");
	if (external_dL_dy && dL_doutput) throw std::runtime_error("forward: with external_dL_dy the caller's buffer is dL_doutput; dL_doutput_dev must be null.");
	if (!x) throw std::runtime_error("forward: input is null.");
	if (!output || (uintptr_t)output % 16 != 0) throw std::runtime_error("forward: output must be a 16-byte aligned device array.");
	if ((uintptr_t)dL_doutput % 16 != 0) throw std::runtime_error("forward: dL_doutput must be 16-byte aligned.");
	check_batch(batch);
	forward(m, stream, batch, x, use_inference_params ? m.opt->inference_params(m.params_fp16) : m.params_fp16, output, nullptr);
	if (external_dL_dy || (!loss_values && !dL_doutput)) return;
	const uint32_t pad = m.mlp.padded_out_width;
	TCNNB_CUDA_CHECK(launch_loss(stream, m.loss_type, ACT_NONE, batch, m.n_out, pad, m.loss_scale, batch * m.n_out, output, y, data_pdf, dL_doutput, loss_values, pad, nullptr));
	++g_kernel_launches;
}

static void ensure_staging(Model& m, uint32_t batch) {
	const size_t need = (size_t)batch * (m.n_in + m.n_out) + 16;
	if (m.pinned_floats < need) {
		if (m.pinned) cudaFreeHost(m.pinned);
		m.pinned = nullptr;
		TCNNB_CUDA_CHECK(cudaMallocHost(&m.pinned, need * sizeof(float)));
		m.pinned_floats = need;
	}
	m.stage_in.resize(std::max(m.stage_in.n, (size_t)batch * m.n_in));
	m.stage_out.resize(std::max(m.stage_out.n, (size_t)batch * m.n_out));
}

static bool host_ptr_is_pinned(Model& m, const void* ptr) {
	for (const void* k : m.known_pinned) if (k == ptr) return true;
	cudaPointerAttributes attr{};
	const bool pinned = cudaPointerGetAttributes(&attr, ptr) == cudaSuccess && attr.type == cudaMemoryTypeHost;
	cudaGetLastError();
	if (pinned) m.known_pinned[m.known_pinned_next++ % 4] = ptr;
	return pinned;
}

// Enqueue one training step on HOST buffers and return at once: host->device copies on the copy stream (they overlap the kernels
// of the step submitted before), the step on the model's compute stream (the binning pass starts when the positions have
// landed, the fused kernel when the targets have), the loss read-back behind it. At most two steps are in flight.
static uint64_t host_step_submit(Model& m, uint32_t batch, uint32_t global_batch, const float* x_host, const float* y_host, bool data_parallel) {
	check_batch(batch);
	check_float_input(m, "the host-buffer training step");
	const uint64_t ticket = m.next_ticket;
	Model::HostSlot& sl = m.slots[ticket & 1u];
	if (sl.busy) throw std::runtime_error("training_step_host_submit: two steps are already in flight; collect ticket " + std::to_string(sl.ticket) + " with tcnnb_training_step_host_wait first.");
	const size_t n_x = (size_t)batch * m.n_in, n_y = (size_t)batch * m.n_out;
	sl.in.resize(std::max(sl.in.n, n_x));
	sl.target.resize(std::max(sl.target.n, n_y));
	if (sl.pinned_floats < 16) {
		TCNNB_CUDA_CHECK(cudaMallocHost(&sl.pinned, 16 * sizeof(float)));
		sl.pinned_floats = 16;
	}
	const float* sx = x_host;
	const float* sy = y_host;
	const bool x_pinned = host_ptr_is_pinned(m, x_host), y_pinned = host_ptr_is_pinned(m, y_host);
	if (!x_pinned || !y_pinned) {  // pageable caller memory: stage through this slot's page-locked buffer
		const size_t need = n_x + n_y + 16;
		if (sl.pinned_floats < need) {
			if (sl.pinned) cudaFreeHost(sl.pinned);
			sl.pinned = nullptr;
			sl.pinned_floats = 0;
			TCNNB_CUDA_CHECK(cudaMallocHost(&sl.pinned, need * sizeof(float)));
			sl.pinned_floats = need;
		}
	}
	cudaStream_t cs = m.copy_stream, s = m.own_stream;
	if (!x_pinned) { std::memcpy(sl.pinned, x_host, n_x * sizeof(float)); sx = sl.pinned; }
	TCNNB_CUDA_CHECK(cudaMemcpyAsync(sl.in.ptr, sx, n_x * sizeof(float), cudaMemcpyHostToDevice, cs));
	TCNNB_CUDA_CHECK(cudaEventRecord(sl.ev_in, cs));
	if (!y_pinned) { std::memcpy(sl.pinned + n_x, y_host, n_y * sizeof(float)); sy = sl.pinned + n_x; }  // while the inputs travel
	TCNNB_CUDA_CHECK(cudaMemcpyAsync(sl.target.ptr, sy, n_y * sizeof(float), cudaMemcpyHostToDevice, cs));
	TCNNB_CUDA_CHECK(cudaEventRecord(sl.ev_target, cs));
	TCNNB_CUDA_CHECK(cudaStreamWaitEvent(s, sl.ev_in, 0));
	float* loss_pinned = sl.pinned + sl.pinned_floats - 1;
	if (data_parallel) {
		TCNNB_CUDA_CHECK(cudaStreamWaitEvent(s, sl.ev_target, 0));
		dp_training_step(m, s, batch, global_batch, sl.in.ptr, sl.target.ptr);
		dp_reduce_loss(m, s);
	} else {
		training_step(m, s, batch, global_batch, sl.in.ptr, sl.target.ptr, true, sl.ev_target);
	}
	TCNNB_CUDA_CHECK(cudaMemcpyAsync(loss_pinned, m.scalars.ptr, sizeof(float), cudaMemcpyDeviceToHost, s));
	TCNNB_CUDA_CHECK(cudaEventRecord(sl.ev_done, s));
	sl.ticket = ticket;
	sl.busy = true;
	++m.next_ticket;
	return ticket;
}

static float host_step_wait(Model& m, uint64_t ticket) {
	Model::HostSlot& sl = m.slots[ticket & 1u];
	if (!sl.busy || sl.ticket != ticket) throw std::runtime_error("training_step_host_wait: ticket " + std::to_string(ticket) + " is not in flight.");
	TCNNB_CUDA_CHECK(cudaEventSynchronize(sl.ev_done));
	sl.busy = false;
	return sl.pinned[sl.pinned_floats - 1];
}

static std::string make_hyperparams(const Model& m) {
	json::Value root = json::Value::object();
	json::Value& enc = root["encoding"];
	if (single_encoding(m.plan, FEAT_GRID)) {
		const GridConfig& g = m.plan.grids[0]->cfg;
		enc["otype"] = json::Value::string("Grid");
		enc["type"] = json::Value::string(g.grid_type == GRID_HASH ? "Hash" : (g.grid_type == GRID_DENSE ? "Dense" : "Tiled"));
		enc["n_levels"] = json::Value::number(g.n_levels);
		enc["n_features_per_level"] = json::Value::number(g.n_features_per_level);
		enc["base_resolution"] = json::Value::number(g.base_resolution);
		enc["log2_hashmap_size"] = json::Value::number(g.log2_hashmap_size);
		enc["per_level_scale"] = json::Value::number(g.per_level_scale);
		enc["interpolation"] = json::Value::string(g.interpolation == INTERP_LINEAR ? "Linear" : (g.interpolation == INTERP_SMOOTHSTEP ? "Smoothstep" : "Nearest"));
		enc["hash"] = json::Value::string("CoherentPrime");
	} else if (single_encoding(m.plan, FEAT_IDENTITY)) {
		enc["otype"] = json::Value::string("Identity");
		enc["scale"] = json::Value::number(m.plan.segs.s[0].scale);
		enc["offset"] = json::Value::number(m.plan.segs.s[0].offset);
	} else {
		enc["otype"] = json::Value::string(m.enc_otype);
		enc["n_nested"] = json::Value::number(m.plan.segs.n);
		enc["n_output_dims"] = json::Value::number(m.plan.width);
	}
	json::Value& net = root["network"];
	net["otype"] = json::Value::string("FullyFusedMLP");
	net["activation"] = json::Value::string(activation_name(m.mlp.activation));
	net["output_activation"] = json::Value::string(activation_name(m.mlp.output_activation));
	net["n_neurons"] = json::Value::number(m.mlp.width);
	net["n_hidden_layers"] = json::Value::number(m.mlp.n_hidden_layers);
	json::Value& loss = root["loss"];
	static const char* loss_names[] = {"L2", "RelativeL2", "L1", "RelativeL1", "Mape", "Smape", "RelativeL2Luminance", "CrossEntropy", "Variance"};
	loss["otype"] = json::Value::string(m.loss_type < sizeof(loss_names) / sizeof(loss_names[0]) ? loss_names[m.loss_type] : m.loss_name.c_str());
	m.opt->write_hyperparams(root["optimizer"]);
	root["n_params"] = json::Value::number((double)m.n_params);
	root["n_mlp_params"] = json::Value::number(m.mlp.n_params);
	root["encoded_width"] = json::Value::number(m.plan.width);
	return json::dump(root);
}

}  // namespace tcnnb

// ==================================================================================================================
// C ABI
// ==================================================================================================================
using namespace tcnnb;

struct tcnnb_model {
	Model impl;
};

extern "C" {

const char* tcnnb_last_error(void) { return g_last_error.c_str(); }
uint32_t tcnnb_batch_size_granularity(void) { return BATCH_GRANULARITY; }
float tcnnb_default_loss_scale(void) { return 128.0f; }
uint32_t tcnnb_abi_version(void) { return 1; }
uint64_t tcnnb_kernel_launch_count(void) { return g_kernel_launches.load(); }

int tcnnb_cuda_device(void) {
	int d = -1;
	if (cudaGetDevice(&d) != cudaSuccess) return -1;
	return d;
}

int tcnnb_set_cuda_device(int device) {
	TCNNB_API_BEGIN
	TCNNB_CUDA_CHECK(cudaSetDevice(device));
	TCNNB_API_END
}

int tcnnb_create_from_config(uint32_t n_input_dims, uint32_t n_output_dims, const char* config_json, uint32_t seed, tcnnb_model** out) {
	TCNNB_API_BEGIN
	if (!out) throw std::runtime_error("tcnnb_create_from_config: out is null");
	*out = nullptr;
	const json::Value cfg = json::parse(config_json ? config_json : "{}");
	std::unique_ptr<tcnnb_model> m{new tcnnb_model{}};
	build_model(m->impl, n_input_dims, n_output_dims, cfg, seed);
	*out = m.release();
	TCNNB_API_END
}

int tcnnb_create_network_trainer(uint32_t n_input_dims, uint32_t n_output_dims, const char* config_json, uint32_t seed, tcnnb_model** out) {
	TCNNB_API_BEGIN
	if (!out) throw std::runtime_error("tcnnb_create_network_trainer: out is null");
	*out = nullptr;
	const json::Value cfg = json::parse(config_json ? config_json : "{}");
	std::unique_ptr<tcnnb_model> m{new tcnnb_model{}};
	build_model(m->impl, n_input_dims, n_output_dims, cfg, seed, /*module_only=*/false, /*half_input=*/true);
	*out = m.release();
	TCNNB_API_END
}

void tcnnb_destroy(tcnnb_model* model) {
#ifdef TCNNB_ENABLE_ABLATION
	if (model && model->impl.dbg_clock.n) {  // dump the phase stamps of the last ws launch
		std::vector<long long> host(model->impl.dbg_clock.n);
		if (cudaMemcpy(host.data(), model->impl.dbg_clock.ptr, host.size() * sizeof(long long), cudaMemcpyDeviceToHost) == cudaSuccess) {
			if (FILE* f = std::fopen(std::getenv("TCNNB_CLOCKS"), "wb")) {
				std::fwrite(host.data(), sizeof(long long), host.size(), f);
				std::fclose(f);
			}
		}
	}
#endif
	delete model;
}

uint64_t tcnnb_n_params(const tcnnb_model* m) { return m->impl.n_params; }
uint64_t tcnnb_n_params_padded(const tcnnb_model* m) { return m->impl.n_params_padded; }
uint64_t tcnnb_n_mlp_params(const tcnnb_model* m) { return m->impl.mlp.n_params; }
uint32_t tcnnb_n_input_dims(const tcnnb_model* m) { return m->impl.n_in; }
uint32_t tcnnb_n_output_dims(const tcnnb_model* m) { return m->impl.n_out; }
uint32_t tcnnb_padded_output_width(const tcnnb_model* m) { return m->impl.mlp.padded_out_width; }
uint32_t tcnnb_encoded_width(const tcnnb_model* m) { return m->impl.plan.width; }
float* tcnnb_params_full_precision(tcnnb_model* m) { return m->impl.params_fp32; }
void* tcnnb_params(tcnnb_model* m) { return m->impl.params_fp16; }
float* tcnnb_mlp_gradient_accumulator(tcnnb_model* m) { return m->impl.dw_accum.ptr; }
void* tcnnb_grid_gradients(tcnnb_model* m) { return m->impl.grads_fp16 + m->impl.mlp.n_params; }

void* tcnnb_param_gradients(tcnnb_model* m) {
	// The MLP part is materialised as fp16 on demand (the fused kernel accumulates it in fp32).
	try {
		// ordered behind the step that produced the gradients: same stream, and the synchronisation is on that stream only
		finalize_mlp_grads(m->impl, m->impl.last_stream, m->impl.grads_fp16);
		TCNNB_CUDA_CHECK(cudaStreamSynchronize(m->impl.last_stream));
	} catch (const std::exception& e) {
		g_last_error = e.what();
		return nullptr;
	}
	return m->impl.grads_fp16;
}

// Level table of the grid when the encoding is one grid; n_levels = 0 for any other encoding, a Composite of one grid included.
int tcnnb_grid_levels(const tcnnb_model* m, uint32_t* n_levels, uint32_t* offsets, float* scales, uint32_t* resolutions) {
	TCNNB_API_BEGIN
	const EncodingPlan& plan = m->impl.plan;
	write_level_table(single_encoding(plan, FEAT_GRID) ? &plan.grids[0]->cfg : nullptr, n_levels, offsets, scales, resolutions);
	TCNNB_API_END
}

const char* tcnnb_hyperparams(tcnnb_model* m) {
	try {
		m->impl.hyperparams_json = make_hyperparams(m->impl);
	} catch (const std::exception& e) {  // nothing may propagate through the C boundary
		g_last_error = e.what();
		m->impl.hyperparams_json = "{}";
	}
	return m->impl.hyperparams_json.c_str();
}

int tcnnb_set_params_full_precision(tcnnb_model* m, const float* params, uint64_t n, int device_ptr) {
	TCNNB_API_BEGIN
	Model& mm = m->impl;
	if (n != mm.n_params) throw std::runtime_error("Can't set fp params because buffer has the wrong size.");  // trainer.h:410-412
	TCNNB_CUDA_CHECK(cudaMemcpy(mm.params_fp32, params, sizeof(float) * n, device_ptr ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
	TCNNB_CUDA_CHECK(launch_cast_params(nullptr, mm.n_params, mm.params_fp32, mm.params_fp16));
	++g_kernel_launches;
	mm.opt->reset_average(mm.params_fp16);
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	TCNNB_API_END
}

// Trainer::params_inference() (trainer.h:401-403): the Ema wrapper's averaged weights when there is one, else the working parameters.
void* tcnnb_params_inference(tcnnb_model* m) { return (void*)m->impl.opt->inference_params(m->impl.params_fp16); }

int tcnnb_set_params(tcnnb_model* m, const void* params_half, uint64_t n, int device_ptr) {
	TCNNB_API_BEGIN
	Model& mm = m->impl;
	if (mm.module_only) throw std::runtime_error("this handle was created with tcnnb_module_create: it owns no parameters.");
	if (n != mm.n_params) throw std::runtime_error("Can't set params because buffer has the wrong size.");  // trainer.h:424-426
	// set_params (trainer.h:423-440): the working-precision parameters are authoritative, fp32 master = (float)fp16
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	TCNNB_CUDA_CHECK(cudaMemcpy(mm.params_fp16, params_half, n * sizeof(__half), device_ptr ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
	half_to_float_kernel<<<(uint32_t)((n + 255) / 256), 256>>>(n, mm.params_fp16, mm.params_fp32);
	++g_kernel_launches;
	mm.opt->reset_average(mm.params_fp16);
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	TCNNB_API_END
}

int tcnnb_optimizer_state(tcnnb_model* m, float** first_moments_dev, float** second_moments_dev, uint32_t** param_steps_dev, uint32_t* current_step, float* base_learning_rate) {
	TCNNB_API_BEGIN
	Model& mm = m->impl;
	Optimizer& opt = *mm.opt;
	if (!opt.allocated()) throw std::runtime_error("this handle was created with tcnnb_module_create: it has no optimizer.");
	if (opt.has_average()) throw std::runtime_error("tcnn_b200: snapshots of the Ema wrapper's state are not built (serialize the parameters only)");
	if (optimizer_state_sharded(mm)) throw std::runtime_error("optimizer state is sharded over the data-parallel ranks: each rank holds the moments of its own slice only");
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	if (param_steps_dev) {
		*param_steps_dev = opt.counters_u32(nullptr);
		TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	}
	if (first_moments_dev) *first_moments_dev = opt.first_moments();
	if (second_moments_dev) *second_moments_dev = opt.second_moments();
	if (current_step) *current_step = opt.step_count();
	if (base_learning_rate) *base_learning_rate = opt.base_learning_rate();
	TCNNB_API_END
}

int tcnnb_set_optimizer_progress(tcnnb_model* m, uint32_t current_step, float base_learning_rate) {
	TCNNB_API_BEGIN
	m->impl.opt->restore_progress(current_step, base_learning_rate);
	TCNNB_API_END
}

// ExponentialDecay's learning-rate factor (exponential_decay.h:136-148 `learning_rate_factor`; 1 without the wrapper). Setting the
// step count recomputes it from the schedule; a snapshot that stores its own factor restores it here afterwards.
float tcnnb_learning_rate_factor(const tcnnb_model* m) { return m->impl.opt->learning_rate_factor(); }

int tcnnb_set_learning_rate_factor(tcnnb_model* m, float factor) {
	TCNNB_API_BEGIN
	m->impl.opt->set_learning_rate_factor(factor);
	TCNNB_API_END
}

int tcnnb_training_step(tcnnb_model* m, tcnnb_stream stream, uint32_t batch_size, const float* input_dev, const float* target_dev, int run_optimizer) {
	TCNNB_API_BEGIN
	training_step(m->impl, (cudaStream_t)stream, batch_size, batch_size, input_dev, target_dev, run_optimizer != 0);
	TCNNB_API_END
}

int tcnnb_training_step_ex(tcnnb_model* m, tcnnb_stream stream, uint32_t batch_size, const float* input_dev, const float* target_dev, const float* data_pdf_dev, int run_optimizer,
                           float* dL_dinput_dev, int use_inference_params, int param_gradients_mode, const void* external_dL_dy_dev) {
	TCNNB_API_BEGIN
	training_step_ex(m->impl, (cudaStream_t)stream, batch_size, input_dev, target_dev, data_pdf_dev, run_optimizer != 0, dL_dinput_dev, use_inference_params != 0, param_gradients_mode,
	                 (const __half*)external_dL_dy_dev);
	TCNNB_API_END
}

int tcnnb_forward(tcnnb_model* m, tcnnb_stream stream, uint32_t batch_size, const float* input_dev, const float* target_dev, const float* data_pdf_dev, int use_inference_params,
                  int prepare_input_gradients, const void* external_dL_dy_dev, void* output_dev, float* loss_values_dev, void* dL_doutput_dev) {
	TCNNB_API_BEGIN
	(void)prepare_input_gradients;  // nothing to prepare: backward recomputes the forward pass, including d(encoded)/d(position)
	trainer_forward(m->impl, (cudaStream_t)stream, batch_size, input_dev, target_dev, data_pdf_dev, use_inference_params != 0, external_dL_dy_dev != nullptr, (__half*)output_dev,
	                loss_values_dev, (__half*)dL_doutput_dev);
	TCNNB_API_END
}

int tcnnb_backward(tcnnb_model* m, tcnnb_stream stream, uint32_t batch_size, const float* input_dev, const void* output_dev, const void* dL_doutput_dev, float* dL_dinput_dev,
                   int use_inference_params, int param_gradients_mode) {
	TCNNB_API_BEGIN
	(void)output_dev;  // the forward pass is recomputed; the saved output is not needed
	if (!dL_doutput_dev) throw std::runtime_error("backward: dL_doutput is null.");
	training_step_ex(m->impl, (cudaStream_t)stream, batch_size, input_dev, nullptr, nullptr, false, dL_dinput_dev, use_inference_params != 0, param_gradients_mode,
	                 (const __half*)dL_doutput_dev);
	TCNNB_API_END
}

int tcnnb_reduce_sum(tcnnb_stream stream, const float* values_dev, uint64_t n_elements, float* sum_out) {
	TCNNB_API_BEGIN
	if (n_elements && !values_dev) throw std::runtime_error("reduce_sum: values are null.");
	cudaStream_t s = (cudaStream_t)stream;
	float* sum_dev = nullptr;
	TCNNB_CUDA_CHECK(cudaMallocAsync(&sum_dev, sizeof(float), s));
	float v = 0;
	cudaError_t e = launch_reduce_sum(s, n_elements, values_dev, sum_dev);
	if (e == cudaSuccess) e = cudaMemcpyAsync(&v, sum_dev, sizeof(float), cudaMemcpyDeviceToHost, s);
	cudaFreeAsync(sum_dev, s);
	TCNNB_CUDA_CHECK(e);
	TCNNB_CUDA_CHECK(cudaStreamSynchronize(s));
	if (n_elements) ++g_kernel_launches;
	if (sum_out) *sum_out = v;
	TCNNB_API_END
}

int tcnnb_training_step_shard(tcnnb_model* m, tcnnb_stream stream, uint32_t shard_batch_size, uint32_t global_batch_size, const float* input_dev, const float* target_dev, int run_optimizer) {
	TCNNB_API_BEGIN
	training_step(m->impl, (cudaStream_t)stream, shard_batch_size, global_batch_size, input_dev, target_dev, run_optimizer != 0);
	TCNNB_API_END
}

int tcnnb_optimizer_step(tcnnb_model* m, tcnnb_stream stream) {
	TCNNB_API_BEGIN
	optimizer_step(m->impl, (cudaStream_t)stream);
	TCNNB_API_END
}

int tcnnb_optimizer_step_ranges(tcnnb_model* m, tcnnb_stream stream, uint32_t n_ranges, const uint64_t* begins, const uint64_t* counts) {
	TCNNB_API_BEGIN
	if (n_ranges > 0 && (!begins || !counts)) throw std::runtime_error("optimizer_step_ranges: null range arrays.");
	optimizer_step(m->impl, (cudaStream_t)stream, n_ranges, begins, counts);
	TCNNB_API_END
}

int tcnnb_loss(tcnnb_model* m, tcnnb_stream stream, float* loss_out) {
	TCNNB_API_BEGIN
	float v = 0;
	TCNNB_CUDA_CHECK(cudaMemcpyAsync(&v, m->impl.scalars.ptr, sizeof(float), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
	TCNNB_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
	if (loss_out) *loss_out = v;
	TCNNB_API_END
}

int tcnnb_inference(tcnnb_model* m, tcnnb_stream stream, uint32_t batch_size, const float* input_dev, float* output_dev) {
	TCNNB_API_BEGIN
	Model& mm = m->impl;
	check_batch(batch_size);
	check_trainer(mm);
	forward(mm, (cudaStream_t)stream, batch_size, input_dev, mm.opt->inference_params(mm.params_fp16), nullptr, output_dev);
	TCNNB_API_END
}

int tcnnb_training_step_host(tcnnb_model* m, uint32_t batch_size, const float* input_host, const float* target_host, float* loss_out) {
	TCNNB_API_BEGIN
	const uint64_t t = host_step_submit(m->impl, batch_size, batch_size, input_host, target_host, false);
	const float loss = host_step_wait(m->impl, t);
	if (loss_out) *loss_out = loss;
	TCNNB_API_END
}

int tcnnb_training_step_host_submit(tcnnb_model* m, uint32_t batch_size, const float* input_host, const float* target_host, uint64_t* ticket_out) {
	TCNNB_API_BEGIN
	const uint64_t t = host_step_submit(m->impl, batch_size, batch_size, input_host, target_host, false);
	if (ticket_out) *ticket_out = t;
	TCNNB_API_END
}

int tcnnb_dp_training_step_host_submit(tcnnb_model* m, uint32_t shard_batch_size, uint32_t global_batch_size, const float* input_host, const float* target_host, uint64_t* ticket_out) {
	TCNNB_API_BEGIN
	if (!m->impl.dp) throw std::runtime_error("dp_training_step_host_submit: call tcnnb_dp_init first.");
	const uint64_t t = host_step_submit(m->impl, shard_batch_size, global_batch_size, input_host, target_host, true);
	if (ticket_out) *ticket_out = t;
	TCNNB_API_END
}

int tcnnb_training_step_host_wait(tcnnb_model* m, uint64_t ticket, float* loss_out) {
	TCNNB_API_BEGIN
	const float loss = host_step_wait(m->impl, ticket);
	if (loss_out) *loss_out = loss;
	TCNNB_API_END
}

int tcnnb_inference_host(tcnnb_model* m, uint32_t batch_size, const float* input_host, float* output_host) {
	TCNNB_API_BEGIN
	Model& mm = m->impl;
	check_batch(batch_size);
	check_trainer(mm);
	check_float_input(mm, "tcnnb_inference_host");
	ensure_staging(mm, batch_size);
	cudaStream_t s = mm.own_stream;
	const size_t n_x = (size_t)batch_size * mm.n_in, n_y = (size_t)batch_size * mm.n_out;
	std::memcpy(mm.pinned, input_host, n_x * sizeof(float));
	TCNNB_CUDA_CHECK(cudaMemcpyAsync(mm.stage_in.ptr, mm.pinned, n_x * sizeof(float), cudaMemcpyHostToDevice, s));
	forward(mm, s, batch_size, mm.stage_in.ptr, mm.opt->inference_params(mm.params_fp16), nullptr, mm.stage_out.ptr);
	TCNNB_CUDA_CHECK(cudaMemcpyAsync(mm.pinned + n_x, mm.stage_out.ptr, n_y * sizeof(float), cudaMemcpyDeviceToHost, s));
	TCNNB_CUDA_CHECK(cudaStreamSynchronize(s));
	std::memcpy(output_host, mm.pinned + n_x, n_y * sizeof(float));
	TCNNB_API_END
}

// Snapshot layout: [u64 n_params][u32 with_optimizer][u32 adam_step][fp16 params][fp32 m][fp32 v][u32 steps]
uint64_t tcnnb_serialize_size(const tcnnb_model* m, int with_optimizer) {
	const uint64_t n = m->impl.n_params;
	return 16 + n * 2 + (with_optimizer ? n * 12 : 0);
}

int tcnnb_serialize(tcnnb_model* m, void* dst_host, uint64_t size, int with_optimizer) {
	TCNNB_API_BEGIN
	Model& mm = m->impl;
	if (size < tcnnb_serialize_size(m, with_optimizer)) throw std::runtime_error("tcnnb_serialize: destination too small");
	if (with_optimizer && mm.opt->has_average()) throw std::runtime_error("tcnn_b200: snapshots of the Ema wrapper's state are not built (serialize with_optimizer = 0)");
	if (with_optimizer && optimizer_state_sharded(mm)) {
		// moments / step counters are current on the owner of a slice only (ZeRO-1): a snapshot of one rank would silently hold stale state
		throw std::runtime_error("tcnnb_serialize: optimizer state is sharded over the data-parallel ranks; serialize with_optimizer = 0 (after tcnnb_dp_sync_full_precision) or from a single-GPU trainer");
	}
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	char* p = (char*)dst_host;
	const uint64_t n = mm.n_params;
	const uint32_t wo = with_optimizer ? 1 : 0, st = mm.opt->step_count();
	std::memcpy(p, &n, 8);
	std::memcpy(p + 8, &wo, 4);
	std::memcpy(p + 12, &st, 4);
	p += 16;
	TCNNB_CUDA_CHECK(cudaMemcpy(p, mm.params_fp16, n * 2, cudaMemcpyDeviceToHost));
	p += n * 2;
	if (with_optimizer) {
		TCNNB_CUDA_CHECK(cudaMemcpy(p, mm.opt->first_moments(), n * 4, cudaMemcpyDeviceToHost));
		p += n * 4;
		TCNNB_CUDA_CHECK(cudaMemcpy(p, mm.opt->second_moments(), n * 4, cudaMemcpyDeviceToHost));
		p += n * 4;
		TCNNB_CUDA_CHECK(cudaMemcpy(p, mm.opt->counters_u32(nullptr), n * 4, cudaMemcpyDeviceToHost));  // uint32 on disk whatever the counters' width
	}
	TCNNB_API_END
}

int tcnnb_deserialize(tcnnb_model* m, const void* src_host, uint64_t size) {
	TCNNB_API_BEGIN
	Model& mm = m->impl;
	if (size < 16) throw std::runtime_error("tcnnb_deserialize: truncated snapshot");
	const char* p = (const char*)src_host;
	uint64_t n;
	uint32_t wo, st;
	std::memcpy(&n, p, 8);
	std::memcpy(&wo, p + 8, 4);
	std::memcpy(&st, p + 12, 4);
	if (n != mm.n_params) throw std::runtime_error("Can't set params because buffer has the wrong size.");  // trainer.h:424-426
	if (size < 16 + n * 2 + (wo ? n * 12 : 0)) throw std::runtime_error("tcnnb_deserialize: truncated snapshot");
	p += 16;
	// set_params (trainer.h:423-440): fp16 params are authoritative, fp32 master = (float)fp16
	TCNNB_CUDA_CHECK(cudaMemcpy(mm.params_fp16, p, n * 2, cudaMemcpyHostToDevice));
	half_to_float_kernel<<<(uint32_t)((n + 255) / 256), 256>>>(n, mm.params_fp16, mm.params_fp32);
	++g_kernel_launches;
	p += n * 2;
	if (wo) {
		TCNNB_CUDA_CHECK(cudaMemcpy(mm.opt->first_moments(), p, n * 4, cudaMemcpyHostToDevice));
		p += n * 4;
		TCNNB_CUDA_CHECK(cudaMemcpy(mm.opt->second_moments(), p, n * 4, cudaMemcpyHostToDevice));
		p += n * 4;
		mm.opt->load_counters_u32((const uint32_t*)p);
		mm.opt->restore_progress(st, mm.opt->base_learning_rate());
	}
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	TCNNB_API_END
}

int tcnnb_dp_unique_id(void* out_id, uint64_t n_bytes) {
	TCNNB_API_BEGIN
	if (!out_id || n_bytes < sizeof(ncclUniqueId)) throw std::runtime_error("dp_unique_id: need a 128-byte buffer.");
	ncclUniqueId id;
	TCNNB_NCCL_CHECK(nccl_api().GetUniqueId(&id));
	std::memcpy(out_id, &id, sizeof(id));
	TCNNB_API_END
}

int tcnnb_dp_init(tcnnb_model* m, const void* id_grads, const void* id_params, int world_size, int rank, int shard_optimizer) {
	TCNNB_API_BEGIN
	Model& mm = m->impl;
	if (world_size < 1 || rank < 0 || rank >= world_size) throw std::runtime_error("dp_init: bad world size / rank.");
	check_float_input(mm, "data-parallel training");
	if (mm.opt->has_average() && world_size > 1) throw std::runtime_error("tcnn_b200: the Ema optimizer wrapper is not built for the data-parallel engines");
	auto d = std::make_unique<DpState>();
	d->world = world_size;
	d->rank = rank;
	// slices must be 16-byte aligned and the network weights must sit inside slice 0, else fall back to replicated Adam
	d->shard_optimizer = shard_optimizer != 0 && mm.n_params_padded % (8 * (size_t)world_size) == 0 && mm.n_params_padded / (size_t)world_size >= mm.mlp.n_params;
	if (world_size > 1) {
		if (!id_grads || !id_params) throw std::runtime_error("dp_init: null NCCL ids.");
		ncclUniqueId a, b;
		std::memcpy(&a, id_grads, sizeof(a));
		std::memcpy(&b, id_params, sizeof(b));
		TCNNB_NCCL_CHECK(nccl_api().CommInitRank(&d->comm_grads, world_size, a, rank));
		TCNNB_NCCL_CHECK(nccl_api().CommInitRank(&d->comm_params, world_size, b, rank));
	}
	TCNNB_CUDA_CHECK(cudaStreamCreateWithFlags(&d->gather_stream, cudaStreamNonBlocking));
	TCNNB_CUDA_CHECK(cudaEventCreateWithFlags(&d->ev_updated, cudaEventDisableTiming));
	TCNNB_CUDA_CHECK(cudaEventCreateWithFlags(&d->ev_gathered, cudaEventDisableTiming));
	mm.dp = std::move(d);
	TCNNB_API_END
}

int tcnnb_dp_attach_symmetric(tcnnb_model* m, const uint64_t* peer_bases, uint64_t multicast_base, uint64_t n_bytes) {
	TCNNB_API_BEGIN
	Model& mm = m->impl;
	if (!mm.dp || mm.dp->world < 2) throw std::runtime_error("dp_attach_symmetric: call tcnnb_dp_init with world_size > 1 first.");
	DpState& d = *mm.dp;
	if (!d.shard_optimizer) throw std::runtime_error("dp_attach_symmetric: needs the sharded optimizer (aligned slices).");
	if (d.world > (int)DP_MAX_RANKS) throw std::runtime_error("dp_attach_symmetric: at most 8 ranks (one NVSwitch domain).");
	if (!peer_bases) throw std::runtime_error("dp_attach_symmetric: peer_bases is null.");
	const size_t np = mm.n_params_padded;
	const size_t need = np * 2 * sizeof(__half) + 256;
	if (n_bytes < need) throw std::runtime_error("dp_attach_symmetric: the symmetric buffer must hold " + std::to_string(need) + " bytes.");
	if (mm.n_params % 8 != 0 || mm.mlp.n_params % 8 != 0 || (np / (size_t)d.world) % 8 != 0) throw std::runtime_error("dp_attach_symmetric: parameter counts must be multiples of 8.");
	DpPeers& p = d.peers;
	p.world = (uint32_t)d.world;
	p.rank = (uint32_t)d.rank;
	for (int r = 0; r < d.world; ++r) {
		if (!peer_bases[r] || peer_bases[r] % 16 != 0) throw std::runtime_error("dp_attach_symmetric: bad peer pointer.");
		char* base = (char*)(uintptr_t)peer_bases[r];
		p.params[r] = (__half*)base;
		p.grads[r] = (__half*)base + np;
		p.flags[r] = (uint32_t*)(base + np * 2 * sizeof(__half));
	}
	p.params_mc = multicast_base ? (__half*)(uintptr_t)multicast_base : nullptr;
	p.grads_mc = multicast_base ? (__half*)(uintptr_t)multicast_base + np : nullptr;
	// move the working parameters into the symmetric region (local copy), clear gradients and flags; the caller synchronises all
	// ranks (host barrier) before the first step
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	TCNNB_CUDA_CHECK(cudaMemcpy(p.params[d.rank], mm.params_fp16, np * sizeof(__half), cudaMemcpyDeviceToDevice));
	TCNNB_CUDA_CHECK(cudaMemset(p.grads[d.rank], 0, np * sizeof(__half) + 256));
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	mm.params_fp16 = p.params[d.rank];
	mm.grads_fp16 = p.grads[d.rank];
	d.epoch = 0;
	d.fused = true;
	TCNNB_API_END
}

int tcnnb_dp_engine(const tcnnb_model* m) {
	const DpState* d = m->impl.dp.get();
	if (!d || d->world < 2) return 0;
	if (d->fused) return d->peers.params_mc ? 3 : 2;
	return 1;
}

int tcnnb_dp_shards_optimizer(const tcnnb_model* m) { return optimizer_state_sharded(m->impl) ? 1 : 0; }

int tcnnb_dp_training_step(tcnnb_model* m, tcnnb_stream stream, uint32_t shard_batch_size, uint32_t global_batch_size, const float* input_dev, const float* target_dev) {
	TCNNB_API_BEGIN
	dp_training_step(m->impl, (cudaStream_t)stream, shard_batch_size, global_batch_size, input_dev, target_dev);
	TCNNB_API_END
}

int tcnnb_dp_sync_full_precision(tcnnb_model* m, tcnnb_stream stream) {
	TCNNB_API_BEGIN
	Model& mm = m->impl;
	if (mm.dp && mm.dp->world > 1 && mm.dp->shard_optimizer && !mm.dp->masters_synced) {
		const size_t chunk = mm.n_params_padded / (size_t)mm.dp->world, lo = chunk * (size_t)mm.dp->rank;
		mm.wait_pending((cudaStream_t)stream);
		TCNNB_NCCL_CHECK(nccl_api().AllGather(mm.params_fp32 + lo, mm.params_fp32, chunk, ncclFloat, mm.dp->comm_grads, (cudaStream_t)stream));
		mm.dp->masters_synced = true;
	}
	TCNNB_API_END
}

int tcnnb_dp_finish(tcnnb_model* m) {
	TCNNB_API_BEGIN
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	m->impl.pending_params_event = nullptr;
	m->impl.dp.reset();
	TCNNB_API_END
}

int tcnnb_generate_random_uniform(tcnnb_stream stream, uint64_t rng_state, uint64_t rng_inc, uint64_t n_elements, float* out_dev, float lower, float upper) {
	TCNNB_API_BEGIN
	if (n_elements && !out_dev) throw std::runtime_error("generate_random_uniform: out is null.");
	Pcg32 rng;
	rng.state = rng_state;
	rng.inc = rng_inc;
	TCNNB_CUDA_CHECK(launch_random_uniform((cudaStream_t)stream, rng, n_elements, out_dev, lower, upper));
	++g_kernel_launches;
	TCNNB_API_END
}

int tcnnb_generate_random_uniform_half(tcnnb_stream stream, uint64_t rng_state, uint64_t rng_inc, uint64_t n_elements, void* out_dev, float lower, float upper) {
	TCNNB_API_BEGIN
	if (n_elements && !out_dev) throw std::runtime_error("generate_random_uniform: out is null.");
	Pcg32 rng;
	rng.state = rng_state;
	rng.inc = rng_inc;
	TCNNB_CUDA_CHECK(launch_random_uniform_half((cudaStream_t)stream, rng, n_elements, (__half*)out_dev, __float2half(lower), __float2half(upper)));
	++g_kernel_launches;
	TCNNB_API_END
}

int tcnnb_transpose(tcnnb_stream stream, uint32_t rows, uint32_t cols, uint32_t element_bytes, const void* src_dev, void* dst_dev) {
	TCNNB_API_BEGIN
	if (element_bytes != 2 && element_bytes != 4) throw std::runtime_error("transpose: element_bytes must be 2 or 4.");
	if (rows == 0 || cols == 0) return 0;
	if (!src_dev || !dst_dev) throw std::runtime_error("transpose: src / dst is null.");
	if (src_dev == dst_dev) throw std::runtime_error("transpose: src and dst must not be the same array.");
	TCNNB_CUDA_CHECK(launch_transpose((cudaStream_t)stream, rows, cols, element_bytes, src_dev, dst_dev));
	++g_kernel_launches;
	TCNNB_API_END
}

// ---- module tier ------------------------------------------------------------------------------------------------------------
int tcnnb_module_create(uint32_t n_input_dims, uint32_t n_output_dims, const char* encoding_json, const char* network_json, tcnnb_model** out) {
	TCNNB_API_BEGIN
	if (!out) throw std::runtime_error("tcnnb_module_create: out is null");
	*out = nullptr;
	const std::string cfg = std::string("{\"encoding\": ") + (encoding_json ? encoding_json : "{}") + ", \"network\": " + (network_json ? network_json : "{}") + "}";
	auto m = std::make_unique<tcnnb_model>();
	build_model(m->impl, n_input_dims, n_output_dims, json::parse(cfg), 1337, /*module_only=*/true);
	*out = m.release();
	TCNNB_API_END
}

int tcnnb_module_initialize_params(tcnnb_model* m, uint64_t seed, float* params_full_precision_dev, float scale) {
	TCNNB_API_BEGIN
	if (!params_full_precision_dev) throw std::runtime_error("module: params_full_precision is null.");
	HostPcg32 rng{seed};  // cpp_api.cu:140-143: pcg32 rng{seed}
	init_params(m->impl, rng, params_full_precision_dev, scale);
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	TCNNB_API_END
}

int tcnnb_module_inference(tcnnb_model* m, tcnnb_stream stream, uint32_t n_elements, const float* input_dev, void* output_dev, const void* params_dev) {
	TCNNB_API_BEGIN
	check_batch(n_elements);
	check_module_ptr(params_dev, "params");
	check_module_ptr(output_dev, "output");
	forward(m->impl, (cudaStream_t)stream, n_elements, input_dev, (const __half*)params_dev, (__half*)output_dev, nullptr);
	TCNNB_API_END
}

int tcnnb_module_forward(tcnnb_model* m, tcnnb_stream stream, uint32_t n_elements, const float* input_dev, void* output_dev, const void* params_dev, int prepare_input_gradients) {
	(void)prepare_input_gradients;  // nothing to prepare: backward recomputes the forward pass, including d(encoded)/d(position)
	return tcnnb_module_inference(m, stream, n_elements, input_dev, output_dev, params_dev);
}

int tcnnb_module_backward(tcnnb_model* m, tcnnb_stream stream, uint32_t n_elements, float* dL_dinput_dev, const void* dL_doutput_dev, void* dL_dparams_dev, const float* input_dev,
                          const void* output_dev, const void* params_dev) {
	TCNNB_API_BEGIN
	(void)output_dev;  // the forward pass is recomputed; the saved output is not needed
	module_backward(m->impl, (cudaStream_t)stream, n_elements, dL_dinput_dev, dL_doutput_dev, dL_dparams_dev, input_dev, params_dev);
	TCNNB_API_END
}

int tcnnb_wait_before_compute(tcnnb_model* m, void* cuda_event) {
	TCNNB_API_BEGIN
	m->impl.pending_params_event = (cudaEvent_t)cuda_event;
	TCNNB_API_END
}

int tcnnb_set_profiling(tcnnb_model* m, int enable) {
	TCNNB_API_BEGIN
	Model& mm = m->impl;
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	for (auto e : mm.prof_events) cudaEventDestroy(e);
	mm.prof_events.clear();
	mm.profiling = enable != 0;
	TCNNB_API_END
}

int tcnnb_read_profile(tcnnb_model* m, float* fused_ms_total, float* optimizer_ms_total, float* binning_ms_total, uint32_t* n_steps) {
	TCNNB_API_BEGIN
	Model& mm = m->impl;
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	float fused = 0, opt = 0, bin = 0;
	const size_t n = mm.prof_events.size() / 4;
	for (size_t i = 0; i < n; ++i) {
		float a = 0, b = 0, c = 0;
		TCNNB_CUDA_CHECK(cudaEventElapsedTime(&c, mm.prof_events[4 * i], mm.prof_events[4 * i + 1]));
		TCNNB_CUDA_CHECK(cudaEventElapsedTime(&a, mm.prof_events[4 * i + 1], mm.prof_events[4 * i + 2]));
		TCNNB_CUDA_CHECK(cudaEventElapsedTime(&b, mm.prof_events[4 * i + 2], mm.prof_events[4 * i + 3]));
		fused += a;
		opt += b;
		bin += c;
	}
	if (binning_ms_total) *binning_ms_total = bin;
	if (fused_ms_total) *fused_ms_total = fused;
	if (optimizer_ms_total) *optimizer_ms_total = opt;
	if (n_steps) *n_steps = (uint32_t)n;
	TCNNB_API_END
}

int tcnnb_debug_set(tcnnb_model* m, const char* key, int value) {
	TCNNB_API_BEGIN
	const std::string k = key ? key : "";
	if (k == "binning") m->impl.binning = value != 0;
	else if (k == "adam_steps32") {  // 32-bit step counters although 16-bit ones give the same updates (tests compare the two layouts)
		if (!m->impl.opt->allocated()) throw std::runtime_error("tcnnb_debug_set(adam_steps32): this handle has no optimizer.");
		m->impl.opt->set_counter_width(value != 0);
	}
	else if (k == "general") {
		// the stand-alone kernels have their own limits (e.g. dL/d(encoded) wider than the layers): only switch when they cover the configuration
		if (value && !m->impl.general) {
			if (const char* why_not = general_path_unsupported(m->impl)) throw std::runtime_error(std::string("tcnnb_debug_set(general): ") + why_not);
		}
		m->impl.force_general = value != 0;
	}
	else throw std::runtime_error("tcnnb_debug_set: unknown key '" + k + "'");
	TCNNB_API_END
}

int tcnnb_set_debug_taps(tcnnb_model* m, const tcnnb_debug_taps* taps) {
	TCNNB_API_BEGIN
	if (taps) m->impl.taps = *taps;
	else m->impl.taps = tcnnb_debug_taps{};
	TCNNB_API_END
}

}  // extern "C"
