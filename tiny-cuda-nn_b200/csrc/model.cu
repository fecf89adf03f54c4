// model.cu -- host side of the hot path and the C ABI declared in include/tcnn_b200.h.
//
// Mirrors, for the HashGrid + FullyFusedMLP path only, what the reference spreads over
//   config.h:53-63              create_from_config
//   src/encoding.cu:132-150     create_encoding ("otype" dispatch, case-insensitive)  + grid.h:1726-1851 (grid JSON keys)
//   src/network.cu:51-141       select_network / create_network
//   src/loss.cu:82-90           create_loss
//   src/optimizer.cu:50-80      create_optimizer + optimizers/adam.h:221-303 (Adam JSON keys)
//   trainer.h:51-87,254-378     Trainer ctor / initialize_params / training_step / loss
//   network_with_input_encoding.h:115-150  parameter layout [MLP | grid]
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

#include <dlfcn.h>
#include <nccl.h>  // types and prototypes only: libnccl is resolved at run time (dlopen), single-GPU users never need it

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <memory>
#include <random>
#include <stdexcept>
#include <string>
#include <vector>

namespace tcnnb {

std::atomic<uint64_t> g_kernel_launches{0};
thread_local std::string g_last_error;

struct MlpConfig {
	std::string otype = "FullyFusedMLP";
	uint32_t in_width = 0;
	uint32_t width = 128;
	uint32_t n_hidden_layers = 5;
	uint32_t out_width = 0;
	uint32_t padded_out_width = 0;
	uint32_t activation = ACT_RELU;
	uint32_t output_activation = ACT_NONE;
	uint32_t n_params = 0;
};

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
	GridConfig grid;
	MlpConfig mlp;
	uint32_t loss_type = LOSS_RELATIVE_L2;
	std::string loss_name = "RelativeL2";
	AdamParams adam;
	uint32_t adam_step_count = 0;
	struct {  // ExponentialDecay wrapper (optimizers/exponential_decay.h)
		bool enabled = false;
		float base = 0.1f, factor = 1.0f;
		uint32_t interval = 10000, start = 10000, end = 10000000;
	} lr_decay;
	struct {  // Ema wrapper (optimizers/ema.h:46-200): exponential moving average of the working weights, used by inference
		bool enabled = false, full_precision = false;
		float decay = 0.99f;
	} ema;
	DeviceBuffer<__half> ema_fp16;  // Trainer::params_inference() (trainer.h:401-403, 497-502)
	DeviceBuffer<float> ema_tmp;
	const __half* inference_params() const { return ema.enabled ? ema_fp16.ptr : params_fp16; }
	float loss_scale = 128.0f;  // default_loss_scale<__half>() (common.h:243)
	int device = 0;
	int n_sms = 132;

	size_t n_params = 0;
	// trainer.h:489-503: one allocation [fp32 master | fp16 params | fp16 gradients]
	DeviceBuffer<char> params_buffer;
	size_t n_params_padded = 0;
	bool module_only = false;  // tcnnb_module: no trainer-owned parameters / optimizer state
	float* params_fp32 = nullptr;
	__half* params_fp16 = nullptr;
	__half* grads_fp16 = nullptr;
	DeviceBuffer<float> first_moments, second_moments;
	DeviceBuffer<uint32_t> param_steps;
	DeviceBuffer<float> dw_accum;   // fp32 MLP weight-gradient accumulator
	DeviceBuffer<float> scalars;    // [0] = loss sum
	DeviceBuffer<long long> dbg_clock;  // TCNNB_CLOCKS=<file> in ablation builds: phase stamps of the last ws launch
	DeviceBuffer<float> level_scales_dev;
	bool enc_identity = false;              // "Identity" encoding instead of a grid (no encoding parameters)
	float identity_scale = 1.0f, identity_offset = 0.0f;
	DeviceBuffer<LevelInfo> levels_dev;     // per-level descriptors for the stand-alone grid kernels (module tier: dL/d(input))
	DeviceBuffer<__half> denc_scratch;      // module tier: dL/d(encoded) rows [n][64] handed from the fused kernel to the input-gradient kernel
	DeviceBuffer<__half> grads_scratch;     // module tier: gradient array when the caller wants dL/d(input) only
	bool mlp_grads_in_accum = false;
	// General (unfused) path: configurations the fused kernel does not cover -- 128 neurons, n_features_per_level in {1, 4, 8}, 4-D
	// inputs, Nearest interpolation, wider encodings / outputs -- run as encoding kernel -> stand-alone MLP kernels -> encoding backward
	// kernel, with the activations of one batch in HBM (the reference's own structure, object.h / network_with_input_encoding.h).
	bool general = false;
	bool force_general = false;  // tcnnb_debug_set("general", 1): run the general path although the fused kernel covers the configuration
	bool use_general() const { return general || force_general; }
	bool plan_only = false;      // an encoding other than one grid / Identity (Composite, Frequency, OneBlob, ...): no fused kernel at all
	EncodingPlan plan;           // segment table of the encoding (general path)
	std::string general_reason;  // which limit of the fused kernel sent this configuration here (hyperparams / diagnostics)
	DeviceBuffer<__half> g_enc, g_hidden, g_out, g_dy, g_grad_hidden, g_denc, g_dy_act;
	DeviceBuffer<float> g_grid_tmp;  // n_features_per_level == 1: fp32 scatter target (grid.h:858-894)
	DeviceBuffer<__half> g_replicas; // private copies of the coarse levels' gradients (grid_kernels.h plan_grid_scatter)
	int grid_replicas_override = -1; // tcnnb_debug_set("grid_replicas", n): experiments (0 / 1 = off)

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
	std::vector<cudaEvent_t> prof_events;  // quadruples: step start, after binning, after fused kernel, after Adam

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

	GridMeta grid_meta() const {
		GridMeta m{};
		m.n_levels = grid.n_levels;
		m.n_features = grid.n_levels * grid.n_features_per_level;
		m.padded_width = grid.padded_width;
		m.interpolation = grid.interpolation;
		for (uint32_t l = 0; l < grid.n_levels; ++l) m.levels[l] = make_level_info(grid, l);
		return m;
	}
};

// initialize_params(rnd, params_full_precision, scale) of NetworkWithInputEncoding (network_with_input_encoding.h:124-130):
// network weights first, then the grid table, one pcg32 stream. `dst` is a DEVICE fp32 array of n_params elements.
static void init_params(Model& m, HostPcg32& rng, float* dst, float scale) {
	const MlpConfig& mlp = m.mlp;
	// MLP: xavier uniform on the host, sequential draws (fully_fused_mlp.cu:868-892, gpu_matrix.h:292-306)
	{
		std::vector<float> w(mlp.n_params);
		std::vector<std::pair<uint32_t, uint32_t>> mats;
		mats.emplace_back(mlp.width, mlp.in_width);
		for (uint32_t i = 0; i + 1 < mlp.n_hidden_layers; ++i) mats.emplace_back(mlp.width, mlp.width);
		mats.emplace_back(mlp.padded_out_width, mlp.width);
		size_t pos = 0;
		for (auto& rc : mats) {
			const float bound = scale * std::sqrt(6.0f / (float)(rc.second + rc.first));
			for (size_t i = 0; i < (size_t)rc.first * rc.second; ++i) w[pos++] = rng.next_float() * 2.0f * bound - bound;
		}
		TCNNB_CUDA_CHECK(cudaMemcpy(dst, w.data(), sizeof(float) * w.size(), cudaMemcpyHostToDevice));
	}
	// grid: U(-1e-4, 1e-4) * scale generated on the device with the jump-ahead pattern (grid.h:1076-1079, random.h:56-69)
	if (m.plan_only) {  // nested encodings draw one after the other from the same stream (composite.h initialize_params)
		for (auto& g : m.plan.grids) {
			TCNNB_CUDA_CHECK(launch_random_uniform(nullptr, rng.device(), g->cfg.n_params, dst + mlp.n_params + g->param_offset, -1e-4f * scale, 1e-4f * scale));
			++g_kernel_launches;
			rng.advance(g->cfg.n_params);
		}
	} else if (m.grid.n_params) {
		TCNNB_CUDA_CHECK(launch_random_uniform(nullptr, rng.device(), m.grid.n_params, dst + mlp.n_params, -1e-4f * scale, 1e-4f * scale));
		++g_kernel_launches;
		rng.advance(m.grid.n_params);
	}
}

static void build_model(Model& m, uint32_t n_in, uint32_t n_out, const json::Value& cfg, uint32_t seed, bool module_only = false) {
	TCNNB_CUDA_CHECK(cudaGetDevice(&m.device));
	cudaDeviceProp prop;
	TCNNB_CUDA_CHECK(cudaGetDeviceProperties(&prop, m.device));
	if (prop.major != 9) {
		throw std::runtime_error("tcnn_b200 requires an sm_90-class GPU (H100); found compute capability " + std::to_string(prop.major) + "." + std::to_string(prop.minor));
	}
	m.n_sms = prop.multiProcessorCount;
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
	const json::Value* opt_ptr = &cfg.sub("optimizer");
	std::string opt_name = opt_ptr->value("otype", "Adam");
	// wrappers around the nested optimizer, in any order: ExponentialDecay (a learning-rate schedule) and Ema (averaged inference weights)
	while (ieq(opt_name, "ExponentialDecay") || ieq(opt_name, "Ema")) {
		if (ieq(opt_name, "ExponentialDecay")) {
			// optimizers/exponential_decay.h:46-160: from step decay_start on, every decay_interval steps (until decay_end) the learning
			// rate is multiplied by decay_base. Host-side bookkeeping only.
			if (m.lr_decay.enabled) throw std::runtime_error("tcnn_b200: one ExponentialDecay wrapper per optimizer");
			m.lr_decay.enabled = true;
			m.lr_decay.base = (float)opt_ptr->value("decay_base", 0.1);
			m.lr_decay.interval = (uint32_t)opt_ptr->value("decay_interval", 10000.0);
			m.lr_decay.start = (uint32_t)opt_ptr->value("decay_start", 10000.0);
			m.lr_decay.end = (uint32_t)opt_ptr->value("decay_end", 10000000.0);
			if (m.lr_decay.interval == 0) throw std::runtime_error("ExponentialDecay: decay_interval must be positive.");
		} else {
			// optimizers/ema.h:46-200: after every step of the nested optimizer, ema = (ema * decay * (1 - decay^(t-1)) + w * (1 - decay)) /
			// (1 - decay^t) on the working-precision weights; network->inference() reads the average (Trainer::params_inference).
			if (m.ema.enabled) throw std::runtime_error("tcnn_b200: one Ema wrapper per optimizer");
			m.ema.enabled = true;
			m.ema.decay = (float)opt_ptr->value("decay", 0.99);
			m.ema.full_precision = opt_ptr->value("full_precision", false);
		}
		opt_ptr = &opt_ptr->sub("nested");
		opt_name = opt_ptr->value("otype", "Adam");
	}
	const json::Value& opt = *opt_ptr;
	if (!ieq(opt_name, "Adam")) {
		throw std::runtime_error("Optimizer '" + opt_name + "' is outside the tcnn_b200 hot path (Adam, optionally inside ExponentialDecay and / or Ema, is built)");
	}
	AdamParams& a = m.adam;
	a.beta1 = (float)opt.value("beta1", (double)a.beta1);
	a.beta2 = (float)opt.value("beta2", (double)a.beta2);
	a.epsilon = (float)opt.value("epsilon", (double)a.epsilon);
	a.learning_rate = (float)opt.value("learning_rate", (double)a.learning_rate);
	a.l2_reg = (float)opt.value("l2_reg", (double)a.l2_reg);
	a.adabound = opt.value("adabound", false);
	a.relative_decay = (float)opt.value("relative_decay", (double)a.relative_decay);
	a.absolute_decay = (float)opt.value("absolute_decay", (double)a.absolute_decay);
	a.clipping_magnitude = (float)opt.value("clipping_magnitude", (double)a.clipping_magnitude);
	a.gradient_clipping_magnitude = (float)opt.value("gradient_clipping_magnitude", (double)a.gradient_clipping_magnitude);
	a.non_matrix_learning_rate_factor = (float)opt.value("non_matrix_learning_rate_factor", (double)a.non_matrix_learning_rate_factor);
	a.non_matrix_l2_reg = (float)opt.value("non_matrix_l2_reg", (double)a.non_matrix_l2_reg);
	a.optimize_matrix_params = opt.value("optimize_matrix_params", true);
	a.optimize_non_matrix_params = opt.value("optimize_non_matrix_params", true);
	a.skip_zero_grad_non_matrix_params = opt.value("skip_zero_grad_non_matrix_params", true);

	// ---- network (src/network.cu:51-141) and encoding alignment (network_with_input_encoding.h:47)
	const json::Value& net = cfg.sub("network");
	MlpConfig& mlp = m.mlp;
	mlp.otype = net.value("otype", "MLP");
	const bool fully_fused = ieq(mlp.otype, "FullyFusedMLP") || ieq(mlp.otype, "MegakernelMLP");
	const bool cutlass = ieq(mlp.otype, "MLP") || ieq(mlp.otype, "CutlassMLP");
	if (!fully_fused && !cutlass) throw std::runtime_error("Invalid network type: " + mlp.otype);
	mlp.width = (uint32_t)net.value("n_neurons", 128.0);
	mlp.n_hidden_layers = (uint32_t)net.value("n_hidden_layers", 5.0);
	mlp.activation = parse_activation(net.value("activation", "ReLU"));
	mlp.output_activation = parse_activation(net.value("output_activation", "None"));
	if (fully_fused && !(mlp.width == 16 || mlp.width == 32 || mlp.width == 64 || mlp.width == 128)) {
		throw std::runtime_error("FullyFusedMLP only supports 16, 32, 64, and 128 neurons, but got " + std::to_string(mlp.width) + ". Use CutlassMLP instead if this is a requirement.");
	}
	if (mlp.n_hidden_layers < 1) throw std::runtime_error("FullyFusedMLP requires at least 1 hidden layer (3 layers in total).");

	const uint32_t alignment = 16;  // FullyFusedMLP / CutlassMLP REQUIRED_ALIGNMENT (src/network.cu:79-98)
	const json::Value& enc_cfg = cfg.sub("encoding");
	if (ieq(enc_cfg.value("otype", "OneBlob"), "Identity")) {
		// Identity encoding (encodings/identity.h:46-67, src/encoding.cu:77-79): feature j = x_j * scale + offset, the features that pad
		// the width up to the network's alignment are ONE. No parameters: the memory warps of the fused kernel write the tile rows
		// directly (BASELINE.json configs[0]: CutlassMLP / FullyFusedMLP 64 x 2 behind Identity).
		m.enc_identity = true;
		m.identity_scale = (float)enc_cfg.value("scale", 1.0);
		m.identity_offset = (float)enc_cfg.value("offset", 0.0);
		m.grid = GridConfig{};
		m.grid.otype = "Identity";
		m.grid.n_pos_dims = n_in;
		m.grid.n_levels = 0;
		m.grid.n_params = 0;
		m.grid.offsets.assign(1, 0u);
		m.grid.padded_width = next_multiple(n_in, alignment);
	} else if (plan_detail::is_grid_otype(to_lower(enc_cfg.value("otype", "OneBlob")))) {
		m.grid = parse_grid(n_in, enc_cfg);
		m.grid.padded_width = next_multiple(m.grid.n_levels * m.grid.n_features_per_level, alignment);
	} else {
		// Composite / Frequency / TriangleWave / OneBlob / SphericalHarmonics (src/encoding.cu:60-120): stand-alone encoding kernels in
		// front of the stand-alone network kernels. `grid` only carries the totals the rest of the model needs.
		m.plan_only = true;
		m.level_scales_dev.resize(128);
		build_encoding_plan(m.plan, n_in, enc_cfg, alignment, m.level_scales_dev.ptr);
		m.grid = GridConfig{};
		m.grid.otype = enc_cfg.value("otype", "OneBlob");
		m.grid.n_pos_dims = n_in;
		m.grid.n_levels = 0;
		m.grid.n_params = (uint32_t)m.plan.n_params;
		m.grid.offsets.assign(1, 0u);
		m.grid.padded_width = m.plan.width;
	}

	mlp.in_width = m.grid.padded_width;
	mlp.out_width = n_out;
	mlp.padded_out_width = next_multiple(n_out, 16u);
	mlp.n_params = mlp.width * mlp.in_width + (mlp.n_hidden_layers - 1) * mlp.width * mlp.width + mlp.padded_out_width * mlp.width;

	// ---- which kernels run this configuration. The fused kernel (fused_ws.cu) covers the benchmarked family; everything else the
	// stand-alone kernels cover takes the general path; the rest fails loudly (no fallback to anything that is not a kernel of this library).
	// FullyFusedMLP's activation set (fully_fused_mlp.cu:689-699): Sine and SiLU need stored pre-activations and are rejected there too.
	for (uint32_t act : {mlp.activation, mlp.output_activation}) {
		if (act == ACT_SINE || act == ACT_SILU) throw std::runtime_error("Unsupported activation.");
	}
	if (m.grid.stochastic_interpolation) throw std::runtime_error("tcnn_b200: stochastic_interpolation is not built");
	{
		const char* why = nullptr;
		if (m.plan_only) why = "an encoding other than one grid / Identity";
		else if (mlp.width > 64) why = "n_neurons > 64";
		else if (mlp.n_hidden_layers > 6) why = "n_hidden_layers > 6";
		else if (mlp.padded_out_width != 16) why = "more than 16 outputs";
		else if (!m.enc_identity && m.grid.n_features_per_level != 2) why = "n_features_per_level != 2";
		else if (m.grid.n_pos_dims != 2 && m.grid.n_pos_dims != 3) why = "input dimensions other than 2 / 3";
		else if (m.grid.padded_width > 64 || m.grid.n_levels > MAX_LEVELS) why = "encoding wider than 64 features";
		else if (fused_ws_smem_bytes(mlp.n_hidden_layers, m.grid.padded_width, true) > 227 * 1024) why = "shared-memory footprint of this depth / encoding width";
		else if (!m.enc_identity && m.grid.interpolation == INTERP_NEAREST) why = "Nearest interpolation";
		if (why) {
			m.general = true;
			m.general_reason = why;
			MlpBackwardArgs probe{};
			probe.width = mlp.width;
			probe.in_width = mlp.in_width;
			probe.out_width = mlp.padded_out_width;
			probe.n_hidden_layers = mlp.n_hidden_layers;
			probe.batch_size = 256;
			probe.dL_dinput = m.grid.n_params == 0 ? nullptr : (__half*)16;  // the encoding's backward pass needs dL/d(encoded)
			const char* why_not = nullptr;
			if (!mlp_backward_supported(probe, &why_not)) throw std::runtime_error(std::string(why_not) + " (general path of tcnn_b200; the fused kernel does not cover this configuration: " + why + ")");
			if (!m.enc_identity && !m.plan_only) {
				const uint32_t F = m.grid.n_features_per_level, D = m.grid.n_pos_dims;
				if (!(F == 1 || F == 2 || F == 4 || F == 8)) throw std::runtime_error("GridEncoding: n_features_per_level must be 1, 2, 4, or 8.");
				if (D < 2 || D > 4) throw std::runtime_error("tcnn_b200: grid encodings cover 2, 3 and 4 input dimensions");
			}
		}
	}

	// ---- per-level scales, evaluated on the device like the reference's kernels (common_device.h:886-891)
	m.level_scales_dev.resize(128);
	if (!m.enc_identity && !m.plan_only) evaluate_level_scales(m.grid, m.level_scales_dev.ptr);
	// one grid / Identity: the segment table of the general path is built for every configuration, so that the general path can run what
	// the fused kernel also covers (tests: both paths must agree; tcnnb_debug_set("general", 1))
	if (!m.plan_only) build_encoding_plan(m.plan, n_in, enc_cfg, alignment, m.level_scales_dev.ptr);

	// ---- parameter buffers (trainer.h:69-87,489-503)
	m.n_params = (size_t)mlp.n_params + m.grid.n_params;
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
		m.first_moments.resize(m.n_params);
		m.first_moments.zero();
		m.second_moments.resize(m.n_params);
		m.second_moments.zero();
		m.param_steps.resize(m.n_params);
		m.param_steps.zero();
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
		if (m.ema.enabled) {  // trainer.h:409-421: the inference parameters start as the initial parameters
			m.ema_fp16.resize(m.n_params_padded);
			TCNNB_CUDA_CHECK(cudaMemcpy(m.ema_fp16.ptr, m.params_fp16, sizeof(__half) * m.n_params_padded, cudaMemcpyDeviceToDevice));
			if (m.ema.full_precision) {
				m.ema_tmp.resize(m.n_params);
				m.ema_tmp.zero();
			}
		}
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

static void check_batch(uint32_t batch) {
	if (batch == 0 || batch % BATCH_GRANULARITY != 0) {
		// object.h:169: CHECK_THROW(input.n() % BATCH_SIZE_GRANULARITY == 0)
		throw std::runtime_error("batch size " + std::to_string(batch) + " must be a non-zero multiple of " + std::to_string(BATCH_GRANULARITY));
	}
}

static FusedStepParams make_params(Model& m, uint32_t batch, uint32_t loss_batch, const float* x, const float* y) {
	FusedStepParams p{};
	p.ablate = m.ablate;
	p.grid = m.grid_meta();
	p.enc_identity = m.enc_identity ? 1u : 0u;
	p.identity_scale = m.identity_scale;
	p.identity_offset = m.identity_offset;
	p.width = m.mlp.width;
	p.n_hidden_layers = m.mlp.n_hidden_layers;
	p.activation = m.mlp.activation;
	p.output_activation = m.mlp.output_activation;
	p.n_out = m.n_out;
	p.n_mlp_params = m.mlp.n_params;
	p.loss_type = m.loss_type;
	p.loss_scale = m.loss_scale;
	p.batch_size = batch;
	p.loss_batch_size = loss_batch;
	p.positions = x;
	p.targets = y;
	p.params = m.params_fp16;
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
	p.dbg_clock = m.dbg_clock.n ? m.dbg_clock.ptr : nullptr;
	return p;
}

// Hyper-parameters of the next optimizer step (advances the step counter; AdaBound bounds per adam.h:161-168).
static AdamParams next_adam_params(Model& m) {
	if (m.lr_decay.enabled) {  // exponential_decay.h:60-70, evaluated with the step count BEFORE this step
		const uint32_t step = m.adam_step_count;
		if (step == 0) m.lr_decay.factor = 1.0f;
		if (step >= m.lr_decay.start && (step - m.lr_decay.start) % m.lr_decay.interval == 0 && step <= m.lr_decay.end) m.lr_decay.factor *= m.lr_decay.base;
	}
	++m.adam_step_count;
	AdamParams a = m.adam;
	a.learning_rate = m.adam.learning_rate * m.lr_decay.factor;
	a.lower_lr_bound = 0;
	a.upper_lr_bound = std::numeric_limits<float>::max();
	if (a.adabound) {
		a.lower_lr_bound = 0.1f - 0.1f / ((1 - a.beta2) * (float)m.adam_step_count + 1);
		a.upper_lr_bound = 0.1f + 0.1f / ((1 - a.beta2) * (float)m.adam_step_count);
	}
	return a;
}

// Adam over the parameter ranges [begin, begin + count) (all parameters when n_ranges == 0). One optimizer step whatever the
// number of ranges: the data-parallel trainer updates the MLP weights everywhere and the grid entries of its own shard only.
static void optimizer_step(Model& m, cudaStream_t stream, uint32_t n_ranges = 0, const uint64_t* begins = nullptr, const uint64_t* counts = nullptr) {
	if (m.module_only) throw std::runtime_error("this handle was created with tcnnb_module_create: it has no optimizer.");
	m.wait_pending(stream);
	const AdamParams a = next_adam_params(m);
	const uint64_t whole_begin = 0, whole_count = m.n_params;
	if (n_ranges == 0) {
		n_ranges = 1;
		begins = &whole_begin;
		counts = &whole_count;
	}
	bool covers_mlp = false;
	for (uint32_t r = 0; r < n_ranges; ++r) {
		const uint64_t b = begins[r], c = counts[r];
		if (b + c > m.n_params) throw std::runtime_error("optimizer_step: parameter range out of bounds.");
		if (c == 0) continue;
		if (b < m.mlp.n_params && b + c < m.mlp.n_params) throw std::runtime_error("optimizer_step: a range may not split the network weights.");
		const uint32_t n_matrix = b < m.mlp.n_params ? (uint32_t)(m.mlp.n_params - b) : 0u;  // matrix weights inside this range
		covers_mlp |= b == 0 && n_matrix > 0;
		if (n_matrix > 0 && b != 0) throw std::runtime_error("optimizer_step: the network weights must be covered from parameter 0.");
		TCNNB_CUDA_CHECK(launch_adam_step(stream, a, (uint32_t)c, n_matrix, m.loss_scale, m.params_fp32 + b, m.params_fp16 + b, m.grads_fp16 + b,
		                                  (m.mlp_grads_in_accum && n_matrix > 0) ? m.dw_accum.ptr : nullptr, m.first_moments.ptr + b, m.second_moments.ptr + b,
		                                  m.param_steps.ptr + b));
		++g_kernel_launches;
	}
	if (covers_mlp) m.mlp_grads_in_accum = false;
	if (m.ema.enabled) {
		if (n_ranges != 1 || begins[0] != 0 || counts[0] != m.n_params) throw std::runtime_error("tcnn_b200: the Ema wrapper is built for whole-vector optimizer steps (not for the sharded data-parallel optimizer)");
		const float t = (float)m.adam_step_count;
		TCNNB_CUDA_CHECK(launch_ema_step(stream, (uint32_t)m.n_params, m.ema.decay, 1.0f - std::pow(m.ema.decay, t - 1.0f), 1.0f / (1.0f - std::pow(m.ema.decay, t)), m.params_fp16, m.ema_fp16.ptr,
		                                 m.ema.full_precision ? m.ema_tmp.ptr : nullptr));
		++g_kernel_launches;
	}
}

static void ensure_levels_dev(Model& m, cudaStream_t stream) {
	if (m.levels_dev.n == 0 && m.grid.n_levels) {
		std::vector<LevelInfo> levels(m.grid.n_levels);
		for (uint32_t l = 0; l < m.grid.n_levels; ++l) levels[l] = make_level_info(m.grid, l);
		m.levels_dev.resize(levels.size());
		TCNNB_CUDA_CHECK(cudaMemcpyAsync(m.levels_dev.ptr, levels.data(), sizeof(LevelInfo) * levels.size(), cudaMemcpyHostToDevice, stream));
		TCNNB_CUDA_CHECK(cudaStreamSynchronize(stream));  // `levels` is a pageable temporary
	}
}

static GridKernelArgs grid_kernel_args(Model& m, uint32_t n, const float* x, uint32_t row_stride) {
	GridKernelArgs a{};
	a.n_pos_dims = m.grid.n_pos_dims;
	a.n_features_per_level = m.grid.n_features_per_level;
	a.n_levels = m.grid.n_levels;
	a.interpolation = m.grid.interpolation;
	a.max_level = 1.0f;
	a.levels_dev = m.levels_dev.ptr;
	a.n_elements = n;
	a.positions = x;
	a.pos_stride = m.grid.n_pos_dims;
	a.row_stride = row_stride;
	a.pad_cols = row_stride - m.grid.n_levels * m.grid.n_features_per_level;
	return a;
}

template <typename T>
static void grow(DeviceBuffer<T>& b, size_t n) {
	if (b.n < n) b.resize(n);
}

// ---- general path: encoding kernel -> stand-alone network kernel (mlp_fused.cu), activations optionally kept for the backward pass
static void general_forward(Model& m, cudaStream_t stream, uint32_t batch, const float* x, const __half* params, __half* out_fp16, float* out_fp32, bool keep_hidden) {
	const MlpConfig& mlp = m.mlp;
	grow(m.g_enc, (size_t)batch * mlp.in_width);
	if (m.plan.has_plain_features()) {
		TCNNB_CUDA_CHECK(launch_feature_forward(stream, m.plan.segs, batch, x, m.n_in, m.g_enc.ptr, mlp.in_width));
		++g_kernel_launches;
	}
	for (auto& g : m.plan.grids) {
		const FeatureSegment& sg = m.plan.segs.s[g->segment];
		GridKernelArgs ga = plan_grid_args(*g, batch, x + sg.in_begin, m.n_in, mlp.in_width);
		ga.pad_cols = sg.n_pad;
		TCNNB_CUDA_CHECK(launch_grid_forward(stream, ga, params + mlp.n_params + g->param_offset, m.g_enc.ptr + sg.out_begin));
		++g_kernel_launches;
	}
	MlpForwardParams p{};
	p.width = mlp.width;
	p.in_width = mlp.in_width;
	p.out_width = mlp.padded_out_width;
	p.n_hidden_layers = mlp.n_hidden_layers;
	p.activation = mlp.activation;
	p.output_activation = mlp.output_activation;
	p.weights = params;
	p.batch_size = batch;
	p.input_fp16 = m.g_enc.ptr;
	p.n_output_dims = m.n_out;
	p.output_fp16 = out_fp16;
	p.output_fp32 = out_fp32;
	if (keep_hidden) {
		grow(m.g_hidden, (size_t)mlp.n_hidden_layers * batch * mlp.width);
		p.hidden_out = m.g_hidden.ptr;
	}
	const char* why = nullptr;
	if (!mlp_forward_supported(p, &why)) throw std::runtime_error(why);
	TCNNB_CUDA_CHECK(launch_mlp_forward(p, (uint32_t)m.n_sms, stream));
	++g_kernel_launches;
	m.last_stream = stream;
}

// Forward + loss (or the caller's dL/d(output)) + backward on the general path. Gradients land where the fused kernel leaves them:
// fp32 network weight-gradient sums in dw_accum, fp16 table gradients in grads + n_mlp_params. `dL_dinput` (fp32 [batch][n_in]) optional.
static void general_backward_pass(Model& m, cudaStream_t stream, uint32_t batch, uint32_t loss_batch, const float* x, const float* y, const __half* params, __half* grads,
                                  const __half* ext_dL_doutput, float* dL_dinput, bool want_param_grads) {
	const MlpConfig& mlp = m.mlp;
	const bool grid_params = m.grid.n_params != 0 && want_param_grads;
	if (grid_params) {
		TCNNB_CUDA_CHECK(cudaMemsetAsync(grads + mlp.n_params, 0, sizeof(__half) * m.grid.n_params, stream));  // GradientMode::Overwrite (grid.h:865-867)
	}
	if (!ext_dL_doutput) TCNNB_CUDA_CHECK(cudaMemsetAsync(m.scalars.ptr, 0, sizeof(float), stream));
	if (m.mlp_grads_in_accum) {
		TCNNB_CUDA_CHECK(cudaMemsetAsync(m.dw_accum.ptr, 0, sizeof(float) * mlp.n_params, stream));
		m.mlp_grads_in_accum = false;
	}
	m.prof_mark(stream);
	m.prof_mark(stream);  // (no binning pass on this path)
	m.wait_pending(stream);
	grow(m.g_out, (size_t)batch * mlp.padded_out_width);
	__half* const out_rows = (m.taps.output && mlp.padded_out_width == 16) ? (__half*)m.taps.output : m.g_out.ptr;  // (the test tap is 16 columns wide)
	general_forward(m, stream, batch, x, params, out_rows, nullptr, true);
	const __half* out = out_rows;

	MlpBackwardArgs a{};
	a.width = mlp.width;
	a.in_width = mlp.in_width;
	a.out_width = mlp.padded_out_width;
	a.n_hidden_layers = mlp.n_hidden_layers;
	a.activation = mlp.activation;
	a.weights = params;
	a.batch_size = batch;
	a.input = m.g_enc.ptr;
	a.hidden = m.g_hidden.ptr;
	a.output = out;
	if (ext_dL_doutput) {  // Module::backward: the caller's dL/d(output) still has to pass the output activation (fully_fused_mlp.cu:755-762)
		a.output_activation = mlp.output_activation;
		a.dL_doutput = ext_dL_doutput;
		if (mlp.output_activation != ACT_NONE) {
			grow(m.g_dy_act, (size_t)batch * mlp.padded_out_width);
			a.grad_output = m.g_dy_act.ptr;
		}
	} else {  // Trainer: loss gradient x loss_scale, through the output activation, in one kernel
		grow(m.g_dy, (size_t)batch * mlp.padded_out_width);
		TCNNB_CUDA_CHECK(launch_loss(stream, m.loss_type, mlp.output_activation, batch, m.n_out, mlp.padded_out_width, m.loss_scale, loss_batch * m.n_out, out, y, m.g_dy.ptr,
		                             m.taps.loss_values, m.scalars.ptr));
		++g_kernel_launches;
		a.output_activation = ACT_NONE;
		a.dL_doutput = m.g_dy.ptr;
	}
	const bool need_denc = grid_params || dL_dinput;
	if (need_denc) {
		grow(m.g_denc, (size_t)batch * mlp.in_width);
		a.dL_dinput = m.g_denc.ptr;
	}
	if (want_param_grads) {
		grow(m.g_grad_hidden, (size_t)mlp.n_hidden_layers * batch * mlp.width);
		a.grad_hidden = m.g_grad_hidden.ptr;
		a.dw_accum = m.dw_accum.ptr;
	}
	const char* why = nullptr;
	if (!mlp_backward_supported(a, &why)) throw std::runtime_error(why);
	uint32_t launches = 0;
	TCNNB_CUDA_CHECK(launch_mlp_backward(a, (uint32_t)m.n_sms, stream, &launches));
	g_kernel_launches += launches;
	if (want_param_grads) m.mlp_grads_in_accum = true;
	if (grid_params) {
		for (auto& g : m.plan.grids) {
			const FeatureSegment& sg = m.plan.segs.s[g->segment];
			float* tmp = nullptr;
			if (g->cfg.n_features_per_level == 1) {
				grow(m.g_grid_tmp, g->cfg.n_params);
				TCNNB_CUDA_CHECK(cudaMemsetAsync(m.g_grid_tmp.ptr, 0, sizeof(float) * g->cfg.n_params, stream));
				tmp = m.g_grid_tmp.ptr;
			}
			GridKernelArgs ga = plan_grid_args(*g, batch, x + sg.in_begin, m.n_in, mlp.in_width);
			GridScatterPlan sp = plan_grid_scatter(g->levels.data(), g->cfg.n_levels, g->cfg.n_features_per_level, g->cfg.n_pos_dims, batch);
			if (m.grid_replicas_override >= 0 && sp.replica_entries) {
				sp.n_replicas = (uint32_t)m.grid_replicas_override;
				sp.scratch_halfs = (size_t)sp.n_replicas * sp.replica_entries * g->cfg.n_features_per_level;
			}
			if (sp.n_replicas > 1) {
				if (m.g_replicas.n < sp.scratch_halfs) {
					m.g_replicas.resize(sp.scratch_halfs);
					m.g_replicas.zero(stream);  // the reduce kernel leaves it zero
				}
				ga.replica_scratch = m.g_replicas.ptr;
				ga.n_replicas = sp.n_replicas;
				ga.replica_entries = sp.replica_entries;
			}
			TCNNB_CUDA_CHECK(launch_grid_backward(stream, ga, m.g_denc.ptr + sg.out_begin, grads + mlp.n_params + g->param_offset, tmp, g->cfg.n_params));
			++g_kernel_launches;
		}
	}
	if (dL_dinput) {
		if (m.plan.composite) TCNNB_CUDA_CHECK(cudaMemsetAsync(dL_dinput, 0, sizeof(float) * (size_t)batch * m.n_in, stream));  // dimensions no nested encoding reads
		if (m.plan.has_plain_features()) {
			TCNNB_CUDA_CHECK(launch_feature_input_gradient(stream, m.plan.segs, batch, x, m.n_in, m.g_denc.ptr, mlp.in_width, dL_dinput));
			++g_kernel_launches;
		}
		for (auto& g : m.plan.grids) {
			const FeatureSegment& sg = m.plan.segs.s[g->segment];
			const GridKernelArgs ga = plan_grid_args(*g, batch, x + sg.in_begin, m.n_in, mlp.in_width);
			TCNNB_CUDA_CHECK(launch_grid_input_gradient(stream, ga, params + mlp.n_params + g->param_offset, m.g_denc.ptr + sg.out_begin, dL_dinput + sg.in_begin));
			++g_kernel_launches;
		}
	}
	m.last_stream = stream;
	m.prof_mark(stream);
}

// `targets_ready`: optional event the fused kernel (the first consumer of `y`) waits for; everything before it in the step --
// gradient zeroing, the binning pass -- only needs `x` and runs while the targets are still in flight.
// Caller-owned arrays of the module tier (cpp_api.h:76-104): working-precision parameters, gradient array, dL/d(output).
struct ModuleIO {
	const __half* params = nullptr;
	__half* grads = nullptr;
	const __half* dL_doutput = nullptr;
	__half* dL_dencoded = nullptr;  // optional [n][64] fp16: the network's input gradient rows, for the input-position gradient
};

static void training_step(Model& m, cudaStream_t stream, uint32_t batch, uint32_t loss_batch, const float* x, const float* y, bool run_optimizer, cudaEvent_t targets_ready = nullptr,
                          const ModuleIO* io = nullptr) {
	check_batch(batch);
	if (!io && m.module_only) throw std::runtime_error("this handle was created with tcnnb_module_create: use the tcnnb_module_* calls.");
	if (m.use_general()) {
		if (io) throw std::runtime_error("internal: the module tier of the general path does not come through here");
		if (targets_ready) TCNNB_CUDA_CHECK(cudaStreamWaitEvent(stream, targets_ready, 0));
		general_backward_pass(m, stream, batch, loss_batch, x, y, m.params_fp16, m.grads_fp16, nullptr, nullptr, true);
		if (run_optimizer) optimizer_step(m, stream);
		m.prof_mark(stream);
		return;
	}
	__half* const grads_base = io ? io->grads : m.grads_fp16;
	// GradientMode::Overwrite: zero the grid gradient table (grid.h:865-867) and the loss accumulator -- inside the binning pass
	// when there is one, else as memsets.
	__half* const grid_grads = grads_base + m.mlp.n_params;
	const size_t grid_grad_bytes = sizeof(__half) * m.grid.n_params;
	const bool bin = m.binning && batch >= 16384 && !m.enc_identity;  // spatial order only matters to the table gathers
	const bool zero_in_binning = bin && (((uintptr_t)grid_grads | grid_grad_bytes) & 15u) == 0;
	if (!zero_in_binning) {
		TCNNB_CUDA_CHECK(cudaMemsetAsync(grid_grads, 0, grid_grad_bytes, stream));
		TCNNB_CUDA_CHECK(cudaMemsetAsync(m.scalars.ptr, 0, sizeof(float), stream));
	}
	if (m.mlp_grads_in_accum) {
		// a previous step left un-consumed weight gradients (run_optimizer == false twice in a row): Overwrite semantics
		TCNNB_CUDA_CHECK(cudaMemsetAsync(m.dw_accum.ptr, 0, sizeof(float) * m.mlp.n_params, stream));
	}
	FusedStepParams p = make_params(m, batch, loss_batch, x, y);
	if (io) {
		p.params = io->params;
		p.grads = io->grads;
		p.ext_dy = io->dL_doutput;
		if (io->dL_dencoded) p.dbg_denc = io->dL_dencoded;
		p.targets = nullptr;
		p.loss_sum = nullptr;
		p.loss_values = nullptr;
	}
	m.prof_mark(stream);
	// Process the batch in (y, z)-column order: same sums, far fewer distinct memory sectors on the coarse levels (binning.cu).
	if (bin) {
		const uint32_t log2_r = binning_log2_resolution(batch, m.grid.n_pos_dims);
		m.bin_keys.resize(std::max(m.bin_keys.n, 2 * (size_t)batch));
		m.bin_perm.resize(std::max(m.bin_perm.n, (size_t)batch));
		{
			const size_t need = 2 * (size_t)binning_n_bins(log2_r, m.grid.n_pos_dims);
			if (m.bin_hist.n != need) {  // layout depends on n_bins: (re)allocate and zero the counters once
				m.bin_hist.resize(need);
				m.bin_hist.zero(stream);
			}
		}
		TCNNB_CUDA_CHECK(launch_binning(stream, m.grid.n_pos_dims, batch, x, log2_r, m.bin_keys.ptr, m.bin_hist.ptr, m.bin_perm.ptr, zero_in_binning ? grid_grads : nullptr,
		                                zero_in_binning ? grid_grad_bytes : 0, zero_in_binning ? (float*)m.scalars.ptr : nullptr));
		g_kernel_launches += 3;
		p.perm = m.bin_perm.ptr;
	}
	m.prof_mark(stream);
	if (targets_ready) TCNNB_CUDA_CHECK(cudaStreamWaitEvent(stream, targets_ready, 0));
	m.wait_pending(stream);  // e.g. the all-gather of the previous data-parallel step: binning above did not need the parameters
	// one persistent 640-thread CTA per SM (fused_ws.cu)
	TCNNB_CUDA_CHECK(launch_fused_ws(p, m.grid.n_pos_dims, true, std::min(batch / TILE_M, (uint32_t)m.n_sms), stream));
	++g_kernel_launches;
	m.last_stream = stream;
	m.prof_mark(stream);
	m.mlp_grads_in_accum = true;
	if (run_optimizer) {
		optimizer_step(m, stream);
	}
	m.prof_mark(stream);
}

static void finalize_mlp_grads(Model& m, cudaStream_t stream) {
	if (m.mlp_grads_in_accum) {
		TCNNB_CUDA_CHECK(launch_mlp_grad_finalize(stream, m.mlp.n_params, m.dw_accum.ptr, m.grads_fp16));
		++g_kernel_launches;
		m.mlp_grads_in_accum = false;
	}
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
		TCNNB_NCCL_CHECK(n.AllReduce(m.grads_fp16 + m.mlp.n_params, m.grads_fp16 + m.mlp.n_params, m.grid.n_params, ncclHalf, ncclSum, d.comm_grads, stream));
		TCNNB_NCCL_CHECK(n.AllReduce(m.dw_accum.ptr, m.dw_accum.ptr, m.mlp.n_params, ncclFloat, ncclSum, d.comm_grads, stream));
		optimizer_step(m, stream);
		return;
	}
	if (m.mlp_grads_in_accum) {  // fp32 network weight-gradient sums -> the fp16 gradient vector (what the reference's buffer holds)
		TCNNB_CUDA_CHECK(launch_mlp_grad_finalize(stream, m.mlp.n_params, m.dw_accum.ptr, m.grads_fp16));
		++g_kernel_launches;
		m.mlp_grads_in_accum = false;
	}
	const size_t chunk = m.n_params_padded / (size_t)d.world, lo = chunk * (size_t)d.rank;
	if (d.fused) {
		// Peer-memory engine: [barrier: every rank's gradient vector is complete] -> ONE kernel on this rank's slice that sums the
		// gradient over the ranks (in the switch with multimem.ld_reduce, else by peer loads), applies Adam and publishes the fp16
		// weights into every replica (multimem.st / peer stores) -> [barrier: all slices have landed everywhere; the gradient
		// vectors may be zeroed again]. No NCCL call on the step.
		TCNNB_CUDA_CHECK(launch_dp_barrier(stream, d.peers, ++d.epoch));
		const AdamParams a = next_adam_params(m);
		TCNNB_CUDA_CHECK(launch_adam_step_dp(stream, a, d.peers, lo, chunk, (uint32_t)m.mlp.n_params, m.n_params, m.loss_scale, m.params_fp32, m.first_moments.ptr, m.second_moments.ptr,
		                                     m.param_steps.ptr));
		TCNNB_CUDA_CHECK(launch_dp_barrier(stream, d.peers, ++d.epoch));
		g_kernel_launches += 3;
		d.masters_synced = false;
		return;
	}
	TCNNB_NCCL_CHECK(n.ReduceScatter(m.grads_fp16, m.grads_fp16 + lo, chunk, ncclHalf, ncclSum, d.comm_grads, stream));
	const uint64_t begin = lo, count = lo < m.n_params ? std::min<uint64_t>(chunk, m.n_params - lo) : 0;
	if (count) optimizer_step(m, stream, 1, &begin, &count);
	else ++m.adam_step_count;
	TCNNB_CUDA_CHECK(cudaEventRecord(d.ev_updated, stream));
	TCNNB_CUDA_CHECK(cudaStreamWaitEvent(d.gather_stream, d.ev_updated, 0));
	TCNNB_NCCL_CHECK(n.AllGather(m.params_fp16 + lo, m.params_fp16, chunk, ncclHalf, d.comm_params, d.gather_stream));
	TCNNB_CUDA_CHECK(cudaEventRecord(d.ev_gathered, d.gather_stream));
	m.pending_params_event = d.ev_gathered;
	d.masters_synced = false;
}

// Sum of the ranks' partial losses (each normalised over the global batch) -> the global loss, in place on every rank.
static void dp_reduce_loss(Model& m, cudaStream_t stream) {
	if (m.dp && m.dp->world > 1) {
		TCNNB_NCCL_CHECK(nccl_api().AllReduce(m.scalars.ptr, m.scalars.ptr, 1, ncclFloat, ncclSum, m.dp->comm_grads, stream));
	}
}

static void launch_inference(Model& m, const FusedStepParams& p, uint32_t batch, cudaStream_t stream) {
	// the warp-specialised kernel without its backward half (measured 0.0885 ms vs 0.127 ms for the bulk-synchronous kernel it replaced)
	TCNNB_CUDA_CHECK(launch_fused_ws(p, m.grid.n_pos_dims, false, std::min(batch / TILE_M, (uint32_t)m.n_sms), stream));
	++g_kernel_launches;
	m.last_stream = stream;
}

static void inference(Model& m, cudaStream_t stream, uint32_t batch, const float* x, float* out) {
	check_batch(batch);
	if (m.module_only) throw std::runtime_error("this handle was created with tcnnb_module_create: use the tcnnb_module_* calls.");
	m.wait_pending(stream);
	if (m.use_general()) {
		general_forward(m, stream, batch, x, m.inference_params(), nullptr, out, false);
		return;
	}
	FusedStepParams p = make_params(m, batch, batch, x, nullptr);
	p.params = m.inference_params();
	p.out_fp32 = out;
	p.loss_sum = nullptr;
	launch_inference(m, p, batch, stream);
}

// ---- module tier (tcnn::cpp::Module for NetworkWithInputEncoding, cpp_api.cu:71-158): caller-owned parameters -------------
static void check_module_ptr(const void* ptr, const char* what) {
	if (!ptr) throw std::runtime_error(std::string("module: ") + what + " is null.");
	if ((uintptr_t)ptr % 16 != 0) throw std::runtime_error(std::string("module: ") + what + " must be 16-byte aligned.");
}

// inference / forward: fp16 [n][padded_output_width] rows (column-major padded x n in the reference's terms, cpp_api.cu:82-83).
// Nothing is saved for the backward pass -- it recomputes the forward inside the fused kernel (the gather + three MMAs per
// tile are cheaper than writing and re-reading 2 x 64 x n fp16 activations, which is what the reference's context holds).
static void module_forward(Model& m, cudaStream_t stream, uint32_t n, const float* x, void* output, const void* params) {
	check_batch(n);
	check_module_ptr(params, "params");
	check_module_ptr(output, "output");
	if (m.use_general()) {
		general_forward(m, stream, n, x, (const __half*)params, (__half*)output, nullptr, false);
		return;
	}
	FusedStepParams p = make_params(m, n, n, x, nullptr);
	p.params = (const __half*)params;
	p.grads = nullptr;
	p.out_fp16 = (__half*)output;
	p.out_fp32 = nullptr;
	p.loss_sum = nullptr;
	launch_inference(m, p, n, stream);
}

// backward: dL_dparams (fp16 [n_params], OVERWRITTEN -- GradientMode::Overwrite, cpp_api.cu:115) from dL_doutput (fp16 [n][padded]).
static void module_backward(Model& m, cudaStream_t stream, uint32_t n, float* dL_dinput, const void* dL_doutput, void* dL_dparams, const float* x, const void* params) {
	if (!dL_dparams && !dL_dinput) return;  // nothing to compute (GradientMode::Ignore)
	check_module_ptr(params, "params");
	check_module_ptr(dL_doutput, "dL_doutput");
	if (m.use_general()) {
		check_batch(n);
		if (dL_dparams) check_module_ptr(dL_dparams, "dL_dparams");
		general_backward_pass(m, stream, n, n, x, nullptr, (const __half*)params, (__half*)dL_dparams, (const __half*)dL_doutput, dL_dinput, dL_dparams != nullptr);
		if (dL_dparams) {
			TCNNB_CUDA_CHECK(launch_mlp_grad_finalize(stream, m.mlp.n_params, m.dw_accum.ptr, (__half*)dL_dparams));
			++g_kernel_launches;
			m.mlp_grads_in_accum = false;
		}
		return;
	}
	ModuleIO io;
	io.params = (const __half*)params;
	io.dL_doutput = (const __half*)dL_doutput;
	if (dL_dparams) {
		check_module_ptr(dL_dparams, "dL_dparams");
		io.grads = (__half*)dL_dparams;
	} else {  // input gradients only: the fused kernel still needs somewhere to scatter
		m.grads_scratch.resize(m.n_params_padded);
		io.grads = m.grads_scratch.ptr;
	}
	if (dL_dinput) {
		// dL/d(input) (cpp_api.cu:104-125 -> NetworkWithInputEncoding::backward -> GridEncoding::backward_impl, grid.h:896-921): the fused
		// kernel hands out the network's input gradient rows, the stand-alone kernel contracts them with d(encoded)/d(position).
		m.denc_scratch.resize(std::max(m.denc_scratch.n, (size_t)n * 64));
		io.dL_dencoded = m.denc_scratch.ptr;
	}
	if (m.mlp_grads_in_accum) {
		TCNNB_CUDA_CHECK(cudaMemsetAsync(m.dw_accum.ptr, 0, sizeof(float) * m.mlp.n_params, stream));
		m.mlp_grads_in_accum = false;
	}
	training_step(m, stream, n, n, x, nullptr, false, nullptr, &io);
	// network weight gradients: fp32 sums -> fp16 entries of the caller's array; re-arms the accumulator
	TCNNB_CUDA_CHECK(launch_mlp_grad_finalize(stream, m.mlp.n_params, m.dw_accum.ptr, io.grads));
	++g_kernel_launches;
	m.mlp_grads_in_accum = false;
	if (dL_dinput) {
		ensure_levels_dev(m, stream);
		GridKernelArgs a{};
		a.n_pos_dims = m.grid.n_pos_dims;
		a.n_features_per_level = m.grid.n_features_per_level;
		a.n_levels = m.grid.n_levels;
		a.interpolation = m.grid.interpolation;
		a.max_level = 1.0f;
		a.levels_dev = m.levels_dev.ptr;
		a.n_elements = n;
		a.positions = x;
		a.pos_stride = m.grid.n_pos_dims;
		a.row_stride = 64;
		TCNNB_CUDA_CHECK(launch_grid_input_gradient(stream, a, (const __half*)params + m.mlp.n_params, m.denc_scratch.ptr, dL_dinput));
		++g_kernel_launches;
	}
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

static void dp_training_step(Model& m, cudaStream_t stream, uint32_t shard_batch, uint32_t global_batch, const float* x, const float* y);
static void dp_reduce_loss(Model& m, cudaStream_t stream);

// Enqueue one training step on HOST buffers and return at once: host->device copies on the copy stream (they overlap the kernels
// of the step submitted before), the step on the model's compute stream (the binning pass starts when the positions have
// landed, the fused kernel when the targets have), the loss read-back behind it. At most two steps are in flight.
static uint64_t host_step_submit(Model& m, uint32_t batch, uint32_t global_batch, const float* x_host, const float* y_host, bool data_parallel) {
	check_batch(batch);
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
	if (m.enc_identity) {
		enc["otype"] = json::Value::string("Identity");
		enc["scale"] = json::Value::number(m.identity_scale);
		enc["offset"] = json::Value::number(m.identity_offset);
	} else if (m.plan_only) {
		enc["otype"] = json::Value::string(m.grid.otype);
		enc["n_nested"] = json::Value::number(m.plan.segs.n);
		enc["n_output_dims"] = json::Value::number(m.plan.width);
	} else {
	enc["otype"] = json::Value::string("Grid");
	enc["type"] = json::Value::string(m.grid.grid_type == GRID_HASH ? "Hash" : (m.grid.grid_type == GRID_DENSE ? "Dense" : "Tiled"));
	enc["n_levels"] = json::Value::number(m.grid.n_levels);
	enc["n_features_per_level"] = json::Value::number(m.grid.n_features_per_level);
	enc["base_resolution"] = json::Value::number(m.grid.base_resolution);
	enc["log2_hashmap_size"] = json::Value::number(m.grid.log2_hashmap_size);
	enc["per_level_scale"] = json::Value::number(m.grid.per_level_scale);
	enc["interpolation"] = json::Value::string(m.grid.interpolation == INTERP_LINEAR ? "Linear" : (m.grid.interpolation == INTERP_SMOOTHSTEP ? "Smoothstep" : "Nearest"));
	enc["hash"] = json::Value::string("CoherentPrime");
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
	json::Value& opt = root["optimizer"];
	opt["otype"] = json::Value::string("Adam");
	opt["learning_rate"] = json::Value::number(m.adam.learning_rate);
	opt["beta1"] = json::Value::number(m.adam.beta1);
	opt["beta2"] = json::Value::number(m.adam.beta2);
	opt["epsilon"] = json::Value::number(m.adam.epsilon);
	opt["l2_reg"] = json::Value::number(m.adam.l2_reg);
	root["n_params"] = json::Value::number((double)m.n_params);
	root["n_mlp_params"] = json::Value::number(m.mlp.n_params);
	root["encoded_width"] = json::Value::number(m.grid.padded_width);
	return json::dump(root);
}

}  // namespace tcnnb

namespace tcnnb {
__global__ void half_to_float_kernel(uint64_t n, const __half* __restrict__ in, float* __restrict__ out) {
	const uint64_t i = threadIdx.x + (uint64_t)blockIdx.x * blockDim.x;
	if (i < n) out[i] = (float)in[i];
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
uint32_t tcnnb_encoded_width(const tcnnb_model* m) { return m->impl.grid.padded_width; }
float* tcnnb_params_full_precision(tcnnb_model* m) { return m->impl.params_fp32; }
void* tcnnb_params(tcnnb_model* m) { return m->impl.params_fp16; }
float* tcnnb_mlp_gradient_accumulator(tcnnb_model* m) { return m->impl.dw_accum.ptr; }
void* tcnnb_grid_gradients(tcnnb_model* m) { return m->impl.grads_fp16 + m->impl.mlp.n_params; }

void* tcnnb_param_gradients(tcnnb_model* m) {
	// The MLP part is materialised as fp16 on demand (the fused kernel accumulates it in fp32).
	try {
		// ordered behind the step that produced the gradients: same stream, and the synchronisation is on that stream only
		finalize_mlp_grads(m->impl, m->impl.last_stream);
		TCNNB_CUDA_CHECK(cudaStreamSynchronize(m->impl.last_stream));
	} catch (const std::exception& e) {
		g_last_error = e.what();
		return nullptr;
	}
	return m->impl.grads_fp16;
}

int tcnnb_grid_levels(const tcnnb_model* m, uint32_t* n_levels, uint32_t* offsets, float* scales, uint32_t* resolutions) {
	TCNNB_API_BEGIN
	const GridConfig& g = m->impl.grid;
	if (n_levels) *n_levels = g.n_levels;
	for (uint32_t l = 0; l < g.n_levels; ++l) {
		if (offsets) offsets[l] = g.offsets[l];
		if (scales) scales[l] = g.scales[l];
		if (resolutions) resolutions[l] = (uint32_t)ceilf(g.scales[l]) + 1;
	}
	if (offsets) offsets[g.n_levels] = g.offsets[g.n_levels];
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
	if (mm.ema.enabled) TCNNB_CUDA_CHECK(cudaMemcpy(mm.ema_fp16.ptr, mm.params_fp16, sizeof(__half) * n, cudaMemcpyDeviceToDevice));  // trainer.h:415-419
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	TCNNB_API_END
}

// Trainer::params_inference() (trainer.h:401-403): the Ema wrapper's averaged weights when there is one, else the working parameters.
void* tcnnb_params_inference(tcnnb_model* m) { return (void*)m->impl.inference_params(); }

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
	if (mm.ema.enabled) TCNNB_CUDA_CHECK(cudaMemcpy(mm.ema_fp16.ptr, mm.params_fp16, sizeof(__half) * n, cudaMemcpyDeviceToDevice));  // trainer.h:428-429
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	TCNNB_API_END
}

int tcnnb_optimizer_state(tcnnb_model* m, float** first_moments_dev, float** second_moments_dev, uint32_t** param_steps_dev, uint32_t* current_step, float* base_learning_rate) {
	TCNNB_API_BEGIN
	Model& mm = m->impl;
	if (mm.module_only) throw std::runtime_error("this handle was created with tcnnb_module_create: it has no optimizer.");
	if (mm.ema.enabled) throw std::runtime_error("tcnn_b200: snapshots of the Ema wrapper's state are not built (serialize the parameters only)");
	if (mm.dp && mm.dp->world > 1 && mm.dp->shard_optimizer) {
		throw std::runtime_error("optimizer state is sharded over the data-parallel ranks: each rank holds the moments of its own slice only");
	}
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	if (first_moments_dev) *first_moments_dev = mm.first_moments.ptr;
	if (second_moments_dev) *second_moments_dev = mm.second_moments.ptr;
	if (param_steps_dev) *param_steps_dev = mm.param_steps.ptr;
	if (current_step) *current_step = mm.adam_step_count;
	if (base_learning_rate) *base_learning_rate = mm.adam.learning_rate;
	TCNNB_API_END
}

int tcnnb_set_optimizer_progress(tcnnb_model* m, uint32_t current_step, float base_learning_rate) {
	TCNNB_API_BEGIN
	m->impl.adam_step_count = current_step;
	m->impl.adam.learning_rate = base_learning_rate;
	TCNNB_API_END
}

int tcnnb_training_step(tcnnb_model* m, tcnnb_stream stream, uint32_t batch_size, const float* input_dev, const float* target_dev, int run_optimizer) {
	TCNNB_API_BEGIN
	training_step(m->impl, (cudaStream_t)stream, batch_size, batch_size, input_dev, target_dev, run_optimizer != 0);
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
	inference(m->impl, (cudaStream_t)stream, batch_size, input_dev, output_dev);
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
	ensure_staging(mm, batch_size);
	cudaStream_t s = mm.own_stream;
	const size_t n_x = (size_t)batch_size * mm.n_in, n_y = (size_t)batch_size * mm.n_out;
	std::memcpy(mm.pinned, input_host, n_x * sizeof(float));
	TCNNB_CUDA_CHECK(cudaMemcpyAsync(mm.stage_in.ptr, mm.pinned, n_x * sizeof(float), cudaMemcpyHostToDevice, s));
	inference(mm, s, batch_size, mm.stage_in.ptr, mm.stage_out.ptr);
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
	if (with_optimizer && mm.ema.enabled) throw std::runtime_error("tcnn_b200: snapshots of the Ema wrapper's state are not built (serialize with_optimizer = 0)");
	if (with_optimizer && mm.dp && mm.dp->world > 1 && mm.dp->shard_optimizer) {
		// moments / step counters are current on the owner of a slice only (ZeRO-1): a snapshot of one rank would silently hold stale state
		throw std::runtime_error("tcnnb_serialize: optimizer state is sharded over the data-parallel ranks; serialize with_optimizer = 0 (after tcnnb_dp_sync_full_precision) or from a single-GPU trainer");
	}
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	char* p = (char*)dst_host;
	const uint64_t n = mm.n_params;
	const uint32_t wo = with_optimizer ? 1 : 0, st = mm.adam_step_count;
	std::memcpy(p, &n, 8);
	std::memcpy(p + 8, &wo, 4);
	std::memcpy(p + 12, &st, 4);
	p += 16;
	TCNNB_CUDA_CHECK(cudaMemcpy(p, mm.params_fp16, n * 2, cudaMemcpyDeviceToHost));
	p += n * 2;
	if (with_optimizer) {
		TCNNB_CUDA_CHECK(cudaMemcpy(p, mm.first_moments.ptr, n * 4, cudaMemcpyDeviceToHost));
		p += n * 4;
		TCNNB_CUDA_CHECK(cudaMemcpy(p, mm.second_moments.ptr, n * 4, cudaMemcpyDeviceToHost));
		p += n * 4;
		TCNNB_CUDA_CHECK(cudaMemcpy(p, mm.param_steps.ptr, n * 4, cudaMemcpyDeviceToHost));
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
		TCNNB_CUDA_CHECK(cudaMemcpy(mm.first_moments.ptr, p, n * 4, cudaMemcpyHostToDevice));
		p += n * 4;
		TCNNB_CUDA_CHECK(cudaMemcpy(mm.second_moments.ptr, p, n * 4, cudaMemcpyHostToDevice));
		p += n * 4;
		TCNNB_CUDA_CHECK(cudaMemcpy(mm.param_steps.ptr, p, n * 4, cudaMemcpyHostToDevice));
		mm.adam_step_count = st;
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
	if (mm.ema.enabled && world_size > 1) throw std::runtime_error("tcnn_b200: the Ema optimizer wrapper is not built for the data-parallel engines");
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

int tcnnb_dp_shards_optimizer(const tcnnb_model* m) { return m->impl.dp && m->impl.dp->world > 1 && m->impl.dp->shard_optimizer ? 1 : 0; }

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
	module_forward(m->impl, (cudaStream_t)stream, n_elements, input_dev, output_dev, params_dev);
	TCNNB_API_END
}

int tcnnb_module_forward(tcnnb_model* m, tcnnb_stream stream, uint32_t n_elements, const float* input_dev, void* output_dev, const void* params_dev, int prepare_input_gradients) {
	TCNNB_API_BEGIN
	(void)prepare_input_gradients;  // nothing to prepare: backward recomputes the forward pass, including d(encoded)/d(position)
	module_forward(m->impl, (cudaStream_t)stream, n_elements, input_dev, output_dev, params_dev);
	TCNNB_API_END
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
	else if (k == "grid_replicas") m->impl.grid_replicas_override = value;
	else if (k == "general") {
		// the stand-alone kernels have their own limits (e.g. dL/d(encoded) wider than the layers): only switch when they cover the configuration
		if (value && !m->impl.general) {
			MlpBackwardArgs probe{};
			probe.width = m->impl.mlp.width;
			probe.in_width = m->impl.mlp.in_width;
			probe.out_width = m->impl.mlp.padded_out_width;
			probe.n_hidden_layers = m->impl.mlp.n_hidden_layers;
			probe.batch_size = 256;
			probe.dL_dinput = m->impl.grid.n_params == 0 ? nullptr : (__half*)16;
			const char* why_not = nullptr;
			if (!mlp_backward_supported(probe, &why_not)) throw std::runtime_error(std::string("tcnnb_debug_set(general): ") + why_not);
		}
		m->impl.force_general = value != 0;
	}  // general path: copies of the coarse levels' gradient (-1 = automatic)
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
