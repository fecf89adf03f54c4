// optimizer.h -- the trainer's optimizer: Adam (optimizers/adam.h) inside any nesting of ExponentialDecay and Ema, with its state and
// its step-counter layout. Host code; the kernels are misc_kernels.cu's.
#pragma once
#include "host_common.h"
#include "json_mini.h"
#include "misc_kernels.h"

namespace tcnnb {

// What the trainer hands the optimizer: whole-vector fp32 masters, fp16 weights and fp16 gradients, the fp32 sums that replace the
// gradients of the first n_matrix (network) weights or null, and the loss scale.
struct OptimizerArrays {
	float* masters;
	__half* weights;
	__half* gradients;
	float* dw_sums;
	uint32_t n_matrix;
	float loss_scale;
};

class Optimizer {
public:
	explicit Optimizer(const json::Value& cfg);  // the "optimizer" JSON (src/optimizer.cu:50-80, adam.h:221-303); no state yet
	// Moments and step counters for n_params parameters; the Ema average starts as `working` ([n_params_padded]).
	void allocate(size_t n_params, size_t n_params_padded, const __half* working);
	bool allocated() const { return n_params_ != 0; }

	// One step over the ranges [begin, begin + count) (all parameters when n_ranges == 0), then Ema's. Returns whether it covered the
	// network weights.
	bool step(cudaStream_t stream, const OptimizerArrays& arrays, uint32_t n_ranges, const uint64_t* begins, const uint64_t* counts);
	// One step over the slice [lo, lo + chunk) of the peer-memory data-parallel engine.
	void step_peers(cudaStream_t stream, const DpPeers& peers, uint64_t lo, uint64_t chunk, const OptimizerArrays& arrays);
	void skip_step() { (void)next_params(); }  // an empty slice: the step count and the decay schedule advance all the same

	// Trainer::params_inference() (trainer.h:401-403); the average restarts from the working weights (trainer.h:415-419, 428-429).
	const __half* inference_params(const __half* working) const { return ema_.enabled ? ema_fp16_.ptr : working; }
	void reset_average(const __half* working) {
		if (ema_.enabled) TCNNB_CUDA_CHECK(cudaMemcpy(ema_fp16_.ptr, working, sizeof(__half) * n_params_padded_, cudaMemcpyDeviceToDevice));
	}
	bool has_average() const { return ema_.enabled; }

	// The counters as uint32: the state itself, or a mirror of 16-bit counters, widened on `stream` unless it is live already. A live
	// mirror is authoritative until counters_written() narrows it back (saturating: exact, see adam_u16_steps_exact).
	uint32_t* counters_u32(cudaStream_t stream);
	void counters_written(cudaStream_t stream);
	void load_counters_u32(const uint32_t* host);  // [n_params]
	void set_counter_width(bool force32);           // 16-bit counters when they are exact and not force32; counts carry over. Synchronous.

	// The step count (the decay factor follows it) and base learning rate set from outside, after the caller may have written the
	// counters through counters_u32().
	void restore_progress(uint32_t step, float base_learning_rate);
	float learning_rate_factor() const { return lr_decay_.factor; }  // ExponentialDecay's (exponential_decay.h:136-148), else 1
	void set_learning_rate_factor(float factor) {
		if (!lr_decay_.enabled) throw std::runtime_error("set_learning_rate_factor: the optimizer has no ExponentialDecay wrapper.");
		lr_decay_.factor = factor;
	}
	uint32_t step_count() const { return step_count_; }
	float base_learning_rate() const { return adam_.learning_rate; }
	float* first_moments() const { return first_moments_.ptr; }
	float* second_moments() const { return second_moments_.ptr; }
	void write_hyperparams(json::Value& opt) const;

private:
	AdamParams next_params();
	float lr_decay_factor_after(uint32_t n_steps) const;
	template <typename F>
	void with_counters(F&& f) {  // the Adam kernels are instantiated for both counter widths
		if (steps16_) f(steps16_buf_.ptr);
		else f(steps32_buf_.ptr);
	}

	AdamParams adam_;
	uint32_t step_count_ = 0;
	struct {  // ExponentialDecay wrapper (optimizers/exponential_decay.h)
		bool enabled = false;
		float base = 0.1f, factor = 1.0f;
		uint32_t interval = 10000, start = 10000, end = 10000000;
	} lr_decay_;
	struct {  // Ema wrapper (optimizers/ema.h:46-200): exponential moving average of the working weights, used by inference
		bool enabled = false, full_precision = false;
		float decay = 0.99f;
	} ema_;
	size_t n_params_ = 0, n_params_padded_ = 0;
	DeviceBuffer<float> first_moments_, second_moments_;
	// Per-parameter step counters: 16-bit (saturating at 65535) when adam_u16_steps_exact() proves the updates identical, else 32-bit;
	// steps32_buf_ is then the mirror.
	bool steps16_ = false, mirror_live_ = false;
	DeviceBuffer<uint16_t> steps16_buf_;
	DeviceBuffer<uint32_t> steps32_buf_;
	DeviceBuffer<__half> ema_fp16_;  // trainer.h:497-502
	DeviceBuffer<float> ema_tmp_;
};

}  // namespace tcnnb
