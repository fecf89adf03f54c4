// optimizer.cu -- the trainer's optimizer (optimizer.h): JSON, state, step sequence and step-counter layout. Defines no kernels: it
// launches the optimizer kernels of misc_kernels.cu.
#include "optimizer.h"

#include <cmath>
#include <limits>

namespace tcnnb {

Optimizer::Optimizer(const json::Value& cfg) {
	const json::Value* opt_ptr = &cfg;
	std::string opt_name = opt_ptr->value("otype", "Adam");
	// wrappers around the nested optimizer, in any order: ExponentialDecay (a learning-rate schedule) and Ema (averaged inference weights)
	while (ieq(opt_name, "ExponentialDecay") || ieq(opt_name, "Ema")) {
		if (ieq(opt_name, "ExponentialDecay")) {
			// optimizers/exponential_decay.h:46-160: from step decay_start on, every decay_interval steps (until decay_end) the learning
			// rate is multiplied by decay_base. Host-side bookkeeping only.
			if (lr_decay_.enabled) throw std::runtime_error("tcnn_b200: one ExponentialDecay wrapper per optimizer");
			lr_decay_.enabled = true;
			lr_decay_.base = (float)opt_ptr->value("decay_base", 0.1);
			lr_decay_.interval = (uint32_t)opt_ptr->value("decay_interval", 10000.0);
			lr_decay_.start = (uint32_t)opt_ptr->value("decay_start", 10000.0);
			lr_decay_.end = (uint32_t)opt_ptr->value("decay_end", 10000000.0);
			if (lr_decay_.interval == 0) throw std::runtime_error("ExponentialDecay: decay_interval must be positive.");
		} else {
			// optimizers/ema.h:46-200: after every step of the nested optimizer, ema = (ema * decay * (1 - decay^(t-1)) + w * (1 - decay)) /
			// (1 - decay^t) on the working-precision weights; network->inference() reads the average (Trainer::params_inference).
			if (ema_.enabled) throw std::runtime_error("tcnn_b200: one Ema wrapper per optimizer");
			ema_.enabled = true;
			ema_.decay = (float)opt_ptr->value("decay", 0.99);
			ema_.full_precision = opt_ptr->value("full_precision", false);
		}
		opt_ptr = &opt_ptr->sub("nested");
		opt_name = opt_ptr->value("otype", "Adam");
	}
	const json::Value& opt = *opt_ptr;
	if (!ieq(opt_name, "Adam")) {
		throw std::runtime_error("Optimizer '" + opt_name + "' is outside the tcnn_b200 hot path (Adam, optionally inside ExponentialDecay and / or Ema, is built)");
	}
	AdamParams& a = adam_;
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
}

void Optimizer::allocate(size_t n_params, size_t n_params_padded, const __half* working) {
	n_params_ = n_params;
	n_params_padded_ = n_params_padded;
	first_moments_.resize(n_params);
	first_moments_.zero();
	second_moments_.resize(n_params);
	second_moments_.zero();
	set_counter_width(false);
	if (ema_.enabled) {  // trainer.h:409-421: the inference parameters start as the initial parameters
		ema_fp16_.resize(n_params_padded);
		reset_average(working);
		if (ema_.full_precision) {
			ema_tmp_.resize(n_params);
			ema_tmp_.zero();
		}
	}
}

// ExponentialDecay's learning-rate factor after `n_steps` uninterrupted steps: the schedule of next_params replayed with the same float
// multiplications, so that a trainer whose step count is restored continues bit-identically. Each decay boundary is visited once; the
// loop stops early once a multiplication no longer changes the factor (0, 1 or a saturated value).
float Optimizer::lr_decay_factor_after(uint32_t n_steps) const {
	float factor = 1.0f;
	if (!lr_decay_.enabled || n_steps == 0) return factor;
	const uint64_t last = std::min<uint64_t>((uint64_t)n_steps - 1, lr_decay_.end);
	for (uint64_t step = lr_decay_.start; step <= last; step += lr_decay_.interval) {
		const float next = factor * lr_decay_.base;
		if (next == factor) break;
		factor = next;
	}
	return factor;
}

// Hyper-parameters of the next optimizer step (advances the step count; AdaBound bounds per adam.h:161-168).
AdamParams Optimizer::next_params() {
	if (lr_decay_.enabled) {  // exponential_decay.h:60-70, evaluated with the step count BEFORE this step
		const uint32_t step = step_count_;
		if (step == 0) lr_decay_.factor = 1.0f;
		if (step >= lr_decay_.start && (step - lr_decay_.start) % lr_decay_.interval == 0 && step <= lr_decay_.end) lr_decay_.factor *= lr_decay_.base;
	}
	++step_count_;
	AdamParams a = adam_;
	a.learning_rate = adam_.learning_rate * lr_decay_.factor;
	a.lower_lr_bound = 0;
	a.upper_lr_bound = std::numeric_limits<float>::max();
	if (a.adabound) {
		a.lower_lr_bound = 0.1f - 0.1f / ((1 - a.beta2) * (float)step_count_ + 1);
		a.upper_lr_bound = 0.1f + 0.1f / ((1 - a.beta2) * (float)step_count_);
	}
	return a;
}

// One optimizer step whatever the number of ranges: the data-parallel trainer updates the network weights everywhere and the grid
// entries of its own shard only.
bool Optimizer::step(cudaStream_t stream, const OptimizerArrays& arrays, uint32_t n_ranges, const uint64_t* begins, const uint64_t* counts) {
	counters_written(stream);
	const AdamParams a = next_params();
	const uint64_t whole_begin = 0, whole_count = n_params_;
	if (n_ranges == 0) {
		n_ranges = 1;
		begins = &whole_begin;
		counts = &whole_count;
	}
	const uint32_t n_mlp = arrays.n_matrix;
	bool covers_mlp = false;
	for (uint32_t r = 0; r < n_ranges; ++r) {
		const uint64_t b = begins[r], c = counts[r];
		if (b + c > n_params_) throw std::runtime_error("optimizer_step: parameter range out of bounds.");
		if (c == 0) continue;
		if (b < n_mlp && b + c < n_mlp) throw std::runtime_error("optimizer_step: a range may not split the network weights.");
		const uint32_t n_matrix = b < n_mlp ? (uint32_t)(n_mlp - b) : 0u;  // matrix weights inside this range
		covers_mlp |= b == 0 && n_matrix > 0;
		if (n_matrix > 0 && b != 0) throw std::runtime_error("optimizer_step: the network weights must be covered from parameter 0.");
		float* const dw = n_matrix > 0 ? arrays.dw_sums : nullptr;
		with_counters([&](auto* steps) {
			TCNNB_CUDA_CHECK(launch_adam_step(stream, a, (uint32_t)c, n_matrix, arrays.loss_scale, arrays.masters + b, arrays.weights + b, arrays.gradients + b, dw,
			                                  first_moments_.ptr + b, second_moments_.ptr + b, steps + b));
		});
		++g_kernel_launches;
	}
	if (ema_.enabled) {
		if (n_ranges != 1 || begins[0] != 0 || counts[0] != n_params_) throw std::runtime_error("tcnn_b200: the Ema wrapper is built for whole-vector optimizer steps (not for the sharded data-parallel optimizer)");
		const float t = (float)step_count_;
		TCNNB_CUDA_CHECK(launch_ema_step(stream, (uint32_t)n_params_, ema_.decay, 1.0f - std::pow(ema_.decay, t - 1.0f), 1.0f / (1.0f - std::pow(ema_.decay, t)), arrays.weights, ema_fp16_.ptr,
		                                 ema_.full_precision ? ema_tmp_.ptr : nullptr));
		++g_kernel_launches;
	}
	return covers_mlp;
}

void Optimizer::step_peers(cudaStream_t stream, const DpPeers& peers, uint64_t lo, uint64_t chunk, const OptimizerArrays& arrays) {
	counters_written(stream);
	const AdamParams a = next_params();
	with_counters([&](auto* steps) {
		TCNNB_CUDA_CHECK(launch_adam_step_dp(stream, a, peers, lo, chunk, arrays.n_matrix, n_params_, arrays.loss_scale, arrays.masters, first_moments_.ptr, second_moments_.ptr, steps));
	});
	++g_kernel_launches;
}

uint32_t* Optimizer::counters_u32(cudaStream_t stream) {
	if (steps16_ && !mirror_live_) {
		steps32_buf_.resize(n_params_);
		TCNNB_CUDA_CHECK(launch_widen_steps(stream, n_params_, steps16_buf_.ptr, steps32_buf_.ptr));
		mirror_live_ = true;
	}
	return steps32_buf_.ptr;
}

void Optimizer::counters_written(cudaStream_t stream) {
	if (steps16_ && mirror_live_) {
		TCNNB_CUDA_CHECK(launch_narrow_steps(stream, n_params_, steps32_buf_.ptr, steps16_buf_.ptr));
		mirror_live_ = false;
	}
}

void Optimizer::load_counters_u32(const uint32_t* host) {
	if (steps16_) steps32_buf_.resize(n_params_);
	TCNNB_CUDA_CHECK(cudaMemcpy(steps32_buf_.ptr, host, n_params_ * sizeof(uint32_t), cudaMemcpyHostToDevice));
	mirror_live_ = steps16_;
	counters_written(nullptr);
}

void Optimizer::set_counter_width(bool force32) {
	bool use16 = false;
	if (!force32) TCNNB_CUDA_CHECK(adam_u16_steps_exact(adam_, &use16));
	const size_t n = n_params_;
	if (use16 == steps16_ && (use16 ? steps16_buf_.n : steps32_buf_.n) == n) return;
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	if (use16) {
		const bool carry = steps32_buf_.n == n;
		steps16_buf_.resize(n);
		if (carry) TCNNB_CUDA_CHECK(launch_narrow_steps(nullptr, n, steps32_buf_.ptr, steps16_buf_.ptr));
		else steps16_buf_.zero();
		steps32_buf_.release();
	} else {
		steps32_buf_.resize(n);
		if (steps16_buf_.n == n) {
			if (!mirror_live_) TCNNB_CUDA_CHECK(launch_widen_steps(nullptr, n, steps16_buf_.ptr, steps32_buf_.ptr));
		} else {
			steps32_buf_.zero();
		}
		steps16_buf_.release();
	}
	steps16_ = use16;
	mirror_live_ = false;
	TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
}

void Optimizer::restore_progress(uint32_t step, float base_learning_rate) {
	if (allocated()) {
		counters_written(nullptr);
		TCNNB_CUDA_CHECK(cudaDeviceSynchronize());
	}
	step_count_ = step;
	lr_decay_.factor = lr_decay_factor_after(step);
	adam_.learning_rate = base_learning_rate;
}

void Optimizer::write_hyperparams(json::Value& opt) const {
	opt["otype"] = json::Value::string("Adam");
	opt["learning_rate"] = json::Value::number(adam_.learning_rate);
	opt["beta1"] = json::Value::number(adam_.beta1);
	opt["beta2"] = json::Value::number(adam_.beta2);
	opt["epsilon"] = json::Value::number(adam_.epsilon);
	opt["l2_reg"] = json::Value::number(adam_.l2_reg);
}

}  // namespace tcnnb
