// A training step split into Trainer::forward / backward (include/tiny-cuda-nn/config.h, declared as in trainer.h:89-157), the way
// applications use it when they need the step's predictions or per-sample losses:
//   - training: forward, the per-element losses ctx->L read on the host (what NRC-style code picks its next samples from) and
//     summed by loss(ctx), backward, optimizer_step;
//   - the application's own loss: forward with external_dL_dy, the gradient written into that buffer from ctx->output, backward with
//     dL_dinput.
// Prints one JSON line that tests/test_gpu_trainer_split.py checks.
#include <tiny-cuda-nn/config.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <memory>
#include <vector>

using namespace tcnn;
using precision_t = network_precision_t;

__global__ void eval_field(uint32_t n_elements, const float* __restrict__ xyz, float* __restrict__ result) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_elements) return;
	const float x = xyz[i * 3 + 0], y = xyz[i * 3 + 1], z = xyz[i * 3 + 2];
	result[i * 3 + 0] = 0.5f + 0.5f * __sinf(9.0f * x) * __cosf(7.0f * y);
	result[i * 3 + 1] = x * z;
	result[i * 3 + 2] = 0.5f + 0.5f * __cosf(11.0f * (y - z));
}

// dL/dy of 0.5 * mean((y - t)^2) x loss scale from the padded fp16 predictions, into the padded fp16 gradient (padding zero)
__global__ void l2_dL_dy(uint32_t n_elements, uint32_t n_out, uint32_t padded, float scale, const precision_t* __restrict__ y, const float* __restrict__ t, precision_t* __restrict__ dy) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_elements * padded) return;
	const uint32_t s = i / padded, c = i % padded;
	dy[i] = (precision_t)(c < n_out ? scale * ((float)y[i] - t[s * n_out + c]) : 0.0f);
}

int main(int argc, char* argv[]) {
	try {
		const uint32_t n_steps = argc >= 2 ? atoi(argv[1]) : 50;
		json config = {
			{"loss", {{"otype", "L2"}}},
			{"optimizer", {{"otype", "Adam"}, {"learning_rate", 1e-2}, {"beta1", 0.9}, {"beta2", 0.99}, {"epsilon", 1e-15}}},
			{"encoding", {{"otype", "HashGrid"}, {"n_levels", 16}, {"n_features_per_level", 2}, {"log2_hashmap_size", 15}, {"base_resolution", 16}, {"per_level_scale", 1.5}}},
			{"network", {{"otype", "FullyFusedMLP"}, {"activation", "ReLU"}, {"output_activation", "None"}, {"n_neurons", 64}, {"n_hidden_layers", 2}}},
		};
		const uint32_t batch = 1 << 14, n_in = 3, n_out = 3;
		TrainableModel model = create_from_config(n_in, n_out, config);
		const uint32_t padded = model.network->padded_output_width();

		cudaStream_t stream;
		CUDA_CHECK_THROW(cudaStreamCreate(&stream));
		default_rng_t rng{1337};
		GPUMatrix<float> x(n_in, batch), target(n_out, batch), dL_dinput(n_in, batch);
		GPUMatrix<precision_t> dL_dy(padded, batch);
		auto draw = [&]() {
			generate_random_uniform<float>(stream, rng, batch * n_in, x.data());
			linear_kernel(eval_field, 0, stream, batch, x.data(), target.data());
		};

		float first_loss = 0, last_loss = 0;
		double max_rel_sum_error = 0;
		uint32_t worst_sample = 0;
		std::vector<float> host_L(padded * batch);
		for (uint32_t step = 0; step < n_steps; ++step) {
			draw();
			std::unique_ptr<Trainer<float, precision_t, precision_t>::ForwardContext> ctx = model.trainer->forward(stream, LOSS_SCALE, x, target);
			const float loss = model.trainer->loss(stream, *ctx);
			CUDA_CHECK_THROW(cudaMemcpyAsync(host_L.data(), ctx->L.data(), sizeof(float) * host_L.size(), cudaMemcpyDeviceToHost, stream));
			CUDA_CHECK_THROW(cudaStreamSynchronize(stream));
			double sum = 0, worst = -1;
			for (uint32_t i = 0; i < batch; ++i) {
				double sample = 0;
				for (uint32_t c = 0; c < padded; ++c) sample += host_L[i * padded + c];
				if (sample > worst) worst = sample, worst_sample = i;
				sum += sample;
			}
			max_rel_sum_error = std::max(max_rel_sum_error, std::abs(sum - loss) / sum);
			if (step == 0) first_loss = loss;
			last_loss = loss;
			model.trainer->backward(stream, *ctx, x);
			model.trainer->optimizer_step(stream, LOSS_SCALE);
		}

		// own loss: the context's dL_doutput is the caller's buffer, filled from the context's predictions before backward
		draw();
		auto ctx = model.trainer->forward(stream, LOSS_SCALE, x, target, nullptr, false, true, &dL_dy);
		const bool is_view = ctx->dL_doutput.data() == dL_dy.data() && ctx->dL_doutput.m() == padded && ctx->dL_doutput.n() == batch;
		const uint32_t n = batch * padded;
		l2_dL_dy<<<(n + 255) / 256, 256, 0, stream>>>(batch, n_out, padded, LOSS_SCALE / (float)(batch * n_out), ctx->output.data(), target.data(), dL_dy.data());
		model.trainer->backward(stream, *ctx, x, &dL_dinput, false, GradientMode::Overwrite);
		const float ext_loss = model.trainer->loss(*ctx);
		std::vector<float> host_dx(n_in * batch);
		CUDA_CHECK_THROW(cudaMemcpy(host_dx.data(), dL_dinput.data(), sizeof(float) * host_dx.size(), cudaMemcpyDeviceToHost));
		double dx_norm = 0;
		for (float v : host_dx) dx_norm += (double)v * v;
		model.trainer->optimizer_step(stream, LOSS_SCALE);
		CUDA_CHECK_THROW(cudaStreamSynchronize(stream));
		printf("{\"first_loss\": %g, \"last_loss\": %g, \"max_rel_sum_error\": %g, \"worst_sample\": %u, \"view\": %s, \"ext_loss\": %g, \"dL_dinput_norm\": %g}\n", first_loss,
		       last_loss, max_rel_sum_error, worst_sample, is_view ? "true" : "false", ext_loss, std::sqrt(dx_norm));
		CUDA_CHECK_THROW(cudaStreamDestroy(stream));
	} catch (const std::exception& e) {
		fprintf(stderr, "shim_trainer_split: %s\n", e.what());
		return 1;
	}
	return 0;
}
