// An application's own loss through Trainer::training_step's full signature (include/tiny-cuda-nn/config.h): gradient accumulation
// over micro-batches. Each step draws 4 micro-batches; for each it runs network->inference, computes the L2 loss's dL/dy itself
// (x loss scale, fp16, padded width) and hands it over as external_dL_dy -- the first micro-batch with GradientMode::Overwrite, the
// others with Accumulate and run_optimizer = false -- and one optimizer_step follows. One more call passes every argument (data_pdf,
// dL_dinput, use_inference_params). Prints one JSON line that tests/test_gpu_trainer_ext.py checks.
#include <tiny-cuda-nn/config.h>

#include <cmath>
#include <cstdio>
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

// dL/dy of 0.5 * mean((y - t)^2) over n_total elements, x loss_scale, into fp16 rows of `padded` columns (padding zero)
__global__ void l2_dL_dy(uint32_t n_elements, uint32_t n_out, uint32_t padded, float scale, const float* __restrict__ y, const float* __restrict__ t, __half* __restrict__ dy) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_elements * padded) return;
	const uint32_t s = i / padded, c = i % padded;
	dy[i] = __float2half(c < n_out ? scale * (y[s * n_out + c] - t[s * n_out + c]) : 0.0f);
}

int main(int argc, char* argv[]) {
	try {
		const uint32_t n_steps = argc >= 2 ? atoi(argv[1]) : 50, n_micro = 4;
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
		GPUMatrix<float> x(n_in, batch), target(n_out, batch), y(n_out, batch), pdf(n_out, batch), dL_dinput(n_in, batch);
		GPUMatrix<precision_t> dL_dy(padded, batch);
		std::vector<float> host_y(n_out * batch), host_t(n_out * batch);

		auto draw = [&]() {
			generate_random_uniform<float>(stream, rng, batch * n_in, x.data());
			linear_kernel(eval_field, 0, stream, batch, x.data(), target.data());
		};
		auto l2 = [&]() {  // mean squared error of the current parameters on the current batch
			model.network->inference(stream, x, y);
			CUDA_CHECK_THROW(cudaMemcpyAsync(host_y.data(), y.data(), sizeof(float) * host_y.size(), cudaMemcpyDeviceToHost, stream));
			CUDA_CHECK_THROW(cudaMemcpyAsync(host_t.data(), target.data(), sizeof(float) * host_t.size(), cudaMemcpyDeviceToHost, stream));
			CUDA_CHECK_THROW(cudaStreamSynchronize(stream));
			double s = 0;
			for (size_t i = 0; i < host_y.size(); ++i) s += (double)(host_y[i] - host_t[i]) * (host_y[i] - host_t[i]);
			return s / host_y.size();
		};

		draw();
		const double first_loss = l2();
		const float scale = LOSS_SCALE / (float)(n_micro * batch * n_out);
		float ext_step_loss = -1.0f;
		for (uint32_t step = 0; step < n_steps; ++step) {
			for (uint32_t k = 0; k < n_micro; ++k) {
				draw();
				model.network->inference(stream, x, y);
				const uint32_t n = batch * padded;
				l2_dL_dy<<<(n + 255) / 256, 256, 0, stream>>>(batch, n_out, padded, scale, y.data(), target.data(), dL_dy.data());
				auto ctx = model.trainer->training_step(stream, x, target, nullptr, false, nullptr, false, k == 0 ? GradientMode::Overwrite : GradientMode::Accumulate, &dL_dy);
				ext_step_loss = model.trainer->loss(stream, *ctx);
			}
			model.trainer->optimizer_step(stream, LOSS_SCALE);
		}
		draw();
		const double last_loss = l2();

		// every argument at once: pdf-weighted loss, input gradients, inference parameters, no optimizer step
		linear_kernel(eval_field, 0, stream, batch, x.data(), pdf.data());  // values in [0, 1]: shift them away from 0 below
		std::vector<float> host_pdf(n_out * batch);
		CUDA_CHECK_THROW(cudaMemcpyAsync(host_pdf.data(), pdf.data(), sizeof(float) * host_pdf.size(), cudaMemcpyDeviceToHost, stream));
		CUDA_CHECK_THROW(cudaStreamSynchronize(stream));
		for (float& p : host_pdf) p = 0.5f + p;
		CUDA_CHECK_THROW(cudaMemcpy(pdf.data(), host_pdf.data(), sizeof(float) * host_pdf.size(), cudaMemcpyHostToDevice));
		auto ctx = model.trainer->training_step(stream, x, target, &pdf, false, &dL_dinput, true, GradientMode::Overwrite, nullptr);
		const float pdf_loss = model.trainer->loss(stream, *ctx);
		std::vector<float> host_dx(n_in * batch);
		CUDA_CHECK_THROW(cudaMemcpy(host_dx.data(), dL_dinput.data(), sizeof(float) * host_dx.size(), cudaMemcpyDeviceToHost));
		double dx_norm = 0;
		for (float v : host_dx) dx_norm += (double)v * v;

		// the shapes Trainer::training_step checks (trainer.h:127-138)
		std::string shape_error;
		try {
			GPUMatrix<precision_t> wrong(n_out, batch);
			model.trainer->training_step(stream, x, target, nullptr, true, nullptr, false, GradientMode::Overwrite, &wrong);
		} catch (const std::runtime_error& e) {
			shape_error = e.what();
		}
		CUDA_CHECK_THROW(cudaStreamSynchronize(stream));
		printf("{\"first_loss\": %g, \"last_loss\": %g, \"ext_step_loss\": %g, \"pdf_loss\": %g, \"dL_dinput_norm\": %g, \"shape_error\": \"%s\"}\n", first_loss, last_loss, ext_step_loss,
		       pdf_loss, std::sqrt(dx_norm), shape_error.c_str());
		CUDA_CHECK_THROW(cudaStreamDestroy(stream));
	} catch (const std::exception& e) {
		fprintf(stderr, "shim_trainer_ext: %s\n", e.what());
		return 1;
	}
	return 0;
}
