// ref_network_trainer -- drives the UNMODIFIED reference's Trainer over a bare network, Trainer(create_network<__half>(json), optimizer,
// loss, seed) (its trainer.h:51-87, src/network.cu:51-141), and dumps what tests/golden/net_trainer_*.npz holds.
// TEST INFRASTRUCTURE ONLY: built by __graft_entry__.build() into oracle/_ref/ next to the reference library objects, run by
// tests/golden/make_golden_net_trainer.sh on a GPU. Nothing under tiny-cuda-nn_b200/ links or calls it.
//
//   ref_network_trainer <otype> <n_neurons> <n_hidden_layers> <batch> <seed> <out dir>
// 32 fp16 inputs x ~ U[0,1), 32 fp32 targets ~ U[0.2,1) (std::mt19937{seed}), RelativeL2, Adam (lr 1e-2, beta 0.9 / 0.99, eps 1e-15,
// l2 1e-6), trainer seed 1337. Ten steps, each training_step(run_optimizer = false), Trainer::loss(ctx), then optimizer_step. Writes
// x.f16 ([batch][32]), y.f32, params_init.f32 (params_full_precision after construction), grads.f16 (the gradient buffer after the
// first step, x loss scale 128), losses.f32 (10) and meta.json.
#include <tiny-cuda-nn/common_device.h>
#include <tiny-cuda-nn/config.h>
#include <tiny-cuda-nn/gpu_memory.h>
#include <tiny-cuda-nn/network.h>
#include <tiny-cuda-nn/trainer.h>

#include <cstdio>
#include <fstream>
#include <random>
#include <string>
#include <sys/stat.h>
#include <vector>

using namespace tcnn;
using T = network_precision_t;

template <typename X>
static void write_bin(const std::string& path, const X* dev, size_t n) {
	std::vector<X> h(n);
	CUDA_CHECK_THROW(cudaMemcpy(h.data(), dev, n * sizeof(X), cudaMemcpyDeviceToHost));
	std::ofstream f{path, std::ios::binary};
	f.write((const char*)h.data(), n * sizeof(X));
}

int main(int argc, char** argv) {
	if (argc < 7) {
		std::fprintf(stderr, "usage: %s <otype> <n_neurons> <n_hidden_layers> <batch> <seed> <out dir>\n", argv[0]);
		return 1;
	}
	const uint32_t n_in = 32, n_out = 32, B = atoi(argv[4]), seed = atoi(argv[5]), n_steps = 10;
	const std::string out = argv[6];
	mkdir(out.c_str(), 0755);
	const json network_opts = {{"otype", argv[1]}, {"n_input_dims", n_in}, {"n_output_dims", n_out}, {"n_neurons", atoi(argv[2])}, {"n_hidden_layers", atoi(argv[3])},
	                           {"activation", "ReLU"}, {"output_activation", "None"}};
	const json loss_opts = {{"otype", "RelativeL2"}};
	const json optimizer_opts = {{"otype", "Adam"}, {"learning_rate", 1e-2}, {"beta1", 0.9}, {"beta2", 0.99}, {"epsilon", 1e-15}, {"l2_reg", 1e-6}};
	try {
		std::shared_ptr<Loss<T>> loss{create_loss<T>(loss_opts)};
		std::shared_ptr<Optimizer<T>> optimizer{create_optimizer<T>(optimizer_opts)};
		std::shared_ptr<Network<T>> network{create_network<T>(network_opts)};
		auto trainer = std::make_shared<Trainer<T, T, T>>(network, optimizer, loss, 1337u);

		std::mt19937 rng{seed};
		std::uniform_real_distribution<float> unit{0.0f, 1.0f};
		std::vector<T> x((size_t)B * n_in);
		std::vector<float> y((size_t)B * n_out);
		for (auto& e : x) e = (T)unit(rng);
		for (auto& e : y) e = 0.2f + 0.8f * unit(rng);
		GPUMatrix<T> x_dev(n_in, B);
		GPUMatrix<float> y_dev(n_out, B);
		CUDA_CHECK_THROW(cudaMemcpy(x_dev.data(), x.data(), x.size() * sizeof(T), cudaMemcpyHostToDevice));
		CUDA_CHECK_THROW(cudaMemcpy(y_dev.data(), y.data(), y.size() * sizeof(float), cudaMemcpyHostToDevice));

		const size_t n_params = trainer->n_params();
		write_bin(out + "/x.f16", x_dev.data(), x.size());
		write_bin(out + "/y.f32", y_dev.data(), y.size());
		write_bin(out + "/params_init.f32", trainer->params_full_precision(), n_params);
		std::vector<float> losses;
		for (uint32_t i = 0; i < n_steps; ++i) {
			auto ctx = trainer->training_step(nullptr, x_dev, y_dev, nullptr, false);
			losses.push_back(trainer->loss(nullptr, *ctx));
			if (i == 0) write_bin(out + "/grads.f16", trainer->param_gradients(), n_params);
			trainer->optimizer_step(nullptr, default_loss_scale<T>());
		}
		CUDA_CHECK_THROW(cudaDeviceSynchronize());
		std::ofstream{out + "/losses.f32", std::ios::binary}.write((const char*)losses.data(), losses.size() * sizeof(float));
		const json meta = {{"network", network_opts}, {"loss", loss_opts}, {"optimizer", optimizer_opts}, {"n_input_dims", n_in}, {"n_output_dims", n_out},
		                   {"padded_output_width", network->padded_output_width()}, {"batch", B}, {"n_params", n_params}, {"seed", seed}, {"trainer_seed", 1337}};
		std::ofstream{out + "/meta.json"} << meta.dump(1);
		std::printf("%s: n_params %zu, losses %f -> %f\n", out.c_str(), n_params, losses.front(), losses.back());
	} catch (const std::exception& e) {
		std::fprintf(stderr, "ref_network_trainer: %s\n", e.what());
		return 2;
	}
	return 0;
}
