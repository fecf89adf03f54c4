// ref_trainer_split -- drives the UNMODIFIED reference through tcnn::create_from_config, Trainer::forward and Trainer::backward (its
// trainer.h:89-153) and dumps inputs and outputs for tests/golden/split_*.npz.
// TEST INFRASTRUCTURE ONLY: built by __graft_entry__.build() into oracle/_ref/ next to the reference library objects, run by
// tests/golden/make_golden_split.sh on a GPU. Nothing under tiny-cuda-nn_b200/ links or calls it.
//
//   ref_trainer_split <config.json> <loss otype> <n_neurons> <output activation> <batch> <seed> <with pdf 0/1> <out dir>
// forward(loss scale 128, x ~ U[0,1)^3, targets ~ U[0.2,1), pdf ~ U[0.2,5] when asked) and backward(GradientMode::Overwrite) on
// the trainer's initial parameters. Writes x.f32, y.f32, pdf.f32 (with pdf), params.f16, output.f16, L.f32 and dL_doutput.f16
// ([batch][padded_output_width] each: the ForwardContext), grads.f16 (the gradient buffer after backward), loss.f32
// (Trainer::loss(ctx)) and meta.json.
#include <tiny-cuda-nn/common_device.h>
#include <tiny-cuda-nn/config.h>
#include <tiny-cuda-nn/gpu_memory.h>

#include <cstdio>
#include <fstream>
#include <random>
#include <string>
#include <sys/stat.h>
#include <vector>

using namespace tcnn;

template <typename T>
static void write_bin(const std::string& path, const T* dev, size_t n) {
	std::vector<T> h(n);
	CUDA_CHECK_THROW(cudaMemcpy(h.data(), dev, n * sizeof(T), cudaMemcpyDeviceToHost));
	std::ofstream f{path, std::ios::binary};
	f.write((const char*)h.data(), n * sizeof(T));
}

int main(int argc, char** argv) {
	if (argc < 9) {
		std::fprintf(stderr, "usage: %s <config.json> <loss otype> <n_neurons> <output activation> <batch> <seed> <with pdf 0/1> <out dir>\n", argv[0]);
		return 1;
	}
	std::ifstream jf{argv[1]};
	json config = json::parse(jf, nullptr, true, true);
	config["loss"] = {{"otype", argv[2]}};
	config["network"]["n_neurons"] = atoi(argv[3]);
	config["network"]["output_activation"] = argv[4];
	const uint32_t B = atoi(argv[5]), seed = atoi(argv[6]), n_in = 3, n_out = 3;
	const bool with_pdf = atoi(argv[7]) != 0;
	const std::string out = argv[8];
	mkdir(out.c_str(), 0755);

	TrainableModel model = create_from_config(n_in, n_out, config);
	std::mt19937 rng{seed};
	std::uniform_real_distribution<float> unit{0.0f, 1.0f};
	std::vector<float> x(B * n_in), y(B * n_out), pdf(B * n_out);
	for (auto& e : x) e = unit(rng);
	for (auto& e : y) e = 0.2f + 0.8f * unit(rng);
	for (auto& e : pdf) e = 0.2f + 4.8f * unit(rng);
	GPUMatrix<float> x_dev(n_in, B), y_dev(n_out, B), pdf_dev(n_out, B);
	CUDA_CHECK_THROW(cudaMemcpy(x_dev.data(), x.data(), x.size() * sizeof(float), cudaMemcpyHostToDevice));
	CUDA_CHECK_THROW(cudaMemcpy(y_dev.data(), y.data(), y.size() * sizeof(float), cudaMemcpyHostToDevice));
	CUDA_CHECK_THROW(cudaMemcpy(pdf_dev.data(), pdf.data(), pdf.size() * sizeof(float), cudaMemcpyHostToDevice));

	const size_t n_params = model.trainer->n_params();
	const uint32_t padded = model.network->padded_output_width();
	write_bin(out + "/params.f16", model.trainer->params(), n_params);
	auto ctx = model.trainer->forward(nullptr, default_loss_scale<network_precision_t>(), x_dev, y_dev, with_pdf ? &pdf_dev : nullptr);
	model.trainer->backward(nullptr, *ctx, x_dev);
	const float loss = model.trainer->loss(nullptr, *ctx);
	CUDA_CHECK_THROW(cudaDeviceSynchronize());

	write_bin(out + "/x.f32", x_dev.data(), x.size());
	write_bin(out + "/y.f32", y_dev.data(), y.size());
	if (with_pdf) write_bin(out + "/pdf.f32", pdf_dev.data(), pdf.size());
	write_bin(out + "/output.f16", ctx->output.data(), (size_t)padded * B);
	write_bin(out + "/L.f32", ctx->L.data(), (size_t)padded * B);
	write_bin(out + "/dL_doutput.f16", ctx->dL_doutput.data(), (size_t)padded * B);
	write_bin(out + "/grads.f16", model.trainer->param_gradients(), n_params);
	std::ofstream{out + "/loss.f32", std::ios::binary}.write((const char*)&loss, sizeof(float));
	json meta = {{"config", config}, {"n_input_dims", n_in}, {"n_output_dims", n_out}, {"padded_output_width", padded}, {"batch", B}, {"n_params", n_params}, {"seed", seed},
	             {"with_pdf", with_pdf}, {"loss", loss}};
	std::ofstream{out + "/meta.json"} << meta.dump(1);
	std::printf("%s: n_params %zu, loss %g\n", out.c_str(), n_params, loss);
	return 0;
}
