// ref_bwd_bwd -- drives the UNMODIFIED reference through tcnn::cpp::create_encoding and Module::backward_backward_input
// (its cpp_api.h:80, src/cpp_api.cu:118-134, grid.h:910-1042) and dumps inputs and outputs for tests/golden/bwdbwd_*.npz.
// TEST INFRASTRUCTURE ONLY: built by __graft_entry__.build() into oracle/_ref/ next to the reference library objects, run by
// tests/golden/make_golden_bwd_bwd.sh on a GPU. Nothing under tiny-cuda-nn_b200/ links or calls it.
//
//   ref_bwd_bwd <encoding.json> <n_input_dims> <batch> <seed> <out dir>
// (all levels active: the type-erased cpp::Module has no set_max_level)
// writes x.f32 [B][D], params.f16 [n_params], dL_doutput.f16 [B][width], dL_ddLdinput.f32 [B][D] (the inputs) and
// dL_dparams.f16, dL_ddLdoutput.f16 [B][width], dL_dinput.f32 [B][D] (the reference's results, all three asked at once), meta.json.
#include <tiny-cuda-nn/common_device.h>
#include <tiny-cuda-nn/cpp_api.h>
#include <tiny-cuda-nn/encoding.h>
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

__global__ void to_half(uint32_t n, const float* in, __half* out) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) out[i] = (__half)in[i];
}

int main(int argc, char** argv) {
	if (argc < 6) {
		std::fprintf(stderr, "usage: %s <encoding.json> <n_input_dims> <batch> <seed> <out dir>\n", argv[0]);
		return 1;
	}
	std::ifstream jf{argv[1]};
	const json config = json::parse(jf, nullptr, true, true);
	const uint32_t D = atoi(argv[2]), B = atoi(argv[3]);
	const uint32_t seed = atoi(argv[4]);
	const std::string out = argv[5];
	mkdir(out.c_str(), 0755);

	std::unique_ptr<cpp::Module> enc{cpp::create_encoding(D, config, cpp::Precision::Fp16)};
	const uint32_t width = enc->n_output_dims();
	const size_t n_params = enc->n_params();
	GPUMemory<float> params_fp32(n_params);
	GPUMemory<__half> params(n_params);
	enc->initialize_params(seed, params_fp32.data(), 50.0f);  // U(-5e-3, 5e-3): features well above fp16 denormals
	to_half<<<(uint32_t)((n_params + 255) / 256), 256>>>((uint32_t)n_params, params_fp32.data(), params.data());

	std::mt19937 rng{seed};
	std::uniform_real_distribution<float> unit{0.0f, 1.0f}, sym{-1.0f, 1.0f};
	std::vector<float> x(B * D), v(B * D);
	std::vector<__half> u((size_t)B * width);
	for (auto& e : x) e = unit(rng);
	for (auto& e : v) e = sym(rng);
	for (auto& e : u) e = (__half)(0.5f * sym(rng));
	GPUMemory<float> x_dev(x.size()), v_dev(v.size()), dinput(x.size());
	GPUMemory<__half> u_dev(u.size()), output(u.size()), ddoutput(u.size()), dparams(n_params);
	x_dev.copy_from_host(x);
	v_dev.copy_from_host(v);
	u_dev.copy_from_host(u);

	cpp::Context ctx = enc->forward(nullptr, B, x_dev.data(), output.data(), params.data(), true);
	enc->backward_backward_input(nullptr, ctx, B, v_dev.data(), x_dev.data(), u_dev.data(), dparams.data(), ddoutput.data(), dinput.data(), params.data());
	CUDA_CHECK_THROW(cudaDeviceSynchronize());

	write_bin(out + "/x.f32", x_dev.data(), x.size());
	write_bin(out + "/params.f16", params.data(), n_params);
	write_bin(out + "/dL_doutput.f16", u_dev.data(), u.size());
	write_bin(out + "/dL_ddLdinput.f32", v_dev.data(), v.size());
	write_bin(out + "/dL_dparams.f16", dparams.data(), n_params);
	write_bin(out + "/dL_ddLdoutput.f16", ddoutput.data(), u.size());
	write_bin(out + "/dL_dinput.f32", dinput.data(), x.size());
	json meta = {{"encoding", config}, {"n_input_dims", D}, {"batch", B}, {"width", width}, {"n_params", n_params}, {"seed", seed}};
	std::ofstream{out + "/meta.json"} << meta.dump(1);
	std::printf("%s: width %u, n_params %zu\n", out.c_str(), width, n_params);
	return 0;
}
