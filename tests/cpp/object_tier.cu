// The C++ object tier (include/tiny-cuda-nn/object.h, network.h, encoding.h, network_with_input_encoding.h, trainer.h) against the C ABI
// tiers it sits on. Each check prints one line "ok <name>" or "FAIL <name>: <why>"; the exit code is the number of failures.
//   network_<otype>:        Network<__half> of create_network -- inference_mixed_precision, forward and dL/dinput bit-equal to the network
//                           tier on the same parameters, dL/dparams up to the order of its atomic sums; row-major matrices bit-equal to column-major ones; inference (fp32) within 1e-4 RAE
//                           of inference_mixed_precision; the trainer's initial parameters equal the network tier's from pcg32{seed_seq}.
//   trainer_<otype>:        a Trainer over the network trains (the loss falls), the object's own inference runs on the trained weights,
//                           row-major inputs give Trainer::forward the same predictions bit for bit, and row-major inputs and targets
//                           train like column-major ones (losses within 1e-3 over ten steps: the weight-gradient and loss sums are atomic).
//   composed_vs_config:     NetworkWithInputEncoding(create_encoding, create_network) trains like create_from_config of the same JSON:
//                           bit-equal initial parameters, the same launches per step, the step-0 loss within 1e-4, the five-step trajectory
//                           within 1e-3 (DESIGN.md section 5.0a: the fp16 scatter atomics of the table gradients), and the component objects
//                           read their parts of the trainer's parameters.
//   not_built:              training an Encoding alone and Encoding::inference with fp32 outputs report "not built".
// tests/test_gpu_object_tier.py runs it.
#include <tiny-cuda-nn/config.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <memory>
#include <random>
#include <string>
#include <vector>

using namespace tcnn;
using T = network_precision_t;

static int g_failures = 0;
static void report(const std::string& name, bool ok, const std::string& why = "") {
	if (ok) std::printf("ok %s\n", name.c_str());
	else std::printf("FAIL %s: %s\n", name.c_str(), why.c_str());
	g_failures += ok ? 0 : 1;
}

template <typename X>
static std::vector<X> host(const X* dev, size_t n) {
	std::vector<X> v(n);
	CUDA_CHECK_THROW(cudaMemcpy(v.data(), dev, n * sizeof(X), cudaMemcpyDeviceToHost));
	return v;
}
template <typename X>
static bool same_bits(const std::vector<X>& a, const std::vector<X>& b) { return a.size() == b.size() && std::memcmp(a.data(), b.data(), a.size() * sizeof(X)) == 0; }

// [rows][cols] -> [cols][rows]
template <typename X>
static std::vector<X> transposed(const std::vector<X>& v, uint32_t rows, uint32_t cols) {
	std::vector<X> t(v.size());
	for (uint32_t r = 0; r < rows; ++r)
		for (uint32_t c = 0; c < cols; ++c) t[(size_t)c * rows + r] = v[(size_t)r * cols + c];
	return t;
}

// Weight gradients: the weight-gradient kernel adds each CTA's fp32 partial sums with red.global.add, so two runs may round a sum to a
// neighbouring fp16 value. Close: at most 0.1 % of the entries differ by more than 2e-3 relative.
static bool grads_close(const std::vector<T>& a, const std::vector<T>& b) {
	if (a.size() != b.size()) return false;
	size_t off = 0;
	for (size_t i = 0; i < a.size(); ++i) {
		const float x = (float)a[i], y = (float)b[i];
		if (std::abs(x - y) > 2e-3f * std::max(std::abs(x), std::abs(y)) + 1e-7f) ++off;
	}
	return off <= a.size() / 1000;
}

// the largest symmetric relative absolute error of test_common.h's vector_match_rae
static double max_rae(const std::vector<T>& a, const std::vector<float>& b, double threshold) {
	double mean = 0;
	for (size_t i = 0; i < a.size(); ++i) mean += (double)(float)a[i] + b[i];
	mean /= 2.0 * a.size();
	double worst = 0;
	for (size_t i = 0; i < a.size(); ++i) {
		const double d1 = (float)a[i], d2 = b[i];
		const double e = (std::abs(d1) < 1e-15 && std::abs(d2) < 1e-15) ? 0 : std::abs(d1 - d2) / (0.5 * (std::abs(d1) + std::abs(d2)) + mean * threshold);
		worst = std::max(worst, e);
	}
	return worst;
}

static json optimizer_json() { return {{"otype", "Adam"}, {"learning_rate", 1e-2}, {"beta1", 0.9}, {"beta2", 0.99}, {"epsilon", 1e-15}, {"l2_reg", 1e-6}}; }

static void check_network(const std::string& otype, uint32_t width, uint32_t depth) {
	const uint32_t n_in = 32, n_out = 32, batch = 1 << 14;
	const json cfg = {{"otype", otype}, {"n_input_dims", n_in}, {"n_output_dims", n_out}, {"n_neurons", width}, {"n_hidden_layers", depth}, {"activation", "ReLU"}, {"output_activation", "None"}};
	std::shared_ptr<Network<T>> network{create_network<T>(cfg)};
	std::shared_ptr<Loss<T>> loss{create_loss<T>({{"otype", "L2"}})};
	std::shared_ptr<Optimizer<T>> optimizer{create_optimizer<T>(optimizer_json())};
	auto trainer = std::make_shared<Trainer<T, T, T>>(network, optimizer, loss, 1337u);
	const std::string tag = "network_" + otype;
	const size_t n_params = network->n_params();
	const uint32_t padded = network->padded_output_width();

	// initial parameters: the network tier's initialize_params from pcg32{seed_seq{1337}} (trainer.h:51-58)
	{
		std::seed_seq seq{1337u};
		std::vector<uint32_t> seeds(2);
		seq.generate(seeds.begin(), seeds.end());
		tcnnb_network* ref = nullptr;
		json keys = cfg;
		keys.erase("n_input_dims");
		keys.erase("n_output_dims");
		TCNNB_CHECK_THROW(tcnnb_network_create(n_in, n_out, keys.dump().c_str(), &ref));
		GPUMemory<float> p(n_params);
		TCNNB_CHECK_THROW(tcnnb_network_initialize_params(ref, seeds.front(), p.data(), 1.0f));
		tcnnb_network_destroy(ref);
		report(tag + "_initial_params", same_bits(host(p.data(), n_params), host(trainer->params_full_precision(), n_params)), "differ from the network tier's");
		report(tag + "_params_shared", network->params() == trainer->params(), "the network does not read the trainer's parameters");
	}

	default_rng_t rng{42};
	GPUMatrix<T> x(n_in, batch), dy(padded, batch);
	x.initialize_uniform(rng, 0.001f, 0.999f);
	dy.initialize_uniform(rng, -LOSS_SCALE, LOSS_SCALE);

	// the network tier on the trainer's parameters
	tcnnb_network* h = nullptr;
	{
		json keys = cfg;
		keys.erase("n_input_dims");
		keys.erase("n_output_dims");
		TCNNB_CHECK_THROW(tcnnb_network_create(n_in, n_out, keys.dump().c_str(), &h));
	}
	const size_t n_hidden = (size_t)tcnnb_network_n_forward_activations(h) * batch * tcnnb_network_width(h);
	GPUMemory<T> ref_out(batch * padded), ref_hidden(n_hidden), ref_dx(batch * n_in), ref_dp(n_params);
	TCNNB_CHECK_THROW(tcnnb_network_forward(h, nullptr, batch, x.data(), ref_out.data(), ref_hidden.data(), network->params()));
	TCNNB_CHECK_THROW(tcnnb_network_backward(h, nullptr, batch, x.data(), ref_out.data(), ref_hidden.data(), dy.data(), network->params(), ref_dx.data(), ref_dp.data()));
	GPUMemory<T> ref_inf(batch * padded);
	TCNNB_CHECK_THROW(tcnnb_network_inference_mixed_precision(h, nullptr, batch, x.data(), ref_inf.data(), network->inference_params()));
	tcnnb_network_destroy(h);
	const auto r_out = host(ref_out.data(), ref_out.size()), r_dx = host(ref_dx.data(), ref_dx.size()), r_dp = host(ref_dp.data(), ref_dp.size());

	GPUMatrix<T> out(padded, batch), dx(n_in, batch);
	network->inference_mixed_precision(x, out);
	report(tag + "_inference_mixed_precision", same_bits(out.to_cpu_vector(), host(ref_inf.data(), ref_inf.size())), "differs from tcnnb_network_inference_mixed_precision");
	{
		auto ctx = network->forward(x, &out);
		network->backward(*ctx, x, out, dy, &dx);
	}
	report(tag + "_forward", same_bits(out.to_cpu_vector(), r_out), "differs from tcnnb_network_forward");
	report(tag + "_backward_input", same_bits(dx.to_cpu_vector(), r_dx), "dL_dinput differs from tcnnb_network_backward");
	report(tag + "_backward_params", grads_close(host(network->gradients(), n_params), r_dp), "dL_dparams differ from tcnnb_network_backward");

	// row-major: the same numbers, transposed
	GPUMatrix<T, RM> x_rm(n_in, batch), dy_rm(padded, batch), out_rm(padded, batch), dx_rm(n_in, batch);
	CUDA_CHECK_THROW(cudaMemcpy(x_rm.data(), transposed(x.to_cpu_vector(), batch, n_in).data(), x.n_bytes(), cudaMemcpyHostToDevice));
	CUDA_CHECK_THROW(cudaMemcpy(dy_rm.data(), transposed(dy.to_cpu_vector(), batch, padded).data(), dy.n_bytes(), cudaMemcpyHostToDevice));
	network->inference_mixed_precision(x_rm, out_rm);
	report(tag + "_rm_inference", same_bits(transposed(out_rm.to_cpu_vector(), padded, batch), host(ref_inf.data(), ref_inf.size())), "row-major output differs");
	{
		auto ctx = network->forward(x_rm, &out_rm);
		network->backward(*ctx, x_rm, out_rm, dy_rm, &dx_rm);
	}
	report(tag + "_rm_forward", same_bits(transposed(out_rm.to_cpu_vector(), padded, batch), r_out), "row-major forward output differs");
	report(tag + "_rm_backward", same_bits(transposed(dx_rm.to_cpu_vector(), n_in, batch), r_dx) && grads_close(host(network->gradients(), n_params), r_dp), "row-major backward differs");

	// inference (fp32) against inference_mixed_precision, the reference's own bar (test_common.h)
	GPUMatrix<float> out_f32(n_out, batch);
	network->inference(x, out_f32);
	network->inference_mixed_precision(x, out);
	{
		const double e = max_rae(out.to_cpu_vector(), out_f32.to_cpu_vector(), 1e-4);
		report(tag + "_inference_fp32", e < 1e-4, "RAE " + std::to_string(e));
	}
}

static void check_trainer(const std::string& otype, uint32_t width, uint32_t depth) {
	const uint32_t n_in = 32, n_out = 32, batch = 1 << 14, n_steps = 10;
	const json cfg = {{"otype", otype}, {"n_input_dims", n_in}, {"n_output_dims", n_out}, {"n_neurons", width}, {"n_hidden_layers", depth}, {"activation", "ReLU"}, {"output_activation", "None"}};
	const std::string tag = "trainer_" + otype;
	default_rng_t rng{7};
	GPUMatrix<T> x(n_in, batch);
	GPUMatrix<float> y(n_out, batch);
	generate_random_uniform<T>(nullptr, rng, x.n_elements(), x.data());
	y.initialize_uniform(rng, 0.0f, 1.0f);
	GPUMatrix<T, RM> x_rm(n_in, batch);
	GPUMatrix<float, RM> y_rm(n_out, batch);
	CUDA_CHECK_THROW(cudaMemcpy(x_rm.data(), transposed(x.to_cpu_vector(), batch, n_in).data(), x.n_bytes(), cudaMemcpyHostToDevice));
	CUDA_CHECK_THROW(cudaMemcpy(y_rm.data(), transposed(y.to_cpu_vector(), batch, n_out).data(), y.n_bytes(), cudaMemcpyHostToDevice));

	std::vector<float> losses[2];
	for (int layout = 0; layout < 2; ++layout) {
		std::shared_ptr<Network<T>> network{create_network<T>(cfg)};
		std::shared_ptr<Loss<T>> loss{create_loss<T>({{"otype", "RelativeL2"}})};
		std::shared_ptr<Optimizer<T>> optimizer{create_optimizer<T>(optimizer_json())};
		Trainer<T, T, T> trainer{network, optimizer, loss, 1337u};
		for (uint32_t i = 0; i < n_steps; ++i) {
			auto ctx = layout == 0 ? trainer.training_step(x, y) : trainer.training_step(x_rm, y_rm);
			losses[layout].push_back(trainer.loss(*ctx));
		}
		if (layout == 1) {
			// row-major input through Trainer::forward: the same predictions as the column-major one (no atomics in the forward pass)
			auto cm = trainer.forward(LOSS_SCALE, x, y);
			const auto cm_out = cm->output.to_cpu_vector();
			auto rm = trainer.forward(LOSS_SCALE, x_rm, y);
			report(tag + "_rm_forward_predictions", same_bits(cm_out, rm->output.to_cpu_vector()), "row-major input gives different predictions");
		}
		if (layout == 0) {
			// the object's own inference runs on the trained weights: the trainer's forward predictions, bit for bit
			GPUMatrix<T> out(network->padded_output_width(), batch);
			network->inference_mixed_precision(x, out, false);
			auto fctx = trainer.forward(LOSS_SCALE, x, y);
			report(tag + "_inference_on_trained_weights", same_bits(out.to_cpu_vector(), fctx->output.to_cpu_vector()), "differs from Trainer::forward's predictions");
		}
	}
	bool finite = true;
	for (float l : losses[0]) finite = finite && std::isfinite(l);
	report(tag + "_trains", finite && losses[0].back() < losses[0].front(), "loss " + std::to_string(losses[0].front()) + " -> " + std::to_string(losses[0].back()));
	// (the two runs differ only by the order of the atomic weight-gradient and loss sums)
	double worst = 0;
	for (uint32_t i = 0; i < n_steps; ++i) worst = std::max(worst, (double)std::abs(losses[0][i] - losses[1][i]) / std::abs(losses[0][i]));
	report(tag + "_rm_equals_cm", worst < 1e-3, "row-major inputs / targets train differently: relative loss difference " + std::to_string(worst));
}

static void check_composed() {
	const json encoding = {{"otype", "HashGrid"}, {"n_levels", 16}, {"n_features_per_level", 2}, {"log2_hashmap_size", 15}, {"base_resolution", 16}, {"per_level_scale", 1.5}};
	const json network = {{"otype", "FullyFusedMLP"}, {"activation", "ReLU"}, {"output_activation", "None"}, {"n_neurons", 64}, {"n_hidden_layers", 2}};
	const json loss_opts = {{"otype", "RelativeL2"}};
	const uint32_t n_in = 3, n_out = 3, batch = 1 << 16, n_steps = 5;
	TrainableModel ref = create_from_config(n_in, n_out, {{"loss", loss_opts}, {"optimizer", optimizer_json()}, {"encoding", encoding}, {"network", network}});

	std::shared_ptr<Encoding<T>> enc{create_encoding<T>(n_in, encoding)};
	json net_cfg = network;
	net_cfg["n_input_dims"] = enc->padded_output_width();
	net_cfg["n_output_dims"] = n_out;
	std::shared_ptr<Network<T>> net{create_network<T>(net_cfg)};
	auto model = std::make_shared<NetworkWithInputEncoding<T>>(enc, net);
	std::shared_ptr<Loss<T>> loss{create_loss<T>(loss_opts)};
	std::shared_ptr<Optimizer<T>> optimizer{create_optimizer<T>(optimizer_json())};
	Trainer<float, T, T> trainer{model, optimizer, loss};

	report("composed_initial_params", same_bits(host(trainer.params_full_precision(), trainer.n_params()), host(ref.trainer->params_full_precision(), ref.trainer->n_params())),
	       "differ from create_from_config's");
	default_rng_t rng{1337};
	GPUMatrix<float> x(n_in, batch), y(n_out, batch);
	report("composed_objects_share_params", net->params() == trainer.params() && enc->params() == trainer.params() + net->n_params(),
	       "the component objects do not read their parts of the trainer's parameters");
	double worst = 0, step0 = 0;
	bool same_launches = true;
	for (uint32_t i = 0; i < n_steps; ++i) {
		generate_random_uniform<float>(nullptr, rng, x.n_elements(), x.data());
		y.initialize_uniform(rng, 0.0f, 1.0f);
		const uint64_t l0 = tcnnb_kernel_launch_count();
		auto c1 = ref.trainer->training_step(x, y);
		const uint64_t l1 = tcnnb_kernel_launch_count();
		auto c2 = trainer.training_step(x, y);
		const uint64_t l2 = tcnnb_kernel_launch_count();
		same_launches = same_launches && (l1 - l0) == (l2 - l1);
		const float a = ref.trainer->loss(*c1), b = trainer.loss(*c2);
		const double rel = (double)std::abs(a - b) / std::max(1e-12, (double)std::abs(a));
		if (i == 0) step0 = rel;
		worst = std::max(worst, rel);
	}
	// step 0 runs on bit-equal parameters; later steps inherit the order of the previous steps' fp16 scatter atomics
	report("composed_step0_loss", step0 < 1e-4, "relative step-0 loss difference " + std::to_string(step0));
	report("composed_launches", same_launches, "a composed model launches a different number of kernels per step");
	// the same kernels on the same data: the runs differ only by the order of the grid's fp16 scatter atomics (DESIGN.md section 5.0a)
	report("composed_losses", worst < 1e-3, "relative loss difference " + std::to_string(worst));
}

static void check_not_built() {
	const json encoding = {{"otype", "HashGrid"}, {"n_levels", 8}, {"n_features_per_level", 2}, {"log2_hashmap_size", 12}, {"base_resolution", 16}};
	std::shared_ptr<Encoding<T>> enc{create_encoding<T>(3, encoding)};
	std::shared_ptr<Loss<T>> loss{create_loss<T>(json::object())};
	std::shared_ptr<Optimizer<T>> optimizer{create_optimizer<T>(json::object())};
	Trainer<float, T, T> trainer{enc, optimizer, loss};
	report("encoding_trainer_params", enc->params() == trainer.params() && enc->params() != nullptr, "the encoding does not read the trainer's parameters");
	GPUMatrix<float> x(3, 256), y(enc->output_width(), 256), out(enc->output_width(), 256);
	default_rng_t rng{1};
	x.initialize_uniform(rng, 0.0f, 1.0f);
	auto throws_not_built = [](const std::function<void()>& f) {
		try {
			f();
		} catch (const std::exception& e) {
			return std::string{e.what()}.find("not built") != std::string::npos;
		}
		return false;
	};
	report("not_built_encoding_training_step", throws_not_built([&] { trainer.training_step(x, y); }), "training an Encoding alone did not report 'not built'");
	report("not_built_encoding_inference_fp32", throws_not_built([&] { enc->inference(x, out); }), "Encoding::inference with fp32 outputs did not report 'not built'");
}

int main() {
	try {
		check_network("FullyFusedMLP", 64, 2);
		check_network("CutlassMLP", 128, 3);
		check_trainer("FullyFusedMLP", 64, 2);
		check_trainer("CutlassMLP", 128, 3);
		check_composed();
		check_not_built();
	} catch (const std::exception& e) {
		std::printf("FAIL exception: %s\n", e.what());
		return 100;
	}
	return g_failures;
}
