// snapshot_decay -- trainer->serialize() / deserialize() under an ExponentialDecay optimizer, in the reference's schema
// (optimizers/exponential_decay.h:136-148) through include/tiny-cuda-nn/config.h (tests/test_cpp_shim_snapshot_decay.py drives it):
//   snapshot_decay <config.json> <n_in> <n_out> <B> <dir> <n_steps> <factor>
// trains n_steps on dir/x.f32, dir/y.f32, serializes with the optimizer, loads that (through msgpack) into a new trainer, and loads
// two documents built by hand in the reference's schema: one storing <factor>, one without a factor. Prints one JSON line with what
// each of them holds.
#include <tiny-cuda-nn/config.h>

#include <cstdio>
#include <fstream>
#include <string>
#include <vector>

using namespace tcnn;

static std::vector<float> read_f32(const std::string& path) {
	std::ifstream f{path, std::ios::binary | std::ios::ate};
	if (!f) throw std::runtime_error{"cannot open " + path};
	std::vector<float> v((size_t)f.tellg() / 4);
	f.seekg(0);
	f.read((char*)v.data(), v.size() * 4);
	return v;
}

static json keys(const json& j) {
	json k = json::array();
	for (auto it = j.begin(); it != j.end(); ++it) k.push_back(it.key());
	return k;
}

int main(int argc, char** argv) {
	try {
		if (argc < 8) {
			fprintf(stderr, "usage: snapshot_decay config n_in n_out B dir n_steps factor\n");
			return 2;
		}
		const std::string dir = argv[5];
		std::ifstream cf{argv[1]};
		const json config = json::parse(cf, nullptr, true, true);
		const uint32_t n_in = atoi(argv[2]), n_out = atoi(argv[3]), B = atoi(argv[4]), n_steps = atoi(argv[6]);
		const float hand_factor = (float)atof(argv[7]);
		auto model = create_from_config(n_in, n_out, config);
		GPUMatrix<float> x(n_in, B), y(n_out, B);
		const std::vector<float> hx = read_f32(dir + "/x.f32"), hy = read_f32(dir + "/y.f32");
		CUDA_CHECK_THROW(cudaMemcpy(x.data(), hx.data(), hx.size() * 4, cudaMemcpyHostToDevice));
		CUDA_CHECK_THROW(cudaMemcpy(y.data(), hy.data(), hy.size() * 4, cudaMemcpyHostToDevice));
		for (uint32_t i = 0; i < n_steps; ++i) model.trainer->training_step(nullptr, x, y);
		const json snap = model.trainer->serialize(true);
		const json& opt = snap.at("optimizer");

		// the snapshot loads into a new trainer (through msgpack, as an application stores it) and serializes back the same
		auto fresh = create_from_config(n_in, n_out, config);
		fresh.trainer->deserialize(json::from_msgpack(json::to_msgpack(snap)));
		const json again = fresh.trainer->serialize(true);

		// exponential_decay.h:136-148 by hand: {"nested": Adam's state with the decayed rate, "learning_rate", "learning_rate_factor"}
		const float base = opt.at("learning_rate").get<float>();
		json nested = opt.at("nested");
		nested["base_learning_rate"] = base * hand_factor;
		json hand = {{"n_params", snap.at("n_params")}, {"params_type", "__half"}, {"params_binary", snap.at("params_binary")},
		             {"optimizer", {{"nested", nested}, {"learning_rate", base}, {"learning_rate_factor", hand_factor}}}};
		auto by_hand = create_from_config(n_in, n_out, config);
		by_hand.trainer->deserialize(hand);
		hand["optimizer"].erase("learning_rate_factor");
		auto without_factor = create_from_config(n_in, n_out, config);
		without_factor.trainer->deserialize(hand);

		const json out = {{"top_keys", keys(opt)},
		                  {"nested_keys", keys(opt.at("nested"))},
		                  {"current_step", opt.at("nested").at("current_step")},
		                  {"learning_rate", base},
		                  {"learning_rate_factor", opt.at("learning_rate_factor")},
		                  {"nested_base_learning_rate", opt.at("nested").at("base_learning_rate")},
		                  {"trainer_factor", tcnnb_learning_rate_factor(model.trainer->handle())},
		                  {"loaded_factor", tcnnb_learning_rate_factor(fresh.trainer->handle())},
		                  {"reserialized_identical", again == snap},
		                  {"hand_factor", tcnnb_learning_rate_factor(by_hand.trainer->handle())},
		                  {"hand_learning_rate", by_hand.trainer->serialize(true).at("optimizer").at("learning_rate")},
		                  {"no_factor_factor", tcnnb_learning_rate_factor(without_factor.trainer->handle())}};
		printf("%s\n", out.dump().c_str());
		return 0;
	} catch (const std::exception& e) {
		fprintf(stderr, "snapshot_decay: %s\n", e.what());
		return 1;
	}
}
