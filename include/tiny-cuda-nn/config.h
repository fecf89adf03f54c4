/* tiny-cuda-nn/config.h -- create_from_config and TrainableModel (reference: config.h:46-63), implemented over the C ABI of libtcnn_b200.
 * Including it (or any header of this directory) brings in the whole object tier: object.h, loss.h, optimizer.h, network.h, encoding.h,
 * network_with_input_encoding.h and trainer.h (Trainer, its training_step of trainer.h:254-357 included).
 *
 * The JSON type is nlohmann::json, as in the reference (`tcnn::json`); it comes from the application's include path
 * (<json/json.hpp> in a tiny-cuda-nn checkout, <nlohmann/json.hpp> elsewhere).
 *
 * Object model. The reference builds loss, optimizer and network separately and ties them together in the Trainer; the C ABI
 * has ONE handle per trainable model. So Loss / Optimizer / NetworkWithInputEncoding here are light objects that carry their JSON
 * options, and the Trainer constructor creates the tcnnb_model from the combined configuration and attaches it to the network, so
 * that network->inference() afterwards runs on the trainer's parameters -- the reference's behaviour (trainer.h:69-87: the
 * trainer owns the parameter buffer and hands pointers into it to the model). A network that is used for inference before any
 * trainer exists gets a model of its own with the default seed. */
#pragma once
#if __has_include(<json/json.hpp>)
#include <json/json.hpp>
#else
#include <nlohmann/json.hpp>
#endif

#include <cctype>
#include <memory>
#include <string>
#include <vector>

#include "common.h"
#include "gpu_matrix.h"
#include "gpu_memory.h"
#include "object.h"
#include "random.h"
#include "trainer.h"

namespace tcnn {

using json = nlohmann::json;

/* config.h:46-63 */
struct TrainableModel {
	std::shared_ptr<Loss<network_precision_t>> loss;
	std::shared_ptr<Optimizer<network_precision_t>> optimizer;
	std::shared_ptr<NetworkWithInputEncoding<network_precision_t>> network;
	std::shared_ptr<Trainer<float, network_precision_t, network_precision_t>> trainer;
};

inline TrainableModel create_from_config(uint32_t n_input_dims, uint32_t n_output_dims, json config) {
	const json loss_opts = config.value("loss", json::object()), optimizer_opts = config.value("optimizer", json::object());
	const json network_opts = config.value("network", json::object()), encoding_opts = config.value("encoding", json::object());
	std::shared_ptr<Loss<network_precision_t>> loss{create_loss<network_precision_t>(loss_opts)};
	std::shared_ptr<Optimizer<network_precision_t>> optimizer{create_optimizer<network_precision_t>(optimizer_opts)};
	auto network = std::make_shared<NetworkWithInputEncoding<network_precision_t>>(n_input_dims, n_output_dims, encoding_opts, network_opts);
	auto trainer = std::make_shared<Trainer<float, network_precision_t, network_precision_t>>(network, optimizer, loss);
	return {loss, optimizer, network, trainer};
}

}  // namespace tcnn
