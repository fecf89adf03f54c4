/* tiny-cuda-nn/optimizer.h -- Optimizer<T> and create_optimizer (reference: optimizer.h:46-90, src/optimizer.cu:50-80). The optimizer runs
 * inside libtcnn_b200's training step; the object carries its JSON options to the Trainer. */
#pragma once
#if __has_include(<json/json.hpp>)
#include <json/json.hpp>
#else
#include <nlohmann/json.hpp>
#endif

#include "common.h"

namespace tcnn {

using json = nlohmann::json;

template <typename T>
class Optimizer {
public:
	explicit Optimizer(const json& opts) : m_opts(opts) {}
	const json& hyperparams() const { return m_opts; }
private:
	json m_opts;
};

template <typename T>
Optimizer<T>* create_optimizer(const json& opts) { return new Optimizer<T>{opts}; } /* src/optimizer.cu:50-80 */

}  // namespace tcnn

#include "config.h"
