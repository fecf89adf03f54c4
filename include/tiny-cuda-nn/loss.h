/* tiny-cuda-nn/loss.h -- Loss<T> and create_loss (reference: loss.h:60-75, src/loss.cu:82-90). The loss runs inside libtcnn_b200's training
 * step; the object carries its JSON options to the Trainer. */
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
class Loss {
public:
	explicit Loss(const json& opts) : m_opts(opts) {}  /* parentheses: brace-initialising a json from a json makes an array */
	const json& hyperparams() const { return m_opts; }
private:
	json m_opts;
};

template <typename T>
Loss<T>* create_loss(const json& opts) { return new Loss<T>{opts}; }           /* src/loss.cu:82-90 */

}  // namespace tcnn

#include "config.h"
