/* tiny-cuda-nn/object.h -- see config.h (the shim keeps these classes in one header). */
#pragma once

namespace tcnn {
/* object.h:116-120 */
enum class GradientMode {
	Ignore,
	Overwrite,
	Accumulate,
};

#ifndef TCNN_B200_CONTEXT_DEFINED  /* cpp_api.h defines the same type */
#define TCNN_B200_CONTEXT_DEFINED
struct Context { /* cpp_api.h:39-47: what a forward pass hands to its backward pass */
	Context() = default;
	virtual ~Context() {}
	Context(const Context&) = delete;
	Context& operator=(const Context&) = delete;
	Context(Context&&) = delete;
	Context& operator=(Context&&) = delete;
};
#endif
}  // namespace tcnn

#include "config.h"
