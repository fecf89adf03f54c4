/* tiny-cuda-nn/object.h -- see config.h (the shim keeps these classes in one header). */
#pragma once

namespace tcnn {
/* object.h:116-120 */
enum class GradientMode {
	Ignore,
	Overwrite,
	Accumulate,
};
}  // namespace tcnn

#include "config.h"
