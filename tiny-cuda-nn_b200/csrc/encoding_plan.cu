// encoding_plan.cu -- runs an EncodingPlan (encoding_plan.h): the feature-encoding kernels (feature_encodings.cu) for the plain
// segments, one stand-alone grid kernel (grid_kernels.cu) per grid, and the reductions / overlapping input-gradient sums of a
// Composite (composite_kernels.cu). Used by the general path of the model (model.cu), the module
// tier's input gradient and the encoding tier (encoding.cu).
#include "encoding_plan.h"

#include "composite_kernels.h"
#include "misc_kernels.h"

namespace tcnnb {

namespace {

// The nested encodings of the plan, each into its own columns of rows [n][row_stride] (the caller's rows under Concatenation,
// plan.nested_out under a reduction).
void nested_forward(const EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const __half* params, __half* rows, uint32_t row_stride, float max_level) {
	if (plan.has_plain_features()) {
		TCNNB_CUDA_CHECK(launch_feature_forward(stream, plan.segs, n, x, plan.n_in, rows, row_stride));
		++g_kernel_launches;
	}
	for (auto& g : plan.grids) {
		const FeatureSegment& sg = plan.segs.s[g->segment];
		GridKernelArgs a = plan_grid_args(*g, n, x + sg.in_begin, plan.n_in, row_stride, max_level);
		a.pad_cols = sg.n_pad;
		TCNNB_CUDA_CHECK(launch_grid_forward(stream, a, params + g->param_offset, rows + sg.out_begin));
		++g_kernel_launches;
	}
}

// Where the nested encodings find dL/d(their outputs): segment sg at column `at_zero ? 0 : sg.out_begin` of rows [n][stride].
struct NestedGradient {
	const __half* rows;
	uint32_t stride;
	bool at_zero;  // Sum: every nested encoding reads dL/d(encoded) itself (composite.h:67-84 copies it K times)
	uint32_t column(const FeatureSegment& sg) const { return at_zero ? 0u : sg.out_begin; }
};

NestedGradient nested_gradient(EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const __half* params, const __half* dL_dencoded, uint32_t row_stride,
                               float max_level, bool nested_out_ready) {
	if (plan.reduction != REDUCE_PRODUCT) return {dL_dencoded, row_stride, plan.reduction == REDUCE_SUM};
	const uint32_t stride = plan.segs.n * plan.width;
	if (!nested_out_ready) {
		grow(plan.nested_out, (size_t)n * stride);
		nested_forward(plan, stream, n, x, params, plan.nested_out.ptr, stride, max_level);
	}
	grow(plan.dL_dnested, (size_t)n * stride);
	TCNNB_CUDA_CHECK(launch_reduce_product_backward(stream, plan.segs.n, plan.width, n, dL_dencoded, row_stride, plan.nested_out.ptr, plan.dL_dnested.ptr));
	++g_kernel_launches;
	return {plan.dL_dnested.ptr, stride, false};
}

void param_gradients(EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const NestedGradient& dy, __half* dL_dparams, float max_level) {
	TCNNB_CUDA_CHECK(cudaMemsetAsync(dL_dparams, 0, sizeof(__half) * plan.n_params, stream));  // GradientMode::Overwrite (grid.h:865-867)
	for (auto& g : plan.grids) {
		const FeatureSegment& sg = plan.segs.s[g->segment];
		const uint32_t F = g->cfg.n_features_per_level;
		GridKernelArgs a = plan_grid_args(*g, n, x + sg.in_begin, plan.n_in, dy.stride, max_level);
		if (max_level >= 1.0f) {  // contended coarse levels scatter into private copies
			const GridScatterPlan sp = plan_grid_scatter(g->levels.data(), g->cfg.n_levels, F, g->cfg.n_pos_dims, n);
			if (sp.n_replicas > 1) {
				if (plan.replicas.n < sp.scratch_halfs) {
					plan.replicas.resize(sp.scratch_halfs);
					plan.replicas.zero(stream);  // the reduce kernel leaves it zero
				}
				a.replica_scratch = plan.replicas.ptr;
				a.n_replicas = sp.n_replicas;
				a.replica_entries = sp.replica_entries;
			}
		}
		float* tmp = nullptr;
		if (F == 1) {
			grow(plan.grad_fp32, g->cfg.n_params);
			tmp = plan.grad_fp32.ptr;
			TCNNB_CUDA_CHECK(cudaMemsetAsync(tmp, 0, sizeof(float) * g->cfg.n_params, stream));
		}
		TCNNB_CUDA_CHECK(launch_grid_backward(stream, a, dy.rows + dy.column(sg), dL_dparams + g->param_offset, tmp, g->cfg.n_params));
		// the scatter, then the replica reduce (F > 1) or the fp32 -> fp16 cast (F == 1) when there is one
		g_kernel_launches += 1 + (a.n_replicas > 1 ? 1 : 0) + (F == 1 ? 1 : 0);
	}
}

void input_gradient(EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const __half* params, const NestedGradient& dy, float* dL_dx, float max_level) {
	if (plan.overlap) {
		// every segment writes its own slab [n][n_in]; one kernel sums the slabs into dL_dx
		const size_t slab = (size_t)n * plan.n_in;
		grow(plan.dx_slabs, slab * plan.segs.n);
		for (uint32_t k = 0; k < plan.segs.n; ++k) {
			const FeatureSegment& sg = plan.segs.s[k];
			if (sg.type == FEAT_GRID || sg.type == FEAT_EMPTY) continue;
			FeatureSegments one{};
			one.n = 1;
			one.s[0] = sg;
			one.s[0].out_begin = dy.column(sg);
			TCNNB_CUDA_CHECK(launch_feature_input_gradient(stream, one, n, x, plan.n_in, dy.rows, dy.stride, plan.dx_slabs.ptr + k * slab));
			++g_kernel_launches;
		}
		for (auto& g : plan.grids) {
			const FeatureSegment& sg = plan.segs.s[g->segment];
			const GridKernelArgs a = plan_grid_args(*g, n, x + sg.in_begin, plan.n_in, dy.stride, max_level);
			TCNNB_CUDA_CHECK(launch_grid_input_gradient(stream, a, params + g->param_offset, dy.rows + dy.column(sg), plan.dx_slabs.ptr + g->segment * slab + sg.in_begin));
			++g_kernel_launches;
		}
		TCNNB_CUDA_CHECK(launch_sum_input_gradients(stream, plan.segs, n, plan.n_in, plan.dx_slabs.ptr, dL_dx));
		++g_kernel_launches;
		return;
	}
	if (plan.zero_dx) TCNNB_CUDA_CHECK(cudaMemsetAsync(dL_dx, 0, sizeof(float) * (size_t)n * plan.n_in, stream));  // dimensions no nested encoding reads
	if (plan.has_plain_features()) {
		FeatureSegments segs = plan.segs;
		for (uint32_t k = 0; k < segs.n; ++k) segs.s[k].out_begin = dy.column(plan.segs.s[k]);
		TCNNB_CUDA_CHECK(launch_feature_input_gradient(stream, segs, n, x, plan.n_in, dy.rows, dy.stride, dL_dx));
		++g_kernel_launches;
	}
	for (auto& g : plan.grids) {
		const FeatureSegment& sg = plan.segs.s[g->segment];
		const GridKernelArgs a = plan_grid_args(*g, n, x + sg.in_begin, plan.n_in, dy.stride, max_level);
		TCNNB_CUDA_CHECK(launch_grid_input_gradient(stream, a, params + g->param_offset, dy.rows + dy.column(sg), dL_dx + sg.in_begin));
		++g_kernel_launches;
	}
}

}  // namespace

void plan_forward(EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const __half* params, __half* encoded, uint32_t row_stride, float max_level) {
	if (!plan.reduced()) {
		nested_forward(plan, stream, n, x, params, encoded, row_stride, max_level);
		return;
	}
	const uint32_t stride = plan.segs.n * plan.width;
	grow(plan.nested_out, (size_t)n * stride);
	nested_forward(plan, stream, n, x, params, plan.nested_out.ptr, stride, max_level);
	TCNNB_CUDA_CHECK(launch_reduce_forward(stream, plan.reduction == REDUCE_PRODUCT, plan.segs.n, plan.width, n, plan.nested_out.ptr, encoded, row_stride));
	++g_kernel_launches;
}

void plan_backward(EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const __half* params, const __half* dL_dencoded, uint32_t row_stride, __half* dL_dparams,
                   float* dL_dx, float max_level, bool nested_out_ready) {
	if (plan.n_params == 0) dL_dparams = nullptr;
	if (!dL_dparams && !dL_dx) return;
	const NestedGradient dy = nested_gradient(plan, stream, n, x, params, dL_dencoded, row_stride, max_level, nested_out_ready);
	if (dL_dparams) param_gradients(plan, stream, n, x, dy, dL_dparams, max_level);
	if (dL_dx) input_gradient(plan, stream, n, x, params, dy, dL_dx, max_level);
}

void plan_param_gradients(EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const __half* params, const __half* dL_dencoded, uint32_t row_stride,
                          __half* dL_dparams, float max_level) {
	plan_backward(plan, stream, n, x, params, dL_dencoded, row_stride, dL_dparams, nullptr, max_level);
}

void plan_input_gradient(EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const __half* params, const __half* dL_dencoded, uint32_t row_stride,
                         float* dL_dx, float max_level) {
	plan_backward(plan, stream, n, x, params, dL_dencoded, row_stride, nullptr, dL_dx, max_level);
}

void plan_backward_backward_input(EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const __half* params, const __half* dL_doutput,
                                  uint32_t row_stride, const float* dL_ddLdinput, __half* dL_dparams, __half* dL_ddLdoutput, float* dL_dinput, float max_level) {
	if (plan.composite || plan.segs.n != 1 || plan.grids.size() != 1) {
		// the reference implements double backward for grid encodings only (object.h:468-482)
		static const char* const names[] = {"Identity", "Frequency", "TriangleWave", "OneBlob", "SphericalHarmonics", "Grid", "Empty"};
		const uint32_t type = plan.segs.n ? plan.segs.s[0].type : 0u;
		const std::string name = plan.composite ? "Composite" : (type < sizeof(names) / sizeof(names[0]) ? names[type] : "Encoding");
		throw std::runtime_error(name + " does not support double backward.");
	}
	const EncodingPlan::Grid& g = *plan.grids.front();
	const FeatureSegment& sg = plan.segs.s[g.segment];
	GridKernelArgs a = plan_grid_args(g, n, x + sg.in_begin, plan.n_in, row_stride, max_level);
	a.pad_cols = sg.n_pad;
	float* tmp = nullptr;
	if (dL_dparams) {
		TCNNB_CUDA_CHECK(cudaMemsetAsync(dL_dparams, 0, sizeof(__half) * plan.n_params, stream));  // GradientMode::Overwrite (grid.h:959-961)
		if (g.cfg.n_features_per_level == 1) {
			grow(plan.grad_fp32, g.cfg.n_params);
			tmp = plan.grad_fp32.ptr;
			TCNNB_CUDA_CHECK(cudaMemsetAsync(tmp, 0, sizeof(float) * g.cfg.n_params, stream));
		}
	}
	if (!dL_dparams && !dL_ddLdoutput && !dL_dinput) return;
	const __half* table = params ? params + g.param_offset : nullptr;
	TCNNB_CUDA_CHECK(launch_grid_backward_backward_input(stream, a, table, dL_doutput ? dL_doutput + sg.out_begin : nullptr, dL_ddLdinput + sg.in_begin,
	                                                     dL_dparams ? dL_dparams + g.param_offset : nullptr, tmp, g.cfg.n_params,
	                                                     dL_ddLdoutput ? dL_ddLdoutput + sg.out_begin : nullptr, dL_dinput ? dL_dinput + sg.in_begin : nullptr));
	// the kernel, and the fp32 -> fp16 cast of the F == 1 parameter gradient; Nearest scatters nothing
	const bool scatter = dL_dparams && g.cfg.interpolation != INTERP_NEAREST;
	g_kernel_launches += ((scatter || dL_ddLdoutput || dL_dinput) ? 1 : 0) + (scatter && g.cfg.n_features_per_level == 1 ? 1 : 0);
}

void init_plan_params(const EncodingPlan& plan, HostPcg32& rng, float* dst, float scale) {
	for (auto& g : plan.grids) {
		TCNNB_CUDA_CHECK(launch_random_uniform(nullptr, rng.device(), g->cfg.n_params, dst + g->param_offset, -1e-4f * scale, 1e-4f * scale));
		++g_kernel_launches;
		rng.advance(g->cfg.n_params);
	}
}

}  // namespace tcnnb
