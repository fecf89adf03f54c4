// encoding_plan.cu -- runs an EncodingPlan (encoding_plan.h): the feature-encoding kernels (feature_encodings.cu) for the plain
// segments and one stand-alone grid kernel (grid_kernels.cu) per grid. Used by the general path of the model (model.cu), the module
// tier's input gradient and the encoding tier (encoding.cu).
#include "encoding_plan.h"

#include "misc_kernels.h"

namespace tcnnb {

void plan_forward(const EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const __half* params, __half* encoded, uint32_t row_stride, float max_level) {
	if (plan.has_plain_features()) {
		TCNNB_CUDA_CHECK(launch_feature_forward(stream, plan.segs, n, x, plan.n_in, encoded, row_stride));
		++g_kernel_launches;
	}
	for (auto& g : plan.grids) {
		const FeatureSegment& sg = plan.segs.s[g->segment];
		GridKernelArgs a = plan_grid_args(*g, n, x + sg.in_begin, plan.n_in, row_stride, max_level);
		a.pad_cols = sg.n_pad;
		TCNNB_CUDA_CHECK(launch_grid_forward(stream, a, params + g->param_offset, encoded + sg.out_begin));
		++g_kernel_launches;
	}
}

void plan_param_gradients(EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const __half* dL_dencoded, uint32_t row_stride, __half* dL_dparams,
                          float max_level) {
	if (plan.n_params == 0) return;
	TCNNB_CUDA_CHECK(cudaMemsetAsync(dL_dparams, 0, sizeof(__half) * plan.n_params, stream));  // GradientMode::Overwrite (grid.h:865-867)
	for (auto& g : plan.grids) {
		const FeatureSegment& sg = plan.segs.s[g->segment];
		const uint32_t F = g->cfg.n_features_per_level;
		GridKernelArgs a = plan_grid_args(*g, n, x + sg.in_begin, plan.n_in, row_stride, max_level);
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
		TCNNB_CUDA_CHECK(launch_grid_backward(stream, a, dL_dencoded + sg.out_begin, dL_dparams + g->param_offset, tmp, g->cfg.n_params));
		// the scatter, then the replica reduce (F > 1) or the fp32 -> fp16 cast (F == 1) when there is one
		g_kernel_launches += 1 + (a.n_replicas > 1 ? 1 : 0) + (F == 1 ? 1 : 0);
	}
}

void plan_input_gradient(const EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const __half* params, const __half* dL_dencoded, uint32_t row_stride,
                         float* dL_dx, float max_level) {
	if (plan.composite) TCNNB_CUDA_CHECK(cudaMemsetAsync(dL_dx, 0, sizeof(float) * (size_t)n * plan.n_in, stream));  // dimensions no nested encoding reads
	if (plan.has_plain_features()) {
		TCNNB_CUDA_CHECK(launch_feature_input_gradient(stream, plan.segs, n, x, plan.n_in, dL_dencoded, row_stride, dL_dx));
		++g_kernel_launches;
	}
	for (auto& g : plan.grids) {
		const FeatureSegment& sg = plan.segs.s[g->segment];
		const GridKernelArgs a = plan_grid_args(*g, n, x + sg.in_begin, plan.n_in, row_stride, max_level);
		TCNNB_CUDA_CHECK(launch_grid_input_gradient(stream, a, params + g->param_offset, dL_dencoded + sg.out_begin, dL_dx + sg.in_begin));
		++g_kernel_launches;
	}
}

void plan_backward_backward_input(EncodingPlan& plan, cudaStream_t stream, uint32_t n, const float* x, const __half* params, const __half* dL_doutput,
                                  uint32_t row_stride, const float* dL_ddLdinput, __half* dL_dparams, __half* dL_ddLdoutput, float* dL_dinput, float max_level) {
	if (plan.composite || plan.segs.n != 1 || plan.grids.size() != 1) {
		// the reference implements double backward for grid encodings only (object.h:468-482)
		static const char* const names[] = {"Identity", "Frequency", "TriangleWave", "OneBlob", "SphericalHarmonics", "Grid"};
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
