/* oracle_cpu.h -- C ABI of the CPU restatement of the reference hot path.
 *
 * TEST INFRASTRUCTURE ONLY. Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load this library. The product (tiny-cuda-nn_b200/) never links,
 * imports or calls it. See oracle/README.md for how the restatement is pinned against the reference.
 *
 * Every function cites the reference file:line (relative to /root/reference) it restates.
 */
#pragma once
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- enums shared with the product's C ABI (same numeric values as include/tcnn_b200.h) ---- */
enum { ORC_GRID_HASH = 0, ORC_GRID_DENSE = 1, ORC_GRID_TILED = 2 };                 /* common.h GridType */
enum { ORC_INTERP_NEAREST = 0, ORC_INTERP_LINEAR = 1, ORC_INTERP_SMOOTHSTEP = 2 };  /* common.h InterpolationType */
enum { ORC_ACT_RELU = 0, ORC_ACT_LEAKY_RELU = 1, ORC_ACT_SILU = 2, ORC_ACT_EXPONENTIAL = 3, ORC_ACT_SINE = 4, ORC_ACT_SIGMOID = 5,
       ORC_ACT_SQUAREPLUS = 6, ORC_ACT_SOFTPLUS = 7, ORC_ACT_TANH = 8, ORC_ACT_NONE = 9 };  /* common.h:133-144 Activation */
enum { ORC_LOSS_L2 = 0, ORC_LOSS_RELATIVE_L2 = 1, ORC_LOSS_L1 = 2, ORC_LOSS_RELATIVE_L1 = 3, ORC_LOSS_MAPE = 4, ORC_LOSS_SMAPE = 5, ORC_LOSS_RELATIVE_L2_LUMINANCE = 6, ORC_LOSS_CROSS_ENTROPY = 7, ORC_LOSS_VARIANCE_IS = 8 };  /* src/loss.cu:57-65 */
enum { ORC_ACCUM_FP32 = 0, ORC_ACCUM_FP16_K16 = 1 };  /* MLP accumulator model: fp32 (wgmma path) or fp16 re-rounded every k=16 (HMMA.F16 path) */

#define ORC_MAX_LEVELS 128

typedef struct {
	uint32_t n_pos_dims;           /* 2, 3 or 4 */
	uint32_t n_levels;
	uint32_t n_features_per_level; /* 1, 2, 4, 8 */
	uint32_t log2_hashmap_size;
	uint32_t base_resolution;
	float per_level_scale;
	uint32_t grid_type;            /* ORC_GRID_* */
	uint32_t interpolation;        /* ORC_INTERP_* */
	uint32_t padded_width;         /* n_levels*F rounded up to the network's alignment (16) */
	/* derived by orc_grid_setup(): */
	uint32_t offsets[ORC_MAX_LEVELS + 1];   /* in grid entries (not params) */
	float scales[ORC_MAX_LEVELS];           /* per-level scale; tests may overwrite with device-evaluated values */
	uint32_t resolutions[ORC_MAX_LEVELS];
	uint32_t n_params;             /* offsets[n_levels] * F */
} orc_grid_t;

typedef struct {
	uint32_t in_width;             /* padded encoding width */
	uint32_t width;                /* hidden width */
	uint32_t n_hidden_layers;      /* >= 1 */
	uint32_t out_width;            /* logical outputs */
	uint32_t padded_out_width;     /* next multiple of 16 */
	uint32_t activation;           /* ORC_ACT_* */
	uint32_t output_activation;
	uint32_t n_params;             /* derived by orc_mlp_setup() */
} orc_mlp_t;

typedef struct {
	float learning_rate, beta1, beta2, epsilon, l2_reg;
	float relative_decay, absolute_decay;
	float clipping_magnitude, gradient_clipping_magnitude;
	float non_matrix_learning_rate_factor, non_matrix_l2_reg;
	int adabound, optimize_matrix_params, optimize_non_matrix_params, skip_zero_grad_non_matrix_params;
} orc_adam_t;

/* ---- pcg32 (dependencies/pcg32/pcg32.h:39-200), state passed explicitly ---- */
typedef struct { uint64_t state, inc; } orc_pcg32_t;
void orc_pcg32_seed(orc_pcg32_t* rng, uint64_t initstate, uint64_t initseq);
uint32_t orc_pcg32_next_uint(orc_pcg32_t* rng);
float orc_pcg32_next_float(orc_pcg32_t* rng);
void orc_pcg32_advance(orc_pcg32_t* rng, int64_t delta);

/* Trainer ctor seeding: std::seed_seq{seed} -> pcg32{seeds[0]} (trainer.h:51-58). */
void orc_trainer_rng(uint32_t seed, orc_pcg32_t* rng);

/* generate_random_uniform (random.h:40-69): thread i advances by 4i and writes i, i+n_thr, ...; advances *rng by n. */
void orc_generate_random_uniform(orc_pcg32_t* rng, uint64_t n_elements, float* out, float lower, float upper);

/* ---- sizing (grid.h:692-737, common_device.h:886-895; fully_fused_mlp.cu:635-672) ---- */
int orc_grid_setup(orc_grid_t* g);
int orc_mlp_setup(orc_mlp_t* m);

/* ---- parameter initialisation (trainer.h:69-87, fully_fused_mlp.cu:868-892, gpu_matrix.h:292-306, grid.h:1076-1079) ----
 * params layout: [MLP weights | grid params] (network_with_input_encoding.h:115-130). *rng is advanced like the reference's. */
void orc_initialize_params(const orc_grid_t* g, const orc_mlp_t* m, orc_pcg32_t* rng, float* params_fp32);

/* fp32 -> fp16 (round-to-nearest-even) bit patterns, as trainer.h:409-421. */
void orc_cast_to_half(uint64_t n, const float* in, uint16_t* out);
void orc_cast_from_half(uint64_t n, const uint16_t* in, float* out);

/* ---- grid encoding (grid.h:49-212 forward, :215-320 backward) ----
 * positions: [B][D] fp32 (column-major D x B). encoded: SoA [padded_width][B] fp16 bits (pad rows = 0).
 * indices (optional, may be NULL): [B][n_levels][2^D] uint32 entry indices *within the level*. */
void orc_grid_forward(const orc_grid_t* g, uint32_t B, const float* positions, const uint16_t* grid_params_fp16,
                      uint16_t* encoded_soa, uint32_t* indices);
/* dL_denc: SoA [padded_width][B] fp16 bits. grad_sum: double[n_params], the exact sum of the fp16-rounded
 * per-corner addends (half)w * dL_denc (grid.h:252-255); the device accumulates the same addends with f16x2 atomics. */
void orc_grid_backward(const orc_grid_t* g, uint32_t B, const float* positions, const uint16_t* dL_denc_soa, double* grad_sum);
/* dL/d(position) [B][D] fp32 from dL/d(encoded) SoA fp16: grid.h:171-210 (dy_dx) + grid.h:322-350 (backward_input). */
void orc_grid_input_gradient(const orc_grid_t* g, uint32_t B, const float* positions, const uint16_t* grid_fp16, const uint16_t* dL_denc_soa, float* dL_dx);

/* ---- MLP (fully_fused_mlp.cu:499-557 forward, :150-259 + :736-837 backward) ----
 * weights fp16 bits, row-major [out][in], matrices in order first/hidden.../last(padded rows).
 * input SoA [in_width][B]; hidden: [n_hidden_layers][B][width] post-activation fp16; output [B][padded_out] fp16. */
void orc_mlp_forward(const orc_mlp_t* m, uint32_t B, int accum_mode, const uint16_t* weights, const uint16_t* input_soa,
                     uint16_t* hidden, uint16_t* output);
/* dL_dout [B][padded_out] fp16; dW: double[n_params] (exact sums of products of fp16 values);
 * dL_din SoA [in_width][B] fp16 bits (may be NULL). */
void orc_mlp_backward(const orc_mlp_t* m, uint32_t B, int accum_mode, const uint16_t* weights, const uint16_t* input_soa,
                      const uint16_t* hidden, const uint16_t* dL_dout, double* dW, uint16_t* dL_din_soa);

/* ---- loss (losses/relative_l2.h:40-76, losses/l2.h:40-75) ----
 * prediction [B][stride] fp16, target [B][dims] fp32 -> values [B][stride] fp32, grads [B][stride] fp16 bits. */
void orc_loss(int loss_type, uint32_t B, uint32_t stride, uint32_t dims, float loss_scale, const uint16_t* prediction,
              const float* target, float* values, uint16_t* grads);

void orc_loss_n(int loss_type, uint32_t B, uint32_t stride, uint32_t dims, float loss_scale, uint32_t n_total, const uint16_t* prediction,
                const float* target, float* values, uint16_t* grads);

/* ---- Adam (optimizers/adam.h:48-129) ---- gradients as fp16 bits (what the reference's buffer holds). */
void orc_adam_step(const orc_adam_t* a, uint64_t n, uint64_t n_matrix, float loss_scale, float* weights_fp32,
                   uint16_t* weights_fp16, const uint16_t* grads_fp16, float* m1, float* m2, uint32_t* steps);

/* ---- whole training step (trainer.h:254-357): forward, loss, backward, optional Adam ----
 * State arrays are caller-owned. grads_fp16 receives fp16(rounded exact sums). Returns sum of loss values. */
typedef struct {
	const orc_grid_t* grid;
	const orc_mlp_t* mlp;
	const orc_adam_t* adam;
	int loss_type;
	int accum_mode;
	float loss_scale;
} orc_model_t;
double orc_training_step(const orc_model_t* model, uint32_t B, const float* positions, const float* targets,
                         float* params_fp32, uint16_t* params_fp16, uint16_t* grads_fp16, float* m1, float* m2,
                         uint32_t* steps, int run_optimizer, float* loss_values /* [B][out_width] or NULL */);
/* Data-parallel shard of a global batch (loss normalised over B_global); grad_sums (optional) = exact double sums. */
double orc_training_step_shard(const orc_model_t* model, uint32_t B, uint32_t B_global, const float* positions, const float* targets,
                               float* params_fp32, uint16_t* params_fp16, uint16_t* grads_fp16, double* grad_sums, float* m1, float* m2,
                               uint32_t* steps, int run_optimizer, float* loss_values);
/* network->inference (object.h:214-282): fp32 [B][out_width]. */
void orc_inference(const orc_model_t* model, uint32_t B, const float* positions, const uint16_t* params_fp16, float* out);

int orc_num_threads(void);

#ifdef __cplusplus
}
#endif
