/* tcnn_b200.h -- C ABI of the Hopper-native (sm_90a) HashGrid + FullyFusedMLP hot path.
 *
 * This is the drop-in boundary: plain C, opaque handles, raw device/host pointers, no torch / C++ types.
 * Each entry point names the reference interface (file:line relative to tiny-cuda-nn's tree) it replaces.
 * The reference's own boundary is C++ in two tiers; this ABI carries both:
 *   - "trainer tier"  == tcnn::create_from_config / Trainer / NetworkWithInputEncoding  (config.h:46-63,
 *                        trainer.h:51-532, network_with_input_encoding.h:42-150)
 *   - "module tier"   == tcnn::cpp::Module, the type-erased API the PyTorch extension binds (cpp_api.h:48-125)
 * the headers under include/tiny-cuda-nn/ (header-only C++ shim over this ABI) restores the reference's C++ names on top.
 *
 * Conventions (identical to the reference):
 *   - inputs are fp32, sample-contiguous: [batch][n_input_dims] == column-major n_input_dims x batch (gpu_matrix.h:226-228)
 *   - batch sizes must be multiples of 256 (common.h:246, object.h:169)
 *   - parameters are one flat buffer [MLP weights | grid table] (network_with_input_encoding.h:115-130), the trainer
 *     owns [fp32 master | fp16 params | fp16 gradients] (trainer.h:489-503)
 *   - all work is stream-ordered on the caller's stream; nothing synchronises except tcnnb_loss and *_host calls
 *   - errors: every call returns 0 on success, non-zero on failure; tcnnb_last_error() returns the message the
 *     reference would have thrown as std::runtime_error (common_host.h:71-110). There is NO CPU fallback.
 *   - threading: like the reference (unsynchronised arenas / streams, SURVEY.md section 8b) a handle is NOT thread-safe; different
 *     handles may be used from different threads. tcnnb_last_error() is per calling thread.
 */
#ifndef TCNN_B200_H
#define TCNN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct tcnnb_model tcnnb_model;   /* TrainableModel{loss, optimizer, network, trainer}  (config.h:46-51) */
typedef void* tcnnb_stream;               /* cudaStream_t */

/* ---- library-level (cpp_api.h:59-86) ---- */
const char* tcnnb_last_error(void);
uint32_t tcnnb_batch_size_granularity(void);             /* cpp_api.h:61  -> 256 */
float tcnnb_default_loss_scale(void);                    /* cpp_api.h:67 / common.h:243 -> 128 for fp16 */
int tcnnb_cuda_device(void);                             /* cpp_api.h:63 */
int tcnnb_set_cuda_device(int device);                   /* cpp_api.h:64 */
uint32_t tcnnb_abi_version(void);

/* ---- construction: tcnn::create_from_config(n_input_dims, n_output_dims, json) + Trainer(..., seed) ----
 * config.h:53-63, trainer.h:51-87. `config_json` is the same JSON document the reference parses
 * ({"loss":{}, "optimizer":{}, "encoding":{}, "network":{}}, keys and defaults per src/encoding.cu, src/network.cu,
 * src/loss.cu, src/optimizer.cu). Parameters are initialised exactly like the reference (same pcg32 streams).
 * Built: encodings Grid / HashGrid / DenseGrid / TiledGrid, Identity, Frequency, TriangleWave, OneBlob, SphericalHarmonics, Composite;
 * networks FullyFusedMLP / CutlassMLP with 16 / 32 / 64 / 128 neurons; all nine losses; Adam, optionally inside ExponentialDecay and / or
 * Ema. The benchmarked family (one grid with 2 features per level or Identity, <= 64 neurons, <= 16 outputs) runs on ONE fused kernel
 * per step, everything else on stand-alone encoding + network kernels (DESIGN.md section 3.5). Unsupported otypes fail loudly. */
int tcnnb_create_from_config(uint32_t n_input_dims, uint32_t n_output_dims, const char* config_json, uint32_t seed, tcnnb_model** out);
void tcnnb_destroy(tcnnb_model* model);
/* ---- Trainer(create_network<__half>(network), optimizer, loss, seed) (trainer.h:51-87, src/network.cu:51-141): a trainer over a network
 * alone, without an encoding. `config_json` is {"loss":{}, "optimizer":{}, "network":{}}; n_input_dims must be a multiple of 16 (the
 * network's input width). Parameters are the network's alone and initialised like the reference's (the same pcg32 stream).
 * Every trainer call of this header applies to the handle -- training_step(_ex), forward / backward, optimizer_step, inference,
 * parameters, snapshots, ExponentialDecay / Ema -- with ONE difference: input_dev and dL_dinput_dev are fp16 rows
 * [batch][n_input_dims] (the network's own input, read in place; pass them cast to float*). Targets, data_pdf and outputs are as for
 * any handle; input and dL_dinput rows must be 16-byte aligned. The host-buffer and data-parallel calls take fp32 inputs and reject such a
 * handle. It always runs the stand-alone
 * network kernels. */
int tcnnb_create_network_trainer(uint32_t n_input_dims, uint32_t n_output_dims, const char* config_json, uint32_t seed, tcnnb_model** out);

/* ---- introspection (network_with_input_encoding.h:132-150, trainer.h:385-407,477-482) ---- */
uint64_t tcnnb_n_params(const tcnnb_model* m);                 /* trainer->n_params() */
/* Allocated length of each of the three parameter regions (>= n_params, multiple of 512; the padding is zero and never
 * touched). The sharded-optimizer data-parallel trainer cuts [0, n_params_padded) into equal slices. */
uint64_t tcnnb_n_params_padded(const tcnnb_model* m);
uint64_t tcnnb_n_mlp_params(const tcnnb_model* m);             /* network part; grid params follow */
uint32_t tcnnb_n_input_dims(const tcnnb_model* m);
uint32_t tcnnb_n_output_dims(const tcnnb_model* m);            /* network->output_width() */
uint32_t tcnnb_padded_output_width(const tcnnb_model* m);      /* network->padded_output_width() */
uint32_t tcnnb_encoded_width(const tcnnb_model* m);            /* encoding->padded_output_width() */
float* tcnnb_params_full_precision(tcnnb_model* m);            /* trainer->params_full_precision(): device fp32 [n_params] */
void* tcnnb_params(tcnnb_model* m);                            /* trainer->params(): device fp16 [n_params] */
/* trainer->param_gradients(): device fp16 [n_params]. The network part is materialised from the fp32 accumulator on the stream
 * of the step that produced it, and THAT stream is synchronised (no other stream is touched). */
void* tcnnb_param_gradients(tcnnb_model* m);
/* Level table of the grid encoding: offsets in entries (n_levels+1), per-level scale and resolution (grid.h:692-737). */
int tcnnb_grid_levels(const tcnnb_model* m, uint32_t* n_levels, uint32_t* offsets, float* scales, uint32_t* resolutions);
/* JSON with the resolved hyper-parameters (object.h hyperparams()); pointer valid until the next call on this model. */
const char* tcnnb_hyperparams(tcnnb_model* m);

/* ---- trainer->set_params_full_precision / set_params (trainer.h:409-440) ---- */
int tcnnb_set_params_full_precision(tcnnb_model* m, const float* params, uint64_t n, int device_ptr);

/* Trainer::params_inference() (trainer.h:401-403): what network->inference() reads -- the Ema optimizer wrapper's averaged fp16 weights
 * (optimizers/ema.h) when the configuration has one, else the working parameters. */
void* tcnnb_params_inference(tcnnb_model* m);
/* trainer->set_params(params, n, device_ptr) (trainer.h:423-440): working-precision (fp16) parameters; the fp32 masters follow. */
int tcnnb_set_params(tcnnb_model* m, const void* params_half, uint64_t n, int device_ptr);
/* Optimizer state for trainer->serialize(true) / deserialize (trainer.h:442-482, optimizers/adam.h:303-325): device pointers to
 * the fp32 first / second moments and the uint32 per-parameter step counters ([n_params] each; valid for the model's lifetime),
 * the optimizer's step counter and base learning rate. Synchronises the device. */
int tcnnb_optimizer_state(tcnnb_model* m, float** first_moments_dev, float** second_moments_dev, uint32_t** param_steps_dev, uint32_t* current_step, float* base_learning_rate);
/* Restores the optimizer's step counter and base learning rate (the undecayed one under ExponentialDecay). ExponentialDecay's
 * learning-rate factor is recomputed from the step counter, exactly as an uninterrupted run reaches it; tcnnb_deserialize does the same. */
int tcnnb_set_optimizer_progress(tcnnb_model* m, uint32_t current_step, float base_learning_rate);
/* ExponentialDecay's current learning-rate factor (optimizers/exponential_decay.h `learning_rate_factor`; 1 without the wrapper): the
 * next step runs at base_learning_rate * factor, times decay_base when that step is a decay boundary. The setter overrides the factor
 * that tcnnb_set_optimizer_progress recomputed, for snapshots that store their own (the reference's ExponentialDecay schema); it fails
 * when the optimizer has no ExponentialDecay wrapper. */
float tcnnb_learning_rate_factor(const tcnnb_model* m);
int tcnnb_set_learning_rate_factor(tcnnb_model* m, float factor);

/* ---- trainer->training_step(stream, input, target, ..., run_optimizer) (trainer.h:254-357) ----
 * input_dev [batch][n_in] fp32, target_dev [batch][n_out] fp32, both device pointers.
 * Runs fwd + loss + bwd (+ Adam when run_optimizer != 0). The loss of this step is fetched with tcnnb_loss. */
int tcnnb_training_step(tcnnb_model* m, tcnnb_stream stream, uint32_t batch_size, const float* input_dev, const float* target_dev, int run_optimizer);
/* trainer->training_step(stream, input, target, data_pdf, run_optimizer, dL_dinput, use_inference_params, param_gradients_mode,
 *                        external_dL_dy)  (trainer.h:254-357). Device pointers; every one but input_dev may be null.
 *   data_pdf_dev        fp32 [batch][n_out], laid out like the targets: every loss divides by the sample's pdf (losses/l2.h etc.; Variance's
 *                       value is factor / pred - factor / pdf with factor = target^2 / pdf / n_total, variance_is.h:69-76).
 *   dL_dinput_dev       fp32 [batch][n_in], overwritten with dL/d(input).
 *   use_inference_params  forward and backward read tcnnb_params_inference (the Ema weights); gradients still go to the trainer.
 *   param_gradients_mode  0 Ignore (the gradient buffer is left as it is), 1 Overwrite (tcnnb_training_step), 2 Accumulate (adds this
 *                       step's gradients onto the buffer, also after tcnnb_param_gradients) -- GradientMode, object.h:116-120.
 *   external_dL_dy_dev  fp16 [batch][padded_output_width], already multiplied by the loss scale (tcnnb_default_loss_scale): replaces
 *                       the loss (trainer.h:127-131), so target_dev and data_pdf_dev are not read. It still passes through the output
 *                       activation's transfer. The reference leaves the loss values of such a step unfilled; tcnnb_loss returns 0.
 * Rejected: handles of tcnnb_module_create, handles with a data-parallel state (tcnnb_dp_init), a null target without
 * external_dL_dy, batches that are not a multiple of tcnnb_batch_size_granularity(). */
int tcnnb_training_step_ex(tcnnb_model* m, tcnnb_stream stream, uint32_t batch_size, const float* input_dev, const float* target_dev, const float* data_pdf_dev,
                           int run_optimizer, float* dL_dinput_dev, int use_inference_params, int param_gradients_mode, const void* external_dL_dy_dev);
/* ---- Trainer::forward / Trainer::backward (trainer.h:89-153): a training step split around a ForwardContext whose buffers the
 * caller owns. The library keeps nothing between the two calls; backward recomputes the forward pass.
 * tcnnb_forward: trainer->forward(stream, loss_scale, input, target, data_pdf, use_inference_params, prepare_input_gradients,
 *                external_dL_dy) (trainer.h:97-139). Device pointers.
 *   output_dev          fp16 [batch][padded_output_width], 16-byte aligned, required: the predictions (ctx.output), with the
 *                       tcnnb_params_inference weights when use_inference_params != 0.
 *   loss_values_dev     fp32 [batch][padded_output_width] (ctx.L): the loss per element, padding columns 0. May be null.
 *   dL_doutput_dev      fp16 [batch][padded_output_width], 16-byte aligned (ctx.dL_doutput): d(loss)/d(output) x the loss scale,
 *                       padding columns 0 -- the loss's own gradient; backward passes it through the output activation. May be null.
 *   target_dev, data_pdf_dev  as in tcnnb_training_step_ex; data_pdf_dev may be null.
 *   external_dL_dy_dev  when non-null the loss is not evaluated: target and pdf are not read, loss_values_dev is left untouched (the
 *                       reference leaves L unfilled), and dL_doutput_dev must be null -- the caller's buffer is the context's
 *                       dL_doutput, handed to tcnnb_backward. Only its presence is read here.
 *   prepare_input_gradients  accepted; nothing to prepare.
 * tcnnb_backward: trainer->backward(stream, ctx, input, dL_dinput, use_inference_params, param_gradients_mode) (trainer.h:147-153).
 *   Back-propagates dL_doutput_dev (fp16 [batch][padded_output_width], read when the call runs, so writes between forward and backward
 *   count) through the output activation into the trainer's gradient buffer, with param_gradients_mode and dL_dinput_dev as in
 *   tcnnb_training_step_ex. output_dev is accepted and not read. The optimizer does not run: tcnnb_optimizer_step does.
 * Rejected like tcnnb_training_step_ex: handles of tcnnb_module_create, data-parallel handles, batches that are not a multiple of
 * tcnnb_batch_size_granularity(), a null target without external_dL_dy, param_gradients_mode outside 0..2; and a non-null
 * dL_doutput_dev together with external_dL_dy_dev. */
int tcnnb_forward(tcnnb_model* m, tcnnb_stream stream, uint32_t batch_size, const float* input_dev, const float* target_dev, const float* data_pdf_dev, int use_inference_params,
                  int prepare_input_gradients, const void* external_dL_dy_dev, void* output_dev, float* loss_values_dev, void* dL_doutput_dev);
int tcnnb_backward(tcnnb_model* m, tcnnb_stream stream, uint32_t batch_size, const float* input_dev, const void* output_dev, const void* dL_doutput_dev, float* dL_dinput_dev,
                   int use_inference_params, int param_gradients_mode);
/* reduce_sum(values, n, stream) (reduce_sum.h:132-146): the fp32 sum of a device array, e.g. trainer->loss(ctx) of a forward context
 * (the sum of ctx.L). Synchronises the stream. */
int tcnnb_reduce_sum(tcnnb_stream stream, const float* values_dev, uint64_t n_elements, float* sum_out);
/* Data-parallel variant: this rank's shard of a global batch; the loss is normalised over global_batch_size
 * (loss n_total, relative_l2.h:62) so that gradient sums over ranks equal the single-GPU gradients. */
int tcnnb_training_step_shard(tcnnb_model* m, tcnnb_stream stream, uint32_t shard_batch_size, uint32_t global_batch_size, const float* input_dev, const float* target_dev, int run_optimizer);
/* trainer->optimizer_step(stream, loss_scale) (trainer.h:155-157): Adam on the current gradient buffers. */
int tcnnb_optimizer_step(tcnnb_model* m, tcnnb_stream stream);
/* The same optimizer step restricted to the parameter ranges [begins[r], begins[r] + counts[r]) (adam.h:48-129 is element-wise,
 * so a range is the reference kernel launched on a sub-span). Used by the sharded-optimizer data-parallel trainer: every rank
 * updates the network weights (a range starting at 0 that covers all of them) and its own slice of the grid table. */
/* generate_random_uniform<float>(stream, rng, n, out, lower, upper) (random.h:40-69) for a pcg32 with the given (state, inc):
 * thread i draws 4 consecutive numbers after advance(4 i), as the reference does. The caller advances its generator by n. */
int tcnnb_generate_random_uniform(tcnnb_stream stream, uint64_t rng_state, uint64_t rng_inc, uint64_t n_elements, float* out_dev, float lower, float upper);
/* generate_random_uniform<__half>: the same draws, each rounded to half and mapped as draw * (upper - lower) + lower in half arithmetic
 * (random.h:40-69 with T = __half). out_dev is fp16 [n_elements]; lower and upper are converted to half first. */
int tcnnb_generate_random_uniform_half(tcnnb_stream stream, uint64_t rng_state, uint64_t rng_inc, uint64_t n_elements, void* out_dev, float lower, float upper);
/* dst [cols][rows] = src [rows][cols] transposed, for 2- or 4-byte elements (fp16 / fp32): converts between the row-major (RM) and
 * column-major (CM) GPUMatrix layouts of the C++ object tier. src and dst must not overlap. Stream-ordered. */
int tcnnb_transpose(tcnnb_stream stream, uint32_t rows, uint32_t cols, uint32_t element_bytes, const void* src_dev, void* dst_dev);

/* ---- module tier: tcnn::cpp::Module as returned by create_network_with_input_encoding (cpp_api.h:76-125, src/cpp_api.cu:71-158) --
 * Parameters, gradients and activations are CALLER-owned device arrays (what the PyTorch extension passes, bindings.cpp:79-171):
 * params / dL_dparams are fp16 [n_params] (network weights first, then the grid table; 16-byte aligned), output / dL_doutput are
 * fp16 [n_elements][padded_output_width] rows, input is fp32 [n_elements][n_input_dims]. The handle is a tcnnb_model without
 * trainer state: destroy with tcnnb_destroy; tcnnb_n_params / tcnnb_padded_output_width / tcnnb_hyperparams apply; the trainer
 * calls do not. Difference from the reference, by design: forward keeps no context -- backward recomputes the forward pass inside
 * the fused kernel, so prepare_input_gradients is accepted and has nothing to prepare. dL_dinput (fp32 [n_elements][n_input_dims],
 * may be null) and dL_dparams (may be null) are overwritten (GradientMode::Overwrite, cpp_api.cu:104-125). */
int tcnnb_module_create(uint32_t n_input_dims, uint32_t n_output_dims, const char* encoding_json, const char* network_json, tcnnb_model** out);
/* Module::initialize_params(seed, params_full_precision, scale) (cpp_api.cu:140-143): pcg32{seed}, network then grid; device fp32 [n_params]. */
int tcnnb_module_initialize_params(tcnnb_model* m, uint64_t seed, float* params_full_precision_dev, float scale);
int tcnnb_module_inference(tcnnb_model* m, tcnnb_stream stream, uint32_t n_elements, const float* input_dev, void* output_dev, const void* params_dev);
int tcnnb_module_forward(tcnnb_model* m, tcnnb_stream stream, uint32_t n_elements, const float* input_dev, void* output_dev, const void* params_dev, int prepare_input_gradients);
int tcnnb_module_backward(tcnnb_model* m, tcnnb_stream stream, uint32_t n_elements, float* dL_dinput_dev, const void* dL_doutput_dev, void* dL_dparams_dev, const float* input_dev,
                          const void* output_dev, const void* params_dev);

/* ---- encoding tier: an encoding on its own ------------------------------------------------------------------------------------
 * tcnn::cpp::create_encoding(n_input_dims, json, Precision::Fp16) (cpp_api.h:124, src/cpp_api.cu:165-174) with the reference's JSON
 * keys (src/encoding.cu:60-120): "Grid" / "HashGrid" / "DenseGrid" / "TiledGrid" (n_features_per_level 1 / 2 / 4 / 8, 2 to 4 input
 * dimensions, Nearest / Linear / Smoothstep), "Identity", "Frequency", "TriangleWave", "OneBlob", "SphericalHarmonics" (degree <= 8) and
 * "Composite" of those (Concatenation; up to 8 nested encodings). Output width = the encoding's own width (no padding: alignment 0;
 * grids: n_levels * n_features_per_level). Caller-owned fp16 parameters [n_params] (nested grids one after the other; 0 for the
 * parameter-free encodings); batches are multiples of 256; stream-ordered. */
typedef struct tcnnb_encoding tcnnb_encoding;
int tcnnb_encoding_create(uint32_t n_input_dims, const char* encoding_json, tcnnb_encoding** out);
void tcnnb_encoding_destroy(tcnnb_encoding* e);
uint64_t tcnnb_encoding_n_params(const tcnnb_encoding* e);
uint32_t tcnnb_encoding_n_input_dims(const tcnnb_encoding* e);
uint32_t tcnnb_encoding_n_output_dims(const tcnnb_encoding* e);
int tcnnb_encoding_grid_levels(const tcnnb_encoding* e, uint32_t* n_levels, uint32_t* offsets, float* scales, uint32_t* resolutions);
/* GridEncoding::set_max_level (grid.h:69-92): fraction in [0, 1] of the levels that is active; the others encode to zero. */
int tcnnb_encoding_set_max_level(tcnnb_encoding* e, float max_level);
/* initialize_params (grid.h:1076-1079): U(-1e-4, 1e-4) * scale from pcg32{seed}; device fp32 [n_params]. */
int tcnnb_encoding_initialize_params(tcnnb_encoding* e, uint64_t seed, float* params_full_precision_dev, float scale);
/* forward == inference: fp32 [n][n_input_dims] -> fp16 [n][n_output_dims]. */
int tcnnb_encoding_forward(tcnnb_encoding* e, tcnnb_stream stream, uint32_t n_elements, const float* input_dev, void* output_dev, const void* params_dev);
/* backward: dL_dparams fp16 [n_params] (OVERWRITTEN) and / or dL_dinput fp32 [n][n_input_dims] from dL_doutput fp16 [n][n_output_dims];
 * either result pointer may be null. params_dev is needed for dL_dinput only. */
int tcnnb_encoding_backward(tcnnb_encoding* e, tcnnb_stream stream, uint32_t n_elements, float* dL_dinput_dev, const void* dL_doutput_dev, void* dL_dparams_dev, const float* input_dev,
                            const void* params_dev);
/* backward_backward_input (cpp_api.h:80; GridEncoding, grid.h:910-1042): the derivatives of a loss on dL_dinput, given
 * dL_ddLdinput fp32 [n][n_input_dims] and the dL_doutput fp16 [n][n_output_dims] of the first backward pass. Every non-null result is
 * OVERWRITTEN: dL_dparams fp16 [n_params], dL_ddLdoutput fp16 [n][n_output_dims], dL_dinput fp32 [n][n_input_dims]. dL_doutput is
 * needed for dL_dparams and dL_dinput, params_dev for dL_ddLdoutput and dL_dinput. Grid / HashGrid / DenseGrid / TiledGrid on their
 * own only: every other encoding (Composite included) fails with "<name> does not support double backward." */
int tcnnb_encoding_backward_backward_input(tcnnb_encoding* e, tcnnb_stream stream, uint32_t n_elements, const float* dL_ddLdinput_dev, const float* input_dev,
                                           const void* dL_doutput_dev, void* dL_dparams_dev, void* dL_ddLdoutput_dev, float* dL_dinput_dev, const void* params_dev);

/* ---- network tier: a FullyFusedMLP on its own -------------------------------------------------------------------------------
 * tcnn::create_network<T>(json) (network.h; src/network.cu:51-141; the object benchmarks/mlp/bench_mlp_ours.cu drives) and
 * tcnn::cpp::create_network (cpp_api.h:122; src/cpp_api.cu:160-162 = the same network behind the Identity encoding).
 * `network_json` carries the reference's keys ("otype", "n_neurons", "n_hidden_layers", "activation", "output_activation"); both
 * "FullyFusedMLP" and "CutlassMLP"/"MLP" run on the wgmma kernel of csrc/mlp_fused.cu (widths 16/32/64/128, any depth >= 1,
 * padded outputs up to 1024, also wider than n_neurons). Parameters are CALLER-owned fp16 device arrays (16-byte aligned) in the reference's layout
 * (fully_fused_mlp.cu:635-672): W_0 [n_neurons][input_width], (n_hidden_layers - 1) x [n_neurons][n_neurons],
 * W_out [padded_output_width][n_neurons], row-major; input_width = n_input_dims rounded up to 16.
 * Hidden activations: FullyFusedMLP's set (everything but Sine / SiLU); "CutlassMLP"/"MLP" also take Sine and SiLU, whose derivative
 * needs the pre-activations: the forward pass then keeps both (cutlass_mlp.cu:162-209), see tcnnb_network_n_forward_activations.
 * Batches are multiples of 256. All work is stream-ordered; nothing synchronises. */
typedef struct tcnnb_network tcnnb_network;
int tcnnb_network_create(uint32_t n_input_dims, uint32_t n_output_dims, const char* network_json, tcnnb_network** out);
void tcnnb_network_destroy(tcnnb_network* n);
uint64_t tcnnb_network_n_params(const tcnnb_network* n);
uint32_t tcnnb_network_input_width(const tcnnb_network* n);          /* n_input_dims rounded up to 16 */
uint32_t tcnnb_network_padded_output_width(const tcnnb_network* n);  /* network->padded_output_width() */
uint32_t tcnnb_network_width(const tcnnb_network* n);
uint32_t tcnnb_network_n_hidden_layers(const tcnnb_network* n);
/* CutlassMLP::num_forward_activations(): the [n][n_neurons] hidden rows tcnnb_network_forward writes and tcnnb_network_backward reads
 * -- n_hidden_layers, or 2 x n_hidden_layers for a Sine / SiLU hidden activation. */
uint32_t tcnnb_network_n_forward_activations(const tcnnb_network* n);
/* Network::initialize_params (fully_fused_mlp.cu:868-892): xavier uniform per matrix from pcg32{seed}; device fp32 [n_params]. A Sine
 * network takes the SIREN initialisation (cutlass_mlp.cu:362-371): 30 / fan_in for W_0, sqrt(6 / fan_in) for the other matrices. */
int tcnnb_network_initialize_params(tcnnb_network* n, uint64_t seed, float* params_full_precision_dev, float scale);
/* network->inference_mixed_precision(stream, input, output) (object.h / network.h): input fp16 [n][n_input_dims] (n_input_dims
 * must be a multiple of 16), output fp16 [n][padded_output_width]. */
int tcnnb_network_inference_mixed_precision(tcnnb_network* n, tcnnb_stream stream, uint32_t n_elements, const void* input_dev, void* output_dev, const void* params_dev);
/* network->forward: the same, and the post-activation hidden layers fp16 [n_hidden_layers][n][n_neurons] are written out
 * (what the reference's ForwardContext holds, fully_fused_mlp.cu:841-854). output_dev may be null. For a Sine / SiLU hidden
 * activation hidden_dev is [2][n_hidden_layers][n][n_neurons]: the post-activations first, then the fp16 pre-activations z, with
 * post = act(z) bit for bit (tcnnb_network_n_forward_activations() rows of [n][n_neurons] in all). */
int tcnnb_network_forward(tcnnb_network* n, tcnnb_stream stream, uint32_t n_elements, const void* input_dev, void* output_dev, void* hidden_dev, const void* params_dev);
/* network->backward (Network<T>::backward, fully_fused_mlp.cu:733-866) from what tcnnb_network_forward was given and wrote:
 * dL_doutput fp16 [n][padded_output_width] -> dL_dinput fp16 [n][n_input_dims] and dL_dparams fp16 [n_params] (OVERWRITTEN);
 * either may be null. output_dev is only read when the network has an output activation; hidden_dev has tcnnb_network_forward's
 * layout (Sine / SiLU: the derivative is taken at the pre-activations of its second half). Three kernels: the dgrad chain on
 * wgmma with the transposed weights read in place (mlp_fused.cu, BWD), the weight-gradient kernel (mlp_wgrad.cu), fp32 -> fp16. */
int tcnnb_network_backward(tcnnb_network* n, tcnnb_stream stream, uint32_t n_elements, const void* input_dev, const void* output_dev, const void* hidden_dev,
                           const void* dL_doutput_dev, const void* params_dev, void* dL_dinput_dev, void* dL_dparams_dev);
/* tcnn::cpp::Module::backward of cpp::create_network (cpp_api.cu:104-125): fp32 input through the Identity encoding; nothing is kept
 * from the forward call (the activations are recomputed). dL_dinput fp32 [n][n_input_dims], dL_dparams fp16; either may be null. */
int tcnnb_network_module_backward(tcnnb_network* n, tcnnb_stream stream, uint32_t n_elements, float* dL_dinput_dev, const void* dL_doutput_dev, void* dL_dparams_dev,
                                  const float* input_dev, const void* params_dev);
/* cpp::create_network semantics: fp32 input [n][n_input_dims] through the Identity encoding (padding features are 1,
 * encodings/identity.h:62-66) -> fp32 output [n][n_output_dims] (object.h:214-282). */
int tcnnb_network_inference(tcnnb_network* n, tcnnb_stream stream, uint32_t n_elements, const float* input_dev, float* output_dev, const void* params_dev);
/* Network<__half>::inference (object.h:214-282): fp16 input [n][n_input_dims] (a multiple of 16) -> fp32 output [n][n_output_dims], the
 * fp16 result of tcnnb_network_inference_mixed_precision trimmed and cast. */
int tcnnb_network_inference_half_input(tcnnb_network* n, tcnnb_stream stream, uint32_t n_elements, const void* input_dev, float* output_dev, const void* params_dev);
/* The same with the module tier's output convention (cpp_api.cu:82-83): fp16 [n][padded_output_width]. This is what
 * tcnn::cpp::Module::inference / forward of create_network returns. */
int tcnnb_network_module_inference(tcnnb_network* n, tcnnb_stream stream, uint32_t n_elements, const float* input_dev, void* output_dev, const void* params_dev);
/* Profiling only: clock64 phase stamps of the following forward / backward-chain launches are written to int64
 * [n_ctas][5 roles][64 events][8 fields] at clocks_dev (null = off): role = consumer warpgroup (4 unused), event = round * n_steps +
 * step, fields 0..3 = waiting for the weights / weights ready / product complete / epilogue done. Not part of the drop-in surface. */
int tcnnb_network_debug_clocks(tcnnb_network* n, void* clocks_dev);
/* Tests only: the following backward passes write g_l = dL/d(pre-activation of hidden layer l), the rows the weight-gradient kernel
 * reads, to grad_hidden_dev (fp16 [n_hidden_layers][n_elements][n_neurons], 16-byte aligned; null = the network's own scratch), with
 * or without dL/dparams. Not part of the drop-in surface. */
int tcnnb_network_debug_grad_hidden(tcnnb_network* n, void* grad_hidden_dev);

/* ---- data parallelism, natively over NCCL (no counterpart in the single-GPU reference; SURVEY.md section 8e) -------------
 * One process per GPU. Rendezvous is the host framework's job (torch.distributed in tcnn_b200/dp.py): rank 0 draws two NCCL
 * ids with tcnnb_dp_unique_id (128 bytes each), broadcasts them, and every rank calls tcnnb_dp_init. libnccl.so.2 is resolved
 * at run time on the first of these calls. A tcnnb_dp_training_step is: fwd+bwd on this rank's shard with the loss normalised
 * over the global batch; then, with shard_optimizer, reduce-scatter of the fp16 gradient vector, Adam on this rank's slice of the
 * (padded) parameter vector, all-gather of the updated fp16 slices on a side stream (the next step's binning pass overlaps it);
 * without, all-reduce of the gradients and the full Adam step on every replica. The zero-gradient skip of adam.h:79-82 is
 * evaluated on the reduced gradients either way, so the working parameters stay identical on all ranks. fp32 masters of a slice
 * are current on its owner only until tcnnb_dp_sync_full_precision gathers them. */
int tcnnb_dp_unique_id(void* out_id, uint64_t n_bytes);
int tcnnb_dp_init(tcnnb_model* m, const void* id_grads, const void* id_params, int world_size, int rank, int shard_optimizer);
int tcnnb_dp_shards_optimizer(const tcnnb_model* m); /* 1 if the sharded optimizer is in effect (aligned slices, world > 1) */
/* Peer-memory engine (single NVSwitch domain, <= 8 ranks). The host framework allocates one SYMMETRIC buffer of at least
 * 4 * tcnnb_n_params_padded + 256 bytes per rank that every rank has mapped (PyTorch: torch.distributed._symmetric_memory.empty +
 * rendezvous) and passes this rank's view of every rank's buffer (peer_bases[world], device pointers as integers) and the NVLS
 * multicast view of the same buffer (0 if the fabric has none). The model moves its working fp16 parameters and its gradient
 * vector into the buffer; from then on tcnnb_dp_training_step replaces reduce-scatter -> Adam -> all-gather by
 *   barrier -> ONE kernel on the rank's slice {gradient summed over the ranks with multimem.ld_reduce (or peer loads), Adam,
 *   updated fp16 weights published to all replicas with multimem.st (or peer stores)} -> barrier,
 * the barriers being flag exchanges over NVLink inside the same buffer. All ranks must call this collectively and synchronise
 * (host barrier) before the next step. The buffer must outlive the model's data-parallel state (tcnnb_dp_finish). */
int tcnnb_dp_attach_symmetric(tcnnb_model* m, const uint64_t* peer_bases, uint64_t multicast_base, uint64_t n_bytes);
/* 0 = not data parallel, 1 = NCCL collectives, 2 = peer-memory engine over peer loads / stores, 3 = over NVLS multicast */
int tcnnb_dp_engine(const tcnnb_model* m);
int tcnnb_dp_training_step(tcnnb_model* m, tcnnb_stream stream, uint32_t shard_batch_size, uint32_t global_batch_size, const float* input_dev, const float* target_dev);
int tcnnb_dp_sync_full_precision(tcnnb_model* m, tcnnb_stream stream);
int tcnnb_dp_finish(tcnnb_model* m); /* destroys the communicators (call before the process group goes away) */

/* Stream-ordering hook for callers that refresh the working parameters on another stream (the data-parallel all-gather):
 * the next kernel of this model that READS the parameters (fused step, inference, optimizer) waits for `cuda_event`
 * (a cudaEvent_t the caller keeps alive until that launch); work that does not read them (the binning pass) is not held back. */
int tcnnb_wait_before_compute(tcnnb_model* m, void* cuda_event);
int tcnnb_optimizer_step_ranges(tcnnb_model* m, tcnnb_stream stream, uint32_t n_ranges, const uint64_t* begins, const uint64_t* counts);
/* Device pointer + element count of the fp32 accumulator that holds the MLP weight gradients between the backward
 * pass and the optimizer (for the data-parallel all-reduce); the grid gradients are tcnnb_param_gradients(). */
float* tcnnb_mlp_gradient_accumulator(tcnnb_model* m);
/* Device pointer to the fp16 gradient table of the grid encoding (n_params - n_mlp_params elements); no side effects. */
void* tcnnb_grid_gradients(tcnnb_model* m);
/* trainer->loss(stream, ctx) (trainer.h:372-378, reduce_sum.h:132-146): sum of the loss values of the last step;
 * synchronises the stream. */
int tcnnb_loss(tcnnb_model* m, tcnnb_stream stream, float* loss_out);

/* ---- network->inference(stream, input, output) (object.h:214-282): fp32 [batch][n_out] ---- */
int tcnnb_inference(tcnnb_model* m, tcnnb_stream stream, uint32_t batch_size, const float* input_dev, float* output_dev);

/* ---- host-buffer entry points (what a foreign-language binding calls with its own arrays) ----
 * Copies inputs host->device (pinned staging inside the model), runs the step, copies the loss / outputs back and
 * synchronises. */
int tcnnb_training_step_host(tcnnb_model* m, uint32_t batch_size, const float* input_host, const float* target_host, float* loss_out);
/* Pipelined form of the same step. _submit enqueues {H2D of inputs and targets, training step, D2H of the loss} and returns a
 * ticket at once; _wait blocks until that step has finished and returns its loss. Up to TWO steps may be in flight, so a caller
 * that submits step i+1 before waiting for step i gets the copies of step i+1 overlapped with the kernels of step i (the copies
 * run on a copy stream; the binning pass of a step starts when its positions have landed, the fused kernel when its targets
 * have). Page-locked caller buffers are copied from directly; pageable ones are staged through pinned memory inside the model
 * and may be reused by the caller as soon as _submit returns. A pinned buffer must stay untouched until its ticket is waited for.
 * The handle is not thread-safe (as the reference's Trainer is not): calls on one model must come from one thread at a time. */
int tcnnb_training_step_host_submit(tcnnb_model* m, uint32_t batch_size, const float* input_host, const float* target_host, uint64_t* ticket_out);
int tcnnb_training_step_host_wait(tcnnb_model* m, uint64_t ticket, float* loss_out);
/* Data-parallel form (after tcnnb_dp_init): this rank's HOST shard of a global batch; the loss returned by _wait is the GLOBAL
 * loss (the partial sums are all-reduced on the device behind the step). */
int tcnnb_dp_training_step_host_submit(tcnnb_model* m, uint32_t shard_batch_size, uint32_t global_batch_size, const float* input_host, const float* target_host, uint64_t* ticket_out);
int tcnnb_inference_host(tcnnb_model* m, uint32_t batch_size, const float* input_host, float* output_host);

/* ---- trainer->serialize / deserialize (trainer.h:442-482): fp16 params (+ optional Adam state) as raw bytes ---- */
uint64_t tcnnb_serialize_size(const tcnnb_model* m, int with_optimizer);
int tcnnb_serialize(tcnnb_model* m, void* dst_host, uint64_t size, int with_optimizer);
int tcnnb_deserialize(tcnnb_model* m, const void* src_host, uint64_t size);

/* ---- test / profiling taps: per-sample intermediates of the fused kernel (null = off). Not part of the drop-in surface. */
typedef struct {
	void* encoded;        /* fp16 [batch][64] */
	void* hidden;         /* fp16 [n_hidden][batch][64] */
	void* output;         /* fp16 [batch][16] */
	void* dL_doutput;     /* fp16 [batch][16] */
	void* grad_hidden;    /* fp16 [n_hidden][batch][64] */
	void* dL_dencoded;    /* fp16 [batch][64] */
	float* loss_values;   /* fp32 [batch][n_out] */
} tcnnb_debug_taps;
int tcnnb_set_debug_taps(tcnnb_model* m, const tcnnb_debug_taps* taps);
/* Test-only switches (not dispatch knobs of the product path): "binning" 0/1 -- run the step without / with the spatial
 * binning pass (tests assert both touch the same table entries); "adam_steps32" 1 -- keep Adam's step counters 32 bits wide
 * although 16-bit ones give the same updates (tests compare the two layouts), 0 -- back to the width the trainer chose. */
int tcnnb_debug_set(tcnnb_model* m, const char* key, int value);
/* Per-kernel device timing for the roofline report: when enabled, CUDA events bracket the binning kernels, the fused fwd+bwd kernel
 * and the optimizer kernel of every training step on the caller's stream; tcnnb_read_profile synchronises and returns the sums. */
int tcnnb_set_profiling(tcnnb_model* m, int enable);
int tcnnb_read_profile(tcnnb_model* m, float* fused_ms_total, float* optimizer_ms_total, float* binning_ms_total, uint32_t* n_steps);
/* Number of kernels this library launched since load (bench.py's gpu_launches). */
uint64_t tcnnb_kernel_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif
