/*
 * xrnerf_b200 — C ABI of the H100-native (sm_90a) volumetric-rendering hot path.
 *
 * Drop-in boundary for the two native interfaces the reference's hot path binds:
 *   #1 `raymarch_cuda`  (pybind module; /root/reference/extensions/ngp_raymarch/include/pybind_api.h:3-95,
 *                        exported in src/pybind_api.cu:6-17) — 10 functions, mirrored 1:1 below (xrb_rm_*);
 *   #2 `tinycudann`     (third-party; call sites /root/reference/xrnerf/models/mlps/hashnerf_mlp.py:36-45,
 *                        :55-79, :107-111) — hash-grid / SH encodings and fully-fused MLPs (xrb_tcnn_*, xrb_ngp_*);
 * plus the fused kernels that replace whole call chains of the reference's Python hot loop
 * (SURVEY §3b/§3c): xrb_ngp_render_* and the NeRF/Mip-NeRF kernels xrb_nerf_*.
 *
 * Conventions (differences from the reference ABI are deliberate and listed in INTEGRATION.md):
 *   - plain pointers + sizes only; every pointer is a DEVICE pointer unless the name ends in `_host`;
 *   - every entry point takes the CUDA stream to launch on (`void *stream` = cudaStream_t) and NEVER
 *     synchronises the device (the reference ends every wrapper with cudaDeviceSynchronize());
 *   - every entry point returns 0 on success, a cudaError_t value (>0) on a CUDA failure, or a negative
 *     XRB_E_* code on bad arguments (the reference surfaces no errors at all);
 *   - the hidden per-translation-unit host RNG of the reference (`static pcg32 rng{9121}`, advanced by 2^32
 *     per API call; raymarch_shared.h:38) is an explicit (seed, n_prior_calls) argument pair;
 *   - sample buffers are laid out in RAY ORDER (exclusive prefix sums) instead of atomic-arrival order; the
 *     (count, base) contract of `numsteps` is unchanged.
 */
#ifndef XRNERF_B200_H
#define XRNERF_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define XRB_OK 0
#define XRB_E_BADARG (-1)
#define XRB_E_UNSUPPORTED (-2)
#define XRB_E_WORKSPACE (-3)

/* activation enum of the reference (raymarch_shared.h:619-625) */
#define XRB_ACT_NONE 0
#define XRB_ACT_RELU 1
#define XRB_ACT_LOGISTIC 2
#define XRB_ACT_EXPONENTIAL 3

/* ---- data-parallel optimiser step over NVLink peer memory (csrc/peer_adam.cu). Replaces, for the Instant-NGP trainer, what the reference gets from torch DDP's gradient all-reduce +
 * torch.optim.Adam on every rank (core/apis/train.py:28-36, hashnerf.py:32-52): one exchange block per rank (flags | bf16 table gradient | fp32 MLP gradients | fp16 working table),
 * allocated with xrb_peer_alloc, its 64-byte IPC handle passed to the other processes by the caller (any transport), opened there with xrb_peer_open.
 *   xrb_peer_publish_grads  my fp32 gradients -> my block, then ready[rank] = step in every block
 *   xrb_peer_adam_step      waits for every rank's gradients, Adam on my slice [rank*per, rank*per+per) of the table from the SUM of all ranks' gradients (mean: / world), new fp16
 *                           values stored into every rank's working table; both MLP groups updated identically on every rank; returns (in stream order) once every rank's slice
 *                           has landed in my working table. `step` is a counter starting at 1 that every rank advances together; opt_step is Adam's bias-correction step.
 * Hyper-parameters as xrb_adam_ema_step. A rank that does not show up within ~10 s makes the kernels give up: xrb_peer_status != 0 (no hang). */
typedef struct { int world, rank; void *base[8]; size_t off_g16, off_gmlp, off_t16; int64_t n_table, per, n_mlp; } xrb_peer_layout;
typedef struct { float *param; void *param_fp16; float *exp_avg, *exp_avg_sq, *ema; int64_t n, g_off; } xrb_peer_mlp_group;
int xrb_peer_alloc(size_t bytes, void **ptr, void *ipc_handle64);
int xrb_peer_open(const void *ipc_handle64, void **ptr);
int xrb_peer_close(void *ptr);
int xrb_peer_free(void *ptr);
int xrb_peer_publish_grads(const xrb_peer_layout *layout, const float *grad_table, const float *grad_mlp, uint32_t step, void *stream);
int xrb_peer_adam_step(const xrb_peer_layout *layout, float *master_slice, float *exp_avg_slice, float *exp_avg_sq_slice, float *ema_slice, const xrb_peer_mlp_group *mlp0,
                       const xrb_peer_mlp_group *mlp1, float lr, float beta1, float beta2, float eps, float weight_decay, int opt_step, float ema_momentum, uint32_t step, void *stream);
int xrb_peer_status(const void *own_block, uint32_t *status_host, void *stream);

/* ABI version, bumped on any signature change; and the compute capability the library was built for (100). */
int xrb_abi_version(void);
int xrb_built_for_sm(void);
/* last error string of the calling thread (static storage) */
const char *xrb_last_error(void);

/* ------------------------------------------------------------------------------------------------
 * Boundary #1 — raymarch_cuda equivalents
 * ---------------------------------------------------------------------------------------------- */

/* replaces generate_grid_samples_nerf_nonuniform_api (pybind_api.h:5-10; src/generate_grid_samples_nerf_nonuniform.cu:44-87).
 * grid f32[8*128^3]; positions f32[n,3]; indices i32[n]. */
int xrb_rm_generate_grid_samples(const float *grid, int ema_step, int n_elements, int max_cascade, float thresh, float aabb0,
                                 float aabb1, uint64_t seed, int64_t n_prior_calls, float *positions, int32_t *indices, void *stream);

/* replaces mark_untrained_density_grid_api (pybind_api.h:12-16; src/mark_untrained_density_grid.cu:53-82).
 * focal f32[I,2]; xforms f32[I,4,3]; grid f32[n_elements] is FULLY written (0 seen / -1 unseen): the reference's
 * dependence on uninitialised memory (SURVEY Appendix B Q1) is removed. */
int xrb_rm_mark_untrained_density_grid(const float *focal, const float *xforms, int n_elements, int n_images, int res0, int res1,
                                       float *grid, void *stream);

/* replaces splat_grid_samples_nerf_max_nearest_neighbor_api (pybind_api.h:18-20). mlp_out f32[n,padded_width]. */
int xrb_rm_splat_grid_samples(const float *mlp_out, const int32_t *indices, int padded_width, int n, float *grid_tmp, void *stream);

/* replaces ema_grid_samples_nerf_api (pybind_api.h:22-23). */
int xrb_rm_ema_grid_samples(const float *grid_tmp, int n_elements, float decay, float *grid, void *stream);

/* replaces update_bitfield_api (pybind_api.h:25-26; src/update_bitfield.cu:74-116). mean f32[>=1] (only [0] written);
 * bitfield u8[8*128^3/8]. Deterministic (fixed-order) mean. */
size_t xrb_rm_update_bitfield_workspace(void);   /* bytes of device scratch (the per-block partial sums of the fixed-order mean) */
int xrb_rm_update_bitfield(const float *grid, float *mean, uint8_t *bitfield, void *workspace, void *stream);

/* replaces rays_sampler_api (pybind_api.h:28-42; src/ray_sampler.cu:118-200).
 * rays_o/rays_d f32[N,3]; bitfield u8[2097152]; coords_out f32[max_samples,7] (rows = pos_warped[3], dt_warped,
 * dir_warped[3]); rays_index i32[N]; numsteps i32[N,2] = (count, base); counters i32[2] = (#rays that got a slot,
 * total samples incl. overflowed rays). metadata/img_ids/xforms are accepted for signature parity and unused,
 * exactly like the reference kernel (ray_sampler.cu:29-38 reads them into dead locals); they may be NULL.
 * workspace: device scratch of xrb_rm_rays_sampler_workspace(N) bytes. */
size_t xrb_rm_rays_sampler_workspace(int n_rays);
int xrb_rm_rays_sampler(const float *rays_o, const float *rays_d, const uint8_t *bitfield, const float *metadata,
                        const int32_t *img_ids, const float *xforms, int n_rays, int max_samples, float aabb0, float aabb1,
                        float near_distance, float cone_angle, uint64_t seed, int64_t n_prior_calls, float *coords_out,
                        int32_t *rays_index, int32_t *numsteps, int32_t *counters, void *workspace, void *stream);

/* replaces compacted_coord_api (pybind_api.h:44-58; src/compacted_coord.cu:79-143). network_output and the
 * activations are accepted and unused (the reference's transmittance loop is dead code, Q3). */
size_t xrb_rm_compacted_coord_workspace(int n_rays);
int xrb_rm_compacted_coord(const float *network_output, const float *coords_in, const int32_t *numsteps, int n_rays,
                           int max_compacted, float *coords_out, int32_t *numsteps_compacted, int32_t *ray_counter,
                           int32_t *step_counter, void *workspace, void *stream);

/* Training bookkeeping (no reference counterpart: the reference never counts them): ADDS to *accum (device i64) the number of rays whose every marched sample
 * survived compacted_coord's truncation (numsteps_compacted.count == numsteps.count), i.e. the rays the step really trains. */
int xrb_ngp_count_trained_rays(const int32_t *numsteps, const int32_t *numsteps_compacted, int n_rays, int64_t *accum, void *stream);

/* replaces calc_rgb_forward_api (pybind_api.h:60-72). raw f32[S,4]; coords f32[S,7]; bg f32[N,3]; rgb f32[N,3]. */
int xrb_rm_calc_rgb_forward(const float *raw, const float *coords, const int32_t *numsteps, const int32_t *numsteps_compacted,
                            const float *bg, int n_rays, int rgb_act, int dens_act, float *rgb_out, void *stream);

/* replaces calc_rgb_backward_api (pybind_api.h:74-86). Writes dL/draw f32[S,4] for the rows owned by rays; the caller
 * zero-fills padding rows (as the reference's Python wrapper does, hashnerf_render.py:122-125). */
int xrb_rm_calc_rgb_backward(const float *raw, const int32_t *numsteps_compacted, const float *coords, const float *grad_rgb,
                             const float *rgb, const float *grid_mean, int n_rays, int rgb_act, int dens_act, float *dl_draw,
                             void *stream);

/* replaces calc_rgb_influence_api (pybind_api.h:88-95). bg3_host: 3 floats on the HOST (as in the reference). */
int xrb_rm_calc_rgb_inference(const float *raw, const float *coords, const int32_t *numsteps, const float *bg3_host, int n_rays,
                              int rgb_act, int dens_act, float *rgb_out, float *alpha_out, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Boundary #2 — tcnn-shaped encodings / networks, and the fused NGP field
 * ---------------------------------------------------------------------------------------------- */

typedef struct {
    int n_levels;            /* 16 */
    int n_features;          /* 2 (only 2 is implemented) */
    int log2_hashmap_size;   /* 19 */
    int base_resolution;     /* 16 */
    float per_level_scale;   /* 2^(log2(2048/16)/15), hashnerf_mlp.py:17-20 */
    int width;               /* n_neurons, 64 (only 64 is implemented) */
    int density_hidden;      /* hidden layers of density_net (config key num_layers / n_hidden_layers), 1..4 */
    int color_hidden;        /* hidden layers of color_net, 1..4 */
} xrb_ngp_config;

/* The hash table as the kernels read it: the fp16 working copy in tcnn's layout (always) and, optionally, its CELL IMAGE — a
 * gather-friendly copy of the first n_packed_levels levels in which every grid cell stores its 8 corner entries as one aligned 32-byte
 * record, so that a sample reads ONE 256-bit word per level instead of 8 scattered 4-byte entries (same values, 8x fewer L1 lines).
 * cell_image == NULL / n_packed_levels == 0: every level is gathered from the table. The image is produced from the fp16 table by
 * xrb_ngp_build_cell_image (xrb_ngp_cell_image_bytes bytes, 32-byte aligned; levels 0..4 = 10.6 MB, ..5 = 27.6 MB, ..6 = 72.6 MB for the
 * reference config) and must be rebuilt when the table changes. It replaces nothing in the reference: tcnn gathers 8 entries per level
 * (call site /root/reference/xrnerf/models/mlps/hashnerf_mlp.py:60). */
typedef struct {
    const void *table_fp16;
    const void *cell_image;
    int n_packed_levels;
} xrb_ngp_table;
size_t xrb_ngp_cell_image_bytes(const xrb_ngp_config *cfg, int n_packed_levels);
int xrb_ngp_build_cell_image(const xrb_ngp_config *cfg, const void *table_fp16, int n_packed_levels, void *cell_image, void *stream);

/* number of scalars in the hash table / density net / colour net parameter vectors, and level offsets */
int64_t xrb_tcnn_hashgrid_num_params(const xrb_ngp_config *cfg);
int64_t xrb_tcnn_density_num_params(const xrb_ngp_config *cfg);
int64_t xrb_tcnn_color_num_params(const xrb_ngp_config *cfg);
int xrb_tcnn_hashgrid_layout(const xrb_ngp_config *cfg, uint32_t *offsets_host /*[n_levels+1]*/, float *scales_host, uint32_t *res_host);

/* fp32 master -> fp16 working copy (what tcnn does on every forward; done once per optimiser step here) */
int xrb_tcnn_cast_params(const float *src, void *dst_fp16, int64_t n, void *stream);
/* packs the density+colour weights (fp32 master, tcnn layout W[out][in]) into the wgmma shared-memory image
 * (128-byte-swizzled K-major tiles) the tensor-core kernels bulk-copy; image size = xrb_ngp_weight_image_bytes(). */
size_t xrb_ngp_weight_image_bytes(const xrb_ngp_config *cfg);
int xrb_ngp_pack_weights(const xrb_ngp_config *cfg, const float *density_params, const float *color_params, void *image, void *stream);

/* tcnn.Encoding(HashGrid).forward: x f32[n,3] in [0,1] -> enc fp16[n, n_levels*n_features] */
int xrb_tcnn_hashgrid_forward(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const float *x, int x_stride, int n, void *enc_fp16, void *stream);
/* tcnn.Encoding(SphericalHarmonics, degree 4).forward: dirs f32[n,3] in [0,1] -> fp16[n,16] */
int xrb_tcnn_sh4_forward(const float *dirs, int dir_stride, int n, void *out_fp16, void *stream);
/* tcnn.Network(FullyFusedMLP).forward, SIMT reference-grade implementation: x fp16[n,in_w] -> y fp16[n,16] */
int xrb_tcnn_mlp_forward(const void *params_fp16, const void *x_fp16, int n, int in_w, int width, int n_hidden, void *y_fp16, void *stream);

/* Backward of the two stand-alone modules (what `tinycudann`'s autograd bindings give the reference when it trains through them,
 * hashnerf_mlp.py:36-45,:60-77): d_enc fp16[n,32] (x grad_scale) -> fp32 table gradient (ACCUMULATED); and for the MLP x fp16[n,32],
 * dy fp16[n,16] -> dx fp16[n,32] (may be NULL) + fp32 parameter gradient (ACCUMULATED, tcnn layout). CUDA-core kernels: the training hot path
 * is the fused field (xrb_ngp_mlp_backward_tc); these exist so that the composable modules are trainable. */
int xrb_tcnn_hashgrid_backward(const xrb_ngp_config *cfg, const float *x, int x_stride, int n, const void *d_enc_fp16, float grad_scale, float *d_table, void *stream);
int xrb_tcnn_mlp_backward(const void *params_fp16, const void *x_fp16, const void *dy_fp16, int n, int in_w, int width, int n_hidden, void *dx_fp16, float *d_params,
                          void *stream);

/* HashNerfMLP.run_mlp (hashnerf_mlp.py:55-79) fused: pts/dirs f32 rows (stride in floats, so `coords[:, :3]` /
 * `coords[:, 4:]` views of a [S,7] buffer work in place) -> raw f32[n,4] = (rgb3, density1).
 * impl: 0 = SIMT (CUDA cores), 1 (or 2) = wgmma tensor-core tiles (weights from `weight_image`).
 * n_rows_dev (optional, device pointer): the effective row count is min(n, *n_rows_dev) — a sample count produced on the device by the
 * march / compaction never has to visit the host. */
int xrb_ngp_mlp_forward(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *density_fp16, const void *color_fp16,
                        const void *weight_image, const float *pts, int pts_stride, const float *dirs, int dirs_stride, int n,
                        const int32_t *n_rows_dev, float *raw, int impl, void *stream);
/* HashNerfMLP.run_density (hashnerf_mlp.py:107-111): -> density f32[n] (raw, pre-activation) */
int xrb_ngp_density_forward(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *density_fp16, const void *weight_image,
                            const float *pts, int pts_stride, int n, float *density, int impl, void *stream);
/* The raw density and its gradient with respect to the warped position (mesh vertex normals), on CUDA cores, one thread per point:
 *   density[i] (f32[n], may be NULL) is bit-identical to xrb_ngp_density_forward with impl = 0 at the same position;
 *   grad[i] (f32[n,3]) is d(raw density)/d(warped position) of that same function, evaluated in fp32 on the fp16 parameters. The fp16 rounding of the
 *   encoding and of the hidden activations is taken as the identity (straight-through); the ReLU masks are the forward's (a unit is live iff its fp16
 *   activation is > 0, as in the CUDA-core backward). Level l contributes scale_l * sum over its 8 corners of dw_c/df * v_c, with v_c the corner's fp16
 *   feature pair and f the in-cell position of the level's grid cell; at a cell face the derivative is the one inside the cell the forward gathered from
 *   (the cell whose lower face it is).
 * Positions must lie in [0,1]^3, as for every field entry point. n == 0 is a no-op that touches no pointer. Returns XRB_E_BADARG for a null cfg, table,
 * density_fp16, pts or grad, n < 0 or pts_stride < 3, and XRB_E_UNSUPPORTED for a config the field does not support, all before any CUDA call. */
int xrb_ngp_density_grad(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *density_fp16, const float *pts, int pts_stride, int n,
                         float *density /* f32[n], may be NULL */, float *grad /* f32[n,3] */, void *stream);

/* Backward of run_mlp: dL/draw f32[n,4] -> fp32 gradients of the three parameter vectors (ACCUMULATED into the
 * outputs with atomics; caller zeroes them). */
int xrb_ngp_mlp_backward(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *density_fp16, const void *color_fp16,
                         const float *pts, int pts_stride, const float *dirs, int dirs_stride, const float *dl_draw, int n,
                         float *d_table, float *d_density, float *d_color, void *stream);

/* The same backward on wgmma tensor-core tiles (csrc/ngp_backward_tc.cu): dX = dZ.W and dW += dZ^T.X per layer as tensor-core instructions, the weight
 * gradients accumulated in registers over the whole launch; fp16 operands (dZ staged with a fixed 2^12 scale), fp32 accumulation. Built for
 * (density_hidden, color_hidden) = (1,1) and (1,2) — the reference config, configs/instant_ngp/nerf_blender_local01.py:113,123 — and returns
 * XRB_E_UNSUPPORTED otherwise. n_rows_dev (optional, device): the effective row count is min(n, *n_rows_dev) (the compacted sample count
 * stays on the device). Same accumulate-into-outputs contract as xrb_ngp_mlp_backward. */
int xrb_ngp_mlp_backward_tc(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *weight_image, const float *pts, int pts_stride,
                            const float *dirs, int dirs_stride, const float *dl_draw, int n, const int32_t *n_rows_dev, float *d_table,
                            float *d_density, float *d_color, void *stream);

/* Fused Adam step on an fp32 master vector + refresh of its fp16 working copy (torch.optim.Adam semantics with
 * L2 weight_decay folded into the gradient; configs/instant_ngp/nerf_blender_local01.py:13-18), with the runner's EMAHook folded into the same
 * pass (configs/instant_ngp/nerf_blender_local01.py:24: momentum 0.05; mmcv EMAHook.after_train_iter: ema = (1 - m) * ema + m * param,
 * m = min(momentum, (1 + iter) / (warm_up + iter)) computed by the caller): ema f32[n] (NULL = no EMA), initialised by the caller as a copy of
 * param (EMAHook.before_run). grad is divided by grad_div first (world size after a sum all-reduce). param_fp16 NULL = no fp16 copy. */
int xrb_adam_ema_step(float *param, void *param_fp16, const float *grad, float *exp_avg, float *exp_avg_sq, int64_t n, float lr,
                      float beta1, float beta2, float eps, float weight_decay, int step, float grad_div, float *ema, float ema_momentum, void *stream);

/* The same step reading a bf16 gradient (the wire format of the sharded data-parallel step in xrnerf_b200/train.py: reduce-scatter of bf16
 * gradients -> this Adam on the rank's own shard of (param, exp_avg, exp_avg_sq, ema) -> all-gather of the refreshed fp16 working copy). */
int xrb_adam_ema_step_bf16grad(float *param, void *param_fp16, const void *grad_bf16, float *exp_avg, float *exp_avg_sq, int64_t n, float lr,
                               float beta1, float beta2, float eps, float weight_decay, int step, float grad_div, float *ema, float ema_momentum,
                               void *stream);
/* fp32 -> bf16 (round to nearest even), n elements */
int xrb_pack_bf16(const float *src, void *dst_bf16, int64_t n, void *stream);
/* HashNerfNetwork.train_step's loss (xrnerf/models/networks/hashnerf.py:39-44, utils/metrics.py:8-16): 5 * HuberLoss(delta, reduction 'sum') over
 * n_elements values; writes d loss / d rgb and ADDS the loss value to *loss_accum (device float), one pass. */
int xrb_ngp_huber5_grad(const float *rgb, const float *target, int64_t n_elements, float delta, float *grad_out, float *loss_accum, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Fused render of a ray batch (inference): replaces the chain
 *   rays_sampler -> HashNerfMLP.run_mlp -> calc_rgb_influence  (ngp_grid_sampler.py:205-228, hashnerf_mlp.py:55-79,
 *   hashnerf_render.py:42-46) without materialising coords[S,7] or raw[S,4] in HBM.
 * rays_o/rays_d f32[N,3]; rgb f32[N,3]; alpha f32[N]; numsteps i32[N,2] (count, base) is also produced;
 * counters i32[2] as in xrb_rm_rays_sampler (counters[1] = total samples marched).
 * Up to 2^21 samples, the field evaluates the marched samples bucketed by position (a counting sort on a 64^3 Morton grid, on the
 * device), not in ray order; every output row is bit-identical to a ray-order evaluation. Larger sample counts are evaluated in ray order.
 * workspace: xrb_ngp_render_workspace(N, max_samples) bytes, 256-byte aligned. It starts with the march workspace, rounded up to
 * 256 bytes, followed by coords f32[max_samples,7], raw f32[max_samples,4] and the field's evaluation order u32[max_samples]
 * (when n = min(counters[1], max_samples) <= 2^21, order[0, n) is a permutation of the rows [0, n)).
 * ev_before_field / ev_after_field: optional cudaEvent_t handles (NULL = none) recorded on `stream` right before the sample-ordering
 * kernels and right after the field kernel, so a caller can time the ordering plus the dominant kernel live inside its own timed
 * region (no library-global state).
 * ---------------------------------------------------------------------------------------------- */
size_t xrb_ngp_render_workspace(int n_rays, int max_samples);
int xrb_ngp_render(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *weight_image, const uint8_t *bitfield,
                   const float *rays_o, const float *rays_d, int n_rays, int max_samples, float aabb0, float aabb1,
                   float near_distance, float cone_angle, uint64_t seed, int64_t n_prior_calls, const float *bg3_host, int rgb_act,
                   int dens_act, float *rgb_out, float *alpha_out, int32_t *numsteps, int32_t *counters, void *workspace,
                   void *ev_before_field, void *ev_after_field, void *stream);

/* Single-launch variant: march + hash encode + MLPs (wgmma) + composite in ONE persistent warp-specialised kernel; no per-sample
 * buffer exists, so there is no max_samples / overflow case. Same arithmetic as xrb_ngp_render (sample positions bit-identical; the
 * composite is a segmented warp scan: fp32 re-association only). `workspace`: xrb_ngp_render_fused_workspace() bytes, 256-byte
 * aligned, ZEROED ONCE by the caller at allocation (the kernel leaves its scheduler words zero on exit); one workspace per stream.
 * n_samples_out i32[n_rays] (samples per ray) may be NULL. alpha_out f32[n_rays]. */
size_t xrb_ngp_render_fused_workspace(void);
int xrb_ngp_render_fused(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *weight_image, const uint8_t *bitfield,
                         const float *rays_o, const float *rays_d, int n_rays, float aabb0, float aabb1, float near_distance,
                         float cone_angle, uint64_t seed, int64_t n_prior_calls, const float *bg3_host, int rgb_act, int dens_act,
                         float *rgb_out, float *alpha_out, int32_t *n_samples_out, void *workspace, void *stream);

/* Depth of the two render paths above: the same call with one more output, depth_out f32[n_rays] (non-NULL), right after alpha_out.
 *   depth = sum_k T_k * alpha_k * t_k
 * over the ray's samples k (T_k: transmittance in front of sample k, alpha_k: its opacity, t_k: its ray parameter), so depth is in the
 * units of t (for unit-norm rays: distance in the frame of [aabb0, aabb1]^3). It is NOT divided by alpha (as NerfRender's depth_map);
 * a ray without samples has depth 0. rgb, alpha and the sample counts are bit-identical to the depth-free call's.
 * xrb_ngp_render_depth rebuilds t_k from the sample row, t_k = ((aabb0 + x_k * (aabb1 - aabb0)) - o) . d / (d . d) with x_k the warped
 * position; xrb_ngp_render_fused_depth uses the marched t_k itself. Both agree to fp32 rounding.
 * Disparity (xrnerf_b200.ngp.disparity) = 1 / max(1e-10, depth / alpha) where alpha > 0 and 0 where alpha == 0: unlike NeRF's disp_map,
 * which is NaN there, so that an image of rays that miss the scene normalises without NaNs. */
int xrb_ngp_render_depth(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *weight_image, const uint8_t *bitfield,
                         const float *rays_o, const float *rays_d, int n_rays, int max_samples, float aabb0, float aabb1,
                         float near_distance, float cone_angle, uint64_t seed, int64_t n_prior_calls, const float *bg3_host, int rgb_act,
                         int dens_act, float *rgb_out, float *alpha_out, float *depth_out, int32_t *numsteps, int32_t *counters, void *workspace,
                         void *ev_before_field, void *ev_after_field, void *stream);
int xrb_ngp_render_fused_depth(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *weight_image, const uint8_t *bitfield,
                               const float *rays_o, const float *rays_d, int n_rays, float aabb0, float aabb1, float near_distance,
                               float cone_angle, uint64_t seed, int64_t n_prior_calls, const float *bg3_host, int rgb_act, int dens_act,
                               float *rgb_out, float *alpha_out, float *depth_out, int32_t *n_samples_out, void *workspace, void *stream);


/* ------------------------------------------------------------------------------------------------
 * NeRF / Mip-NeRF composite + sampling kernels (pure-PyTorch in the reference)
 * ---------------------------------------------------------------------------------------------- */

/* NerfRender.forward (nerf_render.py:47-98) / MipNerfRender (mipnerf_render.py:13-33), forward.
 * raw f32[N,S,4]; z_vals f32[N,S] (mip==0) or f32[N,S+1] (mip==1); rays_d f32[N,3].
 * density_act: XRB_ACT_RELU or 4 (= softplus). Outputs rgb[N,3], disp[N], acc[N], weights[N,S]. */
#define XRB_ACT_SOFTPLUS 4
int xrb_nerf_composite_forward(const float *raw, const float *z_vals, const float *rays_d, int n_rays, int n_samples, int mip,
                               int white_bkgd, float rgb_padding, float density_bias, int density_act, float *rgb, float *disp,
                               float *acc, float *weights, void *stream);
/* The same forward, also writing depth f32[N] = sum_k w_k z_k (the interval mid-points (z_k + z_{k+1})/2 when mip), not divided by acc (the
 * convention of xrb_ngp_render_depth): the value disp is formed from. rgb, disp, acc and weights are bit-identical to xrb_nerf_composite_forward's.
 * Arguments are checked as there; a NULL depth is XRB_E_BADARG. */
int xrb_nerf_composite_forward_depth(const float *raw, const float *z_vals, const float *rays_d, int n_rays, int n_samples, int mip,
                                     int white_bkgd, float rgb_padding, float density_bias, int density_act, float *rgb, float *disp,
                                     float *acc, float *weights, float *depth, void *stream);
/* backward wrt raw of rgb (grad_rgb f32[N,3]); disp/acc/weights are treated as non-differentiated outputs
 * exactly as the reference's losses use them (nerf.py:79-84: loss on rgb only). */
int xrb_nerf_composite_backward(const float *raw, const float *z_vals, const float *rays_d, const float *grad_rgb, int n_rays,
                                int n_samples, int mip, int white_bkgd, float rgb_padding, float density_bias, int density_act,
                                float *d_raw, void *stream);

/* sample_pdf (hierarchical_sample.py:6-53), deterministic (`det`) or with caller-supplied uniforms u f32[N,n_importance].
 * z_vals f32[N,S], weights f32[N,S] -> z_out f32[N,S+n_importance] sorted, pts f32[N,S+n_importance,3] (may be NULL). */
int xrb_nerf_sample_pdf(const float *z_vals, const float *weights, const float *rays_o, const float *rays_d, const float *u,
                        int n_rays, int n_samples, int n_importance, float *z_out, float *pts_out, void *stream);

/* BaseEmbedder.forward (embedders/base.py:57-74): pts f32[M,3], dirs f32[R,3] broadcast over S=M/R samples ->
 * embedded f32[M, 3+6*multires + 3+6*multires_dirs] */
int xrb_nerf_posenc(const float *pts, const float *viewdirs, int64_t n_pts, int samples_per_ray, int multires, int multires_dirs,
                    float *embedded, void *stream);

/* NerfMLP.run_mlp (xrnerf/models/mlps/nerf_mlp.py:70-94; netdepth 8, netwidth 256, skips [4], use_viewdirs) as one persistent wgmma
 * kernel, inference forward. enc_image: the fp16 encoding tile image of n rows with (input_ch, input_ch_dirs) = (63,27) NeRF or (96,27) Mip-NeRF
 * -> raw f32[n,4] = (rgb3, alpha1). weight_image / bias: produced by xrnerf_b200.nerf_mlp.pack_nerf_mlp (fp16 slabs in streaming order; bias = fp32
 * vector + fp16 copy). Each layer's fp32 accumulator is rounded to fp16 before the bias is added in fp16; alpha is a dot product in the epilogue of
 * pts_linears.7. All pointers 16-byte aligned. */
int xrb_nerf_mlp_forward(const void *weight_image, const float *bias, const void *enc_image, int64_t n_rows, int input_ch, int input_ch_dirs, float *raw, void *stream);
/* encoding tile image consumed by xrb_nerf_mlp_forward (per 128-row tile: point-encoding block(s) then direction block, [128x64] fp16, K-major 128B swizzle):
 * size, conversion from an fp32 `embedded` matrix, and BaseEmbedder's positional encoding written directly in that form */
size_t xrb_nerf_enc_image_bytes(int64_t n_rows, int input_ch);
int xrb_nerf_pack_embedded(const float *embedded, int64_t n_rows, int input_ch, int input_ch_dirs, void *enc_image, void *stream);
int xrb_nerf_posenc_tiles(const float *pts, const float *viewdirs, int64_t n_pts, int samples_per_ray, int multires, int multires_dirs, void *enc_image, void *stream);
/* same, from rays: sample positions o + d*z (GetPts, xrnerf/datasets/pipelines/create.py:588-597) are formed in registers; z_vals f32[n_rays, S] */
int xrb_nerf_posenc_tiles_rays(const float *rays_o, const float *rays_d, const float *z_vals, const float *viewdirs, int64_t n_rays, int samples_per_ray, int multires, int multires_dirs,
                               void *enc_image, void *stream);

/* Mip-NeRF cast_rays + MipNerfEmbedder.forward (networks/utils/mip.py:66-129, embedders/mipnerf_embedder.py:43-99, cone, diag):
 * z_vals f32[N,S+1], radii f32[N] -> embedded f32[N*S, 6*(max_deg_point-min_deg_point) + 3 + 6*(max_deg_view-min_deg_view)];
 * means_out/covs_out f32[N,S,3] optional (both or neither). */
int xrb_mip_embed(const float *z_vals, const float *rays_o, const float *rays_d, const float *radii, const float *viewdirs, int n_rays, int n_samples, int min_deg_point,
                  int max_deg_point, int min_deg_view, int max_deg_view, float *embedded, float *means_out, float *covs_out, void *stream);

/* The same cast_rays + IPE + view-direction encoding (networks/utils/mip.py:66-129, embedders/mipnerf_embedder.py:43-99) written straight into the fp16 tile image
 * xrb_nerf_mlp_forward consumes
 * (xrb_nerf_enc_image_bytes(N*S, 6*(max_deg_point-min_deg_point)) bytes): no fp32 `embedded` round trip. Values are the fp16 roundings of xrb_mip_embed's. */
int xrb_mip_ipe_tiles_rays(const float *z_vals, const float *rays_o, const float *rays_d, const float *radii, const float *viewdirs, int64_t n_rays, int n_samples, int min_deg_point,
                           int max_deg_point, int min_deg_view, int max_deg_view, void *enc_image, void *stream);

/* Mip-NeRF resample_along_rays / sorted_piecewise_constant_pdf (networks/utils/mip.py:7-63,:146-176): weights f32[N,S], z_vals f32[N,S+1]
 * -> z_out f32[N,S+1]; u f32[N,S+1] optional (NULL = the deterministic linspace of randomized=False). */
int xrb_mip_resample(const float *z_vals, const float *weights, const float *u, int n_rays, int n_samples, float resample_padding, float *z_out, void *stream);

/* Ray generation on the device (SURVEY §8 a1-a4): GetRays (+ Mip radii) + GetViewdirs (xrnerf/datasets/pipelines/create.py:205-245,:437-448)
 * for convention 0, get_rays_np_hash (xrnerf/datasets/load_data/get_rays.py:35-69) for convention 1. c2w_host: 12 floats on the HOST, row-major [3,4]
 * camera-to-world. pixel_idx i32[n] (row-major pixel numbers) or NULL for the first n pixels. viewdirs / radii may be NULL. */
int xrb_nerf_get_rays(const float *c2w_host, int H, int W, float fx, float fy, float cx, float cy, int convention, const int32_t *pixel_idx, int64_t n, float *rays_o, float *rays_d,
                      float *viewdirs, float *radii, void *stream);
/* The NGP training-ray source on the device (SURVEY §8f-1): replaces the 2.8 GB shuffled host table of HashNerfDataset (datasets/load_data/get_rays.py:72-98,
 * hashnerf_dataset.py:41-44) + HashBatchSample (datasets/pipelines/create.py:153-190) + RandomBGColor (datasets/pipelines/augment.py:290-313).
 * poses f32[I,4,3] (NGP xforms), images_rgba f32[I,H,W,4]; row_idx i64[n] = rows of the (virtual) [I*H*W, 11] table, i.e. a slice of the caller's permutation;
 * u_bg f32[n,3] = the background uniforms, or NULL to draw them on the device from (seed, n_prior_calls). Outputs as the reference's data dict:
 * rays_o, rays_d f32[n,3] (unit dirs), target_s f32[n,3] (blended with the background), alpha f32[n,1], img_ids f32[n,1], bg_color f32[n,3]. */
int xrb_ngp_batch_sample(const float *poses, const float *images_rgba, int n_images, int H, int W, float fx, float fy, float cx, float cy, const int64_t *row_idx, int64_t n,
                         const float *u_bg, uint64_t seed, int64_t n_prior_calls, float *rays_o, float *rays_d, float *target_s, float *alpha, float *img_ids, float *bg_color,
                         void *stream);
/* GetZvals (create.py:502-531, near/far constants) and, with u f32[n_rays, S] != NULL, PerturbZvals (augment.py:269-283) */
int xrb_nerf_zvals(int64_t n_rays, int n_samples, float near_, float far_, int lindisp, const float *u, float *z_vals, void *stream);

/* ------------------------------------------------------------------------------------------------
 * NerfMLP training on tensor cores (csrc/nerf_train.cu): what torch.autograd + cuBLAS do for the reference's NerfMLP (xrnerf/models/mlps/nerf_mlp.py:70-94,
 * trained by networks/nerf.py:71-92 / networks/mipnerf.py:45-74) as wgmma kernels over TILE IMAGES (per 128-row tile, C/64 blocks of [128 x 64] fp16 in the
 * K-major 128-byte-swizzle layout: the encoders' output format, xrb_nerf_enc_image_bytes). The host (xrnerf_b200/nerf_train.py) strings the layers together.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    /* A operand: up to two sources, concatenated block-wise (e.g. the skip layer: point-encoding blocks + 4 hidden blocks); <= 6 blocks in total */
    const void *a_base[2]; uint32_t a_tile_stride[2]; uint32_t a_blk_off[2]; int a_n_blk[2]; int n_a;
    const void *w;                       /* weight slabs (xrb_nerf_tg_pack_weights) */
    /* per weight slab: byte offset in w, bytes (<= 32768), MMA groups using it (A block a_blk0 + j), K-steps of 16 per group (1..4), accumulator column, first-writer flag */
    uint32_t slab_w_off[10]; uint32_t slab_bytes[10]; int slab_n_sub[10]; int slab_a_blk0[10]; int slab_d_col[10]; int slab_first[10]; int slab_n_k[10]; int n_slabs;
    int b_mn;                            /* 0: slabs read K-major (forward: Y = A . W^T); 1: MN-major (input gradient: dX = dZ . W, same slabs) */
    int mma_n;                           /* N of every MMA: the layer width (forward) or 64 (input gradient) */
    int out_cols;                        /* accumulator columns read back (16, 128 or 256) */
    int epi;                             /* 0: + bias, ReLU (relu != 0), fp16 -> y image; 1: + bias -> fp32 yf[row * yf_stride + yf_col + k] * yf_scale, k < yf_n;
                                            2: * [x > 0] -> fp16 y image (x: activation image, out_cols/64 blocks); 3: fp16 -> y image */
    int relu; const float *bias;
    const void *x_base; uint32_t x_tile_stride; uint32_t x_blk_off;
    void *y; uint32_t y_tile_stride; uint32_t y_blk_off;
    float *yf; int yf_stride; int yf_col; int yf_n; float yf_scale;
    int64_t n_rows;
} xrb_tg_layer;
int xrb_nerf_tg_layer(const xrb_tg_layer *layer, void *stream);
/* weight gradient of one layer and one input source: dW[N][K] (fp32, ACCUMULATED) [:, k_off : k_off + k_cols] += dZ^T . X over all rows; db[N] += column sums of dZ
 * when db != NULL. z: dZ image (N/64 blocks per tile, 1 block for N <= 16; zero in the rows >= n_rows), x: input image source (1..4 blocks, k_cols <= 64 x_n_blk).
 * Gradients are unscaled by *scale (the staging scale xrb_nerf_tg_pack_draw wrote; NULL: xrb_nerf_tg_grad_scale()). */
typedef struct {
    const void *z_base; uint32_t z_tile_stride; uint32_t z_blk_off;
    const void *x_base; uint32_t x_tile_stride; uint32_t x_blk_off; int x_n_blk;
    int N, K, k_off, k_cols;
    float *dW; float *db;
    int64_t n_rows;
    const float *scale;
} xrb_tg_dw;
int xrb_nerf_tg_dw(const xrb_tg_dw *layer, void *stream);
/* nn.Linear weight W[N][K_in] (fp32) -> n_kb slabs [n_pad x 64] fp16 (n_pad = N rounded up to 16): slab kb holds input columns [col0[kb], + valid[kb]) (zero beyond) */
int xrb_nerf_tg_pack_weights(const float *W, int N, int K_in, int n_pad, int n_kb, const int *col0_host, const int *valid_host, void *slabs, void *stream);
/* dL/draw f32[n_rows,4] -> the two one-block dZ images of the output heads (d rgb in columns 0..2, d alpha in column 0, every other entry 0), multiplied by
 * the power of two s chosen on the device with max |dL/draw| s in [2^12, 2^13) (xrb_nerf_tg_grad_scale() when dL/draw is all zero or not finite).
 * scale: device f32[2], scale[0] workspace, scale[1] <- s (the xrb_tg_dw.scale of the layers' weight gradients). */
int xrb_nerf_tg_pack_draw(const float *d_raw, int64_t n_rows, void *z_rgb_image, void *z_alpha_image, float *scale, void *stream);
float xrb_nerf_tg_grad_scale(void);

/* ---- NGP mesh export (csrc/mesh.cu; no reference counterpart): the field's density on a lattice, then a triangle mesh of one of its level sets.
 *
 * Lattice of nx x ny x nz points (each size 2..1024) spanning the box [box_min, box_max] (host float[3] each), volumes f32[nz][ny][nx] (x fastest).
 * Point (i, j, k) sits at (X(i), Y(j), Z(k)), per axis with n points from lo to hi:
 *   X(i) = min(lo + i * ((hi - lo) / (n - 1)), hi)      (fp32, each operation rounded once, in this order; the min keeps the last point in the box)
 * A lattice with a size of 0 is empty: every call on it is a no-op that touches no pointer.
 *
 * xrb_ngp_density_lattice: out[k][j][i] <- the raw (pre-activation) density the field returns at lattice point (i, j, k), the very value
 * xrb_ngp_density_forward gives for that position with the same impl. The box must lie in the field's warped domain, 0 <= box_min < box_max <= 1
 * (outside it the dense levels would be addressed past their end); it is checked, with the sizes, before any CUDA call. The positions are
 * staged through `workspace` (xrb_ngp_density_lattice_workspace() bytes, 16-byte aligned, independent of the lattice size) in chunks of
 * consecutive points, each evaluated by the density-only field kernel into its slice of `out`. */
size_t xrb_ngp_density_lattice_workspace(void);
int xrb_ngp_density_lattice(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *density_fp16, const void *weight_image, int nx, int ny, int nz,
                            const float *box_min_host, const float *box_max_host, float *out, int impl, void *workspace, void *stream);
/* Marching cubes of `volume` at `threshold` (not NaN), in two calls on one workspace (xrb_mc_workspace(nx, ny, nz) bytes, 8-byte aligned: 4 bytes per
 * lattice point plus 8 per 256 points plus 16; 0 for bad sizes):
 *   xrb_mc_count  counts <- (V, F), device int32[2] (both -1 when either exceeds INT32_MAX; xrb_mc_emit then writes nothing);
 *   xrb_mc_emit   verts f32[V,3] (box coordinates) and faces int32[F,3] (vertex indices), from the workspace xrb_mc_count filled with the same
 *                 volume, sizes and threshold. box: finite, box_min < box_max.
 * A lattice value v is inside iff v > threshold; a lattice edge is crossing iff exactly one endpoint is inside. Each crossing edge has ONE vertex,
 * shared by every triangle that uses it: the edge from point p along +x, +y or +z belongs to p, and its vertex is
 *   p_out + t * (p_in - p_out),   t = (threshold - v_out) / (v_in - v_out) in [0, 1]
 * on the edge's axis (the other two coordinates are p's), in fp32 with each operation rounded once.
 * Order, independent of the launch: vertices by lattice point (z, then y, then x), then axis x, y, z; triangles by cell (z, y, x; a cell is named
 * by its lowest corner), then in the order of the triangulation table (csrc/mc_table.cuh, generated by scripts/gen_mc_table.py). The table
 * draws the same segments on a face from both cells that share it (a face with two diagonal inside corners cuts each off on its own), so a
 * volume whose boundary points are all outside gives a closed mesh: every edge in exactly two triangles, once in each direction. Triangles wind
 * counter-clockwise seen from outside: their right-hand normals point out of the inside region. No crossing edge gives V = F = 0. */
size_t xrb_mc_workspace(int nx, int ny, int nz);
int xrb_mc_count(const float *volume, int nx, int ny, int nz, float threshold, void *workspace, int32_t *counts, void *stream);
int xrb_mc_emit(const float *volume, int nx, int ny, int nz, float threshold, const float *box_min_host, const float *box_max_host, const void *workspace,
                float *verts, int32_t *faces, void *stream);

/* ---- NeRF mesh export (csrc/nerf_mlp_tc.cu, csrc/nerf.cu; no reference counterpart): the NerfMLP's density on the lattice above, and the gradient of
 * its raw density with respect to the position (vertex normals).
 *
 * xrb_nerf_density_lattice: out[k][j][i] <- raw[:, 3] of xrb_nerf_mlp_forward (same weight_image and bias, from pack_nerf_mlp) on the
 * xrb_nerf_posenc_tiles encoding of lattice point (i, j, k), bit for bit; the view direction does not enter alpha. The lattice positions are the ones
 * above; the box is any finite box with box_min < box_max (the NeRF world frame). The same wgmma kernel with its layer schedule cut after
 * pts_linears.7: it writes each point's encoding into shared memory from the lattice index and stores alpha from the layer-7 epilogue, so it needs
 * no position tensor, encoding image or workspace. Only input_ch = 63, multires = 10 (the reference NeRF configs) is implemented: anything else returns
 * XRB_E_UNSUPPORTED. Sizes, input_ch and box are checked before any CUDA call; weight_image and bias must be 16-byte aligned.
 *
 * xrb_nerf_posenc_grad: grad f32[n,3] <- the gradient with respect to the position through BaseEmbedder's encoding (multires 0..10) of pts f32[n,3].
 * d_enc_image is a tile image of n_terms (1..4) one-block terms per 128-row tile; the gradient with respect to the 3 + 6 multires encoding columns is
 * e = (sum of the terms, fp32) / *scale (device float: the staging scale xrb_nerf_tg_pack_draw wrote, scale[1]), and
 *   grad[i][a] = e[a] + sum_b 2^b (cos(2^b x_a) e[3 + 6b + a] - sin(2^b x_a) e[6 + 6b + a])
 * with the column order of xrb_nerf_posenc. n == 0 is a no-op that touches no pointer. */
int xrb_nerf_density_lattice(const void *weight_image, const float *bias, int input_ch, int multires, int nx, int ny, int nz, const float *box_min_host,
                             const float *box_max_host, float *out, void *stream);
int xrb_nerf_posenc_grad(const float *pts, int64_t n_pts, int multires, const void *d_enc_image, int n_terms, const float *scale, float *grad, void *stream);

/* ---- Mip-NeRF mesh export (csrc/nerf.cu, csrc/nerf_mlp_tc.cu; no reference counterpart). Mip-NeRF's field is defined on Gaussians; a POINT QUERY AT
 * FOOTPRINT sigma >= 0 is MipNerfEmbedder.integrated_pos_enc with mean p and covariance sigma^2 I (an isotropic Gaussian of standard deviation sigma in
 * the rays' world frame): for band k = 0 .. max_deg_point - min_deg_point - 1, deg = min_deg_point + k, axis a, with y = p_a 2^deg and
 * a_k = exp(-0.5 sigma^2 4^deg) (formed once per call, rounded once to fp32), column 3k + a = a_k sin(y) and column 3 n_deg + 3k + a = a_k sin(y + pi/2)
 * (fp32 y + pi/2, as in the reference). A band whose fp32 0.5 ((sigma^2 2^deg) 2^deg) exceeds 20 is zero, the rule of xrb_mip_ipe_tiles_rays.
 * Point degrees: 1 <= max - min, 6 (max - min) <= 128, both in [-100, 100]; sigma finite and >= 0. All three entries check sizes, degrees and sigma
 * before any CUDA call (XRB_E_BADARG), and n == 0 / an empty lattice is a no-op that touches no pointer.
 *
 * xrb_mip_ipe_tiles_points: the point query's encoding of pts f32[n_pts,3] at footprint sigma into point blocks 0 and 1 of the tile image, and
 * MipNerfEmbedder.pos_enc of viewdirs f32[n_pts / samples_per_ray, 3] (identity, then the bands; view degrees 3 + 6 (max - min) <= 64) into block 2, the
 * values xrb_mip_ipe_tiles_rays writes for a direction: the encoding image xrb_nerf_mlp_forward reads (input_ch 96 when 16 point bands). enc_image
 * 16-byte aligned, xrb_nerf_enc_image_bytes(n_pts, 96) bytes.
 *
 * xrb_mip_density_lattice: out[k][j][i] <- raw[:, 3] of xrb_nerf_mlp_forward (input_ch 96, input_ch_dirs 27; weight_image and bias from
 * pack_nerf_mlp) on the xrb_mip_ipe_tiles_points encoding at footprint sigma of lattice point (i, j, k), bit for bit; lattice positions and box as for
 * xrb_nerf_density_lattice. The Mip-NeRF instantiation of the same lattice kernel: it forms each point's IPE in shared memory, so it needs no position
 * tensor, encoding image or workspace. The box is checked before any CUDA call; weight_image and bias must be 16-byte aligned, out 4-byte aligned.
 *
 * xrb_mip_ipe_grad: grad f32[n,3] <- the gradient with respect to the position through the point query's encoding at footprint sigma of pts f32[n,3].
 * d_enc_image is a tile image of n_terms (1..4) two-block terms per 128-row tile (blocks 2t, 2t + 1 = term t); the gradient with respect to the 6 n_deg
 * encoding columns is e = (sum of the terms, fp32) / *scale (device float: the staging scale xrb_nerf_tg_pack_draw wrote, scale[1]), and
 *   grad[i][a] = sum_{live k} a_k 2^deg (cos(y) e[3k + a] + cos(y + pi/2) e[3 n_deg + 3k + a]). d_enc_image must be 16-byte aligned. */
int xrb_mip_ipe_tiles_points(const float *pts, const float *viewdirs, int64_t n_pts, int samples_per_ray, float sigma, int min_deg_point, int max_deg_point, int min_deg_view,
                             int max_deg_view, void *enc_image, void *stream);
int xrb_mip_density_lattice(const void *weight_image, const float *bias, int min_deg_point, int max_deg_point, float sigma, int nx, int ny, int nz,
                            const float *box_min_host, const float *box_max_host, float *out, void *stream);
int xrb_mip_ipe_grad(const float *pts, int64_t n_pts, float sigma, int min_deg_point, int max_deg_point, const void *d_enc_image, int n_terms, const float *scale, float *grad,
                     void *stream);

/* ------------------------------------------------------------------------------------------------
 * Image metrics (csrc/metrics.cu)
 * ---------------------------------------------------------------------------------------------- */

/* SSIM of n image pairs: what the reference's ValidateHook / TestHook ask scikit-image for (hooks/utils.py:20-28, calculate_ssim:
 * structural_similarity(im1, im2, multichannel=True, full=True), 7 x 7 uniform window, K1 = 0.01, K2 = 0.03, sample covariance).
 * x, y f32[n, H, W, C] (contiguous, HWC, 4-byte aligned), H >= 7, W >= 7, 1 <= C <= 4. Each channel is its own 2-D image. Per entry, in double
 * (each fp32 input converted exactly), with ux, uy, uxx, uyy, uxy the 7 x 7 window means (window sum x 1/49) of x, y, x^2, y^2, x y, borders
 * reflected as scipy.ndimage's mode 'reflect' (d c b a | a b c d | d c b a):
 *   vx = cn (uxx - ux^2), vy = cn (uyy - uy^2), vxy = cn (uxy - ux uy), cn = 49/48;  C1 = (0.01 R)^2, C2 = (0.03 R)^2, R = data_range (finite, > 0)
 *   S = ((2 ux uy + C1)(2 vxy + C2)) / ((ux^2 + uy^2 + C1)(vx + vy + C2))
 * every operation rounded once, in this order (no FMA contraction): S(x, x) = 1 and S(x, y) = S(y, x) hold bit for bit.
 * Outputs: mean_full f64[n] <- the mean of S over all H W C entries (calculate_ssim's value), mean_crop f64[n] <- the mean over the entries of the
 * crop [3, H-3) x [3, W-3) (scikit-image's mssim); s_map f32[n, H, W, C] <- S rounded once to fp32, or NULL to skip it.
 * Window sums: horizontal 7-sums left to right, then vertical 7-sums top to bottom; the means sum per-tile partials in a fixed order. An image's
 * results are bit-identical alone, in any batch and from run to run. workspace: xrb_ssim_workspace(n, H, W) bytes (0 for bad sizes), 8-byte
 * aligned, passed with its size. Sizes, channels, data_range, pointers and the workspace size are checked before any CUDA call (XRB_E_BADARG);
 * n == 0 is a no-op that touches no pointer. No allocation inside: capturable in a CUDA graph. */
size_t xrb_ssim_workspace(int n, int height, int width);
int xrb_ssim(const float *x, const float *y, int n, int height, int width, int channels, double data_range, double *mean_full, double *mean_crop, float *s_map,
             void *workspace, size_t workspace_bytes, void *stream);

/* Measurement utility (bench.py's second roofline; no reference counterpart): random reads of 4-, 8- or 32-byte records from a table (L2-resident when
 * it is the size of the fp16 hash table) by SMs x 8 CTAs x 256 threads, `rounds` rounds of 8 independent loads per thread. *loads_issued (host) receives the
 * number of loads of the launch; every 4/8-byte load costs one 32-byte sector, which is what bounds the hash gather. */
int xrb_micro_gather(const void *table, int64_t n_records, int record_bytes, int rounds, int64_t *loads_issued, void *sink, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* XRNERF_B200_H */
