/* plenoctree_b200.h — C ABI of the H100-native (sm_90a) NeRF-SH hot path.
 *
 * The reference (sxyu/plenoctree) has no FFI layer of its own: its boundary for this path is a
 * set of Python call signatures (SURVEY.md §8b).  Each entry point below is what a binding for
 * one of those call sites would call; the reference interface it replaces is cited as
 * file:line relative to the reference tree.  INTEGRATION.md shows the ctypes stubs.
 *
 * Conventions
 *   - every pointer named *_dev is a CUDA device pointer on the current device, *_host is host
 *     memory; `stream` is a cudaStream_t passed as void* (NULL = default stream);
 *   - all functions return 0 on success, non-zero on error; pob_last_error() returns a
 *     thread-local message for the last failure (never NULL);
 *   - nothing here falls back to the CPU: without a CUDA device every compute call fails.
 *   - precision: POB_PREC_FP16 = fp16 operands / fp32 accumulate on wgmma (the numerics class
 *     of the reference's TF32-default XLA GPU path); POB_PREC_FP16X3 = error-compensated 3-pass
 *     split (fp32-class accuracy, 1/3 of the tensor throughput).
 */
#ifndef PLENOCTREE_B200_H
#define PLENOCTREE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define POB_PREC_FP16 1
#define POB_PREC_FP16X3 3

/* flag sigma_activation (nerf_sh/nerf/utils.py:153, models.py:280-281): the density activation of the ray samples
 * and of pob_eval_points_act.  Raw sigma (eval_points_raw, the extraction grids and cell means) never takes one, and
 * the sparsity term of the training step keeps relu on raw sigma whatever the flag (nerf_sh/train.py:77-83). */
#define POB_SIGMA_RELU 0
#define POB_SIGMA_SOFTPLUS 1 /* log(1 + exp(x)), evaluated in fp32 as max(x, 0) + log1p(exp(-|x|)) */

/* flags min_deg_point, max_deg_point, legacy_posenc_order (nerf_sh/nerf/utils.py:119-124,155-159): the point encoder
 * posenc(x, min_deg, max_deg, legacy_order) (nerf_sh/nerf/model_utils.py:145-173) of a model.  Its width
 * W = 3 + 6 (max_deg - min_deg) sets the parameter shapes Dense_0 [W, 256] and Dense_5 [256 + W, 256], so the flat
 * layout, the packed blob's contents and every evaluation depend on it.  Accepted: 0 <= min_deg <= max_deg <= 10
 * (W <= 63), legacy_order 0 or 1.  Feature order, c = 0..2, j = min_deg..max_deg-1:
 *   legacy_order 0: [x, sin(2^j x_c) at 3 + 3(j - min_deg) + c, sin(2^j x_c + pi/2) at 3 + 3L + 3(j - min_deg) + c]
 *   legacy_order 1: [x, sin(2^j x_c) at 3 + 6(j - min_deg) + c, sin(2^j x_c + pi/2) at 3 + 6(j - min_deg) + 3 + c]
 * with L = max_deg - min_deg.
 * The descriptor describes the network beyond sh_deg: it also carries the trunk activation net_activation (POB_NET_*,
 * flag net_activation, nerf_sh/nerf/model_utils.py:69), applied after each of Dense_0..Dense_7.  It changes neither
 * the parameter layout nor the packed blob.  Every entry point taking a `const pob_posenc*` reads NULL as the
 * reference default {0, 10, 0, POB_NET_RELU}, W = 63; the entry points without one use that default, and a
 * zero-filled descriptor is that default too.  Other net_activation values are refused. */
#define POB_NET_RELU 0
#define POB_NET_ELU 1      /* z if z > 0 else expm1(z) */
#define POB_NET_SOFTPLUS 2 /* max(z, 0) + log1p(exp(-|z|)) */
#define POB_NET_TANH 3     /* tanh(z) */
typedef struct pob_posenc {
  int min_deg;
  int max_deg;
  int legacy_order;
  int net_activation;
} pob_posenc;

/* ---------------------------------------------------------------------------------------------
 * Library / device
 * ------------------------------------------------------------------------------------------- */
int pob_abi_version(void);
const char* pob_last_error(void);
/* number of SMs the kernels split their work for (persistent-grid size): the current CUDA device's, or the
 * environment variable POB_SM_COUNT when it is set (read on every call; for tests and diagnosis: it selects the work
 * split of a smaller H100, such as the 114-SM PCIe card or a MIG slice, and changes no code path).  POB_SM_COUNT must
 * be an integer from 16 to the device's SM count; any other value makes every entry point that reads the count (the
 * MLP evaluations, pob_render_rays, the pob_loss_and_grad family, pob_draw_uniforms and the octree entry points) fail
 * with a message naming it, before anything is launched, and this function return -3.  <0 on error */
int pob_sm_count(void);

/* Instrumentation used by bench.py: number of kernels this library has launched so far, and
 * optional CUDA-event timing per kernel class.  pob_timing_read fills ms_out[5] / launches_out[5] for
 * {mlp_fwd, mlp_bwd, mlp_wgrad, per-ray render stages, optimiser (reduce, Adam, pack)} and returns 5;
 * it synchronises with the recorded events. */
long long pob_launch_count(void);
void pob_timing_enable(int on);
int pob_timing_read(double* ms_out, long long* launches_out);
/* all kernel classes: the five of pob_timing_read, then the median cut (pob_quantize_median_cut).  Fills the first
 * min(n, 6) entries of ms_out / launches_out (either may be NULL) and returns 6. */
int pob_timing_read_phases(int n, double* ms_out, long long* launches_out);

/* ---------------------------------------------------------------------------------------------
 * Parameters of one MLP (MLP_0 coarse / MLP_1 fine; nerf_sh/nerf/models.py:83-104).
 * Flat fp32 layout = Dense_0..Dense_9 in order, each kernel [in,out] row-major then bias [out]
 * (nerf_sh/nerf/model_utils.py:60-93; Dense index mapping octree/nerf/models.py:79-102).
 * ------------------------------------------------------------------------------------------- */
/* number of fp32 parameters of one MLP for SH degree sh_deg (-1 = plain RGB head, 3 channels) */
int64_t pob_param_count(int sh_deg);
/* byte size of the packed tensor-core operand blob of one MLP */
int64_t pob_packed_bytes(int sh_deg);
/* flat fp32 parameters -> packed blob (fp16 hi/lo forward images, transposed images, biases) */
int pob_pack_weights(const float* flat_dev, int sh_deg, void* packed_dev, void* stream);
/* the same for a model with point encoder `posenc` (NULL = default): pob_param_count_pe parameters; the blob keeps
 * pob_packed_bytes(sh_deg) bytes and its format */
int64_t pob_param_count_pe(int sh_deg, const pob_posenc* posenc);
int pob_pack_weights_pe(const float* flat_dev, int sh_deg, const pob_posenc* posenc, void* packed_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * NerfModel.eval_points_raw(points, viewdirs=None, coarse=False) -> (raw_rgb[M,3K], raw_sigma[M,1])
 *   JAX:   nerf_sh/nerf/models.py:143-181      torch twin: octree/nerf/models.py:211-252
 * raw_rgb_dev may be NULL (sigma only: octree/extraction.py:271,316 discard rgb).
 * ------------------------------------------------------------------------------------------- */
int pob_eval_points_raw(const void* packed_dev, int sh_deg, const float* points_dev, int64_t m,
                        float* raw_rgb_dev, float* raw_sigma_dev, int precision, void* stream);

/* NerfModel.eval_points(points, viewdirs) -> (rgb[M,3], sigma[M,1])  (models.py:183-214):
 * eval_sh at the per-point view direction, sigmoid / relu.  out_rgbs_dev: [M,4] = (r,g,b,sigma).
 * pob_eval_points is pob_eval_points_act with POB_SIGMA_RELU. */
int pob_eval_points(const void* packed_dev, int sh_deg, const float* points_dev,
                    const float* viewdirs_dev, int64_t m, float* out_rgbs_dev, int precision,
                    void* stream);
/* the same with the density activation sigma_activation (POB_SIGMA_*) in place of relu */
int pob_eval_points_act(const void* packed_dev, int sh_deg, const float* points_dev,
                        const float* viewdirs_dev, int64_t m, float* out_rgbs_dev, int sigma_activation,
                        int precision, void* stream);

/* Dense-grid sweep of octree.extraction (auto_scale / step1: octree/extraction.py:244-320).
 * Evaluates raw sigma (and optionally raw SH coefficients) at the voxel centres
 *   ((i + 0.5)/reso - offset[a]) / scale[a]
 * of the slab ix in [x0, x0+nx), iy in [0,ny), iz in [0,nz), flattened x-major like
 * torch.meshgrid(xx,yy,zz).reshape(3,-1).T.  No host grid, no H2D copies. */
int pob_eval_grid(const void* packed_dev, int sh_deg, int reso, int x0, int nx, int ny, int nz,
                  const float offset[3], const float scale[3], float* raw_rgb_dev,
                  float* raw_sigma_dev, int precision, void* stream);

/* Anti-aliasing pass of octree.extraction step2 (octree/extraction.py:355-394, SH data formats): the caller
 * provides samples_per_cell points per leaf (tree[inds].sample(S), [n_cells*S, 3], cell-major);
 * out_dev [n_cells, 3K+1] = mean over the S samples of cat([raw_rgb, raw_sigma], -1)  (:391-393). */
int pob_eval_cells_mean(const void* packed_dev, int sh_deg, const float* points_dev, int64_t n_cells,
                        int samples_per_cell, float* out_dev, int precision, void* stream);

/* Host-buffer convenience form of pob_eval_points_raw (H2D, kernel, D2H inside the call);
 * the e2e arm of bench.py times this. */
int pob_eval_points_raw_host(const void* packed_dev, int sh_deg, const float* points_host,
                             int64_t m, float* raw_rgb_host, float* raw_sigma_host,
                             int precision);

/* The point, grid and cell evaluators of a model with point encoder `posenc` (NULL = default; the blob packed with
 * the same descriptor).  Each is the entry point above without `_pe`, which is its NULL case; pob_eval_points_pe
 * takes the density activation like pob_eval_points_act. */
int pob_eval_points_raw_pe(const void* packed_dev, int sh_deg, const pob_posenc* posenc, const float* points_dev,
                           int64_t m, float* raw_rgb_dev, float* raw_sigma_dev, int precision, void* stream);
int pob_eval_points_pe(const void* packed_dev, int sh_deg, const pob_posenc* posenc, const float* points_dev,
                       const float* viewdirs_dev, int64_t m, float* out_rgbs_dev, int sigma_activation, int precision,
                       void* stream);
int pob_eval_grid_pe(const void* packed_dev, int sh_deg, const pob_posenc* posenc, int reso, int x0, int nx, int ny,
                     int nz, const float offset[3], const float scale[3], float* raw_rgb_dev, float* raw_sigma_dev,
                     int precision, void* stream);
int pob_eval_cells_mean_pe(const void* packed_dev, int sh_deg, const pob_posenc* posenc, const float* points_dev,
                           int64_t n_cells, int samples_per_cell, float* out_dev, int precision, void* stream);
int pob_eval_points_raw_host_pe(const void* packed_dev, int sh_deg, const pob_posenc* posenc,
                                const float* points_host, int64_t m, float* raw_rgb_host, float* raw_sigma_host,
                                int precision);

/* ---------------------------------------------------------------------------------------------
 * Per-ray stages (exposed individually for parity tests; pob_render_rays chains them).  They take up to
 * 1024 samples per ray: n_samples <= 1024, n_coarse >= 3 and n_coarse + n_fine <= 1024, the bound
 * pob_render_config's num_coarse_samples / num_fine_samples are checked against.
 * ------------------------------------------------------------------------------------------- */
/* model_utils.sample_along_rays (nerf_sh/nerf/model_utils.py:104-142).  z_base[n_samples] is the
 * un-jittered table near*(1-t)+far*t (or the lindisp form) built by the host with the reference
 * expression; t_rand [n_rays,n_samples] in [0,1) replaces random.uniform (NULL = randomized False). */
int pob_sample_coarse(const float* z_base_dev, const float* t_rand_dev, int n_rays, int n_samples,
                      float* z_out_dev, void* stream);

/* The random draws of one randomized training step in ONE launch (replaces jax.random.uniform at
 * nerf_sh/nerf/model_utils.py:137 (t_rand [n_t] ~ U[0,1)), :262 (u [n_u] ~ U[0,1)) and nerf_sh/train.py:79
 * (sp_points [n_sp] ~ U[-radius, radius))): Philox4x32-10 keyed by `seed`, counter = (index, stream, step).  The
 * threefry streams of the reference cannot be reproduced without JAX; parity tests inject their own draws.
 * step_dev (device float, or NULL) overrides `step`, so that a replayed CUDA graph draws fresh numbers. */
int pob_draw_uniforms(uint64_t seed, float step, const float* step_dev, float* t_rand_dev, int64_t n_t,
                      float* u_dev, int64_t n_u, float* sp_points_dev, int64_t n_sp, float sp_radius, void* stream);
/* model_utils.volumetric_rendering (model_utils.py:176-222).  rgbs [n_rays,n_samples,4] = (rgb, sigma)
 * after activations; outputs comp_rgb [n_rays,3], disp, acc [n_rays], weights [n_rays,n_samples]
 * (disp / acc / weights may be NULL). */
int pob_composite(const float* rgbs_dev, const float* z_dev, const float* dirs_dev, int n_rays, int n_samples,
                  int white_bkgd, float* out_rgb_dev, float* out_disp_dev, float* out_acc_dev,
                  float* out_weights_dev, void* stream);
/* reverse-mode of pob_composite composed with the MSE of loss_fn (nerf_sh/train.py:86-96) and with
 * sigmoid'/relu': g_out [n_rays,n_samples,4] = d/d(pre-activation rgb after eval_sh, raw sigma) of
 * gscale/2 * sum (comp_rgb - pixels)^2;  sq_err_sum_dev (may be NULL) += sum (comp_rgb - pixels)^2. */
int pob_composite_bwd(const float* rgbs_dev, const float* z_dev, const float* dirs_dev, const float* comp_rgb_dev,
                      const float* pixels_dev, int n_rays, int n_samples, int white_bkgd, float gscale,
                      float* g_out_dev, float* sq_err_sum_dev, void* stream);
/* model_utils.sample_pdf (model_utils.py:225-314): inverse-CDF resampling from weights[...,1:-1] over the
 * mid-point bins, then the sorted union with the coarse depths.  u: [n_fine] table (u_per_ray = 0,
 * randomized False: linspace(0, 1-eps)) or [n_rays,n_fine] uniforms.  z_out [n_rays, n_coarse+n_fine]. */
int pob_sample_pdf(const float* z_coarse_dev, const float* weights_dev, const float* u_dev, int u_per_ray,
                   int n_rays, int n_coarse, int n_fine, float* z_out_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * NerfModel.__call__(rng_0, rng_1, rays, randomized) -> [(rgb,disp,acc)_coarse, (rgb,disp,acc)_fine]
 *   nerf_sh/nerf/models.py:216-348   (callers: train.py:70, utils.render_image utils.py:331-381)
 * ------------------------------------------------------------------------------------------- */
typedef struct pob_render_config {
  int sh_deg;               /* flag sh_deg            (nerf_sh/nerf/utils.py:135) */
  int num_coarse_samples;   /* flag num_coarse_samples (utils.py:126)             */
  int num_fine_samples;     /* flag num_fine_samples   (utils.py:130); 0 = single level */
  int white_bkgd;           /* flag white_bkgd */
  int max_rays;             /* capacity of the workspace in rays per call */
  int sparsity_npoints;     /* flag sparsity_npoints (training workspace only) */
  /* model_utils.add_gaussian_noise (nerf_sh/nerf/model_utils.py:317-332; flag noise_std, utils.py:137-142):
   * optional per-sample normal draws ALREADY multiplied by noise_std, added to raw sigma before relu at the
   * coarse [n_rays, Nc] and fine [n_rays, Nc+Nf] level; NULL = off (randomized False or noise_std None). */
  const float* sigma_noise_coarse_dev;
  const float* sigma_noise_fine_dev;
  /* flag sigma_activation: POB_SIGMA_* applied to the (noised) raw sigma of the ray samples; 0 = relu.  The
   * sparsity points of the training step keep relu (nerf_sh/train.py:82). */
  int sigma_activation;
  /* flags min_deg_point / max_deg_point / legacy_posenc_order of both MLPs (pob_posenc); NULL = default.  The
   * training step's grad_flat and params_dev follow its flat layout (pob_param_count_pe). */
  const pob_posenc* posenc;
} pob_render_config;

/* bytes of device scratch the render (training=0) / training (training=1) calls need */
int64_t pob_workspace_bytes(const pob_render_config* cfg, int training);

/* out_coarse / out_fine: [n_rays,5] = (r,g,b,disp,acc).  t_rand NULL = randomized False.
 * z_fine_dev (normally NULL): [n_rays, Nc+Nf] sorted depths that replace the sample_pdf stage — lets a
 * caller (and the parity tests) pin the fine-level sample positions. */
int pob_render_rays(const pob_render_config* cfg, const void* packed_coarse_dev, const void* packed_fine_dev,
                    const float* origins_dev, const float* directions_dev, const float* viewdirs_dev,
                    int n_rays, const float* z_base_dev, const float* t_rand_dev, const float* u_dev,
                    int u_per_ray, const float* z_fine_dev, float* out_coarse_dev, float* out_fine_dev,
                    void* workspace_dev, int precision, void* stream);

/* ---------------------------------------------------------------------------------------------
 * train_step (nerf_sh/train.py:51-121), split at the gradient all-reduce:
 *   pob_loss_and_grad = jax.value_and_grad(loss_fn)   (train.py:66-116)
 *   [caller: all-reduce-mean of grad_flat over ranks   (train.py:117) ]
 *   pob_adam_update   = optimizer.apply_gradient       (train.py:119) + operand re-pack
 * ------------------------------------------------------------------------------------------- */
typedef struct pob_train_hparams {
  float sparsity_weight;    /* flag sparsity_weight (utils.py:191) ; 0 disables the term */
  float sparsity_length;    /* flag sparsity_length */
  float loss_scale;         /* power-of-two scale applied to the fp16 gradient chain, divided out of grad_flat */
} pob_train_hparams;

/* grad_flat [num_mlps * pob_param_count] (MLP_0 then MLP_1, reference flat order), per-rank gradient of
 *   mean((rgb_f-px)^2) + mean((rgb_c-px)^2) + sparsity_weight*(1-mean(exp(-len*relu(sigma(p)))))
 * stats [8] (device): [0] sum (rgb_fine-px)^2, [1] sum (rgb_coarse-px)^2, [2] sum exp(-len*relu(sigma)).
 * The backward of MLP_0 (coarse level) is finished first; mlp0_done_event (a cudaEvent_t, or NULL) is recorded on
 * `stream` once grad_flat[0 : pob_param_count) is final, so that the caller can all-reduce that bucket on another
 * stream while the MLP_1 backward (three quarters of the work) is still running (the two branches are independent:
 * stop_gradient, nerf_sh/nerf/model_utils.py:286). */
int pob_loss_and_grad(const pob_render_config* cfg, const pob_train_hparams* hp, const void* packed_coarse_dev,
                      const void* packed_fine_dev, const float* origins_dev, const float* directions_dev,
                      const float* viewdirs_dev, const float* pixels_dev, int n_rays, const float* z_base_dev,
                      const float* t_rand_dev, const float* u_dev, int u_per_ray, const float* z_fine_dev,
                      const float* sp_points_dev, float* grad_flat_dev, float* stats_dev, void* workspace_dev,
                      void* mlp0_done_event, void* stream);

/* bytes of device scratch pob_loss_and_grad_prec needs at `precision`; for POB_PREC_FP16 the same as
 * pob_workspace_bytes(cfg, 1).  -1 on a bad config or precision. */
int64_t pob_train_workspace_bytes(const pob_render_config* cfg, int precision);

/* pob_loss_and_grad at `precision`.  POB_PREC_FP16 is pob_loss_and_grad (params_dev may be NULL).
 * POB_PREC_FP16X3 runs the forward, the data gradient and the weight gradient with error-compensated operands
 * (x = hi + lo, both fp16; every product lo*hi + hi*lo + hi*hi, fp32 accumulation): the render forward of
 * POB_PREC_FP16X3, saving its activations, and a gradient within a few 2^-24 of fp64 per stage.  It needs params_dev
 * (the flat fp32 parameters of all MLPs, [num_mlps * pob_param_count], consistent with the packed blobs as
 * pob_adam_update leaves them) and a workspace of pob_train_workspace_bytes(cfg, POB_PREC_FP16X3) bytes.  The call
 * refuses a workspace whose device allocation (cuMemGetAddressRange) ends before that size; it cannot see the bounds
 * of a block that a caching allocator (torch.empty) cuts out of a larger allocation, so such callers must size the
 * block themselves. */
int pob_loss_and_grad_prec(const pob_render_config* cfg, const pob_train_hparams* hp, const void* packed_coarse_dev,
                           const void* packed_fine_dev, const float* origins_dev, const float* directions_dev,
                           const float* viewdirs_dev, const float* pixels_dev, int n_rays, const float* z_base_dev,
                           const float* t_rand_dev, const float* u_dev, int u_per_ray, const float* z_fine_dev,
                           const float* sp_points_dev, float* grad_flat_dev, float* stats_dev, void* workspace_dev,
                           void* mlp0_done_event, const float* params_dev, int precision, void* stream);

/* flags of pob_loss_and_grad_flags.
 * POB_TRAIN_DISCARD_SAVED_GRADS: the caller will not read the data-gradient tiles (dZ, dO) the call leaves in the
 *   workspace, so the weight gradient drops each of them from L2 once it has loaded it, and they are never written
 *   back to HBM.  After such a call those workspace regions hold undefined bytes; every other region, grad_flat and
 *   stats are as without the flag.  POB_PREC_FP16X3 accepts the flag and ignores it: its weight-gradient passes run
 *   after the data gradient and read every dZ tile twice. */
#define POB_TRAIN_DISCARD_SAVED_GRADS 1
/* pob_loss_and_grad_prec with `flags` (POB_TRAIN_*; 0 is pob_loss_and_grad_prec).  Unknown bits are refused. */
int pob_loss_and_grad_flags(const pob_render_config* cfg, const pob_train_hparams* hp, const void* packed_coarse_dev,
                            const void* packed_fine_dev, const float* origins_dev, const float* directions_dev,
                            const float* viewdirs_dev, const float* pixels_dev, int n_rays, const float* z_base_dev,
                            const float* t_rand_dev, const float* u_dev, int u_per_ray, const float* z_fine_dev,
                            const float* sp_points_dev, float* grad_flat_dev, float* stats_dev, void* workspace_dev,
                            void* mlp0_done_event, const float* params_dev, int precision, int flags, void* stream);

/* flax.optim.Adam (beta1 .9, beta2 .999, eps 1e-8; nerf_sh/nerf/models.py:44) on the flat buffers of
 * num_mlps MLPs, g = grad*grad_mult + weight_decay_coef*param, then re-packs the operand blobs.
 * `step` = number of updates already applied (flax optimizer.state.step).  lr_step_dev (device float[2] = {lr,
 * step}, or NULL) overrides the two host values, so that a captured CUDA graph of the step can be replayed with a
 * new learning rate and step count. */
int pob_adam_update(int sh_deg, int num_mlps, float* params_dev, const float* grads_dev, float* m_dev,
                    float* v_dev, float lr, float step, const float* lr_step_dev, float grad_mult,
                    float weight_decay_coef, void* packed_coarse_dev, void* packed_fine_dev, void* stream);
/* pob_adam_update of a model with point encoder `posenc` (NULL = default): num_mlps * pob_param_count_pe elements,
 * re-packed with the same descriptor */
int pob_adam_update_pe(int sh_deg, const pob_posenc* posenc, int num_mlps, float* params_dev, const float* grads_dev,
                       float* m_dev, float* v_dev, float lr, float step, const float* lr_step_dev, float grad_mult,
                       float weight_decay_coef, void* packed_coarse_dev, void* packed_fine_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * PlenOctree side (SURVEY.md §8 rows a13-middle and a15).  These entry points stand where the
 * reference calls the third-party `svox` extension (absent from the reference tree; the oracle
 * restates its published algorithm, parity unpinned — see oracle/octree_oracle.py):
 *   svox.N3Tree / N3TreeView          octree/extraction.py:330-394,489-509
 *   svox.VolumeRenderer.render_persp  octree/optimization.py:174-229, octree/nerf/utils.py:448-498
 *   svox _C.grid_weight_render        octree/extraction.py:181-214
 * Tree layout (svox N3Tree, keys of tree.npz: octree/compression.py:75-95):
 *   data  [n_nodes, N, N, N, data_dim] fp32, sigma is the LAST channel (octree/extraction.py:391),
 *         SH coefficients channel-major c*K + k before it (same order as raw_rgb of eval_points_raw);
 *   child [n_nodes, N, N, N] int32: index of the child node minus the index of this node, 0 = leaf;
 *   world -> tree coordinates: p * invradius + offset in [0,1]^3.
 * ------------------------------------------------------------------------------------------- */
#define POB_OCTREE_RGBA 0 /* data_dim 4: colour = sigmoid(data[0:3])                              */
#define POB_OCTREE_SH 1   /* data_dim 3K+1: colour = sigmoid(sum_k Y_k(viewdir) * data[c*K+k])    */

typedef struct pob_octree {
  const float* data_dev;
  const int32_t* child_dev;
  int64_t n_nodes;
  int N;          /* branch factor per axis (flag tree_branch_n, octree/extraction.py:100) */
  int data_dim;
  int basis_dim;  /* K */
  int format;     /* POB_OCTREE_* */
  float offset[3];
  float invradius[3];
} pob_octree;

/* svox RenderOptions as VolumeRenderer fills them: step_size = flag renderer_step_size
 * (octree/nerf/utils.py:211-215), background_brightness 1, and sigma_thresh = stop_thresh = 1e-2 when
 * fast=True (evaluation without --no_early_stop, octree/nerf/utils.py:472), 0 otherwise. */
typedef struct pob_octree_opts {
  float step_size;
  float background_brightness;
  float sigma_thresh;
  float stop_thresh;
} pob_octree_opts;

/* perspective camera: c2w = first three rows of the camera-to-world matrix, row-major [3][4]
 * (svox CameraSpec: octree/extraction.py:194-199).  16 floats, also the element type of camera arrays. */
typedef struct pob_camera {
  float c2w[12];
  float fx, fy;
  float width, height;
} pob_camera;

/* NDC description of a forward-facing (LLFF) scene, svox NDCConfig(width, height, focal): the training images' size
 * and focal in pixels (octree/optimization.py:170-174, octree/nerf/utils.py:451-457, octree/extraction.py:187-193).
 * All three must be finite and > 0. */
typedef struct pob_ndc {
  float width, height, focal;
} pob_ndc;

/* The rays the octree march takes for a forward-facing scene: explicit world rays (origins/dirs/vdirs [n_rays,3],
 * cam NULL) or the pixel-row slab [row0, row0+nrows) of a perspective camera (cam != NULL, ray pointers ignored; the
 * pixel rays of pob_octree_render, row-major), turned into NDC as the reference's convert_to_ndc
 * (nerf_sh/nerf/datasets.py:40-60, near = 1): origin moved onto the plane z = -1, then projected.  out_origins_dev /
 * out_dirs_dev [n,3] receive the NDC origins and the NDC directions normalised to unit length; out_vdirs_dev [n,3] the
 * view directions, unchanged (explicit rays) or the pixel's unit world direction (camera), so that SH colours stay a
 * function of the world direction as in NeRF-SH training.  The outputs feed the explicit-ray entry points below
 * (render, backward, depth, compressed trees) unchanged. */
int pob_ndc_rays(const pob_ndc* ndc, const float* origins_dev, const float* dirs_dev, const float* vdirs_dev,
                 int64_t n_rays, const pob_camera* cam, int row0, int nrows, float* out_origins_dev,
                 float* out_dirs_dev, float* out_vdirs_dev, void* stream);

/* VolumeRenderer.forward(rays) / render_persp(c2w, width, height, fx): composite the tree along rays.
 * Either explicit rays (origins/dirs/vdirs [n_rays,3], cam NULL) or a pixel-row slab [row0, row0+nrows) of a
 * perspective camera (cam != NULL, ray pointers ignored; out is [nrows*width, 3] row-major).
 * counters_dev (may be NULL): [2] += {leaf visits, contributing leaf visits} for the roofline accounting. */
int pob_octree_render(const pob_octree* tree, const pob_octree_opts* opts, const float* origins_dev,
                      const float* dirs_dev, const float* vdirs_dev, int64_t n_rays, const pob_camera* cam,
                      int row0, int nrows, float* out_rgb_dev, unsigned long long* counters_dev, void* stream);

/* reverse mode of the above for an upstream gradient grad_out [n,3]: grad_data_dev (same shape as data,
 * ACCUMULATED into) += d<grad_out, rgb>/d data.  Thresholds are ignored like in svox's backward. */
int pob_octree_render_backward(const pob_octree* tree, const pob_octree_opts* opts, const float* origins_dev,
                               const float* dirs_dev, const float* vdirs_dev, int64_t n_rays, const pob_camera* cam,
                               int row0, int nrows, const float* grad_out_dev, float* grad_data_dev, void* stream);

/* pob_octree_render that also returns depth and opacity, the (rgb, disp, acc) of the NeRF-SH renderer minus the
 * disparity (acc / depth, formed by the caller).  out_rgb_dev and counters_dev are bit-identical to
 * pob_octree_render's.  Over the contributing visits i (sigma_i > sigma_thresh), visit i starting at t_i with step
 * dt_i and weight w_i = T_i (1 - exp(-dt_i * delta_scale * sigma_i)):
 *   out_acc_dev   [n] = sum_i w_i                      (the background is not included)
 *   out_depth_dev [n] = sum_i w_i (t_i + dt_i / 2) * delta_scale
 * a distance along the ray's direction vector (explicit rays: the parameter z of origin + z * dir), times
 * 1 / |(x, y, -1)| for a perspective pixel (camera-axis depth).  Early termination rescales both by 1 / (1 - T) like
 * the colour, so a stopped ray has acc = 1; a ray that misses the box has depth = acc = 0. */
int pob_octree_render_depth(const pob_octree* tree, const pob_octree_opts* opts, const float* origins_dev,
                            const float* dirs_dev, const float* vdirs_dev, int64_t n_rays, const pob_camera* cam,
                            int row0, int nrows, float* out_rgb_dev, float* out_depth_dev, float* out_acc_dev,
                            unsigned long long* counters_dev, void* stream);

/* reverse mode of pob_octree_render_depth: grad_data_dev (ACCUMULATED into) += d(<grad_rgb, rgb> + <grad_depth,
 * depth> + <grad_acc, acc>) / d data.  grad_rgb_dev [n,3], grad_depth_dev [n], grad_acc_dev [n]; any of the three
 * may be NULL (zero).  Depth and acc reach sigma only.  Thresholds are ignored like in pob_octree_render_backward. */
int pob_octree_render_depth_backward(const pob_octree* tree, const pob_octree_opts* opts, const float* origins_dev,
                                     const float* dirs_dev, const float* vdirs_dev, int64_t n_rays,
                                     const pob_camera* cam, int row0, int nrows, const float* grad_rgb_dev,
                                     const float* grad_depth_dev, const float* grad_acc_dev, float* grad_data_dev,
                                     void* stream);

/* A compressed PlenOctree, as octree.compression writes it for the web viewer: no `data`; per leaf an fp32 sigma
 * and, for each basis function k, the RGB triple of its coefficients either kept in fp16 (k < retain) or as an index
 * into a 2^bits-entry fp16 palette of that basis function (k >= retain).  With L = n_nodes * N^3 leaves (< 2^32):
 *   sigma_dev    [L] fp32                                 (quantised file key `sigma`)
 *   map_dev      [basis_dim - retain, L] uint16, < 2^bits (`quant_map`; the caller checks the range)
 *   palette_dev  [basis_dim - retain, 2^bits, 3] fp16     (`quant_colors`, as raw fp16 bits)
 *   retained_dev [retain, L, 3] fp16                      (`data_retained`; may be NULL when retain = 0)
 * child, N, format, offset and invradius as in pob_octree; 1 <= bits <= 16, 0 <= retain <= basis_dim.  The tree is
 * read-only: there is no backward or training pass for it. */
typedef struct pob_octree_quant {
  const int32_t* child_dev;
  int64_t n_nodes;
  int N;
  int basis_dim;
  int format;     /* POB_OCTREE_* */
  int retain;
  int bits;
  const float* sigma_dev;
  const uint16_t* map_dev;
  const uint16_t* palette_dev;
  const uint16_t* retained_dev;
  float offset[3];
  float invradius[3];
} pob_octree_quant;

/* pob_octree_render / pob_octree_render_depth on a compressed tree: the same march, ray sources, outputs and counters.
 * On the fp32 tree whose coefficients are the fp16 values the compressed tree decodes to (and the same sigma, child
 * and geometry), the outputs are bit-identical to the fp32 entry points'. */
int pob_octree_render_quant(const pob_octree_quant* tree, const pob_octree_opts* opts, const float* origins_dev,
                            const float* dirs_dev, const float* vdirs_dev, int64_t n_rays, const pob_camera* cam,
                            int row0, int nrows, float* out_rgb_dev, unsigned long long* counters_dev, void* stream);
int pob_octree_render_depth_quant(const pob_octree_quant* tree, const pob_octree_opts* opts, const float* origins_dev,
                                  const float* dirs_dev, const float* vdirs_dev, int64_t n_rays,
                                  const pob_camera* cam, int row0, int nrows, float* out_rgb_dev,
                                  float* out_depth_dev, float* out_acc_dev, unsigned long long* counters_dev,
                                  void* stream);

/* One training image of octree.optimization (octree/optimization.py:201-207) in one launch:
 *   im = render_persp(c2w); mse = mean((clamp(im,0,1) - gt)^2); mse.backward()
 * over the pixel rows [row0,row0+nrows): grad_data += grad_scale * d sum((clamp(im)-gt)^2) / d data,
 * *sq_err_sum_dev += sum((clamp(im)-gt)^2)  (grad_scale = 1/(H*W*3) gives the reference's mean);
 * gt_rgb_dev [nrows*width,3]; out_rgb_dev (may be NULL) receives the rendered slab. */
int pob_octree_train_persp(const pob_octree* tree, const pob_octree_opts* opts, const pob_camera* cam, int row0,
                           int nrows, const float* gt_rgb_dev, float grad_scale, float* grad_data_dev,
                           double* sq_err_sum_dev, float* out_rgb_dev, void* stream);

/* pob_octree_train_persp of a forward-facing scene: each pixel's ray is marched in NDC, as pob_ndc_rays makes it. */
int pob_octree_train_persp_ndc(const pob_octree* tree, const pob_octree_opts* opts, const pob_camera* cam,
                               const pob_ndc* ndc, int row0, int nrows, const float* gt_rgb_dev, float grad_scale,
                               float* grad_data_dev, double* sq_err_sum_dev, float* out_rgb_dev, void* stream);

/* torch.optim.SGD(lr, momentum 0).step() fused with zero_grad (octree/optimization.py:187-189,205-208):
 * data -= lr * grad; grad = 0, touching only entries whose gradient is non-zero. */
int pob_octree_sgd_step(float* data_dev, float* grad_dev, int64_t n, float lr, void* stream);

/* torch.optim.SGD(lr, momentum, dampening 0, nesterov).step() fused with zero_grad (octree/optimization.py:180-181,
 * 205-208), every element: buf = momentum * buf + grad (two roundings, as torch); d = nesterov ? grad + momentum * buf
 * : buf; data -= lr * d; grad = 0.  buf_dev is the caller's momentum buffer (same length as data), zero before the
 * first step.  Entries with grad = buf = 0 are not written.  momentum must be finite and >= 0. */
int pob_octree_sgd_momentum_step(float* data_dev, float* grad_dev, float* buf_dev, int64_t n, float lr, float momentum,
                                 int nesterov, void* stream);

/* torch.optim.Adam(lr, eps) (betas 0.9 / 0.999, no weight decay; octree/optimization.py:190-193, the `--nosgd` branch)
 * fused with zero_grad: m, v are the caller's moment buffers (same shape as data), `step` = updates already applied. */
int pob_octree_adam_step(float* data_dev, float* grad_dev, float* m_dev, float* v_dev, int64_t n, float lr, float step,
                         float eps, void* stream);

/* N3Tree.__getitem__(points): packed leaf index node*N^3 + (i*N + j)*N + k of the leaf holding each world
 * point (points clamped into the volume like svox). */
int pob_octree_query(const pob_octree* tree, const float* points_dev, int64_t n, int64_t* leaf_index_dev,
                     void* stream);

/* calculate_grid_weights (octree/extraction.py:181-214): march all pixels of n_cams cameras (cams_dev: device
 * array of pob_camera) through the dense sigma grid [reso]^3 and max-accumulate the per-voxel compositing
 * weight into max_weight_dev (caller zero-initialises; all cameras in one launch, no per-camera grids).
 * hit_dev (may be NULL): uint8 [reso]^3 set to 1 where any ray contributed. */
int pob_grid_weight_render(const float* sigma_grid_dev, int reso, const pob_camera* cams_dev, int n_cams,
                           int max_width, int max_height, const float offset[3], const float invradius[3],
                           const pob_octree_opts* opts, float* max_weight_dev, uint8_t* hit_dev, void* stream);

/* pob_grid_weight_render of a forward-facing scene (octree/extraction.py:187-193): every pixel's ray is marched
 * through the grid in NDC, as pob_ndc_rays makes it; offset / invradius map NDC coordinates into the grid. */
int pob_grid_weight_render_ndc(const float* sigma_grid_dev, int reso, const pob_camera* cams_dev, int n_cams,
                               int max_width, int max_height, const float offset[3], const float invradius[3],
                               const pob_octree_opts* opts, const pob_ndc* ndc, float* max_weight_dev,
                               uint8_t* hit_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * SH projection of a vanilla NeRF (use_viewdirs) in octree.extraction step2 (octree/extraction.py:217-241,362-394,
 * octree/nerf/sh_proj.py:273-306): coeff[p, c, k] = 4 pi / D * sum_d raw_rgb[p, d, c] Y_k(d) over D directions drawn
 * uniformly on the sphere, Y_k the SH basis of the octree march (sh_basis), the leaf value the mean over its samples.
 * The view branch raw_rgb = W11 relu(W10 [W9 h7 + b9; posenc(d)] + b10) + b11 is split as
 *   a_p = W10_b (W9 h7 + b9) + b10   (per sample point, 128 values; W10_b = Dense_10 kernel rows [0, 256))
 *   t_d = W10_e posenc(d, 0, deg_view, legacy_order)   (per direction; W10_e = rows [256, 256 + 3 + 6 deg_view))
 * so that raw_rgb[p, d] = W11 relu(a_p + t_d) + b11.  All arithmetic is fp32.
 * ------------------------------------------------------------------------------------------- */
/* The point stage in one trunk pass: raw sigma and a_p of m points.  packed_dev is the plain-RGB (sh_deg -1) blob of
 * the vanilla trunk and Dense_8 (rgb columns zero) packed with `posenc` (NULL = default; net_activation must be relu);
 * the fp16 forward evaluates it once, writes raw sigma_dev [m] (the value pob_eval_points_raw gives for that blob) and
 * keeps h7, the trunk's last activation, as fp16 in the workspace; then a_dev [m, 128] = h7 head_w + head_b in fp32
 * with head_w_dev [256, 128] = W9 W10_b and head_b_dev [128] = b9 W10_b + b10 (Dense_9 has no activation).
 * workspace_dev: pob_sh_proj_points_workspace_bytes(m) bytes (-1 for m < 0). */
int64_t pob_sh_proj_points_workspace_bytes(int64_t m);
int pob_sh_proj_points(const void* packed_dev, const pob_posenc* posenc, const float* points_dev, int64_t m,
                       const float* head_w_dev, const float* head_b_dev, void* workspace_dev, float* a_dev,
                       float* sigma_dev, void* stream);
/* The direction sets of table blocks block0 .. block0 + n_blocks - 1, n_dirs directions each: direction d of block b
 * is theta = acos(2u - 1), phi = 2 pi v, (sin theta cos phi, sin theta sin phi, cos theta) with (u, v) uniform in
 * [0, 1) from Philox4x32-10 keyed by `seed`, counter (d, b, stream 0x5348).  A block's set depends on (seed, b) only.
 *   w10e_dev  [3 + 6 deg_view, 128] fp32, W10_e as stored (kernel [in, out]);
 *   dirs_dev  [n_blocks, n_dirs, 3] (may be NULL);  t_dev [n_blocks, 128, n_dirs] = W10_e posenc(d) (stored
 *   direction-minor);  basis_dev [n_blocks, n_dirs, (sh_deg + 1)^2] = Y_k(d).
 * 0 <= n_blocks <= 65535, 0 <= deg_view <= 32, legacy_order 0 / 1 (the posenc feature order of pob_posenc),
 * 0 <= sh_deg <= 4. */
int pob_sh_proj_directions(uint64_t seed, int64_t block0, int n_blocks, int n_dirs, int deg_view, int legacy_order,
                           int sh_deg, const float* w10e_dev, float* dirs_dev, float* t_dev, float* basis_dev,
                           void* stream);
/* Leaf rows of a projected tree.  Cell i (of n_cells) owns sample points [i S, (i + 1) S) (S = samples_per_cell) and
 * uses direction set i / cells_per_block of the tables (pob_sh_proj_directions with the same n_dirs and sh_deg, at
 * least ceil(n_cells / cells_per_block) blocks).
 *   a_dev [n_cells * S, 128] = a_p;  sigma_dev [n_cells * S] raw sigma;  w11_dev [128, 3] (Dense_11 kernel), b11_dev [3]
 *   out_dev [n_cells, 3K + 1], K = (sh_deg + 1)^2: mean over the cell's points of [coeff (channel-major c K + k),
 *   raw sigma] (octree/extraction.py:391-393).
 * Every sum runs in a fixed order: a cell's row depends only on its points and its direction set. */
int pob_sh_proj_cells(int64_t n_cells, int samples_per_cell, int cells_per_block, const float* a_dev,
                      const float* sigma_dev, int n_dirs, int sh_deg, const float* t_dev, const float* basis_dev,
                      const float* w11_dev, const float* b11_dev, float* out_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Vanilla NeRF (use_viewdirs, sh_deg -1) inference: NerfModel.__call__ and eval_points_raw with the view branch
 *   (nerf_sh/nerf/models.py:143-214,216-348, model_utils.py:30-94).  Per MLP the branch is split as in the SH
 *   projection above: a_p = h7 (W9 W10_b) comes out of the tensor-core forward as heads columns 8..135 (column 0 is
 *   raw sigma, 1..7 are zero), t_r = W10_e posenc(viewdir_r, 0, deg_view, legacy_order) + c per ray (or point) with
 *   c = b9 W10_b + b10, and raw_rgb = W11 act(a_p + t_r) + b11, act = the trunk activation (pob_posenc
 *   net_activation), all in fp32 inside the forward's epilogue.  fp16 only; training is not covered.
 * ------------------------------------------------------------------------------------------- */
/* Folded flat parameters of one MLP: Dense_0..Dense_8 in the order of pob_pack_weights_pe (kernel [in,out], bias),
 * then the folded head W9 W10_b [256, 128] (no bias).  The forward rounds it to fp16: a caller that forms it in fp64
 * and rounds it to fp16 itself passes values the packing keeps exactly. */
int64_t pob_vanilla_param_count(const pob_posenc* posenc);
int64_t pob_vanilla_packed_bytes(void);
int pob_pack_vanilla(const float* flat_dev, const pob_posenc* posenc, void* packed_dev, void* stream);

/* The view branch of both MLPs (index 0 coarse, 1 fine), device fp32 arrays: w10e [3 + 6 deg_view, 128] (Dense_10
 * kernel rows [256, 256 + 3 + 6 deg_view)), c [128] = b9 W10_b + b10, w11 [128, 3], b11 [3].  The viewdir encoder
 * takes legacy_order from the config's pob_posenc. */
typedef struct pob_view_mlp {
  const float* w10e_dev;
  const float* c_dev;
  const float* w11_dev;
  const float* b11_dev;
} pob_view_mlp;
typedef struct pob_view_branch {
  int deg_view; /* 0..32 */
  pob_view_mlp mlp[2];
} pob_view_branch;

/* pob_workspace_bytes(cfg, 0) plus the two levels' per-ray tables; -1 on a refused config */
int64_t pob_vanilla_workspace_bytes(const pob_render_config* cfg);
/* pob_render_rays for vanilla blobs (pob_pack_vanilla): the same arguments and outputs; cfg->sh_deg must be -1,
 * precision POB_PREC_FP16; workspace_dev holds pob_vanilla_workspace_bytes(cfg) bytes and is 8-byte aligned (the
 * per-ray tables inside it are read in float2 pairs; cudaMalloc's 256-byte alignment satisfies both). */
int pob_render_rays_vanilla(const pob_render_config* cfg, const pob_view_branch* view, const void* packed_coarse_dev,
                            const void* packed_fine_dev, const float* origins_dev, const float* directions_dev,
                            const float* viewdirs_dev, int n_rays, const float* z_base_dev, const float* t_rand_dev,
                            const float* u_dev, int u_per_ray, const float* z_fine_dev, float* out_coarse_dev,
                            float* out_fine_dev, void* workspace_dev, int precision, void* stream);
/* MLP `mlp` (0 / 1 of view) on m points with one view direction each.  With out_rgbs_dev NULL, eval_points_raw:
 * raw_rgb_dev [m, 3] and raw_sigma_dev [m]; otherwise eval_points: out_rgbs_dev [m, 4] = (sigmoid(raw_rgb),
 * sigma_activation (POB_SIGMA_*) of raw sigma) and the raw pointers are ignored.  table_dev: m * 128 floats of scratch
 * (the per-point t), 8-byte aligned (the forward's epilogue reads it in float2 pairs); 512 bytes per point, so a
 * caller evaluates large point sets in chunks (VanillaNerfModel.eval_points_raw: 2^20 points per call). */
int pob_eval_points_vanilla(const void* packed_dev, const pob_posenc* posenc, const pob_view_branch* view, int mlp,
                            const float* points_dev, const float* viewdirs_dev, int64_t m, float* table_dev,
                            float* raw_rgb_dev, float* raw_sigma_dev, float* out_rgbs_dev, int sigma_activation,
                            void* stream);

/* ---------------------------------------------------------------------------------------------
 * Palette quantisation of compressed trees (octree.compression: median_cut)
 * ------------------------------------------------------------------------------------------- */
/* Median cut of n_basis independent point sets of n points each, byte-identical to the numpy median_cut:
 *   points_dev   [n_basis, n, 3] fp32
 *   weights_dev  [n] fp64 shared by every set, or NULL for the unweighted cut
 *   palette_dev  [n_basis, 2^bits, 3] fp32 out: the (weighted) mean of every box, zero for empty boxes
 *   map_dev      [n_basis, n] uint16 out: the box of every point
 * 0 <= bits <= 16, 0 <= n < 2^31, n_basis >= 1 with n_basis * n < 2^40.  workspace_dev holds
 * pob_quantize_workspace_bytes(n_basis, n, weights != NULL) bytes, 256-byte aligned; the call is deterministic and
 * independent of POB_SM_COUNT.  Every refusal returns before any launch. */
int64_t pob_quantize_workspace_bytes(int64_t n_basis, int64_t n, int weighted);
int pob_quantize_median_cut(const float* points_dev, const double* weights_dev, int64_t n_basis, int64_t n, int bits,
                            float* palette_dev, uint16_t* map_dev, void* workspace_dev, int64_t workspace_bytes,
                            void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PLENOCTREE_B200_H */
