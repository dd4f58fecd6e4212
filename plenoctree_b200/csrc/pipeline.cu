// pipeline.cu — host-side sequencing of the kernels into the two reference-level operations:
//   pob_render_rays    = NerfModel.__call__            (nerf_sh/nerf/models.py:216-348)
//   pob_render_rays_vanilla: the same with use_viewdirs (the view branch in the forward's epilogue)
//   pob_loss_and_grad  = value_and_grad(loss_fn)       (nerf_sh/train.py:66-116)
//   pob_adam_update    = optimizer.apply_gradient      (nerf_sh/train.py:119) + operand re-pack
// Everything is enqueued on the caller's stream; nothing synchronises with the host.
#include <cuda.h>

#include <cstring>
#include <string>

#include "../../include/plenoctree_b200.h"
#include "capi_util.h"
#include "common.cuh"
#include "kernels.h"

namespace {

using namespace pob;

struct Level {
  // sizes
  int N;              // samples per ray (0: no fine level)
  bool last;          // the last level: in training its arrays also carry the sparsity points behind its rays
  long long M;        // samples
  long long tiles;    // 128-row tiles of padded_rows(M)
  // buffers
  float* z;           // [R,N]
  float4* rgbs;       // [M]
  float* weights;     // [R,N]
  float* comp;        // [R,3]
  float* disp;        // [R]
  float* acc;         // [R]
  float4* G;          // [M]
  uint8_t *H, *E, *DZ, *DO;
  uint32_t* mask;
  uint8_t *H_lo, *E_lo, *DZ_lo, *DO_lo;   // x3 training: residual images of H, E, DZ, DO
  float* view_t;      // vanilla rendering: [R, VIEW_H] per-ray view table of the level's MLP
};

struct Workspace {
  Level lv[2];        // coarse, fine
  int levels;         // 1 or 2
  float* partials[2]; // wgrad partials of the two MLPs' launches
  uint32_t* progress; // per tile of level 0, then of level 1: mlp_bwd -> mlp_wgrad progress counters (wgrad_body.cuh)
  size_t progress_bytes;
  // x3 training only, behind everything the fp16 step uses (so that its layout is the fp16 one plus this tail)
  float* partials_x3[2][2];   // [mlp][wgrad pass 1, 2]
  uint8_t* wt_lo[2];          // [mlp] residual of the dgrad weight images, written from params_dev by every call
  size_t total;
};

size_t up(size_t x) { return (x + 1023) / 1024 * 1024; }

// every per-tile array is padded to a multiple of four 128-row tiles (common.cuh: padded_rows)
long long tiles_for(long long M) { return padded_rows(M) / TILE_M; }

// SMs (out of an H100 SXM's 132) that run mlp_bwd during the backward; mlp_wgrad runs on the others.  SH16 training
// step (bench.py --steps 30 --warmup 5) on an H100 80 GB HBM3 at a 700 W power limit (1980 MHz maximum SM clock), with
// train_step discarding dZ / dO from L2 (wgrad_body.cuh), dgrad on 52 / 54 / 56 / 58 / 60 SMs, two sessions of two or
// three runs each: 6.57 / 6.39-6.51 / 6.41-6.54 / 6.45-6.54 / 6.55-6.60 ms.  Without the write-backs the data gradient
// on 60 SMs ended 0.2 ms before the weight gradient (fine level), so SMs move to the weight gradient until, at 52, the
// data gradient becomes the long pole.  The split sets how many CTAs sum each layer's partial gradient (optim.cu:
// wgrad_assign_roles), so changing it changes the gradient's fp32 summation order (DESIGN.md section 6).
// SH25 (heads width 80: a third heads K-slot in the data gradient, a 128-feature dO for the weight gradient) keeps 60:
// its tt step (bench_extras tt_sh25) took 7.13 ms at 56 against 6.84 ms for the kernels before the discard at 60.
constexpr int DGRAD_SMS_OF_132 = 56;
constexpr int DGRAD_SMS_OF_132_NH80 = 60;

// deterministic carve of the caller-provided workspace (x3: the training workspace of the fp16x3 step)
// (vanilla: the render workspace plus the per-ray view tables, behind everything else)
Workspace carve(const pob_render_config& c, int training, uint8_t* base, bool x3 = false, bool vanilla = false) {
  Workspace w;
  memset(&w, 0, sizeof(w));
  size_t off = 0;
  auto take = [&](size_t bytes) {
    uint8_t* p = base ? base + off : nullptr;
    off += up(bytes);
    return p;
  };
  const long long R = c.max_rays;
  w.levels = c.num_fine_samples > 0 ? 2 : 1;
  for (int l = 0; l < 2; ++l) {
    Level& L = w.lv[l];
    L.N = l == 0 ? c.num_coarse_samples : (w.levels == 2 ? c.num_coarse_samples + c.num_fine_samples : 0);
    L.last = l == w.levels - 1;
    const long long Mr = R * L.N;                                      // ray samples
    L.M = Mr + ((training && L.last) ? c.sparsity_npoints : 0);        // + sparsity points (train.py:77-83)
    L.tiles = tiles_for(L.M);
    if (Mr == 0) continue;
    L.z = (float*)take(sizeof(float) * Mr);
    L.rgbs = (float4*)take(sizeof(float4) * L.M);
    L.weights = (float*)take(sizeof(float) * Mr);
    L.comp = (float*)take(sizeof(float) * 3 * R);
    L.disp = (float*)take(sizeof(float) * R);
    L.acc = (float*)take(sizeof(float) * R);
    if (training) {
      L.G = (float4*)take(sizeof(float4) * L.M);
      L.H = take(size_t(L.tiles) * NUM_TRUNK * A_TILE_BYTES);
      L.E = take(size_t(L.tiles) * E_TILE_BYTES);
      L.DZ = take(size_t(L.tiles) * NUM_TRUNK * A_TILE_BYTES);
      L.DO = take(size_t(L.tiles) * 2 * A_CHUNK_BYTES);
      L.mask = (uint32_t*)take(size_t(NUM_TRUNK) * L.tiles * TILE_M * 8 * sizeof(uint32_t));
    }
  }
  if (training) {
    for (int i = 0; i < 2; ++i) w.partials[i] = (float*)take(sizeof(float) * WG_MAX_CTAS * WG_PARTIAL_FLOATS);
    w.progress_bytes = sizeof(uint32_t) * size_t(w.lv[0].tiles + w.lv[1].tiles);
    w.progress = (uint32_t*)take(w.progress_bytes);
  }
  if (training && x3) {
    for (int l = 0; l < 2; ++l) {
      Level& L = w.lv[l];
      if (L.N == 0) continue;
      L.H_lo = take(size_t(L.tiles) * NUM_TRUNK * A_TILE_BYTES);
      L.E_lo = take(size_t(L.tiles) * E_TILE_BYTES);
      L.DZ_lo = take(size_t(L.tiles) * NUM_TRUNK * A_TILE_BYTES);
      L.DO_lo = take(size_t(L.tiles) * 2 * A_CHUNK_BYTES);
    }
    for (int i = 0; i < 2; ++i)
      for (int q = 0; q < 2; ++q) w.partials_x3[i][q] = (float*)take(sizeof(float) * WG_MAX_CTAS * WG_PARTIAL_FLOATS);
    for (int i = 0; i < 2; ++i) w.wt_lo[i] = take(bwd_image_bytes(heads_width(K_of(c.sh_deg))));
  }
  if (vanilla)
    for (int l = 0; l < 2; ++l)
      if (w.lv[l].N > 0) w.lv[l].view_t = (float*)take(sizeof(float) * VIEW_H * size_t(R));
  w.total = off;
  return w;
}

// the config's checks; `net` is then its point encoder and trunk activation
int check_cfg(const char* where, const pob_render_config* c, NetDesc& net) {
  if (!c) return pob_fail(where, "config is NULL");
  if (!valid_deg(c->sh_deg)) return pob_fail(where, "sh_deg must be in [-1, 4]");
  if (c->num_coarse_samples < 3 || c->num_coarse_samples > MAX_RAY_SAMPLES)
    return pob_fail(where, "num_coarse_samples must be in [3, 1024]");
  if (c->num_fine_samples < 0 || c->num_coarse_samples + c->num_fine_samples > MAX_RAY_SAMPLES)
    return pob_fail(where, "num_coarse_samples + num_fine_samples must be <= 1024");
  if (c->max_rays <= 0) return pob_fail(where, "max_rays must be positive");
  if (c->sparsity_npoints < 0) return pob_fail(where, "sparsity_npoints must be >= 0");
  if (int e = pob_check_posenc(where, c->posenc, net)) return e;
  return pob_check_sigma_activation(where, c->sigma_activation);
}

// forward of every level; fills comp/disp/acc (and rgbs, weights, z) of the workspace levels.  The depths of a level
// are the coarse draw, the caller's z_fine or the resampling of the coarse weights.  With `view` the packed blobs are
// vanilla MLPs: each level first tabulates its MLP's view branch for the rays, then runs the vanilla forward.
int forward_levels(const char* where, const pob_render_config& c, NetDesc net, int sms, Workspace& w,
                   const void* const packed[2], const float* o, const float* d, const float* v, int R,
                   const float* z_base, const float* t_rand, const float* u, int u_per_ray, const float* z_fine,
                   int precision, bool save, cudaStream_t st, const float* sp_points = nullptr, long long sp_n = 0,
                   const pob_view_branch* view = nullptr) {
  const float* const noise[2] = {c.sigma_noise_coarse_dev, c.sigma_noise_fine_dev};
  for (int l = 0; l < w.levels; ++l) {
    Level& L = w.lv[l];
    if (l == 0)
      POB_LAUNCH(where, POB_PH_RENDER, st, launch_sample_coarse(z_base, t_rand, R, L.N, L.z, st));
    else if (z_fine)
      POB_CUDA(where, cudaMemcpyAsync(L.z, z_fine, sizeof(float) * size_t(R) * L.N, cudaMemcpyDeviceToDevice, st));
    else
      POB_LAUNCH(where, POB_PH_RENDER, st,
                 launch_sample_pdf(w.lv[0].z, w.lv[0].weights, u, u_per_ray, R, c.num_coarse_samples,
                                   c.num_fine_samples, L.z, st));
    FwdParams p;
    if (view) {
      POB_LAUNCH(where, POB_PH_FWD, st,
                 launch_view_table(v, R, view->deg_view, net.pe.legacy, view->mlp[l].w10e_dev, view->mlp[l].c_dev,
                                   L.view_t, st));
      p = pob_vanilla_params(packed[l], net, *view, l, L.view_t);
    } else {
      p = pob_base_params(packed[l], c.sh_deg, net);
      p.out_mode = OUT_RGBS;
    }
    p.src_mode = SRC_RAYS;
    p.M = (long long)R * L.N;
    p.M_rays = p.M;
    p.origins = o;
    p.directions = d;
    p.viewdirs = v;
    p.zvals = L.z;
    p.n_per_ray = L.N;
    p.out_rgbs = L.rgbs;
    p.sigma_noise = noise[l];
    p.sigma_act = c.sigma_activation;
    if (L.last && sp_n > 0) {     // the sparsity points ride behind the last level's ray samples (same MLP)
      p.M += sp_n;
      p.extra_points = sp_points;
    }
    if (save) {
      p.save_h = L.H;
      p.save_e = L.E;
      p.save_mask = L.mask;
      p.save_h_lo = L.H_lo;   // x3 only (null otherwise)
      p.save_e_lo = L.E_lo;
    }
    POB_LAUNCH(where, POB_PH_FWD, st,
               view ? launch_mlp_fwd_vanilla(p, sms, st) : launch_mlp_fwd(p, precision, sms, st));
    POB_LAUNCH(where, POB_PH_RENDER, st,
               launch_composite_fwd(L.rgbs, L.z, d, R, L.N, c.white_bkgd, L.comp, L.disp, L.acc, L.weights, st));
  }
  return 0;
}

__global__ void pack_outputs_kernel(const float* comp, const float* disp, const float* acc, int R, float* out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  out[5 * r + 0] = comp[3 * r + 0];
  out[5 * r + 1] = comp[3 * r + 1];
  out[5 * r + 2] = comp[3 * r + 2];
  out[5 * r + 3] = disp[r];
  out[5 * r + 4] = acc[r];
}

// The device allocation that holds `ws` must extend to ws + bytes: a workspace sized for the fp16 step (the x3
// tail missing) is refused instead of written past.  The query is the driver's cuMemGetAddressRange, which neither
// synchronises nor enqueues work, so the check is also made under stream capture.  It sees allocations, not the
// blocks a caching allocator cuts out of them: a too-small block inside a larger allocation passes.
int check_workspace_extent(const char* where, const void* ws, size_t bytes) {
  using RangeFn = CUresult (*)(CUdeviceptr*, size_t*, CUdeviceptr);
  static RangeFn range = [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPointByVersion("cuMemGetAddressRange", &fn, 12000, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      fn = nullptr;
    return reinterpret_cast<RangeFn>(fn);
  }();
  if (!range) return pob_fail(where, "cannot query the workspace allocation (cuMemGetAddressRange)");
  CUdeviceptr base = 0;
  size_t size = 0;
  if (range(&base, &size, (CUdeviceptr)ws) != CUDA_SUCCESS)
    return pob_fail(where, "workspace is not a device allocation");
  if ((CUdeviceptr)ws + bytes > base + size)
    return pob_fail(where, "workspace too small for this precision (pob_train_workspace_bytes)");
  return 0;
}

// pob_render_rays and pob_render_rays_vanilla (view != NULL) past their own checks
int render_rays(const char* where, const pob_render_config* cfg, const pob_view_branch* view, NetDesc net, int sms,
                const void* packed_coarse_dev, const void* packed_fine_dev, const float* origins_dev,
                const float* directions_dev, const float* viewdirs_dev, int n_rays, const float* z_base_dev,
                const float* t_rand_dev, const float* u_dev, int u_per_ray, const float* z_fine_dev,
                float* out_coarse_dev, float* out_fine_dev, void* workspace_dev, int precision, void* stream) {
  if (n_rays < 0 || n_rays > cfg->max_rays) return pob_fail(where, "n_rays exceeds cfg->max_rays");
  if (n_rays == 0) return 0;
  if (!origins_dev || !directions_dev || !viewdirs_dev || !z_base_dev || !workspace_dev || !out_coarse_dev)
    return pob_fail(where, "NULL pointer");
  if (cfg->num_fine_samples > 0 && (!packed_fine_dev || (!u_dev && !z_fine_dev) || !out_fine_dev))
    return pob_fail(where, "fine level needs packed_fine, u (or z_fine) and out_fine");
  cudaStream_t st = (cudaStream_t)stream;
  Workspace w = carve(*cfg, 0, (uint8_t*)workspace_dev, false, view != nullptr);
  const void* const packed[2] = {packed_coarse_dev, packed_fine_dev};
  if (int e = forward_levels(where, *cfg, net, sms, w, packed, origins_dev, directions_dev, viewdirs_dev, n_rays,
                             z_base_dev, t_rand_dev, u_dev, u_per_ray, z_fine_dev, precision, false, st, nullptr, 0,
                             view))
    return e;
  const unsigned grid = (n_rays + 255) / 256;
  pob_count_launch(w.levels);
  pack_outputs_kernel<<<grid, 256, 0, st>>>(w.lv[0].comp, w.lv[0].disp, w.lv[0].acc, n_rays, out_coarse_dev);
  if (w.levels == 2)
    pack_outputs_kernel<<<grid, 256, 0, st>>>(w.lv[1].comp, w.lv[1].disp, w.lv[1].acc, n_rays, out_fine_dev);
  POB_CUDA(where, cudaGetLastError());
  return 0;
}

// the config checks of the vanilla entry points: check_cfg, then sh_deg -1
int check_vanilla_cfg(const char* where, const pob_render_config* cfg, NetDesc& net) {
  if (int e = check_cfg(where, cfg, net)) return e;
  if (cfg->sh_deg != -1) return pob_fail(where, "a vanilla NeRF has the plain-RGB head: cfg->sh_deg must be -1");
  return 0;
}

}  // namespace

extern "C" {

int64_t pob_workspace_bytes(const pob_render_config* cfg, int training) {
  NetDesc net;
  if (check_cfg("pob_workspace_bytes", cfg, net)) return -1;
  return (int64_t)carve(*cfg, training, nullptr).total;
}

int64_t pob_train_workspace_bytes(const pob_render_config* cfg, int precision) {
  NetDesc net;
  if (check_cfg("pob_train_workspace_bytes", cfg, net)) return -1;
  if (precision != POB_PREC_FP16 && precision != POB_PREC_FP16X3) {
    pob_fail("pob_train_workspace_bytes", "precision must be POB_PREC_FP16 or POB_PREC_FP16X3");
    return -1;
  }
  return (int64_t)carve(*cfg, 1, nullptr, precision == POB_PREC_FP16X3).total;
}

int pob_render_rays(const pob_render_config* cfg, const void* packed_coarse_dev, const void* packed_fine_dev,
                    const float* origins_dev, const float* directions_dev, const float* viewdirs_dev,
                    int n_rays, const float* z_base_dev, const float* t_rand_dev, const float* u_dev,
                    int u_per_ray, const float* z_fine_dev, float* out_coarse_dev, float* out_fine_dev,
                    void* workspace_dev, int precision, void* stream) {
  const char* where = "pob_render_rays";
  NetDesc net;
  if (int e = check_cfg(where, cfg, net)) return e;
  const int sms = pob_check_common(where, packed_coarse_dev, cfg->sh_deg, precision);
  if (!sms) return 1;
  return render_rays(where, cfg, nullptr, net, sms, packed_coarse_dev, packed_fine_dev, origins_dev, directions_dev,
                     viewdirs_dev, n_rays, z_base_dev, t_rand_dev, u_dev, u_per_ray, z_fine_dev, out_coarse_dev,
                     out_fine_dev, workspace_dev, precision, stream);
}

int64_t pob_vanilla_workspace_bytes(const pob_render_config* cfg) {
  NetDesc net;
  if (check_vanilla_cfg("pob_vanilla_workspace_bytes", cfg, net)) return -1;
  return (int64_t)carve(*cfg, 0, nullptr, false, true).total;
}

int pob_render_rays_vanilla(const pob_render_config* cfg, const pob_view_branch* view, const void* packed_coarse_dev,
                            const void* packed_fine_dev, const float* origins_dev, const float* directions_dev,
                            const float* viewdirs_dev, int n_rays, const float* z_base_dev, const float* t_rand_dev,
                            const float* u_dev, int u_per_ray, const float* z_fine_dev, float* out_coarse_dev,
                            float* out_fine_dev, void* workspace_dev, int precision, void* stream) {
  const char* where = "pob_render_rays_vanilla";
  NetDesc net;
  if (int e = check_vanilla_cfg(where, cfg, net)) return e;
  if (precision != POB_PREC_FP16) return pob_fail(where, "the vanilla forward is fp16: precision must be POB_PREC_FP16");
  if (!packed_coarse_dev) return pob_fail(where, "packed weights pointer is NULL");
  if (int e = pob_check_view(where, view, cfg->num_fine_samples > 0 ? 2 : 1)) return e;
  if (reinterpret_cast<uintptr_t>(workspace_dev) & 7) return pob_fail(where, "workspace_dev must be 8-byte aligned");
  const int sms = pob_sms_or_fail(where);
  if (!sms) return 1;
  return render_rays(where, cfg, view, net, sms, packed_coarse_dev, packed_fine_dev, origins_dev, directions_dev,
                     viewdirs_dev, n_rays, z_base_dev, t_rand_dev, u_dev, u_per_ray, z_fine_dev, out_coarse_dev,
                     out_fine_dev, workspace_dev, precision, stream);
}

int pob_loss_and_grad_flags(const pob_render_config* cfg, const pob_train_hparams* hp, const void* packed_coarse_dev,
                            const void* packed_fine_dev, const float* origins_dev, const float* directions_dev,
                            const float* viewdirs_dev, const float* pixels_dev, int n_rays, const float* z_base_dev,
                            const float* t_rand_dev, const float* u_dev, int u_per_ray, const float* z_fine_dev,
                            const float* sp_points_dev, float* grad_flat_dev, float* stats_dev, void* workspace_dev,
                            void* mlp0_done_event, const float* params_dev, int precision, int flags, void* stream) {
  const char* where = "pob_loss_and_grad";
  if (flags & ~POB_TRAIN_DISCARD_SAVED_GRADS) return pob_fail(where, "unknown bits in flags");
  NetDesc net;
  if (int e = check_cfg(where, cfg, net)) return e;
  if (!hp) return pob_fail(where, "hparams is NULL");
  const int sms = pob_check_common(where, packed_coarse_dev, cfg->sh_deg, precision);
  if (!sms) return 1;
  const bool x3 = precision == POB_PREC_FP16X3;
  if (n_rays <= 0 || n_rays > cfg->max_rays) return pob_fail(where, "n_rays out of range");
  if (!origins_dev || !directions_dev || !viewdirs_dev || !pixels_dev || !z_base_dev || !workspace_dev ||
      !grad_flat_dev || !stats_dev)
    return pob_fail(where, "NULL pointer");
  if (x3 && !params_dev) return pob_fail(where, "POB_PREC_FP16X3 needs params_dev (the flat fp32 parameters)");
  if (cfg->num_fine_samples > 0 && (!packed_fine_dev || (!u_dev && !z_fine_dev)))
    return pob_fail(where, "fine level needs packed_fine and u (or z_fine)");
  const bool sparsity = hp->sparsity_weight > 0.f && cfg->sparsity_npoints > 0;
  if (sparsity && !sp_points_dev) return pob_fail(where, "sparsity term needs sp_points");
  if (!(hp->loss_scale > 0.f)) return pob_fail(where, "loss_scale must be positive");
  cudaStream_t st = (cudaStream_t)stream;
  const int K = K_of(cfg->sh_deg);
  const int W = posenc_width(net.pe);
  const int P = flat_layout(K, W).total;
  Workspace w = carve(*cfg, 1, (uint8_t*)workspace_dev, x3);
  if (x3)
    if (int e = check_workspace_extent(where, workspace_dev, w.total)) return e;
  POB_CUDA(where, cudaMemsetAsync(stats_dev, 0, 8 * sizeof(float), st));
  POB_CUDA(where, cudaMemsetAsync(w.progress, 0, w.progress_bytes, st));
  if (x3) {
    // residual of the transposed weights (the packed blob holds only their hi part)
    for (int mlp = 0; mlp < w.levels; ++mlp)
      POB_LAUNCH(where, POB_PH_OPTIM, st, launch_pack_wt_lo(params_dev + size_t(mlp) * P, K, W, w.wt_lo[mlp], st));
  }
  // The sparsity points (train.py:77-83: eval_points_raw of the fine MLP on uniform points) ride behind the ray
  // samples of the last level: same MLP, same launches, rows [n_rays * N, n_rays * N + sp_n) of its arrays.
  const long long sp_n = sparsity ? cfg->sparsity_npoints : 0;
  const void* const packed[2] = {packed_coarse_dev, packed_fine_dev};
  if (int e = forward_levels(where, *cfg, net, sms, w, packed, origins_dev, directions_dev, viewdirs_dev, n_rays,
                             z_base_dev, t_rand_dev, u_dev, u_per_ray, z_fine_dev, precision, true, st, sp_points_dev,
                             sp_n))
    return e;
  const float gscale = hp->loss_scale * 2.0f / (3.0f * float(n_rays));
  // ---- upstream gradients: stats slot 0 takes the last level's loss, slot 1 the coarse one's of two levels ----
  for (int l = 0; l < w.levels; ++l) {
    Level& L = w.lv[l];
    POB_LAUNCH(where, POB_PH_RENDER, st,
               launch_composite_bwd(L.rgbs, L.z, directions_dev, L.comp, pixels_dev, n_rays, L.N, cfg->white_bkgd,
                                    gscale, cfg->sigma_activation, L.G, stats_dev + (L.last ? 0 : 1), st));
  }
  if (sparsity) {
    Level& L = w.lv[w.levels - 1];
    const long long Mr = (long long)n_rays * L.N;
    const float coef = hp->loss_scale * hp->sparsity_weight * hp->sparsity_length / float(sp_n);
    POB_LAUNCH(where, POB_PH_RENDER, st,
               launch_sparsity_grad(L.rgbs + Mr, int(sp_n), hp->sparsity_length, coef, L.G + Mr, stats_dev + 2, st));
  }
  // ---- backward: per MLP one dgrad launch, then ONE wgrad launch over its saved dZ / h tiles ----
  // MLP_0 (coarse level only) is finished first: its branch of the graph is independent of MLP_1's
  // (stop_gradient, model_utils.py:286), so the caller can all-reduce the MLP_0 bucket of the gradient
  // (mlp0_done_event) while the 3x larger MLP_1 backward is still running.
  // dgrad runs on `dgrad_ctas` SMs and wgrad alongside it on the rest, reading each dZ tile from L2 shortly after it
  // was stored (wgrad_body.cuh).  x3: the data gradient runs on all SMs, then the three wgrad passes (kernels.h:
  // X3_WGRAD_PASSES) one after the other, each on all SMs.  SH16 step (bench.py's workload) on an H100 80 GB HBM3 at a
  // 400 W power limit: 29.1-29.6 ms against 31.8-32.1 ms with the fp16 split (pass 0 beside the data gradient).
  const int NH = heads_width(K);
  const int dgrad_ctas = sms * (NH <= 64 ? DGRAD_SMS_OF_132 : DGRAD_SMS_OF_132_NH80) / 132;
  for (int mlp = 0; mlp < w.levels; ++mlp) {
    Level& L = w.lv[mlp];
    const long long Mr = (long long)n_rays * L.N;
    const long long Mm = Mr + (L.last ? sp_n : 0);
    BwdParams b;
    memset(&b, 0, sizeof(b));
    b.M = Mm;
    b.M_rays = Mr;
    b.G = L.G;
    b.viewdirs = viewdirs_dev;
    b.n_per_ray = L.N;
    FwdParams base = pob_base_params(packed[mlp], cfg->sh_deg, net);
    b.w = base.w;
    b.sh_deg = cfg->sh_deg;
    b.K = base.K;
    b.NH = base.NH;
    b.net_act = net.net_act;
    b.mask = L.mask;
    b.h = L.H;
    b.h_lo = L.H_lo;
    b.save_dz = L.DZ;
    b.save_do = L.DO;
    b.progress = w.progress + (mlp == 0 ? 0 : w.lv[0].tiles);
    b.wt_lo = w.wt_lo[mlp];
    b.save_dz_lo = L.DZ_lo;
    b.save_do_lo = L.DO_lo;
    POB_LAUNCH(where, POB_PH_BWD, st, launch_mlp_bwd(b, precision, x3 ? sms : dgrad_ctas, st));
    const WgradSegment segs[X3_WGRAD_PASSES] = {{L.H, L.DZ, L.E, L.DO},
                                                {L.H, L.DZ_lo, L.E, L.DO_lo},
                                                {L.H_lo, L.DZ, L.E_lo, L.DO}};
    float* const partials[X3_WGRAD_PASSES] = {w.partials[mlp], w.partials_x3[mlp][0], w.partials_x3[mlp][1]};
    const int npass = x3 ? X3_WGRAD_PASSES : 1;
    WgradPass passes[X3_WGRAD_PASSES];
    for (int q = 0; q < npass; ++q) {
      WgradParams g;
      memset(&g, 0, sizeof(g));
      g.seg = segs[q];
      g.seg_tiles = tiles_for(Mm);
      g.NH = NH;
      g.partials = partials[q];
      g.progress = b.progress;
      // fp16x3: the passes run after the data gradient and read dZ twice, so the tiles stay
      g.discard = !x3 && (flags & POB_TRAIN_DISCARD_SAVED_GRADS);
      passes[q].partials = partials[q];
      const int nctas = wgrad_assign_roles(g, (q == 0 && !x3) ? sms - dgrad_ctas : sms, passes[q].role_start,
                                           passes[q].role_count);
      POB_LAUNCH(where, POB_PH_WGRAD, st, launch_mlp_wgrad(g, nctas, st));
    }
    POB_LAUNCH(where, POB_PH_OPTIM, st,
               launch_reduce_grads(passes, npass, K, W, 1.0f / hp->loss_scale, grad_flat_dev + size_t(mlp) * P, st));
    if (mlp == 0 && w.levels == 2 && mlp0_done_event)
      POB_CUDA(where, cudaEventRecord((cudaEvent_t)mlp0_done_event, st));
  }
  return 0;
}

int pob_loss_and_grad_prec(const pob_render_config* cfg, const pob_train_hparams* hp, const void* packed_coarse_dev,
                           const void* packed_fine_dev, const float* origins_dev, const float* directions_dev,
                           const float* viewdirs_dev, const float* pixels_dev, int n_rays, const float* z_base_dev,
                           const float* t_rand_dev, const float* u_dev, int u_per_ray, const float* z_fine_dev,
                           const float* sp_points_dev, float* grad_flat_dev, float* stats_dev, void* workspace_dev,
                           void* mlp0_done_event, const float* params_dev, int precision, void* stream) {
  return pob_loss_and_grad_flags(cfg, hp, packed_coarse_dev, packed_fine_dev, origins_dev, directions_dev,
                                 viewdirs_dev, pixels_dev, n_rays, z_base_dev, t_rand_dev, u_dev, u_per_ray, z_fine_dev,
                                 sp_points_dev, grad_flat_dev, stats_dev, workspace_dev, mlp0_done_event, params_dev,
                                 precision, 0, stream);
}

int pob_loss_and_grad(const pob_render_config* cfg, const pob_train_hparams* hp, const void* packed_coarse_dev,
                      const void* packed_fine_dev, const float* origins_dev, const float* directions_dev,
                      const float* viewdirs_dev, const float* pixels_dev, int n_rays, const float* z_base_dev,
                      const float* t_rand_dev, const float* u_dev, int u_per_ray, const float* z_fine_dev,
                      const float* sp_points_dev, float* grad_flat_dev, float* stats_dev, void* workspace_dev,
                      void* mlp0_done_event, void* stream) {
  return pob_loss_and_grad_prec(cfg, hp, packed_coarse_dev, packed_fine_dev, origins_dev, directions_dev, viewdirs_dev,
                                pixels_dev, n_rays, z_base_dev, t_rand_dev, u_dev, u_per_ray, z_fine_dev, sp_points_dev,
                                grad_flat_dev, stats_dev, workspace_dev, mlp0_done_event, nullptr, POB_PREC_FP16,
                                stream);
}

int pob_adam_update_pe(int sh_deg, const pob_posenc* posenc, int num_mlps, float* params_dev, const float* grads_dev,
                       float* m_dev, float* v_dev, float lr, float step, const float* lr_step_dev, float grad_mult,
                       float weight_decay_coef, void* packed_coarse_dev, void* packed_fine_dev, void* stream) {
  const char* where = "pob_adam_update";
  if (!valid_deg(sh_deg)) return pob_fail(where, "sh_deg must be in [-1, 4]");
  NetDesc net;
  if (int e = pob_check_posenc(where, posenc, net)) return e;
  if (num_mlps < 1 || num_mlps > 2) return pob_fail(where, "num_mlps must be 1 or 2");
  if (!params_dev || !grads_dev || !m_dev || !v_dev || !packed_coarse_dev || (num_mlps == 2 && !packed_fine_dev))
    return pob_fail(where, "NULL pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const long long P = flat_layout(K_of(sh_deg), posenc_width(net.pe)).total;
  POB_LAUNCH(where, POB_PH_OPTIM, st,
             launch_adam(params_dev, grads_dev, m_dev, v_dev, P * num_mlps, lr, step, lr_step_dev, 0.9f, 0.999f, 1e-8f,
                         grad_mult, weight_decay_coef, st));
  if (int e = pob_pack_weights_pe(params_dev, sh_deg, posenc, packed_coarse_dev, stream)) return e;
  if (num_mlps == 2)
    if (int e = pob_pack_weights_pe(params_dev + P, sh_deg, posenc, packed_fine_dev, stream)) return e;
  return 0;
}

int pob_adam_update(int sh_deg, int num_mlps, float* params_dev, const float* grads_dev, float* m_dev,
                    float* v_dev, float lr, float step, const float* lr_step_dev, float grad_mult,
                    float weight_decay_coef, void* packed_coarse_dev, void* packed_fine_dev, void* stream) {
  return pob_adam_update_pe(sh_deg, nullptr, num_mlps, params_dev, grads_dev, m_dev, v_dev, lr, step, lr_step_dev,
                            grad_mult, weight_decay_coef, packed_coarse_dev, packed_fine_dev, stream);
}

}  // extern "C"
