// render.cu — per-ray stages of NerfModel.__call__ that are not GEMMs: stratified sampling,
// volumetric alpha-compositing (forward and backward), inverse-CDF hierarchical resampling with the
// union sort, MSE loss gradient.  All fp32.  A ray is a group of W warps at up to MAX_SEG samples per lane: W = 1
// (four rays per 128-thread block, warp-shuffle scans / reductions) for N <= 256, and W = 4 (one ray per block) for
// 256 < N <= MAX_RAY_SAMPLES, where each scan and reduction adds one cross-warp step through shared memory.  The
// W = 1 instantiations compile to the kernels as they were before W existed.
//
//   sample_along_rays       nerf_sh/nerf/model_utils.py:104-142
//   volumetric_rendering    nerf_sh/nerf/model_utils.py:176-222
//   piecewise_constant_pdf  nerf_sh/nerf/model_utils.py:225-286
//   sample_pdf              nerf_sh/nerf/model_utils.py:289-314
//   loss_fn (MSE part)      nerf_sh/train.py:86-96
#include "common.cuh"
#include "kernels.h"

namespace pob {

namespace {

constexpr int RAYS_PER_BLOCK = 4;
constexpr int MAX_SEG = 8;  // samples per lane
constexpr int WIDE = 4;     // warps per ray for N > 32 * MAX_SEG
static_assert(32 * MAX_SEG * WIDE == MAX_RAY_SAMPLES && WIDE == RAYS_PER_BLOCK, "a wide ray fills one block");
constexpr unsigned FULL = 0xffffffffu;

// the ray of this thread and its index among the ray's 32 * W threads
template <int W>
__device__ __forceinline__ long long ray_of_thread() {
  return blockIdx.x * (long long)(RAYS_PER_BLOCK / W) + (threadIdx.x >> 5) / W;
}
template <int W>
__device__ __forceinline__ int ray_thread() { return threadIdx.x & (32 * W - 1); }
template <int W>
__device__ __forceinline__ void ray_sync() {
  if constexpr (W == 1) __syncwarp(); else __syncthreads();
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}
// exclusive product scan across lanes
__device__ __forceinline__ float warp_excl_prod(float v, int lane) {
  float inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float t = __shfl_up_sync(FULL, inc, o);
    if (lane >= o) inc *= t;
  }
  float ex = __shfl_up_sync(FULL, inc, 1);
  return lane == 0 ? 1.f : ex;
}
// exclusive sum scan across lanes
__device__ __forceinline__ float warp_excl_sum(float v, int lane) {
  float inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float t = __shfl_up_sync(FULL, inc, o);
    if (lane >= o) inc += t;
  }
  float ex = __shfl_up_sync(FULL, inc, 1);
  return lane == 0 ? 0.f : ex;
}
// exclusive suffix sum across lanes (sum over lanes > me)
__device__ __forceinline__ float warp_excl_suffix_sum(float v, int lane) {
  float inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float t = __shfl_down_sync(FULL, inc, o);
    if (lane + o < 32) inc += t;
  }
  float ex = __shfl_down_sync(FULL, inc, 1);
  return lane == 31 ? 0.f : ex;
}

// Cross-warp steps of a W-warp ray (W > 1: one ray per block, warp wid of W).  Each warp's total is the combination
// of its last (prefix) or first (suffix) lane's exclusive scan with that lane's own value.  Every helper owns its
// shared array, so a kernel calls each of them at most once.
// exclusive product over the warps in front of mine, in warp order
template <int W>
__device__ __forceinline__ float warps_front_prod(float warp_total, int lane, int wid) {
  __shared__ float s_tot[W];
  if (lane == 0) s_tot[wid] = warp_total;
  __syncthreads();
  float p = 1.f;
  for (int k = 0; k < wid; ++k) p *= s_tot[k];
  return p;
}
// exclusive sum over the warps in front of mine (front = true, in warp order) or behind it (from the last warp back)
template <int W>
__device__ __forceinline__ float warps_excl_sum(float warp_total, int lane, int wid, bool front) {
  __shared__ float s_tot[W];
  if (lane == 0) s_tot[wid] = warp_total;
  __syncthreads();
  float s = 0.f;
  if (front)
    for (int k = 0; k < wid; ++k) s += s_tot[k];
  else
    for (int k = W - 1; k > wid; --k) s += s_tot[k];
  return s;
}
// sum over all W warps, in warp order, in every thread
template <int W>
__device__ __forceinline__ float warps_sum(float warp_total, int lane, int wid) {
  __shared__ float s_tot[W];
  if (lane == 0) s_tot[wid] = warp_total;
  __syncthreads();
  float s = s_tot[0];
  for (int k = 1; k < W; ++k) s += s_tot[k];
  return s;
}

// ---------------------------------------------------------------------------------------------
// Stratified sampling.  z_base[N] = near*(1-t)+far*t (or the lindisp form) is tabulated by the host
// with the reference's own expression so that no linspace rounding ambiguity enters.
// ---------------------------------------------------------------------------------------------
__global__ void sample_coarse_kernel(const float* __restrict__ z_base, const float* __restrict__ t_rand,
                                     int R, int N, float* __restrict__ z_out) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)R * N) return;
  const int j = int(i % N);
  float z = z_base[j];
  if (t_rand) {
    const float zl = j > 0 ? z_base[j - 1] : z, zu = j < N - 1 ? z_base[j + 1] : z;
    const float lower = j > 0 ? __fmul_rn(0.5f, __fadd_rn(z, zl)) : z;
    const float upper = j < N - 1 ? __fmul_rn(0.5f, __fadd_rn(zu, z)) : z;
    z = __fadd_rn(lower, __fmul_rn(__fsub_rn(upper, lower), t_rand[i]));
  }
  z_out[i] = z;
}

// ---------------------------------------------------------------------------------------------
// Per-ray recomputation shared by the forward and backward compositing kernels
// ---------------------------------------------------------------------------------------------
struct RaySeg {
  float4 c[MAX_SEG];   // (r,g,b,sigma) of my samples
  float z[MAX_SEG];
  float alpha[MAX_SEG], om[MAX_SEG], dist[MAX_SEG];
  float ex[MAX_SEG];   // exp(-sigma * dist): d alpha / d sigma = dist * ex (the backward's factor)
  float T0;            // transmittance in front of my first sample
};

template <int S, int W>
__device__ __forceinline__ void load_ray(const float4* __restrict__ rgbs, const float* __restrict__ z,
                                         const float* __restrict__ dirs, long long ray, int N, int lane,
                                         RaySeg& r) {
  const int seg = ray_thread<W>();
  const float dx = dirs[3 * ray], dy = dirs[3 * ray + 1], dz = dirs[3 * ray + 2];
  const float dnorm = sqrtf(dx * dx + dy * dy + dz * dz);
  float prod = 1.f;
#pragma unroll
  for (int i = 0; i < S; ++i) {
    const int idx = seg * S + i;
    if (idx < N) {
      r.c[i] = rgbs[ray * N + idx];
      r.z[i] = z[ray * N + idx];
      const float zn = (idx + 1 < N) ? z[ray * N + idx + 1] : 0.f;
      float d = (idx + 1 < N) ? __fsub_rn(zn, r.z[i]) : 1e10f;
      d = __fmul_rn(d, dnorm);
      r.dist[i] = d;
      r.ex[i] = expf(-r.c[i].w * d);
      r.alpha[i] = 1.0f - r.ex[i];
      r.om[i] = (1.0f - r.alpha[i]) + 1e-10f;
      prod *= r.om[i];
    } else {
      r.c[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      r.z[i] = 0.f;
      r.dist[i] = 0.f;
      r.ex[i] = 1.f;
      r.alpha[i] = 0.f;
      r.om[i] = 1.f;
    }
  }
  r.T0 = warp_excl_prod(prod, lane);
  if constexpr (W > 1) r.T0 *= warps_front_prod<W>(__shfl_sync(FULL, r.T0 * prod, 31), lane, threadIdx.x >> 5);
}

struct CompositeArgs {
  const float4* rgbs;
  const float* z;
  const float* dirs;
  int R, N, white_bkgd;
  float *out_rgb, *out_disp, *out_acc, *out_weights;
};

template <int S, int W>
__global__ void __launch_bounds__(RAYS_PER_BLOCK * 32)
composite_fwd_kernel(const CompositeArgs a) {
  const int lane = threadIdx.x & 31, seg = ray_thread<W>();
  const long long ray = ray_of_thread<W>();
  if (ray >= a.R) return;
  RaySeg r;
  load_ray<S, W>(a.rgbs, a.z, a.dirs, ray, a.N, lane, r);
  float T = r.T0, cr = 0.f, cg = 0.f, cb = 0.f, depth = 0.f, acc = 0.f;
#pragma unroll
  for (int i = 0; i < S; ++i) {
    const int idx = seg * S + i;
    const float w = r.alpha[i] * T;
    if (idx < a.N) {
      cr += w * r.c[i].x;
      cg += w * r.c[i].y;
      cb += w * r.c[i].z;
      depth += w * r.z[i];
      acc += w;
      if (a.out_weights) a.out_weights[ray * a.N + idx] = w;
    }
    T *= r.om[i];
  }
  cr = warp_sum(cr);
  cg = warp_sum(cg);
  cb = warp_sum(cb);
  depth = warp_sum(depth);
  acc = warp_sum(acc);
  if constexpr (W > 1) {   // the five sums over the W warps, in warp order
    __shared__ float s_part[5][W];
    const int wid = threadIdx.x >> 5;
    if (lane == 0) {
      s_part[0][wid] = cr;
      s_part[1][wid] = cg;
      s_part[2][wid] = cb;
      s_part[3][wid] = depth;
      s_part[4][wid] = acc;
    }
    __syncthreads();
    cr = s_part[0][0], cg = s_part[1][0], cb = s_part[2][0], depth = s_part[3][0], acc = s_part[4][0];
    for (int k = 1; k < W; ++k) {
      cr += s_part[0][k];
      cg += s_part[1][k];
      cb += s_part[2][k];
      depth += s_part[3][k];
      acc += s_part[4][k];
    }
  }
  if (seg == 0) {
    const float inv_eps = 1e10f;
    float disp = acc / depth;
    disp = (disp > 0.f && disp < inv_eps && acc > 1e-10f) ? disp : inv_eps;
    if (a.white_bkgd) {
      cr += 1.0f - acc;
      cg += 1.0f - acc;
      cb += 1.0f - acc;
    }
    a.out_rgb[3 * ray] = cr;
    a.out_rgb[3 * ray + 1] = cg;
    a.out_rgb[3 * ray + 2] = cb;
    if (a.out_disp) a.out_disp[ray] = disp;
    if (a.out_acc) a.out_acc[ray] = acc;
  }
}

// ---------------------------------------------------------------------------------------------
// Backward of compositing + MSE.  Emits, per sample, the gradient w.r.t. the PRE-activation head
// outputs after SH evaluation: (d pre_r, d pre_g, d pre_b, d sigma_raw), already multiplied by
// sigmoid' and relu' (or softplus') — mlp_bwd only has to expand it with the SH basis.
//   dL/dC = gscale * (C - px);   gscale = loss_scale * 2 / (3 * R_global_per_rank)
// ---------------------------------------------------------------------------------------------
struct CompositeBwdArgs {
  const float4* rgbs;
  const float* z;
  const float* dirs;
  const float* comp_rgb;   // [R,3] forward result
  const float* pixels;     // [R,3]
  int R, N, white_bkgd;
  float gscale;
  int sigma_act;           // SigmaAct of rgbs.w: the sigma factor of G.w is relu' = [sigma > 0] or softplus'
  float4* G;               // [R,N]
  float* sq_err_sum;       // += sum_{rays,ch} (C - px)^2   (loss numerator)
};

template <int S, int W>
__global__ void __launch_bounds__(RAYS_PER_BLOCK * 32)
composite_bwd_kernel(const CompositeBwdArgs a) {
  const int lane = threadIdx.x & 31, seg = ray_thread<W>();
  const long long ray = ray_of_thread<W>();
  if (ray >= a.R) return;
  RaySeg r;
  load_ray<S, W>(a.rgbs, a.z, a.dirs, ray, a.N, lane, r);
  const float ex = a.comp_rgb[3 * ray] - a.pixels[3 * ray];
  const float ey = a.comp_rgb[3 * ray + 1] - a.pixels[3 * ray + 1];
  const float ez = a.comp_rgb[3 * ray + 2] - a.pixels[3 * ray + 2];
  const float dcx = a.gscale * ex, dcy = a.gscale * ey, dcz = a.gscale * ez;
  const float bg = a.white_bkgd ? 1.f : 0.f;
  // pass 1: weights, g_i * w_i and its suffix sums
  float T = r.T0;
  float w[S], Tpre[S], gi[S];
  float local = 0.f;
#pragma unroll
  for (int i = 0; i < S; ++i) {
    Tpre[i] = T;
    w[i] = r.alpha[i] * T;
    gi[i] = dcx * (r.c[i].x - bg) + dcy * (r.c[i].y - bg) + dcz * (r.c[i].z - bg);
    local += gi[i] * w[i];
    T *= r.om[i];
  }
  float suffix = warp_excl_suffix_sum(local, lane);  // sum over lanes > me
  if constexpr (W > 1)                                // + sum over the warps behind mine
    suffix += warps_excl_sum<W>(__shfl_sync(FULL, suffix + local, 0), lane, threadIdx.x >> 5, false);
#pragma unroll
  for (int i = S - 1; i >= 0; --i) {
    const int idx = seg * S + i;
    if (idx < a.N) {
      // dL/dalpha_i = g_i T_i - (sum_{k>i} g_k w_k) / (1 - alpha_i + eps)
      const float dalpha = gi[i] * Tpre[i] - suffix / r.om[i];
      // d alpha / d sigma = dist * exp(-sigma dist), from exp's output as autograd forms it: the fp32 1 - alpha
      // carries an absolute error of ~2^-24, which is most of the factor once sigma * dist > ~10 and all of it
      // past ~16.7 (alpha rounds to 1)
      const float dsigma = dalpha * r.dist[i] * r.ex[i];
      float4 g;
      g.x = w[i] * dcx * r.c[i].x * (1.0f - r.c[i].x);
      g.y = w[i] * dcy * r.c[i].y * (1.0f - r.c[i].y);
      g.z = w[i] * dcz * r.c[i].z * (1.0f - r.c[i].z);
      // the activation's derivative at the (noised) raw sigma, from its output: softplus' = -expm1(-sigma)
      g.w = a.sigma_act == SIGMA_SOFTPLUS ? dsigma * softplus_grad_of_output(r.c[i].w) : (r.c[i].w > 0.f ? dsigma : 0.f);
      a.G[ray * a.N + idx] = g;
    }
    suffix += gi[i] * w[i];
  }
  if (seg == 0 && a.sq_err_sum) atomicAdd(a.sq_err_sum, ex * ex + ey * ey + ez * ez);
}

// ---------------------------------------------------------------------------------------------
// Hierarchical resampling: inverse-CDF sampling of Nf new depths from the interior coarse weights,
// then the sorted union with the Nc coarse depths.
// ---------------------------------------------------------------------------------------------
struct PdfArgs {
  const float* z_c;       // [R,Nc]
  const float* weights;   // [R,Nc]
  const float* u;         // [Nf] table (u_per_ray = 0) or [R,Nf]
  int u_per_ray;
  int R, Nc, Nf;
  float* z_out;           // [R, Nc+Nf]
};

// W = 1: one warp per ray, a 256-key union sort.  W = WIDE: one block per ray, bins / cdf / union buffer of 1024
// floats each, a block scan for the cdf and a 1024-key sort under __syncthreads.
template <int W>
__global__ void __launch_bounds__(RAYS_PER_BLOCK * 32) sample_pdf_kernel(const PdfArgs a) {
  constexpr int RB = RAYS_PER_BLOCK / W;   // rays per block
  constexpr int NK = 256 * W;              // sort keys per ray (a power of two >= Nc + Nf)
  constexpr int NT = 32 * W;               // threads per ray
  __shared__ float s_bins[RB][NK];
  __shared__ float s_cdf[RB][NK];
  __shared__ float s_sort[RB][NK];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, seg = ray_thread<W>();
  const long long ray = ray_of_thread<W>();
  if (ray >= a.R) return;
  const int Nc = a.Nc, Nf = a.Nf;
  const int nb = Nc - 1;   // bins (mid points): 63
  const int nw = Nc - 2;   // interior weights:   62
  float* bins = s_bins[wid / W];
  float* cdf = s_cdf[wid / W];
  float* sb = s_sort[wid / W];
  const float* zc = a.z_c + ray * Nc;
  const float* wt = a.weights + ray * Nc;
  for (int i = seg; i < nb; i += NT) bins[i] = __fmul_rn(0.5f, __fadd_rn(zc[i + 1], zc[i]));
  // weights[..., 1:-1], padded so that the sum is at least eps
  const int S = (nw + NT - 1) / NT;
  float wl[MAX_SEG];
  float lsum = 0.f;
#pragma unroll
  for (int i = 0; i < MAX_SEG; ++i) {
    const int idx = seg * S + i;
    wl[i] = (i < S && idx < nw) ? wt[idx + 1] : 0.f;
    lsum += wl[i];
  }
  float wsum = warp_sum(lsum);
  if constexpr (W > 1) wsum = warps_sum<W>(wsum, lane, wid);
  const float padding = fmaxf(0.f, 1e-5f - wsum);
  const float padw = padding / float(nw);
  wsum += padding;
  // pdf and inclusive cumsum over pdf[:-1]
  float run = 0.f;
#pragma unroll
  for (int i = 0; i < MAX_SEG; ++i) {
    const int idx = seg * S + i;
    if (i < S && idx < nw) {
      wl[i] = (wl[i] + padw) / wsum;
      run += wl[i];
    } else {
      wl[i] = 0.f;
    }
  }
  float pre = warp_excl_sum(run, lane);
  if constexpr (W > 1) pre += warps_excl_sum<W>(__shfl_sync(FULL, pre + run, 31), lane, wid, true);
#pragma unroll
  for (int i = 0; i < MAX_SEG; ++i) {
    const int idx = seg * S + i;
    if (i < S && idx < nw) {
      pre += wl[i];
      if (idx < nw - 1) cdf[idx + 1] = fminf(1.f, pre);
    }
  }
  if (seg == 0) {
    cdf[0] = 0.f;
    cdf[nb - 1] = 1.f;
  }
  ray_sync<W>();
  // union buffer: coarse depths first
  for (int i = seg; i < Nc; i += NT) sb[i] = zc[i];
  for (int j = seg; j < Nf; j += NT) {
    const float u = a.u_per_ray ? a.u[ray * Nf + j] : a.u[j];
    // count of cdf entries <= u (cdf is non-decreasing): upper bound
    int lo = 0, hi = nb;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (cdf[mid] <= u) lo = mid + 1; else hi = mid;
    }
    const int i0 = lo > 0 ? lo - 1 : 0;
    const int i1 = lo < nb ? lo : nb - 1;
    const float c0 = cdf[i0], c1 = cdf[i1];
    float t = __fdiv_rn(__fsub_rn(u, c0), __fsub_rn(c1, c0));
    if (t != t) t = 0.f;                      // nan_to_num
    t = fminf(fmaxf(t, 0.f), 1.f);            // +-inf clip like the reference
    const float b0 = bins[i0], b1 = bins[i1];
    sb[Nc + j] = __fadd_rn(b0, __fmul_rn(t, __fsub_rn(b1, b0)));
  }
  for (int i = Nc + Nf + seg; i < NK; i += NT) sb[i] = __int_as_float(0x7f800000);
  ray_sync<W>();
  // bitonic sort of NK keys, 4 compare-exchanges per thread per pass
  for (int k = 2; k <= NK; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int c = seg + NT * q;                // 0..NK/2-1: index of the compare-exchange
        const int i = ((c & ~(j - 1)) << 1) | (c & (j - 1));
        const int p = i | j;
        const bool up = (i & k) == 0;
        const float x = sb[i], y = sb[p];
        if ((x > y) == up) {
          sb[i] = y;
          sb[p] = x;
        }
      }
      ray_sync<W>();
    }
  }
  float* zo = a.z_out + ray * (long long)(Nc + Nf);
  for (int i = seg; i < Nc + Nf; i += NT) zo[i] = sb[i];
}

// sparsity-loss gradient (nerf_sh/train.py:77-83): G.w = coef * exp(-len * relu(s)) * [s > 0]; the forward
// epilogue has already applied the relu (rgbs.w)
__global__ void sparsity_grad_kernel(const float4* __restrict__ rgbs, int n, float length, float coef,
                                     float4* __restrict__ G, float* __restrict__ exp_sum) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float e = 0.f;
  if (i < n) {
    const float s = rgbs[i].w;
    e = expf(-length * s);
    G[i] = make_float4(0.f, 0.f, 0.f, s > 0.f ? coef * e : 0.f);
  }
  e = warp_sum(e);
  if ((threadIdx.x & 31) == 0 && exp_sum) atomicAdd(exp_sum, e);
}

// ---- random draws of one training step (stratified jitter, inverse-CDF uniforms, sparsity points) ----------------
// Philox4x32-10 (Salmon et al., SC'11), counter = (element / 4, stream id, step), key = seed: one launch replaces
// the seven ATen launches (3 x rand + scale / shift) of a step.  The reference draws from jax.random's threefry
// streams, which cannot be reproduced without JAX; parity tests inject their draws instead (SURVEY.md 7.2 RNG).
__global__ void draw_uniforms_kernel(unsigned long long seed, float step_host, const float* __restrict__ step_dev,
                                     float* __restrict__ t_rand, long long n_t, float* __restrict__ u, long long n_u,
                                     float* __restrict__ sp, long long n_sp, float sp_radius) {
  const uint32_t step = uint32_t(step_dev ? __ldg(step_dev) : step_host);
  const long long q4 = (n_t + 3) / 4, r4 = (n_u + 3) / 4, s4 = (n_sp + 3) / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < q4 + r4 + s4;
       i += (long long)gridDim.x * blockDim.x) {
    int stream = 0;
    long long j = i;
    float* dst = t_rand;
    long long n = n_t;
    if (j >= q4) { j -= q4; stream = 1; dst = u; n = n_u; }
    if (stream == 1 && j >= r4) { j -= r4; stream = 2; dst = sp; n = n_sp; }
    const uint4 r = philox4x32_10(make_uint4(uint32_t(j), uint32_t(j >> 32), uint32_t(stream), step),
                                  make_uint2(uint32_t(seed), uint32_t(seed >> 32)));
    float v[4] = {u01(r.x), u01(r.y), u01(r.z), u01(r.w)};
    if (stream == 2) {   // random.uniform(key, (npoints, 3), minval=-radius, maxval=radius)  (train.py:79)
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] = fmaf(v[k], 2.0f * sp_radius, -sp_radius);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (4 * j + k < n) dst[4 * j + k] = v[k];
  }
}

// warps per ray for N samples
int ray_warps(int N) { return N <= 32 * MAX_SEG ? 1 : WIDE; }

// f(S, W): W = ray_warps(N), S = ceil(N / (32 W)) samples per lane (3..8 when W = WIDE)
template <typename F>
cudaError_t dispatch_seg(int N, F&& f) {
  if (N < 1 || N > MAX_RAY_SAMPLES) return cudaErrorInvalidValue;
  using W1 = std::integral_constant<int, 1>;
  using W4 = std::integral_constant<int, WIDE>;
  switch (ray_warps(N) == 1 ? (N + 31) / 32 : (N + 32 * WIDE - 1) / (32 * WIDE) + MAX_SEG) {
    case 1: return f(std::integral_constant<int, 1>(), W1());
    case 2: return f(std::integral_constant<int, 2>(), W1());
    case 3: return f(std::integral_constant<int, 3>(), W1());
    case 4: return f(std::integral_constant<int, 4>(), W1());
    case 5: return f(std::integral_constant<int, 5>(), W1());
    case 6: return f(std::integral_constant<int, 6>(), W1());
    case 7: return f(std::integral_constant<int, 7>(), W1());
    case 8: return f(std::integral_constant<int, 8>(), W1());
    case MAX_SEG + 3: return f(std::integral_constant<int, 3>(), W4());
    case MAX_SEG + 4: return f(std::integral_constant<int, 4>(), W4());
    case MAX_SEG + 5: return f(std::integral_constant<int, 5>(), W4());
    case MAX_SEG + 6: return f(std::integral_constant<int, 6>(), W4());
    case MAX_SEG + 7: return f(std::integral_constant<int, 7>(), W4());
    case MAX_SEG + 8: return f(std::integral_constant<int, 8>(), W4());
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace

cudaError_t launch_sample_coarse(const float* z_base, const float* t_rand, int R, int N, float* z_out,
                                 cudaStream_t st) {
  const long long n = (long long)R * N;
  if (n == 0) return cudaSuccess;
  sample_coarse_kernel<<<unsigned((n + 255) / 256), 256, 0, st>>>(z_base, t_rand, R, N, z_out);
  return cudaGetLastError();
}

cudaError_t launch_composite_fwd(const float4* rgbs, const float* z, const float* dirs, int R, int N,
                                 int white_bkgd, float* out_rgb, float* out_disp, float* out_acc,
                                 float* out_weights, cudaStream_t st) {
  if (R == 0) return cudaSuccess;
  CompositeArgs a{rgbs, z, dirs, R, N, white_bkgd, out_rgb, out_disp, out_acc, out_weights};
  const int rb = RAYS_PER_BLOCK / ray_warps(N);
  const unsigned grid = (R + rb - 1) / rb;
  return dispatch_seg(N, [&](auto s, auto w) {
    composite_fwd_kernel<decltype(s)::value, decltype(w)::value><<<grid, RAYS_PER_BLOCK * 32, 0, st>>>(a);
    return cudaGetLastError();
  });
}

cudaError_t launch_composite_bwd(const float4* rgbs, const float* z, const float* dirs,
                                 const float* comp_rgb, const float* pixels, int R, int N, int white_bkgd,
                                 float gscale, int sigma_act, float4* G, float* sq_err_sum, cudaStream_t st) {
  if (R == 0) return cudaSuccess;
  if (sigma_act != SIGMA_RELU && sigma_act != SIGMA_SOFTPLUS) return cudaErrorInvalidValue;
  CompositeBwdArgs a{rgbs, z, dirs, comp_rgb, pixels, R, N, white_bkgd, gscale, sigma_act, G, sq_err_sum};
  const int rb = RAYS_PER_BLOCK / ray_warps(N);
  const unsigned grid = (R + rb - 1) / rb;
  return dispatch_seg(N, [&](auto s, auto w) {
    composite_bwd_kernel<decltype(s)::value, decltype(w)::value><<<grid, RAYS_PER_BLOCK * 32, 0, st>>>(a);
    return cudaGetLastError();
  });
}

cudaError_t launch_sample_pdf(const float* z_c, const float* weights, const float* u, int u_per_ray, int R,
                              int Nc, int Nf, float* z_out, cudaStream_t st) {
  if (R == 0) return cudaSuccess;
  if (Nc < 3 || Nf < 0 || Nc + Nf > MAX_RAY_SAMPLES) return cudaErrorInvalidValue;
  PdfArgs a{z_c, weights, u, u_per_ray, R, Nc, Nf, z_out};
  if (ray_warps(Nc + Nf) == 1)
    sample_pdf_kernel<1><<<(R + RAYS_PER_BLOCK - 1) / RAYS_PER_BLOCK, RAYS_PER_BLOCK * 32, 0, st>>>(a);
  else
    sample_pdf_kernel<WIDE><<<R, RAYS_PER_BLOCK * 32, 0, st>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_draw_uniforms(unsigned long long seed, float step, const float* step_dev, float* t_rand,
                                 long long n_t, float* u, long long n_u, float* sp, long long n_sp, float sp_radius,
                                 cudaStream_t st) {
  const long long work = (n_t + 3) / 4 + (n_u + 3) / 4 + (n_sp + 3) / 4;
  if (work == 0) return cudaSuccess;
  const int grid = int((work + 255) / 256 < 2048 ? (work + 255) / 256 : 2048);
  draw_uniforms_kernel<<<grid, 256, 0, st>>>(seed, step, step_dev, t_rand, n_t, u, n_u, sp, n_sp, sp_radius);
  return cudaGetLastError();
}

cudaError_t launch_sparsity_grad(const float4* rgbs, int n, float length, float coef, float4* G,
                                 float* exp_sum, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  sparsity_grad_kernel<<<(n + 255) / 256, 256, 0, st>>>(rgbs, n, length, coef, G, exp_sum);
  return cudaGetLastError();
}

}  // namespace pob
