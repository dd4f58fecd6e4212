// optim.cu — gradient finalisation and the optimiser step.
//   reduce_grads : per-CTA wgrad partials -> flat fp32 gradient in reference parameter order
//   adam         : flax.optim.Adam.apply_gradient (nerf_sh/train.py:119, models.py:44)
#include <cstring>

#include "common.cuh"
#include "kernels.h"

namespace pob {

// Work split of the wgrad launch.  The units are the two row halves of each of Dense_1..7 and the transposed
// Dense_0 and heads roles (kernels.h: WgradRole).  A unit's cost is the bytes it streams per 128-sample tile: 96 KB
// for a row half (32 KB of dZ_l, 64 KB of h_{l-1}), 112 KB for Dense_5's (+ the posenc tile), 80 KB for Dense_0 and
// the SH16 heads (16 KB of posenc / dO, 64 KB of dZ_0 / h_7), 96 KB for the SH25 heads.  CTAs go one at a time to
// the unit with the most cost per CTA (the halves of a role in pairs), so that the units finish together.  CTA
// index i of a halved role computes result rows [128 (i & 1), +128) over the tiles i / 2, i / 2 + count / 2, ...;
// CTA i of a transposed role the tiles i, i + count, ...
int wgrad_assign_roles(WgradParams& p, int n_in, int role_start[WG_NUM_ROLES],
                       int role_count[WG_NUM_ROLES]) {
  int n = n_in < WG_MAX_CTAS ? n_in : WG_MAX_CTAS;
  int units = 0;
  for (int r = 0; r < WG_NUM_ROLES; ++r) units += wgrad_role(r).halves;
  if (n < units) n = units;   // one CTA per unit at the very least
  int cost[WG_NUM_ROLES], per_unit[WG_NUM_ROLES];
  for (int r = 0; r < WG_NUM_ROLES; ++r) {
    const WgradRole R = wgrad_role(r);
    const int a_kb = R.halves == 2 ? 32 : (wgrad_split_k(R, p.NH) ? 16 : 32);
    cost[r] = a_kb + 64 + (R.skip ? 16 : 0);
    per_unit[r] = 1;
  }
  for (int left = n - units;;) {
    int best = -1;
    for (int r = 0; r < WG_NUM_ROLES; ++r) {   // cost[r] / per_unit[r] largest; ties: the first
      if (wgrad_role(r).halves > left) continue;
      if (best < 0 || cost[r] * per_unit[best] > cost[best] * per_unit[r]) best = r;
    }
    if (best < 0) break;
    ++per_unit[best];
    left -= wgrad_role(best).halves;
  }
  int cta = 0;
  for (int r = 0; r < WG_NUM_ROLES; ++r) {
    const int c = per_unit[r] * wgrad_role(r).halves;
    role_start[r] = cta;
    role_count[r] = c;
    for (int i = 0; i < c; ++i, ++cta) {
      p.cta_role[cta] = short(r);
      p.cta_index[cta] = short(i);
      p.cta_count[cta] = short(c);
    }
  }
  for (int i = cta; i < WG_MAX_CTAS; ++i) {   // spare CTAs idle (role -1)
    p.cta_role[i] = -1;
    p.cta_index[i] = 0;
    p.cta_count[i] = 2;
  }
  return cta;
}

namespace {

struct ReduceArgs {
  WgradPass pass[X3_WGRAD_PASSES];
  int npass;
  FlatLayout L;
  int K, NH;
  float inv_scale;
  float* grad;
};

// Where element (layer, in i, out o) of a kernel, or (layer, out o) of a bias, lies in its role's partials
// (kernels.h: WgradRole): offset `off`, plus `off2` >= 0 for the second warpgroup's rows of a split-K role; `row_half`
// = the result row half of a halved role (its CTAs with index & 1 == half), -1 for a transposed role (all its CTAs).
struct Loc {
  int role, off, off2, row_half;
};
__device__ __forceinline__ Loc locate(const ReduceArgs& a, int layer, int i, int o, bool is_bias) {
  Loc l;
  l.role = wgrad_role_of(layer);
  const WgradRole R = wgrad_role(l.role);
  l.off2 = -1;
  if (R.halves == 2) {     // D[out feature][in feature]
    l.row_half = o >> 7;
    l.off = is_bias ? 65536 + o
          : i < WIDTH ? o * WIDTH + i
                      : (l.row_half ? 0 : 32768) + (o & 127) * 64 + (i - WIDTH);   // Dense_5's skip rows
  } else {                 // transposed: D[A feature][B feature], A = posenc (Dense_0) or packed heads column
    l.row_half = -1;
    const int r = layer == 0 ? i : layer == 8 ? 0 : heads_column_of_output(o, a.K);
    const int col = layer == 0 ? o : i;
    l.off = is_bias ? 65536 + (layer == 0 ? o : r) : r * WIDTH + col;
    if (!is_bias && wgrad_split_k(R, a.NH)) l.off2 = l.off + 64 * WIDTH;
  }
  return l;
}

// sum over the passes and, in each, over the role's CTAs that computed the element, in CTA order
__device__ __forceinline__ float sum_partials(const ReduceArgs& a, const Loc& l, int npass) {
  float s = 0.f;
  const int step = l.row_half < 0 ? 1 : 2;
  for (int q = 0; q < npass; ++q) {
    const WgradPass& g = a.pass[q];
    const float* p = g.partials + size_t(g.role_start[l.role]) * WG_PARTIAL_FLOATS;
    for (int c = l.row_half < 0 ? 0 : l.row_half; c < g.role_count[l.role]; c += step) {
      s += p[size_t(c) * WG_PARTIAL_FLOATS + l.off];
      if (l.off2 >= 0) s += p[size_t(c) * WG_PARTIAL_FLOATS + l.off2];
    }
  }
  return s;
}

// grid (in tiles of 32, out tiles of 32, 10 layers + 1 bias slice), block (32, 8).  The partials of Dense_1..9 are
// [out][in] (accumulator row = out feature or packed heads column) and the flat gradient is flax's kernel [in][out]:
// every 32x32 tile is read along `in` (coalesced in the partials), summed over the role's CTAs, transposed through
// shared memory and written along `out` (coalesced in the gradient).  Dense_0's partials are [in][out].  (A
// one-thread-per-gradient-element version read with a 1 KB stride: 64 us per step instead of ~15.)
__global__ void reduce_grads_kernel(const __grid_constant__ ReduceArgs a) {
  __shared__ float tile[32][33];
  const int layer = blockIdx.z;
  if (layer == 10) {                      // biases: block x = layer, one thread per output
    const int l = blockIdx.x, o = threadIdx.y * 32 + threadIdx.x;
    if (blockIdx.y != 0 || l >= 10 || o >= a.L.out_dim[l]) return;
    a.grad[a.L.b_off[l] + o] =
        sum_partials(a, locate(a, l, 0, o, true), min(a.npass, X3_BIAS_PASSES)) * a.inv_scale;
    return;
  }
  const int in_dim = a.L.in_dim[layer], out_dim = a.L.out_dim[layer];
  const int i0 = blockIdx.x * 32, o0 = blockIdx.y * 32;
  if (i0 >= in_dim || o0 >= out_dim) return;
  const bool in_major = layer == 0;      // Dense_0's partials are [in][out]: read along `out` instead
  for (int k = threadIdx.y; k < 32; k += 8) {
    const int i = in_major ? i0 + k : i0 + threadIdx.x;
    const int o = in_major ? o0 + threadIdx.x : o0 + k;
    float v = 0.f;
    if (i < in_dim && o < out_dim) v = sum_partials(a, locate(a, layer, i, o, false), a.npass);
    if (in_major) tile[k][threadIdx.x] = v;   // tile[i - i0][o - o0]
    else tile[threadIdx.x][k] = v;
  }
  __syncthreads();
  for (int k = threadIdx.y; k < 32; k += 8) {
    const int i = i0 + k, o = o0 + threadIdx.x;
    if (i < in_dim && o < out_dim) a.grad[a.L.w_off[layer] + i * out_dim + o] = tile[k][threadIdx.x] * a.inv_scale;
  }
}

// lr / step come from the launch arguments or, when lr_step is given, from device memory (replayable CUDA graphs);
// the bias corrections 1 - beta^t are formed in the kernel either way (-expm1f(t log beta): accurate for small t
// where 1 - powf(beta, t) cancels), so that an eager step and a graph-replayed one are bit-identical
__global__ void adam_kernel(float* __restrict__ param, const float* __restrict__ grad, float* __restrict__ m,
                            float* __restrict__ v, long long n, float lr, float step,
                            const float* __restrict__ lr_step, float beta1, float beta2, float eps, float grad_mult,
                            float wd) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (lr_step) {
    lr = __ldg(lr_step);
    step = __ldg(lr_step + 1);
  }
  const float t = step + 1.0f;
  const float bc1 = -expm1f(t * logf(beta1));
  const float bc2 = -expm1f(t * logf(beta2));
  const float p = param[i];
  const float g = grad[i] * grad_mult + wd * p;
  const float mi = (1.0f - beta1) * g + beta1 * m[i];
  const float vi = (1.0f - beta2) * g * g + beta2 * v[i];
  m[i] = mi;
  v[i] = vi;
  const float mh = mi / bc1, vh = vi / bc2;
  param[i] = p - lr * mh / (sqrtf(vh) + eps);
}

}  // namespace

cudaError_t launch_reduce_grads(const WgradPass* passes, int npass, int K, int W, float inv_scale, float* grad_flat,
                                cudaStream_t stream) {
  if (npass < 1 || npass > X3_WGRAD_PASSES) return cudaErrorInvalidValue;
  ReduceArgs a;
  memset(&a, 0, sizeof(a));
  for (int q = 0; q < npass; ++q) a.pass[q] = passes[q];
  a.npass = npass;
  a.L = flat_layout(K, W);   // Dense_0 / Dense_5 rows i < W (+ 256) only: the zero posenc columns are dropped
  a.K = K;
  a.NH = heads_width(K);
  a.inv_scale = inv_scale;
  a.grad = grad_flat;
  reduce_grads_kernel<<<dim3(10, 8, 11), dim3(32, 8), 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_adam(float* param, const float* grad, float* m, float* v, long long n, float lr,
                        float step, const float* lr_step_dev, float beta1, float beta2, float eps, float grad_mult,
                        float weight_decay_coef, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  adam_kernel<<<unsigned((n + 255) / 256), 256, 0, stream>>>(param, grad, m, v, n, lr, step, lr_step_dev, beta1,
                                                              beta2, eps, grad_mult, weight_decay_coef);
  return cudaGetLastError();
}

}  // namespace pob
