// optim.cu — gradient finalisation and the optimiser step.
//   reduce_grads : per-CTA wgrad partials -> flat fp32 gradient in reference parameter order
//   adam         : flax.optim.Adam.apply_gradient (nerf_sh/train.py:119, models.py:44)
#include "common.cuh"
#include "kernels.h"

namespace pob {

// Work split of the wgrad launch.  The kernel is bound by the tile bytes each role streams
// (96 KB per tile and row half for the 256x256 layers, ~40-64 KB for Dense_0 / the skip rows / the heads).  Every
// role gets an even number of CTAs: CTA index i of a role computes result rows [128 (i & 1), +128) over the tiles
// i / 2, i / 2 + count / 2, ...
int wgrad_assign_roles(WgradParams& p, int n_in, int role_start[WG_NUM_ROLES],
                       int role_count[WG_NUM_ROLES]) {
  int n = n_in < WG_MAX_CTAS ? n_in : WG_MAX_CTAS;
  if (n < 2 * WG_NUM_ROLES) n = 2 * WG_NUM_ROLES;  // one CTA per role and row half at the very least
  auto even = [](int x) { return x < 2 ? 2 : x & ~1; };
  int small = even((n * 8) / 100);         // per small role
  const int big = even((n - 3 * small) / 7);
  small = even((n - 7 * big) / 3);
  int cta = 0;
  for (int r = 0; r < WG_NUM_ROLES; ++r) {
    const int c = wgrad_role(r).width == 256 ? big : small;
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
  const float* partials;
  int role_start[WG_NUM_ROLES], role_count[WG_NUM_ROLES];
  FlatLayout L;
  int K, NH;
  float inv_scale;
  float* grad;
};

// role and offset inside a role's partial of element (layer, in i, out o) of a kernel, or (layer, out o) of a bias
__device__ __forceinline__ void locate(const ReduceArgs& a, int layer, int i, int o, bool is_bias, int& role, int& off) {
  role = wgrad_role_of(layer, i);
  const WgradRole R = wgrad_role(role);
  if (R.a_op == WG_H) {    // heads: D[in feature][packed column]
    const int n = layer == 8 ? 0 : heads_column_of_output(o, a.K);
    off = is_bias ? 65536 + n : i * a.NH + n;
  } else {                 // D[out feature][in feature - in0]
    off = is_bias ? 65536 + o : o * R.width + (i - R.in0);
  }
}

// sum over the role's CTAs that computed the element: those of its result row half (a bias taken from B, the heads'
// column sum of dO, comes from row half 0)
__device__ __forceinline__ float sum_partials(const ReduceArgs& a, int role, int off) {
  const WgradRole R = wgrad_role(role);
  const int pitch = wgrad_role_width(R, a.NH);
  const int row = off < 65536 ? off / pitch : (R.bias == WG_BIAS_B ? 0 : off - 65536);
  float s = 0.f;
  const float* p = a.partials + size_t(a.role_start[role]) * WG_PARTIAL_FLOATS + off;
  for (int c = row >> 7; c < a.role_count[role]; c += 2) s += p[size_t(c) * WG_PARTIAL_FLOATS];
  return s;
}

// grid (in tiles of 32, out tiles of 32, 10 layers + 1 bias slice), block (32, 8).  The trunk partials are
// [out][in] (accumulator row = out feature) and the flat gradient is flax's kernel [in][out]: every 32x32 tile is read
// along `in` (coalesced in the partials), summed over the role's CTAs, transposed through shared memory and written
// along `out` (coalesced in the gradient).  (A one-thread-per-gradient-element version read with a 1 KB stride:
// 64 us per step instead of ~15.)
__global__ void reduce_grads_kernel(const __grid_constant__ ReduceArgs a) {
  __shared__ float tile[32][33];
  const int layer = blockIdx.z;
  if (layer == 10) {                      // biases: block x = layer, one thread per output
    const int l = blockIdx.x, o = threadIdx.y * 32 + threadIdx.x;
    if (blockIdx.y != 0 || l >= 10 || o >= a.L.out_dim[l]) return;
    int role, off;
    locate(a, l, 0, o, true, role, off);
    a.grad[a.L.b_off[l] + o] = sum_partials(a, role, off) * a.inv_scale;
    return;
  }
  const int in_dim = a.L.in_dim[layer], out_dim = a.L.out_dim[layer];
  const int i0 = blockIdx.x * 32, o0 = blockIdx.y * 32;
  if (i0 >= in_dim || o0 >= out_dim) return;
  const bool heads = layer >= 8;          // heads partials are [in][out]: read along `out` instead
  for (int k = threadIdx.y; k < 32; k += 8) {
    const int i = heads ? i0 + k : i0 + threadIdx.x;
    const int o = heads ? o0 + threadIdx.x : o0 + k;
    float v = 0.f;
    if (i < in_dim && o < out_dim) {
      int role, off;
      locate(a, layer, i, o, false, role, off);
      v = sum_partials(a, role, off);
    }
    if (heads) tile[k][threadIdx.x] = v;   // tile[i - i0][o - o0]
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

cudaError_t launch_reduce_grads(const float* partials, const int role_start[WG_NUM_ROLES],
                                const int role_count[WG_NUM_ROLES], int K, float inv_scale,
                                float* grad_flat, cudaStream_t stream) {
  ReduceArgs a;
  a.partials = partials;
  for (int r = 0; r < WG_NUM_ROLES; ++r) {
    a.role_start[r] = role_start[r];
    a.role_count[r] = role_count[r];
  }
  a.L = flat_layout(K);
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
