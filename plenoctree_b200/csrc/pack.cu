// pack.cu — flat fp32 parameters (reference order) -> tensor-core operand images.
//
// Flat layout of one MLP (matches the flax pytree MLP_i/Dense_0..Dense_9, kernels [in,out];
// octree/nerf/models.py:75-102 documents the Dense index <-> layer mapping):
//   Dense_0 Wx256, Dense_1..4 256x256, Dense_5 (256+W)x256 ([h4 | posenc] rows), Dense_6..7,
//   Dense_8 256x1 (sigma), Dense_9 256x3K (rgb / SH coefficients, channel-major c*K+k);
//   W = 3 + 6 (max_deg - min_deg) is the posenc width (63 by default).
//
// Forward images  (w_hi / w_lo): sequence of K-major SW64 slots [rows = out feature][32 k],
//   in the order mlp_fwd consumes them.  Heads rows are re-ordered to [sigma, (k, c) ...] so the
//   epilogue can index the SH basis with compile-time constants.
// Backward images (wt_hi): the transposed weights, slots [rows = in feature][32 out features],
//   in the order mlp_bwd consumes them (heads, then Dense_7 .. Dense_1).  Their fp16 residual (wt_lo, same layout)
//   is not part of the blob: the x3 training step writes it into its workspace (launch_pack_wt_lo).
#include "common.cuh"
#include "kernels.h"

namespace pob {

namespace {

struct PackArgs {
  const float* flat;
  FlatLayout L;
  int K, NH, W;
  uint8_t *w_hi, *w_lo, *wt_hi, *wt_lo;
  int dgrad_only;   // write the dgrad slots only (the forward images are left alone)
};

// fp16 hi part and residual of v; either destination may be null
__device__ __forceinline__ void put_hilo(uint8_t* hi, uint8_t* lo, size_t off, float v) {
  __half h = __float2half_rn(v);
  if (hi) *reinterpret_cast<__half*>(hi + off) = h;
  if (lo) *reinterpret_cast<__half*>(lo + off) = __float2half_rn(v - __half2float(h));
}

// heads: the parameter of packed output column n, at flat offset off8 for Dense_8 (sigma) and off9 + (Dense_9 output)
// for the SH coefficients; 0 in the padding columns
__device__ __forceinline__ float heads_param(const PackArgs& a, int off8, int off9, int n) {
  if (n == 0) return a.flat[off8];
  int k, c;
  heads_coeff(n, k, c);
  return k < a.K ? a.flat[off9 + c * a.K + k] : 0.f;
}
// W[in=i -> packed column n]
__device__ __forceinline__ float heads_weight(const PackArgs& a, int i, int n) {
  return heads_param(a, a.L.w_off[8] + i, a.L.w_off[9] + i * (3 * a.K), n);
}

__global__ void pack_weights_kernel(const __grid_constant__ PackArgs a) {
  const int NH = a.NH;
  const long long n_fwd_trunk = (long long)FWD_TRUNK_SLOTS * 256 * 32;
  const long long n_fwd_heads = (long long)FWD_HEAD_SLOTS * NH * 32;
  const int hs = bwd_head_slots(NH);
  const long long n_bwd = (long long)bwd_slots(NH) * 256 * 32;
  const long long total = n_fwd_trunk + n_fwd_heads + n_bwd;
  const long long first = a.dgrad_only ? n_fwd_trunk + n_fwd_heads : 0;
  for (long long t = first + blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    if (t < n_fwd_trunk) {
      const int slot = int(t / (256 * 32));
      const int n = int(t / 32) % 256, kk = int(t % 32);
      // slot -> (layer, j)
      int l = 0, j = slot;
      while (j >= fwd_slots_of_layer(l)) {
        j -= fwd_slots_of_layer(l);
        ++l;
      }
      const int kin = 32 * j + kk;  // input feature index in the layer's [in] axis
      float v = 0.f;
      if (fwd_has_bias_slot(l)) {
        if (j < 8) v = a.flat[a.L.w_off[l] + kin * 256 + n];
        else if (kk == 31) v = a.flat[a.L.b_off[l] + n];       // bias slot: k = 31 <-> posenc column 63 (= 1)
      } else {
        // layers 0 / 5: posenc column pc = kin (minus h4's 256 rows in layer 5) holds Dense row (256 +) pc for
        // pc < W, 0 for pc in [W, 63), and the bias at pc = 63 (the constant-one column)
        const int pc = l == SKIP_LAYER ? kin - WIDTH : kin;
        if (pc < a.W) v = a.flat[a.L.w_off[l] + kin * 256 + n];
        else if (pc == ENC_PAD - 1) v = a.flat[a.L.b_off[l] + n];
      }
      put_hilo(a.w_hi, a.w_lo, size_t(slot) * WSLOT_BYTES + w_slot_offset(n, kk), v);
    } else if (t < n_fwd_trunk + n_fwd_heads) {
      const long long u = t - n_fwd_trunk;
      const int j = int(u / (NH * 32));
      const int n = int(u / 32) % NH, kk = int(u % 32);
      float v = 0.f;
      if (j < 8) v = heads_weight(a, 32 * j + kk, n);
      else if (kk == 31) v = heads_param(a, a.L.b_off[8], a.L.b_off[9], n);   // bias slot
      put_hilo(a.w_hi, a.w_lo, size_t(FWD_TRUNK_SLOTS) * WSLOT_BYTES + size_t(j) * NH * 64 + w_slot_offset(n, kk), v);
    } else {
      const long long u = t - n_fwd_trunk - n_fwd_heads;
      const int slot = int(u / (256 * 32));
      const int i = int(u / 32) % 256, kk = int(u % 32);  // i = in feature (row), kk = out feature
      float v = 0.f;
      if (slot < hs) {
        const int n = 32 * slot + kk;
        if (n < NH) v = heads_weight(a, i, n);
      } else {
        const int l = 7 - (slot - hs) / 8;  // Dense_7 .. Dense_1
        const int ko = 32 * ((slot - hs) % 8) + kk;
        v = a.flat[a.L.w_off[l] + i * 256 + ko];
      }
      put_hilo(a.wt_hi, a.wt_lo, size_t(slot) * WSLOT_BYTES + w_slot_offset(i, kk), v);
    }
  }
}

cudaError_t launch_pack(const float* flat, int K, int W, uint8_t* w_hi, uint8_t* w_lo, uint8_t* wt_hi,
                        uint8_t* wt_lo, int dgrad_only, cudaStream_t stream) {
  PackArgs a;
  a.flat = flat;
  a.L = flat_layout(K, W);
  a.K = K;
  a.W = W;
  a.NH = heads_width(K);
  a.w_hi = w_hi;
  a.w_lo = w_lo;
  a.wt_hi = wt_hi;
  a.wt_lo = wt_lo;
  a.dgrad_only = dgrad_only;
  pack_weights_kernel<<<592, 256, 0, stream>>>(a);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_pack_weights(const float* flat, int K, int W, uint8_t* w_hi, uint8_t* w_lo,
                                uint8_t* wt_hi, cudaStream_t stream) {
  return launch_pack(flat, K, W, w_hi, w_lo, wt_hi, nullptr, 0, stream);
}

cudaError_t launch_pack_wt_lo(const float* flat, int K, int W, uint8_t* wt_lo, cudaStream_t stream) {
  return launch_pack(flat, K, W, nullptr, nullptr, nullptr, wt_lo, 1, stream);
}

}  // namespace pob
