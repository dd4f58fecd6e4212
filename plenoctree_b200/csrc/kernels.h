// kernels.h — internal launch interface between the C-ABI (capi.cu) and the kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace pob {

// ---- packed weights of one MLP (device pointers; produced by launch_pack_weights) ----------
// The biases ride inside the forward slots (common.cuh); the dgrad needs none.
struct MlpPacked {
  const uint8_t* w_hi;    // forward slot images, fp16 "hi" part  (fwd_image_bytes(NH))
  const uint8_t* w_lo;    // forward slot images, fp16 residual   (same layout)
  const uint8_t* wt_hi;   // dgrad slot images (transposed weights), fp16
};

enum SrcMode : int { SRC_POINTS = 0, SRC_RAYS = 1, SRC_GRID = 2 };
// OUT_VANILLA: the vanilla NeRF view branch behind the VANILLA_NH-wide heads (fp16, inference only)
enum OutMode : int { OUT_RAW = 0, OUT_SIGMA = 1, OUT_RGBS = 2, OUT_CELL_MEAN = 3, OUT_VANILLA = 4 };
// density activation of OUT_RGBS (the values of POB_SIGMA_* in the C ABI)
enum SigmaAct : int { SIGMA_RELU = 0, SIGMA_SOFTPLUS = 1 };

// samples per ray the per-ray stages (render.cu) take: 3 <= Nc and Nc + Nf <= MAX_RAY_SAMPLES
constexpr int MAX_RAY_SAMPLES = 1024;

// softplus in fp32, stable for every x: max(x, 0) + log1p(exp(-|x|)).  expf (2 ulp) and log1pf (1 ulp) and the
// final add keep it within 4 * 2^-24 * softplus(x) of the exact value of the fp32 argument, down to where expf's
// output turns denormal (x < -87); DESIGN.md section 3 gives the measured figure.
__device__ __forceinline__ float softplus_f32(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }
// its derivative from its own output: d softplus / dx = sigmoid(x) = 1 - exp(-softplus(x)) = -expm1(-sigma)
__device__ __forceinline__ float softplus_grad_of_output(float sigma) { return -expm1f(-sigma); }

// Trunk activation (flag net_activation, model_utils.py:69; the values of POB_NET_* in the C ABI), applied after
// every Dense_0..Dense_7.  Each one is 1-Lipschitz and its derivative is a function of its output h, so the data
// gradient forms dZ_l = dH_l * f'(h_l) from the h_l tiles the saving forward stores for the weight gradient; only relu
// needs the mask words.  fp32 forms: expm1f (1 ulp), softplus_f32 (above), tanhf (2 ulp): each within
// 4 * 2^-24 * |f(z)| of f at the fp32 argument z.
enum NetAct : int { NET_RELU = 0, NET_ELU = 1, NET_SOFTPLUS = 2, NET_TANH = 3 };
constexpr int NET_ACT_COUNT = 4;
template <int ACT>
__device__ __forceinline__ float net_act_f32(float z) {
  if constexpr (ACT == NET_ELU) return z > 0.f ? z : expm1f(z);
  else if constexpr (ACT == NET_SOFTPLUS) return softplus_f32(z);
  else if constexpr (ACT == NET_TANH) return tanhf(z);
  else return fmaxf(z, 0.f);
}
// f'(z) as a function of h = f(z): elu 1 | h + 1 (= exp(z) for z <= 0), softplus -expm1(-h), tanh (1 - h)(1 + h)
template <int ACT>
__device__ __forceinline__ float net_act_grad_of_output(float h) {
  if constexpr (ACT == NET_ELU) return h > 0.f ? 1.f : h + 1.f;
  else if constexpr (ACT == NET_SOFTPLUS) return softplus_grad_of_output(h);
  else if constexpr (ACT == NET_TANH) return (1.f - h) * (1.f + h);
  else return h > 0.f ? 1.f : 0.f;
}

// The point encoder posenc(x, min_deg, max_deg, legacy) (model_utils.py:145-173; flags min_deg_point, max_deg_point,
// legacy_posenc_order).  Its W = 3 + 6 (max_deg - min_deg) features fill posenc tile columns [0, W); columns [W, 63)
// are 0 and column 63 is the constant 1 that carries the biases.  0 <= min_deg <= max_deg <= POSENC_MAX_DEG keeps
// W <= 63 and the top scale 2^(max_deg - 1) inside posenc_sin's range (common.cuh).
constexpr int POSENC_MAX_DEG = 10;
struct PosencDesc {
  int min_deg, max_deg, legacy;
};
constexpr PosencDesc POSENC_DEFAULT = {0, 10, 0};   // the reference default: W = 63 = ENC_DIM
__host__ __device__ constexpr int posenc_width(PosencDesc pe) { return 3 + 6 * (pe.max_deg - pe.min_deg); }
inline bool posenc_valid(PosencDesc pe) {
  return pe.min_deg >= 0 && pe.min_deg <= pe.max_deg && pe.max_deg <= POSENC_MAX_DEG &&
         (pe.legacy == 0 || pe.legacy == 1);
}
// The network beyond sh_deg (the C ABI's pob_posenc): the point encoder and the trunk activation.
struct NetDesc {
  PosencDesc pe;
  int net_act;   // NetAct
};
inline bool net_act_valid(int a) { return a >= 0 && a < NET_ACT_COUNT; }

struct FwdParams {
  // ---- sample source ----
  int src_mode;
  long long M;                 // number of samples (rows)
  const float* points;         // SRC_POINTS: [M,3]
  const float* origins;        // SRC_RAYS:   [R,3]
  const float* directions;     //             [R,3]
  const float* zvals;          //             [R, n_per_ray]
  int n_per_ray;
  // SRC_RAYS may carry `M - M_rays` free points behind the ray samples (the sparsity-loss points of the training
  // step ride on the main level's launches instead of three 40-CTA launches of their own): rows [M_rays, M)
  long long M_rays;            // SRC_RAYS: R * n_per_ray (== M when there are no extra points)
  const float* extra_points;   // [M - M_rays, 3]
  const float* viewdirs;       // OUT_RGBS: [R,3] (SRC_RAYS) or [M,3] (SRC_POINTS)
  const float* sigma_noise;    // OUT_RGBS, optional [M]: added to raw sigma before relu (model_utils.py:317-332)
  int sigma_act;               // OUT_RGBS: SIGMA_RELU / SIGMA_SOFTPLUS of the ray (or SRC_POINTS) rows; free rows: relu
  // SRC_GRID: voxel centres ((i + 0.5)/reso - offset)/scale, x-major flattening (ix,iy,iz)
  int g_reso;                  // arange length the reference normalises by
  int g_x0, g_nx, g_ny, g_nz;  // slab: ix in [g_x0, g_x0+g_nx), iy in [0,g_ny), iz in [0,g_nz)
  float g_offset[3], g_scale[3];
  // ---- model ----
  MlpPacked w;
  PosencDesc pe;               // point encoder of the model (the packed Dense_0 / Dense_5 rows follow it)
  int sh_deg;                  // -1: 3 raw rgb channels, K = 1
  int K;                       // (sh_deg+1)^2
  int NH;                      // padded heads width, multiple of 16, <= 80
  // ---- outputs ----
  int out_mode;
  float* out_rgb;              // OUT_RAW: [M, 3K] (reference channel-major order c*K+k)
  float* out_sigma;            // OUT_RAW / OUT_SIGMA: [M]
  float4* out_rgbs;            // OUT_RGBS: [M] (sigmoid(rgb), relu(sigma) or softplus(sigma))
  float* out_cell;             // OUT_CELL_MEAN: [M / cell_S, 3K+1] += mean over the cell's samples of
  int cell_S;                  //   cat([raw_rgb, raw_sigma]) (octree/extraction.py:391-393); zeroed by caller
  // ---- training saves (null = off; x3 also needs save_h_lo / save_e_lo) ----
  uint8_t* save_h;             // [ntile][8][64 KB] activation tile images h_0..h_7
  uint8_t* save_e;             // [ntile][16 KB]   posenc tile images
  uint32_t* save_mask;         // [8][ntile*128][8] relu masks (common.cuh: mask_bit); left unwritten by other pe.net_act
  // ---- x3 training saves (NSPLIT = 3): the residual (lo) images beside save_h / save_e ----
  uint8_t* save_h_lo;          // [ntile][8][64 KB]
  uint8_t* save_e_lo;          // [ntile][16 KB]
  // ---- model, continued ----
  int net_act;                 // NetAct of Dense_0..Dense_7
  // ---- OUT_VANILLA: raw_rgb = W11 act(a_p + t_r) + b11 with a_p = heads columns VIEW_COL0.. (act = net_act) ----
  const float* view_t;         // [rows][VIEW_H] fp32: row s / n_per_ray (SRC_RAYS) or s (SRC_POINTS)
  const float* view_w11;       // [VIEW_H][3] (Dense_11 kernel)
  const float* view_b11;       // [3]
  // out_rgbs set: (sigmoid(raw_rgb), density activation of raw sigma (+ noise)); else out_rgb [M,3] and out_sigma [M]
  // take raw_rgb and raw sigma
};

// sh_deg -1 (3 raw rgb channels) to 4, and the coefficients per channel of a degree: K = 1 for -1, else (sh_deg+1)^2
inline bool valid_deg(int sh_deg) { return sh_deg >= -1 && sh_deg <= 4; }
inline int K_of(int sh_deg) { return sh_deg < 0 ? 1 : (sh_deg + 1) * (sh_deg + 1); }
// padded heads width for K spherical-harmonic coefficients per channel
inline int heads_width(int K) { return ((1 + 3 * K) + 15) / 16 * 16; }
// bytes of one forward weight image (hi or lo): the trunk slots, then the heads slots of NH rows
inline size_t fwd_image_bytes(int NH) { return size_t(FWD_TRUNK_SLOTS) * WSLOT_BYTES + size_t(FWD_HEAD_SLOTS) * NH * 64; }
// bytes of one dgrad weight image
inline size_t bwd_image_bytes(int NH) { return size_t(bwd_slots(NH)) * WSLOT_BYTES; }

// precision: 1 = single fp16 pass (10-bit mantissa operands, fp32 accumulate, reduced SFU sine),
//            3 = error-compensated 3-pass split (hi*hi + lo*hi + hi*lo, libdevice sinf)
cudaError_t launch_mlp_fwd(const FwdParams& p, int nsplit, int num_sms, cudaStream_t stream);
// the vanilla view-branch forward (out_mode OUT_VANILLA, FwdParams view_*): fp16 inference only
cudaError_t launch_mlp_fwd_vanilla(const FwdParams& p, int num_sms, cudaStream_t stream);

// forward weight image of a vanilla NeRF MLP (heads VANILLA_NH wide) from its folded flat parameters
// (vanilla_flat_layout); only the fp16 "hi" image: the vanilla forward is fp16 inference
cudaError_t launch_pack_vanilla(const float* flat, int W, uint8_t* w_hi, cudaStream_t stream);

// t[r][j] = sum_e W10_e[e][j] posenc(viewdirs[r], 0, deg_view, legacy)[e] + c[j] of n view directions (projection.cu;
// the same posenc and matvec as the SH projection's direction tables)
cudaError_t launch_view_table(const float* viewdirs, long long n, int deg_view, int legacy, const float* w10e,
                              const float* c, float* t, cudaStream_t stream);
constexpr int MAX_DEG_VIEW = 32;

// flat fp32 parameters of one MLP in reference order (Dense_0..Dense_9: kernel [in,out] then
// bias; flat_layout(K, W), W = posenc_width) -> packed images.  The images do not depend on W: rows [W, 63) of the
// posenc slots are 0.
cudaError_t launch_pack_weights(const float* flat, int K, int W, uint8_t* w_hi, uint8_t* w_lo,
                                uint8_t* wt_hi, cudaStream_t stream);
// the residual (lo) of the dgrad images only, in the layout of wt_hi (bwd_image_bytes(NH)): the x3 data gradient
cudaError_t launch_pack_wt_lo(const float* flat, int K, int W, uint8_t* wt_lo, cudaStream_t stream);



// ---- render.cu ------------------------------------------------------------------------------
cudaError_t launch_sample_coarse(const float* z_base, const float* t_rand, int R, int N, float* z_out,
                                 cudaStream_t st);
cudaError_t launch_composite_fwd(const float4* rgbs, const float* z, const float* dirs, int R, int N,
                                 int white_bkgd, float* out_rgb, float* out_disp, float* out_acc,
                                 float* out_weights, cudaStream_t st);
// sigma_act: the activation rgbs.w went through (SigmaAct); G.w takes its derivative, formed from rgbs.w
cudaError_t launch_composite_bwd(const float4* rgbs, const float* z, const float* dirs,
                                 const float* comp_rgb, const float* pixels, int R, int N, int white_bkgd,
                                 float gscale, int sigma_act, float4* G, float* sq_err_sum, cudaStream_t st);
cudaError_t launch_sample_pdf(const float* z_c, const float* weights, const float* u, int u_per_ray, int R,
                              int Nc, int Nf, float* z_out, cudaStream_t st);
// t_rand [n_t], u [n_u] ~ U[0,1), sp [n_sp] ~ U[-radius, radius): Philox4x32-10 keyed by seed, counter (index, stream, step);
// step_dev (device float, optional) overrides `step` so that a captured graph draws fresh numbers on every replay
cudaError_t launch_draw_uniforms(unsigned long long seed, float step, const float* step_dev, float* t_rand,
                                 long long n_t, float* u, long long n_u, float* sp, long long n_sp, float sp_radius,
                                 cudaStream_t st);
// rgbs[i].w = relu(sigma) of the sparsity points (as the OUT_RGBS epilogue leaves it); G[i] = (0,0,0, dL/dsigma_raw)
cudaError_t launch_sparsity_grad(const float4* rgbs, int n, float length, float coef, float4* G,
                                 float* exp_sum, cudaStream_t st);

// ---- mlp_bwd.cu -----------------------------------------------------------------------------
struct BwdParams {
  long long M;
  const float4* G;          // [M] (d pre_r, d pre_g, d pre_b, d sigma_raw), loss-scaled
  const float* viewdirs;    // [R,3] (n_per_ray > 0) or [M,3] (n_per_ray == 0)
  int n_per_ray;
  long long M_rays;         // rows [M_rays, M) are free points (sigma gradient only): no view direction
  MlpPacked w;
  int sh_deg, K, NH;
  const uint32_t* mask;     // [8][Mpad][8] from mlp_fwd (net_act relu)
  uint8_t* save_dz;         // [ntile][8][64 KB]
  uint8_t* save_do;         // [ntile][32 KB]
  uint32_t* progress;       // [ntile], zeroed: stages of the tile whose stores have completed (wgrad_body.cuh)
  // ---- x3 (nsplit = 3): residual images of the operands and of the saved tiles ----
  const uint8_t* wt_lo;     // residual of w.wt_hi (launch_pack_wt_lo)
  uint8_t* save_dz_lo;      // [ntile][8][64 KB]
  uint8_t* save_do_lo;      // [ntile][32 KB]
  // ---- trunk activation: NET_RELU reads `mask`, the others form f'(h) from `h` (x3: h + h_lo) ----
  int net_act;              // NetAct
  const uint8_t* h;         // [ntile][8][64 KB] h_0..h_7 tile images from mlp_fwd (save_h)
  const uint8_t* h_lo;      // x3: their residual images (save_h_lo)
};
// grid = min(tiles, num_ctas) persistent CTAs.  nsplit 3: dZ_l = hi + lo, every product lo*hi + hi*lo + hi*hi
cudaError_t launch_mlp_bwd(const BwdParams& p, int nsplit, int num_ctas, cudaStream_t stream);

// ---- mlp_wgrad.cu ---------------------------------------------------------------------------
constexpr int WG_PARTIAL_FLOATS = 65536 + 256;
constexpr int WG_MAX_CTAS = 160;
constexpr int WG_NUM_ROLES = 9;

// Roles of the wgrad CTAs.  Role r computes D[A feature][B feature] = sum over samples of A^T B, with A and B read
// from the tile images mlp_fwd and mlp_bwd saved, and the bias gradient as column sums of A or B.  B is always 256
// features wide (h_l or dZ_0), so every MMA is an m64n256.
//  - Dense_1..7 ("halved" roles): A = dZ_l, B = h_{l-1}.  A CTA owns one 128-row half of D, so the role's CTAs come
//    in pairs.  Its partial holds D's rows [128 half, +128) at row pitch 256.  Dense_5 also contracts its A with the
//    posenc tile (the skip rows, inputs 256..318) into a second, 64-wide accumulator; those 128 x 64 go to the rows
//    of the partial its half leaves unused: floats [32768 (1 - half), +8192) at row pitch 64.
//  - Dense_0 and the heads ("transposed" roles): A = posenc or dO (64 or NH features), B = dZ_0 or h_7, so D is the
//    transposed weight gradient.  Every CTA computes all of D; warpgroup w writes partial rows [64 w, +64) at pitch
//    256.  With A <= 64 features (wgrad_split_k) both warpgroups compute the same 64 rows over alternate halves of
//    each stage's samples, and row r of D is the sum of partial rows r and 64 + r; with NH = 80 warpgroup w computes
//    A features [64 w, +64).
// The bias sums follow at WG_PARTIAL_FLOATS - 256, indexed by output feature (the split-K halves already added).
enum WgOperand : int { WG_DZ = 0, WG_H = 1, WG_E = 2, WG_DO = 3 };   // dZ_l, h_l, posenc, dO tile images
enum WgBias : int { WG_BIAS_A = 1, WG_BIAS_B = 2 };
struct WgradRole {
  int dense;            // reference Dense_i (the heads role: Dense_8 and Dense_9, in packed heads columns)
  int a_op, a_layer;    // A operand: result rows
  int b_op, b_layer;    // B operand: result columns
  int halves;           // 2: the CTAs own 128-row halves of D; 1: transposed, every CTA computes all rows
  int skip;             // Dense_5: A is also contracted with the posenc tile
  int bias;
};
__host__ __device__ constexpr WgradRole wgrad_role(int r) {
  //     Dense_i    A               B              halves  skip                bias
  return r < 7 ? WgradRole{r + 1, WG_DZ, r + 1,  WG_H, r,       2, r + 1 == SKIP_LAYER, WG_BIAS_A}   // Dense_1..7
       : r == 7 ? WgradRole{0,    WG_E, 0,       WG_DZ, 0,      1, 0,                   WG_BIAS_B}   // Dense_0^T
       :          WgradRole{8,    WG_DO, 0,      WG_H, 7,       1, 0,                   WG_BIAS_A};  // heads^T
}
// Every tile image mlp_bwd stores (dZ_0..dZ_7, dO) is an operand of exactly one role: the two row halves of a halved
// role load disjoint chunks of its dZ, a transposed role loads all of it, and the CTAs of a role (half) split the
// tiles.  So each stored byte is loaded by exactly one CTA, which may then discard it from L2 (WgradParams::discard).
// A role that read a dZ or dO a second time would read discarded lines: it must not build.
__host__ __device__ constexpr int wgrad_readers(int op, int layer) {
  int n = 0;
  for (int r = 0; r < WG_NUM_ROLES; ++r) {
    const WgradRole W = wgrad_role(r);
    n += (W.a_op == op && W.a_layer == layer) + (W.b_op == op && W.b_layer == layer);
  }
  return n;
}
__host__ __device__ constexpr bool wgrad_reads_saved_grads_once() {
  for (int l = 0; l < NUM_TRUNK; ++l)
    if (wgrad_readers(WG_DZ, l) != 1) return false;
  for (int r = 0; r < WG_NUM_ROLES; ++r)   // a transposed role loads only its first A chunks: all of dO, none of dZ
    if (wgrad_role(r).halves == 1 && wgrad_role(r).a_op == WG_DZ) return false;
  return wgrad_readers(WG_DO, 0) == 1;
}
static_assert(wgrad_reads_saved_grads_once(), "every dZ_l and dO tile must be loaded by exactly one wgrad role");
// role holding Dense_`dense`'s gradient (8 and 9: the heads)
__host__ __device__ constexpr int wgrad_role_of(int dense) { return dense == 0 ? 7 : dense < 8 ? dense - 1 : 8; }
// transposed role whose A (posenc, or dO with NH <= 64) fits one m64: its warpgroups split each stage's samples
__host__ __device__ constexpr bool wgrad_split_k(const WgradRole& R, int NH) {
  return R.halves == 1 && (R.a_op == WG_E || NH <= 64);
}
struct WgradSegment {
  const uint8_t *h, *dz, *e, *d_o;
};
struct WgradParams {
  WgradSegment seg;         // one level's tile arrays (its sparsity points ride behind the ray samples)
  long long seg_tiles;
  int NH;
  float* partials;          // [num_ctas][WG_PARTIAL_FLOATS]
  const uint32_t* progress; // [seg_tiles], advanced by the mlp_bwd launch that writes this segment's dZ / dO
  int discard;              // 1: drop every dZ / dO line from L2 once loaded (no write-back; the images become undefined)
  short cta_role[WG_MAX_CTAS], cta_index[WG_MAX_CTAS], cta_count[WG_MAX_CTAS];
};
// role -> [first CTA, count]; fills the per-CTA tables of `p`; returns number of CTAs to launch
int wgrad_assign_roles(WgradParams& p, int num_sms, int role_start[WG_NUM_ROLES],
                       int role_count[WG_NUM_ROLES]);
// launched with programmatic stream serialization right behind the mlp_bwd launch it consumes (wgrad_body.cuh)
cudaError_t launch_mlp_wgrad(const WgradParams& p, int num_ctas, cudaStream_t stream);

// ---- optim.cu -------------------------------------------------------------------------------
// one mlp_wgrad launch: its partials and its role -> CTA table (wgrad_assign_roles)
struct WgradPass {
  const float* partials;
  int role_start[WG_NUM_ROLES], role_count[WG_NUM_ROLES];
};
// The x3 weight gradient is three launches of mlp_wgrad over the hi / lo tile images (by linearity):
//   pass 0: h hi, dz hi, e hi, d_o hi   -> A_hi B_hi for every role
//   pass 1: h hi, dz lo, e hi, d_o lo   -> A_lo B_hi (Dense_1..7, heads), E_hi dZ0_lo (Dense_0), dZ5_lo E_hi (skip)
//   pass 2: h lo, dz hi, e lo, d_o hi   -> A_hi B_lo (Dense_1..7, heads), E_lo dZ0_hi (Dense_0), dZ5_hi E_lo (skip)
// The bias sums (columns of dZ_l / dO, Dense_0: of dZ_0) of pass 2 repeat pass 0's: only passes 0 and 1 count them.
constexpr int X3_WGRAD_PASSES = 3;
constexpr int X3_BIAS_PASSES = 2;
// partials of `npass` wgrad launches -> flat gradient of one MLP (reference layout flat_layout(K, W)), times
// inv_scale.  Every element sums its passes in order; the biases only the first min(npass, X3_BIAS_PASSES).  The
// rows of posenc columns [W, 64) are not part of the layout: they are dropped.
cudaError_t launch_reduce_grads(const WgradPass* passes, int npass, int K, int W, float inv_scale, float* grad_flat,
                                cudaStream_t stream);
// flax.optim.Adam.apply_gradient on a flat buffer; grad is multiplied by grad_mult first
// lr_step_dev (optional, device [2] = {lr, step}) overrides the host lr / step: a captured graph replays with new values
cudaError_t launch_adam(float* param, const float* grad, float* m, float* v, long long n, float lr,
                        float step, const float* lr_step_dev, float beta1, float beta2, float eps, float grad_mult,
                        float weight_decay_coef, cudaStream_t stream);

// ---- flat parameter layout of one MLP (reference order) -------------------------------------
// Dense_i kernel is [in,out] row-major (flax), followed by its bias [out].  W = posenc width: Dense_0 is [W, 256],
// Dense_5 [256 + W, 256] with rows [h4 | posenc].
struct FlatLayout {
  int w_off[10], b_off[10], in_dim[10], out_dim[10], total;
};
inline FlatLayout flat_layout(int K, int W) {
  FlatLayout L;
  int off = 0;
  for (int i = 0; i < 10; ++i) {
    int in = (i == 0) ? W : (i == SKIP_LAYER ? WIDTH + W : WIDTH);
    int out = (i < 8) ? 256 : (i == 8 ? 1 : 3 * K);
    L.in_dim[i] = in;
    L.out_dim[i] = out;
    L.w_off[i] = off;
    off += in * out;
    L.b_off[i] = off;
    off += out;
  }
  L.total = off;
  return L;
}
// folded flat parameters of a vanilla NeRF MLP: Dense_0..Dense_8 as flat_layout(1, W), then the folded head
// W9 W10_b [256, VIEW_H] (no bias: b9 W10_b + b10 rides in the view table)
inline FlatLayout vanilla_flat_layout(int W) {
  FlatLayout L = flat_layout(1, W);
  L.out_dim[9] = VIEW_H;
  L.b_off[9] = L.w_off[9] + WIDTH * VIEW_H;
  L.total = L.b_off[9];
  return L;
}

// ---- quantize.cu ----------------------------------------------------------------------------
// median cut of compressed-tree palettes (pob_quantize_median_cut): at most 2^16 colours, so at most 2^15 boxes split
// in a round
constexpr int QUANT_MAX_BITS = 16;
constexpr int QUANT_MAX_COLORS = 1 << QUANT_MAX_BITS;
// byte offsets of the workspace arrays of n_basis point sets of n points (256-byte aligned) and the total
struct QuantLayout {
  size_t idx[2], off[2], key[2], pos[2], up, split, wsorted, total, bytes;
};
QuantLayout quant_layout(int64_t n_basis, int64_t n, int weighted);
// every launch of one quantisation, in order on `stream`, each counted and timed under POB_PH_QUANT; the caller has
// checked the arguments.  0, or 1 after a launch error recorded for pob_last_error
int launch_quantize(const float* points, const double* weights, int64_t n, int nb, int bits, float* palette,
                            uint16_t* map, void* workspace, int sms, cudaStream_t stream);

}  // namespace pob
