// projection.cu — SH projection of a vanilla NeRF colour branch (octree.extraction step2 with use_viewdirs:
// octree/extraction.py:217-241,362-394, octree/nerf/sh_proj.py:273-306).
//
// The reference evaluates the whole view branch for every (sample point, direction) pair and projects the raw rgb
// onto the SH basis by Monte Carlo:  coeff[p, c, k] = 4 pi / D * sum_d raw_rgb[p, d, c] Y_k(d).  The branch is
//   z = relu(W10 [bottleneck; posenc(d)] + b10),  raw_rgb = W11 z + b11,  bottleneck = W9 h7 + b9 (no activation),
// so W10 [b; e] = W10_b b + W10_e e splits into a per-point part a_p = W10_b (W9 h7 + b9) + b10 (computed with the
// trunk, see plenoctree_b200/octree/projection.py) and a per-direction part t_d = W10_e posenc(d).  What remains per
// pair is 128 FADD + 128 FMNMX + 3 x 128 FFMA on the CUDA cores, all in fp32:
//
//   pob_sh_proj_directions  one direction set per block of leaves, drawn from (seed, block index) with Philox, and
//                           its tables t_d (stored [128][D]) and Y_k(d) ([D][K]);
//   pob_sh_proj_cells       per leaf: mean over its S sample points of [coeff (c*K + k), raw sigma], the rows of
//                           step2's tree data.
//
// Projection CTA: 256 threads, tiles of 64 points x 64 directions.  Each thread forms a 4 x 4 (point, direction)
// block of raw rgb from shared-memory columns of a_p and t_d (two LDS.128 per hidden unit for 80 FP32 instructions),
// the tile's rgb is summed over each leaf's points in place, and the leaf coefficients sum_d R[d][c] Y_k(d) are
// accumulated in registers by the thread that owns them.  Every sum runs in a fixed order, so the result does not
// depend on the grid or on how many launches (or ranks) the leaves are split over.
#include <cstdint>

#include "../../include/plenoctree_b200.h"
#include "capi_util.h"
#include "common.cuh"
#include "kernels.h"

namespace pob {
namespace {

constexpr int PROJ_H = 128;        // width of the condition layer (net_width_condition)
constexpr int PT = 64;             // points per tile
constexpr int DT = 64;             // directions per tile
constexpr int PROJ_THREADS = 256;  // 16 x 16 threads, 4 x 4 pairs each
constexpr int MAX_K = 25;
// leaf coefficients of one CTA: at most 64 leaves x 3K <= 4800, 19 per thread
constexpr int ACC_PER_THREAD = (PT * 3 * MAX_K + PROJ_THREADS - 1) / PROJ_THREADS;
constexpr int DIRS_PER_CTA = 32;   // direction-table kernel
constexpr int MAX_DEG_VIEW = 32;
constexpr uint32_t PROJ_STREAM = 0x5348u;   // Philox counter word of the direction draws ("SH")

// A direction of block `blk`: theta = acos(2u - 1), phi = 2 pi v (sh_proj.spherical_uniform_sampling), then
// spher2cart, all in fp32 as the reference evaluates them.
__device__ __forceinline__ float3 proj_direction(unsigned long long seed, long long blk, int d) {
  const uint4 r = philox4x32_10(make_uint4(uint32_t(d), uint32_t(blk), uint32_t(blk >> 32), PROJ_STREAM),
                                make_uint2(uint32_t(seed), uint32_t(seed >> 32)));
  const float theta = acosf(__fsub_rn(__fmul_rn(2.0f, u01(r.x)), 1.0f));
  const float phi = __fmul_rn(6.2831854820251465f, u01(r.y));
  const float s = sinf(theta);
  return make_float3(__fmul_rn(s, cosf(phi)), __fmul_rn(s, sinf(phi)), cosf(theta));
}

// grid (ceil(D / 32), n_blocks), 128 threads: thread j forms t_d[j] = sum_e W10_e[e][j] posenc(d)[e] of 32
// directions.  posenc(d, 0, deg_view, legacy) as nerf_sh/nerf/model_utils.py:145-173 (feature order in the header).
__global__ void __launch_bounds__(PROJ_H) proj_directions_kernel(unsigned long long seed, long long block0, int D,
                                                                 int deg_view, int legacy, int sh_deg, int K,
                                                                 const float* __restrict__ w10e,
                                                                 float* __restrict__ dirs, float* __restrict__ tT,
                                                                 float* __restrict__ basis) {
  extern __shared__ float enc[];   // [DIRS_PER_CTA][E]
  __shared__ float3 dsm[DIRS_PER_CTA];
  const int E = 3 + 6 * deg_view;
  const long long b = blockIdx.y;
  const int d0 = blockIdx.x * DIRS_PER_CTA;
  const int nd = min(DIRS_PER_CTA, D - d0);
  const int tid = threadIdx.x;
  if (tid < nd) {
    const int d = d0 + tid;
    const float3 v = proj_direction(seed, block0 + b, d);
    dsm[tid] = v;
    if (dirs) {
      float* o = dirs + (b * D + d) * 3;
      o[0] = v.x, o[1] = v.y, o[2] = v.z;
    }
    float y[25];
    sh_basis(sh_deg, v.x, v.y, v.z, y);
    float* yo = basis + (b * D + d) * K;
#pragma unroll
    for (int k = 0; k < MAX_K; ++k)
      if (k < K) yo[k] = y[k];
  }
  __syncthreads();
  const int L = deg_view;
  for (int i = tid; i < nd * E; i += PROJ_H) {
    const int dd = i / E, e = i - dd * E;
    const float3 v = dsm[dd];
    float f;
    if (e < 3) {
      f = e == 0 ? v.x : (e == 1 ? v.y : v.z);
    } else {
      int q = e - 3, l, c, cosine;
      if (legacy) {
        l = q / 6, cosine = (q % 6) >= 3, c = q % 3;
      } else {
        cosine = q >= 3 * L, q -= cosine ? 3 * L : 0, l = q / 3, c = q % 3;
      }
      const float x = (c == 0 ? v.x : (c == 1 ? v.y : v.z)) * exp2f(float(l));   // exact: a power of two
      f = sinf(cosine ? __fadd_rn(x, 1.5707963705062866f) : x);
    }
    enc[dd * E + e] = f;
  }
  __syncthreads();
  float acc[DIRS_PER_CTA];
#pragma unroll
  for (int dd = 0; dd < DIRS_PER_CTA; ++dd) acc[dd] = 0.f;
  for (int e = 0; e < E; ++e) {
    const float w = __ldg(w10e + (long long)e * PROJ_H + tid);
#pragma unroll
    for (int dd = 0; dd < DIRS_PER_CTA; ++dd) acc[dd] = fmaf(w, enc[min(dd, nd - 1) * E + e], acc[dd]);
  }
  float* row = tT + (b * PROJ_H + tid) * (long long)D + d0;
#pragma unroll
  for (int dd = 0; dd < DIRS_PER_CTA; ++dd)
    if (dd < nd) row[dd] = acc[dd];
}

struct ProjSmem {
  float a[PROJ_H][PT];        // a_p of the point tile, transposed
  float t[PROJ_H][DT];        // t_d of the direction tile
  // raw rgb of the tile; row `first point of a leaf` then holds the leaf's sum.  Rows are padded to DT + 4 floats so
  // that the coefficient phase's reads of different (leaf, channel) rows at the same direction fall in different banks
  float rgb[PT][3][DT + 4];
  float4 w11[PROJ_H];         // (W11[j][0], W11[j][1], W11[j][2], 0)
  float y[DT * MAX_K];        // Y_k(d) of the direction tile, [d][k]
};

// grid (n_table_blocks * ceil(LB / G)), G = leaves per CTA = max(1, 64 / S).
__global__ void __launch_bounds__(PROJ_THREADS, 1)
    proj_cells_kernel(long long n_leaves, int S, int LB, int G, int D, int K, const float* __restrict__ a,
                      const float* __restrict__ sigma, const float* __restrict__ tT, const float* __restrict__ basis,
                      const float* __restrict__ w11, const float* __restrict__ b11, float scale,
                      float* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  ProjSmem& sm = *reinterpret_cast<ProjSmem*>(smem_raw);
  const int cpb = (LB + G - 1) / G;
  const long long blk = blockIdx.x / cpb;
  const int grp = blockIdx.x % cpb;
  const long long leaf0 = blk * LB + (long long)grp * G;
  const int nleaf = int(min((long long)min(G, LB - grp * G), n_leaves - leaf0));
  if (nleaf <= 0) return;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int npts = nleaf * S, nout = nleaf * 3 * K;
  const long long p0 = leaf0 * S;
  const float* tb = tT + blk * PROJ_H * (long long)D;
  const float* yb = basis + blk * (long long)D * K;
  for (int j = tid; j < PROJ_H; j += PROJ_THREADS)
    sm.w11[j] = make_float4(w11[j * 3 + 0], w11[j * 3 + 1], w11[j * 3 + 2], 0.f);
  const float bias0 = b11[0], bias1 = b11[1], bias2 = b11[2];

  float acc[ACC_PER_THREAD];
#pragma unroll
  for (int i = 0; i < ACC_PER_THREAD; ++i) acc[i] = 0.f;

  for (int c0 = 0; c0 < npts; c0 += PT) {
    const int c1 = min(npts, c0 + PT);
    __syncthreads();
    // a tile: lane = point (conflict-free transposed stores), rows beyond the leaves' points are zero
    for (int i = tid; i < PT * PROJ_H; i += PROJ_THREADS) {
      const int p = i % PT, j = i / PT;
      sm.a[j][p] = c0 + p < c1 ? __ldg(a + (p0 + c0 + p) * PROJ_H + j) : 0.f;
    }
    for (int e0 = 0; e0 < D; e0 += DT) {
      const int nd = min(DT, D - e0);
      __syncthreads();
      for (int i = tid; i < PROJ_H * DT; i += PROJ_THREADS) {
        const int d = i % DT, j = i / DT;
        sm.t[j][d] = d < nd ? __ldg(tb + (long long)j * D + e0 + d) : 0.f;
      }
      for (int i = tid; i < DT * K; i += PROJ_THREADS)   // directions past D get Y = 0: they add exact zeros
        sm.y[i] = i < nd * K ? __ldg(yb + (long long)e0 * K + i) : 0.f;
      __syncthreads();

      // raw rgb of the 4 x 4 pairs (points 4 ty + i, directions 4 tx + q)
      float r[4][4][3];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int q = 0; q < 4; ++q) r[i][q][0] = r[i][q][1] = r[i][q][2] = 0.f;
#pragma unroll 4
      for (int j = 0; j < PROJ_H; ++j) {
        const float4 av = *reinterpret_cast<const float4*>(&sm.a[j][ty * 4]);
        const float4 tv = *reinterpret_cast<const float4*>(&sm.t[j][tx * 4]);
        const float4 w = sm.w11[j];
        const float ap[4] = {av.x, av.y, av.z, av.w}, td[4] = {tv.x, tv.y, tv.z, tv.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float z = fmaxf(ap[i] + td[q], 0.f);
            r[i][q][0] = fmaf(w.x, z, r[i][q][0]);
            r[i][q][1] = fmaf(w.y, z, r[i][q][1]);
            r[i][q][2] = fmaf(w.z, z, r[i][q][2]);
          }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int p = ty * 4 + i;
        *reinterpret_cast<float4*>(&sm.rgb[p][0][tx * 4]) =
            make_float4(r[i][0][0] + bias0, r[i][1][0] + bias0, r[i][2][0] + bias0, r[i][3][0] + bias0);
        *reinterpret_cast<float4*>(&sm.rgb[p][1][tx * 4]) =
            make_float4(r[i][0][1] + bias1, r[i][1][1] + bias1, r[i][2][1] + bias1, r[i][3][1] + bias1);
        *reinterpret_cast<float4*>(&sm.rgb[p][2][tx * 4]) =
            make_float4(r[i][0][2] + bias2, r[i][1][2] + bias2, r[i][2][2] + bias2, r[i][3][2] + bias2);
      }
      __syncthreads();

      // sum each leaf's points of this tile into the row of its first point (in point order)
      const int g0 = c0 / S, g1 = (c1 - 1) / S;
      if (S > 1) {
        for (int i = tid; i < (g1 - g0 + 1) * 3 * DT; i += PROJ_THREADS) {
          const int g = g0 + i / (3 * DT), c = (i / DT) % 3, d = i % DT;
          const int first = max(g * S, c0) - c0, last = min(g * S + S, c1) - c0;
          float s = sm.rgb[first][c][d];
          for (int p = first + 1; p < last; ++p) s += sm.rgb[p][c][d];
          sm.rgb[first][c][d] = s;
        }
        __syncthreads();
      }
      // leaf coefficients: acc(g, c, k) += sum_d R_g[d][c] Y_k(d)
#pragma unroll
      for (int i = 0; i < ACC_PER_THREAD; ++i) {
        const int o = tid + i * PROJ_THREADS;
        if (o < nout) {
          const int g = o / (3 * K), c = (o / K) % 3, k = o % K;
          if (g >= g0 && g <= g1) {
            const float* rr = sm.rgb[max(g * S, c0) - c0][c];
            float s = 0.f;
#pragma unroll 8
            for (int d = 0; d < DT; ++d) s = fmaf(rr[d], sm.y[d * K + k], s);
            acc[i] += s;
          }
        }
      }
    }
  }
  const int ld = 3 * K + 1;
#pragma unroll
  for (int i = 0; i < ACC_PER_THREAD; ++i) {
    const int o = tid + i * PROJ_THREADS;
    if (o < nout) {
      const int g = o / (3 * K);
      out[(leaf0 + g) * ld + (o - g * 3 * K)] = acc[i] * scale;
    }
  }
  if (tid < nleaf) {   // raw sigma: the mean over the leaf's points
    const float* sg = sigma + p0 + (long long)tid * S;
    float s = 0.f;
    for (int p = 0; p < S; ++p) s += sg[p];
    out[(leaf0 + tid) * ld + 3 * K] = s / float(S);
  }
}

// a_p = h7 W + b of one 128-row tile of the trunk (grid = tiles, 256 threads, thread = 8 rows x 8 columns): h7 is
// the fp16 tile image the saving forward stores (layouts.py t_tile_offset), W = W9 W10_b [256][128] and b the
// composed bias, fp32 accumulation.
constexpr int A_KC = 32;   // W rows staged per step
__global__ void __launch_bounds__(256) proj_point_a_kernel(const uint8_t* __restrict__ save_h, long long M,
                                                           const float* __restrict__ w, const float* __restrict__ b,
                                                           float* __restrict__ a) {
  extern __shared__ __align__(16) unsigned char smem_a[];
  __half* h = reinterpret_cast<__half*>(smem_a);                            // the 64 KB T image
  float* ws = reinterpret_cast<float*>(smem_a + A_TILE_BYTES);             // [A_KC][128]
  const long long it = blockIdx.x;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const uint4* src = reinterpret_cast<const uint4*>(save_h + (size_t(it) * NUM_TRUNK + (NUM_TRUNK - 1)) * A_TILE_BYTES);
  for (int i = tid; i < A_TILE_BYTES / 16; i += 256) reinterpret_cast<uint4*>(h)[i] = __ldg(src + i);
  float acc[8][8];
#pragma unroll
  for (int r = 0; r < 8; ++r)
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[r][c] = 0.f;
  for (int k0 = 0; k0 < 256; k0 += A_KC) {
    __syncthreads();
    for (int i = tid; i < A_KC * PROJ_H / 4; i += 256)
      reinterpret_cast<float4*>(ws)[i] = __ldg(reinterpret_cast<const float4*>(w + k0 * PROJ_H) + i);
    __syncthreads();
#pragma unroll 4
    for (int k = 0; k < A_KC; ++k) {
      const int col = k0 + k;
      const float4 w0 = *reinterpret_cast<const float4*>(ws + k * PROJ_H + tx * 8);
      const float4 w1 = *reinterpret_cast<const float4*>(ws + k * PROJ_H + tx * 8 + 4);
      const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const int row = ty * 8 + r;
        const uint32_t off = uint32_t(row >> 5) * 16384u + uint32_t(col >> 3) * 512u + uint32_t(row & 31) * 16u +
                             uint32_t(col & 7) * 2u;
        const float hv = __half2float(h[off / 2]);
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[r][c] = fmaf(hv, wv[c], acc[r][c]);
      }
    }
  }
  float bv[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) bv[c] = b[tx * 8 + c];
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const long long row = it * TILE_M + ty * 8 + r;
    if (row < M) {
      float4* o = reinterpret_cast<float4*>(a + row * PROJ_H + tx * 8);
      o[0] = make_float4(acc[r][0] + bv[0], acc[r][1] + bv[1], acc[r][2] + bv[2], acc[r][3] + bv[3]);
      o[1] = make_float4(acc[r][4] + bv[4], acc[r][5] + bv[5], acc[r][6] + bv[6], acc[r][7] + bv[7]);
    }
  }
}

// workspace of pob_sh_proj_points: the saving forward's h_0..h_7 images, posenc images and relu masks
struct PointWs {
  size_t h, e, mask, total;
};
PointWs point_ws(long long m) {
  const long long rows = padded_rows(m), tiles = rows / TILE_M;
  PointWs w;
  w.h = 0;
  w.e = size_t(tiles) * NUM_TRUNK * A_TILE_BYTES;
  w.mask = w.e + size_t(tiles) * (A_TILE_BYTES / 4);
  w.total = w.mask + size_t(NUM_TRUNK) * rows * 8 * sizeof(uint32_t);
  return w;
}

}  // namespace
}  // namespace pob

extern "C" {

int64_t pob_sh_proj_points_workspace_bytes(int64_t m) { return m < 0 ? -1 : int64_t(pob::point_ws(m).total); }

int pob_sh_proj_points(const void* packed_dev, const pob_posenc* posenc, const float* points_dev, int64_t m,
                       const float* head_w_dev, const float* head_b_dev, void* workspace_dev, float* a_dev,
                       float* sigma_dev, void* stream) {
  const char* W = "pob_sh_proj_points";
  if (int e = pob_check_common(W, packed_dev, -1, POB_PREC_FP16)) return e;
  pob::NetDesc net;
  if (int e = pob_check_posenc(W, posenc, net)) return e;
  if (net.net_act != pob::NET_RELU) return pob_fail(W, "the vanilla trunk of the projection is relu");
  if (m < 0) return pob_fail(W, "negative point count");
  if (m == 0) return 0;
  if (!points_dev || !head_w_dev || !head_b_dev || !workspace_dev || !a_dev || !sigma_dev)
    return pob_fail(W, "NULL pointer");
  const int sms = pob_sms_or_fail(W);
  if (!sms) return 1;
  const pob::PointWs ws = pob::point_ws(m);
  uint8_t* base = static_cast<uint8_t*>(workspace_dev);
  pob::FwdParams p = pob_base_params(packed_dev, -1, net);
  p.src_mode = pob::SRC_POINTS;
  p.M = m;
  p.points = points_dev;
  p.out_mode = pob::OUT_SIGMA;
  p.out_sigma = sigma_dev;
  p.save_h = base + ws.h;
  p.save_e = base + ws.e;
  p.save_mask = reinterpret_cast<uint32_t*>(base + ws.mask);
  pob_count_launch(2);
  {
    PobPhaseTimer _t(POB_PH_FWD, (cudaStream_t)stream);
    POB_CUDA(W, pob::launch_mlp_fwd(p, 1, sms, (cudaStream_t)stream));
  }
  const size_t smem = pob::A_TILE_BYTES + size_t(pob::A_KC) * pob::PROJ_H * sizeof(float);
  POB_CUDA(W, cudaFuncSetAttribute(pob::proj_point_a_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  const long long tiles = (m + pob::TILE_M - 1) / pob::TILE_M;
  pob::proj_point_a_kernel<<<unsigned(tiles), 256, smem, (cudaStream_t)stream>>>(base + ws.h, m, head_w_dev,
                                                                                  head_b_dev, a_dev);
  POB_CUDA(W, cudaGetLastError());
  return 0;
}

int pob_sh_proj_directions(uint64_t seed, int64_t block0, int n_blocks, int n_dirs, int deg_view, int legacy_order,
                           int sh_deg, const float* w10e_dev, float* dirs_dev, float* t_dev, float* basis_dev,
                           void* stream) {
  const char* W = "pob_sh_proj_directions";
  if (n_blocks < 0 || n_blocks > 65535 || n_dirs < 1 || block0 < 0)
    return pob_fail(W, "need 0 <= n_blocks <= 65535 (one grid row per block), n_dirs >= 1, block0 >= 0");
  if (deg_view < 0 || deg_view > pob::MAX_DEG_VIEW)
    return pob_fail(W, "deg_view must be in [0, 32] (the posenc scale 2^(deg_view - 1) of a unit direction)");
  if (legacy_order != 0 && legacy_order != 1) return pob_fail(W, "legacy_order must be 0 or 1");
  if (sh_deg < 0 || sh_deg > 4) return pob_fail(W, "sh_deg must be in [0, 4]");
  if (!w10e_dev || !t_dev || !basis_dev) return pob_fail(W, "NULL pointer");
  if (!pob_sms_or_fail(W)) return 1;
  if (n_blocks == 0) return 0;
  const int K = (sh_deg + 1) * (sh_deg + 1);
  const size_t smem = size_t(pob::DIRS_PER_CTA) * (3 + 6 * deg_view) * sizeof(float);
  POB_CUDA(W, cudaFuncSetAttribute(pob::proj_directions_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   int(smem)));
  pob_count_launch();
  const dim3 grid(unsigned((n_dirs + pob::DIRS_PER_CTA - 1) / pob::DIRS_PER_CTA), unsigned(n_blocks));
  pob::proj_directions_kernel<<<grid, pob::PROJ_H, smem, (cudaStream_t)stream>>>(
      seed, block0, n_dirs, deg_view, legacy_order, sh_deg, K, w10e_dev, dirs_dev, t_dev, basis_dev);
  POB_CUDA(W, cudaGetLastError());
  return 0;
}

int pob_sh_proj_cells(int64_t n_cells, int samples_per_cell, int cells_per_block, const float* a_dev,
                      const float* sigma_dev, int n_dirs, int sh_deg, const float* t_dev, const float* basis_dev,
                      const float* w11_dev, const float* b11_dev, float* out_dev, void* stream) {
  const char* W = "pob_sh_proj_cells";
  if (n_cells < 0 || samples_per_cell < 1 || cells_per_block < 1 || n_dirs < 1)
    return pob_fail(W, "need n_cells >= 0, samples_per_cell >= 1, cells_per_block >= 1, n_dirs >= 1");
  if (sh_deg < 0 || sh_deg > 4) return pob_fail(W, "sh_deg must be in [0, 4]");
  if (!a_dev || !sigma_dev || !t_dev || !basis_dev || !w11_dev || !b11_dev || !out_dev)
    return pob_fail(W, "NULL pointer");
  if (!pob_sms_or_fail(W)) return 1;
  if (n_cells == 0) return 0;
  const int K = (sh_deg + 1) * (sh_deg + 1);
  const int G = samples_per_cell >= pob::PT ? 1 : pob::PT / samples_per_cell;
  const long long n_blk = (n_cells + cells_per_block - 1) / cells_per_block;
  const long long ctas = n_blk * ((cells_per_block + G - 1) / G);
  if (ctas > 0x7fffffffLL) return pob_fail(W, "too many cells for one launch");
  const float scale = float(4.0 * 3.14159265358979323846 / (double(n_dirs) * samples_per_cell));
  const size_t smem = sizeof(pob::ProjSmem);
  POB_CUDA(W, cudaFuncSetAttribute(pob::proj_cells_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  pob_count_launch();
  pob::proj_cells_kernel<<<unsigned(ctas), pob::PROJ_THREADS, smem, (cudaStream_t)stream>>>(
      n_cells, samples_per_cell, cells_per_block, G, n_dirs, K, a_dev, sigma_dev, t_dev, basis_dev, w11_dev, b11_dev,
      scale, out_dev);
  POB_CUDA(W, cudaGetLastError());
  return 0;
}

}  // extern "C"
