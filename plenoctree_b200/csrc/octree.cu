// octree.cu — PlenOctree kernels: volume renderer forward / backward (SURVEY §8 row a15), fused
// render + MSE-gradient + scatter training pass, SGD, point query, dense-grid weight render
// (octree.extraction masking_mode "weight").
//
// These replace the third-party svox extension the reference calls (octree/optimization.py:174-229,
// octree/extraction.py:181-214, octree/nerf/utils.py:448-498).  The arithmetic follows svox's published
// per-ray march (oracle/octree_oracle.py restates it).  Everything that decides WHERE a ray samples (ray set-up,
// positions, cell exits, step lengths) is written with __fmul_rn / __fadd_rn so that it rounds exactly like the
// float32 oracle and a ray never lands in a different leaf than the oracle's; the shading arithmetic (SH dot
// products, exp, sigmoid, compositing sums) may contract to FMA and uses the fast exp / reciprocal — the march is
// instruction-issue bound (ncu: sm__throughput 73-79 %, DRAM 5 %), so instruction count is what matters.
//
// Thread mapping (GPU-first, not svox's thread-per-ray): a *group* of G = 4 lanes owns one ray.  All lanes of a
// group walk the tree together (same-address loads broadcast), lane l owns basis functions l, l+G, ...: the 3K
// coefficient gather of a contributing leaf is three coalesced segments per group instead of 3K strided scalar loads
// per thread, the dot products finish with log2(G) shuffles, and the backward scatter issues coalesced RED.ADD.F32.
// Pixels are tiled per CTA so that neighbouring rays share L1 lines.
#include <cstdint>
#include <type_traits>

#include "../../include/plenoctree_b200.h"
#include "capi_util.h"
#include "common.cuh"

namespace pob {
namespace {

// Safety caps (never reached by a valid tree / positive step): a corrupt child array or a step that underflows
// against t must not hang the device.  A march visits one leaf per iteration (a few thousand for a depth-10 tree);
// the cap only has to exceed sqrt(3) / step_size for the smallest step the reference's configurations use
// (renderer_step_size 1e-5, octree/config/syn_sh16.json:16,22,24), since every iteration advances by >= step_size.
constexpr int MAX_MARCH_STEPS = 1 << 20;
constexpr int MAX_TREE_DEPTH = 40;

// Lanes per ray.  The march is instruction-issue bound and every lane of a group repeats the walk, so fewer lanes per
// ray = fewer instructions per ray.  Measured 800x800 / depth-8 SH16: 16 lanes 4.1 ms, 8 lanes 2.25 ms, 4 lanes
// 1.65 ms (2 lanes: 1.52 ms render but 4.7 ms training pass — not kept).
constexpr int G = 4;
// Rays per 256-thread CTA; a perspective camera's CTA renders a TILE_W x TILE_H pixel tile.
constexpr int RPB = 256 / G, TILE_W = 8, TILE_H = RPB / TILE_W;

struct TreeDev {
  const float* data;
  const int32_t* child;
  int N, D, K, rgba;
  float off[3], inv[3];
};

// A compressed (palette-indexed) tree, the format octree.compression writes: the walk uses TreeDev's child /
// N / K / rgba / off / inv (data and D are unused); a leaf's colour coefficient of basis function k is read from
// `retained` for k < retain, else through map[k - retain][leaf] into palette[k - retain].
struct QuantTreeDev : TreeDev {
  const float* sigma;        // [leaves]
  const uint16_t* map;       // [K - retain][leaves]
  const __half* palette;     // [K - retain][ncolors][3]
  const __half* retained;    // [retain][leaves][3]
  int retain, ncolors;
  unsigned long long leaves; // n_nodes * N^3: the plane stride of map / retained (Kq * leaves may pass 2^32)
};

struct Opts {
  float step, bg, sigma_thresh, stop_thresh;
};

struct Cam {
  float c2w[12];
  float fx, fy, width, height;
};

struct RaySrc {
  const float* o;   // explicit rays (world): origins / dirs / vdirs [n,3]; null -> perspective camera
  const float* d;
  const float* v;
  Cam cam;
  int row0;         // first pixel row of the slab this launch renders
  int nrows;
  long long n;      // number of rays (explicit) / pixels in the slab
};

struct Ray {
  float o[3], d[3], invd[3], vdir[3];
  float delta_scale, tmin, tmax;
  bool hit;
};

__device__ __forceinline__ void dda_unit(const float* cen, const float* invd, float& tmin, float& tmax) {
  tmin = 0.0f;
  tmax = 1e9f;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float t1 = __fmul_rn(-cen[i], invd[i]);
    const float t2 = __fadd_rn(t1, invd[i]);
    tmin = fmaxf(tmin, fminf(t1, t2));
    tmax = fminf(tmax, fmaxf(t1, t2));
  }
}

// persp pixel -> world ray (svox render_image_kernel: no +0.5 pixel centre; README.md:184); returns |(x, y, -1)|,
// whose reciprocal turns a distance along the unit ray into camera-axis depth
__device__ __forceinline__ float cam_ray(const Cam& c, int ix, int iy, float* o, float* d) {
  float x = __fsub_rn(float(ix), __fmul_rn(0.5f, c.width)) / c.fx;
  float y = -__fsub_rn(float(iy), __fmul_rn(0.5f, c.height)) / c.fy;
  float z = -1.0f;
  const float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
  x = x / nrm;
  y = y / nrm;
  z = z / nrm;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    d[a] = __fadd_rn(__fadd_rn(__fmul_rn(c.c2w[4 * a + 0], x), __fmul_rn(c.c2w[4 * a + 1], y)),
                     __fmul_rn(c.c2w[4 * a + 2], z));
    o[a] = c.c2w[4 * a + 3];
  }
  return nrm;
}

// NDC description of a forward-facing (LLFF) scene: the training images' width, height and focal (svox NDCConfig)
struct Ndc {
  float width, height, focal;
};

// svox world2ndc as the reference's convert_to_ndc (nerf_sh/nerf/datasets.py:40-60, near = 1) in its operation order:
// the origin moves onto the plane z = -1, then the projection; the NDC direction is then normalised for the march.
// The ray's view direction is not touched: SH colours stay a function of the world direction, as in NeRF-SH training.
__device__ __forceinline__ void world_to_ndc(const Ndc& n, float* o, float* d) {
  const float t = -__fadd_rn(1.0f, o[2]) / d[2];
  float c[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) c[a] = __fadd_rn(o[a], __fmul_rn(t, d[a]));
  const float sx = -(__fmul_rn(2.0f, n.focal) / n.width), sy = -(__fmul_rn(2.0f, n.focal) / n.height);
  const float cx = c[0] / c[2], cy = c[1] / c[2];
  d[0] = __fmul_rn(sx, __fsub_rn(d[0] / d[2], cx));
  d[1] = __fmul_rn(sy, __fsub_rn(d[1] / d[2], cy));
  d[2] = -2.0f / c[2];
  o[0] = __fmul_rn(sx, cx);
  o[1] = __fmul_rn(sy, cy);
  o[2] = __fadd_rn(1.0f, 2.0f / c[2]);
  const float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2])));
#pragma unroll
  for (int a = 0; a < 3; ++a) d[a] = d[a] / nrm;
}

// transform_coord + _get_delta_scale + unit-cube intersection (svox trace_ray prologue)
__device__ __forceinline__ void setup_ray(const float* off, const float* inv, const float* ow, const float* dw,
                                          const float* vw, Ray& r) {
  float nrm2 = 0.f;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    r.o[a] = __fadd_rn(off[a], __fmul_rn(inv[a], ow[a]));
    r.d[a] = __fmul_rn(dw[a], inv[a]);
    r.vdir[a] = vw[a];
  }
  nrm2 = __fadd_rn(__fadd_rn(__fmul_rn(r.d[0], r.d[0]), __fmul_rn(r.d[1], r.d[1])), __fmul_rn(r.d[2], r.d[2]));
  r.delta_scale = 1.0f / sqrtf(nrm2);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    r.d[a] = __fmul_rn(r.d[a], r.delta_scale);
    r.invd[a] = 1.0f / __fadd_rn(r.d[a], 1e-9f);
  }
  dda_unit(r.o, r.invd, r.tmin, r.tmax);
  r.hit = !(r.tmax < 0.f || r.tmin > r.tmax);
}

// svox query_single_from_root: pos in [0,1]^3 -> flat leaf index; pos becomes the position inside the leaf
__device__ __forceinline__ long long query_leaf(const int32_t* __restrict__ child, int N, float* pos, float& cube) {
  const float fN = float(N);
#pragma unroll
  for (int a = 0; a < 3; ++a) pos[a] = fmaxf(0.0f, fminf(1.0f - 1e-6f, pos[a]));
  long long node = 0;
  cube = fN;
  long long idx = 0;
  for (int level = 0; level < MAX_TREE_DEPTH; ++level) {
    int u[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      pos[a] = __fmul_rn(pos[a], fN);
      const float fl = floorf(pos[a]);
      u[a] = int(fl);
      pos[a] = __fsub_rn(pos[a], fl);
    }
    idx = ((node * N + u[0]) * N + u[1]) * N + u[2];
    const int skip = __ldg(child + idx);
    if (skip == 0) return idx;
    cube = cube * fN;
    node += skip;
  }
  return idx;
}

__device__ __forceinline__ unsigned group_mask() {
  const unsigned lane = threadIdx.x & 31;
  return ((1u << G) - 1u) << (lane / G * G);
}

__device__ __forceinline__ float group_sum(float v, unsigned mask) {
#pragma unroll
  for (int s = G / 2; s > 0; s >>= 1) v += __shfl_xor_sync(mask, v, s, G);
  return v;
}

__device__ __forceinline__ float sigmoidf(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }

// ---- leaf lookup with a per-ray path cache --------------------------------------------------------------
// Consecutive samples of a ray fall into neighbouring leaves that share most of their ancestors, yet svox walks
// down from the root for every sample (depth x dependent L2 loads).  For N = 2 the cell digits of a point are the
// binary digits of its coordinates (x*2 and x - floor(x) are exact in fp32), so the walk can resume below the deepest
// ancestor shared with the previous sample: lane k of the group keeps the node entered at level k (the otherwise
// idle lanes are the stack), the shared depth is a count-leading-zeros of the XOR of the integer coordinates, and
// the position inside the leaf is frac(x * 2^(depth+1)) — bit-identical to the iterated form.  Other branch
// factors, and levels deeper than 22, use the plain walk.
struct Marcher {
  unsigned pq0, pq1, pq2;
  static constexpr int PW = 8 / G;   // path registers per lane: levels l, l+G, ... are cached
  static constexpr int CACHED = G * PW;
  int pdepth;     // depth of the previous leaf, -1 = no previous sample
  int path[PW];   // lane l, register j: node entered at level l + j*G (level 0: root)

  __device__ __forceinline__ void init() {
    pdepth = -1;
#pragma unroll
    for (int j = 0; j < PW; ++j) path[j] = 0;
    pq0 = pq1 = pq2 = 0;
  }

  // leaf holding origin + t * dir; returns its flat index and the march length to its exit (+ step)
  // (leaf indices fit 32 bits: n_nodes * N^3 < 2^32 is checked on the host)
  __device__ __forceinline__ unsigned locate(const TreeDev& T, const Ray& r, float step, float t, int l, unsigned mask,
                                             float& delta_t) {
    float pos[3], cube, inv_cube = 0.f;
#pragma unroll
    for (int a = 0; a < 3; ++a) pos[a] = __fadd_rn(r.o[a], __fmul_rn(t, r.d[a]));
    unsigned idx;
    bool pow2 = false;
    if (T.N == 2) {
      pow2 = true;
#pragma unroll
      for (int a = 0; a < 3; ++a) pos[a] = fmaxf(0.0f, fminf(1.0f - 1e-6f, pos[a]));
      const unsigned q0 = __float2uint_rz(pos[0] * 8388608.0f);
      const unsigned q1 = __float2uint_rz(pos[1] * 8388608.0f);
      const unsigned q2 = __float2uint_rz(pos[2] * 8388608.0f);
      int s = 0, node = 0;
      if (pdepth >= 0) {
        const unsigned diff = (q0 ^ pq0) | (q1 ^ pq1) | (q2 ^ pq2);
        const int c = diff ? __clz(int(diff << 9)) : 23;
        s = min(min(c, pdepth), CACHED - 1);
        int sel = path[0];
#pragma unroll
        for (int j = 1; j < PW; ++j)
          if (s / G == j) sel = path[j];
        node = __shfl_sync(mask, sel, s % G, G);
      }
      pq0 = q0;
      pq1 = q1;
      pq2 = q2;
      int k = s;
      idx = 0;
      bool leaf = false;
      for (; k <= 22; ++k) {
        const int sh = 22 - k;
        idx = unsigned(node) * 8u + ((((q0 >> sh) & 1u) << 2) | (((q1 >> sh) & 1u) << 1) | ((q2 >> sh) & 1u));
        const int skip = __ldg(T.child + idx);
        if (skip == 0) {
          leaf = true;
          break;
        }
        node += skip;
        if (l == (k + 1) % G) {
#pragma unroll
          for (int j = 0; j < PW; ++j)
            if ((k + 1) / G == j) path[j] = node;
        }
      }
      if (leaf) {
        pdepth = k;
        cube = __int_as_float((127 + k + 1) << 23);       // 2^(k+1)
        inv_cube = __int_as_float((127 - k - 1) << 23);   // 2^-(k+1), exact
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          const float sc = pos[a] * cube;
          pos[a] = sc - floorf(sc);
        }
      } else {
        // deeper than the 23 cached digits: finish with the plain walk from `node`
        pdepth = 22;
        cube = 8388608.0f;
        pow2 = false;   // the exit length below falls back to the division
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          const float sc = pos[a] * cube;
          pos[a] = sc - floorf(sc);
        }
        for (int level = 23; level < MAX_TREE_DEPTH; ++level) {
          int u[3];
#pragma unroll
          for (int a = 0; a < 3; ++a) {
            pos[a] = pos[a] * 2.0f;
            const float fl = floorf(pos[a]);
            u[a] = int(fl);
            pos[a] = pos[a] - fl;
          }
          cube = cube * 2.0f;
          idx = unsigned(node) * 8u + unsigned(u[0] * 4 + u[1] * 2 + u[2]);
          const int skip = __ldg(T.child + idx);
          if (skip == 0) break;
          node += skip;
        }
      }
    } else {
      idx = unsigned(query_leaf(T.child, T.N, pos, cube));
    }
    float smin, smax;
    dda_unit(pos, r.invd, smin, smax);
    // cube is a power of two for N = 2: multiplying by its (exact) reciprocal equals the IEEE division
    const float len = pow2 ? __fmul_rn(__fsub_rn(smax, smin), inv_cube) : __fsub_rn(smax, smin) / cube;
    delta_t = __fadd_rn(len, step);
    return idx;
  }
};

// ---- leaf fetch: the forward march's policy for where a leaf's sigma and coefficients live ---------------------
// issue() runs before the next leaf is located, finish() after it.  fp32 trees load everything in issue(); compressed
// trees load sigma, the retained coefficients and the palette indices in issue() and the palette entries in finish()
// (a dependent gather, so it waits for the indices while locate() runs).  Both produce fp32 coefficients that the
// shading arithmetic consumes unchanged: lane l owns basis functions l, l+G, ...
template <int KPL>
struct DenseFetch {
  __device__ __forceinline__ float issue(const TreeDev& T, unsigned idx, int l, float* c0, float* c1, float* c2) {
    const int K = T.K, D = T.D;
    const float* __restrict__ val = T.data + size_t(idx) * unsigned(D);
    const float sigma = __ldg(val + D - 1);
#pragma unroll
    for (int j = 0; j < KPL; ++j) {
      const int k = l + j * G;
      c0[j] = c1[j] = c2[j] = 0.f;
      if (k < K) {
        c0[j] = __ldg(val + k);
        c1[j] = __ldg(val + K + k);
        c2[j] = __ldg(val + 2 * K + k);
      }
    }
    return sigma;
  }
  __device__ __forceinline__ void finish(const TreeDev&, int, bool, float*, float*, float*) {}
};

template <int KPL>
struct QuantFetch {
  unsigned m[KPL];   // palette index of basis function l + j*G (palette-coded functions only)

  __device__ __forceinline__ float issue(const QuantTreeDev& T, unsigned idx, int l, float* c0, float* c1, float* c2) {
    const float sigma = __ldg(T.sigma + idx);
#pragma unroll
    for (int j = 0; j < KPL; ++j) {
      const int k = l + j * G;
      c0[j] = c1[j] = c2[j] = 0.f;
      m[j] = 0;
      if (k < T.retain) {
        const __half* p = T.retained + (unsigned long long)k * T.leaves * 3 + size_t(idx) * 3;
        c0[j] = __half2float(__ldg(p));
        c1[j] = __half2float(__ldg(p + 1));
        c2[j] = __half2float(__ldg(p + 2));
      } else if (k < T.K) {
        m[j] = __ldg(T.map + (unsigned long long)(k - T.retain) * T.leaves + idx);
      }
    }
    return sigma;
  }
  // `use`: the leaf contributes (sigma > sigma_thresh); the palette is only read for leaves that are shaded
  __device__ __forceinline__ void finish(const QuantTreeDev& T, int l, bool use, float* c0, float* c1, float* c2) {
    if (!use) return;
#pragma unroll
    for (int j = 0; j < KPL; ++j) {
      const int k = l + j * G;
      if (k >= T.retain && k < T.K) {
        const __half* p = T.palette + ((size_t)(k - T.retain) * unsigned(T.ncolors) + m[j]) * 3;
        c0[j] = __half2float(__ldg(p));
        c1[j] = __half2float(__ldg(p + 1));
        c2[j] = __half2float(__ldg(p + 2));
      }
    }
  }
};

template <class Tree, int KPL>
struct LeafFetch {
  using type = DenseFetch<KPL>;
};
template <int KPL>
struct LeafFetch<QuantTreeDev, KPL> {
  using type = QuantFetch<KPL>;
};

// the three colour channels' SH dot products basis . c of one leaf, summed over the lane group
template <int KPL>
__device__ __forceinline__ void sh_dot(const float* basis_l, const float* c0, const float* c1, const float* c2,
                                       unsigned mask, float& p0, float& p1, float& p2) {
  p0 = p1 = p2 = 0.f;
#pragma unroll
  for (int j = 0; j < KPL; ++j) {
    p0 += basis_l[j] * c0[j];
    p1 += basis_l[j] * c1[j];
    p2 += basis_l[j] * c2[j];
  }
  p0 = group_sum(p0, mask);
  p1 = group_sum(p1, mask);
  p2 = group_sum(p2, mask);
}

// ---- forward march of one ray by one lane group -------------------------------------------------------
// Software-pipelined: the loads of the current leaf (sigma and this lane's three coefficients, issued
// unconditionally; for a compressed tree the palette indices, then the palette entries once the next leaf is
// located) are in flight while the next leaf is located; the march itself never depends on the data.
//
// DEPTH = true also accumulates, over the contributing visits i (sigma_i > sigma_thresh; visit i starts at t_i, has
// step delta_t_i and weight w_i = T_i (1 - exp(-delta_t_i * delta_scale * sigma_i))):
//   dz[0] = depth = sum_i w_i z_i,  z_i = (t_i + delta_t_i / 2) * delta_scale   (midpoint of the visit's
//           constant-density segment, as a parameter along the caller's direction vector)
//   dz[1] = acc   = sum_i w_i                                                   (the background not included)
// Early termination rescales both by 1 / (1 - light) like the colour, so a stopped ray has acc = 1.  A ray that
// misses the box has depth = acc = 0.  The colour, the march and the counters are those of DEPTH = false.
// Tree = QuantTreeDev marches a compressed tree: only the leaf fetch differs (LeafFetch).
template <int KPL, bool DEPTH = false, class Tree = TreeDev>
__device__ __forceinline__ void trace_forward(const Tree& T, const Opts& O, const Ray& r, const float* basis_l, int l,
                                              unsigned mask, float* out, unsigned& visits, unsigned& hits,
                                              float* dz = nullptr) {
  if constexpr (DEPTH) dz[0] = dz[1] = 0.f;
  if (!r.hit) {
    out[0] = out[1] = out[2] = O.bg;
    return;
  }
  out[0] = out[1] = out[2] = 0.f;
  float light = 1.0f;
  float t = r.tmin;
  if (!(t < r.tmax)) {
    out[0] = out[1] = out[2] = O.bg;  // light = 1
    return;
  }
  Marcher m;
  m.init();
  float delta_t;
  unsigned idx = m.locate(T, r, O.step, t, l, mask, delta_t);
  for (int it = 0; it < MAX_MARCH_STEPS; ++it) {
    typename LeafFetch<Tree, KPL>::type fetch;
    float c0[KPL], c1[KPL], c2[KPL];  // lane l owns basis functions l, l+G, ...
    const float sigma = fetch.issue(T, idx, l, c0, c1, c2);
    const float t_next = t + delta_t;
    const bool more = t_next < r.tmax;
    float delta_n = 0.f;
    unsigned idx_n = 0;
    if (more) idx_n = m.locate(T, r, O.step, t_next, l, mask, delta_n);
    fetch.finish(T, l, sigma > O.sigma_thresh, c0, c1, c2);
    ++visits;
    if (sigma > O.sigma_thresh) {
      ++hits;
      const float att = __expf(-delta_t * r.delta_scale * sigma);
      const float weight = light * (1.0f - att);
      float p0, p1, p2;
      sh_dot<KPL>(basis_l, c0, c1, c2, mask, p0, p1, p2);
      out[0] += weight * sigmoidf(p0);
      out[1] += weight * sigmoidf(p1);
      out[2] += weight * sigmoidf(p2);
      if constexpr (DEPTH) {
        dz[0] += weight * ((t + 0.5f * delta_t) * r.delta_scale);
        dz[1] += weight;
      }
      light *= att;
      if (light <= O.stop_thresh) {
        const float scale = 1.0f / (1.0f - light);
        out[0] *= scale;
        out[1] *= scale;
        out[2] *= scale;
        if constexpr (DEPTH) {
          dz[0] *= scale;
          dz[1] *= scale;
        }
        return;
      }
    }
    if (!more) break;
    t = t_next;
    idx = idx_n;
    delta_t = delta_n;
  }
  out[0] += light * O.bg;
  out[1] += light * O.bg;
  out[2] += light * O.bg;
}

// ---- backward march: colour and density gradients in one pass ---------------------------------------
// accum enters as sum_j w_j (c_j . g) + T_end * bg * sum(g) = g . out (svox computes it with an extra march:
// trace_ray_backward pass 1); every contributing leaf then peels its own term off.
// DEPTH = true adds the upstream gradients gz = d loss / d depth and ga = d loss / d acc of trace_forward<DEPTH>: each
// visit's `total` gains z_i gz + ga (the value it composites into g . out + gz depth + ga acc, which the caller passes
// as accum) and only the sigma gradient changes, since depth and acc do not depend on the colour coefficients.
template <int KPL, bool DEPTH = false>
__device__ __forceinline__ void trace_backward(const TreeDev& T, const Opts& O, const Ray& r, const float* basis_l, int l,
                                               unsigned mask, const float* g, float accum,
                                               float* __restrict__ grad, float gz = 0.f, float ga = 0.f) {
  if (!r.hit) return;
  float light = 1.0f;
  float t = r.tmin;
  const int K = T.K, D = T.D;
  if (!(t < r.tmax)) return;
  Marcher m;
  m.init();
  float delta_t;
  unsigned idx = m.locate(T, r, O.step, t, l, mask, delta_t);
  for (int it = 0; it < MAX_MARCH_STEPS; ++it) {
    // DenseFetch::issue's loads, written out with K and D hoisted: calling DenseFetch here changes the generated code
    // of the KPL = 4 and 7 backward and training kernels
    const float* __restrict__ val = T.data + size_t(idx) * unsigned(D);
    const float sigma = __ldg(val + D - 1);
    float c0[KPL], c1[KPL], c2[KPL];  // lane l owns basis functions l, l+G, ...
#pragma unroll
    for (int j = 0; j < KPL; ++j) {
      const int k = l + j * G;
      c0[j] = c1[j] = c2[j] = 0.f;
      if (k < K) {
        c0[j] = __ldg(val + k);
        c1[j] = __ldg(val + K + k);
        c2[j] = __ldg(val + 2 * K + k);
      }
    }
    const float t_next = t + delta_t;
    const bool more = t_next < r.tmax;
    float delta_n = 0.f;
    unsigned idx_n = 0;
    if (more) idx_n = m.locate(T, r, O.step, t_next, l, mask, delta_n);
    if (sigma > 0.0f) {
      const float att = __expf(-delta_t * r.delta_scale * sigma);
      const float weight = light * (1.0f - att);
      float p0, p1, p2;
      sh_dot<KPL>(basis_l, c0, c1, c2, mask, p0, p1, p2);
      const float s0 = sigmoidf(p0), s1 = sigmoidf(p1), s2 = sigmoidf(p2);
      float* gv = grad + size_t(idx) * unsigned(D);
      const float t0 = weight * s0 * (1.0f - s0) * g[0];
      const float t1 = weight * s1 * (1.0f - s1) * g[1];
      const float t2 = weight * s2 * (1.0f - s2) * g[2];
#pragma unroll
      for (int j = 0; j < KPL; ++j) {
        const int k = l + j * G;
        if (k < K) {
          atomicAdd(gv + k, basis_l[j] * t0);
          atomicAdd(gv + K + k, basis_l[j] * t1);
          atomicAdd(gv + 2 * K + k, basis_l[j] * t2);
        }
      }
      float total = s0 * g[0] + s1 * g[1] + s2 * g[2];
      // (rounded separately: with gz = ga = 0 the colour's total keeps its bits)
      if constexpr (DEPTH) total = __fadd_rn(total, __fmaf_rn((t + 0.5f * delta_t) * r.delta_scale, gz, ga));
      light *= att;
      accum -= weight * total;
      if (l == 0) atomicAdd(gv + D - 1, delta_t * r.delta_scale * (total * light - accum));
    }
    if (!more) break;
    t = t_next;
    idx = idx_n;
    delta_t = delta_n;
  }
}

// ---- ray fetch: lane group -> ray index (pixel tiles for the perspective camera) --------------------------
// zscale (optional) receives the factor from a distance along the ray's direction vector to the reported depth:
// 1 for explicit rays, the camera-axis factor 1 / |(x, y, -1)| for a perspective pixel.  NDC = true turns a
// perspective pixel's ray into NDC (world_to_ndc) before the march; its view direction stays the world one.
template <bool NDC = false>
__device__ __forceinline__ bool fetch_ray(const RaySrc& S, const TreeDev& T, Ray& r, long long& out_index,
                                          float* zscale = nullptr, const Ndc& ndc = Ndc{}) {
  const int grp = threadIdx.x / G;
  float o[3], d[3];
  if (S.o != nullptr) {
    const long long i = (long long)blockIdx.x * RPB + grp;
    if (i >= S.n) return false;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      o[a] = __ldg(S.o + 3 * i + a);
      d[a] = __ldg(S.d + 3 * i + a);
    }
    float v[3] = {__ldg(S.v + 3 * i), __ldg(S.v + 3 * i + 1), __ldg(S.v + 3 * i + 2)};
    setup_ray(T.off, T.inv, o, d, v, r);
    out_index = i;
    if (zscale) *zscale = 1.0f;
    return true;
  }
  const int W = int(S.cam.width);
  const int tiles_x = (W + TILE_W - 1) / TILE_W;
  const int tx = blockIdx.x % tiles_x, ty = blockIdx.x / tiles_x;
  const int ix = tx * TILE_W + grp % TILE_W;
  const int iyl = ty * TILE_H + grp / TILE_W;  // row inside the slab
  if (ix >= W || iyl >= S.nrows) return false;
  const float nrm = cam_ray(S.cam, ix, S.row0 + iyl, o, d);
  if constexpr (NDC) {
    const float v[3] = {d[0], d[1], d[2]};
    world_to_ndc(ndc, o, d);
    setup_ray(T.off, T.inv, o, d, v, r);
  } else {
    setup_ray(T.off, T.inv, o, d, d, r);
  }
  out_index = (long long)iyl * W + ix;
  if (zscale) *zscale = 1.0f / nrm;
  return true;
}

template <int KPL>
__device__ __forceinline__ void lane_basis(const TreeDev& T, const Ray& r, int l, float* bl) {
  if (T.rgba) {
#pragma unroll
    for (int j = 0; j < KPL; ++j) bl[j] = 1.0f;
    return;
  }
  float b[25];
  const int deg = T.K >= 25 ? 4 : T.K >= 16 ? 3 : T.K >= 9 ? 2 : T.K >= 4 ? 1 : 0;
  sh_basis(deg, r.vdir[0], r.vdir[1], r.vdir[2], b);
#pragma unroll
  for (int j = 0; j < KPL; ++j) {
    const int want = l + j * G;
    float v = 0.f;
#pragma unroll
    for (int k = 0; k < 25; ++k)
      if (k == want && k < T.K) v = b[k];
    bl[j] = v;
  }
}

// DEPTH = true also stores depth [n] (times fetch_ray's zscale) and acc [n] (trace_forward<DEPTH>); Tree = QuantTreeDev
// renders a compressed tree
template <int KPL, bool DEPTH = false, class Tree = TreeDev>
__global__ void __launch_bounds__(256) octree_render_kernel(Tree T, Opts O, RaySrc S, float* __restrict__ out_rgb,
                                                            unsigned long long* __restrict__ counters,
                                                            float* __restrict__ out_depth, float* __restrict__ out_acc) {
  Ray r;
  long long oi;
  float zscale;
  if (!fetch_ray(S, T, r, oi, DEPTH ? &zscale : nullptr)) return;
  const int l = threadIdx.x % G;
  const unsigned mask = group_mask();
  float bl[KPL];
  lane_basis<KPL>(T, r, l, bl);
  float out[3], dz[2];
  unsigned visits = 0, hits = 0;
  trace_forward<KPL, DEPTH, Tree>(T, O, r, bl, l, mask, out, visits, hits, dz);
  if (l < 3) out_rgb[3 * oi + l] = l == 0 ? out[0] : l == 1 ? out[1] : out[2];
  if constexpr (DEPTH) {
    if (l == 0) {
      out_depth[oi] = dz[0] * zscale;
      out_acc[oi] = dz[1];
    }
  }
  if (counters != nullptr && l == 0) {
    atomicAdd(counters + 0, (unsigned long long)visits);
    atomicAdd(counters + 1, (unsigned long long)hits);
  }
}

// VolumeRenderer backward for an upstream gradient d loss / d rgb  (svox trace_ray_backward).  DEPTH = true adds
// d loss / d depth and d loss / d acc of octree_render_kernel<DEPTH>; each of the three gradient arrays may be null
// (zero).
template <int KPL, bool DEPTH = false>
__global__ void __launch_bounds__(256) octree_backward_kernel(TreeDev T, Opts O, RaySrc S,
                                                              const float* __restrict__ grad_out,
                                                              float* __restrict__ grad_data,
                                                              const float* __restrict__ grad_depth,
                                                              const float* __restrict__ grad_acc) {
  Ray r;
  long long oi;
  float zscale;
  if (!fetch_ray(S, T, r, oi, DEPTH ? &zscale : nullptr)) return;
  const int l = threadIdx.x % G;
  const unsigned mask = group_mask();
  float bl[KPL];
  lane_basis<KPL>(T, r, l, bl);
  float out[3], dz[2];
  unsigned visits = 0, hits = 0;
  Opts Of = O;
  Of.sigma_thresh = 0.f;
  Of.stop_thresh = 0.f;
  trace_forward<KPL, DEPTH>(T, Of, r, bl, l, mask, out, visits, hits, dz);
  if constexpr (!DEPTH) {
    float g[3] = {__ldg(grad_out + 3 * oi), __ldg(grad_out + 3 * oi + 1), __ldg(grad_out + 3 * oi + 2)};
    const float accum = g[0] * out[0] + g[1] * out[1] + g[2] * out[2];
    trace_backward<KPL>(T, Of, r, bl, l, mask, g, accum, grad_data);
  } else {
    float g[3] = {0.f, 0.f, 0.f};
    if (grad_out != nullptr)
      for (int c = 0; c < 3; ++c) g[c] = __ldg(grad_out + 3 * oi + c);
    // the reported depth is zscale * sum_i w_i z_i: its gradient reaches the march's z_i through zscale
    const float gz = grad_depth != nullptr ? __ldg(grad_depth + oi) * zscale : 0.f;
    const float ga = grad_acc != nullptr ? __ldg(grad_acc + oi) : 0.f;
    float accum = g[0] * out[0] + g[1] * out[1] + g[2] * out[2];
    accum = __fadd_rn(accum, __fmaf_rn(gz, dz[0], ga * dz[1]));
    trace_backward<KPL, true>(T, Of, r, bl, l, mask, g, accum, grad_data, gz, ga);
  }
}

// One training pass over a camera slab (octree/optimization.py:201-207 minus the optimiser):
//   im = render_persp(c2w); mse = mean((clamp(im,0,1) - gt)^2); mse.backward()
// g = grad_scale * 2 * (clamp(im) - gt) inside the clamp range, 0 outside (torch.clamp's gradient).
// NDC = true marches the slab's rays in NDC (fetch_ray<NDC>, svox VolumeRenderer(ndc=...)); ndc is unused otherwise.
template <int KPL, bool NDC = false>
__global__ void __launch_bounds__(256) octree_train_kernel(TreeDev T, Opts O, RaySrc S, const float* __restrict__ gt,
                                                           float grad_scale, float* __restrict__ grad_data,
                                                           double* __restrict__ sq_err_sum,
                                                           float* __restrict__ out_rgb, Ndc ndc) {
  Ray r;
  long long oi;
  const bool have = fetch_ray<NDC>(S, T, r, oi, nullptr, ndc);
  float err = 0.f;
  if (have) {
    const int l = threadIdx.x % G;
    const unsigned mask = group_mask();
    float bl[KPL];
    lane_basis<KPL>(T, r, l, bl);
    float out[3];
    unsigned visits = 0, hits = 0;
    trace_forward<KPL>(T, O, r, bl, l, mask, out, visits, hits);
    float g[3];
    float accum = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float cl = fminf(fmaxf(out[c], 0.0f), 1.0f);
      const float diff = cl - __ldg(gt + 3 * oi + c);
      err += diff * diff;
      g[c] = (out[c] >= 0.0f && out[c] <= 1.0f) ? grad_scale * (2.0f * diff) : 0.0f;
      accum += g[c] * out[c];
    }
    if (out_rgb != nullptr && l < 3) out_rgb[3 * oi + l] = l == 0 ? out[0] : l == 1 ? out[1] : out[2];
    if (g[0] != 0.f || g[1] != 0.f || g[2] != 0.f) trace_backward<KPL>(T, O, r, bl, l, mask, g, accum, grad_data);
    if (l != 0) err = 0.f;
  }
  // CTA reduction of the squared error (one double atomic per CTA)
  __shared__ float s_err[8];
  __syncwarp();
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) err += __shfl_xor_sync(0xffffffffu, err, s);
  if ((threadIdx.x & 31) == 0) s_err[threadIdx.x >> 5] = err;
  __syncthreads();
  if (threadIdx.x == 0 && sq_err_sum != nullptr) {
    float tot = 0.f;
    for (int w = 0; w < 8; ++w) tot += s_err[w];
    atomicAdd(sq_err_sum, double(tot));
  }
}

// torch.optim.SGD(momentum=0).step() + zero_grad fused: data -= lr * grad; grad = 0 (octree/optimization.py:205-208)
__global__ void octree_sgd_kernel(float* __restrict__ data, float* __restrict__ grad, long long n, float lr) {
  const long long n4 = n / 4;
  const long long stride = (long long)gridDim.x * blockDim.x;
  float4* d4 = reinterpret_cast<float4*>(data);
  float4* g4 = reinterpret_cast<float4*>(grad);
  // four independent 16-byte gradient loads in flight per thread (the pass is a pure HBM stream)
  for (long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x; i0 < n4; i0 += 4 * stride) {
    float4 g[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long i = i0 + u * stride;
      g[u] = i < n4 ? __ldcs(g4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long i = i0 + u * stride;
      if (g[u].x != 0.f || g[u].y != 0.f || g[u].z != 0.f || g[u].w != 0.f) {
        float4 d = d4[i];
        d.x = d.x - lr * g[u].x;
        d.y = d.y - lr * g[u].y;
        d.z = d.z - lr * g[u].z;
        d.w = d.w - lr * g[u].w;
        d4[i] = d;
        g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  }
  for (long long i = n4 * 4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float g = grad[i];
    if (g != 0.f) {
      data[i] = data[i] - lr * g;
      grad[i] = 0.f;
    }
  }
}

// One element of torch.optim.SGD(lr, momentum=mu, dampening=0, nesterov): b <- mu*b + g with two roundings, as torch's
// buf.mul_(mu).add_(g) (a zero buffer gives fl(fl(mu*0) + g) = g, torch's first-step clone(g)); the direction
// d = nesterov ? g + mu*b : b (one FMA, torch's grad.add(buf, alpha=mu)); data <- data - lr*d (one FMA).
__device__ __forceinline__ void sgd_momentum_elem(float& data, float g, float& b, float lr, float mu, bool nesterov) {
  b = __fadd_rn(__fmul_rn(mu, b), g);
  const float d = nesterov ? __fmaf_rn(mu, b, g) : b;
  data = __fmaf_rn(-lr, d, data);
}

// The SGD-with-momentum step fused with zero_grad (octree/optimization.py:180-181,205-208).  Elements with g = 0 and
// b = 0 are only read (g, b) and keep their bits; elements with g = 0 and b != 0 still move.  Up to 28 B per element
// (read g, b, data; write data, b, g) against the plain step's 16 B.
__global__ void octree_sgd_momentum_kernel(float* __restrict__ data, float* __restrict__ grad, float* __restrict__ buf,
                                           long long n, float lr, float mu, bool nesterov) {
  const long long n4 = n / 4;
  const long long stride = (long long)gridDim.x * blockDim.x;
  float4* d4 = reinterpret_cast<float4*>(data);
  float4* g4 = reinterpret_cast<float4*>(grad);
  float4* b4 = reinterpret_cast<float4*>(buf);
  // four independent 16-byte loads of g and of b in flight per thread, as in octree_sgd_kernel
  for (long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x; i0 < n4; i0 += 4 * stride) {
    float4 g[4], b[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long i = i0 + u * stride;
      g[u] = i < n4 ? __ldcs(g4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
      b[u] = i < n4 ? __ldcs(b4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long i = i0 + u * stride;
      const bool gx = g[u].x != 0.f, gy = g[u].y != 0.f, gz = g[u].z != 0.f, gw = g[u].w != 0.f;
      const bool mx = gx || b[u].x != 0.f, my = gy || b[u].y != 0.f, mz = gz || b[u].z != 0.f,
                 mw = gw || b[u].w != 0.f;
      if (mx || my || mz || mw) {
        float4 d = d4[i];
        float4 bb = b[u];
        if (mx) sgd_momentum_elem(d.x, g[u].x, bb.x, lr, mu, nesterov);
        if (my) sgd_momentum_elem(d.y, g[u].y, bb.y, lr, mu, nesterov);
        if (mz) sgd_momentum_elem(d.z, g[u].z, bb.z, lr, mu, nesterov);
        if (mw) sgd_momentum_elem(d.w, g[u].w, bb.w, lr, mu, nesterov);
        d4[i] = d;
        b4[i] = bb;
        if (gx || gy || gz || gw) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  }
  for (long long i = n4 * 4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float g = grad[i];
    float b = buf[i];
    if (g != 0.f || b != 0.f) {
      float d = data[i];
      sgd_momentum_elem(d, g, b, lr, mu, nesterov);
      data[i] = d;
      buf[i] = b;
      if (g != 0.f) grad[i] = 0.f;
    }
  }
}

// N3Tree.__getitem__(points) (svox query_vertical): world points -> packed leaf index node*N^3 + (i*N+j)*N+k
__global__ void octree_query_kernel(TreeDev T, const float* __restrict__ pts, long long n, long long* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float pos[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) pos[a] = __fadd_rn(T.off[a], __fmul_rn(T.inv[a], __ldg(pts + 3 * i + a)));
  float cube;
  out[i] = query_leaf(T.child, T.N, pos, cube);
}

// svox grid_trace_ray for every pixel of every camera in ONE launch; weights are max-reduced straight into the
// output grid (the reference keeps a per-camera grid and runs torch.max over 2^27 voxels per camera,
// octree/extraction.py:199-212).  Weights are >= 0, so the float max is an integer atomicMax on the bit pattern.
// NDC = true marches every pixel's ray in NDC (octree/extraction.py:187-193, opts.ndc_*); ndc is unused otherwise.
template <bool NDC = false>
__global__ void __launch_bounds__(256) grid_weight_kernel(const float* __restrict__ sigma, int reso, const Cam* __restrict__ cams,
                                                          float off0, float off1, float off2, float inv0, float inv1,
                                                          float inv2, Opts O, float* __restrict__ wmax,
                                                          uint8_t* __restrict__ hit, Ndc ndc) {
  const Cam c = cams[blockIdx.y];
  const int W = int(c.width), H = int(c.height);
  const int tiles_x = (W + 15) / 16;
  const int ix = (blockIdx.x % tiles_x) * 16 + (threadIdx.x & 15);
  const int iy = (blockIdx.x / tiles_x) * 16 + (threadIdx.x >> 4);
  if (ix >= W || iy >= H) return;
  float o[3], d[3];
  cam_ray(c, ix, iy, o, d);
  if constexpr (NDC) world_to_ndc(ndc, o, d);
  const float off[3] = {off0, off1, off2}, inv[3] = {inv0, inv1, inv2};
  Ray r;
  setup_ray(off, inv, o, d, d, r);
  if (!r.hit) return;
  float light = 1.0f;
  float t = r.tmin;
  const float fres = float(reso);
  for (int it = 0; t < r.tmax && it < MAX_MARCH_STEPS; ++it) {
    float pos[3];
    int u[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      pos[a] = __fadd_rn(r.o[a], __fmul_rn(t, r.d[a]));
      pos[a] = fmaxf(0.0f, fminf(1.0f - 1e-6f, pos[a]));
      pos[a] = __fmul_rn(pos[a], fres);
      const float fl = floorf(pos[a]);
      u[a] = int(fl);
      pos[a] = __fsub_rn(pos[a], fl);
    }
    float smin, smax;
    dda_unit(pos, r.invd, smin, smax);
    const float delta_t = __fadd_rn(__fsub_rn(smax, smin) / fres, O.step);
    const long long idx = ((long long)u[0] * reso + u[1]) * reso + u[2];
    const float s = __ldg(sigma + idx);
    if (s > O.sigma_thresh) {
      const float att = __expf(-delta_t * r.delta_scale * s);
      const float weight = light * (1.0f - att);
      light *= att;
      if (weight > wmax[idx]) atomicMax(reinterpret_cast<int*>(wmax + idx), __float_as_int(weight));
      if (hit != nullptr) hit[idx] = 1;
      if (light <= O.stop_thresh) return;
    }
    t += delta_t;
  }
}

// The NDC rays of explicit world rays (S.o != null: origins / dirs / vdirs) or of a perspective camera's pixel-row
// slab (row-major, the pixel order of fetch_ray), one thread per ray: origins and unit directions in NDC
// (world_to_ndc), view directions copied (explicit) or the pixel's unit world direction.  The explicit-ray entry
// points march them unchanged.
__global__ void __launch_bounds__(256) ndc_rays_kernel(RaySrc S, Ndc ndc, float* __restrict__ out_o,
                                                       float* __restrict__ out_d, float* __restrict__ out_v) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S.n) return;
  float o[3], d[3], v[3];
  if (S.o != nullptr) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      o[a] = __ldg(S.o + 3 * i + a);
      d[a] = __ldg(S.d + 3 * i + a);
      v[a] = __ldg(S.v + 3 * i + a);
    }
  } else {
    const int W = int(S.cam.width);
    cam_ray(S.cam, int(i % W), S.row0 + int(i / W), o, d);
#pragma unroll
    for (int a = 0; a < 3; ++a) v[a] = d[a];
  }
  world_to_ndc(ndc, o, d);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    out_o[3 * i + a] = o[a];
    out_d[3 * i + a] = d[a];
    out_v[3 * i + a] = v[a];
  }
}

}  // namespace
}  // namespace pob

// ---------------------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------------------
namespace {

using namespace pob;

// The geometry both tree formats share: branch factor, node count, the 32-bit leaf index, basis_dim per format,
// offset and invradius.  rgba_msg is the format's message for an RGBA tree whose basis_dim is not 1.
template <class Desc>
int tree_geometry(const char* where, const Desc* t, const char* rgba_msg, TreeDev& T) {
  if (t->N < 2 || t->N > 8) return pob_fail(where, "tree branch factor N must be in [2, 8]");
  if (t->n_nodes < 1) return pob_fail(where, "tree has no nodes");
  if (double(t->n_nodes) * t->N * t->N * t->N >= 4294967296.0) return pob_fail(where, "tree too large (leaf index must fit 32 bits)");
  const int K = t->basis_dim;
  if (t->format == POB_OCTREE_RGBA) {
    if (K != 1) return pob_fail(where, rgba_msg);
  } else if (t->format == POB_OCTREE_SH) {
    if (!(K == 1 || K == 4 || K == 9 || K == 16 || K == 25)) return pob_fail(where, "SH basis_dim must be 1,4,9,16,25");
  } else {
    return pob_fail(where, "unsupported data format (RGBA and SH only; SG is out of scope)");
  }
  T.child = t->child_dev;
  T.N = t->N;
  T.K = K;
  T.rgba = t->format == POB_OCTREE_RGBA;
  for (int a = 0; a < 3; ++a) {
    T.off[a] = t->offset[a];
    T.inv[a] = t->invradius[a];
  }
  return 0;
}

int tree_dev(const char* where, const pob_octree* t, TreeDev& T) {
  if (!t) return pob_fail(where, "tree is NULL");
  if (!t->data_dev || !t->child_dev) return pob_fail(where, "tree data/child pointer is NULL");
  if (int rc = tree_geometry(where, t, "RGBA trees have data_dim 4", T)) return rc;
  if (T.rgba && t->data_dim != 4) return pob_fail(where, "RGBA trees have data_dim 4");
  if (!T.rgba && t->data_dim != 3 * T.K + 1) return pob_fail(where, "data_dim must be 3*basis_dim + 1 (sigma last)");
  T.data = t->data_dev;
  T.D = t->data_dim;
  if (!pob_sms_or_fail(where)) return 1;
  return 0;
}

int tree_dev(const char* where, const pob_octree_quant* t, QuantTreeDev& T) {
  if (!t) return pob_fail(where, "tree is NULL");
  if (!t->child_dev || !t->sigma_dev) return pob_fail(where, "tree child/sigma pointer is NULL");
  if (int rc = tree_geometry(where, t, "RGBA trees have basis_dim 1", T)) return rc;
  if (t->bits < 1 || t->bits > 16) return pob_fail(where, "bits must be in [1, 16] (palette indices are uint16)");
  if (t->retain < 0 || t->retain > T.K) return pob_fail(where, "retain must be in [0, basis_dim]");
  if (t->retain > 0 && !t->retained_dev) return pob_fail(where, "retained pointer is NULL with retain > 0");
  if (t->retain < T.K && (!t->map_dev || !t->palette_dev))
    return pob_fail(where, "map/palette pointer is NULL with retain < basis_dim");
  T.data = nullptr;
  T.D = 0;
  T.sigma = t->sigma_dev;
  T.map = t->map_dev;
  T.palette = reinterpret_cast<const __half*>(t->palette_dev);
  T.retained = reinterpret_cast<const __half*>(t->retained_dev);
  T.retain = t->retain;
  T.ncolors = 1 << t->bits;
  T.leaves = (unsigned long long)t->n_nodes * t->N * t->N * t->N;
  if (!pob_sms_or_fail(where)) return 1;
  return 0;
}

int opts_dev(const char* where, const pob_octree_opts* o, Opts& O) {
  if (!o) return pob_fail(where, "options are NULL");
  // every march iteration advances by at least step_size (unit cube): below sqrt(3) / MAX_MARCH_STEPS a diagonal ray
  // would run into the iteration cap and composite the background through the unmarched remainder
  if (!(o->step_size >= 2e-6f))
    return pob_fail(where, "step_size must be >= 2e-6 (the march is capped at 2^20 iterations per ray)");
  O.step = o->step_size;
  O.bg = o->background_brightness;
  O.sigma_thresh = o->sigma_thresh;
  O.stop_thresh = o->stop_thresh;
  return 0;
}

int ndc_dev(const char* where, const pob_ndc* n, Ndc& N) {
  if (!n) return pob_fail(where, "NDC description is NULL");
  if (!(n->width > 0.f && n->height > 0.f && n->focal > 0.f) || !isfinite(n->width) || !isfinite(n->height) ||
      !isfinite(n->focal))
    return pob_fail(where, "NDC width, height and focal must be finite and > 0");
  N.width = n->width;
  N.height = n->height;
  N.focal = n->focal;
  return 0;
}

// explicit rays (cam NULL) or a camera's pixel-row slab; blocks = the march grid (fetch_ray's RPB rays or
// TILE_W x TILE_H pixels per CTA)
int ray_src(const char* where, const float* o, const float* d, const float* v, long long n, const pob_camera* cam,
            int row0, int nrows, RaySrc& S, unsigned& blocks) {
  S.o = o;
  S.d = d;
  S.v = v;
  S.row0 = 0;
  S.nrows = 0;
  S.n = n;
  if (cam == nullptr) {
    if (!o || !d || !v) return pob_fail(where, "ray pointers are NULL");
    if (n < 0) return pob_fail(where, "negative ray count");
    blocks = unsigned((n + RPB - 1) / RPB);
    return 0;
  }
  S.o = S.d = S.v = nullptr;
  for (int i = 0; i < 12; ++i) S.cam.c2w[i] = cam->c2w[i];
  S.cam.fx = cam->fx;
  S.cam.fy = cam->fy;
  S.cam.width = cam->width;
  S.cam.height = cam->height;
  const int W = int(cam->width), H = int(cam->height);
  if (W < 1 || H < 1 || !(cam->fx > 0.f) || !(cam->fy > 0.f)) return pob_fail(where, "bad camera");
  if (row0 < 0 || nrows < 0 || row0 + nrows > H) return pob_fail(where, "pixel-row slab outside the image");
  S.row0 = row0;
  S.nrows = nrows;
  S.n = (long long)nrows * W;
  blocks = unsigned(((W + TILE_W - 1) / TILE_W) * ((nrows + TILE_H - 1) / TILE_H));
  return 0;
}

// What a march launch needs: the tree (TreeDev or QuantTreeDev), the options, the rays, the grid and the stream
template <class Tree>
struct March {
  Tree T;
  Opts O;
  RaySrc S;
  unsigned blocks = 0;
  cudaStream_t st;
};

struct NoChecks {
  int operator()() const { return 0; }
};

// Validates the tree, the options, the caller's own `checks` (which may read M.T and M.O) and the ray source, and
// reports the first failure in that order.
template <class Desc, class Tree, class Checks = NoChecks>
int march_setup(const char* W, const Desc* tree, const pob_octree_opts* opts, const float* origins_dev,
                const float* dirs_dev, const float* vdirs_dev, long long n_rays, const pob_camera* cam, int row0,
                int nrows, void* stream, March<Tree>& M, Checks checks = {}) {
  if (int rc = tree_dev(W, tree, M.T)) return rc;
  if (int rc = opts_dev(W, opts, M.O)) return rc;
  if (int rc = checks()) return rc;
  if (int rc = ray_src(W, origins_dev, dirs_dev, vdirs_dev, n_rays, cam, row0, nrows, M.S, M.blocks)) return rc;
  M.st = (cudaStream_t)stream;
  return 0;
}

// launch(integral_constant KPL) launches the march kernel for the tree's basis functions per lane (K = basis_dim,
// lane l owns l, l+G, ...); an empty grid launches nothing
template <class Tree, class F>
int march_launch(const char* W, const March<Tree>& M, F&& launch) {
  using std::integral_constant;
  if (M.blocks == 0) return 0;
  pob_count_launch();
  const int K = M.T.K;
  if (K <= 4) launch(integral_constant<int, 1>());
  else if (K <= 12) launch(integral_constant<int, 3>());
  else if (K <= 16) launch(integral_constant<int, 4>());
  else launch(integral_constant<int, 7>());
  POB_CUDA(W, cudaGetLastError());
  return 0;
}

// pob_octree_train_persp (ndc NULL) / pob_octree_train_persp_ndc
int train_persp(const char* W, const pob_octree* tree, const pob_octree_opts* opts, const pob_camera* cam,
                const pob_ndc* ndc, int row0, int nrows, const float* gt_rgb_dev, float grad_scale,
                float* grad_data_dev, double* sq_err_sum_dev, float* out_rgb_dev, void* stream) {
  March<TreeDev> M;
  Ndc N{};
  const auto checks = [&] {
    if (ndc != nullptr)
      if (int rc = ndc_dev(W, ndc, N)) return rc;
    if (!cam) return pob_fail(W, "camera is NULL");
    if (M.O.sigma_thresh != 0.f || M.O.stop_thresh != 0.f)
      return pob_fail(W, "training renders with sigma_thresh = stop_thresh = 0 (svox fast=False)");
    return 0;
  };
  if (int rc = march_setup(W, tree, opts, nullptr, nullptr, nullptr, 0, cam, row0, nrows, stream, M, checks)) return rc;
  if (!gt_rgb_dev || !grad_data_dev) return pob_fail(W, "gt / gradient pointer is NULL");
  return march_launch(W, M, [&](auto kpl) {
    if (ndc == nullptr)
      octree_train_kernel<decltype(kpl)::value, false><<<M.blocks, 256, 0, M.st>>>(
          M.T, M.O, M.S, gt_rgb_dev, grad_scale, grad_data_dev, sq_err_sum_dev, out_rgb_dev, N);
    else
      octree_train_kernel<decltype(kpl)::value, true><<<M.blocks, 256, 0, M.st>>>(
          M.T, M.O, M.S, gt_rgb_dev, grad_scale, grad_data_dev, sq_err_sum_dev, out_rgb_dev, N);
  });
}

// pob_grid_weight_render (ndc NULL) / pob_grid_weight_render_ndc
int grid_weights(const char* W, const float* sigma_grid_dev, int reso, const pob_camera* cams_dev, int n_cams,
                 int max_width, int max_height, const float offset[3], const float invradius[3],
                 const pob_octree_opts* opts, const pob_ndc* ndc, float* max_weight_dev, uint8_t* hit_dev,
                 void* stream) {
  Opts O;
  Ndc N{};
  if (int rc = opts_dev(W, opts, O)) return rc;
  if (ndc != nullptr)
    if (int rc = ndc_dev(W, ndc, N)) return rc;
  if (!sigma_grid_dev || !cams_dev || !max_weight_dev) return pob_fail(W, "NULL pointer");
  if (reso < 1 || reso > 2048) return pob_fail(W, "reso must be in [1, 2048]");
  if (n_cams < 0 || n_cams > 65535) return pob_fail(W, "n_cams must be in [0, 65535] per call");
  if (max_width < 1 || max_height < 1) return pob_fail(W, "bad image size");
  if (!pob_sms_or_fail(W)) return 1;
  if (n_cams == 0) return 0;
  dim3 grid(unsigned(((max_width + 15) / 16) * ((max_height + 15) / 16)), unsigned(n_cams));
  pob_count_launch();
  const Cam* cams = reinterpret_cast<const Cam*>(cams_dev);
  if (ndc == nullptr)
    grid_weight_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(
        sigma_grid_dev, reso, cams, offset[0], offset[1], offset[2], invradius[0], invradius[1], invradius[2], O,
        max_weight_dev, hit_dev, N);
  else
    grid_weight_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(
        sigma_grid_dev, reso, cams, offset[0], offset[1], offset[2], invradius[0], invradius[1], invradius[2], O,
        max_weight_dev, hit_dev, N);
  POB_CUDA(W, cudaGetLastError());
  return 0;
}

}  // namespace

extern "C" {

int pob_ndc_rays(const pob_ndc* ndc, const float* origins_dev, const float* dirs_dev, const float* vdirs_dev,
                 int64_t n_rays, const pob_camera* cam, int row0, int nrows, float* out_origins_dev,
                 float* out_dirs_dev, float* out_vdirs_dev, void* stream) {
  const char* W = "pob_ndc_rays";
  Ndc N;
  RaySrc S;
  unsigned tiles = 0;
  if (int rc = ndc_dev(W, ndc, N)) return rc;
  if (int rc = ray_src(W, origins_dev, dirs_dev, vdirs_dev, n_rays, cam, row0, nrows, S, tiles)) return rc;
  if (!out_origins_dev || !out_dirs_dev || !out_vdirs_dev) return pob_fail(W, "output pointer is NULL");
  if (!pob_sms_or_fail(W)) return 1;
  if (S.n == 0) return 0;
  pob_count_launch();
  ndc_rays_kernel<<<unsigned((S.n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(S, N, out_origins_dev, out_dirs_dev,
                                                                                 out_vdirs_dev);
  POB_CUDA(W, cudaGetLastError());
  return 0;
}

int pob_octree_render_quant(const pob_octree_quant* tree, const pob_octree_opts* opts, const float* origins_dev,
                            const float* dirs_dev, const float* vdirs_dev, int64_t n_rays, const pob_camera* cam,
                            int row0, int nrows, float* out_rgb_dev, unsigned long long* counters_dev, void* stream) {
  const char* W = "pob_octree_render_quant";
  March<QuantTreeDev> M;
  if (int rc = march_setup(W, tree, opts, origins_dev, dirs_dev, vdirs_dev, n_rays, cam, row0, nrows, stream, M))
    return rc;
  if (!out_rgb_dev) return pob_fail(W, "output pointer is NULL");
  return march_launch(W, M, [&](auto kpl) {
    octree_render_kernel<decltype(kpl)::value, false, QuantTreeDev><<<M.blocks, 256, 0, M.st>>>(
        M.T, M.O, M.S, out_rgb_dev, counters_dev, nullptr, nullptr);
  });
}

int pob_octree_render_depth_quant(const pob_octree_quant* tree, const pob_octree_opts* opts, const float* origins_dev,
                                  const float* dirs_dev, const float* vdirs_dev, int64_t n_rays,
                                  const pob_camera* cam, int row0, int nrows, float* out_rgb_dev,
                                  float* out_depth_dev, float* out_acc_dev, unsigned long long* counters_dev,
                                  void* stream) {
  const char* W = "pob_octree_render_depth_quant";
  March<QuantTreeDev> M;
  if (int rc = march_setup(W, tree, opts, origins_dev, dirs_dev, vdirs_dev, n_rays, cam, row0, nrows, stream, M))
    return rc;
  if (!out_rgb_dev || !out_depth_dev || !out_acc_dev) return pob_fail(W, "output pointer is NULL");
  return march_launch(W, M, [&](auto kpl) {
    octree_render_kernel<decltype(kpl)::value, true, QuantTreeDev><<<M.blocks, 256, 0, M.st>>>(
        M.T, M.O, M.S, out_rgb_dev, counters_dev, out_depth_dev, out_acc_dev);
  });
}

int pob_octree_render(const pob_octree* tree, const pob_octree_opts* opts, const float* origins_dev,
                      const float* dirs_dev, const float* vdirs_dev, int64_t n_rays, const pob_camera* cam,
                      int row0, int nrows, float* out_rgb_dev, unsigned long long* counters_dev, void* stream) {
  const char* W = "pob_octree_render";
  March<TreeDev> M;
  if (int rc = march_setup(W, tree, opts, origins_dev, dirs_dev, vdirs_dev, n_rays, cam, row0, nrows, stream, M))
    return rc;
  if (!out_rgb_dev) return pob_fail(W, "output pointer is NULL");
  return march_launch(W, M, [&](auto kpl) {
    octree_render_kernel<decltype(kpl)::value><<<M.blocks, 256, 0, M.st>>>(M.T, M.O, M.S, out_rgb_dev, counters_dev,
                                                                           nullptr, nullptr);
  });
}

int pob_octree_render_depth(const pob_octree* tree, const pob_octree_opts* opts, const float* origins_dev,
                            const float* dirs_dev, const float* vdirs_dev, int64_t n_rays, const pob_camera* cam,
                            int row0, int nrows, float* out_rgb_dev, float* out_depth_dev, float* out_acc_dev,
                            unsigned long long* counters_dev, void* stream) {
  const char* W = "pob_octree_render_depth";
  March<TreeDev> M;
  if (int rc = march_setup(W, tree, opts, origins_dev, dirs_dev, vdirs_dev, n_rays, cam, row0, nrows, stream, M))
    return rc;
  if (!out_rgb_dev || !out_depth_dev || !out_acc_dev) return pob_fail(W, "output pointer is NULL");
  return march_launch(W, M, [&](auto kpl) {
    octree_render_kernel<decltype(kpl)::value, true><<<M.blocks, 256, 0, M.st>>>(M.T, M.O, M.S, out_rgb_dev,
                                                                                 counters_dev, out_depth_dev,
                                                                                 out_acc_dev);
  });
}

int pob_octree_render_backward(const pob_octree* tree, const pob_octree_opts* opts, const float* origins_dev,
                               const float* dirs_dev, const float* vdirs_dev, int64_t n_rays, const pob_camera* cam,
                               int row0, int nrows, const float* grad_out_dev, float* grad_data_dev, void* stream) {
  const char* W = "pob_octree_render_backward";
  March<TreeDev> M;
  if (int rc = march_setup(W, tree, opts, origins_dev, dirs_dev, vdirs_dev, n_rays, cam, row0, nrows, stream, M))
    return rc;
  if (!grad_out_dev || !grad_data_dev) return pob_fail(W, "gradient pointer is NULL");
  return march_launch(W, M, [&](auto kpl) {
    octree_backward_kernel<decltype(kpl)::value><<<M.blocks, 256, 0, M.st>>>(M.T, M.O, M.S, grad_out_dev,
                                                                             grad_data_dev, nullptr, nullptr);
  });
}

int pob_octree_render_depth_backward(const pob_octree* tree, const pob_octree_opts* opts, const float* origins_dev,
                                     const float* dirs_dev, const float* vdirs_dev, int64_t n_rays,
                                     const pob_camera* cam, int row0, int nrows, const float* grad_rgb_dev,
                                     const float* grad_depth_dev, const float* grad_acc_dev, float* grad_data_dev,
                                     void* stream) {
  const char* W = "pob_octree_render_depth_backward";
  March<TreeDev> M;
  if (int rc = march_setup(W, tree, opts, origins_dev, dirs_dev, vdirs_dev, n_rays, cam, row0, nrows, stream, M))
    return rc;
  if (!grad_data_dev) return pob_fail(W, "gradient pointer is NULL");
  return march_launch(W, M, [&](auto kpl) {
    octree_backward_kernel<decltype(kpl)::value, true><<<M.blocks, 256, 0, M.st>>>(
        M.T, M.O, M.S, grad_rgb_dev, grad_data_dev, grad_depth_dev, grad_acc_dev);
  });
}

int pob_octree_train_persp(const pob_octree* tree, const pob_octree_opts* opts, const pob_camera* cam, int row0,
                           int nrows, const float* gt_rgb_dev, float grad_scale, float* grad_data_dev,
                           double* sq_err_sum_dev, float* out_rgb_dev, void* stream) {
  return train_persp("pob_octree_train_persp", tree, opts, cam, nullptr, row0, nrows, gt_rgb_dev, grad_scale,
                     grad_data_dev, sq_err_sum_dev, out_rgb_dev, stream);
}

int pob_octree_train_persp_ndc(const pob_octree* tree, const pob_octree_opts* opts, const pob_camera* cam,
                               const pob_ndc* ndc, int row0, int nrows, const float* gt_rgb_dev, float grad_scale,
                               float* grad_data_dev, double* sq_err_sum_dev, float* out_rgb_dev, void* stream) {
  if (!ndc) return pob_fail("pob_octree_train_persp_ndc", "NDC description is NULL");
  return train_persp("pob_octree_train_persp_ndc", tree, opts, cam, ndc, row0, nrows, gt_rgb_dev, grad_scale,
                     grad_data_dev, sq_err_sum_dev, out_rgb_dev, stream);
}

int pob_octree_sgd_step(float* data_dev, float* grad_dev, int64_t n, float lr, void* stream) {
  const char* W = "pob_octree_sgd_step";
  if (!data_dev || !grad_dev) return pob_fail(W, "NULL pointer");
  if (n < 0) return pob_fail(W, "negative size");
  const int sms = pob_sms_or_fail(W);
  if (!sms) return 1;
  if ((reinterpret_cast<uintptr_t>(data_dev) | reinterpret_cast<uintptr_t>(grad_dev)) & 15)
    return pob_fail(W, "data / grad must be 16-byte aligned");
  if (n == 0) return 0;
  pob_count_launch();
  octree_sgd_kernel<<<sms * 16, 256, 0, (cudaStream_t)stream>>>(data_dev, grad_dev, n, lr);
  POB_CUDA(W, cudaGetLastError());
  return 0;
}

int pob_octree_sgd_momentum_step(float* data_dev, float* grad_dev, float* buf_dev, int64_t n, float lr, float momentum,
                                 int nesterov, void* stream) {
  const char* W = "pob_octree_sgd_momentum_step";
  if (!data_dev || !grad_dev || !buf_dev) return pob_fail(W, "NULL pointer");
  if (n < 0) return pob_fail(W, "negative size");
  if (!(momentum >= 0.f) || !isfinite(momentum)) return pob_fail(W, "momentum must be finite and >= 0");
  const int sms = pob_sms_or_fail(W);
  if (!sms) return 1;
  if ((reinterpret_cast<uintptr_t>(data_dev) | reinterpret_cast<uintptr_t>(grad_dev) |
       reinterpret_cast<uintptr_t>(buf_dev)) & 15)
    return pob_fail(W, "data / grad / buf must be 16-byte aligned");
  if (n == 0) return 0;
  pob_count_launch();
  octree_sgd_momentum_kernel<<<sms * 16, 256, 0, (cudaStream_t)stream>>>(data_dev, grad_dev, buf_dev, n, lr, momentum,
                                                                         nesterov != 0);
  POB_CUDA(W, cudaGetLastError());
  return 0;
}

int pob_octree_adam_step(float* data_dev, float* grad_dev, float* m_dev, float* v_dev, int64_t n, float lr, float step,
                         float eps, void* stream) {
  const char* W = "pob_octree_adam_step";
  if (!data_dev || !grad_dev || !m_dev || !v_dev) return pob_fail(W, "NULL pointer");
  if (n < 0) return pob_fail(W, "negative size");
  if (!pob_sms_or_fail(W)) return 1;
  if (n == 0) return 0;
  pob_count_launch();
  POB_CUDA(W, pob::launch_adam(data_dev, grad_dev, m_dev, v_dev, n, lr, step, nullptr, 0.9f, 0.999f, eps, 1.0f,
                               0.0f, (cudaStream_t)stream));
  POB_CUDA(W, cudaMemsetAsync(grad_dev, 0, size_t(n) * sizeof(float), (cudaStream_t)stream));
  return 0;
}

int pob_octree_query(const pob_octree* tree, const float* points_dev, int64_t n, int64_t* leaf_index_dev,
                     void* stream) {
  const char* W = "pob_octree_query";
  TreeDev T;
  if (int rc = tree_dev(W, tree, T)) return rc;
  if (!points_dev || !leaf_index_dev) return pob_fail(W, "NULL pointer");
  if (n <= 0) return n < 0 ? pob_fail(W, "negative size") : 0;
  pob_count_launch();
  octree_query_kernel<<<unsigned((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      T, points_dev, n, reinterpret_cast<long long*>(leaf_index_dev));
  POB_CUDA(W, cudaGetLastError());
  return 0;
}

int pob_grid_weight_render(const float* sigma_grid_dev, int reso, const pob_camera* cams_dev, int n_cams,
                           int max_width, int max_height, const float offset[3], const float invradius[3],
                           const pob_octree_opts* opts, float* max_weight_dev, uint8_t* hit_dev, void* stream) {
  return grid_weights("pob_grid_weight_render", sigma_grid_dev, reso, cams_dev, n_cams, max_width, max_height, offset,
                      invradius, opts, nullptr, max_weight_dev, hit_dev, stream);
}

int pob_grid_weight_render_ndc(const float* sigma_grid_dev, int reso, const pob_camera* cams_dev, int n_cams,
                               int max_width, int max_height, const float offset[3], const float invradius[3],
                               const pob_octree_opts* opts, const pob_ndc* ndc, float* max_weight_dev,
                               uint8_t* hit_dev, void* stream) {
  if (!ndc) return pob_fail("pob_grid_weight_render_ndc", "NDC description is NULL");
  return grid_weights("pob_grid_weight_render_ndc", sigma_grid_dev, reso, cams_dev, n_cams, max_width, max_height,
                      offset, invradius, opts, ndc, max_weight_dev, hit_dev, stream);
}

}  // extern "C"
