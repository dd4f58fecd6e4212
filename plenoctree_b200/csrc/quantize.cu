// quantize.cu — median-cut vector quantisation of the compressed-tree palettes (octree/compression.py: median_cut),
// byte-identical to the numpy implementation for every input.
//
// State of one point set (one SH basis function) between rounds: idx[n], the original point indices grouped by box
// id and, within a box, in ascending index order (the host's stable argsort(box)), and off[2^r + 1], the start of
// every box of round r.  A round is three launches over all (basis, box) pairs of all point sets:
//   quant_sort_boxes  per box: fp32 extents with numpy's NaN propagation, the first-argmax axis, and a stable LSD
//                     radix sort of the box by that axis' key (numpy float order: -0 == +0, NaN last), which is the
//                     host's lexsort((key, seg)) order.  Unweighted: rank >= (size + 1) / 2 goes up.  Weighted: the
//                     sorted weights and np.add.reduceat's total of the box (w[0] + numpy's pairwise sum of the rest).
//   quant_weighted_scan (weighted only) one thread per point set: np.cumsum over the whole sorted array is a
//                     sequential fp64 sum whose rounding depends on every earlier box, so it is reproduced as one:
//                     n dependent fp64 adds per set and round; the sets run side by side.
//   quant_partition   per box: stable partition of idx by the up flags into the children 2 id and 2 id + 1.
// quant_palette then sums every final box in index order in fp64 (np.bincount's order) and scatters the map.
// No float atomics anywhere: the results do not depend on the grid size or on scheduling.
#include <cstdint>

#include "../../include/plenoctree_b200.h"
#include "capi_util.h"
#include "kernels.h"

// the kernels live in pob:: (not an anonymous namespace) so their symbol names stay stable for profiles
namespace pob {

static constexpr int QT = 256;            // threads per CTA of the box kernels
static constexpr int QW = QT / 32;
static constexpr int CTAS_PER_SM = 8;

// numpy's maximum / minimum: NaN if either is NaN
static __device__ __forceinline__ float np_max(float a, float b) { return (a != a || b != b) ? __int_as_float(0x7fc00000) : (a > b ? a : b); }
static __device__ __forceinline__ float np_min(float a, float b) { return (a != a || b != b) ? __int_as_float(0x7fc00000) : (a < b ? a : b); }

// an unsigned key whose order is numpy's sort order of float32: -0 == +0, all NaNs equal and last
static __device__ __forceinline__ uint32_t sort_key(float v) {
  if (v != v) return 0xffffffffu;
  uint32_t u = __float_as_uint(v == 0.f ? 0.f : v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// numpy's pairwise_sum of n doubles: blocks of fewer than 8 summed in order from -0.0, blocks up to 128 with eight
// accumulators, longer runs split at a multiple of 8 below the half and the halves added
static __device__ double np_pairwise_leaf(const double* a, long long n) {
  if (n < 8) {
    double r = -0.0;
    for (long long i = 0; i < n; ++i) r += a[i];
    return r;
  }
  double r0 = a[0], r1 = a[1], r2 = a[2], r3 = a[3], r4 = a[4], r5 = a[5], r6 = a[6], r7 = a[7];
  long long i = 8;
  for (; i < n - (n % 8); i += 8) {
    r0 += a[i + 0]; r1 += a[i + 1]; r2 += a[i + 2]; r3 += a[i + 3];
    r4 += a[i + 4]; r5 += a[i + 5]; r6 += a[i + 6]; r7 += a[i + 7];
  }
  double r = ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7));
  for (; i < n; ++i) r += a[i];
  return r;
}
static __device__ __forceinline__ long long np_pairwise_half(long long n) { return n / 2 - (n / 2) % 8; }
static __device__ double np_pairwise(const double* a, long long n) {
  // the recursion made iterative: a stack of (offset, length, state); 0 = fresh, 1 = left half pending,
  // 2 = right half pending (left sum in acc).  Halving from < 2^32 needs fewer than 32 levels.
  long long off[32], len[32];
  double acc[32];
  int st[32];
  int sp = 0;
  off[0] = 0;
  len[0] = n;
  st[0] = 0;
  double ret = 0.0;
  while (true) {
    const long long o = off[sp], m = len[sp];
    if (st[sp] == 0 && m > 128) {
      st[sp] = 1;
      off[sp + 1] = o;
      len[sp + 1] = np_pairwise_half(m);
      st[sp + 1] = 0;
      ++sp;
      continue;
    }
    if (st[sp] == 0) {
      ret = np_pairwise_leaf(a + o, m);
    } else if (st[sp] == 1) {
      acc[sp] = ret;
      st[sp] = 2;
      const long long h = np_pairwise_half(m);
      off[sp + 1] = o + h;
      len[sp + 1] = m - h;
      st[sp + 1] = 0;
      ++sp;
      continue;
    } else {
      ret = acc[sp] + ret;
    }
    if (sp == 0) return ret;
    --sp;
  }
}

// np.add.reduceat of one segment: the first element, then the pairwise sum of the rest added to it
static __device__ double np_reduceat(const double* a, long long n) { return n == 1 ? a[0] : a[0] + np_pairwise(a + 1, n - 1); }

static __device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

struct QuantParams {
  const float* points;     // [nb][n][3]
  const double* weights;   // [n] or NULL
  int64_t n;
  int nb, round;
  const uint32_t* idx_in;  // [nb][n]
  uint32_t* idx_out;
  const uint32_t* off_in;  // [nb][off_stride]
  uint32_t* off_out;
  int64_t off_stride;      // 2^bits + 1
  uint32_t *key_a, *key_b, *pos_a, *pos_b;   // [nb][n] sort ping-pong
  uint8_t* up;             // [nb][n], by position in idx
  double* wsorted;         // [nb][n] weights in sorted order (weighted)
  double* total;           // [nb][2^15] np.add.reduceat of each box (weighted)
  uint8_t* split;          // [nb][2^15] 1 if the box splits this round
};

// the box of grid item t in round r: point set b, box id
static __device__ __forceinline__ void item_box(long long t, int r, int& b, uint32_t& id) {
  b = int(t >> r);
  id = uint32_t(t & ((1ll << r) - 1));
}

__global__ void __launch_bounds__(QT) quant_sort_boxes(QuantParams p) {
  __shared__ int hist[256];
  __shared__ int wcnt[QW][256];
  __shared__ float red[QW][6];
  __shared__ int s_axis, s_split, s_skip;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long items = (long long)p.nb << p.round;
  const size_t nbox = size_t(1) << 15;
  for (long long t = blockIdx.x; t < items; t += gridDim.x) {
    int b;
    uint32_t id;
    item_box(t, p.round, b, id);
    const uint32_t* off = p.off_in + b * p.off_stride;
    const uint32_t s = off[id], e = off[id + 1], m = e - s;
    if (m == 0) {
      if (tid == 0) p.split[b * nbox + id] = 0;
      continue;
    }
    const size_t base = size_t(b) * p.n;
    const uint32_t* idx = p.idx_in + base + s;
    const float* pts = p.points + size_t(b) * p.n * 3;
    // extents: numpy's maximum.reduceat - minimum.reduceat in fp32
    float mx[3], mn[3];
    for (int c = 0; c < 3; ++c) mx[c] = -__int_as_float(0x7f800000), mn[c] = __int_as_float(0x7f800000);
    for (uint32_t i = tid; i < m; i += QT) {
      const float* q = pts + size_t(idx[i]) * 3;
      for (int c = 0; c < 3; ++c) mx[c] = np_max(mx[c], q[c]), mn[c] = np_min(mn[c], q[c]);
    }
    for (int o = 16; o; o >>= 1)
      for (int c = 0; c < 3; ++c) {
        mx[c] = np_max(mx[c], __shfl_xor_sync(0xffffffffu, mx[c], o));
        mn[c] = np_min(mn[c], __shfl_xor_sync(0xffffffffu, mn[c], o));
      }
    if (lane == 0)
      for (int c = 0; c < 3; ++c) red[warp][c] = mx[c], red[warp][3 + c] = mn[c];
    __syncthreads();
    if (tid == 0) {
      float ext[3];
      for (int c = 0; c < 3; ++c) {
        float a = red[0][c], z = red[0][3 + c];
        for (int w = 1; w < QW; ++w) a = np_max(a, red[w][c]), z = np_min(z, red[w][3 + c]);
        ext[c] = __fsub_rn(a, z);
      }
      int ax = 0;   // np.argmax: the first maximum, a NaN counting as the maximum
      float best = ext[0];
      for (int c = 1; c < 3 && best == best; ++c)
        if (ext[c] != ext[c] || ext[c] > best) ax = c, best = ext[c];
      s_axis = ax;
      s_split = best > 0.f;
      p.split[b * nbox + id] = uint8_t(best > 0.f);
    }
    __syncthreads();
    const int axis = s_axis;
    const bool splittable = s_split;
    // an unweighted box that does not split needs no order; a weighted one does, for the running sum
    if (!splittable && !p.weights) continue;
    uint32_t* kin = p.key_a + base + s;
    uint32_t* pin = p.pos_a + base + s;
    uint32_t* kout = p.key_b + base + s;
    uint32_t* pout = p.pos_b + base + s;
    for (uint32_t i = tid; i < m; i += QT) {
      kin[i] = sort_key(pts[size_t(idx[i]) * 3 + axis]);
      pin[i] = i;
    }
    __syncthreads();
    // stable LSD radix sort of (key, position), 8 bits a pass; a pass whose digit is the same for all is skipped
    for (int pass = 0; pass < 4; ++pass) {
      const int shift = 8 * pass;
      hist[tid] = 0;
      if (tid == 0) s_skip = 0;
      __syncthreads();
      for (uint32_t i = tid; i < m; i += QT) atomicAdd(&hist[(kin[i] >> shift) & 255], 1);
      __syncthreads();
      if (uint32_t(hist[tid]) == m) s_skip = 1;
      // exclusive scan of hist (thread d holds digit d)
      const int h = hist[tid];
      int x = h;
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
      }
      if (lane == 31) wcnt[0][warp] = x;
      __syncthreads();
      const bool skip = s_skip;
      int wpre = 0;
      for (int w = 0; w < warp; ++w) wpre += wcnt[0][w];
      __syncthreads();   // every thread has read s_skip and the warp sums before they are reset
      if (skip) continue;
      hist[tid] = wpre + x - h;   // digit start
      for (int w = 0; w < QW; ++w) wcnt[w][tid] = 0;
      __syncthreads();
      for (uint32_t t0 = 0; t0 < m; t0 += QT) {
        const uint32_t i = t0 + tid;
        const bool valid = i < m;
        const uint32_t k = valid ? kin[i] : 0u;
        const uint32_t ps = valid ? pin[i] : 0u;
        const int d = valid ? int((k >> shift) & 255) : 256;
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int rank = __popc(peers & lanemask_lt());
        if (valid && rank == 0) wcnt[warp][d] = __popc(peers);
        __syncthreads();
        if (valid) {
          int o = hist[d] + rank;
          for (int w = 0; w < warp; ++w) o += wcnt[w][d];
          kout[o] = k;
          pout[o] = ps;
        }
        __syncthreads();
        int sum = 0;
        for (int w = 0; w < QW; ++w) sum += wcnt[w][tid], wcnt[w][tid] = 0;
        hist[tid] += sum;
        __syncthreads();
      }
      uint32_t* tk = kin; kin = kout; kout = tk;
      uint32_t* tp = pin; pin = pout; pout = tp;
    }
    uint32_t* pos_final = p.pos_a + base + s;
    if (!p.weights) {
      const uint32_t k = (m + 1) / 2;   // the lower half keeps the median
      for (uint32_t j = tid; j < m; j += QT) p.up[base + s + pin[j]] = uint8_t(j >= k);
    } else {
      double* ws = p.wsorted + base + s;
      for (uint32_t j = tid; j < m; j += QT) {
        const uint32_t q = pin[j];
        ws[j] = p.weights[idx[q]];
        if (pin != pos_final) pos_final[j] = q;
      }
      __syncthreads();
      if (tid == 0) p.total[b * nbox + id] = splittable ? np_reduceat(ws, m) : 0.0;
    }
    __syncthreads();
  }
}

// the host's weighted threshold, cum - base > 0.5 total with cum = np.cumsum of the whole sorted array: one thread
// per point set walks its boxes in order, adding the sorted weights one by one
__global__ void quant_weighted_scan(QuantParams p) {
  const int b = blockIdx.x;
  if (threadIdx.x != 0) return;
  const size_t base = size_t(b) * p.n;
  const uint32_t* off = p.off_in + b * p.off_stride;
  const double* ws = p.wsorted + base;
  const uint32_t* pos = p.pos_a + base;
  uint8_t* up = p.up + base;
  const size_t nbox = size_t(1) << 15;
  double cum = 0.0;
  const uint32_t boxes = 1u << p.round;
  for (uint32_t id = 0; id < boxes; ++id) {
    const uint32_t s = off[id], e = off[id + 1];
    if (s == e) continue;
    const double cbase = cum;
    const double half = 0.5 * p.total[b * nbox + id];
    const bool splittable = p.split[b * nbox + id];
#pragma unroll 8
    for (uint32_t j = s; j < e; ++j) {
      cum += ws[j];
      up[s + pos[j]] = uint8_t(splittable && j > s && (cum - cbase) > half);
    }
  }
}

// stable partition of each box's indices by their up flags; the children's offsets for the next round
__global__ void __launch_bounds__(QT) quant_partition(QuantParams p) {
  __shared__ int wlow[QW];
  __shared__ int s_low;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long items = (long long)p.nb << p.round;
  const size_t nbox = size_t(1) << 15;
  for (long long t = blockIdx.x; t < items; t += gridDim.x) {
    int b;
    uint32_t id;
    item_box(t, p.round, b, id);
    const uint32_t* off = p.off_in + b * p.off_stride;
    uint32_t* noff = p.off_out + b * p.off_stride;
    const uint32_t s = off[id], e = off[id + 1], m = e - s;
    const size_t base = size_t(b) * p.n;
    const uint32_t* in = p.idx_in + base + s;
    uint32_t* out = p.idx_out + base + s;
    const bool splittable = m > 0 && p.split[b * nbox + id];
    const uint8_t* up = p.up + base + s;
    uint32_t nlow = m;
    if (splittable) {
      int c = 0;
      for (uint32_t i = tid; i < m; i += QT) c += up[i] == 0;
      for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
      if (lane == 0) wlow[warp] = c;
      __syncthreads();
      if (tid == 0) {
        int z = 0;
        for (int w = 0; w < QW; ++w) z += wlow[w];
        s_low = z;
      }
      __syncthreads();
      nlow = uint32_t(s_low);
      uint32_t lo = 0, hi = nlow;   // next slots of the two children
      for (uint32_t t0 = 0; t0 < m; t0 += QT) {
        const uint32_t i = t0 + tid;
        const bool valid = i < m;
        const bool low = valid && up[i] == 0;
        const bool high = valid && !low;
        const unsigned bl = __ballot_sync(0xffffffffu, low), bh = __ballot_sync(0xffffffffu, high);
        __syncthreads();
        if (lane == 0) wlow[warp] = __popc(bl) | (__popc(bh) << 16);
        __syncthreads();
        uint32_t pl = 0, ph = 0, tl = 0, th = 0;
        for (int w = 0; w < QW; ++w) {
          const uint32_t v = uint32_t(wlow[w]);
          if (w < warp) pl += v & 0xffff, ph += v >> 16;
          tl += v & 0xffff, th += v >> 16;
        }
        if (low) out[lo + pl + __popc(bl & lanemask_lt())] = in[i];
        if (high) out[hi + ph + __popc(bh & lanemask_lt())] = in[i];
        lo += tl;
        hi += th;
      }
      __syncthreads();
    } else {
      for (uint32_t i = tid; i < m; i += QT) out[i] = in[i];
    }
    if (tid == 0) {
      noff[2 * id] = s;
      noff[2 * id + 1] = s + nlow;
      if (id + 1 == (1u << p.round)) noff[2 * id + 2] = e;
    }
  }
}

__global__ void quant_init(uint32_t* idx, uint32_t* off, int64_t n, int nb, int64_t off_stride) {
  const long long total = (long long)nb * n;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    idx[i] = uint32_t(i % n);
  if (blockIdx.x == 0)
    for (int b = threadIdx.x; b < nb; b += blockDim.x) {
      off[b * off_stride] = 0;
      off[b * off_stride + 1] = uint32_t(n);
    }
}

// palette = per-box sums in index order (np.bincount) over max(count, 1e-30), zero for empty boxes; the map
__global__ void quant_palette(const float* points, const double* weights, int64_t n, int nb, int bits,
                              const uint32_t* idx_all, const uint32_t* off_all, int64_t off_stride, float* palette,
                              uint16_t* map) {
  const long long colors = 1ll << bits;
  const long long items = (long long)nb * colors;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < items; t += (long long)gridDim.x * blockDim.x) {
    const int b = int(t >> bits);
    const uint32_t id = uint32_t(t & (colors - 1));
    const uint32_t* off = off_all + b * off_stride;
    const uint32_t s = off[id], e = off[id + 1];
    const uint32_t* idx = idx_all + size_t(b) * n;
    const float* pts = points + size_t(b) * n * 3;
    uint16_t* mp = map + size_t(b) * n;
    double cnt = 0.0, sx = 0.0, sy = 0.0, sz = 0.0;
    for (uint32_t j = s; j < e; ++j) {
      const uint32_t i = idx[j];
      const float* q = pts + size_t(i) * 3;
      if (weights) {
        const double w = weights[i];
        cnt = __dadd_rn(cnt, w);
        sx = __dadd_rn(sx, __dmul_rn(double(q[0]), w));
        sy = __dadd_rn(sy, __dmul_rn(double(q[1]), w));
        sz = __dadd_rn(sz, __dmul_rn(double(q[2]), w));
      } else {
        cnt += 1.0;
        sx += double(q[0]);
        sy += double(q[1]);
        sz += double(q[2]);
      }
      mp[i] = uint16_t(id);
    }
    // np.maximum(cnt, 1e-30) keeps a NaN count; cnt == 0 zeroes the row
    const double d = (cnt != cnt || cnt > 1e-30) ? cnt : 1e-30;
    float* out = palette + t * 3;
    const bool zero = cnt == 0.0;
    out[0] = zero ? 0.f : __double2float_rn(__ddiv_rn(sx, d));
    out[1] = zero ? 0.f : __double2float_rn(__ddiv_rn(sy, d));
    out[2] = zero ? 0.f : __double2float_rn(__ddiv_rn(sz, d));
  }
}

static size_t quant_align_up(size_t x) { return (x + 255) / 256 * 256; }

QuantLayout quant_layout(int64_t n_basis, int64_t n, int weighted) {
  QuantLayout L;
  const size_t nn = size_t(n_basis) * size_t(n);
  const size_t offs = size_t(n_basis) * (size_t(QUANT_MAX_COLORS) + 1) * sizeof(uint32_t);
  const size_t boxes = size_t(n_basis) * (QUANT_MAX_COLORS / 2);
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o = quant_align_up(o + bytes); return at; };
  for (int i = 0; i < 2; ++i) L.idx[i] = take(nn * 4);
  for (int i = 0; i < 2; ++i) L.off[i] = take(offs);
  L.key[0] = take(nn * 4);
  L.key[1] = take(nn * 4);
  L.pos[0] = take(nn * 4);
  L.pos[1] = take(nn * 4);
  L.up = take(nn);
  L.split = take(boxes);
  L.wsorted = weighted ? take(nn * 8) : 0;
  L.total = weighted ? take(boxes * 8) : 0;
  L.bytes = o;
  return L;
}

int launch_quantize(const float* points, const double* weights, int64_t n, int nb, int bits, float* palette,
                            uint16_t* map, void* workspace, int sms, cudaStream_t st) {
  const QuantLayout L = quant_layout(nb, n, weights != nullptr);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  uint32_t* idx[2] = {reinterpret_cast<uint32_t*>(ws + L.idx[0]), reinterpret_cast<uint32_t*>(ws + L.idx[1])};
  uint32_t* off[2] = {reinterpret_cast<uint32_t*>(ws + L.off[0]), reinterpret_cast<uint32_t*>(ws + L.off[1])};
  const int64_t off_stride = QUANT_MAX_COLORS + 1;
  const int grid_cap = sms * CTAS_PER_SM;
  const char* where = "pob_quantize_median_cut";
  POB_LAUNCH(where, POB_PH_QUANT, st,
             (quant_init<<<grid_cap, QT, 0, st>>>(idx[0], off[0], n, nb, off_stride), cudaGetLastError()));
  QuantParams p;
  p.points = points;
  p.weights = weights;
  p.n = n;
  p.nb = nb;
  p.off_stride = off_stride;
  p.key_a = reinterpret_cast<uint32_t*>(ws + L.key[0]);
  p.key_b = reinterpret_cast<uint32_t*>(ws + L.key[1]);
  p.pos_a = reinterpret_cast<uint32_t*>(ws + L.pos[0]);
  p.pos_b = reinterpret_cast<uint32_t*>(ws + L.pos[1]);
  p.up = ws + L.up;
  p.split = ws + L.split;
  p.wsorted = weights ? reinterpret_cast<double*>(ws + L.wsorted) : nullptr;
  p.total = weights ? reinterpret_cast<double*>(ws + L.total) : nullptr;
  int cur = 0;
  for (int r = 0; r < bits; ++r) {
    p.round = r;
    p.idx_in = idx[cur];
    p.idx_out = idx[cur ^ 1];
    p.off_in = off[cur];
    p.off_out = off[cur ^ 1];
    const long long items = (long long)nb << r;
    const int grid = int(items < grid_cap ? items : grid_cap);
    POB_LAUNCH(where, POB_PH_QUANT, st, (quant_sort_boxes<<<grid, QT, 0, st>>>(p), cudaGetLastError()));
    if (weights)
      POB_LAUNCH(where, POB_PH_QUANT, st, (quant_weighted_scan<<<nb, 32, 0, st>>>(p), cudaGetLastError()));
    POB_LAUNCH(where, POB_PH_QUANT, st, (quant_partition<<<grid, QT, 0, st>>>(p), cudaGetLastError()));
    cur ^= 1;
  }
  const long long items = (long long)nb << bits;
  const long long pg = (items + 127) / 128;
  const int grid = int(pg < grid_cap ? pg : grid_cap);
  POB_LAUNCH(where, POB_PH_QUANT, st,
             (quant_palette<<<grid, 128, 0, st>>>(points, weights, n, nb, bits, idx[cur], off[cur], off_stride, palette,
                                                  map),
              cudaGetLastError()));
  return 0;
}

}  // namespace pob
