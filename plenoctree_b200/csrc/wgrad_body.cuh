#pragma once
// wgrad_body.cuh — device body of mlp_wgrad.cu: weight-gradient contraction over samples (the wgrad half of jax.value_and_grad,
// nerf_sh/train.py:116):   dW_l[out, in] = sum_s dZ_l[s, out] * h_{l-1}[s, in],  db_l = sum_s dZ_l[s, :]
//
// Every persistent CTA owns one layer ("role") and one half of its 256 result rows for the whole launch: a 128 x 256
// fp32 accumulator is half of an SM's register file (two warpgroups, one m64n256 accumulator each), so the two row
// halves of a role are separate CTAs.  A CTA streams the [sample x feature] tile images that mlp_fwd (h_l, posenc)
// and mlp_bwd (dZ_l, dO) left in global memory; both wgmma operands are read MN-major straight from those images
// (K = samples): no transposes; warp 8 loads them through a ring of 64-sample stages (common.cuh: Ring) whose depth
// depends on the role's bytes per stage.  dZ / dO / posenc tiles are K-major SW128 images (read MN-major with the same
// swizzle), the h_l tiles are "T" images (no swizzle, 128 B core matrices; layouts.py: t_tile_offset).
// CTAs of the same role and row half split the tiles round-robin and each writes an fp32 partial; reduce_grads
// (optim.cu) sums the partials into the flat gradient (deterministic, no atomics).
//
// Roles (kernels.h: wgrad_role): Dense_1..7 (Dense_5: its h4 rows) with A = dZ_l and B = h_{l-1}; Dense_0 and the
// posenc rows of Dense_5 with B = posenc; the heads with A = h_7 and B = dO (a transposed result).
// Bias gradients are column sums of the A (or, for the heads, B) tile, summed by the consumer warps from the staged
// shared-memory tiles while their MMAs run.
//
// Concurrency with mlp_bwd.  The launch runs on the SMs that the mlp_bwd launch of the same level leaves free, right
// behind it (programmatic stream serialization), and reads each dZ / dO tile a few microseconds after it was stored,
// from L2.  Per tile, progress[tile] counts the stages (dO = 0, dZ_7 = 1 .. dZ_0 = 8) whose bulk stores have
// completed: mlp_bwd's warpgroup 0 in the low and warpgroup 1 in the high 16 bits (each warpgroup stores its 64
// rows).  Before the loads of a tile, the loader waits (ld.acquire, nanosleep back-off) until both halves exceed the
// stage it needs, then orders its bulk loads behind that with fence.proxy.async; the writer side is wait_group
// (completion, not .read) -> fence.proxy.async -> red.release.gpu.  h and posenc come from the earlier mlp_fwd launch.
// The two halves are counted apart because the warpgroups may be two stages apart (the weight ring lets one run a
// whole layer ahead), so a sum of both could reach 2 (stage + 1) with one half still missing.
// This cannot deadlock:
//  - this grid starts only once every mlp_bwd CTA has executed griddepcontrol.launch_dependents, so all of them are
//    resident, and none of them ever waits on this grid;
//  - every counter waited on belongs to a tile < seg_tiles, and mlp_bwd completes all nine stages of every such tile,
//    padded tiles included;
//  - if the programmatic launch is not honoured (timing events between the launches, graph capture on an older
//    driver), this grid starts after mlp_bwd has finished and every counter is already full: the result is the same,
//    only serial.
// Each CTA still sums its static share of the tiles in increasing tile order: the gradient is bit-identical from run
// to run.
#include "common.cuh"
#include "kernels.h"

namespace pob {

namespace {

constexpr int WG_THREADS = 288;       // warps 0-7: two consumer warpgroups, warp 8: loads
constexpr int WG_SUB = 64;            // samples per stage
constexpr uint32_t WG_PIECE = WG_SUB * 128;        // 64 samples x 128 B: one 64-feature chunk (SW128) / half a T group pair
constexpr uint32_t WG_A_BYTES = 2 * WG_PIECE;      // the CTA's 128 A features
constexpr uint32_t WG_B_MAX = 4 * WG_PIECE;        // up to 256 B features
constexpr uint32_t WG_SMEM = 4 * (WG_A_BYTES + WG_B_MAX);   // four 48 KB stages of the 256-wide roles
// A stage holds A and the role's B features only, so the narrow roles (Dense_0, Dense_5's posenc rows, the heads:
// 24-32 KB per stage) keep six to eight stages in flight.  Their time per stage is load latency rather than MMAs.
constexpr int WG_MAX_STAGES = 8;
using WgRing = Ring<WG_MAX_STAGES>;

struct RoleInfo {
  int a_op, a_layer, b_op, b_layer;   // kernels.h: WgradRole
  int b_chunks, N;
  int bias_from_b;       // heads: bias = column sums of dO
  int has_bias;
  int a_t, b_t;          // operand is a forward-saved h tile in the T layout (layouts.py: t_tile_offset)
};

__device__ __forceinline__ RoleInfo role_info(int role, int NH) {
  const WgradRole W = wgrad_role(role);
  RoleInfo r;
  r.a_op = W.a_op;
  r.a_layer = W.a_layer;
  r.b_op = W.b_op;
  r.b_layer = W.b_layer;
  r.N = wgrad_role_width(W, NH);
  r.b_chunks = (r.N + 63) / 64;
  r.bias_from_b = W.bias == WG_BIAS_B;
  r.has_bias = W.bias != WG_BIAS_NONE;
  r.a_t = W.a_op == WG_H;
  r.b_t = W.b_op == WG_H;
  return r;
}

// MN-major operand descriptors.  SW128 images: LBO = next 64-feature chunk (8 KB), SBO = next 8 samples (1 KB).
// T images: LBO = next 8 samples (128 B), SBO = next 8 features (512 B).
constexpr uint64_t SW_DESC = make_sdesc_hi(WG_PIECE, 1024, LAYOUT_SW128);
constexpr uint64_t T_DESC = make_sdesc_hi(128, 512, LAYOUT_NONE);

// Consumer warpgroup `wg`: accumulates D[64 A features x NN] over the CTA's stages, then writes its rows of the
// partial.  NN = MMA width (256, 64, or 80 for the heads, whose columns >= NH are never written back).
template <int NN>
__device__ __forceinline__ void wgrad_consume(const RoleInfo& R, uint8_t* smem, WgRing& ring, int nst,
                                              uint32_t stage_bytes, long long n_items, int mh, float* out_w,
                                              float* out_b) {
  const uint32_t warp = warp_id(), lane = lane_id();
  const int wg = int(warp >> 2);
  const int t = int(threadIdx.x & 127);
  const uint32_t sbase = smem_u32(smem);
  float acc[NN / 2];
#pragma unroll
  for (int i = 0; i < NN / 2; ++i) acc[i] = 0.f;

  // bias column sums.  A features (this warpgroup's 64): thread -> feature pair 8*(t/32) + t%8, samples 16*((t%32)/8)..+16
  // of every stage.  B features (heads, CTA row half 0, warpgroup 0): thread t < NH/2 -> pair t, all 64 samples.
  const bool a_bias = R.has_bias && !R.bias_from_b;
  const bool b_bias = R.bias_from_b && mh == 0 && wg == 0 && 2 * t < R.N;
  const int fp = a_bias ? (t >> 5) * 8 + (t & 7) : t;
  const int f = 2 * fp;
  const int s_lo = a_bias ? 16 * ((t & 31) >> 3) : 0, s_n = a_bias ? 16 : 64;
  const uint32_t bias_src = a_bias ? uint32_t(wg) * WG_PIECE : WG_A_BYTES + uint32_t(f >> 6) * WG_PIECE;
  const uint32_t unit = uint32_t((f & 63) >> 3), wsel = uint32_t(f & 7) * 2;
  float s0 = 0.f, s1 = 0.f;

  RingPos pos;
  wgmma_fence();
  for (long long i = 0; i < n_items; ++i) {
    for (int sub = 0; sub < 2; ++sub) {
      ring.wait(pos);
      const uint32_t a0 = sbase + pos.stage * stage_bytes;
      const uint32_t b0 = a0 + WG_A_BYTES;
#pragma unroll
      for (int ks = 0; ks < WG_SUB / 16; ++ks) {
        // SW128: 16 samples = 2 KB.  T: 32-sample group = 8 KB (A half) / 16 KB (B), 16 samples inside it = 256 B.
        const uint64_t ad = R.a_t ? sdesc(T_DESC, a0 + uint32_t(wg) * 4096u + uint32_t(ks >> 1) * 8192u + uint32_t(ks & 1) * 256u)
                                  : sdesc(SW_DESC, a0 + uint32_t(wg) * WG_PIECE + uint32_t(ks) * 2048u);
        const uint64_t bd = R.b_t ? sdesc(T_DESC, b0 + uint32_t(ks >> 1) * 16384u + uint32_t(ks & 1) * 256u)
                                  : sdesc(SW_DESC, b0 + uint32_t(ks) * 2048u);
        if constexpr (NN == 256) wgmma_m64n256<1, 1>(acc, ad, bd, 1u);
        else if constexpr (NN == 80) wgmma_m64n80<1, 1>(acc, ad, bd, 1u);
        else wgmma_m64n64<1, 1>(acc, ad, bd, 1u);
      }
      wgmma_commit();
      if (a_bias || b_bias) {
        const uint8_t* base = smem + pos.stage * stage_bytes + bias_src;
#pragma unroll 4
        for (int r = s_lo; r < s_lo + s_n; ++r) {
          const float2 v = unpack_f16x2(
              *reinterpret_cast<const uint32_t*>(base + r * 128 + ((unit ^ uint32_t(r & 7)) << 4) + wsel));
          s0 += v.x;
          s1 += v.y;
        }
      }
      wgmma_wait<0>();
      ring.release(pos.stage);
      pos.advance(nst);
    }
  }

  // ---- partial of this CTA: rows [128 mh + 64 wg, +64) of D[A feature][B feature], row pitch R.N ----
  const int fr = 16 * int(t >> 5) + int(lane >> 2), fc = 2 * int(lane & 3);
#pragma unroll
  for (int j = 0; j < NN / 8; ++j) {
    const int n = 8 * j + fc;
    if (n < R.N) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = 128 * mh + 64 * wg + fr + 8 * h;
        *reinterpret_cast<float2*>(out_w + size_t(m) * R.N + n) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      }
    }
  }
  if (a_bias) {
    s0 += __shfl_xor_sync(0xffffffffu, s0, 8);
    s1 += __shfl_xor_sync(0xffffffffu, s1, 8);
    s0 += __shfl_xor_sync(0xffffffffu, s0, 16);
    s1 += __shfl_xor_sync(0xffffffffu, s1, 16);
    if ((t & 31) < 8) {
      out_b[128 * mh + 64 * wg + f] = s0;
      out_b[128 * mh + 64 * wg + f + 1] = s1;
    }
  } else if (b_bias) {
    out_b[f] = s0;
    out_b[f + 1] = s1;
  }
}

}  // namespace

// cta indexes cta_role/index/count and the partials
__device__ __forceinline__ void wgrad_body(const WgradParams& p, uint8_t* smem, const int cta) {
  __shared__ __align__(8) WgRing ring;

  const uint32_t warp = warp_id();
  const uint32_t sbase = smem_u32(smem);
  const int role = p.cta_role[cta];
  if (role < 0) return;   // spare CTA
  const int ridx = p.cta_index[cta];
  const int rcnt = p.cta_count[cta];
  const int mh = ridx & 1;                       // result row half
  const int sidx = ridx >> 1, scnt = rcnt >> 1;  // tile split among the role's CTAs of this half
  float* const out_w = p.partials + size_t(cta) * WG_PARTIAL_FLOATS;
  float* const out_b = out_w + 65536;
  const RoleInfo R = role_info(role, p.NH);
  const uint32_t b_bytes = R.b_t ? 4 * WG_PIECE : uint32_t(R.b_chunks) * WG_PIECE;
  // room for every B feature the MMA reads: the heads MMA is 80 wide whenever NH != 64, so NH <= 64 reads a second
  // (unused) chunk.  A multiple of 8 KB, so every stage stays 1 KB aligned.
  const uint32_t b_room = R.N == 256 || R.N == 64 ? b_bytes : 2 * WG_PIECE;
  const uint32_t stage_bytes = WG_A_BYTES + b_room;
  const int nst = min(WG_MAX_STAGES, int(WG_SMEM / stage_bytes));

  // work list: tiles t = sidx + i*scnt
  const long long total_tiles = p.seg_tiles;
  const long long n_items = (total_tiles > sidx) ? (total_tiles - sidx + scnt - 1) / scnt : 0;

  if (threadIdx.x == 0) ring.init(nst);
  __syncthreads();

  if (warp == 8) {
    // ================================ loader ====================================
    // whole-warp control flow, one elected lane issues
    const WgradSegment& sg = p.seg;
    // every role reads one operand mlp_bwd stores: dZ_l (stage 8 - l) or, for the heads, dO (stage 0)
    const uint32_t want = R.a_op == WG_DZ ? uint32_t(NUM_TRUNK + 1 - R.a_layer) : 1u;
    RingPos pos;
    for (long long i = 0; i < n_items; ++i) {
      const long long lt = sidx + i * scnt;
      const uint8_t* a_ptr = (R.a_op == WG_DZ ? sg.dz : sg.h) + (size_t(lt) * NUM_TRUNK + R.a_layer) * A_TILE_BYTES;
      const uint8_t* b_ptr = R.b_op == WG_H ? sg.h + (size_t(lt) * NUM_TRUNK + R.b_layer) * A_TILE_BYTES
                             : R.b_op == WG_E ? sg.e + size_t(lt) * E_TILE_BYTES
                                              : sg.d_o + size_t(lt) * (2 * A_CHUNK_BYTES);
      for (int sub = 0; sub < 2; ++sub) {
        ring.acquire(pos);
        if (elect_one()) {
          // the thread that issues the loads is the one that acquires (once the tile is complete, this is one L2 hit)
          for (uint32_t ns = 32;;) {
            const uint32_t v = ld_acquire_gpu(p.progress + lt);
            if ((v & 0xFFFFu) >= want && (v >> 16) >= want) break;
            __nanosleep(ns);
            if (ns < 512) ns *= 2;
          }
          fence_proxy_async_global();
          const uint32_t bar = ring.arm(pos, WG_A_BYTES + b_bytes);
          const uint32_t dst = sbase + pos.stage * stage_bytes;
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            if (R.a_t)   // T image: this half's 128 features = 8 KB of each 32-sample group
              bulk_g2s(dst + c * WG_PIECE, a_ptr + size_t(2 * sub + c) * 16384 + mh * WG_PIECE, WG_PIECE, bar);
            else         // SW128 image: 64 samples of chunks 2 mh, 2 mh + 1
              bulk_g2s(dst + c * WG_PIECE, a_ptr + size_t(2 * mh + c) * A_CHUNK_BYTES + sub * WG_PIECE, WG_PIECE, bar);
          }
          if (R.b_t) {
            bulk_g2s(dst + WG_A_BYTES, b_ptr + size_t(sub) * 4 * WG_PIECE, 4 * WG_PIECE, bar);
          } else {
            for (int c = 0; c < R.b_chunks; ++c)
              bulk_g2s(dst + WG_A_BYTES + c * WG_PIECE, b_ptr + size_t(c) * A_CHUNK_BYTES + sub * WG_PIECE, WG_PIECE, bar);
          }
        }
        __syncwarp();
        pos.advance(nst);
      }
    }
    return;
  }
  if (R.N == 256) wgrad_consume<256>(R, smem, ring, nst, stage_bytes, n_items, mh, out_w, out_b);
  else if (R.N == 64) wgrad_consume<64>(R, smem, ring, nst, stage_bytes, n_items, mh, out_w, out_b);
  else wgrad_consume<MAX_NH>(R, smem, ring, nst, stage_bytes, n_items, mh, out_w, out_b);
}

}  // namespace pob
