#pragma once
// wgrad_body.cuh — device body of mlp_wgrad.cu: weight-gradient contraction over samples (the wgrad half of jax.value_and_grad,
// nerf_sh/train.py:116):   dW_l[out, in] = sum_s dZ_l[s, out] * h_{l-1}[s, in],  db_l = sum_s dZ_l[s, :]
//
// Every persistent CTA owns one layer ("role", kernels.h: wgrad_role) for the whole launch, and every MMA is an
// m64n256: B is always 256 features (h_l or dZ_0), and each consumer warpgroup holds one 64 x 256 fp32 accumulator.
// A 128 x 256 accumulator is half of an SM's register file, so the 256 x 256 layers Dense_1..7 are split into two
// row halves, computed by separate CTAs (A = dZ_l, B = h_{l-1}; Dense_5 also contracts its A with the posenc tile
// into a second, m64n64 accumulator: the skip rows).  Dense_0 and the heads are computed transposed, as
// posenc^T dZ_0 and dO^T h_7, so that they too are 256 wide: their A is only 64 features (80 for SH25's heads), so
// the two warpgroups of a CTA split each stage's 64 samples between them (two k16 steps each) into separate
// accumulators, which reduce_grads adds; with NH = 80 warpgroup 1 takes heads features 64..79 instead.
// A CTA streams the [sample x feature] tile images that mlp_fwd (h_l, posenc) and mlp_bwd (dZ_l, dO) left in global
// memory; both wgmma operands are read MN-major straight from those images (K = samples): no transposes; warp 8 loads
// them through a ring of 64-sample stages (common.cuh: Ring), four for the halved roles and five for the 40 KB stages
// of the transposed ones.  dZ / dO / posenc tiles are K-major SW128 images (read MN-major with the same swizzle), the
// h_l tiles are "T" images (no swizzle, 128 B core matrices; layouts.py: t_tile_offset).
// CTAs of the same role (and row half) split the tiles round-robin and each writes an fp32 partial; reduce_grads
// (optim.cu) sums the partials into the flat gradient (deterministic, no atomics).
// Bias gradients are column sums of the A tile (dZ_l, dO) or, for Dense_0, of the B tile (dZ_0), summed by the
// consumer warps from the staged shared-memory tiles while their MMAs run.
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

// warps 0-7: two consumer warpgroups (232 registers after setmaxnreg: Dense_5 holds 160 accumulator registers),
// warp 8: loads, warps 9-11 only give their registers back
constexpr int WG_THREADS = 384;
constexpr int WG_SUB = 64;            // samples per stage
constexpr uint32_t WG_PIECE = WG_SUB * 128;        // 64 samples x 128 B: one 64-feature chunk (SW128) / half a T group pair
constexpr uint32_t WG_B_BYTES = 4 * WG_PIECE;      // the 256 B features
// Stage = A (64 or 128 features), B, and for Dense_5 the posenc tile: 40, 48 or 56 KB.  Four 56 KB stages of Dense_5.
constexpr uint32_t WG_SMEM = 4 * (2 * WG_PIECE + WG_B_BYTES + WG_PIECE);
constexpr int WG_MAX_STAGES = 5;
using WgRing = Ring<WG_MAX_STAGES>;
constexpr uint32_t WG_BIAS_BAR = 3;   // named barrier of the 256 consumer threads (1, 2: warpgroup_sync)

struct RoleInfo {
  int a_op, a_layer, b_op, b_layer;   // kernels.h: WgradRole
  int halves, skip, split_k;
  int a_chunks;          // 64-feature chunks of A per stage
  int bias_from_b;       // Dense_0: bias = column sums of dZ_0
  int b_t;               // B is a forward-saved h tile in the T layout (layouts.py: t_tile_offset)
};

__device__ __forceinline__ RoleInfo role_info(int role, int NH) {
  const WgradRole W = wgrad_role(role);
  RoleInfo r;
  r.a_op = W.a_op;
  r.a_layer = W.a_layer;
  r.b_op = W.b_op;
  r.b_layer = W.b_layer;
  r.halves = W.halves;
  r.skip = W.skip;
  r.split_k = wgrad_split_k(W, NH);
  r.a_chunks = W.halves == 2 || !r.split_k ? 2 : 1;
  r.bias_from_b = W.bias == WG_BIAS_B;
  r.b_t = W.b_op == WG_H;
  return r;
}

// MN-major operand descriptors.  SW128 images: LBO = next 64-feature chunk (8 KB), SBO = next 8 samples (1 KB).
// T images: LBO = next 8 samples (128 B), SBO = next 8 features (512 B).
constexpr uint64_t SW_DESC = make_sdesc_hi(WG_PIECE, 1024, LAYOUT_SW128);
constexpr uint64_t T_DESC = make_sdesc_hi(128, 512, LAYOUT_NONE);

// Consumer warpgroup `wg`: accumulates D[64 A features x 256] over the CTA's stages (SKIP: and D'[64 x 64 posenc
// features]), then writes its rows of the partial.  SPLIT_K: both warpgroups read A chunk 0, warpgroup w the k16
// steps 2w, 2w + 1 of every stage; otherwise warpgroup w reads A chunk w and all four.
template <bool SKIP, bool SPLIT_K>
__device__ __forceinline__ void wgrad_consume(const RoleInfo& R, uint8_t* smem, WgRing& ring, int nst,
                                              uint32_t stage_bytes, long long n_items, int mh, float* out_w,
                                              float* out_b) {
  const uint32_t warp = warp_id(), lane = lane_id();
  const int wg = int(warp >> 2);
  const int t = int(threadIdx.x & 127);
  const uint32_t sbase = smem_u32(smem);
  const uint32_t a_bytes = uint32_t(R.a_chunks) * WG_PIECE;
  float acc[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
  float acc2[SKIP ? 32 : 1];
#pragma unroll
  for (int i = 0; i < (SKIP ? 32 : 1); ++i) acc2[i] = 0.f;

  // bias column sums of the samples this warpgroup's MMAs read.
  //  A features (64 per warpgroup): thread -> feature pair 8*(t/32) + t%8, samples s_lo..+s_n with
  //  s_lo = 16*((t%32)/8) of every stage (SPLIT_K: 32 wg + 8*((t%32)/8), 8 samples).
  //  B features (Dense_0, SPLIT_K): thread -> feature pair t of all 256, samples 32 wg..+32.
  const bool b_bias = R.bias_from_b;
  const int f = b_bias ? 2 * t : 2 * ((t >> 5) * 8 + (t & 7));
  const int s_lo = b_bias ? 32 * wg : SPLIT_K ? 32 * wg + 8 * ((t & 31) >> 3) : 16 * ((t & 31) >> 3);
  const int s_n = b_bias ? 32 : SPLIT_K ? 8 : 16;
  const uint32_t bias_src = b_bias ? a_bytes + uint32_t(f >> 6) * WG_PIECE : SPLIT_K ? 0u : uint32_t(wg) * WG_PIECE;
  const uint32_t unit = uint32_t((f & 63) >> 3), wsel = uint32_t(f & 7) * 2;
  float s0 = 0.f, s1 = 0.f;

  RingPos pos;
  wgmma_fence();
  for (long long i = 0; i < n_items; ++i) {
    for (int sub = 0; sub < 2; ++sub) {
      ring.wait(pos);
      const uint32_t a0 = sbase + pos.stage * stage_bytes;
      const uint32_t b0 = a0 + a_bytes;
#pragma unroll
      for (int kk = 0; kk < (SPLIT_K ? 2 : 4); ++kk) {
        const int ks = SPLIT_K ? 2 * wg + kk : kk;
        // SW128: 16 samples = 2 KB.  T: 32-sample group = 16 KB, 16 samples inside it = 256 B.
        const uint64_t ad = sdesc(SW_DESC, a0 + (SPLIT_K ? 0u : uint32_t(wg) * WG_PIECE) + uint32_t(ks) * 2048u);
        const uint64_t bd = R.b_t ? sdesc(T_DESC, b0 + uint32_t(ks >> 1) * 16384u + uint32_t(ks & 1) * 256u)
                                  : sdesc(SW_DESC, b0 + uint32_t(ks) * 2048u);
        wgmma_m64n256<1, 1>(acc, ad, bd, 1u);
        if constexpr (SKIP) wgmma_m64n64<1, 1>(acc2, ad, sdesc(SW_DESC, b0 + WG_B_BYTES + uint32_t(ks) * 2048u), 1u);
      }
      wgmma_commit();
      {
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

  // ---- partial of this CTA: rows [128 mh + 64 wg, +64) of D, row pitch 256 (kernels.h: WgradRole) ----
  const int fr = 16 * int(t >> 5) + int(lane >> 2), fc = 2 * int(lane & 3);
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int n = 8 * j + fc;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = 128 * mh + 64 * wg + fr + 8 * h;
      *reinterpret_cast<float2*>(out_w + size_t(m) * 256 + n) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
    }
  }
  if constexpr (SKIP) {   // the skip rows, in the rows of the partial the other half would use
    float* const out_s = out_w + (mh ? 0 : 32768);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = 8 * j + fc;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = 64 * wg + fr + 8 * h;
        *reinterpret_cast<float2*>(out_s + size_t(m) * 64 + n) = make_float2(acc2[4 * j + 2 * h], acc2[4 * j + 2 * h + 1]);
      }
    }
  }
  if (!b_bias) {   // reduce over the four sample groups of the warp
    s0 += __shfl_xor_sync(0xffffffffu, s0, 8);
    s1 += __shfl_xor_sync(0xffffffffu, s1, 8);
    s0 += __shfl_xor_sync(0xffffffffu, s0, 16);
    s1 += __shfl_xor_sync(0xffffffffu, s1, 16);
  }
  const bool writer = b_bias || (t & 31) < 8;
  if constexpr (SPLIT_K) {
    // both warpgroups summed the same features over different samples: warpgroup 1 hands its sums over through the
    // (by now drained) ring, warpgroup 0 adds them
    float* const red = reinterpret_cast<float*>(smem);
    named_bar_sync(WG_BIAS_BAR, 256);   // no MMA of either warpgroup reads a stage any more
    if (wg == 1 && writer) {
      red[f] = s0;
      red[f + 1] = s1;
    }
    named_bar_sync(WG_BIAS_BAR, 256);
    if (wg == 0 && writer) {
      out_b[f] = s0 + red[f];
      out_b[f + 1] = s1 + red[f + 1];
    }
  } else if (writer) {
    out_b[128 * mh + 64 * wg + f] = s0;
    out_b[128 * mh + 64 * wg + f + 1] = s1;
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
  const RoleInfo R = role_info(role, p.NH);
  const int mh = R.halves == 2 ? ridx & 1 : 0;                         // result row half
  const int sidx = R.halves == 2 ? ridx >> 1 : ridx;                   // tile split among the role's CTAs (of this half)
  const int scnt = R.halves == 2 ? rcnt >> 1 : rcnt;
  float* const out_w = p.partials + size_t(cta) * WG_PARTIAL_FLOATS;
  float* const out_b = out_w + 65536;
  const uint32_t a_bytes = uint32_t(R.a_chunks) * WG_PIECE;
  const uint32_t stage_bytes = a_bytes + WG_B_BYTES + (R.skip ? WG_PIECE : 0u);   // a multiple of 8 KB: 1 KB aligned
  const int nst = min(WG_MAX_STAGES, int(WG_SMEM / stage_bytes));

  // work list: tiles t = sidx + i*scnt
  const long long total_tiles = p.seg_tiles;
  const long long n_items = (total_tiles > sidx) ? (total_tiles - sidx + scnt - 1) / scnt : 0;

  if (threadIdx.x == 0) ring.init(nst);
  __syncthreads();

  if (warp >= 8) {
    // ================================ loader ====================================
    // whole-warp control flow, one elected lane issues
    setmaxnreg_dec<40>();
    if (warp != 8) return;
    const WgradSegment& sg = p.seg;
    // every role reads one operand mlp_bwd stores: dZ_l (stage 8 - l) or, for the heads, dO (stage 0)
    const int dz_layer = R.a_op == WG_DZ ? R.a_layer : R.b_op == WG_DZ ? R.b_layer : -1;
    const uint32_t want = dz_layer >= 0 ? uint32_t(NUM_TRUNK + 1 - dz_layer) : 1u;
    const int a_chunk0 = R.halves == 2 ? 2 * mh : 0;
    // p.discard: once a stage has been consumed, its dZ / dO pieces are dropped from L2.  mlp_bwd stored them a few
    // microseconds earlier and they are still dirty there; nothing reads them again in this launch (kernels.h:
    // wgrad_reads_saved_grads_once), so writing them back to HBM on eviction would be wasted bandwidth.  Ordering:
    // the bulk read of load k is complete -> full barrier of its stage -> every consumer warp's MMAs on the stage
    // have completed and it released the stage -> this warp acquires the stage again (for load k + nst, or after
    // the last load) -> the 32 lanes discard load k's lines, two per lane per 8 KB piece.
    const uint8_t* const saved0 = R.a_op == WG_DZ ? sg.dz + size_t(R.a_layer) * A_TILE_BYTES + size_t(a_chunk0) * A_CHUNK_BYTES
                                  : R.a_op == WG_DO ? sg.d_o
                                                    : sg.dz + size_t(R.b_layer) * A_TILE_BYTES;   // B = dZ_0
    const size_t saved_tile = R.a_op == WG_DO ? 2 * A_CHUNK_BYTES : size_t(NUM_TRUNK) * A_TILE_BYTES;
    const int saved_pieces = R.a_op == WG_E ? 4 : R.a_chunks;
    const uint32_t lane = lane_id();
    auto discard_load = [&](long long k) {   // load k = stage `k & 1` of the CTA's item k / 2
      const uint8_t* const s = saved0 + size_t(sidx + (k >> 1) * scnt) * saved_tile + size_t(k & 1) * WG_PIECE;
      for (int c = 0; c < saved_pieces; ++c) {
        discard_l2_line(s + size_t(c) * A_CHUNK_BYTES + lane * 128u);
        discard_l2_line(s + size_t(c) * A_CHUNK_BYTES + (lane + 32u) * 128u);
      }
    };
    // h tiles come from HBM and are read at most twice (both row halves of a layer), close together: evict_first
    // keeps them from pushing out the dZ / dO lines that mlp_bwd stores for this launch (DESIGN.md section 6)
    const uint64_t stream_l2 = l2_policy_evict_first();
    long long k = 0;   // stage loads issued
    RingPos pos;
    for (long long i = 0; i < n_items; ++i) {
      const long long lt = sidx + i * scnt;
      const uint8_t* a_ptr = R.a_op == WG_DZ ? sg.dz + (size_t(lt) * NUM_TRUNK + R.a_layer) * A_TILE_BYTES
                             : R.a_op == WG_E ? sg.e + size_t(lt) * E_TILE_BYTES
                                              : sg.d_o + size_t(lt) * (2 * A_CHUNK_BYTES);
      const uint8_t* b_ptr = (R.b_op == WG_H ? sg.h : sg.dz) + (size_t(lt) * NUM_TRUNK + R.b_layer) * A_TILE_BYTES;
      const uint8_t* e_ptr = sg.e + size_t(lt) * E_TILE_BYTES;
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
          const uint32_t bar = ring.arm(pos, stage_bytes);
          const uint32_t dst = sbase + pos.stage * stage_bytes;
          // SW128 images: 64 samples of each chunk
          for (int c = 0; c < R.a_chunks; ++c)
            bulk_g2s(dst + c * WG_PIECE, a_ptr + size_t(a_chunk0 + c) * A_CHUNK_BYTES + sub * WG_PIECE, WG_PIECE, bar);
          if (R.b_t) {   // T image: two 32-sample groups of all 256 features
            bulk_g2s_hint(dst + a_bytes, b_ptr + size_t(sub) * WG_B_BYTES, WG_B_BYTES, bar, stream_l2);
          } else {
#pragma unroll
            for (int c = 0; c < 4; ++c)
              bulk_g2s(dst + a_bytes + c * WG_PIECE, b_ptr + size_t(c) * A_CHUNK_BYTES + sub * WG_PIECE, WG_PIECE, bar);
          }
          if (R.skip) bulk_g2s(dst + a_bytes + WG_B_BYTES, e_ptr + sub * WG_PIECE, WG_PIECE, bar);
        }
        __syncwarp();
        if (p.discard && k >= nst) discard_load(k - nst);   // the stage's previous load
        ++k;
        pos.advance(nst);
      }
    }
    // the last nst loads (positions of never-filled stages, j < 0, are free at once)
    if (p.discard)
      for (long long j = k - nst; j < k; ++j) {
        ring.acquire(pos);
        if (j >= 0) discard_load(j);
        pos.advance(nst);
      }
    return;
  }
  setmaxnreg_inc<232>();
  if (R.skip) wgrad_consume<true, false>(R, smem, ring, nst, stage_bytes, n_items, mh, out_w, out_b);
  else if (R.split_k) wgrad_consume<false, true>(R, smem, ring, nst, stage_bytes, n_items, mh, out_w, out_b);
  else wgrad_consume<false, false>(R, smem, ring, nst, stage_bytes, n_items, mh, out_w, out_b);
}

}  // namespace pob
