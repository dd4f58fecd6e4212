// mlp_bwd.cu — data-gradient chain of the NeRF-SH MLP (the dgrad half of jax.value_and_grad in
// nerf_sh/train.py:116), fused per 128-sample tile like mlp_fwd:
//
//   G' (per-sample d pre_rgb[3], d sigma_raw from render.cu)  --SH basis-->  dO [128 x NH]
//   dH_7 = dO . W_heads ;  dZ_l = dH_l * f'(h_l) ;  dH_{l-1} = dZ_l . W_l   (l = 7..1)
//
// f = the trunk activation.  ReLU masks come from the forward pass (1 bit per activation); the other activations form
// f'(h_l) from the forward's saved h_l tiles (kernels.h: net_act_grad_of_output).  The transposed weights come from the
// packed `wt_hi` images.  Every dZ_l tile (and dO) is stored to global memory in the same
// swizzled tile-image format as the forward activations; mlp_wgrad contracts them over samples.
// No gradient w.r.t. the inputs is needed (layer 0 and the skip slice of layer 5 stop here).
//
// Warp roles (384 threads): warps 0-3 and 4-7 = two consumer warpgroups, each owning 64 rows of the tile (wgmma
// m64n256, accumulator in registers), warp 8 = weight producer (a ring of stages, one K-slot of the transposed
// weights each), warps 9 and 10 = store warps of warpgroups 0 and 1 (warp 11 only hands its registers back).  A
// warpgroup writes each stage (dO, dZ_7 .. dZ_0) into its rows of the shared A tile and hands them over; its store
// warp sends the rows to global memory (cp.async.bulk shared -> global), so the 64 KB per tile and GEMM leave the SM
// without occupying the consumer warps.  mlp_wgrad runs alongside on the remaining SMs and reads each stored stage
// back from L2 once the per-tile progress counter says it is complete (wgrad_body.cuh).
//
// NSPLIT = 1 (fp16): eight 16 KB stages.  A warpgroup feeds dZ_l to the next GEMM as a register A fragment and copies
// it into its rows of the A tile behind that GEMM's MMAs.
// NSPLIT = 3 (fp16x3): error-compensated operands.  dO and every dZ_l are formed in fp32 (masked), split into
// x = hi + lo (fp16 each) and stored as two tile images; every K step issues lo*hi + hi*lo + hi*hi against a stage
// holding the K-slot of wt_hi and of wt_lo.  An m64n256 accumulator and two 64-register A fragments do not fit 232
// registers, so A is read from the shared hi and lo tiles (as in the x3 forward): the warpgroup writes dZ_l there
// once its MMAs of the previous GEMM have completed, and the next GEMM reads the rows while the store warp
// bulk-stores both images.
#include <type_traits>

#include "common.cuh"
#include "kernels.h"

namespace pob {

namespace {

constexpr int BWD_THREADS = 384;
constexpr int BWD_PRODUCER_WARP = 8;
constexpr int BWD_STORE_WARP0 = 9;      // warps 9, 10: store warps of warpgroups 0, 1

// dynamic smem map: the A tile (x3: hi and lo tiles), then the weight ring
template <int NSPLIT>
struct BwdSmem {
  static constexpr uint32_t A_HI = 0;
  static constexpr uint32_t A_LO = A_HI + A_TILE_BYTES;                          // x3 only
  static constexpr uint32_t W = NSPLIT == 3 ? A_LO + A_TILE_BYTES : A_HI + A_TILE_BYTES;
  static constexpr uint32_t PARTS = NSPLIT == 3 ? 2 : 1;                        // per stage: wt_hi slot (, wt_lo slot)
  static constexpr uint32_t STAGE_BYTES = PARTS * WSLOT_BYTES;
  static constexpr int STAGES = NSPLIT == 3 ? 3 : 8;
  static constexpr uint32_t TOTAL = W + STAGES * STAGE_BYTES;
  static_assert(TOTAL == (NSPLIT == 3 ? 224u : 192u) * 1024u, "smem map");
};

}  // namespace

// ACT (= p.net_act): relu masks dH_l with the forward's mask words; the other trunk activations multiply it by
// f'(h_l) in fp32, formed from the saved h_l tile images (x3: hi + lo).  A thread reads the h_l elements of its own
// accumulator fragment, the addressing the forward stored them with (t_frag_base); their lines are fetched into L2
// while the GEMM for dH_l runs, as the mask words are loaded for relu.
template <int NSPLIT, int ACT>
__global__ void __launch_bounds__(BWD_THREADS, 1) mlp_bwd_kernel(const __grid_constant__ BwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  using SM = BwdSmem<NSPLIT>;
  __shared__ __align__(8) Ring<SM::STAGES> ring;
  // hand-over of a warpgroup's rows of the A tile: rows_full[g] completes once its 128 threads have written a stage's
  // rows, rows_free[g] once the store warp's bulk stores have read them
  __shared__ __align__(8) uint64_t rows_full[2], rows_free[2];

  const long long mrows = padded_rows(p.M);        // rows of the mask / tile arrays
  const long long num_tiles = mrows / TILE_M;      // padded tiles get zero gradients, not garbage
  const uint32_t warp = warp_id(), lane = lane_id();
  const uint32_t sbase = smem_u32(smem);
  const int NH = p.NH;
  const int do_chunks = (NH + 63) / 64;     // 64-wide chunks of the dO tile image

  // the mlp_wgrad launch behind this one may take the SMs this grid leaves free (wgrad_body.cuh)
  griddep_launch_dependents();
  if (threadIdx.x == 0) {
    ring.init(SM::STAGES);
    for (int g = 0; g < 2; ++g) {
      mbar_init(smem_u32(&rows_full[g]), 128);
      mbar_init(smem_u32(&rows_free[g]), 1);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp >= BWD_PRODUCER_WARP) {
    // whole-warp control flow, one elected lane issues
    setmaxnreg_dec<40>();
    if (warp == BWD_PRODUCER_WARP) {
      RingPos pos;
      const int nslots = bwd_slots(NH);
      for (long long it = blockIdx.x; it < num_tiles; it += gridDim.x) {
        for (int j = 0; j < nslots; ++j) {
          ring.acquire(pos);
          if (elect_one()) {
            const uint32_t bar = ring.arm(pos, SM::STAGE_BYTES);
            const uint32_t dst = sbase + SM::W + pos.stage * SM::STAGE_BYTES;
            bulk_g2s(dst, p.w.wt_hi + size_t(j) * WSLOT_BYTES, WSLOT_BYTES, bar);
            if constexpr (NSPLIT == 3) bulk_g2s(dst + WSLOT_BYTES, p.wt_lo + size_t(j) * WSLOT_BYTES, WSLOT_BYTES, bar);
          }
          __syncwarp();
          pos.advance(SM::STAGES);
        }
      }
    } else if (warp <= BWD_STORE_WARP0 + 1 && lane == 0) {
      // ---- store warp of warpgroup g: every stage of its 64 rows (dO, dZ_7 .. dZ_0; x3: the hi and lo images in
      // one bulk group) leaves the SM as bulk stores.
      // Progress (wgrad_body.cuh reads it): warpgroup 0 counts in the low, warpgroup 1 in the high 16 bits of the
      // tile's counter, one per stage whose bulk stores have completed.  A stage is published once the next one has
      // been committed (wait_group 1), so the rows go back to the warpgroup as soon as they have been read. ----
      const int g = int(warp) - BWD_STORE_WARP0;
      const uint32_t rows_off = uint32_t(g) * 64u * 128u;
      const uint32_t progress_inc = g == 0 ? 1u : 0x10000u;
      const uint32_t full = smem_u32(&rows_full[g]), free = smem_u32(&rows_free[g]);
      uint32_t phase = 0;
      long long pending = -1;       // tile of the most recent committed, not yet published store group
      // fp16: mlp_wgrad reads each stage from L2 shortly after it was stored, while ~4.5 GB of forward-saved h tiles
      // stream through L2 around it; evict_last keeps the stored lines resident until then (DESIGN.md section 6).
      const uint64_t keep_l2 = l2_policy_evict_last();
      auto publish = [&]() {        // pending's group has completed: its writes are visible to this thread
        fence_proxy_async_global();
        red_add_release_gpu(p.progress + pending, progress_inc);
      };
      for (long long it = blockIdx.x; it < num_tiles; it += gridDim.x) {
        for (int st = 0; st <= NUM_TRUNK; ++st) {
          uint8_t* const dst_hi = st == 0 ? p.save_do + size_t(it) * (2 * A_CHUNK_BYTES)
                                          : p.save_dz + (size_t(it) * NUM_TRUNK + (NUM_TRUNK - st)) * A_TILE_BYTES;
          uint8_t* const dst_lo = st == 0 ? p.save_do_lo + size_t(it) * (2 * A_CHUNK_BYTES)
                                          : p.save_dz_lo + (size_t(it) * NUM_TRUNK + (NUM_TRUNK - st)) * A_TILE_BYTES;
          const int nchunks = st == 0 ? do_chunks : 4;
          mbar_wait(full, phase);
          for (int c = 0; c < nchunks; ++c) {
            const uint32_t so = c * A_CHUNK_BYTES + rows_off;
            if constexpr (NSPLIT == 1) {
              bulk_s2g_hint(dst_hi + size_t(c) * A_CHUNK_BYTES + rows_off, sbase + SM::A_HI + so, 64u * 128u, keep_l2);
            } else {
              bulk_s2g(dst_hi + size_t(c) * A_CHUNK_BYTES + rows_off, sbase + SM::A_HI + so, 64u * 128u);
              bulk_s2g(dst_lo + size_t(c) * A_CHUNK_BYTES + rows_off, sbase + SM::A_LO + so, 64u * 128u);
            }
          }
          bulk_commit();
          bulk_wait_read_all();
          mbar_arrive(free);
          if (pending >= 0) {
            bulk_wait_all_but_last();
            publish();
          }
          pending = it;
          phase ^= 1;
        }
      }
      bulk_wait_all();
      if (pending >= 0) publish();
    }
    return;
  }

  // ================================ consumer warpgroups =================================
  setmaxnreg_inc<232>();
  const int wg = int(warp >> 2);
  const int t = int(threadIdx.x & 127);
  const int wq = t >> 5;
  const int fr = 16 * wq + int(lane >> 2);     // fragment rows fr, fr + 8 within the warpgroup's 64 rows
  const int fc = 2 * int(lane & 3);
  uint8_t* const a_hi = smem + SM::A_HI;
  uint8_t* const a_lo = smem + SM::A_LO;
  const uint32_t rows_off = uint32_t(wg) * 64u * 128u;
  constexpr uint64_t A_DESC = make_sdesc_hi(16, 1024, LAYOUT_SW128);
  constexpr uint64_t W_DESC = make_sdesc_hi(16, 512, LAYOUT_SW64);
  RingPos pos;
  float acc[128];
  uint32_t afr[64];        // fp16: dZ_l as the register A operand of the GEMM for dH_{l-1}
  uint32_t mw[2][8];       // relu mask words of h_l for the fragment rows fr, fr + 8

  // the warpgroup's rows of the A tile: wait until the store warp has read the previous stage, and hand a written
  // stage to it (each thread's writes made visible to the async proxy, then one arrival per thread)
  // (the __syncwarp reconverges the warp after the spin: without it ptxas serializes every wgmma of the kernel, C7520)
  uint32_t rows_phase = 0;
  auto rows_acquire = [&]() {
    mbar_wait(smem_u32(&rows_free[wg]), rows_phase ^ 1);
    __syncwarp();
  };
  auto rows_hand_over = [&]() {
    fence_proxy_async_smem();
    mbar_arrive(smem_u32(&rows_full[wg]));
    rows_phase ^= 1;
  };
  // fp16: columns 32c..32c+31 of dZ (afr[8c + i]: k16 step i/4, register i%4) -> the warpgroup's rows of the A tile
  // (a_tile_offset: rows fr and fr + 8 share the swizzle row & 7 = lane / 4)
  uint8_t* const share_base = a_hi + uint32_t(64 * wg + fr) * 128u + uint32_t(fc) * 2u;
  const uint32_t swz = (lane >> 2) << 4;
  auto write_share = [&](int c) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const uint32_t unit = uint32_t(4 * c + 2 * (i >> 2) + ((i >> 1) & 1)) & 7u;   // 16-byte unit of the column
      const uint32_t off = uint32_t(c >> 1) * A_CHUNK_BYTES + uint32_t(i & 1) * 1024u + ((unit << 4) ^ swz);
      *reinterpret_cast<uint32_t*>(share_base + off) = afr[8 * c + i];
    }
  };
  // h_l of this thread's fragment (ACT != relu): element (row fr + 8h, columns 8j + fc, +1) at h_src + t_frag_offset(j, h)
  size_t h_src = 0;
  auto load_masks = [&](int l, long long it) {
    if constexpr (ACT == NET_RELU) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint4* mp = reinterpret_cast<const uint4*>(p.mask + (size_t(l) * mrows + it * TILE_M + 64 * wg + fr + 8 * h) * 8);
        const uint4 m0 = __ldg(mp), m1 = __ldg(mp + 1);
        mw[h][0] = m0.x; mw[h][1] = m0.y; mw[h][2] = m0.z; mw[h][3] = m0.w;
        mw[h][4] = m1.x; mw[h][5] = m1.y; mw[h][6] = m1.z; mw[h][7] = m1.w;
      }
    } else {
      h_src = t_frag_base(it, l, wg, wq, lane);
      // the warp's share of the tile image: 256 contiguous bytes of each 8-column group (512-byte pitch), one group
      // per lane
      const size_t warp_lines = (size_t(it) * NUM_TRUNK + l) * A_TILE_BYTES + uint32_t(2 * wg + (wq >> 1)) * 16384u +
                                uint32_t(wq & 1) * 256u + lane * 512u;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        prefetch_l2(p.h + warp_lines + 128 * i);
        if constexpr (NSPLIT == 3) prefetch_l2(p.h_lo + warp_lines + 128 * i);
      }
    }
  };
  // f'(h) of the fragment pair (row fr + 8h, columns 8j + fc, +1)
  auto act_grad = [&](int j, int h) {
    const uint32_t o = t_frag_offset(j, h);
    float2 hv = unpack_f16x2(__ldg(reinterpret_cast<const uint32_t*>(p.h + h_src + o)));
    if constexpr (NSPLIT == 3) {
      const float2 lv = unpack_f16x2(__ldg(reinterpret_cast<const uint32_t*>(p.h_lo + h_src + o)));
      hv.x += lv.x;
      hv.y += lv.y;
    }
    return make_float2(net_act_grad_of_output<ACT>(hv.x), net_act_grad_of_output<ACT>(hv.y));
  };
  // fp16: dZ = dH * f'(h), fp16 pack of the accumulator (relu: masked).  afr[2j + h] holds 8-column group j of row
  // fr + 8h.
  auto make_dz = [&]() {
    if constexpr (ACT == NET_RELU) {
      acc_to_afrag<false>(acc, afr);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int k = (j & 3) * 4 + (fc >> 1);      // pair index inside the 32-column mask word j / 4
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint32_t m = mw[h][j >> 2];
          afr[2 * j + h] &= ((m >> mask_bit(k, 0)) & 1u ? 0x0000FFFFu : 0u) | ((m >> mask_bit(k, 1)) & 1u ? 0xFFFF0000u : 0u);
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float2 g = act_grad(j, h);
          afr[2 * j + h] = pack_f16x2(acc[4 * j + 2 * h] * g.x, acc[4 * j + 2 * h + 1] * g.y);
        }
      }
    }
  };
  // x3: GEMM over `ns` K-slots, A = the warpgroup's rows of the hi / lo tiles (K-slot j: chunk j/2, half j%2)
  auto gemm = [&](int ns, int mask_layer, long long it) {
    uint32_t prev = 0;
    wgmma_fence();
    for (int j = 0; j < ns; ++j) {
      const uint32_t a_off = uint32_t(j >> 1) * A_CHUNK_BYTES + rows_off + uint32_t(j & 1) * 64u;
      const uint32_t ah = sbase + SM::A_HI + a_off, al = sbase + SM::A_LO + a_off;
      const uint32_t bh = sbase + SM::W + pos.stage * SM::STAGE_BYTES, bl = bh + WSLOT_BYTES;
      ring.wait(pos);
      // per K-slot: without it ptxas injects the warpgroup.arrive after the ring spin itself and serializes every
      // wgmma of the kernel (C7520)
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const uint32_t ko = uint32_t(k) * 32u;
        wgmma_m64n256<0, 0>(acc, sdesc(A_DESC, al + ko), sdesc(W_DESC, bh + ko), (j != 0 || k != 0) ? 1u : 0u);
        wgmma_m64n256<0, 0>(acc, sdesc(A_DESC, ah + ko), sdesc(W_DESC, bl + ko), 1u);
        wgmma_m64n256<0, 0>(acc, sdesc(A_DESC, ah + ko), sdesc(W_DESC, bh + ko), 1u);
      }
      wgmma_commit();
      if (j == 0) load_masks(mask_layer, it);   // loaded while the GEMM runs
      if (j > 0) {
        wgmma_wait<1>();
        ring.release(prev);
      }
      prev = pos.stage;
      pos.advance(SM::STAGES);
    }
    wgmma_wait<0>();
    ring.release(prev);
  };
  // x3: dZ = dH * f'(h) in fp32 (relu: masked), split into hi + lo and written to the warpgroup's rows of the A tiles,
  // then handed to the store warp
  auto store_dz = [&]() {
    rows_acquire();
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int k = (j & 3) * 4 + (fc >> 1);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float v0, v1;
        if constexpr (ACT == NET_RELU) {
          const uint32_t m = mw[h][j >> 2];
          v0 = (m >> mask_bit(k, 0)) & 1u ? acc[4 * j + 2 * h] : 0.f;
          v1 = (m >> mask_bit(k, 1)) & 1u ? acc[4 * j + 2 * h + 1] : 0.f;
        } else {
          const float2 g = act_grad(j, h);
          v0 = acc[4 * j + 2 * h] * g.x;
          v1 = acc[4 * j + 2 * h + 1] * g.y;
        }
        const uint32_t w = pack_f16x2(v0, v1);
        const float2 hv = unpack_f16x2(w);
        const uint32_t off = a_tile_offset(64 * wg + fr + 8 * h, 8 * j + fc);
        *reinterpret_cast<uint32_t*>(a_hi + off) = w;
        *reinterpret_cast<uint32_t*>(a_lo + off) = pack_f16x2(v0 - hv.x, v1 - hv.y);
      }
    }
    rows_hand_over();
    warpgroup_sync(wg);   // every row written before the next GEMM reads them
  };

  for (long long it = blockIdx.x; it < num_tiles; it += gridDim.x) {
    // ---- dO rows from the per-sample gradient and the SH basis (two threads per row, 64 columns each) ----
    {
      const int r = 64 * wg + (t & 63);
      const int hf = t >> 6;
      const long long s = it * TILE_M + r;
      float4 gq = make_float4(0.f, 0.f, 0.f, 0.f);
      float basis[25];
#pragma unroll
      for (int k = 0; k < 25; ++k) basis[k] = 0.f;   // padded rows: 0 * garbage must not become NaN
      basis[0] = 1.f;
      if (s < p.M) {
        gq = p.G[s];
        const long long vi = p.n_per_ray > 0 ? (s < p.M_rays ? s / p.n_per_ray : 0) : s;   // free points: rgb gradient is 0
        const float* vd = p.viewdirs + 3 * vi;
        if (p.sh_deg >= 0) sh_basis(p.sh_deg, __ldg(vd), __ldg(vd + 1), __ldg(vd + 2), basis);
      }
      const float gc[3] = {gq.x, gq.y, gq.z};
      // dO columns 64hf .. 64hf + 63 of row r (x3: fp32 -> hi + lo); the half is a template argument so that the SH
      // basis is indexed with constants and stays in registers
      auto build_do = [&](auto half) {
        constexpr int HF = decltype(half)::value;
#pragma unroll
        for (int uu = 0; uu < 8; ++uu) {            // 16-byte units of 8 columns
          const int u = 8 * HF + uu;
          uint32_t w[4];
          [[maybe_unused]] uint32_t wl[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            float f[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int n = u * 8 + 2 * i + e;
              float v = 0.f;
              if (n == 0) v = gq.w;
              else if (n < 1 + 3 * 25) {
                int k, c;
                heads_coeff(n, k, c);
                if (k < p.K) v = gc[c] * basis[k];   // n < 76: k < 25
              }
              f[e] = v;
            }
            w[i] = pack_f16x2(f[0], f[1]);
            if constexpr (NSPLIT == 3) {
              const float2 hv = unpack_f16x2(w[i]);
              // unfused: lo is the residual of the rounded product f, not of the exact one
              wl[i] = pack_f16x2(__fsub_rn(f[0], hv.x), __fsub_rn(f[1], hv.y));
            }
          }
          const uint32_t off = a_tile_offset(r, 8 * u);
          *reinterpret_cast<uint4*>(a_hi + off) = make_uint4(w[0], w[1], w[2], w[3]);
          if constexpr (NSPLIT == 3) *reinterpret_cast<uint4*>(a_lo + off) = make_uint4(wl[0], wl[1], wl[2], wl[3]);
        }
      };
      rows_acquire();
      if (hf == 0) build_do(std::integral_constant<int, 0>());
      else if (do_chunks > 1) build_do(std::integral_constant<int, 1>());
      rows_hand_over();
      warpgroup_sync(wg);   // every row of dO written before the heads GEMM reads it
    }
    if constexpr (NSPLIT == 1) {
      // ---- heads GEMM: dH_7 = dO . W_heads, A = the dO rows in shared memory ----
      {
        const int ns = bwd_head_slots(NH);
        uint32_t prev = 0;
        wgmma_fence();
        for (int j = 0; j < ns; ++j) {
          const uint32_t a = sbase + SM::A_HI + uint32_t(j >> 1) * A_CHUNK_BYTES + rows_off + uint32_t(j & 1) * 64u;
          const uint32_t b = sbase + SM::W + pos.stage * SM::STAGE_BYTES;
          ring.wait(pos);
          wgmma_m64n256<0, 0>(acc, sdesc(A_DESC, a), sdesc(W_DESC, b), j != 0);
          wgmma_m64n256<0, 0>(acc, sdesc(A_DESC, a + 32), sdesc(W_DESC, b + 32), 1u);
          wgmma_commit();
          if (j == 0) load_masks(NUM_TRUNK - 1, it);   // loaded while the GEMM runs
          if (j > 0) {
            wgmma_wait<1>();
            ring.release(prev);
          }
          prev = pos.stage;
          pos.advance(SM::STAGES);
        }
        wgmma_wait<0>();
        ring.release(prev);
        make_dz();
      }
      // ---- GEMM for dH_l (Dense_{l+1}^T, l = 6 .. 0), A = dZ_{l+1} from registers.  dZ_{l+1} goes to the A tile one
      // K-slot behind the MMAs that read it and is handed to the store warp at the end of the GEMM. ----
      for (int l = NUM_TRUNK - 2; l >= 0; --l) {
        uint32_t prev = 0;
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const uint32_t b = sbase + SM::W + pos.stage * SM::STAGE_BYTES;
          ring.wait(pos);
          wgmma_m64n256_rs(acc, afr[8 * j], afr[8 * j + 1], afr[8 * j + 2], afr[8 * j + 3], sdesc(W_DESC, b), j != 0);
          wgmma_m64n256_rs(acc, afr[8 * j + 4], afr[8 * j + 5], afr[8 * j + 6], afr[8 * j + 7], sdesc(W_DESC, b + 32), 1u);
          wgmma_commit();
          if (j == 0) load_masks(l, it);
          if (j > 0) {
            wgmma_wait<1>();
            ring.release(prev);
            if (j == 1) rows_acquire();
            write_share(j - 1);
          }
          prev = pos.stage;
          pos.advance(SM::STAGES);
        }
        wgmma_wait<0>();
        ring.release(prev);
        write_share(7);
        rows_hand_over();
        make_dz();
      }
      // ---- dZ_0 ----
      rows_acquire();
#pragma unroll
      for (int c = 0; c < 8; ++c) write_share(c);
      rows_hand_over();
    } else {
      // ---- dH_7 = dO . W_heads; then dZ_l, and dH_{l-1} = dZ_l . W_l (l = 7 .. 1), dZ_0 ----
      gemm(bwd_head_slots(NH), NUM_TRUNK - 1, it);
      for (int l = NUM_TRUNK - 1; l >= 0; --l) {
        store_dz();
        if (l > 0) gemm(8, l - 1, it);
      }
    }
  }
}

cudaError_t launch_mlp_bwd(const BwdParams& p, int nsplit, int num_ctas, cudaStream_t stream) {
  if (p.M <= 0) return cudaSuccess;
  if (nsplit != 1 && nsplit != 3) return cudaErrorInvalidValue;
  if (nsplit == 3 && (!p.wt_lo || !p.save_dz_lo || !p.save_do_lo)) return cudaErrorInvalidValue;
  if (p.net_act != NET_RELU && (!p.h || (nsplit == 3 && !p.h_lo))) return cudaErrorInvalidValue;
  const long long tiles = padded_rows(p.M) / TILE_M;
  const int grid = int(tiles < num_ctas ? tiles : num_ctas);
  auto launch = [&](auto act) -> cudaError_t {
    constexpr int A = decltype(act)::value;
    auto kernel = nsplit == 1 ? mlp_bwd_kernel<1, A> : mlp_bwd_kernel<3, A>;
    const uint32_t smem = nsplit == 1 ? BwdSmem<1>::TOTAL : BwdSmem<3>::TOTAL;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    kernel<<<grid, BWD_THREADS, smem, stream>>>(p);
    return cudaGetLastError();
  };
  switch (p.net_act) {
    case NET_RELU: return launch(std::integral_constant<int, NET_RELU>());
    case NET_ELU: return launch(std::integral_constant<int, NET_ELU>());
    case NET_SOFTPLUS: return launch(std::integral_constant<int, NET_SOFTPLUS>());
    case NET_TANH: return launch(std::integral_constant<int, NET_TANH>());
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace pob
