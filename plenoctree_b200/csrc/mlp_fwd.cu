// mlp_fwd.cu — fused NeRF-SH point evaluator for sm_90a.
//
// One persistent CTA per SM evaluates   posenc(x) -> 8 x (Dense256 + ReLU, skip-concat into
// layer 5) -> [sigma | SH coefficient] heads -> (optionally) eval_sh at the view direction +
// sigmoid/relu   for one 128-sample tile per iteration, without the activations ever leaving the SM:
//
//   reference path                                      this kernel
//   -------------------------------------------------   ------------------------------------
//   model_utils.posenc      (model_utils.py:145-173)    consumer warps -> E tile (smem, fp16)
//   model_utils.MLP         (model_utils.py:30-94)      wgmma, fp32 accumulators in registers; fp16: activation
//                                                       (relu / elu / softplus / tanh, ACT) + pack into the next
//                                                       layer's register A operand (x3: epilogue -> smem A tiles)
//   sh.eval_sh + sigmoid/relu (sh.py:54-109,            heads epilogue (registers -> smem staging); the density
//     or softplus              models.py:269-281)       activation is p.sigma_act
//   NerfModel.eval_points_raw (models.py:143-181)       OUT_RAW / OUT_SIGMA
//
// Warp roles (384 threads): warps 0-3 and 4-7 = two consumer warpgroups, each owning 64 rows of the tile
// (one m64n256 accumulator = 128 registers per thread, 232 registers after setmaxnreg), warp 8 = weight producer
// (cp.async.bulk ring, one 16 KB K-slot per stage; warps 9-11 only hand their registers back).  Both warpgroups
// consume every stage; a warpgroup reads and rewrites only its own rows of the activation / posenc tiles, so the two
// synchronise through the weight ring alone.  fp16 chains the layers through registers (the activation tile only
// stages the heads); the training saves of h_l run one K-slot behind layer l+1's MMAs.  NSPLIT = 3 evaluates
// with error-compensated fp16 operands (x = hi + lo; lo*hi + hi*lo + hi*hi per K step), the residual parts in a
// second set of tiles; a stage then holds the K-slot's hi and lo parts (32 KB).  The x3 training forward (SAVE)
// stores h_l's hi and lo from the trunk epilogue and the posenc tile's lo behind the posenc barrier.
#include <type_traits>

#include "common.cuh"
#include "kernels.h"

namespace pob {

namespace {

constexpr int PRODUCER_WARP = 8;
constexpr int FWD_THREADS = 384;
constexpr int HEADS_N = 80;               // heads MMA width: MAX_NH (rows >= NH of a heads slot are never read back)
constexpr int STAGE_PITCH = HEADS_N + 1;  // heads staging: odd pitch -> conflict-free per-row scalar access

// dynamic smem map: activation tile, posenc tile, weight ring.  The x3 mode also keeps the residual (lo) tiles and
// runs a ring of two 32 KB stages.  The training forward (fp16, SAVE) gives those 80 KB to the ring, nine 16 KB
// stages: a stage is handed back only once both warpgroups are done with it, so the ring depth bounds how far one
// warpgroup can run ahead while the other stores its saved tiles.  The non-saving fp16 forward measured no gain from
// the deeper ring and keeps the x3 map, four stages (DESIGN.md §6).
constexpr uint32_t SM_TOTAL = 224 * 1024;
template <int NSPLIT, bool SAVE>
struct Smem {
  static constexpr bool DEEP = NSPLIT == 1 && SAVE;
  static constexpr uint32_t A0 = 0;                                              // activations, fp16 (hi)
  static constexpr uint32_t A1 = A0 + A_TILE_BYTES;                              // residual (x3 only)
  static constexpr uint32_t E0 = DEEP ? A0 + A_TILE_BYTES : A1 + A_TILE_BYTES;
  static constexpr uint32_t E1 = E0 + E_TILE_BYTES;                              // x3 only
  static constexpr uint32_t W = DEEP ? E0 + E_TILE_BYTES : E1 + E_TILE_BYTES;
  static constexpr uint32_t PARTS = NSPLIT == 3 ? 2 : 1;                        // per stage: hi slot (, lo slot)
  static constexpr uint32_t STAGE_BYTES = PARTS * WSLOT_BYTES;
  static constexpr int STAGES = int((SM_TOTAL - W) / STAGE_BYTES);
  static_assert(STAGES == (DEEP ? 9 : NSPLIT == 3 ? 2 : 4), "smem map");
  // Unrolling of the producer's loops (16: full).  Fully unrolled, the x3 producer adds ~2300 instructions to a kernel
  // twice the size of the fp16 one, and the x3 sigma forward ran 7-8 % slower (H100 80 GB HBM3, 700 W).
  static constexpr int PRODUCER_UNROLL = NSPLIT == 3 ? 1 : 16;
};

__device__ __noinline__ void load_point(const FwdParams& p, long long s, float& x, float& y,
                                        float& z) {
  if (s >= p.M) s = p.M - 1;
  if (p.src_mode == SRC_POINTS) {
    const float* q = p.points + 3 * s;
    x = __ldg(q);
    y = __ldg(q + 1);
    z = __ldg(q + 2);
  } else if (p.src_mode == SRC_RAYS && s >= p.M_rays) {
    const float* q = p.extra_points + 3 * (s - p.M_rays);   // free points riding behind the ray samples
    x = __ldg(q);
    y = __ldg(q + 1);
    z = __ldg(q + 2);
  } else if (p.src_mode == SRC_RAYS) {
    long long r = s / p.n_per_ray;
    float t = __ldg(p.zvals + s);
    const float* o = p.origins + 3 * r;
    const float* d = p.directions + 3 * r;
    // cast_rays (model_utils.py:97-101): separate multiply and add, no FMA contraction
    x = __fadd_rn(__ldg(o), __fmul_rn(t, __ldg(d)));
    y = __fadd_rn(__ldg(o + 1), __fmul_rn(t, __ldg(d + 1)));
    z = __fadd_rn(__ldg(o + 2), __fmul_rn(t, __ldg(d + 2)));
  } else {
    // extraction grid (octree/extraction.py:296-304): ((i + 0.5)/reso - offset)/scale
    long long plane = (long long)p.g_ny * p.g_nz;
    int ix = int(s / plane) + p.g_x0;
    int rem = int(s % plane);
    int iy = rem / p.g_nz;
    int iz = rem % p.g_nz;
    float inv = 1.0f / float(p.g_reso);  // reso is a power of two in the reference; see host check
    float ax = __fmul_rn(__fadd_rn(float(ix), 0.5f), inv);
    float ay = __fmul_rn(__fadd_rn(float(iy), 0.5f), inv);
    float az = __fmul_rn(__fadd_rn(float(iz), 0.5f), inv);
    x = __fdiv_rn(__fsub_rn(ax, p.g_offset[0]), p.g_scale[0]);
    y = __fdiv_rn(__fsub_rn(ay, p.g_offset[1]), p.g_scale[1]);
    z = __fdiv_rn(__fsub_rn(az, p.g_offset[2]), p.g_scale[2]);
  }
}

// Positional encoding of one sample into the E tile(s), posenc(x, min_deg, max_deg, legacy) with L = max_deg - min_deg
// (model_utils.py:145-173).  Feature k = 3 + i of the W = 3 + 6L is, for i < 6L and c = i % 3:
//   standard order: [x(3), sin(2^j x_c) j-major (3L), sin(2^j x_c + pi/2) (3L)]
//   legacy order:   [x(3), per degree j: sin(2^j x_c) (3), sin(2^j x_c + pi/2) (3)]
// (the default (0, 10, standard) is [x, 30 sines, 30 cosines]).  Columns [W, 63) are 0 and column 63 = 1 (bias
// carrier).  xb = x_c * 2^j is the exact fp32 product, the cosine the sine of the fp32 sum xb + pi/2, as the
// reference's jnp expression.  unit_lo/unit_hi: which 16-byte units (8 features each) this thread stores.
// GENERIC = false is the default encoder (0, 10, standard) with every index, scale and order a compile-time constant:
// the fixed encoder's code.  The runtime decode of GENERIC = true sits on the forward's critical path (the MMAs wait
// for the tile): compiled into the default's function it cost the default fp16 training step 2.4 %, and beside it
// 0.5 % (H100 80 GB HBM3, 700 W), so the fp16 forwards call a separate instantiation for the default (posenc_row).
// 2^j is built from its exponent bits there, exact for 0 <= j <= 30.
template <int NSPLIT, bool PRECISE, bool GENERIC>
__device__ __noinline__ void posenc_row_of(uint8_t* e_hi, uint8_t* e_lo, int row, float x, float y,
                                           float z, int unit_lo, int unit_hi, PosencDesc pe, uint8_t* e_glob) {
  float f[64];
  f[0] = x;
  f[1] = y;
  f[2] = z;
  const float xyz[3] = {x, y, z};
  const float half_pi = 1.5707963267948966f;
  const int min_deg = GENERIC ? pe.min_deg : 0;
  const bool legacy = GENERIC ? pe.legacy != 0 : false;
  const int L3 = GENERIC ? 3 * (pe.max_deg - pe.min_deg) : 30;   // sines (and cosines) per sample
#pragma unroll
  for (int i = 0; i < ENC_DIM - 3; ++i) {
    const int c = i % 3;                          // the same in both orders: every block is a multiple of 3 wide
    const bool cosine = legacy ? (i % 6) >= 3 : i >= L3;
    const bool on = i < 2 * L3;
    const int j = on ? min_deg + (legacy ? i / 6 : (cosine ? i - L3 : i) / 3) : 0;
    const float sc = GENERIC ? __int_as_float((127 + j) << 23) : float(1 << j);
    const float xb = __fmul_rn(xyz[c], sc);
    const float v = posenc_sin<PRECISE>(cosine ? __fadd_rn(xb, half_pi) : xb);
    f[3 + i] = on ? v : 0.f;
  }
  f[63] = 1.f;   // constant-one column: carries the biases through the tensor cores (common.cuh)
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    if (u < unit_lo || u >= unit_hi) continue;
    uint32_t w[4], wl[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float a = f[8 * u + 2 * i], b = f[8 * u + 2 * i + 1];
      w[i] = pack_f16x2(a, b);
      if (NSPLIT == 3) {
        float2 h = unpack_f16x2(w[i]);
        wl[i] = pack_f16x2(a - h.x, b - h.y);
      }
    }
    const uint32_t off = uint32_t(row) * 128u + (uint32_t(u ^ (row & 7)) << 4);
    *reinterpret_cast<uint4*>(e_hi + off) = make_uint4(w[0], w[1], w[2], w[3]);
    if (NSPLIT == 3) *reinterpret_cast<uint4*>(e_lo + off) = make_uint4(wl[0], wl[1], wl[2], wl[3]);
    if (e_glob) *reinterpret_cast<uint4*>(e_glob + off) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

template <int NSPLIT, bool PRECISE>
__device__ __forceinline__ void posenc_row(uint8_t* e_hi, uint8_t* e_lo, int row, float x, float y, float z,
                                           int unit_lo, int unit_hi, PosencDesc pe, uint8_t* e_glob) {
  // x3 runs the generic code for every encoder: a default instantiation beside libdevice sinf raised its spills
  if (NSPLIT == 1 && pe.min_deg == POSENC_DEFAULT.min_deg && pe.max_deg == POSENC_DEFAULT.max_deg && pe.legacy == 0)
    posenc_row_of<NSPLIT, PRECISE, false>(e_hi, e_lo, row, x, y, z, unit_lo, unit_hi, pe, e_glob);
  else
    posenc_row_of<NSPLIT, PRECISE, true>(e_hi, e_lo, row, x, y, z, unit_lo, unit_hi, pe, e_glob);
}


// fp16 trunk epilogue: activation of the accumulator in fp32, then the fp16 pack into the next A operand.  Relu is
// the fused cvt.rn.relu of acc_to_afrag.
template <int ACT>
__device__ __forceinline__ void act_to_afrag(const float (&acc)[128], uint32_t (&a)[64]) {
  if constexpr (ACT == NET_RELU) {
    acc_to_afrag<true>(acc, a);
  } else {
#pragma unroll
    for (int i = 0; i < 64; ++i) a[i] = pack_f16x2(net_act_f32<ACT>(acc[2 * i]), net_act_f32<ACT>(acc[2 * i + 1]));
  }
}

// heads staging row r (0..63) of warpgroup wg: inside the warpgroup's own (dead after the heads MMAs) rows of the
// activation tile, 16 rows per 8 KB piece
__device__ __forceinline__ float* stage_row(uint8_t* a_tile, int wg, int r) {
  return reinterpret_cast<float*>(a_tile + uint32_t(r >> 4) * A_CHUNK_BYTES + uint32_t(wg) * 8192u) +
         (r & 15) * STAGE_PITCH;
}

}  // namespace

// OUTM (= p.out_mode) is a template parameter so that each instantiation carries only its own heads epilogue, ACT
// (= p.net_act) so that each carries only its trunk activation; the relu instantiations are the relu-only kernel's
// code.  Only relu writes mask words (SAVE): the data gradient of the others reads h_l itself.
template <int NSPLIT, int OUTM, bool SAVE, int ACT>
__global__ void __launch_bounds__(FWD_THREADS, 1) mlp_fwd_kernel(const __grid_constant__ FwdParams p) {
  constexpr bool MASKS = SAVE && ACT == NET_RELU;
  constexpr int HN = OUTM == OUT_VANILLA ? VANILLA_NH : HEADS_N;   // heads MMA width
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr bool PRECISE = (NSPLIT == 3);
  using SM = Smem<NSPLIT, SAVE>;
  __shared__ __align__(8) Ring<SM::STAGES> ring;

  // training launches cover the padded rows: mlp_bwd / mlp_wgrad read every tile of the padded arrays
  const long long num_tiles = SAVE ? padded_rows(p.M) / TILE_M : (p.M + TILE_M - 1) / TILE_M;
  const uint32_t warp = warp_id(), lane = lane_id();
  const uint32_t sbase = smem_u32(smem);
  const int NH = p.NH;

  if (threadIdx.x == 0) ring.init(SM::STAGES);
  __syncthreads();

  if (warp >= PRODUCER_WARP) {
    // =============================== weight producer ===================================
    // whole-warp control flow, one elected lane issues
    setmaxnreg_dec<40>();
    if (warp != PRODUCER_WARP) return;
    RingPos pos;
    for (long long it = blockIdx.x; it < num_tiles; it += gridDim.x) {
      size_t off = 0;
#pragma unroll (SM::PRODUCER_UNROLL)
      for (int l = 0; l <= NUM_TRUNK; ++l) {
        const int ns = (l == NUM_TRUNK) ? FWD_HEAD_SLOTS : fwd_slots_of_layer(l);
        const uint32_t bytes = (l == NUM_TRUNK) ? uint32_t(NH) * 64u : uint32_t(WSLOT_BYTES);
#pragma unroll (SM::PRODUCER_UNROLL)
        for (int j = 0; j < ns; ++j) {
          ring.acquire(pos);
          if (elect_one()) {
            const uint32_t bar = ring.arm(pos, SM::PARTS * bytes);
            const uint32_t dst = sbase + SM::W + pos.stage * SM::STAGE_BYTES;
            bulk_g2s(dst, p.w.w_hi + off, bytes, bar);
            if (NSPLIT == 3) bulk_g2s(dst + WSLOT_BYTES, p.w.w_lo + off, bytes, bar);
          }
          __syncwarp();
          pos.advance(SM::STAGES);
          off += bytes;
        }
      }
    }
    return;
  }

  // ================================ consumer warpgroups =================================
  setmaxnreg_inc<232>();
  const int wg = int(warp >> 2);
  const int t = int(threadIdx.x & 127);
  const int wq = t >> 5;                                   // warp within the warpgroup
  const int fr = 16 * wq + int(lane >> 2);                 // fragment row (and fr + 8) within the warpgroup's rows
  const int fc = 2 * int(lane & 3);                        // fragment column offset within an 8-column group
  uint8_t* const a_hi = smem + SM::A0;
  uint8_t* const a_lo = smem + SM::A1;
  uint8_t* const e_hi = smem + SM::E0;
  uint8_t* const e_lo = smem + SM::E1;
  const uint32_t rows_off = uint32_t(wg) * 64u * 128u;     // this warpgroup's 64 rows inside every 128-row chunk
  constexpr uint64_t A_DESC = make_sdesc_hi(16, 1024, LAYOUT_SW128);
  constexpr uint64_t W_DESC = make_sdesc_hi(16, 512, LAYOUT_SW64);
  RingPos pos;
  float acc[128];
  float hacc[HN / 2];
  uint32_t afr[64];        // fp16: the previous layer's ReLU output as the register A operand (acc_to_afrag)
  long long it = blockIdx.x;

  // shared-memory A operand of k16 group pair kk (columns 32kk..32kk+31) of the posenc tile
  auto e_operand = [&](int kk) {
    return sbase + SM::E0 + uint32_t(kk >> 1) * A_CHUNK_BYTES + rows_off + uint32_t(kk & 1) * 64u;
  };

  // Training save of K-slot c's share of h_lh (columns 32c..32c+31) from the A registers that carried it, once the
  // slot's MMAs have completed: the "T" image and mask word c, whose bits come from the fp16 values (h > 0 <=>
  // fp16(h) != 0 up to fp16 underflow).
  auto save_slot = [&](int lh, int c, uint32_t (&maskw)[4]) {
    uint8_t* const h_glob = p.save_h + t_frag_base(it, lh, wg, wq, lane);
    uint32_t m[2] = {0u, 0u};
#pragma unroll
    for (int i = 0; i < 8; ++i) {            // afr[8c + i]: k16 step i/4 of the slot, register i%4
      const uint32_t w = afr[8 * c + i];
      const int h = i & 1;                    // row fr + 8h
      const int hi8 = (i >> 1) & 1;           // second 8 columns of the k16 step
      *reinterpret_cast<uint32_t*>(h_glob + t_frag_offset(4 * c + 2 * (i >> 2) + hi8, h)) = w;
      if constexpr (MASKS) {
        const int k = 8 * (i >> 2) + 4 * hi8 + int(lane & 3);   // column pair within the mask word
        m[h] |= mask_pair_bits(__vminu2(w, 0x00010001u), k);    // non-negative fp16 pair -> 0/1 per half
      }
    }
    if constexpr (MASKS) mask_quad_reduce(m, c, maskw);
  };

  // fp16 layer l >= 1 (l = NUM_TRUNK: the heads, into hacc): K-slots 0..7 take h_{l-1} from afr, the bias slot and
  // layer 5's skip slots the posenc tile.  The first MMA is issued as soon as h_{l-1} is packed; the training save of
  // h_{l-1} then runs one K-slot behind the MMAs.
  auto chain_layer = [&](auto& d, const int l) {
    constexpr bool HEADS = sizeof(d) == sizeof(hacc);
    const int ns = HEADS ? FWD_HEAD_SLOTS : fwd_slots_of_layer(l);
    uint32_t maskw[4];
    uint32_t prev = 0;
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 10; ++j) {
      if (j == ns) break;
      const uint32_t b = sbase + SM::W + pos.stage * SM::STAGE_BYTES;
      ring.wait(pos);
      if (j < 8) {
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const uint32_t* a = afr + 8 * j + 4 * k;
          const uint64_t bd = sdesc(W_DESC, b + 32u * k);
          const uint32_t sd = (j != 0 || k != 0) ? 1u : 0u;
          if constexpr (HEADS && HN == VANILLA_NH) wgmma_m64n136_rs(d, a[0], a[1], a[2], a[3], bd, sd);
          else if constexpr (HEADS) wgmma_m64n80_rs(d, a[0], a[1], a[2], a[3], bd, sd);
          else wgmma_m64n256_rs(d, a[0], a[1], a[2], a[3], bd, sd);
        }
      } else {
        // the bias slot only multiplies the k16 group [48,64) of the posenc tile (column 63 = 1) with its row k = 31
        const bool bias_slot = fwd_has_bias_slot(l);
        const uint32_t a = e_operand(bias_slot ? 1 : j - 8);
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          if (k == 0 && bias_slot) continue;
          const uint32_t ko = uint32_t(k) * 32u;
          if constexpr (HEADS && HN == VANILLA_NH) wgmma_m64n136<0, 0>(d, sdesc(A_DESC, a + ko), sdesc(W_DESC, b + ko), 1u);
          else if constexpr (HEADS) wgmma_m64n80<0, 0>(d, sdesc(A_DESC, a + ko), sdesc(W_DESC, b + ko), 1u);
          else wgmma_m64n256<0, 0>(d, sdesc(A_DESC, a + ko), sdesc(W_DESC, b + ko), 1u);
        }
      }
      wgmma_commit();
      if (j > 0) {
        // the previous K-slot's MMAs are complete: hand its stage back to the producer, save its share of h_{l-1}
        wgmma_wait<1>();
        ring.release(prev);
        if (SAVE && j <= 8) save_slot(l - 1, j - 1, maskw);
      }
      prev = pos.stage;
      pos.advance(SM::STAGES);
    }
    wgmma_wait<0>();
    ring.release(prev);
    if (MASKS) store_mask_words(p.save_mask, padded_rows(p.M), l - 1, it * TILE_M + 64 * wg + fr, maskw);
  };

  // heads: accumulator fragment -> per-row fp32 staging (column n = packed heads column) inside the warpgroup's own
  // rows of the activation tile, then one thread per row.  The staging rows are rewritten only after the next tile's
  // posenc barrier.
  auto heads_epilogue = [&]() {
#pragma unroll
    for (int j = 0; j < HEADS_N / 8; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float* st = stage_row(a_hi, wg, fr + 8 * h);
        st[8 * j + fc] = hacc[4 * j + 2 * h];
        st[8 * j + fc + 1] = hacc[4 * j + 2 * h + 1];
      }
    }
    warpgroup_sync(wg);
    const int K = p.K;
    const long long row0 = it * TILE_M + 64 * wg;   // first sample of the warpgroup's rows
    if (OUTM == OUT_RGBS) {
      if (t < 64 && row0 + t < p.M) {
        const long long s = row0 + t;
        const float* st = stage_row(a_hi, wg, t);
        float basis[25];
        const long long vi = (p.src_mode == SRC_RAYS) ? (s < p.M_rays ? s / p.n_per_ray : 0) : s;   // free points: any direction
        const float* vd = p.viewdirs + 3 * vi;
        if (p.sh_deg >= 0) sh_basis(p.sh_deg, __ldg(vd), __ldg(vd + 1), __ldg(vd + 2), basis);
        else basis[0] = 1.f;
        float pre[3] = {0.f, 0.f, 0.f};
        for (int k = 0; k < K; ++k) {
#pragma unroll
          for (int c = 0; c < 3; ++c) pre[c] = fmaf(basis[k], st[heads_column(k, c)], pre[c]);
        }
        float sigma_raw = st[0];
        float4 o;
        o.x = 1.f / (1.f + expf(-pre[0]));
        o.y = 1.f / (1.f + expf(-pre[1]));
        o.z = 1.f / (1.f + expf(-pre[2]));
        // ray samples (and SRC_POINTS rows) take the noise and the model's density activation; the free sparsity
        // points behind them keep relu of raw sigma, the value sparsity_grad_kernel reads (train.py:82)
        const bool sample_row = p.src_mode != SRC_RAYS || s < p.M_rays;
        if (p.sigma_noise != nullptr && sample_row) sigma_raw += __ldg(p.sigma_noise + s);  // add_gaussian_noise
        o.w = (p.sigma_act == SIGMA_SOFTPLUS && sample_row) ? softplus_f32(sigma_raw) : fmaxf(sigma_raw, 0.f);
        p.out_rgbs[s] = o;
      }
    } else if (OUTM == OUT_SIGMA || OUTM == OUT_RAW) {
      if (t < 64 && row0 + t < p.M) p.out_sigma[row0 + t] = stage_row(a_hi, wg, t)[0];
      if (OUTM == OUT_RAW) {
        // reference channel-major order
        const int C3 = 3 * K;
        for (int rr = 0; rr < 64 && row0 + rr < p.M; ++rr) {
          const float* st = stage_row(a_hi, wg, rr);
          for (int i = t; i < C3; i += 128) p.out_rgb[(row0 + rr) * C3 + i] = st[heads_column_of_output(i, K)];
        }
      }
    } else if (OUTM == OUT_CELL_MEAN) {
      // extraction step 2 (octree/extraction.py:367-394): out[cell] += cat([raw_rgb, raw_sigma]) / S.
      const int width = 3 * K + 1;
      const float inv = 1.0f / float(p.cell_S);
      auto col_of = [&](int i) { return i == 3 * K ? 0 : heads_column_of_output(i, K); };
      if ((p.cell_S & 31) == 0) {
        // 32 consecutive rows belong to one cell: 64 threads per 32-row half sum over rows, one atomic per column
        const int hf = t >> 6;
        const long long r0 = row0 + 32 * hf;
        if (r0 < p.M) {
          float* dst = p.out_cell + (r0 / p.cell_S) * width;
          for (int i = t & 63; i < width; i += 64) {
            const int n = col_of(i);
            float a = 0.f;
            for (int rr = 0; rr < 32; ++rr) a += stage_row(a_hi, wg, 32 * hf + rr)[n];
            atomicAdd(dst + i, a * inv);
          }
        }
      } else {
        for (int rr = 0; rr < 64 && row0 + rr < p.M; ++rr) {
          float* dst = p.out_cell + ((row0 + rr) / p.cell_S) * width;
          for (int i = t; i < width; i += 128) atomicAdd(dst + i, stage_row(a_hi, wg, rr)[col_of(i)] * inv);
        }
      }
    }
    // reconverge before the next tile's MMAs: after the cell-mean loops ptxas otherwise serializes every wgmma of the
    // kernel (C7520).  The x3 forwards keep their instruction stream.
    if (NSPLIT == 1) __syncwarp();
  };

  // vanilla view branch, in registers: the quad of lanes holding rows fr and fr + 8 holds their 128 a_p columns, 32
  // per lane (8-column groups j = 1..16).  Each lane forms its share of W11 act(a_p + t_r) in a fixed column order, the
  // quad sums the shares with two butterfly shuffles (every lane ends with the same sums), and lane 0 of the quad writes
  // row fr, lane 1 row fr + 8.  No staging, no a_p in memory.
  auto vanilla_epilogue = [&]() {
    const int q = int(lane & 3);
    const long long row0 = it * TILE_M + 64 * wg + fr;
    const float* tr[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      long long s = row0 + 8 * h;
      if (s >= p.M) s = p.M - 1;
      tr[h] = p.view_t + (p.src_mode == SRC_RAYS ? s / p.n_per_ray : s) * VIEW_H;
    }
    float pre[2][3];
#pragma unroll
    for (int h = 0; h < 2; ++h) {   // one row at a time: the softplus condition layer then fits without spilling
      pre[h][0] = pre[h][1] = pre[h][2] = 0.f;
#pragma unroll
      for (int j = VIEW_COL0 / 8; j < HN / 8; ++j) {
        const int col = 8 * j - VIEW_COL0 + fc;   // this lane's column pair of 8-column group j
        const float2 t2 = __ldg(reinterpret_cast<const float2*>(tr[h] + col));
        const float z0 = net_act_f32<ACT>(hacc[4 * j + 2 * h] + t2.x);
        const float z1 = net_act_f32<ACT>(hacc[4 * j + 2 * h + 1] + t2.y);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float w0 = __ldg(p.view_w11 + col * 3 + c), w1 = __ldg(p.view_w11 + (col + 1) * 3 + c);
          pre[h][c] = fmaf(w1, z1, fmaf(w0, z0, pre[h][c]));
        }
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        pre[h][c] += __shfl_xor_sync(0xffffffffu, pre[h][c], 1);
        pre[h][c] += __shfl_xor_sync(0xffffffffu, pre[h][c], 2);
      }
    }
    // raw sigma of rows fr, fr + 8: column 0, held by lane 0 of the quad
    const float sg0 = __shfl_sync(0xffffffffu, hacc[0], int(lane) & ~3);
    const float sg1 = __shfl_sync(0xffffffffu, hacc[2], int(lane) & ~3);
    if (q < 2) {
      const long long s = row0 + 8 * q;
      if (s < p.M) {
        const float r0 = (q ? pre[1][0] : pre[0][0]) + __ldg(p.view_b11);
        const float r1 = (q ? pre[1][1] : pre[0][1]) + __ldg(p.view_b11 + 1);
        const float r2 = (q ? pre[1][2] : pre[0][2]) + __ldg(p.view_b11 + 2);
        float sigma_raw = q ? sg1 : sg0;
        if (p.out_rgbs) {
          if (p.sigma_noise != nullptr) sigma_raw += __ldg(p.sigma_noise + s);   // add_gaussian_noise
          float4 o;
          o.x = 1.f / (1.f + expf(-r0));
          o.y = 1.f / (1.f + expf(-r1));
          o.z = 1.f / (1.f + expf(-r2));
          o.w = p.sigma_act == SIGMA_SOFTPLUS ? softplus_f32(sigma_raw) : fmaxf(sigma_raw, 0.f);
          p.out_rgbs[s] = o;
        } else {
          p.out_rgb[3 * s] = r0;
          p.out_rgb[3 * s + 1] = r1;
          p.out_rgb[3 * s + 2] = r2;
          p.out_sigma[s] = sigma_raw;
        }
      }
    }
    __syncwarp();
  };

  for (; it < num_tiles; it += gridDim.x) {
    // ---- positional encoding of the warpgroup's 64 rows (two threads per row, four 16-byte units each) ----
    {
      const int r = 64 * wg + (t & 63);
      const int u0 = 4 * (t >> 6);
      float x, y, z;
      load_point(p, it * TILE_M + r, x, y, z);
      posenc_row<NSPLIT, PRECISE>(e_hi, e_lo, r, x, y, z, u0, u0 + 4, p.pe,
                                  SAVE ? p.save_e + size_t(it) * E_TILE_BYTES : nullptr);
      fence_proxy_async_smem();
      warpgroup_sync(wg);
      if constexpr (SAVE && NSPLIT == 3) {
        // x3 training save of the posenc residual: the warpgroup's 64 rows of the lo tile (8 KB), as written above
        uint8_t* const dst = p.save_e_lo + size_t(it) * E_TILE_BYTES + rows_off;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const uint32_t o = (uint32_t(i) * 128u + uint32_t(t)) * 16u;
          *reinterpret_cast<uint4*>(dst + o) = *reinterpret_cast<const uint4*>(e_lo + rows_off + o);
        }
      }
    }
    if constexpr (NSPLIT == 1) {
      // ---- fp16: layer 0 from the posenc tile, then every layer's activations stay in registers ----
      uint32_t prev = 0;
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const uint32_t a = e_operand(j);
        const uint32_t b = sbase + SM::W + pos.stage * SM::STAGE_BYTES;
        ring.wait(pos);
        wgmma_m64n256<0, 0>(acc, sdesc(A_DESC, a), sdesc(W_DESC, b), j != 0);
        wgmma_m64n256<0, 0>(acc, sdesc(A_DESC, a + 32), sdesc(W_DESC, b + 32), 1u);
        wgmma_commit();
        if (j > 0) {
          wgmma_wait<1>();
          ring.release(prev);
        }
        prev = pos.stage;
        pos.advance(SM::STAGES);
      }
      wgmma_wait<0>();
      ring.release(prev);
      // activation + fp16 pack of the accumulator (the bias was accumulated by the tensor cores) into the next A
      // operand
      act_to_afrag<ACT>(acc, afr);
      for (int l = 1; l < NUM_TRUNK; ++l) {
        chain_layer(acc, l);
        act_to_afrag<ACT>(acc, afr);
      }
      chain_layer(hacc, NUM_TRUNK);
      if constexpr (OUTM == OUT_VANILLA) vanilla_epilogue();
      else heads_epilogue();
    } else {
      // ---- x3: every operand from shared memory; the epilogue rewrites the warpgroup's rows of the A tiles ----
      for (int l = 0; l <= NUM_TRUNK; ++l) {
        const bool heads = l == NUM_TRUNK;
        const int ns = heads ? FWD_HEAD_SLOTS : fwd_slots_of_layer(l);
        uint32_t prev = 0;
        wgmma_fence();
        for (int j = 0; j < ns; ++j) {
          // A operand of K-slot j: the previous layer's activations, or the posenc tile for layer 0, the skip slots
          // of layer 5, and the bias slot (j == 8) of every other layer, which only multiplies the k16 group
          // [48,64) of the posenc tile (column 63 = 1) with its row k = 31.
          const bool bias_slot = (heads || fwd_has_bias_slot(l)) && j == 8;
          const bool from_e = (l == 0) || j >= 8;
          const int kk = bias_slot ? 1 : ((l == SKIP_LAYER && j >= 8) ? j - 8 : j);
          const uint32_t a_off = uint32_t(kk >> 1) * A_CHUNK_BYTES + rows_off + uint32_t(kk & 1) * 64u;
          const uint32_t ah = sbase + (from_e ? SM::E0 : SM::A0) + a_off;
          const uint32_t al = sbase + (from_e ? SM::E1 : SM::A1) + a_off;
          const uint32_t bh = sbase + SM::W + pos.stage * SM::STAGE_BYTES;
          const uint32_t bl = bh + WSLOT_BYTES;
          ring.wait(pos);
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            if (k == 0 && bias_slot) continue;
            const uint32_t sd = (j != 0 || k != 0) ? 1u : 0u;
            const uint32_t ko = uint32_t(k) * 32u;   // k16 step: +32 bytes inside the swizzled rows
            if (heads) {
              wgmma_m64n80<0, 0>(hacc, sdesc(A_DESC, al + ko), sdesc(W_DESC, bh + ko), sd);
              wgmma_m64n80<0, 0>(hacc, sdesc(A_DESC, ah + ko), sdesc(W_DESC, bl + ko), 1u);
              wgmma_m64n80<0, 0>(hacc, sdesc(A_DESC, ah + ko), sdesc(W_DESC, bh + ko), 1u);
            } else {
              wgmma_m64n256<0, 0>(acc, sdesc(A_DESC, al + ko), sdesc(W_DESC, bh + ko), sd);
              wgmma_m64n256<0, 0>(acc, sdesc(A_DESC, ah + ko), sdesc(W_DESC, bl + ko), 1u);
              wgmma_m64n256<0, 0>(acc, sdesc(A_DESC, ah + ko), sdesc(W_DESC, bh + ko), 1u);
            }
          }
          wgmma_commit();
          if (j > 0) {
            // the previous K-slot's MMAs are complete: hand its stage back to the producer
            wgmma_wait<1>();
            ring.release(prev);
          }
          prev = pos.stage;
          pos.advance(SM::STAGES);
        }
        wgmma_wait<0>();
        ring.release(prev);

        if (!heads) {
          // ---- trunk epilogue: activation + hi/lo fp16 split straight from the accumulator fragment into the next A
          // operands (the bias was accumulated by the tensor cores).  Only this warpgroup's MMAs read these rows.
          // Training (SAVE): the same hi and lo values go to the "T" images of h_l, and (relu) the mask words of h_l
          // take their bits from the sign of the fp32 pre-activation: relu(v) < 2^-25 rounds to hi = lo = 0 but still
          // has a gradient.  The other activations are applied in fp32 before the split. ----
          size_t t_off = 0;
          uint32_t mrow[2] = {0u, 0u}, maskw[4] = {0u, 0u, 0u, 0u};
          if constexpr (SAVE) t_off = t_frag_base(it, l, wg, wq, lane);
#pragma unroll
          for (int j = 0; j < 32; ++j) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = 64 * wg + fr + 8 * h;
              const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
              const uint32_t off = a_tile_offset(row, 8 * j + fc);
              const float f0 = net_act_f32<ACT>(v0), f1 = net_act_f32<ACT>(v1);
              const uint32_t w = ACT == NET_RELU ? pack_f16x2_relu(v0, v1) : pack_f16x2(f0, f1);
              *reinterpret_cast<uint32_t*>(a_hi + off) = w;
              const float2 hv = unpack_f16x2(w);
              const uint32_t wl = pack_f16x2(f0 - hv.x, f1 - hv.y);
              *reinterpret_cast<uint32_t*>(a_lo + off) = wl;
              if constexpr (SAVE) {
                const size_t go = t_off + t_frag_offset(j, h);
                *reinterpret_cast<uint32_t*>(p.save_h + go) = w;
                *reinterpret_cast<uint32_t*>(p.save_h_lo + go) = wl;
              }
              if constexpr (MASKS) {
                const int k = 4 * (j & 3) + (fc >> 1);   // column pair within the mask word
                mrow[h] |= (v0 > 0.f ? 1u << mask_bit(k, 0) : 0u) | (v1 > 0.f ? 1u << mask_bit(k, 1) : 0u);
              }
            }
            if (MASKS && (j & 3) == 3) {
              mask_quad_reduce(mrow, j >> 2, maskw);
              mrow[0] = mrow[1] = 0u;
            }
          }
          if constexpr (MASKS) store_mask_words(p.save_mask, padded_rows(p.M), l, it * TILE_M + 64 * wg + fr, maskw);
          fence_proxy_async_smem();
          warpgroup_sync(wg);
          continue;
        }
        heads_epilogue();
      }
    }
  }
}

// the vanilla view-branch forward (OUT_VANILLA): fp16, no training saves, no free points behind the ray samples
cudaError_t launch_mlp_fwd_vanilla(const FwdParams& p, int num_sms, cudaStream_t stream) {
  if (p.M <= 0) return cudaSuccess;
  if (p.out_mode != OUT_VANILLA || p.NH != VANILLA_NH || p.save_h || !p.view_t || !p.view_w11 || !p.view_b11 ||
      (!p.out_rgbs && (!p.out_rgb || !p.out_sigma)) || (p.src_mode == SRC_RAYS && p.M != p.M_rays) ||
      (p.sigma_act != SIGMA_RELU && p.sigma_act != SIGMA_SOFTPLUS) || !posenc_valid(p.pe))
    return cudaErrorInvalidValue;
  const long long tiles = (p.M + TILE_M - 1) / TILE_M;
  const int grid = int(tiles < num_sms ? tiles : num_sms);
  auto launch = [&](auto kernel) -> cudaError_t {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SM_TOTAL);
    if (e != cudaSuccess) return e;
    kernel<<<grid, FWD_THREADS, SM_TOTAL, stream>>>(p);
    return cudaGetLastError();
  };
  switch (p.net_act) {
    case NET_RELU: return launch(mlp_fwd_kernel<1, OUT_VANILLA, false, NET_RELU>);
    case NET_ELU: return launch(mlp_fwd_kernel<1, OUT_VANILLA, false, NET_ELU>);
    case NET_SOFTPLUS: return launch(mlp_fwd_kernel<1, OUT_VANILLA, false, NET_SOFTPLUS>);
    case NET_TANH: return launch(mlp_fwd_kernel<1, OUT_VANILLA, false, NET_TANH>);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_mlp_fwd(const FwdParams& p, int nsplit, int num_sms, cudaStream_t stream) {
  if (p.M <= 0) return cudaSuccess;
  if (nsplit != 1 && nsplit != 3) return cudaErrorInvalidValue;
  if (p.sigma_act != SIGMA_RELU && p.sigma_act != SIGMA_SOFTPLUS) return cudaErrorInvalidValue;
  if (!posenc_valid(p.pe)) return cudaErrorInvalidValue;
  const bool save = p.save_h != nullptr;
  if (save && (!p.save_e || !p.save_mask || (p.out_mode != OUT_RGBS && p.out_mode != OUT_SIGMA)))
    return cudaErrorInvalidValue;
  // the x3 training forward: the rgbs epilogue of the render path, plus the residual images
  if (save && nsplit == 3 && (!p.save_h_lo || !p.save_e_lo || p.out_mode != OUT_RGBS)) return cudaErrorInvalidValue;
  const long long tiles = save ? padded_rows(p.M) / TILE_M : (p.M + TILE_M - 1) / TILE_M;
  const int grid = int(tiles < num_sms ? tiles : num_sms);
  auto launch = [&](auto kernel) -> cudaError_t {
    cudaError_t e =
        cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SM_TOTAL);
    if (e != cudaSuccess) return e;
    kernel<<<grid, FWD_THREADS, SM_TOTAL, stream>>>(p);
    return cudaGetLastError();
  };
  auto dispatch = [&](auto act) -> cudaError_t {
    constexpr int A = decltype(act)::value;
    switch (p.out_mode) {
      case OUT_RAW:
        return nsplit == 1 ? launch(mlp_fwd_kernel<1, OUT_RAW, false, A>) : launch(mlp_fwd_kernel<3, OUT_RAW, false, A>);
      case OUT_SIGMA:
        if (save) return launch(mlp_fwd_kernel<1, OUT_SIGMA, true, A>);
        return nsplit == 1 ? launch(mlp_fwd_kernel<1, OUT_SIGMA, false, A>)
                           : launch(mlp_fwd_kernel<3, OUT_SIGMA, false, A>);
      case OUT_RGBS:
        if (save)
          return nsplit == 1 ? launch(mlp_fwd_kernel<1, OUT_RGBS, true, A>) : launch(mlp_fwd_kernel<3, OUT_RGBS, true, A>);
        return nsplit == 1 ? launch(mlp_fwd_kernel<1, OUT_RGBS, false, A>) : launch(mlp_fwd_kernel<3, OUT_RGBS, false, A>);
      case OUT_CELL_MEAN:
        return nsplit == 1 ? launch(mlp_fwd_kernel<1, OUT_CELL_MEAN, false, A>)
                           : launch(mlp_fwd_kernel<3, OUT_CELL_MEAN, false, A>);
      default:
        return cudaErrorInvalidValue;
    }
  };
  switch (p.net_act) {
    case NET_RELU: return dispatch(std::integral_constant<int, NET_RELU>());
    case NET_ELU: return dispatch(std::integral_constant<int, NET_ELU>());
    case NET_SOFTPLUS: return dispatch(std::integral_constant<int, NET_SOFTPLUS>());
    case NET_TANH: return dispatch(std::integral_constant<int, NET_TANH>());
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace pob
