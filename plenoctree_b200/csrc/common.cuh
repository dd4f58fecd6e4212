// common.cuh — sm_90a building blocks shared by every kernel of the NeRF-SH hot path.
//
// Everything here is a thin inline-PTX wrapper (mbarrier, bulk async copy = TMA 1-D, wgmma,
// proxy fences) plus the shared-memory operand layouts the tensor-core kernels agree on.  No
// CUTLASS / CuTe types: the descriptor bit layout follows the PTX ISA's wgmma matrix descriptor
// (the same fields as CuTe's GmmaDescriptor) and its canonical K-/MN-major layouts.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace pob {

// ----------------------------------------------------------------------------------
// Geometry shared by all MLP kernels
// ----------------------------------------------------------------------------------
constexpr int TILE_M      = 128;           // samples (rows) per tensor-core tile
constexpr int WIDTH       = 256;           // trunk width (reference net_width)
constexpr int ENC_DIM     = 63;            // posenc(x, 0, 10) feature count
constexpr int ENC_PAD     = 64;            // padded to one 64-wide K chunk
constexpr int NUM_TRUNK   = 8;             // net_depth
constexpr int SKIP_LAYER  = 5;             // layer that consumes [h4, enc] (skip after i=4)
constexpr int KCHUNK      = 64;            // fp16 elements per 128-byte swizzle row
constexpr int A_CHUNK_BYTES = TILE_M * 128;        // one [128 x 64] fp16 K-chunk, SW128
constexpr int A_TILE_BYTES  = 4 * A_CHUNK_BYTES;   // [128 x 256] fp16 = 64 KB
constexpr int E_TILE_BYTES  = A_CHUNK_BYTES;       // [128 x 64]  fp16 = 16 KB
constexpr int WSLOT_K       = 32;                  // K extent of one streamed weight slot
constexpr int WSLOT_BYTES   = WIDTH * WSLOT_K * 2; // [256 x 32] fp16, SW64 = 16 KB
constexpr int MAX_NH        = 80;                  // padded heads width (1 + 3*25 -> 80)
// Rows of every per-sample training array (tile images, relu masks), padded to a multiple of 512 rows; the
// training forward evaluates the padded rows too (clamped to the last sample), so every saved tile is finite.
__host__ __device__ constexpr long long padded_rows(long long M) { return ((M + 511) / 512) * 512; }

// Number of 32-wide K slots each forward layer streams (trunk 0..7, heads = index 8).
// Biases ride on the tensor cores: column 63 of the posenc tile is the constant 1, so for layers 0 and
// 5 (which read the posenc tile anyway) the bias is row k=63 of an existing slot; every other layer
// streams one extra "bias slot" whose only non-zero K row (k = 31) is the bias, multiplied by the
// k16 group [48,64) of the posenc tile.  The epilogue therefore has no bias add at all (a broadcast
// LDS.128 per 4 columns costs 4 shared-memory wavefronts per warp: 2048 cycles per layer).
__host__ __device__ constexpr int fwd_has_bias_slot(int l) { return !(l == 0 || l == SKIP_LAYER); }
__host__ __device__ constexpr int fwd_slots_of_layer(int l) {
  return l == 0 ? 2 : (l == SKIP_LAYER ? 10 : 9);
}
constexpr int FWD_TRUNK_SLOTS = 2 + 9 * 4 + 10 + 9 * 2;       // 66
constexpr int FWD_HEAD_SLOTS = 9;
// K slots of the dgrad image: the heads' ceil(NH/32), then Dense_7 .. Dense_1 with 8 each
__host__ __device__ constexpr int bwd_head_slots(int NH) { return (NH + 31) / 32; }
__host__ __device__ constexpr int bwd_slots(int NH) { return bwd_head_slots(NH) + 7 * 8; }

// Heads column order: packed column 0 is sigma (Dense_8), packed column 1 + 3k + c is SH coefficient k of colour
// channel c, which is Dense_9 output c*K + k in the reference's channel-major order.
__host__ __device__ constexpr int heads_column(int k, int c) { return 1 + 3 * k + c; }
// Dense_9 output o (of 3K) -> packed column
__host__ __device__ constexpr int heads_column_of_output(int o, int K) { return heads_column(o % K, o / K); }
// packed column n >= 1 -> (k, c)
__host__ __device__ constexpr void heads_coeff(int n, int& k, int& c) {
  k = (n - 1) / 3;
  c = (n - 1) % 3;
}

// ----------------------------------------------------------------------------------
// Small helpers
// ----------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ uint32_t warp_id() { return threadIdx.x >> 5; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ----------------------------------------------------------------------------------
// Stage ring of the tensor-core kernels: one producer warp bulk-copies operands into shared-memory stages, the two
// consumer warpgroups read every stage with wgmma.  full[s] completes once stage s's bytes have landed, empty[s]
// once every consumer warp has released it.  The depth (<= MAX_DEPTH) is a compile-time or a run-time value.
// ----------------------------------------------------------------------------------
constexpr uint32_t RING_CONSUMER_WARPS = 8;   // two warpgroups; each warp releases a stage once

struct RingPos {
  uint32_t stage = 0, phase = 0;
  __device__ __forceinline__ void advance(uint32_t depth) {
    if (++stage == depth) {
      stage = 0;
      phase ^= 1;
    }
  }
};

template <int MAX_DEPTH>
struct Ring {
  uint64_t full[MAX_DEPTH];
  uint64_t empty[MAX_DEPTH];

  // one thread; a __syncthreads() after it publishes the barriers
  __device__ __forceinline__ void init(int depth) {
    for (int i = 0; i < depth; ++i) {
      mbar_init(smem_u32(&full[i]), 1);
      mbar_init(smem_u32(&empty[i]), RING_CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  // producer warp: wait until the stage is free.  One elected lane then calls arm() and issues the stage's copies.
  __device__ __forceinline__ void acquire(RingPos pos) { mbar_wait(smem_u32(&empty[pos.stage]), pos.phase ^ 1); }
  // the stage's full barrier, expecting `bytes` of bulk copies (to be completed on it)
  __device__ __forceinline__ uint32_t arm(RingPos pos, uint32_t bytes) {
    const uint32_t bar = smem_u32(&full[pos.stage]);
    mbar_arrive_expect_tx(bar, bytes);
    return bar;
  }
  // consumer: wait until the stage's bytes have landed
  __device__ __forceinline__ void wait(RingPos pos) { mbar_wait(smem_u32(&full[pos.stage]), pos.phase); }
  // consumer warp, once its MMAs reading the stage have completed
  __device__ __forceinline__ void release(uint32_t stage) {
    if (lane_id() == 0) mbar_arrive(smem_u32(&empty[stage]));
  }
};

// ----------------------------------------------------------------------------------
// Proxy fence
// ----------------------------------------------------------------------------------
// generic-proxy st.shared -> visible to the async proxy (wgmma operand reads, bulk stores)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ----------------------------------------------------------------------------------
// Bulk async copies (TMA, 1-D).  SASS: UBLKCP.
// ----------------------------------------------------------------------------------
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes,
                                         uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(dst_smem),
      "l"(src), "r"(bytes), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* dst, uint32_t src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst),
               "r"(src_smem), "r"(bytes)
               : "memory");
}
// L2 cache policies (createpolicy: the whole access gets the priority) and the .L2::cache_hint forms of the bulk copies
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void bulk_g2s_hint(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar,
                                              uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::
          "r"(dst_smem),
      "l"(src), "r"(bytes), "r"(bar), "l"(policy)
      : "memory");
}
__device__ __forceinline__ void bulk_s2g_hint(void* dst, uint32_t src_smem, uint32_t bytes, uint64_t policy) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(dst),
               "r"(src_smem), "r"(bytes), "l"(policy)
               : "memory");
}
// Fetch the line holding p into L2 (no register is written; the later load of the line hits L2).  SASS: CCTL.E.PF2.
__device__ __forceinline__ void prefetch_l2(const void* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}
// Drop the 128-byte line at p (128-byte aligned) from L2 without writing it back: a weak write of an undefined value.
// SASS: CCTL.E.RML2.
__device__ __forceinline__ void discard_l2_line(const void* p) {
  asm volatile("discard.global.L2 [%0], 128;" ::"l"(p) : "memory");
}
__device__ __forceinline__ void bulk_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
// wait until the smem source of all committed bulk stores has been read
__device__ __forceinline__ void bulk_wait_read_all() {
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void bulk_wait_all() {
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}
// wait until every committed bulk store except the most recent group has completed (its global writes performed)
__device__ __forceinline__ void bulk_wait_all_but_last() {
  asm volatile("cp.async.bulk.wait_group 1;" ::: "memory");
}

// ----------------------------------------------------------------------------------
// Cross-CTA hand-over of bulk-copied global data (mlp_bwd -> mlp_wgrad progress counters)
// ----------------------------------------------------------------------------------
// async-proxy global accesses <-> generic-proxy accesses of the same thread
__device__ __forceinline__ void fence_proxy_async_global() {
  asm volatile("fence.proxy.async.global;" ::: "memory");
}
__device__ __forceinline__ void red_add_release_gpu(uint32_t* p, uint32_t v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// programmatic dependent launch: the grid launched after this one with programmatic stream serialization may start
// once every CTA of this grid has executed this (or exited)
__device__ __forceinline__ void griddep_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// ----------------------------------------------------------------------------------
// Named barriers (sub-CTA sync)
// ----------------------------------------------------------------------------------
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ----------------------------------------------------------------------------------
// wgmma — fp16 x fp16 -> fp32, operands from shared memory, accumulator in the registers of one
// warpgroup (4 warps, 128 threads).  SASS: HGMMA.
// ----------------------------------------------------------------------------------
// Shared-memory matrix descriptor:
//   [0,14) addr>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [49,52) base offset (0: atoms 1024-B aligned)
//   [62,64) layout type
// K-major swizzled operands: LBO unused (1), SBO = stride between 8-row groups.
// MN-major SW128: LBO = stride between 64-element atoms along M/N, SBO = stride between 8-row K groups.
// MN-major without swizzle: LBO = stride between 8-row K groups, SBO = stride between 8-element M/N groups.
enum : uint32_t { LAYOUT_NONE = 0, LAYOUT_SW128 = 1, LAYOUT_SW64 = 2, LAYOUT_SW32 = 3 };
__host__ __device__ constexpr uint64_t make_sdesc_hi(uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout) {
  return (uint64_t((lbo_bytes >> 4) & 0x3FFF) << 16) | (uint64_t((sbo_bytes >> 4) & 0x3FFF) << 32) |
         (uint64_t(layout) << 62);
}
__device__ __forceinline__ uint64_t sdesc(uint64_t hi, uint32_t smem_addr) {
  return hi | uint64_t((smem_addr >> 4) & 0x3FFF);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// D[64 x N] (+)= A[64 x 16] * B[16 x N].  TRANS_A / TRANS_B = 1: the operand is MN-major in shared memory.
// Accumulator fragment: thread t of the warpgroup holds rows 16*(t/32) + (t%32)/4 (+8) and, for every
// 8-column group j, columns 8j + 2*(t%4) + {0,1}:  d[4j+0..1] = upper row, d[4j+2..3] = row + 8.
template <int TRANS_A, int TRANS_B>
__device__ __forceinline__ void wgmma_m64n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, %35, %36;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TRANS_A), "n"(TRANS_B));
}
template <int TRANS_A, int TRANS_B>
__device__ __forceinline__ void wgmma_m64n80(float (&d)[40], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %42, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, "
      "%40, %41, p, 1, 1, %43, %44;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
      : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TRANS_A), "n"(TRANS_B));
}
template <int TRANS_A, int TRANS_B>
__device__ __forceinline__ void wgmma_m64n256(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, %131, %132;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TRANS_A), "n"(TRANS_B));
}

// Register-A forms.  The A fragment of k16 step kk is four packed fp16x2 registers: rows r = 16*(t/32) + (t%32)/4 and
// r + 8, columns 16kk + 2*(t%4) + {0,1} and 16kk + 8 + 2*(t%4) + {0,1} -- the pairs an m64nN accumulator holds for
// columns 16kk..16kk+15 (see acc_to_afrag).  B is K-major in shared memory.
__device__ __forceinline__ void wgmma_m64n80_rs(float (&d)[40], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                                 uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %45, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, "
      "{%40, %41, %42, %43}, %44, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_m64n256_rs(float (&d)[128], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                                 uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %133, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "{%128, %129, %130, %131}, %132, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(bdesc), "r"(scale_d));
}

// Register budget per warpgroup (all 128 threads execute it): the weight producer gives registers back, the
// consumers that hold an m64n256 accumulator (128 registers) take them.
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// named barrier over the 128 threads of one warpgroup (ids 1.. are free; 0 is __syncthreads)
__device__ __forceinline__ void warpgroup_sync(uint32_t wg) { named_bar_sync(1 + wg, 128); }

// ----------------------------------------------------------------------------------
// fp32 pair -> packed fp16x2 (element `lo` at the lower address), optional fused ReLU
// ----------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ uint32_t pack_f16x2_relu(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float2 unpack_f16x2(uint32_t v) {
  __half2 h = *reinterpret_cast<__half2*>(&v);
  return __half22float2(h);
}
// m64nN accumulator fragment -> register A fragment of the next GEMM (K = N): a[i] packs acc[2i], acc[2i+1], so the
// four A registers of k16 step kk are a[4kk .. 4kk+3] = acc[8kk .. 8kk+7].  Element for element the same conversion
// as an epilogue that stores the accumulator through pack_f16x2(_relu).
template <bool RELU, int NA>
__device__ __forceinline__ void acc_to_afrag(const float (&acc)[2 * NA], uint32_t (&a)[NA]) {
#pragma unroll
  for (int i = 0; i < NA; ++i) a[i] = RELU ? pack_f16x2_relu(acc[2 * i], acc[2 * i + 1]) : pack_f16x2(acc[2 * i], acc[2 * i + 1]);
}

// ----------------------------------------------------------------------------------
// Operand layouts
// ----------------------------------------------------------------------------------
// Activation tile ("A image"): [nchunk][128 rows][128 B], each row = 64 fp16 of one sample,
// 16-byte units XOR-swizzled with (row & 7)  (= cute Swizzle<3,4,3>, K-major SW128 atom).
// The same bytes are a valid MN-major SW128 operand of the transposed matrix (features x
// samples): LBO = chunk stride, SBO = 1024 (8 samples).
__host__ __device__ __forceinline__ constexpr uint32_t a_tile_offset(int row, int col) {
  // byte offset of element (row, col) of a [128 x 64*nchunk] tile
  return uint32_t(col >> 6) * A_CHUNK_BYTES + uint32_t(row) * 128u +
         ((uint32_t((col >> 3) & 7) ^ uint32_t(row & 7)) << 4) + uint32_t(col & 7) * 2u;
}
// Saved activation tile ("T image", layouts.py: t_tile_offset): [32-row group][8-column group][row & 31][16 B], so
// a warp's store of one 8-column group of an accumulator fragment is one contiguous 512 B.  t_frag_base: byte offset,
// in the [tiles][NUM_TRUNK] T images, of the first fragment element of thread `lane` of warp `wq` of warpgroup `wg`
// (row 64wg + 16wq + lane/4, column 2(lane%4)) in layer `layer`'s tile `it`; t_frag_offset: that element's
// offset in 8-column group g, row + 8h.
__device__ __forceinline__ size_t t_frag_base(long long it, int layer, int wg, int wq, uint32_t lane) {
  return (size_t(it) * NUM_TRUNK + layer) * A_TILE_BYTES + uint32_t(2 * wg + (wq >> 1)) * 16384u +
         uint32_t(16 * (wq & 1) + int(lane >> 2)) * 16u + uint32_t(2 * int(lane & 3)) * 2u;
}
__host__ __device__ __forceinline__ constexpr uint32_t t_frag_offset(int g, int h) {
  return uint32_t(g) * 512u + uint32_t(h) * 128u;
}
// ReLU masks (layouts.py: decode_mask): [layer][row][8] words, 1 bit per activation.  Word c covers columns
// 32c..32c+31; column 32c + 2k + e (pair k = 0..15, e = 0, 1) is bit mask_bit(k, e).
__host__ __device__ constexpr int mask_bit(int k, int e) { return 15 - k + 16 * e; }
// bits of pair k from its two flags held as the halves of one word (bit 0: column 2k, bit 16: column 2k + 1)
__device__ __forceinline__ uint32_t mask_pair_bits(uint32_t flags, int k) {
  static_assert(mask_bit(0, 1) == mask_bit(0, 0) + 16, "a pair's bits are 16 apart");
  return flags << mask_bit(k, 0);
}
// Mask words of an accumulator fragment: the four lanes of a quad hold 4 pairs each of word c of rows fr and fr + 8
// (m[0], m[1]).  OR them over the quad; lane q keeps words 4(q&1)..+3 of row fr + 8(q>>1), word c in maskw[c & 3].
__device__ __forceinline__ void mask_quad_reduce(uint32_t (&m)[2], int c, uint32_t (&maskw)[4]) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    m[h] |= __shfl_xor_sync(0xffffffffu, m[h], 1);
    m[h] |= __shfl_xor_sync(0xffffffffu, m[h], 2);
  }
  const uint32_t q = lane_id() & 3;
  if ((q & 1) == uint32_t(c >> 2)) maskw[c & 3] = (q >> 1) ? m[1] : m[0];
}
// lane q's four words (mask_quad_reduce) -> layer `layer` of a [layers][rows][8] mask array; row: the quad's fragment
// row fr
__device__ __forceinline__ void store_mask_words(uint32_t* mask, long long rows, int layer, long long row,
                                                 const uint32_t (&maskw)[4]) {
  const uint32_t q = lane_id() & 3;
  const long long s = row + 8 * int(q >> 1);
  *reinterpret_cast<uint4*>(mask + (size_t(layer) * rows + s) * 8 + 4 * (q & 1)) =
      make_uint4(maskw[0], maskw[1], maskw[2], maskw[3]);
}
// Weight slot ("W image"): [rows][64 B] = 32 fp16 (K) per output row, 16-byte units
// XOR-swizzled with ((row >> 1) & 3)  (= cute Swizzle<2,4,3>, K-major SW64 atom).
__host__ __device__ __forceinline__ constexpr uint32_t w_slot_offset(int row, int k) {
  return uint32_t(row) * 64u + ((uint32_t((k >> 3) & 3) ^ (uint32_t(row >> 1) & 3u)) << 4) +
         uint32_t(k & 7) * 2u;
}

// accurate-enough sine for the positional encoding: Cody-Waite reduction by 2*pi followed by
// the SFU approximation (abs err ~5e-7 for |x| < 1e4); PRECISE selects libdevice sinf.
template <bool PRECISE>
__device__ __forceinline__ float posenc_sin(float a) {
  if (PRECISE) {
    return sinf(a);
  } else {
    float k = rintf(a * 0.15915494309189535f);
    float r = fmaf(k, -6.2831854820251465f, a);
    r = fmaf(k, 1.7484555314695172e-7f, r);
    return __sinf(r);
  }
}

// Real SH basis, sign/ordering convention of the reference (nerf_sh/nerf/sh.py:54-109).
// basis[k] for k < (deg+1)^2; entries beyond are untouched.
__device__ __forceinline__ void sh_basis(int deg, float x, float y, float z, float (&b)[25]) {
  b[0] = 0.28209479177387814f;
  if (deg > 0) {
    b[1] = -0.4886025119029199f * y;
    b[2] = 0.4886025119029199f * z;
    b[3] = -0.4886025119029199f * x;
    if (deg > 1) {
      float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
      b[4] = 1.0925484305920792f * xy;
      b[5] = -1.0925484305920792f * yz;
      b[6] = 0.31539156525252005f * (2.0f * zz - xx - yy);
      b[7] = -1.0925484305920792f * xz;
      b[8] = 0.5462742152960396f * (xx - yy);
      if (deg > 2) {
        b[9] = -0.5900435899266435f * y * (3.f * xx - yy);
        b[10] = 2.890611442640554f * xy * z;
        b[11] = -0.4570457994644658f * y * (4.f * zz - xx - yy);
        b[12] = 0.3731763325901154f * z * (2.f * zz - 3.f * xx - 3.f * yy);
        b[13] = -0.4570457994644658f * x * (4.f * zz - xx - yy);
        b[14] = 1.445305721320277f * z * (xx - yy);
        b[15] = -0.5900435899266435f * x * (xx - 3.f * yy);
        if (deg > 3) {
          b[16] = 2.5033429417967046f * xy * (xx - yy);
          b[17] = -1.7701307697799304f * yz * (3.f * xx - yy);
          b[18] = 0.9461746957575601f * xy * (7.f * zz - 1.f);
          b[19] = -0.6690465435572892f * yz * (7.f * zz - 3.f);
          b[20] = 0.10578554691520431f * (zz * (35.f * zz - 30.f) + 3.f);
          b[21] = -0.6690465435572892f * xz * (7.f * zz - 3.f);
          b[22] = 0.47308734787878004f * (xx - yy) * (7.f * zz - 1.f);
          b[23] = -1.7701307697799304f * xz * (xx - 3.f * yy);
          b[24] = 0.6258357354491761f * (xx * (xx - 3.f * yy) - yy * (3.f * xx - yy));
        }
      }
    }
  }
}

// Philox4x32-10 (Salmon et al., SC'11): the counter-based generator of pob_draw_uniforms and of the SH projection's
// direction draws.
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, ctr.x), lo0 = 0xD2511F53u * ctr.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr.z), lo1 = 0xCD9E8D57u * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += 0x9E3779B9u;
    key.y += 0xBB67AE85u;
  }
  return ctr;
}
// 24 random bits -> [0, 1): never 1, like random.uniform
__device__ __forceinline__ float u01(uint32_t x) { return float(x >> 8) * (1.0f / 16777216.0f); }

}  // namespace pob
