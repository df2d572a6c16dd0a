// Device code shared by the warp-specialised tensor-core kernels of gemm_tc.cu and attn_tc.cu: tile constants, PTX
// wrappers (mbarrier, TMA, descriptors, elect, register budget, warpgroup barrier), one wgmma K step, frag_rows.
#pragma once
#include "kernels.h"
#include <cuda.h>
#include <cuda_fp16.h>
#include "wgmma.cuh"

namespace b200 {

constexpr int BM = 128;          // rows (pixels) per tile: two m64 warpgroup tiles
constexpr int BKE = 32;          // fp32 elements per K step == one 128-byte swizzle row
constexpr int A_STAGE_BYTES = BM * BKE * 4;   // 16 KiB

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
// Barriers and TMA destinations are given as generic pointers or as 32-bit shared-window addresses (smem_u32).
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) { mbar_expect_tx(smem_u32(bar), bytes); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { mbar_arrive(smem_u32(bar)); }
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must surface as a trapped kernel (launch error), never as a hung GPU.  (No printf here:
// a call anywhere in a kernel makes ptxas serialise its wgmma pipeline.)
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 8000000000LL) __trap();   // ~4 s at 2 GHz
  }
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) { mbar_wait(smem_u32(bar), parity); }

__device__ __forceinline__ void tma_load_4d(const CUtensorMap* tm, void* dst, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* tm, uint32_t dst, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* tm, void* dst, uint64_t* bar, int c0, int c1) {
  tma_load_2d(tm, smem_u32(dst), smem_u32(bar), c0, c1);
}

// TMA store of one box from shared memory, tracked by the issuing thread's bulk groups.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tm, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(tm), "r"(src), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// .read: the stores older than the newest N have finished reading shared memory; without: their writes are done too
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// Shared-memory accesses at 32-bit shared-window addresses.
__device__ __forceinline__ float ld_shared_f32(uint32_t a) {
  float v; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory"); return v;
}
__device__ __forceinline__ float2 ld_shared_f32x2(uint32_t a) {
  float2 v; asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a) : "memory"); return v;
}
__device__ __forceinline__ void st_shared_f32(uint32_t a, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); }
__device__ __forceinline__ void st_shared_f32x2(uint32_t a, float x, float y) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ void st_shared_u16(uint32_t a, uint16_t v) { asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "h"(v) : "memory"); }
__device__ __forceinline__ void st_shared_u32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }

__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// K-major, 128-byte-swizzled operand tile (rows of 128 B, 8-row atoms 1024 B apart) as an sm_90 wgmma descriptor:
// start address >> 4, LBO 16 B (unused for swizzled K-major), SBO 1024 B, layout type 1 = SWIZZLE_128B.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

// One 128-byte K step of an m64nN tile: 4 x K=8 (tf32) or 4 x K=16 (f16); either way +32 B per slice (+2 in the
// descriptor's address field).  `it` counts K steps of the tile: the first one overwrites the accumulator.
template <int N, bool F16>
__device__ __forceinline__ void wgmma_kstep(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, int it) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint32_t acc = (it | k) != 0;
    if constexpr (F16) {
      if constexpr (N == 256) wgmma_f16_n256(d, adesc + 2 * k, bdesc + 2 * k, acc);
      else wgmma_f16_n128(d, adesc + 2 * k, bdesc + 2 * k, acc);
    } else {
      if constexpr (N == 256) wgmma_tf32_n256(d, adesc + 2 * k, bdesc + 2 * k, acc);
      else wgmma_tf32_n128(d, adesc + 2 * k, bdesc + 2 * k, acc);
    }
  }
  wgmma_commit();
}

// One lane of a converged warp (elect.sync): the producer runs as a whole warp with warp-uniform loop state and only
// the TMA instructions predicated on this.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}
// Register budget of the warp-specialised kernels (384 threads, one CTA per SM): the producer warpgroup gives its
// registers to the two MMA warpgroups, whose m64n256 fp32 accumulators take 128 registers per thread.
__device__ __forceinline__ void regs_producer() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;"); }
__device__ __forceinline__ void regs_consumer() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;"); }
__device__ __forceinline__ void wg_barrier(int g) { asm volatile("bar.sync %0, 128;" ::"r"(g + 1) : "memory"); }

// Epilogue of one warp's 16 x BN slice of a row-major accumulator (rows = pixels / tokens, columns = output channels),
// straight from the wgmma fragment: lane l holds rows l/4 and l/4 + 8, column pairs 8j + 2(l%4); a quad of lanes writes
// 32 contiguous bytes of a row.  Specialised like the rest of the epilogue code: RES residual add, MODE store format
// (0 fp32, 1 TF32-rounded fp32, 2 fp16), STATS GroupNorm quad sums of the stored values.
//   gm: global row of the slice's first row; rows_valid: rows of the 16 inside the matrix; n0: first column.
// The 16 rows of a slice belong to one image (rows_per_img % 16 == 0 wherever per-image terms are used).
template <int BN, bool RES, int MODE, bool STATS>
__device__ __forceinline__ void frag_rows(const float (&d)[BN / 2], const Epilogue& e, double* qstats, int n_total,
                                          long long gm, int rows_valid, int n0, int lane) {
  const int ra = lane >> 2, rb = ra + 8;
  const bool va = ra < rows_valid, vb = rb < rows_valid;
  const int img = rows_valid > 0 ? (int)gm / e.rows_per_img : 0;   // row counts stay below 2^31
  const float* rv = e.rowvec ? e.rowvec + (long long)img * e.rowvec_ld : nullptr;
  const float scale = e.scale;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = n0 + 8 * j + 2 * (lane & 3);
    float2 ad = make_float2(0.f, 0.f);
    if (e.bias) ad = __ldg(reinterpret_cast<const float2*>(e.bias + col));
    if (rv) { const float2 t = __ldg(reinterpret_cast<const float2*>(rv + col)); ad.x += t.x; ad.y += t.y; }
    float o0 = d[4 * j] + ad.x, o1 = d[4 * j + 1] + ad.y, o2 = d[4 * j + 2] + ad.x, o3 = d[4 * j + 3] + ad.y;
    if (RES) {
      if (va) { const float2 r = __ldg(reinterpret_cast<const float2*>(e.residual + (gm + ra) * e.ld_res + col)); o0 += r.x; o1 += r.y; }
      if (vb) { const float2 r = __ldg(reinterpret_cast<const float2*>(e.residual + (gm + rb) * e.ld_res + col)); o2 += r.x; o3 += r.y; }
    }
    o0 *= scale; o1 *= scale; o2 *= scale; o3 *= scale;
    if (MODE == 1) { o0 = round_tf32(o0); o1 = round_tf32(o1); o2 = round_tf32(o2); o3 = round_tf32(o3); }
    if (MODE == 2) {
      uint16_t* oh = reinterpret_cast<uint16_t*>(e.out);
      if (va) *reinterpret_cast<uint32_t*>(oh + (gm + ra) * e.ld_out + col) = pack_half2(o0, o1);
      if (vb) *reinterpret_cast<uint32_t*>(oh + (gm + rb) * e.ld_out + col) = pack_half2(o2, o3);
    } else {
      if (va) *reinterpret_cast<float2*>(e.out + (gm + ra) * e.ld_out + col) = make_float2(o0, o1);
      if (vb) *reinterpret_cast<float2*>(e.out + (gm + rb) * e.ld_out + col) = make_float2(o2, o3);
    }
    if (STATS) {
      float s = (va ? o0 + o1 : 0.f) + (vb ? o2 + o3 : 0.f);
      float q = (va ? fmaf(o0, o0, o1 * o1) : 0.f) + (vb ? fmaf(o2, o2, o3 * o3) : 0.f);
#pragma unroll
      for (int m = 4; m <= 16; m <<= 1) { s += __shfl_xor_sync(0xffffffffu, s, m); q += __shfl_xor_sync(0xffffffffu, q, m); }
      s += __shfl_xor_sync(0xffffffffu, s, 1); q += __shfl_xor_sync(0xffffffffu, q, 1);
      if ((lane & ~2) == 0 && rows_valid > 0) {   // lanes 0 and 2: the two column quads of this 8-column group
        double* qd = qstats + ((long long)img * (n_total >> 2) + (col >> 2)) * 2;
        atomicAdd(qd, (double)s); atomicAdd(qd + 1, (double)q);
      }
    }
  }
}

}  // namespace b200
