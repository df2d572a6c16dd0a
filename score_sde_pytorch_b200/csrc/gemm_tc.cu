// wgmma / TMA implicit GEMM for the NCSN++ contractions (3x3 and 1x1 convolutions, NIN projections, the attention
// products) on sm_90a.
//
//   out[b][m, n] = epi( sum_{src, tap, c} A_src(b, m, tap, c) * W(b)[tap][n][koff_src + c]
//                       (+ an optional extra 1x1 phase: the fused skip projection) )
//
// Operands are written by their producers in the contraction's format: fp32 bit patterns rounded to the TF32 grid
// (wgmma .tf32, 32 channels per 128-byte K step) or IEEE fp16 (wgmma .f16, 64 channels per K step); either way 11
// significand bits, fp32 accumulation in registers.  Split TF32 (precision 3, "3xTF32") gives every operand a lo twin
// (x = hi + lo, both on the TF32 grid) and walks each K step three times - A lo x W hi, A hi x W lo, A hi x W hi - into
// the same accumulator: only the producer's tensor-map choice and the K count change; ring, barriers and epilogue do not.
//
// Kernels (persistent, warp-specialised, 384 threads):
//   gemm_tc_kernel<BN>   one CTA per tile: 128 rows x BN columns, or - `swap` - 128 output channels x 256 pixels
//                        (D^T = W X^T) for 128-channel convolutions, 1x1 convolutions, the network head and the 3x3
//                        'same' convolutions on 16- / 32-pixel rows (any output width: one tile per 128-channel slice);
//   attn_tc_kernel<F16>  attn_tc.cuh: QK^T, softmax, PV, NIN_3 + residual in one kernel.
// Roles: warp 0 TMA producer (4-D box of the NHWC tensor shifted by the filter tap - or, in the halo form, three
// W-shifted copies of the tile with its halo per channel chunk - zero halo and tail rows from out-of-bounds fill,
// SWIZZLE_128B, ring with full/empty mbarriers), running as a whole warp with warp-uniform loop state and the TMA
// instructions predicated on one elect.sync lane; warps 1..3 idle (their registers go to the MMA warpgroups);
// warps 4..11 two MMA warpgroups, each issuing m64 x BN wgmma over its 64 rows of the tile and then storing its
// accumulator fragment through an epilogue compiled per (residual, store format, stats) combination - `frag_rows`
// (row-major outputs) or `frag_swap` (swapped tiles) - with bias, time-embedding row, residual, scale,
// fp32 / TF32 / fp16 store and the GroupNorm quad sums fused.
#include "kernels.h"
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_fp16.h>
#include "wgmma.cuh"
#include <mutex>
#include <cstdlib>
#include <cstring>

namespace b200 {

namespace {

constexpr int BM = 128;          // rows (pixels) per tile: two m64 warpgroup tiles
constexpr int BKE = 32;          // fp32 elements per K step == one 128-byte swizzle row
constexpr int A_STAGE_BYTES = BM * BKE * 4;   // 16 KiB

// Halo form of the 3x3 mainloop.  The nine filter taps of one channel chunk read three W-shifted
// copies of the tile *with its one-row halo* (TMA box [chunk, W, rows + 2], origin w = -1 / 0 / +1, zero fill outside the
// image); the operand of tap (dh, dw) is copy[dw] starting (dh + 1) * W pixels in - a multiple of 1024 bytes, so a plain
// swizzled descriptor.  L2 -> shared-memory traffic per chunk: 3 x (rows + 2) / rows tiles instead of 9.
constexpr int HALO_XS = 4;                  // halo copies in flight
constexpr int HALO_X_BYTES = 40 * 1024;     // swapped form: (8 + 2) rows x 32 pixels x 128 B
constexpr int HALO_WS = 4;                  //   its weight-slice ring: 4 x 16 KB   (4 x 40 + 4 x 16 = 224 KB)

struct TcParams {
  CUtensorMap tmA1, tmA2, tmW;
  CUtensorMap tmA3, tmA4, tmW2;            // optional extra 1x1 K phase (fused skip projection): out += [A3|A4] W2^T
  CUtensorMap tmH1, tmH2;                  // halo form: box = [bke channels, W, tile rows + 2, 1] of the two filter sources
  // split TF32: the same maps over the lo twins of every operand (copies of the hi maps otherwise)
  CUtensorMap tmA1l, tmA2l, tmWl, tmA3l, tmA4l, tmW2l, tmH1l, tmH2l;
  int nphase;                              // 3: split TF32, every K step loads (A lo, W hi), (A hi, W lo), (A hi, W hi); else 1
  int halo;                               // 1: 3x3 taps read W-shifted halo copies of the tile (3 loads per channel chunk instead of 9)
  int halo_dh_bytes;                       // W * 128: bytes between the operand windows of consecutive filter rows inside a copy
  int halo_copy_bytes;                     // (tile rows + 2) * W * 128: bytes of one halo copy
  int chunk_major;                         // nine-load loop walks K as (chunk, filter column, filter row): shapes with a halo form
  int conv, H, W, taps, pad, S, stride;   // H, W: OUTPUT spatial size; S = filter width (3 or 1)
  int kchunks1, kchunks2, C1;
  int kchunks3, kchunks4, C3;              // extra phase: channel chunks of its (two-source) input
  int N_total, tiles_n;
  int nbatch, tiles_m_per_batch, M_per_batch;
  int a_batch_rows, w_batch_rows;
  int f16;                                 // 1: A and W are fp16 (wgmma .f16, 64-channel K steps); 0: TF32-grid fp32 (32-channel K steps)
  int bke;                                 // channels per K step: one 128-byte swizzle row = 32 fp32 or 64 fp16
  int swap;                                // 1: operands swapped (D^T = W X^T): 128 output channels x 256 pixels per tile
  double* qstats;                          // optional [img][N_total/4][2] GroupNorm quad sums (sum, sum of squares)
  long long total_tiles;
  Epilogue epi;
};

// ---------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must surface as a trapped kernel (launch error), never as a hung GPU.  (No printf here:
// a call anywhere in a kernel makes ptxas serialise its wgmma pipeline.)
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 8000000000LL) __trap();   // ~4 s at 2 GHz
  }
}

__device__ __forceinline__ void tma_load_4d(const CUtensorMap* tm, void* dst, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* tm, void* dst, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}

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

template <int BN>
struct SmemLayout {
  static constexpr int STAGES = BN == 256 ? 4 : 6;
  static constexpr int B_STAGE_BYTES = BN * BKE * 4;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  static constexpr int HALO_BYTES = HALO_XS * HALO_X_BYTES + HALO_WS * A_STAGE_BYTES;   // the swapped halo form's two rings
  static constexpr int BAR_OFFSET = BN == 256 && HALO_BYTES > RING_BYTES ? HALO_BYTES : RING_BYTES;
  static constexpr int TOTAL = BAR_OFFSET + 256 + 1024;   // barriers + slack for 1024-B alignment
  static_assert(TOTAL <= 232448, "exceeds the 227 KB shared-memory limit of sm_90");
  static_assert(BN != 256 || STAGES >= HALO_XS, "the halo copies use the first HALO_XS stage barriers");
};

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
template <int BN>
__device__ __forceinline__ void frag_rows_dispatch(const float (&d)[BN / 2], const Epilogue& e, double* qstats, int n_total,
                                                   long long gm, int rows_valid, int n0, int lane) {
  const int mode = e.round_tf32;
  const bool has_res = e.residual != nullptr, stats = qstats != nullptr;
#define B200_ROWF(R, M) do { if (stats) frag_rows<BN, R, M, true>(d, e, qstats, n_total, gm, rows_valid, n0, lane); \
                             else frag_rows<BN, R, M, false>(d, e, qstats, n_total, gm, rows_valid, n0, lane); } while (0)
  if (has_res) { if (mode == 0) B200_ROWF(true, 0); else if (mode == 1) B200_ROWF(true, 1); else B200_ROWF(true, 2); }
  else { if (mode == 0) B200_ROWF(false, 0); else if (mode == 1) B200_ROWF(false, 1); else B200_ROWF(false, 2); }
#undef B200_ROWF
}

// Epilogue of one warp's 16-channel x 256-pixel slice of a swapped tile (D^T = W X^T: rows = output channels, columns =
// pixels of ONE image).  Lane l holds channels c0 + l/4 and c0 + l/4 + 8 of pixel pairs 8j + 2(l%4); eight lanes cover 32
// contiguous bytes of a pixel's channel vector.
template <bool RES, int MODE, bool STATS>
__device__ __forceinline__ void frag_swap(const float (&d)[128], const Epilogue& e, double* qstats, int n_total,
                                          int c0, long long pix0, int img, int lane) {
  const int ca = c0 + (lane >> 2), cb = ca + 8;
  const float adda = (e.bias ? __ldg(e.bias + ca) : 0.f) + (e.rowvec ? __ldg(e.rowvec + img * e.rowvec_ld + ca) : 0.f);
  const float addb = (e.bias ? __ldg(e.bias + cb) : 0.f) + (e.rowvec ? __ldg(e.rowvec + img * e.rowvec_ld + cb) : 0.f);
  const float scale = e.scale;
  float sa = 0.f, qa = 0.f, sb = 0.f, qb = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const long long px = pix0 + 8 * j + 2 * (lane & 3);
    float o[4] = {d[4 * j] + adda, d[4 * j + 1] + adda, d[4 * j + 2] + addb, d[4 * j + 3] + addb};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const long long pix = px + (i & 1);
      const int ch = i < 2 ? ca : cb;
      if (RES) o[i] += __ldg(e.residual + pix * e.ld_res + ch);
      o[i] *= scale;
      if (MODE == 1) o[i] = round_tf32(o[i]);
      if (MODE == 2) {
        uint16_t h;
        asm("cvt.rn.f16.f32 %0, %1;" : "=h"(h) : "f"(o[i]));
        reinterpret_cast<uint16_t*>(e.out)[pix * e.ld_out + ch] = h;
      } else e.out[pix * e.ld_out + ch] = o[i];
    }
    if (STATS) {
      sa += o[0] + o[1]; qa = fmaf(o[0], o[0], fmaf(o[1], o[1], qa));
      sb += o[2] + o[3]; qb = fmaf(o[2], o[2], fmaf(o[3], o[3], qb));
    }
  }
  if (STATS) {
#pragma unroll
    for (int m = 1; m <= 8; m <<= 1) {   // pixel lanes (1, 2), then the four channels of a quad (4, 8)
      sa += __shfl_xor_sync(0xffffffffu, sa, m); qa += __shfl_xor_sync(0xffffffffu, qa, m);
      sb += __shfl_xor_sync(0xffffffffu, sb, m); qb += __shfl_xor_sync(0xffffffffu, qb, m);
    }
    if ((lane & 15) == 0) {
      double* qd = qstats + ((long long)img * (n_total >> 2) + (ca >> 2)) * 2;
      atomicAdd(qd, (double)sa); atomicAdd(qd + 1, (double)qa);
      qd = qstats + ((long long)img * (n_total >> 2) + (cb >> 2)) * 2;
      atomicAdd(qd, (double)sb); atomicAdd(qd + 1, (double)qb);
    }
  }
}

// ---------------------------------------------------------------------------
// Kernel
// ---------------------------------------------------------------------------
// Consumer side of gemm_tc_kernel: one MMA warpgroup (g = 0, 1) owns accumulator rows 64g .. 64g + 63 of every tile.
// A K step is released to the producer once the wgmma after it has been issued (wait_group 1), so the tensor core
// always has the next step queued while the previous one's slot is handed back.
template <int BN, bool F16>
__device__ __forceinline__ void gemm_tc_consumer(const TcParams& p, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                                 uint64_t* wfull_bar, uint64_t* wempty_bar, int g, int wq, int lane) {
  using L = SmemLayout<BN>;
  const int kiters = ((p.kchunks1 + p.kchunks2) * p.taps + p.kchunks3 + p.kchunks4) * p.nphase;
  const Epilogue& e = p.epi;
  uint32_t stage = 0, phase = 0, ws = 0, wphase = 0;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    float acc[BN / 2];
    if (BN == 256 && p.halo) {
      // halo form: A = the 16 KB weight slice (128 output channels), B = 256 pixel rows of a halo copy starting one filter
      // row (W pixels) further in per dh; the slice's slot is released per tap, the copy's after its three taps
      const uint32_t wring = smem_u32(smem + HALO_XS * HALO_X_BYTES);
      int it = 0, pend_ws = -1, pend_x = -1;
      for (int src = 0; src < 4; ++src) {
        const int nch = src == 0 ? p.kchunks1 : src == 1 ? p.kchunks2 : src == 2 ? p.kchunks3 : p.kchunks4;
        const int ncopies = (src < 2 ? 3 * nch : nch) * p.nphase, ntap = src < 2 ? 3 : 1;
        for (int c = 0; c < ncopies; ++c) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t sx = smem_u32(smem + stage * HALO_X_BYTES);
          for (int dhi = 0; dhi < ntap; ++dhi, ++it) {
            mbar_wait(&wfull_bar[ws], wphase);
            const uint64_t adesc = make_smem_desc(wring + ws * A_STAGE_BYTES + g * (A_STAGE_BYTES / 2));
            const uint64_t bdesc = make_smem_desc(sx + (src < 2 ? dhi * p.halo_dh_bytes : 0));
            wgmma_kstep<BN, F16>(acc, adesc, bdesc, it);
            wgmma_wait<1>();
            if (lane == 0) {
              if (pend_ws >= 0) mbar_arrive(&wempty_bar[pend_ws]);
              if (pend_x >= 0) mbar_arrive(&empty_bar[pend_x]);
            }
            pend_ws = (int)ws; pend_x = dhi == ntap - 1 ? (int)stage : -1;
            if (++ws == HALO_WS) { ws = 0; wphase ^= 1; }
          }
          if (++stage == HALO_XS) { stage = 0; phase ^= 1; }
        }
      }
      wgmma_wait<0>();
      if (lane == 0) {
        if (pend_ws >= 0) mbar_arrive(&wempty_bar[pend_ws]);
        if (pend_x >= 0) mbar_arrive(&empty_bar[pend_x]);
      }
    } else {
      int pend = -1;
      for (int it = 0; it < kiters; ++it) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * L::STAGE_BYTES);
        wgmma_kstep<BN, F16>(acc, make_smem_desc(sa + g * (A_STAGE_BYTES / 2)), make_smem_desc(sa + A_STAGE_BYTES), it);
        wgmma_wait<1>();
        if (lane == 0 && pend >= 0) mbar_arrive(&empty_bar[pend]);
        pend = (int)stage;
        if (++stage == L::STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (lane == 0 && pend >= 0) mbar_arrive(&empty_bar[pend]);
    }

    // ---- epilogue: this warp's 16 accumulator rows ----
    const int rw = g * 64 + wq * 16;                       // first tile row of this warp
    if constexpr (BN == 256) {
      if (p.swap) {
        // swapped operands (128-channel layers, 1x1 convolutions, the head): rows = output channels, columns = 256 pixels
        const int c0 = (int)(tile % p.tiles_n) * 128 + rw;
        const int pix0 = (tile / p.tiles_n) * 256;
        const int img = pix0 / e.rows_per_img;     // rows_per_img % 256 == 0: one image per tile
        if (e.out_nchw) {
          // Network head (ncsnpp.py:374-380): the 128-row weight tile is zero-padded above the n_valid image channels;
          // (acc + bias) / sigma[img] is written as NCHW
          const float dv = e.per_img_div ? __ldg(e.per_img_div + img * e.div_stride) : 1.f;
          const int hw = e.rows_per_img, pix_in_img = (int)(pix0 - (long long)img * hw);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int co = c0 + (lane >> 2) + 8 * h;
            if (co < e.n_valid) {
              const float add = e.bias ? __ldg(e.bias + co) : 0.f;
              float* dst = e.out + ((long long)img * e.n_valid + co) * hw + pix_in_img + 2 * (lane & 3);
#pragma unroll
              for (int j = 0; j < 32; ++j)
                *reinterpret_cast<float2*>(dst + 8 * j) = make_float2((acc[4 * j + 2 * h] + add) / dv, (acc[4 * j + 2 * h + 1] + add) / dv);
            }
          }
        } else {
          const int mode = e.round_tf32;
          const bool has_res = e.residual != nullptr, stats = p.qstats != nullptr;
#define B200_SWAPF(R, M) do { if (stats) frag_swap<R, M, true>(acc, e, p.qstats, p.N_total, c0, pix0, img, lane); \
                              else frag_swap<R, M, false>(acc, e, p.qstats, p.N_total, c0, pix0, img, lane); } while (0)
          if (has_res) { if (mode == 0) B200_SWAPF(true, 0); else if (mode == 1) B200_SWAPF(true, 1); else B200_SWAPF(true, 2); }
          else { if (mode == 0) B200_SWAPF(false, 0); else if (mode == 1) B200_SWAPF(false, 1); else B200_SWAPF(false, 2); }
#undef B200_SWAPF
        }
        continue;
      }
    }
    const int nt = (int)(tile % p.tiles_n);
    const int mg = tile / p.tiles_n;
    const int b = (int)(mg / p.tiles_m_per_batch);
    const int mt = (int)(mg % p.tiles_m_per_batch);
    const int row0 = mt * BM + rw;
    const int rows_valid = min(16, max(0, p.M_per_batch - row0));
    frag_rows_dispatch<BN>(acc, e, p.qstats, p.N_total, (long long)b * p.M_per_batch + row0, rows_valid, nt * BN, lane);
  }
}

template <int BN>
__global__ void __launch_bounds__(384, 1) gemm_tc_kernel(const __grid_constant__ TcParams p) {
  using L = SmemLayout<BN>;
  constexpr int STAGES = L::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* wfull_bar = empty_bar + STAGES;      // halo form: the weight-slice ring has its own barriers
  uint64_t* wempty_bar = wfull_bar + HALO_WS;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp index provably warp-uniform

  if (threadIdx.x == 0) {
    // empty slots: one arrival per MMA warp (8)
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
    for (int s = 0; s < HALO_WS; ++s) { mbar_init(&wfull_bar[s], 1); mbar_init(&wempty_bar[s], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  pdl_wait(); pdl_trigger();   // barriers are set up; nothing above touched global memory (common.cuh)

  const int HW = p.H * p.W;
  const int bke = p.bke;

  if (warp < 4) {
    regs_producer();
    if (warp != 0) return;
    // ======================= TMA producer (whole warp; one elected lane issues, see elect_one) =======================
    const bool issue = elect_one();
    const int alo_ph = p.nphase == 3 ? 0 : -1;   // split TF32: the product phase that reads the pixel / row operand's lo twin
    uint32_t stage = 0, phase = 0;
    if (BN == 256 && p.halo) {
      // halo form (swapped operands, one image per 256-pixel tile, W <= 32): per channel chunk three halo copies, each
      // followed by the three 16 KB weight slices of its filter column
      uint32_t ws = 0, wphase = 0;
      uint8_t* const wring = smem + HALO_XS * HALO_X_BYTES;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int nt = (int)(tile % p.tiles_n);
        const int p0 = (tile / p.tiles_n) * 256;
        const int img0 = (int)(p0 / HW), h0 = (int)(p0 % HW) / p.W;
        const int wrow0 = nt * 128;
        for (int src = 0; src < 4; ++src) {
          const int nch = src == 0 ? p.kchunks1 : src == 1 ? p.kchunks2 : src == 2 ? p.kchunks3 : p.kchunks4;
          if (nch == 0) continue;
          const int wcol0 = src == 1 ? p.C1 : src == 3 ? p.C3 : 0;
          for (int kc = 0; kc < nch; ++kc) {
            if (src < 2) {
              for (int dwi = 0; dwi < 3; ++dwi) {
                // split TF32: the copy + its three weight slices once per product (pixels lo / hi / hi, weights hi / lo / hi)
                for (int ph = 0; ph < p.nphase; ++ph) {
                  const CUtensorMap* tmH = ph == alo_ph ? (src == 0 ? &p.tmH1l : &p.tmH2l) : (src == 0 ? &p.tmH1 : &p.tmH2);
                  const CUtensorMap* tmW = ph == 1 ? &p.tmWl : &p.tmW;
                  mbar_wait(&empty_bar[stage], phase ^ 1);
                  if (issue) {
                    mbar_expect_tx(&full_bar[stage], (uint32_t)p.halo_copy_bytes);
                    tma_load_4d(tmH, smem + stage * HALO_X_BYTES, &full_bar[stage], kc * bke, dwi - 1, h0 - 1, img0);
                  }
                  if (++stage == HALO_XS) { stage = 0; phase ^= 1; }
                  for (int dhi = 0; dhi < 3; ++dhi) {
                    mbar_wait(&wempty_bar[ws], wphase ^ 1);
                    if (issue) {
                      mbar_expect_tx(&wfull_bar[ws], A_STAGE_BYTES);
                      tma_load_2d(tmW, wring + ws * A_STAGE_BYTES, &wfull_bar[ws], wcol0 + kc * bke, wrow0 + (dhi * 3 + dwi) * p.N_total);
                    }
                    if (++ws == HALO_WS) { ws = 0; wphase ^= 1; }
                  }
                }
              }
            } else {
              // extra 1x1 phase (fused skip projection): the plain 256-pixel tile as two 128-pixel boxes, its own weights
              const int h1 = h0 + 128 / p.W;
              for (int ph = 0; ph < p.nphase; ++ph) {
                const CUtensorMap* tmA = ph == alo_ph ? (src == 2 ? &p.tmA3l : &p.tmA4l) : (src == 2 ? &p.tmA3 : &p.tmA4);
                mbar_wait(&empty_bar[stage], phase ^ 1);
                if (issue) {
                  mbar_expect_tx(&full_bar[stage], 2 * A_STAGE_BYTES);
                  tma_load_4d(tmA, smem + stage * HALO_X_BYTES, &full_bar[stage], kc * bke, 0, h0, img0);
                  tma_load_4d(tmA, smem + stage * HALO_X_BYTES + A_STAGE_BYTES, &full_bar[stage], kc * bke, 0, h1, img0);
                }
                if (++stage == HALO_XS) { stage = 0; phase ^= 1; }
                mbar_wait(&wempty_bar[ws], wphase ^ 1);
                if (issue) {
                  mbar_expect_tx(&wfull_bar[ws], A_STAGE_BYTES);
                  tma_load_2d(ph == 1 ? &p.tmW2l : &p.tmW2, wring + ws * A_STAGE_BYTES, &wfull_bar[ws], wcol0 + kc * bke, wrow0);
                }
                if (++ws == HALO_WS) { ws = 0; wphase ^= 1; }
              }
            }
          }
        }
      }
    } else
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const int nt = (int)(tile % p.tiles_n);
      const int mg = tile / p.tiles_n;
      const int b = (int)(mg / p.tiles_m_per_batch);
      const int mt = (int)(mg % p.tiles_m_per_batch);
      int img0 = 0, h0 = 0, w0 = 0;
      if (p.conv) {
        const int p0 = (long long)mt * BM;
        img0 = (int)(p0 / HW);
        const int rem = (int)(p0 % HW);
        h0 = rem / p.W; w0 = rem % p.W;
      }
      const int arow0 = b * p.a_batch_rows + mt * BM;
      const int wrow0 = b * p.w_batch_rows + nt * (p.swap ? 128 : BN);
      int img1 = 0, h1 = 0, w1 = 0;                     // swap mode: second 128-pixel box of the 256-pixel tile
      if (p.swap) {
        const int p0 = (long long)mt * 256;
        img0 = (int)(p0 / HW); h0 = (int)(p0 % HW) / p.W; w0 = (int)(p0 % HW) % p.W;
        const int p1 = p0 + 128;
        img1 = (int)(p1 / HW); h1 = (int)(p1 % HW) / p.W; w1 = (int)(p1 % HW) % p.W;
      }
      // sources 0,1: the (two-source) filter input, all taps; sources 2,3: the extra 1x1 phase (centre tap, own weights)
      for (int src = 0; src < 4; ++src) {
        const int nch = src == 0 ? p.kchunks1 : src == 1 ? p.kchunks2 : src == 2 ? p.kchunks3 : p.kchunks4;
        if (nch == 0) continue;
        const CUtensorMap* tmAh = src == 0 ? &p.tmA1 : src == 1 ? &p.tmA2 : src == 2 ? &p.tmA3 : &p.tmA4;
        const CUtensorMap* tmWh = src < 2 ? &p.tmW : &p.tmW2;
        const CUtensorMap* tmAl = src == 0 ? &p.tmA1l : src == 1 ? &p.tmA2l : src == 2 ? &p.tmA3l : &p.tmA4l;
        const CUtensorMap* tmWl = src < 2 ? &p.tmWl : &p.tmW2l;
        const int wcol0 = src == 1 ? p.C1 : src == 3 ? p.C3 : 0;
        const int ntaps = src < 2 ? p.taps : 1;
        // K order.  Default: filter tap, then channel chunk - consecutive loads sweep the channel vector of the same shifted
        // pixels (contiguous 128-byte segments of every pixel row).  Shapes that have a halo form (p.chunk_major) walk K the way that form must -
        // channel chunk, filter column, filter row - so that halo on / off and row-major launches of such shapes add
        // the same products in the same order.
        const int nouter = p.chunk_major ? nch : ntaps, ninner = p.chunk_major ? ntaps : nch;
        for (int o = 0; o < nouter; ++o) {
          for (int i = 0; i < ninner; ++i) {
            const int kc = p.chunk_major ? o : i, t = p.chunk_major ? i : o;
            const int tap = (ntaps == 1 || !p.chunk_major) ? t : (t % p.S) * p.S + t / p.S;
            const int dh = src < 2 ? tap / p.S - p.pad : 0, dw = src < 2 ? tap % p.S - p.pad : 0;
            for (int ph = 0; ph < p.nphase; ++ph) {   // split TF32: (A lo, W hi), (A hi, W lo), (A hi, W hi)
              const CUtensorMap* tmA = ph == alo_ph ? tmAl : tmAh;
              const CUtensorMap* tmW = ph == 1 ? tmWl : tmWh;
              mbar_wait(&empty_bar[stage], phase ^ 1);
              uint8_t* sa = smem + stage * L::STAGE_BYTES;
              uint8_t* sb = sa + A_STAGE_BYTES;
              if (issue) {
                mbar_expect_tx(&full_bar[stage], L::STAGE_BYTES);
                if (p.swap) {
                  // first 16 KiB: 128 output channels x 32 k of W (MMA A); next 32 KiB: 256 pixels x 32 k (MMA B)
                  tma_load_2d(tmW, sa, &full_bar[stage], wcol0 + kc * bke, wrow0 + tap * p.N_total);
                  tma_load_4d(tmA, sb, &full_bar[stage], kc * bke, w0 + dw, h0 + dh, img0);
                  tma_load_4d(tmA, sb + A_STAGE_BYTES, &full_bar[stage], kc * bke, w1 + dw, h1 + dh, img1);
                } else {
                  if (p.conv) tma_load_4d(tmA, sa, &full_bar[stage], kc * bke, w0 * p.stride + dw, h0 * p.stride + dh, img0);
                  else tma_load_4d(tmA, sa, &full_bar[stage], kc * bke, arow0, 0, 0);
                  tma_load_2d(tmW, sb, &full_bar[stage], wcol0 + kc * bke, wrow0 + tap * p.N_total);
                }
              }
              if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
          }
        }
      }
    }
  } else {
    regs_consumer();
    const int g = (warp >> 2) - 1, wq = warp & 3;   // MMA warpgroup and warp within it
    if (p.f16) gemm_tc_consumer<BN, true>(p, smem, full_bar, empty_bar, wfull_bar, wempty_bar, g, wq, lane);
    else gemm_tc_consumer<BN, false>(p, smem, full_bar, empty_bar, wfull_bar, wempty_bar, g, wq, lane);
  }
}

#include "attn_tc.cuh"

// ---------------------------------------------------------------------------
// Host side: tensor maps, plan, launch
// ---------------------------------------------------------------------------
PFN_cuTensorMapEncodeTiled_v12000 get_encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qr) == cudaSuccess &&
        qr == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(f);
  });
  return fn;
}

int encode_map(CUtensorMap* tm, const float* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
               const uint32_t* box, const uint32_t* elem_strides = nullptr, bool f16 = false) {
  auto fn = get_encode_fn();
  B200_REQUIRE(fn != nullptr, "gemm_tc: cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "gemm_tc: operand base %p not 16-byte aligned", (const void*)base);
  uint32_t estr[5] = {1, 1, 1, 1, 1};
  if (elem_strides) for (int i = 0; i < rank; ++i) estr[i] = elem_strides[i];
  CUresult r = fn(tm, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<float*>(base), dims,
                  strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B200_REQUIRE(r == CUDA_SUCCESS, "gemm_tc: cuTensorMapEncodeTiled failed with CUresult %d "
               "(rank %d dims %llu,%llu,%llu,%llu box %u,%u,%u,%u)", (int)r, rank,
               (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)(rank > 2 ? dims[2] : 0),
               (unsigned long long)(rank > 3 ? dims[3] : 0), box[0], box[1], rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
  return 0;
}

int num_sms() {
  static int n = 0;
  if (!n) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); if (n <= 0) n = 132; }
  return n;
}

}  // namespace

struct TcGemmPlan {
  TcParams prm;
  int bn;
};

static int tc_configure();

bool tc_gemm_supported(const TcGemmDesc& d, const char** why) {
  static const char* w;
  auto fail = [&](const char* m) { w = m; if (why) *why = w; return false; };
  const int bke = d.f16 ? 64 : BKE;
  if (d.C1 % bke || d.C2 % bke || d.C1 <= 0) return fail("channel counts must be multiples of 32 (tf32) / 64 (f16)");
  if (d.N_total % 128) return fail("N must be a multiple of 128");
  if (d.taps != 1 && d.taps != 9) return fail("only 1x1 and 3x3 filters");
  if (d.conv) {
    if (d.nbatch != 1) return fail("conv mode is unbatched");
    if (d.stride > 2) return fail("stride must be 1 or 2");
    if (d.stride == 2 && d.a2) return fail("strided conv is single-source");
    const int HW = d.H * d.W;
    if (HW >= BM) {
      if (d.W >= BM) { if (d.W % BM) return fail("image width does not tile 128 pixels"); }
      else if ((BM % d.W) || (d.H % (BM / d.W))) return fail("image rows do not tile 128 pixels");
    } else if (BM % HW) return fail("image size does not divide 128 pixels");
  } else {
    if (d.nbatch > 1 && (d.M_per_batch % BM)) return fail("batched gemm needs M_per_batch % 128 == 0");
    if (d.a_ld % (d.f16 ? 8 : 4)) return fail("A row pitch must be a multiple of 16 bytes");
  }
  if (d.a3) {
    if (!d.conv || d.stride == 2 || !d.w2) return fail("extra 1x1 phase needs a stride-1 convolution and its weights");
    if (d.C3 % bke || d.C3 <= 0 || (d.a4 && d.C4 % bke)) return fail("extra-phase channel counts must be multiples of 32 (tf32) / 64 (f16)");
  }
  if (d.epi.out_nchw) {   // network head: zero-padded 128-row weight tile, swapped form, NCHW store of the real channels
    if (!(d.conv && d.N_total == 128 && d.epi.n_valid > 0 && d.epi.n_valid <= 32 && (d.H * d.W) % 256 == 0 && (d.W <= BM || d.W % BM == 0) && d.stride != 2 &&
          !d.qstats && !d.epi.residual && !d.epi.rowvec && d.epi.round_tf32 == 0))
      return fail("NCHW head needs a 128-row padded weight tile, HW % 256 == 0 and a plain epilogue");
  } else if (d.epi.per_img_div) return fail("per-image divisor only with the NCHW head epilogue");
  // a 32-row epilogue block spans two images only for 4x4 images (rows_per_img == 16)
  if ((d.qstats || d.epi.rowvec) && !(d.epi.rows_per_img % 32 == 0 || d.epi.rows_per_img == 16)) return fail("per-image epilogue terms need rows_per_img % 32 == 0 or == 16");
  if (d.epi.ld_out % 4 || (d.epi.residual && d.epi.ld_res % 4)) return fail("output pitch must be a multiple of 4 elements");
  if (d.epi.round_tf32 == 2 && d.epi.ld_out % 8) return fail("fp16 output pitch must be a multiple of 8 elements");
  if (d.split && d.f16) return fail("split TF32 takes TF32 operands, not fp16");
  if (d.split && (!d.a1_lo || (d.a2 && !d.a2_lo) || (d.a3 && !d.a3_lo) || (d.a4 && !d.a4_lo) || !d.w_lo || (d.a3 && !d.w2_lo)))
    return fail("split TF32 needs the lo twin of every operand");
  return true;
}

int tc_gemm_plan_create(const TcGemmDesc& d, TcGemmPlan** out) {
  const char* why = nullptr;
  B200_REQUIRE(tc_gemm_supported(d, &why), "gemm_tc: unsupported shape: %s", why ? why : "?");
  if (int r = tc_configure()) return r;
  TcGemmPlan* pl = new TcGemmPlan();
  TcParams& p = pl->prm;
  memset(&p, 0, sizeof(p));
  pl->bn = (d.N_total % 256 == 0) ? 256 : 128;
  p.conv = d.conv; p.H = d.conv ? d.H : 1; p.W = d.conv ? d.W : 1; p.taps = d.taps;
  p.S = d.taps == 9 ? 3 : 1; p.pad = (d.taps == 9 && !d.valid_pad) ? 1 : 0;
  p.stride = d.stride == 2 ? 2 : 1;
  p.f16 = d.f16 ? 1 : 0;
  p.nphase = d.split ? 3 : 1;

  const bool f16 = d.f16 != 0;
  // every map is encoded over the hi operand and, in split-TF32 plans, once more over its lo twin
  auto encode_pair = [&](CUtensorMap* tm, CUtensorMap* tml, const float* base, const float* lo, int rank, const uint64_t* dims,
                         const uint64_t* str, const uint32_t* box, const uint32_t* estr) {
    if (int r = encode_map(tm, base, rank, dims, str, box, estr, f16)) return r;
    if (!d.split) { *tml = *tm; return 0; }
    return encode_map(tml, lo, rank, dims, str, box, estr, f16);
  };
  const int bke = f16 ? 64 : BKE;            // elements per 128-byte K step
  const uint64_t es = f16 ? 2 : 4;           // operand element size
  p.bke = bke;
  {
    // Form selection:
    //  * swapped operands (D^T = W X^T: 128 output channels x 256 pixels per tile) for 128-channel outputs, whose
    //    M=128,N=128 MMAs are issue-bound, and for 1x1 convolutions (output-bound launches: the swapped form's
    //    epilogue writes whole channel vectors of a pixel); the NCHW head exists only in this form;
    //  * 3x3 'same' filters on 16- / 32-pixel rows with more output channels take the swapped form too, as tiles_n
    //    128-channel halves of each 256-pixel tile: it has the halo form (about 29 KB brought into shared memory per
    //    K step of a 128 x 256 tile instead of 48 KB).  It has as many tiles as the row-major plan, except below ~34
    //    images at 16x16 (~9 at 32x32), where the row-major plan would split into 128-column tiles; those small launches
    //    stay swapped all the same, because a swapped tile's wgmma sums are not bitwise those of a row-major tile, and
    //    every batch size should compute each output as the large-batch plan does;
    //  * launches too small to give every SM a 256-column tile are cut into 128-column tiles: twice the CTAs at work.
    const long long Mtot = (long long)d.nimg * d.H * d.W;
    // (image rows wider than 128 pixels - the 256..1024-pixel families - are cut into 128-pixel boxes like any other: the
    // two boxes of a 256-pixel tile are then two halves of one row or of consecutive rows)
    const bool halo_geom = d.taps == 9 && p.pad == 1 && (d.W == 16 || d.W == 32) && (d.Hin == 0 || d.Hin == d.H) &&
                           (d.Win == 0 || d.Win == d.W);
    const bool can_swap = d.conv && p.stride == 1 && (d.N_total % 256 != 0 || d.taps == 1 || halo_geom) && (d.H * d.W) % 256 == 0 &&
                          (d.W <= BM || d.W % BM == 0) && Mtot % 256 == 0 && d.epi.rows_per_img % 256 == 0;
    p.swap = can_swap ? 1 : 0;
    if (d.epi.out_nchw && !p.swap) { delete pl; B200_REQUIRE(false, "gemm_tc: the NCHW head needs the swapped-operand form"); }
    if (p.swap) pl->bn = 256;
    p.qstats = d.qstats;
    const int tmb = d.conv ? 1 : (d.M_per_batch + BM - 1) / BM;
    const long long m_tiles = d.conv ? (Mtot + BM - 1) / BM : (long long)d.nbatch * tmb;
    const long long n_tiles = d.N_total % 256 == 0 ? d.N_total / 256 : d.N_total / 128;
    if (!p.swap && pl->bn == 256 && m_tiles * n_tiles <= num_sms() / 2) pl->bn = 128;
  }
  p.kchunks1 = d.C1 / bke; p.kchunks2 = d.a2 ? d.C2 / bke : 0; p.C1 = d.C1;
  p.N_total = d.N_total; p.tiles_n = p.swap ? d.N_total / 128 : d.N_total / pl->bn;
  p.a_batch_rows = d.a_batch_rows; p.w_batch_rows = d.w_batch_rows;
  p.epi = d.epi;

  int rc = 0;
  if (d.conv) {
    const int HW = d.H * d.W;
    const long long M = (long long)d.nimg * HW;
    p.nbatch = 1; p.M_per_batch = (int)M; p.tiles_m_per_batch = p.swap ? (int)(M / 256) : (int)((M + BM - 1) / BM);
    uint32_t box[4];
    if (HW >= BM) { box[1] = std::min(d.W, BM); box[2] = BM / box[1]; box[3] = 1; }
    else { box[1] = d.W; box[2] = d.H; box[3] = BM / HW; }
    box[0] = (uint32_t)bke;
    // stride 2: the box *traverses* 2x as many pixels and TMA keeps every other one
    const uint32_t estr[4] = {1, (uint32_t)p.stride, (uint32_t)p.stride, 1};
    box[1] *= p.stride; box[2] *= p.stride;
    const int Hin = d.Hin ? d.Hin : d.H, Win = d.Win ? d.Win : d.W;
    for (int s = 0; s < 2; ++s) {
      const float* base = s ? d.a2 : d.a1;
      const int C = s ? d.C2 : d.C1;
      if (!base) continue;
      uint64_t dims[4] = {(uint64_t)C, (uint64_t)Win, (uint64_t)Hin, (uint64_t)d.nimg};
      uint64_t str[3] = {(uint64_t)C * es, (uint64_t)Win * C * es, (uint64_t)Hin * Win * C * es};
      rc = encode_pair(s ? &p.tmA2 : &p.tmA1, s ? &p.tmA2l : &p.tmA1l, base, s ? d.a2_lo : d.a1_lo, 4, dims, str, box, estr);
      if (rc) { delete pl; return rc; }
    }
  } else {
    p.nbatch = d.nbatch; p.M_per_batch = d.M_per_batch; p.tiles_m_per_batch = (d.M_per_batch + BM - 1) / BM;
    uint32_t box[4] = {(uint32_t)bke, BM, 1, 1};
    for (int s = 0; s < 2; ++s) {
      const float* base = s ? d.a2 : d.a1;
      if (!base) continue;
      uint64_t dims[4] = {(uint64_t)(s ? d.C2 : d.C1), (uint64_t)d.a_rows, 1, 1};
      uint64_t str[3] = {(uint64_t)d.a_ld * es, (uint64_t)d.a_ld * es * d.a_rows, (uint64_t)d.a_ld * es * d.a_rows};
      rc = encode_pair(s ? &p.tmA2 : &p.tmA1, s ? &p.tmA2l : &p.tmA1l, base, s ? d.a2_lo : d.a1_lo, 4, dims, str, box, nullptr);
      if (rc) { delete pl; return rc; }
    }
  }
  if (!d.a2) { p.tmA2 = p.tmA1; p.tmA2l = p.tmA1l; }
  p.tmA3 = p.tmA1; p.tmA4 = p.tmA1; p.tmA3l = p.tmA1l; p.tmA4l = p.tmA1l;
  p.tmH1 = p.tmA1; p.tmH2 = p.tmA1; p.tmH1l = p.tmA1l; p.tmH2l = p.tmA1l;
  {
    // Halo form: 'same'-padded stride-1 3x3 filters on 16- or 32-pixel-wide images, where the CTA's tile
    // (256 pixels, swapped form) is whole rows of ONE image: 3 loads of (rows + 2) x W pixels per
    // channel chunk instead of 9 loads of rows x W - the plain form is bound by the L2 -> SM fill rate, not the tensor pipe.
    const int tile_px = p.swap ? 256 : BM;
    const bool halo = !d.no_halo && d.conv && d.taps == 9 && p.pad == 1 && p.stride == 1 && p.swap &&
                      (d.W == 16 || d.W == 32) && (d.H * d.W) % tile_px == 0 && (d.Hin == 0 || d.Hin == d.H) && (d.Win == 0 || d.Win == d.W);
    // every launch of a shape that has a halo form walks K in that form's order, swapped or row-major, halo on or off: the
    // A/B of the two mainloops is bit-identical, and a row-major launch of such a shape (one the swapped form does not
    // take) adds the same products in the same order
    const bool halo_shape = d.conv && d.taps == 9 && p.pad == 1 && p.stride == 1 && (d.W == 16 || d.W == 32) && (d.H * d.W) % tile_px == 0 &&
                            (d.Hin == 0 || d.Hin == d.H) && (d.Win == 0 || d.Win == d.W);
    p.chunk_major = halo_shape ? 1 : 0;
    if (halo) {
      const int rows = tile_px / d.W;
      p.halo = 1; p.halo_dh_bytes = d.W * 128; p.halo_copy_bytes = (rows + 2) * d.W * 128;
      B200_REQUIRE(p.halo_copy_bytes <= HALO_X_BYTES, "gemm_tc: halo copy of %d bytes does not fit its slot", p.halo_copy_bytes);
      uint32_t box[4] = {(uint32_t)bke, (uint32_t)d.W, (uint32_t)(rows + 2), 1};
      for (int s = 0; s < 2; ++s) {
        const float* base = s ? d.a2 : d.a1;
        const int C = s ? d.C2 : d.C1;
        if (!base) continue;
        uint64_t dims[4] = {(uint64_t)C, (uint64_t)d.W, (uint64_t)d.H, (uint64_t)d.nimg};
        uint64_t str[3] = {(uint64_t)C * es, (uint64_t)d.W * C * es, (uint64_t)d.H * d.W * C * es};
        rc = encode_pair(s ? &p.tmH2 : &p.tmH1, s ? &p.tmH2l : &p.tmH1l, base, s ? d.a2_lo : d.a1_lo, 4, dims, str, box, nullptr);
        if (rc) { delete pl; return rc; }
      }
    }
  }
  if (d.a3) {
    // extra 1x1 phase: same pixel box as the main input (stride 1, same spatial size), its own channel counts
    const int HW = d.H * d.W;
    uint32_t box[4];
    if (HW >= BM) { box[1] = std::min(d.W, BM); box[2] = BM / box[1]; box[3] = 1; }
    else { box[1] = d.W; box[2] = d.H; box[3] = BM / HW; }
    box[0] = (uint32_t)bke;
    for (int s = 0; s < 2; ++s) {
      const float* base = s ? d.a4 : d.a3;
      const int C = s ? d.C4 : d.C3;
      if (!base) continue;
      uint64_t dims[4] = {(uint64_t)C, (uint64_t)d.W, (uint64_t)d.H, (uint64_t)d.nimg};
      uint64_t str[3] = {(uint64_t)C * es, (uint64_t)d.W * C * es, (uint64_t)d.H * d.W * C * es};
      rc = encode_pair(s ? &p.tmA4 : &p.tmA3, s ? &p.tmA4l : &p.tmA3l, base, s ? d.a4_lo : d.a3_lo, 4, dims, str, box, nullptr);
      if (rc) { delete pl; return rc; }
    }
    p.kchunks3 = d.C3 / bke; p.kchunks4 = d.a4 ? d.C4 / bke : 0; p.C3 = d.C3;
  }
  {
    uint64_t dims[2] = {(uint64_t)d.K_total, (uint64_t)d.w_rows};
    uint64_t str[1] = {(uint64_t)(d.w_ld ? d.w_ld : d.K_total) * es};
    uint32_t box[2] = {(uint32_t)bke, (uint32_t)(p.swap ? 128 : pl->bn)};
    rc = encode_pair(&p.tmW, &p.tmWl, d.w, d.w_lo, 2, dims, str, box, nullptr);
    if (rc) { delete pl; return rc; }
    p.tmW2 = p.tmW; p.tmW2l = p.tmWl;
    if (d.a3) {
      const uint64_t K3 = (uint64_t)d.C3 + (d.a4 ? d.C4 : 0);
      uint64_t dims2[2] = {K3, (uint64_t)d.N_total};
      uint64_t str2[1] = {K3 * es};
      rc = encode_pair(&p.tmW2, &p.tmW2l, d.w2, d.w2_lo, 2, dims2, str2, box, nullptr);
      if (rc) { delete pl; return rc; }
    }
  }
  p.total_tiles = (long long)p.nbatch * p.tiles_m_per_batch * p.tiles_n;
  *out = pl;
  return 0;
}

void tc_gemm_plan_destroy(TcGemmPlan* p) { delete p; }
const char* tc_gemm_form(const TcGemmPlan* p) {
  if (p->prm.nphase == 3) {
    if (p->prm.swap) return p->prm.halo ? "swap-halo 3xtf32" : "swap 3xtf32";
    return p->bn == 256 ? "single256 3xtf32" : "single128 3xtf32";
  }
  if (p->prm.swap) return p->prm.halo ? "swap-halo" : "swap";
  return p->bn == 256 ? "single256" : "single128";
}
void tc_gemm_set_rowvec_ld(TcGemmPlan* p, long long ld) { p->prm.epi.rowvec_ld = ld; }
void tc_gemm_set_head(TcGemmPlan* p, float* out_nchw, const float* per_img_div, long long div_stride) {
  p->prm.epi.out = out_nchw; p->prm.epi.per_img_div = per_img_div; p->prm.epi.div_stride = div_stride;
}
// ---- fused attention core (attn_tc.cuh) ----
struct TcAttnPlan { AttnParams prm; bool f16; };

bool tc_attn_supported(int T, int C) { return T == AT_T && C == AT_C; }

int tc_attn_plan_create(const TcAttnDesc& d, TcAttnPlan** out) {
  B200_REQUIRE(tc_attn_supported(d.T, d.C), "attn_tc: only T=256, C=256 (got T=%d C=%d)", d.T, d.C);
  B200_REQUIRE(d.qk && d.vT && d.w3 && d.bv && d.b3 && d.x && d.out && d.nimg > 0, "attn_tc: null argument");
  if (int r = tc_configure()) return r;
  TcAttnPlan* pl = new TcAttnPlan();
  AttnParams& p = pl->prm;
  memset(&p, 0, sizeof(p));
  pl->f16 = d.f16 != 0;
  const bool f16 = pl->f16;
  const uint64_t es = f16 ? 2 : 4;
  const uint32_t bka = f16 ? 64 : 32;
  int rc = 0;
  {
    uint64_t dims[2] = {(uint64_t)2 * AT_C, (uint64_t)d.nimg * AT_T};
    uint64_t str[1] = {(uint64_t)2 * AT_C * es};
    uint32_t boxq[2] = {bka, (uint32_t)BM}, boxk[2] = {bka, 256};
    rc = encode_map(&p.tmQ, d.qk, 2, dims, str, boxq, nullptr, f16);
    if (!rc) rc = encode_map(&p.tmK, d.qk, 2, dims, str, boxk, nullptr, f16);
  }
  if (!rc) {
    uint64_t dims[2] = {(uint64_t)AT_T, (uint64_t)d.nimg * AT_C};
    uint64_t str[1] = {(uint64_t)AT_T * es};
    uint32_t box[2] = {bka, 256};
    rc = encode_map(&p.tmVT, d.vT, 2, dims, str, box, nullptr, f16);
  }
  if (!rc) {
    uint64_t dims[2] = {(uint64_t)AT_C, (uint64_t)AT_C};
    uint64_t str[1] = {(uint64_t)AT_C * es};
    uint32_t box[2] = {bka, 256};
    rc = encode_map(&p.tmW3, d.w3, 2, dims, str, box, nullptr, f16);
  }
  if (rc) { delete pl; return rc; }
  p.bv = d.bv; p.b3 = d.b3; p.x = d.x; p.out = d.out; p.qstats = d.qstats; p.nimg = d.nimg;
  p.logit_scale = (float)((1.0 / std::sqrt((double)AT_C)) * 1.4426950408889634);
  p.out_scale = d.out_scale;
  *out = pl;
  return 0;
}
void tc_attn_plan_destroy(TcAttnPlan* p) { delete p; }
int tc_attn_launch(const TcAttnPlan* pl, cudaStream_t st) {
  const long long tiles = 2LL * pl->prm.nimg;
  const int grid = (int)std::min<long long>(tiles, num_sms());
  if (pl->f16) launch_kernel(attn_tc_kernel<true>, dim3(grid), dim3(384), AttnSmem<true>::TOTAL, st, pl->prm);
  else launch_kernel(attn_tc_kernel<false>, dim3(grid), dim3(384), AttnSmem<false>::TOTAL, st, pl->prm);
  B200_CHECK_LAUNCH();
  return 0;
}

// Opt in to the large dynamic shared-memory carve-out once, outside any stream capture.
static int tc_configure() {
  static bool configured = false;
  if (configured) return 0;
  B200_CHECK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemLayout<256>::TOTAL));
  B200_CHECK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemLayout<128>::TOTAL));
  B200_CHECK_CUDA(cudaFuncSetAttribute(attn_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnSmem<false>::TOTAL));
  B200_CHECK_CUDA(cudaFuncSetAttribute(attn_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnSmem<true>::TOTAL));
  configured = true;
  return 0;
}

template <int BN>
static int launch_impl(const TcGemmPlan* pl, cudaStream_t st) {
  const int grid = (int)std::min<long long>(pl->prm.total_tiles, num_sms());
  launch_kernel(gemm_tc_kernel<BN>, dim3(grid), dim3(384), SmemLayout<BN>::TOTAL, st, pl->prm);
  B200_CHECK_LAUNCH();
  return 0;
}

int tc_gemm_launch(const TcGemmPlan* pl, cudaStream_t st) {
  if (pl->prm.total_tiles == 0) return 0;
  return pl->bn == 256 ? launch_impl<256>(pl, st) : launch_impl<128>(pl, st);
}

}  // namespace b200
