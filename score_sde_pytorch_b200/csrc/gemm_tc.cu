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
// the same accumulator: only the producer's tensor-map choice (phase_maps) and the K count change; ring, barriers and
// epilogue do not.
//
// gemm_tc_kernel<BN> (persistent, warp-specialised, 384 threads; the fused attention core is in attn_tc.cu): one CTA per
// tile of 128 rows x BN columns, or - `swap` - 128 output channels x 256 pixels (D^T = W X^T) for 128-channel
// convolutions, 1x1 convolutions, the network head and the 3x3 'same' convolutions on 16- / 32-pixel rows.
//   warp 0       TMA producer (whole warp, TMA instructions predicated on one elect.sync lane; SWIZZLE_128B, zero halo and
//                tail rows from out-of-bounds fill): produce_taps, one box shifted by the filter tap per K step, or
//                produce_halo, three W-shifted copies of the tile with its halo per channel chunk;
//   warps 1..3   idle (their registers go to the MMA warpgroups);
//   warps 4..11  two MMA warpgroups, m64 x BN wgmma over 64 rows each: consume_ring or consume_halo per tile, then
//                store_tile (NCHW head, or stage_epilogue - compiled per orientation x residual x store format x stats -
//                through shared memory and TMA stores that drain during the next tile's mainloop).
#include "tc_common.cuh"
#include <cudaTypedefs.h>
#include <array>
#include <mutex>
#include <cstring>

namespace b200 {

namespace {

// Halo form of the 3x3 mainloop.  The nine filter taps of one channel chunk read three W-shifted
// copies of the tile *with its one-row halo* (TMA box [chunk, W, rows + 2], origin w = -1 / 0 / +1, zero fill outside the
// image); the operand of tap (dh, dw) is copy[dw] starting (dh + 1) * W pixels in - a multiple of 1024 bytes, so a plain
// swizzled descriptor.  L2 -> shared-memory traffic per chunk: 3 x (rows + 2) / rows tiles instead of 9.
constexpr int HALO_XS = 3;                  // halo copies in flight (each feeds 3 K steps)
constexpr int HALO_X_BYTES = 40 * 1024;     // swapped form: (8 + 2) rows x 32 pixels x 128 B
constexpr int HALO_WS = 4;                  //   its weight-slice ring: 4 x 16 KB   (3 x 40 + 4 x 16 = 184 KB)

struct TcParams {
  // [.][0] hi, [.][1] split-TF32 lo twin.  a: sources 0, 1 = the filter input, 2, 3 = the extra 1x1 K phase (fused skip
  // projection, weights w[1]); h: halo form, box [bke, W, tile rows + 2, 1].  Maps a plan lacks copy a[0] (w[1]: w[0]).
  CUtensorMap a[4][2], w[2][2], h[2][2];
  CUtensorMap out_map, res_map;            // staged epilogue: [rows][N_total] output (store) and fp32 residual (load)
  int nphase;                              // 3: split TF32, every K step loads (A lo, W hi), (A hi, W lo), (A hi, W hi); else 1
  int halo;                               // 1: 3x3 taps read W-shifted halo copies of the tile (3 loads per channel chunk instead of 9)
  int halo_dh_bytes;                       // W * 128: bytes between the operand windows of consecutive filter rows inside a copy
  int halo_copy_bytes;                     // (tile rows + 2) * W * 128: bytes of one halo copy
  int chunk_major;                         // nine-load loop walks K as (chunk, filter column, filter row): shapes with a halo form
  int conv, H, W, taps, pad, S, stride;   // H, W: OUTPUT spatial size; S = filter width (3 or 1)
  int kchunks[4];                          // channel chunks of each source (0: no such source)
  int wcol[4];                             // first weight column of each source: 0, C1 in w[0]; 0, C3 in w[1]
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

// The maps of product phase `ph` of a K step: split TF32 runs (A lo, W hi), (A hi, W lo), (A hi, W hi), small terms
// first; the other formats run phase 0 alone, on the hi maps.
struct PhaseMaps { const CUtensorMap* a; const CUtensorMap* w; };
__device__ __forceinline__ PhaseMaps phase_maps(const TcParams& p, const CUtensorMap (&a)[2], const CUtensorMap (&w)[2], int ph) {
  return {&a[p.nphase == 3 && ph == 0], &w[ph == 1]};
}


// Staged epilogue.  Each MMA warpgroup owns two STG_BUF-byte shared-memory buffers and stores its 64 accumulator rows in
// rounds: its warps write one round's values into a buffer, laid out as rows of the output, and one thread (the
// warpgroup's leader) TMA-stores it while the warps fill the other buffer.  The last stores of a tile drain while the
// next tile's mainloop runs.  A round is 32 output columns of the 64 rows (row-major tiles: one box of 64 pixels x 32
// channels) or 32 pixels of the 64 output channels (swapped tiles: two boxes of 32 pixels x 32 channels).  Box rows hold
// 32 elements: 128 B with the 128-byte swizzle for fp32 (output and residual), 64 B with the 64-byte swizzle for fp16
// output, so the fragment writes do not bank-conflict.  The TMA store clips at the tensor map's bounds (the M tail, an
// output pitch wider than N).  The residual of round r + 1 is TMA-loaded into the other buffer while round r is
// computed (round 0 at tile start, before the mainloop), and each value's result overwrites its residual in place.
// (Also prefetching a tile's later residual rounds into L2 at tile start measured slower on H100: 832 instead of 732 us
// for `conv3x3 128->128 @32 +res` at batch 1024.)
constexpr int STG_BUF = 8 * 1024;
constexpr int STG_BYTES = 2 * 2 * STG_BUF;   // two warpgroups x two buffers

// Read-only global load kept in program order with the epilogue's other asm (shared-memory accesses, barriers): the
// compiler would otherwise hoist the bias / row-vector loads of later rounds and spill them next to the accumulator.
__device__ __forceinline__ float2 ldg_f32x2_ordered(const float* a) {
  float2 v;
  asm volatile("ld.global.nc.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(a));
  return v;
}

// byte offset of element (row r, column c) of a staged box with 32-element rows
template <bool F16>
__device__ __forceinline__ uint32_t stg_off(int r, int c) {
  if (F16) return r * 64 + ((((c >> 3) ^ (r >> 1)) & 3) << 4) + (c & 7) * 2;
  return r * 128 + ((((c >> 2) ^ r) & 7) << 4) + (c & 3) * 4;
}

// One warpgroup's output region in one tile, swapped (SWAP) or row-major: box k of round r starts at global
// (column, row) (box_col(r, k), box_row(r)).
template <bool SWAP>
struct StageTile {
  int col0, row0;
  static constexpr int nbox() { return SWAP ? 2 : 1; }
  __device__ __forceinline__ int box_col(int r, int k) const { return col0 + 32 * (SWAP ? k : r); }
  __device__ __forceinline__ int box_row(int r) const { return row0 + (SWAP ? 32 * r : 0); }
  static constexpr int box_bytes(int es) { return (SWAP ? 32 : 64) * 32 * es; }
};

template <int BN, bool SWAP>
__device__ __forceinline__ StageTile<SWAP> stage_tile(const TcParams& p, int tile, int g) {
  const int nt = tile % p.tiles_n, mg = tile / p.tiles_n;
  if (SWAP) return {nt * 128 + 64 * g, mg * 256};
  const int b = mg / p.tiles_m_per_batch, mt = mg % p.tiles_m_per_batch;
  return {nt * BN, b * p.M_per_batch + mt * BM + 64 * g};
}

// Leader: the residual of round r into buffer `buf`, completing on `bar` (shared-window addresses).
template <bool SWAP>
__device__ __forceinline__ void load_residual(const TcParams& p, const StageTile<SWAP>& t, int r, uint32_t buf, uint32_t bar) {
  mbar_expect_tx(bar, STG_BUF);
  for (int k = 0; k < t.nbox(); ++k) tma_load_2d(&p.res_map, buf + k * t.box_bytes(4), bar, t.box_col(r, k), t.box_row(r));
}

// The epilogue of one warp's 16 accumulator rows, specialised by operand orientation (SWAP), residual add (RES), store
// format (MODE: 0 fp32, 1 TF32-rounded fp32, 2 fp16) and GroupNorm quad sums of the stored values (STATS).  Each value is
// (acc + (bias + rowvec) + residual) * scale, then rounded, as it always was; only where it is written changed.
//   SWAP: rows = output channels c0 + 16wq .. of ONE image, columns = the tile's 256 pixels.  Lane l holds channels
//         l/4 and l/4 + 8 of pixel pairs 8j + 2(l%4).
//   else: rows = pixels / tokens, columns = output channels; lane l holds rows l/4 and l/4 + 8, column pairs 8j + 2(l%4).
//         rows_valid: rows of the warp's 16 inside the matrix (GroupNorm sums only: the TMA store clips the rest).
template <int BN, bool SWAP, bool RES, int MODE, bool STATS>
__device__ __forceinline__ void stage_epilogue(const TcParams& p, const float (&d)[BN / 2], const StageTile<SWAP>& t, uint32_t stg,
                                               uint32_t rbar, uint32_t& rpar, int rows_valid, int g, int wq, int lane,
                                               bool leader) {
  constexpr bool H = MODE == 2;
  constexpr int ES = H ? 2 : 4;
  constexpr int ROUNDS = SWAP ? 8 : BN / 32;
  const Epilogue& e = p.epi;
  const float scale = e.scale;
  const int q = lane & 3;
  // row-major: the warp's two rows in the box; swapped: its two channels in box wq / 2
  const int ra = (SWAP ? 16 * (wq & 1) : 16 * wq) + (lane >> 2), rb = ra + 8;
  const int kbox = SWAP ? wq >> 1 : 0;
  const bool va = ra - 16 * wq < rows_valid, vb = rb - 16 * wq < rows_valid;
  int img;
  float adda = 0.f, addb = 0.f;
  const float* rv = nullptr;
  if (SWAP) {
    img = t.row0 / e.rows_per_img;     // rows_per_img % 256 == 0: one image per tile
    const int ca = t.col0 + 32 * kbox + ra, cb = ca + 8;
    adda = (e.bias ? __ldg(e.bias + ca) : 0.f) + (e.rowvec ? __ldg(e.rowvec + img * e.rowvec_ld + ca) : 0.f);
    addb = (e.bias ? __ldg(e.bias + cb) : 0.f) + (e.rowvec ? __ldg(e.rowvec + img * e.rowvec_ld + cb) : 0.f);
  } else {
    img = rows_valid > 0 ? (t.row0 + 16 * wq) / e.rows_per_img : 0;   // the 16 rows of a warp belong to one image
    rv = e.rowvec ? e.rowvec + (long long)img * e.rowvec_ld : nullptr;
  }
  // Offsets of the thread's values in a box, output and fp32 residual layouts.  The swizzle repeats every 8 rows and
  // only permutes 16-byte chunks within a row, so
  //   swapped:   the four values of pixel rows 2q + {0, 1}; column group jj is 8jj rows further on;
  //   row-major: rows ra and rb at column 2q; column group jj (8 columns = 2 fp32 / 1 fp16 chunks further) flips
  //              chunk-index bits, i.e. XORs the offset with jj << 5 (fp32) or jj << 4 (fp16).
  uint32_t ooff[SWAP ? 4 : 2], roff[SWAP ? 4 : 2];
#pragma unroll
  for (int i = 0; i < (SWAP ? 4 : 2); ++i) {
    const int row = SWAP ? 2 * q + (i & 1) : (i ? rb : ra), col = SWAP ? (i < 2 ? ra : rb) : 2 * q;
    ooff[i] = stg_off<H>(row, col);
    roff[i] = stg_off<false>(row, col);
  }
  // writes the four values of fragment column group jj of the round: fp32, or fp16 pairs h01 = (v0, v1), h23 = (v2, v3)
  // (cvt.rn.f16x2 rounds each half as cvt.rn.f16 does)
  auto put = [&](uint32_t obox, int jj, const float* v, uint32_t h01, uint32_t h23) {
    if (SWAP) {
      if (H) {
        st_shared_u16(obox + ooff[0] + jj * 8 * 64, (uint16_t)h01); st_shared_u16(obox + ooff[1] + jj * 8 * 64, (uint16_t)(h01 >> 16));
        st_shared_u16(obox + ooff[2] + jj * 8 * 64, (uint16_t)h23); st_shared_u16(obox + ooff[3] + jj * 8 * 64, (uint16_t)(h23 >> 16));
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) st_shared_f32(obox + ooff[i] + jj * 8 * 128, v[i]);
      }
    } else if (H) {
      st_shared_u32(obox + (ooff[0] ^ (jj << 4)), h01);
      st_shared_u32(obox + (ooff[1] ^ (jj << 4)), h23);
    } else {
      st_shared_f32x2(obox + (ooff[0] ^ (jj << 5)), v[0], v[1]);
      st_shared_f32x2(obox + (ooff[1] ^ (jj << 5)), v[2], v[3]);
    }
  };
  float sa = 0.f, qa = 0.f, sb = 0.f, qb = 0.f;
#pragma unroll
  for (int r = 0; r < ROUNDS; ++r) {
    const int b = r & 1;
    const uint32_t buf = stg + b * STG_BUF;
    if (leader) {
      bulk_wait_read<0>();   // the store of round r - 1 has read the other buffer
      if (RES && r + 1 < ROUNDS) load_residual(p, t, r + 1, stg + (b ^ 1) * STG_BUF, rbar + 8 * (b ^ 1));
    }
    if (RES) { mbar_wait(rbar + 8 * b, (rpar >> b) & 1); rpar ^= 1u << b; }
    const uint32_t rbox = buf + kbox * t.box_bytes(4);
    const uint32_t obox = buf + kbox * t.box_bytes(ES);
    // fp16 values overlay the round's fp32 residual: they are held, packed, until every thread has read its own
    uint32_t hp[RES && H ? 8 : 1];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = 4 * r + jj;
      float v[4];
      if (SWAP) {
        // pixel rows 8jj + 2q + {0, 1} of the box: the swizzle repeats every 8 rows, so 8jj rows past the jj = 0 offsets
        v[0] = d[4 * j] + adda; v[1] = d[4 * j + 1] + adda; v[2] = d[4 * j + 2] + addb; v[3] = d[4 * j + 3] + addb;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if (RES) v[i] += ld_shared_f32(rbox + roff[i] + jj * 1024);
          v[i] *= scale;
          if (MODE == 1) v[i] = round_tf32(v[i]);
        }
        if (STATS) {
          sa += v[0] + v[1]; qa = fmaf(v[0], v[0], fmaf(v[1], v[1], qa));
          sb += v[2] + v[3]; qb = fmaf(v[2], v[2], fmaf(v[3], v[3], qb));
        }
      } else {
        const int col = t.col0 + 8 * j + 2 * q;
        float2 ad = make_float2(0.f, 0.f);
        if (e.bias) ad = ldg_f32x2_ordered(e.bias + col);
        if (rv) { const float2 u = ldg_f32x2_ordered(rv + col); ad.x += u.x; ad.y += u.y; }
        v[0] = d[4 * j] + ad.x; v[1] = d[4 * j + 1] + ad.y; v[2] = d[4 * j + 2] + ad.x; v[3] = d[4 * j + 3] + ad.y;
        if (RES) {
          const float2 ua = ld_shared_f32x2(rbox + (roff[0] ^ (jj << 5)));
          const float2 ub = ld_shared_f32x2(rbox + (roff[1] ^ (jj << 5)));
          v[0] += ua.x; v[1] += ua.y; v[2] += ub.x; v[3] += ub.y;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          v[i] *= scale;
          if (MODE == 1) v[i] = round_tf32(v[i]);
        }
        if (STATS) {
          float s = (va ? v[0] + v[1] : 0.f) + (vb ? v[2] + v[3] : 0.f);
          float qq = (va ? fmaf(v[0], v[0], v[1] * v[1]) : 0.f) + (vb ? fmaf(v[2], v[2], v[3] * v[3]) : 0.f);
#pragma unroll
          for (int m = 4; m <= 16; m <<= 1) { s += __shfl_xor_sync(0xffffffffu, s, m); qq += __shfl_xor_sync(0xffffffffu, qq, m); }
          s += __shfl_xor_sync(0xffffffffu, s, 1); qq += __shfl_xor_sync(0xffffffffu, qq, 1);
          if ((lane & ~2) == 0 && rows_valid > 0) {   // lanes 0 and 2: the two column quads of this 8-column group
            double* qd = p.qstats + ((long long)img * (p.N_total >> 2) + (col >> 2)) * 2;
            atomicAdd(qd, (double)s); atomicAdd(qd + 1, (double)qq);
          }
        }
      }
      const uint32_t h01 = H ? pack_half2(v[0], v[1]) : 0u, h23 = H ? pack_half2(v[2], v[3]) : 0u;
      if constexpr (RES && H) { hp[2 * jj] = h01; hp[2 * jj + 1] = h23; }
      else put(obox, jj, v, h01, h23);
    }
    if constexpr (RES && H) {
      wg_barrier(g);
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) put(obox, jj, nullptr, hp[2 * jj], hp[2 * jj + 1]);
    }
    fence_async_smem();   // generic-proxy writes -> the TMA store's reads
    wg_barrier(g);
    if (leader) {
      for (int k = 0; k < t.nbox(); ++k) tma_store_2d(&p.out_map, buf + k * t.box_bytes(ES), t.box_col(r, k), t.box_row(r));
      bulk_commit();
    }
  }
  if (SWAP && STATS) {
#pragma unroll
    for (int m = 1; m <= 8; m <<= 1) {   // pixel lanes (1, 2), then the four channels of a quad (4, 8)
      sa += __shfl_xor_sync(0xffffffffu, sa, m); qa += __shfl_xor_sync(0xffffffffu, qa, m);
      sb += __shfl_xor_sync(0xffffffffu, sb, m); qb += __shfl_xor_sync(0xffffffffu, qb, m);
    }
    if ((lane & 15) == 0) {
      const int ca = t.col0 + 32 * kbox + ra, cb = ca + 8;
      double* qd = p.qstats + ((long long)img * (p.N_total >> 2) + (ca >> 2)) * 2;
      atomicAdd(qd, (double)sa); atomicAdd(qd + 1, (double)qa);
      qd = p.qstats + ((long long)img * (p.N_total >> 2) + (cb >> 2)) * 2;
      atomicAdd(qd, (double)sb); atomicAdd(qd + 1, (double)qb);
    }
  }
}

template <int BN>
struct SmemLayout {
  static constexpr int STAGES = BN == 256 ? 4 : 6;
  static constexpr int B_STAGE_BYTES = BN * BKE * 4;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  static constexpr int HALO_BYTES = HALO_XS * HALO_X_BYTES + HALO_WS * A_STAGE_BYTES;   // the swapped halo form's two rings
  static constexpr int STG_OFFSET = BN == 256 && HALO_BYTES > RING_BYTES ? HALO_BYTES : RING_BYTES;   // epilogue staging
  static constexpr int BAR_OFFSET = STG_OFFSET + STG_BYTES;
  // barrier arrays (byte offsets from the aligned base): ring full / empty, halo weight-slice full / empty, residual loads
  static constexpr int FULL_BAR = BAR_OFFSET, EMPTY_BAR = FULL_BAR + 8 * STAGES, WFULL_BAR = EMPTY_BAR + 8 * STAGES;
  static constexpr int WEMPTY_BAR = WFULL_BAR + 8 * HALO_WS, RES_BAR = WEMPTY_BAR + 8 * HALO_WS;
  static constexpr int TOTAL = BAR_OFFSET + 256 + 1024;   // barriers + slack for 1024-B alignment
  static_assert(TOTAL <= 232448, "exceeds the 227 KB shared-memory limit of sm_90");
  static_assert(BN != 256 || STAGES >= HALO_XS, "the halo copies use the first HALO_XS stage barriers");
  static_assert(STG_OFFSET % 1024 == 0 && STG_BUF % 1024 == 0, "staged boxes need the 128-byte swizzle's 1024-B alignment");
  static_assert(RES_BAR + 4 * 8 <= BAR_OFFSET + 256, "barriers overflow their 256 bytes");
};

// Producer stages run on warp 0 as a whole; only the elected lane (`issue`) issues TMA instructions.
// Nine-load form, swapped or row-major: per K step one ring slot with the W box and the A box(es) shifted by the tap.
template <int BN>
__device__ __forceinline__ void produce_taps(const TcParams& p, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, bool issue) {
  using L = SmemLayout<BN>;
  const int HW = p.H * p.W, bke = p.bke;
  uint32_t stage = 0, phase = 0;
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
      const int nch = p.kchunks[src];
      if (nch == 0) continue;
      const int wcol0 = p.wcol[src];
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
          for (int ph = 0; ph < p.nphase; ++ph) {
            const PhaseMaps m = phase_maps(p, p.a[src], p.w[src >> 1], ph);
            mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* sa = smem + stage * L::STAGE_BYTES;
            uint8_t* sb = sa + A_STAGE_BYTES;
            if (issue) {
              mbar_expect_tx(&full_bar[stage], L::STAGE_BYTES);
              if (p.swap) {
                // first 16 KiB: 128 output channels x 32 k of W (MMA A); next 32 KiB: 256 pixels x 32 k (MMA B)
                tma_load_2d(m.w, sa, &full_bar[stage], wcol0 + kc * bke, wrow0 + tap * p.N_total);
                tma_load_4d(m.a, sb, &full_bar[stage], kc * bke, w0 + dw, h0 + dh, img0);
                tma_load_4d(m.a, sb + A_STAGE_BYTES, &full_bar[stage], kc * bke, w1 + dw, h1 + dh, img1);
              } else {
                if (p.conv) tma_load_4d(m.a, sa, &full_bar[stage], kc * bke, w0 * p.stride + dw, h0 * p.stride + dh, img0);
                else tma_load_4d(m.a, sa, &full_bar[stage], kc * bke, arow0, 0, 0);
                tma_load_2d(m.w, sb, &full_bar[stage], wcol0 + kc * bke, wrow0 + tap * p.N_total);
              }
            }
            if (++stage == L::STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  }
}

// Halo form (swapped operands, one image per 256-pixel tile, W <= 32): per channel chunk three halo copies (ring of
// HALO_XS slots on the stage barriers), each followed by the three 16 KB weight slices of its filter column (ring of
// HALO_WS slots with their own barriers).
__device__ __forceinline__ void produce_halo(const TcParams& p, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                             uint64_t* wfull_bar, uint64_t* wempty_bar, bool issue) {
  const int HW = p.H * p.W, bke = p.bke;
  uint32_t stage = 0, phase = 0, ws = 0, wphase = 0;
  uint8_t* const wring = smem + HALO_XS * HALO_X_BYTES;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const int nt = (int)(tile % p.tiles_n);
    const int p0 = (tile / p.tiles_n) * 256;
    const int img0 = (int)(p0 / HW), h0 = (int)(p0 % HW) / p.W;
    const int wrow0 = nt * 128;
    for (int src = 0; src < 4; ++src) {
      const int nch = p.kchunks[src];
      if (nch == 0) continue;
      const int wcol0 = p.wcol[src];
      for (int kc = 0; kc < nch; ++kc) {
        if (src < 2) {
          for (int dwi = 0; dwi < 3; ++dwi) {
            // split TF32: the copy + its three weight slices once per product phase
            for (int ph = 0; ph < p.nphase; ++ph) {
              const PhaseMaps m = phase_maps(p, p.h[src], p.w[0], ph);
              mbar_wait(&empty_bar[stage], phase ^ 1);
              if (issue) {
                mbar_expect_tx(&full_bar[stage], (uint32_t)p.halo_copy_bytes);
                tma_load_4d(m.a, smem + stage * HALO_X_BYTES, &full_bar[stage], kc * bke, dwi - 1, h0 - 1, img0);
              }
              if (++stage == HALO_XS) { stage = 0; phase ^= 1; }
              for (int dhi = 0; dhi < 3; ++dhi) {
                mbar_wait(&wempty_bar[ws], wphase ^ 1);
                if (issue) {
                  mbar_expect_tx(&wfull_bar[ws], A_STAGE_BYTES);
                  tma_load_2d(m.w, wring + ws * A_STAGE_BYTES, &wfull_bar[ws], wcol0 + kc * bke, wrow0 + (dhi * 3 + dwi) * p.N_total);
                }
                if (++ws == HALO_WS) { ws = 0; wphase ^= 1; }
              }
            }
          }
        } else {
          // extra 1x1 phase (fused skip projection): the plain 256-pixel tile as two 128-pixel boxes, its own weights
          const int h1 = h0 + 128 / p.W;
          for (int ph = 0; ph < p.nphase; ++ph) {
            const PhaseMaps m = phase_maps(p, p.a[src], p.w[1], ph);
            mbar_wait(&empty_bar[stage], phase ^ 1);
            if (issue) {
              mbar_expect_tx(&full_bar[stage], 2 * A_STAGE_BYTES);
              tma_load_4d(m.a, smem + stage * HALO_X_BYTES, &full_bar[stage], kc * bke, 0, h0, img0);
              tma_load_4d(m.a, smem + stage * HALO_X_BYTES + A_STAGE_BYTES, &full_bar[stage], kc * bke, 0, h1, img0);
            }
            if (++stage == HALO_XS) { stage = 0; phase ^= 1; }
            mbar_wait(&wempty_bar[ws], wphase ^ 1);
            if (issue) {
              mbar_expect_tx(&wfull_bar[ws], A_STAGE_BYTES);
              tma_load_2d(m.w, wring + ws * A_STAGE_BYTES, &wfull_bar[ws], wcol0 + kc * bke, wrow0);
            }
            if (++ws == HALO_WS) { ws = 0; wphase ^= 1; }
          }
        }
      }
    }
  }
}

// MMA stages: warpgroup g (0, 1) owns accumulator rows 64g .. 64g + 63 of every tile.  A K step is released to the
// producer once the wgmma after it has been issued (wait_group 1), so the tensor core always has the next step queued
// while the previous one's slot is handed back.
// The MMA warps address shared memory through 32-bit shared-window addresses (sm: the aligned base, SmemLayout
// offsets): generic pointers would hold two registers each next to the 128-register accumulator.
// One tile from the nine-load ring.
template <int BN, bool F16>
__device__ __forceinline__ void consume_ring(const TcParams& p, uint32_t sm, float (&acc)[BN / 2], int kiters, uint32_t& stage,
                                             uint32_t& phase, int g, int lane) {
  using L = SmemLayout<BN>;
  int pend = -1;
  for (int it = 0; it < kiters; ++it) {
    mbar_wait(sm + L::FULL_BAR + 8 * stage, phase);
    const uint32_t sa = sm + stage * L::STAGE_BYTES;
    wgmma_kstep<BN, F16>(acc, make_smem_desc(sa + g * (A_STAGE_BYTES / 2)), make_smem_desc(sa + A_STAGE_BYTES), it);
    wgmma_wait<1>();
    if (lane == 0 && pend >= 0) mbar_arrive(sm + L::EMPTY_BAR + 8 * pend);
    pend = (int)stage;
    if (++stage == L::STAGES) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  if (lane == 0 && pend >= 0) mbar_arrive(sm + L::EMPTY_BAR + 8 * pend);
}

// One tile of the halo form: A = the 16 KB weight slice (128 output channels), B = 256 pixel rows of a halo copy starting
// one filter row (W pixels) further in per dh; the slice's slot is released per tap, the copy's after its three taps.
template <int BN, bool F16>
__device__ __forceinline__ void consume_halo(const TcParams& p, uint32_t sm, float (&acc)[BN / 2], uint32_t& stage,
                                             uint32_t& phase, uint32_t& ws, uint32_t& wphase, int g, int lane) {
  using L = SmemLayout<BN>;
  const uint32_t wring = sm + HALO_XS * HALO_X_BYTES;
  int it = 0, pend_ws = -1, pend_x = -1;
  for (int src = 0; src < 4; ++src) {
    const int nch = p.kchunks[src];
    const int ncopies = (src < 2 ? 3 * nch : nch) * p.nphase, ntap = src < 2 ? 3 : 1;
    for (int c = 0; c < ncopies; ++c) {
      mbar_wait(sm + L::FULL_BAR + 8 * stage, phase);
      const uint32_t sx = sm + stage * HALO_X_BYTES;
      for (int dhi = 0; dhi < ntap; ++dhi, ++it) {
        mbar_wait(sm + L::WFULL_BAR + 8 * ws, wphase);
        const uint64_t adesc = make_smem_desc(wring + ws * A_STAGE_BYTES + g * (A_STAGE_BYTES / 2));
        const uint64_t bdesc = make_smem_desc(sx + (src < 2 ? dhi * p.halo_dh_bytes : 0));
        wgmma_kstep<BN, F16>(acc, adesc, bdesc, it);
        wgmma_wait<1>();
        if (lane == 0) {
          if (pend_ws >= 0) mbar_arrive(sm + L::WEMPTY_BAR + 8 * pend_ws);
          if (pend_x >= 0) mbar_arrive(sm + L::EMPTY_BAR + 8 * pend_x);
        }
        pend_ws = (int)ws; pend_x = dhi == ntap - 1 ? (int)stage : -1;
        if (++ws == HALO_WS) { ws = 0; wphase ^= 1; }
      }
      if (++stage == HALO_XS) { stage = 0; phase ^= 1; }
    }
  }
  wgmma_wait<0>();
  if (lane == 0) {
    if (pend_ws >= 0) mbar_arrive(sm + L::WEMPTY_BAR + 8 * pend_ws);
    if (pend_x >= 0) mbar_arrive(sm + L::EMPTY_BAR + 8 * pend_x);
  }
}

// Epilogue of one tile: warp wq of MMA warpgroup g stores its 16 accumulator rows (tile rows 64g + 16wq ..).
// Network head (swapped operands, NCHW store):
template <int BN>
__device__ __forceinline__ void store_head(const TcParams& p, const float (&acc)[BN / 2], int tile, int g, int wq, int lane) {
  const Epilogue& e = p.epi;
  // ncsnpp.py:374-380: the 128-row weight tile is zero-padded above the n_valid image channels; (acc + bias) / sigma[img]
  // is written as NCHW
  const int c0 = (int)(tile % p.tiles_n) * 128 + g * 64 + wq * 16;
  const int pix0 = (tile / p.tiles_n) * 256;
  const int img = pix0 / e.rows_per_img;     // rows_per_img % 256 == 0: one image per tile
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
}

// Every other tile: the staged epilogue.
template <int BN, bool SWAP, bool RES, int MODE, bool STATS>
__device__ __forceinline__ void store_tile(const TcParams& p, const float (&acc)[BN / 2], int tile, int g, int wq, int lane,
                                           uint32_t stg, uint32_t rbar, uint32_t& rpar, bool leader) {
  const StageTile<SWAP> t = stage_tile<BN, SWAP>(p, tile, g);
  const int mt = (int)((tile / p.tiles_n) % p.tiles_m_per_batch);
  const int rows_valid = min(16, max(0, p.M_per_batch - (mt * BM + g * 64 + wq * 16)));   // row-major tiles only
  stage_epilogue<BN, SWAP, RES, MODE, STATS>(p, acc, t, stg, rbar, rpar, rows_valid, g, wq, lane, leader);
}

// The MMA warps' tile loop.  store(acc, tile, stg, rbar, rpar, leader) is one compiled epilogue variant, chosen once
// per launch: each variant's loop gets its own register allocation next to the 128-register accumulator.
template <int BN, bool F16, class Store>
__device__ __forceinline__ void gemm_tc_consumer(const TcParams& p, uint32_t sm, int g, int wq, int lane, Store&& store) {
  using L = SmemLayout<BN>;
  const int kiters = ((p.kchunks[0] + p.kchunks[1]) * p.taps + p.kchunks[2] + p.kchunks[3]) * p.nphase;
  // the leader (thread 0 of the warpgroup: wq == 0, lane 0) issues the epilogue's TMA and owns its bulk groups; read from
  // threadIdx where it is used rather than held across the loop
  auto leader = [] { return (threadIdx.x & 127) == 0; };
  const uint32_t stg = sm + L::STG_OFFSET + g * 2 * STG_BUF;   // this warpgroup's staging buffers
  const uint32_t rbar = sm + L::RES_BAR + g * 2 * 8;            // and their residual barriers
  uint32_t stage = 0, phase = 0, ws = 0, wphase = 0, rpar = 0;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    if (leader() && p.epi.residual) {   // round 0's residual into buffer 0 (stg, rbar: the warpgroup's buffers, barriers)
      if (BN == 256 && p.swap) load_residual(p, stage_tile<BN, true>(p, tile, g), 0, stg, rbar);
      else load_residual(p, stage_tile<BN, false>(p, tile, g), 0, stg, rbar);
    }
    float acc[BN / 2];
    if (BN == 256 && p.halo) consume_halo<BN, F16>(p, sm, acc, stage, phase, ws, wphase, g, lane);
    else consume_ring<BN, F16>(p, sm, acc, kiters, stage, phase, g, lane);
    store(acc, tile, stg, rbar, rpar, leader());
  }
  if (leader()) bulk_wait<0>();   // every store has landed before the CTA exits (dependent launches run under PDL)
}

// The tile loop with one staged-epilogue variant.  (Functions and by-value captures throughout: a lambda object or a
// captured reference that is not inlined away lives in local memory.)
template <int BN, bool F16, bool SWAP, bool RES, int MODE, bool STATS>
__device__ __forceinline__ void gemm_tc_staged(const TcParams& p, uint32_t sm, int g, int wq, int lane) {
  gemm_tc_consumer<BN, F16>(p, sm, g, wq, lane, [&p, g, wq, lane](const float (&acc)[BN / 2], int tile, uint32_t stg,
                                                                uint32_t rbar, uint32_t& rpar, bool leader) {
    store_tile<BN, SWAP, RES, MODE, STATS>(p, acc, tile, g, wq, lane, stg, rbar, rpar, leader);
  });
}

// Staged-epilogue variant v = 6 RES + 2 MODE + STATS (residual add, store format Epilogue::round_tf32, GroupNorm quad
// sums): each of the 12 is its own compiled tile loop.
template <int BN, bool F16, bool SWAP, int V = 0>
__device__ __forceinline__ void gemm_tc_select(const TcParams& p, uint32_t sm, int g, int wq, int lane, int v) {
  if constexpr (V < 12) {
    if (v == V) gemm_tc_staged<BN, F16, SWAP, (V >= 6), (V / 2) % 3, (V & 1) != 0>(p, sm, g, wq, lane);
    else gemm_tc_select<BN, F16, SWAP, V + 1>(p, sm, g, wq, lane, v);
  }
}

// Selects the epilogue (head, or orientation x staged variant) and runs the tile loop.
template <int BN, bool F16>
__device__ __forceinline__ void gemm_tc_mma(const TcParams& p, uint32_t sm, int g, int wq, int lane) {
  if constexpr (BN == 256) {
    if (p.swap && p.epi.out_nchw) {
      gemm_tc_consumer<BN, F16>(p, sm, g, wq, lane, [&p, g, wq, lane](const float (&acc)[BN / 2], int tile, uint32_t, uint32_t, uint32_t&, bool) {
        store_head<BN>(p, acc, tile, g, wq, lane);
      });
      return;
    }
  }
  const int v = (p.epi.residual ? 6 : 0) + 2 * p.epi.round_tf32 + (p.qstats ? 1 : 0);
  if constexpr (BN == 256) {
    if (p.swap) { gemm_tc_select<BN, F16, true>(p, sm, g, wq, lane, v); return; }
  }
  gemm_tc_select<BN, F16, false>(p, sm, g, wq, lane, v);
}

// ---------------------------------------------------------------------------
// Kernel
// ---------------------------------------------------------------------------
template <int BN>
__global__ void __launch_bounds__(384, 1) gemm_tc_kernel(const __grid_constant__ TcParams p) {
  using L = SmemLayout<BN>;
  constexpr int STAGES = L::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::FULL_BAR);
  uint64_t* empty_bar = reinterpret_cast<uint64_t*>(smem + L::EMPTY_BAR);
  uint64_t* wfull_bar = reinterpret_cast<uint64_t*>(smem + L::WFULL_BAR);     // halo form: the weight-slice ring has its own barriers
  uint64_t* wempty_bar = reinterpret_cast<uint64_t*>(smem + L::WEMPTY_BAR);
  uint64_t* res_bar = reinterpret_cast<uint64_t*>(smem + L::RES_BAR);         // staged epilogue: residual loads, two per MMA warpgroup

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp index provably warp-uniform

  if (threadIdx.x == 0) {
    // empty slots: one arrival per MMA warp (8)
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
    for (int s = 0; s < HALO_WS; ++s) { mbar_init(&wfull_bar[s], 1); mbar_init(&wempty_bar[s], 8); }
    for (int s = 0; s < 4; ++s) mbar_init(&res_bar[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  pdl_wait(); pdl_trigger();   // barriers are set up; nothing above touched global memory (common.cuh)

  if (warp < 4) {
    regs_producer();
    if (warp != 0) return;
    const bool issue = elect_one();
    if (BN == 256 && p.halo) produce_halo(p, smem, full_bar, empty_bar, wfull_bar, wempty_bar, issue);
    else produce_taps<BN>(p, smem, full_bar, empty_bar, issue);
  } else {
    regs_consumer();
    const int g = (warp >> 2) - 1, wq = warp & 3;   // MMA warpgroup and warp within it
    if (p.f16) gemm_tc_mma<BN, true>(p, smem_u32(smem), g, wq, lane);
    else gemm_tc_mma<BN, false>(p, smem_u32(smem), g, wq, lane);
  }
}

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

}  // namespace

int encode_map(CUtensorMap* tm, const float* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
               const uint32_t* box, const uint32_t* elem_strides, bool f16, CUtensorMapSwizzle swizzle) {
  auto fn = get_encode_fn();
  B200_REQUIRE(fn != nullptr, "gemm_tc: cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "gemm_tc: operand base %p not 16-byte aligned", (const void*)base);
  uint32_t estr[5] = {1, 1, 1, 1, 1};
  if (elem_strides) for (int i = 0; i < rank; ++i) estr[i] = elem_strides[i];
  CUresult r = fn(tm, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<float*>(base), dims,
                  strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
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

struct TcGemmPlan { TcParams prm; int bn; };

// Opt in to the large dynamic shared-memory carve-out once, outside any stream capture.
static int tc_configure() {
  static bool configured = false;
  if (configured) return 0;
  B200_CHECK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemLayout<256>::TOTAL));
  B200_CHECK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemLayout<128>::TOTAL));
  configured = true;
  return 0;
}

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
  if (d.epi.round_tf32 < 0 || d.epi.round_tf32 > 2) return fail("store format must be 0 (fp32), 1 (TF32 grid) or 2 (fp16)");
  if (d.epi.round_tf32 == 2 && d.epi.ld_out % 8) return fail("fp16 output pitch must be a multiple of 8 elements");
  // the epilogue's TMA store and residual load
  if (!d.epi.out_nchw && (reinterpret_cast<uintptr_t>(d.epi.out) & 15)) return fail("output must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(d.epi.residual) & 15) return fail("residual must be 16-byte aligned");
  if (d.split && d.f16) return fail("split TF32 takes TF32 operands, not fp16");
  if (d.split && (!d.a1_lo || (d.a2 && !d.a2_lo) || (d.a3 && !d.a3_lo) || (d.a4 && !d.a4_lo) || !d.w_lo || (d.a3 && !d.w2_lo)))
    return fail("split TF32 needs the lo twin of every operand");
  return true;
}

// 'same'-padded stride-1 3x3 filters on 16- or 32-pixel-wide images, read at their output size: the shapes that have a
// halo form.
static bool has_halo_shape(const TcGemmDesc& d) {
  return d.conv && d.taps == 9 && !d.valid_pad && d.stride != 2 && (d.W == 16 || d.W == 32) && (d.Hin == 0 || d.Hin == d.H) &&
         (d.Win == 0 || d.Win == d.W);
}

struct TcForm { int bn; bool swap, halo, chunk_major; };   // tile columns, swapped operands, halo mainloop, K order

static TcForm choose_form(const TcGemmDesc& d) {
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
  // (image rows wider than 128 pixels - the 256..1024-pixel families - are cut into 128-pixel boxes like any other: the
  // two boxes of a 256-pixel tile are then two halves of one row or of consecutive rows)
  const bool halo_shape = has_halo_shape(d);
  const long long Mtot = (long long)d.nimg * d.H * d.W;
  TcForm f;
  f.swap = d.conv && d.stride != 2 && (d.N_total % 256 != 0 || d.taps == 1 || halo_shape) && (d.H * d.W) % 256 == 0 &&
           (d.W <= BM || d.W % BM == 0) && Mtot % 256 == 0 && d.epi.rows_per_img % 256 == 0;
  f.bn = f.swap || d.N_total % 256 == 0 ? 256 : 128;
  if (!f.swap && f.bn == 256) {
    const long long m_tiles = d.conv ? (Mtot + BM - 1) / BM : (long long)d.nbatch * ((d.M_per_batch + BM - 1) / BM);
    if (m_tiles * (d.N_total / 256) <= num_sms() / 2) f.bn = 128;
  }
  // Every launch of a shape that has a halo form walks K in that form's order, swapped or row-major, halo on or off: the
  // A/B of the two mainloops is bit-identical, and a row-major launch of such a shape (one the swapped form does not
  // take) adds the same products in the same order.  The halo form itself needs the swapped tile: 256 pixels, whole
  // rows of ONE image - 3 loads of (rows + 2) x W pixels per channel chunk instead of 9 loads of rows x W, as the plain
  // form is bound by the L2 -> SM fill rate, not the tensor pipe.
  f.chunk_major = halo_shape && (d.H * d.W) % (f.swap ? 256 : BM) == 0;
  f.halo = f.chunk_major && f.swap && !d.no_halo;
  return f;
}

// TMA box [channels, W, rows, images] of a 128-pixel tile: part of an image row, whole rows, or whole images.
static std::array<uint32_t, 4> pixel_box(int H, int W, int bke) {
  if (H * W >= BM) return {(uint32_t)bke, (uint32_t)std::min(W, BM), (uint32_t)(BM / std::min(W, BM)), 1};
  return {(uint32_t)bke, (uint32_t)W, (uint32_t)H, (uint32_t)(BM / (H * W))};
}

int tc_gemm_plan_create(const TcGemmDesc& d, TcGemmPlan** out) {
  const char* why = nullptr;
  B200_REQUIRE(tc_gemm_supported(d, &why), "gemm_tc: unsupported shape: %s", why ? why : "?");
  if (int r = tc_configure()) return r;
  const TcForm form = choose_form(d);
  B200_REQUIRE(!d.epi.out_nchw || form.swap, "gemm_tc: the NCHW head needs the swapped-operand form");
  TcParams p;
  memset(&p, 0, sizeof(p));
  p.conv = d.conv; p.H = d.conv ? d.H : 1; p.W = d.conv ? d.W : 1; p.taps = d.taps;
  p.S = d.taps == 9 ? 3 : 1; p.pad = (d.taps == 9 && !d.valid_pad) ? 1 : 0;
  p.stride = d.stride == 2 ? 2 : 1;
  p.f16 = d.f16 ? 1 : 0;
  p.nphase = d.split ? 3 : 1;
  p.swap = form.swap; p.halo = form.halo; p.chunk_major = form.chunk_major;
  p.qstats = d.qstats;

  const bool f16 = d.f16 != 0;
  const int bke = f16 ? 64 : BKE;            // elements per 128-byte K step
  const uint64_t es = f16 ? 2 : 4;           // operand element size
  p.bke = bke;
  p.kchunks[0] = d.C1 / bke; p.kchunks[1] = d.a2 ? d.C2 / bke : 0; p.wcol[1] = d.C1;
  p.N_total = d.N_total; p.tiles_n = form.swap ? d.N_total / 128 : d.N_total / form.bn;
  p.a_batch_rows = d.a_batch_rows; p.w_batch_rows = d.w_batch_rows;
  p.epi = d.epi;

  // every map is encoded over the hi operand and, in split-TF32 plans, once more over its lo twin
  auto encode_pair = [&](CUtensorMap (&tm)[2], const float* hi, const float* lo, int rank, const uint64_t* dims,
                         const uint64_t* str, const uint32_t* box, const uint32_t* estr) {
    if (int r = encode_map(&tm[0], hi, rank, dims, str, box, estr, f16)) return r;
    if (!d.split) { tm[1] = tm[0]; return 0; }
    return encode_map(&tm[1], lo, rank, dims, str, box, estr, f16);
  };
  // an NHWC activation [nimg][H][W][C]
  auto encode_nhwc = [&](CUtensorMap (&tm)[2], const float* hi, const float* lo, int C, int H, int W, const uint32_t* box,
                         const uint32_t* estr) {
    const uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)d.nimg};
    const uint64_t str[3] = {(uint64_t)C * es, (uint64_t)W * C * es, (uint64_t)H * W * C * es};
    return encode_pair(tm, hi, lo, 4, dims, str, box, estr);
  };
  const float* const src_hi[4] = {d.a1, d.a2, d.a3, d.a3 ? d.a4 : nullptr};
  const float* const src_lo[4] = {d.a1_lo, d.a2_lo, d.a3_lo, d.a4_lo};
  const int src_c[4] = {d.C1, d.C2, d.C3, d.C4};

  if (d.conv) {
    const long long M = (long long)d.nimg * d.H * d.W;
    p.nbatch = 1; p.M_per_batch = (int)M; p.tiles_m_per_batch = form.swap ? (int)(M / 256) : (int)((M + BM - 1) / BM);
    // stride 2: the box *traverses* 2x as many pixels and TMA keeps every other one
    std::array<uint32_t, 4> box = pixel_box(d.H, d.W, bke);
    box[1] *= p.stride; box[2] *= p.stride;
    const uint32_t estr[4] = {1, (uint32_t)p.stride, (uint32_t)p.stride, 1};
    const int Hin = d.Hin ? d.Hin : d.H, Win = d.Win ? d.Win : d.W;
    for (int s = 0; s < 2; ++s)
      if (int r = src_hi[s] ? encode_nhwc(p.a[s], src_hi[s], src_lo[s], src_c[s], Hin, Win, box.data(), estr) : 0) return r;
  } else {
    p.nbatch = d.nbatch; p.M_per_batch = d.M_per_batch; p.tiles_m_per_batch = (d.M_per_batch + BM - 1) / BM;
    const uint32_t box[4] = {(uint32_t)bke, BM, 1, 1};
    for (int s = 0; s < 2; ++s) {
      if (!src_hi[s]) continue;
      const uint64_t dims[4] = {(uint64_t)src_c[s], (uint64_t)d.a_rows, 1, 1};
      const uint64_t str[3] = {(uint64_t)d.a_ld * es, (uint64_t)d.a_ld * es * d.a_rows, (uint64_t)d.a_ld * es * d.a_rows};
      if (int r = encode_pair(p.a[s], src_hi[s], src_lo[s], 4, dims, str, box, nullptr)) return r;
    }
  }
  if (form.halo) {
    const int rows = 256 / d.W;
    p.halo_dh_bytes = d.W * 128; p.halo_copy_bytes = (rows + 2) * d.W * 128;
    B200_REQUIRE(p.halo_copy_bytes <= HALO_X_BYTES, "gemm_tc: halo copy of %d bytes does not fit its slot", p.halo_copy_bytes);
    const uint32_t box[4] = {(uint32_t)bke, (uint32_t)d.W, (uint32_t)(rows + 2), 1};
    for (int s = 0; s < 2; ++s)
      if (int r = src_hi[s] ? encode_nhwc(p.h[s], src_hi[s], src_lo[s], src_c[s], d.H, d.W, box, nullptr) : 0) return r;
  }
  if (d.a3) {
    // extra 1x1 phase: same pixel box as the main input (stride 1, same spatial size), its own channel counts
    const std::array<uint32_t, 4> box = pixel_box(d.H, d.W, bke);
    for (int s = 2; s < 4; ++s)
      if (int r = src_hi[s] ? encode_nhwc(p.a[s], src_hi[s], src_lo[s], src_c[s], d.H, d.W, box.data(), nullptr) : 0) return r;
    p.kchunks[2] = d.C3 / bke; p.kchunks[3] = d.a4 ? d.C4 / bke : 0; p.wcol[3] = d.C3;
  }
  const uint64_t wdims[2] = {(uint64_t)d.K_total, (uint64_t)d.w_rows};
  const uint64_t wstr[1] = {(uint64_t)(d.w_ld ? d.w_ld : d.K_total) * es};
  const uint32_t wbox[2] = {(uint32_t)bke, (uint32_t)(form.swap ? 128 : form.bn)};
  if (int r = encode_pair(p.w[0], d.w, d.w_lo, 2, wdims, wstr, wbox, nullptr)) return r;
  if (d.a3) {
    const uint64_t K3 = (uint64_t)d.C3 + (d.a4 ? d.C4 : 0);
    const uint64_t dims2[2] = {K3, (uint64_t)d.N_total};
    const uint64_t str2[1] = {K3 * es};
    if (int r = encode_pair(p.w[1], d.w2, d.w2_lo, 2, dims2, str2, wbox, nullptr)) return r;
  }
  // staged epilogue: the output and the residual as [rows][N_total] matrices of pitch ld_out / ld_res, in the epilogue's
  // boxes (32 columns x 64 rows, or x 32 pixels in the swapped form); rows past M and columns past N are clipped
  if (!d.epi.out_nchw) {
    const uint64_t rows = d.conv ? (uint64_t)d.nimg * d.H * d.W : (uint64_t)d.nbatch * d.M_per_batch;
    const uint64_t dims[2] = {(uint64_t)d.N_total, rows};
    const uint32_t box[2] = {32, form.swap ? 32u : 64u};
    const bool oh = d.epi.round_tf32 == 2;
    const uint64_t ostr[1] = {(uint64_t)d.epi.ld_out * (oh ? 2 : 4)};
    if (int r = encode_map(&p.out_map, d.epi.out, 2, dims, ostr, box, nullptr, oh, oh ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B))
      return r;
    if (d.epi.residual) {
      const uint64_t rstr[1] = {(uint64_t)d.epi.ld_res * 4};
      if (int r = encode_map(&p.res_map, d.epi.residual, 2, dims, rstr, box, nullptr, false)) return r;
    }
  }
  // the maps the plan does not have (the kernel never reads them) copy a[0], or w[0]
  for (int s = 1; s < 4; ++s)
    if (!src_hi[s]) memcpy(p.a[s], p.a[0], sizeof(p.a[0]));
  for (int s = 0; s < 2; ++s)
    if (!form.halo || !src_hi[s]) memcpy(p.h[s], p.a[0], sizeof(p.h[s]));
  if (!d.a3) memcpy(p.w[1], p.w[0], sizeof(p.w[1]));
  p.total_tiles = (long long)p.nbatch * p.tiles_m_per_batch * p.tiles_n;
  *out = new TcGemmPlan{p, form.bn};
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
