// Few-channel 3x3 / 1x1 stride-1 convolutions (Cin a multiple of 16, Cout 16 / 32 / 64) on NHWC fp32 tensors.
//
// These are the 1024..128-pixel levels of the high-resolution family (nf = 16: 16, 32, 64 channels;
// /root/reference/configs/ve/ffhq_ncsnpp_continuous.py:71-94).  Their output tiles are far too narrow for the
// wgmma tiling (N = 128 / 256 columns, K steps of 32 TF32 elements) and they are memory-bound by construction:
// 16 -> 16 channels is 36 FLOP per byte.  What they need is enough contraction rate to stay at the HBM roofline,
// which the strict-fp32 CUDA-core kernel (conv_simt.cu: 6 - 28 TFLOP/s on these shapes, 73 % of an FFHQ-1024
// evaluation) does not have and warp-level TF32 MMAs do:
//   * a CTA owns an 8 x 32 pixel output tile of one image; it stages the (8+2) x (32+2) pixel halo of one
//     16-channel slab, rounded to the TF32 grid on the way in (one RN rounding per operand, like every TF32 layer of
//     the engine), and the [tap][Cout][16] slab of the packed weights;
//   * warp w computes row w of the tile: two m16 pixel blocks x Cout/8 n8 blocks, K walked as (tap, slab, k8);
//   * all fragment loads are 128-bit: a lane reads channels 4t..4t+3 of its pixel / output row and the MMA's k slots
//     are *defined* as (t -> 4t+2s, t+4 -> 4t+2s+1) for k8 step s.  The sum over k does not care about the order as
//     long as A and B agree, so one LDS.128 feeds two MMAs and no shared-memory padding is needed (a quarter warp
//     reads 32 consecutive words);
//   * two persistent CTAs per SM (<= 81 KB shared, <= 128 registers); the next 16-channel input slab arrives by
//     cp.async while the current one is multiplied.
// The epilogue is conv_simt's: + bias + per-image row vector + residual, * scale, optional TF32-grid store.
#include "kernels.h"

namespace b200 {

namespace {

constexpr int LC_TH = 8, LC_TW = 32, LC_KC = 16, LC_THREADS = 256;

__device__ __forceinline__ void mma_tf32_m16n8k8(float (&d)[4], float a0, float a1, float a2, float a3, float b0, float b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(__float_as_uint(a0)), "r"(__float_as_uint(a1)), "r"(__float_as_uint(a2)), "r"(__float_as_uint(a3)),
                 "r"(__float_as_uint(b0)), "r"(__float_as_uint(b1)));
}

__device__ __forceinline__ float4 round4_tf32(float4 v) {
  v.x = round_tf32(v.x); v.y = round_tf32(v.y); v.z = round_tf32(v.z); v.w = round_tf32(v.w);
  return v;
}

__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gsrc, bool valid) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  const int bytes = valid ? 16 : 0;           // src-size 0: the 16 destination bytes are zero-filled (the padding ring)
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(d), "l"(gsrc), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// Persistent CTAs: a CTA walks (tile, 16-channel slab) work items.  The input slab of item i+1 is in flight (cp.async into
// the other buffer) while item i's MMAs run; a thread rounds the 16-byte pieces it copied itself to the TF32 grid in place
// before the barrier that publishes the buffer.  Single-slab layers (Cin = 16) load their weights once per CTA; the
// others re-stage the [tap][Cout][16] weight slab of each item from L2.
template <int TAPS, int NB>
__global__ void __launch_bounds__(LC_THREADS, 2) conv_lowc_kernel(const SimtConv p, int num_tiles, int w_slabs) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  constexpr int HALO = TAPS == 9 ? 1 : 0;
  constexpr int PH = LC_TH + 2 * HALO, PW = LC_TW + 2 * HALO;
  constexpr int N = NB * 8;
  constexpr int A_FLOATS = PH * PW * LC_KC;
  constexpr int A_PIECES = PH * PW * 4;                                   // 16-byte pieces of one input slab
  constexpr int A_ITERS = (A_PIECES + LC_THREADS - 1) / LC_THREADS;
  constexpr int B_PIECES = TAPS * N * 4;
  extern __shared__ __align__(16) float lc_smem[];
  float* sA0 = lc_smem;                         // 2 x [PH][PW][16]  input slab with halo
  float* sB = lc_smem + 2 * A_FLOATS;           // [TAPS][N][16]     weight slab, TF32 grid

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int tiles_x = p.W / LC_TW, tiles_y = p.H / LC_TH, tiles_img = tiles_x * tiles_y;
  const int Cin = p.C1 + p.C2, slabs = Cin / LC_KC;
  const int ld1 = (int)(p.ld1 ? p.ld1 : p.C1), ld2 = (int)(p.ld2 ? p.ld2 : p.C2), wld = (int)(p.w_ld ? p.w_ld : Cin);
  const int my_tiles = (int)blockIdx.x < num_tiles ? (num_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  const long long img_pix = (long long)p.H * p.W;

  // weight slab `slab` ([tap][N][16 channels]) into dst; piece e = 4 floats of row e/4 (= tap * N + n) of the [tap][N][Cin] weights
  auto stage_weights = [&](int slab, float* dst) {
    for (int e = tid; e < B_PIECES; e += LC_THREADS) {
      const float4 v = round4_tf32(__ldg(reinterpret_cast<const float4*>(p.w + (e >> 2) * wld + slab * LC_KC + 4 * (e & 3))));
      *reinterpret_cast<float4*>(dst + 4 * e) = v;
    }
  };
  // all slabs stay resident when they fit the launch's shared memory (w_slabs == slabs: staged once per CTA, e.g. 32 -> 32
  // channels = 36 KB); otherwise one slab at a time, re-staged from L2 for every work item
  const bool resident = w_slabs == slabs;
  // copies of one (tile, slab) work item into `dst`: piece e = floats 4e..4e+3 of the [PH][PW][16] slab.  A thread's
  // pieces are e = tid + 256 k: channel quad q = tid & 3 for all of them, slab pixel (tid >> 2) + 64 k.
  const int q4 = 4 * (tid & 3), pix0 = tid >> 2;
  auto issue = [&](int img, int ty, int tx, int slab, float* dst) {
    const int c0 = slab * LC_KC;
    const bool one = c0 < p.C1;
    const int ld = one ? ld1 : ld2;
    const int y0 = ty * LC_TH - HALO, x0 = tx * LC_TW - HALO;
    // (tile origin may lie one pixel outside the image: only dereferenced for in-bounds pixels)
    const float* src = (one ? p.x1 + c0 : p.x2 + (c0 - p.C1)) + (img * img_pix + (long long)y0 * p.W + x0) * ld + q4;
    float* d = dst + 4 * tid;
    if (HALO == 0 || (ty > 0 && ty < tiles_y - 1 && tx > 0 && tx < tiles_x - 1)) {
#pragma unroll
      for (int k = 0; k < A_ITERS; ++k) {
        const int pix = pix0 + 64 * k;
        if (k < A_ITERS - 1 || pix < PH * PW) {
          const int py = pix / PW, px = pix - py * PW;
          cp_async16(d + 4 * LC_THREADS * k, src + (py * p.W + px) * ld, true);
        }
      }
    } else {
#pragma unroll
      for (int k = 0; k < A_ITERS; ++k) {
        const int pix = pix0 + 64 * k;
        if (k < A_ITERS - 1 || pix < PH * PW) {
          const int py = pix / PW, px = pix - py * PW, iy = y0 + py, ix = x0 + px;
          const bool ok = iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
          cp_async16(d + 4 * LC_THREADS * k, ok ? src + (py * p.W + px) * ld : p.x1, ok);
        }
      }
    }
    cp_async_commit();
  };
  auto decompose = [&](int tile, int& img, int& ty, int& tx) {
    img = tile / tiles_img; const int r = tile - img * tiles_img; ty = r / tiles_x; tx = r - ty * tiles_x;
  };

  float acc[2][NB][4];
#pragma unroll
  for (int mb = 0; mb < 2; ++mb)
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mb][nb][i] = 0.f;

  // GroupNorm quad sums of the output (p.qstats): per-CTA fp64 accumulators [N/4][2] for the image the CTA is working
  // on, flushed to global memory when the image changes and at the end (a CTA's tiles come in image order)
  __shared__ double sQ[2 * NB * 2];
  int q_img = -1;
  auto flush_stats = [&](int next_img) {         // CTA-uniform call sites only
    __syncthreads();
    if (tid < 2 * NB * 2) {
      if (q_img >= 0 && sQ[tid] != 0.0) atomicAdd(p.qstats + ((long long)q_img * (2 * NB) * 2 + tid), sQ[tid]);
      sQ[tid] = 0.0;
    }
    __syncthreads();
    q_img = next_img;
  };

  int img = 0, ty = 0, tx = 0, nimg = 0, nty = 0, ntx = 0;     // current / next tile of this CTA
  if (my_tiles > 0) { decompose(blockIdx.x, img, ty, tx); issue(img, ty, tx, 0, sA0); }
  if (resident) for (int sl = 0; sl < slabs; ++sl) stage_weights(sl, sB + sl * (B_PIECES * 4));
  int buf = 0;
  for (int k = 0, tile = blockIdx.x; k < my_tiles; ++k, tile += gridDim.x, img = nimg, ty = nty, tx = ntx) {
    if (k + 1 < my_tiles) decompose(tile + gridDim.x, nimg, nty, ntx);
    for (int slab = 0; slab < slabs; ++slab, buf ^= 1) {
      float* sA = sA0 + buf * A_FLOATS;
      {                                            // next work item: the next slab of this tile, else the next tile's first
        const bool same = slab + 1 < slabs;
        if (same || k + 1 < my_tiles) {
          issue(same ? img : nimg, same ? ty : nty, same ? tx : ntx, same ? slab + 1 : 0, sA0 + (buf ^ 1) * A_FLOATS);
          cp_async_wait<1>();
        } else {
          cp_async_wait<0>();
        }
      }
      if (!p.gn_scale) {
#pragma unroll
        for (int kk = 0; kk < A_ITERS; ++kk) {     // round this thread's own pieces of the current item
          const int e = tid + kk * LC_THREADS;
          if (e < A_PIECES) {
            float4* q4p = reinterpret_cast<float4*>(sA + 4 * e);
            *q4p = round4_tf32(*q4p);
          }
        }
      } else {
        // GroupNorm + SiLU on load: y = fma(x, scale, shift) of this thread's channel quad (the same four channels for
        // all of its pieces), SiLU, TF32 rounding - the arithmetic of gn_apply_stream_kernel's TF32-grid mode.  The
        // padding ring must stay zero AFTER the transform (the reference pads the normalised tensor), so border tiles
        // re-derive which pieces lie outside the image.
        const int cidx = img * Cin + slab * LC_KC + q4;
        const float4 sc = __ldg(reinterpret_cast<const float4*>(p.gn_scale + cidx));
        const float4 sh = __ldg(reinterpret_cast<const float4*>(p.gn_shift + cidx));
        const bool interior = HALO == 0 || (ty > 0 && ty < tiles_y - 1 && tx > 0 && tx < tiles_x - 1);
        const int y0 = ty * LC_TH - HALO, x0 = tx * LC_TW - HALO;
#pragma unroll
        for (int kk = 0; kk < A_ITERS; ++kk) {
          const int pix = pix0 + 64 * kk;
          if (kk < A_ITERS - 1 || pix < PH * PW) {
            float4* q4p = reinterpret_cast<float4*>(sA + 4 * (tid + kk * LC_THREADS));
            float4 v = *q4p;
            v.x = fmaf(v.x, sc.x, sh.x); v.y = fmaf(v.y, sc.y, sh.y); v.z = fmaf(v.z, sc.z, sh.z); v.w = fmaf(v.w, sc.w, sh.w);
            if (p.gn_act) { v.x = silu_fast(v.x); v.y = silu_fast(v.y); v.z = silu_fast(v.z); v.w = silu_fast(v.w); }
            if (!interior) {
              const int py = pix / PW, px = pix - py * PW, iy = y0 + py, ix = x0 + px;
              if (!(iy >= 0 && iy < p.H && ix >= 0 && ix < p.W)) v = make_float4(0.f, 0.f, 0.f, 0.f);
            }
            *q4p = round4_tf32(v);
          }
        }
      }
      if (!resident) stage_weights(slab, sB);      // (the barrier that closed the previous item freed sB)
      const float* sBs = resident ? sB + slab * (B_PIECES * 4) : sB;
      __syncthreads();

#pragma unroll
      for (int tap = 0; tap < TAPS; ++tap) {
        const int dy = TAPS == 9 ? tap / 3 : 0, dx = TAPS == 9 ? tap % 3 : 0;
        float4 av[2][2];
#pragma unroll
        for (int mb = 0; mb < 2; ++mb)
#pragma unroll
          for (int h = 0; h < 2; ++h)
            av[mb][h] = *reinterpret_cast<const float4*>(sA + ((warp + dy) * PW + mb * 16 + g + 8 * h + dx) * LC_KC + 4 * t);
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) {
          const float4 bv = *reinterpret_cast<const float4*>(sBs + (tap * N + nb * 8 + g) * LC_KC + 4 * t);
#pragma unroll
          for (int mb = 0; mb < 2; ++mb) {
            mma_tf32_m16n8k8(acc[mb][nb], av[mb][0].x, av[mb][1].x, av[mb][0].y, av[mb][1].y, bv.x, bv.y);
            mma_tf32_m16n8k8(acc[mb][nb], av[mb][0].z, av[mb][1].z, av[mb][0].w, av[mb][1].w, bv.z, bv.w);
          }
        }
      }
      __syncthreads();                             // this buffer and sB may be overwritten from here on
    }

    // ---- epilogue: lane (g, t) holds pixels g / g+8 of each m16 block and output channels 2t, 2t+1 of each n8 block ----
    const Epilogue& e = p.epi;
    if (p.qstats && img != q_img) flush_stats(img);
    float qs[NB], qq[NB];
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) { qs[nb] = 0.f; qq[nb] = 0.f; }
    const int oy = ty * LC_TH + warp;
    float2 add[NB];                                // bias + per-image row vector of this lane's channels
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) {
      const int n = nb * 8 + 2 * t;
      add[nb] = make_float2(0.f, 0.f);
      if (e.bias) { const float2 b = __ldg(reinterpret_cast<const float2*>(e.bias + n)); add[nb].x += b.x; add[nb].y += b.y; }
      if (e.rowvec) { const float2 rv = __ldg(reinterpret_cast<const float2*>(e.rowvec + img * e.rowvec_ld + n)); add[nb].x += rv.x; add[nb].y += rv.y; }
    }
#pragma unroll
    for (int mb = 0; mb < 2; ++mb)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int ox = tx * LC_TW + mb * 16 + g + 8 * h;
        const long long gm = (img * img_pix + (long long)oy * p.W + ox);
        float* orow = e.out + gm * e.ld_out + 2 * t;
        const float* rrow = e.residual ? e.residual + gm * e.ld_res + 2 * t : nullptr;
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) {
          float v0 = acc[mb][nb][2 * h] + add[nb].x, v1 = acc[mb][nb][2 * h + 1] + add[nb].y;
          acc[mb][nb][2 * h] = 0.f; acc[mb][nb][2 * h + 1] = 0.f;
          if (rrow) { const float2 rr = __ldg(reinterpret_cast<const float2*>(rrow + nb * 8)); v0 += rr.x; v1 += rr.y; }
          v0 *= e.scale; v1 *= e.scale;
          if (e.round_tf32) { v0 = round_tf32(v0); v1 = round_tf32(v1); }
          *reinterpret_cast<float2*>(orow + nb * 8) = make_float2(v0, v1);
          qs[nb] += v0 + v1; qq[nb] = fmaf(v0, v0, fmaf(v1, v1, qq[nb]));
        }
      }
    if (p.qstats) {
      // lane (g, t): channels 2t, 2t+1 of each n8 block -> lanes t = 0,1 share quad 2nb, t = 2,3 quad 2nb+1; fold the
      // lane pair, then the eight pixel lanes g; lanes 0 and 2 add the warp's 32-pixel totals to the CTA accumulators
#pragma unroll
      for (int nb = 0; nb < NB; ++nb) {
        float a = qs[nb], b = qq[nb];
        a += __shfl_xor_sync(0xffffffffu, a, 1);  b += __shfl_xor_sync(0xffffffffu, b, 1);
        a += __shfl_xor_sync(0xffffffffu, a, 4);  b += __shfl_xor_sync(0xffffffffu, b, 4);
        a += __shfl_xor_sync(0xffffffffu, a, 8);  b += __shfl_xor_sync(0xffffffffu, b, 8);
        a += __shfl_xor_sync(0xffffffffu, a, 16); b += __shfl_xor_sync(0xffffffffu, b, 16);
        if (lane == 0 || lane == 2) {
          const int quad = 2 * nb + (lane >> 1);
          atomicAdd(&sQ[2 * quad], (double)a); atomicAdd(&sQ[2 * quad + 1], (double)b);
        }
      }
    }
  }
  if (p.qstats) flush_stats(-1);
}

int lc_num_sms() {
  static int n = 0;
  if (!n) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); if (n <= 0) n = 132; }
  return n;
}

template <int TAPS, int NB>
int launch_lowc(const SimtConv& p, cudaStream_t st) {
  constexpr int HALO = TAPS == 9 ? 1 : 0;
  constexpr int a_bytes = 2 * (LC_TH + 2 * HALO) * (LC_TW + 2 * HALO) * LC_KC * (int)sizeof(float);
  constexpr int slab_bytes = TAPS * NB * 8 * LC_KC * (int)sizeof(float);
  constexpr int max_smem = a_bytes + 36 * 1024;   // two CTAs per SM: <= 43.5 + 36 KB each (one 64-channel 3x3 slab is 36 KB)
  const int slabs = (p.C1 + p.C2) / LC_KC;
  const int w_slabs = (a_bytes + slabs * slab_bytes <= max_smem) ? slabs : 1;
  const int smem = a_bytes + w_slabs * slab_bytes;
  static bool configured = false;   // one attribute call per instantiation (same value every time: benign if raced)
  if (!configured) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(conv_lowc_kernel<TAPS, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    configured = true;
  }
  const long long tiles = (long long)p.nbatch * (p.H / LC_TH) * (p.W / LC_TW);
  B200_REQUIRE(tiles > 0 && tiles < (1LL << 30), "conv_lowc: %lld tiles", tiles);
  const int grid = (int)std::min<long long>(tiles, 2LL * lc_num_sms());
  launch_kernel(conv_lowc_kernel<TAPS, NB>, dim3(grid), dim3(LC_THREADS), smem, st, p, (int)tiles, w_slabs);
  B200_CHECK_LAUNCH();
  return 0;
}

bool aligned(const void* q, uintptr_t a) { return (reinterpret_cast<uintptr_t>(q) & (a - 1)) == 0; }

}  // namespace

bool conv_lowc_supported(const SimtConv& p) {
  const bool geom = (p.R == 3 && p.S == 3 && p.pad == 1) || (p.R == 1 && p.S == 1 && p.pad == 0);
  const long long ld1 = p.ld1 ? p.ld1 : p.C1, ld2 = p.ld2 ? p.ld2 : p.C2, wld = p.w_ld ? p.w_ld : p.C1 + p.C2;
  return geom && p.stride == 1 && p.dilation <= 1 && !p.in_nchw && p.in_scale == 1.f && p.in_shift == 0.f && p.OH == p.H && p.OW == p.W &&
         p.H % LC_TH == 0 && p.W % LC_TW == 0 && p.C1 > 0 && p.C1 % LC_KC == 0 && p.C2 >= 0 && p.C2 % LC_KC == 0 &&
         (p.N == 16 || p.N == 32 || p.N == 64) && p.a_batched && p.w_batch_stride == 0 && ld1 % 4 == 0 && ld2 % 4 == 0 &&
         wld % 4 == 0 && !p.epi.out_nchw && !p.epi.per_img_div && (p.epi.round_tf32 == 0 || p.epi.round_tf32 == 1) &&
         p.epi.ld_out % 2 == 0 && p.epi.ld_res % 2 == 0 && p.epi.rowvec_ld % 2 == 0;
}

int launch_conv_lowc(const SimtConv& p, cudaStream_t st) {
  B200_REQUIRE(p.x1 && p.w && p.epi.out, "conv_lowc: null operand");
  B200_REQUIRE(conv_lowc_supported(p), "conv_lowc: unsupported shape (C %d+%d -> %d, %dx%d, %dx%d filter)", p.C1, p.C2, p.N, p.H,
               p.W, p.R, p.S);
  B200_REQUIRE((p.x2 != nullptr) == (p.C2 > 0), "conv_lowc: second source / channel count mismatch");
  B200_REQUIRE(aligned(p.qstats, 8), "conv_lowc: quad sums must be 8-byte aligned");
  B200_REQUIRE((p.gn_scale == nullptr) == (p.gn_shift == nullptr) && aligned(p.gn_scale, 16) && aligned(p.gn_shift, 16),
               "conv_lowc: GroupNorm scale and shift come together, 16-byte aligned");
  B200_REQUIRE(aligned(p.x1, 16) && aligned(p.x2, 16) && aligned(p.w, 16) && aligned(p.epi.out, 8) && aligned(p.epi.residual, 8) &&
               aligned(p.epi.bias, 8) && aligned(p.epi.rowvec, 8), "conv_lowc: operands must be 16-byte, epilogue terms 8-byte aligned");
  if (p.R == 3) {
    if (p.N == 16) return launch_lowc<9, 2>(p, st);
    if (p.N == 32) return launch_lowc<9, 4>(p, st);
    return launch_lowc<9, 8>(p, st);
  }
  if (p.N == 16) return launch_lowc<1, 2>(p, st);
  if (p.N == 32) return launch_lowc<1, 4>(p, st);
  return launch_lowc<1, 8>(p, st);
}

}  // namespace b200
