// HBM-bound kernels of the NCSN++ forward: GroupNorm statistics / apply(+SiLU),
// FIR resampling (upfirdn2d), fused bias+activation, row softmax, the
// time-embedding path, layout/packing utilities.
//
// All activations are NHWC fp32 ([image][pixel][channel], channel contiguous) so a
// 128-bit access covers 4 channels of one pixel and a GroupNorm group (4/8/12/16
// channels here) never straddles a float4.
#include "common.cuh"
#include "kernels.h"
#include <cuda_fp16.h>

namespace b200 {

// ============================================================================
// GroupNorm.  Reference semantics: nn.GroupNorm(min(C/4,32), C, eps=1e-6)
// (layerspp.py:67,219,231; ncsnpp.py:226) -> biased variance over (C/G)*H*W.
//
// Statistics are carried as fp64 "quad sums": for every image and every aligned group of 4
// channels the pair (sum x, sum x^2).  Any GroupNorm group of this network (4/8/12/16 channels,
// always quad aligned, possibly straddling the two sources of a U-Net channel concat,
// ncsnpp.py:318) is a sum of 1-4 quads, so a tensor's quad sums serve every consumer.  They are
// produced for free by the tensor-core contraction's epilogue (gemm_tc.cu) for tensors it writes, or
// by gn_quad_stats_kernel below for the rest; gn_apply_kernel turns them into mean / rstd once
// per thread and streams the tensor exactly once (read + write, optional TF32-rounded raw copy).
// ============================================================================
constexpr int GN_THREADS = 384;   // divisible by C/4 for every channel count of the network (32, 64, 96, 128)

__global__ void __launch_bounds__(GN_THREADS) gn_quad_stats_kernel(
    const float* __restrict__ x, int C, int HW_img, double* __restrict__ qsums /* [B][C/4][2] */) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  extern __shared__ double sred[];   // [lanes][Q][2]
  const int Q = C >> 2, b = blockIdx.x;
  // gridDim.y > 1 (few large images: one CTA per image would leave the GPU idle): each CTA sums a slice of the pixels and
  // ADDS its fp64 partials to qsums, which the caller has zeroed (the engine zeroes its whole statistics region per forward)
  const int per = (HW_img + gridDim.y - 1) / gridDim.y, pix0 = blockIdx.y * per;
  const int HW = max(0, min(HW_img, pix0 + per) - pix0);
  const bool accumulate = gridDim.y > 1;
  const float* px = x + ((long long)b * HW_img + pix0) * C;
  if (GN_THREADS % Q == 0) {
    // deterministic: thread owns quad q for pixels lane, lane+L, ...; fixed-order fold over lanes
    const int L = GN_THREADS / Q, q = threadIdx.x % Q, lane = threadIdx.x / Q;
    double s = 0.0, ss = 0.0;
    int pix = lane;
    for (; pix + 3 * L < HW; pix += 4 * L) {
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = __ldg(reinterpret_cast<const float4*>(px + (long long)(pix + u * L) * C + 4 * q));
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        s += ((double)v[u].x + (double)v[u].y) + ((double)v[u].z + (double)v[u].w);
        ss += ((double)v[u].x * v[u].x + (double)v[u].y * v[u].y) + ((double)v[u].z * v[u].z + (double)v[u].w * v[u].w);
      }
    }
    for (; pix < HW; pix += L) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(px + (long long)pix * C + 4 * q));
      s += ((double)v.x + (double)v.y) + ((double)v.z + (double)v.w);
      ss += ((double)v.x * v.x + (double)v.y * v.y) + ((double)v.z * v.z + (double)v.w * v.w);
    }
    sred[(lane * Q + q) * 2] = s; sred[(lane * Q + q) * 2 + 1] = ss;
    __syncthreads();
    if (threadIdx.x < Q) {
      double a = 0.0, c = 0.0;
      for (int l = 0; l < L; ++l) { a += sred[(l * Q + threadIdx.x) * 2]; c += sred[(l * Q + threadIdx.x) * 2 + 1]; }
      double* dst = qsums + ((long long)b * Q + threadIdx.x) * 2;
      if (accumulate) { atomicAdd(dst, a); atomicAdd(dst + 1, c); }
      else { dst[0] = a; dst[1] = c; }
    }
  } else {
    // generic channel counts: shared-memory fp64 atomics
    for (int i = threadIdx.x; i < 2 * Q; i += blockDim.x) sred[i] = 0.0;
    __syncthreads();
    for (long long u = threadIdx.x; u < (long long)HW * Q; u += blockDim.x) {
      const int q = (int)(u % Q);
      const float4 v = __ldg(reinterpret_cast<const float4*>(px + (u / Q) * C + 4 * q));
      atomicAdd(&sred[2 * q], ((double)v.x + (double)v.y) + ((double)v.z + (double)v.w));
      atomicAdd(&sred[2 * q + 1], ((double)v.x * v.x + (double)v.y * v.y) + ((double)v.z * v.z + (double)v.w * v.w));
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * Q; i += blockDim.x) {
      if (accumulate) atomicAdd(&qsums[(long long)b * 2 * Q + i], sred[i]);
      else qsums[(long long)b * 2 * Q + i] = sred[i];
    }
  }
}

int launch_gn_quad_stats(const float* x, int C, int B, int HW, double* qsums, cudaStream_t st, bool qsums_zeroed) {
  B200_REQUIRE(C % 4 == 0, "gn_quad_stats: C=%d must be a multiple of 4", C);
  const int Q = C / 4;
  const size_t smem = (GN_THREADS % Q == 0) ? (size_t)GN_THREADS * 2 * sizeof(double) : (size_t)2 * Q * sizeof(double);
  B200_REQUIRE(smem <= 48 * 1024, "gn_quad_stats: C=%d too large", C);
  // few, large images (high-resolution networks at small batch): several CTAs per image, accumulating into zeroed sums
  int splits = 1;
  if (qsums_zeroed && B < 296 && HW >= 4096) splits = (int)std::min<long long>(std::min<long long>(512, HW / 1024), (592 + B - 1) / B);
  launch_kernel(gn_quad_stats_kernel, dim3(B, splits), dim3(GN_THREADS), smem, st, x, C, HW, qsums);
  B200_CHECK_LAUNCH();
  return 0;
}

// mean / rstd of the group containing concat-channel c0 from the quad sums of the two sources
__device__ __forceinline__ float2 group_mean_rstd(const double* __restrict__ q1, int C1, const double* __restrict__ q2, int C2,
                                                  int b, int c0, int cpg, double n, float eps) {
  const int g0 = (c0 / cpg) * cpg;
  double s = 0.0, ss = 0.0;
  for (int c = g0; c < g0 + cpg; c += 4) {
    const double* src = (c < C1) ? q1 + ((long long)b * (C1 >> 2) + (c >> 2)) * 2
                                 : q2 + ((long long)b * (C2 >> 2) + ((c - C1) >> 2)) * 2;
    s += src[0]; ss += src[1];
  }
  const double mean = s / n;
  double var = ss / n - mean * mean;
  if (var < 0.0) var = 0.0;
  return make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
}

// y = v * sc + sh with sc = rstd * gamma, sh = beta - mean * sc folded per channel by the caller
__device__ __forceinline__ float4 gn_affine4(float4 v, float4 sc, float4 sh, int act) {
  float4 o;
  o.x = fmaf(v.x, sc.x, sh.x); o.y = fmaf(v.y, sc.y, sh.y); o.z = fmaf(v.z, sc.z, sh.z); o.w = fmaf(v.w, sc.w, sh.w);
  if (act) { o.x = silu_fast(o.x); o.y = silu_fast(o.y); o.z = silu_fast(o.z); o.w = silu_fast(o.w); }
  return o;
}
__device__ __forceinline__ float4 gn_norm4(float4 v, float2 mr, float4 ga, float4 be, int act, int round_out) {
  float4 o;
  o.x = (v.x - mr.x) * mr.y * ga.x + be.x;
  o.y = (v.y - mr.x) * mr.y * ga.y + be.y;
  o.z = (v.z - mr.x) * mr.y * ga.z + be.z;
  o.w = (v.w - mr.x) * mr.y * ga.w + be.w;
  if (act) { o.x = silu_f(o.x); o.y = silu_f(o.y); o.z = silu_f(o.z); o.w = silu_f(o.w); }
  (void)round_out;   // the store applies the operand mode (store_operand4)
  return o;
}

// grid = (pixel splits, images).  blockDim % (C/4) == 0: a thread keeps one channel quad (so its
// group statistics, gamma and beta are loaded once) and walks pixels with 4 loads in flight.
template <bool XH>   // XH: x1 holds fp16 elements (the mid-block conv output in fp16 operand mode)
__global__ void __launch_bounds__(GN_THREADS) gn_apply_kernel(
    const float* __restrict__ x1, int C1, const float* __restrict__ x2, int C2,
    const double* __restrict__ q1, const double* __restrict__ q2,
    const float* __restrict__ gamma, const float* __restrict__ beta,
    int HW, int G, float eps, int act, int round_out, float* __restrict__ y, float* __restrict__ raw) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const int C = C1 + C2, Q = C >> 2, cpg = C / G, b = blockIdx.y;
  const int per = (HW + gridDim.x - 1) / gridDim.x;
  const int p0 = blockIdx.x * per, p1 = min(HW, p0 + per);
  const double n = (double)HW * cpg;
  const long long ib = (long long)b * HW;
  if (blockDim.x % Q == 0) {
    const int L = blockDim.x / Q, c0 = (threadIdx.x % Q) << 2, lane = threadIdx.x / Q;
    const bool first = c0 < C1;
    const float* src = first ? x1 + ib * C1 + c0 : x2 + ib * C2 + (c0 - C1);
    const int Cs = first ? C1 : C2;
    // XH: 8-byte fp16 loads, widened here (single-source launches only, checked by the launcher)
    const uint16_t* srch = reinterpret_cast<const uint16_t*>(x1) + ib * C1 + c0;
    auto load4 = [&](int px) -> float4 {
      if (XH) {
        const uint2 u = __ldg(reinterpret_cast<const uint2*>(srch + (long long)px * Cs));
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
        const float2 b2 = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
        return make_float4(a.x, a.y, b2.x, b2.y);
      }
      return __ldg(reinterpret_cast<const float4*>(src + (long long)px * Cs));
    };
    // The first batch of loads is issued BEFORE the (fp64 divide / sqrt) statistics so that their latency hides it.
    constexpr int U = 4;
    float4 v[U];
    int pix = p0 + lane;
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (pix + u * L < p1) v[u] = load4(pix + u * L);
    const float2 mr = group_mean_rstd(q1, C1, q2, C2, b, c0, cpg, n, eps);
    const float4 ga = __ldg(reinterpret_cast<const float4*>(gamma + c0));
    const float4 be = __ldg(reinterpret_cast<const float4*>(beta + c0));
    const bool fast = round_out != 0;       // the stored value keeps 11 significand bits: approximate SiLU is exact enough
    const float4 sc = make_float4(mr.y * ga.x, mr.y * ga.y, mr.y * ga.z, mr.y * ga.w);
    const float4 sh = make_float4(fmaf(-mr.x, sc.x, be.x), fmaf(-mr.x, sc.y, be.y), fmaf(-mr.x, sc.z, be.z), fmaf(-mr.x, sc.w, be.w));
    while (pix < p1) {
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (pix + u * L < p1) {
          const long long o = (ib + pix + u * L) * C + c0;
          store_operand4(y, o, fast ? gn_affine4(v[u], sc, sh, act) : gn_norm4(v[u], mr, ga, be, act, round_out), round_out);
          if (raw) store_operand4(raw, o, v[u], round_out);
        }
      }
      pix += U * L;
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (pix + u * L < p1) v[u] = load4(pix + u * L);
    }
  } else {
    for (long long u = (long long)p0 * Q + threadIdx.x; u < (long long)p1 * Q; u += blockDim.x) {
      const int pix = (int)(u / Q), c0 = (int)(u % Q) << 2;
      const float4 v = (c0 < C1) ? __ldg(reinterpret_cast<const float4*>(x1 + (ib + pix) * C1 + c0))
                                 : __ldg(reinterpret_cast<const float4*>(x2 + (ib + pix) * C2 + (c0 - C1)));
      const float2 mr = group_mean_rstd(q1, C1, q2, C2, b, c0, cpg, n, eps);
      const float4 ga = __ldg(reinterpret_cast<const float4*>(gamma + c0));
      const float4 be = __ldg(reinterpret_cast<const float4*>(beta + c0));
      const long long o = (ib + pix) * C + c0;
      store_operand4(y, o, gn_norm4(v, mr, ga, be, act, round_out), round_out);
      if (raw) store_operand4(raw, o, v, round_out);
    }
  }
}

// ---- lean streaming form -------------------------------------------------------------------------------
// The generic kernel above is instruction-bound (about 26 instructions per element): per-element guards, 64-bit index multiplies, both SiLU paths
// compiled into one loop, and an fp64 divide + square root per thread.  Here every launch property is a template
// parameter, the per-quad scale / shift (rstd*gamma, beta - mean*rstd*gamma) are computed once per CTA into shared
// memory (fp64 only for mean and variance; the reciprocal square root is taken in fp32), the main loop runs
// unguarded over full batches of four pixels with pointer increments, and a short guarded tail finishes.
//   XH: x1 holds fp16;  MODE: store format of y / raw (0 fp32 exact SiLU, 1 TF32 grid, 2 fp16; 1, 2 use the
//   approximate SiLU);  ACT: SiLU;  RAW: also store the rounded copy of the input.
template <bool XH, int MODE, bool ACT, bool RAW>
__global__ void __launch_bounds__(GN_THREADS) gn_apply_stream_kernel(
    const float* __restrict__ x1, int C1, const float* __restrict__ x2, int C2,
    const double* __restrict__ q1, const double* __restrict__ q2,
    const float* __restrict__ gamma, const float* __restrict__ beta,
    int HW, int G, float eps, double inv_n, float* __restrict__ y, float* __restrict__ raw) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  __shared__ float4 s_sc[128], s_sh[128];
  const int C = C1 + C2, Q = C >> 2, cpg = C / G, b = blockIdx.y;
  if (threadIdx.x < Q) {
    const int c0 = threadIdx.x << 2, g0 = (c0 / cpg) * cpg;
    double s = 0.0, ss = 0.0;
    for (int c = g0; c < g0 + cpg; c += 4) {
      const double* src = (c < C1) ? q1 + ((long long)b * (C1 >> 2) + (c >> 2)) * 2
                                   : q2 + ((long long)b * (C2 >> 2) + ((c - C1) >> 2)) * 2;
      s += src[0]; ss += src[1];
    }
    const double mean = s * inv_n;
    const float var = fmaxf((float)(ss * inv_n - mean * mean), 0.f);
    const float rstd = rsqrtf(var + eps), mu = (float)mean;
    const float4 ga = __ldg(reinterpret_cast<const float4*>(gamma + c0));
    const float4 be = __ldg(reinterpret_cast<const float4*>(beta + c0));
    const float4 sc = make_float4(rstd * ga.x, rstd * ga.y, rstd * ga.z, rstd * ga.w);
    s_sc[threadIdx.x] = sc;
    s_sh[threadIdx.x] = make_float4(fmaf(-mu, sc.x, be.x), fmaf(-mu, sc.y, be.y), fmaf(-mu, sc.z, be.z), fmaf(-mu, sc.w, be.w));
  }
  __syncthreads();
  const int per = (HW + gridDim.x - 1) / gridDim.x;
  const int p0 = blockIdx.x * per, p1 = min(HW, p0 + per);
  const int L = blockDim.x / Q, qd = threadIdx.x % Q, lane = threadIdx.x / Q, c0 = qd << 2;
  const float4 sc = s_sc[qd], sh = s_sh[qd];
  const long long ib = (long long)b * HW;
  const bool first = c0 < C1;
  const int Cs = first ? C1 : C2;
  int pix = p0 + lane;
  // element offsets advance by a fixed stride per pixel step
  const float* src = first ? x1 + (ib + pix) * C1 + c0 : x2 + (ib + pix) * C2 + (c0 - C1);
  const uint16_t* srch = reinterpret_cast<const uint16_t*>(x1) + (ib + pix) * C1 + c0;
  const long long sstep = (long long)L * Cs, ostep = (long long)L * C;
  long long o = (ib + pix) * C + c0;
  auto load4 = [&](long long off) -> float4 {
    if (XH) {
      const uint2 u = __ldg(reinterpret_cast<const uint2*>(srch + off));
      const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
      const float2 c2 = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
      return make_float4(a.x, a.y, c2.x, c2.y);
    }
    return __ldg(reinterpret_cast<const float4*>(src + off));
  };
  auto emit = [&](float4 v, long long oo) {
    float4 r;
    r.x = fmaf(v.x, sc.x, sh.x); r.y = fmaf(v.y, sc.y, sh.y); r.z = fmaf(v.z, sc.z, sh.z); r.w = fmaf(v.w, sc.w, sh.w);
    if (ACT) {
      if (MODE == 0) { r.x = silu_f(r.x); r.y = silu_f(r.y); r.z = silu_f(r.z); r.w = silu_f(r.w); }
      else { r.x = silu_fast(r.x); r.y = silu_fast(r.y); r.z = silu_fast(r.z); r.w = silu_fast(r.w); }
    }
    store_operand4(y, oo, r, MODE);
    if (RAW) store_operand4(raw, oo, v, MODE);
  };
  for (; pix + 3 * L < p1; pix += 4 * L) {
    float4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = load4(u * sstep);
#pragma unroll
    for (int u = 0; u < 4; ++u) emit(v[u], o + u * ostep);
    src += 4 * sstep; srch += 4 * sstep; o += 4 * ostep;
  }
  for (; pix < p1; pix += L) {
    emit(load4(0), o);
    src += sstep; srch += sstep; o += ostep;
  }
}

template <bool XH, int MODE>
static void gn_stream_launch(dim3 grid, int threads, cudaStream_t st, int act, bool has_raw, const float* x1, int C1, const float* x2,
                             int C2, const double* q1, const double* q2, const float* gamma, const float* beta, int HW, int G,
                             float eps, double inv_n, float* y, float* raw) {
#define B200_GNS(A, R) launch_kernel(gn_apply_stream_kernel<XH, MODE, A, R>, dim3(grid), dim3(threads), 0, st, x1, C1, x2, C2, q1, q2, gamma, beta, HW, G, eps, inv_n, y, raw)
  if (act) { if (has_raw) B200_GNS(true, true); else B200_GNS(true, false); }
  else { if (has_raw) B200_GNS(false, true); else B200_GNS(false, false); }
#undef B200_GNS
}

int launch_gn_apply(const float* x1, int C1, const float* x2, int C2, const double* q1, const double* q2,
                    const float* gamma, const float* beta, int B, int HW, int G, float eps, int act,
                    int round_out, float* y, float* raw, cudaStream_t st, int x1_f16) {
  const int C = C1 + C2;
  B200_REQUIRE(C % 4 == 0 && C1 % 4 == 0 && C % G == 0 && (C / G) % 4 == 0,
               "gn_apply: C=%d (C1=%d) G=%d must give 4-aligned groups", C, C1, G);
  const int Q = C / 4;
  // Small CTAs (the smallest multiple of the quad count >= 128 threads: 128 or 192 here): finer-grained tail, and
  // several fit in the registers a persistent tensor-core CTA leaves free.
  int threads = GN_THREADS;
  for (int t = 128; t <= GN_THREADS; t += 32) if (t % Q == 0) { threads = t; break; }
  B200_REQUIRE(!x1_f16 || (threads % Q == 0 && !raw), "gn_apply: fp16 input needs the quad-per-thread path (C=%d) and no raw copy", C);
  // aim for ~16 float4 per thread (four 4-deep batches), at least one block per image
  const long long per_img_units = (long long)HW * Q;
  const int work = 16;
  // (few, very large images - the 1024-pixel family at batch 2 - need more than 64 CTAs per image to fill the chip)
  const long long max_splits = std::max<long long>(64, (132LL * 16 + B - 1) / B);
  int splits = (int)std::max<long long>(1, std::min<long long>(per_img_units / ((long long)threads * work), max_splits));
  splits = std::min(splits, HW);
  dim3 grid(splits, B);
  B200_REQUIRE(!x1_f16 || C2 == 0, "gn_apply: fp16 input is single-source");
  if (threads % Q == 0 && Q <= 128 && (!x1_f16 || round_out == 2)) {
    const double inv_n = 1.0 / ((double)HW * (C / G));
    if (x1_f16) gn_stream_launch<true, 2>(grid, threads, st, act, raw != nullptr, x1, C1, x2, C2, q1, q2, gamma, beta, HW, G, eps, inv_n, y, raw);
    else if (round_out == 2) gn_stream_launch<false, 2>(grid, threads, st, act, raw != nullptr, x1, C1, x2, C2, q1, q2, gamma, beta, HW, G, eps, inv_n, y, raw);
    else if (round_out == 1) gn_stream_launch<false, 1>(grid, threads, st, act, raw != nullptr, x1, C1, x2, C2, q1, q2, gamma, beta, HW, G, eps, inv_n, y, raw);
    else gn_stream_launch<false, 0>(grid, threads, st, act, raw != nullptr, x1, C1, x2, C2, q1, q2, gamma, beta, HW, G, eps, inv_n, y, raw);
    B200_CHECK_LAUNCH();
    return 0;
  }
  if (x1_f16) launch_kernel(gn_apply_kernel<true>, dim3(grid), dim3(threads), 0, st, x1, C1, x2, C2, q1, q2, gamma, beta, HW, G, eps, act, round_out, y, raw);
  else launch_kernel(gn_apply_kernel<false>, dim3(grid), dim3(threads), 0, st, x1, C1, x2, C2, q1, q2, gamma, beta, HW, G, eps, act, round_out, y, raw);
  B200_CHECK_LAUNCH();
  return 0;
}

// ---- GroupNorm for group sizes that are not a multiple of four channels -------------------------------------------------
// nn.GroupNorm(min(C/4, 32), C) gives 6 channels per group for C = 192 (the 128+64 concatenation of FFHQ-1024's up
// path): such groups straddle the aligned channel quads the fused statistics are kept in.  These rare layers take a plain
// two-kernel path: per-(image, group) mean / rstd in fp64, then an elementwise apply over the (two-source) tensor.
__global__ void __launch_bounds__(256) gn_generic_stats_kernel(const float* __restrict__ x1, int C1, const float* __restrict__ x2, int C2,
                                                               int HW, int G, double* __restrict__ part) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  // grid (group, image, pixel split): each CTA reduces its pixel range of one group to one (sum, sum of squares) pair
  const int C = C1 + C2, cpg = C / G, g = blockIdx.x, b = blockIdx.y, S = gridDim.z;
  const int per = (HW + S - 1) / S, p0 = blockIdx.z * per, p1 = min(HW, p0 + per);
  double s = 0.0, ss = 0.0;
  for (int pix = p0 + threadIdx.x; pix < p1; pix += blockDim.x) {
    float fs = 0.f, fq = 0.f;                  // <= a few dozen channels per pixel: fp32 inside the pixel, fp64 across pixels
    for (int k = 0; k < cpg; ++k) {
      const int c = g * cpg + k;
      const float v = c < C1 ? __ldg(x1 + ((long long)b * HW + pix) * C1 + c) : __ldg(x2 + ((long long)b * HW + pix) * C2 + (c - C1));
      fs += v; fq = fmaf(v, v, fq);
    }
    s += fs; ss += fq;
  }
  __shared__ double sh[2][8];
  s = warp_sum_d(s); ss = warp_sum_d(ss);
  if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = s; sh[1][threadIdx.x >> 5] = ss; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, q = 0.0;
    for (int w = 0; w < 8; ++w) { a += sh[0][w]; q += sh[1][w]; }
    double* dst = part + (((long long)b * G + g) * S + blockIdx.z) * 2;
    dst[0] = a; dst[1] = q;
  }
}
// one thread per (image, group): fold the pixel-split partials (fixed order: deterministic) into mean / rstd
__global__ void gn_generic_finish_kernel(const double* __restrict__ part, int BG, int S, double n, float eps, float2* __restrict__ mr) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= BG) return;
  double a = 0.0, q = 0.0;
  for (int k = 0; k < S; ++k) { a += part[((long long)i * S + k) * 2]; q += part[((long long)i * S + k) * 2 + 1]; }
  const double mean = a / n;
  const float var = fmaxf((float)(q / n - mean * mean), 0.f);
  mr[i] = make_float2((float)mean, rsqrtf(var + eps));
}
__global__ void __launch_bounds__(256) gn_generic_apply_kernel(const float* __restrict__ x1, int C1, const float* __restrict__ x2, int C2,
                                                               const float2* __restrict__ mr, const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, int B, int HW, int G, int act,
                                                               int round_out, float* __restrict__ y, float* __restrict__ raw) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const int C = C1 + C2, cpg = C / G;
  const long long total = (long long)B * HW * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long bp = i / C;                            // b * HW + pix
    const int b = (int)(bp / HW);
    const float v = c < C1 ? x1[bp * C1 + c] : x2[bp * C2 + (c - C1)];
    const float2 m = mr[(long long)b * G + c / cpg];
    float o = (v - m.x) * m.y * __ldg(gamma + c) + __ldg(beta + c);
    if (act) o = round_out ? silu_fast(o) : silu_f(o);
    store_operand1(y, i, o, round_out);
    if (raw) store_operand1(raw, i, v, round_out);
  }
}
// pixel splits of the statistics pass, and the workspace (in floats) the two-kernel path needs:
// [B*G] float2 mean/rstd, then [B*G][splits] (sum, sum of squares) fp64 partials
static int gn_generic_splits(int HW) { return (int)std::max(1, std::min(64, HW / 1024)); }
long long gn_generic_workspace_floats(int B, int HW, int G) { return 2LL * B * G + 4LL * B * G * gn_generic_splits(HW); }

int launch_gn_generic(const float* x1, int C1, const float* x2, int C2, const float* gamma, const float* beta, int B, int HW, int G,
                      float eps, int act, int round_out, float* y, float* raw, float* mr_ws, cudaStream_t st) {
  const int C = C1 + C2;
  B200_REQUIRE(C % G == 0 && mr_ws, "gn_generic: C=%d G=%d", C, G);
  const int S = gn_generic_splits(HW);
  float2* mr = reinterpret_cast<float2*>(mr_ws);
  double* part = reinterpret_cast<double*>(mr_ws + 2LL * B * G);
  launch_kernel(gn_generic_stats_kernel, dim3(G, B, S), dim3(256), 0, st, x1, C1, x2, C2, HW, G, part);
  launch_kernel(gn_generic_finish_kernel, dim3((B * G + 127) / 128), dim3(128), 0, st, (const double*)part, B * G, S,
                (double)HW * (C / G), eps, mr);
  const long long total = (long long)B * HW * C;
  const int grid = (int)std::min<long long>((total + 255) / 256, 132LL * 32);
  launch_kernel(gn_generic_apply_kernel, dim3(grid), dim3(256), 0, st, x1, C1, x2, C2, (const float2*)mr, gamma, beta, B, HW, G, act, round_out, y, raw);
  B200_CHECK_LAUNCH();
  return 0;
}

// GroupNorm folded into per-(image, channel) affine coefficients: scale = rstd * gamma, shift = beta - mean * scale,
// from the same fp64 quad sums and with the same fp32 operations as gn_apply_stream_kernel (so a consumer that applies
// fma(x, scale, shift) reproduces that kernel bit for bit).  Consumed by the few-channel convolutions that normalise their
// input on load (conv_lowc.cu): the [B][C] tables are ~1e-3 of the activation bytes, the normalised tensor is never stored.
__global__ void __launch_bounds__(128) gn_coeff_kernel(const double* __restrict__ q1, int C1, const double* __restrict__ q2, int C2,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta, int G,
                                                       float eps, double inv_n, float* __restrict__ scale, float* __restrict__ shift) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const int C = C1 + C2, Q = C >> 2, cpg = C / G, b = blockIdx.y;
  const int qd = blockIdx.x * blockDim.x + threadIdx.x;
  if (qd >= Q) return;
  const int c0 = qd << 2, g0 = (c0 / cpg) * cpg;
  double s = 0.0, ss = 0.0;
  for (int c = g0; c < g0 + cpg; c += 4) {
    const double* src = (c < C1) ? q1 + ((long long)b * (C1 >> 2) + (c >> 2)) * 2
                                 : q2 + ((long long)b * (C2 >> 2) + ((c - C1) >> 2)) * 2;
    s += src[0]; ss += src[1];
  }
  const double mean = s * inv_n;
  const float var = fmaxf((float)(ss * inv_n - mean * mean), 0.f);
  const float rstd = rsqrtf(var + eps), mu = (float)mean;
  const float4 ga = __ldg(reinterpret_cast<const float4*>(gamma + c0));
  const float4 be = __ldg(reinterpret_cast<const float4*>(beta + c0));
  const float4 sc = make_float4(rstd * ga.x, rstd * ga.y, rstd * ga.z, rstd * ga.w);
  *reinterpret_cast<float4*>(scale + (long long)b * C + c0) = sc;
  *reinterpret_cast<float4*>(shift + (long long)b * C + c0) =
      make_float4(fmaf(-mu, sc.x, be.x), fmaf(-mu, sc.y, be.y), fmaf(-mu, sc.z, be.z), fmaf(-mu, sc.w, be.w));
}

int launch_gn_coeff(int C1, int C2, const double* q1, const double* q2, const float* gamma, const float* beta, int B, int HW,
                    int G, float eps, float* scale, float* shift, cudaStream_t st) {
  const int C = C1 + C2;
  B200_REQUIRE(C % 4 == 0 && C1 % 4 == 0 && C % G == 0 && (C / G) % 4 == 0, "gn_coeff: C=%d (C1=%d) G=%d must give 4-aligned groups", C, C1, G);
  B200_REQUIRE(q1 && (C2 == 0 || q2) && scale && shift, "gn_coeff: null pointer");
  const double inv_n = 1.0 / ((double)HW * (C / G));
  dim3 grid((C / 4 + 127) / 128, B);
  launch_kernel(gn_coeff_kernel, dim3(grid), dim3(128), 0, st, q1, C1, q2, C2, gamma, beta, G, eps, inv_n, scale, shift);
  B200_CHECK_LAUNCH();
  return 0;
}

// ============================================================================
// upfirdn2d: zero-insert upsample (up), zero pad, correlate with the flipped FIR,
// decimate (down).  Successor of the reference's native op
// (op/upfirdn2d_kernel.cu:49-207, host dispatch :209-369); same tensor convention
// [major, in_h, in_w, minor] -> [major, out_h, out_w, minor].  The reference always
// calls it with major=N*C, minor=1 (op/upfirdn2d.py:99); the engine calls it with
// major=N, minor=C, i.e. directly on NHWC, so a thread produces VEC consecutive
// channels of one output pixel with 128-bit accesses and the FIR taps in registers.
//   out[oy,ox] = sum_{a,b} k[kh-1-a, kw-1-b] * u[oy*down_y + a, ox*down_x + b]
//   u[Y,X] = x[(Y-pad_y0)/up_y, (X-pad_x0)/up_x] when divisible and in range, else 0.
// ============================================================================
struct FirParams {
  int major, in_h, in_w, minor, out_h, out_w;
  int kh, kw, up_x, up_y, down_x, down_y, pad_x0, pad_y0;
  int round_out;
  float k[64];   // row-major [kh][kw], kh*kw <= 64
};

template <int VEC>
__global__ void __launch_bounds__(256) upfirdn2d_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                       const FirParams p) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const int mv = p.minor / VEC;
  const long long total = (long long)p.major * p.out_h * p.out_w * mv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int cm = (int)(i % mv) * VEC;
    long long t = i / mv;
    const int ox = (int)(t % p.out_w); t /= p.out_w;
    const int oy = (int)(t % p.out_h);
    const int n = (int)(t / p.out_h);
    float acc[VEC];
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[v] = 0.f;
    for (int a = 0; a < p.kh; ++a) {
      const int Y = oy * p.down_y + a - p.pad_y0;
      if (Y < 0 || (Y % p.up_y) != 0) continue;
      const int iy = Y / p.up_y;
      if (iy >= p.in_h) continue;
      for (int b = 0; b < p.kw; ++b) {
        const int X = ox * p.down_x + b - p.pad_x0;
        if (X < 0 || (X % p.up_x) != 0) continue;
        const int ix = X / p.up_x;
        if (ix >= p.in_w) continue;
        const float w = p.k[(p.kh - 1 - a) * p.kw + (p.kw - 1 - b)];
        const float* src = x + (((long long)n * p.in_h + iy) * p.in_w + ix) * p.minor + cm;
        if (VEC == 4) {
          const float4 v = __ldg(reinterpret_cast<const float4*>(src));
          acc[0] += w * v.x; acc[1] += w * v.y; acc[2] += w * v.z; acc[3] += w * v.w;
        } else {
          acc[0] += w * __ldg(src);
        }
      }
    }
    const long long o = (((long long)n * p.out_h + oy) * p.out_w + ox) * p.minor + cm;
    if (VEC == 4) store_operand4(y, o, make_float4(acc[0], acc[1], acc[2], acc[3]), p.round_out);
    else store_operand1(y, o, acc[0], p.round_out);
  }
}

// Fast path for the three parameterisations NCSN++ uses (4x4 FIR, NHWC with minor % 4 == 0):
//   UP=2 (pad 2,1): polyphase, 2x2 live taps per output;  DOWN=2 (pad 1,1): 4x4 taps, stride 2;
//   UP=DOWN=1 (pad 2,2): 4x4 taps.  All index arithmetic is compile-time; one thread = one output float4.
template <int UP, int DOWN>
__global__ void __launch_bounds__(256) fir4_nhwc_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                       const FirParams p) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  // grid = (x chunks over out_w * minor/4, out_h, images): no 64-bit div/mod chain per thread (the flat-index
  // version spent more instructions decoding its index than filtering)
  const int mv = p.minor >> 2;
  const unsigned xi = blockIdx.x * blockDim.x + threadIdx.x;
  if (xi >= (unsigned)(p.out_w * mv)) return;
  const int cm = (int)(xi % (unsigned)mv) << 2, ox = (int)(xi / (unsigned)mv);
  const int oy = blockIdx.y, n = blockIdx.z;
  const float* xin = x + (long long)n * p.in_h * p.in_w * p.minor + cm;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int Y = oy * DOWN + a - p.pad_y0;
    if (UP == 2 && (Y & 1)) continue;
    const int iy = UP == 2 ? (Y >> 1) : Y;
    if (Y < 0 || iy >= p.in_h) continue;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int X = ox * DOWN + b - p.pad_x0;
      if (UP == 2 && (X & 1)) continue;
      const int ix = UP == 2 ? (X >> 1) : X;
      if (X < 0 || ix >= p.in_w) continue;
      const float w = p.k[(3 - a) * 4 + (3 - b)];
      const float4 v = __ldg(reinterpret_cast<const float4*>(xin + ((long long)iy * p.in_w + ix) * p.minor));
      acc.x += w * v.x; acc.y += w * v.y; acc.z += w * v.z; acc.w += w * v.w;
    }
  }
  store_operand4(y, (((long long)n * p.out_h + oy) * p.out_w + ox) * p.minor + cm, acc, p.round_out);
}

// 2x upsampling (up=2, pad0=2, 4x4 FIR), one thread per INPUT pixel quad: the 3x3 input neighbourhood is loaded
// once (9 float4) and produces the 2x2 output block (4 float4), 2.25 loads per output instead of 4.
//   out[2i+ay][2j+ax] = sum over the two live taps per axis:  ay=0: (a=0, iy=i-1), (a=2, iy=i);  ay=1: (a=1, iy=i), (a=3, iy=i+1)
__global__ void __launch_bounds__(256) fir4_up2_nhwc_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                           const FirParams p) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const int mv = p.minor >> 2;
  const unsigned xi = blockIdx.x * blockDim.x + threadIdx.x;   // grid = (x chunks over in_w * minor/4, in_h, images)
  if (xi >= (unsigned)(p.in_w * mv)) return;
  const int cm = (int)(xi % (unsigned)mv) << 2, j = (int)(xi / (unsigned)mv);
  const int i = blockIdx.y, n = blockIdx.z;
  const float* xin = x + (long long)n * p.in_h * p.in_w * p.minor + cm;
  float4 v[3][3];
#pragma unroll
  for (int dy = 0; dy < 3; ++dy)
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) {
      const int iy = i + dy - 1, ix = j + dx - 1;
      v[dy][dx] = (iy >= 0 && iy < p.in_h && ix >= 0 && ix < p.in_w)
                      ? __ldg(reinterpret_cast<const float4*>(xin + ((long long)iy * p.in_w + ix) * p.minor))
                      : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  const long long yout = (long long)n * p.out_h * p.out_w * p.minor + cm;
#pragma unroll
  for (int ay = 0; ay < 2; ++ay)
#pragma unroll
    for (int ax = 0; ax < 2; ++ax) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int ty = 0; ty < 2; ++ty)
#pragma unroll
        for (int tx = 0; tx < 2; ++tx) {
          const int a = ay + 2 * ty, b = ax + 2 * tx;          // live taps of this output phase
          const int dy = ay + ty, dx = ax + tx;                // neighbourhood slot: iy = i - 1 + dy
          const float w = p.k[(3 - a) * 4 + (3 - b)];
          const float4 u = v[dy][dx];
          acc.x += w * u.x; acc.y += w * u.y; acc.z += w * u.z; acc.w += w * u.w;
        }
      store_operand4(y, yout + ((long long)(2 * i + ay) * p.out_w + (2 * j + ax)) * p.minor, acc, p.round_out);
    }
}

// ---- planar (minor == 1) 4x4 FIR: the reference's own tensor convention [N*C, H, W, 1] (op/upfirdn2d.py:99) ----
// The NHWC kernels above put channels on the fast axis; with one channel per "pixel" a thread instead produces four
// consecutive outputs along W of one plane row, so its global accesses run along the contiguous axis and it stores 128 bits.
// out[oy, ox] = sum_{a,b} kf[a][b] * u[oy*D + a, ox*D + b], kf = flipped FIR, u = x zero-inserted by U and padded by p0.
template <int UP, int DOWN>
__global__ void __launch_bounds__(128) fir4_planar_kernel(const float* __restrict__ x, float* __restrict__ y, const FirParams p) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const int qw = (p.out_w + 3) >> 2;                      // four-output groups per row
  const long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (q >= (long long)p.major * p.out_h * qw) return;
  const int ox0 = (int)(q % qw) * 4;
  const long long t = q / qw;
  const int oy = (int)(t % p.out_h);
  const long long n = t / p.out_h;
  const float* xp = x + n * p.in_h * p.in_w;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  if (UP == 1) {
    constexpr int NC = 3 * DOWN + 4;                       // input columns feeding four outputs
    const int c0 = ox0 * DOWN - p.pad_x0;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int iy = oy * DOWN + a - p.pad_y0;
      if (iy < 0 || iy >= p.in_h) continue;
      const float* row = xp + (long long)iy * p.in_w;
      float v[NC];
#pragma unroll
      for (int c = 0; c < NC; ++c) { const int ix = c0 + c; v[c] = (ix >= 0 && ix < p.in_w) ? __ldg(row + ix) : 0.f; }
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[j] = fmaf(p.k[(3 - a) * 4 + (3 - b)], v[j * DOWN + b], acc[j]);
    }
  } else {
    // zero-insertion by 2: only taps with (oy + a - p0) and (ox + b - p0) even meet an input sample
    const int a0 = (oy + p.pad_y0) & 1;
#pragma unroll
    for (int aa = 0; aa < 2; ++aa) {
      const int a = a0 + 2 * aa, Y = oy + a - p.pad_y0;
      if (Y < 0) continue;
      const int iy = Y >> 1;
      if (iy >= p.in_h) continue;
      const float* row = xp + (long long)iy * p.in_w;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int ox = ox0 + j, b0 = (ox + p.pad_x0) & 1;
#pragma unroll
        for (int bb = 0; bb < 2; ++bb) {
          const int b = b0 + 2 * bb, X = ox + b - p.pad_x0;
          if (X < 0) continue;
          const int ix = X >> 1;
          if (ix < p.in_w) acc[j] = fmaf(p.k[(3 - a) * 4 + (3 - b)], __ldg(row + ix), acc[j]);
        }
      }
    }
  }
  float* dst = y + (n * p.out_h + oy) * p.out_w + ox0;
  if (ox0 + 3 < p.out_w && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0)) {
    float4 o = make_float4(acc[0], acc[1], acc[2], acc[3]);
    if (p.round_out == 1) { o.x = round_tf32(o.x); o.y = round_tf32(o.y); o.z = round_tf32(o.z); o.w = round_tf32(o.w); }
    *reinterpret_cast<float4*>(dst) = o;
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) if (ox0 + j < p.out_w) dst[j] = p.round_out == 1 ? round_tf32(acc[j]) : acc[j];
  }
}

int launch_upfirdn2d(const float* x, const float* kernel_host, float* y, int major, int in_h, int in_w,
                     int minor, int kh, int kw, int up_x, int up_y, int down_x, int down_y,
                     int pad_x0, int pad_x1, int pad_y0, int pad_y1, int round_out, cudaStream_t st) {
  B200_REQUIRE(kh * kw <= 64 && kh > 0 && kw > 0, "upfirdn2d: FIR %dx%d exceeds 64 taps", kh, kw);
  B200_REQUIRE(up_x > 0 && up_y > 0 && down_x > 0 && down_y > 0, "upfirdn2d: up/down must be positive");
  FirParams p;
  p.major = major; p.in_h = in_h; p.in_w = in_w; p.minor = minor;
  p.out_h = (in_h * up_y + pad_y0 + pad_y1 - kh) / down_y + 1;
  p.out_w = (in_w * up_x + pad_x0 + pad_x1 - kw) / down_x + 1;
  p.kh = kh; p.kw = kw; p.up_x = up_x; p.up_y = up_y; p.down_x = down_x; p.down_y = down_y;
  p.pad_x0 = pad_x0; p.pad_y0 = pad_y0; p.round_out = round_out;
  for (int i = 0; i < kh * kw; ++i) p.k[i] = kernel_host[i];
  B200_REQUIRE(p.out_h > 0 && p.out_w > 0, "upfirdn2d: empty output %dx%d", p.out_h, p.out_w);
  const bool vec = (minor % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) % 16 == 0);
  const long long total = (long long)major * p.out_h * p.out_w * (vec ? minor / 4 : minor);
  if (total == 0) return 0;
  if (vec && kh == 4 && kw == 4 && up_x == up_y && down_x == down_y && pad_x0 == pad_y0 && pad_x0 >= 0 && major <= 65535 &&
      p.out_h <= 65535 && (long long)p.out_w * (minor / 4) < (1LL << 31)) {
    const int mv = minor / 4;
    const int threads = (p.out_w * mv >= 256) ? 256 : 128;
    const dim3 grid((unsigned)((p.out_w * mv + threads - 1) / threads), (unsigned)p.out_h, (unsigned)major);
    if (up_x == 2 && down_x == 1 && pad_x0 == 2 && p.out_h == 2 * in_h && p.out_w == 2 * in_w) {
      const int tin = (in_w * mv >= 256) ? 256 : 128;
      launch_kernel(fir4_up2_nhwc_kernel, dim3(dim3((unsigned)((in_w * mv + tin - 1) / tin), (unsigned)in_h, (unsigned)major)), dim3(tin), 0, st, x, y, p);
      B200_CHECK_LAUNCH();
      return 0;
    }
    if (up_x == 2 && down_x == 1) { launch_kernel(fir4_nhwc_kernel<2, 1>, dim3(grid), dim3(threads), 0, st, x, y, p); B200_CHECK_LAUNCH(); return 0; }
    if (up_x == 1 && down_x == 2) { launch_kernel(fir4_nhwc_kernel<1, 2>, dim3(grid), dim3(threads), 0, st, x, y, p); B200_CHECK_LAUNCH(); return 0; }
    if (up_x == 1 && down_x == 1) { launch_kernel(fir4_nhwc_kernel<1, 1>, dim3(grid), dim3(threads), 0, st, x, y, p); B200_CHECK_LAUNCH(); return 0; }
  }
  if (minor == 1 && kh == 4 && kw == 4 && up_x == up_y && down_x == down_y && pad_x0 == pad_y0 && round_out != 2 &&
      ((up_x == 1 && (down_x == 1 || down_x == 2)) || (up_x == 2 && down_x == 1)) &&
      (long long)major * p.out_h * ((p.out_w + 3) / 4) < (1LL << 37)) {
    // the reference's own layout ([N*C, H, W, 1]): four outputs along W per thread (VERDICT r01 task 9d)
    const int tx = 128;
    const long long quads = (long long)major * p.out_h * ((p.out_w + 3) / 4);
    const unsigned pg = (unsigned)((quads + tx - 1) / tx);
    if (up_x == 2) launch_kernel(fir4_planar_kernel<2, 1>, dim3(pg), dim3(tx), 0, st, x, y, p);
    else if (down_x == 2) launch_kernel(fir4_planar_kernel<1, 2>, dim3(pg), dim3(tx), 0, st, x, y, p);
    else launch_kernel(fir4_planar_kernel<1, 1>, dim3(pg), dim3(tx), 0, st, x, y, p);
    B200_CHECK_LAUNCH();
    return 0;
  }
  const int grid = (int)std::min<long long>((total + 255) / 256, 132LL * 64);
  if (vec) launch_kernel(upfirdn2d_kernel<4>, dim3(grid), dim3(256), 0, st, x, y, p);
  else launch_kernel(upfirdn2d_kernel<1>, dim3(grid), dim3(256), 0, st, x, y, p);
  B200_CHECK_LAUNCH();
  return 0;
}

// ============================================================================
// fused bias + activation (successor of op/fused_bias_act_kernel.cu:19-98):
// y = act(x + b[(i / step_b) % size_b]) * scale, act 1 = linear, 3 = leaky-relu(alpha);
// grad 1 gates on `ref` instead of x (first derivative), grad 2 yields zeros.
// ============================================================================
__global__ void __launch_bounds__(256) fused_bias_act_kernel(
    const float* __restrict__ x, const float* __restrict__ b, const float* __restrict__ ref,
    float* __restrict__ y, long long n, int step_b, int size_b, int act, int grad, float alpha, float scale) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    float v = x[i];
    if (b) v += __ldg(&b[(i / step_b) % size_b]);
    const float r = ref ? ref[i] : 0.f;
    float o;
    if (grad == 2) o = 0.f;
    else if (act == 3) o = ((grad == 1 ? r : v) > 0.f) ? v : v * alpha;
    else o = v;
    y[i] = o * scale;
  }
}

int launch_fused_bias_act(const float* x, const float* b, const float* ref, float* y, long long n,
                          int step_b, int size_b, int act, int grad, float alpha, float scale,
                          cudaStream_t st) {
  if (n == 0) return 0;
  B200_REQUIRE(act == 1 || act == 3, "fused_bias_act: act=%d unsupported (1 linear, 3 lrelu)", act);
  B200_REQUIRE(!b || (step_b > 0 && size_b > 0), "fused_bias_act: bad bias geometry");
  const int grid = (int)std::min<long long>((n + 255) / 256, 132LL * 64);
  launch_kernel(fused_bias_act_kernel, dim3(grid), dim3(256), 0, st, x, b, ref, y, n, step_b, size_b, act, grad, alpha, scale);
  B200_CHECK_LAUNCH();
  return 0;
}

// ============================================================================
// Row softmax for the attention logits (layerspp.py:82-85): rows of length T,
// logits pre-multiplied by `scale` = C^-1/2.  One warp per row, values held in
// registers (T <= 1024), warp-shuffle max/sum.
// ============================================================================
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ s, float* __restrict__ p,
                                                          long long rows, int T, float scale, int round_out) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const int lane = threadIdx.x & 31;
  const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* src = s + row * T;
  float v[32];
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int c = lane + j * 32;
    v[j] = (c < T) ? src[c] * scale : -INFINITY;
    mx = fmaxf(mx, v[j]);
  }
  mx = warp_max(mx);
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int c = lane + j * 32;
    v[j] = (c < T) ? expf(v[j] - mx) : 0.f;
    sum += v[j];
  }
  sum = warp_sum(sum);
  float* dst = p + row * T;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int c = lane + j * 32;
    if (c < T) {
      float o = v[j] / sum;
      dst[c] = round_out ? round_tf32(o) : o;
    }
  }
}

// T == 256 (the 16x16 attention of NCSN++): one warp per row, two 128-bit accesses per lane each way,
// two rows per warp iteration in flight.
__global__ void __launch_bounds__(256) softmax_rows256_kernel(const float* __restrict__ s, float* __restrict__ p,
                                                             long long rows, float scale, int round_out) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const int lane = threadIdx.x & 31;
  const long long warp_id = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long row = warp_id * 2; row < rows; row += nwarps * 2) {
    float4 a[2][2];
    const bool two = row + 1 < rows;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float4* src = reinterpret_cast<const float4*>(s + (row + (two ? r : 0)) * 256);
      a[r][0] = __ldg(src + lane); a[r][1] = __ldg(src + 32 + lane);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float* e = reinterpret_cast<float*>(a[r]);
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 8; ++i) { e[i] *= scale; mx = fmaxf(mx, e[i]); }
      mx = warp_max(mx);
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) { e[i] = expf(e[i] - mx); sum += e[i]; }
      sum = warp_sum(sum);
#pragma unroll
      for (int i = 0; i < 8; ++i) { e[i] = e[i] / sum; if (round_out) e[i] = round_tf32(e[i]); }
      if (r == 0 || two) {
        float4* dst = reinterpret_cast<float4*>(p + (row + r) * 256);
        dst[lane] = a[r][0]; dst[32 + lane] = a[r][1];
      }
    }
  }
}

int launch_softmax_rows(const float* s, float* p, long long rows, int T, float scale, int round_out,
                        cudaStream_t st) {
  B200_REQUIRE(T > 0 && T <= 1024, "softmax_rows: T=%d out of range (1..1024)", T);
  const int wpb = 8;
  if (T == 256 && ((reinterpret_cast<uintptr_t>(s) | reinterpret_cast<uintptr_t>(p)) & 15) == 0) {
    const long long blocks = std::min<long long>((rows / 2 + wpb - 1) / wpb + 1, 132LL * 16);
    launch_kernel(softmax_rows256_kernel, dim3((unsigned)blocks), dim3(wpb * 32), 0, st, s, p, rows, scale, round_out);
    B200_CHECK_LAUNCH();
    return 0;
  }
  launch_kernel(softmax_rows_kernel, dim3((unsigned)((rows + wpb - 1) / wpb)), dim3(wpb * 32), 0, st, s, p, rows, T, scale, round_out);
  B200_CHECK_LAUNCH();
  return 0;
}

// ============================================================================
// Time-embedding path (ncsnpp.py:236-255, layerspp.py:39-41).
// fourier: emb[r] = [sin(p), cos(p)], p = ((log(sigma_r) * W_j) * 2) * fp32(pi) with the
// reference's operation order; accurate sinf/cosf/logf (phases reach ~1e3 rad).
// ============================================================================
// positional != 0: sinusoidal embedding of the label itself (models/layers.py:515-529): emb = [sin(t f_j), cos(t f_j)],
// f = exp(-j log(10000) / (half - 1)) precomputed by the host with the reference's torch ops; W then holds `nf` = half
// frequencies and a row of emb has 2 * nf entries.
__global__ void fourier_embed_kernel(const float* __restrict__ sigma, long long sigma_stride,
                                     const float* __restrict__ W, int nf, float* __restrict__ emb, int positional) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const int r = blockIdx.x;
  const float t = sigma[r * sigma_stride];
  const float lv = positional ? t : logf(t);
  for (int j = threadIdx.x; j < nf; j += blockDim.x) {
    const float ph = positional ? lv * W[j] : ((lv * W[j]) * 2.0f) * 3.14159265358979323846f;
    emb[(long long)r * 2 * nf + j] = sinf(ph);
    emb[(long long)r * 2 * nf + nf + j] = cosf(ph);
  }
}

int launch_fourier_embed(const float* sigma, long long sigma_stride, const float* W, int nf, int rows,
                         float* emb, cudaStream_t st, int positional) {
  launch_kernel(fourier_embed_kernel, dim3(rows), dim3(128), 0, st, sigma, sigma_stride, W, nf, emb, positional);
  B200_CHECK_LAUNCH();
  return 0;
}

// y[r][n] = sum_k act(x[r][k]) * W[n][k] + b[n]   (torch Linear layout, fp32 exact).
// A CTA stages up to RB rows of act(x) in shared memory; each warp owns output
// columns and reuses every W row it loads for all staged rows.
constexpr int LIN_RB = 8;
__global__ void __launch_bounds__(256) linear_rows_kernel(
    const float* __restrict__ x, long long ldx, const float* __restrict__ W, const float* __restrict__ bias,
    int rows, int N, int K, int act_in, float* __restrict__ y, long long ldy) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  extern __shared__ float sx[];   // [LIN_RB][K]
  const int r0 = blockIdx.y * LIN_RB;
  const int nr = min(LIN_RB, rows - r0);
  for (int i = threadIdx.x; i < nr * K; i += blockDim.x) {
    const int r = i / K, k = i % K;
    float v = x[(long long)(r0 + r) * ldx + k];
    sx[r * K + k] = act_in ? silu_f(v) : v;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int n = blockIdx.x * nwarps + warp; n < N; n += gridDim.x * nwarps) {
    float acc[LIN_RB];
#pragma unroll
    for (int r = 0; r < LIN_RB; ++r) acc[r] = 0.f;
    const float* w = W + (long long)n * K;
    for (int k = lane; k < K; k += 32) {
      const float wv = __ldg(&w[k]);
#pragma unroll
      for (int r = 0; r < LIN_RB; ++r)
        if (r < nr) acc[r] += sx[r * K + k] * wv;
    }
#pragma unroll
    for (int r = 0; r < LIN_RB; ++r) {
      const float t = warp_sum(acc[r]);
      if (lane == 0 && r < nr) y[(long long)(r0 + r) * ldy + n] = t + (bias ? bias[n] : 0.f);
    }
  }
}

int launch_linear_rows(const float* x, long long ldx, const float* W, const float* bias, int rows, int N,
                       int K, int act_in, float* y, long long ldy, cudaStream_t st) {
  B200_REQUIRE(K * LIN_RB * 4 <= 96 * 1024, "linear_rows: K=%d too large for the row stage", K);
  const size_t smem = (size_t)LIN_RB * K * sizeof(float);
  if (smem > 48 * 1024)
    B200_CHECK_CUDA(cudaFuncSetAttribute(linear_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(std::min(ceil_div(N, 8), 132 * 4), ceil_div(rows, LIN_RB));   // 4 CTAs per H100 SM
  launch_kernel(linear_rows_kernel, dim3(grid), dim3(256), smem, st, x, ldx, W, bias, rows, N, K, act_in, y, ldy);
  B200_CHECK_LAUNCH();
  return 0;
}

// ============================================================================
// Utilities
// ============================================================================
__global__ void fill_from_table_kernel(const float* __restrict__ table, const int* __restrict__ step,
                                       float* __restrict__ dst, int n) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const float v = table[*step];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = v;
}
int launch_fill_from_table(const float* table, const int* step, float* dst, int n, cudaStream_t st) {
  launch_kernel(fill_from_table_kernel, dim3(ceil_div(n, 256)), dim3(256), 0, st, table, step, dst, n);
  B200_CHECK_LAUNCH();
  return 0;
}

__global__ void nhwc_to_nchw_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int HW, int C) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const long long total = (long long)B * HW * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(i % HW);
    const long long t = i / HW;
    const int c = (int)(t % C);
    const long long b = t / C;
    dst[i] = src[(b * HW + p) * C + c];
  }
}
int launch_nhwc_to_nchw(const float* src, float* dst, int B, int HW, int C, cudaStream_t st) {
  const long long total = (long long)B * HW * C;
  launch_kernel(nhwc_to_nchw_kernel, dim3((int)std::min<long long>((total + 255) / 256, 132LL * 64)), dim3(256), 0, st, src, dst, B, HW, C);
  B200_CHECK_LAUNCH();
  return 0;
}

// operand-format copy of an fp32 activation (the DDPM Downsample convolution reads a block output directly)
__global__ void __launch_bounds__(256) store_operand_kernel(const float4* __restrict__ x, float* __restrict__ y, long long n4, int mode) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x)
    store_operand4(y, 4 * i, __ldg(x + i), mode);
}
int launch_store_operand(const float* x, float* y, long long n, int mode, cudaStream_t st) {
  B200_REQUIRE(n % 4 == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) % 16) == 0,
               "store_operand: %lld elements / pointer alignment not float4-aligned", n);
  const long long n4 = n / 4;
  if (n4 == 0) return 0;
  launch_kernel(store_operand_kernel, dim3((int)std::min<long long>((n4 + 255) / 256, 132LL * 16)), dim3(256), 0, st,
                reinterpret_cast<const float4*>(x), y, n4, mode);
  B200_CHECK_LAUNCH();
  return 0;
}

// dst[tap*dt + o*dO + i] = src[o*so + i*si + tap*st]  (OIHW conv weights: so=I*R*S, si=R*S, st=1;
// NIN W[in][out]: taps=1, so=1, si=out).  Default destination [tap][o][i] (dt=O*I, dO=I); the
// flat-K packing of the input convolution uses dt=I, dO=row pitch.  Optional TF32 rounding; with `lo` (split TF32) dst
// holds hi = rna_tf32(w) and lo, at the same index, rna_tf32(w - hi).
__global__ void pack_weight_kernel(const float* __restrict__ src, float* __restrict__ dst, int taps, int O, int I,
                                   long long so, long long si, long long stp, int round_out, long long dt, long long dO,
                                   float* __restrict__ lo) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const long long total = (long long)taps * O * I;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(idx % I);
    const long long t = idx / I;
    const int o = (int)(t % O);
    const int tap = (int)(t / O);
    const float v = src[o * so + i * si + tap * stp];
    const long long d = tap * dt + o * dO + i;
    store_operand1(dst, d, v, round_out);
    if (lo) lo[d] = round_tf32(v - round_tf32(v));
  }
}
int launch_pack_weight(const float* src, float* dst, int taps, int O, int I, long long so, long long si,
                       long long stp, int round_out, cudaStream_t st, long long dt, long long dO, float* lo) {
  B200_REQUIRE(!lo || round_out == 1, "pack_weight: the split-TF32 lo copy goes with TF32-rounded weights");
  const long long total = (long long)taps * O * I;
  if (dt == 0) { dt = (long long)O * I; dO = I; }
  launch_kernel(pack_weight_kernel, dim3((int)std::min<long long>((total + 255) / 256, 132LL * 16)), dim3(256), 0, st,
      src, dst, taps, O, I, so, si, stp, round_out, dt, dO, lo);
  B200_CHECK_LAUNCH();
  return 0;
}

// split TF32 pair of an fp32 operand (precision 3): hi = rna_tf32(x), lo = rna_tf32(x - hi); x = hi + lo to ~2^-22 relative
__global__ void __launch_bounds__(256) split_tf32_kernel(const float4* __restrict__ x, float4* __restrict__ hi,
                                                         float4* __restrict__ lo, long long n4) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = __ldg(x + i);
    const float4 h = make_float4(round_tf32(v.x), round_tf32(v.y), round_tf32(v.z), round_tf32(v.w));
    hi[i] = h;
    lo[i] = make_float4(round_tf32(v.x - h.x), round_tf32(v.y - h.y), round_tf32(v.z - h.z), round_tf32(v.w - h.w));
  }
}
int launch_split_tf32(const float* x, float* hi, float* lo, long long n, cudaStream_t st) {
  B200_REQUIRE(n % 4 == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(hi) | reinterpret_cast<uintptr_t>(lo)) % 16) == 0,
               "split_tf32: %lld elements / pointer alignment not float4-aligned", n);
  const long long n4 = n / 4;
  if (n4 == 0) return 0;
  launch_kernel(split_tf32_kernel, dim3((int)std::min<long long>((n4 + 255) / 256, 132LL * 16)), dim3(256), 0, st,
                reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(hi), reinterpret_cast<float4*>(lo), n4);
  B200_CHECK_LAUNCH();
  return 0;
}

// ============================================================================
// Input convolution as one K=32 contraction: patches[b*HW + pix][tap*C + c] = x[b][c][pix + tap offset]
// (zero outside the image, zero for k >= 9*C), TF32-rounded, from the NCHW network input.
// 9*C <= 32 (C = 3 for images).  The 3->nf 3x3 conv (ncsnpp.py:268) then runs on the tensor cores as a
// [B*HW, 32] x [nf, 32]^T product instead of a 27-deep CUDA-core loop.
// ============================================================================
template <int C>   // image channels (9*C <= 32); compile-time so the patch lives in registers
__global__ void __launch_bounds__(256) im2col3x3_nchw_kernel(const float* __restrict__ x, float* __restrict__ patches,
                                                            int B, int Hin, int Win, int H, int W, int stride, int pad,
                                                            int mode /* 1: 32 TF32 floats per row, 2: 64 halves per row */) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  // One thread per output pixel: consecutive lanes read consecutive pixels of one channel plane (coalesced; the first
  // version gave each lane a different (tap, channel) and paid ~64 L1 wavefronts per pixel), then the thread writes
  // its whole 128-byte row.
  const long long pg = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (pg >= (long long)B * H * W) return;
  const int px = (int)(pg % W), py = (int)((pg / W) % H), b = (int)(pg / ((long long)W * H));
  float v[32];
#pragma unroll
  for (int k = 0; k < 32; ++k) v[k] = 0.f;
  const float* xb = x + (long long)b * C * Hin * Win;
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) {
    const int iy = py * stride + tap / 3 - pad, ix = px * stride + tap % 3 - pad;
    const bool in = iy >= 0 && iy < Hin && ix >= 0 && ix < Win;
#pragma unroll
    for (int c = 0; c < C; ++c)
      v[tap * C + c] = in ? __ldg(xb + ((long long)c * Hin + iy) * Win + ix) : 0.f;
  }
  if (mode == 2) {
    uint16_t* row = reinterpret_cast<uint16_t*>(patches) + pg * 64;
#pragma unroll
    for (int q = 0; q < 4; ++q)
      *reinterpret_cast<uint4*>(row + 8 * q) = make_uint4(pack_half2(v[8 * q], v[8 * q + 1]), pack_half2(v[8 * q + 2], v[8 * q + 3]),
                                                          pack_half2(v[8 * q + 4], v[8 * q + 5]), pack_half2(v[8 * q + 6], v[8 * q + 7]));
#pragma unroll
    for (int q = 4; q < 8; ++q) *reinterpret_cast<uint4*>(row + 8 * q) = make_uint4(0u, 0u, 0u, 0u);
  } else {
    float* row = patches + pg * 32;   // mode 1: TF32 grid; mode 0: fp32 as read (split TF32 plans split the patches after)
#pragma unroll
    for (int q = 0; q < 8; ++q)
      store_operand4(row, 4 * q, make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]), mode);
  }
}

int launch_im2col3x3_nchw(const float* x, float* patches, int B, int C, int Hin, int Win, int H, int W, int stride,
                          int pad, int mode, cudaStream_t st) {
  B200_REQUIRE(C >= 1 && C <= 3, "im2col3x3: %d channels unsupported (1..3 image channels)", C);
  B200_REQUIRE(mode >= 0 && mode <= 2, "im2col3x3: operand mode %d", mode);
  const long long total = (long long)B * H * W;
  const unsigned blocks = (unsigned)((total + 255) / 256);
  switch (C) {
    case 1: launch_kernel(im2col3x3_nchw_kernel<1>, dim3(blocks), dim3(256), 0, st, x, patches, B, Hin, Win, H, W, stride, pad, mode); break;
    case 2: launch_kernel(im2col3x3_nchw_kernel<2>, dim3(blocks), dim3(256), 0, st, x, patches, B, Hin, Win, H, W, stride, pad, mode); break;
    default: launch_kernel(im2col3x3_nchw_kernel<3>, dim3(blocks), dim3(256), 0, st, x, patches, B, Hin, Win, H, W, stride, pad, mode); break;
  }
  B200_CHECK_LAUNCH();
  return 0;
}

// ============================================================================
// Output head: 3x3 'same' convolution to N <= 4 channels (ncsnpp.py:374) on NHWC input, written
// straight to NCHW with bias and the 1/sigma scaling (ncsnpp.py:377-379) fused.  Memory-bound
// (reads the activation once through L1, 9x tap reuse between neighbouring threads); the 9*N*C
// weights sit in shared memory and are read as broadcast float4s.
// ============================================================================
template <int N, int LPP>
__global__ void __launch_bounds__(256) conv3x3_small_n_kernel(const float* __restrict__ x, const float* __restrict__ w /* [9][N][C] */,
                                                             const float* __restrict__ bias, const float* __restrict__ div,
                                                             long long div_stride, float* __restrict__ out_nchw,
                                                             int B, int H, int W, int C, int x_f16,
                                                             const float* __restrict__ add_nchw) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  // LPP (eight; two for <= 32 channels, whose pixel vector is only 4 - 8 float4s) lanes share one output pixel: lane
  // `part` takes the float4s part, part+LPP, ... of the pixel's channel
  // vector, so a warp-wide 128-bit load covers 4 pixels x 128 contiguous bytes (4 cache lines per instruction
  // instead of 32 with one pixel per lane, which was L1-wavefront bound); the partial dot products are folded with
  // three shuffles per output channel.
  extern __shared__ float sw[];   // [9][N][C]
  if (x_f16 && LPP == 8) {
    // fp16 input: lane `part` owns 8 consecutive channels per 64-channel block.  Its two weight float4s are stored
    // so that the eight lanes of a pixel read 128 contiguous bytes per LDS.128 (conflict-free), i.e. within a block
    // channel c = 8*part + 4*k + e sits at float ((2*blk + k)*8 + part)*4 + e.
    for (int i = threadIdx.x; i < 9 * N * C; i += blockDim.x) {
      const int c = i % C, row = i / C, blk = c >> 6, prt = (c >> 3) & 7, k = (c >> 2) & 1, e = c & 3;
      sw[row * C + (((2 * blk + k) * 8 + prt) << 2) + e] = w[i];
    }
  } else {
    for (int i = threadIdx.x; i < 9 * N * C; i += blockDim.x) sw[i] = w[i];
  }
  __syncthreads();
  const long long gt = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long pg = gt / LPP;
  const int part = (int)(gt & (LPP - 1));
  const bool live = pg < (long long)B * H * W;
  const long long pgc = live ? pg : 0;
  const int px = (int)(pgc % W), py = (int)((pgc / W) % H), b = (int)(pgc / ((long long)W * H));
  float acc[N];
#pragma unroll
  for (int n = 0; n < N; ++n) acc[n] = 0.f;
  const float* xb = x + (long long)b * H * W * C;
  const int nq = C >> 2;                                  // float4s per pixel
  if (x_f16 && LPP == 8) {
    // fp16 activations (operand mode 2): a lane's 128-bit load carries 8 channels, half the L1/L2 bytes of the
    // nine-fold tap re-reads that bound this kernel
    const uint16_t* xh = reinterpret_cast<const uint16_t*>(x) + (long long)b * H * W * C;
    const int n8 = C >> 3;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int iy = py + tap / 3 - 1, ix = px + tap % 3 - 1;
      if (!live || iy < 0 || iy >= H || ix < 0 || ix >= W) continue;
      const uint4* src = reinterpret_cast<const uint4*>(xh + ((long long)iy * W + ix) * C);
      const float4* wt = reinterpret_cast<const float4*>(sw + tap * N * C);
      for (int c8 = part; c8 < n8; c8 += 16) {
        uint4 a[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) a[u] = (c8 + 8 * u < n8) ? __ldg(src + c8 + 8 * u) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          if (c8 + 8 * u >= n8) break;
          const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&a[u].x));
          const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&a[u].y));
          const float2 f2 = __half22float2(*reinterpret_cast<const __half2*>(&a[u].z));
          const float2 f3 = __half22float2(*reinterpret_cast<const __half2*>(&a[u].w));
#pragma unroll
          for (int n = 0; n < N; ++n) {
            const int blk = (c8 + 8 * u) >> 3;       // c8 + 8u = 8*blk + part
            const float4 w0 = wt[n * nq + (2 * blk) * 8 + part], w1 = wt[n * nq + (2 * blk + 1) * 8 + part];
            acc[n] = fmaf(f0.x, w0.x, fmaf(f0.y, w0.y, fmaf(f1.x, w0.z, fmaf(f1.y, w0.w, acc[n]))));
            acc[n] = fmaf(f2.x, w1.x, fmaf(f2.y, w1.y, fmaf(f3.x, w1.z, fmaf(f3.y, w1.w, acc[n]))));
          }
        }
      }
    }
  } else
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) {
    const int iy = py + tap / 3 - 1, ix = px + tap % 3 - 1;
    if (!live || iy < 0 || iy >= H || ix < 0 || ix >= W) continue;
    const float4* src = reinterpret_cast<const float4*>(xb + ((long long)iy * W + ix) * C);
    const float4* wt = reinterpret_cast<const float4*>(sw + tap * N * C);
    for (int c4 = part; c4 < nq; c4 += 4 * LPP) {          // up to four 128-bit loads in flight
      float4 a[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) a[u] = (c4 + LPP * u < nq) ? __ldg(src + c4 + LPP * u) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (c4 + LPP * u >= nq) break;
#pragma unroll
        for (int n = 0; n < N; ++n) {
          const float4 ww = wt[n * nq + c4 + LPP * u];
          acc[n] = fmaf(a[u].x, ww.x, fmaf(a[u].y, ww.y, fmaf(a[u].z, ww.z, fmaf(a[u].w, ww.w, acc[n]))));
        }
      }
    }
  }
#pragma unroll
  for (int n = 0; n < N; ++n) {
#pragma unroll
    for (int o = 1; o < LPP; o <<= 1) acc[n] += __shfl_xor_sync(0xffffffffu, acc[n], o);
  }
  if (live && part == 0) {
    const float dv = div ? __ldg(div + b * div_stride) : 1.f;
#pragma unroll
    for (int n = 0; n < N; ++n) {
      float v = acc[n] + (bias ? __ldg(bias + n) : 0.f);
      const long long oi = (((long long)b * N + n) * H + py) * W + px;
      if (add_nchw) v = __ldg(add_nchw + oi) + v;      // output_skip: pyramid = upsample(pyramid) + conv (ncsnpp.py:341)
      if (div) v = v / dv;
      out_nchw[oi] = v;
    }
  }
}

int launch_conv3x3_small_n(const float* x, const float* w, const float* bias, const float* div, long long div_stride,
                           float* out_nchw, int B, int H, int W, int C, int N, int x_f16, cudaStream_t st, const float* add_nchw) {
  B200_REQUIRE(N >= 1 && N <= 4 && C % (x_f16 ? 64 : 4) == 0, "conv3x3_small_n: N=%d C=%d unsupported", N, C);
  const size_t smem = (size_t)9 * N * C * sizeof(float);
  B200_REQUIRE(smem <= 96 * 1024, "conv3x3_small_n: weights (%zu B) exceed shared memory", smem);
  const bool two = !x_f16 && C <= 32;                     // lanes per output pixel: 2 for short channel vectors, else 8
  const long long total = (long long)B * H * W * (two ? 2 : 8);
  const unsigned blocks = (unsigned)((total + 255) / 256);
#define B200_LAUNCH_SMALLN(NN)                                                                                      \
  do {                                                                                                              \
    if (smem > 48 * 1024)                                                                                           \
      B200_CHECK_CUDA(cudaFuncSetAttribute(conv3x3_small_n_kernel<NN, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    if (two) launch_kernel(conv3x3_small_n_kernel<NN, 2>, dim3(blocks), dim3(256), smem, st, x, w, bias, div, div_stride, out_nchw, B, H, W, C, x_f16, add_nchw); \
    else launch_kernel(conv3x3_small_n_kernel<NN, 8>, dim3(blocks), dim3(256), smem, st, x, w, bias, div, div_stride, out_nchw, B, H, W, C, x_f16, add_nchw); \
  } while (0)
  switch (N) {
    case 1: B200_LAUNCH_SMALLN(1); break;
    case 2: B200_LAUNCH_SMALLN(2); break;
    case 3: B200_LAUNCH_SMALLN(3); break;
    default: B200_LAUNCH_SMALLN(4); break;
  }
#undef B200_LAUNCH_SMALLN
  B200_CHECK_LAUNCH();
  return 0;
}

// ============================================================================
// Attention core for small token counts (T = H*W <= 64, e.g. the 4x4 bottleneck block, or the 8x8, 512-channel one of
// FFHQ-1024): one CTA per image forms logits = q k^T * C^-1/2 (layerspp.py:82), softmax over keys (:83-85) and
// h = P v (:86).  qkv is the [B*T, 3C] output of the fused projection (bias included).  q and k are staged in shared
// memory one slab of Cc channels at a time (Cc = C when everything fits: one slab, the original single-pass order);
// the logits accumulate across slabs; v is read through L2 in the last phase (each element once per CTA).
// ============================================================================
__global__ void __launch_bounds__(256) attn_small_kernel(const float* __restrict__ qkv, float* __restrict__ out,
                                                        int T, int C, int Cc, float scale, int round_out) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  extern __shared__ float sm[];            // q[TQ][Cc] (room for T rows) k[T][Cc] p[TQ][T]
  float* sq = sm; float* sk = sq + T * Cc; float* sp = sk + T * Cc;
  // grid (image, query-row block): few images (the batch-2 1024-pixel network) are split over row blocks so that more
  // than `images` SMs work; every output element is computed by the same instruction sequence whatever the split
  const int b = blockIdx.x, TQ = T / gridDim.y, r0 = blockIdx.y * TQ;
  const float* src = qkv + (long long)b * T * 3 * C;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int c0 = 0; c0 < C; c0 += Cc) {
    __syncthreads();
    for (int i = threadIdx.x; i < T * Cc / 4; i += blockDim.x) {
      const int t = i / (Cc / 4), c = (i % (Cc / 4)) * 4;
      if (t < TQ) *reinterpret_cast<float4*>(sq + t * Cc + c) = __ldg(reinterpret_cast<const float4*>(src + (long long)(r0 + t) * 3 * C + c0 + c));
      *reinterpret_cast<float4*>(sk + t * Cc + c) = __ldg(reinterpret_cast<const float4*>(src + (long long)t * 3 * C + C + c0 + c));
    }
    __syncthreads();
    const bool first = c0 == 0, last = c0 + Cc >= C;
    for (int e = warp; e < TQ * T; e += nw) {         // one warp per logit
      const int i = e / T, j = e % T;
      float a = 0.f;
      for (int c = lane; c < Cc; c += 32) a = fmaf(sq[i * Cc + c], sk[j * Cc + c], a);
      a = warp_sum(a);
      if (lane == 0) {
        const float acc = first ? a : sp[e] + a;
        sp[e] = last ? acc * scale : acc;
      }
    }
  }
  __syncthreads();
  for (int i = warp; i < TQ; i += nw) {             // softmax of row i
    float mx = -INFINITY;
    for (int j = lane; j < T; j += 32) mx = fmaxf(mx, sp[i * T + j]);
    mx = warp_max(mx);
    float sum = 0.f;
    for (int j = lane; j < T; j += 32) { const float ev = expf(sp[i * T + j] - mx); sp[i * T + j] = ev; sum += ev; }
    sum = warp_sum(sum);
    for (int j = lane; j < T; j += 32) sp[i * T + j] = sp[i * T + j] / sum;
  }
  __syncthreads();
  const float* sv = src + 2 * C;                    // v[j][c] at sv[j * 3C + c]
  for (int i = threadIdx.x; i < TQ * C; i += blockDim.x) {
    const int t = i / C, c = i % C;
    float a = 0.f;
    for (int j = 0; j < T; ++j) a = fmaf(sp[t * T + j], __ldg(sv + (long long)j * 3 * C + c), a);
    store_operand1(out, ((long long)b * T + r0 + t) * C + c, a, round_out);
  }
}

// channels per staged slab: the largest C / 2^k (a multiple of 4) whose q, k slabs and the logits fit 160 KB
static int attn_small_slab(int T, int C) {
  int Cc = C;
  while (Cc % 8 == 0 && ((size_t)2 * T * Cc + (size_t)T * T) * sizeof(float) > 160 * 1024) Cc /= 2;
  return Cc;
}
bool attn_small_supported(int T, int C) {
  if (T < 1 || T > 64 || C < 4 || C % 4 != 0) return false;
  const int Cc = attn_small_slab(T, C);
  return C % Cc == 0 && ((size_t)2 * T * Cc + (size_t)T * T) * sizeof(float) <= 160 * 1024;
}

// called at plan time (outside any stream capture): opt in to > 48 KB of dynamic shared memory
int launch_attn_small_configure(int T, int C) {
  B200_REQUIRE(attn_small_supported(T, C), "attn_small: T=%d C=%d unsupported", T, C);
  const size_t smem = ((size_t)2 * T * attn_small_slab(T, C) + (size_t)T * T) * sizeof(float);
  static size_t configured = 0;
  if (smem > 48 * 1024 && smem > configured) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(attn_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = smem;
  }
  return 0;
}

int launch_attn_small(const float* qkv, float* out, int B, int T, int C, float scale, int round_out, cudaStream_t st) {
  B200_REQUIRE(attn_small_supported(T, C), "attn_small: T=%d C=%d unsupported", T, C);
  const int Cc = attn_small_slab(T, C);
  const size_t smem = ((size_t)2 * T * Cc + (size_t)T * T) * sizeof(float);
  int TQ = T;                                       // query rows per CTA
  if (B < 32 && T % 4 == 0) TQ = 4; else if (B < 128 && T % 8 == 0) TQ = 8;
  launch_kernel(attn_small_kernel, dim3(B, T / TQ), dim3(256), smem, st, qkv, out, T, C, Cc, scale, round_out);
  B200_CHECK_LAUNCH();
  return 0;
}

}  // namespace b200
