// Forward-mode tangent kernels of the network's nonlinear ops (the JVP pass of b200_ncsnpp_jvp).
//
// Every linear op of the network (3x3 / 1x1 / stride-2 convolutions, NIN projections, nearest upsampling, 2x2 mean
// pooling, skip concatenation, residual add and scale) acts on a tangent through the forward kernels the engine already
// has, without bias and without the time-embedding row.  Only GroupNorm(+SiLU) and the attention softmax need their own
// tangent:
//   GroupNorm:  xh = (x - mu) r,  dxh = r (dx - mean_g(dx) - xh mean_g(dx xh)),  dy = gamma dxh
//   SiLU:       s = y sigmoid(y),  ds = dy sigmoid(y) (1 + y (1 - sigmoid(y)))
//   softmax:    P = softmax(scale S),  dP = P (scale dS - rowsum(P scale dS))
// Reductions are deterministic: fixed per-thread order, fp64 accumulation, fixed-order block fold.
#include "common.cuh"
#include "kernels.h"

namespace b200 {
namespace {

constexpr int GNT_THREADS = 256;

// fixed-order sum of two doubles over the block (warp shuffles, then warp 0 folds the per-warp partials in order)
__device__ __forceinline__ double2 block_sum2(double a, double b, double2* sh) {
  a = warp_sum_d(a); b = warp_sum_d(b);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = make_double2(a, b);
  __syncthreads();
  double2 r = make_double2(0.0, 0.0);
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { r.x += sh[w].x; r.y += sh[w].y; }
  return r;
}

// grid (group, image): one CTA walks its group's HW x cpg elements twice (tangent means, then the store).
// Statistics of the primal pass: quad sums q1/q2 (GroupNorm on whole channel quads) or the generic path's
// per-(image, group) mean / rstd table `mr`.
__global__ void __launch_bounds__(GNT_THREADS) gn_tangent_kernel(
    const float* __restrict__ x1, const float* __restrict__ d1, int C1, const float* __restrict__ x2,
    const float* __restrict__ d2, int C2, const double* __restrict__ q1, const double* __restrict__ q2,
    const float2* __restrict__ mr, const float* __restrict__ gamma, const float* __restrict__ beta, int HW, int G,
    float eps, int act, int round_out, float* __restrict__ dy, float* __restrict__ draw) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  __shared__ double2 sh[GNT_THREADS / 32];
  __shared__ float s_mu, s_r;
  const int C = C1 + C2, cpg = C / G, g = blockIdx.x, b = blockIdx.y;
  const long long ib = (long long)b * HW;
  if (threadIdx.x == 0) {
    if (mr) { const float2 m = mr[(long long)b * G + g]; s_mu = m.x; s_r = m.y; }
    else {   // same fp64 group sums and fp32 rstd as gn_apply_stream_kernel
      double s = 0.0, ss = 0.0;
      for (int c = g * cpg; c < (g + 1) * cpg; c += 4) {
        const double* src = (c < C1) ? q1 + ((long long)b * (C1 >> 2) + (c >> 2)) * 2
                                     : q2 + ((long long)b * (C2 >> 2) + ((c - C1) >> 2)) * 2;
        s += src[0]; ss += src[1];
      }
      const double inv_n = 1.0 / ((double)HW * cpg), mean = s * inv_n;
      const float var = fmaxf((float)(ss * inv_n - mean * mean), 0.f);
      s_mu = (float)mean; s_r = rsqrtf(var + eps);
    }
  }
  __syncthreads();
  const float mu = s_mu, r = s_r;
  const long long n = (long long)HW * cpg;
  auto at = [&](long long u, const float* a, const float* bb) -> float {
    const long long pix = u / cpg; const int c = g * cpg + (int)(u % cpg);
    return c < C1 ? __ldg(a + (ib + pix) * C1 + c) : __ldg(bb + (ib + pix) * C2 + (c - C1));
  };
  double s1 = 0.0, s2 = 0.0;
  for (long long u = threadIdx.x; u < n; u += blockDim.x) {
    const float xh = (at(u, x1, x2) - mu) * r, dv = at(u, d1, d2);
    s1 += (double)dv; s2 += (double)dv * (double)xh;
  }
  const double2 m = block_sum2(s1, s2, sh);
  const float m1 = (float)(m.x / (double)n), m2 = (float)(m.y / (double)n);
  for (long long u = threadIdx.x; u < n; u += blockDim.x) {
    const long long pix = u / cpg; const int c = g * cpg + (int)(u % cpg);
    const float xh = (at(u, x1, x2) - mu) * r, dv = at(u, d1, d2);
    const float ga = __ldg(gamma + c);
    float t = ga * (r * (dv - m1 - xh * m2));
    if (act) {
      const float y = fmaf(ga, xh, __ldg(beta + c));
      const float sg = 1.0f / (1.0f + expf(-y));
      t = t * sg * (1.0f + y * (1.0f - sg));
    }
    const long long o = (ib + pix) * C + c;
    store_operand1(dy, o, t, round_out);
    if (draw) store_operand1(draw, o, dv, round_out);
  }
}

// one warp per row: dP = P (scale dS - sum_k P scale dS), written over dS
__global__ void __launch_bounds__(256) softmax_tangent_kernel(const float* __restrict__ p, float* __restrict__ ds, long long rows,
                                                             int T, float scale, int round_out) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const int lane = threadIdx.x & 31;
  const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* pr = p + row * T;
  float* dr = ds + row * T;
  float pv[32], dv[32];
  float acc = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int c = lane + j * 32;
    pv[j] = c < T ? pr[c] : 0.f;
    dv[j] = c < T ? dr[c] * scale : 0.f;
    acc = fmaf(pv[j], dv[j], acc);
  }
  acc = warp_sum(acc);
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int c = lane + j * 32;
    if (c < T) {
      const float o = pv[j] * (dv[j] - acc);
      dr[c] = round_out ? round_tf32(o) : o;
    }
  }
}

}  // namespace

int launch_gn_tangent(const float* x1, const float* d1, int C1, const float* x2, const float* d2, int C2, const double* q1,
                      const double* q2, const float* mr, const float* gamma, const float* beta, int B, int HW, int G, float eps,
                      int act, int round_out, float* dy, float* draw, cudaStream_t st) {
  const int C = C1 + C2;
  B200_REQUIRE(C % G == 0 && x1 && d1 && (C2 == 0 || (x2 && d2)), "gn_tangent: C=%d G=%d or missing operand", C, G);
  B200_REQUIRE(mr || (q1 && C1 % 4 == 0 && (C / G) % 4 == 0 && (C2 == 0 || q2)), "gn_tangent: no primal statistics");
  B200_REQUIRE(round_out == 0 || round_out == 1, "gn_tangent: store mode %d (fp16 operands have no tangent pass)", round_out);
  launch_kernel(gn_tangent_kernel, dim3(G, B), dim3(GNT_THREADS), 0, st, x1, d1, C1, x2, d2, C2, q1, q2,
                reinterpret_cast<const float2*>(mr), gamma, beta, HW, G, eps, act, round_out, dy, draw);
  B200_CHECK_LAUNCH();
  return 0;
}

int launch_softmax_tangent(const float* p, float* ds, long long rows, int T, float scale, int round_out, cudaStream_t st) {
  B200_REQUIRE(T > 0 && T <= 1024, "softmax_tangent: T=%d out of range (1..1024)", T);
  const int wpb = 8;
  launch_kernel(softmax_tangent_kernel, dim3((unsigned)((rows + wpb - 1) / wpb)), dim3(wpb * 32), 0, st, p, ds, rows, T, scale, round_out);
  B200_CHECK_LAUNCH();
  return 0;
}

}  // namespace b200
