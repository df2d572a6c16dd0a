// Elementwise and pooling kernels of the NCSNv2 score network (the reference's models/ncsnv2.py, models/layers.py:133-310,
// 453-507, models/normalization.py:157-183), on NHWC fp32 activations:
//   * InstanceNorm2dPlus (+ ELU): per-(image, channel) sums in fp64 by a streaming pass, then one apply pass that derives
//     the channel statistics of its image and writes ELU(IN++(x)) in the operand format of the next contraction;
//   * ELU into an operand format (the RCU blocks' and the CRP block's activations);
//   * the CRP block's 5x5 stride-1 max pool (implicit -inf padding), optionally writing the running sum path + x;
//   * the MSF block's bilinear (align_corners=True) upsample of a half-resolution branch, added into the sum.
#include "kernels.h"

namespace b200 {

namespace {

__device__ __forceinline__ float elu_f(float x) { return x > 0.f ? x : expm1f(x); }   // nn.ELU(alpha=1)

// (sum, sum of squares) in fp64 over the pixels [z * chunk, (z + 1) * chunk) of image b, channel c, written to
// out[((b * gridDim.z + z) * C + c) * 2].  One CTA per (image, 32-channel slice, pixel slice z): lane = channel, the 8
// rows of the CTA stride the pixels, then a fixed-order reduction over the rows.
__global__ void __launch_bounds__(256) in_stats_kernel(const float* __restrict__ x, int C, int HW, int chunk,
                                                       double* __restrict__ out) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  __shared__ double red[2][8][33];
  const int b = blockIdx.x, c = blockIdx.y * 32 + threadIdx.x, z = blockIdx.z;
  const int p0 = z * chunk, p1 = min(HW, p0 + chunk);
  double s = 0.0, ss = 0.0;
  if (c < C) {
    const float* xb = x + (long long)b * HW * C + c;
    for (int p = p0 + threadIdx.y; p < p1; p += 8) {
      const double v = __ldg(xb + (long long)p * C);
      s += v; ss = fma(v, v, ss);
    }
  }
  red[0][threadIdx.y][threadIdx.x] = s; red[1][threadIdx.y][threadIdx.x] = ss;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    double a = 0.0, q = 0.0;
#pragma unroll
    for (int r = 0; r < 8; ++r) { a += red[0][r][threadIdx.x]; q += red[1][r][threadIdx.x]; }
    const long long o = (((long long)b * gridDim.z + z) * C + c) * 2;
    out[o] = a; out[o + 1] = q;
  }
}

// stats[b][c] = the sum of the S pixel-slice partials part[b][0..S-1][c], added in slice order
__global__ void in_stats_reduce_kernel(const double* __restrict__ part, int B, int C, int S, double* __restrict__ stats) {
  pdl_wait(); pdl_trigger();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)B * C; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / C, c = i % C;
    double a = 0.0, q = 0.0;
    for (int z = 0; z < S; ++z) {
      const long long o = ((b * S + z) * C + c) * 2;
      a += part[o]; q += part[o + 1];
    }
    stats[i * 2] = a; stats[i * 2 + 1] = q;
  }
}

// y = act(gamma_c ((x - mu) / sqrt(var + eps) + alpha_c (mu - m) / sqrt(v + eps)) + beta_c), stored in operand format
// `mode`.  m and v (unbiased) are the mean and variance of the channel means mu[b][:]; every CTA of image b derives them
// from the fp64 sums in the same order, so the result does not depend on the grid.
constexpr int IN_MAXC = 512;
__global__ void __launch_bounds__(256) in_apply_kernel(const float* __restrict__ x, const double* __restrict__ stats,
                                                       const float* __restrict__ alpha, const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, int C, int HW, float eps, int act,
                                                       int mode, float* __restrict__ y) {
  pdl_wait(); pdl_trigger();
  __shared__ float s_mu[IN_MAXC], s_sc[IN_MAXC], s_sh[IN_MAXC];
  __shared__ double s_red[256];
  __shared__ double s_m, s_rv;
  const int b = blockIdx.y, tid = threadIdx.x;
  const double inv_n = __drcp_rn((double)HW);   // (reciprocals and rsqrt keep the double division / sqrt slow paths out)
  const double* st = stats + (long long)b * C * 2;
  // m: mean of the channel means
  double a = 0.0;
  for (int c = tid; c < C; c += 256) a += st[2 * c] * inv_n;
  s_red[tid] = a;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) { if (tid < w) s_red[tid] += s_red[tid + w]; __syncthreads(); }
  if (tid == 0) s_m = s_red[0] * __drcp_rn((double)C);
  __syncthreads();
  const double m = s_m;
  a = 0.0;
  for (int c = tid; c < C; c += 256) { const double d = st[2 * c] * inv_n - m; a = fma(d, d, a); }
  __syncthreads();
  s_red[tid] = a;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) { if (tid < w) s_red[tid] += s_red[tid + w]; __syncthreads(); }
  if (tid == 0) s_rv = rsqrt(s_red[0] * __drcp_rn((double)(C - 1)) + (double)eps);   // torch.var: correction 1
  __syncthreads();
  for (int c = tid; c < C; c += 256) {
    const double mu = st[2 * c] * inv_n;
    const double var = fmax(st[2 * c + 1] * inv_n - mu * mu, 0.0);   // biased, as nn.InstanceNorm2d
    const double g = gamma[c];
    s_mu[c] = (float)mu;
    s_sc[c] = (float)(g * rsqrt(var + (double)eps));
    s_sh[c] = (float)(g * alpha[c] * (mu - m) * s_rv + beta[c]);
  }
  __syncthreads();
  const long long n4 = (long long)HW * C / 4;
  const float4* xb = reinterpret_cast<const float4*>(x + (long long)b * HW * C);
  const long long ybase = (long long)b * HW * C;
  for (long long i = blockIdx.x * 256LL + tid; i < n4; i += (long long)gridDim.x * 256) {
    const int c = (int)((i * 4) % C);
    float4 v = __ldg(xb + i);
    v.x = fmaf(v.x - s_mu[c], s_sc[c], s_sh[c]);
    v.y = fmaf(v.y - s_mu[c + 1], s_sc[c + 1], s_sh[c + 1]);
    v.z = fmaf(v.z - s_mu[c + 2], s_sc[c + 2], s_sh[c + 2]);
    v.w = fmaf(v.w - s_mu[c + 3], s_sc[c + 3], s_sh[c + 3]);
    if (act) { v.x = elu_f(v.x); v.y = elu_f(v.y); v.z = elu_f(v.z); v.w = elu_f(v.w); }
    store_operand4(y, ybase + i * 4, v, mode);
  }
}

__global__ void elu_operand_kernel(const float4* __restrict__ x, float* __restrict__ y, long long n4, int mode) {
  pdl_wait(); pdl_trigger();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 v = __ldg(x + i);
    v.x = elu_f(v.x); v.y = elu_f(v.y); v.z = elu_f(v.z); v.w = elu_f(v.w);
    store_operand4(y, 4 * i, v, mode);
  }
}

// nn.MaxPool2d(5, stride=1, padding=2) over NHWC channel quads: out-of-image taps are skipped (the implicit -inf padding).
// With `add`, also sum = x + add at the centre pixel (the CRP block's running x = path + x, fp32).
__global__ void maxpool5_kernel(const float* __restrict__ x, int B, int H, int W, int C, int mode, float* __restrict__ y,
                                const float* __restrict__ add, float* __restrict__ sum) {
  pdl_wait(); pdl_trigger();
  const int C4 = C / 4;
  const long long total = (long long)B * H * W * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    const long long pix = i / C4;
    const int xx = (int)(pix % W), yy = (int)((pix / W) % H);
    const long long img = pix / ((long long)W * H);
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int dy = -2; dy <= 2; ++dy) {
      const int iy = yy + dy;
      if (iy < 0 || iy >= H) continue;
      for (int dx = -2; dx <= 2; ++dx) {
        const int ix = xx + dx;
        if (ix < 0 || ix >= W) continue;
        const float4 v = __ldg(reinterpret_cast<const float4*>(x + ((img * H + iy) * W + ix) * C) + c4);
        m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
      }
    }
    store_operand4(y, i * 4, m, mode);
    if (add) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(x) + i), b = __ldg(reinterpret_cast<const float4*>(add) + i);
      reinterpret_cast<float4*>(sum)[i] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
  }
}

// acc[b][y][x][c] += bilinear(lo)[b][y][x][c], F.interpolate(mode='bilinear', align_corners=True) from Hl x Wl to H x W
// (source coordinate = dst * (in - 1) / (out - 1), as upsample_bilinear2d computes it in fp32)
__global__ void bilinear_add_kernel(const float* __restrict__ lo, int B, int Hl, int Wl, int C, float* __restrict__ acc, int H,
                                    int W) {
  pdl_wait(); pdl_trigger();
  const int C4 = C / 4;
  const float sh = H > 1 ? (float)(Hl - 1) / (float)(H - 1) : 0.f, sw = W > 1 ? (float)(Wl - 1) / (float)(W - 1) : 0.f;
  const long long total = (long long)B * H * W * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    const long long pix = i / C4;
    const int xx = (int)(pix % W), yy = (int)((pix / W) % H);
    const long long img = pix / ((long long)W * H);
    const float ry = sh * yy, rx = sw * xx;
    const int y0 = (int)ry, x0 = (int)rx;
    const int y1 = y0 + (y0 < Hl - 1 ? 1 : 0), x1 = x0 + (x0 < Wl - 1 ? 1 : 0);
    const float ly = ry - y0, lx = rx - x0, hy = 1.f - ly, hx = 1.f - lx;
    auto at = [&](int iy, int ix) { return __ldg(reinterpret_cast<const float4*>(lo + ((img * Hl + iy) * Wl + ix) * C) + c4); };
    const float4 a = at(y0, x0), b = at(y0, x1), c = at(y1, x0), d = at(y1, x1);
    float4 o = reinterpret_cast<float4*>(acc)[i];
    o.x += hy * (hx * a.x + lx * b.x) + ly * (hx * c.x + lx * d.x);
    o.y += hy * (hx * a.y + lx * b.y) + ly * (hx * c.y + lx * d.y);
    o.z += hy * (hx * a.z + lx * b.z) + ly * (hx * c.z + lx * d.z);
    o.w += hy * (hx * a.w + lx * b.w) + ly * (hx * c.w + lx * d.w);
    reinterpret_cast<float4*>(acc)[i] = o;
  }
}

int grid_for(long long items) { return (int)std::max<long long>(1, std::min<long long>((items + 255) / 256, 132LL * 16)); }
bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

// Pixel slices per image: one per 512 pixels, at most IN_MAX_SLICES, so large images (128x128 at batch 1: 32 slices
// instead of one CTA walking 16384 pixels per channel slice) still spread over the SMs.
static int in_stats_slices(int HW) { return std::max(1, std::min(IN_MAX_SLICES, HW / 512)); }

long long in_stats_doubles(int B, int HW, int C) {
  const int S = in_stats_slices(HW);
  return 2LL * B * C * (S > 1 ? 1 + S : 1);
}

int launch_in_stats(const float* x, int B, int HW, int C, double* stats, cudaStream_t st) {
  B200_REQUIRE(x && stats && B > 0 && HW > 0 && C > 0, "in_stats: bad argument");
  const int S = in_stats_slices(HW), chunk = (HW + S - 1) / S;
  double* part = S > 1 ? stats + 2LL * B * C : stats;   // one slice: the CTAs write the sums themselves
  launch_kernel(in_stats_kernel, dim3(B, (C + 31) / 32, S), dim3(32, 8), 0, st, x, C, HW, chunk, part);
  B200_CHECK_LAUNCH();
  if (S > 1) {
    launch_kernel(in_stats_reduce_kernel, dim3(grid_for((long long)B * C)), dim3(256), 0, st, (const double*)part, B, C, S, stats);
    B200_CHECK_LAUNCH();
  }
  return 0;
}

int launch_in_apply(const float* x, const double* stats, const float* alpha, const float* gamma, const float* beta, int B,
                    int HW, int C, float eps, int act, int mode, float* y, cudaStream_t st) {
  B200_REQUIRE(x && stats && alpha && gamma && beta && y, "in_apply: null argument");
  B200_REQUIRE(C % 4 == 0 && C >= 2 && C <= IN_MAXC && aligned16(x) && aligned16(y), "in_apply: C=%d unsupported (multiple of 4, <= %d)",
               C, IN_MAXC);
  B200_REQUIRE(mode >= 0 && mode <= 2, "in_apply: store mode %d unknown", mode);
  const long long n4 = (long long)HW * C / 4;
  const int gx = (int)std::max<long long>(1, std::min<long long>((n4 + 1023) / 1024, std::max(1, 132 * 8 / B)));
  launch_kernel(in_apply_kernel, dim3(gx, B), dim3(256), 0, st, x, stats, alpha, gamma, beta, C, HW, eps, act, mode, y);
  B200_CHECK_LAUNCH();
  return 0;
}

int launch_elu_operand(const float* x, float* y, long long n, int mode, cudaStream_t st) {
  B200_REQUIRE(n % 4 == 0 && aligned16(x) && aligned16(y), "elu_operand: %lld elements / pointer alignment not float4-aligned", n);
  if (n == 0) return 0;
  launch_kernel(elu_operand_kernel, dim3(grid_for(n / 4)), dim3(256), 0, st, reinterpret_cast<const float4*>(x), y, n / 4, mode);
  B200_CHECK_LAUNCH();
  return 0;
}

int launch_maxpool5(const float* x, int B, int H, int W, int C, int mode, float* y, const float* add, float* sum, cudaStream_t st) {
  B200_REQUIRE(x && y && C % 4 == 0 && aligned16(x) && aligned16(y), "maxpool5: C=%d must be a multiple of 4", C);
  B200_REQUIRE(!add == !sum && (!add || (aligned16(add) && aligned16(sum))), "maxpool5: add and sum go together");
  launch_kernel(maxpool5_kernel, dim3(grid_for((long long)B * H * W * C / 4)), dim3(256), 0, st, x, B, H, W, C, mode, y, add, sum);
  B200_CHECK_LAUNCH();
  return 0;
}

int launch_bilinear_add(const float* lo, int B, int Hl, int Wl, int C, float* acc, int H, int W, cudaStream_t st) {
  B200_REQUIRE(lo && acc && C % 4 == 0 && aligned16(lo) && aligned16(acc), "bilinear_add: C=%d must be a multiple of 4", C);
  B200_REQUIRE(Hl >= 1 && Wl >= 1 && H >= Hl && W >= Wl, "bilinear_add: %dx%d -> %dx%d is not an upsample", Hl, Wl, H, W);
  launch_kernel(bilinear_add_kernel, dim3(grid_for((long long)B * H * W * C / 4)), dim3(256), 0, st, lo, B, Hl, Wl, C, acc, H, W);
  B200_CHECK_LAUNCH();
  return 0;
}

}  // namespace b200
