// Strict-fp32 CUDA-core implicit GEMM.  It serves three purposes:
//   * the layers whose shape does not fit the tensor-core tiling (3->128 input conv read
//     straight from NCHW, 128->3 output conv written straight to NCHW with the 1/sigma
//     scaling fused, FIR-padded stride-2 pyramid convs, 4x4-resolution attention);
//   * an exact-fp32 execution mode of the whole network (precision="fp32") used to
//     separate logic errors from TF32 rounding when checking parity with the oracle;
//   * the reference point the tensor-core path is validated against on the device.
// K is walked flat over (tap, channel) so tiny channel counts (Cin=3) do not waste
// the K tile; operands are staged k-major in shared memory and every thread keeps a
// TM x TN register tile.
#include "kernels.h"

namespace b200 {

namespace {

constexpr int BK = 16;

template <int BM, int BN, int TM, int TN>
__global__ void __launch_bounds__(256) conv_simt_kernel(const SimtConv p) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  static_assert((BM / TM) * (BN / TN) == 256, "256 threads per CTA");
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  __shared__ int s_oy[BM], s_ox[BM];

  const int Cin = p.C1 + p.C2;
  const int K = p.R * p.S * Cin;
  const int rows_per_img = p.OH * p.OW;
  const int tiles_m = (rows_per_img + BM - 1) / BM;
  const int tiles_n = (p.N + BN - 1) / BN;
  const long long tiles_total = (long long)p.nbatch * tiles_m * tiles_n;
  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  const long long ld1 = p.ld1 ? p.ld1 : p.C1, ld2 = p.ld2 ? p.ld2 : p.C2, wld = p.w_ld ? p.w_ld : Cin;
  const bool vecA = !p.in_nchw && (p.C1 % 4 == 0) && (p.C2 % 4 == 0) && (ld1 % 4 == 0) && (ld2 % 4 == 0);
  const bool vecB = (Cin % 4 == 0) && (wld % 4 == 0);
  const int dil = p.dilation > 1 ? p.dilation : 1;   // filter tap spacing (the NCSNv2 dilated blocks)

  for (long long tile = blockIdx.x; tile < tiles_total; tile += gridDim.x) {
    const int nt = (int)(tile % tiles_n);
    const int mt = (int)((tile / tiles_n) % tiles_m);
    const int img = (int)(tile / ((long long)tiles_n * tiles_m));
    const int m0 = mt * BM, n0 = nt * BN;
    __syncthreads();
    for (int i = tid; i < BM; i += 256) {
      const int m = m0 + i;
      if (m < rows_per_img) { s_oy[i] = m / p.OW; s_ox[i] = m % p.OW; }
      else { s_oy[i] = -(1 << 20); s_ox[i] = 0; }
    }
    __syncthreads();

    const long long a_img = p.a_batched ? img : 0;
    const float* a1 = p.x1 + a_img * (long long)p.H * p.W * ld1;
    const float* a2 = p.x2 ? p.x2 + a_img * (long long)p.H * p.W * ld2 : nullptr;
    const float* wb = p.w + (long long)img * p.w_batch_stride;

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
      for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < K; k0 += BK) {
      // ---- stage A: BM rows x 16 k (4 consecutive k per item) ----
      for (int e = tid; e < BM * 4; e += 256) {
        const int i = e >> 2, kg = (e & 3) << 2;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        const int kk = k0 + kg;
        const int oy = s_oy[i];
        if (oy >= 0 && kk < K) {
          if (vecA) {
            const int tap = kk / Cin, c = kk % Cin;
            const int iy = oy * p.stride + (tap / p.S) * dil - p.pad, ix = s_ox[i] * p.stride + (tap % p.S) * dil - p.pad;
            if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) {
              const long long pix = (long long)iy * p.W + ix;
              const float4 q = (c < p.C1) ? __ldg(reinterpret_cast<const float4*>(a1 + pix * ld1 + c))
                                          : __ldg(reinterpret_cast<const float4*>(a2 + pix * ld2 + (c - p.C1)));
              v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
            }
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const int k = kk + j;
              if (k >= K) break;
              const int tap = k / Cin, c = k % Cin;
              const int iy = oy * p.stride + (tap / p.S) * dil - p.pad, ix = s_ox[i] * p.stride + (tap % p.S) * dil - p.pad;
              if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) {
                float t;
                if (p.in_nchw) t = __ldg(a1 + ((long long)c * p.H + iy) * p.W + ix);   // same per-image offset
                else if (c < p.C1) t = __ldg(a1 + ((long long)iy * p.W + ix) * ld1 + c);
                else t = __ldg(a2 + ((long long)iy * p.W + ix) * ld2 + (c - p.C1));
                v[j] = t * p.in_scale + p.in_shift;
              }
            }
          }
        }
        As[kg + 0][i] = v[0]; As[kg + 1][i] = v[1]; As[kg + 2][i] = v[2]; As[kg + 3][i] = v[3];
      }
      // ---- stage B: BN cols x 16 k ----
      for (int e = tid; e < BN * 4; e += 256) {
        const int j = e >> 2, kg = (e & 3) << 2;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        const int kk = k0 + kg, n = n0 + j;
        if (n < p.N && kk < K) {
          if (vecB) {
            const int tap = kk / Cin, c = kk % Cin;
            const float4 q = __ldg(reinterpret_cast<const float4*>(wb + ((long long)tap * p.N + n) * wld + c));
            v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
          } else {
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int k = kk + jj;
              if (k >= K) break;
              const int tap = k / Cin, c = k % Cin;
              v[jj] = __ldg(wb + ((long long)tap * p.N + n) * wld + c);
            }
          }
        }
        Bs[kg + 0][j] = v[0]; Bs[kg + 1][j] = v[1]; Bs[kg + 2][j] = v[2]; Bs[kg + 3][j] = v[3];
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < BK; ++k) {
        float a[TM], b[TN];
#pragma unroll
        for (int i = 0; i < TM; ++i) a[i] = As[k][ty * TM + i];
#pragma unroll
        for (int j = 0; j < TN; ++j) b[j] = Bs[k][tx * TN + j];
#pragma unroll
        for (int i = 0; i < TM; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }

    // ---- epilogue ----
    const Epilogue& e = p.epi;
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int m = m0 + ty * TM + i;
      if (m >= rows_per_img) continue;
      const long long gm = (long long)img * rows_per_img + m;   // global output row
      const float dv = e.per_img_div ? __ldg(e.per_img_div + img * e.div_stride) : 1.f;
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        const int n = n0 + tx * TN + j;
        if (n >= p.N) continue;
        float v = acc[i][j];
        if (e.bias) v += __ldg(e.bias + n);
        if (e.rowvec) v += __ldg(e.rowvec + img * e.rowvec_ld + n);
        if (e.residual) v += __ldg(e.residual + gm * e.ld_res + n);
        v *= e.scale;
        if (e.per_img_div) v = v / dv;
        if (e.round_tf32) v = round_tf32(v);
        if (e.out_nchw) e.out[((long long)img * p.N + n) * rows_per_img + m] = v;
        else e.out[gm * e.ld_out + n] = v;
      }
    }
  }
}

}  // namespace

int launch_conv_simt(const SimtConv& p, cudaStream_t st) {
  B200_REQUIRE(p.x1 && p.w && p.epi.out, "conv_simt: null operand");
  B200_REQUIRE(!(p.in_nchw && p.x2), "conv_simt: NCHW input cannot be two-source");
  B200_REQUIRE(!p.gn_scale && !p.qstats, "conv_simt: GroupNorm on load / fused quad sums are implemented by the few-channel kernel only");
  B200_REQUIRE(p.in_nchw || (p.in_scale == 1.f && p.in_shift == 0.f) || (p.C1 % 4 != 0),
               "conv_simt: input affine is only wired for the scalar-load path");
  const int rows_per_img = p.OH * p.OW;
  if (p.N <= 8) {
    constexpr int BM = 256, BN = 8;
    const long long tiles = (long long)p.nbatch * ceil_div(rows_per_img, BM) * ceil_div(p.N, BN);
    const int grid = (int)std::min<long long>(tiles, 132LL * 8);
    launch_kernel(conv_simt_kernel<BM, BN, 1, 8>, dim3(grid), dim3(256), 0, st, p);
  } else {
    constexpr int BM = 64, BN = 64;
    const long long tiles = (long long)p.nbatch * ceil_div(rows_per_img, BM) * ceil_div(p.N, BN);
    const int grid = (int)std::min<long long>(tiles, 132LL * 8);
    launch_kernel(conv_simt_kernel<BM, BN, 4, 4>, dim3(grid), dim3(256), 0, st, p);
  }
  B200_CHECK_LAUNCH();
  return 0;
}

}  // namespace b200
