// Device-resident pieces of the probability-flow ODE solver (sampling.py:414-485 and likelihood.py:84-113 in the reference).
//
// The reference integrates dx/dt = f(x,t) - 1/2 g(t)^2 score(x,t) with scipy.integrate.solve_ivp(method=m): the state
// lives in a float64 numpy array on the HOST, every right-hand side copies it to the GPU (as float32), evaluates the
// network, and copies the drift back - two PCIe crossings of the whole state per function evaluation, plus numpy's
// stage arithmetic on one host core.  Here the float64 state, the Runge-Kutta stage derivatives (RK23: 4, RK45: 7,
// DOP853: 13) and all stage / error arithmetic stay in HBM; the host keeps scipy's step-size controller (a handful of
// float64 scalars, score_sde_pytorch_b200/ode.py) and reads back the sum of squares behind the error norm once per
// attempted step (one double; two for DOP853's two error estimators).
//
// Arithmetic follows the reference's: stage states and y_new in float64 (numpy), the network input and the drift in
// float32 with torch's operation order (sde_lib.py:93-100: drift - diffusion^2 * score * 0.5, unfused), the drift widened
// to float64 for the stage sums (scipy's fun wrapper).  Reductions are deterministic (fixed-order two-pass).
#include "kernels.h"
#include "../../include/scoresde_b200.h"

namespace b200 {
namespace {

constexpr int ODE_THREADS = 256;
constexpr int ODE_MAX_BLOCKS = 1024;

// DOP853: 12 stage weights, 13 error weights.  The coefficient loops run unrolled to this bound (guarded by nk) so the
// coefficients are read from the kernel parameters at fixed offsets, not from a per-thread local copy.
constexpr int ODE_MAX_COEF = 16;
struct OdeCoef { double c[ODE_MAX_COEF]; };

// y_stage = y + h * sum_j c[j] K[j];  optional float64 copy (y_new), float32 copy (network input)
__global__ void __launch_bounds__(ODE_THREADS) ode_stage_kernel(const double* __restrict__ y, const double* __restrict__ K,
                                                                long long n, OdeCoef coef, int nk, double h,
                                                                double* __restrict__ y_out, float* __restrict__ x32) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    double acc = 0.0;
#pragma unroll
    for (int j = 0; j < ODE_MAX_COEF; ++j)                                         // np.dot(K[:s].T, a[:s])
      if (j < nk) acc += K[(long long)j * n + i] * coef.c[j];
    const double v = nk ? y[i] + acc * h : y[i];                                   // y + dy, dy = dot * h
    if (y_out) y_out[i] = v;
    if (x32) x32[i] = (float)v;                                                    // .type(torch.float32)
  }
}

// K_s = (double) drift, drift = c_f * x - (g2 * score) * 0.5, score = std > 0 ? -(out / std) : out     (all fp32, unfused)
// scal = {c_f, g2, std}: device scalars produced by the SDE's own torch ops on a one-element tensor (no host sync)
__global__ void __launch_bounds__(ODE_THREADS) ode_drift_kernel(const float* __restrict__ x32, const float* __restrict__ out,
                                                                long long n, const float* __restrict__ scal,
                                                                double* __restrict__ k_out) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const float c_f = scal[0], g2 = scal[1], sd = scal[2];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float score = out[i];
    if (sd > 0.f) score = -__fdiv_rn(score, sd);
    const float drift = __fsub_rn(__fmul_rn(c_f, x32[i]), __fmul_rn(__fmul_rn(g2, score), 0.5f));
    k_out[i] = (double)drift;
  }
}

// k_out[img] = sum_i eps_i * (J_drift eps)_i with (J_drift eps) = c_f * eps - (g2 * dscore) * 0.5, dscore the score's
// tangent (-(jvp / std) for VP / sub-VP, jvp for VE) in the drift kernel's fp32 operation order; one CTA per image,
// fixed-order fp64 reduction
__device__ __forceinline__ void block_sum_to(double v, double* dst);
__global__ void __launch_bounds__(ODE_THREADS) ode_div_kernel(const float* __restrict__ eps, const float* __restrict__ jvp,
                                                              long long per_img, const float* __restrict__ scal,
                                                              double* __restrict__ k_out) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const float c_f = scal[0], g2 = scal[1], sd = scal[2];
  const long long base = (long long)blockIdx.x * per_img;
  double s = 0.0;
  for (long long i = threadIdx.x; i < per_img; i += blockDim.x) {
    const float e = eps[base + i];
    float ds = jvp[base + i];
    if (sd > 0.f) ds = -__fdiv_rn(ds, sd);
    const float jd = __fsub_rn(__fmul_rn(c_f, e), __fmul_rn(__fmul_rn(g2, ds), 0.5f));
    s += (double)e * (double)jd;
  }
  block_sum_to(s, k_out + blockIdx.x);
}

__device__ __forceinline__ void block_sum_to(double v, double* dst) {
  __shared__ double sh[ODE_THREADS / 32];
  v = warp_sum_d(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    double t = threadIdx.x < ODE_THREADS / 32 ? sh[threadIdx.x] : 0.0;
    t = warp_sum_d(t);
    if (threadIdx.x == 0) *dst = t;
  }
}

// block_sum_to for two values at once (one barrier): each sum in block_sum_to's order
__device__ __forceinline__ void block_sum2_to(double a, double b, double* dst_a, double* dst_b) {
  __shared__ double sh[2][ODE_THREADS / 32];
  a = warp_sum_d(a);
  b = warp_sum_d(b);
  if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = a; sh[1][threadIdx.x >> 5] = b; }
  __syncthreads();
  if (threadIdx.x < 32) {
    double ta = threadIdx.x < ODE_THREADS / 32 ? sh[0][threadIdx.x] : 0.0;
    double tb = threadIdx.x < ODE_THREADS / 32 ? sh[1][threadIdx.x] : 0.0;
    ta = warp_sum_d(ta);
    tb = warp_sum_d(tb);
    if (threadIdx.x == 0) { *dst_a = ta; *dst_b = tb; }
  }
}

// partial[b] = sum over this block's elements of ((h * sum_j e[j] K[j][i]) / (atol + max(|y|, |y_new|) * rtol))^2
__global__ void __launch_bounds__(ODE_THREADS) ode_error_kernel(const double* __restrict__ y, const double* __restrict__ y_new,
                                                                const double* __restrict__ K, long long n, OdeCoef e, int nk,
                                                                double h, double rtol, double atol, double* __restrict__ partial) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  double s = 0.0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    double acc = 0.0;
#pragma unroll
    for (int j = 0; j < ODE_MAX_COEF; ++j)
      if (j < nk) acc += K[(long long)j * n + i] * e.c[j];
    const double scale = atol + fmax(fabs(y[i]), fabs(y_new[i])) * rtol;
    const double r = acc * h / scale;
    s += r * r;
  }
  block_sum_to(s, partial + blockIdx.x);
}

// DOP853's two estimators from one read of K: partial5[b] / partial3[b] = sum over this block's elements of
// ((sum_j e5[j] K[j][i]) / scale)^2 / ((sum_j e3[j] K[j][i]) / scale)^2, scale = atol + max(|y|, |y_new|) * rtol
__global__ void __launch_bounds__(ODE_THREADS) ode_error2_kernel(const double* __restrict__ y, const double* __restrict__ y_new,
                                                                 const double* __restrict__ K, long long n, OdeCoef e5,
                                                                 OdeCoef e3, int nk, double rtol, double atol,
                                                                 double* __restrict__ partial5, double* __restrict__ partial3) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  double s5 = 0.0, s3 = 0.0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    double acc5 = 0.0, acc3 = 0.0;
#pragma unroll
    for (int j = 0; j < ODE_MAX_COEF; ++j) {
      if (j < nk) {
        const double k = K[(long long)j * n + i];
        acc5 += k * e5.c[j];
        acc3 += k * e3.c[j];
      }
    }
    const double scale = atol + fmax(fabs(y[i]), fabs(y_new[i])) * rtol;
    const double r5 = acc5 / scale, r3 = acc3 / scale;
    s5 += r5 * r5;
    s3 += r3 * r3;
  }
  block_sum2_to(s5, s3, partial5 + blockIdx.x, partial3 + blockIdx.x);
}

// partial[b] = sum of ((v - v2) / (atol + |y0| * rtol))^2     (v2 optional) : the norms of select_initial_step
__global__ void __launch_bounds__(ODE_THREADS) ode_scaled_sq_kernel(const double* __restrict__ v, const double* __restrict__ v2,
                                                                    const double* __restrict__ y0, long long n, double rtol,
                                                                    double atol, double* __restrict__ partial) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  double s = 0.0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double d = v2 ? v[i] - v2[i] : v[i];
    const double r = d / (atol + fabs(y0[i]) * rtol);
    s += r * r;
  }
  block_sum_to(s, partial + blockIdx.x);
}

__global__ void __launch_bounds__(ODE_THREADS) ode_final_sum_kernel(const double* __restrict__ partial, int nb, double* __restrict__ out) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  double s = 0.0;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) s += partial[i];
  block_sum_to(s, out);
}

int ode_grid(long long n) { return (int)std::max<long long>(1, std::min<long long>((n + ODE_THREADS - 1) / ODE_THREADS, ODE_MAX_BLOCKS)); }

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

int b200_ode_stage_f64(const double* y, const double* k, long long n, const double* coef_host, int nk, double h,
                       double* y_out, float* x32, void* stream) {
  B200_REQUIRE(y && n > 0 && nk >= 0 && nk <= ODE_MAX_COEF && (nk == 0 || (k && coef_host)), "ode_stage: bad argument");
  OdeCoef c; for (int j = 0; j < ODE_MAX_COEF; ++j) c.c[j] = j < nk ? coef_host[j] : 0.0;
  launch_kernel(ode_stage_kernel, dim3(ode_grid(n)), dim3(ODE_THREADS), 0, static_cast<cudaStream_t>(stream), y, k, n, c, nk, h, y_out, x32);
  B200_CHECK_LAUNCH();
  return 0;
}

int b200_ode_drift_f64(const float* x32, const float* net_out, long long n, const float* scalars_dev, double* k_out, void* stream) {
  B200_REQUIRE(x32 && net_out && scalars_dev && k_out && n > 0, "ode_drift: null argument");
  launch_kernel(ode_drift_kernel, dim3(ode_grid(n)), dim3(ODE_THREADS), 0, static_cast<cudaStream_t>(stream), x32, net_out, n, scalars_dev, k_out);
  B200_CHECK_LAUNCH();
  return 0;
}

int b200_ode_div_f64(const float* eps, const float* jvp_out, int nimg, long long per_img, const float* scalars_dev,
                     double* k_out, void* stream) {
  B200_REQUIRE(eps && jvp_out && scalars_dev && k_out && nimg > 0 && per_img > 0, "ode_div: bad argument");
  launch_kernel(ode_div_kernel, dim3(nimg), dim3(ODE_THREADS), 0, static_cast<cudaStream_t>(stream), eps, jvp_out, per_img,
                scalars_dev, k_out);
  B200_CHECK_LAUNCH();
  return 0;
}

// ws[0..7]: results; ws + 8: block partials (two arrays of ODE_MAX_BLOCKS for b200_ode_error_sumsq2_f64)
long long b200_ode_workspace_doubles(void) { return 2 * ODE_MAX_BLOCKS + 8; }

int b200_ode_error_sumsq_f64(const double* y, const double* y_new, const double* k, long long n, const double* e_host, int nk,
                             double h, double rtol, double atol, double* ws, void* stream) {
  B200_REQUIRE(y && y_new && k && e_host && ws && n > 0 && nk > 0 && nk <= ODE_MAX_COEF, "ode_error: bad argument");
  OdeCoef c; for (int j = 0; j < ODE_MAX_COEF; ++j) c.c[j] = j < nk ? e_host[j] : 0.0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int g = ode_grid(n);
  launch_kernel(ode_error_kernel, dim3(g), dim3(ODE_THREADS), 0, st, y, y_new, k, n, c, nk, h, rtol, atol, ws + 8);
  launch_kernel(ode_final_sum_kernel, dim3(1), dim3(ODE_THREADS), 0, st, ws + 8, g, ws);
  B200_CHECK_LAUNCH();
  return 0;
}

int b200_ode_error_sumsq2_f64(const double* y, const double* y_new, const double* k, long long n, const double* e5_host,
                              const double* e3_host, int nk, double rtol, double atol, double* ws, void* stream) {
  B200_REQUIRE(y && y_new && k && e5_host && e3_host && ws && n > 0 && nk > 0 && nk <= ODE_MAX_COEF, "ode_error2: bad argument");
  OdeCoef c5, c3;
  for (int j = 0; j < ODE_MAX_COEF; ++j) { c5.c[j] = j < nk ? e5_host[j] : 0.0; c3.c[j] = j < nk ? e3_host[j] : 0.0; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int g = ode_grid(n);
  double* p5 = ws + 8;
  double* p3 = ws + 8 + ODE_MAX_BLOCKS;
  launch_kernel(ode_error2_kernel, dim3(g), dim3(ODE_THREADS), 0, st, y, y_new, k, n, c5, c3, nk, rtol, atol, p5, p3);
  launch_kernel(ode_final_sum_kernel, dim3(1), dim3(ODE_THREADS), 0, st, p5, g, ws);
  launch_kernel(ode_final_sum_kernel, dim3(1), dim3(ODE_THREADS), 0, st, p3, g, ws + 1);
  B200_CHECK_LAUNCH();
  return 0;
}

int b200_ode_scaled_sumsq_f64(const double* v, const double* v2, const double* y0, long long n, double rtol, double atol,
                              double* ws, void* stream) {
  B200_REQUIRE(v && y0 && ws && n > 0, "ode_scaled_sumsq: bad argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int g = ode_grid(n);
  launch_kernel(ode_scaled_sq_kernel, dim3(g), dim3(ODE_THREADS), 0, st, v, v2, y0, n, rtol, atol, ws + 8);
  launch_kernel(ode_final_sum_kernel, dim3(1), dim3(ODE_THREADS), 0, st, ws + 8, g, ws);
  B200_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
