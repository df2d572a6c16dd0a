// Predictor / corrector state updates with the Gaussian noise generated in-kernel.
//
// Reference semantics:
//   LangevinCorrector.update_fn        sampling.py:262-282
//   ReverseDiffusionPredictor.update_fn sampling.py:195-200 (+ sde_lib.py:102-107, 246-254)
//   EulerMaruyamaPredictor.update_fn   sampling.py:181-187 (+ sde_lib.py:93-100)
// each of which draws z = torch.randn_like(x) on the CUDA generator.  To produce the
// same samples as the reference under the same torch.cuda.manual_seed, the noise here
// is generated with the identical counter layout: torch's normal_ kernel launches
// `grid` x 256 threads (grid = min(SMs * (maxThreadsPerSM/256), ceil(numel/256))),
// thread t seeds Philox4x32-10 with (seed, subsequence=t, offset) and for loop l
// writes its four Box-Muller normals to elements t + T*ii + 4*T*l (T = grid*256),
// advancing the generator offset by 4*ceil(numel/(4T)) per call.  Because the noise
// is a pure function of (seed, offset, element) it is recomputed where needed (norm
// pass, update pass) and never touches HBM.
#include "kernels.h"
#include <curand_kernel.h>

namespace b200 {

int philox_map_init(PhiloxMap* m, long long numel, unsigned long long seed) {
  int dev = 0, sms = 0, tpsm = 0;
  B200_CHECK_CUDA(cudaGetDevice(&dev));
  B200_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  B200_CHECK_CUDA(cudaDeviceGetAttribute(&tpsm, cudaDevAttrMaxThreadsPerMultiProcessor, dev));
  const int block = 256;
  long long grid = (numel + block - 1) / block;
  grid = std::min<long long>(grid, (long long)sms * (tpsm / block));
  if (grid < 1) grid = 1;
  m->seed = seed; m->numel = numel; m->grid = (int)grid; m->block = block;
  m->inc = (unsigned long long)((numel - 1) / ((long long)block * grid * 4) + 1) * 4;
  return 0;
}

namespace {

__device__ __forceinline__ float4 philox_normal4(unsigned long long seed, unsigned long long subseq,
                                                 unsigned long long offset) {
  curandStatePhilox4_32_10_t st;
  curand_init(seed, subseq, offset, &st);
  return curand_normal4(&st);
}

__device__ __forceinline__ unsigned long long step_offset(const unsigned long long* offset_dev, const int* step,
                                                          unsigned long long calls_per_step,
                                                          unsigned long long call_idx, unsigned long long inc) {
  const unsigned long long s = step ? (unsigned long long)(*step) : 0ull;
  return *offset_dev + (s * calls_per_step + call_idx) * inc;
}

// noise value of flat element e under torch's layout (4x redundant Philox; used only by the norm pass)
__device__ __forceinline__ float noise_at(const PhiloxMap& m, unsigned long long off, long long e) {
  const long long T = (long long)m.grid * m.block;
  const long long l = e / (4 * T), r = e % (4 * T);
  const int ii = (int)(r / T);
  const float4 z = philox_normal4(m.seed, (unsigned long long)(r % T), off + 4ull * l);
  return ii == 0 ? z.x : ii == 1 ? z.y : ii == 2 ? z.z : z.w;
}

__global__ void __launch_bounds__(256) randn_torch_kernel(PhiloxMap m, const unsigned long long* offset_dev,
                                                          unsigned long long offset_add, float* out) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const long long T = (long long)m.grid * m.block;
  const long long L = (m.numel + 4 * T - 1) / (4 * T);
  const unsigned long long off = *offset_dev + offset_add;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < T * L;
       i += (long long)gridDim.x * blockDim.x) {
    const long long t = i % T, l = i / T;
    const float4 z = philox_normal4(m.seed, (unsigned long long)t, off + 4ull * l);
    const long long e0 = t + 4 * T * l;
    if (e0 < m.numel) out[e0] = z.x;
    if (e0 + T < m.numel) out[e0 + T] = z.y;
    if (e0 + 2 * T < m.numel) out[e0 + 2 * T] = z.z;
    if (e0 + 3 * T < m.numel) out[e0 + 3 * T] = z.w;
  }
}

// One CTA per image: ||out_b||_2 and ||z_b||_2 (sampling.py:276-277, before the batch mean).
__global__ void __launch_bounds__(256) pc_norms_kernel(const float* __restrict__ out, const float* __restrict__ noise,
                                                       PhiloxMap m, const unsigned long long* offset_dev,
                                                       const int* step, unsigned long long cps,
                                                       unsigned long long cidx, int per_img, float* __restrict__ norms) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  __shared__ double red[2][8];
  const int b = blockIdx.x;
  const unsigned long long off = noise ? 0ull : step_offset(offset_dev, step, cps, cidx, m.inc);
  double so = 0.0, sz = 0.0;
  for (int j = threadIdx.x; j < per_img; j += blockDim.x) {
    const long long e = (long long)b * per_img + j;
    const float o = out[e];
    const float z = noise ? noise[e] : noise_at(m, off, e);
    so += (double)o * o;
    sz += (double)z * z;
  }
  so = warp_sum_d(so); sz = warp_sum_d(sz);
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = so; red[1][threadIdx.x >> 5] = sz; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, c = 0.0;
    for (int w = 0; w < 8; ++w) { a += red[0][w]; c += red[1][w]; }
    norms[b] = (float)sqrt(a);
    norms[gridDim.x + b] = (float)sqrt(c);
  }
}

__global__ void __launch_bounds__(256) pc_means_kernel(const float* __restrict__ norms, int B, float* __restrict__ means) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  __shared__ double red[2][8];
  double a = 0.0, c = 0.0;
  for (int i = threadIdx.x; i < B; i += blockDim.x) { a += norms[i]; c += norms[B + i]; }
  a = warp_sum_d(a); c = warp_sum_d(c);
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = a; red[1][threadIdx.x >> 5] = c; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double x = 0.0, y = 0.0;
    for (int w = 0; w < 8; ++w) { x += red[0][w]; y += red[1][w]; }
    means[0] = (float)(x / B);   // mean_b ||out_b||
    means[1] = (float)(y / B);   // mean_b ||z_b||
  }
}

// mode 0: Langevin  x_mean = x + eps*g, x = x_mean + sqrt(2 eps) z, g = score_scale*out,
//                   eps = (snr * mean||z|| / mean||g||)^2 * 2 * alpha
// mode 1: predictor x_mean = pa*x + pb*out, x = x_mean + pc*z   (add_noise=0 -> x = x_mean)
__global__ void __launch_bounds__(256) pc_apply_kernel(float* __restrict__ x, float* __restrict__ x_mean,
                                                       const float* __restrict__ out, const float* __restrict__ noise,
                                                       PhiloxMap m, const unsigned long long* offset_dev, const int* step,
                                                       unsigned long long cps, unsigned long long cidx,
                                                       const float* __restrict__ means, float snr, PcStepScalars sc,
                                                       int mode, int add_noise) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const long long T = (long long)m.grid * m.block;
  const long long L = (m.numel + 4 * T - 1) / (4 * T);
  const int s = step ? *step : 0;
  float ca, cb, cz;
  if (mode == 0) {
    const float ss = sc.score_scale ? sc.score_scale[s] : 1.f;
    const float alpha = sc.alpha ? sc.alpha[s] : 1.f;
    const float grad_norm = fabsf(ss) * means[0], noise_norm = means[1];
    const float r = snr * noise_norm / grad_norm;
    const float eps = r * r * 2.f * alpha;
    ca = 1.f; cb = eps * ss; cz = sqrtf(eps * 2.f);
  } else {
    ca = sc.pa ? sc.pa[s] : 1.f; cb = sc.pb[s]; cz = sc.pc ? sc.pc[s] : 0.f;
  }
  const unsigned long long off = (noise || !add_noise) ? 0ull : step_offset(offset_dev, step, cps, cidx, m.inc);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < T * L;
       i += (long long)gridDim.x * blockDim.x) {
    const long long t = i % T, l = i / T;
    float z[4] = {0.f, 0.f, 0.f, 0.f};
    if (add_noise && !noise) {
      const float4 q = philox_normal4(m.seed, (unsigned long long)t, off + 4ull * l);
      z[0] = q.x; z[1] = q.y; z[2] = q.z; z[3] = q.w;
    }
#pragma unroll
    for (int ii = 0; ii < 4; ++ii) {
      const long long e = t + T * ii + 4 * T * l;
      if (e >= m.numel) continue;
      const float zz = (add_noise && noise) ? noise[e] : z[ii];
      const float xm = ca * x[e] + cb * out[e];
      if (x_mean) x_mean[e] = xm;
      x[e] = add_noise ? xm + cz * zz : xm;
    }
  }
}

__global__ void step_increment_kernel(int* step) { pdl_wait(); pdl_trigger(); *step += 1; }

int apply_grid(const PhiloxMap& m) {
  const long long T = (long long)m.grid * m.block;
  const long long L = (m.numel + 4 * T - 1) / (4 * T);
  return (int)std::min<long long>((T * L + 255) / 256, 132LL * 16);
}

}  // namespace

int launch_randn_torch(const PhiloxMap& m, const unsigned long long* offset_dev, unsigned long long offset_add,
                       float* out, cudaStream_t st) {
  if (m.numel == 0) return 0;
  launch_kernel(randn_torch_kernel, dim3(apply_grid(m)), dim3(256), 0, st, m, offset_dev, offset_add, out);
  B200_CHECK_LAUNCH();
  return 0;
}

int launch_pc_norms(const float* out, const float* noise, const PhiloxMap& m, const unsigned long long* offset_dev,
                    const int* step, unsigned long long calls_per_step, unsigned long long call_idx,
                    int B, int per_img, float* norms, float* means, cudaStream_t st) {
  launch_kernel(pc_norms_kernel, dim3(B), dim3(256), 0, st, out, noise, m, offset_dev, step, calls_per_step, call_idx, per_img, norms);
  B200_CHECK_LAUNCH();
  launch_kernel(pc_means_kernel, dim3(1), dim3(256), 0, st, norms, B, means);
  B200_CHECK_LAUNCH();
  return 0;
}

int launch_langevin_apply(float* x, float* x_mean, const float* out, const float* noise, const PhiloxMap& m,
                          const unsigned long long* offset_dev, const int* step,
                          unsigned long long calls_per_step, unsigned long long call_idx,
                          const float* means, float snr, PcStepScalars sc, cudaStream_t st) {
  launch_kernel(pc_apply_kernel, dim3(apply_grid(m)), dim3(256), 0, st, x, x_mean, out, noise, m, offset_dev, step, calls_per_step,
                                                 call_idx, means, snr, sc, 0, 1);
  B200_CHECK_LAUNCH();
  return 0;
}

int launch_predictor_apply(float* x, float* x_mean, const float* out, const float* noise, const PhiloxMap& m,
                           const unsigned long long* offset_dev, const int* step,
                           unsigned long long calls_per_step, unsigned long long call_idx,
                           PcStepScalars sc, int add_noise, cudaStream_t st) {
  B200_REQUIRE(sc.pb != nullptr, "predictor_apply: pb table missing");
  launch_kernel(pc_apply_kernel, dim3(apply_grid(m)), dim3(256), 0, st, x, x_mean, out, noise, m, offset_dev, step, calls_per_step,
                                                 call_idx, nullptr, 0.f, sc, 1, add_noise);
  B200_CHECK_LAUNCH();
  return 0;
}

int launch_step_increment(int* step, cudaStream_t st) {
  launch_kernel(step_increment_kernel, dim3(1), dim3(1), 0, st, step);
  B200_CHECK_LAUNCH();
  return 0;
}

}  // namespace b200
