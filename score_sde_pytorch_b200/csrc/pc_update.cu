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
  m->nhwc = 0; m->C = 1; m->HW = 1;
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

// NCHW element that receives draw p (the draw's position in memory), and its inverse
__device__ __forceinline__ long long draw_elem(const PhiloxMap& m, long long p) {
  if (!m.nhwc) return p;
  const long long chw = m.C * m.HW, b = p / chw, r = p - b * chw, hw = r / m.C;
  return b * chw + (r - hw * m.C) * m.HW + hw;
}

__device__ __forceinline__ long long draw_index(const PhiloxMap& m, long long e) {
  if (!m.nhwc) return e;
  const long long chw = m.C * m.HW, b = e / chw, r = e - b * chw, c = r / m.HW;
  return b * chw + (r - c * m.HW) * m.C + c;
}

// noise value of draw e under torch's layout (4x redundant Philox; used by the norm pass and the constraint blend,
// whose per-pixel threads need channels that torch's layout hands to different threads)
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
    const float z = noise ? noise[e] : noise_at(m, off, draw_index(m, e));
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
      const long long p = t + T * ii + 4 * T * l;
      if (p >= m.numel) continue;
      const long long e = draw_elem(m, p);
      const float zz = (add_noise && noise) ? noise[e] : z[ii];
      const float xm = ca * x[e] + cb * out[e];
      if (x_mean) x_mean[e] = xm;
      x[e] = add_noise ? xm + cz * zz : xm;
    }
  }
}

// Data-consistency step of controllable generation (controllable_generation.py:43-52 inpainting, :137-146 colorization),
// one thread per pixel (b, h, w) over its C channels.  In latent space y = decouple(x) (identity when inpainting,
// y_j = sum_i x_i M_ij when colorizing), with a = mean coefficient and s = std of the data marginal at this step:
//   y' = y*(1-m) + (a*known + s*z)*m,  x = couple(y'),  x_mean = couple(decouple(x)*(1-m) + (a*known)*m)
// z is the blend's own torch.randn_like draw, regenerated per element (in the state's memory order: the reference's
// colorization state is the channels-last output of its einsum, see PhiloxMap::nhwc).  Every product and sum is rounded separately
// (no FMA contraction) in the reference's operation order, so the inpainting blend is bit-equal to the eager ops.
__device__ __forceinline__ void mat3(const float* M, const float v[3], float y[3]) {   // y_j = sum_i v_i M[i*3+j]
#pragma unroll
  for (int j = 0; j < 3; ++j)
    y[j] = __fadd_rn(__fadd_rn(__fmul_rn(v[0], M[j]), __fmul_rn(v[1], M[3 + j])), __fmul_rn(v[2], M[6 + j]));
}

__device__ __forceinline__ float blend(float y, float k, float m, float a, float s, float z) {
  return __fadd_rn(__fmul_rn(y, __fsub_rn(1.f, m)), __fmul_rn(__fadd_rn(__fmul_rn(a, k), __fmul_rn(z, s)), m));
}

__device__ __forceinline__ float blend_mean(float y, float k, float m, float a) {
  return __fadd_rn(__fmul_rn(y, __fsub_rn(1.f, m)), __fmul_rn(__fmul_rn(a, k), m));
}

__global__ void __launch_bounds__(256) pc_constrain_kernel(float* __restrict__ x, float* __restrict__ x_mean,
                                                           const float* __restrict__ known, const float* __restrict__ mask,
                                                           PhiloxMap m, const unsigned long long* offset_dev, const int* step,
                                                           unsigned long long cps, unsigned long long cidx,
                                                           const float* __restrict__ cm, const float* __restrict__ cs,
                                                           PcColorTransform ct, int colorize, int C, long long HW) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const int s_idx = step ? *step : 0;
  const float a = cm[s_idx], s = cs[s_idx];
  const unsigned long long off = step_offset(offset_dev, step, cps, cidx, m.inc);
  const long long npix = m.numel / C;
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < npix; p += (long long)gridDim.x * blockDim.x) {
    const long long b = p / HW, hw = p - b * HW;
    const long long e0 = b * C * HW + hw;   // flat NCHW index of channel 0 at this pixel
    if (colorize) {
      float v[3], y[3], k[3], mk[3];
#pragma unroll
      for (int j = 0; j < 3; ++j) { v[j] = x[e0 + j * HW]; k[j] = known[e0 + j * HW]; mk[j] = mask[e0 + j * HW]; }
      mat3(ct.M, v, y);
#pragma unroll
      for (int j = 0; j < 3; ++j) y[j] = blend(y[j], k[j], mk[j], a, s, noise_at(m, off, draw_index(m, e0 + j * HW)));
      mat3(ct.Minv, y, v);                     // x' = couple(y')
#pragma unroll
      for (int j = 0; j < 3; ++j) x[e0 + j * HW] = v[j];
      mat3(ct.M, v, y);                        // decouple(x'), not y': the reference re-derives it from the blended x
#pragma unroll
      for (int j = 0; j < 3; ++j) y[j] = blend_mean(y[j], k[j], mk[j], a);
      mat3(ct.Minv, y, v);
#pragma unroll
      for (int j = 0; j < 3; ++j) x_mean[e0 + j * HW] = v[j];
    } else {
      for (int c = 0; c < C; ++c) {
        const long long e = e0 + c * HW;
        const float k = known[e], mk = mask[e];
        const float xn = blend(x[e], k, mk, a, s, noise_at(m, off, draw_index(m, e)));
        x[e] = xn;
        x_mean[e] = blend_mean(xn, k, mk, a);
      }
    }
  }
}

// Multistep ODE update (b200_pc_config.predictor == 2), one element:  M = mq x + mr out,
// x' = pa x + pb M (+ c1 M_prev) (+ c2 M_prev2), every product and sum rounded separately in this order, so an eager fp32
// loop over the same tables reproduces it.  A zero coefficient skips its history term: the slots hold stale values
// (or nothing yet) during the warm-up steps.
__device__ __forceinline__ float multistep_elem(float x, float o, float* m0, const float* m1, const float* m2, float mq,
                                                float mr, float pa, float pb, float c1, float c2) {
  const float M = __fadd_rn(__fmul_rn(mq, x), __fmul_rn(mr, o));
  *m0 = M;
  float xn = __fadd_rn(__fmul_rn(pa, x), __fmul_rn(pb, M));
  if (c1 != 0.f) xn = __fadd_rn(xn, __fmul_rn(c1, *m1));
  if (c2 != 0.f) xn = __fadd_rn(xn, __fmul_rn(c2, *m2));
  return xn;
}

__global__ void __launch_bounds__(256) pc_multistep_kernel(float* __restrict__ x, float* __restrict__ x_mean,
                                                           const float* __restrict__ out, float* __restrict__ hist,
                                                           long long numel, const int* __restrict__ step,
                                                           PcMultistepScalars sc) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  const int s = *step;
  const float mq = sc.mq[s], mr = sc.mr[s], pa = sc.pa[s], pb = sc.pb[s], c1 = sc.pm1[s], c2 = sc.pm2[s];
  float* h0 = hist + (long long)(s % 3) * numel;            // M_s
  const float* h1 = hist + (long long)((s + 2) % 3) * numel; // M_{s-1}
  const float* h2 = hist + (long long)((s + 1) % 3) * numel; // M_{s-2}
  const long long n4 = numel >> 2;   // numel % 4 == 0 (launch_pc_multistep)
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 xv = reinterpret_cast<const float4*>(x)[i], ov = __ldg(reinterpret_cast<const float4*>(out) + i);
    const float4 a = c1 != 0.f ? reinterpret_cast<const float4*>(h1)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 b = c2 != 0.f ? reinterpret_cast<const float4*>(h2)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 m, r;
    r.x = multistep_elem(xv.x, ov.x, &m.x, &a.x, &b.x, mq, mr, pa, pb, c1, c2);
    r.y = multistep_elem(xv.y, ov.y, &m.y, &a.y, &b.y, mq, mr, pa, pb, c1, c2);
    r.z = multistep_elem(xv.z, ov.z, &m.z, &a.z, &b.z, mq, mr, pa, pb, c1, c2);
    r.w = multistep_elem(xv.w, ov.w, &m.w, &a.w, &b.w, mq, mr, pa, pb, c1, c2);
    reinterpret_cast<float4*>(h0)[i] = m;
    reinterpret_cast<float4*>(x)[i] = r;
    if (x_mean) reinterpret_cast<float4*>(x_mean)[i] = r;
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

int launch_pc_constrain(float* x, float* x_mean, const float* known, const float* mask, const PhiloxMap& m,
                        const unsigned long long* offset_dev, const int* step,
                        unsigned long long calls_per_step, unsigned long long call_idx,
                        const float* cm, const float* cs, const PcColorTransform& ct, int colorize, int C, long long HW,
                        cudaStream_t st) {
  B200_REQUIRE(x && x_mean && known && mask && cm && cs, "pc_constrain: null argument");
  B200_REQUIRE(C > 0 && HW > 0 && m.numel % (C * HW) == 0, "pc_constrain: %lld elements are not whole %dx%lld images",
               m.numel, C, HW);
  B200_REQUIRE(!colorize || C == 3, "pc_constrain: colorization needs 3 channels, got %d", C);
  const long long npix = m.numel / C;
  const int grid = (int)std::min<long long>((npix + 255) / 256, 132LL * 16);
  launch_kernel(pc_constrain_kernel, dim3(grid), dim3(256), 0, st, x, x_mean, known, mask, m, offset_dev, step,
                calls_per_step, call_idx, cm, cs, ct, colorize, C, HW);
  B200_CHECK_LAUNCH();
  return 0;
}

int launch_pc_multistep(float* x, float* x_mean, const float* out, float* hist, long long numel, const int* step,
                        PcMultistepScalars sc, cudaStream_t st) {
  B200_REQUIRE(x && out && hist && step && sc.mq && sc.mr && sc.pa && sc.pb && sc.pm1 && sc.pm2,
               "pc_multistep: null argument");
  auto aligned = [](const void* p) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  B200_REQUIRE(aligned(x) && aligned(x_mean) && aligned(out) && aligned(hist) && numel % 4 == 0,
               "pc_multistep: x, x_mean, out and hist must be 16-byte aligned with numel %% 4 == 0 (numel %lld)", numel);
  if (numel == 0) return 0;
  const int grid = (int)std::min<long long>((numel / 4 + 255) / 256, 132LL * 8);
  launch_kernel(pc_multistep_kernel, dim3(grid), dim3(256), 0, st, x, x_mean, out, hist, numel, step, sc);
  B200_CHECK_LAUNCH();
  return 0;
}

int launch_step_increment(int* step, cudaStream_t st) {
  launch_kernel(step_increment_kernel, dim3(1), dim3(1), 0, st, step);
  B200_CHECK_LAUNCH();
  return 0;
}

}  // namespace b200
