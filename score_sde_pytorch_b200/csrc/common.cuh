// Shared helpers for the sm_90a kernels of the score-SDE sampling engine.
// Error reporting follows the C-ABI contract in include/scoresde_b200.h:
// every entry point returns 0 on success, non-zero on failure, and the text is
// available from b200_last_error().
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include <string>
#include <utility>

namespace b200 {

// ---- error plumbing --------------------------------------------------------
void set_error(const char* fmt, ...);           // defined in api.cu
const char* last_error();

#define B200_CHECK_CUDA(expr)                                                        \
  do {                                                                               \
    cudaError_t _e = (expr);                                                         \
    if (_e != cudaSuccess) {                                                         \
      (void)cudaGetLastError(); /* clear the sticky last-error so later launches are not blamed */ \
      ::b200::set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr,           \
                        cudaGetErrorString(_e));                                     \
      return 1;                                                                      \
    }                                                                                \
  } while (0)

#define B200_CHECK_LAUNCH()  B200_CHECK_CUDA(cudaGetLastError())

#define B200_REQUIRE(cond, ...)                                                      \
  do {                                                                               \
    if (!(cond)) {                                                                   \
      ::b200::set_error(__VA_ARGS__);                                                \
      return 2;                                                                      \
    }                                                                                \
  } while (0)

static inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

// ---- device helpers --------------------------------------------------------
__device__ __forceinline__ float round_tf32(float x) {
  // round-to-nearest (ties away) to the 10-bit-mantissa TF32 grid, kept as fp32 bits.
  // wgmma .tf32 ignores the low 13 mantissa bits of its operands; pre-rounding
  // makes that truncation a no-op so the only error is one RN rounding per operand.
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// Operand-grid stores.  Tensors that feed a tensor-core contraction are written by their producer in one of
// three forms, selected by an integer `mode` that travels with the launch:
//   0  fp32 as computed;
//   1  fp32 rounded to the TF32 grid (operands of wgmma .tf32);
//   2  IEEE fp16, round-to-nearest-even (operands of wgmma .f16).  Same 11-bit significand as TF32, half the
//      bytes in HBM and shared memory; `base` then addresses __half elements and `idx` counts halves.
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));   // low half = a, high half = b
  return r;
}
__device__ __forceinline__ void store_operand4(float* base, long long idx, float4 v, int mode) {
  if (mode == 2) {
    uint2 u; u.x = pack_half2(v.x, v.y); u.y = pack_half2(v.z, v.w);
    *reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(base) + idx) = u;
  } else {
    if (mode == 1) { v.x = round_tf32(v.x); v.y = round_tf32(v.y); v.z = round_tf32(v.z); v.w = round_tf32(v.w); }
    *reinterpret_cast<float4*>(base + idx) = v;
  }
}
__device__ __forceinline__ void store_operand1(float* base, long long idx, float v, int mode) {
  if (mode == 2) {
    uint16_t h;
    asm("cvt.rn.f16.f32 %0, %1;" : "=h"(h) : "f"(v));
    reinterpret_cast<uint16_t*>(base)[idx] = h;
  } else {
    base[idx] = mode == 1 ? round_tf32(v) : v;
  }
}

__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }
// SiLU for outputs that are rounded to an 11-bit significand right after (operand modes 1, 2): ex2.approx +
// rcp.approx (relative error ~1e-6, two orders below the rounding) instead of the IEEE exp/divide sequences,
// which made this HBM-streaming kernel instruction-bound (~25 -> ~8 instructions per element).
// (Written out as the two MUFU ops: __fdividef / __expf wrap them in range-scaling code, 9-10 instructions per element
// instead of 5.)
__device__ __forceinline__ float silu_fast(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return x * r;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- programmatic dependent launch (PDL) ---------------------------------------------------------------------------
// Every kernel of this library starts with griddepcontrol.wait - which returns once the preceding kernel of the stream has
// completed and its memory is visible, i.e. ordinary stream order - followed by griddepcontrol.launch_dependents, which
// lets the NEXT kernel's CTAs be scheduled as soon as all of this kernel's CTAs are running.  The tensor-core kernels put
// the pair after their prologue (barrier init), so that prologue and the launch latency of kernel k+1
// overlap the tail of kernel k (464 launches per PC step).  Without the launch attribute both instructions are no-ops.
// Host side: launch_kernel() adds cudaLaunchAttributeProgrammaticStreamSerialization when the calling engine asked for it
// (b200_ncsnpp_config.pdl; a thread-local scope set by the forward / PC-loop entry points - nothing process-global).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
bool pdl_active();                                   // api.cu
struct PdlScope { bool prev; explicit PdlScope(bool on); ~PdlScope(); };
template <typename... KP, typename... A>
inline void launch_kernel(void (*kern)(KP...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at = {};
  at.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at.val.programmaticStreamSerializationAllowed = 1;
  const bool on = pdl_active();
  cfg.attrs = on ? &at : nullptr; cfg.numAttrs = on ? 1 : 0;
  (void)cudaLaunchKernelEx(&cfg, kern, static_cast<KP>(args)...);   // a failure is picked up by B200_CHECK_LAUNCH()
}

// ---- the one contraction descriptor both conv back-ends implement ----------
// out[b][m, n] = epi( sum_{tap, c} A(b, m, tap, c) * W(b)[tap][n][c] )
//   conv mode : m enumerates NHWC pixels of all images, A is the (zero padded,
//               optionally two-source channel-concatenated) input neighbourhood;
//   gemm mode : A is a row-major [rows, K] matrix (optionally batched).
// epi(v) = (v + bias[n] + rowvec[img(m)][n] + residual[m][n]) * scale
//          then / per_img_div[img(m)], then optional TF32 rounding.
struct Epilogue {
  const float* bias;        // [N] or null
  const float* rowvec;      // per-image row vector (time-embedding bias) or null
  long long rowvec_ld;      // stride between images in rowvec (0 = same row for every image)
  const float* residual;    // [M, ld_res] or null
  long long ld_res;
  const float* per_img_div; // [images] divide (scale_by_sigma) or null
  long long div_stride;     // 0 = same divisor for every image
  float scale;              // multiplies after the adds (1/sqrt(2) for skip_rescale)
  int round_tf32;           // store mode of `out`: 0 fp32, 1 fp32 on the TF32 grid, 2 fp16 (see store_operand4)
  int rows_per_img;         // H_out*W_out in conv mode, rows per batch item in gemm mode
  float* out;
  long long ld_out;         // elements between consecutive rows of out (NHWC: C_out_total)
  int out_nchw;             // conv mode only: write [img][n][pix] instead of [m][n]
  int n_valid;              // out_nchw on the tensor-core path: only output channels < n_valid exist (0 = all)
};

}  // namespace b200
