// Fused attention core for the 16x16-resolution AttnBlockpp (layerspp.py:74-91) with T = 256 tokens and
// C = 256 channels per image (TF32 or fp16 operands) or C = 512 channels (fp16 operands): logits, softmax, P.V, the
// output projection NIN_3, the residual add, the 1/sqrt(2) rescale and the next GroupNorm's quad sums in ONE kernel, so
// the [T,T] logits / probabilities and the attention output never touch HBM.
//
// One tile = 128 query rows of one image (two tiles per image); persistent CTAs, 384 threads:
//   warp 0         TMA producer (one elected lane issues): one load per 128-byte K block through a ring of 48 KB slots
//                  ({Q 128 rows + K 256 keys}, V^T 256 channels, W3 256 output channels), running ahead across phases;
//   warps 4..11    two MMA warpgroups, warpgroup g owning query rows 64g .. 64g + 63 of the tile, chained
//                  m64 x n256 wgmma contractions with the accumulator in registers:
//                    S = Q K^T    then softmax in registers (a row lives in one quad of lanes): E = exp((s-max)/sqrt(C))
//                                 rounded to the operand format into the K-major SWIZZLE_128B operand buffer;
//                    O = E V      (A operand = E from shared memory), then O' = O / rowsum + b_v (softmax rows sum to 1,
//                                 so V's bias is added after P.V) rounded into the same buffer;
//                    Y = O' W3^T  (A operand = O'), then (Y + b_3 + x) / sqrt(2), GroupNorm quad sums, direct stores.
//                  At C = 512 every product with N = C runs as two n256 halves (an m64n512 accumulator would take 256
//                  registers per thread): O = E V high channel half first, so O'_hi goes to operand K blocks 4..7 while
//                  E still sits in blocks 0..3, then the low half, whose O'_lo overwrites E; Y = O' W3^T one half of the
//                  output columns at a time, each with its own epilogue.
// A warpgroup only reads and writes its own 64 rows of the operand buffer, so it synchronises with itself alone.
//
// Deferred normalisation: the reference rounds nothing; here E (not E/rowsum) is the operand and the division
// happens in fp32 on the accumulator - one rounding per operand, as everywhere else in the engine.

#include "tc_common.cuh"
#include <cmath>
#include <cstring>

namespace b200 {

namespace {

// Operand formats: TF32-grid fp32 (wgmma .tf32; a 128-byte K block = 32 elements) or fp16 (wgmma .f16; 64 elements per
// K block).  The operand buffer holds E (T wide) and O' (C wide, C >= T) for 128 rows: C / BKA K blocks of 16 KB.
//   TF32, C = 256: 8 K blocks (128 KB), 2-stage ring;  fp16, C = 256: 4 K blocks (64 KB), 3-stage ring;
//   fp16, C = 512: 8 K blocks (128 KB), 2-stage ring - the TF32 C = 256 layout.  (TF32 at C = 512 would need 256 KB.)
constexpr int AT_T = 256;
template <bool F16, int C>
struct AttnSmem {
  static constexpr int BKA = F16 ? 64 : 32;                         // elements per K block
  static constexpr int KB = C / BKA;                                // K blocks of a contraction over channels (and of the operand buffer)
  static constexpr int TKB = AT_T / BKA;                            // K blocks of a contraction over tokens
  static constexpr int NH = C / 256;                                // n256 halves of a product with N = C
  static constexpr int PBUF = 0;                                    // KB x (128 rows x 128 B)
  static constexpr int RING = KB * 16384;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + 256 * 128;     // 16 KB + 32 KB
  static constexpr int STAGES = F16 && C == 256 ? 3 : 2;
  static constexpr int BAR_OFFSET = RING + STAGES * STAGE_BYTES;
  static constexpr int TOTAL = BAR_OFFSET + 256 + 1024;
  static_assert(C % 256 == 0 && C >= AT_T, "the operand buffer holds E (T wide) in the K blocks of O' (C wide)");
  static_assert(TOTAL <= 232448, "exceeds the 227 KB shared-memory limit of sm_90");
};

struct AttnParams {
  CUtensorMap tmQ, tmK, tmVT, tmW3;
  const float* bv;          // [C] bias of NIN_2 (added after P.V)
  const float* b3;          // [C] bias of NIN_3
  const float* x;           // [B*T][C] block input (residual)
  float* out;               // [B*T][C]
  double* qstats;           // optional [B][C/4][2]
  float logit_scale;        // C^-0.5 * log2(e)
  float out_scale;          // 1/sqrt(2) with skip_rescale, else 1
  int nimg;
};

// address of 16-byte chunk `c16` (0..7) of row r in K-block kb of the swizzled operand buffer
__device__ __forceinline__ uint8_t* pbuf_chunk(uint8_t* pbuf, int kb, int r, int c16) {
  return pbuf + kb * 16384 + (r >> 3) * 1024 + (r & 7) * 128 + ((c16 ^ (r & 7)) << 4);
}
// write K elements k, k + 1 (k even) of operand row r: TF32-rounded fp32 or fp16
template <bool F16>
__device__ __forceinline__ void pbuf_store2(uint8_t* pbuf, int r, int k, float a, float b) {
  if (F16) {
    const uint32_t sa = smem_u32(pbuf_chunk(pbuf, k >> 6, r, (k & 63) >> 3)) + (k & 7) * 2;
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(sa), "r"(pack_half2(a, b)) : "memory");
  } else {
    const uint32_t sa = smem_u32(pbuf_chunk(pbuf, k >> 5, r, (k & 31) >> 2)) + (k & 3) * 4;
    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(sa), "r"(__float_as_uint(round_tf32(a))), "r"(__float_as_uint(round_tf32(b))) : "memory");
  }
}

// Operand-buffer stores of one thread at C = 512 (fp16): its rows ra and rb = ra + 8 share the swizzle phase ra % 8, so
// column pair j (K elements 8j + 2 (lane % 4) + {0, 1}) of row ra sits at sw[j % 8] + (j / 8) * 16 KB, and of row rb
// 1 KB further.  The eight addresses pass through an opaque move: without it the compiler folds the K-block, row and
// lane offsets into 128 distinct addresses, hoists them out of the tile loop and spills them beside the accumulator.
struct PbufRowsF16 {
  uint32_t sw[8];
  __device__ __forceinline__ void init(uint8_t* pbuf, int ra, int lane) {
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      sw[c] = smem_u32(pbuf_chunk(pbuf, 0, ra, c)) + 4 * (lane & 3);
      asm volatile("mov.b32 %0, %0;" : "+r"(sw[c]));
    }
  }
  __device__ __forceinline__ void store2(int rb, int j, float a, float b) const {
    const uint32_t sa = sw[j & 7] + (j >> 3) * 16384 + rb * 1024;
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(sa), "r"(pack_half2(a, b)) : "memory");
  }
};

// One contraction of the tile: NK ring slots, B operand from the slot, A from the slot (S = Q K^T) or the operand buffer.
template <bool F16, int C, int NK>
__device__ __forceinline__ void attn_phase(float (&acc)[128], bool a_ring, uint8_t* ring, uint8_t* pbuf, uint64_t* full_bar,
                                           uint64_t* empty_bar, uint32_t& stage, uint32_t& phase, int g, int lane) {
  using L = AttnSmem<F16, C>;
  int pend = -1;
#pragma unroll 1
  for (int kc = 0; kc < NK; ++kc) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sa = smem_u32(ring + stage * L::STAGE_BYTES);
    const uint32_t a = a_ring ? sa : smem_u32(pbuf + kc * 16384);
    wgmma_kstep<256, F16>(acc, make_smem_desc(a + g * (A_STAGE_BYTES / 2)), make_smem_desc(sa + A_STAGE_BYTES), kc);
    wgmma_wait<1>();
    if (lane == 0 && pend >= 0) mbar_arrive(&empty_bar[pend]);
    pend = (int)stage;
    if (++stage == L::STAGES) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  if (lane == 0) mbar_arrive(&empty_bar[pend]);
}

template <bool F16, int C>
__global__ void __launch_bounds__(384, 1) attn_tc_kernel(const __grid_constant__ AttnParams p) {
  using L = AttnSmem<F16, C>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* pbuf = smem + L::PBUF;
  uint8_t* ring = smem + L::RING;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + L::STAGES;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp index provably warp-uniform
  if (threadIdx.x == 0) {
    for (int s = 0; s < L::STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }   // one arrival per MMA warp
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  pdl_wait(); pdl_trigger();   // prologue done; nothing above touched global memory (common.cuh)
  const long long total_tiles = 2LL * p.nimg;
  constexpr int KB = L::KB, TKB = L::TKB, NH = L::NH;
  constexpr int BKA = L::BKA;

  if (warp < 4) {
    regs_producer();
    if (warp != 0) return;
    // ======================= TMA producer (whole warp; one elected lane issues - see elect_one in tc_common.cuh) =======================
    const bool issue = elect_one();
    uint32_t stage = 0, phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int b = (int)(tile >> 1), qh = (int)(tile & 1);
      for (int ph = 0; ph < 3; ++ph) {                       // Q K^T, E V, O' W3^T
        for (int h = 0; h < (ph == 0 ? 1 : NH); ++h) {       // n256 halves of E V (high channels first) and O' W3^T
          for (int kc = 0; kc < (ph == 1 ? TKB : KB); ++kc) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* sa = ring + stage * L::STAGE_BYTES;
            uint8_t* sb = sa + A_STAGE_BYTES;
            if (!issue) {
            } else if (ph == 0) {
              mbar_expect_tx(&full_bar[stage], L::STAGE_BYTES);
              tma_load_2d(&p.tmQ, sa, &full_bar[stage], kc * BKA, b * AT_T + qh * BM);
              tma_load_2d(&p.tmK, sb, &full_bar[stage], C + kc * BKA, b * AT_T);
            } else if (ph == 1) {
              mbar_expect_tx(&full_bar[stage], 256 * 128);
              tma_load_2d(&p.tmVT, sb, &full_bar[stage], kc * BKA, b * C + (NH - 1 - h) * 256);
            } else {
              mbar_expect_tx(&full_bar[stage], 256 * 128);
              tma_load_2d(&p.tmW3, sb, &full_bar[stage], kc * BKA, h * 256);
            }
            if (++stage == L::STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }
  regs_consumer();
  // ======================= MMA warpgroups: softmax / convert / final =======================
  const int g = (warp >> 2) - 1, wq = warp & 3;
  const int ra = g * 64 + wq * 16 + (lane >> 2), rb = ra + 8;   // the two query rows of the tile this thread holds
  PbufRowsF16 rows;
  if constexpr (C == 512) rows.init(pbuf, ra, lane);
  // operand-buffer store of K elements k, k + 1 (k = 8j + 2 (lane % 4)) of row r (ra or rb)
  auto store2 = [&](int r, int k, float a, float b) {
    if constexpr (C == 512) rows.store2(r == rb, k >> 3, a, b);
    else pbuf_store2<F16>(pbuf, r, k, a, b);
  };
  uint32_t stage = 0, phase = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int b = (int)(tile >> 1), qh = (int)(tile & 1);
    float acc[128];
    // ---- S = Q K^T, softmax over each row's 256 logits (a quad of lanes holds a row) ----
    attn_phase<F16, C, KB>(acc, true, ring, pbuf, full_bar, empty_bar, stage, phase, g, lane);
    float mxa = -INFINITY, mxb = -INFINITY;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      mxa = fmaxf(mxa, fmaxf(acc[4 * j], acc[4 * j + 1]));
      mxb = fmaxf(mxb, fmaxf(acc[4 * j + 2], acc[4 * j + 3]));
    }
#pragma unroll
    for (int m = 1; m <= 2; m <<= 1) {
      mxa = fmaxf(mxa, __shfl_xor_sync(0xffffffffu, mxa, m));
      mxb = fmaxf(mxb, __shfl_xor_sync(0xffffffffu, mxb, m));
    }
    const float moffa = mxa * p.logit_scale, moffb = mxb * p.logit_scale;
    float suma = 0.f, sumb = 0.f;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int k = 8 * j + 2 * (lane & 3);
      const float e0 = exp2f(fmaf(acc[4 * j], p.logit_scale, -moffa)), e1 = exp2f(fmaf(acc[4 * j + 1], p.logit_scale, -moffa));
      const float e2 = exp2f(fmaf(acc[4 * j + 2], p.logit_scale, -moffb)), e3 = exp2f(fmaf(acc[4 * j + 3], p.logit_scale, -moffb));
      suma += e0 + e1; sumb += e2 + e3;
      store2(ra, k, e0, e1);
      store2(rb, k, e2, e3);
    }
#pragma unroll
    for (int m = 1; m <= 2; m <<= 1) {
      suma += __shfl_xor_sync(0xffffffffu, suma, m);
      sumb += __shfl_xor_sync(0xffffffffu, sumb, m);
    }
    const float inva = 1.0f / suma, invb = 1.0f / sumb;
    fence_async_smem();                               // E (generic-proxy writes) -> visible to the tensor core
    wg_barrier(g);
    // ---- O = E V;  O' = O / rowsum + b_v -> operand buffer (K = channel), one n256 channel half at a time, high half
    //      first: its O' lands in K blocks past E's, so only the last half has to wait for E to die ----
#pragma unroll
    for (int h = NH - 1; h >= 0; --h) {
      attn_phase<F16, C, TKB>(acc, false, ring, pbuf, full_bar, empty_bar, stage, phase, g, lane);
      if (h == 0) wg_barrier(g);                      // every warp of the warpgroup is done reading E
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int ch = 256 * h + 8 * j + 2 * (lane & 3);
        const float2 t = __ldg(reinterpret_cast<const float2*>(p.bv + ch));
        store2(ra, ch, fmaf(acc[4 * j], inva, t.x), fmaf(acc[4 * j + 1], inva, t.y));
        store2(rb, ch, fmaf(acc[4 * j + 2], invb, t.x), fmaf(acc[4 * j + 3], invb, t.y));
      }
    }
    fence_async_smem();
    wg_barrier(g);
    // ---- Y = O' W3^T;  final: (Y + b_3 + x) * out_scale, quad sums, store - one n256 half of the output columns at a time ----
#pragma unroll
    for (int h = 0; h < NH; ++h) {
      attn_phase<F16, C, KB>(acc, false, ring, pbuf, full_bar, empty_bar, stage, phase, g, lane);
      if (h == NH - 1) wg_barrier(g);                 // O' is dead: the next tile's E may overwrite it
      Epilogue ep;
      ep.bias = p.b3; ep.rowvec = nullptr; ep.rowvec_ld = 0; ep.residual = p.x; ep.ld_res = C; ep.per_img_div = nullptr;
      ep.div_stride = 0; ep.scale = p.out_scale; ep.round_tf32 = 0; ep.rows_per_img = AT_T; ep.out = p.out; ep.ld_out = C;
      ep.out_nchw = 0; ep.n_valid = 0;
      const long long gm = (long long)b * AT_T + qh * BM + g * 64 + wq * 16;
      if (p.qstats) frag_rows<256, true, 0, true>(acc, ep, p.qstats, C, gm, 16, 256 * h, lane);
      else frag_rows<256, true, 0, false>(acc, ep, p.qstats, C, gm, 16, 256 * h, lane);
    }
  }
}

}  // namespace

struct TcAttnPlan { AttnParams prm; bool f16; int C; };

bool tc_attn_supported(int T, int C, bool f16) { return T == AT_T && (C == 256 || (C == 512 && f16)); }

// Opt in to the large dynamic shared-memory carve-out once, outside any stream capture.
static int attn_configure() {
  static bool configured = false;
  if (configured) return 0;
  B200_CHECK_CUDA(cudaFuncSetAttribute(attn_tc_kernel<false, 256>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnSmem<false, 256>::TOTAL));
  B200_CHECK_CUDA(cudaFuncSetAttribute(attn_tc_kernel<true, 256>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnSmem<true, 256>::TOTAL));
  B200_CHECK_CUDA(cudaFuncSetAttribute(attn_tc_kernel<true, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnSmem<true, 512>::TOTAL));
  configured = true;
  return 0;
}

int tc_attn_plan_create(const TcAttnDesc& d, TcAttnPlan** out) {
  B200_REQUIRE(tc_attn_supported(d.T, d.C, d.f16 != 0), "attn_tc: only T=256 with C=256, or C=512 with fp16 operands (got T=%d C=%d %s)",
               d.T, d.C, d.f16 ? "fp16" : "tf32");
  B200_REQUIRE(d.qk && d.vT && d.w3 && d.bv && d.b3 && d.x && d.out && d.nimg > 0, "attn_tc: null argument");
  if (int r = attn_configure()) return r;
  AttnParams p;
  memset(&p, 0, sizeof(p));
  const bool f16 = d.f16 != 0;
  const int C = d.C;
  // [rows][cols] row-major operand, boxes of one 128-byte K block x box_rows rows
  auto encode = [&](CUtensorMap* tm, const float* base, uint64_t cols, uint64_t rows, uint32_t box_rows) {
    const uint64_t dims[2] = {cols, rows}, str[1] = {cols * (f16 ? 2 : 4)};
    const uint32_t box[2] = {f16 ? 64u : 32u, box_rows};
    return encode_map(tm, base, 2, dims, str, box, nullptr, f16);
  };
  if (int r = encode(&p.tmQ, d.qk, 2 * (uint64_t)C, (uint64_t)d.nimg * AT_T, BM)) return r;
  if (int r = encode(&p.tmK, d.qk, 2 * (uint64_t)C, (uint64_t)d.nimg * AT_T, 256)) return r;
  if (int r = encode(&p.tmVT, d.vT, AT_T, (uint64_t)d.nimg * C, 256)) return r;
  if (int r = encode(&p.tmW3, d.w3, C, C, 256)) return r;
  p.bv = d.bv; p.b3 = d.b3; p.x = d.x; p.out = d.out; p.qstats = d.qstats; p.nimg = d.nimg;
  p.logit_scale = (float)((1.0 / std::sqrt((double)C)) * 1.4426950408889634);
  p.out_scale = d.out_scale;
  *out = new TcAttnPlan{p, f16, C};
  return 0;
}
void tc_attn_plan_destroy(TcAttnPlan* p) { delete p; }
int tc_attn_launch(const TcAttnPlan* pl, cudaStream_t st) {
  const long long tiles = 2LL * pl->prm.nimg;
  const int grid = (int)std::min<long long>(tiles, num_sms());
  if (pl->C == 512) launch_kernel(attn_tc_kernel<true, 512>, dim3(grid), dim3(384), AttnSmem<true, 512>::TOTAL, st, pl->prm);
  else if (pl->f16) launch_kernel(attn_tc_kernel<true, 256>, dim3(grid), dim3(384), AttnSmem<true, 256>::TOTAL, st, pl->prm);
  else launch_kernel(attn_tc_kernel<false, 256>, dim3(grid), dim3(384), AttnSmem<false, 256>::TOTAL, st, pl->prm);
  B200_CHECK_LAUNCH();
  return 0;
}

}  // namespace b200
