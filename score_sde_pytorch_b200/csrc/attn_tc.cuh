// Fused attention core for the 16x16-resolution AttnBlockpp (layerspp.py:74-91) with T = 256 tokens and
// C = 256 channels per image: logits, softmax, P.V, the output projection NIN_3, the residual add, the 1/sqrt(2)
// rescale and the next GroupNorm's quad sums in ONE kernel, so the [T,T] logits / probabilities and the
// attention output never touch HBM.  Included by gemm_tc.cu inside its anonymous namespace (PTX wrappers,
// descriptors, fragment epilogue).
//
// One tile = 128 query rows of one image (two tiles per image); persistent CTAs, 384 threads:
//   warp 0         TMA producer (one elected lane issues): 24 loads per tile through a ring of 48 KB slots
//                  (8 x {Q 128x32 + K 256x32}, 8 x V^T 256x32 keys, 8 x W3 256x32), running ahead across phases;
//   warps 4..11    two MMA warpgroups, warpgroup g owning query rows 64g .. 64g + 63 of the tile, three chained
//                  m64 x n256 x k256 wgmma contractions with the accumulator in registers:
//                    S = Q K^T    then softmax in registers (a row lives in one quad of lanes): E = exp((s-max)/sqrt(C))
//                                 rounded to the operand format into the K-major SWIZZLE_128B operand buffer;
//                    O = E V      (A operand = E from shared memory), then O' = O / rowsum + b_v (softmax rows sum to 1,
//                                 so V's bias is added after P.V) rounded into the same buffer;
//                    Y = O' W3^T  (A operand = O'), then (Y + b_3 + x) / sqrt(2), GroupNorm quad sums, direct stores.
// A warpgroup only reads and writes its own 64 rows of the operand buffer, so it synchronises with itself alone.
//
// Deferred normalisation: the reference rounds nothing; here E (not E/rowsum) is the operand and the division
// happens in fp32 on the accumulator - one rounding per operand, as everywhere else in the engine.

// Operand formats: TF32-grid fp32 (kind::tf32; a 128-byte K block = 32 elements, 8 K blocks per contraction,
// 128 KB operand buffer, 2-stage ring) or fp16 (kind::f16; 64 elements per K block, 4 K blocks, 64 KB operand
// buffer, 3-stage ring).
constexpr int AT_T = 256, AT_C = 256;
template <bool F16>
struct AttnSmem {
  static constexpr int KB = F16 ? 4 : 8;                            // 128-byte K blocks per contraction (K = 256 elements)
  static constexpr int BKA = F16 ? 64 : 32;                         // elements per K block
  static constexpr int PBUF = 0;                                    // KB x (128 rows x 128 B)
  static constexpr int RING = KB * 16384;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + 256 * 128;     // 16 KB + 32 KB
  static constexpr int STAGES = F16 ? 3 : 2;
  static constexpr int BAR_OFFSET = RING + STAGES * STAGE_BYTES;
  static constexpr int TOTAL = BAR_OFFSET + 256 + 1024;
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

// One contraction of the tile: KB ring slots, B operand from the slot, A from the slot (phase 0) or the operand buffer.
template <bool F16>
__device__ __forceinline__ void attn_phase(float (&acc)[128], int ph, uint8_t* ring, uint8_t* pbuf, uint64_t* full_bar,
                                           uint64_t* empty_bar, uint32_t& stage, uint32_t& phase, int g, int lane) {
  using L = AttnSmem<F16>;
  int pend = -1;
#pragma unroll 1
  for (int kc = 0; kc < L::KB; ++kc) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sa = smem_u32(ring + stage * L::STAGE_BYTES);
    const uint32_t a = ph == 0 ? sa : smem_u32(pbuf + kc * 16384);
    wgmma_kstep<256, F16>(acc, make_smem_desc(a + g * (A_STAGE_BYTES / 2)), make_smem_desc(sa + A_STAGE_BYTES), kc);
    wgmma_wait<1>();
    if (lane == 0 && pend >= 0) mbar_arrive(&empty_bar[pend]);
    pend = (int)stage;
    if (++stage == L::STAGES) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  if (lane == 0) mbar_arrive(&empty_bar[pend]);
}

template <bool F16>
__global__ void __launch_bounds__(384, 1) attn_tc_kernel(const __grid_constant__ AttnParams p) {
  using L = AttnSmem<F16>;
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
  constexpr int KB = L::KB;        // K blocks in every phase (C = T = 256 elements)
  constexpr int BKA = L::BKA;

  if (warp < 4) {
    regs_producer();
    if (warp != 0) return;
    // ======================= TMA producer (whole warp; one elected lane issues - see elect_one in gemm_tc.cu) =======================
    const bool issue = elect_one();
    uint32_t stage = 0, phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int b = (int)(tile >> 1), qh = (int)(tile & 1);
      for (int ph = 0; ph < 3; ++ph) {
        for (int kc = 0; kc < KB; ++kc) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = ring + stage * L::STAGE_BYTES;
          uint8_t* sb = sa + A_STAGE_BYTES;
          if (!issue) {
          } else if (ph == 0) {
            mbar_expect_tx(&full_bar[stage], L::STAGE_BYTES);
            tma_load_2d(&p.tmQ, sa, &full_bar[stage], kc * BKA, b * AT_T + qh * BM);
            tma_load_2d(&p.tmK, sb, &full_bar[stage], AT_C + kc * BKA, b * AT_T);
          } else if (ph == 1) {
            mbar_expect_tx(&full_bar[stage], 256 * 128);
            tma_load_2d(&p.tmVT, sb, &full_bar[stage], kc * BKA, b * AT_C);
          } else {
            mbar_expect_tx(&full_bar[stage], 256 * 128);
            tma_load_2d(&p.tmW3, sb, &full_bar[stage], kc * BKA, 0);
          }
          if (++stage == L::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }
  regs_consumer();
  // ======================= MMA warpgroups: softmax / convert / final =======================
  const int g = (warp >> 2) - 1, wq = warp & 3;
  const int ra = g * 64 + wq * 16 + (lane >> 2), rb = ra + 8;   // the two query rows of the tile this thread holds
  uint32_t stage = 0, phase = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int b = (int)(tile >> 1), qh = (int)(tile & 1);
    float acc[128];
    // ---- S = Q K^T, softmax over each row's 256 logits (a quad of lanes holds a row) ----
    attn_phase<F16>(acc, 0, ring, pbuf, full_bar, empty_bar, stage, phase, g, lane);
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
      pbuf_store2<F16>(pbuf, ra, k, e0, e1);
      pbuf_store2<F16>(pbuf, rb, k, e2, e3);
    }
#pragma unroll
    for (int m = 1; m <= 2; m <<= 1) {
      suma += __shfl_xor_sync(0xffffffffu, suma, m);
      sumb += __shfl_xor_sync(0xffffffffu, sumb, m);
    }
    const float inva = 1.0f / suma, invb = 1.0f / sumb;
    fence_async_smem();                               // E (generic-proxy writes) -> visible to the tensor core
    wg_barrier(g);
    // ---- O = E V;  O' = O / rowsum + b_v -> operand buffer (K = channel) ----
    attn_phase<F16>(acc, 1, ring, pbuf, full_bar, empty_bar, stage, phase, g, lane);
    wg_barrier(g);                                    // every warp of the warpgroup is done reading E
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int ch = 8 * j + 2 * (lane & 3);
      const float2 t = __ldg(reinterpret_cast<const float2*>(p.bv + ch));
      pbuf_store2<F16>(pbuf, ra, ch, fmaf(acc[4 * j], inva, t.x), fmaf(acc[4 * j + 1], inva, t.y));
      pbuf_store2<F16>(pbuf, rb, ch, fmaf(acc[4 * j + 2], invb, t.x), fmaf(acc[4 * j + 3], invb, t.y));
    }
    fence_async_smem();
    wg_barrier(g);
    // ---- Y = O' W3^T;  final: (Y + b_3 + x) * out_scale, quad sums, store ----
    attn_phase<F16>(acc, 2, ring, pbuf, full_bar, empty_bar, stage, phase, g, lane);
    wg_barrier(g);                                    // O' is dead: the next tile's E may overwrite it
    Epilogue ep;
    ep.bias = p.b3; ep.rowvec = nullptr; ep.rowvec_ld = 0; ep.residual = p.x; ep.ld_res = AT_C; ep.per_img_div = nullptr;
    ep.div_stride = 0; ep.scale = p.out_scale; ep.round_tf32 = 0; ep.rows_per_img = AT_T; ep.out = p.out; ep.ld_out = AT_C;
    ep.out_nchw = 0; ep.n_valid = 0;
    const long long gm = (long long)b * AT_T + qh * BM + g * 64 + wq * 16;
    if (p.qstats) frag_rows<256, true, 0, true>(acc, ep, p.qstats, AT_C, gm, 16, 0, lane);
    else frag_rows<256, true, 0, false>(acc, ep, p.qstats, AT_C, gm, 16, 0, lane);
  }
}
