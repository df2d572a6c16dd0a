// Flash-style fp16 attention core for the attention shapes the fused core (attn_tc.cu) does not cover: T tokens (a
// multiple of 128, 128 .. 4096) x C = 128 / 256 / 512 channels per image.  Per image
//   O = softmax(q k^T / sqrt(C)) v + b_v,   written as fp16 [B*T][C], the operand of the NIN_3 contraction that follows.
// The [T, T] logits never leave the chip: each query row runs over the keys in blocks of 64 with a running max and a
// running sum in fp32 (online softmax), and the unnormalised probabilities feed P.V from registers.
//
// One tile = RT query rows of one image; persistent CTAs, 384 threads:
//   warp 0         TMA producer (one elected lane issues): the tile's Q once, then per key block j the K block
//                  (64 keys x C) and the V^T block (C channels x 64 keys) into two rings of mbarrier-guarded slots;
//   warps 4..11    two MMA warpgroups.  C <= 256: RT = 128, warpgroup g owns query rows 64g .. 64g + 63 and all C
//                  output channels (an m64nC fp32 accumulator, at most 128 registers).  C = 512: RT = 64, both
//                  warpgroups own all 64 rows and warpgroup g the output channels 256g .. 256g + 255, so the
//                  accumulator stays at 128 registers; each warpgroup computes the (same) logits itself.
//   Per key block:  S = Q K^T       m64n64 over C / 64 K steps, A = Q and B = K from shared memory;
//                   m' = max(m, rowmax(S) / sqrt(C)),  P = exp(S / sqrt(C) - m'),  l = l e^(m - m') + rowsum(P),
//                   O = O e^(m - m')  (base-2 exponentials, log2(e) folded into the logit scale);
//                   O += P V        m64nN over 64 keys, A = P (fp16) from registers, B = V^T from shared memory.
//   End of tile:    O / l + b_v rounded to fp16 and stored straight from the fragment.
// As in the fused core, P is rounded to fp16 as the operand while l sums the fp32 values, and the division happens on
// the fp32 accumulator: one rounding per operand.  No atomics: every output element is written by one thread.
//
// Shared memory: Q (RT x C fp16), STAGES K slots and STAGES V^T slots of 64 x C fp16 each, barriers.
//   C = 128: 32 KB + 4 x (16 + 16) KB;  C = 256: 64 KB + 2 x (32 + 32) KB;  C = 512: 64 KB + 1 x (64 + 64) KB.
// Every buffer is a stack of 128-byte-swizzled boxes of 64 fp16 (one 128-byte K block) by rows.

#include "tc_common.cuh"
#include <cmath>
#include <cstring>

namespace b200 {

namespace {

constexpr int FB = 64;   // keys per block (one 128-byte K block of the P.V contraction)

template <int C>
struct FlashSmem {
  static constexpr int RT = C == 512 ? 64 : 128;                  // query rows per tile
  static constexpr int NO = C == 512 ? 256 : C;                   // output channels per warpgroup
  static constexpr int NV = C == 512 ? 256 : C;                   // V^T rows per TMA box (a box has at most 256 rows)
  static constexpr int KCH = C / 64;                              // 128-byte K blocks of the logit contraction
  static constexpr int Q_BYTES = RT * C * 2;
  static constexpr int SLOT = FB * C * 2;                         // one K block or one V^T block
  static constexpr int STAGES = C == 128 ? 4 : C == 256 ? 2 : 1;
  static constexpr int Q = 0;
  static constexpr int KRING = Q_BYTES;
  static constexpr int VRING = KRING + STAGES * SLOT;
  static constexpr int BAR_OFFSET = VRING + STAGES * SLOT;
  static constexpr int TOTAL = BAR_OFFSET + 256 + 1024;
  static_assert(TOTAL <= 232448, "exceeds the 227 KB shared-memory limit of sm_90");
};

// m64 x NO += P (64 keys, fp16 from registers) x V^T block; P's k16 slice t is S fragment columns 16t .. 16t + 15
template <int NO>
__device__ __forceinline__ void pv_product(float (&o)[NO / 2], const uint32_t (&pa)[16], uint64_t vdesc) {
  wgmma_fence();
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const uint32_t a[4] = {pa[4 * t], pa[4 * t + 1], pa[4 * t + 2], pa[4 * t + 3]};
    if constexpr (NO == 256) wgmma_f16_rs_n256(o, a, vdesc + 2 * t, 1);
    else wgmma_f16_rs_n128(o, a, vdesc + 2 * t, 1);
  }
  wgmma_commit();
  wgmma_wait<0>();
}

template <int C>
__global__ void __launch_bounds__(384, 1) attn_flash_kernel(const __grid_constant__ AttnFlashPlan p) {
  using L = FlashSmem<C>;
  constexpr int RT = L::RT, NO = L::NO, KCH = L::KCH, STAGES = L::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* qbuf = smem + L::Q;
  uint8_t* kring = smem + L::KRING;
  uint8_t* vring = smem + L::VRING;
  uint64_t* k_full = reinterpret_cast<uint64_t*>(smem + L::BAR_OFFSET);
  uint64_t* k_empty = k_full + STAGES;
  uint64_t* v_full = k_empty + STAGES;
  uint64_t* v_empty = v_full + STAGES;
  uint64_t* q_full = v_empty + STAGES;
  uint64_t* q_empty = q_full + 1;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&k_full[s], 1); mbar_init(&k_empty[s], 8);     // one arrival per MMA warp
      mbar_init(&v_full[s], 1); mbar_init(&v_empty[s], 8);
    }
    mbar_init(q_full, 1); mbar_init(q_empty, 8);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  pdl_wait(); pdl_trigger();   // prologue done; nothing above touched global memory (common.cuh)
  const int T = p.T, nkb = T / FB, tiles_per_img = T / RT;
  const long long total_tiles = (long long)p.nimg * tiles_per_img;

  if (warp < 4) {
    regs_producer();
    if (warp != 0) return;
    // ======================= TMA producer (whole warp; one elected lane issues) =======================
    const bool issue = elect_one();
    uint32_t ks = 0, kph = 0, vs = 0, vph = 0, qph = 0;
    for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int b = (int)(tile / tiles_per_img), row0 = (int)(tile % tiles_per_img) * RT;
      mbar_wait(q_empty, qph ^ 1);
      if (issue) {
        mbar_expect_tx(q_full, L::Q_BYTES);
        for (int kc = 0; kc < KCH; ++kc) tma_load_2d(&p.tmQ, qbuf + kc * RT * 128, q_full, kc * 64, b * T + row0);
      }
      qph ^= 1;
      for (int j = 0; j < nkb; ++j) {
        mbar_wait(&k_empty[ks], kph ^ 1);
        if (issue) {
          uint8_t* dst = kring + ks * L::SLOT;
          mbar_expect_tx(&k_full[ks], L::SLOT);
          for (int kc = 0; kc < KCH; ++kc) tma_load_2d(&p.tmK, dst + kc * FB * 128, &k_full[ks], C + kc * 64, b * T + j * FB);
        }
        if (++ks == STAGES) { ks = 0; kph ^= 1; }
        mbar_wait(&v_empty[vs], vph ^ 1);
        if (issue) {
          uint8_t* dst = vring + vs * L::SLOT;
          mbar_expect_tx(&v_full[vs], L::SLOT);
          for (int h = 0; h < C / L::NV; ++h) tma_load_2d(&p.tmV, dst + h * L::NV * 128, &v_full[vs], j * FB, b * C + h * L::NV);
        }
        if (++vs == STAGES) { vs = 0; vph ^= 1; }
      }
    }
    return;
  }
  regs_consumer();
  // ======================= MMA warpgroups: logits, online softmax, P.V, final =======================
  const int g = (warp >> 2) - 1, wq = warp & 3;
  const int qrow = C == 512 ? 0 : 64 * g;     // first query row of this warpgroup within the tile
  const int ncol = C == 512 ? 256 * g : 0;    // first output channel of this warpgroup
  const float ls = p.logit_scale;
  uint32_t ks = 0, kph = 0, vs = 0, vph = 0, qph = 0;
  for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int b = (int)(tile / tiles_per_img), row0 = (int)(tile % tiles_per_img) * RT;
    float o[NO / 2];
#pragma unroll
    for (int i = 0; i < NO / 2; ++i) o[i] = 0.f;
    float ma = -INFINITY, mb = -INFINITY, la = 0.f, lb = 0.f;   // running max (scaled logits) and partial row sums
    mbar_wait(q_full, qph);
    qph ^= 1;
    const uint32_t qa = smem_u32(qbuf) + qrow * 128;
#pragma unroll 1
    for (int j = 0; j < nkb; ++j) {
      // ---- S = Q K^T for 64 keys ----
      float s[32];
      mbar_wait(&k_full[ks], kph);
      const uint32_t kb = smem_u32(kring + ks * L::SLOT);
      wgmma_fence();
#pragma unroll
      for (int kc = 0; kc < KCH; ++kc)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_f16_n64(s, make_smem_desc(qa + kc * RT * 128) + 2 * k, make_smem_desc(kb + kc * FB * 128) + 2 * k, (kc | k) != 0);
      wgmma_commit();
      wgmma_wait<0>();
      if (lane == 0) {
        mbar_arrive(&k_empty[ks]);
        if (j == nkb - 1) mbar_arrive(q_empty);   // the next tile's Q may land
      }
      if (++ks == STAGES) { ks = 0; kph ^= 1; }
      // ---- online softmax: rows ra (s[4i], s[4i+1]) and rb (s[4i+2], s[4i+3]) are held by a quad of lanes ----
      float xa = -INFINITY, xb = -INFINITY;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        xa = fmaxf(xa, fmaxf(s[4 * i], s[4 * i + 1]));
        xb = fmaxf(xb, fmaxf(s[4 * i + 2], s[4 * i + 3]));
      }
#pragma unroll
      for (int m = 1; m <= 2; m <<= 1) {
        xa = fmaxf(xa, __shfl_xor_sync(0xffffffffu, xa, m));
        xb = fmaxf(xb, __shfl_xor_sync(0xffffffffu, xb, m));
      }
      const float na = fmaxf(ma, xa * ls), nb = fmaxf(mb, xb * ls);
      const float ca = exp2f(ma - na), cb = exp2f(mb - nb);   // 0 on the first block (ma = -inf)
      ma = na; mb = nb;
      float sa = 0.f, sb = 0.f;
      uint32_t pa[16];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float e0 = exp2f(fmaf(s[4 * i], ls, -na)), e1 = exp2f(fmaf(s[4 * i + 1], ls, -na));
        const float e2 = exp2f(fmaf(s[4 * i + 2], ls, -nb)), e3 = exp2f(fmaf(s[4 * i + 3], ls, -nb));
        sa += e0 + e1; sb += e2 + e3;
        pa[2 * i] = pack_half2(e0, e1);       // (row ra, key 8i + 2(lane % 4)): a[0] / a[2] of k16 slice i / 2
        pa[2 * i + 1] = pack_half2(e2, e3);   // (row rb, same keys):            a[1] / a[3]
      }
      la = fmaf(la, ca, sa); lb = fmaf(lb, cb, sb);
#pragma unroll
      for (int i = 0; i < NO / 8; ++i) { o[4 * i] *= ca; o[4 * i + 1] *= ca; o[4 * i + 2] *= cb; o[4 * i + 3] *= cb; }
      // ---- O += P V ----
      mbar_wait(&v_full[vs], vph);
      pv_product<NO>(o, pa, make_smem_desc(smem_u32(vring + vs * L::SLOT) + ncol * 128));
      if (lane == 0) mbar_arrive(&v_empty[vs]);
      if (++vs == STAGES) { vs = 0; vph ^= 1; }
    }
    // ---- O / l + b_v -> fp16 [B*T][C] ----
#pragma unroll
    for (int m = 1; m <= 2; m <<= 1) {
      la += __shfl_xor_sync(0xffffffffu, la, m);
      lb += __shfl_xor_sync(0xffffffffu, lb, m);
    }
    const float ia = 1.0f / la, ib = 1.0f / lb;
#pragma unroll
    for (int i = 0; i < NO / 8; ++i) { o[4 * i] *= ia; o[4 * i + 1] *= ia; o[4 * i + 2] *= ib; o[4 * i + 3] *= ib; }
    Epilogue ep = {};
    ep.bias = p.bv; ep.scale = 1.f; ep.rows_per_img = T; ep.out = reinterpret_cast<float*>(p.out); ep.ld_out = C;
    const long long gm = (long long)b * T + row0 + qrow + wq * 16;
    frag_rows<NO, false, 2, false>(o, ep, nullptr, C, gm, 16, ncol, lane);
  }
}

}  // namespace

bool attn_flash_supported(int T, int C) {
  return T >= 128 && T <= 4096 && T % 128 == 0 && (C == 128 || C == 256 || C == 512);
}

// Opt in to the large dynamic shared-memory carve-out once, outside any stream capture.
static int flash_configure() {
  static bool configured = false;
  if (configured) return 0;
  B200_CHECK_CUDA(cudaFuncSetAttribute(attn_flash_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, FlashSmem<128>::TOTAL));
  B200_CHECK_CUDA(cudaFuncSetAttribute(attn_flash_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, FlashSmem<256>::TOTAL));
  B200_CHECK_CUDA(cudaFuncSetAttribute(attn_flash_kernel<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, FlashSmem<512>::TOTAL));
  configured = true;
  return 0;
}

int attn_flash_plan(const void* qk, const void* vT, const float* bv, void* out, int nimg, int T, int C, AttnFlashPlan* pl) {
  B200_REQUIRE(attn_flash_supported(T, C),
               "attention_flash_f16: implemented for T a multiple of 128 in [128, 4096] and C in {128, 256, 512} (got T=%d C=%d)", T, C);
  B200_REQUIRE(qk && vT && bv && out && nimg > 0, "attention_flash_f16: null argument or nimg < 1 (T=%d C=%d nimg=%d)", T, C, nimg);
  if (int r = flash_configure()) return r;
  AttnFlashPlan p;
  memset(&p, 0, sizeof(p));
  // [rows][cols] row-major fp16 operand, boxes of one 128-byte K block (64 elements) x box_rows rows
  auto encode = [&](CUtensorMap* tm, const void* base, uint64_t cols, uint64_t rows, uint32_t box_rows) {
    const uint64_t dims[2] = {cols, rows}, str[1] = {cols * 2};
    const uint32_t box[2] = {64u, box_rows};
    return encode_map(tm, static_cast<const float*>(base), 2, dims, str, box, nullptr, true);
  };
  const uint32_t rt = C == 512 ? 64 : 128;
  if (int r = encode(&p.tmQ, qk, 2 * (uint64_t)C, (uint64_t)nimg * T, rt)) return r;
  if (int r = encode(&p.tmK, qk, 2 * (uint64_t)C, (uint64_t)nimg * T, FB)) return r;
  if (int r = encode(&p.tmV, vT, (uint64_t)T, (uint64_t)nimg * C, C == 512 ? 256 : C)) return r;
  p.bv = bv; p.out = out; p.nimg = nimg; p.T = T; p.C = C;
  p.logit_scale = (float)((1.0 / std::sqrt((double)C)) * 1.4426950408889634);
  *pl = p;
  return 0;
}

int attn_flash_launch(const AttnFlashPlan& p, cudaStream_t st) {
  const long long tiles = (long long)p.nimg * (p.T / (p.C == 512 ? 64 : 128));
  const int grid = (int)std::min<long long>(tiles, num_sms());
  if (p.C == 128) launch_kernel(attn_flash_kernel<128>, dim3(grid), dim3(384), FlashSmem<128>::TOTAL, st, p);
  else if (p.C == 256) launch_kernel(attn_flash_kernel<256>, dim3(grid), dim3(384), FlashSmem<256>::TOTAL, st, p);
  else launch_kernel(attn_flash_kernel<512>, dim3(grid), dim3(384), FlashSmem<512>::TOTAL, st, p);
  B200_CHECK_LAUNCH();
  return 0;
}

}  // namespace b200
