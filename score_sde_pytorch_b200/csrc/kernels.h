// Internal launch interface between the engine (engine.cu), the C-ABI (api.cu)
// and the kernel translation units.  Every launcher returns 0 on success and has
// already recorded the message for b200_last_error() otherwise.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <algorithm>
#include "common.cuh"

namespace b200 {

// ---- elementwise.cu --------------------------------------------------------
int launch_gn_quad_stats(const float* x, int C, int B, int HW, double* qsums, cudaStream_t st, bool qsums_zeroed = false);
int launch_gn_apply(const float* x1, int C1, const float* x2, int C2, const double* q1, const double* q2,
                    const float* gamma, const float* beta, int B, int HW, int G, float eps, int act,
                    int round_out, float* y, float* raw, cudaStream_t st, int x1_f16 = 0);
int launch_gn_generic(const float* x1, int C1, const float* x2, int C2, const float* gamma, const float* beta, int B, int HW, int G,
                      float eps, int act, int round_out, float* y, float* raw, float* mr_ws, cudaStream_t st);
long long gn_generic_workspace_floats(int B, int HW, int G);   // size of mr_ws
int launch_gn_coeff(int C1, int C2, const double* q1, const double* q2, const float* gamma, const float* beta, int B, int HW,
                    int G, float eps, float* scale, float* shift, cudaStream_t st);
int launch_upfirdn2d(const float* x, const float* kernel_host, float* y, int major, int in_h, int in_w,
                     int minor, int kh, int kw, int up_x, int up_y, int down_x, int down_y,
                     int pad_x0, int pad_x1, int pad_y0, int pad_y1, int round_out, cudaStream_t st);
int launch_fused_bias_act(const float* x, const float* b, const float* ref, float* y, long long n,
                          int step_b, int size_b, int act, int grad, float alpha, float scale,
                          cudaStream_t st);
int launch_softmax_rows(const float* s, float* p, long long rows, int T, float scale, int round_out,
                        cudaStream_t st);
int launch_fourier_embed(const float* sigma, long long sigma_stride, const float* W, int nf, int rows,
                         float* emb, cudaStream_t st, int positional = 0);
int launch_linear_rows(const float* x, long long ldx, const float* W, const float* bias, int rows, int N,
                       int K, int act_in, float* y, long long ldy, cudaStream_t st);
int launch_fill_from_table(const float* table, const int* step, float* dst, int n, cudaStream_t st);
int launch_nhwc_to_nchw(const float* src, float* dst, int B, int HW, int C, cudaStream_t st);
// y = x in tensor-core operand format `mode` (store_operand4: 1 TF32 grid, 2 fp16); n % 4 == 0, 16-byte aligned pointers
int launch_store_operand(const float* x, float* y, long long n, int mode, cudaStream_t st);
// lo (split TF32, round_out 1 only): dst gets hi = rna_tf32(w), lo the same layout of rna_tf32(w - hi)
int launch_pack_weight(const float* src, float* dst, int taps, int O, int I, long long so, long long si,
                       long long stp, int round_out, cudaStream_t st, long long dt = 0, long long dO = 0, float* lo = nullptr);
// split TF32 pair of an fp32 tensor: hi = rna_tf32(x), lo = rna_tf32(x - hi); n % 4 == 0, 16-byte aligned pointers
int launch_split_tf32(const float* x, float* hi, float* lo, long long n, cudaStream_t st);
int launch_im2col3x3_nchw(const float* x, float* patches, int B, int C, int Hin, int Win, int H, int W, int stride,
                          int pad, int mode, cudaStream_t st);
bool attn_small_supported(int T, int C);   // T <= 64 tokens; q / k staged in channel slabs when 2*T*C floats exceed shared memory
int launch_attn_small_configure(int T, int C);
int launch_attn_small(const float* qkv, float* out, int B, int T, int C, float scale, int round_out, cudaStream_t st);
int launch_conv3x3_small_n(const float* x, const float* w, const float* bias, const float* div, long long div_stride,
                           float* out_nchw, int B, int H, int W, int C, int N, int x_f16, cudaStream_t st,
                           const float* add_nchw = nullptr);

// ---- tangent.cu : forward-mode tangents of the nonlinear ops (b200_ncsnpp_jvp) --------------------------------------
// GroupNorm(+SiLU) tangent of a (two-source) NHWC tensor: x = primal input, d = its tangent; the primal statistics come from
// the quad sums q1/q2 or, for groups that are not channel quads, the generic path's mean / rstd table mr (float2 per
// (image, group)).  dy (and draw, the tangent of the input in operand format, optional) are stored in mode round_out (0, 1).
int launch_gn_tangent(const float* x1, const float* d1, int C1, const float* x2, const float* d2, int C2, const double* q1,
                      const double* q2, const float* mr, const float* gamma, const float* beta, int B, int HW, int G, float eps,
                      int act, int round_out, float* dy, float* draw, cudaStream_t st);
// dP = P (scale dS - rowsum(P scale dS)) over rows of length T, written over ds
int launch_softmax_tangent(const float* p, float* ds, long long rows, int T, float scale, int round_out, cudaStream_t st);

// ---- conv_simt.cu : strict-fp32 CUDA-core implicit GEMM (any shape) ---------
struct SimtConv {
  // A operand
  const float* x1; int C1;          // first source (NHWC, or NCHW when in_nchw)
  const float* x2; int C2;          // optional second source, channel-concatenated after x1
  long long ld1, ld2;               // pixel pitch of each source in elements (0 = C1 / C2)
  int in_nchw;                      // x1 is [img][C1][H][W] (network input); x2 must be null
  float in_scale, in_shift;         // a*x+b applied to in-bounds input samples (2x-1 centring)
  int H, W;                         // input spatial size (gemm mode: H=rows per batch, W=1)
  int R, S, stride, pad;            // filter geometry (gemm mode: 1,1,1,0)
  int OH, OW;                       // output spatial size
  int nbatch;                       // images (conv) or batch items (gemm)
  long long a_batch_stride;         // elements between batch items of A (conv: H*W*C per source, implied)
  int a_batched;                    // gemm mode: 0 = A shared by all batch items
  // W operand: [tap][N][Cin] (Cin contiguous), optionally one per batch item
  const float* w; int N; long long w_batch_stride;
  long long w_ld;                   // row pitch of W in elements (0 = Cin)
  // GroupNorm (+ SiLU) applied to the input while it is staged (conv_lowc.cu only): per-(image, concatenated channel)
  // y = fma(x, gn_scale, gn_shift) as written by launch_gn_coeff, then SiLU when gn_act; null = plain input
  const float* gn_scale; const float* gn_shift; int gn_act;
  // GroupNorm quad sums of the stored output, accumulated by the epilogue (conv_lowc.cu only): [image][N/4][2] fp64
  // (sum, sum of squares), zeroed by the caller; null = none
  double* qstats;
  Epilogue epi;
  int dilation;                     // filter taps dilation apart (0 or 1: dense); 'same' convolutions then pad by dilation
};
int launch_conv_simt(const SimtConv& p, cudaStream_t st);

// ---- conv_lowc.cu : few-channel stride-1 3x3 / 1x1 convolutions on warp-level TF32 MMAs (same descriptor) ----
// Cin % 16 == 0, Cout in {16, 32, 64}, H % 8 == 0, W % 32 == 0, NHWC fp32 in and out; operands are rounded to the
// TF32 grid while they are staged.  `conv_lowc_supported` looks at shapes and flags only (usable while planning).
bool conv_lowc_supported(const SimtConv& p);
int launch_conv_lowc(const SimtConv& p, cudaStream_t st);

// ---- gemm_tc.cu : wgmma / TMA implicit GEMM (TF32 or fp16 operands) --------
// TMA tensor map (SWIZZLE_128B unless told otherwise, zero out-of-bounds fill) over fp32 or fp16 elements; also used by
// attn_tc.cu and attn_flash.cu
int encode_map(CUtensorMap* tm, const float* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
               const uint32_t* box, const uint32_t* elem_strides = nullptr, bool f16 = false,
               CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B);
int num_sms();   // of the current device
struct TcGemmPlan;   // opaque, owns the encoded tensor maps
struct TcGemmDesc {
  // A: NHWC activations, values already on the TF32 grid.
  const float* a1; int C1; const float* a2; int C2;     // two-source channel concat (a2 may be null)
  int conv;                 // 1: 4-D box gather with zero halo; 0: plain row-major [rows, K]
  int H, W, nimg;           // conv: OUTPUT spatial size and image count; gemm: unused
  int taps;                 // 9 (3x3) or 1
  int stride;               // conv: 1 (default when 0) or 2 (TMA element strides gather every other pixel)
  int valid_pad;            // conv: 1 = no padding (VALID, input is Hin x Win), 0 = 'same' padding
  int Hin, Win;             // conv: input spatial size (0 = same as H, W)
  long long a_rows;         // gemm: total rows of A; a_ld = row pitch in elements
  long long a_ld;
  int a_batch_rows;         // gemm: rows to advance per batch item (0 = shared)
  // W: [tap][N_total][K_total] row-major (K contiguous), TF32 grid.
  const float* w; int N_total; int K_total; long long w_rows;
  long long w_ld;           // row pitch of W in elements (0 = K_total)
  int w_batch_rows;         // rows to advance per batch item (0 = shared)
  int nbatch; int M_per_batch;   // gemm: rows of output per batch item; conv: nbatch=1, M=nimg*H*W
  // optional extra 1x1 phase accumulated into the same tile (a resblock's skip projection fused into its second
  // 3x3 convolution): out += [a3 | a4] w2^T, w2 = [N_total][C3 + C4]; same spatial size as the output, stride 1
  const float* a3; int C3; const float* a4; int C4; const float* w2;
  int f16;                  // 1: a1..a4, w, w2 hold fp16 elements (wgmma .f16, 64-channel K steps); pitches stay in elements
  int no_halo;              // halo form of the 3x3 mainloop (three W-shifted halo copies per channel chunk instead of nine shifted
                            // tiles): 0 = in the swapped form, 1 = never (same K order either way)
  double* qstats;           // optional GroupNorm quad sums [img][N_total/4][2] accumulated by the epilogue (mode 1)
  Epilogue epi;
  // split TF32 ("3xTF32"): every operand x is the pair hi = rna_tf32(x) (a1..a4, w, w2) and lo = rna_tf32(x - hi) (the
  // *_lo twins, same shape and pitch), and each K step runs three products into one fp32 accumulator:
  // lo_A hi_W + hi_A lo_W + hi_A hi_W (small terms first).  TF32 operands only.
  int split;
  const float *a1_lo, *a2_lo, *a3_lo, *a4_lo, *w_lo, *w2_lo;
  // conv, 3x3 'same' stride 1: filter tap (r, s) reads pixel (y + dilation (r - 1), x + dilation (s - 1)), TMA's
  // out-of-bounds fill being the zero padding (0 or 1: dense).  Dilated filters run the nine-load mainloop only.
  int dilation;
};
int tc_gemm_plan_create(const TcGemmDesc& d, TcGemmPlan** out);
void tc_gemm_plan_destroy(TcGemmPlan* p);
int tc_gemm_launch(const TcGemmPlan* p, cudaStream_t st);
bool tc_gemm_supported(const TcGemmDesc& d, const char** why);
void tc_gemm_set_head(TcGemmPlan* p, float* out_nchw, const float* per_img_div, long long div_stride);   // per-call pointers of the NCHW head
void tc_gemm_set_rowvec_ld(TcGemmPlan* p, long long ld);   // epi.rowvec_ld of a built plan
const char* tc_gemm_form(const TcGemmPlan* p);   // "single256" | "single128" | "swap[-halo]", + " 3xtf32" for split TF32

// ---- attn_tc.cu : fused attention core (logits, softmax, P.V, NIN_3, residual, rescale, quad sums), T=256 x C=256 --
// (TF32 or fp16 operands) and T=256 x C=512 (fp16 operands)
struct TcAttnPlan;
struct TcAttnDesc {
  const float* qk;          // [nimg*T][2C]: q | k rows (TF32 grid)
  const float* vT;          // [nimg][C][T]: v transposed, without its bias (TF32 grid)
  const float* w3;          // [C][C] NIN_3 as [out][in] (TF32 grid)
  const float* bv;          // [C] bias of NIN_2
  const float* b3;          // [C] bias of NIN_3
  const float* x;           // [nimg*T][C] block input (residual)
  float* out;               // [nimg*T][C]
  double* qstats;           // optional GroupNorm quad sums of out
  int nimg, T, C;
  float out_scale;
  int f16;                  // 1: qk, vT, w3 hold fp16 elements
};
bool tc_attn_supported(int T, int C, bool f16);
int tc_attn_plan_create(const TcAttnDesc& d, TcAttnPlan** out);
void tc_attn_plan_destroy(TcAttnPlan* p);
int tc_attn_launch(const TcAttnPlan* p, cudaStream_t st);

// ---- attn_flash.cu : flash-style fp16 attention core O = softmax(q k^T / sqrt(C)) v + b_v (online softmax, the logits
// never leave the chip) for T % 128 == 0, 128 <= T <= 4096, C in {128, 256, 512}.  qk = [nimg*T][2C] (q | k), vT =
// [nimg][C][T] (v^T without b_v), out = [nimg*T][C], all fp16; bv fp32.  The plan is a value (tensor maps + arguments).
struct AttnFlashPlan {
  CUtensorMap tmQ, tmK, tmV;
  const float* bv;
  void* out;
  float logit_scale;        // C^-0.5 * log2(e)
  int nimg, T, C;
};
bool attn_flash_supported(int T, int C);
int attn_flash_plan(const void* qk, const void* vT, const float* bv, void* out, int nimg, int T, int C, AttnFlashPlan* pl);
int attn_flash_launch(const AttnFlashPlan& p, cudaStream_t st);

// ---- ncsnv2.cu : InstanceNorm2dPlus, ELU, the CRP max pool and the MSF bilinear sum (NHWC fp32 activations) ----------
// stats [B][C][2] fp64 (sum, sum of squares over HW), written (not accumulated; no zeroing needed), in a buffer of
// in_stats_doubles(B, HW, C) doubles: large images are summed in up to IN_MAX_SLICES pixel slices, whose partials follow
// the [B][C][2] sums and are added in slice order
constexpr int IN_MAX_SLICES = 32;
long long in_stats_doubles(int B, int HW, int C);
int launch_in_stats(const float* x, int B, int HW, int C, double* stats, cudaStream_t st);
// y = act ? ELU(IN++(x)) : IN++(x) in operand format `mode` (0 fp32, 1 TF32 grid, 2 fp16); C % 4 == 0, C <= 512
int launch_in_apply(const float* x, const double* stats, const float* alpha, const float* gamma, const float* beta, int B,
                    int HW, int C, float eps, int act, int mode, float* y, cudaStream_t st);
int launch_elu_operand(const float* x, float* y, long long n, int mode, cudaStream_t st);
// y = maxpool5x5_s1_p2(x) in operand format `mode`; with add: sum = x + add (fp32)
int launch_maxpool5(const float* x, int B, int H, int W, int C, int mode, float* y, const float* add, float* sum, cudaStream_t st);
// acc += bilinear upsample (align_corners=True) of lo [B][Hl][Wl][C] to H x W
int launch_bilinear_add(const float* lo, int B, int Hl, int Wl, int C, float* acc, int H, int W, cudaStream_t st);

// ---- pc_update.cu -----------------------------------------------------------
struct PhiloxMap {          // torch.randn_like's launch geometry for `numel` elements
  unsigned long long seed;
  long long numel;
  int grid, block;          // torch's grid/block => thread stride for element ownership
  unsigned long long inc;   // Philox offset consumed per randn call
  // torch draws a dense tensor in memory order: with nhwc = 1 the state is channels-last (C x HW images), so draw p
  // lands on the NCHW element of memory position p.  philox_map_init sets nhwc = 0 (contiguous NCHW).
  int nhwc, C;
  long long HW;
};
int philox_map_init(PhiloxMap* m, long long numel, unsigned long long seed);
int launch_randn_torch(const PhiloxMap& m, const unsigned long long* offset_dev, unsigned long long offset_add,
                       float* out, cudaStream_t st);
struct PcStepScalars {       // device tables indexed by the step counter
  const float* score_scale;  // multiplies the network output to give the score (VE: 1, VP: -1/std)
  const float* alpha;        // Langevin alpha_i
  const float* pa;           // predictor: x_mean = pa*x + pb*out
  const float* pb;
  const float* pc;           // x = x_mean + pc*z
};
int launch_pc_norms(const float* out, const float* noise, const PhiloxMap& m, const unsigned long long* offset_dev,
                    const int* step, unsigned long long calls_per_step, unsigned long long call_idx,
                    int B, int per_img, float* norms, float* means, cudaStream_t st);
int launch_langevin_apply(float* x, float* x_mean, const float* out, const float* noise, const PhiloxMap& m,
                          const unsigned long long* offset_dev, const int* step,
                          unsigned long long calls_per_step, unsigned long long call_idx,
                          const float* means, float snr, PcStepScalars sc, cudaStream_t st);
int launch_predictor_apply(float* x, float* x_mean, const float* out, const float* noise, const PhiloxMap& m,
                           const unsigned long long* offset_dev, const int* step,
                           unsigned long long calls_per_step, unsigned long long call_idx,
                           PcStepScalars sc, int add_noise, cudaStream_t st);
struct PcColorTransform {    // decouple(v)_j = sum_i v_i M[i*3+j]; couple uses Minv the same way
  float M[9], Minv[9];
};
// controllable generation's data-consistency blend (inpainting: colorize = 0, no channel transform); cm/cs are the
// device tables of the data marginal's mean coefficient and std, z is the randn_like draw at call `call_idx`
int launch_pc_constrain(float* x, float* x_mean, const float* known, const float* mask, const PhiloxMap& m,
                        const unsigned long long* offset_dev, const int* step,
                        unsigned long long calls_per_step, unsigned long long call_idx,
                        const float* cm, const float* cs, const PcColorTransform& ct, int colorize, int C, long long HW,
                        cudaStream_t st);
struct PcMultistepScalars {  // device tables of the multistep ODE update (b200_pc_config.predictor == 2)
  const float *mq, *mr;      // M = mq*x + mr*out
  const float *pa, *pb, *pm1, *pm2;   // x' = pa*x + pb*M + pm1*M_prev + pm2*M_prev2
};
// hist: three slots of numel floats; step s writes its M into slot s % 3 and reads M_{s-1}, M_{s-2} from the others
int launch_pc_multistep(float* x, float* x_mean, const float* out, float* hist, long long numel, const int* step,
                        PcMultistepScalars sc, cudaStream_t st);
int launch_step_increment(int* step, cudaStream_t st);

}  // namespace b200
