/* scoresde_b200 — C ABI of the score-SDE sampling engine (sm_90a, H100).
 *
 * Drop-in boundary for the native surface of yang-song/score_sde_pytorch on the
 * predictor–corrector sampling path.  Every entry point takes plain pointers and
 * sizes (device pointers unless noted), an explicit CUDA stream (`void*` holding
 * a cudaStream_t; NULL = default stream), never allocates device memory per call
 * (workspaces are sized by a query and supplied by the caller, so calls are
 * CUDA-graph capturable) and returns 0 on success.  On failure the return value
 * is non-zero and b200_last_error() describes it (thread-local).
 *
 * The reference interface each group replaces is cited as file:line relative to
 * the reference repository.
 */
#ifndef SCORESDE_B200_H_
#define SCORESDE_B200_H_

#ifdef __cplusplus
extern "C" {
#endif

#define B200_API __attribute__((visibility("default")))

/* ---- library ---------------------------------------------------------------- */
B200_API const char* b200_last_error(void);
B200_API int b200_version(void);                  /* 10000*major + 100*minor + patch */
B200_API int b200_device_sm_count(int* out);      /* multiProcessorCount of the current device */

/* ---- FIR resampling ----------------------------------------------------------
 * Replaces the pybind11 op `upfirdn2d(Tensor input[major,in_h,in_w,minor], Tensor
 * kernel[kh,kw], up_x, up_y, down_x, down_y, pad_x0, pad_x1, pad_y0, pad_y1)`
 * (op/upfirdn2d.cpp:12-19 -> op/upfirdn2d_kernel.cu:209-369).  Same tensor
 * convention and output size rule (op/upfirdn2d.py:106-107):
 *   out_h = (in_h*up_y + pad_y0 + pad_y1 - kh) / down_y + 1 (likewise out_w).
 * `kernel` is a HOST pointer to kh*kw floats (<= 64 taps).  x/y are device fp32. */
B200_API int b200_upfirdn2d_f32(const float* x, const float* kernel_host, float* y,
                                int major, int in_h, int in_w, int minor, int kh, int kw,
                                int up_x, int up_y, int down_x, int down_y,
                                int pad_x0, int pad_x1, int pad_y0, int pad_y1, void* stream);

/* ---- fused bias + activation -------------------------------------------------
 * Replaces `fused_bias_act(Tensor input, Tensor bias, Tensor refer, int act, int grad,
 * float alpha, float scale)` (op/fused_bias_act.cpp:11-17 -> fused_bias_act_kernel.cu:52-98).
 * y[i] = act(x[i] + b[(i/step_b) % size_b]) * scale; act 1 = linear, 3 = leaky-relu;
 * grad 0/1/2 as in the reference kernel (:36-46).  b / ref may be NULL. */
B200_API int b200_fused_bias_act_f32(const float* x, const float* b, const float* ref, float* y,
                                     long long n, int step_b, int size_b, int act, int grad,
                                     float alpha, float scale, void* stream);

/* ---- GroupNorm(+SiLU), softmax, Gaussian noise: building blocks exported for tests ---- */
B200_API int b200_groupnorm_nhwc_f32(const float* x1, int c1, const float* x2, int c2,
                                     const float* gamma, const float* beta, int batch, int hw, int groups,
                                     float eps, int silu, int round_tf32,
                                     float* stats_ws /* 16*batch*(c1+c2)/4 bytes: fp64 quad sums */,
                                     float* y, float* raw_or_null, void* stream);
B200_API int b200_softmax_rows_f32(const float* s, float* p, long long rows, int t, float scale,
                                   int round_tf32, void* stream);
/* torch.randn-compatible N(0,1) fill: the values torch.randn(numel, device='cuda') would
 * produce for generator state (seed, offset); *offset_inc_out = offset consumed. */
B200_API int b200_randn_like_torch_f32(float* out, long long numel, unsigned long long seed,
                                       unsigned long long offset, unsigned long long* offset_inc_out,
                                       unsigned long long* offset_ws_dev /* 8 B device scratch */, void* stream);

/* ---- one contraction (3x3 / 1x1 convolution on NHWC, 'same' padding, stride 1) ----
 * Exported so the tensor-core path can be checked against the CUDA-core path and torch.
 * w_packed is [taps][c_out][c_in] (see b200_pack_conv_weight_f32). impl: 0 = fp32 CUDA cores,
 * 1 = tensor-core TF32 (inputs must already be TF32-representable for exactness claims),
 * 2 = tensor-core fp16: x1, x2 and w_packed hold IEEE fp16 elements (same layouts; round_tf32 = 2 packs / stores fp16);
 *     out is fp32 unless round_tf32 == 2;
 * 3 = warp-level TF32 MMAs for few-channel layers (c1, c2 multiples of 16, c_out 16 / 32 / 64, h % 8 == 0, w % 32 == 0):
 *     fp32 in and out, operands rounded to the TF32 grid while staged (the 16..64-channel levels of the nf = 16
 *     high-resolution networks, configs/ve/ffhq_ncsnpp_continuous.py:71-94);
 * 4 / 5 = as 1 / 2 with the halo form of the 3x3 mainloop disabled (nine shifted tile loads per channel chunk;
 *     b200_ncsnpp_config.no_halo = 1): A/B checks, bit-identical results. */
B200_API int b200_conv_nhwc_f32(const float* x1, int c1, const float* x2, int c2, int batch, int h, int w,
                                const float* w_packed, const float* bias, int c_out, int ksize,
                                const float* rowvec, long long rowvec_ld, const float* residual, float scale,
                                int round_tf32, float* out, int impl, void* stream);
/* 3x3 convolution with a fused 1x1 skip projection (a BigGAN resblock's tail, layerspp.py:268-274):
 * out = (conv3x3(x; w) + bias + [s1 | s2] w_skip^T + bias_skip + residual) * scale, tensor-core path only.
 * w_skip is [c_out][cs1 + cs2]; s1/s2 are NHWC tensors of the output's spatial size. */
B200_API int b200_conv_skip_nhwc_f32(const float* x, int c, const float* s1, int cs1, const float* s2, int cs2,
                                     int batch, int h, int w, const float* w_packed, const float* bias,
                                     const float* w_skip, const float* bias_skip, int c_out, const float* residual,
                                     float scale, int round_tf32, float* out, void* stream);
/* NCSNv2 building blocks on NHWC fp32 tensors (kernel tests; the engine's family 2 plans the same kernels).
 * Dilated 3x3 'same' convolution (padding = dilation), out = conv + bias (+ residual), stored in mode round_out
 * (0 fp32, 1 TF32 grid, 2 fp16 - tensor-core impls only); w_packed as b200_pack_conv_weight_f32 (ksize 3).
 * impl 0 = CUDA cores (strict fp32), 1 = tensor cores on TF32-grid operands, 2 = tensor cores on fp16 operands. */
B200_API int b200_conv_dilated_nhwc_f32(const float* x, int c, int batch, int h, int w, const float* w_packed, const float* bias,
                                        int c_out, int dilation, const float* residual, int round_out, float* out, int impl,
                                        void* stream);
/* InstanceNorm2dPlus (models/normalization.py:157-183, eps 1e-5) of x [batch][hw][c], then ELU when act, stored in mode
 * round_out; stats_ws holds batch * c * 66 doubles (the [batch][c][2] sums and up to 32 pixel slices of partial sums). */
B200_API int b200_instnorm_plus_nhwc_f32(const float* x, int batch, int hw, int c, const float* alpha, const float* gamma,
                                         const float* beta, int act, int round_out, float* y, double* stats_ws, void* stream);
/* nn.MaxPool2d(5, stride 1, padding 2) of x [batch][h][w][c] into y (mode round_out); with add: sum = x + add */
B200_API int b200_maxpool5_nhwc_f32(const float* x, int batch, int h, int w, int c, int round_out, float* y, const float* add,
                                    float* sum, void* stream);
/* acc [batch][h][w][c] += F.interpolate(lo [batch][hl][wl][c], (h, w), mode='bilinear', align_corners=True) */
B200_API int b200_bilinear_add_nhwc_f32(const float* lo, int batch, int hl, int wl, int c, float* acc, int h, int w, void* stream);
B200_API int b200_pack_conv_weight_f32(const float* w_oihw, float* w_packed, int c_out, int c_in, int ksize,
                                       int round_tf32, void* stream);
/* Fused attention core of AttnBlockpp (layerspp.py:82-91) for T=256 tokens x C=256 channels per image, or T=256 x
 * C=512 with fp16 operands (a TF32 C=512 core is not implemented and returns an error naming shape and format):
 * out = (softmax(q k^T / sqrt(C)) v + b_v) W3^T + b_3 + x) * out_scale, tensor cores only.
 * qk = [nimg*T][2C] (q | k), vT = [nimg][C][T] (v transposed, without b_v), w3 = [C_out][C_in]; TF32-representable
 * fp32 (operand_f16 = 0) or IEEE fp16 elements (operand_f16 = 1).
 * qstats (optional, zero-initialised by the caller) receives out's GroupNorm quad sums [nimg][C/4][2]. */
B200_API int b200_attention_core_f32(const float* qk, const float* vT, const float* w3, const float* bv,
                                     const float* b3, const float* x, float* out, double* qstats, int nimg,
                                     int t, int c, float out_scale, int operand_f16, void* stream);
/* Flash-style fp16 attention core of AttnBlockpp (layerspp.py:82-86) for T tokens (a multiple of 128, 128 <= T <= 4096)
 * x C in {128, 256, 512} channels per image: out = softmax(q k^T / sqrt(C)) v + b_v, with an online softmax (the
 * [T][T] logits never reach memory), tensor cores only.  qk = [nimg*T][2C] (q | k), vT = [nimg][C][T] (v transposed,
 * without b_v), out = [nimg*T][C]: IEEE fp16 elements; bv = [C] fp32.  Other shapes, null pointers and nimg < 1
 * return an error naming the shape.  Deterministic: no atomics. */
B200_API int b200_attention_flash_f16(const void* qk, const void* vT, const float* bv, void* out, int nimg, int t,
                                      int c, void* stream);
/* batched C[b] = A[b] (M x K, pitch lda) * W[b]^T (N x K, pitch ldw), row-major out pitch ldo. */
B200_API int b200_gemm_nt_f32(const float* a, long long lda, int a_batch_rows, const float* w, long long ldw,
                              int w_batch_rows, int nbatch, int m, int n, int k, const float* bias,
                              int round_tf32, float* out, long long ldo, int impl, void* stream);

/* ---- NCSN++ score network ----------------------------------------------------
 * Replaces models/ncsnpp.py:38-381 (+ models/layerspp.py, models/layers.py:29-124,515-555,
 * models/up_or_down_sampling.py, op/) for configurations with Fourier embedding,
 * (or positional) embedding, BigGAN residual blocks, FIR or naive resampling, progressive in {'none','output_skip'}
 * and progressive_input in {'none','residual','input_skip'} (Combine method 'sum').  forward(x[B,C,H,W], time_cond[B]) -> [B,C,H,W]
 * like NCSNpp.forward (models/ncsnpp.py:232).  With family = 1 the same handle type runs the DDPM network
 * (models/ddpm.py:39-181, DDPM.forward :110-181); every entry point below, the PC loop included, works unchanged. */
typedef struct b200_ncsnpp b200_ncsnpp_t;

typedef struct {
  int image_size, num_channels, nf, num_res_blocks;
  int num_levels;  int ch_mult[8];
  int num_attn_resolutions;  int attn_resolutions[8];
  int centered, scale_by_sigma, skip_rescale, conditional;
  int progressive_input;        /* 0 = none, 1 = residual, 2 = input_skip (Combine 'sum', layerspp.py:44-59) */
  int fir_taps;  float fir_kernel[8];   /* separable taps, e.g. {1,3,3,1} */
  int precision;                /* 0 = tensor cores on TF32-rounded fp32 operands where shapes allow, 1 = strict fp32
                                 * CUDA cores, 2 = tensor cores on fp16 operands (same 11-bit significand as TF32,
                                 * fp32 accumulation; activations between layers stay fp32), 3 = split TF32 ("3xTF32"):
                                 * tensor cores on hi + lo pairs of TF32 values (hi = rna_tf32(x), lo = rna_tf32(x - hi)),
                                 * three products per K step (lo*hi + hi*lo + hi*hi) into fp32 accumulators - close to fp32
                                 * accuracy for about 3x the MMA work of 0.  Producers write fp32; a split pass in front of
                                 * each tensor-core contraction makes the pairs of its activation operands ("split 3xtf32"
                                 * ops), the weight blob holds a hi and a lo copy of every contraction weight (so
                                 * b200_ncsnpp_weights_bytes is larger; the parameter table is that of precision 0).
                                 * Attention runs as separate contractions, the few-channel levels of the nf = 16
                                 * networks and the head on CUDA cores; contraction labels carry "3xtf32".  Other values
                                 * are rejected by b200_ncsnpp_create. */
  int keep_activations;         /* debug: never recycle activation buffers so b200_ncsnpp_tap works */
  int lanes;                    /* 0/1: one plan over the whole batch (default); 2: two half-batch plans on two
                                 * streams (batches >= 128).  Off by default. */
  int cuda_core_head;           /* 1: the output convolution (ncsnpp.py:374-380) runs on CUDA cores with an fp32 input in
                                 * every precision mode (costs ~1.4 % of a step, buys back ~1e-4 of rel-L2); 0: tensor cores */
  int embedding_type;          /* 0: Gaussian Fourier features of log(sigma) (layerspp.py:32-41, all_modules[0].W); 1: sinusoidal
                                 * positional embedding of the time label (layers.py:515-529, ncsnpp.py:242-247): no module,
                                 * the frequency table is the pseudo-parameter "pos_freqs" [nf/2] */
  int naive_resample;           /* 0: FIR up/down-sampling in the resblocks (fir=True); 1: nearest-neighbour 2x upsampling and
                                 * 2x2 mean downsampling (fir=False, up_or_down_sampling.py:59-69; the DDPM++ family) */
  int progressive;              /* 0 = none; 1 = output_skip (ncsnpp.py:190-203, 325-341, 366-367): every level adds
                                 * conv3x3(SiLU(GroupNorm(h))) in image channels to the upsampled pyramid, which is the output
                                 * (the high-resolution NCSN++ family: configs/ve/{ffhq,celebahq}_*_ncsnpp_continuous.py) */
  int pdl;                      /* 1: every launch of a forward / PC iteration carries the programmatic-dependent-launch attribute
                                 * (each kernel waits for its predecessor with griddepcontrol.wait after its own prologue, so launch
                                 * latency and barrier init of kernel k+1 overlap the tail of kernel k) */
  int no_halo;                  /* 0 (default): swapped-form 3x3 'same' convolutions on 16- / 32-pixel-wide images read three
                                 * W-shifted halo copies of their tile per channel chunk (csrc/gemm_tc.cu "halo form": 2.4x fewer
                                 * L2 -> shared-memory bytes than one shifted tile per filter tap); 1: one shifted tile per tap
                                 * everywhere (kept for A/B).  Results are bit-identical in both modes (same products, same order).
                                 * Other values are rejected by b200_ncsnpp_create. */
  int family;                   /* 0 = NCSN++ / DDPM++ (models/ncsnpp.py, the default); 1 = DDPM (models/ddpm.py:39-181): ResnetBlockDDPM
                                 * with the NIN_0 skip (layers.py:619-662), AttnBlock (:558-581), Downsample / Upsample with_conv
                                 * (:584-616), residual scale 1, GroupNorm with 32 groups everywhere (channel counts must be multiples
                                 * of 32), sinusoidal time embedding through the "pos_freqs" pseudo-parameter.  Family 1 reads
                                 * image_size, num_channels, nf, num_res_blocks, num_levels, ch_mult, num_attn_resolutions,
                                 * attn_resolutions, centered and the execution fields (precision, keep_activations, lanes,
                                 * cuda_core_head, pdl, no_halo, tangent); it requires
                                 * conditional = 1 and scale_by_sigma = 0, and ignores skip_rescale, progressive_input, progressive,
                                 * fir_taps / fir_kernel, naive_resample and embedding_type.
                                 * 2 = NCSNv2 (models/ncsnv2.py: NCSNv2 'ncsnv2_64' with num_levels = 4, NCSNv2_128 with
                                 * num_levels = 5): ResidualBlocks with InstanceNorm2dPlus + ELU, dilated 3x3 convolutions and
                                 * ConvMeanPool, RefineBlocks (RCU, MSF with bilinear sums, CRP with 5x5 max pooling), output
                                 * divided by the per-image label, which the caller sets to sigmas[y].  Family 2 reads image_size,
                                 * num_channels, nf, num_levels, centered and the execution fields; it ignores the rest, refuses
                                 * tangent = 1 and precision = 3, and records module taps as 0 = begin_conv, then every
                                 * ResidualBlock, then every RefineBlock in forward order. */
  int tangent;                  /* 0 (default): the forward alone.  1: the plan also carries the forward-mode tangent pass of
                                 * b200_ncsnpp_jvp: after each op its tangent op (the same contraction on the tangent buffers
                                 * without bias and time-embedding row, or a GroupNorm(+SiLU) / softmax tangent kernel).  Taken
                                 * by family 1 (DDPM) and by family 0 with naive_resample = 1, progressive = 0 and
                                 * progressive_input = 0 (the DDPM++ configs), at precision 0, 1 or 3 with lanes <= 1; anything
                                 * else is rejected by b200_ncsnpp_create.  A tangent plan runs attention as separate
                                 * contractions, the skip projections as their own contraction, and keeps the few-channel
                                 * levels on the CUDA-core kernel (op labels name the form). */
} b200_ncsnpp_config;

B200_API int b200_ncsnpp_create(const b200_ncsnpp_config* cfg, b200_ncsnpp_t** out);
B200_API void b200_ncsnpp_destroy(b200_ncsnpp_t* h);
/* Parameter table in the reference's state_dict order and naming (all_modules.{i}.…). */
B200_API int b200_ncsnpp_num_params(const b200_ncsnpp_t* h);
B200_API int b200_ncsnpp_param_info(const b200_ncsnpp_t* h, int index, char* name, int name_cap,
                                    long long shape[4], int* ndim);
B200_API long long b200_ncsnpp_weights_bytes(const b200_ncsnpp_t* h);
B200_API int b200_ncsnpp_bind_weights(b200_ncsnpp_t* h, void* blob_dev);
/* Repack one parameter (reference layout, fp32, device) into the bound blob. */
B200_API int b200_ncsnpp_load_param(b200_ncsnpp_t* h, int index, const float* src_dev, void* stream);
B200_API long long b200_ncsnpp_workspace_bytes(b200_ncsnpp_t* h, int batch);
B200_API int b200_ncsnpp_bind_workspace(b200_ncsnpp_t* h, int batch, void* ws_dev, long long ws_bytes);
/* labels_uniform != 0: every image has the label labels[0] (the sampler's case,
 * sampling.py:404-405) — the time-embedding path is then evaluated for one row. */
B200_API int b200_ncsnpp_forward(b200_ncsnpp_t* h, const float* x_nchw, const float* labels,
                                 int labels_uniform, float* out_nchw, void* stream);
/* debug (keep_activations=1): copy the output of all_modules[index] as NCHW into dst. */
B200_API int b200_ncsnpp_tap(b200_ncsnpp_t* h, int module_index, float* dst_nchw, long long dst_cap_elems,
                             int shape_out[4], void* stream);
B200_API long long b200_ncsnpp_launches_per_forward(const b200_ncsnpp_t* h);
/* Forward plus Jacobian-vector product (engine created with tangent = 1): out = net(x), jvp_out = J_net(x) v, all NCHW
 * [B,C,H,W].  Replaces the autograd VJP of the Hutchinson-Skilling estimator (likelihood.py:26-35): for a fixed eps,
 * eps . (J^T eps) = eps . (J eps), so the divergence needs one forward-mode pass and no backward graph.  The engine's
 * b200_ncsnpp_forward is not available on a tangent engine; profile_forward / profile_ops there run this pass with v = x
 * and both results written to out. */
B200_API int b200_ncsnpp_jvp(b200_ncsnpp_t* h, const float* x_nchw, const float* labels, int labels_uniform,
                             const float* v_nchw, float* out_nchw, float* jvp_out_nchw, void* stream);
/* debug (tangent = 1, keep_activations = 1): the tangent of all_modules[index]'s output, as b200_ncsnpp_tap */
B200_API int b200_ncsnpp_tap_tangent(b200_ncsnpp_t* h, int module_index, float* dst_nchw, long long dst_cap_elems,
                                     int shape_out[4], void* stream);
/* One eager forward with a CUDA-event pair around every op; per-kind totals (kind 0 tensor-core
 * contraction, 1 CUDA-core contraction, 2 GroupNorm, 3 FIR, 4 softmax, 5 time embedding, 6 misc):
 * device milliseconds, algorithmic FLOPs (2*M*N*K of the contractions) and op counts. */
B200_API int b200_ncsnpp_profile_forward(b200_ncsnpp_t* h, const float* x_nchw, const float* labels,
                                         int labels_uniform, float* out_nchw, void* stream,
                                         float ms_by_kind[8], double flops_by_kind[8], long long ops_by_kind[8]);
/* Per-op view of the bound plan (both half-batch lanes, lane 0 first): a shape label, the kind index used by
 * b200_ncsnpp_profile_forward, the algorithmic FLOPs, and one CUDA-event-timed duration per op (run serially). */
B200_API long long b200_ncsnpp_num_ops(const b200_ncsnpp_t* h);
B200_API int b200_ncsnpp_op_info(const b200_ncsnpp_t* h, long long index, char* name, int name_cap, int* kind,
                                 double* flops);
/* algorithmic HBM bytes of op `index` (operands read once + outputs written once; 0 for ops that do not report it) */
B200_API int b200_ncsnpp_op_bytes(const b200_ncsnpp_t* h, long long index, double* bytes);
B200_API int b200_ncsnpp_profile_ops(b200_ncsnpp_t* h, const float* x, const float* labels, int labels_uniform,
                                     float* out, void* stream, float* ms_per_op, long long cap);

/* ---- predictor–corrector loop --------------------------------------------------
 * Replaces the body of pc_sampler (sampling.py:390-409) with
 * shared_corrector_update_fn/LangevinCorrector (:344-352, :262-282) and
 * shared_predictor_update_fn/ReverseDiffusion|EulerMaruyama (:333-341, :181-200)
 * + get_score_fn (models/utils.py:129-178) for an engine-backed model.
 * Per-step scalars are supplied as host tables of length n_steps (built by the host
 * with the SDE's own torch ops so they are bit-equal to the reference's):
 *   label[i]       network time label (VE: sigma(t_i), VP: 999 t_i)
 *   score_scale[i] score = score_scale * net_out   (VE: 1, VP: -1/std(t_i))
 *   alpha[i]       Langevin alpha (VE: 1)
 *   pa,pb,pc[i]    predictor: x_mean = pa*x + pb*net_out ; x = x_mean + pc*z
 */
typedef struct b200_pc b200_pc_t;
typedef struct {
  int n_steps;                 /* sde.N */
  int corrector;               /* 0 none, 1 langevin (norm-based step size, sampling.py:262-282), 2 affine corrector: annealed
                                * Langevin dynamics (:286-319), whose step size depends on the step only: x_mean = ca x + cb out,
                                * x = x_mean + cc z */
  int predictor;               /* 0 none, 1 affine (reverse_diffusion / euler_maruyama / ancestral_sampling: x_mean = pa x + pb out,
                                * x = x_mean + pc z) */
  int n_corrector_steps;       /* config.sampling.n_steps_each */
  float snr;
  const float *label, *score_scale, *alpha, *pa, *pb, *pc;   /* HOST tables [n_steps] */
  const float *ca, *cb, *cc;   /* HOST tables [n_steps] of the affine corrector (corrector == 2), else NULL */
  /* controllable generation (controllable_generation.py:8-198): after the corrector block and again after the predictor
   * block (even a None one) the state is blended with a fresh draw from the data marginal, in the latent space
   * y = decouple(x):  y' = y*(1-mask) + (cm*known + cs*z)*mask,  x = couple(y'),
   * x_mean = couple(decouple(x)*(1-mask) + cm*known*mask).  Each blend draws one randn_like(x). */
  int constraint;              /* 0 off, 1 inpaint (decouple = identity), 2 colorize (decouple(v)_j = sum_i v_i color_m[3i+j]) */
  const float *cm, *cs;        /* HOST tables [n_steps]: mean coefficient and std of sde.marginal_prob at t_i */
  float color_m[9], color_minv[9];   /* colorize: M and M^-1, row-major */
  int noise_nhwc;              /* 1: every randn_like draw fills the state in channels-last memory order, as torch does for
                                * a channels-last x (the reference's colorization state is its einsum's channels-last
                                * output for batches > 1); 0: NCHW order */
} b200_pc_config;

B200_API int b200_pc_create(b200_ncsnpp_t* model, const b200_pc_config* cfg, int batch, b200_pc_t** out);
B200_API void b200_pc_destroy(b200_pc_t* pc);
B200_API long long b200_pc_workspace_bytes(const b200_pc_t* pc);
B200_API int b200_pc_bind_workspace(b200_pc_t* pc, void* ws_dev, long long ws_bytes, void* stream);
/* Run iterations [first_step, first_step+num_steps) on x (NCHW, in place); x_mean receives the
 * last predictor (or corrector) mean.  Noise comes from the in-kernel Philox stream equal to
 * torch's CUDA generator at (seed, offset); *offset_out = offset after the run.
 * use_graph != 0 replays one captured CUDA graph per iteration. */
B200_API int b200_pc_run(b200_pc_t* pc, float* x, float* x_mean, int first_step, int num_steps,
                         unsigned long long seed, unsigned long long offset, unsigned long long* offset_out,
                         int use_graph, void* stream);
/* Constrained plans: the blend's `known` (the data; for colorization already decouple(gray)) and `mask`, both full
 * NCHW device tensors of the batch shape.  Rebinding other pointers re-captures the graph on the next run.
 * `stream` matches b200_pc_bind_workspace's signature; nothing is enqueued on it. */
B200_API int b200_pc_bind_constraint(b200_pc_t* pc, const float* known, const float* mask, void* stream);
/* One iteration with caller-supplied noise tensors (NCHW, may be NULL when unused).  Not for constrained plans. */
B200_API int b200_pc_step_external(b200_pc_t* pc, float* x, float* x_mean, int step,
                                   const float* noise_corrector, const float* noise_predictor, void* stream);
B200_API long long b200_pc_launches_per_step(const b200_pc_t* pc);

/* ---- probability-flow ODE: device-resident explicit Runge-Kutta (RK23, RK45, DOP853) ------------
 * Replaces the host-side state and stage arithmetic of sampling.py:414-485 and likelihood.py:84-113
 * (scipy.integrate.solve_ivp on a float64 numpy array: two PCIe crossings of the whole state per function evaluation).
 * The float64 state y, y_new and the stage derivatives K[n_stages + 1][n] stay in device memory; scipy's step-size
 * controller runs on the host (score_sde_pytorch_b200/ode.py) and reads back one double per attempted step (two for
 * DOP853).  All pointers are device pointers except coef_host / e_host / e5_host / e3_host (<= 16 doubles, passed by
 * value into the launch). */
/* y_stage = y + h * sum_{j<nk} coef[j] * K[j] (float64; nk = 0: y itself); optional float64 copy (y_out) and float32
 * copy (x32: the network input, `.type(torch.float32)` in the reference's ode_func) */
B200_API int b200_ode_stage_f64(const double* y, const double* k, long long n, const double* coef_host, int nk, double h,
                                double* y_out, float* x32, void* stream);
/* K_s = (double) drift, drift = c_f * x32 - (g2 * score) * 0.5f, score = std > 0 ? -(net_out / std) : net_out, in unfused
 * fp32 like rsde.sde with probability_flow=True (sde_lib.py:93-100) over get_score_fn (models/utils.py:129-178);
 * scalars_dev = {c_f, g2, std} */
B200_API int b200_ode_drift_f64(const float* x32, const float* net_out, long long n, const float* scalars_dev, double* k_out,
                                void* stream);
/* Divergence of the drift for the likelihood ODE (likelihood.py:66-67, 95): k_out[img] (float64, the logp slots of a stage
 * derivative) = sum_i eps_i (c_f eps_i - 0.5 g2 dscore_i), dscore = -(jvp_out / std) (std > 0) or jvp_out, with
 * jvp_out = J_net eps from b200_ncsnpp_jvp; same scalars_dev as b200_ode_drift_f64.  Deterministic fp64 sum per image. */
B200_API int b200_ode_div_f64(const float* eps, const float* jvp_out, int nimg, long long per_img, const float* scalars_dev,
                              double* k_out, void* stream);
/* ws[0] = sum_i ((h * sum_{j<nk} e[j] K[j][i]) / (atol + max(|y_i|, |y_new_i|) * rtol))^2   (RungeKutta._estimate_error_norm);
 * ws: b200_ode_workspace_doubles() doubles; deterministic two-pass reduction */
B200_API long long b200_ode_workspace_doubles(void);
B200_API int b200_ode_error_sumsq_f64(const double* y, const double* y_new, const double* k, long long n, const double* e_host,
                                      int nk, double h, double rtol, double atol, double* ws, void* stream);
/* DOP853._estimate_error_norm's two sums from one read of K, scale_i = atol + max(|y_i|, |y_new_i|) * rtol:
 * ws[0] = sum_i ((sum_{j<nk} e5[j] K[j][i]) / scale_i)^2,  ws[1] = sum_i ((sum_{j<nk} e3[j] K[j][i]) / scale_i)^2;
 * each the same deterministic two-pass reduction as b200_ode_error_sumsq_f64 */
B200_API int b200_ode_error_sumsq2_f64(const double* y, const double* y_new, const double* k, long long n,
                                       const double* e5_host, const double* e3_host, int nk, double rtol, double atol,
                                       double* ws, void* stream);
/* ws[0] = sum_i (((v - v2)_i) / (atol + |y0_i| * rtol))^2, v2 optional: the three norms of scipy's select_initial_step */
B200_API int b200_ode_scaled_sumsq_f64(const double* v, const double* v2, const double* y0, long long n, double rtol, double atol,
                                       double* ws, void* stream);

/* ---- denoising score matching losses: the evaluation step ---------------------------------------
 * Device pieces of losses.py:55-150 (get_sde_loss_fn / get_smld_loss_fn / get_ddpm_loss_fn) around the engine's network
 * evaluation, used by score_sde_pytorch_b200/losses.py.  Per-image scalars are device arrays [nimg] computed with the SDE's own
 * torch ops (sde.marginal_prob, sde.sde), as the reference does. */
/* out = mean_coef[img] * x + noise_coef[img] * z (mean_coef NULL: 1): losses.py:86-87, :111-112, :133-134; separate fp32
 * roundings like the reference's unfused torch ops, i.e. bit-equal to it */
B200_API int b200_dsm_perturb_f32(const float* x, const float* z, const float* mean_coef, const float* noise_coef, float* out,
                                  int nimg, long long n_per_img, void* stream);
/* losses[img] = reduce(residual^2) over the image, reduce = mean (reduce_mean != 0) or 0.5 * sum (losses.py:71); residual by
 * mode: 0 score * w + z (:90), 1 score + z / w (:94), 2 score + (z * w) / w2 (SMLD, w = sigma, w2 = sigma^2, :110-115),
 * 3 score - z (DDPM, :136).  ws: b200_dsm_workspace_doubles(nimg, n_per_img) doubles; deterministic fixed-order fp64 sums. */
B200_API long long b200_dsm_workspace_doubles(int nimg, long long n_per_img);
B200_API int b200_dsm_loss_f32(const float* score, const float* z, const float* w, const float* w2, float* losses, int nimg,
                               long long n_per_img, int mode, int reduce_mean, double* ws, void* stream);

#ifdef __cplusplus
}
#endif
#endif  /* SCORESDE_B200_H_ */
