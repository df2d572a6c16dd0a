// C-ABI entry points that are not part of the engine object: error text, the
// successors of the reference's two native ops, and single-kernel building blocks
// exported so tests can check each device kernel against torch / the oracle.
#include "kernels.h"
#include "../../include/scoresde_b200.h"
#include <cstring>

namespace b200 {
namespace { thread_local bool tl_pdl = false; }
bool pdl_active() { return tl_pdl; }
PdlScope::PdlScope(bool on) : prev(tl_pdl) { tl_pdl = on; }
PdlScope::~PdlScope() { tl_pdl = prev; }


static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }

}  // namespace b200

using namespace b200;

extern "C" {

const char* b200_last_error(void) { return last_error(); }
int b200_version(void) { return 200; }   // 0.2.0

int b200_device_sm_count(int* out) {
  int dev = 0, n = 0;
  B200_CHECK_CUDA(cudaGetDevice(&dev));
  B200_CHECK_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  if (out) *out = n;
  return 0;
}

int b200_upfirdn2d_f32(const float* x, const float* kernel_host, float* y, int major, int in_h, int in_w, int minor,
                       int kh, int kw, int up_x, int up_y, int down_x, int down_y, int pad_x0, int pad_x1,
                       int pad_y0, int pad_y1, void* stream) {
  B200_REQUIRE(x && kernel_host && y, "upfirdn2d: null pointer");
  B200_REQUIRE(major >= 0 && in_h > 0 && in_w > 0 && minor > 0, "upfirdn2d: bad shape [%d,%d,%d,%d]", major, in_h, in_w, minor);
  return launch_upfirdn2d(x, kernel_host, y, major, in_h, in_w, minor, kh, kw, up_x, up_y, down_x, down_y, pad_x0,
                          pad_x1, pad_y0, pad_y1, 0, static_cast<cudaStream_t>(stream));
}

int b200_fused_bias_act_f32(const float* x, const float* b, const float* ref, float* y, long long n, int step_b,
                            int size_b, int act, int grad, float alpha, float scale, void* stream) {
  B200_REQUIRE(n == 0 || (x && y), "fused_bias_act: null pointer");
  return launch_fused_bias_act(x, b, ref, y, n, step_b, size_b, act, grad, alpha, scale, static_cast<cudaStream_t>(stream));
}

int b200_groupnorm_nhwc_f32(const float* x1, int c1, const float* x2, int c2, const float* gamma, const float* beta,
                            int batch, int hw, int groups, float eps, int silu, int round_tf32, float* stats_ws,
                            float* y, float* raw, void* stream) {
  B200_REQUIRE(x1 && gamma && beta && stats_ws && y, "groupnorm: null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // stats_ws holds the fp64 quad sums of both sources: [batch][c1/4][2] then [batch][c2/4][2]
  double* q1 = reinterpret_cast<double*>(stats_ws);
  double* q2 = q1 + (long long)batch * (c1 / 4) * 2;
  if (int r = launch_gn_quad_stats(x1, c1, batch, hw, q1, st)) return r;
  if (x2) { if (int r = launch_gn_quad_stats(x2, c2, batch, hw, q2, st)) return r; }
  return launch_gn_apply(x1, c1, x2, x2 ? c2 : 0, q1, q2, gamma, beta, batch, hw, groups, eps, silu, round_tf32, y, raw, st);
}

int b200_softmax_rows_f32(const float* s, float* p, long long rows, int t, float scale, int round_tf32, void* stream) {
  B200_REQUIRE(s && p, "softmax: null pointer");
  return launch_softmax_rows(s, p, rows, t, scale, round_tf32, static_cast<cudaStream_t>(stream));
}

int b200_randn_like_torch_f32(float* out, long long numel, unsigned long long seed, unsigned long long offset,
                              unsigned long long* inc_out, unsigned long long* offset_ws, void* stream) {
  B200_REQUIRE(out && offset_ws, "randn: null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PhiloxMap m;
  if (int r = philox_map_init(&m, numel, seed)) return r;
  B200_CHECK_CUDA(cudaMemcpyAsync(offset_ws, &offset, 8, cudaMemcpyHostToDevice, st));
  B200_CHECK_CUDA(cudaStreamSynchronize(st));
  if (inc_out) *inc_out = m.inc;
  return launch_randn_torch(m, offset_ws, 0, out, st);
}

int b200_pack_conv_weight_f32(const float* w_oihw, float* w_packed, int c_out, int c_in, int ksize, int round_tf32,
                              void* stream) {
  B200_REQUIRE(w_oihw && w_packed && ksize > 0, "pack_conv_weight: bad argument");
  const int taps = ksize * ksize;
  return launch_pack_weight(w_oihw, w_packed, taps, c_out, c_in, (long long)c_in * taps, taps, 1, round_tf32,
                            static_cast<cudaStream_t>(stream));
}

int b200_conv_nhwc_f32(const float* x1, int c1, const float* x2, int c2, int batch, int h, int w,
                       const float* w_packed, const float* bias, int c_out, int ksize, const float* rowvec,
                       long long rowvec_ld, const float* residual, float scale, int round_tf32, float* out, int impl,
                       void* stream) {
  B200_REQUIRE(x1 && w_packed && out, "conv_nhwc: null pointer");
  B200_REQUIRE(ksize == 1 || ksize == 3, "conv_nhwc: ksize %d unsupported", ksize);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Epilogue ep; memset(&ep, 0, sizeof(ep));
  ep.bias = bias; ep.rowvec = rowvec; ep.rowvec_ld = rowvec_ld; ep.residual = residual; ep.ld_res = c_out;
  ep.scale = scale; ep.round_tf32 = round_tf32; ep.rows_per_img = h * w; ep.out = out; ep.ld_out = c_out;
  if (!x2) c2 = 0;
  if (impl == 1 || impl == 2 || impl == 4 || impl == 5) {   // 4 / 5: as 1 / 2 without the halo form
    TcGemmDesc d; memset(&d, 0, sizeof(d));
    d.f16 = impl == 2 || impl == 5; d.no_halo = impl >= 4 ? 1 : 0;
    d.a1 = x1; d.C1 = c1; d.a2 = x2; d.C2 = c2; d.conv = 1; d.H = h; d.W = w; d.nimg = batch; d.taps = ksize * ksize;
    d.w = w_packed; d.N_total = c_out; d.K_total = c1 + c2; d.w_rows = (long long)ksize * ksize * c_out; d.nbatch = 1;
    d.epi = ep;
    TcGemmPlan* pl = nullptr;
    if (int r = tc_gemm_plan_create(d, &pl)) return r;
    const int r = tc_gemm_launch(pl, st);
    tc_gemm_plan_destroy(pl);
    return r;
  }
  SimtConv s; memset(&s, 0, sizeof(s));
  s.x1 = x1; s.C1 = c1; s.x2 = x2; s.C2 = c2; s.in_scale = 1.f; s.H = h; s.W = w; s.R = s.S = ksize; s.stride = 1;
  s.pad = ksize / 2; s.OH = h; s.OW = w; s.nbatch = batch; s.a_batched = 1; s.w = w_packed; s.N = c_out; s.epi = ep;
  if (impl == 3) return launch_conv_lowc(s, st);
  B200_REQUIRE(impl == 0, "conv_nhwc: impl %d unknown", impl);
  return launch_conv_simt(s, st);
}

int b200_conv_dilated_nhwc_f32(const float* x, int c, int batch, int h, int w, const float* w_packed, const float* bias,
                               int c_out, int dilation, const float* residual, int round_out, float* out, int impl,
                               void* stream) {
  B200_REQUIRE(x && w_packed && out && dilation >= 1, "conv_dilated_nhwc: bad argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Epilogue ep; memset(&ep, 0, sizeof(ep));
  ep.bias = bias; ep.residual = residual; ep.ld_res = c_out; ep.scale = 1.f; ep.round_tf32 = round_out;
  ep.rows_per_img = h * w; ep.out = out; ep.ld_out = c_out;
  if (impl == 1 || impl == 2) {
    TcGemmDesc d; memset(&d, 0, sizeof(d));
    d.f16 = impl == 2; d.a1 = x; d.C1 = c; d.conv = 1; d.H = h; d.W = w; d.nimg = batch; d.taps = 9; d.dilation = dilation;
    d.w = w_packed; d.N_total = c_out; d.K_total = c; d.w_rows = 9LL * c_out; d.nbatch = 1; d.epi = ep;
    TcGemmPlan* pl = nullptr;
    if (int r = tc_gemm_plan_create(d, &pl)) return r;
    const int r = tc_gemm_launch(pl, st);
    tc_gemm_plan_destroy(pl);
    return r;
  }
  B200_REQUIRE(impl == 0, "conv_dilated_nhwc: impl %d unknown", impl);
  SimtConv s; memset(&s, 0, sizeof(s));
  s.x1 = x; s.C1 = c; s.in_scale = 1.f; s.H = h; s.W = w; s.R = s.S = 3; s.stride = 1; s.pad = dilation; s.dilation = dilation;
  s.OH = h; s.OW = w; s.nbatch = batch; s.a_batched = 1; s.w = w_packed; s.N = c_out; s.epi = ep;
  return launch_conv_simt(s, st);
}

int b200_instnorm_plus_nhwc_f32(const float* x, int batch, int hw, int c, const float* alpha, const float* gamma,
                                const float* beta, int act, int round_out, float* y, double* stats_ws, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int r = launch_in_stats(x, batch, hw, c, stats_ws, st)) return r;
  return launch_in_apply(x, stats_ws, alpha, gamma, beta, batch, hw, c, 1e-5f, act, round_out, y, st);
}

int b200_maxpool5_nhwc_f32(const float* x, int batch, int h, int w, int c, int round_out, float* y, const float* add, float* sum,
                           void* stream) {
  return launch_maxpool5(x, batch, h, w, c, round_out, y, add, sum, static_cast<cudaStream_t>(stream));
}

int b200_bilinear_add_nhwc_f32(const float* lo, int batch, int hl, int wl, int c, float* acc, int h, int w, void* stream) {
  return launch_bilinear_add(lo, batch, hl, wl, c, acc, h, w, static_cast<cudaStream_t>(stream));
}

int b200_conv_skip_nhwc_f32(const float* x, int c, const float* s1, int cs1, const float* s2, int cs2, int batch, int h,
                            int w, const float* w_packed, const float* bias, const float* w_skip,
                            const float* bias_skip, int c_out, const float* residual, float scale, int round_tf32,
                            float* out, void* stream) {
  B200_REQUIRE(x && s1 && w_packed && w_skip && out, "conv_skip_nhwc: null pointer");
  Epilogue ep; memset(&ep, 0, sizeof(ep));
  ep.bias = bias; ep.rowvec = bias_skip; ep.rowvec_ld = 0; ep.residual = residual; ep.ld_res = c_out;
  ep.scale = scale; ep.round_tf32 = round_tf32; ep.rows_per_img = h * w; ep.out = out; ep.ld_out = c_out;
  TcGemmDesc d; memset(&d, 0, sizeof(d));
  d.a1 = x; d.C1 = c; d.conv = 1; d.H = h; d.W = w; d.nimg = batch; d.taps = 9;
  d.w = w_packed; d.N_total = c_out; d.K_total = c; d.w_rows = 9LL * c_out; d.nbatch = 1;
  d.a3 = s1; d.C3 = cs1; d.a4 = s2; d.C4 = s2 ? cs2 : 0; d.w2 = w_skip;
  d.epi = ep;
  TcGemmPlan* pl = nullptr;
  if (int r = tc_gemm_plan_create(d, &pl)) return r;
  const int r = tc_gemm_launch(pl, static_cast<cudaStream_t>(stream));
  tc_gemm_plan_destroy(pl);
  return r;
}

int b200_attention_core_f32(const float* qk, const float* vT, const float* w3, const float* bv, const float* b3,
                            const float* x, float* out, double* qstats, int nimg, int t, int c, float out_scale,
                            int operand_f16, void* stream) {
  B200_REQUIRE(tc_attn_supported(t, c, operand_f16 != 0),
               "attention_core: implemented for T=256 with C=256 (tf32 or fp16 operands) or C=512 (fp16 operands only); "
               "got T=%d C=%d with %s operands", t, c, operand_f16 ? "fp16" : "tf32");
  TcAttnDesc d; memset(&d, 0, sizeof(d));
  d.qk = qk; d.vT = vT; d.w3 = w3; d.bv = bv; d.b3 = b3; d.x = x; d.out = out; d.qstats = qstats;
  d.nimg = nimg; d.T = t; d.C = c; d.out_scale = out_scale; d.f16 = operand_f16 ? 1 : 0;
  TcAttnPlan* pl = nullptr;
  if (int r = tc_attn_plan_create(d, &pl)) return r;
  const int r = tc_attn_launch(pl, static_cast<cudaStream_t>(stream));
  tc_attn_plan_destroy(pl);
  return r;
}

int b200_attention_flash_f16(const void* qk, const void* vT, const float* bv, void* out, int nimg, int t, int c,
                              void* stream) {
  AttnFlashPlan pl;
  if (int r = attn_flash_plan(qk, vT, bv, out, nimg, t, c, &pl)) return r;
  return attn_flash_launch(pl, static_cast<cudaStream_t>(stream));
}

int b200_gemm_nt_f32(const float* a, long long lda, int a_batch_rows, const float* w, long long ldw, int w_batch_rows,
                     int nbatch, int m, int n, int k, const float* bias, int round_tf32, float* out, long long ldo,
                     int impl, void* stream) {
  B200_REQUIRE(a && w && out && nbatch > 0, "gemm_nt: bad argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Epilogue ep; memset(&ep, 0, sizeof(ep));
  ep.bias = bias; ep.scale = 1.f; ep.round_tf32 = round_tf32; ep.rows_per_img = m; ep.out = out; ep.ld_out = ldo;
  if (impl == 1 || impl == 2) {
    TcGemmDesc d; memset(&d, 0, sizeof(d));
    d.f16 = impl == 2;
    d.a1 = a; d.C1 = k; d.conv = 0; d.taps = 1; d.a_ld = lda; d.a_batch_rows = a_batch_rows;
    d.a_rows = a_batch_rows ? (long long)a_batch_rows * (nbatch - 1) + m : m;
    d.w = w; d.N_total = n; d.K_total = k; d.w_ld = ldw; d.w_batch_rows = w_batch_rows;
    d.w_rows = w_batch_rows ? (long long)w_batch_rows * (nbatch - 1) + n : n;
    d.nbatch = nbatch; d.M_per_batch = m; d.epi = ep;
    TcGemmPlan* pl = nullptr;
    if (int r = tc_gemm_plan_create(d, &pl)) return r;
    const int r = tc_gemm_launch(pl, st);
    tc_gemm_plan_destroy(pl);
    return r;
  }
  SimtConv s; memset(&s, 0, sizeof(s));
  s.x1 = a; s.C1 = k; s.ld1 = lda; s.in_scale = 1.f; s.H = m; s.W = 1; s.R = s.S = 1; s.stride = 1; s.pad = 0;
  s.OH = m; s.OW = 1; s.nbatch = nbatch; s.a_batched = a_batch_rows != 0; s.w = w; s.N = n;
  s.w_batch_stride = (long long)w_batch_rows * ldw; s.w_ld = ldw; s.epi = ep;
  B200_REQUIRE(!a_batch_rows || a_batch_rows == m, "gemm_nt(simt): a_batch_rows must be 0 or m");
  return launch_conv_simt(s, st);
}

int b200_tc_contract_f32(const b200_tc_test_desc* t, char* form, int form_len, void* stream) {
  B200_REQUIRE(t, "tc_contract: null descriptor");
  B200_REQUIRE(t->struct_bytes == (int)sizeof(b200_tc_test_desc),
               "tc_contract: descriptor of %d bytes, the library's b200_tc_test_desc has %d", t->struct_bytes,
               (int)sizeof(b200_tc_test_desc));
  auto f = [](const void* p) { return static_cast<const float*>(p); };
  TcGemmDesc d; memset(&d, 0, sizeof(d));
  d.a1 = f(t->a1); d.C1 = t->c1; d.a2 = f(t->a2); d.C2 = t->c2;
  d.conv = t->conv; d.H = t->h; d.W = t->w; d.nimg = t->nimg; d.taps = t->taps; d.stride = t->stride;
  d.valid_pad = t->valid_pad; d.Hin = t->hin; d.Win = t->win; d.dilation = t->dilation; d.no_halo = t->no_halo; d.f16 = t->f16;
  d.a_rows = t->a_rows; d.a_ld = t->a_ld; d.a_batch_rows = t->a_batch_rows;
  d.w = f(t->wt); d.N_total = t->n_total; d.K_total = t->k_total; d.w_rows = t->w_rows; d.w_ld = t->w_ld;
  d.w_batch_rows = t->w_batch_rows; d.nbatch = t->nbatch; d.M_per_batch = t->m_per_batch;
  d.a3 = f(t->a3); d.C3 = t->c3; d.a4 = f(t->a4); d.C4 = t->c4; d.w2 = f(t->w2);
  d.split = t->split; d.a1_lo = f(t->a1_lo); d.a2_lo = f(t->a2_lo); d.a3_lo = f(t->a3_lo); d.a4_lo = f(t->a4_lo);
  d.w_lo = f(t->w_lo); d.w2_lo = f(t->w2_lo);
  d.qstats = t->qstats;
  Epilogue& ep = d.epi;
  ep.bias = t->bias; ep.rowvec = t->rowvec; ep.rowvec_ld = t->rowvec_ld; ep.residual = t->residual; ep.ld_res = t->ld_res;
  ep.per_img_div = t->per_img_div; ep.div_stride = t->div_stride; ep.scale = t->scale; ep.round_tf32 = t->store_mode;
  ep.rows_per_img = t->rows_per_img; ep.out = static_cast<float*>(t->out); ep.ld_out = t->ld_out; ep.out_nchw = t->out_nchw;
  ep.n_valid = t->n_valid;
  TcGemmPlan* pl = nullptr;
  if (int r = tc_gemm_plan_create(d, &pl)) return r;
  if (form && form_len > 0) { strncpy(form, tc_gemm_form(pl), form_len - 1); form[form_len - 1] = '\0'; }
  const int r = tc_gemm_launch(pl, static_cast<cudaStream_t>(stream));
  tc_gemm_plan_destroy(pl);
  return r;
}

int b200_conv_lowc_gn_f32(const float* x1, int c1, const float* x2, int c2, int batch, int h, int w, const float* w_packed,
                          int c_out, int ksize, const double* q1, const double* q2, const float* gamma, const float* beta,
                          int groups, float eps, int silu, float* coeff_ws, const float* bias, const float* rowvec,
                          long long rowvec_ld, const float* residual, float scale, int round_tf32, float* out, double* qstats,
                          void* stream) {
  B200_REQUIRE(x1 && w_packed && q1 && gamma && beta && coeff_ws && out, "conv_lowc_gn: null pointer");
  B200_REQUIRE(ksize == 1 || ksize == 3, "conv_lowc_gn: ksize %d unsupported", ksize);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!x2) c2 = 0;
  float* gn_scale = coeff_ws;
  float* gn_shift = coeff_ws + (long long)batch * (c1 + c2);
  if (int r = launch_gn_coeff(c1, c2, q1, q2, gamma, beta, batch, h * w, groups, eps, gn_scale, gn_shift, st)) return r;
  SimtConv s; memset(&s, 0, sizeof(s));
  s.x1 = x1; s.C1 = c1; s.x2 = x2; s.C2 = c2; s.in_scale = 1.f; s.H = h; s.W = w; s.R = s.S = ksize; s.stride = 1;
  s.pad = ksize / 2; s.OH = h; s.OW = w; s.nbatch = batch; s.a_batched = 1; s.w = w_packed; s.N = c_out;
  s.gn_scale = gn_scale; s.gn_shift = gn_shift; s.gn_act = silu ? 1 : 0; s.qstats = qstats;
  s.epi.bias = bias; s.epi.rowvec = rowvec; s.epi.rowvec_ld = rowvec_ld; s.epi.residual = residual; s.epi.ld_res = c_out;
  s.epi.scale = scale; s.epi.round_tf32 = round_tf32; s.epi.rows_per_img = h * w; s.epi.out = out; s.epi.ld_out = c_out;
  return launch_conv_lowc(s, st);
}

int b200_head_small_n_f32(const void* x, int x_f16, int batch, int h, int w, int c, const float* w_packed, const float* bias,
                          int n, const float* div, long long div_stride, float* out_nchw, void* stream) {
  B200_REQUIRE(x && w_packed && out_nchw, "head_small_n: null pointer");
  return launch_conv3x3_small_n(static_cast<const float*>(x), w_packed, bias, div, div_stride, out_nchw, batch, h, w, c, n,
                                x_f16, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
