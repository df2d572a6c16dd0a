// NCSN++ execution engine: builds the layer graph from the model configuration in the
// same order as the reference constructor (models/ncsnpp.py:68-230), owns the packed
// weight blob layout, plans activation buffers inside a caller-provided workspace and
// replays the forward pass (models/ncsnpp.py:232-381) as a fixed sequence of kernel
// launches on the caller's stream.  Nothing here allocates device memory.
#include "kernels.h"
#include "../../include/scoresde_b200.h"
#include <cmath>
#include <cstring>
#include <functional>
#include <map>
#include <string>
#include <vector>

using namespace b200;

namespace {

// M_DOWN / M_UP: the DDPM family's Downsample / Upsample with_conv (layers.py:584-616)
// M_NRES / M_NREF / M_NHEAD: the NCSNv2 family's ResidualBlock, RefineBlock and output head (models/ncsnv2.py, layers.py)
enum ModKind { M_FOURIER, M_LINEAR, M_CONV_IN, M_RESBLOCK, M_ATTN, M_PYR_DOWN, M_GN_OUT, M_CONV_OUT, M_COMBINE, M_DOWN, M_UP,
               M_NRES, M_NREF, M_NHEAD };
enum PackKind { PK_COPY = 0, PK_CONV = 1, PK_NIN = 2, PK_CONV_FLAT32 = 3, PK_CONV_PAD128 = 4 };

struct Param {
  std::string name;
  int ndim; long long shape[4];
  long long off, count;      // location in the packed blob (floats)
  int pack, taps, O, I, round;   // round: packed format (store_operand4 mode; 3 = split TF32, a hi and a lo copy)
  long long lo = -1;             // split TF32: location of the lo copy (same packed layout as the hi copy at off)
};

struct Mod {
  ModKind kind; int index;
  int cin1 = 0, cin2 = 0, cout = 0, up = 0, down = 0, res = 0, has_conv2 = 0;
  int dense_row = 0;
  bool tc0 = false, tc1 = false, tc2 = false, tcattn = false;
  // parameter indices
  int gn0w = -1, gn0b = -1, c0w = -1, c0b = -1, dw = -1, db = -1, gn1w = -1, gn1b = -1, c1w = -1, c1b = -1, c2w = -1, c2b = -1;
  int nw[4] = {-1, -1, -1, -1}, nb[4] = {-1, -1, -1, -1};
  int w = -1, b = -1;
  // NCSNv2 (family 2).  M_NRES: dilation, InstanceNorm2dPlus parameters in[k] = {alpha, gamma, beta} of normalize1 (k = 0)
  // and normalize2 (k = 1), conv1 (c0w, c0b), conv2 (c1w, c1b), shortcut (c2w, c2b; -1 when the identity).  M_NREF: the
  // RCU convolutions of each input (adapt[i], 4 each) and of the output (outc, 2 per block), the MSF convolutions
  // (msfw / msfb, one per input when there are two) and the CRP convolutions (crp).  M_NHEAD: normalizer in[0], end_conv (w, b).
  int dil = 1;
  int in[2][3] = {{-1, -1, -1}, {-1, -1, -1}};
  int nin = 0;
  std::vector<int> adapt[2], outc, msfw, msfb, crp;
};

struct Tensor {
  float* p = nullptr; int C = 0, H = 0, W = 0; long long bytes = 0;
  double* qs = nullptr;   // GroupNorm quad sums [B][C/4][2]
  bool f16 = false;       // elements are IEEE fp16 (mid-block conv output in fp16 operand mode)
  float* d = nullptr;     // tangent of the same shape (tangent plans: allocated right after the primal elements)
};

class Arena {
 public:
  explicit Arena(bool keep) : keep_(keep) {}
  long long alloc(long long bytes) {
    bytes = (bytes + 1023) & ~1023LL;
    if (!keep_) {
      for (size_t i = 0; i < free_.size(); ++i) {
        if (free_[i].second >= bytes) {
          const long long off = free_[i].first;
          if (free_[i].second == bytes) free_.erase(free_.begin() + i);
          else { free_[i].first += bytes; free_[i].second -= bytes; }
          return off;
        }
      }
    }
    const long long off = top_;
    top_ += bytes;
    return off;
  }
  void release(long long off, long long bytes) {
    if (keep_ || bytes == 0) return;
    bytes = (bytes + 1023) & ~1023LL;
    size_t i = 0;
    while (i < free_.size() && free_[i].first < off) ++i;
    free_.insert(free_.begin() + i, {off, bytes});
    if (i + 1 < free_.size() && free_[i].first + free_[i].second == free_[i + 1].first) {
      free_[i].second += free_[i + 1].second; free_.erase(free_.begin() + i + 1);
    }
    if (i > 0 && free_[i - 1].first + free_[i - 1].second == free_[i].first) {
      free_[i - 1].second += free_[i].second; free_.erase(free_.begin() + i);
    }
    // give the tail back to the bump pointer
    if (!free_.empty() && free_.back().first + free_.back().second == top_) { top_ = free_.back().first; free_.pop_back(); }
  }
  long long high_water() const { return std::max(top_, hw_); }
  void note() { hw_ = std::max(hw_, top_); }
 private:
  bool keep_;
  long long top_ = 0, hw_ = 0;
  std::vector<std::pair<long long, long long>> free_;
};

__global__ void affine_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, float shift, float scale) {
  pdl_wait(); pdl_trigger();   // programmatic dependent launch: see common.cuh
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = (x[i] + shift) * scale;
}

}  // namespace

struct b200_ncsnpp {
  b200_ncsnpp_config cfg;
  std::vector<Param> params;
  std::vector<Mod> mods;
  long long wcount = 0;
  float* wblob = nullptr;
  int sumC = 0; long long dense_w_off = 0, dense_b_off = 0;
  float fir2d[64]; int firn = 0;
  // plan
  int B = 0; char* ws = nullptr; long long ws_bytes = 0;
  struct Op { int kind; double flops; std::function<int(cudaStream_t)> fn; std::string name; double bytes; /* algorithmic HBM bytes: operands read once + outputs written once */ };
  std::vector<Op> ops;
  // Two half-batch "lanes" (ops2 = the second half's plan, empty when the batch is not split).  The lanes are
  // independent within one network evaluation, so forward() issues them on two streams: while one lane's
  // HBM-bound GroupNorm/FIR pass streams, the other lane's tensor-core contraction owns the tensor pipes.
  std::vector<Op> ops2;
  int B0 = 0;                                  // images in lane 0 (lane 1 holds B - B0)
  cudaStream_t lane_stream = nullptr; cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  const float* in_x_l[2] = {nullptr, nullptr}; const float* in_labels_l[2] = {nullptr, nullptr}; float* out_l[2] = {nullptr, nullptr};

  std::vector<TcGemmPlan*> tcplans;
  std::vector<TcAttnPlan*> attnplans;
  std::map<int, Tensor> taps;
  long long launches = 0;
  // per-call arguments read by the closures
  const float* in_x = nullptr; const float* in_labels = nullptr; float* out = nullptr; int uniform = 0;
  const float* in_v = nullptr; float* tout = nullptr;   // b200_ncsnpp_jvp: tangent direction and J v (tangent plans)

  const float* W(int pi) const { return wblob + params[pi].off; }
  const float* Wlo(int pi) const { return params[pi].lo >= 0 ? wblob + params[pi].lo : nullptr; }   // split TF32 lo copy
  ~b200_ncsnpp() {
    for (auto* p : tcplans) tc_gemm_plan_destroy(p);
    for (auto* p : attnplans) tc_attn_plan_destroy(p);
    if (lane_stream) cudaStreamDestroy(lane_stream);
    if (ev_fork) cudaEventDestroy(ev_fork);
    if (ev_join) cudaEventDestroy(ev_join);
  }
};

namespace {

int add_param(b200_ncsnpp* e, const std::string& name, std::vector<long long> shape, int pack, int taps, int O,
              int I, int round, long long fixed_off = -1, long long reserve = 0) {
  Param p;
  p.name = name; p.ndim = (int)shape.size();
  p.count = 1;
  for (int i = 0; i < 4; ++i) { p.shape[i] = i < p.ndim ? shape[i] : 1; p.count *= p.shape[i]; }
  p.pack = pack; p.taps = taps; p.O = O; p.I = I; p.round = round;
  if (fixed_off >= 0) p.off = fixed_off;   // (split TF32: the caller places the lo copy)
  else {
    const long long n = (std::max(p.count, reserve) + 63) & ~63LL;
    p.off = e->wcount; e->wcount += n;
    if (round == 3) { p.lo = e->wcount; e->wcount += n; }
  }
  e->params.push_back(p);
  return (int)e->params.size() - 1;
}

// Tensor-core convolution descriptor with the fields every contraction of the engine shares: A = a1 [C1] (+ a2 [C2])
// over nimg images of H x W output pixels, W [taps][N][C1 + C2], one batch item, output pitch N, the engine's operand
// format and halo mode.  The gemm sites switch conv off and set their own batch geometry.
TcGemmDesc tc_desc(const b200_ncsnpp* e, const float* a1, int C1, const float* a2, int C2, int H, int W, int nimg, int taps,
                   const float* w, int N) {
  TcGemmDesc d; memset(&d, 0, sizeof(d));
  d.f16 = e->cfg.precision == 2; d.no_halo = e->cfg.no_halo;
  d.a1 = a1; d.C1 = C1; d.a2 = a2; d.C2 = C2; d.conv = 1; d.H = H; d.W = W; d.nimg = nimg; d.taps = taps;
  d.w = w; d.N_total = N; d.K_total = C1 + C2; d.w_rows = (long long)taps * N; d.nbatch = 1; d.epi.ld_out = N;
  return d;
}

// precision: 0 = tensor cores on TF32-grid fp32 operands, 1 = strict fp32 CUDA cores, 2 = tensor cores on fp16 operands
// (same 11-bit significand as TF32, fp32 accumulation; half the operand bytes and twice the MMA rate), 3 = split TF32
// ("3xTF32"): tensor cores on hi / lo TF32 pairs of fp32 operands, three products per K step, close to fp32 accuracy.
// In precision 3 producers write plain fp32 (as in precision 1); a split pass in front of each tensor-core contraction
// writes the hi / lo pair of each activation operand, and the weight blob holds a hi and a lo copy of every contraction
// weight.  The attention blocks run as separate contractions, the few-channel levels and the head on CUDA cores.
bool tc_ok(const b200_ncsnpp* e, int C1, int C2, int Cout, int H, int W, int taps) {
  if (e->cfg.precision == 1) return false;
  return tc_gemm_supported(tc_desc(e, nullptr, C1, C2 ? (const float*)1 : nullptr, C2, H, W, 1, taps, nullptr, Cout), nullptr);
}

bool has_attn(const b200_ncsnpp_config& c, int res) {
  for (int i = 0; i < c.num_attn_resolutions; ++i) if (c.attn_resolutions[i] == res) return true;
  return false;
}

// NCSNv2 walk (family 2): the level table of NCSNv2 (models/ncsnv2.py:43-100; num_levels = 4, the 'ncsnv2_64' network)
// and NCSNv2_128 (:221-276; num_levels = 5).  Level l has two ResidualBlocks with chans[l] output channels and filter
// dilation dil[l]; the first block of levels l > 0 is resample='down' (a 2x2 mean after its convolutions when dil[l] = 1,
// no resampling when dilated).  refine k (k = 1..L) takes [layer L-k (, the previous refine output)] to feat[k-1] channels.
struct NcsnWalk { int L; int chans[5]; int dil[5]; int feat[5]; };
NcsnWalk ncsnv2_walk(int L, int nf) {
  if (L == 4) return {4, {nf, 2 * nf, 2 * nf, 2 * nf}, {1, 1, 2, 4}, {2 * nf, 2 * nf, nf, nf}};
  return {5, {nf, 2 * nf, 2 * nf, 4 * nf, 4 * nf}, {1, 1, 1, 2, 4}, {4 * nf, 2 * nf, 2 * nf, nf, nf}};
}

int build_graph_ncsnv2(b200_ncsnpp* e) {
  const b200_ncsnpp_config& c = e->cfg;
  const int nf = c.nf, ch = c.num_channels, R = c.image_size;
  const NcsnWalk wk = ncsnv2_walk(c.num_levels, nf);
  const bool tcmode = c.precision != 1;
  const int om = c.precision == 2 ? 2 : 1;
  // a 3x3 / 1x1 convolution weight OIHW -> [tap][O][I], packed in the operand format when it runs on the tensor cores
  // (Param::round != 0 marks those; the walk reads it back)
  auto conv_param = [&](const std::string& name, int cin, int cout, int taps, int res, int dil, bool bias, int* pb) {
    TcGemmDesc d = tc_desc(e, nullptr, cin, nullptr, 0, res, res, 1, taps, nullptr, cout);
    d.dilation = dil;
    const bool tc = tcmode && tc_gemm_supported(d, nullptr);
    const int k = taps == 9 ? 3 : 1;
    const int pw = add_param(e, name + ".weight", {cout, cin, k, k}, PK_CONV, taps, cout, cin, tc ? om : 0);
    if (pb) *pb = bias ? add_param(e, name + ".bias", {cout}, PK_COPY, 0, 0, 0, 0) : -1;
    return pw;
  };
  auto in_params = [&](const std::string& name, int C, int (&dst)[3]) {   // InstanceNorm2dPlus: alpha, gamma, beta
    for (int k = 0; k < 3; ++k) dst[k] = add_param(e, name + (k == 0 ? ".alpha" : k == 1 ? ".gamma" : ".beta"), {C}, PK_COPY, 0, 0, 0, 0);
  };
  // begin_conv (ncsnv2.py:55): the input convolution of the shared walk (im2col + one K=32 contraction on the tensor cores)
  { Mod m; m.kind = M_CONV_IN; m.index = 0; m.cin1 = ch; m.cout = nf; m.res = R;
    m.tc0 = tcmode && (9 * ch <= 32) && (nf % 128 == 0);
    const int om_in = c.precision == 2 ? 2 : 1;
    m.w = m.tc0 ? add_param(e, "begin_conv.weight", {nf, ch, 3, 3}, PK_CONV_FLAT32, 9, nf, ch, om_in, -1, (long long)nf * 32)
                : add_param(e, "begin_conv.weight", {nf, ch, 3, 3}, PK_CONV, 9, nf, ch, 0);
    m.b = add_param(e, "begin_conv.bias", {nf}, PK_COPY, 0, 0, 0, 0); e->mods.push_back(m); }
  // normalizer and end_conv are registered right after begin_conv (ncsnv2.py:57-58) and run last
  Mod head; head.kind = M_NHEAD; head.index = -1; head.cin1 = nf; head.cout = ch; head.res = R;
  in_params("normalizer", nf, head.in[0]);
  head.w = add_param(e, "end_conv.weight", {ch, nf, 3, 3}, PK_CONV, 9, ch, nf, 0);
  head.b = add_param(e, "end_conv.bias", {ch}, PK_COPY, 0, 0, 0, 0);
  // ResidualBlock (layers.py:453-507) in its registration order: conv1, normalize2, conv2, shortcut, normalize1
  int res = R, cin = nf, idx = 1;
  std::vector<int> level_res;
  for (int l = 0; l < wk.L; ++l) {
    for (int b = 0; b < 2; ++b) {
      Mod m; m.kind = M_NRES; m.index = idx++; m.cin1 = cin; m.cout = wk.chans[l]; m.dil = wk.dil[l]; m.res = res;
      m.down = (l > 0 && b == 0) ? 1 : 0;
      const std::string nm = "res" + std::to_string(l + 1) + "." + std::to_string(b);
      const int d = m.dil, mid = m.down ? cin : m.cout;
      m.c0w = conv_param(nm + ".conv1", cin, mid, 9, res, d, true, &m.c0b);
      in_params(nm + ".normalize2", mid, m.in[1]);
      const bool meanpool = m.down && d == 1;   // ConvMeanPool (layers.py:351-369): the convolution at full resolution
      m.c1w = conv_param(nm + (meanpool ? ".conv2.conv" : ".conv2"), mid, m.cout, 9, res, d, true, &m.c1b);
      if (m.cout != cin || m.down) {
        // ConvMeanPool with a 1x1 filter, ncsn_conv1x1, or the dilated 3x3 (conv_shortcut, layers.py:462-484)
        const int taps = d > 1 ? 9 : 1;
        m.c2w = conv_param(nm + (meanpool ? ".shortcut.conv" : ".shortcut"), cin, m.cout, taps, res, d, true, &m.c2b);
      }
      in_params(nm + ".normalize1", cin, m.in[0]);
      e->mods.push_back(m);
      if (meanpool) res /= 2;
      cin = m.cout;
    }
    level_res.push_back(res);
  }
  // RefineBlock (layers.py:277-310) in its registration order: adapt_convs, output_convs, msf, crp
  for (int k = 1; k <= wk.L; ++k) {
    Mod m; m.kind = M_NREF; m.index = idx++;
    const int lay = wk.L - k, F = wk.feat[k - 1];
    const int ins[2] = {wk.chans[lay], k > 1 ? wk.feat[k - 2] : 0};
    const int rin[2] = {level_res[lay], k > 1 ? level_res[lay + 1] : 0};
    m.nin = k > 1 ? 2 : 1; m.cin1 = ins[0]; m.cout = F; m.res = level_res[lay];
    const bool end = k == wk.L;   // the output RCU has three blocks
    const std::string nm = "refine" + std::to_string(k);
    for (int i = 0; i < m.nin; ++i)
      for (int bl = 1; bl <= 2; ++bl)
        for (int st = 1; st <= 2; ++st)
          m.adapt[i].push_back(conv_param(nm + ".adapt_convs." + std::to_string(i) + "." + std::to_string(bl) + "_" +
                                          std::to_string(st) + "_conv", ins[i], ins[i], 9, rin[i], 1, false, nullptr));
    for (int bl = 1; bl <= (end ? 3 : 1); ++bl)
      for (int st = 1; st <= 2; ++st)
        m.outc.push_back(conv_param(nm + ".output_convs." + std::to_string(bl) + "_" + std::to_string(st) + "_conv", F, F, 9,
                                    m.res, 1, false, nullptr));
    if (m.nin > 1)
      for (int i = 0; i < 2; ++i) {
        int pb = -1;
        m.msfw.push_back(conv_param(nm + ".msf.convs." + std::to_string(i), ins[i], F, 9, rin[i], 1, true, &pb));
        m.msfb.push_back(pb);
      }
    for (int i = 0; i < 2; ++i) m.crp.push_back(conv_param(nm + ".crp.convs." + std::to_string(i), F, F, 9, m.res, 1, false, nullptr));
    e->mods.push_back(m);
  }
  e->mods.push_back(head);
  return 0;
}

int build_graph(b200_ncsnpp* e) {
  if (e->cfg.family == 2) return build_graph_ncsnv2(e);
  const b200_ncsnpp_config& c = e->cfg;
  const bool ddpm = c.family == 1;
  B200_REQUIRE(c.num_levels >= 1 && c.num_levels <= 8, "ncsnpp: num_levels=%d out of range", c.num_levels);
  B200_REQUIRE(c.nf % 4 == 0 && c.nf >= 8, "ncsnpp: nf=%d must be a multiple of 4", c.nf);
  if (ddpm) {   // every GroupNorm has 32 groups (layers.py:562, 625, 633; ddpm.py:104)
    B200_REQUIRE(c.nf % 32 == 0, "ddpm: nf=%d must be a multiple of 32 (GroupNorm with 32 groups)", c.nf);
    for (int i = 0; i < c.num_levels; ++i)
      B200_REQUIRE(c.ch_mult[i] >= 1 && (c.nf * c.ch_mult[i]) % 32 == 0, "ddpm: level %d has %d channels, not a multiple of 32", i, c.nf * c.ch_mult[i]);
  }
  B200_REQUIRE(c.conditional, "ncsnpp: unconditional models are not supported by the engine");
  B200_REQUIRE(c.fir_taps >= 1 && c.fir_taps <= 8, "ncsnpp: fir kernel length %d unsupported", c.fir_taps);
  B200_REQUIRE((c.image_size >> (c.num_levels - 1)) >= 1 && c.image_size % (1 << (c.num_levels - 1)) == 0,
               "ncsnpp: image_size=%d not divisible by 2^(levels-1)", c.image_size);
  // 2-D FIR = outer(k,k)/sum  (up_or_down_sampling.py:181-188)
  {
    double s = 0; for (int i = 0; i < c.fir_taps; ++i) s += c.fir_kernel[i];
    e->firn = c.fir_taps;
    for (int i = 0; i < c.fir_taps; ++i)
      for (int j = 0; j < c.fir_taps; ++j) {
        float kk = c.fir_kernel[i] * c.fir_kernel[j];
        e->fir2d[i * c.fir_taps + j] = kk / (float)(s * s);
      }
  }
  const int nf = c.nf, L = c.num_levels, nrb = c.num_res_blocks, ch = c.num_channels;
  const bool tcmode = c.precision != 1;
  // packed format of tensor-core weights (store_operand4 mode; 3: split TF32, a hi and a lo copy)
  const int om = c.precision == 2 ? 2 : c.precision == 3 ? 3 : 1;
  const int flatk = om == 2 ? 64 : 32;          // elements of one 128-byte K step (im2col contraction depth)
  std::vector<int> all_res(L);
  for (int i = 0; i < L; ++i) all_res[i] = c.image_size >> i;
  // The positional embedding has no module in all_modules (ncsnpp.py:79-83): its Mod below takes no index, so every
  // later module's index is its position in `mods` minus one.
  const int ishift = c.embedding_type == 1 ? 1 : 0;
  auto cur = [&]() { return (int)e->mods.size() - ishift; };
  auto nm = [&](const char* suffix) { return "all_modules." + std::to_string(cur()) + "." + suffix; };
  auto nmi = [&](int idx, const std::string& suffix) { return "all_modules." + std::to_string(idx) + "." + suffix; };

  // --- first pass: count Dense_0 rows so their packed rows are contiguous ---
  // (done lazily: dense region is reserved after the walk; Dense params get fixed offsets then)
  struct DenseFix { int pw, pb, row, cout; };
  std::vector<DenseFix> dense;

  {  // sigmas buffer is a state_dict key of the reference (ncsnpp.py:42) but unused on this path
    // (it is fp64 there; the host skips it when loading)
  }
  B200_REQUIRE(c.embedding_type == 0 || c.embedding_type == 1, "ncsnpp: embedding_type=%d unknown", c.embedding_type);
  B200_REQUIRE(!(c.embedding_type == 1 && c.scale_by_sigma), "ncsnpp: positional embedding with scale_by_sigma is not supported");
  B200_REQUIRE(!(c.naive_resample && c.progressive_input == 1), "ncsnpp: the residual input pyramid needs FIR resampling");
  B200_REQUIRE(c.progressive_input >= 0 && c.progressive_input <= 2, "ncsnpp: progressive_input=%d unknown", c.progressive_input);
  B200_REQUIRE(c.progressive == 0 || c.progressive == 1, "ncsnpp: progressive=%d unknown (0 none, 1 output_skip)", c.progressive);
  B200_REQUIRE((c.progressive == 0 && c.progressive_input != 2) || c.num_channels <= 4,
               "ncsnpp: the output_skip / input_skip pyramids carry the image channels (<= 4), got %d", c.num_channels);
  // 0: Fourier projection (all_modules[0].W [nf]) or the positional frequency table (pseudo-parameter [nf/2])
  const int emb_dim = c.embedding_type == 1 ? nf : 2 * nf;
  if (c.embedding_type == 1) {
    B200_REQUIRE(nf % 2 == 0 && nf >= 4, "ncsnpp: positional embedding needs an even nf >= 4");
    Mod m; m.kind = M_FOURIER; m.index = -1; m.w = add_param(e, "pos_freqs", {nf / 2}, PK_COPY, 0, 0, 0, 0); e->mods.push_back(m);
  } else {
    Mod m; m.kind = M_FOURIER; m.index = cur(); m.w = add_param(e, nm("W"), {nf}, PK_COPY, 0, 0, 0, 0); e->mods.push_back(m);
  }
  { Mod m; m.kind = M_LINEAR; m.index = cur(); m.cin1 = emb_dim; m.cout = 4 * nf;
    m.w = add_param(e, nm("weight"), {4 * nf, emb_dim}, PK_COPY, 0, 0, 0, 0); m.b = add_param(e, nm("bias"), {4 * nf}, PK_COPY, 0, 0, 0, 0); e->mods.push_back(m); }
  { Mod m; m.kind = M_LINEAR; m.index = cur(); m.cin1 = 4 * nf; m.cout = 4 * nf;
    m.w = add_param(e, nm("weight"), {4 * nf, 4 * nf}, PK_COPY, 0, 0, 0, 0); m.b = add_param(e, nm("bias"), {4 * nf}, PK_COPY, 0, 0, 0, 0); e->mods.push_back(m); }

  // NCSN++: ResnetBlockBigGANpp (layerspp.py:214-274); DDPM: ResnetBlockDDPM (layers.py:619-662), whose skip projection is
  // NIN_0 (W [in][out], packed like a 1x1 convolution) instead of Conv_2, and which never resamples
  auto add_resblock = [&](int cin1, int cin2, int cout, int up, int down, int res_in) {
    Mod m; m.kind = M_RESBLOCK; m.index = cur();
    const int cin = cin1 + cin2;
    m.cin1 = cin1; m.cin2 = cin2; m.cout = cout; m.up = up; m.down = down; m.res = res_in;
    m.has_conv2 = (cin != cout) || up || down;
    const int ro = up ? res_in * 2 : down ? res_in / 2 : res_in;
    m.tc0 = tc_ok(e, cin, 0, cout, ro, ro, 9);
    m.tc1 = tc_ok(e, cout, 0, cout, ro, ro, 9);
    m.tc2 = m.has_conv2 && tc_ok(e, cin, 0, cout, ro, ro, 1);
    m.gn0w = add_param(e, nm("GroupNorm_0.weight"), {cin}, PK_COPY, 0, 0, 0, 0);
    m.gn0b = add_param(e, nm("GroupNorm_0.bias"), {cin}, PK_COPY, 0, 0, 0, 0);
    m.c0w = add_param(e, nm("Conv_0.weight"), {cout, cin, 3, 3}, PK_CONV, 9, cout, cin, m.tc0 ? om : 0);
    m.c0b = add_param(e, nm("Conv_0.bias"), {cout}, PK_COPY, 0, 0, 0, 0);
    m.dw = add_param(e, nm("Dense_0.weight"), {cout, 4 * nf}, PK_COPY, 0, 0, 0, 0, 0);   // offset fixed below
    m.db = add_param(e, nm("Dense_0.bias"), {cout}, PK_COPY, 0, 0, 0, 0, 0);
    m.dense_row = e->sumC;
    dense.push_back({m.dw, m.db, e->sumC, cout});
    e->sumC += cout;
    m.gn1w = add_param(e, nm("GroupNorm_1.weight"), {cout}, PK_COPY, 0, 0, 0, 0);
    m.gn1b = add_param(e, nm("GroupNorm_1.bias"), {cout}, PK_COPY, 0, 0, 0, 0);
    m.c1w = add_param(e, nm("Conv_1.weight"), {cout, cout, 3, 3}, PK_CONV, 9, cout, cout, m.tc1 ? om : 0);
    m.c1b = add_param(e, nm("Conv_1.bias"), {cout}, PK_COPY, 0, 0, 0, 0);
    if (m.has_conv2 && ddpm) {
      m.c2w = add_param(e, nm("NIN_0.W"), {cin, cout}, PK_NIN, 1, cout, cin, m.tc2 ? om : 0);
      m.c2b = add_param(e, nm("NIN_0.b"), {cout}, PK_COPY, 0, 0, 0, 0);
    } else if (m.has_conv2) {
      m.c2w = add_param(e, nm("Conv_2.weight"), {cout, cin, 1, 1}, PK_CONV, 1, cout, cin, m.tc2 ? om : 0);
      m.c2b = add_param(e, nm("Conv_2.bias"), {cout}, PK_COPY, 0, 0, 0, 0);
    }
    e->mods.push_back(m);
  };
  // DDPM Downsample (pad (0,1,0,1) + 3x3 stride-2 VALID conv) and Upsample (nearest 2x + 3x3 conv): Conv_0 is C -> C
  auto add_resample = [&](ModKind kind, int C, int res_in) {
    Mod m; m.kind = kind; m.index = cur(); m.cin1 = C; m.cout = C; m.res = res_in;
    const int ro = kind == M_UP ? 2 * res_in : res_in / 2;
    m.tc0 = tc_ok(e, C, 0, C, ro, ro, 9);
    m.w = add_param(e, nm("Conv_0.weight"), {C, C, 3, 3}, PK_CONV, 9, C, C, m.tc0 ? om : 0);
    m.b = add_param(e, nm("Conv_0.bias"), {C}, PK_COPY, 0, 0, 0, 0);
    e->mods.push_back(m);
  };
  auto add_attn = [&](int C, int res) {
    Mod m; m.kind = M_ATTN; m.index = cur(); m.cin1 = C; m.cout = C; m.res = res;
    const int T = res * res;
    m.tcattn = tcmode && (C % 128 == 0) && (T % 128 == 0) && (T <= 1024);
    // fp16 operands: the logits/probabilities never leave the chip, so only the fused core (T = 256) and the flash core
    // (attn_flash.cu: T % 128 == 0 up to 4096, C = 128 / 256 / 512) are implemented
    if (om == 2) m.tcattn = tc_attn_supported(T, C, true) || attn_flash_supported(T, C);
    // few tokens (T <= 64: the 4x4 block of CIFAR-10, the 8x8, 512-channel bottleneck of FFHQ-1024): one CTA per image
    // (attn_small_kernel); otherwise the block runs as separate contractions
    const bool small_ok = attn_small_supported(T, C);
    m.tc0 = tcmode && (C % 128 == 0) && (m.tcattn || (small_ok && !c.tangent && c.precision != 3));   // q/k/v projections on tensor cores
    // (tangent and split-TF32 plans run every attention block as separate contractions: no small-token core, no fused core)
    m.gn0w = add_param(e, nm("GroupNorm_0.weight"), {C}, PK_COPY, 0, 0, 0, 0);
    m.gn0b = add_param(e, nm("GroupNorm_0.bias"), {C}, PK_COPY, 0, 0, 0, 0);
    // q,k,v projection weights packed as one [3C][C] block (rows: q, k, v), biases as one [3C] vector; split TF32: the lo
    // copies as a second [3C][C] block right after it
    const bool tcproj = m.tc0;
    const long long wbase = e->wcount; e->wcount += 3LL * C * C * (tcproj && om == 3 ? 2 : 1);
    const long long bbase = e->wcount; e->wcount += (3LL * C + 63) & ~63LL;
    for (int k = 0; k < 3; ++k) {
      m.nw[k] = add_param(e, nmi(m.index, "NIN_" + std::to_string(k) + ".W"), {C, C}, PK_NIN, 1, C, C, tcproj ? om : 0,
                          wbase + (long long)k * C * C / ((tcproj && om == 2) ? 2 : 1));   // fp16: the three blocks stay contiguous as [3C][C] halves
      if (tcproj && om == 3) e->params[m.nw[k]].lo = wbase + 3LL * C * C + (long long)k * C * C;
      m.nb[k] = add_param(e, nmi(m.index, "NIN_" + std::to_string(k) + ".b"), {C}, PK_COPY, 0, 0, 0, 0, bbase + (long long)k * C);
    }
    m.tc2 = tc_ok(e, C, 0, C, res, res, 1) && (om != 2 || m.tcattn || T <= 64);   // output projection as a 1x1 conv over pixels
    m.nw[3] = add_param(e, nmi(m.index, "NIN_3.W"), {C, C}, PK_NIN, 1, C, C, m.tc2 ? om : 0);
    m.nb[3] = add_param(e, nmi(m.index, "NIN_3.b"), {C}, PK_COPY, 0, 0, 0, 0);
    e->mods.push_back(m);
  };

  // input conv
  { Mod m; m.kind = M_CONV_IN; m.index = cur(); m.cin1 = ch; m.cout = nf; m.res = c.image_size;
    // on tensor cores the 3x3 input conv is one K=32 contraction over im2col patches: weights packed [nf][32]
    m.tc0 = tcmode && (9 * ch <= 32) && (nf % 128 == 0);
    // nf = 16 / 32 / 64 (the high-resolution family) in TF32 mode: the same patches, contracted by the few-channel kernel
    m.tc1 = !m.tc0 && c.precision == 0 && (9 * ch <= 32) && (nf == 16 || nf == 32 || nf == 64) && c.image_size % 32 == 0;
    m.w = (m.tc0 || m.tc1) ? add_param(e, nm("weight"), {nf, ch, 3, 3}, PK_CONV_FLAT32, 9, nf, ch, om, -1, (long long)nf * 32)
                : add_param(e, nm("weight"), {nf, ch, 3, 3}, PK_CONV, 9, nf, ch, 0);
    m.b = add_param(e, nm("bias"), {nf}, PK_COPY, 0, 0, 0, 0); e->mods.push_back(m); }
  std::vector<int> hs_c = {nf};
  int in_ch = nf, pyr_ch = ch;
  for (int lvl = 0; lvl < L; ++lvl) {
    for (int b = 0; b < nrb; ++b) {
      const int out_ch = nf * c.ch_mult[lvl];
      add_resblock(in_ch, 0, out_ch, 0, 0, all_res[lvl]);
      in_ch = out_ch;
      if (has_attn(c, all_res[lvl])) add_attn(in_ch, all_res[lvl]);
      hs_c.push_back(in_ch);
    }
    if (lvl != L - 1) {
      if (ddpm) add_resample(M_DOWN, in_ch, all_res[lvl]);
      else add_resblock(in_ch, 0, in_ch, 0, 1, all_res[lvl]);
      if (c.progressive_input == 2) {
        // Combine(dim1 = image channels, dim2 = in_ch, method 'sum') (layerspp.py:44-59, ncsnpp.py:163-166): Conv_0 is a 1x1
        Mod m; m.kind = M_COMBINE; m.index = cur(); m.cin1 = ch; m.cout = in_ch; m.res = all_res[lvl] / 2;
        m.w = add_param(e, nm("Conv_0.weight"), {in_ch, ch, 1, 1}, PK_CONV, 1, in_ch, ch, 0);
        m.b = add_param(e, nm("Conv_0.bias"), {in_ch}, PK_COPY, 0, 0, 0, 0);
        e->mods.push_back(m);
      }
      if (c.progressive_input == 1) {
        Mod m; m.kind = M_PYR_DOWN; m.index = cur(); m.cin1 = pyr_ch; m.cout = in_ch; m.res = all_res[lvl];
        // FIR-padded stride-2 VALID conv: on the tensor cores via TMA element strides when the channel counts tile
        m.tc0 = tc_ok(e, pyr_ch, 0, in_ch, all_res[lvl] / 2, all_res[lvl] / 2, 9);
        // image-channel pyramid level (3 channels): im2col patches + one K=32 contraction, like the input conv
        m.tc2 = tcmode && (9 * pyr_ch <= 32) && tc_ok(e, flatk, 0, in_ch, all_res[lvl] / 2, all_res[lvl] / 2, 1);
        m.w = m.tc2 ? add_param(e, nm("Conv2d_0.weight"), {in_ch, pyr_ch, 3, 3}, PK_CONV_FLAT32, 9, in_ch, pyr_ch, om, -1, (long long)in_ch * 32)
                    : add_param(e, nm("Conv2d_0.weight"), {in_ch, pyr_ch, 3, 3}, PK_CONV, 9, in_ch, pyr_ch, m.tc0 ? om : 0);
        m.b = add_param(e, nm("Conv2d_0.bias"), {in_ch}, PK_COPY, 0, 0, 0, 0);
        e->mods.push_back(m);
        pyr_ch = in_ch;
      }
      hs_c.push_back(in_ch);
    }
  }
  in_ch = hs_c.back();
  add_resblock(in_ch, 0, in_ch, 0, 0, all_res[L - 1]);
  add_attn(in_ch, all_res[L - 1]);
  add_resblock(in_ch, 0, in_ch, 0, 0, all_res[L - 1]);
  for (int lvl = L - 1; lvl >= 0; --lvl) {
    for (int b = 0; b < nrb + 1; ++b) {
      const int out_ch = nf * c.ch_mult[lvl];
      const int skip = hs_c.back(); hs_c.pop_back();
      add_resblock(in_ch, skip, out_ch, 0, 0, all_res[lvl]);
      in_ch = out_ch;
    }
    if (has_attn(c, all_res[lvl])) add_attn(in_ch, all_res[lvl]);
    if (c.progressive == 1) {
      // output_skip (ncsnpp.py:190-203, 325-341): GroupNorm + SiLU + conv3x3 (in_ch -> image channels) at every level;
      // the image-channel pyramid is upsampled and summed, and IS the network output
      { Mod m; m.kind = M_GN_OUT; m.index = cur(); m.cin1 = in_ch; m.res = all_res[lvl];
        m.w = add_param(e, nm("weight"), {in_ch}, PK_COPY, 0, 0, 0, 0); m.b = add_param(e, nm("bias"), {in_ch}, PK_COPY, 0, 0, 0, 0); e->mods.push_back(m); }
      { Mod m; m.kind = M_CONV_OUT; m.index = cur(); m.cin1 = in_ch; m.cout = ch; m.res = all_res[lvl]; m.tc0 = false;
        m.w = add_param(e, nm("weight"), {ch, in_ch, 3, 3}, PK_CONV, 9, ch, in_ch, 0);
        m.b = add_param(e, nm("bias"), {ch}, PK_COPY, 0, 0, 0, 0); e->mods.push_back(m); }
    }
    if (lvl != 0) {
      if (ddpm) add_resample(M_UP, in_ch, all_res[lvl]);
      else add_resblock(in_ch, 0, in_ch, 1, 0, all_res[lvl]);
    }
  }
  B200_REQUIRE(hs_c.empty(), "ncsnpp: internal skip-stack mismatch");
  if (c.progressive != 1) {
  { Mod m; m.kind = M_GN_OUT; m.index = cur(); m.cin1 = in_ch;
    m.w = add_param(e, nm("weight"), {in_ch}, PK_COPY, 0, 0, 0, 0); m.b = add_param(e, nm("bias"), {in_ch}, PK_COPY, 0, 0, 0, 0); e->mods.push_back(m); }
  { Mod m; m.kind = M_CONV_OUT; m.index = cur(); m.cin1 = in_ch; m.cout = ch; m.res = c.image_size;
    // Head on tensor cores: the ch (3) output channels become rows 0..ch-1 of a zero-padded 128-row weight tile
    // ([9][128][in_ch]; bias padded likewise), run as a swapped-operand convolution whose epilogue stores only those
    // rows, as NCHW, divided by sigma.  2.3x faster than the CUDA-core head despite the 125 idle rows.
    // cfg.cuda_core_head = 1 keeps the head on CUDA cores with an fp32 input (it is the one convolution with no later
    // layer to average its operand rounding: +1e-4 of the parity budget on tensor cores).
    // (split TF32 keeps the head on CUDA cores: strict fp32, no zero-padded pair of weight tiles)
    m.tc0 = !c.cuda_core_head && tcmode && c.precision != 3 && ch <= 32 && tc_ok(e, in_ch, 0, 128, c.image_size, c.image_size, 9) && (c.image_size * c.image_size) % 256 == 0 &&
            (c.image_size <= 128 || c.image_size % 128 == 0);
    m.w = m.tc0 ? add_param(e, nm("weight"), {ch, in_ch, 3, 3}, PK_CONV_PAD128, 9, ch, in_ch, om, -1, 9LL * 128 * in_ch)
                : add_param(e, nm("weight"), {ch, in_ch, 3, 3}, PK_CONV, 9, ch, in_ch, 0);
    m.b = add_param(e, nm("bias"), {ch}, PK_COPY, 0, 0, 0, 0, -1, m.tc0 ? 128 : 0); e->mods.push_back(m); }
  }

  // contiguous Dense_0 block: one [sumC][4nf] matrix + [sumC] bias for a single batched linear
  e->dense_w_off = e->wcount; e->wcount += ((long long)e->sumC * 4 * nf + 63) & ~63LL;
  e->dense_b_off = e->wcount; e->wcount += (e->sumC + 63) & ~63LL;
  for (auto& d : dense) {
    e->params[d.pw].off = e->dense_w_off + (long long)d.row * 4 * nf;
    e->params[d.pb].off = e->dense_b_off + d.row;
  }
  return 0;
}

// ---------------------------------------------------------------------------
// Plan builder
// ---------------------------------------------------------------------------
// GroupNorm coefficient tables for the few-channel convolutions that normalise while staging their input
struct Coef { float* scale = nullptr; float* shift = nullptr; long long bytes = 0; };

// optional arguments of conv(), set by name: conv(..., Conv().taps(1).residual(x).scale(s).stats())
struct Conv {
  int taps_ = 9, stride_ = 1, Hin_ = 0, round_ = 0, row_ = -1, skip_w_ = -1, skip_b_ = -1;
  Tensor residual_, skip1_, skip2_;
  float scale_ = 1.f; bool stats_ = false; const Coef* gn_ = nullptr;
  Conv& taps(int t) { taps_ = t; return *this; }                        // 9 (3x3) or 1 (1x1)
  Conv& stride(int s, int Hin) { stride_ = s; Hin_ = Hin; return *this; }   // stride 2: VALID over Hin x Hin inputs
  Conv& residual(const Tensor& r) { residual_ = r; return *this; }      // out = (acc + bias + residual) * scale
  Conv& scale(float s) { scale_ = s; return *this; }
  Conv& round(int r) { round_ = r; return *this; }                      // output format (store_operand4 mode)
  Conv& stats() { stats_ = true; return *this; }                        // GroupNorm quad sums of the output, when fused
  Conv& temb(int dense_row) { row_ = dense_row; return *this; }         // + this block's Dense_0 row of the time embedding
  // fused skip projection: the 1x1 conv (weights pw, bias pb) of x1 (+ x2) as extra K steps (tensor-core path)
  Conv& skip(const Tensor& x1, const Tensor& x2, int pw, int pb) { skip1_ = x1; skip2_ = x2; skip_w_ = pw; skip_b_ = pb; return *this; }
  Conv& gn(const Coef& c) { gn_ = &c; return *this; }                   // GroupNorm+SiLU on load (few-channel kernel)
  int dil_ = 1;
  Conv& dilation(int d) { dil_ = d; return *this; }                     // 3x3 'same' filter taps d pixels apart (padding d)
};

struct Builder {
  b200_ncsnpp* e; int B; char* base; bool dry; Arena arena; int rc = 0;
  char* stats_base = nullptr; long long stats_top = 0;   // bump region for GroupNorm quad sums, zeroed once per forward
  bool fused_stats = false;
  bool lowc_gn = false;                        // the few-channel convolutions (conv_lowc.cu, TF32 mode) apply GroupNorm+SiLU while staging their input
  int lane = 0;                                // which half-batch plan this builder fills (ops or ops2)
  int om = 1;                                  // operand store mode of tensor-core inputs: 1 TF32-grid fp32, 2 fp16, 0 fp32 (split TF32)
  bool split = false;                          // split TF32 (precision 3): contractions read hi / lo pairs made by split_pair()
  std::string next_name;                       // label of the next op (shape summary for the per-op profile)
  double next_bytes = 0.0;                     // algorithmic HBM bytes of the next op
  bool tan = false;                            // tangent plan (cfg.tangent): every tensor carries its tangent in Tensor::d
  bool tan_op = false;                         // the op being added is a tangent op (labelled "tangent[...]"); set by tangent()
  size_t mi = 3;                               // next module of e->mods to plan (0..2: the time embedding)
  const float* dense_all_ = nullptr;           // Dense_0 rows of every resblock [B][sumC]
  Tensor pyr; bool pyr_nchw = true, pyr_owned = false; long long pyr_bytes = 0;   // input pyramid (progressive_input)
  float* opyr = nullptr; long long opyr_bytes = 0;      // output_skip pyramid [B][ch][H][W] of the previous (coarser) level
  void name(const char* fmt, ...) {
    char buf[160]; va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap); next_name = buf;
  }
  Builder(b200_ncsnpp* e_, int B_, char* base_, bool dry_, int lane_ = 0) : e(e_), B(B_), base(base_), dry(dry_), arena(e_->cfg.keep_activations != 0), lane(lane_) {
    fused_stats = e_->cfg.precision != 1 && e_->cfg.family != 2;   // (NCSNv2's InstanceNorm statistics take a pass of their own)
    split = e_->cfg.precision == 3;
    om = e_->cfg.precision == 2 ? 2 : split ? 0 : 1;
    tan = e_->cfg.tangent != 0;
    lowc_gn = e_->cfg.precision == 0 && !tan;
    if (dry_) stats_base = reinterpret_cast<char*>(uintptr_t(1) << 40);   // any non-null base: only offsets matter in a dry run
  }
  // the tangent of t as a tensor of its own (for the linear ops, which run the forward kernels on it)
  static Tensor tg(const Tensor& t) { Tensor r = t; r.p = t.d; r.d = nullptr; r.qs = nullptr; return r; }
  double* qalloc(int C) {
    const long long bytes = ((long long)B * (C / 4) * 2 * 8 + 255) & ~255LL;
    double* p = reinterpret_cast<double*>(stats_base + stats_top);
    stats_top += bytes;
    return p;
  }

  Tensor talloc(int C, int H, int W) {
    Tensor t; t.C = C; t.H = H; t.W = W; t.bytes = (long long)B * H * W * C * 4 * (tan ? 2 : 1);
    const long long off = arena.alloc(t.bytes); arena.note();
    t.p = reinterpret_cast<float*>(base + off);
    if (tan) t.d = t.p + (long long)B * H * W * C;
    return t;
  }
  float* falloc(long long floats, long long* bytes_out) {
    *bytes_out = floats * 4;
    const long long off = arena.alloc(*bytes_out); arena.note();
    return reinterpret_cast<float*>(base + off);
  }
  void tfree(Tensor& t) { if (t.p) arena.release((char*)t.p - base, t.bytes); t.p = nullptr; t.d = nullptr; }
  // a plain buffer and, in tangent plans, its tangent twin (*dp; nullptr otherwise): one allocation of twice the size
  float* falloc2(long long floats, long long* bytes_out, float** dp) {
    float* p = falloc(floats * (tan ? 2 : 1), bytes_out);
    *dp = tan ? p + floats : nullptr;
    return p;
  }
  void ffree(float* p, long long bytes) { arena.release((char*)p - base, bytes); }

  // split TF32: hi = rna_tf32(x) and lo = rna_tf32(x - hi) of the n fp32 elements at x, one split pass into a temporary
  // [hi | lo] buffer.  The caller releases it once the contraction that reads it is planned (later ops, which may reuse
  // the memory, run after that contraction).
  struct Pair { const float* hi = nullptr; const float* lo = nullptr; float* buf = nullptr; long long bytes = 0; };
  Pair split_pair(const float* x, long long n, const char* what) {
    Pair s;
    if (!x) return s;
    if (n % 4) { set_error("ncsnpp: split TF32 operand of %lld elements (not a multiple of 4)", n); rc = 2; return s; }
    s.buf = falloc(2 * n, &s.bytes);
    float* hi = s.buf; float* lo = s.buf + n;
    s.hi = hi; s.lo = lo;
    name("split 3xtf32 %s", what);
    next_bytes = n * 12.0;
    op(1, [=](cudaStream_t st) { return launch_split_tf32(x, hi, lo, n, st); }, 6);
    return s;
  }
  void release(Pair& s) { if (s.buf) ffree(s.buf, s.bytes); s = Pair(); }

  // kind: 0 tensor-core contraction, 1 CUDA-core contraction, 2 GroupNorm, 3 FIR, 4 softmax, 5 time embedding, 6 misc
  void op(int launches, std::function<int(cudaStream_t)> f, int kind = 6, double flops = 0.0) {
    if (dry) return;
    e->launches += launches;
    static const char* kind_names[] = {"tensor-core contraction", "cuda-core contraction", "groupnorm", "fir", "softmax", "time embedding", "misc", "mma.sync contraction"};
    std::string label = next_name.empty() ? std::string(kind_names[kind & 7]) : next_name;
    // tangent ops of a tangent plan: their own launch on the tangent buffers ("separate" form; no 2B-image contraction)
    if (tan_op) label = "tangent[separate]: " + label;
    (lane ? e->ops2 : e->ops).push_back({kind, flops, std::move(f), label, next_bytes});
    next_name.clear(); next_bytes = 0.0;
  }

  // A linear op and, in tangent plans, its tangent twin: emit(false) adds the op on the primal buffers, emit(true) the same
  // op on the tangent buffers (Tensor::d, no bias, J v into tout), which op() labels "tangent[separate]: " + the label.
  template <class F> void twin(F emit) {
    emit(false);
    if (tan) tangent([&] { emit(true); });
  }
  // ops of tangent plans that are not copies of a primal op: gn_tangent, softmax_tangent, the attention product rule
  template <class F> void tangent(F emit) { tan_op = true; emit(); tan_op = false; }

  const Mod& next() { return e->mods[mi++]; }
  // the block output nh replaces the running activation h (freed) and is recorded as module m's output
  void advance(Tensor& h, const Mod& m, const Tensor& nh) { tfree(h); h = nh; tap(m.index, h); }

  // CUDA-core / few-channel convolution descriptor over the B images of this plan: x1 [B][H][W][C1] -> [B][OH][OW][N] with
  // `taps` (9: 3x3, 'same' padding at stride 1, VALID at stride 2; 1: 1x1), weights w [taps][N][C1]; unit epilogue
  SimtConv simt_desc(const float* x1, int C1, int H, int W, int taps, int stride, int OH, int OW, const float* w, int N) const {
    SimtConv s; memset(&s, 0, sizeof(s));
    s.x1 = x1; s.C1 = C1; s.in_scale = 1.f; s.H = H; s.W = W; s.R = s.S = (taps == 9 ? 3 : 1); s.stride = stride;
    s.pad = (taps == 9 && stride == 1 ? 1 : 0); s.OH = OH; s.OW = OW; s.nbatch = B; s.a_batched = 1; s.w = w; s.N = N;
    s.epi.scale = 1.f; s.epi.rows_per_img = OH * OW; s.epi.ld_out = N; s.epi.ld_res = N;
    return s;
  }

  // make sure tensor t has quad sums: produced by its tensor-core epilogue, else by one streaming pass
  void ensure_qs(Tensor& t) {
    if (t.qs || !t.p) return;
    t.qs = qalloc(t.C);
    const Tensor tt = t; const int Bc = B;
    name("gn_quad_stats %d @%d", t.C, t.H);
    op(1, [=](cudaStream_t st) { return launch_gn_quad_stats(tt.p, tt.C, Bc, tt.H * tt.W, tt.qs, st, /*qsums_zeroed=*/true); }, 2);
  }
  // GroupNorm group count: min(C/4, 32) in NCSN++ (layerspp.py:219, 235), 32 everywhere in DDPM (layers.py:562, 625, 633)
  int groups(int C) const { return e->cfg.family == 1 ? 32 : std::min(C / 4, 32); }
  // draw: tangent of the raw copy (tangent plans)
  void gn(Tensor& x1, Tensor& x2, int pgw, int pgb, int act, int round, Tensor y, float* raw, float* draw = nullptr) {
    const int C = x1.C + x2.C, G = groups(C), HW = x1.H * x1.W;
    if ((C / G) % 4 != 0) {
      // groups that are not whole channel quads (C = 192 -> 6 channels per group): the generic two-kernel path
      if (x1.f16 || x2.f16) { set_error("ncsnpp: GroupNorm with %d-channel groups on an fp16 tensor", C / G); rc = 2; return; }
      long long mb; float* mr = falloc(gn_generic_workspace_floats(B, HW, G), &mb);
      const float *g = e->W(pgw), *bt = e->W(pgb);
      const Tensor a = x1, b = x2; const int Bc = B;
      name("gn_generic %d+%d @%d (%d-channel groups)", x1.C, x2.C, x1.H, C / G);
      op(3, [=](cudaStream_t st) { return launch_gn_generic(a.p, a.C, b.p, b.C, g, bt, Bc, HW, G, 1e-6f, act, round, y.p, raw, mr, st); }, 2);
      if (tan) gn_tangent(x1, x2, g, bt, act, round, y, draw, mr, G, HW);   // reads the primal mean / rstd table
      ffree(mr, mb);
      return;
    }
    ensure_qs(x1); ensure_qs(x2);
    const float *g = e->W(pgw), *bt = e->W(pgb);
    const Tensor a = x1, b = x2; const int Bc = B;
    name("gn_apply %d+%d @%d%s%s%s", x1.C, x2.C, x1.H, act ? " silu" : "", raw ? " +raw" : "", x1.f16 ? " f16-in" : "");
    op(1, [=](cudaStream_t st) {
      return launch_gn_apply(a.p, a.C, b.p, b.C, a.qs, b.qs, g, bt, Bc, HW, G, 1e-6f, act, round, y.p, raw, st, a.f16 ? 1 : 0);
    }, 2);
    if (tan) gn_tangent(x1, x2, g, bt, act, round, y, draw, nullptr, G, HW);   // reads the primal quad sums
  }
  void gn_tangent(const Tensor& a, const Tensor& b, const float* g, const float* bt, int act, int round, const Tensor& y, float* draw,
                  const float* mr, int G, int HW) {
    const int Bc = B;
    name("gn_tangent %d+%d @%d%s%s (%s stats)", a.C, b.C, a.H, act ? " silu" : "", draw ? " +raw" : "", mr ? "generic" : "quad");
    tangent([&] {
      op(1, [=](cudaStream_t st) {
        return launch_gn_tangent(a.p, a.d, a.C, b.p, b.d, b.C, a.qs, b.qs, mr, g, bt, Bc, HW, G, 1e-6f, act, round, y.d, draw, st);
      }, 2);
    });
  }

  Coef gncoef(Tensor& x1, Tensor& x2, int pgw, int pgb) {
    const int C = x1.C + x2.C, G = groups(C), HW = x1.H * x1.W;
    ensure_qs(x1); ensure_qs(x2);
    Coef c;
    c.scale = falloc(2LL * B * C, &c.bytes); c.shift = c.scale + (long long)B * C;
    const float *g = e->W(pgw), *bt = e->W(pgb);
    const Tensor a = x1, b = x2; const int Bc = B; const Coef cc = c;
    name("gn_coeff %d+%d @%d", x1.C, x2.C, x1.H);
    op(1, [=](cudaStream_t st) { return launch_gn_coeff(a.C, b.C, a.qs, b.qs, g, bt, Bc, HW, G, 1e-6f, cc.scale, cc.shift, st); }, 2);
    return c;
  }
  // 2x resampling of a resblock (layerspp.py:244-256).  fir=True: upsample_2d / downsample_2d with the configured FIR
  // (up_or_down_sampling.py:218-224, 252-257); fir=False: naive_upsample_2d (nearest-neighbour repeat) and
  // naive_downsample_2d (2x2 mean) (:59-69), expressed as the same upfirdn2d with a 2x2 box: up=2, pad (1,0), taps 1
  // -> out[2i] = out[2i+1] = x[i]; down=2, pad (0,0), taps 1/4 -> the mean of each 2x2 cell.
  void resample2x(const float* x, int H, int C, bool up, int round, float* y) {
    if (e->cfg.naive_resample) {
      fir(x, B, H, H, C, up ? 2 : 1, up ? 1 : 2, up ? 1 : 0, 0, round, y, up ? 1.f : 0.25f, /*box=*/true);
      return;
    }
    const int p = e->firn - 2;
    if (up) fir(x, B, H, H, C, 2, 1, (p + 1) / 2 + 1, p / 2, round, y, 4.f);
    else fir(x, B, H, H, C, 1, 2, (p + 1) / 2, p / 2, round, y, 1.f);
  }

  // the same 2x resampling on [planes][H][W] tensors (image-channel pyramids kept NCHW): Downsample / Upsample with
  // with_conv=False (layerspp.py:113-126, 150-163): downsample_2d / upsample_2d, or avg_pool2d / nearest when fir=False
  void resample2x_planes(const float* x, int planes, int H, bool up, float* y) {
    if (e->cfg.naive_resample) { fir(x, planes, H, H, 1, up ? 2 : 1, up ? 1 : 2, up ? 1 : 0, 0, 0, y, up ? 1.f : 0.25f, /*box=*/true); return; }
    const int p = e->firn - 2;
    if (up) fir(x, planes, H, H, 1, 2, 1, (p + 1) / 2 + 1, p / 2, 0, y, 4.f);
    else fir(x, planes, H, H, 1, 1, 2, (p + 1) / 2, p / 2, 0, y, 1.f);
  }

  void fir(const float* x, int major, int H, int W, int minor, int up, int down, int pad0, int pad1, int round, float* y,
           float gain, bool box = false) {
    // kernel taps scaled by `gain` (x factor^2 when upsampling, up_or_down_sampling.py:220)
    std::vector<float> k(box ? 4 : e->firn * e->firn);
    for (size_t i = 0; i < k.size(); ++i) k[i] = box ? gain : e->fir2d[i] * gain;
    const int n = box ? 2 : e->firn;
    name("fir up%d down%d %d @%d", up, down, minor == 1 ? major / B : minor, H);
    op(1, [=](cudaStream_t st) {
      return launch_upfirdn2d(x, k.data(), y, major, H, W, minor, n, n, up, up, down, down, pad0, pad1, pad0, pad1, round, st);
    }, 3);
  }

  // 3x3 / 1x1 convolution on NHWC tensors into out (out.C channels), stride 1 'same' or stride 2 VALID.  In tangent plans
  // it is followed by its tangent: the same contraction over the tangents of the operands and of the residual, without
  // bias, time-embedding row or GroupNorm sums.
  void conv(bool use_tc, const Tensor& a1, const Tensor& a2, int pw, int pb, Tensor& out, const Conv& o = Conv()) {
    twin([&](bool d) {
      if (!d) return conv_op(use_tc, a1, a2, pw, pb, out, o);
      Conv t = o; t.residual_ = tg(o.residual_); t.row_ = -1; t.stats_ = false;
      Tensor dout = tg(out);
      conv_op(use_tc, tg(a1), tg(a2), pw, -1, dout, t);
    });
  }
  void conv_op(bool use_tc, const Tensor& a1, const Tensor& a2, int pw, int pb, Tensor& out, const Conv& o) {
    const int Cout = out.C, taps = o.taps_, stride = o.stride_, Hin = o.Hin_, dense_row = o.row_;
    const Tensor &x3 = o.skip1_, &x4 = o.skip2_;
    const float* residual = o.residual_.p;
    Epilogue ep; memset(&ep, 0, sizeof(ep));
    ep.bias = pb >= 0 ? e->W(pb) : nullptr;   // pb < 0: no bias (tangent ops)
    ep.rowvec = nullptr;   // patched at launch (depends on the per-call buffers)
    ep.residual = residual; ep.ld_res = Cout; ep.scale = o.scale_; ep.round_tf32 = o.round_;
    ep.rows_per_img = out.H * out.W; ep.out = out.p; ep.ld_out = Cout;
    b200_ncsnpp* eng = e;
    const float* dense_all = dense_all_;
    const int sumC = e->sumC;
    const double cflops = 2.0 * B * out.H * out.W * (double)Cout * ((a1.C + a2.C) * taps + x3.C + x4.C);
    if (x3.p && !use_tc) { set_error("ncsnpp: fused skip projection needs the tensor-core path"); rc = 2; return; }
    if (o.gn_ && use_tc) { set_error("ncsnpp: conv(): GroupNorm coefficients go with the few-channel kernel (the tensor-core path reads normalised operands)"); rc = 2; return; }
    if (use_tc) {
      TcGemmDesc d = tc_desc(e, a1.p, a1.C, a2.p, a2.C, out.H, out.W, B, taps, e->W(pw), Cout);
      d.stride = stride; d.valid_pad = stride == 2 ? 1 : 0; d.Hin = Hin ? Hin : out.H; d.Win = Hin ? Hin : out.W;
      d.dilation = o.dil_;
      if (dense_row >= 0) ep.rowvec = dense_all + dense_row;
      if (x3.p) {   // fused skip projection: its bias rides in the (image-independent) row-vector slot
        if (dense_row >= 0) { set_error("ncsnpp: fused skip projection on a conv with a time-embedding bias"); rc = 2; return; }
        d.a3 = x3.p; d.C3 = x3.C; d.a4 = x4.p; d.C4 = x4.C; d.w2 = e->W(o.skip_w_);
        ep.rowvec = e->W(o.skip_b_); ep.rowvec_ld = 0;
      }
      if (o.stats_ && fused_stats && (ep.rows_per_img % 32 == 0 || ep.rows_per_img == 16)) { out.qs = qalloc(Cout); d.qstats = out.qs; }
      d.epi = ep;
      if (split) {   // every activation operand as a hi / lo pair, the weights' lo copies from the blob
        const Tensor* src[4] = {&a1, &a2, &x3, &x4};
        Pair pr[4];
        for (int s = 0; s < 4; ++s) {
          const Tensor& t = *src[s];
          pr[s] = split_pair(t.p, (long long)B * t.H * t.W * t.C, s < 2 ? "conv input" : "skip input");
        }
        if (rc) return;
        d.split = 1;
        d.a1 = pr[0].hi; d.a1_lo = pr[0].lo; d.a2 = pr[1].hi; d.a2_lo = pr[1].lo;
        d.a3 = pr[2].hi; d.a3_lo = pr[2].lo; d.a4 = pr[3].hi; d.a4_lo = pr[3].lo;
        d.w_lo = e->Wlo(pw); d.w2_lo = x3.p ? e->Wlo(o.skip_w_) : nullptr;
        for (auto& q : pr) release(q);
      }
      if (dry) return;
      TcGemmPlan* pl = nullptr;
      if (int r = tc_gemm_plan_create(d, &pl)) { rc = r; return; }
      e->tcplans.push_back(pl);
      name("conv%s %d+%d->%d @%d%s%s%s [%s]", taps == 9 ? "3x3" : "1x1", a1.C, a2.C, Cout, out.H, stride == 2 ? " s2" : "",
           x3.p ? " +skipproj" : "", residual ? " +res" : "", tc_gemm_form(pl));
      if (o.dil_ > 1) next_name += " d" + std::to_string(o.dil_);
      if (x3.p) next_name += " " + std::to_string(x3.C + x4.C);
      {
        const double es = om == 2 ? 2.0 : split ? 8.0 : 4.0, px = (double)B * out.H * out.W;   // split TF32: hi + lo
        const double in_px = (double)B * (Hin ? (double)Hin * Hin : (double)out.H * out.W);
        next_bytes = in_px * (a1.C + a2.C) * es + px * (x3.C + x4.C) * es + px * Cout * (o.round_ == 2 ? 2.0 : 4.0) +
                     (residual ? px * Cout * 4.0 : 0.0) + ((double)taps * (a1.C + a2.C) + x3.C + x4.C) * Cout * es;
      }
      op(1, [=](cudaStream_t st) {
        if (dense_row >= 0) tc_gemm_set_rowvec_ld(pl, eng->uniform ? 0 : sumC);
        return tc_gemm_launch(pl, st);
      }, 0, cflops);
    } else {
      SimtConv s = simt_desc(a1.p, a1.C, a1.H, a1.W, taps, 1, a1.H, a1.W, e->W(pw), Cout);
      s.x2 = a2.p; s.C2 = a2.C;
      if (o.dil_ > 1) { s.dilation = o.dil_; s.pad = o.dil_; }
      if (dense_row >= 0) ep.rowvec = dense_all + dense_row;
      s.epi = ep;
      // few-channel levels of the nf = 16 networks: warp-level TF32 MMAs keep them at the HBM roofline (conv_lowc.cu);
      // strict-fp32 mode and every other shape stay on the CUDA-core kernel
      // (tangent and split-TF32 plans keep every level on the CUDA-core kernel)
      const bool lowc = e->cfg.precision != 1 && !split && !tan && !a1.f16 && !a2.f16 && sumC % 2 == 0 && conv_lowc_supported(s);
      if (o.stats_ && lowc && fused_stats) { out.qs = qalloc(Cout); s.qstats = out.qs; }   // the epilogue sums what the next GroupNorm needs
      if (o.gn_) {
        if (!lowc) { set_error("ncsnpp: GroupNorm on load planned for a convolution the few-channel kernel does not take"); rc = 2; return; }
        s.gn_scale = o.gn_->scale; s.gn_shift = o.gn_->shift; s.gn_act = 1;
      }
      name("conv%s %s%d+%d->%d @%d [%s]", taps == 9 ? "3x3" : "1x1", o.gn_ ? "gn+silu " : "", a1.C, a2.C, Cout, out.H, lowc ? "mma.sync tf32" : "cuda-core");
      if (o.dil_ > 1) next_name += " d" + std::to_string(o.dil_);
      next_bytes = (double)B * out.H * out.W * ((a1.C + a2.C) * 4.0 + Cout * 4.0 + (residual ? Cout * 4.0 : 0.0)) +
                   (double)taps * (a1.C + a2.C) * Cout * 4.0;
      op(1, [=](cudaStream_t st) {
        SimtConv c = s;
        if (dense_row >= 0) c.epi.rowvec_ld = eng->uniform ? 0 : sumC;
        return lowc ? launch_conv_lowc(c, st) : launch_conv_simt(c, st);
      }, lowc ? 7 : 1, cflops);
    }
  }

  // batched C[b] = A[b] * W[b]^T.  Split TF32: a_lo / w_lo are the lo twins of A / W when the caller has them (weights, an
  // operand split once for two products); a null twin makes this contraction split its operand itself.
  void gemm(bool use_tc, const float* A, long long lda, long long a_rows, int a_batch_rows, const float* Wm, long long ldw,
            long long w_rows, int w_batch_rows, int nbatch, int M, int N, int K, const float* bias,
            const float* residual, long long ld_res, float scale, int round, float* out, long long ldo,
            double* qstats = nullptr, int rows_per_img = 1 << 30, const float* a_lo = nullptr, const float* w_lo = nullptr) {
    Epilogue ep; memset(&ep, 0, sizeof(ep));
    ep.bias = bias; ep.residual = residual; ep.ld_res = ld_res; ep.scale = scale; ep.round_tf32 = round;
    ep.rows_per_img = rows_per_img; ep.out = out; ep.ld_out = ldo;
    if (use_tc) {
      TcGemmDesc d = tc_desc(e, A, K, nullptr, 0, 0, 0, 0, 1, Wm, N);
      d.conv = 0; d.a_rows = a_rows; d.a_ld = lda; d.a_batch_rows = a_batch_rows;
      d.w_rows = w_rows; d.w_ld = ldw; d.w_batch_rows = w_batch_rows; d.nbatch = nbatch; d.M_per_batch = M; d.qstats = qstats; d.epi = ep;
      if (split) {   // the rows the contraction reads: (rows - 1) pitches + K elements from the base
        Pair pa, pw;
        if (!a_lo) { pa = split_pair(A, (a_rows - 1) * lda + K, "gemm A"); d.a1 = pa.hi; a_lo = pa.lo; }
        if (!w_lo) { pw = split_pair(Wm, (w_rows - 1) * ldw + K, "gemm W"); d.w = pw.hi; w_lo = pw.lo; }
        if (rc) return;
        d.split = 1; d.a1_lo = a_lo; d.w_lo = w_lo;
        release(pa); release(pw);
      }
      if (dry) return;
      TcGemmPlan* pl = nullptr;
      if (int r = tc_gemm_plan_create(d, &pl)) { rc = r; return; }
      e->tcplans.push_back(pl);
      name("gemm %dx(%dx%dx%d)%s [%s]", nbatch, M, N, K, residual ? " +res" : "", tc_gemm_form(pl));
      {
        const double es = om == 2 ? 2.0 : split ? 8.0 : 4.0;
        next_bytes = (double)(a_batch_rows ? nbatch : 1) * M * K * es + (double)(w_batch_rows ? nbatch : 1) * N * K * es +
                     (double)nbatch * M * N * (round == 2 ? 2.0 : 4.0) + (residual ? (double)nbatch * M * N * 4.0 : 0.0);
      }
      op(1, [=](cudaStream_t st) { return tc_gemm_launch(pl, st); }, 0, 2.0 * nbatch * (double)M * N * K);
    } else {
      SimtConv s = simt_desc(A, K, M, 1, 1, 1, M, 1, Wm, N);
      s.ld1 = lda; s.nbatch = nbatch; s.a_batched = a_batch_rows != 0;
      s.w_batch_stride = (long long)w_batch_rows * ldw; s.w_ld = ldw;
      ep.rows_per_img = M; s.epi = ep;
      op(1, [=](cudaStream_t st) { return launch_conv_simt(s, st); }, 1, 2.0 * nbatch * (double)M * N * K);
    }
  }

  void tap(int idx, const Tensor& t) { if (!dry) e->taps[idx] = t; }

  // would conv() run this stride-1 convolution on the few-channel kernel (conv_lowc.cu: TF32 mode, fp32 tensors)?
  bool lowc_ok(int C1, int C2, int Cout, int H, int taps) const {
    if (e->cfg.precision != 0 || e->sumC % 2 != 0) return false;
    SimtConv s = simt_desc(nullptr, C1, H, H, taps, 1, H, H, nullptr, Cout);
    s.C2 = C2;
    return conv_lowc_supported(s);
  }

  Tensor resblock(const Mod& m, Tensor& x1, Tensor& x2) {
    Tensor none;
    const int Cin = x1.C + x2.C, H = x1.H, Ho = m.up ? 2 * H : m.down ? H / 2 : H;
    const bool resample = m.up || m.down;
    const float inv_s2 = e->cfg.skip_rescale ? 1.0f / (float)std::sqrt(2.0) : 1.0f;
    const bool h1_f16 = om == 2 && m.tc0 && m.tc1 && fused_stats && (Ho * Ho) % 32 == 0 && (m.cout % 128 == 0);
    // few-channel levels (TF32 mode): both 3x3 convolutions normalise their input while they stage it, so neither
    // GroupNorm writes a tensor (quad-aligned groups only: the coefficient kernel works on channel quads)
    const int G0 = groups(Cin), G1 = groups(m.cout);
    const bool lc0 = lowc_gn && !m.tc0 && !resample && !x1.f16 && !x2.f16 && Cin % G0 == 0 && (Cin / G0) % 4 == 0 && x1.C % 4 == 0 &&
                     lowc_ok(x1.C, x2.C, m.cout, H, 9);
    const bool lc1 = lowc_gn && !m.tc1 && m.cout % G1 == 0 && (m.cout / G1) % 4 == 0 && lowc_ok(m.cout, 0, m.cout, Ho, 9);
    Tensor a0, raw;   // raw: operand-format copy of the (concatenated) block input for the tensor-core skip conv
    if (!lc0) {
      a0 = talloc(Cin, H, H);
      if (m.has_conv2 && m.tc2 && !resample) raw = talloc(Cin, H, H);
      gn(x1, x2, m.gn0w, m.gn0b, 1, (m.tc0 && !resample) ? om : 0, a0, raw.p, raw.d);
    }
    Tensor xr;
    if (resample) {
      if (x2.p) { set_error("ncsnpp: resampling block with a two-source input"); rc = 2; return Tensor(); }
      Tensor a0r = talloc(Cin, Ho, Ho);
      xr = talloc(Cin, Ho, Ho);
      xr.f16 = m.tc2 && om == 2;
      twin([&](bool d) {
        resample2x(d ? a0.d : a0.p, H, Cin, m.up != 0, m.tc0 ? om : 0, d ? a0r.d : a0r.p);
        resample2x(d ? x1.d : x1.p, H, Cin, m.up != 0, m.tc2 ? om : 0, d ? xr.d : xr.p);
      });
      tfree(a0); a0 = a0r;
    }
    Tensor h1 = talloc(m.cout, Ho, Ho);
    // fp16 operand mode: the mid-block tensor (Conv_0 output, only ever read by GroupNorm_1) is stored as fp16;
    // its GroupNorm sums are accumulated from the fp32 accumulators in the epilogue.
    h1.f16 = h1_f16;
    if (lc0) {
      Coef c0 = gncoef(x1, x2, m.gn0w, m.gn0b);
      conv(false, x1, x2, m.c0w, m.c0b, h1, Conv().temb(m.dense_row).stats().gn(c0));
      ffree(c0.scale, c0.bytes);
    } else {
      conv(m.tc0, a0, none, m.c0w, m.c0b, h1, Conv().temb(m.dense_row).round(h1_f16 ? 2 : 0).stats());
      tfree(a0);
    }
    if (h1_f16 && !h1.qs) { set_error("ncsnpp: fp16 mid-block tensor without fused GroupNorm sums"); rc = 2; return Tensor(); }
    Tensor a1; Coef c1;
    if (lc1) {
      c1 = gncoef(h1, none, m.gn1w, m.gn1b);
    } else {
      a1 = talloc(m.cout, Ho, Ho);
      gn(h1, none, m.gn1w, m.gn1b, 1, m.tc1 ? om : 0, a1, nullptr);
      tfree(h1);
    }
    Tensor s;
    Tensor residual = x1;
    // Fused skip projection (default): Conv_2(x) (layerspp.py:270) is accumulated inside the second 3x3 convolution
    // as extra K steps instead of a separate launch + a residual round trip through HBM.  (Tangent plans: its bias rides
    // in the row-vector slot, so the skip projection stays a contraction of its own there.)
    if (m.has_conv2 && m.tc1 && m.tc2 && (resample || raw.p) && !tan) {
      Tensor out = talloc(m.cout, Ho, Ho);
      Tensor e1 = resample ? xr : raw;
      e1.f16 = false;   // conv() addresses operands by the engine-wide operand mode
      conv(true, a1, none, m.c1w, m.c1b, out, Conv().scale(inv_s2).stats().skip(e1, none, m.c2w, m.c2b));
      tfree(a1); tfree(raw); tfree(xr);
      return out;
    }
    if (m.has_conv2) {
      s = talloc(m.cout, Ho, Ho);
      if (resample) conv(m.tc2, xr, none, m.c2w, m.c2b, s, Conv().taps(1));
      else if (m.tc2 && raw.p) conv(true, raw, none, m.c2w, m.c2b, s, Conv().taps(1));
      else conv(m.tc2, x1, x2, m.c2w, m.c2b, s, Conv().taps(1));
      residual = s;
      tfree(raw); tfree(xr);
    } else if (x2.p) { set_error("ncsnpp: concat input without a skip convolution"); rc = 2; return Tensor(); }
    Tensor out = talloc(m.cout, Ho, Ho);
    if (lc1) {
      conv(false, h1, none, m.c1w, m.c1b, out, Conv().residual(residual).scale(inv_s2).stats().gn(c1));
      ffree(c1.scale, c1.bytes); tfree(h1);
    } else {
      conv(m.tc1, a1, none, m.c1w, m.c1b, out, Conv().residual(residual).scale(inv_s2).stats());
      tfree(a1);
    }
    tfree(s);
    return out;
  }

  Tensor attn(const Mod& m, Tensor& x) {
    Tensor none;
    const int C = x.C, T = x.H * x.W;
    const float inv_s2 = e->cfg.skip_rescale ? 1.0f / (float)std::sqrt(2.0) : 1.0f;
    const bool tc = m.tcattn;
    const bool small = !m.tcattn && m.tc0 && T <= 64;   // few tokens: projections on tensor cores, core in one CTA per image
    const float* Wqkv = e->W(m.nw[0]);          // [3C][C] (fp32 slots; fp16 elements when om == 2)
    // Wv = rows 2C.. of the packed block: the offset counts ELEMENTS of the operand format
    const float* wv = om == 2 && m.tc0 ? reinterpret_cast<const float*>(reinterpret_cast<const uint16_t*>(Wqkv) + 2LL * C * C)
                                        : Wqkv + 2LL * C * C;
    const float* bqkv = e->W(m.nb[0]);          // [3C]
    const float sc = 1.0f / std::sqrt((float)C);   // int(C) ** -0.5
    const long long BT = (long long)B * T;
    const int Bc = B;
    Tensor a = talloc(C, x.H, x.W);
    gn(x, none, m.gn0w, m.gn0b, 0, (tc || small) ? om : 0, a, nullptr);
    long long ob; float* O = nullptr;
    float* dO = nullptr;   // tangent of O (tangent plans)
    if (small) {
      long long qb; float* qkv = falloc(BT * 3 * C, &qb);
      // q | k | v = a [Wq; Wk; Wv]^T + [bq; bk; bv]   (layerspp.py:78-80) as one N=3C contraction
      gemm(true, a.p, C, BT, 0, Wqkv, C, 3LL * C, 0, 1, (int)BT, 3 * C, C, bqkv, nullptr, 0, 1.f, 0, qkv, 3 * C);
      tfree(a);
      O = falloc(BT * C, &ob);
      const int rnd = m.tc2 ? om : 0;
      if (!dry) { if (int r = launch_attn_small_configure(T, C)) { rc = r; } }
      name("attn_small T=%d C=%d", T, C);
      op(1, [=](cudaStream_t st) { return launch_attn_small(qkv, O, Bc, T, C, sc, rnd, st); }, 4);
      ffree(qkv, qb);
    } else {
      long long qkb, vtb, sb;
      float *dqk = nullptr, *dvT = nullptr, *dS = nullptr;   // tangents (tangent plans)
      float* qk = falloc2((long long)B * T * 2 * C, &qkb, &dqk);
      float* vT = falloc2((long long)B * C * T, &vtb, &dvT);
      twin([&](bool d) {   // tangent: dq, dk, dv, the projections of da without bias
        // q,k = a Wq^T + bq | a Wk^T + bk   (layerspp.py:78-79) in one N=2C contraction
        gemm(tc, d ? a.d : a.p, C, BT, 0 /* rows enumerated flat */, Wqkv, C, 2LL * C, 0, 1, (int)BT, 2 * C, C, d ? nullptr : bqkv,
             nullptr, 0, 1.f, tc ? om : 0, d ? dqk : qk, 2 * C, nullptr, 1 << 30, nullptr, e->Wlo(m.nw[0]));
        // v^T[b][c][t] = sum_i Wv[c][i] a[b][t][i]   (bias bv is added after the PV product: softmax rows sum to 1)
        gemm(tc, wv, C, C, 0, d ? a.d : a.p, C, BT, T, B, C, T, C, nullptr, nullptr, 0, 1.f, tc ? om : 0, d ? dvT : vT, T, nullptr, 1 << 30,
             e->Wlo(m.nw[0]) ? e->Wlo(m.nw[0]) + 2LL * C * C : nullptr);
      });
      tfree(a);
      // Fused core (default): logits, softmax, P.V, NIN_3, residual, rescale and quad sums in one kernel; the
      // [T,T] logits/probabilities and the attention output stay on chip.  Other shapes: the flash core in fp16 operand mode
      // (logits on chip, O through HBM into NIN_3), separate launches otherwise.
      if (om == 2 && !(tc && m.tc2 && (tc_attn_supported(T, C, true) || attn_flash_supported(T, C)))) {
        set_error("ncsnpp: fp16 operand mode needs the fused attention core (T=%d C=%d)", T, C); rc = 2; return Tensor();
      }
      if (tc && m.tc2 && tc_attn_supported(T, C, om == 2) && !tan && !split) {
        Tensor out = talloc(C, x.H, x.W);
        if (fused_stats) out.qs = qalloc(C);
        if (!dry) {
          TcAttnDesc d; memset(&d, 0, sizeof(d));
          d.qk = qk; d.vT = vT; d.w3 = e->W(m.nw[3]); d.bv = bqkv + 2 * C; d.b3 = e->W(m.nb[3]); d.x = x.p; d.out = out.p;
          d.qstats = out.qs; d.nimg = B; d.T = T; d.C = C; d.out_scale = inv_s2; d.f16 = om == 2;
          TcAttnPlan* pl = nullptr;
          if (int r = tc_attn_plan_create(d, &pl)) { rc = r; return Tensor(); }
          e->attnplans.push_back(pl);
          name("attention core T=%d C=%d (QK^T, softmax, PV, NIN_3 +res) [fused]", T, C);
          next_bytes = (double)B * T * C * ((om == 2 ? 2.0 : 4.0) * 3 + 8.0) + (double)C * C * (om == 2 ? 2.0 : 4.0);
          op(1, [=](cudaStream_t st) { return tc_attn_launch(pl, st); }, 0, 2.0 * B * T * ((double)T * C * 2 + (double)C * C));
        }
        ffree(qk, qkb); ffree(vT, vtb);
        return out;
      }
      if (om == 2) {   // flash core: logits, online softmax and P.V on chip; O (fp16) feeds NIN_3 below
        O = falloc(BT * C, &ob);
        if (!dry) {
          AttnFlashPlan pl;
          if (int r = attn_flash_plan(qk, vT, bqkv + 2 * C, O, B, T, C, &pl)) { rc = r; return Tensor(); }
          name("attention flash T=%d C=%d (QK^T, online softmax, PV) [fused f16]", T, C);
          next_bytes = (double)B * T * C * 2.0 * 4;   // q, k, v^T in, O out
          op(1, [=](cudaStream_t st) { return attn_flash_launch(pl, st); }, 0, 4.0 * B * (double)T * T * C);
        }
        ffree(qk, qkb); ffree(vT, vtb);
      } else {
        float* S = falloc2(BT * T, &sb, &dS);
        // logits[b][q][k] = q . k   (layerspp.py:82), scaled inside the softmax (split TF32: q | k split once for both operands)
        Pair qkp;
        if (tc && split) qkp = split_pair(qk, (long long)B * T * 2 * C, "q|k");
        const float* qkh = qkp.hi ? qkp.hi : qk;
        gemm(tc, qkh, 2 * C, BT, T, qkh + C, 2 * C, BT, T, B, T, T, C, nullptr, nullptr, 0, 1.f, 0, S, T, nullptr, 1 << 30,
             qkp.lo, qkp.lo ? qkp.lo + C : nullptr);
        release(qkp);
        if (tan) {   // dS = dq k^T + q dk^T
          long long tb; float* t1 = falloc(BT * T, &tb);
          tangent([&] {
            gemm(tc, dqk, 2 * C, BT, T, qk + C, 2 * C, BT, T, B, T, T, C, nullptr, nullptr, 0, 1.f, 0, t1, T, nullptr, 1 << 30);
            gemm(tc, qk, 2 * C, BT, T, dqk + C, 2 * C, BT, T, B, T, T, C, nullptr, t1, T, 1.f, 0, dS, T, nullptr, 1 << 30);
          });
          ffree(t1, tb);
        }
        ffree(qk, qkb);
        name("softmax T=%d", T);
        const int prnd = tc ? om : 0;   // probabilities in the operand format of the P.V contraction (fp32 when split TF32)
        op(1, [=](cudaStream_t st) { return launch_softmax_rows(S, S, (long long)Bc * T, T, sc, prnd, st); }, 4);
        if (tan) {   // dP = P (sc dS - rowsum(P sc dS)), over dS
          name("softmax_tangent T=%d", T);
          tangent([&] { op(1, [=](cudaStream_t st) { return launch_softmax_tangent(S, dS, (long long)Bc * T, T, sc, prnd, st); }, 4); });
        }
        O = falloc2(BT * C, &ob, &dO);
        // h[b][q][c] = sum_k P[q][k] v[k][c] + bv[c]   (layerspp.py:86)
        gemm(tc, S, T, BT, T, vT, T, (long long)B * C, C, B, T, C, T, bqkv + 2 * C, nullptr, 0, 1.f, m.tc2 ? om : 0, O, C);
        if (tan) {   // dO = dP v + P dv
          long long tb; float* t2 = falloc(BT * C, &tb);
          tangent([&] {
            gemm(tc, dS, T, BT, T, vT, T, (long long)B * C, C, B, T, C, T, nullptr, nullptr, 0, 1.f, 0, t2, C);
            gemm(tc, S, T, BT, T, dvT, T, (long long)B * C, C, B, T, C, T, nullptr, t2, C, 1.f, m.tc2 ? om : 0, dO, C);
          });
          ffree(t2, tb);
        }
        ffree(S, sb); ffree(vT, vtb);
      }
    }
    Tensor out = talloc(C, x.H, x.W);
    Tensor Ot; Ot.p = O; Ot.C = C; Ot.H = x.H; Ot.W = x.W; Ot.d = dO;
    conv(m.tc2, Ot, none, m.nw[3], m.nb[3], out, Conv().taps(1).residual(x).scale(inv_s2).stats());   // NIN_3 + (x+h)/sqrt2 (:87-91)
    ffree(O, ob);
    return out;
  }

  // DDPM Downsample(with_conv) (layers.py:599-616): F.pad(x, (0,1,0,1)) then a 3x3 stride-2 VALID convolution.  The
  // convolution reads the unpadded input: the taps of the last output row / column that fall on row / column H are the
  // padding zeros (TMA's out-of-bounds fill on the tensor cores, the bounds check of the CUDA-core kernel otherwise).
  Tensor downsample(const Mod& m, Tensor& x) {
    const int H = x.H, Ho = H / 2;
    Tensor out = talloc(m.cout, Ho, Ho);
    if (m.tc0 && split) {
      conv(true, x, Tensor(), m.w, m.b, out, Conv().stats().stride(2, H));   // the contraction's split pass reads the fp32 block output
    } else if (m.tc0) {
      // the block output is fp32; the tensor cores read it in the operand format (TF32 grid / fp16)
      Tensor xo = talloc(x.C, H, H);
      const long long n = (long long)B * H * H * x.C; const int omc = om;
      twin([&](bool d) {
        const float* src = d ? x.d : x.p; float* dst = d ? xo.d : xo.p;
        name("operand copy %d @%d", x.C, H);
        next_bytes = (double)n * (4.0 + (om == 2 ? 2.0 : 4.0));
        op(1, [=](cudaStream_t st) { return launch_store_operand(src, dst, n, omc, st); }, 6);
      });
      conv(true, xo, Tensor(), m.w, m.b, out, Conv().stats().stride(2, H));
      tfree(xo);
    } else {
      twin([&](bool d) {
        SimtConv s = simt_desc(d ? x.d : x.p, x.C, H, H, 9, 2, Ho, Ho, e->W(m.w), m.cout);
        s.epi.bias = d ? nullptr : e->W(m.b); s.epi.out = d ? out.d : out.p;
        name("conv3x3 s2 %d->%d @%d [cuda-core]", x.C, m.cout, Ho);
        op(1, [=](cudaStream_t st) { return launch_conv_simt(s, st); }, 1, 2.0 * B * Ho * Ho * (double)m.cout * x.C * 9);
      });
    }
    return out;
  }

  // DDPM Upsample(with_conv) (layers.py:584-596): nearest 2x (the 2x2 box upfirdn2d, written in the convolution's operand
  // format) then a 3x3 'same' convolution
  Tensor upsample(const Mod& m, Tensor& x) {
    const int H = x.H, Ho = 2 * H;
    Tensor u = talloc(x.C, Ho, Ho);
    twin([&](bool d) { fir(d ? x.d : x.p, B, H, H, x.C, 2, 1, 1, 0, m.tc0 ? om : 0, d ? u.d : u.p, 1.f, /*box=*/true); });
    Tensor out = talloc(m.cout, Ho, Ho);
    conv(m.tc0, u, Tensor(), m.w, m.b, out, Conv().stats());
    tfree(u);
    return out;
  }

  // ---- time embedding (ncsnpp.py:236-255) + all Dense_0(act(temb)) rows (layerspp.py:263) ----
  void time_embedding() {
    const b200_ncsnpp_config& c = e->cfg;
    const int nf = c.nf, sumC = e->sumC, Bc = B, ln = lane;
    b200_ncsnpp* eng = e;
    long long eb, t1b, t2b, db;
    const int positional = c.embedding_type == 1 ? 1 : 0, emb_dim = positional ? nf : 2 * nf;
    float* emb = falloc((long long)B * 2 * nf, &eb);
    float* t1 = falloc((long long)B * 4 * nf, &t1b);
    float* t2 = falloc((long long)B * 4 * nf, &t2b);
    float* dense_all = falloc((long long)B * sumC, &db);
    dense_all_ = dense_all;
    const Mod &mf = e->mods[0], &l1 = e->mods[1], &l2 = e->mods[2];
    const float *Wf = e->W(mf.w), *W1 = e->W(l1.w), *b1 = e->W(l1.b), *W2 = e->W(l2.w), *b2 = e->W(l2.b);
    const float *Wd = e->wblob + e->dense_w_off, *bd = e->wblob + e->dense_b_off;
    op(4, [=](cudaStream_t st) {
      const int rows = eng->uniform ? 1 : Bc;
      if (int r = launch_fourier_embed(eng->in_labels_l[ln], 1, Wf, positional ? nf / 2 : nf, rows, emb, st, positional)) return r;
      if (int r = launch_linear_rows(emb, emb_dim, W1, b1, rows, 4 * nf, emb_dim, 0, t1, 4 * nf, st)) return r;
      if (int r = launch_linear_rows(t1, 4 * nf, W2, b2, rows, 4 * nf, 4 * nf, 1, t2, 4 * nf, st)) return r;
      return launch_linear_rows(t2, 4 * nf, Wd, bd, rows, sumC, 4 * nf, 1, dense_all, sumC, st);
    }, 5);
  }

  // ---- input (ncsnpp.py:259-268): 2x-1 when the data is not centred (its tangent: v, or 2v), NCHW; then the input conv.
  // The input also is the bottom of the input pyramid. ----
  Tensor input_conv() {
    const b200_ncsnpp_config& c = e->cfg;
    const int nf = c.nf, R = c.image_size, ch = c.num_channels, ln = lane, centered = c.centered;
    b200_ncsnpp* eng = e;
    const Mod& m = next();
    long long xcb; float* dxc = nullptr;
    float* xc = falloc2((long long)B * ch * R * R, &xcb, &dxc);
    const long long n = (long long)B * ch * R * R;
    twin([&](bool d) {
      float* dst = d ? dxc : xc;
      const float shift = d ? 0.0f : -0.5f;
      op(1, [=](cudaStream_t st) {
        const float* src = d ? eng->in_v : eng->in_x_l[ln];
        if (centered) return cudaMemcpyAsync(dst, src, n * 4, cudaMemcpyDeviceToDevice, st) == cudaSuccess ? 0 : (set_error("memcpy failed"), 1);
        launch_kernel(affine_kernel, dim3((int)std::min<long long>((n + 255) / 256, 4096)), dim3(256), 0, st, src, dst, n, shift, 2.0f);
        return cudaGetLastError() == cudaSuccess ? 0 : (set_error("affine launch failed"), 1);
      });
    });
    pyr.p = xc; pyr.C = ch; pyr.H = R; pyr.W = R;
    Tensor h0 = talloc(nf, R, R);
    if (m.tc0 || m.tc1) {
      // im2col patches [B*R*R][32] (TF32 grid) then one K=32 contraction with the flat-packed weights (tensor cores, or the
      // few-channel kernel for nf <= 64)
      float* dpatches = nullptr;
      long long pb; float* patches = falloc2((long long)B * R * R * 32, &pb, &dpatches);   // 128 B per pixel: 32 fp32 or 64 fp16
      const int Bc = B, omc = om;
      twin([&](bool d) {
        const float* src = d ? dxc : xc; float* dst = d ? dpatches : patches;
        name("im2col 3x3 %d @%d", ch, R);
        op(1, [=](cudaStream_t st) { return launch_im2col3x3_nchw(src, dst, Bc, ch, R, R, R, R, 1, 1, omc, st); }, 6);
      });
      Tensor pt; pt.p = patches; pt.C = om == 2 ? 64 : 32; pt.H = R; pt.W = R;   // patches as a one-K-step NHWC image: a 1x1 conv
      pt.d = dpatches;
      conv(m.tc0, pt, Tensor(), m.w, m.b, h0, Conv().taps(1).stats());
      ffree(patches, pb);
    } else {
      twin([&](bool d) {
        SimtConv s = simt_desc(d ? dxc : xc, ch, R, R, 9, 1, R, R, e->W(m.w), nf);
        s.in_nchw = 1; s.epi.bias = d ? nullptr : e->W(m.b); s.epi.out = d ? h0.d : h0.p;
        op(1, [=](cudaStream_t st) { return launch_conv_simt(s, st); }, 1, 2.0 * B * R * R * (double)nf * ch * 9);
      });
    }
    tap(m.index, h0);
    return h0;
  }

  // ---- one level of the input pyramid (ncsnpp.py:289-301), after the level's downsampling block h ----
  Tensor input_pyramid(Tensor h) {
    const b200_ncsnpp_config& c = e->cfg;
    const int ch = c.num_channels;
    const Mod& m = next();
    if (m.kind == M_COMBINE) {
      // input_skip (ncsnpp.py:289-292): the image pyramid is downsampled (no parameters) and a 1x1 convolution of it is
      // added to h: Combine(method='sum') (layerspp.py:44-59)
      const int Hin = pyr.H, Hn = Hin / 2;
      long long nb; float* npyr = falloc((long long)B * ch * Hn * Hn, &nb);
      resample2x_planes(pyr.p, B * ch, Hin, false, npyr);
      if (pyr_owned) ffree(pyr.p, pyr_bytes);
      pyr.p = npyr; pyr.H = pyr.W = Hn; pyr_owned = true; pyr_bytes = nb;
      if (Hn != h.H) { set_error("ncsnpp: input pyramid geometry mismatch (%d vs %d)", Hn, h.H); rc = 2; return Tensor(); }
      Tensor out = talloc(m.cout, h.H, h.W);
      SimtConv s = simt_desc(npyr, ch, Hn, Hn, 1, 1, Hn, Hn, e->W(m.w), m.cout);
      s.in_nchw = 1; s.epi.bias = e->W(m.b); s.epi.residual = h.p; s.epi.out = out.p;
      name("combine sum: conv1x1 %d->%d @%d +h [cuda-core]", ch, m.cout, Hn);
      op(1, [=](cudaStream_t st) { return launch_conv_simt(s, st); }, 1, 2.0 * B * Hn * Hn * (double)m.cout * ch);
      advance(h, m, out);
      return h;
    }
    // residual (M_PYR_DOWN): Downsample(fir, with_conv): FIR with pad (2,2) then 3x3 stride-2 VALID conv + bias
    // (up_or_down_sampling.py:170-178, Conv2d.forward :44-56), then (pyr + h)/sqrt2 (ncsnpp.py:297-301)
    const int Hin = pyr.H, p = (e->firn - 2) + 2;
    const int Hp = Hin + ((p + 1) / 2) + (p / 2) - e->firn + 1;
    long long fb; float* fbuf = falloc((long long)B * pyr.C * Hp * Hp, &fb);
    const bool tcp = m.tc0 && !pyr_nchw;
    const bool flat = m.tc2 && pyr_nchw;
    if (pyr_nchw) fir(pyr.p, B * pyr.C, Hin, Hin, 1, 1, 1, (p + 1) / 2, p / 2, 0, fbuf, 1.f);
    else fir(pyr.p, B, Hin, Hin, pyr.C, 1, 1, (p + 1) / 2, p / 2, tcp ? om : 0, fbuf, 1.f);
    Tensor np = talloc(m.cout, h.H, h.W);
    if ((Hp - 3) / 2 + 1 != h.H) { set_error("ncsnpp: pyramid geometry mismatch (%d vs %d)", (Hp - 3) / 2 + 1, h.H); rc = 2; return Tensor(); }
    const float ps = c.skip_rescale ? 1.0f / (float)std::sqrt(2.0) : 1.0f;
    if (flat) {
      long long pb2; float* patches = falloc((long long)B * h.H * h.W * 32, &pb2);
      const int Bc = B, pc = pyr.C, oh = h.H, ow = h.W, omc = om;
      name("im2col 3x3 s2 %d @%d", pc, oh);
      op(1, [=](cudaStream_t st) { return launch_im2col3x3_nchw(fbuf, patches, Bc, pc, Hp, Hp, oh, ow, 2, 0, omc, st); }, 6);
      Tensor pt; pt.p = patches; pt.C = om == 2 ? 64 : 32; pt.H = h.H; pt.W = h.W;
      conv(true, pt, Tensor(), m.w, m.b, np, Conv().taps(1).residual(h).scale(ps).stats());
      ffree(patches, pb2);
    } else if (tcp) {
      Tensor fin; fin.p = fbuf; fin.C = pyr.C; fin.H = Hp; fin.W = Hp;
      conv(true, fin, Tensor(), m.w, m.b, np, Conv().residual(h).scale(ps).stats().stride(2, Hp));
    } else {
      SimtConv s = simt_desc(fbuf, pyr.C, Hp, Hp, 9, 2, h.H, h.W, e->W(m.w), m.cout);
      s.in_nchw = pyr_nchw ? 1 : 0; s.epi.bias = e->W(m.b); s.epi.residual = h.p; s.epi.scale = ps; s.epi.out = np.p;
      op(1, [=](cudaStream_t st) { return launch_conv_simt(s, st); }, 1, 2.0 * B * h.H * h.W * (double)m.cout * pyr.C * 9);
    }
    ffree(fbuf, fb);
    if (pyr_owned) tfree(pyr);
    tfree(h);
    pyr = np; pyr_nchw = false; pyr_owned = false;   // h aliases the pyramid from here on (it lives in hs)
    // (no debug tap: the reference module's own output is the pre-combine conv result, which is never materialised)
    return np;
  }

  // ---- middle (ncsnpp.py:305-311): resblock, attention, resblock ----
  Tensor middle(Tensor& x) {
    Tensor none;
    const Mod& m0 = next(); Tensor h = resblock(m0, x, none); if (rc) return h;
    tap(m0.index, h);
    const Mod& ma = next(); Tensor h2 = attn(ma, h); if (rc) return h2;
    advance(h, ma, h2);
    const Mod& m1 = next(); Tensor h3 = resblock(m1, h, none); if (rc) return h3;
    advance(h, m1, h3);
    return h;
  }

  // ---- one output_skip level (ncsnpp.py:325-341): pyramid = upsample(pyramid) + conv3x3(SiLU(GroupNorm(h))) in image
  // channels; the level-0 sum is the network output (divided by sigma when scale_by_sigma, :377-379) ----
  void output_skip(Tensor& h, bool last) {
    const b200_ncsnpp_config& c = e->cfg;
    const int ch = c.num_channels, Hl = h.H, ln = lane;
    b200_ncsnpp* eng = e;
    const Mod& mg = next(); const Mod& mo = next();
    Tensor a = talloc(h.C, Hl, Hl);
    const int hf16 = (om == 2 && h.C % 64 == 0) ? 1 : 0;
    Tensor none; gn(h, none, mg.w, mg.b, 1, hf16 ? 2 : 0, a, nullptr);
    long long ub = 0; float* up = nullptr;
    if (opyr) {
      up = falloc((long long)B * ch * Hl * Hl, &ub);
      resample2x_planes(opyr, B * ch, Hl / 2, true, up);
      ffree(opyr, opyr_bytes); opyr = nullptr;
    }
    long long nb = 0; float* dst = nullptr;
    if (!last) dst = falloc((long long)B * ch * Hl * Hl, &nb);
    const float *wo = e->W(mo.w), *bo = e->W(mo.b);
    const Tensor ain = a; const int Bc2 = B, sbs = c.scale_by_sigma;
    if (ch > 4) { set_error("ncsnpp: output_skip needs <= 4 image channels"); rc = 2; return; }
    name("conv3x3 %d->%d @%d nchw-out +pyramid [small-n]", a.C, ch, Hl);
    op(1, [=](cudaStream_t st) {
      return launch_conv3x3_small_n(ain.p, wo, bo, (last && sbs) ? eng->in_labels_l[ln] : nullptr, eng->uniform ? 0 : 1,
                                    last ? eng->out_l[ln] : dst, Bc2, Hl, Hl, ain.C, ch, hf16, st, up);
    }, 1, 2.0 * B * Hl * Hl * (double)ch * a.C * 9);
    tfree(a);
    if (up) ffree(up, ub);
    opyr = dst; opyr_bytes = nb;
  }

  // ---- output head (ncsnpp.py:371-379): GroupNorm, SiLU, 3x3 conv to the image channels, stored NCHW, / sigma.  Its
  // tangent writes J v into tout. ----
  void head(Tensor& h) {
    const b200_ncsnpp_config& c = e->cfg;
    const int R = c.image_size, ch = c.num_channels, ln = lane, Bc = B, sbs = c.scale_by_sigma;
    b200_ncsnpp* eng = e;
    const Mod& mg = next(); const Mod& mo = next();
    Tensor a = talloc(h.C, h.H, h.W);
    // fp16 operand mode: the head's input is stored as fp16 too (the CUDA-core head is bound by its nine-fold
    // tap re-reads through L1/L2, so half the bytes is half the time); same 11-bit rounding as every other conv input
    const int head_f16 = (!mo.tc0 && om == 2 && ch <= 4 && h.C % 64 == 0) ? 1 : 0;
    Tensor none; gn(h, none, mg.w, mg.b, 1, mo.tc0 ? om : head_f16 ? 2 : 0, a, nullptr);
    tfree(h);
    const float *wo = e->W(mo.w), *bo = e->W(mo.b);
    const double flops = 2.0 * B * R * R * (double)ch * a.C * 9;
    twin([&](bool d) {
      const float* x = d ? a.d : a.p;
      const float* bias = d ? nullptr : bo;
      if (mo.tc0) {
        if (dry) return;
        TcGemmDesc desc = tc_desc(e, x, a.C, nullptr, 0, R, R, B, 9, wo, 128);
        desc.stride = 1;
        desc.epi.bias = bias; desc.epi.scale = 1.f; desc.epi.rows_per_img = R * R; desc.epi.out_nchw = 1; desc.epi.n_valid = ch;
        desc.epi.out = reinterpret_cast<float*>(uintptr_t(16));   // patched per call (tc_gemm_set_head)
        TcGemmPlan* pl = nullptr;
        if (int r = tc_gemm_plan_create(desc, &pl)) { rc = r; return; }
        e->tcplans.push_back(pl);
        name("conv3x3 %d->%d(pad 128) @%d nchw-out /sigma [%s]", a.C, ch, R, tc_gemm_form(pl));
        next_bytes = (double)B * R * R * (a.C * (om == 2 ? 2.0 : 4.0) + ch * 4.0);
        op(1, [=](cudaStream_t st) {
          tc_gemm_set_head(pl, d ? eng->tout : eng->out_l[ln], sbs ? eng->in_labels_l[ln] : nullptr, eng->uniform ? 0 : 1);
          return tc_gemm_launch(pl, st);
        }, 0, flops);
      } else if (ch <= 4) {
        const int C = a.C;
        name("conv3x3 %d->%d @%d nchw-out [small-n]", C, ch, R);
        op(1, [=](cudaStream_t st) {
          return launch_conv3x3_small_n(x, wo, bias, sbs ? eng->in_labels_l[ln] : nullptr, eng->uniform ? 0 : 1,
                                        d ? eng->tout : eng->out_l[ln], Bc, R, R, C, ch, head_f16, st);
        }, 1, flops);
      } else {
        SimtConv s = simt_desc(x, a.C, R, R, 9, 1, R, R, wo, ch);
        s.epi.bias = bias; s.epi.out_nchw = 1;
        op(1, [=](cudaStream_t st) {
          SimtConv cc = s;
          cc.epi.out = d ? eng->tout : eng->out_l[ln];
          if (sbs) { cc.epi.per_img_div = eng->in_labels_l[ln]; cc.epi.div_stride = eng->uniform ? 0 : 1; }
          return launch_conv_simt(cc, st);
        }, 1, flops);
      }
    });
    tfree(a);
  }

  // ===== NCSNv2 (family 2) =====
  // would the contraction with packed weight pi run on the tensor cores (its weights are packed in the operand format)?
  bool on_tc(int pi) const { return pi >= 0 && e->params[pi].round != 0; }
  int mode_for(int pi) const { return on_tc(pi) ? om : 0; }
  // InstanceNorm2dPlus (normalization.py:157-183) of x with parameters p = {alpha, gamma, beta}, then ELU, into y in
  // store mode `mode`: one fp64 statistics pass and one apply pass
  void in_elu(const Tensor& x, const int (&p)[3], int mode, const Tensor& y) {
    long long sb; double* stats = reinterpret_cast<double*>(falloc(2 * in_stats_doubles(B, x.H * x.W, x.C), &sb));   // (floats)
    const Tensor xx = x; const int Bc = B, HW = x.H * x.W;
    const float *al = e->W(p[0]), *ga = e->W(p[1]), *be = e->W(p[2]);
    name("in++ stats %d @%d", x.C, x.H);
    next_bytes = (double)B * HW * x.C * 4.0;
    const int nl = in_stats_doubles(B, HW, x.C) > 2LL * B * x.C ? 2 : 1;   // pixel slices + their reduction
    op(nl, [=](cudaStream_t st) { return launch_in_stats(xx.p, Bc, HW, xx.C, stats, st); }, 2);
    name("in++ apply elu %d @%d%s", x.C, x.H, mode == 2 ? " f16-out" : "");
    next_bytes = (double)B * HW * x.C * (4.0 + (mode == 2 ? 2.0 : 4.0));
    op(1, [=](cudaStream_t st) { return launch_in_apply(xx.p, stats, al, ga, be, Bc, HW, xx.C, 1e-5f, 1, mode, y.p, st); }, 2);
    ffree(reinterpret_cast<float*>(stats), sb);
  }
  Tensor elu(const Tensor& x, int mode) {
    Tensor y = talloc(x.C, x.H, x.W);
    const long long n = (long long)B * x.H * x.W * x.C;
    const float* src = x.p;
    name("elu %d @%d%s", x.C, x.H, mode == 2 ? " f16-out" : "");
    next_bytes = n * (4.0 + (mode == 2 ? 2.0 : 4.0));
    op(1, [=](cudaStream_t st) { return launch_elu_operand(src, y.p, n, mode, st); }, 6);
    return y;
  }
  // x itself when the contraction reads fp32 (CUDA cores), else a copy in the operand format
  Tensor operand(const Tensor& x, bool tc, bool* owned) {
    *owned = tc;
    if (!tc) return x;
    Tensor y = talloc(x.C, x.H, x.W);
    const long long n = (long long)B * x.H * x.W * x.C; const int omc = om; const float* src = x.p;
    name("operand copy %d @%d", x.C, x.H);
    next_bytes = (double)n * (4.0 + (om == 2 ? 2.0 : 4.0));
    op(1, [=](cudaStream_t st) { return launch_store_operand(src, y.p, n, omc, st); }, 6);
    return y;
  }

  // ResidualBlock (layers.py:453-507): normalize1, ELU, conv1, normalize2, ELU, conv2, + shortcut.  conv2 adds the shortcut
  // (the identity, a 1x1 / dilated 3x3 convolution of x) in its epilogue; a resample='down' block at dilation 1
  // (ConvMeanPool, layers.py:351-369) then takes the 2x2 mean of that sum.
  Tensor nres(const Mod& m, const Tensor& x) {
    Tensor none;
    const int H = x.H, mid = m.down ? m.cin1 : m.cout, d = m.dil;
    const bool meanpool = m.down && d == 1;
    Tensor a = talloc(m.cin1, H, H);
    in_elu(x, m.in[0], mode_for(m.c0w), a);
    Tensor t = talloc(mid, H, H);
    conv(on_tc(m.c0w), a, none, m.c0w, m.c0b, t, Conv().dilation(d));
    tfree(a);
    Tensor a2 = talloc(mid, H, H);
    in_elu(t, m.in[1], mode_for(m.c1w), a2);
    tfree(t);
    Tensor sc;
    if (m.c2w >= 0) {
      bool owned; Tensor xo = operand(x, on_tc(m.c2w), &owned);
      sc = talloc(m.cout, H, H);
      conv(on_tc(m.c2w), xo, none, m.c2w, m.c2b, sc, Conv().taps(d > 1 ? 9 : 1).dilation(d));
      if (owned) tfree(xo);
    }
    Tensor full = talloc(m.cout, H, H);
    conv(on_tc(m.c1w), a2, none, m.c1w, m.c1b, full, Conv().dilation(d).residual(sc.p ? sc : x));
    tfree(a2); tfree(sc);
    if (!meanpool) return full;
    Tensor out = talloc(m.cout, H / 2, H / 2);
    fir(full.p, B, H, H, m.cout, 1, 2, 0, 0, 0, out.p, 0.25f, /*box=*/true);   // mean of each 2x2 cell
    tfree(full);
    return out;
  }

  // RCUBlock(features, n_blocks, 2) (layers.py:183-204): per block x = conv(ELU(conv(ELU(x)))) + x, 3x3 without bias.
  // The last block's output is stored in mode `out_mode` (the operand of an MSF convolution), the rest fp32.  x stays owned by
  // the caller.
  Tensor rcu(const Tensor& x, const std::vector<int>& convs, int out_mode) {
    Tensor none, cur = x;
    const int nblk = (int)convs.size() / 2;
    for (int k = 0; k < nblk; ++k) {
      const int c1 = convs[2 * k], c2 = convs[2 * k + 1];
      Tensor e1 = elu(cur, mode_for(c1));
      Tensor t = talloc(x.C, x.H, x.W);
      conv(on_tc(c1), e1, none, c1, -1, t);
      tfree(e1);
      Tensor e2 = elu(t, mode_for(c2));
      tfree(t);
      Tensor nx = talloc(x.C, x.H, x.W);
      conv(on_tc(c2), e2, none, c2, -1, nx, Conv().residual(cur).round(k == nblk - 1 ? out_mode : 0));
      tfree(e2);
      if (k > 0) tfree(cur);
      cur = nx;
    }
    return cur;
  }

  // RefineBlock (layers.py:277-310): adapt RCUs, MSF (layers.py:236-250: a 3x3 conv with bias of each input, bilinearly
  // resized to the first input's size, summed into zeros in input order), CRP (layers.py:133-154, max pooling), output RCU
  Tensor refine(const Mod& m, const Tensor* xs) {
    Tensor none, h;
    Tensor hs[2];
    for (int i = 0; i < m.nin; ++i) {
      // an MSF input is only read by its MSF convolution: the RCU's last epilogue writes it in that operand format
      const int msf_tc = m.nin > 1 && on_tc(m.msfw[i]) && on_tc(m.adapt[i][3]);
      hs[i] = rcu(xs[i], m.adapt[i], msf_tc ? om : 0);
      if (m.nin > 1 && on_tc(m.msfw[i]) && !msf_tc) {   // CUDA-core RCU feeding a tensor-core MSF convolution
        bool owned; Tensor o = operand(hs[i], true, &owned);
        tfree(hs[i]); hs[i] = o;
      }
    }
    if (m.nin > 1) {
      const int F = m.cout, Ho = hs[0].H;
      Tensor h0 = talloc(F, Ho, Ho);
      conv(on_tc(m.msfw[0]), hs[0], none, m.msfw[0], m.msfb[0], h0);
      tfree(hs[0]);
      if (hs[1].H == Ho) {   // same size: the interpolation is the identity, 0 + h0 + h1 = conv1 + bias + h0 in the epilogue
        h = talloc(F, Ho, Ho);
        conv(on_tc(m.msfw[1]), hs[1], none, m.msfw[1], m.msfb[1], h, Conv().residual(h0));
        tfree(h0);
      } else {
        Tensor h1 = talloc(F, hs[1].H, hs[1].W);
        conv(on_tc(m.msfw[1]), hs[1], none, m.msfw[1], m.msfb[1], h1);
        const int Bc = B, Hl = h1.H, Fc = F;
        name("bilinear 2x +sum %d @%d", F, Ho);
        next_bytes = (double)B * F * (Hl * Hl + 2.0 * Ho * Ho) * 4.0;
        op(1, [=](cudaStream_t st) { return launch_bilinear_add(h1.p, Bc, Hl, Hl, Fc, h0.p, Ho, Ho, st); }, 3);
        tfree(h1);
        h = h0;
      }
      tfree(hs[1]);
    } else {
      h = hs[0];
    }
    // CRP: x = ELU(x); path = x; twice: path = conv(maxpool(path)); x = path + x.  The second pool also writes
    // x1 = path1 + ELU(x), which the last convolution adds in its epilogue.
    const int F = h.C, H = h.H, Bc = B;
    Tensor xa = elu(h, 0);
    tfree(h);
    Tensor pool0 = talloc(F, H, H);
    { const int md = mode_for(m.crp[0]); name("maxpool5x5 %d @%d", F, H); next_bytes = (double)B * H * H * F * 8.0;
      op(1, [=](cudaStream_t st) { return launch_maxpool5(xa.p, Bc, H, H, F, md, pool0.p, nullptr, nullptr, st); }, 6); }
    Tensor path1 = talloc(F, H, H);
    conv(on_tc(m.crp[0]), pool0, none, m.crp[0], -1, path1);
    tfree(pool0);
    Tensor pool1 = talloc(F, H, H), x1 = talloc(F, H, H);
    { const int md = mode_for(m.crp[1]); name("maxpool5x5 +sum %d @%d", F, H); next_bytes = (double)B * H * H * F * 16.0;
      op(1, [=](cudaStream_t st) { return launch_maxpool5(path1.p, Bc, H, H, F, md, pool1.p, xa.p, x1.p, st); }, 6); }
    tfree(path1); tfree(xa);
    Tensor x2 = talloc(F, H, H);
    conv(on_tc(m.crp[1]), pool1, none, m.crp[1], -1, x2, Conv().residual(x1));
    tfree(pool1); tfree(x1);
    Tensor out = rcu(x2, m.outc, 0);
    tfree(x2);
    return out;
  }

  // output (ncsnv2.py:124-132): normalizer, ELU, end_conv, / sigmas[y] (the caller passes sigma per image as the label)
  void nhead(const Mod& m, Tensor& h) {
    const int R = h.H, ch = m.cout, ln = lane, Bc = B, C = h.C;
    b200_ncsnpp* eng = e;
    Tensor a = talloc(C, R, R);
    in_elu(h, m.in[0], 0, a);
    tfree(h);
    const float *wo = e->W(m.w), *bo = e->W(m.b);
    name("conv3x3 %d->%d @%d nchw-out /sigma [small-n]", C, ch, R);
    next_bytes = (double)B * R * R * (C + ch) * 4.0;
    op(1, [=](cudaStream_t st) {
      return launch_conv3x3_small_n(a.p, wo, bo, eng->in_labels_l[ln], eng->uniform ? 0 : 1, eng->out_l[ln], Bc, R, R, C, ch, 0, st);
    }, 1, 2.0 * B * R * R * (double)ch * C * 9);
    tfree(a);
  }

  // the forward pass of NCSNv2 / NCSNv2_128 (ncsnv2.py:107-132, 278-312) as a walk over e->mods
  int build_ncsnv2() {
    mi = 0;
    const int L = e->cfg.num_levels;
    Tensor x = input_conv();   // 2x - 1 (unless centred), begin_conv
    if (rc) return rc;
    std::vector<Tensor> layers;
    for (int l = 0; l < L; ++l) {
      const Mod& m0 = next(); Tensor a = nres(m0, x); if (rc) return rc;
      tap(m0.index, a);
      if (l == 0) tfree(x);   // begin_conv's output; later levels keep their input in `layers`
      const Mod& m1 = next(); Tensor b = nres(m1, a); if (rc) return rc;
      tap(m1.index, b);
      tfree(a);
      layers.push_back(b); x = b;
    }
    Tensor ref;
    for (int k = 1; k <= L; ++k) {
      const Mod& m = next();
      const Tensor xs[2] = {layers[L - k], ref};
      Tensor r = refine(m, xs); if (rc) return rc;
      tap(m.index, r);
      tfree(layers[L - k]); tfree(ref);
      ref = r;
    }
    const Mod& mh = next();
    nhead(mh, ref);
    if (mi != e->mods.size()) { set_error("ncsnv2: plan walked %zu of %zu modules", mi, e->mods.size()); return 2; }
    return rc;
  }

  // the forward pass (models/ncsnpp.py:232-381) as a walk over e->mods
  int build() {
    if (e->cfg.family == 2) return build_ncsnv2();
    const b200_ncsnpp_config& c = e->cfg;
    const int L = c.num_levels;
    Tensor none;
    time_embedding();
    std::vector<Tensor> hs = {input_conv()};
    for (int lvl = 0; lvl < L; ++lvl) {
      for (int b = 0; b < c.num_res_blocks; ++b) {
        const Mod& m = next();
        Tensor h = resblock(m, hs.back(), none); if (rc) return rc;
        tap(m.index, h);
        if (mi < e->mods.size() && e->mods[mi].kind == M_ATTN && e->mods[mi].res == h.H && has_attn(c, h.H)) {
          const Mod& ma = next();
          Tensor h2 = attn(ma, h); if (rc) return rc;
          advance(h, ma, h2);
        }
        hs.push_back(h);
      }
      if (lvl != L - 1) {
        const Mod& m = next();
        Tensor h = m.kind == M_DOWN ? downsample(m, hs.back()) : resblock(m, hs.back(), none); if (rc) return rc;
        tap(m.index, h);
        if (c.progressive_input) { h = input_pyramid(h); if (rc) return rc; }
        hs.push_back(h);
      }
    }
    Tensor h = middle(hs.back()); if (rc) return rc;
    // ---- up path (ncsnpp.py:316-364) ----
    for (int lvl = L - 1; lvl >= 0; --lvl) {
      for (int b = 0; b < c.num_res_blocks + 1; ++b) {
        const Mod& m = next();
        Tensor skip = hs.back(); hs.pop_back();
        Tensor h2 = resblock(m, h, skip); if (rc) return rc;
        advance(h, m, h2);
        tfree(skip);
      }
      if (e->mods[mi].kind == M_ATTN) {
        const Mod& ma = next();
        Tensor h2 = attn(ma, h); if (rc) return rc;
        advance(h, ma, h2);
      }
      if (c.progressive == 1) { output_skip(h, lvl == 0); if (rc) return rc; }
      if (lvl != 0) {
        const Mod& m = next();
        Tensor h2 = m.kind == M_UP ? upsample(m, h) : resblock(m, h, none); if (rc) return rc;
        advance(h, m, h2);
      }
    }
    // with output_skip the pyramid already is the output
    if (c.progressive != 1) { head(h); if (rc) return rc; }
    if (mi != e->mods.size()) { set_error("ncsnpp: plan walked %zu of %zu modules", mi, e->mods.size()); return 2; }
    if (!dry && stats_top > 0) {
      // the epilogue-accumulated GroupNorm sums start from zero every forward: one memset of the whole region
      char* sb = stats_base; const long long sn = stats_top;
      e->launches += 1;
      auto& lops = lane ? e->ops2 : e->ops;
      lops.insert(lops.begin(), b200_ncsnpp::Op{6, 0.0, [=](cudaStream_t st) {
        return cudaMemsetAsync(sb, 0, (size_t)sn, st) == cudaSuccess ? 0 : (set_error("stats memset failed"), 1);
      }, "zero GroupNorm sums", 0.0});
    }
    return rc;
  }
};

}  // namespace

// ===========================================================================
// C ABI: model
// ===========================================================================
extern "C" {

int b200_ncsnpp_create(const b200_ncsnpp_config* cfg, b200_ncsnpp_t** out) {
  B200_REQUIRE(cfg && out, "ncsnpp_create: null argument");
  B200_REQUIRE(cfg->no_halo == 0 || cfg->no_halo == 1, "ncsnpp_create: no_halo=%d unknown (0 halo form, 1 one tile per tap)",
               cfg->no_halo);
  B200_REQUIRE(cfg->family >= 0 && cfg->family <= 2, "ncsnpp_create: family=%d unknown (0 NCSN++, 1 DDPM, 2 NCSNv2)", cfg->family);
  B200_REQUIRE(cfg->precision >= 0 && cfg->precision <= 3, "ncsnpp_create: precision=%d unknown (0 tf32, 1 fp32, 2 f16, 3 split tf32)",
               cfg->precision);
  if (cfg->family == 1) {
    B200_REQUIRE(cfg->conditional, "ncsnpp_create: DDPM (family 1) needs conditional = 1 (the reference's own constructor fails "
                 "without time conditioning, models/ddpm.py:58-71)");
    B200_REQUIRE(!cfg->scale_by_sigma, "ncsnpp_create: DDPM (family 1) with scale_by_sigma = 1 (configs/ve/cifar10_ddpm.py) is not "
                 "supported by the engine");
  }
  if (cfg->family == 2) {
    B200_REQUIRE(!cfg->tangent, "ncsnpp_create: family = 2 (NCSNv2) has no forward-mode tangent pass (tangent = 1)");
    B200_REQUIRE(cfg->precision != 3, "ncsnpp_create: family = 2 (NCSNv2) runs in precision 0 (tf32), 1 (fp32) or 2 (f16), not "
                 "3 (split tf32)");
    B200_REQUIRE(cfg->num_levels == 4 || cfg->num_levels == 5, "ncsnpp_create: family = 2 (NCSNv2) has num_levels = 4 (ncsnv2_64) "
                 "or 5 (ncsnv2_128), got %d", cfg->num_levels);
    B200_REQUIRE(cfg->nf >= 4 && cfg->nf % 4 == 0 && cfg->nf * (cfg->num_levels == 5 ? 4 : 2) <= 512,
                 "ncsnpp_create: family = 2 (NCSNv2) needs nf a multiple of 4 with at most 512 channels per level, got nf=%d", cfg->nf);
    B200_REQUIRE(cfg->num_channels >= 1 && cfg->num_channels <= 4, "ncsnpp_create: family = 2 (NCSNv2) takes 1..4 image channels, "
                 "got %d", cfg->num_channels);
    B200_REQUIRE(cfg->image_size >= 8 && cfg->image_size % (cfg->num_levels == 5 ? 8 : 4) == 0,
                 "ncsnpp_create: family = 2 (NCSNv2): image_size=%d does not halve %d times", cfg->image_size, cfg->num_levels == 5 ? 3 : 2);
  }
  if (cfg->tangent) {
    // the forward-mode tangent pass (b200_ncsnpp_jvp) covers DDPM and the DDPM++ family; everything else is refused here
    // rather than approximated
    B200_REQUIRE(cfg->tangent == 1, "ncsnpp_create: tangent=%d unknown (0 or 1)", cfg->tangent);
    B200_REQUIRE(cfg->precision != 2, "ncsnpp_create: tangent = 1 with precision = %d: the tangent pass "
                 "runs in precision 0 (tf32), 1 (fp32) or 3 (split tf32), not on fp16 operands", cfg->precision);
    B200_REQUIRE(cfg->lanes <= 1, "ncsnpp_create: tangent = 1 with lanes = %d: the tangent pass runs one lane", cfg->lanes);
    if (cfg->family == 0) {
      B200_REQUIRE(cfg->naive_resample, "ncsnpp_create: tangent = 1 with naive_resample = 0: FIR resampling has no tangent pass");
      B200_REQUIRE(cfg->progressive == 0, "ncsnpp_create: tangent = 1 with progressive = %d: the output_skip pyramid has no "
                   "tangent pass", cfg->progressive);
      B200_REQUIRE(cfg->progressive_input == 0, "ncsnpp_create: tangent = 1 with progressive_input = %d: the input pyramid has "
                   "no tangent pass", cfg->progressive_input);
    }
  }
  b200_ncsnpp* e = new b200_ncsnpp();
  e->cfg = *cfg;
  if (cfg->family == 1) {
    // the fields DDPM ignores take the values that describe it on the shared paths: residual scale 1, no pyramids,
    // sinusoidal embedding (ddpm.py:116), and a unit FIR that no DDPM layer reads
    b200_ncsnpp_config& c = e->cfg;
    c.skip_rescale = 0; c.progressive_input = 0; c.progressive = 0; c.embedding_type = 1; c.naive_resample = 1;
    c.fir_taps = 1; c.fir_kernel[0] = 1.f;
  }
  if (cfg->family == 2) {
    // NCSNv2 reads image_size, num_channels, nf, num_levels, centered and the execution fields; the rest takes the values
    // that keep the shared paths inert: no pyramids, no time embedding, a unit FIR no layer reads
    b200_ncsnpp_config& c = e->cfg;
    c.skip_rescale = 0; c.progressive_input = 0; c.progressive = 0; c.embedding_type = 0; c.naive_resample = 1;
    c.fir_taps = 1; c.fir_kernel[0] = 1.f; c.scale_by_sigma = 1; c.conditional = 1; c.num_res_blocks = 2;
  }
  if (int r = build_graph(e)) { delete e; return r; }
  *out = e;
  return 0;
}

void b200_ncsnpp_destroy(b200_ncsnpp_t* h) { delete h; }

int b200_ncsnpp_num_params(const b200_ncsnpp_t* h) { return h ? (int)h->params.size() : 0; }

int b200_ncsnpp_param_info(const b200_ncsnpp_t* h, int index, char* name, int name_cap, long long shape[4], int* ndim) {
  B200_REQUIRE(h && index >= 0 && index < (int)h->params.size(), "param_info: index %d out of range", index);
  const Param& p = h->params[index];
  if (name && name_cap > 0) { strncpy(name, p.name.c_str(), name_cap - 1); name[name_cap - 1] = 0; }
  if (shape) for (int i = 0; i < 4; ++i) shape[i] = p.shape[i];
  if (ndim) *ndim = p.ndim;
  return 0;
}

long long b200_ncsnpp_weights_bytes(const b200_ncsnpp_t* h) { return h ? h->wcount * 4 + 256 : 0; }

int b200_ncsnpp_bind_weights(b200_ncsnpp_t* h, void* blob) {
  B200_REQUIRE(h && blob, "bind_weights: null argument");
  B200_REQUIRE(h->ops.empty(), "bind_weights: rebind after planning is not supported");
  // the blob is over-allocated by 256 B (b200_ncsnpp_weights_bytes) so any base can be aligned here
  h->wblob = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(blob) + 255) & ~uintptr_t(255));
  return 0;
}

int b200_ncsnpp_load_param(b200_ncsnpp_t* h, int index, const float* src, void* stream) {
  B200_REQUIRE(h && h->wblob, "load_param: weights not bound");
  B200_REQUIRE(index >= 0 && index < (int)h->params.size(), "load_param: index %d out of range", index);
  const Param& p = h->params[index];
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* dst = h->wblob + p.off;
  if (p.pack == PK_COPY) {
    B200_CHECK_CUDA(cudaMemcpyAsync(dst, src, p.count * 4, cudaMemcpyDeviceToDevice, st));
    return 0;
  }
  // split TF32 (round 3): the hi copy on the TF32 grid at off, the lo copy in the same layout at p.lo
  const int rnd = p.round == 3 ? 1 : p.round;
  float* lo = p.round == 3 ? h->wblob + p.lo : nullptr;
  if (p.pack == PK_CONV_FLAT32)   // OIHW (3x3, I*9 <= 32) -> [O][32] with k = tap*I + i (rest of the row stays zero)
    return launch_pack_weight(src, dst, p.taps, p.O, p.I, (long long)p.I * p.taps, p.taps, 1, rnd, st, p.I, p.round == 2 ? 64 : 32, lo);
  if (p.pack == PK_CONV_PAD128)   // OIHW -> [tap][128][I], rows >= O stay zero
    return launch_pack_weight(src, dst, p.taps, p.O, p.I, (long long)p.I * p.taps, p.taps, 1, rnd, st, 128LL * p.I, p.I, lo);
  if (p.pack == PK_CONV)   // OIHW -> [tap][O][I]
    return launch_pack_weight(src, dst, p.taps, p.O, p.I, (long long)p.I * p.taps, p.taps, 1, rnd, st, 0, 0, lo);
  // NIN W[in][out] -> [out][in]
  return launch_pack_weight(src, dst, 1, p.O, p.I, 1, p.O, 0, rnd, st, 0, 0, lo);
}

namespace {
// Lane split of a batch (cfg.lanes == 2): two halves when the batch is large
// enough for every launch of a half to fill the GPU; one lane otherwise, by default, and always with
// keep_activations (its taps address whole-batch tensors).
int lane0_images(const b200_ncsnpp* h, int batch) {
  const int lanes = h->cfg.lanes;
  if (lanes < 2 || h->cfg.keep_activations || batch < 128) return batch;
  return (batch + 1) / 2;
}
long long lane_bytes(b200_ncsnpp* h, int images, long long* arena_out) {
  Builder b(h, images, nullptr, true);
  if (b.build()) return -1;
  const long long a = (b.arena.high_water() + 1023) & ~1023LL;
  if (arena_out) *arena_out = a;
  return a + ((b.stats_top + 1023) & ~1023LL);
}
}  // namespace

long long b200_ncsnpp_workspace_bytes(b200_ncsnpp_t* h, int batch) {
  if (!h || batch <= 0) return -1;
  const int b0 = lane0_images(h, batch);
  long long total = lane_bytes(h, b0, nullptr);
  if (total < 0) return -1;
  if (b0 < batch) { const long long t1 = lane_bytes(h, batch - b0, nullptr); if (t1 < 0) return -1; total += t1; }
  return total + 2048;   // + slack to align any caller pointer to 1024 B
}

int b200_ncsnpp_bind_workspace(b200_ncsnpp_t* h, int batch, void* ws, long long ws_bytes) {
  B200_REQUIRE(h && ws && batch > 0, "bind_workspace: bad argument");
  B200_REQUIRE(h->wblob, "bind_workspace: bind the weight blob first");
  const long long need = b200_ncsnpp_workspace_bytes(h, batch);
  B200_REQUIRE(need >= 0, "bind_workspace: planning failed: %s", last_error());
  B200_REQUIRE(ws_bytes >= need, "bind_workspace: workspace too small (%lld < %lld bytes)", ws_bytes, need);
  for (auto* p : h->tcplans) tc_gemm_plan_destroy(p);
  for (auto* p : h->attnplans) tc_attn_plan_destroy(p);
  h->attnplans.clear();
  h->tcplans.clear(); h->ops.clear(); h->ops2.clear(); h->taps.clear(); h->launches = 0;
  h->B = batch; h->ws_bytes = ws_bytes;
  h->ws = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(ws) + 1023) & ~uintptr_t(1023));
  h->B0 = lane0_images(h, batch);
  char* base = h->ws;
  for (int lane = 0; lane < (h->B0 < batch ? 2 : 1); ++lane) {
    const int images = lane ? batch - h->B0 : h->B0;
    long long arena_bytes = 0;
    const long long lb = lane_bytes(h, images, &arena_bytes);
    if (lb < 0) return 1;
    Builder b(h, images, base, false, lane);
    b.stats_base = base + arena_bytes;   // quad sums live after the lane's activation arena
    if (int r = b.build()) { h->ops.clear(); h->ops2.clear(); return r; }
    base += lb;
  }
  if (!h->ops2.empty() && !h->lane_stream) {
    B200_CHECK_CUDA(cudaStreamCreateWithFlags(&h->lane_stream, cudaStreamNonBlocking));
    B200_CHECK_CUDA(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
    B200_CHECK_CUDA(cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming));
  }
  return 0;
}

namespace {
void set_call_args(b200_ncsnpp* h, const float* x, const float* labels, int uniform, float* out) {
  h->in_x = x; h->in_labels = labels; h->out = out; h->uniform = uniform;
  const long long per_img = (long long)h->cfg.num_channels * h->cfg.image_size * h->cfg.image_size;
  h->in_x_l[0] = x; h->in_labels_l[0] = labels; h->out_l[0] = out;
  h->in_x_l[1] = x + h->B0 * per_img; h->in_labels_l[1] = uniform ? labels : labels + h->B0; h->out_l[1] = out + h->B0 * per_img;
}

// op i of the plan: lane 0's ops, then lane 1's; nullptr when out of range
const b200_ncsnpp::Op* op_at(const b200_ncsnpp* h, long long i) {
  if (!h || i < 0) return nullptr;
  const long long n0 = (long long)h->ops.size();
  if (i < n0) return &h->ops[i];
  return i - n0 < (long long)h->ops2.size() ? &h->ops2[i - n0] : nullptr;
}

// every op of both lanes serially on ONE stream, each between two events: each launch is timed alone (no overlap), which is
// what a per-kernel roofline needs.  ms[i] receives op i's time.
int time_ops(b200_ncsnpp* h, const float* x, const float* labels, int uniform, float* out, void* stream, float* ms, const char* who) {
  set_call_args(h, x, labels, uniform, out);
  h->in_v = x; h->tout = out;   // tangent plans: the JVP pass along v = x
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long n = (long long)(h->ops.size() + h->ops2.size());
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& e : ev) B200_CHECK_CUDA(cudaEventCreate(&e));
  int rc = 0;
  B200_CHECK_CUDA(cudaEventRecord(ev[0], st));
  for (long long i = 0; i < n && !rc; ++i) {
    rc = op_at(h, i)->fn(st);
    cudaEventRecord(ev[i + 1], st);
  }
  if (!rc && cudaStreamSynchronize(st) != cudaSuccess) { set_error("%s: stream sync failed", who); rc = 1; }
  if (!rc) for (long long i = 0; i < n; ++i) cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]);
  for (auto& e : ev) cudaEventDestroy(e);
  return rc;
}
}  // namespace

int b200_ncsnpp_forward(b200_ncsnpp_t* h, const float* x, const float* labels, int uniform, float* out, void* stream) {
  B200_REQUIRE(h && x && labels && out, "forward: null argument");
  B200_REQUIRE(!h->ops.empty(), "forward: no plan bound (call b200_ncsnpp_bind_workspace)");
  B200_REQUIRE(!h->cfg.tangent, "forward: the engine was created with tangent = 1; call b200_ncsnpp_jvp");
  PdlScope pdl(h->cfg.pdl != 0);            // launches of this call carry the programmatic-dependent-launch attribute
  set_call_args(h, x, labels, uniform, out);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (h->ops2.empty()) {
    for (auto& o : h->ops) if (int r = o.fn(st)) return r;
    return 0;
  }
  // fork: lane 1 runs on the engine's side stream, ordered after everything already queued on `st`
  // (event record/wait pairs are also what stream capture turns into parallel graph branches)
  B200_CHECK_CUDA(cudaEventRecord(h->ev_fork, st));
  B200_CHECK_CUDA(cudaStreamWaitEvent(h->lane_stream, h->ev_fork, 0));
  const size_t n = std::max(h->ops.size(), h->ops2.size());
  int rc = 0;
  for (size_t i = 0; i < n && !rc; ++i) {       // interleaved issue so eager (non-graph) launches overlap too
    if (i < h->ops.size()) rc = h->ops[i].fn(st);
    if (!rc && i < h->ops2.size()) rc = h->ops2[i].fn(h->lane_stream);
  }
  // join (also on failure, so a capture in progress is left well-formed)
  const cudaError_t e1 = cudaEventRecord(h->ev_join, h->lane_stream);
  const cudaError_t e2 = cudaStreamWaitEvent(st, h->ev_join, 0);
  if (rc) return rc;
  B200_CHECK_CUDA(e1); B200_CHECK_CUDA(e2);
  return 0;
}

int b200_ncsnpp_jvp(b200_ncsnpp_t* h, const float* x, const float* labels, int uniform, const float* v, float* out, float* jvp_out,
                    void* stream) {
  B200_REQUIRE(h && x && labels && v && out && jvp_out, "jvp: null argument");
  B200_REQUIRE(h->cfg.tangent, "jvp: the engine was not created with tangent = 1");
  B200_REQUIRE(!h->ops.empty(), "jvp: no plan bound (call b200_ncsnpp_bind_workspace)");
  PdlScope pdl(h->cfg.pdl != 0);
  set_call_args(h, x, labels, uniform, out);
  h->in_v = v; h->tout = jvp_out;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (auto& o : h->ops) if (int r = o.fn(st)) return r;   // one lane (b200_ncsnpp_create rejects lanes = 2 with tangent = 1)
  return 0;
}

int b200_ncsnpp_profile_forward(b200_ncsnpp_t* h, const float* x, const float* labels, int uniform, float* out,
                                void* stream, float ms_by_kind[8], double flops_by_kind[8], long long ops_by_kind[8]) {
  B200_REQUIRE(h && x && labels && out && ms_by_kind, "profile_forward: null argument");
  B200_REQUIRE(!h->ops.empty(), "profile_forward: no plan bound");
  for (int k = 0; k < 8; ++k) { ms_by_kind[k] = 0.f; if (flops_by_kind) flops_by_kind[k] = 0.0; if (ops_by_kind) ops_by_kind[k] = 0; }
  std::vector<float> ms(h->ops.size() + h->ops2.size());
  if (int rc = time_ops(h, x, labels, uniform, out, stream, ms.data(), "profile_forward")) return rc;
  for (size_t i = 0; i < ms.size(); ++i) {
    const b200_ncsnpp::Op& o = *op_at(h, (long long)i);
    const int k = o.kind & 7;
    ms_by_kind[k] += ms[i];
    if (flops_by_kind) flops_by_kind[k] += o.flops;
    if (ops_by_kind) ops_by_kind[k] += 1;
  }
  return 0;
}

long long b200_ncsnpp_num_ops(const b200_ncsnpp_t* h) { return h ? (long long)(h->ops.size() + h->ops2.size()) : 0; }

int b200_ncsnpp_op_info(const b200_ncsnpp_t* h, long long index, char* name, int name_cap, int* kind, double* flops) {
  const b200_ncsnpp::Op* o = op_at(h, index);
  B200_REQUIRE(o, "op_info: index out of range");
  if (name && name_cap > 0) { strncpy(name, o->name.c_str(), name_cap - 1); name[name_cap - 1] = 0; }
  if (kind) *kind = o->kind;
  if (flops) *flops = o->flops;
  return 0;
}

int b200_ncsnpp_op_bytes(const b200_ncsnpp_t* h, long long index, double* bytes) {
  const b200_ncsnpp::Op* o = op_at(h, index);
  B200_REQUIRE(o && bytes, "op_bytes: index out of range");
  *bytes = o->bytes;
  return 0;
}

int b200_ncsnpp_profile_ops(b200_ncsnpp_t* h, const float* x, const float* labels, int uniform, float* out, void* stream,
                            float* ms_per_op, long long cap) {
  B200_REQUIRE(h && x && labels && out && ms_per_op, "profile_ops: null argument");
  B200_REQUIRE(!h->ops.empty(), "profile_ops: no plan bound");
  const long long n = (long long)(h->ops.size() + h->ops2.size());
  B200_REQUIRE(cap >= n, "profile_ops: need room for %lld ops", n);
  return time_ops(h, x, labels, uniform, out, stream, ms_per_op, "profile_ops");
}

int b200_ncsnpp_tap(b200_ncsnpp_t* h, int module_index, float* dst, long long cap, int shape_out[4], void* stream) {
  B200_REQUIRE(h && h->cfg.keep_activations, "tap: engine was not created with keep_activations=1");
  auto it = h->taps.find(module_index);
  B200_REQUIRE(it != h->taps.end(), "tap: module %d has no recorded activation", module_index);
  const Tensor& t = it->second;
  const long long n = (long long)h->B * t.C * t.H * t.W;
  if (shape_out) { shape_out[0] = h->B; shape_out[1] = t.C; shape_out[2] = t.H; shape_out[3] = t.W; }
  B200_REQUIRE(cap >= n, "tap: destination too small (%lld < %lld)", cap, n);
  return launch_nhwc_to_nchw(t.p, dst, h->B, t.H * t.W, t.C, static_cast<cudaStream_t>(stream));
}

int b200_ncsnpp_tap_tangent(b200_ncsnpp_t* h, int module_index, float* dst, long long cap, int shape_out[4], void* stream) {
  B200_REQUIRE(h && h->cfg.keep_activations && h->cfg.tangent, "tap_tangent: engine was not created with keep_activations=1, tangent=1");
  auto it = h->taps.find(module_index);
  B200_REQUIRE(it != h->taps.end() && it->second.d, "tap_tangent: module %d has no recorded tangent", module_index);
  const Tensor& t = it->second;
  const long long n = (long long)h->B * t.C * t.H * t.W;
  if (shape_out) { shape_out[0] = h->B; shape_out[1] = t.C; shape_out[2] = t.H; shape_out[3] = t.W; }
  B200_REQUIRE(cap >= n, "tap_tangent: destination too small (%lld < %lld)", cap, n);
  return launch_nhwc_to_nchw(t.d, dst, h->B, t.H * t.W, t.C, static_cast<cudaStream_t>(stream));
}

long long b200_ncsnpp_launches_per_forward(const b200_ncsnpp_t* h) { return h ? h->launches : 0; }

}  // extern "C"

// ===========================================================================
// C ABI: predictor-corrector loop
// ===========================================================================
// per-step schedule tables of a PC plan (b200_pc_config: label .. cs, mq .. pm2); cm and cs only in constrained plans,
// mq .. pm2 only in multistep plans (predictor == 2)
enum PcTable { PC_LABEL, PC_SS, PC_ALPHA, PC_PA, PC_PB, PC_PC, PC_CA, PC_CB, PC_CC, PC_CM, PC_CS, PC_MQ, PC_MR, PC_PM1, PC_PM2,
               PC_TABLES };

static bool pc_table_used(const b200_pc_config& c, int k) {
  if (k >= PC_MQ) return c.predictor == 2;
  if (k >= PC_CM) return c.constraint != 0;
  return true;
}

struct b200_pc {
  b200_ncsnpp* model; b200_pc_config cfg; int B; long long numel, per_img;
  std::vector<float> h_tab[PC_TABLES];   // host copies, uploaded by b200_pc_bind_workspace
  // workspace carve-up
  char* ws = nullptr; float* d_tab[PC_TABLES] = {}; float *labels, *net_out, *norms, *means;
  float* hist = nullptr;   // multistep plans: three slots of numel floats (the last three data / noise predictions)
  int* d_step; unsigned long long* d_offset;
  PhiloxMap map;
  const float* known = nullptr; const float* mask = nullptr;   // constrained plans: bound by b200_pc_bind_constraint
  PcColorTransform color{};
  cudaGraphExec_t gexec = nullptr; float* graph_x = nullptr; float* graph_xm = nullptr; cudaStream_t graph_stream = nullptr;
  const float* graph_known = nullptr; const float* graph_mask = nullptr;
  unsigned long long graph_seed = 0;
  cudaStream_t cap_stream = nullptr;   // the legacy default stream cannot be captured: capture on a private one
  long long launches_per_step = 0;
  ~b200_pc() { if (gexec) cudaGraphExecDestroy(gexec); if (cap_stream) cudaStreamDestroy(cap_stream); }
};

namespace {

long long pc_ws_layout(b200_pc* pc, char* base) {
  long long off = 0;
  auto take = [&](long long bytes) { long long o = off; off += (bytes + 255) & ~255LL; return base ? base + o : nullptr; };
  const int N = pc->cfg.n_steps;
  for (int k = 0; k < PC_TABLES; ++k) if (pc_table_used(pc->cfg, k)) pc->d_tab[k] = (float*)take(N * 4LL);
  pc->labels = (float*)take(pc->B * 4LL); pc->net_out = (float*)take(pc->numel * 4LL);
  pc->norms = (float*)take(2LL * pc->B * 4); pc->means = (float*)take(256);
  pc->d_step = (int*)take(256); pc->d_offset = (unsigned long long*)take(256);
  if (pc->cfg.predictor == 2) pc->hist = (float*)take(3 * pc->numel * 4LL);
  return off;
}

// randn_like calls per iteration: the corrector's inner steps, the noisy predictor, and the two constraint blends
// (the multistep ODE update draws none)
unsigned long long pc_calls_per_step(const b200_pc_config& c) {
  return (unsigned long long)((c.corrector ? c.n_corrector_steps : 0) + (c.predictor == 1 ? 1 : 0) + (c.constraint ? 2 : 0));
}

int pc_constrain(b200_pc* pc, float* x, float* x_mean, unsigned long long cps, unsigned long long call, cudaStream_t st) {
  const b200_ncsnpp_config& mc = pc->model->cfg;
  return launch_pc_constrain(x, x_mean, pc->known, pc->mask, pc->map, pc->d_offset, pc->d_step, cps, call, pc->d_tab[PC_CM],
                             pc->d_tab[PC_CS], pc->color, pc->cfg.constraint == 2, mc.num_channels,
                             (long long)mc.image_size * mc.image_size, st);
}

// one PC iteration at step *d_step; noise_c/noise_p non-null -> external noise
int pc_iteration(b200_pc* pc, float* x, float* x_mean, const float* noise_c, const float* noise_p, cudaStream_t st) {
  b200_ncsnpp* m = pc->model;
  const b200_pc_config& c = pc->cfg;
  float* const* t = pc->d_tab;
  PcStepScalars sc{t[PC_SS], t[PC_ALPHA], t[PC_PA], t[PC_PB], t[PC_PC]};
  const unsigned long long cps = pc_calls_per_step(c);
  if (int r = launch_fill_from_table(t[PC_LABEL], pc->d_step, pc->labels, pc->B, st)) return r;
  if (c.predictor == 2) {
    PcMultistepScalars ms{t[PC_MQ], t[PC_MR], t[PC_PA], t[PC_PB], t[PC_PM1], t[PC_PM2]};
    if (int r = b200_ncsnpp_forward(m, x, pc->labels, 1, pc->net_out, st)) return r;
    if (int r = launch_pc_multistep(x, x_mean, pc->net_out, pc->hist, pc->numel, pc->d_step, ms, st)) return r;
    return launch_step_increment(pc->d_step, st);
  }
  unsigned long long call = 0;
  if (c.corrector == 2) {
    // affine corrector (annealed Langevin dynamics, sampling.py:286-319): the step size is a per-step scalar, so the update is
    // the predictor's kernel with the corrector's own tables; every inner step draws fresh noise like the reference's loop
    PcStepScalars cs{t[PC_SS], t[PC_ALPHA], t[PC_CA], t[PC_CB], t[PC_CC]};
    for (int k = 0; k < c.n_corrector_steps; ++k) {
      if (int r = b200_ncsnpp_forward(m, x, pc->labels, 1, pc->net_out, st)) return r;
      if (int r = launch_predictor_apply(x, x_mean, pc->net_out, noise_c, pc->map, pc->d_offset, pc->d_step, cps, call, cs, 1, st)) return r;
      ++call;
    }
  } else if (c.corrector) {
    for (int k = 0; k < c.n_corrector_steps; ++k) {
      if (int r = b200_ncsnpp_forward(m, x, pc->labels, 1, pc->net_out, st)) return r;
      if (int r = launch_pc_norms(pc->net_out, noise_c, pc->map, pc->d_offset, pc->d_step, cps, call, pc->B,
                                  (int)pc->per_img, pc->norms, pc->means, st)) return r;
      if (int r = launch_langevin_apply(x, x_mean, pc->net_out, noise_c, pc->map, pc->d_offset, pc->d_step, cps, call,
                                        pc->means, c.snr, sc, st)) return r;
      ++call;
    }
  }
  if (c.constraint) {
    // controllable_generation.py:43-52 / :137-146 after the corrector update, which a NoneCorrector makes the identity
    if (int r = pc_constrain(pc, x, x_mean, cps, call, st)) return r;
    ++call;
  }
  if (c.predictor) {
    if (int r = b200_ncsnpp_forward(m, x, pc->labels, 1, pc->net_out, st)) return r;
    if (int r = launch_predictor_apply(x, x_mean, pc->net_out, noise_p, pc->map, pc->d_offset, pc->d_step, cps, call,
                                       sc, 1, st)) return r;
    ++call;
  }
  if (c.constraint) {
    // the blend after the predictor writes this iteration's x_mean, also for a NonePredictor
    if (int r = pc_constrain(pc, x, x_mean, cps, call, st)) return r;
  } else if (!c.predictor && x_mean) {
    // NonePredictor.update_fn returns (x, x) (sampling.py:241-250): the "mean" handed to the denoise step of
    // pc_sampler (:409) is the noisy state after the corrector, not the last Langevin mean
    B200_CHECK_CUDA(cudaMemcpyAsync(x_mean, x, (size_t)pc->numel * 4, cudaMemcpyDeviceToDevice, st));
  }
  return launch_step_increment(pc->d_step, st);
}

}  // namespace

extern "C" {

int b200_pc_create(b200_ncsnpp_t* model, const b200_pc_config* cfg, int batch, b200_pc_t** out) {
  B200_REQUIRE(model && cfg && out && batch > 0, "pc_create: bad argument");
  B200_REQUIRE(model->B == batch && !model->ops.empty(), "pc_create: model is not planned for batch %d", batch);
  B200_REQUIRE(cfg->n_steps > 0 && cfg->label && cfg->pb, "pc_create: missing schedule tables");
  B200_REQUIRE(cfg->corrector >= 0 && cfg->corrector <= 2, "pc_create: corrector %d unsupported", cfg->corrector);
  B200_REQUIRE(cfg->corrector != 2 || (cfg->ca && cfg->cb && cfg->cc), "pc_create: affine corrector without its tables");
  B200_REQUIRE(cfg->predictor >= 0 && cfg->predictor <= 2, "pc_create: predictor %d unsupported", cfg->predictor);
  B200_REQUIRE(cfg->predictor != 2 || (cfg->corrector == 0 && cfg->constraint == 0),
               "pc_create: the multistep ODE update (predictor 2) takes no corrector and no constraint");
  B200_REQUIRE(cfg->constraint >= 0 && cfg->constraint <= 2, "pc_create: constraint %d unsupported", cfg->constraint);
  B200_REQUIRE(!cfg->constraint || (cfg->cm && cfg->cs), "pc_create: constraint without its cm/cs tables");
  B200_REQUIRE(cfg->noise_nhwc == 0 || cfg->noise_nhwc == 1, "pc_create: noise_nhwc %d unsupported", cfg->noise_nhwc);
  B200_REQUIRE(cfg->constraint != 2 || model->cfg.num_channels == 3,
               "pc_create: colorization needs 3 channels, the model has %d", model->cfg.num_channels);
  b200_pc* pc = new b200_pc();
  pc->model = model; pc->cfg = *cfg; pc->B = batch;
  const b200_ncsnpp_config& mc = model->cfg;
  pc->per_img = (long long)mc.num_channels * mc.image_size * mc.image_size;
  pc->numel = pc->per_img * batch;
  const int N = cfg->n_steps;
  // a table the caller leaves null takes its default: label 0, score_scale 1, alpha 1, the predictor's and the
  // corrector's x_mean = 1 x + 0 out, x = x_mean + 0 z, and the constraint's marginal 1 known + 0 z
  // and the multistep update's M = 0 x + 1 out without history terms
  const float* src[PC_TABLES] = {cfg->label, cfg->score_scale, cfg->alpha, cfg->pa, cfg->pb, cfg->pc, cfg->ca, cfg->cb, cfg->cc,
                                 cfg->cm, cfg->cs, cfg->mq, cfg->mr, cfg->pm1, cfg->pm2};
  const float dflt[PC_TABLES] = {0.f, 1.f, 1.f, 1.f, 0.f, 0.f, 1.f, 0.f, 0.f, 1.f, 0.f, 0.f, 1.f, 0.f, 0.f};
  for (int k = 0; k < PC_TABLES; ++k) {
    if (!pc_table_used(*cfg, k)) continue;
    pc->h_tab[k].assign(N, dflt[k]);
    if (src[k]) memcpy(pc->h_tab[k].data(), src[k], N * 4);
  }
  if (cfg->constraint) {
    memcpy(pc->color.M, cfg->color_m, sizeof(pc->color.M));
    memcpy(pc->color.Minv, cfg->color_minv, sizeof(pc->color.Minv));
  }
  pc->cfg.label = pc->cfg.score_scale = pc->cfg.alpha = pc->cfg.pa = pc->cfg.pb = pc->cfg.pc = nullptr;
  pc->cfg.ca = pc->cfg.cb = pc->cfg.cc = pc->cfg.cm = pc->cfg.cs = nullptr;
  pc->cfg.mq = pc->cfg.mr = pc->cfg.pm1 = pc->cfg.pm2 = nullptr;
  const long long cps = (cfg->corrector ? cfg->n_corrector_steps : 0) + (cfg->predictor ? 1 : 0);   // network evaluations
  const long long tail = cfg->constraint ? (cfg->predictor ? 1 : 0) + 2   /* predictor apply, two blends */
                                         : 1 /* predictor apply, or the x -> x_mean copy */;
  pc->launches_per_step = cps * model->launches + (cfg->corrector == 1 ? cfg->n_corrector_steps * 3 : cfg->corrector == 2 ? cfg->n_corrector_steps : 0) +
                          tail + 2;
  *out = pc;
  return 0;
}

void b200_pc_destroy(b200_pc_t* pc) { delete pc; }

long long b200_pc_workspace_bytes(const b200_pc_t* pc) {
  if (!pc) return -1;
  b200_pc tmp = *pc; tmp.gexec = nullptr; tmp.cap_stream = nullptr;
  return pc_ws_layout(&tmp, nullptr) + 512;
}

int b200_pc_bind_workspace(b200_pc_t* pc, void* ws, long long bytes, void* stream) {
  B200_REQUIRE(pc && ws, "pc_bind_workspace: null argument");
  char* base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~uintptr_t(255));
  const long long need = pc_ws_layout(pc, base) + (base - static_cast<char*>(ws));
  B200_REQUIRE(bytes >= need, "pc_bind_workspace: workspace too small (%lld < %lld)", bytes, need);
  pc->ws = base;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int N = pc->cfg.n_steps;
  for (int k = 0; k < PC_TABLES; ++k)
    if (pc->d_tab[k]) B200_CHECK_CUDA(cudaMemcpyAsync(pc->d_tab[k], pc->h_tab[k].data(), N * 4, cudaMemcpyHostToDevice, st));
  B200_CHECK_CUDA(cudaStreamSynchronize(st));
  if (pc->gexec) { cudaGraphExecDestroy(pc->gexec); pc->gexec = nullptr; }
  if (int r = philox_map_init(&pc->map, pc->numel, 0)) return r;
  const b200_ncsnpp_config& mc = pc->model->cfg;
  pc->map.nhwc = pc->cfg.noise_nhwc; pc->map.C = mc.num_channels; pc->map.HW = (long long)mc.image_size * mc.image_size;
  return 0;
}

int b200_pc_run(b200_pc_t* pc, float* x, float* x_mean, int first_step, int num_steps, unsigned long long seed,
                unsigned long long offset, unsigned long long* offset_out, int use_graph, void* stream) {
  B200_REQUIRE(pc && pc->ws && x, "pc_run: not bound");
  PdlScope pdl(pc->model->cfg.pdl != 0);
  B200_REQUIRE(first_step >= 0 && num_steps >= 0 && first_step + num_steps <= pc->cfg.n_steps,
               "pc_run: steps [%d,%d) outside the %d-step schedule", first_step, first_step + num_steps, pc->cfg.n_steps);
  B200_REQUIRE(!pc->cfg.constraint || (pc->known && pc->mask), "pc_run: constrained plan without b200_pc_bind_constraint");
  B200_REQUIRE(!pc->cfg.constraint || x_mean, "pc_run: a constrained plan needs x_mean");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  pc->map.seed = seed;
  // the noise offset of step s is *d_offset + (s*cps + call)*inc, so rebase for first_step
  const unsigned long long cps = pc_calls_per_step(pc->cfg);
  const unsigned long long base = offset - (unsigned long long)first_step * cps * pc->map.inc;
  B200_CHECK_CUDA(cudaMemcpyAsync(pc->d_offset, &base, 8, cudaMemcpyHostToDevice, st));
  B200_CHECK_CUDA(cudaMemcpyAsync(pc->d_step, &first_step, 4, cudaMemcpyHostToDevice, st));
  B200_CHECK_CUDA(cudaStreamSynchronize(st));   // host sources above are stack variables
  if (use_graph && num_steps > 0) {
    if (!pc->gexec || pc->graph_x != x || pc->graph_xm != x_mean || pc->graph_seed != seed || pc->graph_stream != st ||
        pc->graph_known != pc->known || pc->graph_mask != pc->mask) {
      if (pc->gexec) { cudaGraphExecDestroy(pc->gexec); pc->gexec = nullptr; }
      cudaGraph_t g = nullptr;
      if (!pc->cap_stream) B200_CHECK_CUDA(cudaStreamCreateWithFlags(&pc->cap_stream, cudaStreamNonBlocking));
      B200_CHECK_CUDA(cudaStreamBeginCapture(pc->cap_stream, cudaStreamCaptureModeThreadLocal));
      const int r = pc_iteration(pc, x, x_mean, nullptr, nullptr, pc->cap_stream);
      const cudaError_t ce = cudaStreamEndCapture(pc->cap_stream, &g);
      if (r) { if (g) cudaGraphDestroy(g); return r; }
      B200_CHECK_CUDA(ce);
      B200_CHECK_CUDA(cudaGraphInstantiate(&pc->gexec, g, 0));
      cudaGraphDestroy(g);
      pc->graph_x = x; pc->graph_xm = x_mean; pc->graph_stream = st; pc->graph_seed = seed;
      pc->graph_known = pc->known; pc->graph_mask = pc->mask;
    }
    for (int i = 0; i < num_steps; ++i) B200_CHECK_CUDA(cudaGraphLaunch(pc->gexec, st));
  } else {
    for (int i = 0; i < num_steps; ++i) if (int r = pc_iteration(pc, x, x_mean, nullptr, nullptr, st)) return r;
  }
  if (offset_out) *offset_out = offset + (unsigned long long)num_steps * cps * pc->map.inc;
  return 0;
}

int b200_pc_bind_constraint(b200_pc_t* pc, const float* known, const float* mask, void* stream) {
  (void)stream;
  B200_REQUIRE(pc && known && mask, "pc_bind_constraint: null argument");
  B200_REQUIRE(pc->cfg.constraint, "pc_bind_constraint: the plan was created with constraint = 0");
  pc->known = known; pc->mask = mask;   // a changed pointer re-captures the graph on the next b200_pc_run
  return 0;
}

int b200_pc_step_external(b200_pc_t* pc, float* x, float* x_mean, int step, const float* noise_c,
                          const float* noise_p, void* stream) {
  B200_REQUIRE(pc && pc->ws && x, "pc_step_external: not bound");
  B200_REQUIRE(!pc->cfg.constraint, "pc_step_external: not available for constrained (inpainting / colorization) plans; "
               "use b200_pc_run");
  PdlScope pdl(pc->model->cfg.pdl != 0);
  B200_REQUIRE(step >= 0 && step < pc->cfg.n_steps, "pc_step_external: step %d out of range", step);
  B200_REQUIRE(!pc->cfg.corrector || noise_c, "pc_step_external: corrector noise missing");
  B200_REQUIRE(pc->cfg.predictor != 1 || noise_p, "pc_step_external: predictor noise missing");
  B200_REQUIRE(pc->cfg.n_corrector_steps <= 1 || !pc->cfg.corrector, "pc_step_external: supports n_steps_each <= 1");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  B200_CHECK_CUDA(cudaMemcpyAsync(pc->d_step, &step, 4, cudaMemcpyHostToDevice, st));
  B200_CHECK_CUDA(cudaStreamSynchronize(st));
  return pc_iteration(pc, x, x_mean, noise_c, noise_p, st);
}

long long b200_pc_launches_per_step(const b200_pc_t* pc) { return pc ? pc->launches_per_step : 0; }

}  // extern "C"
