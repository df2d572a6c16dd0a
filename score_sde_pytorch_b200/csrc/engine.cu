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

namespace b200 {
void tc_gemm_set_rowvec_ld(TcGemmPlan* p, long long ld);
}
using namespace b200;

namespace {

// M_DOWN / M_UP: the DDPM family's Downsample / Upsample with_conv (layers.py:584-616)
enum ModKind { M_FOURIER, M_LINEAR, M_CONV_IN, M_RESBLOCK, M_ATTN, M_PYR_DOWN, M_GN_OUT, M_CONV_OUT, M_COMBINE, M_DOWN, M_UP };
enum PackKind { PK_COPY = 0, PK_CONV = 1, PK_NIN = 2, PK_CONV_FLAT32 = 3, PK_CONV_PAD128 = 4 };

struct Param {
  std::string name;
  int ndim; long long shape[4];
  long long off, count;      // location in the packed blob (floats)
  int pack, taps, O, I, round;
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
};

struct Tensor {
  float* p = nullptr; int C = 0, H = 0, W = 0; long long bytes = 0;
  double* qs = nullptr;   // GroupNorm quad sums [B][C/4][2]
  bool f16 = false;       // elements are IEEE fp16 (mid-block conv output in fp16 operand mode)
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

  const float* W(int pi) const { return wblob + params[pi].off; }
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
  if (fixed_off >= 0) p.off = fixed_off;
  else { p.off = e->wcount; e->wcount += (std::max(p.count, reserve) + 63) & ~63LL; }
  e->params.push_back(p);
  return (int)e->params.size() - 1;
}

// precision: 0 = tensor cores on TF32-grid fp32 operands, 1 = strict fp32 CUDA cores, 2 = tensor cores on fp16 operands
// (same 11-bit significand as TF32, fp32 accumulation; half the operand bytes and twice the MMA rate)
bool tc_ok(const b200_ncsnpp* e, int C1, int C2, int Cout, int H, int W, int taps) {
  if (e->cfg.precision == 1) return false;
  TcGemmDesc d; memset(&d, 0, sizeof(d));
  d.f16 = e->cfg.precision == 2;
  d.C1 = C1; d.C2 = C2; d.a2 = C2 ? (const float*)1 : nullptr; d.conv = 1; d.H = H; d.W = W; d.nimg = 1; d.taps = taps;
  d.N_total = Cout; d.K_total = C1 + C2; d.nbatch = 1; d.epi.ld_out = Cout; d.epi.ld_res = Cout;
  return tc_gemm_supported(d, nullptr);
}

int build_graph(b200_ncsnpp* e) {
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
  const int om = c.precision == 2 ? 2 : 1;      // operand store mode of tensor-core inputs (store_operand4)
  const int flatk = om == 2 ? 64 : 32;          // elements of one 128-byte K step (im2col contraction depth)
  std::vector<int> all_res(L);
  for (int i = 0; i < L; ++i) all_res[i] = c.image_size >> i;
  auto has_attn = [&](int r) { for (int i = 0; i < c.num_attn_resolutions; ++i) if (c.attn_resolutions[i] == r) return true; return false; };
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
    // fp16 operands: the logits/probabilities never leave the chip, so only the fused core is implemented
    if (om == 2 && !tc_attn_supported(T, C)) m.tcattn = false;
    // few tokens (T <= 64: the 4x4 block of CIFAR-10, the 8x8, 512-channel bottleneck of FFHQ-1024): one CTA per image
    // (attn_small_kernel); otherwise the block runs as separate contractions
    const bool small_ok = attn_small_supported(T, C);
    m.tc0 = tcmode && (C % 128 == 0) && (m.tcattn || small_ok);   // q/k/v projections on tensor cores
    m.gn0w = add_param(e, nm("GroupNorm_0.weight"), {C}, PK_COPY, 0, 0, 0, 0);
    m.gn0b = add_param(e, nm("GroupNorm_0.bias"), {C}, PK_COPY, 0, 0, 0, 0);
    // q,k,v projection weights packed as one [3C][C] block (rows: q, k, v), biases as one [3C] vector
    const long long wbase = e->wcount; e->wcount += 3LL * C * C;
    const long long bbase = e->wcount; e->wcount += (3LL * C + 63) & ~63LL;
    const bool tcproj = m.tc0;
    for (int k = 0; k < 3; ++k) {
      m.nw[k] = add_param(e, nmi(m.index, "NIN_" + std::to_string(k) + ".W"), {C, C}, PK_NIN, 1, C, C, tcproj ? om : 0,
                          wbase + (long long)k * C * C / ((tcproj && om == 2) ? 2 : 1));   // fp16: the three blocks stay contiguous as [3C][C] halves
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
      if (has_attn(all_res[lvl])) add_attn(in_ch, all_res[lvl]);
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
    if (has_attn(all_res[lvl])) add_attn(in_ch, all_res[lvl]);
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
    m.tc0 = !c.cuda_core_head && tcmode && ch <= 32 && tc_ok(e, in_ch, 0, 128, c.image_size, c.image_size, 9) && (c.image_size * c.image_size) % 256 == 0 &&
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
struct Builder {
  b200_ncsnpp* e; int B; char* base; bool dry; Arena arena; int rc = 0;
  char* stats_base = nullptr; long long stats_top = 0;   // bump region for GroupNorm quad sums, zeroed once per forward
  bool fused_stats = false;
  bool lowc_gn = false;                        // the few-channel convolutions (conv_lowc.cu, TF32 mode) apply GroupNorm+SiLU while staging their input
  int lane = 0;                                // which half-batch plan this builder fills (ops or ops2)
  int om = 1;                                  // operand store mode of tensor-core inputs: 1 TF32-grid fp32, 2 fp16
  std::string next_name;                       // label of the next op (shape summary for the per-op profile)
  double next_bytes = 0.0;                     // algorithmic HBM bytes of the next op
  void name(const char* fmt, ...) {
    char buf[160]; va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap); next_name = buf;
  }
  Builder(b200_ncsnpp* e_, int B_, char* base_, bool dry_, int lane_ = 0) : e(e_), B(B_), base(base_), dry(dry_), arena(e_->cfg.keep_activations != 0), lane(lane_) {
    fused_stats = e_->cfg.precision != 1;
    om = e_->cfg.precision == 2 ? 2 : 1;
    lowc_gn = e_->cfg.precision == 0 && e_->cfg.separate_groupnorm != 2;
    if (dry_) stats_base = reinterpret_cast<char*>(uintptr_t(1) << 40);   // any non-null base: only offsets matter in a dry run
  }
  double* qalloc(int C) {
    const long long bytes = ((long long)B * (C / 4) * 2 * 8 + 255) & ~255LL;
    double* p = reinterpret_cast<double*>(stats_base + stats_top);
    stats_top += bytes;
    return p;
  }

  Tensor talloc(int C, int H, int W) {
    Tensor t; t.C = C; t.H = H; t.W = W; t.bytes = (long long)B * H * W * C * 4;
    const long long off = arena.alloc(t.bytes); arena.note();
    t.p = reinterpret_cast<float*>(base + off);
    return t;
  }
  float* falloc(long long floats, long long* bytes_out) {
    *bytes_out = floats * 4;
    const long long off = arena.alloc(*bytes_out); arena.note();
    return reinterpret_cast<float*>(base + off);
  }
  void tfree(Tensor& t) { if (t.p) arena.release((char*)t.p - base, t.bytes); t.p = nullptr; }
  void ffree(float* p, long long bytes) { arena.release((char*)p - base, bytes); }

  // kind: 0 tensor-core contraction, 1 CUDA-core contraction, 2 GroupNorm, 3 FIR, 4 softmax, 5 time embedding, 6 misc
  void op(int launches, std::function<int(cudaStream_t)> f, int kind = 6, double flops = 0.0) {
    if (dry) return;
    e->launches += launches;
    static const char* kind_names[] = {"tensor-core contraction", "cuda-core contraction", "groupnorm", "fir", "softmax", "time embedding", "misc", "mma.sync contraction"};
    (lane ? e->ops2 : e->ops).push_back({kind, flops, std::move(f), next_name.empty() ? std::string(kind_names[kind & 7]) : next_name, next_bytes});
    next_name.clear(); next_bytes = 0.0;
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
  void gn(Tensor& x1, Tensor& x2, int pgw, int pgb, int act, int round, Tensor y, float* raw) {
    const int C = x1.C + x2.C, G = groups(C), HW = x1.H * x1.W;
    if ((C / G) % 4 != 0) {
      // groups that are not whole channel quads (C = 192 -> 6 channels per group): the generic two-kernel path
      if (x1.f16 || x2.f16) { set_error("ncsnpp: GroupNorm with %d-channel groups on an fp16 tensor", C / G); rc = 2; return; }
      long long mb; float* mr = falloc(gn_generic_workspace_floats(B, HW, G), &mb);
      const float *g = e->W(pgw), *bt = e->W(pgb);
      const Tensor a = x1, b = x2; const int Bc = B;
      name("gn_generic %d+%d @%d (%d-channel groups)", x1.C, x2.C, x1.H, C / G);
      op(3, [=](cudaStream_t st) { return launch_gn_generic(a.p, a.C, b.p, b.C, g, bt, Bc, HW, G, 1e-6f, act, round, y.p, raw, mr, st); }, 2);
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
  }

  // ---- GroupNorm coefficient tables for the few-channel convolutions that normalise while staging their input ----
  struct Coef { float* scale = nullptr; float* shift = nullptr; long long bytes = 0; };
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

  // 3x3 / 1x1 'same' convolution on NHWC tensors, stride 1.
  void conv(bool use_tc, Tensor a1, Tensor a2, int taps, int pw, int pb, int Cout, int dense_row /* -1 = none */,
            const float* residual, float scale, int round, Tensor& out, bool want_stats = false, int stride = 1,
            int Hin = 0, Tensor x3 = Tensor(), Tensor x4 = Tensor(), int pw2 = -1, int pb2 = -1, const Coef* gnc = nullptr) {
    Epilogue ep; memset(&ep, 0, sizeof(ep));
    ep.bias = e->W(pb);
    ep.rowvec = nullptr;   // patched at launch (depends on the per-call buffers)
    ep.residual = residual; ep.ld_res = Cout; ep.scale = scale; ep.round_tf32 = round;
    ep.rows_per_img = out.H * out.W; ep.out = out.p; ep.ld_out = Cout;
    b200_ncsnpp* eng = e;
    const float* dense_all = dense_all_;
    const int sumC = e->sumC;
    const double cflops = 2.0 * B * out.H * out.W * (double)Cout * ((a1.C + a2.C) * taps + x3.C + x4.C);
    if (x3.p && !use_tc) { set_error("ncsnpp: fused skip projection needs the tensor-core path"); rc = 2; return; }
    if (gnc && use_tc) { set_error("ncsnpp: conv(): GroupNorm coefficients go with the few-channel kernel (the tensor-core path reads normalised operands)"); rc = 2; return; }
    if (use_tc) {
      TcGemmDesc d; memset(&d, 0, sizeof(d));
      d.a1 = a1.p; d.C1 = a1.C; d.a2 = a2.p; d.C2 = a2.C; d.conv = 1; d.H = out.H; d.W = out.W; d.nimg = B; d.taps = taps;
      d.stride = stride; d.valid_pad = stride == 2 ? 1 : 0; d.Hin = Hin ? Hin : out.H; d.Win = Hin ? Hin : out.W;
      d.w = e->W(pw); d.N_total = Cout; d.K_total = a1.C + a2.C; d.w_rows = (long long)taps * Cout; d.nbatch = 1;
      d.f16 = om == 2; d.no_halo = e->cfg.no_halo;
      if (dense_row >= 0) ep.rowvec = dense_all + dense_row;
      if (x3.p) {   // fused skip projection: its bias rides in the (image-independent) row-vector slot
        if (dense_row >= 0) { set_error("ncsnpp: fused skip projection on a conv with a time-embedding bias"); rc = 2; return; }
        d.a3 = x3.p; d.C3 = x3.C; d.a4 = x4.p; d.C4 = x4.C; d.w2 = e->W(pw2);
        ep.rowvec = e->W(pb2); ep.rowvec_ld = 0;
      }
      if (want_stats && fused_stats && (ep.rows_per_img % 32 == 0 || ep.rows_per_img == 16)) { out.qs = qalloc(Cout); d.qstats = out.qs; }
      d.epi = ep;
      if (dry) return;
      TcGemmPlan* pl = nullptr;
      if (int r = tc_gemm_plan_create(d, &pl)) { rc = r; return; }
      e->tcplans.push_back(pl);
      name("conv%s %d+%d->%d @%d%s%s%s [%s]", taps == 9 ? "3x3" : "1x1", a1.C, a2.C, Cout, out.H, stride == 2 ? " s2" : "",
           x3.p ? " +skipproj" : "", residual ? " +res" : "", tc_gemm_form(pl));
      if (x3.p) next_name += " " + std::to_string(x3.C + x4.C);
      {
        const double es = om == 2 ? 2.0 : 4.0, px = (double)B * out.H * out.W;
        const double in_px = (double)B * (Hin ? (double)Hin * Hin : (double)out.H * out.W);
        next_bytes = in_px * (a1.C + a2.C) * es + px * (x3.C + x4.C) * es + px * Cout * (round == 2 ? 2.0 : 4.0) +
                     (residual ? px * Cout * 4.0 : 0.0) + ((double)taps * (a1.C + a2.C) + x3.C + x4.C) * Cout * es;
      }
      op(1, [=](cudaStream_t st) {
        if (dense_row >= 0) tc_gemm_set_rowvec_ld(pl, eng->uniform ? 0 : sumC);
        return tc_gemm_launch(pl, st);
      }, 0, cflops);
    } else {
      SimtConv s; memset(&s, 0, sizeof(s));
      s.x1 = a1.p; s.C1 = a1.C; s.x2 = a2.p; s.C2 = a2.C; s.in_scale = 1.f; s.in_shift = 0.f;
      s.H = a1.H; s.W = a1.W; s.R = s.S = (taps == 9 ? 3 : 1); s.stride = 1; s.pad = (taps == 9 ? 1 : 0);
      s.OH = a1.H; s.OW = a1.W; s.nbatch = B; s.a_batched = 1; s.w = e->W(pw); s.N = Cout;
      if (dense_row >= 0) ep.rowvec = dense_all + dense_row;
      s.epi = ep;
      // few-channel levels of the nf = 16 networks: warp-level TF32 MMAs keep them at the HBM roofline (conv_lowc.cu);
      // strict-fp32 mode and every other shape stay on the CUDA-core kernel
      const bool lowc = e->cfg.precision != 1 && !a1.f16 && !a2.f16 && sumC % 2 == 0 && conv_lowc_supported(s);
      if (want_stats && lowc && fused_stats) { out.qs = qalloc(Cout); s.qstats = out.qs; }   // the epilogue sums what the next GroupNorm needs
      if (gnc) {
        if (!lowc) { set_error("ncsnpp: GroupNorm on load planned for a convolution the few-channel kernel does not take"); rc = 2; return; }
        s.gn_scale = gnc->scale; s.gn_shift = gnc->shift; s.gn_act = 1;
      }
      name("conv%s %s%d+%d->%d @%d [%s]", taps == 9 ? "3x3" : "1x1", gnc ? "gn+silu " : "", a1.C, a2.C, Cout, out.H, lowc ? "mma.sync tf32" : "cuda-core");
      next_bytes = (double)B * out.H * out.W * ((a1.C + a2.C) * 4.0 + Cout * 4.0 + (residual ? Cout * 4.0 : 0.0)) +
                   (double)taps * (a1.C + a2.C) * Cout * 4.0;
      op(1, [=](cudaStream_t st) {
        SimtConv c = s;
        if (dense_row >= 0) c.epi.rowvec_ld = eng->uniform ? 0 : sumC;
        return lowc ? launch_conv_lowc(c, st) : launch_conv_simt(c, st);
      }, lowc ? 7 : 1, cflops);
    }
  }

  // batched C[b] = A[b] * W[b]^T
  void gemm(bool use_tc, const float* A, long long lda, long long a_rows, int a_batch_rows, const float* Wm, long long ldw,
            long long w_rows, int w_batch_rows, int nbatch, int M, int N, int K, const float* bias,
            const float* residual, long long ld_res, float scale, int round, float* out, long long ldo,
            double* qstats = nullptr, int rows_per_img = 1 << 30) {
    Epilogue ep; memset(&ep, 0, sizeof(ep));
    ep.bias = bias; ep.residual = residual; ep.ld_res = ld_res; ep.scale = scale; ep.round_tf32 = round;
    ep.rows_per_img = rows_per_img; ep.out = out; ep.ld_out = ldo;
    if (use_tc) {
      TcGemmDesc d; memset(&d, 0, sizeof(d));
      d.a1 = A; d.C1 = K; d.conv = 0; d.taps = 1; d.a_rows = a_rows; d.a_ld = lda; d.a_batch_rows = a_batch_rows;
      d.w = Wm; d.N_total = N; d.K_total = K; d.w_rows = w_rows; d.w_ld = ldw; d.w_batch_rows = w_batch_rows;
      d.nbatch = nbatch; d.M_per_batch = M; d.qstats = qstats; d.epi = ep;
      d.f16 = om == 2;
      if (dry) return;
      TcGemmPlan* pl = nullptr;
      if (int r = tc_gemm_plan_create(d, &pl)) { rc = r; return; }
      e->tcplans.push_back(pl);
      name("gemm %dx(%dx%dx%d)%s [%s]", nbatch, M, N, K, residual ? " +res" : "", tc_gemm_form(pl));
      {
        const double es = om == 2 ? 2.0 : 4.0;
        next_bytes = (double)(a_batch_rows ? nbatch : 1) * M * K * es + (double)(w_batch_rows ? nbatch : 1) * N * K * es +
                     (double)nbatch * M * N * (round == 2 ? 2.0 : 4.0) + (residual ? (double)nbatch * M * N * 4.0 : 0.0);
      }
      op(1, [=](cudaStream_t st) { return tc_gemm_launch(pl, st); }, 0, 2.0 * nbatch * (double)M * N * K);
    } else {
      SimtConv s; memset(&s, 0, sizeof(s));
      s.x1 = A; s.C1 = K; s.ld1 = lda; s.in_scale = 1.f; s.H = M; s.W = 1; s.R = s.S = 1; s.stride = 1; s.pad = 0;
      s.OH = M; s.OW = 1; s.nbatch = nbatch; s.a_batched = a_batch_rows != 0; s.w = Wm; s.N = N;
      s.w_batch_stride = (long long)w_batch_rows * ldw; s.w_ld = ldw;
      ep.rows_per_img = M; s.epi = ep;
      op(1, [=](cudaStream_t st) { return launch_conv_simt(s, st); }, 1, 2.0 * nbatch * (double)M * N * K);
    }
  }

  const float* dense_all_ = nullptr;
  void tap(int idx, const Tensor& t) { if (!dry) e->taps[idx] = t; }

  // would conv() run this stride-1 convolution on the few-channel kernel (conv_lowc.cu: TF32 mode, fp32 tensors)?
  bool lowc_ok(int C1, int C2, int Cout, int H, int taps) const {
    if (e->cfg.precision != 0 || e->sumC % 2 != 0) return false;
    SimtConv s; memset(&s, 0, sizeof(s));
    s.C1 = C1; s.C2 = C2; s.in_scale = 1.f; s.H = H; s.W = H; s.R = s.S = (taps == 9 ? 3 : 1); s.stride = 1; s.pad = (taps == 9 ? 1 : 0);
    s.OH = H; s.OW = H; s.nbatch = B; s.a_batched = 1; s.N = Cout; s.epi.ld_out = Cout; s.epi.ld_res = Cout;
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
      gn(x1, x2, m.gn0w, m.gn0b, 1, (m.tc0 && !resample) ? om : 0, a0, raw.p);
    }
    Tensor xr;
    if (resample) {
      if (x2.p) { set_error("ncsnpp: resampling block with a two-source input"); rc = 2; return Tensor(); }
      Tensor a0r = talloc(Cin, Ho, Ho);
      xr = talloc(Cin, Ho, Ho);
      xr.f16 = m.tc2 && om == 2;
      resample2x(a0.p, H, Cin, m.up != 0, m.tc0 ? om : 0, a0r.p);
      resample2x(x1.p, H, Cin, m.up != 0, m.tc2 ? om : 0, xr.p);
      tfree(a0); a0 = a0r;
    }
    Tensor h1 = talloc(m.cout, Ho, Ho);
    // fp16 operand mode: the mid-block tensor (Conv_0 output, only ever read by GroupNorm_1) is stored as fp16;
    // its GroupNorm sums are accumulated from the fp32 accumulators in the epilogue.
    h1.f16 = h1_f16;
    if (lc0) {
      Coef c0 = gncoef(x1, x2, m.gn0w, m.gn0b);
      conv(false, x1, x2, 9, m.c0w, m.c0b, m.cout, m.dense_row, nullptr, 1.f, 0, h1, /*want_stats=*/true, 1, 0, Tensor(), Tensor(), -1, -1, &c0);
      ffree(c0.scale, c0.bytes);
    } else {
      conv(m.tc0, a0, Tensor(), 9, m.c0w, m.c0b, m.cout, m.dense_row, nullptr, 1.f, h1_f16 ? 2 : 0, h1, /*want_stats=*/true);
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
    const float* residual = x1.p;
    // Fused skip projection (default): Conv_2(x) (layerspp.py:270) is accumulated inside the second 3x3 convolution
    // as extra K steps instead of a separate launch + a residual round trip through HBM.
    if (m.has_conv2 && m.tc1 && m.tc2 && (resample || raw.p)) {
      Tensor out = talloc(m.cout, Ho, Ho);
      Tensor e1 = resample ? xr : raw, e2 = Tensor();
      e1.f16 = false;   // conv() addresses operands by the engine-wide operand mode
      conv(true, a1, Tensor(), 9, m.c1w, m.c1b, m.cout, -1, nullptr, inv_s2, 0, out, /*want_stats=*/true, 1, 0, e1, e2, m.c2w, m.c2b);
      tfree(a1); tfree(raw); tfree(xr);
      return out;
    }
    if (m.has_conv2) {
      s = talloc(m.cout, Ho, Ho);
      if (resample) conv(m.tc2, xr, Tensor(), 1, m.c2w, m.c2b, m.cout, -1, nullptr, 1.f, 0, s);
      else if (m.tc2 && raw.p) conv(true, raw, Tensor(), 1, m.c2w, m.c2b, m.cout, -1, nullptr, 1.f, 0, s);
      else if (m.tc2) conv(true, x1, x2, 1, m.c2w, m.c2b, m.cout, -1, nullptr, 1.f, 0, s);
      else conv(false, x1, x2, 1, m.c2w, m.c2b, m.cout, -1, nullptr, 1.f, 0, s);
      residual = s.p;
      tfree(raw); tfree(xr);
    } else if (x2.p) { set_error("ncsnpp: concat input without a skip convolution"); rc = 2; return Tensor(); }
    Tensor out = talloc(m.cout, Ho, Ho);
    if (lc1) {
      conv(false, h1, Tensor(), 9, m.c1w, m.c1b, m.cout, -1, residual, inv_s2, 0, out, /*want_stats=*/true, 1, 0, Tensor(), Tensor(), -1, -1, &c1);
      ffree(c1.scale, c1.bytes); tfree(h1);
    } else {
      conv(m.tc1, a1, Tensor(), 9, m.c1w, m.c1b, m.cout, -1, residual, inv_s2, 0, out, /*want_stats=*/true);
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
      float* qk = falloc((long long)B * T * 2 * C, &qkb);
      float* vT = falloc((long long)B * C * T, &vtb);
      // q,k = a Wq^T + bq | a Wk^T + bk   (layerspp.py:78-79) in one N=2C contraction
      gemm(tc, a.p, C, BT, 0 /* rows enumerated flat */, Wqkv, C, 2LL * C, 0, 1, (int)BT, 2 * C, C, bqkv, nullptr, 0, 1.f, tc ? om : 0, qk, 2 * C);
      // v^T[b][c][t] = sum_i Wv[c][i] a[b][t][i]   (bias bv is added after the PV product: softmax rows sum to 1)
      gemm(tc, wv, C, C, 0, a.p, C, BT, T, B, C, T, C, nullptr, nullptr, 0, 1.f, tc ? om : 0, vT, T, nullptr, 1 << 30);
      tfree(a);
      // Fused core (default): logits, softmax, P.V, NIN_3, residual, rescale and quad sums in one kernel; the
      // [T,T] logits/probabilities and the attention output stay on chip; other token counts (tf32 mode) use separate launches.
      if (om == 2 && !(tc && m.tc2 && tc_attn_supported(T, C))) {
        set_error("ncsnpp: fp16 operand mode needs the fused attention core (T=%d C=%d)", T, C); rc = 2; return Tensor();
      }
      if (tc && m.tc2 && tc_attn_supported(T, C)) {
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
      float* S = falloc(BT * T, &sb);
      // logits[b][q][k] = q . k   (layerspp.py:82), scaled inside the softmax
      gemm(tc, qk, 2 * C, BT, T, qk + C, 2 * C, BT, T, B, T, T, C, nullptr, nullptr, 0, 1.f, 0, S, T, nullptr, 1 << 30);
      ffree(qk, qkb);
      name("softmax T=%d", T);
      op(1, [=](cudaStream_t st) { return launch_softmax_rows(S, S, (long long)Bc * T, T, sc, tc ? 1 : 0, st); }, 4);
      O = falloc(BT * C, &ob);
      // h[b][q][c] = sum_k P[q][k] v[k][c] + bv[c]   (layerspp.py:86)
      gemm(tc, S, T, BT, T, vT, T, (long long)B * C, C, B, T, C, T, bqkv + 2 * C, nullptr, 0, 1.f, m.tc2 ? 1 : 0, O, C);
      ffree(S, sb); ffree(vT, vtb);
    }
    Tensor out = talloc(C, x.H, x.W);
    Tensor Ot; Ot.p = O; Ot.C = C; Ot.H = x.H; Ot.W = x.W;
    conv(m.tc2, Ot, Tensor(), 1, m.nw[3], m.nb[3], C, -1, x.p, inv_s2, 0, out, /*want_stats=*/true);   // NIN_3 + (x+h)/sqrt2 (:87-91)
    ffree(O, ob);
    return out;
  }

  // DDPM Downsample(with_conv) (layers.py:599-616): F.pad(x, (0,1,0,1)) then a 3x3 stride-2 VALID convolution.  The
  // convolution reads the unpadded input: the taps of the last output row / column that fall on row / column H are the
  // padding zeros (TMA's out-of-bounds fill on the tensor cores, the bounds check of the CUDA-core kernel otherwise).
  Tensor downsample(const Mod& m, Tensor& x) {
    const int H = x.H, Ho = H / 2;
    Tensor out = talloc(m.cout, Ho, Ho);
    if (m.tc0) {
      // the block output is fp32; the tensor cores read it in the operand format (TF32 grid / fp16)
      Tensor xo = talloc(x.C, H, H);
      const float* src = x.p; float* dst = xo.p; const long long n = (long long)B * H * H * x.C; const int omc = om;
      name("operand copy %d @%d", x.C, H);
      next_bytes = (double)n * (4.0 + (om == 2 ? 2.0 : 4.0));
      op(1, [=](cudaStream_t st) { return launch_store_operand(src, dst, n, omc, st); }, 6);
      conv(true, xo, Tensor(), 9, m.w, m.b, m.cout, -1, nullptr, 1.f, 0, out, /*want_stats=*/true, /*stride=*/2, /*Hin=*/H);
      tfree(xo);
    } else {
      SimtConv s; memset(&s, 0, sizeof(s));
      s.x1 = x.p; s.C1 = x.C; s.in_scale = 1.f; s.H = H; s.W = H; s.R = s.S = 3; s.stride = 2; s.pad = 0;
      s.OH = Ho; s.OW = Ho; s.nbatch = B; s.a_batched = 1; s.w = e->W(m.w); s.N = m.cout;
      s.epi.bias = e->W(m.b); s.epi.scale = 1.f; s.epi.rows_per_img = Ho * Ho; s.epi.out = out.p; s.epi.ld_out = m.cout;
      name("conv3x3 s2 %d->%d @%d [cuda-core]", x.C, m.cout, Ho);
      op(1, [=](cudaStream_t st) { return launch_conv_simt(s, st); }, 1, 2.0 * B * Ho * Ho * (double)m.cout * x.C * 9);
    }
    return out;
  }

  // DDPM Upsample(with_conv) (layers.py:584-596): nearest 2x (the 2x2 box upfirdn2d, written in the convolution's operand
  // format) then a 3x3 'same' convolution
  Tensor upsample(const Mod& m, Tensor& x) {
    const int H = x.H, Ho = 2 * H;
    Tensor u = talloc(x.C, Ho, Ho);
    fir(x.p, B, H, H, x.C, 2, 1, 1, 0, m.tc0 ? om : 0, u.p, 1.f, /*box=*/true);
    Tensor out = talloc(m.cout, Ho, Ho);
    conv(m.tc0, u, Tensor(), 9, m.w, m.b, m.cout, -1, nullptr, 1.f, 0, out, /*want_stats=*/true);
    tfree(u);
    return out;
  }

  int build() {
    const b200_ncsnpp_config& c = e->cfg;
    const int nf = c.nf, R = c.image_size, ch = c.num_channels, sumC = e->sumC;
    b200_ncsnpp* eng = e;
    const int Bc = B;
    const int ln = lane;
    // ---- time embedding (ncsnpp.py:236-255) + all Dense_0(act(temb)) rows (layerspp.py:263) ----
    long long eb, t1b, t2b, db, xcb;
    const int positional = c.embedding_type == 1 ? 1 : 0, emb_dim = positional ? nf : 2 * nf;
    float* emb = falloc((long long)B * 2 * nf, &eb);
    float* t1 = falloc((long long)B * 4 * nf, &t1b);
    float* t2 = falloc((long long)B * 4 * nf, &t2b);
    float* dense_all = falloc((long long)B * sumC, &db);
    dense_all_ = dense_all;
    {
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
    // ---- input (ncsnpp.py:259-268) ----
    float* xc = falloc((long long)B * ch * R * R, &xcb);   // 2x-1 when data is not centred; NCHW
    {
      const long long n = (long long)B * ch * R * R;
      const int centered = c.centered;
      op(1, [=](cudaStream_t st) {
        if (centered) return cudaMemcpyAsync(xc, eng->in_x_l[ln], n * 4, cudaMemcpyDeviceToDevice, st) == cudaSuccess ? 0 : (set_error("memcpy failed"), 1);
        launch_kernel(affine_kernel, dim3((int)std::min<long long>((n + 255) / 256, 4096)), dim3(256), 0, st, eng->in_x_l[ln], xc, n, -0.5f, 2.0f);
        return cudaGetLastError() == cudaSuccess ? 0 : (set_error("affine launch failed"), 1);
      });
    }
    size_t mi = 3;
    std::vector<Tensor> hs;
    {
      const Mod& m = e->mods[mi++];
      Tensor h0 = talloc(nf, R, R);
      if (m.tc0 || m.tc1) {
        // im2col patches [B*R*R][32] (TF32 grid) then one K=32 contraction with the flat-packed weights (tensor cores, or the
        // few-channel kernel for nf <= 64)
        long long pb; float* patches = falloc((long long)B * R * R * 32, &pb);   // 128 B per pixel: 32 fp32 or 64 fp16
        const int Bc = B, omc = om;
        name("im2col 3x3 %d @%d", ch, R);
        op(1, [=](cudaStream_t st) { return launch_im2col3x3_nchw(xc, patches, Bc, ch, R, R, R, R, 1, 1, omc, st); }, 6);
        Tensor pt; pt.p = patches; pt.C = om == 2 ? 64 : 32; pt.H = R; pt.W = R;   // patches as a one-K-step NHWC image: a 1x1 conv
        conv(m.tc0, pt, Tensor(), 1, m.w, m.b, nf, -1, nullptr, 1.f, 0, h0, /*want_stats=*/true);
        ffree(patches, pb);
      } else {
        SimtConv s; memset(&s, 0, sizeof(s));
        s.x1 = xc; s.C1 = ch; s.in_nchw = 1; s.in_scale = 1.f; s.H = R; s.W = R; s.R = s.S = 3; s.stride = 1; s.pad = 1;
        s.OH = R; s.OW = R; s.nbatch = B; s.a_batched = 1; s.w = e->W(m.w); s.N = nf;
        s.epi.bias = e->W(m.b); s.epi.scale = 1.f; s.epi.rows_per_img = R * R; s.epi.out = h0.p; s.epi.ld_out = nf;
        op(1, [=](cudaStream_t st) { return launch_conv_simt(s, st); }, 1, 2.0 * B * R * R * (double)nf * ch * 9);
      }
      hs.push_back(h0);
      tap(m.index, h0);
    }
    // input pyramid (progressive_input='residual', ncsnpp.py:289-301): starts as the network input
    Tensor pyr; pyr.p = xc; pyr.C = ch; pyr.H = R; pyr.W = R; bool pyr_nchw = true; bool pyr_owned = false; long long pyr_bytes = 0;
    const int L = c.num_levels;
    for (int lvl = 0; lvl < L; ++lvl) {
      for (int b = 0; b < c.num_res_blocks; ++b) {
        const Mod& m = e->mods[mi++];
        Tensor none; Tensor h = resblock(m, hs.back(), none); if (rc) return rc;
        tap(m.index, h);
        if (mi < e->mods.size() && e->mods[mi].kind == M_ATTN && e->mods[mi].res == h.H && lvl_has_attn(h.H)) {
          const Mod& ma = e->mods[mi++];
          Tensor h2 = attn(ma, h); if (rc) return rc;
          tfree(h); h = h2; tap(ma.index, h);
        }
        hs.push_back(h);
      }
      if (lvl != L - 1) {
        const Mod& m = e->mods[mi++];
        Tensor none; Tensor h = m.kind == M_DOWN ? downsample(m, hs.back()) : resblock(m, hs.back(), none); if (rc) return rc;
        tap(m.index, h);
        if (c.progressive_input == 2) {
          // input_skip (ncsnpp.py:289-292): the image pyramid is downsampled (no parameters) and a 1x1 convolution of it is
          // added to h: Combine(method='sum') (layerspp.py:44-59)
          const Mod& mc = e->mods[mi++];
          const int Hin = pyr.H, Hn = Hin / 2;
          long long nb; float* npyr = falloc((long long)B * ch * Hn * Hn, &nb);
          resample2x_planes(pyr.p, B * ch, Hin, false, npyr);
          if (pyr_owned) ffree(pyr.p, pyr_bytes);
          pyr.p = npyr; pyr.H = pyr.W = Hn; pyr_owned = true; pyr_bytes = nb;
          if (Hn != h.H) { set_error("ncsnpp: input pyramid geometry mismatch (%d vs %d)", Hn, h.H); return 2; }
          Tensor out = talloc(mc.cout, h.H, h.W);
          SimtConv sc; memset(&sc, 0, sizeof(sc));
          sc.x1 = npyr; sc.C1 = ch; sc.in_nchw = 1; sc.in_scale = 1.f; sc.H = Hn; sc.W = Hn; sc.R = sc.S = 1; sc.stride = 1; sc.pad = 0;
          sc.OH = Hn; sc.OW = Hn; sc.nbatch = B; sc.a_batched = 1; sc.w = e->W(mc.w); sc.N = mc.cout;
          sc.epi.bias = e->W(mc.b); sc.epi.residual = h.p; sc.epi.ld_res = mc.cout; sc.epi.scale = 1.f;
          sc.epi.rows_per_img = Hn * Hn; sc.epi.out = out.p; sc.epi.ld_out = mc.cout;
          name("combine sum: conv1x1 %d->%d @%d +h [cuda-core]", ch, mc.cout, Hn);
          op(1, [=](cudaStream_t st) { return launch_conv_simt(sc, st); }, 1, 2.0 * B * Hn * Hn * (double)mc.cout * ch);
          tfree(h);
          h = out; tap(mc.index, h);
        }
        if (c.progressive_input == 1) {
          const Mod& mp = e->mods[mi++];
          // Downsample(fir, with_conv): FIR with pad (2,2) then 3x3 stride-2 VALID conv + bias
          // (up_or_down_sampling.py:170-178, Conv2d.forward :44-56), then (pyr + h)/sqrt2 (ncsnpp.py:297-301)
          const int Hin = pyr.H, p = (e->firn - 2) + 2;
          const int Hp = Hin + ((p + 1) / 2) + (p / 2) - e->firn + 1;
          long long fb; float* fbuf = falloc((long long)B * pyr.C * Hp * Hp, &fb);
          const bool tcp = mp.tc0 && !pyr_nchw;
          const bool flat = mp.tc2 && pyr_nchw;
          if (pyr_nchw) fir(pyr.p, B * pyr.C, Hin, Hin, 1, 1, 1, (p + 1) / 2, p / 2, 0, fbuf, 1.f);
          else fir(pyr.p, B, Hin, Hin, pyr.C, 1, 1, (p + 1) / 2, p / 2, tcp ? om : 0, fbuf, 1.f);
          Tensor np = talloc(mp.cout, h.H, h.W);
          if ((Hp - 3) / 2 + 1 != h.H) { set_error("ncsnpp: pyramid geometry mismatch (%d vs %d)", (Hp - 3) / 2 + 1, h.H); return 2; }
          const float ps = c.skip_rescale ? 1.0f / (float)std::sqrt(2.0) : 1.0f;
          if (flat) {
            long long pb2; float* patches = falloc((long long)B * h.H * h.W * 32, &pb2);
            const int Bc = B, pc = pyr.C, oh = h.H, ow = h.W, omc = om;
            name("im2col 3x3 s2 %d @%d", pc, oh);
            op(1, [=](cudaStream_t st) { return launch_im2col3x3_nchw(fbuf, patches, Bc, pc, Hp, Hp, oh, ow, 2, 0, omc, st); }, 6);
            Tensor pt; pt.p = patches; pt.C = om == 2 ? 64 : 32; pt.H = h.H; pt.W = h.W;
            conv(true, pt, Tensor(), 1, mp.w, mp.b, mp.cout, -1, h.p, ps, 0, np, /*want_stats=*/true);
            ffree(patches, pb2);
          } else if (tcp) {
            Tensor fin; fin.p = fbuf; fin.C = pyr.C; fin.H = Hp; fin.W = Hp;
            conv(true, fin, Tensor(), 9, mp.w, mp.b, mp.cout, -1, h.p, ps, 0, np, /*want_stats=*/true, /*stride=*/2, /*Hin=*/Hp);
          } else {
            SimtConv s; memset(&s, 0, sizeof(s));
            s.x1 = fbuf; s.C1 = pyr.C; s.in_nchw = pyr_nchw ? 1 : 0; s.in_scale = 1.f; s.H = Hp; s.W = Hp; s.R = s.S = 3; s.stride = 2; s.pad = 0;
            s.OH = h.H; s.OW = h.W; s.nbatch = B; s.a_batched = 1; s.w = e->W(mp.w); s.N = mp.cout;
            s.epi.bias = e->W(mp.b); s.epi.residual = h.p; s.epi.ld_res = mp.cout; s.epi.scale = ps;
            s.epi.rows_per_img = h.H * h.W; s.epi.out = np.p; s.epi.ld_out = mp.cout;
            op(1, [=](cudaStream_t st) { return launch_conv_simt(s, st); }, 1, 2.0 * B * h.H * h.W * (double)mp.cout * pyr.C * 9);
          }
          ffree(fbuf, fb);
          if (pyr_owned) tfree(pyr);
          tfree(h);
          h = np; pyr = np; pyr_nchw = false; pyr_owned = false;   // h aliases the pyramid from here on (it lives in hs)
          // (no debug tap: the reference module's own output is the pre-combine conv result, which is never materialised)
        }
        hs.push_back(h);
      }
    }
    // ---- middle (ncsnpp.py:305-311) ----
    Tensor h;
    {
      Tensor none; const Mod& m0 = e->mods[mi++]; h = resblock(m0, hs.back(), none); if (rc) return rc; tap(m0.index, h);
      const Mod& ma = e->mods[mi++]; Tensor h2 = attn(ma, h); if (rc) return rc; tfree(h); h = h2; tap(ma.index, h);
      const Mod& m1 = e->mods[mi++]; Tensor h3 = resblock(m1, h, none); if (rc) return rc; tfree(h); h = h3; tap(m1.index, h);
    }
    // ---- up path (ncsnpp.py:316-364) ----
    float* opyr = nullptr; long long opyr_bytes = 0;      // output_skip pyramid [B][ch][H][W] of the previous (coarser) level
    for (int lvl = L - 1; lvl >= 0; --lvl) {
      for (int b = 0; b < c.num_res_blocks + 1; ++b) {
        const Mod& m = e->mods[mi++];
        Tensor skip = hs.back(); hs.pop_back();
        Tensor h2 = resblock(m, h, skip); if (rc) return rc;
        tfree(h); tfree(skip);
        h = h2; tap(m.index, h);
      }
      if (e->mods[mi].kind == M_ATTN) {
        const Mod& ma = e->mods[mi++]; Tensor h2 = attn(ma, h); if (rc) return rc; tfree(h); h = h2; tap(ma.index, h);
      }
      if (c.progressive == 1) {
        // output_skip (ncsnpp.py:325-341): pyramid = upsample(pyramid) + conv3x3(SiLU(GroupNorm(h))) in image channels;
        // the level-0 sum is the network output (divided by sigma when scale_by_sigma, :377-379)
        const Mod& mg = e->mods[mi++]; const Mod& mo = e->mods[mi++];
        const int Hl = h.H;
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
        if (lvl != 0) dst = falloc((long long)B * ch * Hl * Hl, &nb);
        const float *wo = e->W(mo.w), *bo = e->W(mo.b);
        const Tensor ain = a; const int Bc2 = B, sbs = c.scale_by_sigma, last = lvl == 0;
        if (ch > 4) { set_error("ncsnpp: output_skip needs <= 4 image channels"); return 2; }
        name("conv3x3 %d->%d @%d nchw-out +pyramid [small-n]", a.C, ch, Hl);
        op(1, [=](cudaStream_t st) {
          return launch_conv3x3_small_n(ain.p, wo, bo, (last && sbs) ? eng->in_labels_l[ln] : nullptr, eng->uniform ? 0 : 1,
                                        last ? eng->out_l[ln] : dst, Bc2, Hl, Hl, ain.C, ch, hf16, st, up);
        }, 1, 2.0 * B * Hl * Hl * (double)ch * a.C * 9);
        tfree(a);
        if (up) ffree(up, ub);
        opyr = dst; opyr_bytes = nb;
      }
      if (lvl != 0) {
        Tensor none; const Mod& m = e->mods[mi++];
        Tensor h2 = m.kind == M_UP ? upsample(m, h) : resblock(m, h, none); if (rc) return rc;
        tfree(h); h = h2; tap(m.index, h);
      }
    }
    // ---- output head (ncsnpp.py:371-379); with output_skip the pyramid already is the output ----
    if (c.progressive != 1) {
      const Mod& mg = e->mods[mi++];
      Tensor a = talloc(h.C, h.H, h.W);
      // fp16 operand mode: the head's input is stored as fp16 too (the CUDA-core head is bound by its nine-fold
      // tap re-reads through L1/L2, so half the bytes is half the time); same 11-bit rounding as every other conv input
      const Mod& mo = e->mods[mi];
      const int head_f16 = (!mo.tc0 && om == 2 && ch <= 4 && h.C % 64 == 0) ? 1 : 0;
      Tensor none; gn(h, none, mg.w, mg.b, 1, mo.tc0 ? om : head_f16 ? 2 : 0, a, nullptr);
      tfree(h);
      ++mi;
      const int sbs = c.scale_by_sigma;
      const float *wo = e->W(mo.w), *bo = e->W(mo.b);
      const Tensor ain = a; const int Bc = B;
      if (mo.tc0) {
        TcGemmDesc d; memset(&d, 0, sizeof(d));
        d.a1 = a.p; d.C1 = a.C; d.conv = 1; d.H = R; d.W = R; d.nimg = B; d.taps = 9; d.stride = 1;
        d.w = wo; d.N_total = 128; d.K_total = a.C; d.w_rows = 9LL * 128; d.nbatch = 1; d.f16 = om == 2; d.no_halo = e->cfg.no_halo;
        d.epi.bias = bo; d.epi.scale = 1.f; d.epi.rows_per_img = R * R; d.epi.out_nchw = 1; d.epi.n_valid = ch; d.epi.ld_out = 128;
        d.epi.out = reinterpret_cast<float*>(uintptr_t(16));   // patched per call (tc_gemm_set_head)
        if (!dry) {
          TcGemmPlan* pl = nullptr;
          if (int r = tc_gemm_plan_create(d, &pl)) { rc = r; return r; }
          e->tcplans.push_back(pl);
          name("conv3x3 %d->%d(pad 128) @%d nchw-out /sigma [%s]", a.C, ch, R, tc_gemm_form(pl));
          next_bytes = (double)B * R * R * (a.C * (om == 2 ? 2.0 : 4.0) + ch * 4.0);
          op(1, [=](cudaStream_t st) {
            tc_gemm_set_head(pl, eng->out_l[ln], sbs ? eng->in_labels_l[ln] : nullptr, eng->uniform ? 0 : 1);
            return tc_gemm_launch(pl, st);
          }, 0, 2.0 * B * R * R * (double)ch * a.C * 9);
        }
      } else if (ch <= 4) {
        name("conv3x3 %d->%d @%d nchw-out [small-n]", a.C, ch, R);
        op(1, [=](cudaStream_t st) {
          return launch_conv3x3_small_n(ain.p, wo, bo, sbs ? eng->in_labels_l[ln] : nullptr, eng->uniform ? 0 : 1, eng->out_l[ln],
                                        Bc, R, R, ain.C, ch, head_f16, st);
        }, 1, 2.0 * B * R * R * (double)ch * a.C * 9);
      } else {
        SimtConv s; memset(&s, 0, sizeof(s));
        s.x1 = a.p; s.C1 = a.C; s.in_scale = 1.f; s.H = R; s.W = R; s.R = s.S = 3; s.stride = 1; s.pad = 1;
        s.OH = R; s.OW = R; s.nbatch = B; s.a_batched = 1; s.w = wo; s.N = ch;
        s.epi.bias = bo; s.epi.scale = 1.f; s.epi.rows_per_img = R * R; s.epi.out_nchw = 1; s.epi.ld_out = ch;
        op(1, [=](cudaStream_t st) {
          SimtConv cc = s;
          cc.epi.out = eng->out_l[ln];
          if (sbs) { cc.epi.per_img_div = eng->in_labels_l[ln]; cc.epi.div_stride = eng->uniform ? 0 : 1; }
          return launch_conv_simt(cc, st);
        }, 1, 2.0 * B * R * R * (double)ch * a.C * 9);
      }
      tfree(a);
    }
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
    (void)eb; (void)t1b; (void)t2b; (void)db; (void)xcb;
    return rc;
  }

  bool lvl_has_attn(int r) const {
    for (int i = 0; i < e->cfg.num_attn_resolutions; ++i) if (e->cfg.attn_resolutions[i] == r) return true;
    return false;
  }
};

}  // namespace

// ===========================================================================
// C ABI: model
// ===========================================================================
extern "C" {

int b200_ncsnpp_create(const b200_ncsnpp_config* cfg, b200_ncsnpp_t** out) {
  B200_REQUIRE(cfg && out, "ncsnpp_create: null argument");
  B200_REQUIRE(cfg->separate_groupnorm != 0, "ncsnpp_create: separate_groupnorm = 0 (GroupNorm applied on load by the tensor-core "
               "convolution) is not available in this build; use 1 or 2");
  B200_REQUIRE(cfg->family == 0 || cfg->family == 1, "ncsnpp_create: family=%d unknown (0 NCSN++, 1 DDPM)", cfg->family);
  if (cfg->family == 1) {
    B200_REQUIRE(cfg->conditional, "ncsnpp_create: DDPM (family 1) needs conditional = 1 (the reference's own constructor fails "
                 "without time conditioning, models/ddpm.py:58-71)");
    B200_REQUIRE(!cfg->scale_by_sigma, "ncsnpp_create: DDPM (family 1) with scale_by_sigma = 1 (configs/ve/cifar10_ddpm.py) is not "
                 "supported by the engine");
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
  if (p.pack == PK_CONV_FLAT32)   // OIHW (3x3, I*9 <= 32) -> [O][32] with k = tap*I + i (rest of the row stays zero)
    return launch_pack_weight(src, dst, p.taps, p.O, p.I, (long long)p.I * p.taps, p.taps, 1, p.round, st, p.I, p.round == 2 ? 64 : 32);
  if (p.pack == PK_CONV_PAD128)   // OIHW -> [tap][128][I], rows >= O stay zero
    return launch_pack_weight(src, dst, p.taps, p.O, p.I, (long long)p.I * p.taps, p.taps, 1, p.round, st, 128LL * p.I, p.I);
  if (p.pack == PK_CONV)   // OIHW -> [tap][O][I]
    return launch_pack_weight(src, dst, p.taps, p.O, p.I, (long long)p.I * p.taps, p.taps, 1, p.round, st);
  // NIN W[in][out] -> [out][in]
  return launch_pack_weight(src, dst, 1, p.O, p.I, 1, p.O, 0, p.round, st);
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
}  // namespace

int b200_ncsnpp_forward(b200_ncsnpp_t* h, const float* x, const float* labels, int uniform, float* out, void* stream) {
  B200_REQUIRE(h && x && labels && out, "forward: null argument");
  B200_REQUIRE(!h->ops.empty(), "forward: no plan bound (call b200_ncsnpp_bind_workspace)");
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

int b200_ncsnpp_profile_forward(b200_ncsnpp_t* h, const float* x, const float* labels, int uniform, float* out,
                                void* stream, float ms_by_kind[8], double flops_by_kind[8], long long ops_by_kind[8]) {
  B200_REQUIRE(h && x && labels && out && ms_by_kind, "profile_forward: null argument");
  B200_REQUIRE(!h->ops.empty(), "profile_forward: no plan bound");
  set_call_args(h, x, labels, uniform, out);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (int k = 0; k < 8; ++k) { ms_by_kind[k] = 0.f; if (flops_by_kind) flops_by_kind[k] = 0.0; if (ops_by_kind) ops_by_kind[k] = 0; }
  // both lanes serially on ONE stream: each launch is timed alone (no overlap), which is what a per-kernel roofline needs
  std::vector<const b200_ncsnpp::Op*> all;
  for (auto& o : h->ops) all.push_back(&o);
  for (auto& o : h->ops2) all.push_back(&o);
  std::vector<cudaEvent_t> ev(all.size() + 1);
  for (auto& e : ev) B200_CHECK_CUDA(cudaEventCreate(&e));
  int rc = 0;
  B200_CHECK_CUDA(cudaEventRecord(ev[0], st));
  for (size_t i = 0; i < all.size() && !rc; ++i) {
    rc = all[i]->fn(st);
    cudaEventRecord(ev[i + 1], st);
  }
  if (!rc && cudaStreamSynchronize(st) != cudaSuccess) { set_error("profile_forward: stream sync failed"); rc = 1; }
  if (!rc) {
    for (size_t i = 0; i < all.size(); ++i) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, ev[i], ev[i + 1]);
      const int k = all[i]->kind & 7;
      ms_by_kind[k] += ms;
      if (flops_by_kind) flops_by_kind[k] += all[i]->flops;
      if (ops_by_kind) ops_by_kind[k] += 1;
    }
  }
  for (auto& e : ev) cudaEventDestroy(e);
  return rc;
}

long long b200_ncsnpp_num_ops(const b200_ncsnpp_t* h) { return h ? (long long)(h->ops.size() + h->ops2.size()) : 0; }

int b200_ncsnpp_op_info(const b200_ncsnpp_t* h, long long index, char* name, int name_cap, int* kind, double* flops) {
  B200_REQUIRE(h && index >= 0 && index < (long long)(h->ops.size() + h->ops2.size()), "op_info: index out of range");
  const b200_ncsnpp::Op& o = index < (long long)h->ops.size() ? h->ops[index] : h->ops2[index - h->ops.size()];
  if (name && name_cap > 0) { strncpy(name, o.name.c_str(), name_cap - 1); name[name_cap - 1] = 0; }
  if (kind) *kind = o.kind;
  if (flops) *flops = o.flops;
  return 0;
}

int b200_ncsnpp_op_bytes(const b200_ncsnpp_t* h, long long index, double* bytes) {
  B200_REQUIRE(h && bytes && index >= 0 && index < (long long)(h->ops.size() + h->ops2.size()), "op_bytes: index out of range");
  *bytes = (index < (long long)h->ops.size() ? h->ops[index] : h->ops2[index - h->ops.size()]).bytes;
  return 0;
}

int b200_ncsnpp_profile_ops(b200_ncsnpp_t* h, const float* x, const float* labels, int uniform, float* out, void* stream,
                            float* ms_per_op, long long cap) {
  B200_REQUIRE(h && x && labels && out && ms_per_op, "profile_ops: null argument");
  B200_REQUIRE(!h->ops.empty(), "profile_ops: no plan bound");
  const long long n = (long long)(h->ops.size() + h->ops2.size());
  B200_REQUIRE(cap >= n, "profile_ops: need room for %lld ops", n);
  set_call_args(h, x, labels, uniform, out);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& e : ev) B200_CHECK_CUDA(cudaEventCreate(&e));
  int rc = 0;
  B200_CHECK_CUDA(cudaEventRecord(ev[0], st));
  for (long long i = 0; i < n && !rc; ++i) {
    rc = (i < (long long)h->ops.size() ? h->ops[i] : h->ops2[i - h->ops.size()]).fn(st);
    cudaEventRecord(ev[i + 1], st);
  }
  if (!rc && cudaStreamSynchronize(st) != cudaSuccess) { set_error("profile_ops: stream sync failed"); rc = 1; }
  if (!rc) for (long long i = 0; i < n; ++i) cudaEventElapsedTime(&ms_per_op[i], ev[i], ev[i + 1]);
  for (auto& e : ev) cudaEventDestroy(e);
  return rc;
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

long long b200_ncsnpp_launches_per_forward(const b200_ncsnpp_t* h) { return h ? h->launches : 0; }

}  // extern "C"

// ===========================================================================
// C ABI: predictor-corrector loop
// ===========================================================================
struct b200_pc {
  b200_ncsnpp* model; b200_pc_config cfg; int B; long long numel, per_img;
  std::vector<float> h_label, h_ss, h_alpha, h_pa, h_pb, h_pc, h_ca, h_cb, h_cc;
  // workspace carve-up
  char* ws = nullptr; float *d_label, *d_ss, *d_alpha, *d_pa, *d_pb, *d_pc, *d_ca, *d_cb, *d_cc, *labels, *net_out, *norms, *means;
  int* d_step; unsigned long long* d_offset;
  PhiloxMap map;
  cudaGraphExec_t gexec = nullptr; float* graph_x = nullptr; float* graph_xm = nullptr; cudaStream_t graph_stream = nullptr;
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
  pc->d_label = (float*)take(N * 4LL); pc->d_ss = (float*)take(N * 4LL); pc->d_alpha = (float*)take(N * 4LL);
  pc->d_pa = (float*)take(N * 4LL); pc->d_pb = (float*)take(N * 4LL); pc->d_pc = (float*)take(N * 4LL);
  pc->d_ca = (float*)take(N * 4LL); pc->d_cb = (float*)take(N * 4LL); pc->d_cc = (float*)take(N * 4LL);
  pc->labels = (float*)take(pc->B * 4LL); pc->net_out = (float*)take(pc->numel * 4LL);
  pc->norms = (float*)take(2LL * pc->B * 4); pc->means = (float*)take(256);
  pc->d_step = (int*)take(256); pc->d_offset = (unsigned long long*)take(256);
  return off;
}

// one PC iteration at step *d_step; noise_c/noise_p non-null -> external noise
int pc_iteration(b200_pc* pc, float* x, float* x_mean, const float* noise_c, const float* noise_p, cudaStream_t st) {
  b200_ncsnpp* m = pc->model;
  const b200_pc_config& c = pc->cfg;
  PcStepScalars sc{pc->d_ss, pc->d_alpha, pc->d_pa, pc->d_pb, pc->d_pc};
  const unsigned long long cps = (unsigned long long)((c.corrector ? c.n_corrector_steps : 0) + (c.predictor ? 1 : 0));
  if (int r = launch_fill_from_table(pc->d_label, pc->d_step, pc->labels, pc->B, st)) return r;
  unsigned long long call = 0;
  if (c.corrector == 2) {
    // affine corrector (annealed Langevin dynamics, sampling.py:286-319): the step size is a per-step scalar, so the update is
    // the predictor's kernel with the corrector's own tables; every inner step draws fresh noise like the reference's loop
    PcStepScalars cs{pc->d_ss, pc->d_alpha, pc->d_ca, pc->d_cb, pc->d_cc};
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
  if (c.predictor) {
    if (int r = b200_ncsnpp_forward(m, x, pc->labels, 1, pc->net_out, st)) return r;
    if (int r = launch_predictor_apply(x, x_mean, pc->net_out, noise_p, pc->map, pc->d_offset, pc->d_step, cps, call,
                                       sc, 1, st)) return r;
  }
  if (!c.predictor && x_mean) {
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
  B200_REQUIRE(cfg->predictor == 0 || cfg->predictor == 1, "pc_create: predictor %d unsupported", cfg->predictor);
  b200_pc* pc = new b200_pc();
  pc->model = model; pc->cfg = *cfg; pc->B = batch;
  const b200_ncsnpp_config& mc = model->cfg;
  pc->per_img = (long long)mc.num_channels * mc.image_size * mc.image_size;
  pc->numel = pc->per_img * batch;
  const int N = cfg->n_steps;
  auto cp = [&](std::vector<float>& dst, const float* src, float dflt) { dst.assign(N, dflt); if (src) memcpy(dst.data(), src, N * 4); };
  cp(pc->h_label, cfg->label, 0.f); cp(pc->h_ss, cfg->score_scale, 1.f); cp(pc->h_alpha, cfg->alpha, 1.f);
  cp(pc->h_pa, cfg->pa, 1.f); cp(pc->h_pb, cfg->pb, 0.f); cp(pc->h_pc, cfg->pc, 0.f);
  cp(pc->h_ca, cfg->ca, 1.f); cp(pc->h_cb, cfg->cb, 0.f); cp(pc->h_cc, cfg->cc, 0.f);
  pc->cfg.label = pc->cfg.score_scale = pc->cfg.alpha = pc->cfg.pa = pc->cfg.pb = pc->cfg.pc = nullptr;
  pc->cfg.ca = pc->cfg.cb = pc->cfg.cc = nullptr;
  const long long cps = (cfg->corrector ? cfg->n_corrector_steps : 0) + (cfg->predictor ? 1 : 0);
  pc->launches_per_step = cps * model->launches + (cfg->corrector == 1 ? cfg->n_corrector_steps * 3 : cfg->corrector == 2 ? cfg->n_corrector_steps : 0) +
                          1 /* predictor apply, or the x -> x_mean copy */ + 2;
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
  B200_CHECK_CUDA(cudaMemcpyAsync(pc->d_label, pc->h_label.data(), N * 4, cudaMemcpyHostToDevice, st));
  B200_CHECK_CUDA(cudaMemcpyAsync(pc->d_ss, pc->h_ss.data(), N * 4, cudaMemcpyHostToDevice, st));
  B200_CHECK_CUDA(cudaMemcpyAsync(pc->d_alpha, pc->h_alpha.data(), N * 4, cudaMemcpyHostToDevice, st));
  B200_CHECK_CUDA(cudaMemcpyAsync(pc->d_pa, pc->h_pa.data(), N * 4, cudaMemcpyHostToDevice, st));
  B200_CHECK_CUDA(cudaMemcpyAsync(pc->d_pb, pc->h_pb.data(), N * 4, cudaMemcpyHostToDevice, st));
  B200_CHECK_CUDA(cudaMemcpyAsync(pc->d_pc, pc->h_pc.data(), N * 4, cudaMemcpyHostToDevice, st));
  B200_CHECK_CUDA(cudaMemcpyAsync(pc->d_ca, pc->h_ca.data(), N * 4, cudaMemcpyHostToDevice, st));
  B200_CHECK_CUDA(cudaMemcpyAsync(pc->d_cb, pc->h_cb.data(), N * 4, cudaMemcpyHostToDevice, st));
  B200_CHECK_CUDA(cudaMemcpyAsync(pc->d_cc, pc->h_cc.data(), N * 4, cudaMemcpyHostToDevice, st));
  B200_CHECK_CUDA(cudaStreamSynchronize(st));
  if (pc->gexec) { cudaGraphExecDestroy(pc->gexec); pc->gexec = nullptr; }
  return philox_map_init(&pc->map, pc->numel, 0);
}

int b200_pc_run(b200_pc_t* pc, float* x, float* x_mean, int first_step, int num_steps, unsigned long long seed,
                unsigned long long offset, unsigned long long* offset_out, int use_graph, void* stream) {
  B200_REQUIRE(pc && pc->ws && x, "pc_run: not bound");
  PdlScope pdl(pc->model->cfg.pdl != 0);
  B200_REQUIRE(first_step >= 0 && num_steps >= 0 && first_step + num_steps <= pc->cfg.n_steps,
               "pc_run: steps [%d,%d) outside the %d-step schedule", first_step, first_step + num_steps, pc->cfg.n_steps);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  pc->map.seed = seed;
  // the noise offset of step s is *d_offset + (s*cps + call)*inc, so rebase for first_step
  const unsigned long long cps = (unsigned long long)((pc->cfg.corrector ? pc->cfg.n_corrector_steps : 0) + (pc->cfg.predictor ? 1 : 0));
  const unsigned long long base = offset - (unsigned long long)first_step * cps * pc->map.inc;
  B200_CHECK_CUDA(cudaMemcpyAsync(pc->d_offset, &base, 8, cudaMemcpyHostToDevice, st));
  B200_CHECK_CUDA(cudaMemcpyAsync(pc->d_step, &first_step, 4, cudaMemcpyHostToDevice, st));
  B200_CHECK_CUDA(cudaStreamSynchronize(st));   // host sources above are stack variables
  if (use_graph && num_steps > 0) {
    if (!pc->gexec || pc->graph_x != x || pc->graph_xm != x_mean || pc->graph_seed != seed || pc->graph_stream != st) {
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
    }
    for (int i = 0; i < num_steps; ++i) B200_CHECK_CUDA(cudaGraphLaunch(pc->gexec, st));
  } else {
    for (int i = 0; i < num_steps; ++i) if (int r = pc_iteration(pc, x, x_mean, nullptr, nullptr, st)) return r;
  }
  if (offset_out) *offset_out = offset + (unsigned long long)num_steps * cps * pc->map.inc;
  return 0;
}

int b200_pc_step_external(b200_pc_t* pc, float* x, float* x_mean, int step, const float* noise_c,
                          const float* noise_p, void* stream) {
  B200_REQUIRE(pc && pc->ws && x, "pc_step_external: not bound");
  PdlScope pdl(pc->model->cfg.pdl != 0);
  B200_REQUIRE(step >= 0 && step < pc->cfg.n_steps, "pc_step_external: step %d out of range", step);
  B200_REQUIRE(!pc->cfg.corrector || noise_c, "pc_step_external: corrector noise missing");
  B200_REQUIRE(!pc->cfg.predictor || noise_p, "pc_step_external: predictor noise missing");
  B200_REQUIRE(pc->cfg.n_corrector_steps <= 1 || !pc->cfg.corrector, "pc_step_external: supports n_steps_each <= 1");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  B200_CHECK_CUDA(cudaMemcpyAsync(pc->d_step, &step, 4, cudaMemcpyHostToDevice, st));
  B200_CHECK_CUDA(cudaStreamSynchronize(st));
  return pc_iteration(pc, x, x_mean, noise_c, noise_p, st);
}

long long b200_pc_launches_per_step(const b200_pc_t* pc) { return pc ? pc->launches_per_step : 0; }

}  // extern "C"
