// C ABI of linetr_b200 (see include/linetr_b200.h): checkpoint folding/packing, workspace
// carving and the launch sequence of the line-descriptor forward and the matcher.
#include "../../include/linetr_b200.h"
#include "../../include/linetr_b200_debug.h"

#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <unordered_map>

#include "common.cuh"
#include "encoder_kernels.cuh"
#include "tc_weight.cuh"
#include "gemm_img.cuh"
#include "token_fused.cuh"
#include "sig_attention_tc.cuh"
#include "tokenizer_kernels.cuh"
#include "match_kernels.cuh"
#include "match_tc.cuh"
#include "line_gt.cuh"
#include "triplet.cuh"
#include "homography.cuh"
#include "warp.cuh"
#include "essential.cuh"
#include "fundamental.cuh"
#include "absolute_pose.cuh"
#include "triangulation.cuh"
#include "tracks.cuh"
#include "bundle.cuh"
#include "global_poses.cuh"
#include "retrieval.cuh"
#include "photometric.cuh"

namespace ltr {

thread_local std::string g_last_error;
std::atomic<int64_t> g_launches{0};
Profiler g_prof;
std::mutex g_state_mutex;

int set_error(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}

const char* kernel_class_name(int kc) {
  static const char* names[KC_COUNT] = {"small_mlp", "linear", "img_convert", "sig_attention", "final_norm",
                                         "dist", "segmean", "argmin", "mutual", "token_fused",
                                         "tokenize", "desc_tiles", "match_tc", "match_exact", "match_tail", "line_gt",
                                         "triplet", "homography", "warp", "essential", "photometric",
                                         "fundamental", "absolute_pose", "triangulate", "tracks",
                                         "bundle", "global_poses", "retrieval", "debug"};
  return (kc >= 0 && kc < KC_COUNT) ? names[kc] : "?";
}

cudaEvent_t Profiler::get() {
  if (!pool.empty()) {
    cudaEvent_t e = pool.back();
    pool.pop_back();
    return e;
  }
  cudaEvent_t e;
  cudaEventCreate(&e);
  return e;
}

// ------------------------------------------------------------------ packed model
// One wide linear layer: fp32 bias and the packed split-bf16 tile image of the folded matrix.
struct Lin {
  const float* b = nullptr;
  TcWeight tw;
};

// Positional encoders (IN -> 32 -> 64 -> 128 -> 256 -> 256), each packed in the form its kernels read.
struct WordPosEnc {   // token_fused_kernel: first layer on CUDA cores, the other four as tensor-core images
  const float *w1 = nullptr, *b1 = nullptr;
  Lin l2;             // 32 -> 64 with K zero-padded to one 64-wide k-block; l2.b is the kernel's fp32 b2
  Lin l3, l4, l5;
};
struct LinePosEnc {   // small_mlp_kernel (narrow head), then two image GEMMs (128 -> 256 relu, 256 -> 256)
  SmallMlpWeights head;
  Lin l4, l5;
};

struct SigLayer {
  Lin qkv;    // [768,256] head-major rows, q rows pre-scaled by 1/8
  Lin mlp1;   // [512,512] BN folded, attention output projection (`merge`) folded into the o-half
  Lin mlp2;   // [256,512]
};

}  // namespace ltr

struct LtrModel {
  int device = 0;
  LtrConfig cfg{};
  float* arena = nullptr;
  uint16_t* tc_arena = nullptr;
  size_t arena_floats = 0;
  ltr::WordPosEnc wpe{};
  ltr::LinePosEnc lpe{};
  float *U = nullptr, *s_cls = nullptr, *cls = nullptr;
  ltr::Lin wv, wfc, w1, w2, wf;  // wv: 4 heads of [64,256]; wfc bias includes the CLS residual
  float *ln1g = nullptr, *ln1b = nullptr, *ln2g = nullptr, *ln2b = nullptr;
  std::vector<ltr::SigLayer> sig;
};

namespace ltr {

using TensorMap = std::unordered_map<std::string, std::pair<const float*, int64_t>>;

struct LinOff { size_t b, tc; int N, K; };

struct HostPack {
  std::vector<float> buf;
  std::vector<uint16_t> tc;  // packed split-bf16 images: hi at off, lo at off + N*K
  size_t add(const std::vector<double>& v) {
    size_t off = (buf.size() + 63) / 64 * 64;  // 256-byte alignment of every tensor
    buf.resize(off + v.size());
    for (size_t i = 0; i < v.size(); ++i) buf[off + i] = (float)v[i];
    return off;
  }
  // wide layer [N,K]: bias + tensor-core image
  LinOff add_lin(const std::vector<double>& W, const std::vector<double>& b, int N, int K) {
    LinOff o{add(b), 0, N, K};
    size_t off = (tc.size() + 511) / 512 * 512;  // 1024-byte alignment
    tc.resize(off + 2 * (size_t)N * K);
    pack_tc_weight(W.data(), N, K, tc.data() + off, tc.data() + off + (size_t)N * K);
    o.tc = off;
    return o;
  }
};

static Lin bind_lin(const LinOff& o, float* fbase, uint16_t* tbase) {
  Lin l;
  l.b = fbase + o.b;
  l.tw.hi = reinterpret_cast<const __nv_bfloat16*>(tbase + o.tc);
  l.tw.lo = reinterpret_cast<const __nv_bfloat16*>(tbase + o.tc + (size_t)o.N * o.K);
  l.tw.N = o.N;
  l.tw.K = o.K;
  return l;
}

static bool fetch(const TensorMap& tm, const std::string& name, int64_t numel, const float** out, std::string& err) {
  auto it = tm.find(name);
  if (it == tm.end()) { err = "missing checkpoint tensor '" + name + "'"; return false; }
  if (it->second.second != numel) {
    err = "checkpoint tensor '" + name + "' has " + std::to_string(it->second.second) + " elements, expected " +
          std::to_string(numel);
    return false;
  }
  *out = it->second.first;
  return true;
}

// Conv1d(k=1)/Linear [out,in] (+ eval BatchNorm1d at bn_prefix, eps 1e-5) -> folded W, b in fp64.
static bool fold_layer(const TensorMap& tm, const std::string& conv, const std::string& bn, int out, int in,
                       std::vector<double>& W, std::vector<double>& b, std::string& err) {
  const float *w, *bias;
  if (!fetch(tm, conv + ".weight", (int64_t)out * in, &w, err) || !fetch(tm, conv + ".bias", out, &bias, err)) return false;
  W.assign((size_t)out * in, 0.0);
  b.assign(out, 0.0);
  for (int o = 0; o < out; ++o) {
    double s = 1.0, shift = 0.0;
    if (!bn.empty()) {
      const float *g, *be, *mu, *var;
      if (!fetch(tm, bn + ".weight", out, &g, err) || !fetch(tm, bn + ".bias", out, &be, err) ||
          !fetch(tm, bn + ".running_mean", out, &mu, err) || !fetch(tm, bn + ".running_var", out, &var, err))
        return false;
      s = (double)g[o] / std::sqrt((double)var[o] + 1e-5);
      shift = (double)be[o] - (double)mu[o] * s;
    }
    for (int i = 0; i < in; ++i) W[(size_t)o * in + i] = (double)w[(size_t)o * in + i] * s;
    b[o] = (double)bias[o] * s + shift;
  }
  return true;
}

// The five layers of a positional encoder, eval-BatchNorm folded into the first four.
static bool fold_pos_encoder(const TensorMap& tm, const std::string& prefix, int in, std::vector<double> (&W)[5],
                             std::vector<double> (&b)[5], std::string& err) {
  const int ch[6] = {in, 32, 64, 128, 256, 256};
  for (int l = 0; l < 5; ++l) {
    std::string conv = prefix + "." + std::to_string(3 * l);
    std::string bn = (l < 4) ? prefix + "." + std::to_string(3 * l + 1) : std::string();
    if (!fold_layer(tm, conv, bn, ch[l + 1], ch[l], W[l], b[l], err)) return false;
  }
  return true;
}

struct WordPosOff { size_t w1, b1; LinOff l2, l3, l4, l5; };
struct LinePosOff { size_t w[3], b[3]; LinOff l4, l5; };

static bool pack_word_pos(const TensorMap& tm, HostPack& hp, WordPosOff& o, std::string& err) {
  std::vector<double> W[5], b[5];
  if (!fold_pos_encoder(tm, "klenc.word_position_enc.encoder", 3, W, b, err)) return false;
  std::vector<double> W2((size_t)64 * 64, 0.0);
  for (int r = 0; r < 64; ++r)
    for (int i = 0; i < 32; ++i) W2[(size_t)r * 64 + i] = W[1][(size_t)r * 32 + i];
  o.w1 = hp.add(W[0]);
  o.b1 = hp.add(b[0]);
  o.l2 = hp.add_lin(W2, b[1], 64, 64);
  o.l3 = hp.add_lin(W[2], b[2], 128, 64);
  o.l4 = hp.add_lin(W[3], b[3], 256, 128);
  o.l5 = hp.add_lin(W[4], b[4], 256, 256);
  return true;
}

static bool pack_line_pos(const TensorMap& tm, HostPack& hp, LinePosOff& o, std::string& err) {
  std::vector<double> W[5], b[5];
  if (!fold_pos_encoder(tm, "klenc.line_position_enc.encoder", 5, W, b, err)) return false;
  for (int l = 0; l < 3; ++l) {
    o.w[l] = hp.add(W[l]);
    o.b[l] = hp.add(b[l]);
  }
  o.l4 = hp.add_lin(W[3], b[3], 256, 128);
  o.l5 = hp.add_lin(W[4], b[4], 256, 256);
  return true;
}

static cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// ------------------------------------------------------------------ workspace
struct EncodeWs {
  // line stage
  ActImg z, ctx, y1i, g, l128, l256, lpos;  // images [R, 1024 / 256 / 256 / 1024 / 128 / 256 / 256]
  // signature stage
  ActImg xm, hm;       // images [R, 512] = [x | attention output], [R, 512]
  ActImg qkv;          // image [R, 768]: k-block h = q of head h, 4 + h = k, 8 + h = v
  float* yf;           // fp32 [R, 256] (final projection when the channel-first layout is requested)
  int64_t bytes;
};

static EncodeWs carve(const LtrModel* m, int n_lines, char* base) {
  EncodeWs w{};
  int64_t off = 0;
  auto take = [&](int64_t bytes) {
    char* p = base + off;
    off = align_up(off + bytes, 1024);
    return p;
  };
  auto takef = [&](int64_t floats) { return reinterpret_cast<float*>(take(floats * 4)); };
  auto takei = [&](int64_t rows, int K) {
    const int64_t mpad = align_up(rows, 256);
    ActImg a;
    a.hi = reinterpret_cast<__nv_bfloat16*>(take(mpad * K * 2));
    a.lo = reinterpret_cast<__nv_bfloat16*>(take(mpad * K * 2));
    a.kblocks = K / 64;
    return a;
  };
  const int64_t R = n_lines;
  w.z = takei(R, 1024);
  w.ctx = takei(R, 256);
  w.y1i = takei(R, 256);
  w.g = takei(R, m->cfg.d_inner);   // FFN hidden activation [R, d_inner]
  w.l128 = takei(R, 128);
  w.l256 = takei(R, 256);
  w.lpos = takei(R, 256);
  w.xm = takei(R, 512);
  w.hm = takei(R, 512);
  w.qkv = takei(R, 768);
  w.yf = takef(R * 256);
  w.bytes = off;
  return w;
}

// One wide layer on the tensor-core engine: A image k-blocks [a_kb0, a_kb0 + K/64) -> fp32 rows C
// (optional) and/or image O k-blocks from o_kb0 (optional); R = fp32 residual.
static GemmImgArgs gemm_args(const Lin& L, const ActImg& A, int a_kb0, int M, int act, float* C, int ldc,
                             const ActImg* O = nullptr, int o_kb0 = 0, const float* R = nullptr, int ldr = 0,
                             const ActImg* Rimg = nullptr, int r_kb0 = 0, int a_kb_nb = 0) {
  GemmImgArgs a{};
  a.A = A; a.a_kb0 = a_kb0; a.W = L.tw; a.bias = L.b; a.R = R; a.ldr = ldr; a.C = C; a.ldc = ldc;
  if (O) { a.O = *O; a.o_kb0 = o_kb0; }
  if (Rimg) { a.Rimg = *Rimg; a.r_kb0 = r_kb0; }
  a.M = M; a.act = act; a.a_kb_nb = a_kb_nb;
  return a;
}

static int gemm(const Lin& L, const ActImg& A, int a_kb0, int M, int act, cudaStream_t s, float* C, int ldc,
                const ActImg* O = nullptr, int o_kb0 = 0, const float* R = nullptr, int ldr = 0,
                const ActImg* Rimg = nullptr, int r_kb0 = 0, int bn_hint = 0, int a_kb_nb = 0) {
  return launch_gemm_img(gemm_args(L, A, a_kb0, M, act, C, ldc, O, o_kb0, R, ldr, Rimg, r_kb0, a_kb_nb), s, bn_hint);
}

static int launch_small_mlp(const SmallMlpWeights& w, const float* in0, const float* in1, const float* in2, ActImg out,
                            int rows, float width, float height, cudaStream_t s) {
  if (rows <= 0) return 0;
  const int groups = cdiv(rows, SM_ROWS);
  int grid = cdiv(groups, SM_WARPS);
  if (grid > 132 * 3) grid = 132 * 3;
  const float scale = fmaxf(width, height) * 0.7f;
  return launch(KC_SMALL_MLP, true, small_mlp_kernel, dim3(grid), dim3(SM_WARPS * 32), sizeof(SmallMlpSmem), s, w, in0, in1,
                in2, out, rows, width / 2.f, height / 2.f, scale);
}

static ActImg tiles_image(void* tiles, int64_t n_lines) {
  ActImg a;
  const int64_t plane = align_up(n_lines, 128) * MT_D;   // bf16 elements per plane
  a.hi = reinterpret_cast<__nv_bfloat16*>(tiles);
  a.lo = a.hi + plane;
  a.kblocks = MT_KB;
  return a;
}

// Fewest 128-row tiles for which an encode chains its row-local GEMMs (gemm_chain_kernel: one CTA per m-tile, so it
// needs about as many m-tiles as SMs to pay).  128 = bench.py cfg1, the smallest batch measured faster chained on
// H100 (a layer chain at 64 and 96 tiles was slower than its three launches, tools/gemm_chain_bench.py).
// LTR_CHAIN_MIN_TILES overrides it, 0 = never chain; read at every call so that one process can run both paths.
static int chain_min_tiles() {
  const char* e = std::getenv("LTR_CHAIN_MIN_TILES");
  if (e && *e) {
    char* end = nullptr;
    const long v = std::strtol(e, &end, 10);
    if (*end == '\0' && v >= 0) return v == 0 || v > INT_MAX ? INT_MAX : (int)v;
  }
  return 128;
}

static int encode_impl(LtrModel* m, const LtrEncodeInput& in, float* out_cf, float* out_rows, void* out_tiles,
                       const EncodeWs& w, cudaStream_t s) {
  const int R = in.n_lines, T = in.n_tokens;
  const int* cu = in.cu_lines_dev;
  // ---- token stage: one fused persistent kernel (narrow MLP, 3 tensor-core layers, + desc, CLS pooling) ----
  {
    TokenFusedArgs a{};
    a.pnt = in.pnt; a.score = in.score; a.desc = in.desc;
    a.w1 = m->wpe.w1; a.b1 = m->wpe.b1; a.b2 = m->wpe.l2.b;
    a.W2 = m->wpe.l2.tw; a.W3 = m->wpe.l3.tw; a.W4 = m->wpe.l4.tw; a.W5 = m->wpe.l5.tw;
    a.b3 = m->wpe.l3.b; a.b4 = m->wpe.l4.b; a.b5 = m->wpe.l5.b;
    a.U = m->U; a.s_cls = m->s_cls; a.cls = m->cls;
    a.z = w.z; a.R = R; a.T = T;
    a.cx = in.image_width / 2.f; a.cy = in.image_height / 2.f;
    a.scale = fmaxf(in.image_width, in.image_height) * 0.7f;
    LTR_TRY(launch_token_fused(a, s));
  }
  // ---- line stage: V projection (block diagonal over heads), fc + CLS residual, LN, FFN, LN, + line pos ----
  LTR_TRY(gemm(m->wv, w.z, 0, R, ACT_NONE, s, nullptr, 0, &w.ctx, 0, nullptr, 0, nullptr, 0, 64, 4));
  // line positional encoder first (its output is added in the w_2 epilogue)
  LTR_TRY(launch_small_mlp(m->lpe.head, in.sublines, in.resp, in.angle, w.l128, R, in.image_width, in.image_height, s));
  LTR_TRY(gemm(m->lpe.l4, w.l128, 0, R, ACT_RELU, s, nullptr, 0, &w.l256, 0));
  LTR_TRY(gemm(m->lpe.l5, w.l256, 0, R, ACT_NONE, s, nullptr, 0, &w.lpos, 0));
  // The row-local GEMM runs fc -> w_1 -> w_2 -> qkv(0) and, per signature layer, mlp1 -> mlp2 -> qkv(l+1) (or
  // final_proj) go out as one gemm_chain_kernel launch each when the batch fills the GPU with m-tiles; small batches
  // keep one launch per layer, which spreads the n-blocks of a layer over more SMs.
  const bool chain = !out_cf && cdiv(R, 128) >= chain_min_tiles();
  GemmImgArgs pend[CHAIN_MAX_OPS];
  int n_pend = 0;
  auto flush = [&]() -> int {
    const int n = n_pend;
    n_pend = 0;
    if (n == 0) return 0;
    return n == 1 ? launch_gemm_img(pend[0], s) : launch_gemm_chain(pend, n, s);
  };
  auto row_local = [&](const GemmImgArgs& a) -> int {   // queued for the current chain, or launched now
    if (!chain) return launch_gemm_img(a, s);
    pend[n_pend++] = a;
    return 0;
  };
  {
    // fc (+ CLS residual folded into the bias) -> LayerNorm in the epilogue -> y1.  y1 and the line position code live
    // only as split-bf16 images (hi + lo: ~2^-17 relative): the FFN residual and the post-norm addend are read back
    // from them, row by row, straight into registers
    GemmImgArgs fc = gemm_args(m->wfc, w.ctx, 0, R, ACT_NONE, nullptr, 0, &w.y1i, 0);
    fc.norm = NORM_LAYER; fc.eps = 1e-6f; fc.ng = m->ln1g; fc.nbeta = m->ln1b;
    GemmImgArgs w1 = gemm_args(m->w1, w.y1i, 0, R, ACT_GELU, nullptr, 0, &w.g, 0);
    // sentence = klines_pos + LN(y1 + ffn)  -> image xm[:, :256] (the running descriptor), all in the w_2 epilogue
    GemmImgArgs w2 = gemm_args(m->w2, w.g, 0, R, ACT_NONE, nullptr, 0, &w.xm, 0, nullptr, 0, &w.y1i, 0);
    w2.norm = NORM_LAYER; w2.eps = 1e-6f; w2.ng = m->ln2g; w2.nbeta = m->ln2b; w2.NaddImg = w.lpos; w2.nadd_kb0 = 0;
    if (m->cfg.d_inner % 256 == 0 && m->cfg.d_inner <= 64 * CHAIN_MAX_KB) {   // w_1 output fits the chain's k-block barriers
      LTR_TRY(row_local(fc));
      LTR_TRY(row_local(w1));
      LTR_TRY(row_local(w2));
    } else {
      LTR_TRY(launch_gemm_img(fc, s));
      LTR_TRY(launch_gemm_img(w1, s));
      LTR_TRY(launch_gemm_img(w2, s));
    }
  }
  // ---- line signature layers ----
  int max_l = in.lines_per_image;
  if (in.cu_lines_host) {
    max_l = 0;
    for (int i = 0; i < in.n_images; ++i) max_l = std::max(max_l, in.cu_lines_host[i + 1] - in.cu_lines_host[i]);
  }
  ActImg tiles{};
  if (out_tiles) tiles = tiles_image(out_tiles, R);
  GemmImgArgs fin = gemm_args(m->wf, w.xm, 0, R, ACT_NONE, out_rows, 256, out_tiles ? &tiles : nullptr, 0);
  fin.norm = NORM_L2; fin.eps = 1e-6f;   // final_proj + F.normalize in one epilogue (rows-only output)
  for (size_t li = 0; li < m->sig.size(); ++li) {
    const SigLayer& L = m->sig[li];
    LTR_TRY(row_local(gemm_args(L.qkv, w.xm, 0, R, ACT_NONE, nullptr, 0, &w.qkv, 0)));
    LTR_TRY(flush());
    // o -> xm[:, 256:]
    LTR_TRY(launch_sig_attention_tc(w.qkv, w.xm, 256, cu, in.lines_per_image, max_l, in.n_images, s));
    // x += delta: the running descriptor lives ONLY as the split-bf16 image xm[:, :256] (hi + lo carries
    // ~2^-17 relative precision; an fp32 copy would double the store traffic of this epilogue)
    LTR_TRY(row_local(gemm_args(L.mlp1, w.xm, 0, R, ACT_RELU, nullptr, 0, &w.hm, 0)));
    LTR_TRY(row_local(gemm_args(L.mlp2, w.hm, 0, R, ACT_NONE, nullptr, 0, &w.xm, 0, nullptr, 0, &w.xm, 0)));
  }
  if (!out_cf) {   // rows (+ matcher tile image): projection + L2 normalisation in one launch
    LTR_TRY(row_local(fin));
    return flush();
  }
  LTR_TRY(gemm(m->wf, w.xm, 0, R, ACT_NONE, s, w.yf, 256));
  if (max_l > 0)
    LTR_TRY(launch(KC_FINAL_NORM, true, final_norm_kernel, dim3(cdiv(max_l, 32), in.n_images), dim3(256), 0, s,
                   (const float*)w.yf, out_rows, out_cf, cu, in.lines_per_image));
  return 0;
}

static int run_nn(const NNArgs& a, int n_pairs, int max_k0, int max_k1, cudaStream_t s) {
  if (max_k0 <= 0) {
    LTR_CUDA_TRY(cudaMemsetAsync(a.counts, 0, sizeof(int) * n_pairs, s));
    return 0;
  }
  // row_argmin_kernel also zeroes counts[pair]
  LTR_TRY(launch(KC_ARGMIN, true, row_argmin_kernel, dim3(cdiv(max_k0, 8), n_pairs), dim3(256), 0, s, a));
  if (a.mutual && max_k1 > 0)
    LTR_TRY(launch(KC_ARGMIN, true, col_argmin_kernel, dim3(cdiv(max_k1, 32), n_pairs), dim3(256), 0, s, a));
  return launch(KC_MUTUAL, true, mutual_kernel, dim3(cdiv(max_k0, 256), n_pairs), dim3(256), 0, s, a);
}

// Images per launch of the tokenizer kernels: their table travels as a kernel parameter (40 bytes each, 5 KB in
// all: above the classic 4 KB, within the 32 KB parameter limit CUDA 12.1 brought to sm_70 and newer).
constexpr int kTokImagesPerLaunch = 128;

// The two tokenizer launches for the sublines [s_begin, s_end) of images I.first ...
template <int NI>
static int launch_tokenize(const TokLines& L, const TokImages<NI>& I, int s_begin, int s_end, int align_corners,
                           float* sublines, float* pnt, float* mask, float* resp, float* angle, float* desc, float* score,
                           cudaStream_t s) {
  const long long n_tok = (long long)(s_end - s_begin) * L.T;
  if (n_tok <= 0) return LTR_OK;
  LTR_TRY(launch(KC_TOKENIZE, false, tok_points_kernel<NI>, dim3(cdiv(n_tok, 256)), dim3(256), 0, s, L, I, s_begin, s_end, pnt,
                 mask, sublines, resp, angle));
  return launch(KC_TOKENIZE, false, tok_sample_kernel<NI>, dim3(cdiv(n_tok, 8)), dim3(256), 0, s, L, I, s_begin, s_end,
                align_corners, pnt, desc, score);
}

}  // namespace ltr

using namespace ltr;

extern "C" {

int ltr_abi_version(void) { return LTR_ABI_VERSION; }
const char* ltr_last_error(void) { return g_last_error.c_str(); }
int64_t ltr_launch_count(void) { return g_launches.load(); }
void ltr_reset_launch_count(void) { g_launches.store(0); }

void ltr_profile_begin(void) {
  std::lock_guard<std::mutex> lk(g_state_mutex);
  for (auto& r : g_prof.recs) { g_prof.pool.push_back(r.a); g_prof.pool.push_back(r.b); }
  g_prof.recs.clear();
  g_prof.on = true;
}

int ltr_profile_end(const char** names, float* ms, int32_t* launches, int32_t max_classes) {
  g_prof.on = false;
  cudaDeviceSynchronize();
  float tot[KC_COUNT] = {0};
  int cnt[KC_COUNT] = {0};
  std::lock_guard<std::mutex> lk(g_state_mutex);
  for (auto& r : g_prof.recs) {
    float t = 0.f;
    if (cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess) { tot[r.kc] += t; cnt[r.kc]++; }
    g_prof.pool.push_back(r.a);
    g_prof.pool.push_back(r.b);
  }
  g_prof.recs.clear();
  int n = 0;
  for (int k = 0; k < KC_COUNT && n < max_classes; ++k) {
    if (!cnt[k]) continue;
    names[n] = kernel_class_name(k);
    ms[n] = tot[k];
    launches[n] = cnt[k];
    ++n;
  }
  return n;
}

int ltr_create(const LtrTensor* tensors, int32_t n_tensors, const LtrConfig* cfg, int32_t device, LtrModel** out) {
  if (!tensors || !cfg || !out) return set_error(LTR_E_INVALID, "ltr_create: null argument");
  if (cfg->d_model != 256 || cfg->n_heads != 4)
    return set_error(LTR_E_UNSUPPORTED, "ltr_create: kernels are specialised for d_model=256, n_heads=4");
  if (cfg->d_inner <= 0 || cfg->d_inner % 128 || cfg->n_desc_layers < 1 || cfg->n_sig_layers < 0)
    return set_error(LTR_E_INVALID, "ltr_create: bad d_inner / layer counts");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return set_error(LTR_E_CUDA, "ltr_create: no CUDA device (there is no CPU fallback)");
  if (device < 0 || device >= ndev) return set_error(LTR_E_INVALID, "ltr_create: bad device index");
  LTR_CUDA_TRY(cudaSetDevice(device));

  TensorMap tm;
  for (int i = 0; i < n_tensors; ++i) tm[tensors[i].name] = {tensors[i].data, tensors[i].numel};
  std::string err;
  HostPack hp;
  const int D = 256, DI = cfg->d_inner;
  WordPosOff wpe_o{};
  LinePosOff lpe_o{};
  if (!pack_word_pos(tm, hp, wpe_o, err) || !pack_line_pos(tm, hp, lpe_o, err)) return set_error(LTR_E_INVALID, err);

  // ---- descriptive layer (only the last one is live) ----
  const std::string dl = "klenc.desc_layers." + std::to_string(cfg->n_desc_layers - 1);
  const float *cls, *wq, *bq, *wk, *bk, *wv, *bv, *wfc, *bfc, *ln1g, *ln1b, *w1, *b1, *w2, *b2, *ln2g, *ln2b;
  if (!fetch(tm, "klenc.cls_token", D, &cls, err) ||
      !fetch(tm, dl + ".slf_attn.w_qs.weight", D * D, &wq, err) || !fetch(tm, dl + ".slf_attn.w_qs.bias", D, &bq, err) ||
      !fetch(tm, dl + ".slf_attn.w_ks.weight", D * D, &wk, err) || !fetch(tm, dl + ".slf_attn.w_ks.bias", D, &bk, err) ||
      !fetch(tm, dl + ".slf_attn.w_vs.weight", D * D, &wv, err) || !fetch(tm, dl + ".slf_attn.w_vs.bias", D, &bv, err) ||
      !fetch(tm, dl + ".slf_attn.fc.weight", D * D, &wfc, err) || !fetch(tm, dl + ".slf_attn.fc.bias", D, &bfc, err) ||
      !fetch(tm, dl + ".slf_attn.layer_norm.weight", D, &ln1g, err) ||
      !fetch(tm, dl + ".slf_attn.layer_norm.bias", D, &ln1b, err) ||
      !fetch(tm, dl + ".pos_ffn.w_1.weight", (int64_t)DI * D, &w1, err) || !fetch(tm, dl + ".pos_ffn.w_1.bias", DI, &b1, err) ||
      !fetch(tm, dl + ".pos_ffn.w_2.weight", (int64_t)D * DI, &w2, err) || !fetch(tm, dl + ".pos_ffn.w_2.bias", D, &b2, err) ||
      !fetch(tm, dl + ".pos_ffn.layer_norm.weight", D, &ln2g, err) ||
      !fetch(tm, dl + ".pos_ffn.layer_norm.bias", D, &ln2b, err))
    return set_error(LTR_E_INVALID, err);
  (void)bk;  // the key bias shifts all scores of a head equally: cancels in the softmax
  auto vec = [](const float* p, size_t n) { return std::vector<double>(p, p + n); };
  // q_cls = W_q cls + b_q ;  u_h = W_k,h^T q_h / sqrt(64) ;  s_cls,h = cls . u_h
  std::vector<double> q(D), U(4 * D, 0.0), scls(4, 0.0);
  for (int o = 0; o < D; ++o) {
    double a = bq[o];
    for (int i = 0; i < D; ++i) a += (double)wq[o * D + i] * cls[i];
    q[o] = a;
  }
  for (int h = 0; h < 4; ++h) {
    for (int c = 0; c < D; ++c) {
      double a = 0;
      for (int d = 0; d < 64; ++d) a += (double)wk[(h * 64 + d) * D + c] * q[h * 64 + d];
      U[h * D + c] = a / 8.0;
    }
    for (int c = 0; c < D; ++c) scls[h] += (double)cls[c] * U[h * D + c];
  }
  std::vector<double> bfc_cls(D);
  for (int i = 0; i < D; ++i) bfc_cls[i] = (double)bfc[i] + cls[i];  // fc bias + CLS residual (line_attention.py:72)
  size_t oU = hp.add(U), oS = hp.add(scls), oC = hp.add(vec(cls, D));
  // V projection of the pooled per-head inputs z = [z_0 | z_1 | z_2 | z_3]: output channels h*64..h*64+63
  // only see z_h, i.e. a block-diagonal GEMM - run as N = 256, K = 256 with 64-wide n-blocks whose A
  // k-blocks start at 4*h (GemmImgArgs::a_kb_nb).
  LinOff oWv = hp.add_lin(vec(wv, D * D), vec(bv, D), D, D);
  LinOff oWfc = hp.add_lin(vec(wfc, D * D), bfc_cls, D, D);
  size_t oL1g = hp.add(vec(ln1g, D)), oL1b = hp.add(vec(ln1b, D));
  LinOff oW1 = hp.add_lin(vec(w1, (size_t)DI * D), vec(b1, DI), DI, D);
  LinOff oW2 = hp.add_lin(vec(w2, (size_t)D * DI), vec(b2, D), D, DI);
  size_t oL2g = hp.add(vec(ln2g, D)), oL2b = hp.add(vec(ln2b, D));

  // ---- signature layers ----
  struct SigOff { LinOff qkv, mlp1, mlp2; };
  std::vector<SigOff> so(cfg->n_sig_layers);
  for (int li = 0; li < cfg->n_sig_layers; ++li) {
    const std::string p = "selfattn.layers." + std::to_string(li);
    std::vector<double> Wqkv((size_t)768 * D), bqkv(768);
    for (int t = 0; t < 3; ++t) {
      const float *w, *b;
      if (!fetch(tm, p + ".attn.proj." + std::to_string(t) + ".weight", D * D, &w, err) ||
          !fetch(tm, p + ".attn.proj." + std::to_string(t) + ".bias", D, &b, err))
        return set_error(LTR_E_INVALID, err);
      const double sc = (t == 0) ? 0.125 : 1.0;  // scores / sqrt(64), line_transformer.py:134
      for (int h = 0; h < 4; ++h)
        for (int d = 0; d < 64; ++d) {
          const int oldr = d * 4 + h, newr = t * 256 + h * 64 + d;  // view(b, dim, heads, n), :151
          for (int i = 0; i < D; ++i) Wqkv[(size_t)newr * D + i] = (double)w[oldr * D + i] * sc;
          bqkv[newr] = (double)b[oldr] * sc;
        }
    }
    const float *wm, *bm;
    if (!fetch(tm, p + ".attn.merge.weight", D * D, &wm, err) || !fetch(tm, p + ".attn.merge.bias", D, &bm, err))
      return set_error(LTR_E_INVALID, err);
    std::vector<double> Wm((size_t)D * D);
    for (int o = 0; o < D; ++o)
      for (int h = 0; h < 4; ++h)
        for (int d = 0; d < 64; ++d) Wm[(size_t)o * D + h * 64 + d] = wm[o * D + d * 4 + h];
    std::vector<double> W1, B1, W2, B2;
    if (!fold_layer(tm, p + ".mlp.0", p + ".mlp.1", 2 * D, 2 * D, W1, B1, err) ||
        !fold_layer(tm, p + ".mlp.3", "", D, 2 * D, W2, B2, err))
      return set_error(LTR_E_INVALID, err);
    // Fold the attention output projection (`merge`) into the first MLP layer:
    //   mlp1([x | merge(o)]) = W1a x + W1b (Wm o + bm) + b1 = [W1a | W1b Wm] [x | o] + (b1 + W1b bm)
    // so the attention kernel writes o straight into the second half of the MLP input and the
    // merge GEMM (one launch + one activation round trip per layer) disappears.
    std::vector<double> W1f((size_t)2 * D * 2 * D), B1f(2 * D);
    for (int o = 0; o < 2 * D; ++o) {
      double bacc = B1[o];
      for (int i = 0; i < D; ++i) W1f[(size_t)o * 2 * D + i] = W1[(size_t)o * 2 * D + i];
      for (int j = 0; j < D; ++j) {
        double a = 0.0;
        for (int i = 0; i < D; ++i) a += W1[(size_t)o * 2 * D + D + i] * Wm[(size_t)i * D + j];
        W1f[(size_t)o * 2 * D + D + j] = a;
      }
      for (int i = 0; i < D; ++i) bacc += W1[(size_t)o * 2 * D + D + i] * (double)bm[i];
      B1f[o] = bacc;
    }
    so[li] = {hp.add_lin(Wqkv, bqkv, 768, D), hp.add_lin(W1f, B1f, 2 * D, 2 * D), hp.add_lin(W2, B2, D, 2 * D)};
  }
  std::vector<double> Wf, Bf;
  if (!fold_layer(tm, "final_proj", "", D, D, Wf, Bf, err)) return set_error(LTR_E_INVALID, err);
  LinOff oWf = hp.add_lin(Wf, Bf, D, D);

  LtrModel* m = new LtrModel();
  m->device = device;
  m->cfg = *cfg;
  m->arena_floats = hp.buf.size();
  cudaError_t ce = cudaMalloc(&m->arena, hp.buf.size() * sizeof(float));
  if (ce == cudaSuccess) ce = cudaMemcpy(m->arena, hp.buf.data(), hp.buf.size() * sizeof(float), cudaMemcpyHostToDevice);
  if (ce == cudaSuccess) ce = cudaMalloc(&m->tc_arena, hp.tc.size() * sizeof(uint16_t));
  if (ce == cudaSuccess) ce = cudaMemcpy(m->tc_arena, hp.tc.data(), hp.tc.size() * sizeof(uint16_t), cudaMemcpyHostToDevice);
  if (ce != cudaSuccess) {
    if (m->arena) cudaFree(m->arena);
    if (m->tc_arena) cudaFree(m->tc_arena);
    delete m;
    return set_error(LTR_E_CUDA, std::string("ltr_create: ") + cudaGetErrorString(ce));
  }
  float* B = m->arena;
  uint16_t* TB = m->tc_arena;
  m->wpe = {B + wpe_o.w1, B + wpe_o.b1, bind_lin(wpe_o.l2, B, TB), bind_lin(wpe_o.l3, B, TB), bind_lin(wpe_o.l4, B, TB),
            bind_lin(wpe_o.l5, B, TB)};
  m->lpe.head = {B + lpe_o.w[0], B + lpe_o.b[0], B + lpe_o.w[1], B + lpe_o.b[1], B + lpe_o.w[2], B + lpe_o.b[2]};
  m->lpe.l4 = bind_lin(lpe_o.l4, B, TB);
  m->lpe.l5 = bind_lin(lpe_o.l5, B, TB);
  m->U = B + oU; m->s_cls = B + oS; m->cls = B + oC;
  m->wv = bind_lin(oWv, B, TB);
  m->wfc = bind_lin(oWfc, B, TB);
  m->ln1g = B + oL1g; m->ln1b = B + oL1b;
  m->w1 = bind_lin(oW1, B, TB);
  m->w2 = bind_lin(oW2, B, TB);
  m->ln2g = B + oL2g; m->ln2b = B + oL2b;
  for (auto& o : so)
    m->sig.push_back({bind_lin(o.qkv, B, TB), bind_lin(o.mlp1, B, TB), bind_lin(o.mlp2, B, TB)});
  m->wf = bind_lin(oWf, B, TB);
  *out = m;
  return LTR_OK;
}

void ltr_destroy(LtrModel* m) {
  if (!m) return;
  cudaSetDevice(m->device);
  if (m->arena) cudaFree(m->arena);
  if (m->tc_arena) cudaFree(m->tc_arena);
  delete m;
}

int64_t ltr_encode_workspace_bytes(const LtrModel* m, int32_t n_images, int32_t n_lines, int32_t n_tokens) {
  (void)n_images;
  if (!m || n_lines < 0 || n_tokens < 1) return set_error(LTR_E_INVALID, "ltr_encode_workspace_bytes: bad argument");
  return carve(m, n_lines, nullptr).bytes + 256;
}

int64_t ltr_desc_tiles_bytes(int32_t n_lines) {
  if (n_lines < 0) return set_error(LTR_E_INVALID, "ltr_desc_tiles_bytes: bad argument");
  return align_up(n_lines, 128) * MT_D * 2 * 2;   // hi + lo plane, bf16
}

int ltr_encode(LtrModel* m, const LtrEncodeInput* in, const LtrEncodeOutput* out, void* workspace, int64_t workspace_bytes,
               void* stream) {
  if (!m || !in || !out) return set_error(LTR_E_INVALID, "ltr_encode: null argument");
  if (in->n_lines == 0 || in->n_images == 0) return LTR_OK;
  if (in->n_tokens < 1 || in->n_tokens > 128) return set_error(LTR_E_UNSUPPORTED, "ltr_encode: n_tokens must be in 1..128");
  if (!in->sublines || !in->resp || !in->angle || !in->pnt || !in->desc || !in->score)
    return set_error(LTR_E_INVALID, "ltr_encode: null input tensor");
  if ((in->cu_lines_host == nullptr) != (in->cu_lines_dev == nullptr))
    return set_error(LTR_E_INVALID, "ltr_encode: cu_lines_host and cu_lines_dev must be given together");
  if (!in->cu_lines_host && (int64_t)in->lines_per_image * in->n_images != in->n_lines)
    return set_error(LTR_E_INVALID, "ltr_encode: uniform batch needs n_lines == n_images * lines_per_image");
  if (in->cu_lines_host && (in->cu_lines_host[0] != 0 || in->cu_lines_host[in->n_images] != in->n_lines))
    return set_error(LTR_E_INVALID, "ltr_encode: cu_lines must start at 0 and end at n_lines");
  if (!(in->image_width > 0.f) || !(in->image_height > 0.f)) return set_error(LTR_E_INVALID, "ltr_encode: bad image shape");
  if (out->desc_tiles && (out->desc_cf || !out->desc_rows))
    return set_error(LTR_E_UNSUPPORTED, "ltr_encode: desc_tiles needs desc_rows and no desc_cf");
  if (out->desc_tiles && (reinterpret_cast<uintptr_t>(out->desc_tiles) & 15))
    return set_error(LTR_E_INVALID, "ltr_encode: desc_tiles must be 16-byte aligned");
  LTR_CUDA_TRY(cudaSetDevice(m->device));
  char* base = reinterpret_cast<char*>(align_up(reinterpret_cast<int64_t>(workspace), 256));
  EncodeWs w = carve(m, in->n_lines, base);
  if (!workspace || (base - (char*)workspace) + w.bytes > workspace_bytes)
    return set_error(LTR_E_WORKSPACE, "ltr_encode: workspace too small, need " + std::to_string(w.bytes + 256));
  return encode_impl(m, *in, out->desc_cf, out->desc_rows, out->desc_tiles, w, as_stream(stream));
}

// ---- tensor-core matcher plumbing (d == 256) ----
struct MatchPlan {
  int mx[2], tmax[2], total[2];
  bool direct[2];       // side uses the caller's tile image (written by ltr_encode)
  ActImg img[2];
  uint2* slot[2];
  float* sq[2];
  int* done;
  int64_t bytes;
};

// Scratch carve-up of one match.  ix == nullptr: a batch of pairs; a side either reads the caller's tile image
// (written by ltr_encode) or is converted into the scratch.  ix != nullptr: a pair list over image pools; both operands
// are the caller's image-aligned tile images, so the scratch is the per-(pair, line) argmin slots (not needed with
// key-line merging, whose decisions run on dist_key).
static MatchPlan plan_match(const LtrMatchInput& in, const LtrPairIndex* ix, char* base) {
  MatchPlan pl{};
  const int P = in.n_pairs;
  const int n[2] = {in.n0, in.n1};
  const int mxn[2] = {in.max_n0, in.max_n1};
  const int tot[2] = {ix ? ix->total_out0 : in.total_n0, ix ? ix->total_out1 : in.total_n1};
  const void* tiles[2] = {ix ? ix->tiles0 : in.tiles0, ix ? ix->tiles1 : in.tiles1};
  const int64_t tl[2] = {ix ? (int64_t)ix->n_tiles0 * 128 : in.tiles_lines0,
                         ix ? (int64_t)ix->n_tiles1 * 128 : in.tiles_lines1};
  const int tr0[2] = {in.tiles_row0_0, in.tiles_row0_1};
  const bool varlen = in.cu0 != nullptr;
  const bool slots = !ix || in.sub_off0 == nullptr;
  int64_t off = 0;
  auto take = [&](int64_t bytes) {
    char* p = base + off;
    off = align_up(off + bytes, 1024);
    return p;
  };
  for (int s = 0; s < 2; ++s) {
    pl.mx[s] = varlen ? mxn[s] : n[s];
    pl.tmax[s] = cdiv(pl.mx[s], 128);
    pl.total[s] = varlen ? tot[s] : P * n[s];
    pl.direct[s] = ix || (tiles[s] && !varlen && in.dist_mode == 0 && n[s] % 128 == 0 && tr0[s] % 128 == 0 && tr0[s] >= 0 &&
                          (int64_t)tr0[s] + (int64_t)P * n[s] <= align_up(tl[s], 128));
    if (pl.direct[s]) {
      pl.img[s] = tiles_image(const_cast<void*>(tiles[s]), tl[s]);
    } else {
      const int64_t plane = (int64_t)P * pl.tmax[s] * 128 * MT_D;   // bf16 elements
      pl.img[s].hi = reinterpret_cast<__nv_bfloat16*>(take(plane * 2));
      pl.img[s].lo = reinterpret_cast<__nv_bfloat16*>(take(plane * 2));
      pl.img[s].kblocks = MT_KB;
    }
    pl.slot[s] = slots ? reinterpret_cast<uint2*>(take((int64_t)std::max(pl.total[s], 1) * 8)) : nullptr;
    pl.sq[s] = !ix && in.dist_mode == 1 ? reinterpret_cast<float*>(take((int64_t)std::max(pl.total[s], 1) * 4)) : nullptr;
  }
  pl.done = reinterpret_cast<int*>(take(256));
  pl.bytes = off;
  return pl;
}

static const char* check_match_input(const LtrMatchInput* in) {
  if (in->d <= 0 || in->d % 16) return "ltr_match: descriptor dim must be a multiple of 16";
  const bool seg = in->sub_off0 != nullptr || in->sub_off1 != nullptr;
  if (seg && (!in->sub_off0 || !in->sub_off1 || !in->cuk0 || !in->cuk1 || !in->cu0 || !in->cu1))
    return "ltr_match: keyline merging needs sub_off0/1, cuk0/1 and cu0/1";
  if ((in->cu0 == nullptr) != (in->cu1 == nullptr)) return "ltr_match: cu0/cu1 must be given together";
  if (in->dist_mode != 0 && in->dist_mode != 1) return "ltr_match: dist_mode must be 0 or 1";
  if (in->dist_mode == 1 && (in->d != MT_D || seg)) return "ltr_match: dist_mode 1 needs d == 256 and no keyline merging";
  if (in->d == MT_D && in->cu0 && (in->total_n0 < 0 || in->total_n1 < 0)) return "ltr_match: total_n0/total_n1 required with cu0/cu1";
  return nullptr;
}

// a descriptor dimension that is not a multiple of 16 is a valid request the kernels do not serve
static int match_input_code(const LtrMatchInput* in) { return in->d > 0 && in->d % 16 ? LTR_E_UNSUPPORTED : LTR_E_INVALID; }

// The matcher kernels put the pair count in grid y or z, and segmean_kernel covers side 0's key lines with grid y in
// blocks of 8: counts above what those grid dimensions hold are valid requests the kernels do not serve, refused
// (LTR_E_UNSUPPORTED) before any CUDA call.  Callers with more pairs split them into calls (engine.plan_chunks).
constexpr int kMaxGridYZ = 65535;
static int check_grid_limits(const char* who, int64_t n_pairs, bool seg, int64_t max_k0) {
  if (n_pairs > kMaxGridYZ) return set_error(LTR_E_UNSUPPORTED, std::string(who) + ": at most 65535 pairs per call");
  if (seg && max_k0 > 8LL * kMaxGridYZ)
    return set_error(LTR_E_UNSUPPORTED, std::string(who) + ": key-line merging takes at most 8 * 65535 side-0 key lines per pair");
  return LTR_OK;
}
static int check_match_limits(const char* who, const LtrMatchInput* in) {
  return check_grid_limits(who, in->n_pairs, in->sub_off0 != nullptr, in->max_k0);
}

}  // extern "C"

// launch sequence of the tensor-core matcher; returns 0 or an error code.  ix != nullptr: pair list over image
// pools (ltr_match_indexed), both sides read the caller's image-aligned tiles
static int run_match_tc(const LtrMatchInput& in, const LtrMatchOutput& out, const MatchPlan& pl, bool seg, long long stride_key,
                        cudaStream_t s, const LtrPairIndex* ix = nullptr) {
  const int P = in.n_pairs;
  const bool want_nn = out.matches0 != nullptr && !seg;
  const bool both = want_nn && in.mutual;
  if (pl.mx[0] > 0 && pl.mx[1] > 0) {
    if (!pl.direct[0] || !pl.direct[1]) {
      DescTilesArgs da{};
      da.layout = in.layout;
      const float* d[2] = {in.desc0, in.desc1};
      const int* cu[2] = {in.cu0, in.cu1};
      const int n[2] = {in.n0, in.n1};
      int tm = 0;
      for (int sd = 0; sd < 2; ++sd) {
        da.d[sd] = d[sd]; da.cu[sd] = cu[sd]; da.n[sd] = n[sd]; da.img[sd] = pl.img[sd];
        da.tmax[sd] = pl.direct[sd] ? 0 : pl.tmax[sd];
        da.sq[sd] = pl.sq[sd];
        tm = std::max(tm, da.tmax[sd]);
      }
      LTR_TRY(launch(KC_DESC_TILES, true, desc_tiles_kernel, dim3(tm * 4, P, 2), dim3(256), 0, s, da));
    }
    MatchTcArgs ma{};
    const int* cu[2] = {in.cu0, in.cu1};
    const int n[2] = {in.n0, in.n1};
    const int tr0[2] = {in.tiles_row0_0, in.tiles_row0_1};
    for (int sd = 0; sd < 2; ++sd) {
      ma.s[sd].img = pl.img[sd]; ma.s[sd].cu = cu[sd]; ma.s[sd].n = n[sd];
      ma.s[sd].tile_mode = pl.direct[sd] ? 1 : 0; ma.s[sd].tile_row0 = pl.direct[sd] ? tr0[sd] : 0;
      ma.s[sd].tmax = pl.tmax[sd]; ma.s[sd].sq = pl.sq[sd]; ma.s[sd].slot = pl.slot[sd];
      if (ix) {
        ma.s[sd].tile_mode = 2; ma.s[sd].tile_row0 = 0;
        ma.s[sd].pimg = sd ? ix->img1 : ix->img0;
        ma.s[sd].tile_off = sd ? ix->tile_off1 : ix->tile_off0;
        ma.s[sd].out_off = sd ? ix->out_off1 : ix->out_off0;
      }
    }
    ma.dist_mode = in.dist_mode;
    ma.thr = in.nn_thresh;
    ma.dist = seg ? out.dist_sub : out.dist_key;
    ma.dist_stride = seg ? (long long)pl.mx[0] * pl.mx[1] : stride_key;
    ma.counts = want_nn ? out.counts : nullptr;
    ma.done = want_nn ? pl.done : nullptr;
    ma.n_pairs = P;
    LTR_TRY(launch(KC_MATCH_TC, true, match_tc_kernel, dim3(pl.tmax[0] + (both ? pl.tmax[1] : 0), P), dim3(MT_THREADS),
                   (size_t)MT_SMEM, s, ma));
  } else if (want_nn) {
    LTR_CUDA_TRY(cudaMemsetAsync(out.counts, 0, sizeof(int) * P, s));
    LTR_CUDA_TRY(cudaMemsetAsync(pl.done, 0, sizeof(int), s));
  }
  if (want_nn && pl.mx[0] > 0 && pl.mx[1] > 0) {
    // exact fp32 re-check of the lines whose tensor-core result match_tc_kernel flagged, written back into their slots
    MatchExactArgs xa{};
    xa.d[0] = in.desc0; xa.d[1] = in.desc1; xa.layout = in.layout;
    xa.cu[0] = in.cu0; xa.cu[1] = in.cu1; xa.n[0] = in.n0; xa.n[1] = in.n1;
    xa.sq[0] = pl.sq[0]; xa.sq[1] = pl.sq[1]; xa.dist_mode = in.dist_mode;
    xa.slot[0] = pl.slot[0]; xa.slot[1] = pl.slot[1];
    xa.thr = in.nn_thresh; xa.mutual = in.mutual;
    if (ix) {
      xa.pimg[0] = ix->img0; xa.pimg[1] = ix->img1;
      xa.out_off[0] = ix->out_off0; xa.out_off[1] = ix->out_off1;
    }
    const int windows = std::min(cdiv(std::max(pl.mx[0], in.mutual ? pl.mx[1] : 0), MX_WIN), 65535);
    LTR_TRY(launch(KC_MATCH_EXACT, true, match_exact_kernel, dim3(P, 2, windows), dim3(256), (size_t)MX_SMEM, s, xa));
  }
  if (want_nn && pl.mx[0] > 0) {
    MatchTailArgs ta{};
    ta.cu[0] = in.cu0; ta.cu[1] = in.cu1; ta.n[0] = in.n0; ta.n[1] = in.n1;
    ta.slot[0] = pl.slot[0]; ta.slot[1] = pl.slot[1];
    ta.thr = in.nn_thresh; ta.mutual = in.mutual;
    ta.matches0 = out.matches0; ta.scores0 = out.scores0; ta.nn1 = out.nn1; ta.counts = out.counts;
    ta.max0 = pl.mx[0];
    ta.done = pl.done; ta.n_pairs = P; ta.world = 1;
    if (ix) {
      ta.pimg[0] = ix->img0; ta.pimg[1] = ix->img1;
      ta.out_off[0] = ix->out_off0; ta.out_off[1] = ix->out_off1;
    }
    if (out.gather && out.gather->world > 1) {
      const LtrPeerGather& g = *out.gather;
      ta.mc_base = reinterpret_cast<int*>(g.mc_base);
      ta.peer_bases = reinterpret_cast<int* const*>(g.peer_bases);
      ta.rank = g.rank; ta.world = g.world; ta.gslot = g.slot; ta.epoch = g.epoch;
    }
    LTR_TRY(launch(KC_MATCH_TAIL, true, match_tail_kernel, dim3(cdiv(pl.mx[0] + (in.mutual ? pl.mx[1] : 0), 256), P),
                   dim3(256), 0, s, ta));
  }
  return 0;
}

static int launch_segmean(const SegMeanArgs& a, int max_k0, int max_k1, int n_pairs, cudaStream_t s) {
  return launch(KC_SEGMEAN, false, segmean_kernel, dim3(cdiv(max_k1, 32), cdiv(max_k0, 8), n_pairs), dim3(256), 0, s, a);
}

// the output checks both matcher entries share; `who` (the entry's name) prefixes the message
static int check_match_output(const char* who, const LtrMatchInput& in, const LtrMatchOutput& out) {
  const std::string w(who);
  if (out.matches0 && (!out.scores0 || !out.nn1 || !out.counts))
    return set_error(LTR_E_INVALID, w + ": matches0 needs scores0, nn1 and counts");
  if (!out.matches0 && !out.dist_key) return set_error(LTR_E_INVALID, w + ": nothing to compute (matches0 and dist_key are NULL)");
  if (in.sub_off0 && (!out.dist_sub || !out.dist_key)) return set_error(LTR_E_INVALID, w + ": keyline merging needs dist_sub and dist_key");
  return LTR_OK;
}

// Everything after an entry's own checks: the match of a batch of pairs (ix == nullptr, ltr_match) or of a pair list
// over two image pools (ltr_match_indexed).  d != 256 (ltr_match only) runs the fp32 FMA distance tiles instead of the
// tensor-core matcher.  `who` prefixes every error message.
static int run_match(const char* who, const LtrMatchInput& in, const LtrPairIndex* ix, const LtrMatchOutput& out,
                     int32_t device, void* stream) {
  const bool seg = in.sub_off0 != nullptr;
  const int mx0 = in.cu0 ? in.max_n0 : in.n0, mx1 = in.cu1 ? in.max_n1 : in.n1;
  const int mk0 = seg ? in.max_k0 : mx0, mk1 = seg ? in.max_k1 : mx1;
  const long long stride_key = in.dist_pair_stride > 0 ? in.dist_pair_stride : (long long)mk0 * mk1;
  const bool null_desc = mx0 > 0 && mx1 > 0 && (!in.desc0 || !in.desc1);
  // a pair list is refused before any CUDA call; ltr_match selects its device first
  if (ix && null_desc) return set_error(LTR_E_INVALID, std::string(who) + ": null descriptors");
  LTR_CUDA_TRY(cudaSetDevice(device));
  if (null_desc) return set_error(LTR_E_INVALID, std::string(who) + ": null descriptors");
  cudaStream_t s = as_stream(stream);
  if (in.d == MT_D) {
    // a slot keeps a line index in 30 bits (match_tc.cuh)
    if (mx0 >= (1 << 30) || mx1 >= (1 << 30))
      return set_error(LTR_E_INVALID, std::string(who) + ": a pair side has 2^30 lines or more");
    char* base = reinterpret_cast<char*>(align_up(reinterpret_cast<int64_t>(out.workspace), 1024));
    MatchPlan pl = plan_match(in, ix, base);
    if (!out.workspace || (base - (char*)out.workspace) + pl.bytes > out.workspace_bytes)
      return set_error(LTR_E_WORKSPACE, std::string(who) + ": workspace too small, need " + std::to_string(pl.bytes + 1024));
    LTR_TRY(run_match_tc(in, out, pl, seg, stride_key, s, ix));
    if (!seg) return LTR_OK;
  } else if (mx0 > 0 && mx1 > 0) {
    // generic descriptor dimension: fp32 FMA distance tiles
    DistArgs da{};
    da.d0 = in.desc0; da.d1 = in.desc1; da.layout = in.layout; da.d = in.d;
    da.cu0 = in.cu0; da.cu1 = in.cu1; da.n0 = in.n0; da.n1 = in.n1;
    da.out = seg ? out.dist_sub : out.dist_key;
    da.stride = seg ? (long long)mx0 * mx1 : stride_key;
    dim3 grid(cdiv(mx0, DK_BM), cdiv(mx1, DK_BN), in.n_pairs);
    LTR_TRY(launch(KC_DIST, true, in.layout == LTR_LAYOUT_CHANNEL_FIRST ? dist_kernel<true> : dist_kernel<false>, grid,
                   dim3(DK_THREADS), 0, s, da));
  }
  if (seg && mx0 > 0 && mx1 > 0 && mk0 > 0 && mk1 > 0)
    LTR_TRY(launch_segmean({out.dist_sub, (long long)mx0 * mx1, out.dist_key, stride_key, in.cuk0, in.cuk1, in.sub_off0,
                            in.sub_off1, ix ? ix->img0 : nullptr, ix ? ix->img1 : nullptr},
                           mk0, mk1, in.n_pairs, s));
  if (!out.matches0) return LTR_OK;
  // a pair list's per-pair output offsets play the role cuk0/cuk1 play for a batch: the NN kernels need no indirection
  NNArgs na{};
  na.dist = out.dist_key; na.stride = stride_key;
  na.cuk0 = ix ? ix->out_off0 : seg ? in.cuk0 : in.cu0; na.cuk1 = ix ? ix->out_off1 : seg ? in.cuk1 : in.cu1;
  na.n0 = in.n0; na.n1 = in.n1; na.thr = in.nn_thresh; na.mutual = in.mutual;
  na.matches0 = out.matches0; na.scores0 = out.scores0; na.nn1 = out.nn1; na.counts = out.counts;
  return run_nn(na, in.n_pairs, mk0, mk1, s);
}

extern "C" {

int64_t ltr_match_workspace_bytes(const LtrMatchInput* in) {
  if (!in) return set_error(LTR_E_INVALID, "ltr_match_workspace_bytes: null argument");
  if (const char* e = check_match_input(in)) return set_error(match_input_code(in), e);
  if (int rc = check_match_limits("ltr_match_workspace_bytes", in)) return rc;
  if (in->n_pairs <= 0 || in->d != MT_D) return 0;
  return plan_match(*in, nullptr, nullptr).bytes + 1024;
}

int ltr_match(const LtrMatchInput* in, const LtrMatchOutput* out, int32_t device, void* stream) {
  if (!in || !out) return set_error(LTR_E_INVALID, "ltr_match: null argument");
  if (in->n_pairs <= 0) return LTR_OK;
  if (const char* e = check_match_input(in)) return set_error(match_input_code(in), e);
  LTR_TRY(check_match_limits("ltr_match", in));
  LTR_TRY(check_match_output("ltr_match", *in, *out));
  const bool seg = in->sub_off0 != nullptr;
  const bool tc = in->d == MT_D;
  const bool want_nn = out->matches0 != nullptr;
  if (out->gather && out->gather->world > 1) {
    const LtrPeerGather& g = *out->gather;
    if (seg || !tc || !want_nn) return set_error(LTR_E_UNSUPPORTED, "ltr_match: gather needs d == 256, no keyline merging, matches0");
    if ((!g.mc_base && !g.peer_bases) || g.rank < 0 || g.rank >= g.world || g.slot < 0 || g.slot >= LTR_GATHER_SLOTS || g.epoch <= 0)
      return set_error(LTR_E_INVALID, "ltr_match: bad LtrPeerGather");
    if ((in->cu0 ? in->max_n0 : in->n0) <= 0) return set_error(LTR_E_UNSUPPORTED, "ltr_match: gather needs a non-empty side 0");
  }
  if (!tc && !out->dist_key) return set_error(LTR_E_INVALID, "ltr_match: dist_key is required when d != 256");
  return run_match("ltr_match", *in, nullptr, *out, device, stream);
}

int64_t ltr_image_tiles_bytes(int32_t n_images, const int32_t* cu_host) {
  if (n_images < 0 || (n_images > 0 && !cu_host)) return set_error(LTR_E_INVALID, "ltr_image_tiles_bytes: bad argument");
  int64_t tiles = 0;
  for (int i = 0; i < n_images; ++i) {
    const int L = cu_host[i + 1] - cu_host[i];
    if (L < 0) return set_error(LTR_E_INVALID, "ltr_image_tiles_bytes: cu must not decrease");
    tiles += cdiv(L, 128);
  }
  return tiles * 128 * MT_D * 2 * 2;   // hi + lo plane, bf16
}

int ltr_image_tiles(const float* desc, int32_t layout, const int32_t* cu_dev, const int32_t* tile_off_dev, int32_t n_images,
                    int32_t max_n, int32_t n_tiles, void* out, int32_t device, void* stream) {
  if (n_images < 0 || max_n < 0 || n_tiles < 0) return set_error(LTR_E_INVALID, "ltr_image_tiles: negative count");
  if (layout != LTR_LAYOUT_ROWS && layout != LTR_LAYOUT_CHANNEL_FIRST) return set_error(LTR_E_INVALID, "ltr_image_tiles: bad layout");
  if (n_images == 0 || max_n == 0 || n_tiles == 0) return LTR_OK;
  if (!desc || !cu_dev || !tile_off_dev || !out) return set_error(LTR_E_INVALID, "ltr_image_tiles: null argument");
  if (reinterpret_cast<uintptr_t>(out) & 15) return set_error(LTR_E_INVALID, "ltr_image_tiles: out must be 16-byte aligned");
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  DescTilesArgs da{};
  da.layout = layout;
  da.d[0] = desc; da.cu[0] = cu_dev; da.tile_off[0] = tile_off_dev;
  da.img[0] = tiles_image(out, (int64_t)n_tiles * 128);
  da.tmax[0] = cdiv(max_n, 128);
  return launch(KC_DESC_TILES, true, desc_tiles_kernel, dim3(da.tmax[0] * 4, n_images, 1), dim3(256), 0, s, da);
}

static const char* check_match_indexed(const LtrMatchInput* in, const LtrPairIndex* ix) {
  if (in->cu0 == nullptr || in->cu1 == nullptr) return "ltr_match_indexed: cu0 and cu1 (image offsets of the pools) are required";
  const bool seg = in->sub_off0 != nullptr || in->sub_off1 != nullptr;
  if (seg && (!in->sub_off0 || !in->sub_off1 || !in->cuk0 || !in->cuk1))
    return "ltr_match_indexed: keyline merging needs sub_off0/1 and cuk0/1";
  if (!ix->img0 || !ix->img1 || !ix->out_off0 || !ix->out_off1) return "ltr_match_indexed: img0/1 and out_off0/1 are required";
  if (in->max_n0 < 0 || in->max_n1 < 0 || ix->n_tiles0 < 0 || ix->n_tiles1 < 0 || ix->total_out0 < 0 || ix->total_out1 < 0)
    return "ltr_match_indexed: negative count";
  if (in->max_n0 > 0 && in->max_n1 > 0 && (!ix->tiles0 || !ix->tiles1 || !ix->tile_off0 || !ix->tile_off1))
    return "ltr_match_indexed: tiles0/1 and tile_off0/1 (ltr_image_tiles) are required";
  return nullptr;
}

int64_t ltr_match_indexed_workspace_bytes(const LtrMatchInput* in, const LtrPairIndex* idx) {
  if (!in || !idx) return set_error(LTR_E_INVALID, "ltr_match_indexed_workspace_bytes: null argument");
  if (const char* e = check_match_indexed(in, idx)) return set_error(LTR_E_INVALID, e);
  if (int rc = check_match_limits("ltr_match_indexed_workspace_bytes", in)) return rc;
  if (in->n_pairs <= 0) return 0;
  return plan_match(*in, idx, nullptr).bytes + 1024;
}

int ltr_match_indexed(const LtrMatchInput* in, const LtrPairIndex* idx, const LtrMatchOutput* out, int32_t device, void* stream) {
  if (!in || !idx || !out) return set_error(LTR_E_INVALID, "ltr_match_indexed: null argument");
  if (in->d != MT_D || in->dist_mode != 0)
    return set_error(LTR_E_UNSUPPORTED, "ltr_match_indexed: needs d == 256 and dist_mode 0");
  if (out->gather && out->gather->world > 1) return set_error(LTR_E_UNSUPPORTED, "ltr_match_indexed: gather is not supported");
  if (in->n_pairs <= 0) return LTR_OK;
  if (const char* e = check_match_indexed(in, idx)) return set_error(LTR_E_INVALID, e);
  LTR_TRY(check_match_limits("ltr_match_indexed", in));
  LTR_TRY(check_match_output("ltr_match_indexed", *in, *out));
  return run_match("ltr_match_indexed", *in, idx, *out, device, stream);
}

int ltr_gather_wait(const void* local_base, int32_t world, int32_t n_pairs, int32_t slot, int32_t epoch, int32_t* out,
                    int32_t device, void* stream) {
  if (!local_base || !out || world < 1 || world > 256 || n_pairs < 1 || slot < 0 || slot >= LTR_GATHER_SLOTS)
    return set_error(LTR_E_INVALID, "ltr_gather_wait: bad argument");
  LTR_CUDA_TRY(cudaSetDevice(device));
  return launch(KC_MUTUAL, true, gather_wait_kernel, dim3(1), dim3(256), 0, as_stream(stream),
                reinterpret_cast<const int*>(local_base), world, n_pairs, slot, epoch, out);
}

int ltr_match_distmat(const float* dist, int32_t n_pairs, int32_t n0, int32_t n1, int64_t dist_pair_stride, float nn_thresh,
                      int32_t mutual, int32_t* matches0, float* scores0, int32_t* nn1, int32_t* counts, int32_t device,
                      void* stream) {
  if (n_pairs <= 0) return LTR_OK;
  LTR_TRY(check_grid_limits("ltr_match_distmat", n_pairs, false, 0));
  if (!matches0 || !scores0 || !nn1 || !counts) return set_error(LTR_E_INVALID, "ltr_match_distmat: null output");
  if (n0 > 0 && n1 > 0 && !dist) return set_error(LTR_E_INVALID, "ltr_match_distmat: null distance matrix");
  LTR_CUDA_TRY(cudaSetDevice(device));
  NNArgs na{};
  na.dist = dist; na.stride = dist_pair_stride > 0 ? dist_pair_stride : (long long)n0 * n1;
  na.n0 = n0; na.n1 = n1; na.thr = nn_thresh; na.mutual = mutual;
  na.matches0 = matches0; na.scores0 = scores0; na.nn1 = nn1; na.counts = counts;
  return run_nn(na, n_pairs, n0, n1, as_stream(stream));
}

int ltr_merge_sublines(const float* dist_sub, int64_t stride_sub, int32_t n_pairs, const int32_t* cuk0,
                       const int32_t* cuk1, const int32_t* sub_off0, const int32_t* sub_off1, int32_t max_k0,
                       int32_t max_k1, float* dist_key, int64_t stride_key, int32_t device, void* stream) {
  if (n_pairs <= 0 || max_k0 <= 0 || max_k1 <= 0) return LTR_OK;
  LTR_TRY(check_grid_limits("ltr_merge_sublines", n_pairs, true, max_k0));
  if (!dist_sub || !cuk0 || !cuk1 || !sub_off0 || !sub_off1 || !dist_key)
    return set_error(LTR_E_INVALID, "ltr_merge_sublines: null argument");
  LTR_CUDA_TRY(cudaSetDevice(device));
  return launch_segmean({dist_sub, stride_sub, dist_key, stride_key, cuk0, cuk1, sub_off0, sub_off1}, max_k0, max_k1, n_pairs,
                        as_stream(stream));
}

int ltr_tokenize_batch(const LtrTokenizeBatchInput* in, float* sublines, float* pnt, float* mask, float* resp,
                       float* angle, float* desc, float* score, int32_t device, void* stream) {
  if (!in) return set_error(LTR_E_INVALID, "ltr_tokenize_batch: null argument");
  if (in->n_images < 0 || in->n_keylines < 0 || in->n_sublines < 0)
    return set_error(LTR_E_INVALID, "ltr_tokenize_batch: negative count");
  // a batch without key lines has empty outputs, whose pointers may be NULL
  if (in->n_images == 0 || in->n_sublines == 0 || in->n_keylines == 0) return LTR_OK;
  if (!sublines || !pnt || !mask || !resp || !angle || !desc || !score)
    return set_error(LTR_E_INVALID, "ltr_tokenize_batch: null output");
  if (in->n_tokens < 1 || in->n_tokens > 128 || in->desc_channels != 256)
    return set_error(LTR_E_UNSUPPORTED, "ltr_tokenize_batch: n_tokens in 1..128 and 256 descriptor channels required");
  if (!in->sp || !in->ep || !in->ep_clipped || !in->length || !in->angle || !in->n_tok || !in->sub0 || !in->sub2line ||
      !in->line_image || !in->images || !in->cu_sublines)
    return set_error(LTR_E_INVALID, "ltr_tokenize_batch: null input array");
  const int32_t* cu = in->cu_sublines;
  if (cu[0] != 0 || cu[in->n_images] != in->n_sublines)
    return set_error(LTR_E_INVALID, "ltr_tokenize_batch: cu_sublines must start at 0 and end at n_sublines");
  for (int i = 0; i < in->n_images; ++i) {
    if (cu[i + 1] < cu[i]) return set_error(LTR_E_INVALID, "ltr_tokenize_batch: cu_sublines must not decrease");
    if (cu[i + 1] > cu[i] && (!in->images[i].dense_desc || !in->images[i].dense_score))
      return set_error(LTR_E_INVALID, "ltr_tokenize_batch: null map of an image with key lines");
  }
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  TokLines L{in->sp, in->ep, in->ep_clipped, in->length, in->angle, in->n_tok, in->sub0, in->sub2line, in->line_image,
             in->n_keylines, in->n_sublines, in->n_tokens};
  const auto image = [](const LtrTokenizeImage& g) {
    return TokImage{g.dense_desc, g.dense_score, g.token_distance, g.desc_h, g.desc_w, g.score_h, g.score_w};
  };
  if (in->n_images == 1) {   // one image: a 40-byte table, and every line is in it
    TokImages<1> I{{image(in->images[0])}, 0};
    return launch_tokenize(L, I, 0, in->n_sublines, in->align_corners, sublines, pnt, mask, resp, angle, desc, score, s);
  }
  for (int i0 = 0; i0 < in->n_images; i0 += kTokImagesPerLaunch) {
    const int i1 = std::min(in->n_images, i0 + kTokImagesPerLaunch);
    TokImages<kTokImagesPerLaunch> I{};
    I.first = i0;
    for (int i = i0; i < i1; ++i) I.im[i - i0] = image(in->images[i]);
    LTR_TRY(launch_tokenize(L, I, cu[i0], cu[i1], in->align_corners, sublines, pnt, mask, resp, angle, desc, score, s));
  }
  return LTR_OK;
}

int ltr_line_gt(const LtrLineGtInput* in, const LtrLineGtOutput* out, int32_t device, void* stream) {
  if (!in || !out) return set_error(LTR_E_INVALID, "ltr_line_gt: null argument");
  if (in->n_pairs < 0 || in->max_n0 < 0 || in->max_n1 < 0) return set_error(LTR_E_INVALID, "ltr_line_gt: negative count");
  if (out->assign && out->assign_stride < (int64_t)in->max_n0 * in->max_n1)
    return set_error(LTR_E_INVALID, "ltr_line_gt: assign_stride < max_n0 * max_n1");
  if (in->n_pairs == 0) return LTR_OK;
  if (!out->n_gt) return set_error(LTR_E_INVALID, "ltr_line_gt: null n_gt");
  if (in->pred0 && !out->tfpn) return set_error(LTR_E_INVALID, "ltr_line_gt: pred0 needs tfpn");
  if (!in->cu0 || !in->cu1 || !in->homography || !in->homography_inv)
    return set_error(LTR_E_INVALID, "ltr_line_gt: null input array");
  if ((in->max_n0 > 0 && !in->segs0) || (in->max_n1 > 0 && !in->segs1))
    return set_error(LTR_E_INVALID, "ltr_line_gt: null segments");
  for (const void* p : {(const void*)in->segs0, (const void*)in->segs1, (const void*)in->proj0, (const void*)in->proj1})
    if (reinterpret_cast<uintptr_t>(p) & 15) return set_error(LTR_E_INVALID, "ltr_line_gt: segments must be 16-byte aligned");
  if (cdiv(in->max_n0, LG_ROWS) > 65535) return set_error(LTR_E_INVALID, "ltr_line_gt: too many side-0 segments per pair");
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  LTR_CUDA_TRY(cudaMemsetAsync(out->n_gt, 0, sizeof(int32_t) * in->n_pairs, s));
  if (in->pred0) LTR_CUDA_TRY(cudaMemsetAsync(out->tfpn, 0, sizeof(int32_t) * 4 * in->n_pairs, s));
  if (in->max_n0 == 0) return LTR_OK;
  LineGtArgs a{in->segs0, in->segs1, in->cu0, in->cu1, in->homography, in->homography_inv, in->proj0, in->proj1, in->pred0,
               in->thres_reprojected, in->thres_angdiff, in->min_overlap_ratio, out->assign, (long long)out->assign_stride,
               out->n_gt, out->tfpn};
  const dim3 grid(in->n_pairs, cdiv(in->max_n0, LG_ROWS));
  return launch(KC_LINE_GT, true, out->assign ? line_gt_kernel<true> : line_gt_kernel<false>, grid, dim3(LG_ROWS), 0, s, a);
}

int ltr_triplet_loss(const LtrTripletInput* in, const LtrTripletOutput* out, int32_t device, void* stream) {
  if (!in || !out) return set_error(LTR_E_INVALID, "ltr_triplet_loss: null argument");
  if (in->d != MT_D) return set_error(LTR_E_UNSUPPORTED, "ltr_triplet_loss: descriptor dim must be 256");
  if (in->layout != LTR_LAYOUT_ROWS && in->layout != LTR_LAYOUT_CHANNEL_FIRST) return set_error(LTR_E_INVALID, "ltr_triplet_loss: bad layout");
  if (in->n_pairs < 0 || in->n0 < 0 || in->n1 < 0 || in->max_n0 < 0 || in->max_n1 < 0 || in->assign_ld < 0 || in->assign_stride < 0)
    return set_error(LTR_E_INVALID, "ltr_triplet_loss: negative count");
  if ((in->cu0 == nullptr) != (in->cu1 == nullptr)) return set_error(LTR_E_INVALID, "ltr_triplet_loss: cu0/cu1 must be given together");
  if (in->n_groups < 1 || (!in->group_off && in->n_groups != 1))
    return set_error(LTR_E_INVALID, "ltr_triplet_loss: n_groups must be >= 1 (1 without group_off)");
  const int mx0 = in->cu0 ? in->max_n0 : in->n0, mx1 = in->cu1 ? in->max_n1 : in->n1;
  if (mx0 >= (1 << 30) || mx1 >= (1 << 30)) return set_error(LTR_E_INVALID, "ltr_triplet_loss: a pair side has 2^30 lines or more");
  if (in->assign_ld > 0 && in->assign_ld < mx1) return set_error(LTR_E_INVALID, "ltr_triplet_loss: assign_ld < max_n1");
  if (in->assign_stride < (int64_t)mx0 * (in->assign_ld ? in->assign_ld : mx1))
    return set_error(LTR_E_INVALID, "ltr_triplet_loss: assign_stride < max_n0 * row pitch");
  if (in->n_pairs == 0) return LTR_OK;
  if (!out->pos || !out->neg || !out->state || !out->loss || !out->hardest_pos || !out->hardest_neg || !out->n_valid)
    return set_error(LTR_E_INVALID, "ltr_triplet_loss: null output");
  if (in->pred0 && !out->tfpn) return set_error(LTR_E_INVALID, "ltr_triplet_loss: pred0 needs tfpn");
  const bool lines = mx0 > 0 || mx1 > 0;
  if (lines && (!in->desc0 || !in->desc1 || !in->assign)) return set_error(LTR_E_INVALID, "ltr_triplet_loss: null descriptors or assign");
  if (in->layout == LTR_LAYOUT_ROWS && ((reinterpret_cast<uintptr_t>(in->desc0) | reinterpret_cast<uintptr_t>(in->desc1)) & 15))
    return set_error(LTR_E_INVALID, "ltr_triplet_loss: row descriptors must be 16-byte aligned");
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  if (in->pred0) LTR_CUDA_TRY(cudaMemsetAsync(out->tfpn, 0, sizeof(int32_t) * 4 * in->n_pairs, s));
  if (lines) {
    TripletArgs a{};
    a.d[0] = in->desc0; a.d[1] = in->desc1; a.layout = in->layout;
    a.cu[0] = in->cu0; a.cu[1] = in->cu1; a.n[0] = in->n0; a.n[1] = in->n1;
    a.assign = in->assign; a.assign_stride = in->assign_stride; a.assign_ld = in->assign_ld;
    a.match_thr = in->match_thr; a.unmatch_thr = in->unmatch_thr;
    a.pred0 = in->pred0;
    a.pos = out->pos; a.neg = out->neg; a.state = out->state; a.tfpn = out->tfpn;
    const int windows = std::min(cdiv(std::max(mx0, mx1), MX_R), 65535);
    LTR_TRY(launch(KC_TRIPLET, true, triplet_mine_kernel, dim3(in->n_pairs, 2, windows), dim3(256), (size_t)MX_SMEM, s, a));
  }
  TripletReduceArgs r{};
  r.cu[0] = in->cu0; r.cu[1] = in->cu1; r.n[0] = in->n0; r.n[1] = in->n1;
  r.group_off = in->group_off; r.n_pairs = in->n_pairs;
  r.pos = out->pos; r.neg = out->neg; r.state = out->state;
  r.loss = out->loss; r.hardest_pos = out->hardest_pos; r.hardest_neg = out->hardest_neg; r.n_valid = out->n_valid;
  return launch(KC_TRIPLET, true, triplet_reduce_kernel, dim3(in->n_groups), dim3(256), 0, s, r);
}

int ltr_homography(const LtrHomographyInput* in, const LtrHomographyOutput* out, int32_t device, void* stream) {
  if (!in || !out) return set_error(LTR_E_INVALID, "ltr_homography: null argument");
  if (in->n_pairs < 0 || in->max_rows_p < 0 || in->max_rows_l < 0)
    return set_error(LTR_E_INVALID, "ltr_homography: negative count");
  if (in->n_hypotheses < 1 || cdiv(in->n_hypotheses, HG_THREADS) > 65535)
    return set_error(LTR_E_INVALID, "ltr_homography: n_hypotheses must be in [1, 65535 * 128]");
  if (!(in->thresh > 0.0) || !std::isfinite(in->thresh)) return set_error(LTR_E_INVALID, "ltr_homography: thresh must be > 0");
  const int rows_p = in->use_points ? in->max_rows_p : 0, rows_l = in->use_lines ? in->max_rows_l : 0;
  const long long smem = hg_smem_bytes(rows_p, rows_l, true);
  if (smem > HG_SMEM_MAX)
    return set_error(LTR_E_UNSUPPORTED, "ltr_homography: a pair's correspondences need " + std::to_string(smem) +
                                             " bytes of shared memory (18 per keypoint row, 58 per segment row), over " +
                                             std::to_string(HG_SMEM_MAX));
  if (in->n_pairs == 0) return LTR_OK;
  if (!out->H || !out->valid || !out->n_inliers_p || !out->n_inliers_l || !out->hypothesis || !out->hypothesis_inliers ||
      !out->key)
    return set_error(LTR_E_INVALID, "ltr_homography: null output");
  if (!in->cu_p || !in->cu_l) return set_error(LTR_E_INVALID, "ltr_homography: null offsets");
  if (in->max_rows_p > 0 && (!in->matches_p || !out->inliers_p)) return set_error(LTR_E_INVALID, "ltr_homography: null point matches");
  if (in->max_rows_l > 0 && (!in->matches_l || !out->inliers_l)) return set_error(LTR_E_INVALID, "ltr_homography: null line matches");
  if (rows_p > 0 && (!in->pts0 || !in->pts1 || !in->pts_off0 || !in->pts_off1 || !in->n_pts1))
    return set_error(LTR_E_INVALID, "ltr_homography: null keypoint pools");
  if (rows_l > 0 && (!in->segs0 || !in->segs1 || !in->seg_off0 || !in->seg_off1 || !in->n_segs1))
    return set_error(LTR_E_INVALID, "ltr_homography: null segment pools");
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  HomographyArgs a{in->pts0, in->pts1, in->pts_off0, in->pts_off1, in->n_pts1, in->matches_p, in->cu_p,
                   in->segs0, in->segs1, in->seg_off0, in->seg_off1, in->n_segs1, in->matches_l, in->cu_l,
                   rows_p, rows_l, in->use_points != 0, in->use_lines != 0, in->thresh * in->thresh, in->n_hypotheses, (unsigned long long)in->seed,
                   reinterpret_cast<unsigned long long*>(out->key), out->H, out->valid, out->inliers_p, out->inliers_l,
                   out->n_inliers_p, out->n_inliers_l, out->hypothesis, out->hypothesis_inliers};
  LTR_CUDA_TRY(cudaMemsetAsync(out->key, 0, sizeof(uint64_t) * in->n_pairs, s));
  LTR_TRY(launch(KC_HOMOGRAPHY, true, homography_hyp_kernel, dim3(in->n_pairs, cdiv(in->n_hypotheses, HG_THREADS)),
                 dim3(HG_THREADS), (size_t)hg_smem_bytes(rows_p, rows_l, false), s, a));
  return launch(KC_HOMOGRAPHY, true, homography_refit_kernel, dim3(in->n_pairs), dim3(HG_REFIT_THREADS), (size_t)smem, s, a);
}

int ltr_essential(const LtrEssentialInput* in, const LtrEssentialOutput* out, int32_t device, void* stream) {
  if (!in || !out) return set_error(LTR_E_INVALID, "ltr_essential: null argument");
  if (in->n_pairs < 0 || in->max_rows_p < 0) return set_error(LTR_E_INVALID, "ltr_essential: negative count");
  if (in->n_hypotheses < 1 || cdiv(in->n_hypotheses, ESS_THREADS) > 65535)
    return set_error(LTR_E_INVALID, "ltr_essential: n_hypotheses must be in [1, 65535 * 128]");
  if (!(in->thresh > 0.0) || !std::isfinite(in->thresh)) return set_error(LTR_E_INVALID, "ltr_essential: thresh must be > 0");
  if (!(in->dist_thresh > 0.0)) return set_error(LTR_E_INVALID, "ltr_essential: dist_thresh must be > 0");
  const long long smem = ess_smem_bytes(in->max_rows_p, true);
  if (smem > ESS_SMEM_MAX)
    return set_error(LTR_E_UNSUPPORTED, "ltr_essential: a pair's correspondences need " + std::to_string(smem) +
                                            " bytes of shared memory (33 per keypoint row), over " +
                                            std::to_string(ESS_SMEM_MAX));
  if (in->n_pairs == 0) return LTR_OK;
  if (!out->E || !out->R || !out->t || !out->valid || !out->n_inliers || !out->n_cheirality || !out->hypothesis ||
      !out->hypothesis_inliers || !out->key)
    return set_error(LTR_E_INVALID, "ltr_essential: null output");
  if (!in->cu_p || !in->K0 || !in->K1) return set_error(LTR_E_INVALID, "ltr_essential: null offsets or intrinsics");
  if (in->max_rows_p > 0 && (!in->matches_p || !out->inliers_p || !in->pts0 || !in->pts1 || !in->pts_off0 ||
                             !in->pts_off1 || !in->n_pts1))
    return set_error(LTR_E_INVALID, "ltr_essential: null keypoint pools or matches");
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  EssentialArgs a{in->pts0, in->pts1, in->pts_off0, in->pts_off1, in->n_pts1, in->matches_p, in->cu_p, in->K0, in->K1,
                  in->max_rows_p, in->thresh, in->dist_thresh, in->n_hypotheses, (unsigned long long)in->seed,
                  reinterpret_cast<unsigned long long*>(out->key), out->E, out->R, out->t, out->valid, out->inliers_p,
                  out->n_inliers, out->n_cheirality, out->hypothesis, out->hypothesis_inliers};
  LTR_CUDA_TRY(cudaMemsetAsync(out->key, 0, sizeof(uint64_t) * in->n_pairs, s));
  LTR_TRY(launch(KC_ESSENTIAL, true, essential_hyp_kernel, dim3(in->n_pairs, cdiv(in->n_hypotheses, ESS_THREADS)),
                 dim3(ESS_THREADS), (size_t)ess_smem_bytes(in->max_rows_p, false), s, a));
  return launch(KC_ESSENTIAL, true, essential_pose_kernel, dim3(in->n_pairs), dim3(ESS_POSE_THREADS), (size_t)smem, s, a);
}

int ltr_fundamental(const LtrFundamentalInput* in, const LtrFundamentalOutput* out, int32_t device, void* stream) {
  if (!in || !out) return set_error(LTR_E_INVALID, "ltr_fundamental: null argument");
  if (in->n_pairs < 0 || in->max_rows_p < 0) return set_error(LTR_E_INVALID, "ltr_fundamental: negative count");
  if (in->n_hypotheses < 1 || cdiv(in->n_hypotheses, FM_THREADS) > 65535)
    return set_error(LTR_E_INVALID, "ltr_fundamental: n_hypotheses must be in [1, 65535 * 128]");
  if (!(in->thresh > 0.0) || !std::isfinite(in->thresh)) return set_error(LTR_E_INVALID, "ltr_fundamental: thresh must be > 0");
  if (!(in->min_overlap >= 0.0 && in->min_overlap <= 1.0))
    return set_error(LTR_E_INVALID, "ltr_fundamental: min_overlap must be in [0, 1]");
  const long long smem = fm_smem_bytes(in->max_rows_p, true);
  if (smem > FM_SMEM_MAX)
    return set_error(LTR_E_UNSUPPORTED, "ltr_fundamental: a pair's correspondences need " + std::to_string(smem) +
                                            " bytes of shared memory (18 per keypoint row), over " +
                                            std::to_string(FM_SMEM_MAX));
  if (in->n_pairs == 0) return LTR_OK;
  if (!out->F || !out->valid || !out->refit || !out->n_inliers || !out->n_lines_consistent || !out->hypothesis ||
      !out->hypothesis_inliers || !out->key)
    return set_error(LTR_E_INVALID, "ltr_fundamental: null output");
  if (!in->cu_p || !in->cu_l) return set_error(LTR_E_INVALID, "ltr_fundamental: null offsets");
  if (in->max_rows_p > 0 && (!in->matches_p || !out->inliers_p || !in->pts0 || !in->pts1 || !in->pts_off0 ||
                             !in->pts_off1 || !in->n_pts1))
    return set_error(LTR_E_INVALID, "ltr_fundamental: null keypoint pools or matches");
  if (in->max_rows_l > 0 && (!in->matches_l || !out->lines_consistent || !in->segs0 || !in->segs1 || !in->seg_off0 ||
                             !in->seg_off1 || !in->n_segs1))
    return set_error(LTR_E_INVALID, "ltr_fundamental: null segment pools or line matches");
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  FundamentalArgs a{in->pts0, in->pts1, in->pts_off0, in->pts_off1, in->n_pts1, in->matches_p, in->cu_p,
                    in->segs0, in->segs1, in->seg_off0, in->seg_off1, in->n_segs1, in->matches_l, in->cu_l,
                    in->max_rows_p, in->thresh * in->thresh, in->min_overlap, in->n_hypotheses,
                    (unsigned long long)in->seed, reinterpret_cast<unsigned long long*>(out->key), out->F, out->valid,
                    out->inliers_p, out->lines_consistent, out->refit, out->n_inliers, out->n_lines_consistent,
                    out->hypothesis, out->hypothesis_inliers};
  LTR_CUDA_TRY(cudaMemsetAsync(out->key, 0, sizeof(uint64_t) * in->n_pairs, s));
  LTR_TRY(launch(KC_FUNDAMENTAL, true, fundamental_hyp_kernel, dim3(in->n_pairs, cdiv(in->n_hypotheses, FM_THREADS)),
                 dim3(FM_THREADS), (size_t)fm_smem_bytes(in->max_rows_p, false), s, a));
  return launch(KC_FUNDAMENTAL, true, fundamental_fit_kernel, dim3(in->n_pairs), dim3(FM_FIT_THREADS), (size_t)smem, s, a);
}

// ltr_absolute_pose is this body with no line hypotheses; `who` names the entry in its errors.
static int absolute_pose(const char* who, const LtrAbsPoseInput* in, const LtrAbsPoseOutput* out, int n_line_hyp,
                         int32_t device, void* stream) {
  const std::string w = who;
  if (!in || !out) return set_error(LTR_E_INVALID, w + ": null argument");
  if (in->n_pairs < 0 || in->n_groups < 0 || in->max_rows_p < 0 || in->max_rows_l < 0)
    return set_error(LTR_E_INVALID, w + ": negative count");
  if (n_line_hyp < 0 || n_line_hyp > AP_LINE_MAX_HYP)
    return set_error(LTR_E_INVALID, w + ": n_line_hypotheses must be in [0, 2^21]");
  if (in->n_hypotheses < (n_line_hyp ? 0 : 1) || cdiv(in->n_hypotheses, AP_THREADS) > 65535)
    return set_error(LTR_E_INVALID, w + (n_line_hyp ? ": n_hypotheses must be in [0, 65535 * 128]"
                                                    : ": n_hypotheses must be in [1, 65535 * 128]"));
  if (n_line_hyp && !in->use_lines)
    return set_error(LTR_E_INVALID, w + ": line hypotheses need use_lines");
  if (!(in->thresh > 0.0) || !std::isfinite(in->thresh))
    return set_error(LTR_E_INVALID, w + ": thresh must be finite and > 0");
  const int rows_l = in->use_lines ? in->max_rows_l : 0;
  const long long smem = ap_smem_bytes(in->max_rows_p, rows_l);
  if (smem > AP_SMEM_MAX)
    return set_error(LTR_E_UNSUPPORTED, w + ": a group's correspondences need " + std::to_string(smem) +
                                            " bytes of shared memory (32 per keypoint row, 64 per segment row), over " +
                                            std::to_string(AP_SMEM_MAX));
  if (in->n_groups == 0) return LTR_OK;
  if (!out->R || !out->t || !out->valid || !out->refit || !out->n_inliers_p || !out->n_inliers_l || !out->hypothesis ||
      !out->hypothesis_inliers || !out->key)
    return set_error(LTR_E_INVALID, w + ": null output");
  if (!in->groups || !in->K0 || !in->cu_p || !in->cu_l || !out->inliers_p || !out->inliers_l)
    return set_error(LTR_E_INVALID, w + ": null groups, intrinsics, offsets or masks");
  if (in->max_rows_p > 0 && (!in->pts0 || !in->pts_off0 || !in->matches_p || !in->X1 || !in->x_off1 || !in->n_x1))
    return set_error(LTR_E_INVALID, w + ": null keypoint pools, 3D points or matches");
  if (rows_l > 0 && (!in->segs0 || !in->seg_off0 || !in->matches_l || !in->L1 || !in->l_off1 || !in->n_l1))
    return set_error(LTR_E_INVALID, w + ": null segment pools, 3D segments or line matches");
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  AbsPoseArgs a{in->pts0, in->pts_off0, in->matches_p, in->cu_p, in->X1, in->x_off1, in->n_x1,
                in->segs0, in->seg_off0, in->matches_l, in->cu_l, in->L1, in->l_off1, in->n_l1,
                in->groups, in->K0, in->max_rows_p, rows_l, in->thresh * in->thresh, in->n_hypotheses, n_line_hyp,
                (unsigned long long)in->seed, reinterpret_cast<unsigned long long*>(out->key), out->R, out->t,
                out->valid, out->refit, out->inliers_p, out->inliers_l, out->n_inliers_p, out->n_inliers_l,
                out->hypothesis, out->hypothesis_inliers};
  LTR_CUDA_TRY(cudaMemsetAsync(out->key, 0, sizeof(uint64_t) * in->n_groups, s));
  if (in->n_hypotheses)
    LTR_TRY(launch(KC_ABSOLUTE_POSE, true, abspose_hyp_kernel, dim3(in->n_groups, cdiv(in->n_hypotheses, AP_THREADS)),
                   dim3(AP_THREADS), (size_t)smem, s, a));
  if (n_line_hyp)
    LTR_TRY(launch(KC_ABSOLUTE_POSE, true, abspose_line_hyp_kernel,
                   dim3(in->n_groups, cdiv(AP_LINE_SOLVERS * n_line_hyp, AP_THREADS)), dim3(AP_THREADS), (size_t)smem,
                   s, a));
  return launch(KC_ABSOLUTE_POSE, true, abspose_fit_kernel, dim3(in->n_groups), dim3(AP_FIT_THREADS), (size_t)smem, s, a);
}

int ltr_absolute_pose(const LtrAbsPoseInput* in, const LtrAbsPoseOutput* out, int32_t device, void* stream) {
  return absolute_pose("ltr_absolute_pose", in, out, 0, device, stream);
}

int ltr_absolute_pose_lines(const LtrAbsPoseInput* in, const LtrAbsPoseOutput* out, int32_t n_line_hypotheses,
                            int32_t device, void* stream) {
  return absolute_pose("ltr_absolute_pose_lines", in, out, n_line_hypotheses, device, stream);
}

static_assert(LTR_TRI_MAX_VIEWS == ltr::TRI_MAX_VIEWS, "LTR_TRI_MAX_VIEWS and the kernels' bound differ");

int ltr_triangulate(const LtrTriangulateInput* in, const LtrTriangulateOutput* out, int32_t device, void* stream) {
  if (!in || !out) return set_error(LTR_E_INVALID, "ltr_triangulate: null argument");
  if (in->n_images < 0 || in->n_pairs < 0 || in->total_p < 0 || in->total_l < 0 || in->n_inv_p < 0 ||
      in->n_inv_l < 0 || in->n_blocks < 0 || in->max_views < 0)
    return set_error(LTR_E_INVALID, "ltr_triangulate: negative count");
  if (in->max_views > LTR_TRI_MAX_VIEWS)
    return set_error(LTR_E_UNSUPPORTED, "ltr_triangulate: an image takes part in " + std::to_string(in->max_views) +
                                            " pairs, over " + std::to_string(LTR_TRI_MAX_VIEWS));
  if (!(in->thresh > 0.0) || !std::isfinite(in->thresh))
    return set_error(LTR_E_INVALID, "ltr_triangulate: thresh must be finite and > 0");
  if (!(in->min_angle >= 0.0 && in->min_angle < 90.0))
    return set_error(LTR_E_INVALID, "ltr_triangulate: min_angle must be in [0, 90) degrees");
  if (in->min_views < 1 || in->min_views > LTR_TRI_MAX_VIEWS + 1)
    return set_error(LTR_E_INVALID, "ltr_triangulate: min_views must be in [1, LTR_TRI_MAX_VIEWS + 1]");
  if (in->n_images == 0 || in->n_blocks == 0) return LTR_OK;
  if (!in->kp_off || !in->seg_off || !in->K || !in->R || !in->t || !in->view_off || !in->block_off)
    return set_error(LTR_E_INVALID, "ltr_triangulate: null offsets or cameras");
  if (!out->points3d || !out->lines3d || !out->n_views_p || !out->n_views_l)
    return set_error(LTR_E_INVALID, "ltr_triangulate: null output");
  if (in->n_pairs > 0 && (!in->pairs || !in->views || !in->cu_p || !in->cu_l || !in->inv_off_p || !in->inv_off_l))
    return set_error(LTR_E_INVALID, "ltr_triangulate: null pairs, observations or match offsets");
  if ((in->total_p > 0 && !in->matches_p) || (in->total_l > 0 && !in->matches_l) || (in->n_inv_p > 0 && !out->inv_p) ||
      (in->n_inv_l > 0 && !out->inv_l))
    return set_error(LTR_E_INVALID, "ltr_triangulate: null matches or index workspace");
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  const double rad = in->min_angle * (M_PI / 180.0), sn = std::sin(rad);
  TriArgs a{in->kpts, in->kp_off, in->segs, in->seg_off, in->K, in->R, in->t, in->pairs, in->matches_p, in->cu_p,
            in->matches_l, in->cu_l, in->views, in->view_off, in->block_off, in->inv_off_p, in->inv_off_l, out->inv_p,
            out->inv_l, in->n_images, in->n_pairs, in->total_p, in->total_l, in->thresh * in->thresh, std::cos(rad),
            sn * sn, in->min_views, out->points3d, out->lines3d, out->n_views_p, out->n_views_l};
  if (in->n_inv_p > 0) LTR_CUDA_TRY(cudaMemsetAsync(out->inv_p, 0x7f, sizeof(int32_t) * in->n_inv_p, s));
  if (in->n_inv_l > 0) LTR_CUDA_TRY(cudaMemsetAsync(out->inv_l, 0x7f, sizeof(int32_t) * in->n_inv_l, s));
  const long long rows = (long long)in->total_p + in->total_l;
  if (rows > 0)
    LTR_TRY(launch(KC_TRIANGULATE, true, tri_scatter_kernel, dim3(cdiv(rows, TRI_SCATTER_THREADS)), dim3(TRI_SCATTER_THREADS),
                   0, s, a));
  const int smem = (in->max_views > 0 ? in->max_views : 1) * TRI_THREADS * (int)sizeof(float4);
  return launch(KC_TRIANGULATE, true, tri_kernel, dim3(in->n_blocks), dim3(TRI_THREADS), (size_t)smem, s, a);
}

static_assert(LTR_TRK_MAX_OBS == ltr::TRK_MAX_OBS && LTR_TRK_OK == ltr::TRK_OK && LTR_TRK_TOO_LONG == ltr::TRK_TOO_LONG &&
                  LTR_TRK_NO_CANDIDATE == ltr::TRK_NO_CANDIDATE && LTR_TRK_TOO_FEW == ltr::TRK_TOO_FEW,
              "the LTR_TRK_* constants and the kernels' differ");

int ltr_tracks(const LtrTracksInput* in, const LtrTracksOutput* out, int32_t device, void* stream) {
  if (!in || !out) return set_error(LTR_E_INVALID, "ltr_tracks: null argument");
  if (in->n_images < 0 || in->n_pairs < 0 || in->total_p < 0 || in->total_l < 0 || in->n_kp < 0 || in->n_kl < 0)
    return set_error(LTR_E_INVALID, "ltr_tracks: negative count");
  if ((long long)in->n_kp + in->n_kl > INT_MAX / 5)
    return set_error(LTR_E_UNSUPPORTED, "ltr_tracks: too many rows for 32-bit node indices");
  if (!(in->thresh > 0.0) || !std::isfinite(in->thresh) || !(in->epi_thresh > 0.0) || !std::isfinite(in->epi_thresh))
    return set_error(LTR_E_INVALID, "ltr_tracks: thresh and epi_thresh must be finite and > 0");
  if (!(in->min_angle >= 0.0 && in->min_angle < 90.0))
    return set_error(LTR_E_INVALID, "ltr_tracks: min_angle must be in [0, 90) degrees");
  if (!std::isfinite(in->min_overlap)) return set_error(LTR_E_INVALID, "ltr_tracks: min_overlap must be finite");
  if (in->min_views < 1) return set_error(LTR_E_INVALID, "ltr_tracks: min_views must be >= 1");
  if (in->n_images == 0 || (in->n_kp == 0 && in->n_kl == 0)) return LTR_OK;
  if (!in->kp_off || !in->seg_off || !in->K || !in->R || !in->t)
    return set_error(LTR_E_INVALID, "ltr_tracks: null offsets or cameras");
  if (in->n_pairs > 0 && (!in->pairs || !in->F || !in->cu_p || !in->cu_l))
    return set_error(LTR_E_INVALID, "ltr_tracks: null pairs, fundamental matrices or match offsets");
  if ((in->total_p > 0 && (!in->matches_p || !in->kpts)) || (in->total_l > 0 && (!in->matches_l || !in->segs)))
    return set_error(LTR_E_INVALID, "ltr_tracks: null matches or rows");
  if (!out->track_p || !out->track_l || !out->n_tracks_p || !out->n_tracks_l || !out->track_off_p ||
      !out->track_off_l || !out->obs_p || !out->obs_l || !out->points3d || !out->lines3d || !out->n_obs_p ||
      !out->n_obs_l || !out->n_inliers_p || !out->n_inliers_l || !out->n_images_p || !out->n_images_l ||
      !out->status_p || !out->status_l || !out->inlier_p || !out->inlier_l || !out->row_points3d ||
      !out->row_lines3d || !out->n_views_p || !out->n_views_l || !out->workspace)
    return set_error(LTR_E_INVALID, "ltr_tracks: null output or workspace");
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  const double rad = in->min_angle * (M_PI / 180.0), sn = std::sin(rad);
  const int nodes = in->n_kp + in->n_kl;
  int* ws = out->workspace;
  TrkArgs a{in->kpts, in->kp_off, in->segs, in->seg_off, in->K, in->R, in->t, in->F, in->pairs, in->matches_p,
            in->cu_p, in->matches_l, in->cu_l, in->n_images, in->n_pairs, in->total_p, in->total_l,
            {in->n_kp, in->n_kl}, in->thresh * in->thresh, in->epi_thresh * in->epi_thresh, in->min_overlap,
            std::cos(rad), sn * sn, in->min_views, ws, ws + nodes, ws + 2 * nodes, ws + 3 * nodes, ws + 4 * nodes,
            {out->track_p, out->track_l}, {out->n_tracks_p, out->n_tracks_l}, {out->track_off_p, out->track_off_l},
            {out->obs_p, out->obs_l}, {out->n_obs_p, out->n_obs_l}, {out->n_inliers_p, out->n_inliers_l},
            {out->n_images_p, out->n_images_l}, {out->status_p, out->status_l}, out->points3d, out->lines3d,
            out->row_points3d, out->row_lines3d, {out->inlier_p, out->inlier_l}, {out->n_views_p, out->n_views_l}};
  const dim3 node_grid(cdiv(nodes, TRK_ROW_THREADS)), rows(TRK_ROW_THREADS);
  LTR_TRY(launch(KC_TRACKS, true, trk_init_kernel, node_grid, rows, 0, s, a));
  const long long edges = (long long)in->total_p + in->total_l;
  if (edges > 0) LTR_TRY(launch(KC_TRACKS, true, trk_edge_kernel, dim3(cdiv(edges, TRK_ROW_THREADS)), rows, 0, s, a));
  LTR_TRY(launch(KC_TRACKS, true, trk_root_kernel, node_grid, rows, 0, s, a));
  LTR_TRY(launch(KC_TRACKS, true, trk_scan_kernel, dim3(2), dim3(TRK_SCAN_THREADS), 0, s, a));
  LTR_TRY(launch(KC_TRACKS, true, trk_assign_kernel, node_grid, rows, 0, s, a));
  // persistent: enough CTAs for the larger bound, at most 8 per SM
  const int bound = std::max(in->n_kp / 2, in->n_kl / 2);
  const int ctas = std::max(1, std::min(bound, 8 * device_sm_count()));
  return launch(KC_TRACKS, true, trk_kernel, dim3(ctas, 2), dim3(TRK_THREADS), 0, s, a);
}

static_assert(LTR_BA_MAX_IMAGES == ltr::BA_MAX_IMAGES && LTR_BA_IN == ltr::BA_IN &&
                  LTR_BA_NOT_VALID == ltr::BA_NOT_VALID && LTR_BA_SAME_IMAGE == ltr::BA_SAME_IMAGE &&
                  LTR_BA_DEGENERATE == ltr::BA_DEGENERATE && LTR_BA_STOP_ITERS == ltr::BA_STOP_ITERS &&
                  LTR_BA_STOP_FTOL == ltr::BA_STOP_FTOL && LTR_BA_STOP_LAMBDA == ltr::BA_STOP_LAMBDA,
              "the LTR_BA_* constants and the kernels' differ");

int ltr_bundle_adjust(const LtrBundleInput* in, const LtrBundleOutput* out, int32_t device, void* stream) {
  if (!in || !out) return set_error(LTR_E_INVALID, "ltr_bundle_adjust: null argument");
  if (in->n_images < 1 || in->n_kp < 0 || in->n_kl < 0 || in->t_p < 1 || in->t_l < 1)
    return set_error(LTR_E_INVALID, "ltr_bundle_adjust: n_images and the track bounds must be >= 1, rows >= 0");
  if (in->n_images > LTR_BA_MAX_IMAGES)
    return set_error(LTR_E_UNSUPPORTED, "ltr_bundle_adjust: more than LTR_BA_MAX_IMAGES images");
  if ((long long)in->n_kp + in->n_kl > INT_MAX / 64)
    return set_error(LTR_E_UNSUPPORTED, "ltr_bundle_adjust: too many rows");
  if (in->n_fixed < 1 || in->n_fixed > in->n_images)
    return set_error(LTR_E_INVALID, "ltr_bundle_adjust: at least one image must be fixed");
  if (in->max_iters < 0 || in->max_iters > LTR_BA_MAX_ITERS)
    return set_error(LTR_E_INVALID, "ltr_bundle_adjust: max_iters must lie in [0, LTR_BA_MAX_ITERS]");
  if (!std::isfinite(in->ftol) || !(in->ftol >= 0.0))
    return set_error(LTR_E_INVALID, "ltr_bundle_adjust: ftol must be finite and >= 0");
  if (!in->kp_off || !in->seg_off || !in->K || !in->R || !in->t || !in->hold || !in->fixed || !in->n_tracks_p ||
      !in->n_tracks_l || !in->track_off_p || !in->track_off_l || !in->status_p || !in->status_l || !in->points3d ||
      !in->lines3d || !in->kpts || !in->segs || !in->obs_p || !in->obs_l || !in->inlier_p || !in->inlier_l ||
      !in->track_p || !in->track_l || !in->n_views_p || !in->n_views_l)
    return set_error(LTR_E_INVALID, "ltr_bundle_adjust: null input");
  if (!out->R || !out->t || !out->points3d || !out->lines3d || !out->status_p || !out->status_l || !out->residual_p ||
      !out->residual_l || !out->row_points3d || !out->row_lines3d || !out->n_views_p || !out->n_views_l ||
      !out->stats || !out->workspace)
    return set_error(LTR_E_INVALID, "ltr_bundle_adjust: null output or workspace");
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  const int n = in->n_images, rows = in->n_kp + in->n_kl, trk = in->t_p + in->t_l;
  char* w = static_cast<char*>(out->workspace);
  auto take = [&](size_t bytes) {
    char* p = w;
    w += bytes;
    return p;
  };
  BaArgs a{};
  a.kpts = in->kpts; a.kp_off = in->kp_off; a.segs = in->segs; a.seg_off = in->seg_off;
  a.K = in->K; a.R0 = in->R; a.t0 = in->t; a.hold = in->hold; a.fixed = in->fixed;
  a.n_images = n; a.n_fixed = in->n_fixed; a.n_nodes[0] = in->n_kp; a.n_nodes[1] = in->n_kl;
  a.t_bound[0] = in->t_p; a.t_bound[1] = in->t_l; a.max_iters = in->max_iters; a.ftol = in->ftol;
  a.n_tracks[0] = in->n_tracks_p; a.n_tracks[1] = in->n_tracks_l;
  a.track_off[0] = in->track_off_p; a.track_off[1] = in->track_off_l; a.obs[0] = in->obs_p; a.obs[1] = in->obs_l;
  a.trk_status[0] = in->status_p; a.trk_status[1] = in->status_l; a.inlier[0] = in->inlier_p;
  a.inlier[1] = in->inlier_l; a.track_row[0] = in->track_p; a.track_row[1] = in->track_l;
  a.n_views_in[0] = in->n_views_p; a.n_views_in[1] = in->n_views_l; a.X_in[0] = in->points3d;
  a.X_in[1] = in->lines3d;
  a.R = out->R; a.t = out->t; a.X_out[0] = out->points3d; a.X_out[1] = out->lines3d; a.status[0] = out->status_p;
  a.status[1] = out->status_l; a.residual[0] = out->residual_p; a.residual[1] = out->residual_l;
  a.row_points = out->row_points3d; a.row_lines = out->row_lines3d; a.n_views[0] = out->n_views_p;
  a.n_views[1] = out->n_views_l; a.stats = out->stats;
  a.row = reinterpret_cast<double*>(take(8ull * BA_ROW * rows));
  a.trk = reinterpret_cast<double*>(take(8ull * BA_TRK * trk));
  a.A = reinterpret_cast<double*>(take(8ull * 36 * n * n));
  a.cam = reinterpret_cast<double*>(take(8ull * BA_CAM * n));
  a.rhs = reinterpret_cast<double*>(take(8ull * 12 * n));
  a.sd = reinterpret_cast<double*>(take(8ull * 16));
  a.list = reinterpret_cast<int*>(take(4ull * 2 * rows));
  a.mask = reinterpret_cast<unsigned*>(take(4ull * 4 * trk));
  a.list_off = reinterpret_cast<int*>(take(4ull * (n + 1)));
  a.col = reinterpret_cast<int*>(take(4ull * 6 * n));
  a.si = reinterpret_cast<int*>(take(4ull * 23));
  a.part = reinterpret_cast<uint8_t*>(take(n));
  const int sms = device_sm_count();
  const dim3 tg(std::max(1, std::min(cdiv(trk, BA_THREADS), 4 * sms))), tb(BA_THREADS);
  LTR_TRY(launch(KC_BUNDLE, true, ba_start_kernel, dim3(1), dim3(BA_COST_THREADS), 0, s, a));
  LTR_TRY(launch(KC_BUNDLE, true, ba_init_kernel, tg, tb, 0, s, a));
  LTR_TRY(launch(KC_BUNDLE, true, ba_setup_kernel, dim3(1), dim3(BA_COST_THREADS), 0, s, a));
  for (int it = 0; it < in->max_iters; ++it) {
    LTR_TRY(launch(KC_BUNDLE, true, ba_track_kernel, tg, tb, 0, s, a));
    LTR_TRY(launch(KC_BUNDLE, true, ba_reduce_kernel, dim3(n, n), dim3(64), 0, s, a));
    LTR_TRY(launch(KC_BUNDLE, true, ba_solve_kernel, dim3(1), dim3(BA_CTA_THREADS), 0, s, a));
    LTR_TRY(launch(KC_BUNDLE, true, ba_update_kernel, tg, tb, 0, s, a));
    LTR_TRY(launch(KC_BUNDLE, true, ba_accept_kernel, dim3(1), dim3(BA_COST_THREADS), 0, s, a));
  }
  const dim3 fg(std::max(1, std::min(cdiv(std::max(rows, trk), BA_THREADS), 4 * sms)));
  return launch(KC_BUNDLE, true, ba_finish_kernel, fg, tb, 0, s, a);
}

int ltr_global_poses(const LtrGlobalPoseInput* in, const LtrGlobalPoseOutput* out, int32_t device, void* stream) {
  if (!in || !out) return set_error(LTR_E_INVALID, "ltr_global_poses: null argument");
  if (in->n_images < 1 || in->n_pairs < 0)
    return set_error(LTR_E_INVALID, "ltr_global_poses: n_images must be >= 1 and n_pairs >= 0");
  if (in->n_images > LTR_GP_MAX_IMAGES)
    return set_error(LTR_E_UNSUPPORTED, "ltr_global_poses: more than LTR_GP_MAX_IMAGES images");
  if ((long long)in->n_pairs > (long long)in->n_images * (in->n_images - 1) / 2)
    return set_error(LTR_E_INVALID, "ltr_global_poses: more pairs than distinct image pairs");
  if (in->anchor >= in->n_images)
    return set_error(LTR_E_INVALID, "ltr_global_poses: anchor out of range");
  if (in->rot_iters < 0 || in->rot_iters > LTR_GP_MAX_ITERS || in->pos_iters < 0 || in->pos_iters > LTR_GP_MAX_ITERS)
    return set_error(LTR_E_INVALID, "ltr_global_poses: iteration counts must lie in [0, LTR_GP_MAX_ITERS]");
  if (!std::isfinite(in->rot_tan) || !(in->rot_tan > 0.0) || !std::isfinite(in->dir_cos) || !std::isfinite(in->ftol) ||
      !(in->ftol >= 0.0))
    return set_error(LTR_E_INVALID, "ltr_global_poses: rot_tan must be finite > 0, dir_cos finite, ftol finite >= 0");
  if (in->n_pairs && (!in->pairs || !in->R || !in->t || !in->valid || !in->n_cheirality))
    return set_error(LTR_E_INVALID, "ltr_global_poses: null input");
  if (!out->R || !out->t || !out->registered || !out->edge_status || !out->support || !out->rot_residual ||
      !out->dir_cos || !out->stats || !out->workspace)
    return set_error(LTR_E_INVALID, "ltr_global_poses: null output or workspace");
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  const int n = in->n_images, P = in->n_pairs;
  char* w = static_cast<char*>(out->workspace);
  auto take = [&](size_t bytes) {
    char* p = w;
    w += bytes;
    return p;
  };
  GpArgs a{};
  a.pairs = in->pairs; a.Rp = in->R; a.tp = in->t; a.valid = in->valid; a.ncheir = in->n_cheirality;
  a.n = n; a.P = P; a.min_inliers = in->min_inliers; a.anchor_in = in->anchor < 0 ? -1 : in->anchor;
  a.rot_iters = in->rot_iters; a.pos_iters = in->pos_iters; a.rot_tan = in->rot_tan; a.dir_cos = in->dir_cos;
  a.ftol = in->ftol;
  a.R = out->R; a.t = out->t; a.registered = out->registered; a.status = out->edge_status; a.support = out->support;
  a.rot_res = out->rot_residual; a.dcos = out->dir_cos; a.stats = out->stats;
  a.edge = reinterpret_cast<double*>(take(8ull * GP_EDGE * P));
  a.cam = reinterpret_cast<double*>(take(8ull * GP_CAM * n));
  a.table = reinterpret_cast<int*>(take(4ull * n * n));
  a.inc = reinterpret_cast<int*>(take(4ull * n * std::max(n - 1, 1)));
  a.deg = reinterpret_cast<int*>(take(4ull * n));
  a.comp = reinterpret_cast<int*>(take(4ull * n));
  a.si = reinterpret_cast<int*>(take(4ull * 16));
  LTR_TRY(launch(KC_GLOBAL_POSES, true, gp_graph_kernel, dim3(1), dim3(GP_THREADS), 0, s, a));
  if (P) LTR_TRY(launch(KC_GLOBAL_POSES, true, gp_support_kernel, dim3(P), dim3(GP_MAX_IMAGES), 0, s, a));
  return launch(KC_GLOBAL_POSES, true, gp_solve_kernel, dim3(1), dim3(GP_THREADS), gp_smem_bytes(n), s, a);
}

static int rt_check_rows(const char* who, const float* desc, const int32_t* cu, int32_t layout, int32_t rows) {
  if (layout != LTR_LAYOUT_ROWS && layout != LTR_LAYOUT_CHANNEL_FIRST)
    return set_error(LTR_E_INVALID, std::string(who) + ": layout must be LTR_LAYOUT_ROWS or LTR_LAYOUT_CHANNEL_FIRST");
  if (rows < 0) return set_error(LTR_E_INVALID, std::string(who) + ": negative row count");
  if (!cu || (rows > 0 && !desc)) return set_error(LTR_E_INVALID, std::string(who) + ": null descriptors or offsets");
  return LTR_OK;
}

int ltr_kmeans_update(const LtrKmeansInput* in, const LtrKmeansOutput* out, int32_t device, void* stream) {
  if (!in || !out) return set_error(LTR_E_INVALID, "ltr_kmeans_update: null argument");
  if (in->K < 1 || in->K > LTR_RT_MAX_CLUSTERS)
    return set_error(LTR_E_UNSUPPORTED, "ltr_kmeans_update: K must lie in [1, LTR_RT_MAX_CLUSTERS]");
  if (in->n_images < 1) return set_error(LTR_E_INVALID, "ltr_kmeans_update: n_images must be >= 1");
  if (int rc = rt_check_rows("ltr_kmeans_update", in->desc, in->cu, in->layout, in->n_rows)) return rc;
  if (in->init_rows ? in->n_rows < in->K : (!in->centroids_in || (in->n_rows > 0 && !in->assign)))
    return set_error(LTR_E_INVALID, "ltr_kmeans_update: fewer rows than clusters, or null centroids or assignments");
  if (!out->centroids || !out->centroids_cf || !out->tiles || !out->counts || (in->scores && !out->cost) || !out->workspace)
    return set_error(LTR_E_INVALID, "ltr_kmeans_update: null output or workspace");
  if (out->workspace_bytes < LTR_RT_KMEANS_WORKSPACE_BYTES(in->n_rows, in->K))
    return set_error(LTR_E_WORKSPACE, "ltr_kmeans_update: workspace too small");
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  int* cstart = static_cast<int*>(out->workspace);
  int* perm = cstart + in->K + 1;
  const int K = in->K;
  RtKmeansArgs a{};
  a.rows = RtRows{in->desc, in->cu, in->layout, in->n_images};
  a.K = K; a.cstart = cstart; a.perm = perm; a.init_rows = in->init_rows; a.cent_in = in->centroids_in;
  a.cent = out->centroids; a.cent_cf = out->centroids_cf; a.counts = out->counts;
  a.img.hi = static_cast<__nv_bfloat16*>(out->tiles);
  a.img.lo = a.img.hi + (size_t)cdiv(K, 128) * 4 * IMG_TILE_ELEMS;
  a.img.kblocks = 4;
  if (!in->init_rows) {
    RtBucketArgs b{in->assign, nullptr, 1, in->n_rows, K, cstart, perm, in->scores, in->scores ? out->cost : nullptr};
    LTR_TRY(launch(KC_RETRIEVAL, true, rt_bucket_kernel, dim3(1), dim3(RT_BUCKET_THREADS), 0, s, b));
  }
  return launch(KC_RETRIEVAL, true, rt_kmeans_kernel, dim3(K), dim3(256), 0, s, a);
}

int ltr_vlad(const LtrVladInput* in, const LtrVladOutput* out, int32_t device, void* stream) {
  if (!in || !out) return set_error(LTR_E_INVALID, "ltr_vlad: null argument");
  if (in->k_p < 1 || in->k_p > LTR_RT_MAX_CLUSTERS || in->k_l < 1 || in->k_l > LTR_RT_MAX_CLUSTERS)
    return set_error(LTR_E_UNSUPPORTED, "ltr_vlad: k_p and k_l must lie in [1, LTR_RT_MAX_CLUSTERS]");
  if (in->n_images < 1) return set_error(LTR_E_INVALID, "ltr_vlad: n_images must be >= 1");
  if (int rc = rt_check_rows("ltr_vlad", in->desc_p, in->cu_p, in->layout_p, in->rows_p)) return rc;
  if (int rc = rt_check_rows("ltr_vlad", in->desc_l, in->cu_l, in->layout_l, in->rows_l)) return rc;
  if (!(std::isfinite(in->w_p) && in->w_p >= 0.0 && std::isfinite(in->w_l) && in->w_l >= 0.0))
    return set_error(LTR_E_INVALID, "ltr_vlad: the part weights must be finite and >= 0");
  if (!in->centroids_p || !in->centroids_l || (in->rows_p && !in->assign_p) || (in->rows_l && !in->assign_l))
    return set_error(LTR_E_INVALID, "ltr_vlad: null centroids or assignments");
  if (!out->desc || !out->tiles || !out->workspace) return set_error(LTR_E_INVALID, "ltr_vlad: null output or workspace");
  if (out->workspace_bytes < LTR_RT_VLAD_WORKSPACE_BYTES(in->n_images, in->rows_p, in->rows_l, in->k_p, in->k_l))
    return set_error(LTR_E_WORKSPACE, "ltr_vlad: workspace too small");
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  const int n = in->n_images, D = RT_DL * (in->k_p + in->k_l);
  int* w = static_cast<int*>(out->workspace);
  RtVladArgs a{};
  const float* desc[2] = {in->desc_p, in->desc_l};
  const int32_t* cu[2] = {in->cu_p, in->cu_l};
  const int32_t layout[2] = {in->layout_p, in->layout_l}, rows[2] = {in->rows_p, in->rows_l}, K[2] = {in->k_p, in->k_l};
  const int32_t* assign[2] = {in->assign_p, in->assign_l};
  const float* cent[2] = {in->centroids_p, in->centroids_l};
  const double wt[2] = {in->w_p, in->w_l};
  RtBucketArgs b[2];
  for (int pi = 0; pi < 2; ++pi) {
    RtPart& p = a.part[pi];
    p.rows = RtRows{desc[pi], cu[pi], layout[pi], n};
    p.K = K[pi]; p.cent = cent[pi]; p.sw = std::sqrt(wt[pi]); p.col0 = pi ? RT_DL * in->k_p : 0;
    int* cstart = w;
    w += (size_t)n * K[pi] + 1;
    int* perm = w;
    w += rows[pi];
    p.cstart = cstart; p.perm = perm;
    b[pi] = RtBucketArgs{assign[pi], cu[pi], n, rows[pi], K[pi], cstart, perm, nullptr, nullptr};
  }
  a.n_images = n; a.D = D; a.desc = out->desc;
  a.img.hi = static_cast<__nv_bfloat16*>(out->tiles);
  a.img.lo = a.img.hi + (size_t)cdiv(n, 128) * (D / 64) * IMG_TILE_ELEMS;
  a.img.kblocks = D / 64;
  for (int pi = 0; pi < 2; ++pi)
    LTR_TRY(launch(KC_RETRIEVAL, true, rt_bucket_kernel, dim3(n), dim3(RT_BUCKET_THREADS), 0, s, b[pi]));
  return launch(KC_RETRIEVAL, true, rt_vlad_kernel, dim3(cdiv(n, 128) * 128), dim3(256), 0, s, a);
}

int ltr_retrieve(const LtrRetrieveInput* in, const LtrRetrieveOutput* out, int32_t device, void* stream) {
  if (!in || !out) return set_error(LTR_E_INVALID, "ltr_retrieve: null argument");
  if (in->Q < 1 || in->N < 1) return set_error(LTR_E_INVALID, "ltr_retrieve: Q and N must be >= 1");
  if (in->k < 1 || in->k > LTR_RT_MAX_K) return set_error(LTR_E_UNSUPPORTED, "ltr_retrieve: k must lie in [1, LTR_RT_MAX_K]");
  if (in->D < 64 || in->D % 64 || in->D > 2 * RT_DL * LTR_RT_MAX_CLUSTERS)
    return set_error(LTR_E_UNSUPPORTED, "ltr_retrieve: D must be a positive multiple of 64, at most 2 * 256 * LTR_RT_MAX_CLUSTERS");
  if (cdiv(in->Q, 128) > 65535) return set_error(LTR_E_UNSUPPORTED, "ltr_retrieve: more than 65535 query tiles");
  if (!in->q || !in->q_tiles || !in->db || !in->db_tiles) return set_error(LTR_E_INVALID, "ltr_retrieve: null input");
  if (!out->idx || !out->score || !out->n_full || !out->workspace)
    return set_error(LTR_E_INVALID, "ltr_retrieve: null output or workspace");
  if (out->workspace_bytes < LTR_RT_WORKSPACE_BYTES(in->Q, in->N, in->k))
    return set_error(LTR_E_WORKSPACE, "ltr_retrieve: workspace too small");
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  const int nt = cdiv(in->N, 128), kbs = in->D / 64;
  const size_t nc = (size_t)in->Q * nt * in->k;
  RtScreenArgs a{};
  auto img = [&](const void* t, int rows) {
    ActImg m;
    m.hi = static_cast<__nv_bfloat16*>(const_cast<void*>(t));
    m.lo = m.hi + (size_t)cdiv(rows, 128) * kbs * IMG_TILE_ELEMS;
    m.kblocks = kbs;
    return m;
  };
  a.q = img(in->q_tiles, in->Q); a.db = img(in->db_tiles, in->N);
  a.Q = in->Q; a.N = in->N; a.kb = kbs; a.k = in->k; a.exclude_self = in->exclude_self != 0; a.n_tiles = nt;
  a.cand_score = static_cast<float*>(out->workspace);
  a.cand_idx = reinterpret_cast<int*>(a.cand_score + nc);
  a.drop = reinterpret_cast<float*>(a.cand_idx + nc);
  a.n_full = out->n_full;
  RtMergeArgs m{in->q, in->db, in->Q, in->N, in->D, in->k, a.exclude_self, nt, a.cand_score, a.cand_idx, a.drop,
                out->idx, out->score, out->n_full};
  LTR_TRY(launch(KC_RETRIEVAL, true, rt_screen_kernel, dim3(nt, cdiv(in->Q, 128)), dim3(RT_THREADS), (size_t)RT_SMEM, s, a));
  return launch(KC_RETRIEVAL, true, rt_merge_kernel, dim3(in->Q), dim3(RT_MERGE_THREADS), 0, s, m);
}

int ltr_rt_tiles(const float* x, int32_t n, int32_t D, void* tiles, int32_t device, void* stream) {
  if (n < 1 || D < 64 || D % 64 || !x || !tiles)
    return set_error(LTR_E_INVALID, "ltr_rt_tiles: n must be >= 1, D a positive multiple of 64, pointers not null");
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  ActImg img;
  img.hi = static_cast<__nv_bfloat16*>(tiles);
  img.lo = img.hi + (size_t)cdiv(n, 128) * (D / 64) * IMG_TILE_ELEMS;
  img.kblocks = D / 64;
  return launch(KC_RETRIEVAL, true, rt_tiles_kernel, dim3(cdiv(n, 128) * 128), dim3(256), 0, s, x, n, D, img);
}

int ltr_warp_pairs(const uint8_t* gray, const uint8_t* colour, int32_t n_images, int32_t height, int32_t width,
                   int32_t channels, const int32_t* src_index_host, const int32_t* src_index, const double* inv_maps,
                   int32_t n_pairs, uint8_t* warped, uint8_t* mask, int32_t device, void* stream) {
  if (n_images < 1 || n_pairs < 0) return set_error(LTR_E_INVALID, "ltr_warp_pairs: n_images must be >= 1 and n_pairs >= 0");
  if (height < 1 || width < 1 || height > WP_MAX_SIDE || width > WP_MAX_SIDE)
    return set_error(LTR_E_UNSUPPORTED, "ltr_warp_pairs: height and width must be in [1, 32767]");
  if (channels != 1 && channels != 3) return set_error(LTR_E_UNSUPPORTED, "ltr_warp_pairs: channels must be 1 or 3");
  if (n_pairs == 0) return LTR_OK;
  if (!gray || !colour || !src_index_host || !src_index || !inv_maps || !warped || !mask)
    return set_error(LTR_E_INVALID, "ltr_warp_pairs: null argument");
  for (int32_t p = 0; p < n_pairs; ++p)
    if (src_index_host[p] < 0 || src_index_host[p] >= n_images)
      return set_error(LTR_E_INVALID, "ltr_warp_pairs: src_index[" + std::to_string(p) + "] = " +
                                          std::to_string(src_index_host[p]) + " is not an image index");
  const int tiles_x = cdiv(width, WP_TW), tiles = tiles_x * cdiv(height, WP_TH);
  if ((long long)tiles * n_pairs > INT_MAX) return set_error(LTR_E_UNSUPPORTED, "ltr_warp_pairs: too many output tiles");
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  WarpArgs a{gray, colour, src_index, inv_maps, warped, mask, n_images, height, width, channels,
             std::min(1024 / std::min(16, (int)height), (int)width), tiles_x, tiles};
  return launch(KC_WARP, true, warp_pairs_kernel, dim3(tiles * n_pairs), dim3(WP_THREADS), 0, s, a);
}

static bool ph_is_int(double v, double lo, double hi) { return std::isfinite(v) && v == std::floor(v) && v >= lo && v <= hi; }

// Host check of one image's parameter vector; an empty string when it is inside the contract.
static std::string ph_check_params(const double* p, int32_t max_ellipses) {
  for (int s : {PH_P_BRIGHT, PH_P_CONTRAST, PH_P_NOISE, PH_P_SPECKLE})
    if (!ph_is_int(p[s], 0, 2)) return "an application count must be 0, 1 or 2";
  for (int j = 0; j < 2; ++j) {
    if (!ph_is_int(p[PH_P_BRIGHT + 1 + j], -255, 255)) return "a brightness delta must be an integer in [-255, 255]";
    if (!std::isfinite(p[PH_P_CONTRAST + 1 + j])) return "a contrast alpha is not finite";
    if (!(p[PH_P_NOISE + 1 + j] >= 0 && std::isfinite(p[PH_P_NOISE + 1 + j]))) return "a noise stddev must be finite and >= 0";
    if (!(p[PH_P_SPECKLE + 1 + j] >= 0 && p[PH_P_SPECKLE + 1 + j] <= 1)) return "an impulse probability must lie in [0, 1]";
  }
  if (!ph_is_int(p[PH_P_BLUR], 0, 1) || !ph_is_int(p[PH_P_SHADE], 0, 1)) return "the blur and shade flags must be 0 or 1";
  for (int k = 0; k < 9; ++k)
    if (!std::isfinite(p[PH_P_KERNEL + k])) return "a motion-blur tap is not finite";
  if (!ph_is_int(p[PH_P_KEY_LO], 0, 4294967295.0) || !ph_is_int(p[PH_P_KEY_HI], 0, 4294967295.0))
    return "the noise key halves must be integers in [0, 2^32)";
  if (p[PH_P_SHADE] != 0) {
    if (!ph_is_int(p[PH_P_KSIZE], 1, PH_MAX_KSIZE) || ((int)p[PH_P_KSIZE] % 2) == 0)
      return "the shade's kernel size must be odd and in [1, 149]";
    if (!std::isfinite(p[PH_P_TRANSPARENCY])) return "the transparency is not finite";
    if (!ph_is_int(p[PH_P_N_ELLIPSES], 0, max_ellipses)) return "the ellipse count must lie in [0, max_ellipses]";
  }
  return "";
}

int ltr_photometric(const uint8_t* in, uint8_t* out, int32_t n_images, int32_t height, int32_t width,
                    const double* params_host, const double* params, int32_t n_params, const int32_t* ellipses,
                    int32_t max_ellipses, const float* taps, void* workspace, int64_t workspace_bytes, int32_t device,
                    void* stream) {
  if (n_images < 0 || max_ellipses < 0)
    return set_error(LTR_E_INVALID, "ltr_photometric: n_images and max_ellipses must be >= 0");
  if (n_params != PH_NPARAM)
    return set_error(LTR_E_INVALID, "ltr_photometric: n_params must be LTR_PHOTOMETRIC_PARAMS (" +
                                        std::to_string(PH_NPARAM) + "), got " + std::to_string(n_params));
  if (height < 1 || width < 1 || height > 32767 || width > 32767)
    return set_error(LTR_E_UNSUPPORTED, "ltr_photometric: height and width must be in [1, 32767]");
  if (n_images > 65535) return set_error(LTR_E_UNSUPPORTED, "ltr_photometric: at most 65535 images per call");
  if (n_images == 0) return LTR_OK;
  if (!in || !out || !params_host || !params || !taps || !workspace || (max_ellipses > 0 && !ellipses))
    return set_error(LTR_E_INVALID, "ltr_photometric: null argument");
  const int64_t plane = (int64_t)n_images * height * width, a1 = align_up(plane, 256);
  if (workspace_bytes < 2 * a1 + 4 * plane)
    return set_error(LTR_E_WORKSPACE, "ltr_photometric: the workspace needs LTR_PHOTOMETRIC_WORKSPACE_BYTES(n, h, w)");
  for (int32_t i = 0; i < n_images; ++i) {
    const std::string why = ph_check_params(params_host + (size_t)i * PH_NPARAM, max_ellipses);
    if (!why.empty()) return set_error(LTR_E_INVALID, "ltr_photometric: image " + std::to_string(i) + ": " + why);
  }
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  PhotoArgs a{in, out, params, ellipses, taps, ws, ws + a1, reinterpret_cast<float*>(ws + 2 * a1),
              height, width, max_ellipses};
  LTR_CUDA_TRY(cudaMemsetAsync(a.mask, 0, (size_t)plane, s));
  LTR_TRY(launch(KC_PHOTOMETRIC, true, photo_stage1_kernel, dim3(cdiv(width, PS_TW), cdiv(height, PS_TH), n_images),
                 dim3(PS_THREADS), 0, s, a));
  if (max_ellipses > 0)
    LTR_TRY(launch(KC_PHOTOMETRIC, true, photo_ellipse_kernel, dim3(max_ellipses, n_images), dim3(PE_THREADS), 0, s, a));
  LTR_TRY(launch(KC_PHOTOMETRIC, true, photo_blur_row_kernel, dim3(cdiv(width, PR_W), cdiv(height, PR_ROWS), n_images),
                 dim3(PR_ROWS * 32), 0, s, a));
  return launch(KC_PHOTOMETRIC, true, photo_blur_col_kernel, dim3(cdiv(width, PC_W), cdiv(height, PC_H), n_images),
                dim3(PC_W * (PC_H / PC_Q)), 0, s, a);
}

struct NormSpec { int norm; float eps; const float* g; const float* beta; const float* add; int ldadd; };

// res_image: the residual res [m, n] (row stride ldr) is split into the output image first and read from there (Rimg);
// the output image, if any, is then written in place over it
static int linear_img_impl(const float* x, int32_t ldx, const float* w_host, const float* bias, const float* res, int32_t ldr,
                           float* y, int32_t ldy, float* y_from_image, int32_t m, int32_t n, int32_t k, int32_t act,
                           int32_t bn_hint, int32_t device, void* stream, const NormSpec& ns, bool res_image = false) {
  if (!x || !w_host || (!y && !y_from_image)) return set_error(LTR_E_INVALID, "ltr_linear_img: null argument");
  if (n % 64 || k % 64) return set_error(LTR_E_UNSUPPORTED, "ltr_linear_img: n and k must be multiples of 64");
  LTR_CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = as_stream(stream);
  std::vector<double> W((size_t)n * k);
  for (size_t i = 0; i < W.size(); ++i) W[i] = w_host[i];
  std::vector<uint16_t> img(2 * (size_t)n * k);
  pack_tc_weight(W.data(), n, k, img.data(), img.data() + (size_t)n * k);
  const size_t mpad = (size_t)cdiv(m, 256) * 256;
  uint16_t *dw = nullptr, *da = nullptr, *dout = nullptr;
  cudaError_t ce = cudaMalloc(&dw, img.size() * 2);
  if (ce == cudaSuccess) ce = cudaMalloc(&da, 2 * mpad * k * 2);
  if (ce == cudaSuccess) ce = cudaMalloc(&dout, 2 * mpad * n * 2);
  if (ce == cudaSuccess) ce = cudaMemcpyAsync(dw, img.data(), img.size() * 2, cudaMemcpyHostToDevice, s);
  if (ce == cudaSuccess) ce = cudaMemsetAsync(da, 0, 2 * mpad * k * 2, s);
  int rc = 0;
  if (ce == cudaSuccess) {
    ActImg A{reinterpret_cast<__nv_bfloat16*>(da), reinterpret_cast<__nv_bfloat16*>(da + mpad * k), k / 64};
    ActImg O{reinterpret_cast<__nv_bfloat16*>(dout), reinterpret_cast<__nv_bfloat16*>(dout + mpad * n), n / 64};
    rc = launch(KC_IMG_CONVERT, false, to_image_kernel, dim3(cdiv((long long)m * (k / 8), 256)), dim3(256), 0, s, x, ldx, m, k,
                A, 0);
    if (rc == 0 && res_image)
      rc = launch(KC_IMG_CONVERT, false, to_image_kernel, dim3(cdiv((long long)m * (n / 8), 256)), dim3(256), 0, s, res, ldr, m,
                  n, O, 0);
    GemmImgArgs a{};
    a.A = A; a.a_kb0 = 0; a.bias = bias; a.C = y; a.ldc = ldy; a.M = m; a.act = act;
    if (res_image) { a.Rimg = O; a.r_kb0 = 0; } else { a.R = res; a.ldr = ldr; }
    a.W.hi = reinterpret_cast<const __nv_bfloat16*>(dw);
    a.W.lo = reinterpret_cast<const __nv_bfloat16*>(dw + (size_t)n * k);
    a.W.N = n; a.W.K = k;
    if (y_from_image) { a.O = O; a.o_kb0 = 0; }
    a.norm = ns.norm; a.eps = ns.eps; a.ng = ns.g; a.nbeta = ns.beta; a.nadd = ns.add; a.ldadd = ns.ldadd;
    if (rc == 0) rc = launch_gemm_img(a, s, bn_hint);
    if (rc == 0 && y_from_image)
      rc = launch(KC_IMG_CONVERT, false, from_image_kernel, dim3(cdiv((long long)m * n, 256)), dim3(256), 0, s, O, 0,
                  y_from_image, n, m, n);
    ce = cudaStreamSynchronize(s);
  }
  cudaFree(dw); cudaFree(da); cudaFree(dout);
  if (rc != 0) return rc;
  if (ce != cudaSuccess) return set_error(LTR_E_CUDA, std::string("ltr_linear_img: ") + cudaGetErrorString(ce));
  return LTR_OK;
}

int ltr_linear_img(const float* x, int32_t ldx, const float* w_host, const float* bias, const float* res, int32_t ldr,
                   float* y, int32_t ldy, float* y_from_image, int32_t m, int32_t n, int32_t k, int32_t act,
                   int32_t bn_hint, int32_t device, void* stream) {
  return linear_img_impl(x, ldx, w_host, bias, res, ldr, y, ldy, y_from_image, m, n, k, act, bn_hint, device, stream,
                         NormSpec{NORM_NONE, 0.f, nullptr, nullptr, nullptr, 0});
}

int ltr_debug_linear_img_res(const float* x, int32_t ldx, const float* w_host, const float* bias, const float* res,
                             float* y, float* y_from_image, int32_t m, int32_t n, int32_t k, int32_t act,
                             int32_t bn_hint, int32_t device, void* stream) {
  if (!res || (y != nullptr) == (y_from_image != nullptr))
    return set_error(LTR_E_INVALID, "ltr_debug_linear_img_res: res and exactly one of y, y_from_image required");
  return linear_img_impl(x, ldx, w_host, bias, res, n, y, n, y_from_image, m, n, k, act, bn_hint, device, stream,
                         NormSpec{NORM_NONE, 0.f, nullptr, nullptr, nullptr, 0}, true);
}

int ltr_linear_img_norm(const float* x, int32_t ldx, const float* w_host, const float* bias, const float* res, int32_t ldr,
                        int32_t norm, float eps, const float* gamma, const float* beta, const float* add, int32_t ldadd,
                        float* y, int32_t ldy, float* y_from_image, int32_t m, int32_t k, int32_t device, void* stream) {
  if (norm != NORM_LAYER && norm != NORM_L2) return set_error(LTR_E_INVALID, "ltr_linear_img_norm: norm must be 1 (LayerNorm) or 2 (L2)");
  if (norm == NORM_LAYER && (!gamma || !beta)) return set_error(LTR_E_INVALID, "ltr_linear_img_norm: LayerNorm needs gamma and beta");
  return linear_img_impl(x, ldx, w_host, bias, res, ldr, y, ldy, y_from_image, m, 256, k, ACT_NONE, 256, device, stream,
                         NormSpec{norm, eps, gamma, beta, add, ldadd});
}

// Micro-benchmark of the image GEMM engine: average device ms per launch of an [m,k]x[n,k]^T
// problem with zero-filled operands (timing only).  out_mode: 0 fp32 rows, 1 image, 2 both.
// debug: arm / read the clock64 stamps kernels of CTA 0 leave in g_dbg_trace (see LTR_DBG_STAMP)
void ltr_debug_trace_arm(int32_t on) {
  int v = on;
  cudaMemcpyToSymbol(g_dbg_on, &v, sizeof(int));
  if (on) {
    static unsigned long long zeros[128] = {0};
    cudaMemcpyToSymbol(g_dbg_trace, zeros, sizeof(zeros));
  }
}
int ltr_debug_trace_read(unsigned long long* out128) {
  cudaDeviceSynchronize();
  return cudaMemcpyFromSymbol(out128, g_dbg_trace, 128 * sizeof(unsigned long long)) == cudaSuccess ? 0 : -2;
}

int ltr_debug_encode_images(const LtrModel* m, int32_t n_lines, void* workspace, void* hi[11], void* lo[11],
                            int32_t kblocks[11]) {
  if (!m || n_lines < 0 || !workspace || !hi || !lo || !kblocks)
    return set_error(LTR_E_INVALID, "ltr_debug_encode_images: bad argument");
  char* base = reinterpret_cast<char*>(align_up(reinterpret_cast<int64_t>(workspace), 256));   // as ltr_encode
  const EncodeWs w = carve(m, n_lines, base);
  const ActImg* img[10] = {&w.z, &w.ctx, &w.l128, &w.l256, &w.lpos, &w.y1i, &w.g, &w.xm, &w.hm, &w.qkv};
  for (int i = 0; i < 10; ++i) {
    hi[i] = img[i]->hi;
    lo[i] = img[i]->lo;
    kblocks[i] = img[i]->kblocks;
  }
  hi[10] = w.yf;
  lo[10] = nullptr;
  kblocks[10] = 0;
  return LTR_OK;
}

int ltr_debug_sig_attention(const void* qkv_hi, const void* qkv_lo, void* out_hi, void* out_lo, int32_t n_images,
                            int32_t launches, void* stream) {
  if (!qkv_hi || !qkv_lo || !out_hi || !out_lo || n_images <= 0 || launches < 0)
    return set_error(LTR_E_INVALID, "ltr_debug_sig_attention: bad argument");
  auto img = [](const void* hi, const void* lo, int kb) {
    return ActImg{reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(hi)), reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(lo)), kb};
  };
  const ActImg qkv = img(qkv_hi, qkv_lo, 12), out = img(out_hi, out_lo, 8);
  for (int i = 0; i < launches; ++i)
    LTR_TRY(launch_sig_attention_tc(qkv, out, 256, nullptr, 128, 128, n_images, static_cast<cudaStream_t>(stream)));
  return LTR_OK;
}

// Test hooks of the relative-pose estimator's fp64 pieces: one thread per item, the estimator's __device__ functions.
static __global__ void debug_sturm_roots_kernel(const double* poly, int n, double* roots, int* count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double p[11], r[10];
  for (int j = 0; j < 11; ++j) p[j] = poly[11ll * i + j];
  const int c = ess_roots(p, r);
  for (int j = 0; j < 10; ++j) roots[10ll * i + j] = j < c ? r[j] : __longlong_as_double(0x7ff8000000000000ll);
  count[i] = c;
}

static __global__ void debug_essential_solve_kernel(const double* q, int n, double* E, int* root_index, int* n_sol) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double4 s[5];
  for (int j = 0; j < 5; ++j)
    s[j] = make_double4(q[20ll * i + 4 * j], q[20ll * i + 4 * j + 1], q[20ll * i + 4 * j + 2], q[20ll * i + 4 * j + 3]);
  double Es[90];
  int jr[10];
  const int ns = ess_solve(s, Es, jr);
  for (int j = 0; j < 90; ++j) E[90ll * i + j] = j < 9 * ns ? Es[j] : __longlong_as_double(0x7ff8000000000000ll);
  for (int j = 0; j < 10; ++j) root_index[10ll * i + j] = j < ns ? jr[j] : -1;
  n_sol[i] = ns;
}

// Test hooks of the fundamental-matrix and absolute-pose estimators' fp64 pieces, in the same form.
static __global__ void debug_fundamental_solve_kernel(const double* q, int n, double* F, int* root_index, int* n_sol) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double4 s[FM_SAMPLE];
  for (int j = 0; j < FM_SAMPLE; ++j)
    s[j] = make_double4(q[28ll * i + 4 * j], q[28ll * i + 4 * j + 1], q[28ll * i + 4 * j + 2], q[28ll * i + 4 * j + 3]);
  double Fs[9 * FM_MAX_SOLUTIONS];
  int jr[FM_MAX_SOLUTIONS];
  const int ns = fm_solve(s, Fs, jr);
  for (int j = 0; j < 9 * FM_MAX_SOLUTIONS; ++j)
    F[27ll * i + j] = j < 9 * ns ? Fs[j] : __longlong_as_double(0x7ff8000000000000ll);
  for (int j = 0; j < FM_MAX_SOLUTIONS; ++j) root_index[3ll * i + j] = j < ns ? jr[j] : -1;
  n_sol[i] = ns;
}

static __global__ void debug_p3p_kernel(const double* jb, const double* X, int n, double* R, double* t, int* root_index,
                                        int* n_sol) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double j[9], x[9];
  for (int e = 0; e < 9; ++e) {
    j[e] = jb[9ll * i + e];
    x[e] = X[9ll * i + e];
  }
  double Rs[9 * AP_MAX_SOLUTIONS], ts[3 * AP_MAX_SOLUTIONS];
  int jr[AP_MAX_SOLUTIONS];
  const int ns = ap_p3p(j, x, Rs, ts, jr);
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  for (int e = 0; e < 9 * AP_MAX_SOLUTIONS; ++e) R[36ll * i + e] = e < 9 * ns ? Rs[e] : nan;
  for (int e = 0; e < 3 * AP_MAX_SOLUTIONS; ++e) t[12ll * i + e] = e < 3 * ns ? ts[e] : nan;
  for (int e = 0; e < AP_MAX_SOLUTIONS; ++e) root_index[4ll * i + e] = e < ns ? jr[e] : -1;
  n_sol[i] = ns;
}

// One thread per sample of line solver s: j, X [n, 2 - s, 3], normals [n, s + 1, 3], end points [n, s + 1, 2, 3].
static __global__ void debug_line_pose_kernel(int s, const double* jb, const double* Xb, const double* nb,
                                              const double* Eb, int n, double* R, double* t, int* root_index,
                                              int* n_sol) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int np = ap_line_np(s), nl = ap_line_nl(s);
  double j[6], X[6], nn[9], E[18];
  for (int e = 0; e < 3 * np; ++e) {
    j[e] = jb[3ll * np * i + e];
    X[e] = Xb[3ll * np * i + e];
  }
  for (int e = 0; e < 3 * nl; ++e) nn[e] = nb[3ll * nl * i + e];
  for (int e = 0; e < 6 * nl; ++e) E[e] = Eb[6ll * nl * i + e];
  double Rs[9 * AP_LINE_MAX_SOLUTIONS], ts[3 * AP_LINE_MAX_SOLUTIONS];
  int jr[AP_LINE_MAX_SOLUTIONS];
  const int ns = ap_line_pose(s, j, X, nn, E, Rs, ts, jr);
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  for (int e = 0; e < 9 * AP_LINE_MAX_SOLUTIONS; ++e) R[72ll * i + e] = e < 9 * ns ? Rs[e] : nan;
  for (int e = 0; e < 3 * AP_LINE_MAX_SOLUTIONS; ++e) t[24ll * i + e] = e < 3 * ns ? ts[e] : nan;
  for (int e = 0; e < AP_LINE_MAX_SOLUTIONS; ++e) root_index[8ll * i + e] = e < ns ? jr[e] : -1;
  n_sol[i] = ns;
}

static __global__ void debug_fundamental_lines_kernel(const double* F, const float* s0, const float* s1, int n,
                                                      double min_overlap, double* r1, double* r0, uint8_t* ok) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double f[9];
  for (int e = 0; e < 9; ++e) f[e] = F[9ll * i + e];
  double a, b;
  fm_line_ratios(f, s0 + 4ll * i, s1 + 4ll * i, a, b);
  r1[i] = a;
  r0[i] = b;
  ok[i] = fm_ratios_consistent(a, b, min_overlap);
}

// One CTA of 1024 threads per system, the rc_cholesky_solve<1024> instantiation of ba_solve_kernel and gp_solve_kernel.
// shared: A (square, ld m) and x are copied into dynamic shared memory first, as gp_solve_kernel keeps them, and copied
// back after; else the solve works in place on the caller's A (leading dimension ld) and x, as ba_solve_kernel does.
constexpr int DEBUG_CHOL_THREADS = 1024;
static __global__ void __launch_bounds__(DEBUG_CHOL_THREADS) debug_cholesky_kernel(double* A, int m, int ld, double* x,
                                                                                   int k, int shared, uint8_t* ok) {
  extern __shared__ double s_dyn[];
  __shared__ int s_fail;
  const int tid = threadIdx.x;
  double* Ag = A + (size_t)blockIdx.x * m * ld;
  double* xg = x + (size_t)blockIdx.x * m * k;
  double* As = Ag;
  double* xs = xg;
  int lds = ld;
  if (shared) {
    As = s_dyn;
    xs = As + (size_t)m * m;
    lds = m;
    for (int e = tid; e < m * m; e += DEBUG_CHOL_THREADS) As[e] = Ag[(size_t)ld * (e / m) + e % m];
    for (int e = tid; e < m * k; e += DEBUG_CHOL_THREADS) xs[e] = xg[e];
  }
  double* scol = shared ? xs + (size_t)m * k : s_dyn;
  if (tid == 0) s_fail = 0;
  __syncthreads();
  const bool fail = rc_cholesky_solve<DEBUG_CHOL_THREADS>(As, lds, m, xs, k, scol, &s_fail);
  if (shared) {
    for (int e = tid; e < m * m; e += DEBUG_CHOL_THREADS) Ag[(size_t)ld * (e / m) + e % m] = As[e];
    for (int e = tid; e < m * k; e += DEBUG_CHOL_THREADS) xg[e] = xs[e];
  }
  if (tid == 0) ok[blockIdx.x] = !fail;
}

int ltr_debug_sturm_roots(const double* poly, int32_t n, double* roots, int32_t* count, int32_t device, void* stream) {
  if (n < 0 || (n > 0 && (!poly || !roots || !count))) return set_error(LTR_E_INVALID, "ltr_debug_sturm_roots: bad argument");
  if (n == 0) return LTR_OK;
  LTR_CUDA_TRY(cudaSetDevice(device));
  return launch(KC_DEBUG, false, debug_sturm_roots_kernel, dim3(cdiv(n, 128)), dim3(128), 0, as_stream(stream), poly, n,
                roots, count);
}

int ltr_debug_essential_solve(const double* q, int32_t n, double* E, int32_t* root_index, int32_t* n_solutions,
                              int32_t device, void* stream) {
  if (n < 0 || (n > 0 && (!q || !E || !root_index || !n_solutions)))
    return set_error(LTR_E_INVALID, "ltr_debug_essential_solve: bad argument");
  if (n == 0) return LTR_OK;
  LTR_CUDA_TRY(cudaSetDevice(device));
  return launch(KC_DEBUG, false, debug_essential_solve_kernel, dim3(cdiv(n, 128)), dim3(128), 0, as_stream(stream), q, n, E,
                root_index, n_solutions);
}

int ltr_debug_fundamental_solve(const double* q, int32_t n, double* F, int32_t* root_index, int32_t* n_solutions,
                                int32_t device, void* stream) {
  if (n < 0 || (n > 0 && (!q || !F || !root_index || !n_solutions)))
    return set_error(LTR_E_INVALID, "ltr_debug_fundamental_solve: bad argument");
  if (n == 0) return LTR_OK;
  LTR_CUDA_TRY(cudaSetDevice(device));
  return launch(KC_DEBUG, false, debug_fundamental_solve_kernel, dim3(cdiv(n, 128)), dim3(128), 0, as_stream(stream), q, n, F,
                root_index, n_solutions);
}

int ltr_debug_p3p(const double* j, const double* X, int32_t n, double* R, double* t, int32_t* root_index,
                  int32_t* n_solutions, int32_t device, void* stream) {
  if (n < 0 || (n > 0 && (!j || !X || !R || !t || !root_index || !n_solutions)))
    return set_error(LTR_E_INVALID, "ltr_debug_p3p: bad argument");
  if (n == 0) return LTR_OK;
  LTR_CUDA_TRY(cudaSetDevice(device));
  return launch(KC_DEBUG, false, debug_p3p_kernel, dim3(cdiv(n, 128)), dim3(128), 0, as_stream(stream), j, X, n, R, t,
                root_index, n_solutions);
}

int ltr_debug_line_pose(int32_t solver, const double* j, const double* X, const double* n, const double* E, int32_t count,
                        double* R, double* t, int32_t* root_index, int32_t* n_solutions, int32_t device, void* stream) {
  if (solver < 0 || solver >= AP_LINE_SOLVERS || count < 0 ||
      (count > 0 && ((solver < 2 && (!j || !X)) || !n || !E || !R || !t || !root_index || !n_solutions)))
    return set_error(LTR_E_INVALID, "ltr_debug_line_pose: bad argument");
  if (count == 0) return LTR_OK;
  LTR_CUDA_TRY(cudaSetDevice(device));
  return launch(KC_DEBUG, false, debug_line_pose_kernel, dim3(cdiv(count, 128)), dim3(128), 0, as_stream(stream),
                (int)solver, j, X, n, E, (int)count, R, t, root_index, n_solutions);
}

int ltr_debug_fundamental_lines(const double* F, const float* s0, const float* s1, int32_t n, double min_overlap,
                                double* r1, double* r0, uint8_t* ok, int32_t device, void* stream) {
  if (n < 0 || (n > 0 && (!F || !s0 || !s1 || !r1 || !r0 || !ok)) || !(min_overlap >= 0.0 && min_overlap <= 1.0))
    return set_error(LTR_E_INVALID, "ltr_debug_fundamental_lines: bad argument");
  if (n == 0) return LTR_OK;
  LTR_CUDA_TRY(cudaSetDevice(device));
  return launch(KC_DEBUG, false, debug_fundamental_lines_kernel, dim3(cdiv(n, 128)), dim3(128), 0, as_stream(stream), F, s0,
                s1, n, min_overlap, r1, r0, ok);
}

int ltr_debug_cholesky_solve(double* A, int32_t n, int32_t m, int32_t ld, double* x, int32_t k, int32_t shared,
                             uint8_t* ok, int32_t device, void* stream) {
  if (n < 0 || m < 0 || m > DEBUG_CHOL_THREADS || k < 1 || k > 6 || ld < m || (shared != 0 && shared != 1) ||
      (shared && m > GP_MAX_IMAGES - 1) || (n > 0 && (!ok || (m > 0 && (!A || !x)))))
    return set_error(LTR_E_INVALID, "ltr_debug_cholesky_solve: bad argument");
  if (n == 0) return LTR_OK;
  LTR_CUDA_TRY(cudaSetDevice(device));
  const size_t smem = 8 * (shared ? (size_t)m * m + (size_t)m * k + m : (size_t)(m > 0 ? m : 1));
  return launch(KC_DEBUG, false, debug_cholesky_kernel, dim3(n), dim3(DEBUG_CHOL_THREADS), smem, as_stream(stream), A, m, ld, x,
                k, shared, ok);
}

float ltr_gemm_bench(int32_t m, int32_t n, int32_t k, int32_t bn_hint, int32_t out_mode, int32_t iters, int32_t device) {
  if (cudaSetDevice(device) != cudaSuccess) return -1.f;
  const size_t mpad = (size_t)cdiv(m, 256) * 256;
  uint16_t *dw = nullptr, *da = nullptr, *dout = nullptr;
  float* dc = nullptr;
  cudaMalloc(&dw, 2 * (size_t)n * k * 2);
  cudaMalloc(&da, 2 * mpad * k * 2);
  cudaMalloc(&dout, 2 * mpad * n * 2);
  cudaMalloc(&dc, mpad * n * 4);
  cudaMemset(dw, 0, 2 * (size_t)n * k * 2);
  cudaMemset(da, 0, 2 * mpad * k * 2);
  GemmImgArgs a{};
  a.A = ActImg{reinterpret_cast<__nv_bfloat16*>(da), reinterpret_cast<__nv_bfloat16*>(da + mpad * k), k / 64};
  a.W.hi = reinterpret_cast<const __nv_bfloat16*>(dw);
  a.W.lo = reinterpret_cast<const __nv_bfloat16*>(dw + (size_t)n * k);
  a.W.N = n; a.W.K = k; a.M = m; a.act = 1;
  if (out_mode == 0 || out_mode == 2) { a.C = dc; a.ldc = n; }
  if (out_mode == 1 || out_mode == 2) a.O = ActImg{reinterpret_cast<__nv_bfloat16*>(dout), reinterpret_cast<__nv_bfloat16*>(dout + mpad * n), n / 64};
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int i = 0; i < 3; ++i) launch_gemm_img(a, 0, bn_hint);
  cudaEventRecord(e0, 0);
  for (int i = 0; i < iters; ++i) launch_gemm_img(a, 0, bn_hint);
  cudaEventRecord(e1, 0);
  cudaEventSynchronize(e1);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  cudaFree(dw); cudaFree(da); cudaFree(dout); cudaFree(dc);
  return cudaGetLastError() == cudaSuccess ? ms / iters : -1.f;
}

// One signature layer's row-local GEMMs at m rows (zero-filled operands, timing only):
// mlp1 [512 x 512] ReLU -> hm, mlp2 [256 x 512] + x -> xm[:, :256] in place, qkv [768 x 256] -> qkv image,
// as one gemm_chain_kernel launch (chained != 0) or three gemm_img_kernel launches.  Average device ms per layer.
float ltr_gemm_chain_bench(int32_t m, int32_t chained, int32_t iters, int32_t device) {
  if (m <= 0 || iters <= 0 || cudaSetDevice(device) != cudaSuccess) return -1.f;
  const size_t mpad = (size_t)cdiv(m, 256) * 256;
  const int Ns[3] = {512, 256, 768}, Ks[3] = {512, 512, 256}, acts[3] = {ACT_RELU, ACT_NONE, ACT_NONE};
  uint16_t* dw[3] = {nullptr, nullptr, nullptr};
  uint16_t *dxm = nullptr, *dhm = nullptr, *dqkv = nullptr;
  bool ok = true;
  for (int i = 0; i < 3; ++i) ok = ok && cudaMalloc(&dw[i], 2 * (size_t)Ns[i] * Ks[i] * 2) == cudaSuccess;
  ok = ok && cudaMalloc(&dxm, 2 * mpad * 512 * 2) == cudaSuccess && cudaMalloc(&dhm, 2 * mpad * 512 * 2) == cudaSuccess &&
       cudaMalloc(&dqkv, 2 * mpad * 768 * 2) == cudaSuccess;
  float ms = -1.f;
  if (ok) {
    for (int i = 0; i < 3; ++i) cudaMemset(dw[i], 0, 2 * (size_t)Ns[i] * Ks[i] * 2);
    cudaMemset(dxm, 0, 2 * mpad * 512 * 2);
    auto img = [&](uint16_t* p, int K) {
      return ActImg{reinterpret_cast<__nv_bfloat16*>(p), reinterpret_cast<__nv_bfloat16*>(p + mpad * K), K / 64};
    };
    const ActImg xm = img(dxm, 512), hm = img(dhm, 512), qkv = img(dqkv, 768);
    const ActImg A[3] = {xm, hm, xm}, O[3] = {hm, xm, qkv};
    GemmImgArgs ops[3];
    for (int i = 0; i < 3; ++i) {
      GemmImgArgs a{};
      a.A = A[i]; a.O = O[i]; a.M = m; a.act = acts[i];
      a.W.hi = reinterpret_cast<const __nv_bfloat16*>(dw[i]);
      a.W.lo = reinterpret_cast<const __nv_bfloat16*>(dw[i] + (size_t)Ns[i] * Ks[i]);
      a.W.N = Ns[i]; a.W.K = Ks[i];
      ops[i] = a;
    }
    ops[1].Rimg = xm;   // x += delta
    auto layer = [&]() {
      if (chained) return launch_gemm_chain(ops, 3, 0);
      for (int i = 0; i < 3; ++i)
        if (int rc = launch_gemm_img(ops[i], 0)) return rc;
      return 0;
    };
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    int rc = 0;
    for (int i = 0; i < 3 && !rc; ++i) rc = layer();
    cudaEventRecord(e0, 0);
    for (int i = 0; i < iters && !rc; ++i) rc = layer();
    cudaEventRecord(e1, 0);
    cudaEventSynchronize(e1);
    if (!rc && cudaGetLastError() == cudaSuccess && cudaEventElapsedTime(&ms, e0, e1) == cudaSuccess) ms /= iters;
    else ms = -1.f;
    cudaEventDestroy(e0); cudaEventDestroy(e1);
  }
  for (int i = 0; i < 3; ++i) cudaFree(dw[i]);
  cudaFree(dxm); cudaFree(dhm); cudaFree(dqkv);
  return ms;
}

}  // extern "C"
