// GPU line tokenizer: the step that FEEDS the hot path (SURVEY.md 8f row 1).
// Replaces the per-line / per-token Python loops of line_tokenizer (reference
// models/line_process.py:100-196) and sample_descriptors (:86-98): token positions along each key
// line, split of long lines into sublines, masks, responses, angles, bilinear sampling +
// L2 normalisation of the dense 256-d descriptor map, score lookup.
//
// The host prepares per key line (vectorised numpy, no loops): end points in float64, the
// clipped end point, n_tokens = ceil(length / token_distance), first subline index, image index.
// One launch pair covers many images (ltr_tokenize_batch); each image has its own maps, sizes and
// token_distance, and its sublines land at its rows of the concatenated output.  Token
// positions, subline cut points and responses are computed in float64 in the CPU glue's numpy order,
// one explicitly rounded operation per numpy operation (__dmul_rn / __dadd_rn / __ddiv_rn / __dsqrt_rn, so
// nvcc cannot contract a product and a sum into one fma; squares are products, as in the glue, where the
// reference's scalar m ** 2 goes through libm pow), then rounded once to fp32: they, the masks and the
// score lookups are bit-identical to the CPU glue.  That order is part of the contract.  Sampled
// descriptors agree to fp32 rounding (bound: tests/tokenizer_model.py).  Key lines must have finite,
// non-negative coordinates and run left to right (start x <= end x, as change_cv2_T_np orders them), so no
// token rounds to a negative score row or column; the host refuses other lines (keyline_geometry).
#pragma once
#include "common.cuh"

namespace ltr {

// Per image: the token spacing and the SuperPoint maps the image's tokens are sampled from.
struct TokImage {
  const float* dense;     // [256, Hc, Wc]
  const float* score;     // [H, W]
  double token_distance;
  int Hc, Wc, H, W;
};

// The images of one launch, passed by value (__grid_constant__: indexed in place, never copied to local
// memory).  Key line k belongs to im[line_image[k] - first]; a one-image table (NI = 1) holds every line.
template <int NI>
struct TokImages {
  TokImage im[NI];
  int first;
};

struct TokLines {
  const double* sp;       // [K,2] start point (x, y)
  const double* ep;       // [K,2] end point BEFORE the in-place clip (direction of the line)
  const double* epc;      // [K,2] end point after clip to (width-0.6, height-0.6)
  const double* length;   // [K] length_klines (detector length, NOT the geometric one)
  const float* angle;     // [K,2]
  const int* n_tok;       // [K]
  const int* sub0;        // [K+1] first subline of each key line (prefix sum of n_sub, over all images)
  const int* sub2line;    // [S]
  const int* line_image;  // [K] image of each key line
  int K, S, T;
};

template <int NI>
__device__ __forceinline__ const TokImage& image_of_line(const TokLines& L, const TokImages<NI>& I, int k) {
  if constexpr (NI == 1) return I.im[0];
  else return I.im[L.line_image[k] - I.first];
}

// point at distance d from sp along the line (reference point_on_line, line_process.py:43-59), every operation
// rounded as numpy rounds it: m = vy / vx, dx = sqrt(d**2 / (1 + m**2)), dy = m * dx, then + sp.  Explicit
// intrinsics keep nvcc from contracting 1 + m * m into one fma, which rounds once less than numpy.
__device__ __forceinline__ void point_on_line_f64(double spx, double spy, double epx, double epy, double d, double& x, double& y) {
  const double vx = __dsub_rn(epx, spx), vy = __dsub_rn(epy, spy);
  double dx, dy;
  if (vx != 0.0) {
    const double m = __ddiv_rn(vy, vx);
    dx = __dsqrt_rn(__ddiv_rn(__dmul_rn(d, d), __dadd_rn(1.0, __dmul_rn(m, m))));
    dy = __dmul_rn(m, dx);
  } else {
    dx = 0.0;
    dy = (vy > 0.0) ? d : -d;
  }
  x = __dadd_rn(dx, spx);
  y = __dadd_rn(dy, spy);
}

// token i of key line k (i < n_tok): i < n_tok-1 -> point at i*token_distance, last -> clipped end point
__device__ __forceinline__ void token_of_line(const TokLines& L, double token_distance, int k, int i, double& x, double& y) {
  if (i < L.n_tok[k] - 1) {
    point_on_line_f64(L.sp[2 * k], L.sp[2 * k + 1], L.ep[2 * k], L.ep[2 * k + 1], __dmul_rn((double)i, token_distance), x, y);
  } else {
    x = L.epc[2 * k];
    y = L.epc[2 * k + 1];
  }
}

// one thread per (subline, token slot) of sublines [s_begin, s_end): pnt [S,T,2], mask [S,T+1,1]; slot 0
// threads also write the subline end points [S,2,2], resp [S,1], angle [S,2]
template <int NI>
__global__ void __launch_bounds__(256)
tok_points_kernel(TokLines L, const __grid_constant__ TokImages<NI> I, int s_begin, int s_end, float* __restrict__ pnt,
                  float* __restrict__ mask, float* __restrict__ sublines, float* __restrict__ resp, float* __restrict__ angle) {
  const long long idx = (long long)s_begin * L.T + (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= (long long)s_end * L.T) return;
  const int s = (int)(idx / L.T), j = (int)(idx % L.T);
  const int k = L.sub2line[s];
  const double td = image_of_line(L, I, k).token_distance;
  const int sl = s - L.sub0[k];          // subline index within the key line
  const int n_sub = L.sub0[k + 1] - L.sub0[k];
  const int i = sl * L.T + j;
  const bool live = i < L.n_tok[k];
  double x = 0.0, y = 0.0;
  if (live) token_of_line(L, td, k, i, x, y);
  pnt[2 * idx] = (float)x;
  pnt[2 * idx + 1] = (float)y;
  mask[(long long)s * (L.T + 1) + 1 + j] = live ? 1.f : 0.f;
  if (j == 0) {
    mask[(long long)s * (L.T + 1)] = 1.f;
    double ax, ay, bx, by;
    if (sl == 0) { ax = L.sp[2 * k]; ay = L.sp[2 * k + 1]; } else token_of_line(L, td, k, sl * L.T - 1, ax, ay);
    if (sl == n_sub - 1) { bx = L.epc[2 * k]; by = L.epc[2 * k + 1]; } else token_of_line(L, td, k, (sl + 1) * L.T - 1, bx, by);
    sublines[4 * s + 0] = (float)ax; sublines[4 * s + 1] = (float)ay;
    sublines[4 * s + 2] = (float)bx; sublines[4 * s + 3] = (float)by;
    // numpy: sqrt(((b - a) ** 2).sum()) / (token_distance * max_tokens), both squares rounded before the sum
    const double dxx = __dsub_rn(bx, ax), dyy = __dsub_rn(by, ay);
    resp[s] = (float)__ddiv_rn(__dsqrt_rn(__dadd_rn(__dmul_rn(dxx, dxx), __dmul_rn(dyy, dyy))),
                               __dmul_rn(td, (double)L.T));
    angle[2 * s] = L.angle[2 * k];
    angle[2 * s + 1] = L.angle[2 * k + 1];
  }
}

// one warp per token of sublines [s_begin, s_end): bilinear sample of its image's dense [C=256, Hc, Wc] at the
// token (torch grid_sample, mode bilinear, zeros padding), L2 normalise over channels, nearest score lookup.
template <int NI>
__global__ void __launch_bounds__(256)
tok_sample_kernel(TokLines L, const __grid_constant__ TokImages<NI> I, int s_begin, int s_end, int align_corners,
                  const float* __restrict__ pnt, float* __restrict__ desc, float* __restrict__ score) {
  const long long t = (long long)s_begin * L.T + (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= (long long)s_end * L.T) return;
  const TokImage& im = image_of_line(L, I, L.sub2line[t / L.T]);
  const float* __restrict__ dense = im.dense;
  const int Hc = im.Hc, Wc = im.Wc;
  const float px = pnt[2 * t], py = pnt[2 * t + 1];
  // reference sample_descriptors: (kp - s/2 + 0.5) / (w*s - s/2 - 0.5) * 2 - 1 with s = 8, fp32 arithmetic
  const float gx = ((px - 4.0f) + 0.5f) / ((float)Wc * 8.0f - 4.0f - 0.5f) * 2.0f - 1.0f;
  const float gy = ((py - 4.0f) + 0.5f) / ((float)Hc * 8.0f - 4.0f - 0.5f) * 2.0f - 1.0f;
  float ix, iy;
  if (align_corners) {
    ix = (gx + 1.f) / 2.f * (float)(Wc - 1);
    iy = (gy + 1.f) / 2.f * (float)(Hc - 1);
  } else {
    ix = ((gx + 1.f) * (float)Wc - 1.f) / 2.f;
    iy = ((gy + 1.f) * (float)Hc - 1.f) / 2.f;
  }
  const float fx = floorf(ix), fy = floorf(iy);
  const int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
  const float wnw = ((float)x1 - ix) * ((float)y1 - iy), wne = (ix - (float)x0) * ((float)y1 - iy);
  const float wsw = ((float)x1 - ix) * (iy - (float)y0), wse = (ix - (float)x0) * (iy - (float)y0);
  const bool inx0 = x0 >= 0 && x0 < Wc, inx1 = x1 >= 0 && x1 < Wc, iny0 = y0 >= 0 && y0 < Hc, iny1 = y1 >= 0 && y1 < Hc;
  const long long plane = (long long)Hc * Wc;
  float v[8];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float* ch = dense + (long long)(lane + 32 * i) * plane;
    float a = 0.f;
    if (inx0 && iny0) a += ch[y0 * Wc + x0] * wnw;
    if (inx1 && iny0) a += ch[y0 * Wc + x1] * wne;
    if (inx0 && iny1) a += ch[y1 * Wc + x0] * wsw;
    if (inx1 && iny1) a += ch[y1 * Wc + x1] * wse;
    v[i] = a;
    ss = fmaf(a, a, ss);
  }
  ss = warp_sum(ss);
  const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
#pragma unroll
  for (int i = 0; i < 8; ++i) desc[t * 256 + lane + 32 * i] = v[i] * inv;
  if (lane == 0) {
    int rx = (int)rintf(px), ry = (int)rintf(py);   // torch.round: half to even
    rx = min(rx, im.W - 1);
    ry = min(ry, im.H - 1);
    score[t] = im.score[(long long)ry * im.W + rx];
  }
}

}  // namespace ltr
