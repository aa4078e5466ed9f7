// Homography ground truth for line matches and per-pair TP/FP/FN/TN of predicted matches.
// Reference: the builder's mat_assign_sublines (dataloaders/build_homography_dataset.py:210-234) from
// find_line_matches / calculate_line_overlaps (dataloaders/utils/util_lines.py:67-171), scored like
// Evaluate_PR.calc_TFPN (evaluations/evaluate_pr.py:10-22).
//
// The reference evaluates every distance, length and ratio as numpy float32 scalars, so every + - * / sqrt
// here is an explicitly rounded fp32 intrinsic (no FMA contraction) in the reference's evaluation order: the
// values are then bit-identical.  The one exception is the angle (numpy's float32 arctan2 / degrees are not
// correctly rounded and vary with the host's SIMD path): it is computed in fp64, so the angle decision may
// differ from the reference only where the reference's |ang_diff - thres_angdiff| is tiny.
#pragma once
#include <cfloat>
#include "common.cuh"

namespace ltr {

constexpr int LG_ROWS = 128;   // side-0 rows per CTA, one per thread
constexpr int LG_COLS = 32;    // side-1 lines staged through shared memory per step

struct LineGtArgs {
  const float* segs0; const float* segs1;     // [S, 2, 2] pixels (start xy, end xy)
  const int* cu0; const int* cu1;             // [P+1]
  const double* H; const double* Hinv;        // [P, 3, 3] image 0 -> 1 and its inverse
  const float* proj0; const float* proj1;     // optional caller projections (segs0 by H, segs1 by Hinv)
  const int* pred0;                           // optional [S0]: local side-1 index or -1
  float thr_reproj; double thr_ang; double min_overlap;
  float* assign; long long stride;            // optional dense [n0_p, n1_p] at p * stride
  int* n_gt;                                  // [P]
  int* tfpn;                                  // [P, 4] when pred0 is given
};

struct Seg { float sx, sy, ex, ey; };

// One line in the role of `line0` of find_line_matches / calc_overlap: everything that depends on it alone.
struct RefLine {
  Seg s;
  float a, b, c, d;   // point-line numerator terms (y2-y1, x2-x1, x2*y1, y2*x1)
  float len;          // sqrt((x2-x1)^2 + (y2-y1)^2); also the point-line denominator (same two squares)
  double ang;         // degrees(atan2(dx, dy)) in fp64 (x and y swapped as in the reference)
};

__device__ __forceinline__ float sq_rn(float x) { return __fmul_rn(x, x); }

__device__ __forceinline__ float pp_dist(float x0, float y0, float x1, float y1) {
  return __fsqrt_rn(__fadd_rn(sq_rn(__fsub_rn(x1, x0)), sq_rn(__fsub_rn(y1, y0))));
}

__device__ __forceinline__ double seg_angle(const Seg& s) {
  return atan2((double)__fsub_rn(s.ex, s.sx), (double)__fsub_rn(s.ey, s.sy)) * (180.0 / 3.14159265358979323846);
}

__device__ __forceinline__ RefLine ref_line(const Seg& s) {
  RefLine r;
  r.s = s;
  r.a = __fsub_rn(s.ey, s.sy);
  r.b = __fsub_rn(s.ex, s.sx);
  r.c = __fmul_rn(s.ex, s.sy);
  r.d = __fmul_rn(s.ey, s.sx);
  r.len = __fsqrt_rn(__fadd_rn(sq_rn(r.a), sq_rn(r.b)));
  r.ang = seg_angle(s);
  return r;
}

// |(y2-y1)*x0 - (x2-x1)*y0 + x2*y1 - y2*x1| / sqrt(...): a zero-length line gives 0/0 = NaN, which fails every
// comparison (so the "both far" skip does not fire), as in the reference.
__device__ __forceinline__ float pl_dist(const RefLine& l, float x0, float y0) {
  const float num = __fsub_rn(__fadd_rn(__fsub_rn(__fmul_rn(l.a, x0), __fmul_rn(l.b, y0)), l.c), l.d);
  return __fdiv_rn(fabsf(num), l.len);
}

// find_line_matches(line0, line1) followed by calc_overlap(line0, line1) on the same pair: the overlap ratio
// (>= 0) if line1 matches line0, else -1.  len1 / ang1 belong to line1.
__device__ __forceinline__ float match_overlap(const RefLine& l0, const Seg& l1, float len1, double ang1, float thr_r,
                                               double thr_a) {
  const float d0 = pl_dist(l0, l1.sx, l1.sy), d1 = pl_dist(l0, l1.ex, l1.ey);
  if (d0 > thr_r && d1 > thr_r) return -1.f;
  const double ad = fmod(fabs(ang1 - l0.ang), 180.0);
  if (ad > thr_a) return -1.f;
  const float len0 = l0.len;
  const float s0s1 = pp_dist(l0.s.sx, l0.s.sy, l1.sx, l1.sy), e0s1 = pp_dist(l0.s.ex, l0.s.ey, l1.sx, l1.sy);
  const float s0e1 = pp_dist(l0.s.sx, l0.s.sy, l1.ex, l1.ey), e0e1 = pp_dist(l0.s.ex, l0.s.ey, l1.ex, l1.ey);
  const bool sp_in = s0s1 < len0 && e0s1 < len0;
  const bool ep_in = s0e1 < len0 && e0e1 < len0;
  if (sp_in && ep_in) return __fdiv_rn(len1, len0);
  if (sp_in) return __fdiv_rn(s0e1 > e0e1 ? e0s1 : s0s1, len0);
  if (ep_in) return __fdiv_rn(s0s1 > e0s1 ? e0e1 : s0e1, len0);
  const float mx = fmaxf(fmaxf(s0s1, e0s1), fmaxf(s0e1, e0e1));
  return mx > __fadd_rn(len0, len1) ? -1.f : 1.f;   // find_line_matches rejects what calc_overlap would score 0
}

// cv2.perspectiveTransform of one point: fp64, w = 1 / (x*m6 + y*m7 + m8) unless |w| <= FLT_EPSILON -> (0, 0).
__device__ __forceinline__ void project(const double* __restrict__ m, float x, float y, float& ox, float& oy) {
  const double X = x, Y = y;
  const double w = __dadd_rn(__dadd_rn(__dmul_rn(X, m[6]), __dmul_rn(Y, m[7])), m[8]);
  if (fabs(w) > (double)FLT_EPSILON) {
    const double r = __ddiv_rn(1.0, w);
    ox = (float)__dmul_rn(__dadd_rn(__dadd_rn(__dmul_rn(X, m[0]), __dmul_rn(Y, m[1])), m[2]), r);
    oy = (float)__dmul_rn(__dadd_rn(__dadd_rn(__dmul_rn(X, m[3]), __dmul_rn(Y, m[4])), m[5]), r);
  } else {
    ox = 0.f;
    oy = 0.f;
  }
}

__device__ __forceinline__ Seg load_seg(const float* __restrict__ p, long long i) {
  const float4 v = *reinterpret_cast<const float4*>(p + 4 * i);
  return Seg{v.x, v.y, v.z, v.w};
}

__device__ __forceinline__ Seg project_seg(const double* __restrict__ m, const Seg& s) {
  Seg o;
  project(m, s.sx, s.sy, o.sx, o.sy);
  project(m, s.ex, s.ey, o.ex, o.ey);
  return o;
}

// Evaluate_PR.calc_TFPN, one row of a pair: n_tp += TP (the predicted column is ground truth), n_pos += positive (the
// row has ground truth), n_tn += TN.  TN is literal calc_TFPN: the row's count of columns with neither a prediction nor
// ground truth equals the number of ROWS.
__device__ __forceinline__ void tfpn_row(bool any_gt, bool tp, int neither, int n_rows, int& n_tp, int& n_pos, int& n_tn) {
  n_tp += tp;
  n_pos += any_gt ? 1 : 0;
  n_tn += neither == n_rows;
}

// A block's row sums into the pair's TP, FP = negatives - TN, FN = positives - TP, TN.
__device__ __forceinline__ void tfpn_add(int* o, int rows, int pos, int tp, int tn) {
  atomicAdd(o + 0, tp);
  atomicAdd(o + 1, rows - pos - tn);
  atomicAdd(o + 2, pos - tp);
  atomicAdd(o + 3, tn);
}

// Grid (pairs, ceil(max_n0 / 128)), 128 threads: thread t owns side-0 row blockIdx.y*128 + t of pair blockIdx.x and
// keeps its whole ground-truth row, so the per-row TP / TN / positive tests need no atomics; one atomic per count
// and block.  Side 1 goes through shared memory 32 lines at a time; in dense mode the 128 x 32 block of the
// assignment is transposed there too so that rows are stored coalesced.
template <bool DENSE>
__global__ void __launch_bounds__(LG_ROWS) line_gt_kernel(LineGtArgs a) {
  __shared__ RefLine s_l1[LG_COLS];      // side-1 lines in the line0 role (direction 1)
  __shared__ Seg s_p1[LG_COLS];          // their projections into image 0 (direction 0's line1)
  __shared__ float s_plen1[LG_COLS];
  __shared__ double s_pang1[LG_COLS];
  __shared__ float s_out[DENSE ? LG_ROWS : 1][LG_COLS + 1];
  __shared__ int s_red[4][LG_ROWS / 32];
  pdl_launch_dependents();
  pdl_wait();
  const int pair = blockIdx.x, t = threadIdx.x;
  const int b0 = a.cu0[pair], n0 = a.cu0[pair + 1] - b0;
  const int b1 = a.cu1[pair], n1 = a.cu1[pair + 1] - b1;
  const int row0 = blockIdx.y * LG_ROWS;
  if (row0 >= n0) return;
  const int i = row0 + t;
  const bool live = i < n0;
  const double* __restrict__ Hm = a.H + 9 * pair;
  const double* __restrict__ Hi = a.Hinv + 9 * pair;

  // this thread's side-0 line (direction 0's line0) and its projection into image 1 (direction 1's line1)
  RefLine l0{};
  Seg p0{};
  float plen0 = 0.f;
  double pang0 = 0.0;
  if (live) {
    const Seg s = load_seg(a.segs0, b0 + i);
    l0 = ref_line(s);
    p0 = a.proj0 ? load_seg(a.proj0, b0 + i) : project_seg(Hm, s);
    plen0 = pp_dist(p0.sx, p0.sy, p0.ex, p0.ey);
    pang0 = seg_angle(p0);
  }
  int pred = -1;
  if (a.pred0 && live) {
    pred = a.pred0[b0 + i];
    if (pred >= n1) pred = -1;
  }
  bool any_gt = false, tp = false;
  int neither = 0, n_gt = 0;
  float* out = DENSE ? a.assign + (long long)pair * a.stride : nullptr;

  for (int j0 = 0; j0 < n1; j0 += LG_COLS) {
    const int nj = min(LG_COLS, n1 - j0);
    __syncthreads();   // previous step's readers are done with the staging buffers
    if (t < nj) {
      const Seg s = load_seg(a.segs1, b1 + j0 + t);
      s_l1[t] = ref_line(s);
      const Seg p = a.proj1 ? load_seg(a.proj1, b1 + j0 + t) : project_seg(Hi, s);
      s_p1[t] = p;
      s_plen1[t] = pp_dist(p.sx, p.sy, p.ex, p.ey);
      s_pang1[t] = seg_angle(p);
    }
    __syncthreads();
    if (live) {
      for (int jj = 0; jj < nj; ++jj) {
        float v = 0.f;
        const float o0 = match_overlap(l0, s_p1[jj], s_plen1[jj], s_pang1[jj], a.thr_reproj, a.thr_ang);
        if (o0 >= 0.f) {
          const float o1 = match_overlap(s_l1[jj], p0, plen0, pang0, a.thr_reproj, a.thr_ang);
          if (o1 >= 0.f) v = o0 > o1 ? o0 : o1;
        }
        const bool gt = v > 0.f;
        const int j = j0 + jj;
        any_gt |= gt;
        n_gt += (double)v > a.min_overlap;
        if (j == pred) tp = gt;
        else neither += !gt;
        if (DENSE) s_out[t][jj] = v;
      }
    }
    if (DENSE) {
      __syncthreads();
      // warp w stores rows w, w+4, ... of the block: lanes along the 32 columns
      const int lane = t & 31, w = t >> 5;
      for (int r = w; r < LG_ROWS && row0 + r < n0; r += LG_ROWS / 32)
        if (lane < nj) out[(long long)(row0 + r) * n1 + j0 + lane] = s_out[r][lane];
    }
  }

  // per-pair counts: n_gt; with predictions the calc_TFPN row terms
  int c[4] = {0, 0, 0, 0};
  if (live) {
    c[0] = n_gt;
    tfpn_row(any_gt, tp, neither, n0, c[1], c[2], c[3]);
  }
  const int lane = t & 31, w = t >> 5;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    int v = c[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) s_red[k][w] = v;
  }
  __syncthreads();
  if (t == 0) {
    int s[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      s[k] = 0;
#pragma unroll
      for (int q = 0; q < LG_ROWS / 32; ++q) s[k] += s_red[k][q];
    }
    atomicAdd(a.n_gt + pair, s[0]);
    if (a.pred0) tfpn_add(a.tfpn + 4 * pair, min(LG_ROWS, n0 - row0), s[2], s[1], s[3]);
  }
}

}  // namespace ltr
