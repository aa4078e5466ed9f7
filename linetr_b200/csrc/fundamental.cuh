// Fundamental matrices of a batch of uncalibrated image pairs: seven-point RANSAC, an eight-point refit, and the
// epipolar check of the line matches (ltr_fundamental).
//
// Model (DESIGN.md "Fundamental matrices"; restated in numpy by linetr_b200.geometry.ransac_fundamental_host):
//   F maps image 0 to image 1: x1^T F x0 = 0 in pixels.
//   correspondences of pair p: the matched side-0 keypoints in row order with their partners, normalised per side as
//   the homography's points are (centre and half the larger extent of the side's bounding box, hg_stage_pair).
//   hypothesis k: 7 distinct correspondences drawn as the homography's (hg_draw), then the seven-point solver: the
//   null basis F1, F2 of the 7 epipolar rows (rc_null_basis), the cubic det(F2 + a (F1 - F2)) expanded along the first
//   row, its real roots a_j (ascending) by the Sturm chain and bisection (ess_roots); solution j is F2 + a_j (F1 - F2)
//   (a solution where F1 - F2 alone is singular, a = infinity, is not returned).  F = T1^T F^ T0, scaled to unit
//   Frobenius norm with its largest |entry| positive.  Every operation up to here is explicitly rounded fp64.
//   inlier: cv2's FM error, the larger squared distance of x1 to F x0 and of x0 to F^T x1 in pixels, below thresh^2,
//   evaluated as (x1^T F x0)^2 < thresh^2 min(|(F x0)_xy|^2, |(F^T x1)_xy|^2); a zero line normal is an outlier.
//   winner: most inliers, then lowest k, then lowest j (atomicMax of (count << 32) | ~(3 k + j)).
//   refit (at least 8 winner inliers): smallest eigenvector of A^T A over the winner's inliers (normalised epipolar
//   rows, hg_smallest_eigvec), rank 2 by removing F^'s smallest singular direction (Jacobi eigenvectors of F^T F),
//   denormalised and scaled as above; kept iff its inlier count >= the hypothesis'.
//   line check of matched key lines s0 = (a0, b0), s1 = (a1, b1) under the kept F: per side, the epipolar lines of the
//   other segment's end points cut the segment's line at positions ta, tb (its start at 0, its end at 1); the overlap
//   ratio is |[min, max] n [0, 1]| / min(max - min, 1).  A side whose intersection has |w| <= FLT_EPSILON |X| or whose
//   positions coincide cannot reject; consistent iff no side's ratio is below min_overlap.
//
// Kernels:
//   fundamental_hyp_kernel  grid (pair, chunk of FM_THREADS hypotheses): stage the pair's correspondences, one
//                           hypothesis per thread (solver + up to 3 solutions scored against every staged row), one
//                           atomicMax per CTA.
//   fundamental_fit_kernel  grid (pair): the winner again, both inlier passes, the refit, the outputs, and the line
//                           check of the pair's match rows (row-parallel, from global memory).
#pragma once
#include "common.cuh"
#include "rn_fp64.cuh"
#include "ransac_common.cuh"
#include "homography.cuh"

namespace ltr {

constexpr int FM_THREADS = 128;          // hypotheses per CTA
constexpr int FM_FIT_THREADS = 256;
constexpr int FM_SAMPLE = 7;
constexpr int FM_MAX_SOLUTIONS = 3;
constexpr int FM_MIN_REFIT = 8;          // winner inliers needed for the eight-point refit
constexpr int FM_SMEM_MAX = 200 * 1024;

struct FundamentalArgs {
  const float* pts0; const float* pts1;   // [*, 2] keypoint pools
  const int* pts_off0; const int* pts_off1; const int* n_pts1;
  const int* matches_p; const int* cu_p;
  const float* segs0; const float* segs1; // [*, 2, 2] segment pools
  const int* seg_off0; const int* seg_off1; const int* n_segs1;
  const int* matches_l; const int* cu_l;
  int rows;                               // staging rows per pair
  double thresh2, min_overlap;
  int n_hyp;
  unsigned long long seed;
  unsigned long long* key;
  double* F; uint8_t* valid; uint8_t* inl; uint8_t* lines_ok; uint8_t* refit;
  int* n_inl; int* n_lines_ok; int* hyp_index; int* hyp_inliers;
};

// Dynamic shared memory of one pair: the pixel rows (16 bytes each), plus two flag bytes per row in the fit kernel.
static inline long long fm_smem_bytes(long long rows, bool fit) { return hg_smem_bytes(rows, 0, fit); }

// The point-only view of the arguments that the homography's staging reads (same compaction and normalisation).
__device__ __forceinline__ HomographyArgs fm_point_args(const FundamentalArgs& a) {
  HomographyArgs h{};
  h.pts0 = a.pts0; h.pts1 = a.pts1; h.pts_off0 = a.pts_off0; h.pts_off1 = a.pts_off1; h.n_pts1 = a.n_pts1;
  h.matches_p = a.matches_p; h.cu_p = a.cu_p;
  h.rows_p = a.rows; h.rows_l = 0; h.use_p = 1; h.use_l = 0;
  return h;
}

// The seven-point solver on 7 normalised correspondences q[s] = (x0, y0, x1, y1): up to 3 normalised F^ (row-major,
// Fs[9 s]) with their root indices jr[s].  -> solution count.
__device__ __noinline__ int fm_solve(const double4* q, double* Fs, int* jr) {
  double e[9][2];
  if (!rc_null_basis<FM_SAMPLE>(q, e)) return 0;
  // F(a) = F2 + a D, D = F1 - F2: entry i is the polynomial c[i] = [F2_i, D_i] in a
  double c[9][2];
  for (int i = 0; i < 9; ++i) {
    c[i][0] = e[i][1];
    c[i][1] = RC_S(e[i][0], e[i][1]);
  }
  // det F(a) = (c0 (c4 c8 - c5 c7) - c1 (c3 c8 - c5 c6)) + c2 (c3 c7 - c4 c6), ascending coefficients
  double poly[11], x3[3], y3[3], t[4];
  ess_pmul(c[4], 2, c[8], 2, x3); ess_pmul(c[5], 2, c[7], 2, y3);
  for (int i = 0; i < 3; ++i) x3[i] = RC_S(x3[i], y3[i]);
  ess_pmul(c[0], 2, x3, 3, poly);
  ess_pmul(c[3], 2, c[8], 2, x3); ess_pmul(c[5], 2, c[6], 2, y3);
  for (int i = 0; i < 3; ++i) x3[i] = RC_S(x3[i], y3[i]);
  ess_pmul(c[1], 2, x3, 3, t);
  for (int i = 0; i < 4; ++i) poly[i] = RC_S(poly[i], t[i]);
  ess_pmul(c[3], 2, c[7], 2, x3); ess_pmul(c[4], 2, c[6], 2, y3);
  for (int i = 0; i < 3; ++i) x3[i] = RC_S(x3[i], y3[i]);
  ess_pmul(c[2], 2, x3, 3, t);
  for (int i = 0; i < 4; ++i) poly[i] = RC_A(poly[i], t[i]);
  for (int i = 4; i < 11; ++i) poly[i] = 0.0;
  double roots[10];
  const int nr = ess_roots(poly, roots);
  int ns = 0;
  for (int j = 0; j < nr; ++j) {
    double* F = Fs + 9 * ns;
    bool fin = true;
    for (int i = 0; i < 9; ++i) {
      F[i] = RC_A(c[i][0], RC_M(roots[j], c[i][1]));
      fin &= isfinite(F[i]);
    }
    if (fin) jr[ns++] = j;
  }
  return ns;
}

// Normalised f (9) -> pixel F = T1^T F^ T0, scaled to unit Frobenius norm with its largest |entry| (the first on a
// tie) positive; false for a zero or non-finite result.
__device__ __forceinline__ bool fm_to_pixels(const HgPair& sp, const double* f, double* F) {
  const double t0x = -RC_M(sp.c0x, sp.i0), t0y = -RC_M(sp.c0y, sp.i0);
  const double t1x = -RC_M(sp.c1x, sp.i1), t1y = -RC_M(sp.c1y, sp.i1);
  double M[9], G[9];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    M[3 * i] = RC_M(f[3 * i], sp.i0);
    M[3 * i + 1] = RC_M(f[3 * i + 1], sp.i0);
    M[3 * i + 2] = RC_A(RC_A(RC_M(f[3 * i], t0x), RC_M(f[3 * i + 1], t0y)), f[3 * i + 2]);
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    G[j] = RC_M(M[j], sp.i1);
    G[3 + j] = RC_M(M[3 + j], sp.i1);
    G[6 + j] = RC_A(RC_A(RC_M(t1x, M[j]), RC_M(t1y, M[3 + j])), M[6 + j]);
  }
  double s = 0.0;
  int im = 0;
#pragma unroll
  for (int j = 0; j < 9; ++j) {
    s = RC_A(s, RC_M(G[j], G[j]));
    if (fabs(G[j]) > fabs(G[im])) im = j;
  }
  const double nrm = __dsqrt_rn(s);
  if (!(nrm > 0.0) || !isfinite(nrm)) return false;
  const bool neg = G[im] < 0.0;
#pragma unroll
  for (int j = 0; j < 9; ++j) {
    const double v = RC_D(G[j], nrm);
    F[j] = neg ? -v : v;
  }
  return true;
}

// Hypothesis k of pair p: its pixel solutions Fs[9 s] (unit norm) with root indices jr[s].  -> solution count.
__device__ __forceinline__ int fm_hypothesis(const HgStage& st, const HgPair& sp, unsigned long long seed, int p, int k,
                                             double* Fs, int* jr) {
  int idx[FM_SAMPLE];
  if (!hg_draw<FM_SAMPLE>(seed, p, k, sp.np, idx)) return 0;
  double4 q[FM_SAMPLE];
  for (int s = 0; s < FM_SAMPLE; ++s) {
    const float4 r = st.pt[idx[s]];
    q[s] = make_double4(RC_M(RC_S(r.x, sp.c0x), sp.i0), RC_M(RC_S(r.y, sp.c0y), sp.i0),
                        RC_M(RC_S(r.z, sp.c1x), sp.i1), RC_M(RC_S(r.w, sp.c1y), sp.i1));
  }
  double Fh[9 * FM_MAX_SOLUTIONS];
  int jh[FM_MAX_SOLUTIONS];
  const int nh = fm_solve(q, Fh, jh);
  int ns = 0;
  for (int s = 0; s < nh; ++s)
    if (fm_to_pixels(sp, Fh + 9 * s, Fs + 9 * ns)) jr[ns++] = jh[s];
  return ns;
}

// cv2's FM error below t2, without the division: (x1^T F x0)^2 < t2 min(|(F x0)_xy|^2, |(F^T x1)_xy|^2).
__device__ __forceinline__ bool fm_inlier(const double* F, const float4 q, double t2) {
  const double x0 = q.x, y0 = q.y, x1 = q.z, y1 = q.w;
  const double u0 = RC_A(RC_A(RC_M(F[0], x0), RC_M(F[1], y0)), F[2]);
  const double u1 = RC_A(RC_A(RC_M(F[3], x0), RC_M(F[4], y0)), F[5]);
  const double u2 = RC_A(RC_A(RC_M(F[6], x0), RC_M(F[7], y0)), F[8]);
  const double w0 = RC_A(RC_A(RC_M(F[0], x1), RC_M(F[3], y1)), F[6]);
  const double w1 = RC_A(RC_A(RC_M(F[1], x1), RC_M(F[4], y1)), F[7]);
  const double num = RC_A(RC_A(RC_M(x1, u0), RC_M(y1, u1)), u2);
  const double a = RC_A(RC_M(u0, u0), RC_M(u1, u1)), b = RC_A(RC_M(w0, w0), RC_M(w1, w1));
  const double m = a < b ? a : b;
  return m > 0.0 && RC_M(num, num) < RC_M(t2, m);
}

__global__ void __launch_bounds__(FM_THREADS) fundamental_hyp_kernel(FundamentalArgs a) {
  extern __shared__ __align__(16) unsigned char fm_smem[];
  __shared__ HgPair sp;
  __shared__ int warp_cnt[FM_THREADS / 32];
  __shared__ float red[FM_THREADS / 32 * 8];
  __shared__ unsigned long long wbest[FM_THREADS / 32];
  pdl_launch_dependents();
  pdl_wait();
  const int p = blockIdx.x;
  const HgStage st = hg_stage_ptrs(fm_smem, a.rows, 0);
  hg_stage_pair<FM_THREADS>(fm_point_args(a), p, st, sp, warp_cnt, red);
  const int n = sp.np;
  if (n < FM_SAMPLE) return;
  const int k = blockIdx.y * FM_THREADS + threadIdx.x;
  unsigned long long key = 0;
  if (k < a.n_hyp) {
    double Fs[9 * FM_MAX_SOLUTIONS];
    int jr[FM_MAX_SOLUTIONS];
    const int ns = fm_hypothesis(st, sp, a.seed, p, k, Fs, jr);
    for (int s = 0; s < ns; ++s) {
      double F[9];
#pragma unroll
      for (int i = 0; i < 9; ++i) F[i] = Fs[9 * s + i];
      unsigned cnt = 0;
      for (int d = 0; d < n; ++d) cnt += fm_inlier(F, st.pt[d], a.thresh2);
      const unsigned long long kk =
          ((unsigned long long)cnt << 32) | (unsigned long long)(~(unsigned)(FM_MAX_SOLUTIONS * k + jr[s]));
      key = kk > key ? kk : key;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long t = __shfl_xor_sync(0xffffffffu, key, o);
    key = t > key ? t : key;
  }
  if ((threadIdx.x & 31) == 0) wbest[threadIdx.x >> 5] = key;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < FM_THREADS / 32; ++i) key = wbest[i] > key ? wbest[i] : key;
    if (key) atomicMax(a.key + p, key);
  }
}

// Block-wide inlier flags of F (shared) into fl; returns the inlier count to every thread.
template <int NT>
__device__ __forceinline__ int fm_mark(const HgStage& st, int n, const double* sF, double t2, uint8_t* fl, int* red) {
  double F[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) F[i] = sF[i];
  int c = 0;
  for (int d = threadIdx.x; d < n; d += NT) {
    const bool in = fm_inlier(F, st.pt[d], t2);
    fl[d] = in;
    c += in;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = c;
  __syncthreads();
  int t = 0;
  for (int i = 0; i < NT / 32; ++i) t += red[i];
  return t;
}

// Rank 2: f (3 x 3, row-major) minus its smallest singular direction, F - (F v) v^T with v the eigenvector of the
// smallest eigenvalue of F^T F (cyclic Jacobi).
__device__ __noinline__ void fm_rank2(double* f) {
  double S[3][3], V[3][3];
  for (int i = 0; i < 3; ++i)
    for (int k = 0; k < 3; ++k) {
      S[i][k] = f[i] * f[k] + f[3 + i] * f[3 + k] + f[6 + i] * f[6 + k];
      V[i][k] = i == k ? 1.0 : 0.0;
    }
  rc_jacobi3(S, V);
  int m = 0;
  for (int i = 1; i < 3; ++i)
    if (S[i][i] < S[m][m]) m = i;
  const double v0 = V[0][m], v1 = V[1][m], v2 = V[2][m];
  for (int r = 0; r < 3; ++r) {
    const double fv = f[3 * r] * v0 + f[3 * r + 1] * v1 + f[3 * r + 2] * v2;
    f[3 * r] -= fv * v0;
    f[3 * r + 1] -= fv * v1;
    f[3 * r + 2] -= fv * v2;
  }
}

// Overlap ratio of one side: the lines la, lb (epipolar lines of the other segment's end points) cut the line through
// segment (p, q) at positions ta, tb (p at 0, q at 1).  -> |[min, max] n [0, 1]| / min(max - min, 1), or NaN when the
// side cannot reject (an intersection with |w| <= FLT_EPSILON |X|, or ta == tb).
__device__ __forceinline__ double fm_side_ratio(const double* la, const double* lb, double px, double py, double qx,
                                                double qy) {
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  const double l0 = RC_S(py, qy), l1 = RC_S(qx, px), l2 = RC_S(RC_M(px, qy), RC_M(qx, py));
  const double dx = RC_S(qx, px), dy = RC_S(qy, py);
  const double len2 = RC_A(RC_M(dx, dx), RC_M(dy, dy));
  double t[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const double* m = e ? lb : la;
    const double X0 = RC_S(RC_M(m[1], l2), RC_M(m[2], l1));
    const double X1 = RC_S(RC_M(m[2], l0), RC_M(m[0], l2));
    const double X2 = RC_S(RC_M(m[0], l1), RC_M(m[1], l0));
    const double nrm = __dsqrt_rn(RC_A(RC_A(RC_M(X0, X0), RC_M(X1, X1)), RC_M(X2, X2)));
    if (!(fabs(X2) > RC_M(HG_FLT_EPS, nrm))) return nan;
    const double x = RC_D(X0, X2), y = RC_D(X1, X2);
    t[e] = RC_D(RC_A(RC_M(RC_S(x, px), dx), RC_M(RC_S(y, py), dy)), len2);
  }
  const double lo = t[0] < t[1] ? t[0] : t[1], hi = t[0] < t[1] ? t[1] : t[0];
  if (!(hi > lo)) return nan;
  const double a = lo > 0.0 ? lo : 0.0, b = hi < 1.0 ? hi : 1.0;
  const double ov = b > a ? RC_S(b, a) : 0.0;
  const double span = RC_S(hi, lo);
  return RC_D(ov, span < 1.0 ? span : 1.0);
}

// Both side ratios of one matched key-line pair under F: r1 in image 1 (F a0, F b0 against s1), r0 in image 0
// (F^T a1, F^T b1 against s0); NaN where the side cannot reject.
__device__ __forceinline__ void fm_line_ratios(const double* F, const float* s0, const float* s1, double& r1,
                                               double& r0) {
  const double a0x = s0[0], a0y = s0[1], b0x = s0[2], b0y = s0[3];
  const double a1x = s1[0], a1y = s1[1], b1x = s1[2], b1y = s1[3];
  double la[3], lb[3];
  // image 1: F a0, F b0 against s1
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    la[r] = RC_A(RC_A(RC_M(F[3 * r], a0x), RC_M(F[3 * r + 1], a0y)), F[3 * r + 2]);
    lb[r] = RC_A(RC_A(RC_M(F[3 * r], b0x), RC_M(F[3 * r + 1], b0y)), F[3 * r + 2]);
  }
  r1 = fm_side_ratio(la, lb, a1x, a1y, b1x, b1y);
  // image 0: F^T a1, F^T b1 against s0
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    la[c] = RC_A(RC_A(RC_M(F[c], a1x), RC_M(F[3 + c], a1y)), F[6 + c]);
    lb[c] = RC_A(RC_A(RC_M(F[c], b1x), RC_M(F[3 + c], b1y)), F[6 + c]);
  }
  r0 = fm_side_ratio(la, lb, a0x, a0y, b0x, b0y);
}

// The decision on the two ratios: consistent iff no side's ratio is below min_overlap (a NaN side cannot reject).
__device__ __forceinline__ bool fm_ratios_consistent(double r1, double r0, double min_overlap) {
  return !(r1 < min_overlap) && !(r0 < min_overlap);
}

// The line check of one matched key-line pair under F: false iff a side's ratio is below min_overlap.
__device__ __forceinline__ bool fm_line_consistent(const double* F, const float* s0, const float* s1, double min_overlap) {
  double r1, r0;
  fm_line_ratios(F, s0, s1, r1, r0);
  return fm_ratios_consistent(r1, r0, min_overlap);
}

__global__ void __launch_bounds__(FM_FIT_THREADS) fundamental_fit_kernel(FundamentalArgs a) {
  constexpr int NT = FM_FIT_THREADS, NW = NT / 32;
  extern __shared__ __align__(16) unsigned char fm_smem[];
  __shared__ HgPair sp;
  __shared__ int warp_cnt[NW];
  __shared__ float red[NW * 8];
  __shared__ int redi[NW];
  __shared__ double ata[NW][45];
  __shared__ double sF[2][9];
  __shared__ int s_ok[2];
  pdl_launch_dependents();
  pdl_wait();
  const int p = blockIdx.x;
  const HgStage st = hg_stage_ptrs(fm_smem, a.rows, 0);
  hg_stage_pair<NT>(fm_point_args(a), p, st, sp, warp_cnt, red);
  const int n = sp.np;
  uint8_t* flh = reinterpret_cast<uint8_t*>(st.l);
  uint8_t* flr = flh + a.rows;
  const unsigned long long key = a.key[p];
  const unsigned kj = ~(unsigned)(key & 0xffffffffull);
  const int k = (int)(kj / FM_MAX_SOLUTIONS), j = (int)(kj % FM_MAX_SOLUTIONS);
  if (threadIdx.x == 0) {
    s_ok[0] = s_ok[1] = 0;
    if (n >= FM_SAMPLE && key != 0) {
      double Fs[9 * FM_MAX_SOLUTIONS];
      int jr[FM_MAX_SOLUTIONS];
      const int ns = fm_hypothesis(st, sp, a.seed, p, k, Fs, jr);
      for (int s = 0; s < ns; ++s)
        if (jr[s] == j) {
          for (int i = 0; i < 9; ++i) sF[0][i] = Fs[9 * s + i];
          s_ok[0] = 1;
        }
    }
  }
  __syncthreads();
  const bool valid = s_ok[0];
  int cnt = 0;
  const uint8_t* fl = flh;
  if (valid) {
    const int ch = fm_mark<NT>(st, n, sF[0], a.thresh2, flh, redi);
    cnt = ch;
    if (ch >= FM_MIN_REFIT) {
      // A^T A over the hypothesis' inliers (normalised epipolar rows): thread t sums rows t, t + NT, ... in order,
      // then a fixed tree
      double acc[45];
#pragma unroll
      for (int e = 0; e < 45; ++e) acc[e] = 0.0;
      for (int d = threadIdx.x; d < n; d += NT) {
        if (!flh[d]) continue;
        const float4 q = st.pt[d];
        const double x = RC_M(RC_S(q.x, sp.c0x), sp.i0), y = RC_M(RC_S(q.y, sp.c0y), sp.i0);
        const double u = RC_M(RC_S(q.z, sp.c1x), sp.i1), v = RC_M(RC_S(q.w, sp.c1y), sp.i1);
        const double r[9] = {u * x, u * y, u, v * x, v * y, v, x, y, 1.0};
        int e = 0;
#pragma unroll
        for (int i = 0; i < 9; ++i)
#pragma unroll
          for (int jj = i; jj < 9; ++jj, ++e) acc[e] += r[i] * r[jj];
      }
#pragma unroll
      for (int e = 0; e < 45; ++e) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[e] += __shfl_xor_sync(0xffffffffu, acc[e], o);
      }
      if ((threadIdx.x & 31) == 0)
#pragma unroll
        for (int e = 0; e < 45; ++e) ata[threadIdx.x >> 5][e] = acc[e];
      __syncthreads();
      if (threadIdx.x == 0) {
        double M[81], f[9];
        int e = 0;
        for (int i = 0; i < 9; ++i)
          for (int jj = i; jj < 9; ++jj, ++e) {
            double v = 0.0;
            for (int w = 0; w < NW; ++w) v += ata[w][e];
            M[9 * i + jj] = v;
            M[9 * jj + i] = v;
          }
        hg_smallest_eigvec(M, f);
        fm_rank2(f);
        s_ok[1] = fm_to_pixels(sp, f, sF[1]);
      }
      __syncthreads();
      if (s_ok[1]) {
        const int cr = fm_mark<NT>(st, n, sF[1], a.thresh2, flr, redi);
        if (cr >= ch) {
          cnt = cr;
          fl = flr;
        } else if (threadIdx.x == 0) {
          s_ok[1] = 0;
        }
      }
    }
  }
  __syncthreads();
  const int kept = s_ok[1];
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  if (threadIdx.x < 9) a.F[9ll * p + threadIdx.x] = valid ? sF[kept][threadIdx.x] : nan;
  if (threadIdx.x == 0) {
    a.valid[p] = valid;
    a.refit[p] = valid && kept;
    a.n_inl[p] = cnt;
    a.hyp_index[p] = valid ? (int)kj : -1;
    a.hyp_inliers[p] = valid ? (int)(key >> 32) : 0;
  }
  // point masks aligned with the match rows (0 for unmatched rows and invalid pairs)
  const int pb = a.cu_p[p], pe = a.cu_p[p + 1];
  if (valid) {
    hg_compact<NT>(a.matches_p, pb, pe, a.n_pts1[p], warp_cnt, [&](int i, int, int ci) {
      a.inl[pb + i] = ci >= 0 ? fl[ci] : 0;
    });
  } else {
    for (int r = pb + threadIdx.x; r < pe; r += NT) a.inl[r] = 0;
  }
  // line check, one match row per thread (0 for unmatched rows and invalid pairs)
  const int lb = a.cu_l[p], le = a.cu_l[p + 1];
  int nl = 0;
  if (lb < le) {
    double F[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) F[i] = valid ? sF[kept][i] : 0.0;
    const int n1 = a.n_segs1[p];
    const float* __restrict__ l0 = a.segs0 + 4ll * a.seg_off0[p];
    const float* __restrict__ l1 = a.segs1 + 4ll * a.seg_off1[p];
    for (int r = lb + threadIdx.x; r < le; r += NT) {
      const int m = a.matches_l[r];
      const bool ok = valid && m >= 0 && m < n1 && fm_line_consistent(F, l0 + 4ll * (r - lb), l1 + 4ll * m,
                                                                     a.min_overlap);
      a.lines_ok[r] = ok;
      nl += ok;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) nl += __shfl_xor_sync(0xffffffffu, nl, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) redi[threadIdx.x >> 5] = nl;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int i = 0; i < NW; ++i) t += redi[i];
    a.n_lines_ok[p] = t;
  }
}

}  // namespace ltr
