// Relative pose of a batch of calibrated image pairs: five-point RANSAC essential matrices and the pose (ltr_essential).
//
// Model (DESIGN.md "Relative pose"; restated in numpy by linetr_b200.geometry.ransac_essential_host):
//   correspondences of pair p: the matched side-0 keypoints in row order with their partners, in normalised
//   coordinates x = (k - c) / f per axis (K0 for side 0, K1 for side 1).
//   threshold: f_mean = (((K0[0,0] + K1[1,1]) + K0[0,0]) + K1[1,1]) / 4 (the reference's mean), t_n = thresh / f_mean;
//   an inlier has (x1^T E x0)^2 < t_n^2 ((E x0)_0^2 + (E x0)_1^2 + (E^T x1)_0^2 + (E^T x1)_1^2) (Sampson error < t_n^2).
//   hypothesis k: 5 distinct correspondences drawn as the homography's (hg_draw), then Nister's five-point solver:
//   Householder QR of the 9 x 5 transpose of the epipolar rows -> null basis X, Y, Z, W; the 10 x 20 cubic constraints
//   of E = x X + y Y + z Z + W; Gauss-Jordan with partial pivoting; the 3 x 3 hidden-variable matrix B(z) and its
//   degree-10 determinant; its real roots by a Sturm chain and bisection; (x, y) from B(z)'s null vector.  Solution j
//   of hypothesis k is real root j (ascending).  Every operation up to here is explicitly rounded fp64 (no FMA).
//   winner: most inliers, then lowest k, then lowest j (atomicMax of (count << 32) | ~(10 k + j)).
//   outputs: E scaled to unit Frobenius norm (largest |entry| positive), its four (R, t) candidates, the one with the
//   most inliers in front of both cameras (depths from the 2 x 2 normal equations of d1 x1 = d0 R x0 + t, within
//   (0, dist_thresh)).  No refit.
//
// Kernels:
//   essential_hyp_kernel   grid (pair, chunk of ESS_THREADS hypotheses): stage the pair's normalised correspondences in
//                          shared memory, one hypothesis per thread (solver + every solution scored against every
//                          staged row), one atomicMax per CTA.
//   essential_pose_kernel  grid (pair): the winner again, inlier flags, decomposition, cheirality, the outputs.
#pragma once
#include "common.cuh"
#include "rn_fp64.cuh"
#include "ransac_common.cuh"

namespace ltr {

constexpr int ESS_THREADS = 128;          // hypotheses per CTA
constexpr int ESS_POSE_THREADS = 256;
constexpr int ESS_ROW_BYTES = 32;         // shared bytes per correspondence: a0, b0, a1, b1 fp64
constexpr int ESS_SMEM_MAX = 200 * 1024;

struct EssentialArgs {
  const float* pts0; const float* pts1;   // [*, 2] keypoint pools
  const int* pts_off0; const int* pts_off1; const int* n_pts1;
  const int* matches_p; const int* cu_p;
  const double* K0; const double* K1;     // [P, 3, 3]
  int rows;                               // staging rows per pair
  double thresh, dist_thresh;
  int n_hyp;
  unsigned long long seed;
  unsigned long long* key;
  double* E; double* R; double* t; uint8_t* valid; uint8_t* inl;
  int* n_inl; int* n_cheir; int* hyp_index; int* hyp_inliers;
};

// Dynamic shared memory of one pair: the rows, plus one flag byte per row in the pose kernel.
static inline long long ess_smem_bytes(long long rows, bool pose) { return rows * (ESS_ROW_BYTES + (pose ? 1 : 0)); }

// Products of monomials in (x, y, z): degree 1 [x, y, z, 1], degree 2 [x^2, xy, xz, x, y^2, yz, y, z^2, z, 1], degree 3
// [x^3, y^3, x^2y, xy^2, x^2z, x^2, y^2z, y^2, xyz, xy | xz^2, xz, x, yz^2, yz, y, z^3, z^2, z, 1].
__constant__ unsigned char ESS_MUL11[4][4] = {{0, 1, 2, 3}, {1, 4, 5, 6}, {2, 5, 7, 8}, {3, 6, 8, 9}};
__constant__ unsigned char ESS_MUL21[10][4] = {{0, 2, 4, 5},     {2, 3, 8, 9},     {4, 8, 10, 11}, {5, 9, 11, 12},
                                               {3, 1, 6, 7},     {8, 6, 13, 14},   {9, 7, 14, 15}, {10, 13, 16, 17},
                                               {11, 14, 17, 18}, {12, 15, 18, 19}};

// Stage pair p's normalised correspondences; returns their count to every thread.  Ends with __syncthreads.
template <int NT>
__device__ int ess_stage_pair(const EssentialArgs& a, int p, double4* rows, int* warp_cnt, int* s_n) {
  if (a.cu_p[p + 1] - a.cu_p[p] > a.rows) {   // more rows than the caller's bound: not staged, so invalid
    if (threadIdx.x == 0) *s_n = 0;
    __syncthreads();
    return 0;
  }
  const double* K0 = a.K0 + 9ll * p;
  const double* K1 = a.K1 + 9ll * p;
  const double f0x = K0[0], c0x = K0[2], f0y = K0[4], c0y = K0[5];
  const double f1x = K1[0], c1x = K1[2], f1y = K1[4], c1y = K1[5];
  const float* __restrict__ x0 = a.pts0 + 2ll * a.pts_off0[p];
  const float* __restrict__ x1 = a.pts1 + 2ll * a.pts_off1[p];
  const int n = hg_compact<NT>(a.matches_p, a.cu_p[p], a.cu_p[p + 1], a.n_pts1[p], warp_cnt, [&](int i, int m, int ci) {
    if (ci < 0) return;
    rows[ci] = make_double4(RC_D(RC_S((double)x0[2 * i], c0x), f0x), RC_D(RC_S((double)x0[2 * i + 1], c0y), f0y),
                            RC_D(RC_S((double)x1[2 * m], c1x), f1x), RC_D(RC_S((double)x1[2 * m + 1], c1y), f1y));
  });
  if (threadIdx.x == 0) *s_n = n;
  __syncthreads();
  return n;
}

// t_n^2 of pair p.
__device__ __forceinline__ double ess_t2(const EssentialArgs& a, int p) {
  const double* K0 = a.K0 + 9ll * p;
  const double* K1 = a.K1 + 9ll * p;
  const double fm = RC_D(RC_A(RC_A(RC_A(K0[0], K1[4]), K0[0]), K1[4]), 4.0);
  const double tn = RC_D(a.thresh, fm);
  return RC_M(tn, tn);
}

__device__ __forceinline__ void ess_mul11(const double* x, const double* y, double* out) {
#pragma unroll
  for (int m = 0; m < 10; ++m) out[m] = 0.0;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) out[ESS_MUL11[i][j]] = RC_A(out[ESS_MUL11[i][j]], RC_M(x[i], y[j]));
}

__device__ __forceinline__ void ess_sub(double* x, const double* y, int n) {
  for (int i = 0; i < n; ++i) x[i] = RC_S(x[i], y[i]);
}

// out (20) = x (degree 2) * y (degree 1)
__device__ __forceinline__ void ess_mul21(const double* x, const double* y, double* out) {
  for (int m = 0; m < 20; ++m) out[m] = 0.0;
  for (int i = 0; i < 10; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) out[ESS_MUL21[i][j]] = RC_A(out[ESS_MUL21[i][j]], RC_M(x[i], y[j]));
}

// The five-point solver on 5 normalised correspondences q[s] = (a0, b0, a1, b1): up to 10 E (row-major, Es[9 s]) with
// their root indices jr[s].  -> solution count.
__device__ __noinline__ int ess_solve(const double4* q, double* Es, int* jr) {
  // null basis X, Y, Z, W of the 5 epipolar rows; e[i] = entry i of E as a polynomial [x, y, z, 1]
  double e[9][4];
  if (!rc_null_basis<5>(q, e)) return 0;
  // the 10 x 20 constraints: det E, then (2 E E^T - tr(E E^T) I) E row-major
  double C[10][20];
  {
    double t1[10], t2[10], u[20];
    ess_mul11(e[4], e[8], t1); ess_mul11(e[5], e[7], t2); ess_sub(t1, t2, 10); ess_mul21(t1, e[0], C[0]);
    ess_mul11(e[3], e[8], t1); ess_mul11(e[5], e[6], t2); ess_sub(t1, t2, 10); ess_mul21(t1, e[1], u);
    ess_sub(C[0], u, 20);
    ess_mul11(e[3], e[7], t1); ess_mul11(e[4], e[6], t2); ess_sub(t1, t2, 10); ess_mul21(t1, e[2], u);
    for (int m = 0; m < 20; ++m) C[0][m] = RC_A(C[0][m], u[m]);
    double L[6][10];   // (0,0) (0,1) (0,2) (1,1) (1,2) (2,2) of E E^T, then 2 E E^T - tr I
    int w = 0;
    for (int i = 0; i < 3; ++i)
      for (int k = i; k < 3; ++k, ++w) {
        ess_mul11(e[3 * i], e[3 * k], L[w]);
        ess_mul11(e[3 * i + 1], e[3 * k + 1], t1);
        for (int m = 0; m < 10; ++m) L[w][m] = RC_A(L[w][m], t1[m]);
        ess_mul11(e[3 * i + 2], e[3 * k + 2], t1);
        for (int m = 0; m < 10; ++m) L[w][m] = RC_A(L[w][m], t1[m]);
      }
    double tr[10];
    for (int m = 0; m < 10; ++m) tr[m] = RC_A(RC_A(L[0][m], L[3][m]), L[5][m]);
    for (int w2 = 0; w2 < 6; ++w2) {
      const bool diag = w2 == 0 || w2 == 3 || w2 == 5;
      for (int m = 0; m < 10; ++m) L[w2][m] = diag ? RC_S(RC_M(L[w2][m], 2.0), tr[m]) : RC_M(L[w2][m], 2.0);
    }
    const int li[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        double* row = C[1 + 3 * i + j];
        ess_mul21(L[li[i][0]], e[j], row);
        ess_mul21(L[li[i][1]], e[3 + j], u);
        for (int m = 0; m < 20; ++m) row[m] = RC_A(row[m], u[m]);
        ess_mul21(L[li[i][2]], e[6 + j], u);
        for (int m = 0; m < 20; ++m) row[m] = RC_A(row[m], u[m]);
      }
  }
  // Gauss-Jordan on the first 10 columns
  for (int c = 0; c < 10; ++c) {
    int piv = c;
    double best = fabs(C[c][c]);
    for (int r = c + 1; r < 10; ++r)
      if (fabs(C[r][c]) > best) { best = fabs(C[r][c]); piv = r; }
    if (!(best > 0.0)) return 0;
    if (piv != c)
      for (int j = 0; j < 20; ++j) { const double tmp = C[c][j]; C[c][j] = C[piv][j]; C[piv][j] = tmp; }
    const double pv = C[c][c];
    for (int j = c + 1; j < 20; ++j) C[c][j] = RC_D(C[c][j], pv);
    for (int r = 0; r < 10; ++r) {
      if (r == c) continue;
      const double f = C[r][c];
      for (int j = c + 1; j < 20; ++j) C[r][j] = RC_S(C[r][j], RC_M(f, C[c][j]));
    }
  }
  // hidden-variable matrix B(z): rows x^2z - z x^2, y^2z - z y^2, xyz - z xy; B[r] = bx (4), by (4), b1 (5)
  double B[3][13];
  for (int r = 0; r < 3; ++r) {
    const double* ru = C[4 + 2 * r] + 10;
    const double* rl = C[5 + 2 * r] + 10;
    double* b = B[r];
    b[0] = -ru[2]; b[1] = RC_S(rl[2], ru[1]); b[2] = RC_S(rl[1], ru[0]); b[3] = rl[0];
    b[4] = -ru[5]; b[5] = RC_S(rl[5], ru[4]); b[6] = RC_S(rl[4], ru[3]); b[7] = rl[3];
    b[8] = -ru[9]; b[9] = RC_S(rl[9], ru[8]); b[10] = RC_S(rl[8], ru[7]); b[11] = RC_S(rl[7], ru[6]); b[12] = rl[6];
  }
  double poly[11];
  {
    double x8[8], y8[8], t[11];
    // t0 = B00 (B11 B22 - B12 B21)
    ess_pmul(B[1] + 4, 4, B[2] + 8, 5, x8); ess_pmul(B[1] + 8, 5, B[2] + 4, 4, y8); ess_sub(x8, y8, 8);
    ess_pmul(B[0], 4, x8, 8, poly);
    // t1 = B01 (B10 B22 - B12 B20)
    ess_pmul(B[1], 4, B[2] + 8, 5, x8); ess_pmul(B[1] + 8, 5, B[2], 4, y8); ess_sub(x8, y8, 8);
    ess_pmul(B[0] + 4, 4, x8, 8, t);
    ess_sub(poly, t, 11);
    // t2 = B02 (B10 B21 - B11 B20)
    ess_pmul(B[1], 4, B[2] + 4, 4, x8); ess_pmul(B[1] + 4, 4, B[2], 4, y8); ess_sub(x8, y8, 7);
    ess_pmul(B[0] + 8, 5, x8, 7, t);
    for (int i = 0; i < 11; ++i) poly[i] = RC_A(poly[i], t[i]);
  }
  double roots[10];
  const int nr = ess_roots(poly, roots);
  int ns = 0;
  for (int j = 0; j < nr; ++j) {
    const double z = roots[j];
    double rw[3][3];
    for (int r = 0; r < 3; ++r) {
      rw[r][0] = ess_horner(B[r], 3, z);
      rw[r][1] = ess_horner(B[r] + 4, 3, z);
      rw[r][2] = ess_horner(B[r] + 8, 4, z);
    }
    double best[3], c[3];
    rc_cross3(rw[0], rw[1], best);
    rc_cross3(rw[0], rw[2], c);
    if (fabs(c[2]) > fabs(best[2])) { best[0] = c[0]; best[1] = c[1]; best[2] = c[2]; }
    rc_cross3(rw[1], rw[2], c);
    if (fabs(c[2]) > fabs(best[2])) { best[0] = c[0]; best[1] = c[1]; best[2] = c[2]; }
    if (!(fabs(best[2]) > 0.0)) continue;
    const double x = RC_D(best[0], best[2]), y = RC_D(best[1], best[2]);
    double* E = Es + 9 * ns;
    bool fin = true;
    for (int i = 0; i < 9; ++i) {
      E[i] = RC_A(RC_A(RC_A(RC_M(x, e[i][0]), RC_M(y, e[i][1])), RC_M(z, e[i][2])), e[i][3]);
      fin &= isfinite(E[i]);
    }
    if (!fin) continue;
    jr[ns++] = j;
  }
  return ns;
}

__device__ __forceinline__ bool ess_inlier(const double* e, const double4 q, double t2) {
  const double u0 = RC_A(RC_A(RC_M(e[0], q.x), RC_M(e[1], q.y)), e[2]);
  const double u1 = RC_A(RC_A(RC_M(e[3], q.x), RC_M(e[4], q.y)), e[5]);
  const double u2 = RC_A(RC_A(RC_M(e[6], q.x), RC_M(e[7], q.y)), e[8]);
  const double w0 = RC_A(RC_A(RC_M(e[0], q.z), RC_M(e[3], q.w)), e[6]);
  const double w1 = RC_A(RC_A(RC_M(e[1], q.z), RC_M(e[4], q.w)), e[7]);
  const double num = RC_A(RC_A(RC_M(q.z, u0), RC_M(q.w, u1)), u2);
  const double den = RC_A(RC_A(RC_A(RC_M(u0, u0), RC_M(u1, u1)), RC_M(w0, w0)), RC_M(w1, w1));
  return RC_M(num, num) < RC_M(t2, den);
}

__global__ void __launch_bounds__(ESS_THREADS) essential_hyp_kernel(EssentialArgs a) {
  extern __shared__ __align__(16) unsigned char es_smem[];
  __shared__ int warp_cnt[ESS_THREADS / 32];
  __shared__ int s_n;
  __shared__ unsigned long long wbest[ESS_THREADS / 32];
  pdl_launch_dependents();
  pdl_wait();
  const int p = blockIdx.x;
  const double4* rows = reinterpret_cast<const double4*>(es_smem);
  const int n = ess_stage_pair<ESS_THREADS>(a, p, reinterpret_cast<double4*>(es_smem), warp_cnt, &s_n);
  if (n < 5) return;
  const int k = blockIdx.y * ESS_THREADS + threadIdx.x;
  unsigned long long key = 0;
  int idx[5];
  if (k < a.n_hyp && hg_draw<5>(a.seed, p, k, n, idx)) {
    const double t2 = ess_t2(a, p);
    double4 q[5];
    for (int s = 0; s < 5; ++s) q[s] = rows[idx[s]];
    double Es[90];
    int jr[10];
    const int ns = ess_solve(q, Es, jr);
    for (int s = 0; s < ns; ++s) {
      double e[9];
#pragma unroll
      for (int i = 0; i < 9; ++i) e[i] = Es[9 * s + i];
      unsigned cnt = 0;
      for (int d = 0; d < n; ++d) cnt += ess_inlier(e, rows[d], t2);
      const unsigned long long kk =
          ((unsigned long long)cnt << 32) | (unsigned long long)(~(unsigned)(10 * k + jr[s]));
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
    for (int i = 1; i < ESS_THREADS / 32; ++i) key = wbest[i] > key ? wbest[i] : key;
    if (key) atomicMax(a.key + p, key);
  }
}

// Unit-Frobenius E (largest |entry| positive) -> its four (R, t) candidates in OpenCV's order (R1, t), (R2, t),
// (R1, -t), (R2, -t): V from a cyclic Jacobi eigen-decomposition of E^T E, U from E V.  cand[c] = R (9), t (3).
__device__ __noinline__ void ess_decompose(const double* E, double (*cand)[12]) {
  double S[3][3], V[3][3];
  for (int i = 0; i < 3; ++i)
    for (int k = 0; k < 3; ++k) {
      S[i][k] = E[i] * E[k] + E[3 + i] * E[3 + k] + E[6 + i] * E[6 + k];
      V[i][k] = i == k ? 1.0 : 0.0;
    }
  rc_jacobi3(S, V);
  int i0 = 0, i2 = 0;
  for (int i = 1; i < 3; ++i) {
    if (S[i][i] > S[i0][i0]) i0 = i;
    if (S[i][i] < S[i2][i2]) i2 = i;
  }
  if (i2 == i0) i2 = (i0 + 2) % 3;
  const int i1 = 3 - i0 - i2;
  double v1[3], v2[3], v3[3], u1[3], u2[3], u3[3];
  for (int k = 0; k < 3; ++k) { v1[k] = V[k][i0]; v2[k] = V[k][i1]; }
  rc_cross3(v1, v2, v3);
  for (int r = 0; r < 3; ++r) {
    u1[r] = E[3 * r] * v1[0] + E[3 * r + 1] * v1[1] + E[3 * r + 2] * v1[2];
    u2[r] = E[3 * r] * v2[0] + E[3 * r + 1] * v2[1] + E[3 * r + 2] * v2[2];
  }
  double n1 = sqrt(u1[0] * u1[0] + u1[1] * u1[1] + u1[2] * u1[2]);
  for (int r = 0; r < 3; ++r) u1[r] /= n1;
  const double d = u1[0] * u2[0] + u1[1] * u2[1] + u1[2] * u2[2];
  for (int r = 0; r < 3; ++r) u2[r] -= d * u1[r];
  const double n2 = sqrt(u2[0] * u2[0] + u2[1] * u2[1] + u2[2] * u2[2]);
  for (int r = 0; r < 3; ++r) u2[r] /= n2;
  rc_cross3(u1, u2, u3);
  // R1 = U W V^T = -u2 v1^T + u1 v2^T + u3 v3^T, R2 = U W^T V^T = u2 v1^T - u1 v2^T + u3 v3^T, t = u3
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      const double a = u1[r] * v2[c] - u2[r] * v1[c], b = u3[r] * v3[c];
      cand[0][3 * r + c] = cand[2][3 * r + c] = a + b;
      cand[1][3 * r + c] = cand[3][3 * r + c] = b - a;
    }
  for (int r = 0; r < 3; ++r) {
    cand[0][9 + r] = cand[1][9 + r] = u3[r];
    cand[2][9 + r] = cand[3][9 + r] = -u3[r];
  }
}

// Depths of d1 x1 = d0 R x0 + t from the 2 x 2 normal equations; true when both lie in (0, dist).
__device__ __forceinline__ bool ess_in_front(const double* c, const double4 q, double dist) {
  const double ax = RC_A(RC_A(RC_M(c[0], q.x), RC_M(c[1], q.y)), c[2]);
  const double ay = RC_A(RC_A(RC_M(c[3], q.x), RC_M(c[4], q.y)), c[5]);
  const double az = RC_A(RC_A(RC_M(c[6], q.x), RC_M(c[7], q.y)), c[8]);
  const double aa = RC_A(RC_A(RC_M(ax, ax), RC_M(ay, ay)), RC_M(az, az));
  const double ab = RC_A(RC_A(RC_M(ax, q.z), RC_M(ay, q.w)), az);
  const double bb = RC_A(RC_A(RC_M(q.z, q.z), RC_M(q.w, q.w)), 1.0);
  const double at = RC_A(RC_A(RC_M(ax, c[9]), RC_M(ay, c[10])), RC_M(az, c[11]));
  const double bt = RC_A(RC_A(RC_M(q.z, c[9]), RC_M(q.w, c[10])), c[11]);
  const double det = RC_S(RC_M(ab, ab), RC_M(aa, bb));
  const double d0 = RC_D(RC_S(RC_M(at, bb), RC_M(ab, bt)), det);
  const double d1 = RC_D(RC_S(RC_M(ab, at), RC_M(aa, bt)), det);
  return d0 > 0.0 && d0 < dist && d1 > 0.0 && d1 < dist;
}

__global__ void __launch_bounds__(ESS_POSE_THREADS) essential_pose_kernel(EssentialArgs a) {
  constexpr int NT = ESS_POSE_THREADS, NW = NT / 32;
  extern __shared__ __align__(16) unsigned char es_smem[];
  __shared__ int warp_cnt[NW];
  __shared__ int s_n, s_ok, s_best;
  __shared__ int red[NW][5];
  __shared__ double sE[9], sEu[9];   // the winning solution, scaled to unit norm
  __shared__ double cand[4][12];
  pdl_launch_dependents();
  pdl_wait();
  const int p = blockIdx.x;
  const double4* rows = reinterpret_cast<const double4*>(es_smem);
  const int n = ess_stage_pair<NT>(a, p, reinterpret_cast<double4*>(es_smem), warp_cnt, &s_n);
  uint8_t* fl = es_smem + (size_t)a.rows * ESS_ROW_BYTES;
  const unsigned long long key = a.key[p];
  const unsigned kj = ~(unsigned)(key & 0xffffffffull);
  const int k = (int)(kj / 10u), j = (int)(kj % 10u);
  if (threadIdx.x == 0) {
    s_ok = 0;
    int idx[5];
    if (n >= 5 && key != 0 && hg_draw<5>(a.seed, p, k, n, idx)) {
      double4 q[5];
      for (int s = 0; s < 5; ++s) q[s] = rows[idx[s]];
      double Es[90];
      int jr[10];
      const int ns = ess_solve(q, Es, jr);
      for (int s = 0; s < ns; ++s)
        if (jr[s] == j) {
          for (int i = 0; i < 9; ++i) sE[i] = Es[9 * s + i];
          s_ok = 1;
        }
    }
  }
  __syncthreads();
  const bool valid = s_ok;
  int cnt = 0, cc[4] = {0, 0, 0, 0};
  if (valid) {
    const double t2 = ess_t2(a, p);
    double e[9];
    for (int i = 0; i < 9; ++i) e[i] = sE[i];
    for (int d = threadIdx.x; d < n; d += NT) {
      const bool in = ess_inlier(e, rows[d], t2);
      fl[d] = in;
      cnt += in;
    }
    if (threadIdx.x == 0) {
      // unit Frobenius norm, largest |entry| positive
      double f = 0.0;
      for (int i = 0; i < 9; ++i) f += e[i] * e[i];
      f = sqrt(f);
      int im = 0;
      for (int i = 1; i < 9; ++i)
        if (fabs(e[i]) > fabs(e[im])) im = i;
      const double sc = e[im] > 0.0 ? 1.0 / f : -1.0 / f;
      for (int i = 0; i < 9; ++i) sEu[i] = e[i] * sc;
      ess_decompose(sEu, cand);
    }
    __syncthreads();
    for (int d = threadIdx.x; d < n; d += NT) {
      if (!fl[d]) continue;
      const double4 q = rows[d];
#pragma unroll
      for (int c = 0; c < 4; ++c) cc[c] += ess_in_front(cand[c], q, a.dist_thresh);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
#pragma unroll
    for (int c = 0; c < 4; ++c) cc[c] += __shfl_xor_sync(0xffffffffu, cc[c], o);
  }
  if ((threadIdx.x & 31) == 0) {
    red[threadIdx.x >> 5][0] = cnt;
#pragma unroll
    for (int c = 0; c < 4; ++c) red[threadIdx.x >> 5][1 + c] = cc[c];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int tot[5] = {0, 0, 0, 0, 0};
    for (int w = 0; w < NW; ++w)
      for (int i = 0; i < 5; ++i) tot[i] += red[w][i];
    int b = 0;
    for (int c = 1; c < 4; ++c)
      if (tot[1 + c] > tot[1 + b]) b = c;
    s_best = b;
    a.valid[p] = valid;
    a.n_inl[p] = valid ? tot[0] : 0;
    a.n_cheir[p] = valid ? tot[1 + b] : 0;
    a.hyp_index[p] = valid ? (int)kj : -1;
    a.hyp_inliers[p] = valid ? (int)(key >> 32) : 0;
  }
  __syncthreads();
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  if (threadIdx.x < 9) {
    a.E[9ll * p + threadIdx.x] = valid ? sEu[threadIdx.x] : nan;
    a.R[9ll * p + threadIdx.x] = valid ? cand[s_best][threadIdx.x] : nan;
  } else if (threadIdx.x < 12) {
    a.t[3ll * p + threadIdx.x - 9] = valid ? cand[s_best][threadIdx.x] : nan;
  }
  // masks aligned with the match rows (0 for unmatched rows and invalid pairs)
  const int pb = a.cu_p[p], pe = a.cu_p[p + 1];
  if (valid) {
    hg_compact<NT>(a.matches_p, pb, pe, a.n_pts1[p], warp_cnt, [&](int i, int, int ci) {
      a.inl[pb + i] = ci >= 0 ? fl[ci] : 0;
    });
  } else {
    for (int r = pb + threadIdx.x; r < pe; r += NT) a.inl[r] = 0;
  }
}

}  // namespace ltr
