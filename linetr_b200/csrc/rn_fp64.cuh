// Explicitly rounded fp64 for the parity-bound geometry stages (the RANSAC estimators, absolute pose, triangulation,
// tracks and bundle adjustment).  Every operation is one of the correctly rounded intrinsics below, never contracted
// into an FMA, so a kernel gives the same bits as a numpy model that does the same operations in the same order.  The
// camera primitives shared by those stages live here once, and linetr_b200/_posed.py restates them in numpy; a new
// parity-bound stage takes its camera math from both.
#pragma once
#include "common.cuh"

#define RC_M __dmul_rn
#define RC_A __dadd_rn
#define RC_S __dsub_rn
#define RC_D __ddiv_rn

namespace ltr {

// Largest g in [0, n) with off[g] <= x (off non-decreasing, off[0] <= x < off[n]).
__device__ __forceinline__ int rc_segment(const int* __restrict__ off, int n, int x) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ double rc_dot3(const double* a, const double* b) {
  return RC_A(RC_A(RC_M(a[0], b[0]), RC_M(a[1], b[1])), RC_M(a[2], b[2]));
}

// M v for a row-major 3 x 3 M
__device__ __forceinline__ void rc_mv3(const double* M, const double* v, double* o) {
  for (int i = 0; i < 3; ++i) o[i] = rc_dot3(M + 3 * i, v);
}

__device__ __forceinline__ void rc_cross3(const double* x, const double* y, double* c) {
  c[0] = RC_S(RC_M(x[1], y[2]), RC_M(x[2], y[1]));
  c[1] = RC_S(RC_M(x[2], y[0]), RC_M(x[0], y[2]));
  c[2] = RC_S(RC_M(x[0], y[1]), RC_M(x[1], y[0]));
}

// The camera centre C = -R^T t of the world -> camera pose X_cam = R X + t (R row-major).
__device__ __forceinline__ void rc_centre(const double* R, const double* t, double* C) {
  for (int j = 0; j < 3; ++j) C[j] = -RC_A(RC_A(RC_M(R[j], t[0]), RC_M(R[3 + j], t[1])), RC_M(R[6 + j], t[2]));
}

// The world ray r = R^T ((x - cx) / fx, (y - cy) / fy, 1) of pixel (x, y): X(s) = C + s r has depth s.
__device__ __forceinline__ void rc_ray(const double* R, double fx, double fy, double cx, double cy, float x, float y,
                                       double* r) {
  const double nx = RC_D(RC_S((double)x, cx), fx), ny = RC_D(RC_S((double)y, cy), fy);
  for (int k = 0; k < 3; ++k) r[k] = RC_A(RC_A(RC_M(R[k], nx), RC_M(R[3 + k], ny)), R[6 + k]);
}

// The segment (x0, y0, x1, y1) as a unit pixel line in camera-ray form through the intrinsics c = (fx, fy, cx, cy):
// the line scaled to a^2 + b^2 = 1, then (a fx, b fy, a cx + b cy + c), so n . P / P_z is the signed pixel distance
// of the projection of the camera point P.  c is read last: the four values by argument would move those loads ahead
// and change the kernels' code.
__device__ __forceinline__ void rc_line_normal(const double* c, float4 s, double* n) {
  const double x0 = s.x, y0 = s.y, x1 = s.z, y1 = s.w;
  const double a = RC_S(y0, y1), b = RC_S(x1, x0), cc = RC_S(RC_M(x0, y1), RC_M(x1, y0));
  const double rn = RC_D(1.0, __dsqrt_rn(RC_A(RC_M(a, a), RC_M(b, b))));
  const double la = RC_M(a, rn), lb = RC_M(b, rn), lc = RC_M(cc, rn);
  n[0] = RC_M(la, c[0]);
  n[1] = RC_M(lb, c[1]);
  n[2] = RC_A(RC_A(RC_M(la, c[2]), RC_M(lb, c[3])), lc);
}

// The point X + u d of the world line through X with direction d closest to the ray C + s r, w = X - C.
__device__ __forceinline__ void rc_closest_on_line(const double* X, const double* d, const double* w, const double* r,
                                                   double* out) {
  const double aa = rc_dot3(d, d), b = rc_dot3(d, r), cc = rc_dot3(r, r), dd = rc_dot3(d, w), ee = rc_dot3(r, w);
  const double u = RC_D(RC_S(RC_M(b, ee), RC_M(cc, dd)), RC_S(RC_M(aa, cc), RC_M(b, b)));
  for (int k = 0; k < 3; ++k) out[k] = RC_A(X[k], RC_M(u, d[k]));
}

// Cayley map Q = ((1 - w.w) I + 2 [w]x + 2 w w^T) / (1 + w.w), row-major: the rotation update R <- Q R.
__device__ __forceinline__ void rc_cayley(const double* w, double* Q) {
  const double ww = RC_A(RC_A(RC_M(w[0], w[0]), RC_M(w[1], w[1])), RC_M(w[2], w[2]));
  const double den = RC_A(1.0, ww), s = RC_S(1.0, ww);
  const double wx[9] = {0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0};
  for (int i = 0; i < 3; ++i)
    for (int k = 0; k < 3; ++k)
      Q[3 * i + k] = RC_D(RC_A(RC_A(i == k ? s : 0.0, RC_M(2.0, RC_M(w[i], w[k]))), RC_M(2.0, wx[3 * i + k])), den);
}

// The dense SPD solver of one CTA of NT threads (_posed.cholesky_solve): a right-looking Cholesky of the m x m matrix
// A (leading dimension ld; the lower triangle is read and L written over it), then the forward and back substitutions
// of the k right-hand sides x [m, k] in place.  A and x may be global or shared.  s_col holds m doubles of shared
// memory; *s_fail (shared) enters as 1 to skip the call, and leaves as 1 iff a pivot was not > 0, with x untouched.
// Barriers: every thread reads the pivot A[c][c], so thread 0 writes its root l there only after the barrier that
// follows the column's scaling; the trailing update reads columns > c, and the next column's pivot read and the solves
// come after a later barrier.  On a failed pivot A keeps the columns before it as L, the pivot and the trailing lower
// triangle as its Schur complement; the upper triangle is never touched.
template <int NT>
__device__ __forceinline__ bool rc_cholesky_solve(double* A, int ld, int m, double* x, int k, double* s_col,
                                                  int* s_fail) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  // column c, then every later lower element once, in column order
  for (int c = 0; c < m && !*s_fail; ++c) {
    const double piv = A[(size_t)ld * c + c];
    if (!(piv > 0.0)) {
      __syncthreads();
      if (tid == 0) *s_fail = 1;
      break;
    }
    const double l = __dsqrt_rn(piv);
    for (int i = c + 1 + tid; i < m; i += NT) {
      const double v = RC_D(A[(size_t)ld * i + c], l);
      A[(size_t)ld * i + c] = v;
      s_col[i] = v;
    }
    __syncthreads();
    if (tid == 0) A[(size_t)ld * c + c] = l;
    // one warp per row of the trailing block, lanes over its columns c < j <= i
    for (int i = c + 1 + wid; i < m; i += NT / 32) {
      const double li = s_col[i];
      double* Ai = A + (size_t)ld * i;
      for (int j = c + 1 + lane; j <= i; j += 32) Ai[j] = RC_S(Ai[j], RC_M(li, s_col[j]));
    }
    __syncthreads();
  }
  __syncthreads();
  const bool fail = *s_fail != 0;
  if (fail) return true;
  for (int c = 0; c < m; ++c) {
    if (tid < k) x[(size_t)k * c + tid] = RC_D(x[(size_t)k * c + tid], A[(size_t)ld * c + c]);
    __syncthreads();
    for (int e = c * k + k + tid; e < m * k; e += NT) {
      const int i = e / k;
      x[e] = RC_S(x[e], RC_M(A[(size_t)ld * i + c], x[(size_t)k * c + e % k]));
    }
    __syncthreads();
  }
  for (int c = m - 1; c >= 0; --c) {
    if (tid < k) x[(size_t)k * c + tid] = RC_D(x[(size_t)k * c + tid], A[(size_t)ld * c + c]);
    __syncthreads();
    for (int e = tid; e < c * k; e += NT) {
      const int i = e / k;
      x[e] = RC_S(x[e], RC_M(A[(size_t)ld * c + i], x[(size_t)k * c + e % k]));
    }
    __syncthreads();
  }
  return false;
}

}  // namespace ltr
