// Absolute pose of query images from point and line matches to database images with 3D coordinates: P3P RANSAC over
// the point matches, scored and refined with the line matches too (ltr_absolute_pose).
//
// Model (DESIGN.md "Absolute pose"; restated in numpy by linetr_b200.localization.ransac_absolute_pose_host):
//   side 0 is the query, side 1 a database image whose keypoint / key-line rows have world coordinates (fp64, NaN: no
//   3D); the pose maps world to query camera, X_cam = R X + t.  Group g is the run of pairs [groups[g], groups[g+1])
//   of one query; its correspondences are its pairs' point rows in pair and row order (a matched side-0 keypoint whose
//   partner has finite 3D), then its line rows (a matched side-0 segment whose partner has two finite end points).
//   World coordinates are shifted by the midpoint c of the bounding box of the group's staged 3D coordinates.
//   hypothesis k: 3 distinct point rows drawn as the homography's (hg_draw), then Grunert's P3P: bearings of
//   ((k - c) / f, 1), the quartic in v = s3 / s1 (Haralick et al. 1994, section 2.1), its real roots by the Sturm chain
//   and bisection (ess_roots), u from the back-substitution, s1 = sqrt(b^2 / (1 + v^2 - 2 v cos beta)); a root with a
//   zero divisor or u, v <= 0 is dropped; R from the triads of the camera and world points, t = P1 - R X1.  Solution j
//   is real root j.  A sample whose world cross-product norm is at most AP_COLLINEAR_EPS times its edge lengths has
//   none.  Every operation is explicitly rounded fp64.
//   inlier (pixels through K0): a point iff depth > 0 and |fx Px - (kx - cx) Pz|^2 + |fy Py - (ky - cy) Pz|^2 <
//   thresh^2 Pz^2 (the squared reprojection error below thresh^2 without the division); a line iff both end points
//   have depth > 0 and (n . P)^2 < thresh^2 Pz^2 for each, n the query line through s0 in camera-ray form.
//   line hypotheses (ltr_absolute_pose_lines): hypothesis k of line solver s (0 P2P1L, 1 P1P2L, 2 P3L) draws 2 - s
//   point rows and s + 1 line rows and solves them through two bilinear trigonometric equations (ap_line_pose), up to
//   8 solutions; its index is 4 n_hyp + 8 (s n_line_hyp + k) + j.
//   winner: most inliers (points and lines), then lowest index (atomicMax of (count << 32) | ~index, 4 k + j for P3P).
//   refit (at least AP_MIN_REFIT winner inliers): Levenberg-Marquardt over the winner's inliers, R <- cay(w) R,
//   t <- t + dt, J^T J and J^T r summed in a fixed order, the damped 6 x 6 system by Gaussian elimination with partial
//   pivoting, a fixed budget and damping schedule; kept iff its inlier count >= the hypothesis'.
//
// Kernels:
//   abspose_hyp_kernel  grid (group, chunk of AP_THREADS hypotheses): stage the group's rows, one hypothesis per
//                       thread (P3P + up to 4 solutions scored against every staged row), one atomicMax per CTA.
//   abspose_line_hyp_kernel  grid (group, chunk of AP_THREADS over 3 n_line_hyp): the same for the line hypotheses
//                       (up to 8 solutions each), into the same key; launched only with n_line_hyp > 0.
//   abspose_fit_kernel  grid (group): the winner again, the block-parallel refit, the masks, counts and pose.
#pragma once
#include "common.cuh"
#include "rn_fp64.cuh"
#include "ransac_common.cuh"

namespace ltr {

constexpr int AP_THREADS = 128;            // hypotheses per CTA
constexpr int AP_FIT_THREADS = 256;
constexpr int AP_SAMPLE = 3;
constexpr int AP_MAX_SOLUTIONS = 4;
constexpr int AP_MIN_REFIT = 3;            // winner inliers needed for the refit
constexpr int AP_LM_ITERS = 20;            // Levenberg-Marquardt steps (fixed budget)
constexpr double AP_LM_LAMBDA0 = 1e-3;     // initial damping (A_ii + lambda A_ii)
constexpr double AP_LM_ACCEPT = 0.1;       // damping factor after a step that lowers the cost
constexpr double AP_LM_REJECT = 10.0;      // damping factor after one that does not
constexpr double AP_COLLINEAR_EPS = 1e-10;
// Line hypotheses (ap_line_pose): solver s = 0 P2P1L, 1 P1P2L, 2 P3L samples 2 - s point and s + 1 line rows and
// gives up to AP_LINE_MAX_SOLUTIONS poses (the real roots of a degree-8 polynomial).
constexpr int AP_LINE_SOLVERS = 3;
constexpr int AP_LINE_MAX_SOLUTIONS = 8;
constexpr int AP_LINE_MAX_HYP = 1 << 21;   // n_line_hypotheses bound: the index space fits int32, the grid y 65535
constexpr double AP_BEARING_EPS = 1e-10;    // P2P1L: |j1 x j2| of the unit bearings at most this rejects the sample
constexpr double AP_POINT_LINE_EPS = 1e-10; // P1P2L: |n1 . j1| / |n1| at most this (the point on line 1) rejects it
constexpr double AP_CONCURRENT_EPS = 1e-10; // P3L: |n1 . (n2 x n3)| at most this times |n1| |n2| |n3| rejects it
constexpr int AP_PT_BYTES = 32;            // shared bytes per point row: query pixel fp32, world point fp64
constexpr int AP_LN_BYTES = 64;            // per line row: query segment fp32, two world end points fp64
constexpr int AP_SMEM_MAX = 200 * 1024;
constexpr int AP_TERMS = 28;               // J^T J (upper triangle, 21), J^T r (6), r^T r

struct AbsPoseArgs {
  const float* pts0; const int* pts_off0;    // [*, 2] query keypoint pool, per-pair first row
  const int* matches_p; const int* cu_p;
  const double* X1; const int* x_off1; const int* n_x1;   // [*, 3] world points of the database keypoints
  const float* segs0; const int* seg_off0;   // [*, 2, 2] query segment pool
  const int* matches_l; const int* cu_l;
  const double* L1; const int* l_off1; const int* n_l1;   // [*, 2, 3] world end points of the database key lines
  const int* groups; const double* K0;       // [G + 1] pair offsets, [G, 3, 3]
  int rows_p, rows_l;                        // staging rows per group (rows_l 0: lines unused)
  double thresh2;
  int n_hyp;
  int n_line_hyp;                            // hypotheses per line solver
  unsigned long long seed;
  unsigned long long* key;
  double* R; double* t; uint8_t* valid; uint8_t* refit; uint8_t* inl_p; uint8_t* inl_l;
  int* n_inl_p; int* n_inl_l; int* hyp_index; int* hyp_inliers;
};

// Dynamic shared memory of one group (both kernels).
static inline long long ap_smem_bytes(long long rows_p, long long rows_l) {
  return rows_p * AP_PT_BYTES + rows_l * AP_LN_BYTES;
}

struct ApGroup {
  int np, nl;
  double fx, fy, cx, cy;
  double c[3];   // the world shift
};

struct ApStage {
  float4* s0;   // [rows_l] query segments
  float2* k;    // [rows_p] query pixels
  double* X;    // [3 rows_p] shifted world points
  double* E;    // [6 rows_l] shifted world end points
};

__device__ __forceinline__ ApStage ap_stage_ptrs(unsigned char* base, int rows_p, int rows_l) {
  ApStage st;
  st.s0 = reinterpret_cast<float4*>(base);
  st.k = reinterpret_cast<float2*>(st.s0 + rows_l);
  st.X = reinterpret_cast<double*>(st.k + rows_p);
  st.E = st.X + 3 * rows_p;
  return st;
}

// Stage group g's rows and its frame.  Ends with __syncthreads.
template <int NT>
__device__ void ap_stage_group(const AbsPoseArgs& a, int g, const ApStage& st, ApGroup& sg, int* warp_cnt, double* red) {
  const int pb = a.groups[g], pe = a.groups[g + 1];
  // A group with more match rows than the staging bounds is left without correspondences (so invalid) rather than
  // written past its shared memory: the bounds come from the caller.
  if (a.cu_p[pe] - a.cu_p[pb] > a.rows_p || (a.rows_l && a.cu_l[pe] - a.cu_l[pb] > a.rows_l)) {
    if (threadIdx.x == 0) sg.np = sg.nl = 0;
    __syncthreads();
    return;
  }
  int np = 0, nl = 0;
  if (a.rows_p) {
    for (int p = pb; p < pe; ++p) {
      const float* __restrict__ x0 = a.pts0 + 2ll * a.pts_off0[p];
      const double* __restrict__ X1 = a.X1 + 3ll * a.x_off1[p];
      const int n1 = a.n_x1[p], base = np;
      np += rc_compact_if<NT>(
          a.matches_p, a.cu_p[p], a.cu_p[p + 1], warp_cnt,
          [&](int m) {
            return m >= 0 && m < n1 && isfinite(X1[3 * m]) && isfinite(X1[3 * m + 1]) && isfinite(X1[3 * m + 2]);
          },
          [&](int i, int m, int ci) {
            if (ci < 0) return;
            st.k[base + ci] = make_float2(x0[2 * i], x0[2 * i + 1]);
#pragma unroll
            for (int e = 0; e < 3; ++e) st.X[3 * (base + ci) + e] = X1[3 * m + e];
          });
    }
  }
  if (a.rows_l) {
    for (int p = pb; p < pe; ++p) {
      const float* __restrict__ l0 = a.segs0 + 4ll * a.seg_off0[p];
      const double* __restrict__ L1 = a.L1 + 6ll * a.l_off1[p];
      const int n1 = a.n_l1[p], base = nl;
      nl += rc_compact_if<NT>(
          a.matches_l, a.cu_l[p], a.cu_l[p + 1], warp_cnt,
          [&](int m) {
            bool ok = m >= 0 && m < n1;
            for (int e = 0; ok && e < 6; ++e) ok = isfinite(L1[6 * m + e]);
            return ok;
          },
          [&](int i, int m, int ci) {
            if (ci < 0) return;
            st.s0[base + ci] = make_float4(l0[4 * i], l0[4 * i + 1], l0[4 * i + 2], l0[4 * i + 3]);
#pragma unroll
            for (int e = 0; e < 6; ++e) st.E[6 * (base + ci) + e] = L1[6 * m + e];
          });
    }
  }
  // bounding box of the staged world coordinates: min x, y, z, then -max x, y, z
  double v[6];
#pragma unroll
  for (int e = 0; e < 6; ++e) v[e] = INFINITY;
  auto add = [&](const double* X) {
#pragma unroll
    for (int e = 0; e < 3; ++e) {
      v[e] = fmin(v[e], X[e]);
      v[3 + e] = fmin(v[3 + e], -X[e]);
    }
  };
  for (int i = threadIdx.x; i < np; i += NT) add(st.X + 3 * i);
  for (int i = threadIdx.x; i < 2 * nl; i += NT) add(st.E + 3 * i);
#pragma unroll
  for (int e = 0; e < 6; ++e)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[e] = fmin(v[e], __shfl_xor_sync(0xffffffffu, v[e], o));
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0)
#pragma unroll
    for (int e = 0; e < 6; ++e) red[w * 6 + e] = v[e];
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < NT / 32; ++i)
      for (int e = 0; e < 6; ++e) red[e] = fmin(red[e], red[i * 6 + e]);
    for (int e = 0; e < 3; ++e) sg.c[e] = np + nl ? RC_M(RC_A(red[e], -red[3 + e]), 0.5) : 0.0;
    const double* K = a.K0 + 9ll * g;
    sg.fx = K[0]; sg.cx = K[2]; sg.fy = K[4]; sg.cy = K[5];
    sg.np = np;
    sg.nl = nl;
  }
  __syncthreads();
  const double c0 = sg.c[0], c1 = sg.c[1], c2 = sg.c[2];
  for (int i = threadIdx.x; i < np; i += NT) {
    st.X[3 * i] = RC_S(st.X[3 * i], c0);
    st.X[3 * i + 1] = RC_S(st.X[3 * i + 1], c1);
    st.X[3 * i + 2] = RC_S(st.X[3 * i + 2], c2);
  }
  for (int i = threadIdx.x; i < 2 * nl; i += NT) {
    st.E[3 * i] = RC_S(st.E[3 * i], c0);
    st.E[3 * i + 1] = RC_S(st.E[3 * i + 1], c1);
    st.E[3 * i + 2] = RC_S(st.E[3 * i + 2], c2);
  }
  __syncthreads();
}

// Grunert's P3P on unit bearings j[3 s .. 3 s + 2] and world points X[3 s ..] of the sample's points s = 0, 1, 2: up
// to 4 poses (Rs[9 i] row-major, ts[3 i]) with their root indices jr[i].  -> solution count.
__device__ __noinline__ int ap_p3p(const double* j, const double* X, double* Rs, double* ts, int* jr) {
  double d1[3], d2[3], d3[3];
#pragma unroll
  for (int e = 0; e < 3; ++e) {
    d1[e] = RC_S(X[3 + e], X[e]);
    d2[e] = RC_S(X[6 + e], X[e]);
    d3[e] = RC_S(X[6 + e], X[3 + e]);
  }
  const double c2 = rc_dot3(d1, d1), b2 = rc_dot3(d2, d2), a2 = rc_dot3(d3, d3);
  double cr[3];
  rc_cross3(d1, d2, cr);
  const double n1 = __dsqrt_rn(c2), n2 = __dsqrt_rn(b2), ncr = __dsqrt_rn(rc_dot3(cr, cr));
  if (!(ncr > RC_M(RC_M(AP_COLLINEAR_EPS, n1), n2))) return 0;   // collinear world points
  const double ca = rc_dot3(j + 3, j + 6), cb = rc_dot3(j, j + 6), cg = rc_dot3(j, j + 3);
  const double p = RC_D(RC_S(a2, c2), b2), q = RC_D(RC_A(a2, c2), b2);
  const double rc = RC_D(c2, b2), ra = RC_D(a2, b2), rbc = RC_D(RC_S(b2, c2), b2), rba = RC_D(RC_S(b2, a2), b2);
  const double ca2 = RC_M(ca, ca), cb2 = RC_M(cb, cb), cg2 = RC_M(cg, cg);
  const double pm1 = RC_S(p, 1.0), pp1 = RC_A(p, 1.0), omq = RC_S(1.0, q);
  double poly[11];
  poly[4] = RC_S(RC_M(pm1, pm1), RC_M(RC_M(4.0, rc), ca2));
  poly[3] = RC_M(4.0, RC_A(RC_S(RC_M(RC_M(p, RC_S(1.0, p)), cb), RC_M(RC_M(omq, ca), cg)),
                           RC_M(RC_M(RC_M(2.0, rc), ca2), cb)));
  poly[2] = RC_M(2.0, RC_A(RC_S(RC_A(RC_A(RC_S(RC_M(p, p), 1.0), RC_M(RC_M(2.0, RC_M(p, p)), cb2)),
                                     RC_M(RC_M(2.0, rbc), ca2)),
                                RC_M(RC_M(RC_M(RC_M(4.0, q), ca), cb), cg)),
                           RC_M(RC_M(2.0, rba), cg2)));
  poly[1] = RC_M(4.0, RC_S(RC_A(-RC_M(RC_M(p, pp1), cb), RC_M(RC_M(RC_M(2.0, ra), cg2), cb)), RC_M(RC_M(omq, ca), cg)));
  poly[0] = RC_S(RC_M(pp1, pp1), RC_M(RC_M(4.0, ra), cg2));
  for (int i = 5; i < 11; ++i) poly[i] = 0.0;
  double roots[10];
  const int nr = ess_roots(poly, roots);
  double e1[3], e2[3], e3[3];
#pragma unroll
  for (int e = 0; e < 3; ++e) {
    e1[e] = RC_D(d1[e], n1);
    e3[e] = RC_D(cr[e], ncr);
  }
  rc_cross3(e3, e1, e2);
  int ns = 0;
  for (int r = 0; r < nr && r < AP_MAX_SOLUTIONS; ++r) {
    const double v = roots[r], v2 = RC_M(v, v);
    const double num = RC_A(RC_S(RC_M(pm1, v2), RC_M(RC_M(RC_M(2.0, p), cb), v)), pp1);
    const double den = RC_M(2.0, RC_S(cg, RC_M(v, ca)));
    const double den1 = RC_S(RC_A(1.0, v2), RC_M(RC_M(2.0, v), cb));
    if (den == 0.0 || !(den1 > 0.0)) continue;
    const double u = RC_D(num, den);
    if (!(u > 0.0) || !(v > 0.0)) continue;
    const double s1 = __dsqrt_rn(RC_D(b2, den1)), s2 = RC_M(u, s1), s3 = RC_M(v, s1);
    double P1[3], f1[3], f2[3];
#pragma unroll
    for (int e = 0; e < 3; ++e) {
      P1[e] = RC_M(s1, j[e]);
      f1[e] = RC_S(RC_M(s2, j[3 + e]), P1[e]);
      f2[e] = RC_S(RC_M(s3, j[6 + e]), P1[e]);
    }
    double cc[3], g1[3], g2[3], g3[3];
    rc_cross3(f1, f2, cc);
    const double m1 = __dsqrt_rn(rc_dot3(f1, f1)), mc = __dsqrt_rn(rc_dot3(cc, cc));
#pragma unroll
    for (int e = 0; e < 3; ++e) {
      g1[e] = RC_D(f1[e], m1);
      g3[e] = RC_D(cc[e], mc);
    }
    rc_cross3(g3, g1, g2);
    double* R = Rs + 9 * ns;
    double* t = ts + 3 * ns;
    bool fin = true;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        R[3 * i + k] = RC_A(RC_A(RC_M(g1[i], e1[k]), RC_M(g2[i], e2[k])), RC_M(g3[i], e3[k]));
        fin &= isfinite(R[3 * i + k]);
      }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      t[i] = RC_S(P1[i], RC_A(RC_A(RC_M(R[3 * i], X[0]), RC_M(R[3 * i + 1], X[1])), RC_M(R[3 * i + 2], X[2])));
      fin &= isfinite(t[i]);
    }
    if (fin) jr[ns++] = r;
  }
  return ns;
}

// Hypothesis k of group g: its poses (shifted frame) with root indices.  -> solution count.
__device__ __forceinline__ int ap_hypothesis(const ApStage& st, const ApGroup& sg, unsigned long long seed, int g, int k,
                                             double* Rs, double* ts, int* jr) {
  int idx[AP_SAMPLE];
  if (!hg_draw<AP_SAMPLE>(seed, g, k, sg.np, idx)) return 0;
  double j[9], X[9];
  for (int s = 0; s < AP_SAMPLE; ++s) {
    const float2 kk = st.k[idx[s]];
    const double qx = RC_D(RC_S(kk.x, sg.cx), sg.fx), qy = RC_D(RC_S(kk.y, sg.cy), sg.fy);
    const double nb = __dsqrt_rn(RC_A(RC_A(RC_M(qx, qx), RC_M(qy, qy)), 1.0));
    j[3 * s] = RC_D(qx, nb);
    j[3 * s + 1] = RC_D(qy, nb);
    j[3 * s + 2] = RC_D(1.0, nb);
#pragma unroll
    for (int e = 0; e < 3; ++e) X[3 * s + e] = st.X[3 * idx[s] + e];
  }
  return ap_p3p(j, X, Rs, ts, jr);
}

// ---- line hypotheses: P2P1L, P1P2L and P3L through one pair of bilinear trigonometric equations
// The rotation between a world triad H and a camera triad G (rows) is R' = Rz(a) Rx(b), R = G^T R' H.  Each solver
// gives two equations [cos a, sin a, 1] M_i [cos b, sin b, 1]^T = 0; tau = tan(b / 2) makes row r of M_i the
// quadratic q_ir = M_i[r][0] (1 - tau^2) + 2 M_i[r][1] tau + M_i[r][2] (1 + tau^2), A_i, B_i, C_i = rows 0, 1, 2, and
// with D = A1 B2 - A2 B1, X = B1 C2 - B2 C1, Y = A2 C1 - A1 C2 (cos a, sin a) = (X, Y) / D on X^2 + Y^2 - D^2 = 0.
// b = pi (tau = inf) is not found.

// Point and line rows of a sample of solver s.
__host__ __device__ constexpr int ap_line_np(int s) { return 2 - s; }
__host__ __device__ constexpr int ap_line_nl(int s) { return s + 1; }

// The coefficients of n' . Rz(a) Rx(b) E' in M (row-major; rows cos a, sin a, 1; columns cos b, sin b, 1).
__device__ __forceinline__ void ap_trig_terms(const double* n, const double* E, double* M) {
  M[0] = RC_M(n[1], E[1]);
  M[1] = -RC_M(n[1], E[2]);
  M[2] = RC_M(n[0], E[0]);
  M[3] = -RC_M(n[0], E[1]);
  M[4] = RC_M(n[0], E[2]);
  M[5] = RC_M(n[1], E[0]);
  M[6] = RC_M(n[2], E[2]);
  M[7] = RC_M(n[2], E[1]);
  M[8] = 0.0;
}

// c = a b (ascending coefficients; a has na, b nb), each c[k] summed over a's index ascending from 0.
__device__ __forceinline__ void ap_pmul(const double* a, int na, const double* b, int nb, double* c) {
  for (int k = 0; k < na + nb - 1; ++k) {
    double acc = 0.0;
    for (int i = 0; i < na; ++i)
      if (k - i >= 0 && k - i < nb) acc = RC_A(acc, RC_M(a[i], b[k - i]));
    c[k] = acc;
  }
}

// The quartics D, X, Y [5] and p = (X^2 + Y^2) - D^2 [11] (degree 8, zero-padded) of M1, M2 [9].
__device__ __noinline__ void ap_trig_poly(const double* M1, const double* M2, double* D, double* X, double* Y,
                                          double* p) {
  double q[2][3][3];   // q[i][r]: row r of M_i as a quadratic in tau
  for (int i = 0; i < 2; ++i) {
    const double* M = i ? M2 : M1;
    for (int r = 0; r < 3; ++r) {
      q[i][r][0] = RC_A(M[3 * r], M[3 * r + 2]);
      q[i][r][1] = RC_M(2.0, M[3 * r + 1]);
      q[i][r][2] = RC_S(M[3 * r + 2], M[3 * r]);
    }
  }
  double u[5], v[5];
  ap_pmul(q[0][0], 3, q[1][1], 3, u);
  ap_pmul(q[1][0], 3, q[0][1], 3, v);
  for (int k = 0; k < 5; ++k) D[k] = RC_S(u[k], v[k]);
  ap_pmul(q[0][1], 3, q[1][2], 3, u);
  ap_pmul(q[1][1], 3, q[0][2], 3, v);
  for (int k = 0; k < 5; ++k) X[k] = RC_S(u[k], v[k]);
  ap_pmul(q[1][0], 3, q[0][2], 3, u);
  ap_pmul(q[0][0], 3, q[1][2], 3, v);
  for (int k = 0; k < 5; ++k) Y[k] = RC_S(u[k], v[k]);
  double xx[9], yy[9], dd[9];
  ap_pmul(X, 5, X, 5, xx);
  ap_pmul(Y, 5, Y, 5, yy);
  ap_pmul(D, 5, D, 5, dd);
  for (int k = 0; k < 9; ++k) p[k] = RC_S(RC_A(xx[k], yy[k]), dd[k]);
  p[9] = p[10] = 0.0;
}

__device__ __forceinline__ double ap_horner4(const double* c, double x) {
  double v = c[4];
  for (int k = 3; k >= 0; --k) v = RC_A(RC_M(v, x), c[k]);
  return v;
}

// (cos a, sin a, cos b, sin b) at the root tau of p.  -> false where D(tau) == 0.
__device__ __forceinline__ bool ap_trig_angles(const double* D, const double* X, const double* Y, double tau,
                                               double* cs) {
  const double d = ap_horner4(D, tau);
  if (d == 0.0) return false;
  const double c = RC_D(ap_horner4(X, tau), d), s = RC_D(ap_horner4(Y, tau), d);
  const double nr = __dsqrt_rn(RC_A(RC_M(c, c), RC_M(s, s)));
  const double t2 = RC_M(tau, tau), den = RC_A(1.0, t2);
  cs[0] = RC_D(c, nr);
  cs[1] = RC_D(s, nr);
  cs[2] = RC_D(RC_S(1.0, t2), den);
  cs[3] = RC_D(RC_M(2.0, tau), den);
  return true;
}

// T rows (f, u, v): the unit f, then u = f x e / |f x e| for the coordinate axis e least aligned with f (the first of
// the smallest |f_k|), v = f x u; a right-handed orthonormal frame.
__device__ __forceinline__ void ap_triad(const double* f, double* T) {
  int k = 0;
  if (fabs(f[1]) < fabs(f[k])) k = 1;
  if (fabs(f[2]) < fabs(f[k])) k = 2;
  double e[3] = {0.0, 0.0, 0.0}, c[3];
  e[k] = 1.0;
  rc_cross3(f, e, c);
  const double nc = __dsqrt_rn(rc_dot3(c, c));
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    T[i] = f[i];
    T[3 + i] = RC_D(c[i], nc);
  }
  rc_cross3(T, T + 3, T + 6);
}

// The unit vector of v.  -> |v|.
__device__ __forceinline__ double ap_unit(const double* v, double* u) {
  const double n = __dsqrt_rn(rc_dot3(v, v));
#pragma unroll
  for (int i = 0; i < 3; ++i) u[i] = RC_D(v[i], n);
  return n;
}

__device__ __forceinline__ void ap_sub3(const double* a, const double* b, double* c) {
#pragma unroll
  for (int i = 0; i < 3; ++i) c[i] = RC_S(a[i], b[i]);
}

// Line solver s on unit bearings j [ap_line_np(s)][3] and world points X (same shape) of the sample's points, camera-
// ray line normals n [ap_line_nl(s)][3] and world end points E [ap_line_nl(s)][2][3] of its lines (DESIGN.md
// "Absolute pose"): up to 8 poses (Rs[9 i] row-major, ts[3 i]) with their root indices jr[i].  -> solution count.
__device__ __noinline__ int ap_line_pose(int s, const double* j, const double* X, const double* n, const double* E,
                                         double* Rs, double* ts, int* jr) {
  double G[9], H[9], M[18], w[3], c[3], aux[3];
  if (s == 0) {   // P2P1L: h1 along X2 - X1; g1 = j1, g3 = j1 x j2 / |j1 x j2|
    ap_sub3(X + 3, X, w);
    ap_unit(w, c);
    const double L = __dsqrt_rn(rc_dot3(w, w));
    ap_triad(c, H);
    rc_cross3(j, j + 3, c);
    const double sg = __dsqrt_rn(rc_dot3(c, c));
    if (!(sg > AP_BEARING_EPS)) return 0;
    const double gs = RC_D(rc_dot3(j, j + 3), sg);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      G[i] = j[i];
      G[6 + i] = RC_D(c[i], sg);
    }
    rc_cross3(G + 6, G, G + 3);
    double np_[3], Ep[3];
    rc_mv3(G, n, np_);
    const double Ln = RC_M(L, np_[0]);
    for (int e = 0; e < 2; ++e) {
      ap_sub3(E + 3 * e, X, w);
      rc_mv3(H, w, Ep);
      double* Me = M + 9 * e;
      ap_trig_terms(np_, Ep, Me);
      Me[2] = RC_S(Me[2], Ln);
      Me[5] = RC_A(Me[5], RC_M(Ln, gs));
    }
    aux[0] = L;
    aux[1] = gs;
    aux[2] = sg;
  } else {        // P1P2L, P3L: g3 along n1, h1 along line 1's direction
    ap_unit(n, c);
    double T[9];   // (g3, g1, g2)
    ap_triad(c, T);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      G[i] = T[3 + i];
      G[3 + i] = T[6 + i];
      G[6 + i] = T[i];
    }
    ap_sub3(E + 3, E, w);
    ap_unit(w, c);
    ap_triad(c, H);
    double np_[3], Ep[3];
    if (s == 1) {   // P1P2L: line 2's direction; line 2's end point a with s1 from line 1's end point a
      const double m1 = rc_dot3(G + 6, j), m2 = rc_dot3(n + 3, j);
      if (!(fabs(m1) > AP_POINT_LINE_EPS)) return 0;
      rc_mv3(G, n + 3, np_);
      ap_sub3(E + 9, E + 6, w);
      rc_mv3(H, w, Ep);
      ap_trig_terms(np_, Ep, M);
#pragma unroll
      for (int i = 0; i < 3; ++i) np_[i] = RC_M(m1, np_[i]);
      ap_sub3(E + 6, X, w);
      rc_mv3(H, w, Ep);
      ap_trig_terms(np_, Ep, M + 9);
      ap_sub3(E, X, w);
      rc_mv3(H, w, Ep);
      M[15] = RC_S(M[15], RC_M(m2, Ep[2]));
      M[16] = RC_S(M[16], RC_M(m2, Ep[1]));
      aux[0] = m1;
      aux[1] = Ep[1];
      aux[2] = Ep[2];
    } else {        // P3L: the directions of lines 2 and 3
      double cr[3];
      rc_cross3(n + 3, n + 6, cr);
      const double det = rc_dot3(n, cr);
      const double n1 = __dsqrt_rn(rc_dot3(n, n)), n2 = __dsqrt_rn(rc_dot3(n + 3, n + 3)),
                   n3 = __dsqrt_rn(rc_dot3(n + 6, n + 6));
      if (!(fabs(det) > RC_M(RC_M(RC_M(AP_CONCURRENT_EPS, n1), n2), n3))) return 0;
      for (int e = 0; e < 2; ++e) {
        rc_mv3(G, n + 3 * (e + 1), np_);
        ap_sub3(E + 6 * (e + 1) + 3, E + 6 * (e + 1), w);
        rc_mv3(H, w, Ep);
        ap_trig_terms(np_, Ep, M + 9 * e);
      }
    }
  }
  double D[5], Xq[5], Yq[5], p[11], roots[10];
  ap_trig_poly(M, M + 9, D, Xq, Yq, p);
  const int nr = ess_roots(p, roots);
  int ns = 0;
  for (int r = 0; r < nr && r < AP_LINE_MAX_SOLUTIONS; ++r) {
    double cs[4];
    if (!ap_trig_angles(D, Xq, Yq, roots[r], cs)) continue;
    const double ca = cs[0], sa = cs[1], cb = cs[2], sb = cs[3];
    double s1 = 0.0;
    if (s == 0) {
      const double s2 = RC_D(RC_M(aux[0], sa), aux[2]);
      s1 = RC_M(aux[0], RC_S(RC_M(aux[1], sa), ca));
      if (!(s1 > 0.0) || !(s2 > 0.0)) continue;
    } else if (s == 1) {
      s1 = RC_D(-RC_A(RC_M(sb, aux[1]), RC_M(cb, aux[2])), aux[0]);
      if (!(s1 > 0.0)) continue;
    }
    const double Rp[9] = {ca, -RC_M(sa, cb), RC_M(sa, sb), sa, RC_M(ca, cb), -RC_M(ca, sb), 0.0, sb, cb};
    double W[9];
    double* R = Rs + 9 * ns;
    double* t = ts + 3 * ns;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int k = 0; k < 3; ++k)
        W[3 * i + k] = RC_A(RC_A(RC_M(Rp[3 * i], H[k]), RC_M(Rp[3 * i + 1], H[3 + k])), RC_M(Rp[3 * i + 2], H[6 + k]));
    bool fin = true;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        R[3 * i + k] = RC_A(RC_A(RC_M(G[i], W[k]), RC_M(G[3 + i], W[3 + k])), RC_M(G[6 + i], W[6 + k]));
        fin &= isfinite(R[3 * i + k]);
      }
    if (s < 2) {   // t = s1 j1 - R X1
#pragma unroll
      for (int i = 0; i < 3; ++i) t[i] = RC_S(RC_M(s1, j[i]), rc_dot3(R + 3 * i, X));
    } else {       // n_i . t = -n_i . R A_i by Gaussian elimination with partial pivoting (first largest |pivot|)
      double A[3][4];
      for (int i = 0; i < 3; ++i) {
        double RA[3];
        rc_mv3(R, E + 6 * i, RA);
        for (int k = 0; k < 3; ++k) A[i][k] = n[3 * i + k];
        A[i][3] = -rc_dot3(n + 3 * i, RA);
      }
      for (int cc = 0; cc < 3; ++cc) {
        int piv = cc;
        double best = fabs(A[cc][cc]);
        for (int q = cc + 1; q < 3; ++q)
          if (fabs(A[q][cc]) > best) { best = fabs(A[q][cc]); piv = q; }
        if (piv != cc)
          for (int k = cc; k < 4; ++k) { const double tmp = A[cc][k]; A[cc][k] = A[piv][k]; A[piv][k] = tmp; }
        for (int q = cc + 1; q < 3; ++q) {
          const double f = RC_D(A[q][cc], A[cc][cc]);
          for (int k = cc + 1; k < 4; ++k) A[q][k] = RC_S(A[q][k], RC_M(f, A[cc][k]));
        }
      }
      for (int i = 2; i >= 0; --i) {
        double acc = A[i][3];
        for (int k = i + 1; k < 3; ++k) acc = RC_S(acc, RC_M(A[i][k], t[k]));
        t[i] = RC_D(acc, A[i][i]);
      }
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) fin &= isfinite(t[i]);
    if (fin) jr[ns++] = r;
  }
  return ns;
}

__device__ __forceinline__ bool ap_line_rows_ok(int s, int np, int nl) {
  return np >= ap_line_np(s) && nl >= ap_line_nl(s);
}

// Line hypothesis k of solver s of group g: its poses (shifted frame) with root indices.  -> solution count.  The
// point rows are drawn with seed + 2 s + 1, the line rows with seed + 2 s + 2.
__device__ __forceinline__ int ap_line_hypothesis(const ApStage& st, const ApGroup& sg, unsigned long long seed, int g,
                                                  int s, int k, double* Rs, double* ts, int* jr) {
  if (!ap_line_rows_ok(s, sg.np, sg.nl)) return 0;
  int ip[2], il[3];
  bool ok = true;
  if (s == 0) ok = hg_draw<2>(seed + 1, g, k, sg.np, ip) && hg_draw<1>(seed + 2, g, k, sg.nl, il);
  else if (s == 1) ok = hg_draw<1>(seed + 3, g, k, sg.np, ip) && hg_draw<2>(seed + 4, g, k, sg.nl, il);
  else ok = hg_draw<3>(seed + 6, g, k, sg.nl, il);
  if (!ok) return 0;
  double j[6], X[6], n[9], E[18];
  const int np = ap_line_np(s), nl = ap_line_nl(s);
  for (int q = 0; q < np; ++q) {
    const float2 kk = st.k[ip[q]];
    const double qx = RC_D(RC_S(kk.x, sg.cx), sg.fx), qy = RC_D(RC_S(kk.y, sg.cy), sg.fy);
    const double nb = __dsqrt_rn(RC_A(RC_A(RC_M(qx, qx), RC_M(qy, qy)), 1.0));
    j[3 * q] = RC_D(qx, nb);
    j[3 * q + 1] = RC_D(qy, nb);
    j[3 * q + 2] = RC_D(1.0, nb);
    for (int e = 0; e < 3; ++e) X[3 * q + e] = st.X[3 * ip[q] + e];
  }
  const double cam[4] = {sg.fx, sg.fy, sg.cx, sg.cy};
  for (int q = 0; q < nl; ++q) {
    rc_line_normal(cam, st.s0[il[q]], n + 3 * q);
    for (int e = 0; e < 6; ++e) E[6 * q + e] = st.E[6 * il[q] + e];
  }
  return ap_line_pose(s, j, X, n, E, Rs, ts, jr);
}

// Camera coordinates of world point X under pose C (R row-major, then t): Y = R X, P = Y + t.
__device__ __forceinline__ void ap_cam(const double* C, const double* X, double* Y, double* P) {
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    Y[i] = RC_A(RC_A(RC_M(C[3 * i], X[0]), RC_M(C[3 * i + 1], X[1])), RC_M(C[3 * i + 2], X[2]));
    P[i] = RC_A(Y[i], C[9 + i]);
  }
}

// Staged row d (points, then lines) is an inlier of pose C.
__device__ __forceinline__ bool ap_inlier(const ApStage& st, const ApGroup& sg, const double* C, double t2, int d) {
  double Y[3], P[3];
  if (d < sg.np) {
    ap_cam(C, st.X + 3 * d, Y, P);
    const float2 k = st.k[d];
    const double ex = RC_S(RC_M(sg.fx, P[0]), RC_M(RC_S(k.x, sg.cx), P[2]));
    const double ey = RC_S(RC_M(sg.fy, P[1]), RC_M(RC_S(k.y, sg.cy), P[2]));
    return P[2] > 0.0 && RC_A(RC_M(ex, ex), RC_M(ey, ey)) < RC_M(t2, RC_M(P[2], P[2]));
  }
  const int i = d - sg.np;
  double n[3];
  const double cam[4] = {sg.fx, sg.fy, sg.cx, sg.cy};
  rc_line_normal(cam, st.s0[i], n);
  bool ok = true;
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    ap_cam(C, st.E + 6 * i + 3 * e, Y, P);
    const double dd = RC_A(RC_A(RC_M(n[0], P[0]), RC_M(n[1], P[1])), RC_M(n[2], P[2]));
    ok &= P[2] > 0.0 && RC_M(dd, dd) < RC_M(t2, RC_M(P[2], P[2]));
  }
  return ok;
}

__global__ void __launch_bounds__(AP_THREADS) abspose_hyp_kernel(AbsPoseArgs a) {
  extern __shared__ __align__(16) unsigned char ap_smem[];
  __shared__ ApGroup sg;
  __shared__ int warp_cnt[AP_THREADS / 32];
  __shared__ double red[AP_THREADS / 32 * 6];
  __shared__ unsigned long long wbest[AP_THREADS / 32];
  pdl_launch_dependents();
  pdl_wait();
  const int g = blockIdx.x;
  const ApStage st = ap_stage_ptrs(ap_smem, a.rows_p, a.rows_l);
  ap_stage_group<AP_THREADS>(a, g, st, sg, warp_cnt, red);
  if (sg.np < AP_SAMPLE) return;
  const int n = sg.np + sg.nl;
  const int k = blockIdx.y * AP_THREADS + threadIdx.x;
  unsigned long long key = 0;
  if (k < a.n_hyp) {
    double Rs[9 * AP_MAX_SOLUTIONS], ts[3 * AP_MAX_SOLUTIONS];
    int jr[AP_MAX_SOLUTIONS];
    const int ns = ap_hypothesis(st, sg, a.seed, g, k, Rs, ts, jr);
    for (int s = 0; s < ns; ++s) {
      double C[12];
#pragma unroll
      for (int i = 0; i < 9; ++i) C[i] = Rs[9 * s + i];
#pragma unroll
      for (int i = 0; i < 3; ++i) C[9 + i] = ts[3 * s + i];
      unsigned cnt = 0;
      for (int d = 0; d < n; ++d) cnt += ap_inlier(st, sg, C, a.thresh2, d);
      const unsigned long long kk =
          ((unsigned long long)cnt << 32) | (unsigned long long)(~(unsigned)(AP_MAX_SOLUTIONS * k + jr[s]));
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
    for (int i = 1; i < AP_THREADS / 32; ++i) key = wbest[i] > key ? wbest[i] : key;
    if (key) atomicMax(a.key + g, key);
  }
}

// Thread h = s n_line_hyp + k runs hypothesis k of line solver s, index 4 n_hyp + 8 h + j.
__global__ void __launch_bounds__(AP_THREADS) abspose_line_hyp_kernel(AbsPoseArgs a) {
  extern __shared__ __align__(16) unsigned char ap_smem[];
  __shared__ ApGroup sg;
  __shared__ int warp_cnt[AP_THREADS / 32];
  __shared__ double red[AP_THREADS / 32 * 6];
  __shared__ unsigned long long wbest[AP_THREADS / 32];
  pdl_launch_dependents();
  pdl_wait();
  const int g = blockIdx.x;
  const ApStage st = ap_stage_ptrs(ap_smem, a.rows_p, a.rows_l);
  ap_stage_group<AP_THREADS>(a, g, st, sg, warp_cnt, red);
  if (sg.nl < 1) return;
  const int n = sg.np + sg.nl;
  const int h = blockIdx.y * AP_THREADS + threadIdx.x;
  unsigned long long key = 0;
  if (h < AP_LINE_SOLVERS * a.n_line_hyp) {
    double Rs[9 * AP_LINE_MAX_SOLUTIONS], ts[3 * AP_LINE_MAX_SOLUTIONS];
    int jr[AP_LINE_MAX_SOLUTIONS];
    const int ns = ap_line_hypothesis(st, sg, a.seed, g, h / a.n_line_hyp, h % a.n_line_hyp, Rs, ts, jr);
    const unsigned base = AP_MAX_SOLUTIONS * (unsigned)a.n_hyp + AP_LINE_MAX_SOLUTIONS * (unsigned)h;
    for (int s = 0; s < ns; ++s) {
      double C[12];
#pragma unroll
      for (int i = 0; i < 9; ++i) C[i] = Rs[9 * s + i];
#pragma unroll
      for (int i = 0; i < 3; ++i) C[9 + i] = ts[3 * s + i];
      unsigned cnt = 0;
      for (int d = 0; d < n; ++d) cnt += ap_inlier(st, sg, C, a.thresh2, d);
      const unsigned long long kk = ((unsigned long long)cnt << 32) | (unsigned long long)(~(base + jr[s]));
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
    for (int i = 1; i < AP_THREADS / 32; ++i) key = wbest[i] > key ? wbest[i] : key;
    if (key) atomicMax(a.key + g, key);
  }
}

// The winner's pose C (shifted frame) from its index kj: hypothesis kj / 4, root kj % 4 of P3P below 4 n_hyp, else
// line hypothesis (kj - 4 n_hyp) / 8, root (kj - 4 n_hyp) % 8.  -> false when that solution does not exist.
__device__ __noinline__ bool ap_winner_pose(const AbsPoseArgs& a, const ApStage& st, const ApGroup& sg, int g,
                                            unsigned kj, double* C) {
  double Rs[9 * AP_LINE_MAX_SOLUTIONS], ts[3 * AP_LINE_MAX_SOLUTIONS];
  int jr[AP_LINE_MAX_SOLUTIONS], ns = 0, j;
  const unsigned p3p = AP_MAX_SOLUTIONS * (unsigned)a.n_hyp;
  if (kj < p3p) {
    j = (int)(kj % AP_MAX_SOLUTIONS);
    if (sg.np >= AP_SAMPLE) ns = ap_hypothesis(st, sg, a.seed, g, (int)(kj / AP_MAX_SOLUTIONS), Rs, ts, jr);
  } else {
    const int h = (int)((kj - p3p) / AP_LINE_MAX_SOLUTIONS);
    j = (int)((kj - p3p) % AP_LINE_MAX_SOLUTIONS);
    if (h < AP_LINE_SOLVERS * a.n_line_hyp)
      ns = ap_line_hypothesis(st, sg, a.seed, g, h / a.n_line_hyp, h % a.n_line_hyp, Rs, ts, jr);
  }
  for (int s = 0; s < ns; ++s)
    if (jr[s] == j) {
      for (int i = 0; i < 9; ++i) C[i] = Rs[9 * s + i];
      for (int i = 0; i < 3; ++i) C[9 + i] = ts[3 * s + i];
      return true;
    }
  return false;
}

// Block-wide inlier counts (points, lines) of pose C (shared), returned to every thread.
template <int NT>
__device__ __forceinline__ int2 ap_count(const ApStage& st, const ApGroup& sg, const double* sC, double t2, int2* red) {
  double C[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) C[i] = sC[i];
  int cp = 0, cl = 0;
  for (int d = threadIdx.x; d < sg.np + sg.nl; d += NT) {
    const bool in = ap_inlier(st, sg, C, t2, d);
    if (d < sg.np) cp += in; else cl += in;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    cp += __shfl_xor_sync(0xffffffffu, cp, o);
    cl += __shfl_xor_sync(0xffffffffu, cl, o);
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = make_int2(cp, cl);
  __syncthreads();
  int2 t = make_int2(0, 0);
  for (int i = 0; i < NT / 32; ++i) { t.x += red[i].x; t.y += red[i].y; }
  return t;
}

// The two residual components of staged row d at pose C (a point's pixel x / y residuals, a line's two signed end-point
// distances in pixels) and, with JAC, their Jacobian rows in (w, dt) of R <- cay(w) R, t <- t + dt at w = 0: for a
// component with gradient g in the camera point, (2 (R X) x g, g).
template <bool JAC>
__device__ __forceinline__ void ap_residual(const ApStage& st, const ApGroup& sg, const double* C, int d, double* r,
                                            double (*J)[6]) {
  double Y[3], P[3], g[3];
  auto jac = [&](double* Jr) {
    double c[3];
    rc_cross3(Y, g, c);
#pragma unroll
    for (int e = 0; e < 3; ++e) {
      Jr[e] = RC_M(2.0, c[e]);
      Jr[3 + e] = g[e];
    }
  };
  if (d < sg.np) {
    ap_cam(C, st.X + 3 * d, Y, P);
    const float2 k = st.k[d];
    const double iz = __drcp_rn(P[2]);
    const double xn = RC_M(P[0], iz), yn = RC_M(P[1], iz);
    r[0] = RC_S(RC_M(sg.fx, xn), RC_S(k.x, sg.cx));
    r[1] = RC_S(RC_M(sg.fy, yn), RC_S(k.y, sg.cy));
    if (JAC) {
      g[0] = RC_M(sg.fx, iz); g[1] = 0.0; g[2] = -RC_M(RC_M(sg.fx, xn), iz);
      jac(J[0]);
      g[0] = 0.0; g[1] = RC_M(sg.fy, iz); g[2] = -RC_M(RC_M(sg.fy, yn), iz);
      jac(J[1]);
    }
    return;
  }
  const int i = d - sg.np;
  double n[3];
  const double cam[4] = {sg.fx, sg.fy, sg.cx, sg.cy};
  rc_line_normal(cam, st.s0[i], n);
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    ap_cam(C, st.E + 6 * i + 3 * e, Y, P);
    const double iz = __drcp_rn(P[2]);
    r[e] = RC_M(RC_A(RC_A(RC_M(n[0], P[0]), RC_M(n[1], P[1])), RC_M(n[2], P[2])), iz);
    if (JAC) {
      g[0] = RC_M(n[0], iz); g[1] = RC_M(n[1], iz); g[2] = -RC_M(RC_S(r[e], n[2]), iz);
      jac(J[e]);
    }
  }
}

// The refit's sums over the rows that are inliers of pose H, evaluated at pose C: with FULL the AP_TERMS terms (J^T J
// upper triangle row-major, J^T r, r^T r), else r^T r alone.  Thread t sums rows t, t + NT, ... in order, each warp
// folds its lanes with the xor butterfly, then thread 0 adds the warps in order into out.  Ends with __syncthreads.
template <int NT, bool FULL>
__device__ void ap_sums(const ApStage& st, const ApGroup& sg, const double* sH, const double* sC, double t2,
                        double* red, double* out) {
  constexpr int M = FULL ? AP_TERMS : 1;
  double H[12], C[12], acc[M];
#pragma unroll
  for (int i = 0; i < 12; ++i) {
    H[i] = sH[i];
    C[i] = sC[i];
  }
#pragma unroll
  for (int e = 0; e < M; ++e) acc[e] = 0.0;
  for (int d = threadIdx.x; d < sg.np + sg.nl; d += NT) {
    if (!ap_inlier(st, sg, H, t2, d)) continue;
    double r[2], J[2][6];
    ap_residual<FULL>(st, sg, C, d, r, J);
    if (FULL) {
      int e = 0;
#pragma unroll
      for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int k = i; k < 6; ++k, ++e)
          acc[e] = RC_A(acc[e], RC_A(RC_M(J[0][i], J[0][k]), RC_M(J[1][i], J[1][k])));
#pragma unroll
      for (int i = 0; i < 6; ++i) acc[21 + i] = RC_A(acc[21 + i], RC_A(RC_M(J[0][i], r[0]), RC_M(J[1][i], r[1])));
    }
    acc[M - 1] = RC_A(acc[M - 1], RC_A(RC_M(r[0], r[0]), RC_M(r[1], r[1])));
  }
#pragma unroll
  for (int e = 0; e < M; ++e)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[e] = RC_A(acc[e], __shfl_xor_sync(0xffffffffu, acc[e], o));
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int e = 0; e < M; ++e) red[(threadIdx.x >> 5) * M + e] = acc[e];
  __syncthreads();
  if (threadIdx.x == 0)
    for (int e = 0; e < M; ++e) {
      double v = 0.0;
      for (int w = 0; w < NT / 32; ++w) v = RC_A(v, red[w * M + e]);
      out[e] = v;
    }
  __syncthreads();
}

// One damped step from the sums S at pose C: (A + lam diag A) x = -J^T r by Gaussian elimination with partial pivoting
// (first largest |pivot|), then R <- cay(w) R, t <- t + dt into Cn.  -> false for a zero pivot or a non-finite result.
__device__ __noinline__ bool ap_lm_step(const double* S, double lam, const double* C, double* Cn) {
  double A[6][7];
  int e = 0;
  for (int i = 0; i < 6; ++i)
    for (int k = i; k < 6; ++k, ++e) A[i][k] = A[k][i] = S[e];
  for (int i = 0; i < 6; ++i) {
    A[i][i] = RC_A(A[i][i], RC_M(lam, A[i][i]));
    A[i][6] = -S[21 + i];
  }
  for (int c = 0; c < 6; ++c) {
    int piv = c;
    double best = fabs(A[c][c]);
    for (int r = c + 1; r < 6; ++r)
      if (fabs(A[r][c]) > best) { best = fabs(A[r][c]); piv = r; }
    if (!(best > 0.0)) return false;
    if (piv != c)
      for (int k = c; k < 7; ++k) { const double t = A[c][k]; A[c][k] = A[piv][k]; A[piv][k] = t; }
    for (int r = c + 1; r < 6; ++r) {
      const double f = RC_D(A[r][c], A[c][c]);
      for (int k = c + 1; k < 7; ++k) A[r][k] = RC_S(A[r][k], RC_M(f, A[c][k]));
    }
  }
  double x[6];
  for (int i = 5; i >= 0; --i) {
    double acc = A[i][6];
    for (int k = i + 1; k < 6; ++k) acc = RC_S(acc, RC_M(A[i][k], x[k]));
    x[i] = RC_D(acc, A[i][i]);
    if (!isfinite(x[i])) return false;
  }
  double Q[9];
  rc_cayley(x, Q);
  bool fin = true;
  for (int i = 0; i < 3; ++i) {
    for (int k = 0; k < 3; ++k) {
      Cn[3 * i + k] = RC_A(RC_A(RC_M(Q[3 * i], C[k]), RC_M(Q[3 * i + 1], C[3 + k])), RC_M(Q[3 * i + 2], C[6 + k]));
      fin &= isfinite(Cn[3 * i + k]);
    }
    Cn[9 + i] = RC_A(C[9 + i], x[3 + i]);
    fin &= isfinite(Cn[9 + i]);
  }
  return fin;
}

__global__ void __launch_bounds__(AP_FIT_THREADS) abspose_fit_kernel(AbsPoseArgs a) {
  constexpr int NT = AP_FIT_THREADS, NW = NT / 32;
  extern __shared__ __align__(16) unsigned char ap_smem[];
  __shared__ ApGroup sg;
  __shared__ int warp_cnt[NW];
  __shared__ double red[NW * AP_TERMS];
  __shared__ int2 red2[NW];
  __shared__ double sC[3][12];     // the hypothesis, the refit's current pose, its candidate
  __shared__ double sS[AP_TERMS];  // sums at the current pose
  __shared__ double s_cost;        // r^T r at the candidate
  __shared__ int s_ok[3];          // valid, candidate usable, candidate accepted
  pdl_launch_dependents();
  pdl_wait();
  const int g = blockIdx.x;
  const ApStage st = ap_stage_ptrs(ap_smem, a.rows_p, a.rows_l);
  ap_stage_group<NT>(a, g, st, sg, warp_cnt, red);
  const unsigned long long key = a.key[g];
  const unsigned kj = ~(unsigned)(key & 0xffffffffull);
  if (threadIdx.x == 0) {
    s_ok[0] = key != 0 && ap_winner_pose(a, st, sg, g, kj, sC[0]);
    if (s_ok[0])
      for (int i = 0; i < 12; ++i) sC[1][i] = sC[0][i];
  }
  __syncthreads();
  const bool valid = s_ok[0];
  int kept = 0;
  if (valid) {
    const int2 ch = ap_count<NT>(st, sg, sC[0], a.thresh2, red2);
    if (ch.x + ch.y >= AP_MIN_REFIT) {
      ap_sums<NT, true>(st, sg, sC[0], sC[1], a.thresh2, red, sS);
      double lam = AP_LM_LAMBDA0;   // thread 0's
      for (int it = 0; it < AP_LM_ITERS; ++it) {
        if (threadIdx.x == 0) s_ok[1] = ap_lm_step(sS, lam, sC[1], sC[2]);
        __syncthreads();
        if (s_ok[1]) ap_sums<NT, false>(st, sg, sC[0], sC[2], a.thresh2, red, &s_cost);
        if (threadIdx.x == 0) {
          s_ok[2] = s_ok[1] && s_cost < sS[AP_TERMS - 1];
          if (s_ok[2]) {
            for (int i = 0; i < 12; ++i) sC[1][i] = sC[2][i];
            lam = RC_M(lam, AP_LM_ACCEPT);
          } else {
            lam = RC_M(lam, AP_LM_REJECT);
          }
        }
        __syncthreads();
        if (s_ok[2]) ap_sums<NT, true>(st, sg, sC[0], sC[1], a.thresh2, red, sS);
      }
      const int2 cr = ap_count<NT>(st, sg, sC[1], a.thresh2, red2);
      kept = cr.x + cr.y >= ch.x + ch.y;
    }
  }
  const double* C = sC[kept];
  // masks aligned with the match rows (0 for rows without a correspondence, unused lines and invalid groups)
  const int pb = a.groups[g], pe = a.groups[g + 1];
  int cp = 0, cl = 0, base = 0;
  for (int p = pb; p < pe; ++p) {
    const int rb = a.cu_p[p], re = a.cu_p[p + 1];
    if (valid) {
      const double* __restrict__ X1 = a.X1 + 3ll * a.x_off1[p];
      const int n1 = a.n_x1[p];
      base += rc_compact_if<NT>(
          a.matches_p, rb, re, warp_cnt,
          [&](int m) {
            return m >= 0 && m < n1 && isfinite(X1[3 * m]) && isfinite(X1[3 * m + 1]) && isfinite(X1[3 * m + 2]);
          },
          [&](int i, int, int ci) {
            const bool in = ci >= 0 && ap_inlier(st, sg, C, a.thresh2, base + ci);
            a.inl_p[rb + i] = in;
            cp += in;
          });
    } else {
      for (int r = rb + threadIdx.x; r < re; r += NT) a.inl_p[r] = 0;
    }
  }
  base = sg.np;
  for (int p = pb; p < pe; ++p) {
    const int rb = a.cu_l[p], re = a.cu_l[p + 1];
    if (valid && a.rows_l) {
      const double* __restrict__ L1 = a.L1 + 6ll * a.l_off1[p];
      const int n1 = a.n_l1[p];
      base += rc_compact_if<NT>(
          a.matches_l, rb, re, warp_cnt,
          [&](int m) {
            bool ok = m >= 0 && m < n1;
            for (int e = 0; ok && e < 6; ++e) ok = isfinite(L1[6 * m + e]);
            return ok;
          },
          [&](int i, int, int ci) {
            const bool in = ci >= 0 && ap_inlier(st, sg, C, a.thresh2, base + ci);
            a.inl_l[rb + i] = in;
            cl += in;
          });
    } else {
      for (int r = rb + threadIdx.x; r < re; r += NT) a.inl_l[r] = 0;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    cp += __shfl_xor_sync(0xffffffffu, cp, o);
    cl += __shfl_xor_sync(0xffffffffu, cl, o);
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red2[threadIdx.x >> 5] = make_int2(cp, cl);
  __syncthreads();
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  if (threadIdx.x < 9) a.R[9ll * g + threadIdx.x] = valid ? C[threadIdx.x] : nan;
  if (threadIdx.x < 3) {
    const int i = threadIdx.x;
    const double rc = RC_A(RC_A(RC_M(C[3 * i], sg.c[0]), RC_M(C[3 * i + 1], sg.c[1])), RC_M(C[3 * i + 2], sg.c[2]));
    a.t[3ll * g + i] = valid ? RC_S(C[9 + i], rc) : nan;
  }
  if (threadIdx.x == 0) {
    int2 t = make_int2(0, 0);
    for (int i = 0; i < NW; ++i) { t.x += red2[i].x; t.y += red2[i].y; }
    a.valid[g] = valid;
    a.refit[g] = valid && kept;
    a.n_inl_p[g] = t.x;
    a.n_inl_l[g] = t.y;
    a.hyp_index[g] = valid ? (int)kj : -1;
    a.hyp_inliers[g] = valid ? (int)(key >> 32) : 0;
  }
}

}  // namespace ltr
