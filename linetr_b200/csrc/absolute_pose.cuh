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
//   winner: most inliers (points and lines), then lowest k, then lowest j (atomicMax of (count << 32) | ~(4 k + j)).
//   refit (at least AP_MIN_REFIT winner inliers): Levenberg-Marquardt over the winner's inliers, R <- cay(w) R,
//   t <- t + dt, J^T J and J^T r summed in a fixed order, the damped 6 x 6 system by Gaussian elimination with partial
//   pivoting, a fixed budget and damping schedule; kept iff its inlier count >= the hypothesis'.
//
// Kernels:
//   abspose_hyp_kernel  grid (group, chunk of AP_THREADS hypotheses): stage the group's rows, one hypothesis per
//                       thread (P3P + up to 4 solutions scored against every staged row), one atomicMax per CTA.
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
  const int k = (int)(kj / AP_MAX_SOLUTIONS), j = (int)(kj % AP_MAX_SOLUTIONS);
  if (threadIdx.x == 0) {
    s_ok[0] = 0;
    if (sg.np >= AP_SAMPLE && key != 0) {
      double Rs[9 * AP_MAX_SOLUTIONS], ts[3 * AP_MAX_SOLUTIONS];
      int jr[AP_MAX_SOLUTIONS];
      const int ns = ap_hypothesis(st, sg, a.seed, g, k, Rs, ts, jr);
      for (int s = 0; s < ns; ++s)
        if (jr[s] == j) {
          for (int i = 0; i < 9; ++i) sC[0][i] = sC[1][i] = Rs[9 * s + i];
          for (int i = 0; i < 3; ++i) sC[0][9 + i] = sC[1][9 + i] = ts[3 * s + i];
          s_ok[0] = 1;
        }
    }
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
