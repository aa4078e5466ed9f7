// Triangulation of posed images' keypoints and key-line end points from their pair matches (ltr_triangulate).
//
// Model (DESIGN.md "Triangulation"; restated in numpy by linetr_b200.triangulation.triangulate_host):
//   image i has intrinsics K_i (zero skew) and the world -> camera pose X_cam = R_i X + t_i, centre C_i = -R_i^T t_i.
//   Every keypoint row and every key-line end point of every image (the anchor a) is lifted along its own ray,
//   X(s) = C_a + s r, r = R_a^T ((x - cx) / fx, (y - cy) / fy, 1), so s is the depth along the optical axis.
//   observations: each pair that contains a gives at most one partner row, in pair order: matches[k] when a is side 0,
//   the lowest side-0 row that matched k when a is side 1 (tri_scatter_kernel builds that index).  In partner camera v,
//   P(s) = A + s B with A = R_v C_a + t_v and B = R_v r, and every residual is (alpha + s beta) / (gamma + s delta)
//   pixels: a point's x / y reprojection errors (fx Px - (u - cx) Pz) / Pz and (fy Py - (w - cy) Pz) / Pz, an end
//   point's signed distance n . P / Pz to the partner segment's line n (unit pixel line in camera-ray form).
//   candidate of partner o: a point's least-squares root of its two numerators, -(ax bx + ay by) / (bx^2 + by^2), an
//   end point's plane intersection -alpha / beta; kept iff depth > 0 and the triangulation angle >= min_angle (point:
//   B . P <= cos(min_angle) |B| |P|, the angle at X between the two rays; end point: beta^2 >= sin^2(min_angle)
//   |n|^2 |B|^2, the angle between the anchor ray and the partner plane; a line needs both end points).
//   support: partner q supports depth s iff its depth Pz > 0 and its residual is <= thresh (a point: the squared
//   reprojection error <= thresh^2, without the division; a line: at both end points).  Winner: the most supporters,
//   ties to the lowest o.  Refit: TRI_GN_ITERS one-dimensional Gauss-Newton steps over the winner's supporters'
//   residuals (a line's end points separately), stopped early when J^T J is not > 0 or the step is not finite; kept
//   iff its depth is > 0 and it has at least as many supporters.  Valid iff 1 + supporters >= min_views: X = C_a + s r
//   and n_views = 1 + supporters, else NaN and 0.  Every operation is explicitly rounded fp64, every sum in a fixed
//   order.
//
// Kernels:
//   tri_scatter_kernel  1D grid over the point and line match rows of every pair: atomicMin of the side-0 row into
//                       the side-1 -> side-0 index (filled with TRI_NONE by cudaMemsetAsync beforehand).
//   tri_kernel          1D grid over TRI_THREADS-row blocks of each image's keypoints, then of its key lines
//                       (block_off): one row per thread; the anchor's partner cameras are staged in shared memory,
//                       and each thread's partner pixels in dynamic shared memory.
#pragma once
#include "common.cuh"
#include "rn_fp64.cuh"

namespace ltr {

constexpr int TRI_THREADS = 128;
constexpr int TRI_SCATTER_THREADS = 256;
constexpr int TRI_MAX_VIEWS = 64;          // LTR_TRI_MAX_VIEWS: pairs per image (the support mask is 64 bits)
constexpr int TRI_GN_ITERS = 5;
constexpr int TRI_NONE = 0x7f7f7f7f;       // an empty slot of the side-1 -> side-0 index (memset byte 0x7f)
constexpr int TRI_CAM = 16;                // staged doubles per partner: fx, fy, cx, cy, R_v (9), A (3)

struct TriArgs {
  const float* kpts; const int* kp_off;      // [*, 2] keypoints of image i from row kp_off[i], [n + 1]
  const float* segs; const int* seg_off;     // [*, 4] key lines (start xy, end xy), [n + 1]
  const double* K; const double* R; const double* t;   // [n, 3, 3], [n, 3, 3], [n, 3]
  const int* pairs;                          // [P, 2]
  const int* matches_p; const int* cu_p;     // pair p's side-0 keypoint rows are [cu_p[p], cu_p[p + 1])
  const int* matches_l; const int* cu_l;
  const int* views; const int* view_off;     // image i's observations [view_off[i], view_off[i + 1]): pair << 1 | side
  const int* block_off;                      // [2n + 1]: blocks of image i's keypoints, then of image i's key lines
  const int* inv_off_p; const int* inv_off_l;   // [P + 1] side-1 -> side-0 index of pair p from inv_*[inv_off_*[p]]
  int* inv_p; int* inv_l;
  int n_images, n_pairs, total_p, total_l;
  double thresh2, cos_min, sin2_min;
  int min_views;
  double* points3d; double* lines3d; int* n_views_p; int* n_views_l;
};

// A point observation's residual terms in partner camera c (TRI_CAM doubles): x numerator ax + s bx, y numerator
// ay + s by, denominator A[2] + s B[2]; B = R_v r.
struct TriPt { double ax, bx, ay, by, B[3]; };

__device__ __forceinline__ TriPt tri_point_terms(const double* c, const double* r, float2 px) {
  TriPt o;
  rc_mv3(c + 4, r, o.B);
  const double* A = c + 13;
  const double dx = RC_S((double)px.x, c[2]), dy = RC_S((double)px.y, c[3]);
  o.ax = RC_S(RC_M(c[0], A[0]), RC_M(dx, A[2]));
  o.bx = RC_S(RC_M(c[0], o.B[0]), RC_M(dx, o.B[2]));
  o.ay = RC_S(RC_M(c[1], A[1]), RC_M(dy, A[2]));
  o.by = RC_S(RC_M(c[1], o.B[1]), RC_M(dy, o.B[2]));
  return o;
}

__device__ __forceinline__ bool tri_point_supports(const TriPt& o, double Az, double s, double t2) {
  const double pz = RC_A(Az, RC_M(s, o.B[2]));
  const double ex = RC_A(o.ax, RC_M(s, o.bx)), ey = RC_A(o.ay, RC_M(s, o.by));
  return pz > 0.0 && RC_A(RC_M(ex, ex), RC_M(ey, ey)) <= RC_M(t2, RC_M(pz, pz));
}

// An end point's residual terms: numerator alpha + s beta, denominator A[2] + s delta.
struct TriEnd { double beta, delta, BB; };

__device__ __forceinline__ TriEnd tri_end_terms(const double* c, const double* n, const double* r) {
  double B[3];
  rc_mv3(c + 4, r, B);
  return TriEnd{rc_dot3(n, B), B[2], rc_dot3(B, B)};
}

__device__ __forceinline__ bool tri_end_supports(double alpha, const TriEnd& e, double Az, double s, double t2) {
  const double pz = RC_A(Az, RC_M(s, e.delta));
  const double v = RC_A(alpha, RC_M(s, e.beta));
  return pz > 0.0 && RC_M(v, v) <= RC_M(t2, RC_M(pz, pz));
}

// One Gauss-Newton term (alpha + s beta) / (gamma + s delta) into J^T J and J^T r.
__device__ __forceinline__ void tri_gn_term(double a, double b, double g, double d, double s, double& jj, double& jr) {
  const double den = RC_A(g, RC_M(s, d));
  const double r = RC_D(RC_A(a, RC_M(s, b)), den);
  const double J = RC_D(RC_S(b, RC_M(r, d)), den);
  jj = RC_A(jj, RC_M(J, J));
  jr = RC_A(jr, RC_M(J, r));
}

__device__ __forceinline__ bool tri_gn_step(double jj, double jr, double& s) {
  if (!(jj > 0.0)) return false;
  const double sn = RC_S(s, RC_D(jr, jj));
  if (!isfinite(sn)) return false;
  s = sn;
  return true;
}

__global__ void __launch_bounds__(TRI_SCATTER_THREADS) tri_scatter_kernel(const TriArgs a) {
  pdl_launch_dependents();
  const long long r = (long long)blockIdx.x * TRI_SCATTER_THREADS + threadIdx.x;
  const bool lines = r >= a.total_p;
  const int row = (int)(lines ? r - a.total_p : r);
  pdl_wait();
  if (r >= (long long)a.total_p + a.total_l) return;
  const int* cu = lines ? a.cu_l : a.cu_p;
  const int* inv_off = lines ? a.inv_off_l : a.inv_off_p;
  const int p = rc_segment(cu, a.n_pairs, row);
  const int m = (lines ? a.matches_l : a.matches_p)[row];
  if (m >= 0 && m < inv_off[p + 1] - inv_off[p]) atomicMin((lines ? a.inv_l : a.inv_p) + inv_off[p] + m, row - cu[p]);
}

__global__ void __launch_bounds__(TRI_THREADS) tri_kernel(const TriArgs a) {
  __shared__ double s_cam[TRI_MAX_VIEWS][TRI_CAM];
  __shared__ int s_obs[TRI_MAX_VIEWS][2];      // partner row source (pair << 1 | side), partner image
  extern __shared__ float4 s_px[];             // [V][TRI_THREADS] each thread's partner pixel / segment
  pdl_launch_dependents();
  const int tid = threadIdx.x;
  const int g = rc_segment(a.block_off, 2 * a.n_images, blockIdx.x);
  const bool lines = g >= a.n_images;
  const int img = lines ? g - a.n_images : g;
  const int* off = lines ? a.seg_off : a.kp_off;
  const int k = (blockIdx.x - a.block_off[g]) * TRI_THREADS + tid, n_rows = off[img + 1] - off[img];
  const int vb = a.view_off[img], V = a.view_off[img + 1] - vb;
  const double* Ra = a.R + 9 * img;
  const double* ta = a.t + 3 * img;
  double C[3];
  rc_centre(Ra, ta, C);
  for (int o = tid; o < V; o += TRI_THREADS) {
    const int code = a.views[vb + o], p = code >> 1, side = code & 1;
    const int v = a.pairs[2 * p + 1 - side];
    const double* Kv = a.K + 9 * v;
    double* c = s_cam[o];
    c[0] = Kv[0]; c[1] = Kv[4]; c[2] = Kv[2]; c[3] = Kv[5];
    for (int e = 0; e < 9; ++e) c[4 + e] = a.R[9 * v + e];
    rc_mv3(c + 4, C, c + 13);
    for (int e = 0; e < 3; ++e) c[13 + e] = RC_A(c[13 + e], a.t[3 * v + e]);
    s_obs[o][0] = code;
    s_obs[o][1] = v;
  }
  __syncthreads();
  pdl_wait();
  if (k >= n_rows) return;
  const double* Ka = a.K + 9 * img;
  const double fx = Ka[0], fy = Ka[4], cx = Ka[2], cy = Ka[5];
  const double t2 = a.thresh2;
  // partner rows
  for (int o = 0; o < V; ++o) {
    const int code = s_obs[o][0], p = code >> 1, v = s_obs[o][1];
    int j, nv;
    const int* poff = lines ? a.seg_off : a.kp_off;
    nv = poff[v + 1] - poff[v];
    if (code & 1) {
      j = (lines ? a.inv_l : a.inv_p)[(lines ? a.inv_off_l : a.inv_off_p)[p] + k];
    } else {
      j = lines ? a.matches_l[a.cu_l[p] + k] : a.matches_p[a.cu_p[p] + k];
    }
    float4 px = make_float4(__int_as_float(0x7fc00000), 0.f, 0.f, 0.f);
    if (j >= 0 && j < nv) {
      if (lines) {
        px = reinterpret_cast<const float4*>(a.segs)[poff[v] + j];
      } else {
        const float2 q = reinterpret_cast<const float2*>(a.kpts)[poff[v] + j];
        px.x = q.x; px.y = q.y;
      }
    }
    s_px[o * TRI_THREADS + tid] = px;
  }
  if (!lines) {
    const float2 q = reinterpret_cast<const float2*>(a.kpts)[off[img] + k];
    double r[3];
    rc_ray(Ra, fx, fy, cx, cy, q.x, q.y, r);
    int best = -1;
    double s_best = 0.0;
    unsigned long long mask = 0ull;
    for (int o = 0; o < V; ++o) {
      const double* c = s_cam[o];
      const float4 po = s_px[o * TRI_THREADS + tid];
      const TriPt t = tri_point_terms(c, r, make_float2(po.x, po.y));
      const double s = -RC_D(RC_A(RC_M(t.ax, t.bx), RC_M(t.ay, t.by)), RC_A(RC_M(t.bx, t.bx), RC_M(t.by, t.by)));
      if (!(s > 0.0)) continue;
      double P[3];
      for (int e = 0; e < 3; ++e) P[e] = RC_A(c[13 + e], RC_M(s, t.B[e]));
      if (!(rc_dot3(t.B, P) <= RC_M(a.cos_min, __dsqrt_rn(RC_M(rc_dot3(t.B, t.B), rc_dot3(P, P)))))) continue;
      unsigned long long m = 0ull;
      int cnt = 0;
      for (int q = 0; q < V; ++q) {
        const float4 pq = s_px[q * TRI_THREADS + tid];
        const bool sup = tri_point_supports(tri_point_terms(s_cam[q], r, make_float2(pq.x, pq.y)), s_cam[q][15], s, t2);
        m |= (unsigned long long)sup << q;
        cnt += sup;
      }
      if (cnt > best) {
        best = cnt;
        s_best = s;
        mask = m;
      }
    }
    int nvw = 0;
    double X[3] = {__longlong_as_double(0x7ff8000000000000ll), __longlong_as_double(0x7ff8000000000000ll),
                   __longlong_as_double(0x7ff8000000000000ll)};
    if (best >= 0) {
      double s = s_best;
      for (int it = 0; it < TRI_GN_ITERS; ++it) {
        double jj = 0.0, jr = 0.0;
        for (int q = 0; q < V; ++q) {
          if (!((mask >> q) & 1ull)) continue;
          const float4 pq = s_px[q * TRI_THREADS + tid];
          const TriPt t = tri_point_terms(s_cam[q], r, make_float2(pq.x, pq.y));
          const double gz = s_cam[q][15];
          tri_gn_term(t.ax, t.bx, gz, t.B[2], s, jj, jr);
          tri_gn_term(t.ay, t.by, gz, t.B[2], s, jj, jr);
        }
        if (!tri_gn_step(jj, jr, s)) break;
      }
      if (s > 0.0) {
        int cnt = 0;
        for (int q = 0; q < V; ++q) {
          const float4 pq = s_px[q * TRI_THREADS + tid];
          cnt += tri_point_supports(tri_point_terms(s_cam[q], r, make_float2(pq.x, pq.y)), s_cam[q][15], s, t2);
        }
        if (cnt >= best) {
          best = cnt;
          s_best = s;
        }
      }
      if (1 + best >= a.min_views) {
        nvw = 1 + best;
        for (int e = 0; e < 3; ++e) X[e] = RC_A(C[e], RC_M(s_best, r[e]));
      }
    }
    const long long row = off[img] + k;
    for (int e = 0; e < 3; ++e) a.points3d[3 * row + e] = X[e];
    a.n_views_p[row] = nvw;
  } else {
    const float4 sg = reinterpret_cast<const float4*>(a.segs)[off[img] + k];
    double r0[3], r1[3];
    rc_ray(Ra, fx, fy, cx, cy, sg.x, sg.y, r0);
    rc_ray(Ra, fx, fy, cx, cy, sg.z, sg.w, r1);
    int best = -1;
    double b0 = 0.0, b1 = 0.0;
    unsigned long long mask = 0ull;
    for (int o = 0; o < V; ++o) {
      const double* c = s_cam[o];
      double n[3];
      rc_line_normal(c, s_px[o * TRI_THREADS + tid], n);
      const double alpha = rc_dot3(n, c + 13), nn = rc_dot3(n, n);
      const TriEnd e0 = tri_end_terms(c, n, r0), e1 = tri_end_terms(c, n, r1);
      const double s0 = -RC_D(alpha, e0.beta), s1 = -RC_D(alpha, e1.beta);
      if (!(s0 > 0.0 && s1 > 0.0)) continue;
      if (!(RC_M(e0.beta, e0.beta) >= RC_M(a.sin2_min, RC_M(nn, e0.BB)) &&
            RC_M(e1.beta, e1.beta) >= RC_M(a.sin2_min, RC_M(nn, e1.BB))))
        continue;
      unsigned long long m = 0ull;
      int cnt = 0;
      for (int q = 0; q < V; ++q) {
        const double* cq = s_cam[q];
        double nq[3];
        rc_line_normal(cq, s_px[q * TRI_THREADS + tid], nq);
        const double aq = rc_dot3(nq, cq + 13);
        const bool sup = tri_end_supports(aq, tri_end_terms(cq, nq, r0), cq[15], s0, t2) &&
                         tri_end_supports(aq, tri_end_terms(cq, nq, r1), cq[15], s1, t2);
        m |= (unsigned long long)sup << q;
        cnt += sup;
      }
      if (cnt > best) {
        best = cnt;
        b0 = s0;
        b1 = s1;
        mask = m;
      }
    }
    int nvw = 0;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    double X[6] = {nan, nan, nan, nan, nan, nan};
    if (best >= 0) {
      double s[2] = {b0, b1};
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const double* r = e ? r1 : r0;
        for (int it = 0; it < TRI_GN_ITERS; ++it) {
          double jj = 0.0, jr = 0.0;
          for (int q = 0; q < V; ++q) {
            if (!((mask >> q) & 1ull)) continue;
            const double* cq = s_cam[q];
            double nq[3];
            rc_line_normal(cq, s_px[q * TRI_THREADS + tid], nq);
            const TriEnd t = tri_end_terms(cq, nq, r);
            tri_gn_term(rc_dot3(nq, cq + 13), t.beta, cq[15], t.delta, s[e], jj, jr);
          }
          if (!tri_gn_step(jj, jr, s[e])) break;
        }
      }
      if (s[0] > 0.0 && s[1] > 0.0) {
        int cnt = 0;
        for (int q = 0; q < V; ++q) {
          const double* cq = s_cam[q];
          double nq[3];
          rc_line_normal(cq, s_px[q * TRI_THREADS + tid], nq);
          const double aq = rc_dot3(nq, cq + 13);
          cnt += tri_end_supports(aq, tri_end_terms(cq, nq, r0), cq[15], s[0], t2) &&
                 tri_end_supports(aq, tri_end_terms(cq, nq, r1), cq[15], s[1], t2);
        }
        if (cnt >= best) {
          best = cnt;
          b0 = s[0];
          b1 = s[1];
        }
      }
      if (1 + best >= a.min_views) {
        nvw = 1 + best;
        for (int e = 0; e < 3; ++e) {
          X[e] = RC_A(C[e], RC_M(b0, r0[e]));
          X[3 + e] = RC_A(C[e], RC_M(b1, r1[e]));
        }
      }
    }
    const long long row = off[img] + k;
    for (int e = 0; e < 6; ++e) a.lines3d[6 * row + e] = X[e];
    a.n_views_l[row] = nvw;
  }
}

}  // namespace ltr
