// Tracks of posed image sets (ltr_tracks): the pair matches that agree with the known poses join the rows of every
// image into point and line tracks, and each track gets one robust multi-view world point or world line.
//
// Model (DESIGN.md "Tracks"; restated in numpy by linetr_b200.tracks.triangulate_tracks_host):
//   nodes: image i's keypoint k is point node kp_off[i] + k, its key line k line node seg_off[i] + k (two graphs).
//   edges: a match row of pair p = (i, j) with m in [0, rows of j) is an edge iff it agrees with the pixel fundamental
//   matrix F[p] of the poses (staged by the caller): fm_inlier(F, q, epi_thresh^2) for a point, fm_line_consistent(F,
//   s0, s1, min_overlap) for a key line.
//   components: lock-free union-find (the larger root is linked under the smaller with atomicCAS), then full path
//   compression, so every component's label is its minimum node whatever order the atomics ran in.  A track is a
//   component of >= 2 nodes; track ids ascend with the minimum node (an integer prefix sum over the roots); its
//   observations obs[track_off[t] .. track_off[t + 1]) ascend by node.
//   estimate (tracks of at most TRK_MAX_OBS observations, o = 0 .. V - 1 in track order): candidate (i, j), i < j, is
//   the two-view estimate of ltr_triangulate with anchor i and partner j (a point's least-squares depth, a key line's
//   two plane intersections; depth > 0 and the min_angle rule).  Observation q supports a world point X iff its depth
//   P_z > 0, P = R_q X + t_q, and its squared reprojection error <= thresh^2 (a key line: the signed distance of both
//   end points to q's infinite line).  Winner: the largest (supporters << 32) | ~(i * TRK_MAX_OBS + j).  Refit:
//   TRK_GN_ITERS Gauss-Newton steps on the world point (a key line: each anchor end point separately) in a frame centred
//   on the anchor camera, 3 x 3 normal equations solved by Gaussian elimination with first-largest partial pivoting;
//   kept iff every winner supporter keeps P_z > 0 and the supporter count does not fall.  Inliers are the supporters of
//   the kept estimate; the track is valid iff inliers >= min_views.  Every operation is explicitly rounded fp64, every
//   sum in a fixed order.
//
// Kernels (launched in this order, PDL-chained):
//   trk_init_kernel    per node: parent = self, size = 0, slot counter = 0; per-row outputs NaN / 0.
//   trk_edge_kernel    per match row: the epipolar check, then the union.
//   trk_root_kernel    per node: path compression to the root, atomicAdd of the component size.
//   trk_scan_kernel    one CTA per graph: exclusive prefix sum over the roots of >= 2 nodes -> track ids, track_off,
//                      the track count (device scalar).
//   trk_assign_kernel  per node: its track id, and an observation slot (atomicAdd; order fixed by the next kernel).
//   trk_kernel         persistent grid (x: CTAs, y: graph) over the tracks up to the device track count: sorts the
//                      track's observations, then candidates, winner, refit and the outputs.
#pragma once
#include "common.cuh"
#include "rn_fp64.cuh"
#include "fundamental.cuh"
#include "triangulation.cuh"

namespace ltr {

constexpr int TRK_THREADS = 128;
constexpr int TRK_ROW_THREADS = 256;
constexpr int TRK_SCAN_THREADS = 1024;
constexpr int TRK_SCAN_ITEMS = 8;
constexpr int TRK_MAX_OBS = 64;          // LTR_TRK_MAX_OBS: one 64-bit support mask per candidate
constexpr int TRK_GN_ITERS = 5;
constexpr int TRK_CAM = 28;              // staged doubles per observation: fx fy cx cy, R (9), t (3), C (3), r0, r1, n
enum { TRK_OK = 0, TRK_TOO_LONG = 1, TRK_NO_CANDIDATE = 2, TRK_TOO_FEW = 3 };

struct TrkArgs {
  const float* kpts; const int* kp_off;      // [*, 2] keypoints of image i from row kp_off[i], [n + 1]
  const float* segs; const int* seg_off;     // [*, 4] key lines, [n + 1]
  const double* K; const double* R; const double* t; const double* F;   // [n,3,3], [n,3,3], [n,3], [P,9]
  const int* pairs;                          // [P, 2]
  const int* matches_p; const int* cu_p;
  const int* matches_l; const int* cu_l;
  int n_images, n_pairs, total_p, total_l;
  int n_nodes[2];                            // keypoint rows, key-line rows
  double thresh2, epi2, min_overlap, cos_min, sin2_min;
  int min_views;
  int* parent; int* size; int* root_id; int* fill; int* obs_raw;   // workspace over both graphs' nodes
  int* track_row[2]; int* n_tracks[2]; int* track_off[2]; int* obs[2];
  int* n_obs[2]; int* n_inliers[2]; int* n_imgs[2]; int* status[2];
  double* points3d; double* lines3d;         // [T_p, 3], [T_l, 2, 3]
  double* row_points; double* row_lines;     // [n_nodes[0], 3], [n_nodes[1], 2, 3]
  uint8_t* inlier[2]; int* n_views[2];
};

__device__ __forceinline__ int trk_find(const int* par, int x) {
  int p = __ldcg(par + x);
  while (p != x) {
    x = p;
    p = __ldcg(par + x);
  }
  return x;
}

// Union of the components of a and b: the larger root goes under the smaller (parent[x] <= x always holds, so a
// component's root is its minimum node).
__device__ __forceinline__ void trk_unite(int* par, int a, int b) {
  for (;;) {
    a = trk_find(par, a);
    b = trk_find(par, b);
    if (a == b) return;
    const int hi = a > b ? a : b, lo = a > b ? b : a;
    if (atomicCAS(par + hi, hi, lo) == hi) return;
  }
}

__global__ void __launch_bounds__(TRK_ROW_THREADS) trk_init_kernel(const TrkArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const int x = blockIdx.x * TRK_ROW_THREADS + threadIdx.x;
  if (x >= a.n_nodes[0] + a.n_nodes[1]) return;
  a.parent[x] = x;
  a.size[x] = 0;
  a.fill[x] = 0;
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  const int g = x >= a.n_nodes[0], row = g ? x - a.n_nodes[0] : x;
  a.inlier[g][row] = 0;
  a.n_views[g][row] = 0;
  if (g) {
    for (int e = 0; e < 6; ++e) a.row_lines[6ll * row + e] = nan;
  } else {
    for (int e = 0; e < 3; ++e) a.row_points[3ll * row + e] = nan;
  }
}

__global__ void __launch_bounds__(TRK_ROW_THREADS) trk_edge_kernel(const TrkArgs a) {
  pdl_launch_dependents();
  const long long r = (long long)blockIdx.x * TRK_ROW_THREADS + threadIdx.x;
  const bool lines = r >= a.total_p;
  const int row = (int)(lines ? r - a.total_p : r);
  pdl_wait();
  if (r >= (long long)a.total_p + a.total_l) return;
  const int* cu = lines ? a.cu_l : a.cu_p;
  const int* off = lines ? a.seg_off : a.kp_off;
  const int p = rc_segment(cu, a.n_pairs, row);
  const int i = a.pairs[2 * p], j = a.pairs[2 * p + 1];
  const int k = row - cu[p], m = (lines ? a.matches_l : a.matches_p)[row];
  if (!(m >= 0 && m < off[j + 1] - off[j])) return;
  double F[9];
  for (int e = 0; e < 9; ++e) F[e] = a.F[9 * p + e];
  const int u = off[i] + k, v = off[j] + m;
  bool edge;
  if (lines) {
    edge = fm_line_consistent(F, a.segs + 4ll * u, a.segs + 4ll * v, a.min_overlap);
  } else {
    const float2 q0 = reinterpret_cast<const float2*>(a.kpts)[u], q1 = reinterpret_cast<const float2*>(a.kpts)[v];
    edge = fm_inlier(F, make_float4(q0.x, q0.y, q1.x, q1.y), a.epi2);
  }
  const int base = lines ? a.n_nodes[0] : 0;
  if (edge) trk_unite(a.parent, base + u, base + v);
}

__global__ void __launch_bounds__(TRK_ROW_THREADS) trk_root_kernel(const TrkArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const int x = blockIdx.x * TRK_ROW_THREADS + threadIdx.x;
  if (x >= a.n_nodes[0] + a.n_nodes[1]) return;
  const int r = trk_find(a.parent, x);
  a.parent[x] = r;
  atomicAdd(a.size + r, 1);
}

// One CTA per graph: tracks and observations before each root, in node order (a 64-bit (tracks << 32) + observations
// exclusive block scan per chunk of TRK_SCAN_THREADS * TRK_SCAN_ITEMS nodes, with the running total carried).
__global__ void __launch_bounds__(TRK_SCAN_THREADS) trk_scan_kernel(const TrkArgs a) {
  __shared__ unsigned long long s_warp[TRK_SCAN_THREADS / 32];
  pdl_launch_dependents();
  pdl_wait();
  const int g = blockIdx.x, base = g ? a.n_nodes[0] : 0, N = a.n_nodes[g];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  unsigned long long carry = 0;
  for (int c0 = 0; c0 < N; c0 += TRK_SCAN_THREADS * TRK_SCAN_ITEMS) {
    const int b = c0 + tid * TRK_SCAN_ITEMS;
    int sz[TRK_SCAN_ITEMS];
    unsigned long long mine = 0;
#pragma unroll
    for (int e = 0; e < TRK_SCAN_ITEMS; ++e) {
      const int x = b + e;
      sz[e] = 0;
      if (x < N && a.parent[base + x] == base + x && a.size[base + x] >= 2) sz[e] = a.size[base + x];
      if (sz[e]) mine += (1ull << 32) + (unsigned long long)sz[e];
    }
    unsigned long long v = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += y;
    }
    if (lane == 31) s_warp[wid] = v;
    __syncthreads();
    if (wid == 0) {
      unsigned long long w = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += y;
      }
      s_warp[lane] = w;
    }
    __syncthreads();
    unsigned long long run = carry + (wid ? s_warp[wid - 1] : 0ull) + (v - mine);
#pragma unroll
    for (int e = 0; e < TRK_SCAN_ITEMS; ++e) {
      if (!sz[e]) continue;
      const int id = (int)(run >> 32);
      a.root_id[base + b + e] = id;
      a.track_off[g][id] = (int)(run & 0xffffffffull);
      run += (1ull << 32) + (unsigned long long)sz[e];
    }
    carry += s_warp[TRK_SCAN_THREADS / 32 - 1];
    __syncthreads();
  }
  if (tid == 0) {
    a.n_tracks[g][0] = (int)(carry >> 32);
    a.track_off[g][carry >> 32] = (int)(carry & 0xffffffffull);
  }
}

__global__ void __launch_bounds__(TRK_ROW_THREADS) trk_assign_kernel(const TrkArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const int x = blockIdx.x * TRK_ROW_THREADS + threadIdx.x;
  if (x >= a.n_nodes[0] + a.n_nodes[1]) return;
  const int g = x >= a.n_nodes[0], base = g ? a.n_nodes[0] : 0, row = x - base;
  const int r = a.parent[x];
  int id = -1;
  if (a.size[r] >= 2) {
    id = a.root_id[r];
    const int slot = atomicAdd(a.fill + base + id, 1);
    a.obs_raw[base + a.track_off[g][id] + slot] = row;
  }
  a.track_row[g][row] = id;
}

// Observation q supports the world point X: depth P_z > 0 (P = R_q X + t_q) and squared reprojection error <= t2.
__device__ __forceinline__ bool trk_point_supports(const double* c, float2 px, const double* X, double t2) {
  double P[3];
  rc_mv3(c + 4, X, P);
  for (int e = 0; e < 3; ++e) P[e] = RC_A(P[e], c[13 + e]);
  const double dx = RC_S((double)px.x, c[2]), dy = RC_S((double)px.y, c[3]);
  const double ex = RC_S(RC_M(c[0], P[0]), RC_M(dx, P[2])), ey = RC_S(RC_M(c[1], P[1]), RC_M(dy, P[2]));
  return P[2] > 0.0 && RC_A(RC_M(ex, ex), RC_M(ey, ey)) <= RC_M(t2, RC_M(P[2], P[2]));
}

// Observation q supports the world end point X: P_z > 0 and (n_q . P)^2 <= t2 P_z^2 (q's line normal at c + 25).
__device__ __forceinline__ bool trk_end_supports(const double* c, const double* X, double t2) {
  double P[3];
  rc_mv3(c + 4, X, P);
  for (int e = 0; e < 3; ++e) P[e] = RC_A(P[e], c[13 + e]);
  const double v = rc_dot3(c + 25, P);
  return P[2] > 0.0 && RC_M(v, v) <= RC_M(t2, RC_M(P[2], P[2]));
}

// The depth P_z of world point X in observation q.
__device__ __forceinline__ double trk_depth(const double* c, const double* X) {
  return RC_A(rc_dot3(c + 10, X), c[15]);
}

// Partner j as ltr_triangulate's camera relative to anchor i (TRI_CAM doubles: fx fy cx cy, R_j, A = R_j C_i + t_j).
__device__ __forceinline__ void trk_partner(const double* ci, const double* cj, double* o) {
  for (int e = 0; e < 13; ++e) o[e] = cj[e];
  rc_mv3(cj + 4, ci + 16, o + 13);
  for (int e = 0; e < 3; ++e) o[13 + e] = RC_A(o[13 + e], cj[13 + e]);
}

// Candidate (i, j) of a point track -> the world point X; false when it fails the depth or angle rule.
__device__ __forceinline__ bool trk_point_candidate(const double (*cam)[TRK_CAM], float2 pj, int i, int j,
                                                    double cos_min, double* X) {
  double c[TRI_CAM];
  trk_partner(cam[i], cam[j], c);
  const double* r = cam[i] + 19;
  const TriPt t = tri_point_terms(c, r, pj);
  const double s = -RC_D(RC_A(RC_M(t.ax, t.bx), RC_M(t.ay, t.by)), RC_A(RC_M(t.bx, t.bx), RC_M(t.by, t.by)));
  if (!(s > 0.0)) return false;
  double P[3];
  for (int e = 0; e < 3; ++e) P[e] = RC_A(c[13 + e], RC_M(s, t.B[e]));
  if (!(rc_dot3(t.B, P) <= RC_M(cos_min, __dsqrt_rn(RC_M(rc_dot3(t.B, t.B), rc_dot3(P, P)))))) return false;
  for (int e = 0; e < 3; ++e) X[e] = RC_A(cam[i][16 + e], RC_M(s, r[e]));
  return true;
}

// Candidate (i, j) of a line track -> anchor i's world end points X [6]; false on the depth or angle rule.
__device__ __forceinline__ bool trk_line_candidate(const double (*cam)[TRK_CAM], int i, int j, double sin2_min,
                                                   double* X) {
  double c[TRI_CAM];
  trk_partner(cam[i], cam[j], c);
  const double* n = cam[j] + 25;
  const double* r0 = cam[i] + 19;
  const double* r1 = cam[i] + 22;
  const double alpha = rc_dot3(n, c + 13), nn = rc_dot3(n, n);
  const TriEnd e0 = tri_end_terms(c, n, r0), e1 = tri_end_terms(c, n, r1);
  const double s0 = -RC_D(alpha, e0.beta), s1 = -RC_D(alpha, e1.beta);
  if (!(s0 > 0.0 && s1 > 0.0)) return false;
  if (!(RC_M(e0.beta, e0.beta) >= RC_M(sin2_min, RC_M(nn, e0.BB)) &&
        RC_M(e1.beta, e1.beta) >= RC_M(sin2_min, RC_M(nn, e1.BB))))
    return false;
  for (int e = 0; e < 3; ++e) {
    X[e] = RC_A(cam[i][16 + e], RC_M(s0, r0[e]));
    X[3 + e] = RC_A(cam[i][16 + e], RC_M(s1, r1[e]));
  }
  return true;
}

// One residual (num / den) with d num / dY = b and d den / dY = R_q row 2 into the normal equations (h: 00 01 02 11 12
// 22, g: J^T r).
__device__ __forceinline__ void trk_gn_term(double num, double den, const double* b, const double* d, double* h,
                                            double* g) {
  const double r = RC_D(num, den);
  double J[3];
  for (int k = 0; k < 3; ++k) J[k] = RC_D(RC_S(b[k], RC_M(r, d[k])), den);
  h[0] = RC_A(h[0], RC_M(J[0], J[0]));
  h[1] = RC_A(h[1], RC_M(J[0], J[1]));
  h[2] = RC_A(h[2], RC_M(J[0], J[2]));
  h[3] = RC_A(h[3], RC_M(J[1], J[1]));
  h[4] = RC_A(h[4], RC_M(J[1], J[2]));
  h[5] = RC_A(h[5], RC_M(J[2], J[2]));
  for (int k = 0; k < 3; ++k) g[k] = RC_A(g[k], RC_M(J[k], r));
}

// A point's two pixel residual terms in observation c at the anchor-frame point Y (A = R_q C_anchor + t_q).
__device__ __forceinline__ void trk_pixel_terms(const double* c, const double* A, float2 px, const double* Y, double* h,
                                                double* g) {
  double P[3];
  rc_mv3(c + 4, Y, P);
  for (int e = 0; e < 3; ++e) P[e] = RC_A(P[e], A[e]);
  const double dx = RC_S((double)px.x, c[2]), dy = RC_S((double)px.y, c[3]);
  const double* R = c + 4;
  double b[3];
  for (int k = 0; k < 3; ++k) b[k] = RC_S(RC_M(c[0], R[k]), RC_M(dx, R[6 + k]));
  trk_gn_term(RC_S(RC_M(c[0], P[0]), RC_M(dx, P[2])), P[2], b, R + 6, h, g);
  for (int k = 0; k < 3; ++k) b[k] = RC_S(RC_M(c[1], R[3 + k]), RC_M(dy, R[6 + k]));
  trk_gn_term(RC_S(RC_M(c[1], P[1]), RC_M(dy, P[2])), P[2], b, R + 6, h, g);
}

// The signed-distance residual n . P / P_z of observation c at Y.
__device__ __forceinline__ void trk_line_term(const double* c, const double* A, const double* Y, double* h, double* g) {
  double P[3];
  rc_mv3(c + 4, Y, P);
  for (int e = 0; e < 3; ++e) P[e] = RC_A(P[e], A[e]);
  const double* R = c + 4;
  const double* n = c + 25;
  double b[3];
  for (int k = 0; k < 3; ++k) b[k] = RC_A(RC_A(RC_M(n[0], R[k]), RC_M(n[1], R[3 + k])), RC_M(n[2], R[6 + k]));
  trk_gn_term(rc_dot3(n, P), P[2], b, R + 6, h, g);
}

// Y -= H^-1 g by Gaussian elimination with first-largest partial pivoting; false (Y unchanged) on a zero pivot or a
// non-finite step.
__device__ __forceinline__ bool trk_solve_step(const double* h, const double* g, double* Y) {
  double M[3][4] = {{h[0], h[1], h[2], g[0]}, {h[1], h[3], h[4], g[1]}, {h[2], h[4], h[5], g[2]}};
  for (int c = 0; c < 3; ++c) {
    int p = c;
    for (int r = c + 1; r < 3; ++r)
      if (fabs(M[r][c]) > fabs(M[p][c])) p = r;
    if (!(fabs(M[p][c]) > 0.0)) return false;
    if (p != c)
      for (int k = 0; k < 4; ++k) {
        const double tmp = M[c][k];
        M[c][k] = M[p][k];
        M[p][k] = tmp;
      }
    for (int r = c + 1; r < 3; ++r) {
      const double f = RC_D(M[r][c], M[c][c]);
      for (int k = c + 1; k < 4; ++k) M[r][k] = RC_S(M[r][k], RC_M(f, M[c][k]));
    }
  }
  double d[3];
  d[2] = RC_D(M[2][3], M[2][2]);
  d[1] = RC_D(RC_S(M[1][3], RC_M(M[1][2], d[2])), M[1][1]);
  d[0] = RC_D(RC_S(RC_S(M[0][3], RC_M(M[0][1], d[1])), RC_M(M[0][2], d[2])), M[0][0]);
  double Yn[3];
  for (int k = 0; k < 3; ++k) {
    Yn[k] = RC_S(Y[k], d[k]);
    if (!isfinite(Yn[k])) return false;
  }
  for (int k = 0; k < 3; ++k) Y[k] = Yn[k];
  return true;
}

__global__ void __launch_bounds__(TRK_THREADS) trk_kernel(const TrkArgs a) {
  __shared__ double s_cam[TRK_MAX_OBS][TRK_CAM];
  __shared__ float4 s_px[TRK_MAX_OBS];
  __shared__ int s_node[TRK_MAX_OBS];
  __shared__ unsigned long long s_key[TRK_THREADS / 32];
  __shared__ int s_nimg;
  __shared__ double s_X[6];
  __shared__ unsigned long long s_mask;
  __shared__ int s_valid, s_ninl;
  pdl_launch_dependents();
  pdl_wait();
  const int g = blockIdx.y, tid = threadIdx.x;
  const bool lines = g == 1;
  const int base = lines ? a.n_nodes[0] : 0;
  const int* off = lines ? a.seg_off : a.kp_off;
  const int n_tracks = *a.n_tracks[g];
  const double t2 = a.thresh2, nan = __longlong_as_double(0x7ff8000000000000ll);
  const float2* kp = reinterpret_cast<const float2*>(a.kpts);
  const float4* sg = reinterpret_cast<const float4*>(a.segs);
  for (int id = blockIdx.x; id < n_tracks; id += gridDim.x) {
    const int o0 = a.track_off[g][id], V = a.track_off[g][id + 1] - o0;
    const int* raw = a.obs_raw + base + o0;
    int* obs = a.obs[g] + o0;
    if (tid == 0) s_nimg = 0;
    // the observations in node order (slots were taken in any order)
    for (int q = tid; q < V; q += TRK_THREADS) {
      const int node = raw[q];
      int rk = 0;
      for (int u = 0; u < V; ++u) rk += raw[u] < node;
      obs[rk] = node;
      if (V <= TRK_MAX_OBS) s_node[rk] = node;
    }
    __syncthreads();
    for (int q = tid; q < V; q += TRK_THREADS) {
      const int img = rc_segment(off, a.n_images, obs[q]);
      if (q == 0 || img != rc_segment(off, a.n_images, obs[q - 1])) atomicAdd(&s_nimg, 1);
    }
    __syncthreads();
    if (tid == 0) {
      a.n_obs[g][id] = V;
      a.n_imgs[g][id] = s_nimg;
    }
    if (V > TRK_MAX_OBS) {
      if (tid == 0) {
        a.status[g][id] = TRK_TOO_LONG;
        a.n_inliers[g][id] = 0;
        if (lines) for (int e = 0; e < 6; ++e) a.lines3d[6ll * id + e] = nan;
        else for (int e = 0; e < 3; ++e) a.points3d[3ll * id + e] = nan;
      }
      __syncthreads();
      continue;
    }
    // stage each observation's camera, centre, ray(s) and pixel / line normal
    if (tid < V) {
      const int node = s_node[tid], v = rc_segment(off, a.n_images, node);
      double* c = s_cam[tid];
      const double* Kv = a.K + 9 * v;
      c[0] = Kv[0]; c[1] = Kv[4]; c[2] = Kv[2]; c[3] = Kv[5];
      for (int e = 0; e < 9; ++e) c[4 + e] = a.R[9 * v + e];
      for (int e = 0; e < 3; ++e) c[13 + e] = a.t[3 * v + e];
      const double* Rv = c + 4;
      rc_centre(Rv, c + 13, c + 16);
      if (lines) {
        const float4 s = sg[node];
        s_px[tid] = s;
        rc_ray(Rv, c[0], c[1], c[2], c[3], s.x, s.y, c + 19);
        rc_ray(Rv, c[0], c[1], c[2], c[3], s.z, s.w, c + 22);
        rc_line_normal(c, s, c + 25);
      } else {
        const float2 q = kp[node];
        s_px[tid] = make_float4(q.x, q.y, 0.f, 0.f);
        rc_ray(Rv, c[0], c[1], c[2], c[3], q.x, q.y, c + 19);
      }
    }
    __syncthreads();
    // candidates (i, j), i < j: the most supporters, ties to the lowest i * TRK_MAX_OBS + j
    unsigned long long key = 0;
    for (int cidx = tid; cidx < V * V; cidx += TRK_THREADS) {
      const int i = cidx / V, j = cidx - i * V;
      if (j <= i) continue;
      double X[6];
      unsigned cnt = 0;
      if (lines) {
        if (!trk_line_candidate(s_cam, i, j, a.sin2_min, X)) continue;
        for (int q = 0; q < V; ++q) cnt += trk_end_supports(s_cam[q], X, t2) && trk_end_supports(s_cam[q], X + 3, t2);
      } else {
        if (!trk_point_candidate(s_cam, make_float2(s_px[j].x, s_px[j].y), i, j, a.cos_min, X)) continue;
        for (int q = 0; q < V; ++q)
          cnt += trk_point_supports(s_cam[q], make_float2(s_px[q].x, s_px[q].y), X, t2);
      }
      const unsigned long long k = ((unsigned long long)cnt << 32) | (unsigned long long)(~(unsigned)(i * TRK_MAX_OBS + j));
      key = k > key ? k : key;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long y = __shfl_xor_sync(0xffffffffu, key, o);
      key = y > key ? y : key;
    }
    if ((tid & 31) == 0) s_key[tid >> 5] = key;
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < TRK_THREADS / 32; ++w) key = s_key[w] > key ? s_key[w] : key;
      int status = TRK_NO_CANDIDATE, ninl = 0;
      unsigned long long mask = 0;
      double X[6] = {nan, nan, nan, nan, nan, nan};
      if (key) {
        const unsigned idx = ~(unsigned)(key & 0xffffffffull);
        const int i = idx / TRK_MAX_OBS, j = idx % TRK_MAX_OBS, best = (int)(key >> 32);
        const double* ci = s_cam[i];
        double A[3];
        if (lines) {
          trk_line_candidate(s_cam, i, j, a.sin2_min, X);
          for (int q = 0; q < V; ++q)
            mask |= (unsigned long long)(trk_end_supports(s_cam[q], X, t2) && trk_end_supports(s_cam[q], X + 3, t2)) << q;
          double Xr[6];
          for (int e = 0; e < 2; ++e) {
            double Y[3];
            for (int k = 0; k < 3; ++k) Y[k] = RC_S(X[3 * e + k], ci[16 + k]);
            const float2 pe = e ? make_float2(s_px[i].z, s_px[i].w) : make_float2(s_px[i].x, s_px[i].y);
            for (int it = 0; it < TRK_GN_ITERS; ++it) {
              double h[6] = {0, 0, 0, 0, 0, 0}, gr[3] = {0, 0, 0};
              rc_mv3(ci + 4, ci + 16, A);
              for (int k = 0; k < 3; ++k) A[k] = RC_A(A[k], ci[13 + k]);
              trk_pixel_terms(ci, A, pe, Y, h, gr);
              for (int q = 0; q < V; ++q) {
                if (q == i || !((mask >> q) & 1ull)) continue;
                rc_mv3(s_cam[q] + 4, ci + 16, A);
                for (int k = 0; k < 3; ++k) A[k] = RC_A(A[k], s_cam[q][13 + k]);
                trk_line_term(s_cam[q], A, Y, h, gr);
              }
              if (!trk_solve_step(h, gr, Y)) break;
            }
            for (int k = 0; k < 3; ++k) Xr[3 * e + k] = RC_A(ci[16 + k], Y[k]);
          }
          bool front = true;
          unsigned long long mr = 0;
          for (int q = 0; q < V; ++q) {
            if ((mask >> q) & 1ull) front = front && trk_depth(s_cam[q], Xr) > 0.0 && trk_depth(s_cam[q], Xr + 3) > 0.0;
            mr |= (unsigned long long)(trk_end_supports(s_cam[q], Xr, t2) && trk_end_supports(s_cam[q], Xr + 3, t2)) << q;
          }
          if (front && __popcll(mr) >= best) {
            for (int e = 0; e < 6; ++e) X[e] = Xr[e];
            mask = mr;
          }
        } else {
          trk_point_candidate(s_cam, make_float2(s_px[j].x, s_px[j].y), i, j, a.cos_min, X);
          for (int q = 0; q < V; ++q)
            mask |= (unsigned long long)trk_point_supports(s_cam[q], make_float2(s_px[q].x, s_px[q].y), X, t2) << q;
          double Y[3];
          for (int k = 0; k < 3; ++k) Y[k] = RC_S(X[k], ci[16 + k]);
          for (int it = 0; it < TRK_GN_ITERS; ++it) {
            double h[6] = {0, 0, 0, 0, 0, 0}, gr[3] = {0, 0, 0};
            for (int q = 0; q < V; ++q) {
              if (!((mask >> q) & 1ull)) continue;
              rc_mv3(s_cam[q] + 4, ci + 16, A);
              for (int k = 0; k < 3; ++k) A[k] = RC_A(A[k], s_cam[q][13 + k]);
              trk_pixel_terms(s_cam[q], A, make_float2(s_px[q].x, s_px[q].y), Y, h, gr);
            }
            if (!trk_solve_step(h, gr, Y)) break;
          }
          double Xr[3];
          for (int k = 0; k < 3; ++k) Xr[k] = RC_A(ci[16 + k], Y[k]);
          bool front = true;
          unsigned long long mr = 0;
          for (int q = 0; q < V; ++q) {
            if ((mask >> q) & 1ull) front = front && trk_depth(s_cam[q], Xr) > 0.0;
            mr |= (unsigned long long)trk_point_supports(s_cam[q], make_float2(s_px[q].x, s_px[q].y), Xr, t2) << q;
          }
          if (front && __popcll(mr) >= best) {
            for (int k = 0; k < 3; ++k) X[k] = Xr[k];
            mask = mr;
          }
        }
        ninl = __popcll(mask);
        status = ninl >= a.min_views ? TRK_OK : TRK_TOO_FEW;
      }
      if (status != TRK_OK)
        for (int e = 0; e < 6; ++e) X[e] = nan;
      a.status[g][id] = status;
      a.n_inliers[g][id] = ninl;
      if (lines) for (int e = 0; e < 6; ++e) a.lines3d[6ll * id + e] = X[e];
      else for (int e = 0; e < 3; ++e) a.points3d[3ll * id + e] = X[e];
      for (int e = 0; e < 6; ++e) s_X[e] = X[e];
      s_mask = mask;
      s_valid = status == TRK_OK;
      s_ninl = ninl;
    }
    __syncthreads();
    // per-row outputs: every inlier row, valid or not; coordinates for the rows of a valid track
    if (tid < V && ((s_mask >> tid) & 1ull)) {
      const int row = s_node[tid];
      a.inlier[g][row] = 1;
      if (s_valid) {
        a.n_views[g][row] = s_ninl;
        if (lines) {
          const double* c = s_cam[tid];
          double d[3], w[3];
          for (int k = 0; k < 3; ++k) {
            d[k] = RC_S(s_X[3 + k], s_X[k]);
            w[k] = RC_S(s_X[k], c[16 + k]);
          }
          for (int e = 0; e < 2; ++e) rc_closest_on_line(s_X, d, w, c + 19 + 3 * e, a.row_lines + 6ll * row + 3 * e);
        } else {
          for (int k = 0; k < 3; ++k) a.row_points[3ll * row + k] = s_X[k];
        }
      }
    }
    __syncthreads();
  }
}

}  // namespace ltr
