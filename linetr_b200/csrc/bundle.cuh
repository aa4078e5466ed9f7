// Bundle adjustment of posed image sets (ltr_bundle_adjust): the camera poses, the world points of the point tracks
// and the world lines of the line tracks of ltr_tracks refined together by Levenberg-Marquardt with a Schur complement
// onto the cameras.
//
// Model (DESIGN.md "Bundle adjustment"; restated in numpy by linetr_b200.bundle.bundle_adjust_host):
//   participation: a track takes part iff its ltr_tracks status is TRK_OK, its inlier rows lie in distinct images and
//   the Cholesky of its undamped initial landmark block has every pivot d_c > BA_DEGENERATE_PIVOT * V_cc.
//   residuals (pixels): a point row's two reprojection errors (f P_xy - (x - c) P_z) / P_z; a key-line row the signed
//   distances n . P / P_z of the track's two world end points to the row's line (P = R (X - C)).
//   parameters: camera R <- cay(w) R, C <- C + dC; point X <- X + dX; line X_a <- X_a + u1 da1 + u2 da2 (X_b likewise),
//   u1 = normalize(d x e_k) with e_k the first-smallest |d_k| of d = X_b - X_a, u2 = normalize(d x u1).
//   gauge: fixed images keep their pose; with exactly one fixed image, the lowest free image with a participating row
//   holds the centre coordinate hold[k] (chosen by the caller from the input).
//   step: (A + lambda diag A) on both blocks; per-track Cholesky of the landmark block, Y = W V^-1 per row; reduced
//   block (I, J), I >= J: delta_IJ U_I - sum_t Y_tI W_tJ^T in ascending track order; dense right-looking Cholesky,
//   forward and back substitution; landmark steps -V^-1 (g_t + sum_rows W^T dc).  Accepted iff every factorization
//   succeeds, every participating depth stays > 0 and the cost falls; lambda x0.1 / x10; stop on a relative decrease
//   <= ftol after an accepted step, lambda > 1e32 or max_iters iterations.  Every operation is explicitly rounded fp64
//   (no contraction; DMMA is not used: its accumulation order has no host twin), every sum in a fixed order.
//
// Kernels (PDL-chained; once the stop flag is set the iteration kernels return at once):
//   ba_start_kernel    one CTA: camera state (R, C = -R^T t), scalars.
//   ba_init_kernel     per track: status, image mask, the degeneracy test, initial cost.
//   ba_setup_kernel    one CTA: camera columns and gauge, per-image lists of (track, row) ascending by track, the
//                      initial cost reduction.
//   per iteration:
//     ba_track_kernel  per track: residuals, Jacobians, the damped landmark block's Cholesky, W and Y per row.
//     ba_reduce_kernel per image pair (I, J), I >= J: one block of the reduced camera matrix (and I's right-hand side).
//     ba_solve_kernel  one CTA: Cholesky, the two triangular solves, the candidate cameras.
//     ba_update_kernel per track: landmark step, candidate landmark, candidate cost and depths.
//     ba_accept_kernel one CTA: cost reduction, accept / reject, commit, lambda, stop.
//   ba_finish_kernel   outputs: poses, per-track coordinates and status, per-row residuals and rows(), stats.
#pragma once
#include "common.cuh"
#include "rn_fp64.cuh"
#include "triangulation.cuh"
#include "tracks.cuh"

namespace ltr {

constexpr int BA_MAX_IMAGES = 128;       // LTR_BA_MAX_IMAGES: a track's image set is a 128-bit mask
constexpr int BA_THREADS = 128;
constexpr int BA_CTA_THREADS = 1024;     // the one-CTA solve
constexpr int BA_COST_THREADS = 256;     // the cost reduction (_posed.block_sum)
constexpr int BA_ROW = 64;               // doubles per row: r (2), Jc (2 x 6), W (6 x 4), Y (6 x 4)
constexpr int BA_TRK = 40;               // doubles per track: X (6), X_new (6), g (4), L (16), cost (1)
constexpr int BA_CAM = 48;               // doubles per image: R (9), C (3), R_new (9), C_new (3), dcam (6)
constexpr double BA_LAMBDA0 = 1e-3, BA_ACCEPT = 0.1, BA_REJECT = 10.0, BA_LAMBDA_MAX = 1e32;
constexpr double BA_DEGENERATE_PIVOT = 1e-12;
enum { BA_IN = 0, BA_NOT_VALID = 1, BA_SAME_IMAGE = 2, BA_DEGENERATE = 3 };
enum { BA_STOP_ITERS = 0, BA_STOP_FTOL = 1, BA_STOP_LAMBDA = 2 };
enum { BA_S_COST = 0, BA_S_COST_NEW, BA_S_LAMBDA, BA_S_INIT };                       // double scalars
enum { BA_I_ITER = 0, BA_I_ACC, BA_I_STOP, BA_I_REASON, BA_I_FAIL, BA_I_M, BA_I_K, BA_I_NTRK };   // int scalars

struct BaArgs {
  const float* kpts; const int* kp_off;      // [*, 2] keypoints of image i from row kp_off[i], [n + 1]
  const float* segs; const int* seg_off;     // [*, 4] key lines, [n + 1]
  const double* K; const double* R0; const double* t0;   // input poses
  const int* hold; const int* fixed;     // [n] held centre coordinate, fixed flags
  int n_images, n_fixed, n_nodes[2], t_bound[2], max_iters;
  double ftol;
  // the tracks
  const int* n_tracks[2]; const int* track_off[2]; const int* obs[2]; const int* trk_status[2];
  const uint8_t* inlier[2]; const int* track_row[2]; const int* n_views_in[2];
  const double* X_in[2];                     // points3d [T_p, 3], lines3d [T_l, 2, 3]
  // outputs
  double* R; double* t; double* X_out[2]; int* status[2]; double* residual[2];
  double* row_points; double* row_lines; int* n_views[2]; double* stats;
  // workspace
  double* row; double* trk; double* cam; double* A; double* rhs; double* sd;
  int* list; int* list_off; int* col; uint8_t* part; unsigned* mask; int* si;
};

__device__ __forceinline__ int ba_width(int g) { return g ? 6 : 3; }
__device__ __forceinline__ int ba_k(int g) { return g ? 4 : 3; }

// Track c of the concatenated order (point tracks, then line tracks) -> kind g and local id; -1 past the counts.
__device__ __forceinline__ int ba_split(const BaArgs& a, int c, int& id) {
  const int np = *a.n_tracks[0];
  if (c < np) { id = c; return 0; }
  id = c - np;
  return id < *a.n_tracks[1] ? 1 : -1;
}
__device__ __forceinline__ double* ba_trk(const BaArgs& a, int g, int id) {
  return a.trk + (size_t)BA_TRK * (g ? a.t_bound[0] + id : id);
}
__device__ __forceinline__ double* ba_rowp(const BaArgs& a, int g, int row) {
  return a.row + (size_t)BA_ROW * (g ? a.n_nodes[0] + row : row);
}
__device__ __forceinline__ int ba_image(const BaArgs& a, int g, int row) {
  return rc_segment(g ? a.seg_off : a.kp_off, a.n_images, row);
}

// A row's observation: fx fy cx cy, then (x - cx, y - cy) of a keypoint or the pixel line normal of a key line.
struct BaObs { double fx, fy, cx, cy, ob[3]; };

__device__ __forceinline__ BaObs ba_obs(const BaArgs& a, int g, int row, int img) {
  BaObs o;
  const double* Kv = a.K + 9 * img;
  o.fx = Kv[0]; o.fy = Kv[4]; o.cx = Kv[2]; o.cy = Kv[5];
  if (g) {
    const double c[4] = {o.fx, o.fy, o.cx, o.cy};
    rc_line_normal(c, reinterpret_cast<const float4*>(a.segs)[row], o.ob);
  } else {
    const float2 q = reinterpret_cast<const float2*>(a.kpts)[row];
    o.ob[0] = RC_S((double)q.x, o.cx);
    o.ob[1] = RC_S((double)q.y, o.cy);
    o.ob[2] = 0.0;
  }
  return o;
}

// The in-plane basis u1, u2 of a line's end points X [6].
__device__ __forceinline__ void ba_basis(const double* X, double* u1, double* u2) {
  double d[3], e[3] = {0.0, 0.0, 0.0}, v[3];
  for (int k = 0; k < 3; ++k) d[k] = RC_S(X[3 + k], X[k]);
  int k = 0;
  if (fabs(d[1]) < fabs(d[k])) k = 1;
  if (fabs(d[2]) < fabs(d[k])) k = 2;
  e[k] = 1.0;
  rc_cross3(d, e, v);
  const double nv = __dsqrt_rn(rc_dot3(v, v));
  for (int j = 0; j < 3; ++j) u1[j] = RC_D(v[j], nv);
  rc_cross3(d, u1, v);
  const double nw = __dsqrt_rn(rc_dot3(v, v));
  for (int j = 0; j < 3; ++j) u2[j] = RC_D(v[j], nw);
}

// Camera Jacobian (w, C) and world Jacobian of a residual with dr/dP = gp.
__device__ __forceinline__ void ba_jac(const double* R, const double* P, const double* gp, double* Jc, double* gX) {
  for (int k = 0; k < 3; ++k) gX[k] = RC_A(RC_A(RC_M(R[k], gp[0]), RC_M(R[3 + k], gp[1])), RC_M(R[6 + k], gp[2]));
  double c[3];
  rc_cross3(P, gp, c);
  for (int k = 0; k < 3; ++k) {
    Jc[k] = RC_M(2.0, c[k]);
    Jc[3 + k] = -gX[k];
  }
}

// One row's two residuals r, camera Jacobians Jc [2][6] and landmark Jacobians Jl [2][4] at camera (R, C) and world
// point(s) X; returns whether every depth is > 0.  u1 / u2: the line's basis.
__device__ __forceinline__ bool ba_terms(const double* R, const double* C, const BaObs& o, int g, const double* X,
                                         const double* u1, const double* u2, double* r, double (*Jc)[6],
                                         double (*Jl)[4]) {
  bool front = true;
  for (int e = 0; e < (g ? 2 : 1); ++e) {
    double D[3], P[3];
    for (int k = 0; k < 3; ++k) D[k] = RC_S(X[3 * e + k], C[k]);
    rc_mv3(R, D, P);
    front = front && P[2] > 0.0;
    if (g) {
      const double rr = RC_D(rc_dot3(o.ob, P), P[2]);
      const double gp[3] = {RC_D(o.ob[0], P[2]), RC_D(o.ob[1], P[2]), RC_D(RC_S(o.ob[2], rr), P[2])};
      double gX[3];
      ba_jac(R, P, gp, Jc[e], gX);
      r[e] = rr;
      const double ja = rc_dot3(gX, u1), jb = rc_dot3(gX, u2);
      Jl[e][0] = e ? 0.0 : ja;
      Jl[e][1] = e ? 0.0 : jb;
      Jl[e][2] = e ? ja : 0.0;
      Jl[e][3] = e ? jb : 0.0;
    } else {
      const double rx = RC_D(RC_S(RC_M(o.fx, P[0]), RC_M(o.ob[0], P[2])), P[2]);
      const double ry = RC_D(RC_S(RC_M(o.fy, P[1]), RC_M(o.ob[1], P[2])), P[2]);
      const double gx[3] = {RC_D(o.fx, P[2]), 0.0, RC_D(-RC_A(o.ob[0], rx), P[2])};
      const double gy[3] = {0.0, RC_D(o.fy, P[2]), RC_D(-RC_A(o.ob[1], ry), P[2])};
      ba_jac(R, P, gx, Jc[0], Jl[0]);
      ba_jac(R, P, gy, Jc[1], Jl[1]);
      r[0] = rx;
      r[1] = ry;
    }
  }
  return front;
}

// Cholesky of the k x k block V (row-major 4 x 4 storage) into L; false unless every pivot d_c > rel V_cc.
__device__ __forceinline__ bool ba_chol(const double* V, int k, double rel, double* L) {
  bool ok = true;
  for (int c = 0; c < k; ++c) {
    double d = V[5 * c];
    for (int p = 0; p < c; ++p) d = RC_S(d, RC_M(L[4 * c + p], L[4 * c + p]));
    ok = ok && d > RC_M(rel, V[5 * c]);
    L[5 * c] = d > 0.0 ? __dsqrt_rn(d) : __longlong_as_double(0x7ff8000000000000ll);
    for (int r = c + 1; r < k; ++r) {
      double s = V[4 * r + c];
      for (int p = 0; p < c; ++p) s = RC_S(s, RC_M(L[4 * r + p], L[4 * c + p]));
      L[4 * r + c] = RC_D(s, L[5 * c]);
    }
  }
  return ok;
}

__device__ __forceinline__ void ba_cholsolve(const double* L, int k, const double* b, double* x) {
  double y[4];
  for (int c = 0; c < k; ++c) {
    double s = b[c];
    for (int p = 0; p < c; ++p) s = RC_S(s, RC_M(L[4 * c + p], y[p]));
    y[c] = RC_D(s, L[5 * c]);
  }
  for (int c = k - 1; c >= 0; --c) {
    double s = y[c];
    for (int p = c + 1; p < k; ++p) s = RC_S(s, RC_M(L[4 * p + c], x[p]));
    x[c] = RC_D(s, L[5 * c]);
  }
}

// The participating rows of track id of kind g, in observation order: calls f(row) for each inlier row.
template <class F>
__device__ __forceinline__ void ba_rows(const BaArgs& a, int g, int id, F&& f) {
  const int o0 = a.track_off[g][id], o1 = a.track_off[g][id + 1];
  for (int o = o0; o < o1; ++o) {
    const int row = a.obs[g][o];
    if (a.inlier[g][row]) f(row);
  }
}

// Landmark block V and gradient of a track at cameras cam (offset co: current or candidate) and world point(s) X;
// optionally stores each row's terms.  Returns the cost sum r^2 over its rows and whether every depth is > 0.
__device__ __forceinline__ double ba_track_terms(const BaArgs& a, int g, int id, int co, const double* X, double* V,
                                                 double* gr, bool store, bool& front) {
  double u1[3] = {0, 0, 0}, u2[3] = {0, 0, 0};
  if (g) ba_basis(X, u1, u2);
  const int k = ba_k(g);
  for (int e = 0; e < 16; ++e) V[e] = 0.0;
  for (int e = 0; e < 4; ++e) gr[e] = 0.0;
  double cost = 0.0;
  front = true;
  ba_rows(a, g, id, [&](int row) {
    const int img = ba_image(a, g, row);
    const BaObs o = ba_obs(a, g, row, img);
    const double* cm = a.cam + (size_t)BA_CAM * img + co;
    double r[2], Jc[2][6], Jl[2][4];
    front = ba_terms(cm, cm + 9, o, g, X, u1, u2, r, Jc, Jl) && front;
    for (int q = 0; q < 2; ++q) {
      for (int x = 0; x < k; ++x) {
        for (int y = x; y < k; ++y) V[4 * x + y] = RC_A(V[4 * x + y], RC_M(Jl[q][x], Jl[q][y]));
        gr[x] = RC_A(gr[x], RC_M(Jl[q][x], r[q]));
      }
      cost = RC_A(cost, RC_M(r[q], r[q]));
    }
    if (store) {
      double* rp = ba_rowp(a, g, row);
      rp[0] = r[0];
      rp[1] = r[1];
      for (int q = 0; q < 2; ++q)
        for (int x = 0; x < 6; ++x) rp[2 + 6 * q + x] = Jc[q][x];
      for (int x = 0; x < 6; ++x)
        for (int y = 0; y < k; ++y) rp[14 + 4 * x + y] = RC_A(RC_M(Jc[0][x], Jl[0][y]), RC_M(Jc[1][x], Jl[1][y]));
    }
  });
  for (int x = 0; x < k; ++x)
    for (int y = 0; y < x; ++y) V[4 * x + y] = V[4 * y + x];
  return cost;
}

__device__ __forceinline__ bool ba_stopped(const BaArgs& a) { return *(volatile int*)(a.si + BA_I_STOP) != 0; }

// The block-sum of the per-track costs (slot 32 of each track) in the concatenated track order.
__device__ __forceinline__ double ba_cost_sum(const BaArgs& a, int slot) {
  __shared__ double s_w[BA_COST_THREADS / 32];
  const int tid = threadIdx.x;
  const int total = *a.n_tracks[0] + *a.n_tracks[1];
  double acc = 0.0;
  for (int c = tid; c < total; c += BA_COST_THREADS) {
    int id;
    const int g = ba_split(a, c, id);
    acc = RC_A(acc, ba_trk(a, g, id)[slot]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc = RC_A(acc, __shfl_xor_sync(0xffffffffu, acc, o));
  if ((tid & 31) == 0) s_w[tid >> 5] = acc;
  __syncthreads();
  double out = 0.0;
  for (int w = 0; w < BA_COST_THREADS / 32; ++w) out = RC_A(out, s_w[w]);
  __syncthreads();
  return out;
}

__global__ void __launch_bounds__(BA_COST_THREADS) ba_start_kernel(const BaArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = threadIdx.x;
  if (i < a.n_images) {
    double* cm = a.cam + (size_t)BA_CAM * i;
    const double* R = a.R0 + 9 * i;
    const double* t = a.t0 + 3 * i;
    for (int e = 0; e < 9; ++e) cm[e] = R[e];
    rc_centre(R, t, cm + 9);
    for (int e = 24; e < 30; ++e) cm[e] = 0.0;
    a.part[i] = 0;
  }
  if (i < 8) a.si[i] = 0;
}

__global__ void __launch_bounds__(BA_THREADS) ba_init_kernel(const BaArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const int total = *a.n_tracks[0] + *a.n_tracks[1];
  for (int c = blockIdx.x * BA_THREADS + threadIdx.x; c < total; c += gridDim.x * BA_THREADS) {
    int id;
    const int g = ba_split(a, c, id);
    double* tr = ba_trk(a, g, id);
    unsigned* mk = a.mask + 4 * (size_t)c;
    for (int w = 0; w < 4; ++w) mk[w] = 0u;
    tr[32] = 0.0;
    int st = BA_NOT_VALID;
    if (a.trk_status[g][id] == TRK_OK) {
      st = BA_IN;
      int prev = -1;
      ba_rows(a, g, id, [&](int row) {
        const int img = ba_image(a, g, row);
        if (img == prev) st = BA_SAME_IMAGE;
        prev = img;
      });
    }
    if (st == BA_IN) {
      const int w = ba_width(g);
      for (int e = 0; e < w; ++e) tr[e] = a.X_in[g][(size_t)w * id + e];
      double V[16], gr[4], L[16];
      bool front;
      const double cost = ba_track_terms(a, g, id, 0, tr, V, gr, false, front);
      if (!ba_chol(V, ba_k(g), BA_DEGENERATE_PIVOT, L)) {
        st = BA_DEGENERATE;
      } else {
        tr[32] = cost;
        ba_rows(a, g, id, [&](int row) {
          const int img = ba_image(a, g, row);
          mk[img >> 5] |= 1u << (img & 31);
          a.part[img] = 1;
        });
        atomicAdd(a.si + BA_I_NTRK, 1);
      }
    }
    a.status[g][id] = st;
  }
}

__global__ void __launch_bounds__(BA_COST_THREADS) ba_setup_kernel(const BaArgs a) {
  __shared__ int s_cnt[BA_MAX_IMAGES];
  pdl_launch_dependents();
  pdl_wait();
  const int tid = threadIdx.x, n = a.n_images;
  const int total = *a.n_tracks[0] + *a.n_tracks[1];
  if (tid == 0) {
    int m = 0, kimg = -1;
    for (int i = 0; i < n; ++i) {
      const bool sys = !a.fixed[i] && a.part[i];
      if (sys && kimg < 0 && a.n_fixed == 1) kimg = i;
      for (int e = 0; e < 6; ++e) {
        const bool held = i == kimg && e == 3 + a.hold[i];
        a.col[6 * i + e] = sys && !held ? m++ : -1;
      }
    }
    a.si[BA_I_M] = m;
    a.si[BA_I_K] = kimg;
  }
  // per-image lists of (track, row), ascending by track
  if (tid < n) {
    int cnt = 0;
    for (int c = 0; c < total; ++c) cnt += (a.mask[4 * (size_t)c + (tid >> 5)] >> (tid & 31)) & 1u;
    s_cnt[tid] = cnt;
  }
  __syncthreads();
  if (tid == 0) {
    int s = 0;
    for (int i = 0; i < n; ++i) {
      a.list_off[i] = s;
      s += s_cnt[i];
    }
    a.list_off[n] = s;
  }
  __syncthreads();
  if (tid < n) {
    int pos = a.list_off[tid];
    for (int c = 0; c < total; ++c) {
      if (!((a.mask[4 * (size_t)c + (tid >> 5)] >> (tid & 31)) & 1u)) continue;
      int id;
      const int g = ba_split(a, c, id);
      int hit = -1;
      ba_rows(a, g, id, [&](int row) {
        if (ba_image(a, g, row) == tid) hit = row;
      });
      a.list[2 * pos] = c;
      a.list[2 * pos + 1] = g ? a.n_nodes[0] + hit : hit;
      ++pos;
    }
  }
  const double cost = ba_cost_sum(a, 32);
  if (tid == 0) {
    a.sd[BA_S_COST] = cost;
    a.sd[BA_S_INIT] = cost;
    a.sd[BA_S_LAMBDA] = BA_LAMBDA0;
    if (a.max_iters == 0) a.si[BA_I_STOP] = 1;
  }
}

__global__ void __launch_bounds__(BA_THREADS) ba_track_kernel(const BaArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  if (ba_stopped(a)) return;
  const double lam = a.sd[BA_S_LAMBDA];
  const int total = *a.n_tracks[0] + *a.n_tracks[1];
  for (int c = blockIdx.x * BA_THREADS + threadIdx.x; c < total; c += gridDim.x * BA_THREADS) {
    int id;
    const int g = ba_split(a, c, id);
    if (a.status[g][id] != BA_IN) continue;
    double* tr = ba_trk(a, g, id);
    const int k = ba_k(g);
    double V[16], gr[4];
    bool front;
    ba_track_terms(a, g, id, 0, tr, V, gr, true, front);
    for (int x = 0; x < k; ++x) V[5 * x] = RC_A(V[5 * x], RC_M(lam, V[5 * x]));
    double* L = tr + 16;
    if (!ba_chol(V, k, 0.0, L)) atomicExch(a.si + BA_I_FAIL, 1);
    for (int x = 0; x < k; ++x) tr[12 + x] = gr[x];
    ba_rows(a, g, id, [&](int row) {
      double* rp = ba_rowp(a, g, row);
      for (int x = 0; x < 6; ++x) ba_cholsolve(L, k, rp + 14 + 4 * x, rp + 38 + 4 * x);
    });
  }
}

// Block (I, J), I >= J, of the reduced camera matrix (threads 0..35: entry (a, b)) and, for I == J, its right-hand
// side (threads 36..41).
__global__ void __launch_bounds__(64) ba_reduce_kernel(const BaArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  if (ba_stopped(a)) return;
  const int I = blockIdx.y, J = blockIdx.x, tid = threadIdx.x;
  if (J > I || a.fixed[I] || a.fixed[J] || !a.part[I] || !a.part[J] || tid >= 42) return;
  const double lam = a.sd[BA_S_LAMBDA];
  const int ld = 6 * a.n_images;
  const int* li = a.list + 2 * a.list_off[I];
  const int ni = a.list_off[I + 1] - a.list_off[I];
  const int p = tid < 36 ? tid / 6 : tid - 36, q = tid < 36 ? tid % 6 : 0;
  auto kk = [&](int c) { return c < *a.n_tracks[0] ? 3 : 4; };
  auto dot = [&](const double* y, const double* w, int k) {
    double d = RC_M(y[0], w[0]);
    for (int e = 1; e < k; ++e) d = RC_A(d, RC_M(y[e], w[e]));
    return d;
  };
  if (I == J) {
    double s = 0.0;
    for (int e = 0; e < ni; ++e) {
      const double* rp = a.row + (size_t)BA_ROW * li[2 * e + 1];
      s = tid < 36 ? RC_A(s, RC_A(RC_M(rp[2 + p], rp[2 + q]), RC_M(rp[8 + p], rp[8 + q])))
                   : RC_A(s, RC_A(RC_M(rp[2 + p], rp[0]), RC_M(rp[8 + p], rp[1])));
    }
    if (tid < 36 && p == q) s = RC_A(s, RC_M(lam, s));
    for (int e = 0; e < ni; ++e) {
      const int c = li[2 * e];
      const double* rp = a.row + (size_t)BA_ROW * li[2 * e + 1];
      if (tid < 36) {
        s = RC_S(s, dot(rp + 38 + 4 * p, rp + 14 + 4 * q, kk(c)));
      } else {
        int id;
        const int g = ba_split(a, c, id);
        s = RC_S(s, dot(rp + 38 + 4 * p, ba_trk(a, g, id) + 12, kk(c)));
      }
    }
    const int cp = a.col[6 * I + p];
    if (cp < 0) return;
    if (tid < 36) {
      const int cq = a.col[6 * I + q];
      if (cq >= 0 && cp >= cq) a.A[(size_t)ld * cp + cq] = s;
    } else {
      a.rhs[cp] = -s;
    }
    return;
  }
  if (tid >= 36) return;
  const int* lj = a.list + 2 * a.list_off[J];
  const int nj = a.list_off[J + 1] - a.list_off[J];
  double s = 0.0;
  for (int x = 0, y = 0; x < ni && y < nj;) {
    const int cx = li[2 * x], cy = lj[2 * y];
    if (cx < cy) { ++x; continue; }
    if (cy < cx) { ++y; continue; }
    const double* ri = a.row + (size_t)BA_ROW * li[2 * x + 1];
    const double* rj = a.row + (size_t)BA_ROW * lj[2 * y + 1];
    s = RC_S(s, dot(ri + 38 + 4 * p, rj + 14 + 4 * q, kk(cx)));
    ++x;
    ++y;
  }
  const int cp = a.col[6 * I + p], cq = a.col[6 * J + q];
  if (cp >= 0 && cq >= 0) a.A[(size_t)ld * cp + cq] = s;
}

__global__ void __launch_bounds__(BA_CTA_THREADS) ba_solve_kernel(const BaArgs a) {
  __shared__ int s_fail;
  __shared__ double s_col[6 * BA_MAX_IMAGES];
  pdl_launch_dependents();
  pdl_wait();
  if (ba_stopped(a)) return;
  const int tid = threadIdx.x, m = a.si[BA_I_M];
  double* x = a.rhs;
  // a failed landmark factorization already rejects the step: the camera step is then zero, as on the host
  if (tid == 0) s_fail = a.si[BA_I_FAIL] != 0;
  __syncthreads();
  const bool fail = rc_cholesky_solve<BA_CTA_THREADS>(a.A, 6 * a.n_images, m, x, 1, s_col, &s_fail);
  if (fail && tid == 0) atomicExch(a.si + BA_I_FAIL, 1);
  // candidate cameras
  if (tid < a.n_images) {
    double* cm = a.cam + (size_t)BA_CAM * tid;
    double w[6];
    for (int e = 0; e < 6; ++e) {
      const int cc = a.col[6 * tid + e];
      w[e] = cc >= 0 && !fail ? x[cc] : 0.0;
      cm[24 + e] = w[e];
    }
    if (a.col[6 * tid] >= 0) {
      double Q[9];
      rc_cayley(w, Q);
      for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 3; ++k)
          cm[12 + 3 * i + k] =
              RC_A(RC_A(RC_M(Q[3 * i], cm[k]), RC_M(Q[3 * i + 1], cm[3 + k])), RC_M(Q[3 * i + 2], cm[6 + k]));
      for (int k = 0; k < 3; ++k) cm[21 + k] = RC_A(cm[9 + k], w[3 + k]);
    } else {
      for (int e = 0; e < 12; ++e) cm[12 + e] = cm[e];
    }
  }
}

__global__ void __launch_bounds__(BA_THREADS) ba_update_kernel(const BaArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  if (ba_stopped(a)) return;
  const int total = *a.n_tracks[0] + *a.n_tracks[1];
  for (int c = blockIdx.x * BA_THREADS + threadIdx.x; c < total; c += gridDim.x * BA_THREADS) {
    int id;
    const int g = ba_split(a, c, id);
    double* tr = ba_trk(a, g, id);
    tr[32] = 0.0;
    if (a.status[g][id] != BA_IN) continue;
    const int k = ba_k(g);
    double s[4];
    for (int x = 0; x < k; ++x) s[x] = tr[12 + x];
    ba_rows(a, g, id, [&](int row) {
      const double* rp = ba_rowp(a, g, row);
      const double* dc = a.cam + (size_t)BA_CAM * ba_image(a, g, row) + 24;
      for (int x = 0; x < k; ++x) {
        double dd = RC_M(rp[14 + x], dc[0]);
        for (int y = 1; y < 6; ++y) dd = RC_A(dd, RC_M(rp[14 + 4 * y + x], dc[y]));
        s[x] = RC_A(s[x], dd);
      }
    });
    double dl[4];
    ba_cholsolve(tr + 16, k, s, dl);
    for (int x = 0; x < k; ++x) dl[x] = -dl[x];
    double* Xn = tr + 6;
    if (g) {
      double u1[3], u2[3];
      ba_basis(tr, u1, u2);
      for (int e = 0; e < 3; ++e) {
        Xn[e] = RC_A(tr[e], RC_A(RC_M(u1[e], dl[0]), RC_M(u2[e], dl[1])));
        Xn[3 + e] = RC_A(tr[3 + e], RC_A(RC_M(u1[e], dl[2]), RC_M(u2[e], dl[3])));
      }
    } else {
      for (int e = 0; e < 3; ++e) Xn[e] = RC_A(tr[e], dl[e]);
    }
    double V[16], gr[4];
    bool front;
    tr[32] = ba_track_terms(a, g, id, 12, Xn, V, gr, false, front);
    if (!front) atomicExch(a.si + BA_I_FAIL, 1);
  }
}

__global__ void __launch_bounds__(BA_COST_THREADS) ba_accept_kernel(const BaArgs a) {
  __shared__ int s_acc;
  pdl_launch_dependents();
  pdl_wait();
  if (ba_stopped(a)) return;
  const int tid = threadIdx.x;
  const double cnew = ba_cost_sum(a, 32);
  if (tid == 0) {
    const double cost = a.sd[BA_S_COST];
    double lam = a.sd[BA_S_LAMBDA];
    const int it = a.si[BA_I_ITER] + 1;
    a.si[BA_I_ITER] = it;
    const bool acc = !a.si[BA_I_FAIL] && cnew < cost;
    int stop = 0;
    if (acc) {
      const double rel = RC_D(RC_S(cost, cnew), cost);
      a.sd[BA_S_COST] = cnew;
      lam = RC_M(lam, BA_ACCEPT);
      a.si[BA_I_ACC] += 1;
      if (rel <= a.ftol) {
        stop = 1;
        a.si[BA_I_REASON] = BA_STOP_FTOL;
      }
    } else {
      lam = RC_M(lam, BA_REJECT);
      if (lam > BA_LAMBDA_MAX) {
        stop = 1;
        a.si[BA_I_REASON] = BA_STOP_LAMBDA;
      }
    }
    if (it >= a.max_iters) stop = 1;
    a.sd[BA_S_LAMBDA] = lam;
    a.si[BA_I_FAIL] = 0;
    if (stop) a.si[BA_I_STOP] = 1;
    s_acc = acc;
  }
  __syncthreads();
  if (!s_acc) return;
  for (int i = tid; i < a.n_images; i += BA_COST_THREADS) {
    double* cm = a.cam + (size_t)BA_CAM * i;
    for (int e = 0; e < 12; ++e) cm[e] = cm[12 + e];
  }
  const int total = *a.n_tracks[0] + *a.n_tracks[1];
  for (int c = tid; c < total; c += BA_COST_THREADS) {
    int id;
    const int g = ba_split(a, c, id);
    if (a.status[g][id] != BA_IN) continue;
    double* tr = ba_trk(a, g, id);
    for (int e = 0; e < 6; ++e) tr[e] = tr[6 + e];
  }
}

// The output pose of image i: the state if it moved, else the input bits.
__device__ __forceinline__ void ba_pose(const BaArgs& a, int i, double* R, double* t) {
  const double* cm = a.cam + (size_t)BA_CAM * i;
  if (a.col[6 * i] >= 0 && a.si[BA_I_ACC] > 0) {
    for (int e = 0; e < 9; ++e) R[e] = cm[e];
    for (int e = 0; e < 3; ++e) t[e] = -rc_dot3(cm + 3 * e, cm + 9);
  } else {
    for (int e = 0; e < 9; ++e) R[e] = a.R0[9 * i + e];
    for (int e = 0; e < 3; ++e) t[e] = a.t0[3 * i + e];
  }
}

__global__ void __launch_bounds__(BA_THREADS) ba_finish_kernel(const BaArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  const int gtid = blockIdx.x * BA_THREADS + threadIdx.x, stride = gridDim.x * BA_THREADS;
  if (gtid < a.n_images) {
    double R[9], t[3];
    ba_pose(a, gtid, R, t);
    for (int e = 0; e < 9; ++e) a.R[9 * gtid + e] = R[e];
    for (int e = 0; e < 3; ++e) a.t[3 * gtid + e] = t[e];
  }
  if (gtid == 0) {
    const double st[8] = {a.sd[BA_S_INIT], a.sd[BA_S_COST], a.sd[BA_S_LAMBDA], (double)a.si[BA_I_ITER],
                          (double)a.si[BA_I_ACC], (double)a.si[BA_I_REASON], (double)a.list_off[a.n_images],
                          (double)a.si[BA_I_NTRK]};
    for (int e = 0; e < 8; ++e) a.stats[e] = st[e];
  }
  const int total = *a.n_tracks[0] + *a.n_tracks[1];
  for (int c = gtid; c < total; c += stride) {
    int id;
    const int g = ba_split(a, c, id);
    const int w = ba_width(g);
    const bool in = a.status[g][id] == BA_IN;
    for (int e = 0; e < w; ++e) a.X_out[g][(size_t)w * id + e] = in ? ba_trk(a, g, id)[e] : a.X_in[g][(size_t)w * id + e];
  }
  const int rows = a.n_nodes[0] + a.n_nodes[1];
  for (int x = gtid; x < rows; x += stride) {
    const int g = x >= a.n_nodes[0], row = g ? x - a.n_nodes[0] : x;
    const int id = a.track_row[g][row];
    a.n_views[g][row] = a.n_views_in[g][row];
    const bool inl = id >= 0 && a.inlier[g][row];
    double res = nan;
    if (inl && a.status[g][id] == BA_IN) {
      const double* X = ba_trk(a, g, id);
      double u1[3] = {0, 0, 0}, u2[3] = {0, 0, 0};
      if (g) ba_basis(X, u1, u2);
      const int img = ba_image(a, g, row);
      const BaObs o = ba_obs(a, g, row, img);
      const double* cm = a.cam + (size_t)BA_CAM * img;
      double r[2], Jc[2][6], Jl[2][4];
      ba_terms(cm, cm + 9, o, g, X, u1, u2, r, Jc, Jl);
      res = g ? fmax(fabs(r[0]), fabs(r[1])) : __dsqrt_rn(RC_A(RC_M(r[0], r[0]), RC_M(r[1], r[1])));
    }
    a.residual[g][row] = res;
    const bool ok = inl && a.trk_status[g][id] == TRK_OK;
    if (!g) {
      const double* Xp = ok && a.status[0][id] == BA_IN ? ba_trk(a, 0, id) : a.X_in[0] + 3ll * (ok ? id : 0);
      for (int e = 0; e < 3; ++e) a.row_points[3ll * row + e] = ok ? Xp[e] : nan;
      continue;
    }
    if (!ok) {
      for (int e = 0; e < 6; ++e) a.row_lines[6ll * row + e] = nan;
      continue;
    }
    const double* Xf = a.status[1][id] == BA_IN ? ba_trk(a, 1, id) : a.X_in[1] + 6ll * id;
    const int img = ba_image(a, 1, row);
    double R[9], t[3], C[3], d[3], w[3];
    ba_pose(a, img, R, t);
    rc_centre(R, t, C);
    for (int k = 0; k < 3; ++k) {
      d[k] = RC_S(Xf[3 + k], Xf[k]);
      w[k] = RC_S(Xf[k], C[k]);
    }
    const double* Kv = a.K + 9 * img;
    const float4 s = reinterpret_cast<const float4*>(a.segs)[row];
    for (int e = 0; e < 2; ++e) {
      double rr[3];
      rc_ray(R, Kv[0], Kv[4], Kv[2], Kv[5], e ? s.z : s.x, e ? s.w : s.y, rr);
      rc_closest_on_line(Xf, d, w, rr, a.row_lines + 6ll * row + 3 * e);
    }
  }
}

}  // namespace ltr
