// Global poses of an unposed image set (ltr_global_poses): one world -> camera pose per image from the relative poses
// of its pairs, by rotation averaging and BATA camera positions.
//
// Model (DESIGN.md "Global poses"; restated in numpy by linetr_b200.global_poses.global_poses_host), with cayinv(Q) =
// vee(Q - Q^T) / (1 + tr Q) (|cayinv| = +inf where 1 + tr Q <= 0):
//   graph: usable edges (valid, n_cheirality >= min_inliers); the largest component (ties: the lowest image) is
//   registered, the anchor defaults to its lowest image; an explicit anchor registers its own component.
//   loop support: per usable edge (i, j), the images k whose triangle |cayinv(R_ij^T R_kj R_ik)| <= tan(rot / 2).
//   rotations: Prim's maximum spanning tree from the anchor on (support, n_cheirality, -p), chained; IRLS on
//   r_p = cayinv(R_j^T R_p R_i) - (w_j - w_i), R_k <- R_k cay(w_k): GP_L1_ITERS L1 steps, then Geman-McClure steps
//   accepted iff the cost falls, until a relative decrease <= ftol, a rejection or rot_iters.
//   rigidity: drop images with < 2 rotation-inlier edges to kept images or all edge directions parallel to the first
//   (never the anchor, never below three images), then keep those connected to the anchor.
//   positions (BATA): C_anchor = 0, sum <dC_p, v_p> = E, v_p = -R_j^T t_p; C by one factorization and six right-hand
//   sides, s_p = max(<dC_p, v_p>, 0) / |dC_p|^2, Geman-McClure weights; stops as the rotations with pos_iters.
//   Every operation is explicitly rounded fp64, every sum in a fixed order: a Laplacian row over the image's edges in
//   ascending pair index, the other reductions as _posed.block_sum over GP_THREADS threads.
//
// Kernels (PDL-chained):
//   gp_graph_kernel    one CTA: the n x n edge table, the components, the registered component and the anchor.
//   gp_support_kernel  one CTA per pair, one thread per third image: the loop support.
//   gp_solve_kernel    one persistent CTA of GP_THREADS: the tree, the rotation IRLS, the rigidity pruning, BATA and
//                      the outputs.  The normal matrix (at most 127 x 127) lives in shared memory.
#pragma once
#include "common.cuh"
#include "rn_fp64.cuh"

namespace ltr {

constexpr int GP_MAX_IMAGES = 128;       // LTR_GP_MAX_IMAGES
constexpr int GP_THREADS = 1024;
constexpr int GP_L1_ITERS = 5;
constexpr double GP_L1_EPS = 1e-9;
constexpr double GP_SIGMA_ROT = 0.04366094290851206;     // tan(2.5 deg)
constexpr double GP_SIGMA_POS = 0.1;
constexpr double GP_PARALLEL_SIN = 0.03489949670250097;  // sin(2 deg)
enum { GP_EDGE_UNUSED = 0, GP_EDGE_OUTSIDE, GP_EDGE_ROT_OUTLIER, GP_EDGE_DIR_OUTLIER, GP_EDGE_INLIER };
constexpr int GP_EDGE = 16;              // doubles per edge: c (3), res, c' (3), res', wt, v (3), s, w, s', w'
constexpr int GP_CAM = 24;               // doubles per image: R (9), R' (9), C (3), C' (3)
// shared memory of gp_solve_kernel: A [m, m], x [m, 6], a [m, 3], s_col [m]
inline size_t gp_smem_bytes(int n) {
  const size_t m = n > 1 ? n - 1 : 1;
  return 8 * (m * m + 10 * m);
}

struct GpArgs {
  const int* pairs; const double* Rp; const double* tp; const uint8_t* valid; const int* ncheir;
  int n, P, min_inliers, anchor_in, rot_iters, pos_iters;
  double rot_tan, dir_cos, ftol;
  double* R; double* t; uint8_t* registered; int* status; int* support; double* rot_res; double* dcos; double* stats;
  // workspace
  double* edge; double* cam;
  int* table; int* inc; int* deg; int* comp; int* si;
};
enum { GP_I_ANCHOR = 0, GP_I_NCOMP, GP_I_LABEL };

__device__ __forceinline__ bool gp_usable(const GpArgs& a, int p) {
  return a.valid[p] != 0 && a.ncheir[p] >= a.min_inliers;
}

// A B of row-major rotations, each entry rc_dot3 of a row and a column (global_poses._mm)
__device__ __forceinline__ void gp_mm(const double* A, const double* B, double* O) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      O[3 * r + c] = RC_A(RC_A(RC_M(A[3 * r], B[c]), RC_M(A[3 * r + 1], B[3 + c])), RC_M(A[3 * r + 2], B[6 + c]));
}

__device__ __forceinline__ void gp_transpose(const double* A, double* O) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) O[3 * r + c] = A[3 * c + r];
}

// The rotation of edge e from image i to its other image: R_e, or R_e^T when i is its side 1.
__device__ __forceinline__ void gp_rel(const GpArgs& a, int e, int i, double* O) {
  const double* Re = a.Rp + 9 * (size_t)e;
  if (a.pairs[2 * e] == i) {
    for (int k = 0; k < 9; ++k) O[k] = Re[k];
  } else {
    gp_transpose(Re, O);
  }
}

// cayinv(A^T (B C)) -> c, and |c| (+inf with c = 0 where 1 + tr <= 0)
__device__ __forceinline__ double gp_loop(const double* A, const double* B, const double* C, double* c) {
  double M[9], At[9], Q[9];
  gp_mm(B, C, M);
  gp_transpose(A, At);
  gp_mm(At, M, Q);
  const double v[3] = {RC_S(Q[7], Q[5]), RC_S(Q[2], Q[6]), RC_S(Q[3], Q[1])};
  const double den = RC_A(RC_A(RC_A(1.0, Q[0]), Q[4]), Q[8]);
  if (!(den > 0.0)) {
    c[0] = c[1] = c[2] = 0.0;
    return __longlong_as_double(0x7ff0000000000000ll);
  }
  for (int k = 0; k < 3; ++k) c[k] = RC_D(v[k], den);
  return __dsqrt_rn(rc_dot3(c, c));
}

// Geman-McClure cost q / (s2 + q) and weight s2 / (s2 + q)^2 of a squared residual q (+inf: 1 and 0)
__device__ __forceinline__ double gp_gm(double q, double s2, double* wt) {
  if (isinf(q)) {
    *wt = 0.0;
    return 1.0;
  }
  const double d = RC_A(s2, q);
  *wt = RC_D(s2, RC_M(d, d));
  return RC_D(q, d);
}

// _posed.block_sum of one value per thread-strided row over GP_THREADS threads; every thread gets the sum.
__device__ __forceinline__ double gp_block_sum(double acc, double* s_w) {
  const int tid = threadIdx.x;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc = RC_A(acc, __shfl_xor_sync(0xffffffffu, acc, o));
  __syncthreads();
  if ((tid & 31) == 0) s_w[tid >> 5] = acc;
  __syncthreads();
  double out = 0.0;
  for (int w = 0; w < GP_THREADS / 32; ++w) out = RC_A(out, s_w[w]);
  return out;
}

// The CTA-wide sum of one integer per thread; every thread gets it.
__device__ __forceinline__ int gp_count(int v, int* s_cnt) {
  __syncthreads();
  if (threadIdx.x == 0) *s_cnt = 0;
  __syncthreads();
  if (v) atomicAdd(s_cnt, v);
  __syncthreads();
  return *s_cnt;
}

__global__ void __launch_bounds__(GP_THREADS) gp_graph_kernel(const GpArgs a) {
  __shared__ int s_label[GP_MAX_IMAGES], s_next[GP_MAX_IMAGES], s_size[GP_MAX_IMAGES];
  pdl_launch_dependents();
  pdl_wait();
  const int n = a.n, tid = threadIdx.x;
  for (int e = tid; e < n * n; e += GP_THREADS) a.table[e] = -1;
  if (tid < n) s_label[tid] = tid;
  __syncthreads();
  for (int p = tid; p < a.P; p += GP_THREADS) {
    if (!gp_usable(a, p)) continue;
    const int i = a.pairs[2 * p], j = a.pairs[2 * p + 1];
    a.table[n * i + j] = p;
    a.table[n * j + i] = p;
  }
  __syncthreads();
  // minimum-label propagation: every label ends as the lowest image of its component
  for (;;) {
    int changed = 0;
    if (tid < n) {
      int l = s_label[tid];
      for (int b = 0; b < n; ++b)
        if (a.table[n * tid + b] >= 0) l = min(l, s_label[b]);
      l = s_label[l] < l ? s_label[l] : l;
      s_next[tid] = l;
      changed = l != s_label[tid];
    }
    changed = __syncthreads_or(changed);
    if (tid < n) s_label[tid] = s_next[tid];
    __syncthreads();
    if (!changed) break;
  }
  if (tid < n) s_size[tid] = 0;
  __syncthreads();
  if (tid < n) atomicAdd(&s_size[s_label[tid]], 1);
  __syncthreads();
  if (tid == 0) {
    int best = 0;
    for (int i = 1; i < n; ++i)
      if (s_size[i] > s_size[best]) best = i;
    // an explicit anchor registers its own component (global_poses refuses one outside the largest), so the tree
    // below always reaches every image of the component from the anchor
    if (a.anchor_in >= 0) best = s_label[a.anchor_in];
    a.si[GP_I_ANCHOR] = a.anchor_in >= 0 ? a.anchor_in : best;
    a.si[GP_I_NCOMP] = s_size[best];
    a.si[GP_I_LABEL] = best;
  }
  __syncthreads();
  if (tid < n) a.comp[tid] = s_label[tid] == a.si[GP_I_LABEL];
}

// One CTA per pair, one thread per third image k.
__global__ void __launch_bounds__(GP_MAX_IMAGES) gp_support_kernel(const GpArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const int p = blockIdx.x, k = threadIdx.x, n = a.n;
  const bool use = gp_usable(a, p);
  const int i = a.pairs[2 * p], j = a.pairs[2 * p + 1];
  bool ok = false;
  if (use && k < n && k != i && k != j) {
    const int e1 = a.table[n * i + k], e2 = a.table[n * k + j];
    if (e1 >= 0 && e2 >= 0) {
      double Rik[9], Rkj[9], c[3];
      gp_rel(a, e1, i, Rik);
      gp_rel(a, e2, k, Rkj);
      ok = gp_loop(a.Rp + 9 * (size_t)p, Rkj, Rik, c) <= a.rot_tan;
    }
  }
  const int cnt = __syncthreads_count(ok);
  if (k == 0) a.support[p] = use ? cnt : -1;
}

// The residuals of every component edge at the rotations of slot `o` (0: R, 9: R') into the edge slot `eo` (0: c,
// res; 4: c', res'), and their Geman-McClure cost.
__device__ double gp_rot_residuals(const GpArgs& a, int o, int eo, double* s_w) {
  const double s2 = RC_M(GP_SIGMA_ROT, GP_SIGMA_ROT);
  double acc = 0.0;
  for (int p = threadIdx.x; p < a.P; p += GP_THREADS) {
    const int i = a.pairs[2 * p], j = a.pairs[2 * p + 1];
    if (!gp_usable(a, p) || !a.comp[i]) continue;
    double* ed = a.edge + (size_t)GP_EDGE * p;
    const double r = gp_loop(a.cam + GP_CAM * j + o, a.Rp + 9 * (size_t)p, a.cam + GP_CAM * i + o, ed + eo);
    ed[eo + 3] = r;
    double wt;
    acc = RC_A(acc, gp_gm(RC_M(r, r), s2, &wt));
  }
  return gp_block_sum(acc, s_w);
}

// The anchor-free weighted Laplacian A [m, m] of the edges with act(p) and weight wt(p), and the right-hand sides
// x [m, k] (k = 3 or 6): per image row, sums over its incident edges in ascending pair index, + on side 1, - on side 0.
template <class Act, class Wt, class Rhs>
__device__ __forceinline__ void gp_assemble(const GpArgs& a, const int* col, int m, double* A, double* x, int k,
                                            Act act, Wt wt, Rhs rhs) {
  for (int e = threadIdx.x; e < m * m; e += GP_THREADS) A[e] = 0.0;
  __syncthreads();
  const int n = a.n;
  for (int i = threadIdx.x; i < n; i += GP_THREADS) {
    const int ci = col[i];
    if (ci < 0) continue;
    double d = 0.0, b[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    const int* li = a.inc + (size_t)(n - 1 > 0 ? n - 1 : 1) * i;
    for (int q = 0; q < a.deg[i]; ++q) {
      const int p = li[q];
      if (!act(p)) continue;
      const double w = wt(p);
      d = RC_A(d, w);
      const bool side1 = a.pairs[2 * p + 1] == i;
      const int other = side1 ? a.pairs[2 * p] : a.pairs[2 * p + 1];
      if (col[other] >= 0) A[(size_t)m * ci + col[other]] = -w;
      for (int e = 0; e < k; ++e) {
        const double term = rhs(p, e);
        b[e] = side1 ? RC_A(b[e], term) : RC_S(b[e], term);
      }
    }
    A[(size_t)m * ci + ci] = d;
    for (int e = 0; e < k; ++e) x[k * ci + e] = b[e];
  }
  __syncthreads();
}

__global__ void __launch_bounds__(GP_THREADS, 1) gp_solve_kernel(const GpArgs a) {
  extern __shared__ double s_dyn[];
  __shared__ double s_w[GP_THREADS / 32];
  __shared__ int s_col[GP_MAX_IMAGES], s_col2[GP_MAX_IMAGES], s_kept[GP_MAX_IMAGES], s_reg[GP_MAX_IMAGES];
  __shared__ int s_drop[GP_MAX_IMAGES], s_intree[GP_MAX_IMAGES], s_order[GP_MAX_IMAGES], s_oedge[GP_MAX_IMAGES];
  __shared__ long long s_best[GP_MAX_IMAGES];
  __shared__ int s_bedge[GP_MAX_IMAGES], s_fail, s_u, s_m, s_m2, s_cnt;
  pdl_launch_dependents();
  pdl_wait();
  const int n = a.n, P = a.P, tid = threadIdx.x;
  const int anchor = a.si[GP_I_ANCHOR], ncomp = a.si[GP_I_NCOMP];
  const int mcap = n > 1 ? n - 1 : 1;
  double* A = s_dyn;
  double* x = A + (size_t)mcap * mcap;
  double* av = x + 6 * mcap;
  double* scol = av + 3 * mcap;
  // incidence lists of the component edges, ascending; columns
  if (tid < n) {
    int d = 0;
    if (a.comp[tid])
      for (int p = 0; p < P; ++p)
        if ((a.pairs[2 * p] == tid || a.pairs[2 * p + 1] == tid) && gp_usable(a, p)) a.inc[(size_t)mcap * tid + d++] = p;
    a.deg[tid] = d;
    s_intree[tid] = tid == anchor;
    s_best[tid] = -1;
    s_bedge[tid] = -1;
    double* cm = a.cam + GP_CAM * tid;
    for (int e = 0; e < 9; ++e) cm[e] = (e % 4 == 0) ? 1.0 : 0.0;
  }
  if (tid == 0) {
    int m = 0;
    for (int i = 0; i < n; ++i) s_col[i] = (a.comp[i] && i != anchor) ? m++ : -1;
    s_m = m;
    s_u = anchor;
  }
  __syncthreads();
  // Prim from the anchor, key (support, n_cheirality, -p)
  for (int step = 0; step + 1 < ncomp; ++step) {
    const int u = s_u;
    if (tid < n && !s_intree[tid]) {
      const int e = a.table[n * u + tid];
      if (e >= 0) {
        const long long key = ((long long)max(a.support[e], 0) << 45) | ((long long)max(a.ncheir[e], 0) << 13) |
                              (long long)(8191 - e);
        if (key > s_best[tid]) {
          s_best[tid] = key;
          s_bedge[tid] = e;
        }
      }
    }
    __syncthreads();
    if (tid == 0) {
      int b = -1;
      long long bk = -1;
      for (int i = 0; i < n; ++i)
        if (!s_intree[i] && s_best[i] > bk) { bk = s_best[i]; b = i; }
      s_intree[b] = 1;
      s_order[step] = b;
      s_oedge[step] = s_bedge[b];
      s_u = b;
    }
    __syncthreads();
  }
  if (tid == 0) {
    for (int step = 0; step + 1 < ncomp; ++step) {
      const int b = s_order[step], e = s_oedge[step];
      const int par = a.pairs[2 * e] + a.pairs[2 * e + 1] - b;
      double Rr[9];
      gp_rel(a, e, par, Rr);
      gp_mm(Rr, a.cam + GP_CAM * par, a.cam + GP_CAM * b);
    }
  }
  __syncthreads();
  // rotation IRLS
  const int m = s_m;
  const double s2r = RC_M(GP_SIGMA_ROT, GP_SIGMA_ROT);
  double cost = gp_rot_residuals(a, 0, 0, s_w);
  int it_r = 0;
  auto ce = [&](int p) { return gp_usable(a, p) && a.comp[a.pairs[2 * p]] != 0; };
  while (m > 0 && it_r < a.rot_iters) {
    const bool l1 = it_r < GP_L1_ITERS;
    for (int p = tid; p < P; p += GP_THREADS) {
      double* ed = a.edge + (size_t)GP_EDGE * p;
      double w = 0.0;
      if (ce(p)) {
        if (l1) w = RC_D(1.0, fmax(ed[3], GP_L1_EPS));
        else gp_gm(RC_M(ed[3], ed[3]), s2r, &w);
      }
      ed[8] = w;
    }
    __syncthreads();
    gp_assemble(a, s_col, m, A, x, 3, ce, [&](int p) { return a.edge[(size_t)GP_EDGE * p + 8]; },
                [&](int p, int e) {
                  // Geman-McClure steps take the gradient's exact J^T r = +-(1 + |r|^2) r; the normal matrix, and the
                  // L1 steps' gradient, keep J's leading term [-I, +I]
                  const double* ed = a.edge + (size_t)GP_EDGE * p;
                  if (l1) return RC_M(ed[8], ed[e]);
                  return isinf(ed[3]) ? 0.0 : RC_M(RC_M(ed[8], RC_A(1.0, RC_M(ed[3], ed[3]))), ed[e]);
                });
    if (tid == 0) s_fail = 0;
    __syncthreads();
    if (rc_cholesky_solve<GP_THREADS>(A, m, m, x, 3, scol, &s_fail)) break;
    if (tid < n) {
      double* cm = a.cam + GP_CAM * tid;
      if (s_col[tid] >= 0) {
        double Q[9];
        rc_cayley(x + 3 * s_col[tid], Q);
        gp_mm(cm, Q, cm + 9);
      } else {
        for (int e = 0; e < 9; ++e) cm[9 + e] = cm[e];
      }
    }
    __syncthreads();
    const double cnew = gp_rot_residuals(a, 9, 4, s_w);
    ++it_r;
    bool accept = l1 || cnew < cost, stop = !accept;
    if (accept && !l1) stop = RC_D(RC_S(cost, cnew), cost) <= a.ftol;
    if (accept) {
      cost = cnew;
      if (tid < n)
        for (int e = 0; e < 9; ++e) a.cam[GP_CAM * tid + e] = a.cam[GP_CAM * tid + 9 + e];
      for (int p = tid; p < P; p += GP_THREADS) {
        double* ed = a.edge + (size_t)GP_EDGE * p;
        for (int e = 0; e < 4; ++e) ed[e] = ed[4 + e];
      }
    }
    __syncthreads();
    if (stop) break;
  }
  // rigidity
  auto ie = [&](int p) { return ce(p) && a.edge[(size_t)GP_EDGE * p + 3] <= a.rot_tan; };
  for (int p = tid; p < P; p += GP_THREADS) {
    double* ed = a.edge + (size_t)GP_EDGE * p;
    const int j = a.pairs[2 * p + 1];
    if (ce(p)) rc_centre(a.cam + GP_CAM * j, a.tp + 3 * (size_t)p, ed + 9);
    ed[12] = 1.0;
    ed[13] = 1.0;
  }
  if (tid < n) s_kept[tid] = a.comp[tid];
  __syncthreads();
  const double sin2 = RC_M(GP_PARALLEL_SIN, GP_PARALLEL_SIN);
  for (;;) {
    const int nk = __syncthreads_count(tid < n && s_kept[tid]);
    if (nk <= 2) break;
    int drop = 0;
    if (tid < n && s_kept[tid] && tid != anchor) {
      const int* li = a.inc + (size_t)mcap * tid;
      int cnt = 0, first = -1;
      bool allpar = true;
      for (int q = 0; q < a.deg[tid]; ++q) {
        const int p = li[q];
        const int other = a.pairs[2 * p] + a.pairs[2 * p + 1] - tid;
        if (!ie(p) || !s_kept[other]) continue;
        ++cnt;
        if (first < 0) { first = p; continue; }
        const double* v0 = a.edge + (size_t)GP_EDGE * first + 9;
        const double* v = a.edge + (size_t)GP_EDGE * p + 9;
        double cr[3];
        rc_cross3(v0, v, cr);
        allpar = allpar && rc_dot3(cr, cr) <= RC_M(sin2, RC_M(rc_dot3(v0, v0), rc_dot3(v, v)));
      }
      drop = cnt < 2 || allpar;
    }
    if (tid < n) s_drop[tid] = drop;
    if (!__syncthreads_or(drop)) break;
    if (tid < n && s_drop[tid]) s_kept[tid] = 0;
    __syncthreads();
  }
  if (tid < n) s_reg[tid] = tid == anchor;
  __syncthreads();
  for (;;) {
    int grow = 0;
    if (tid < n && s_kept[tid] && !s_reg[tid]) {
      const int* li = a.inc + (size_t)mcap * tid;
      for (int q = 0; q < a.deg[tid] && !grow; ++q) {
        const int p = li[q];
        const int other = a.pairs[2 * p] + a.pairs[2 * p + 1] - tid;
        grow = ie(p) && s_kept[other] && s_reg[other];
      }
    }
    if (!__syncthreads_or(grow)) break;
    if (grow) s_reg[tid] = 1;
    __syncthreads();
  }
  if (tid == 0) {
    int m2 = 0;
    for (int i = 0; i < n; ++i) s_col2[i] = (s_reg[i] && i != anchor) ? m2++ : -1;
    s_m2 = m2;
  }
  for (int e = tid; e < 3 * n; e += GP_THREADS) a.cam[GP_CAM * (e / 3) + 18 + e % 3] = 0.0;
  __syncthreads();
  // positions (BATA)
  const int m2 = s_m2;
  auto pe = [&](int p) { return ie(p) && s_reg[a.pairs[2 * p]] && s_reg[a.pairs[2 * p + 1]]; };
  int ec = 0;
  for (int p = tid; p < P; p += GP_THREADS) ec += pe(p);
  const int ecount = gp_count(ec, &s_cnt);
  const double s2p = RC_M(GP_SIGMA_POS, GP_SIGMA_POS);
  double pcost = ecount ? __longlong_as_double(0x7ff0000000000000ll) : 0.0;
  int it_p = 0;
  while (ecount && it_p < a.pos_iters) {
    gp_assemble(a, s_col2, m2, A, x, 6, pe,
                [&](int p) { const double* ed = a.edge + (size_t)GP_EDGE * p; return RC_M(RC_M(ed[13], ed[12]), ed[12]); },
                [&](int p, int e) {
                  const double* ed = a.edge + (size_t)GP_EDGE * p;
                  return e < 3 ? RC_M(RC_M(ed[13], ed[12]), ed[9 + e]) : ed[9 + e - 3];
                });
    for (int e = tid; e < 3 * m2; e += GP_THREADS) av[e] = x[6 * (e / 3) + 3 + e % 3];
    if (tid == 0) s_fail = 0;
    __syncthreads();
    if (rc_cholesky_solve<GP_THREADS>(A, m2, m2, x, 6, scol, &s_fail)) break;
    double pb = 0.0, pa = 0.0;
    for (int r = tid; r < m2; r += GP_THREADS) {
      pb = RC_A(pb, rc_dot3(av + 3 * r, x + 6 * r));
      pa = RC_A(pa, rc_dot3(av + 3 * r, x + 6 * r + 3));
    }
    const double ab = gp_block_sum(pb, s_w);
    const double aa = gp_block_sum(pa, s_w);
    const double lam = RC_D(RC_S(ab, (double)ecount), aa);
    if (tid < n) {
      double* cm = a.cam + GP_CAM * tid;
      const int c2 = s_col2[tid];
      for (int e = 0; e < 3; ++e) cm[21 + e] = c2 >= 0 ? RC_S(x[6 * c2 + e], RC_M(lam, x[6 * c2 + 3 + e])) : 0.0;
    }
    __syncthreads();
    double acc = 0.0;
    for (int p = tid; p < P; p += GP_THREADS) {
      if (!pe(p)) continue;
      double* ed = a.edge + (size_t)GP_EDGE * p;
      const double* Ci = a.cam + GP_CAM * a.pairs[2 * p] + 21;
      const double* Cj = a.cam + GP_CAM * a.pairs[2 * p + 1] + 21;
      double dC[3], er[3];
      for (int e = 0; e < 3; ++e) dC[e] = RC_S(Cj[e], Ci[e]);
      const double dd = rc_dot3(dC, dC), dv = rc_dot3(dC, ed + 9);
      const double s = dd > 0.0 ? RC_D(dv > 0.0 ? dv : 0.0, dd) : 0.0;
      for (int e = 0; e < 3; ++e) er[e] = RC_S(RC_M(s, dC[e]), ed[9 + e]);
      double w;
      acc = RC_A(acc, gp_gm(rc_dot3(er, er), s2p, &w));
      ed[14] = s;
      ed[15] = w;
    }
    const double cnew = gp_block_sum(acc, s_w);
    ++it_p;
    const bool accept = cnew < pcost;
    const bool stop = !accept || RC_D(RC_S(pcost, cnew), pcost) <= a.ftol;
    if (accept) {
      pcost = cnew;
      if (tid < n)
        for (int e = 0; e < 3; ++e) a.cam[GP_CAM * tid + 18 + e] = a.cam[GP_CAM * tid + 21 + e];
      for (int p = tid; p < P; p += GP_THREADS) {
        double* ed = a.edge + (size_t)GP_EDGE * p;
        ed[12] = ed[14];
        ed[13] = ed[15];
      }
    }
    __syncthreads();
    if (stop) break;
  }
  // outputs
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  int inl = 0;
  for (int p = tid; p < P; p += GP_THREADS) {
    const double* ed = a.edge + (size_t)GP_EDGE * p;
    int st = GP_EDGE_UNUSED;
    double dc = nan;
    if (gp_usable(a, p)) st = GP_EDGE_OUTSIDE;
    if (ce(p) && !ie(p)) st = GP_EDGE_ROT_OUTLIER;
    if (pe(p)) {
      const double* Ci = a.cam + GP_CAM * a.pairs[2 * p] + 18;
      const double* Cj = a.cam + GP_CAM * a.pairs[2 * p + 1] + 18;
      double dC[3];
      for (int e = 0; e < 3; ++e) dC[e] = RC_S(Cj[e], Ci[e]);
      const double dv = rc_dot3(dC, ed + 9), nrm = __dsqrt_rn(rc_dot3(dC, dC));
      st = dv > RC_M(a.dir_cos, nrm) ? GP_EDGE_INLIER : GP_EDGE_DIR_OUTLIER;
      dc = RC_D(dv, nrm);
    }
    inl += st == GP_EDGE_INLIER;
    a.status[p] = st;
    a.rot_res[p] = ce(p) ? ed[3] : nan;
    a.dcos[p] = dc;
  }
  const int n_inl = gp_count(inl, &s_cnt);
  if (tid < n) {
    const double* cm = a.cam + GP_CAM * tid;
    double* Ro = a.R + 9 * tid;
    double* to = a.t + 3 * tid;
    a.registered[tid] = s_reg[tid];
    if (tid == anchor) {
      for (int e = 0; e < 9; ++e) Ro[e] = (e % 4 == 0) ? 1.0 : 0.0;
      for (int e = 0; e < 3; ++e) to[e] = 0.0;
    } else if (s_reg[tid]) {
      for (int e = 0; e < 9; ++e) Ro[e] = cm[e];
      for (int e = 0; e < 3; ++e) to[e] = -rc_dot3(cm + 3 * e, cm + 18);
    } else {
      for (int e = 0; e < 9; ++e) Ro[e] = nan;
      for (int e = 0; e < 3; ++e) to[e] = nan;
    }
  }
  const int nreg = __syncthreads_count(tid < n && s_reg[tid]);
  if (tid == 0) {
    a.stats[0] = it_r;
    a.stats[1] = cost;
    a.stats[2] = it_p;
    a.stats[3] = pcost;
    a.stats[4] = nreg;
    a.stats[5] = n_inl;
    a.stats[6] = anchor;
  }
}

}  // namespace ltr
