// RANSAC homographies from point and line matches for a batch of image pairs (ltr_homography).
//
// Model (DESIGN.md "Homography estimation"; restated in numpy by linetr_b200.geometry.ransac_homography_host):
//   correspondences of pair p: the matched side-0 keypoints in row order, then the matched side-0 key lines in row
//   order (index d < n_points: point d, else line d - n_points); per side, normalised coordinates
//   (x - c) * (1 / s) with c the midpoint of that side's bounding box (points and segment end points) and s half its
//   larger extent (1 when 0).  A point gives the two DLT rows, a line l1^T H p = 0 for both end points p of s0, l1 the
//   line through s1 with l1x^2 + l1y^2 = 1.
//   hypothesis k: 4 distinct correspondences drawn with
//       s = splitmix64(seed + splitmix64(p << 32 | k)),  draw j = splitmix64(s + j) mod n,  j = 0, 1, ...
//   a duplicate is redrawn with the next j (at most HG_MAX_DRAWS draws, then the hypothesis is rejected); the 8 rows
//   are solved with h33 = 1 by Gaussian elimination with partial pivoting (first largest |pivot|), rejected for a
//   pivot below 1e-12, a non-finite result or |H33| < 1e-12 after H = T1^-1 H^ T0.
//   residuals in pixels of image 1, fp64 with every operation explicitly rounded (no FMA contraction):
//   point |pi(H x0) - x1|^2, line max of the squared distances of pi(H a0), pi(H b0) to the line through s1; an outlier
//   where a projected |w| <= FLT_EPSILON; an inlier iff residual < thresh^2.
//   winner: most inliers, lowest k on a tie (atomicMax of (count << 32) | ~k).
//   refit: smallest eigenvector (cyclic Jacobi, fp64) of A^T A over the winner's inliers (fixed summation order),
//   kept iff its inlier count >= the hypothesis'.
//
// Kernels:
//   homography_hyp_kernel    grid (pair, chunk of HG_THREADS hypotheses): stage the pair's correspondences in shared
//                            memory (ballot + prefix compaction of the match rows), one hypothesis per thread scored
//                            against all of them, one atomicMax per CTA.
//   homography_refit_kernel  grid (pair): the winner again, A^T A, Jacobi, both inlier passes, the outputs.
#pragma once
#include "common.cuh"
#include "rn_fp64.cuh"
#include "ransac_common.cuh"

namespace ltr {

constexpr int HG_THREADS = 128;         // hypotheses per CTA
constexpr int HG_REFIT_THREADS = 256;
constexpr int HG_PT_BYTES = 16;         // shared bytes per point: x0, y0, x1, y1 fp32
constexpr int HG_LN_BYTES = 56;         // per line: s0, s1 (4 fp32 each) and the pixel line through s1 (3 fp64)
constexpr int HG_SMEM_MAX = 200 * 1024; // staging capacity of one pair (see hg_smem_bytes)
constexpr double HG_FLT_EPS = 1.1920928955078125e-07;

struct HomographyArgs {
  const float* pts0; const float* pts1;   // [*, 2] keypoint pools
  const int* pts_off0; const int* pts_off1; const int* n_pts1;
  const int* matches_p; const int* cu_p;
  const float* segs0; const float* segs1; // [*, 2, 2] segment pools
  const int* seg_off0; const int* seg_off1; const int* n_segs1;
  const int* matches_l; const int* cu_l;
  int rows_p, rows_l;                     // staging rows per pair (0 when the kind is not used)
  int use_p, use_l;
  double thresh2;
  int n_hyp;
  unsigned long long seed;
  unsigned long long* key;
  double* H; uint8_t* valid; uint8_t* inl_p; uint8_t* inl_l;
  int* n_inl_p; int* n_inl_l; int* hyp_index; int* hyp_inliers;
};

// Dynamic shared memory of one pair: points, then s0 / s1, then the pixel lines; the refit kernel adds two flag bytes
// per correspondence.
static inline long long hg_smem_bytes(long long rows_p, long long rows_l, bool refit) {
  long long b = rows_p * HG_PT_BYTES + rows_l * HG_LN_BYTES;
  if (refit) b += 2 * (rows_p + rows_l);
  return b;
}

struct HgPair {
  int np, nl;
  double c0x, c0y, i0, s0, c1x, c1y, i1, s1;   // per side: centre, 1 / scale, scale
};

struct HgStage {
  float4* pt;   // [rows_p]
  float4* a;    // [rows_l] s0
  float4* b;    // [rows_l] s1
  double* l;    // [3 * rows_l]
};

__device__ __forceinline__ HgStage hg_stage_ptrs(unsigned char* base, int rows_p, int rows_l) {
  HgStage st;
  st.pt = reinterpret_cast<float4*>(base);
  st.a = st.pt + rows_p;
  st.b = st.a + rows_l;
  st.l = reinterpret_cast<double*>(st.b + rows_l);
  return st;
}

// Stage pair p's correspondences and its normalisation.  Ends with __syncthreads.
template <int NT>
__device__ void hg_stage_pair(const HomographyArgs& a, int p, const HgStage& st, HgPair& sp, int* warp_cnt, float* red) {
  // A pair with more match rows than the staging bounds is left without correspondences (so invalid) rather than
  // written past its shared memory: the bounds come from the caller.
  if ((a.use_p && a.cu_p[p + 1] - a.cu_p[p] > a.rows_p) || (a.use_l && a.cu_l[p + 1] - a.cu_l[p] > a.rows_l)) {
    if (threadIdx.x == 0) sp.np = sp.nl = 0;
    __syncthreads();
    return;
  }
  int np = 0, nl = 0;
  if (a.rows_p) {
    const float* __restrict__ x0 = a.pts0 + 2ll * a.pts_off0[p];
    const float* __restrict__ x1 = a.pts1 + 2ll * a.pts_off1[p];
    np = hg_compact<NT>(a.matches_p, a.cu_p[p], a.cu_p[p + 1], a.n_pts1[p], warp_cnt, [&](int i, int m, int ci) {
      if (ci >= 0) st.pt[ci] = make_float4(x0[2 * i], x0[2 * i + 1], x1[2 * m], x1[2 * m + 1]);
    });
  }
  if (a.rows_l) {
    const float* __restrict__ l0 = a.segs0 + 4ll * a.seg_off0[p];
    const float* __restrict__ l1 = a.segs1 + 4ll * a.seg_off1[p];
    nl = hg_compact<NT>(a.matches_l, a.cu_l[p], a.cu_l[p + 1], a.n_segs1[p], warp_cnt, [&](int i, int m, int ci) {
      if (ci < 0) return;
      const float4 s1 = make_float4(l1[4 * m], l1[4 * m + 1], l1[4 * m + 2], l1[4 * m + 3]);
      st.a[ci] = make_float4(l0[4 * i], l0[4 * i + 1], l0[4 * i + 2], l0[4 * i + 3]);
      st.b[ci] = s1;
      const double ax = s1.x, ay = s1.y, bx = s1.z, by = s1.w;
      const double la = RC_S(ay, by), lb = RC_S(bx, ax), lc = RC_S(RC_M(ax, by), RC_M(bx, ay));
      const double r = __drcp_rn(__dsqrt_rn(RC_A(RC_M(la, la), RC_M(lb, lb))));
      st.l[3 * ci] = RC_M(la, r);
      st.l[3 * ci + 1] = RC_M(lb, r);
      st.l[3 * ci + 2] = RC_M(lc, r);
    });
  }
  // bounding boxes: min x0, min y0, -max x0, -max y0, then side 1
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = INFINITY;
  auto add = [&](float x, float y, int side) {
    v[4 * side] = fminf(v[4 * side], x);
    v[4 * side + 1] = fminf(v[4 * side + 1], y);
    v[4 * side + 2] = fminf(v[4 * side + 2], -x);
    v[4 * side + 3] = fminf(v[4 * side + 3], -y);
  };
  for (int i = threadIdx.x; i < np; i += NT) {
    const float4 q = st.pt[i];
    add(q.x, q.y, 0);
    add(q.z, q.w, 1);
  }
  for (int i = threadIdx.x; i < nl; i += NT) {
    const float4 q = st.a[i], r = st.b[i];
    add(q.x, q.y, 0);
    add(q.z, q.w, 0);
    add(r.x, r.y, 1);
    add(r.z, r.w, 1);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[j] = fminf(v[j], __shfl_xor_sync(0xffffffffu, v[j], o));
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0)
#pragma unroll
    for (int j = 0; j < 8; ++j) red[w * 8 + j] = v[j];
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < NT / 32; ++i)
      for (int j = 0; j < 8; ++j) red[j] = fminf(red[j], red[i * 8 + j]);
    double c[2][2], s[2];
    for (int side = 0; side < 2; ++side) {
      const double lx = red[4 * side], ly = red[4 * side + 1], hx = -red[4 * side + 2], hy = -red[4 * side + 3];
      c[side][0] = RC_M(RC_A(lx, hx), 0.5);
      c[side][1] = RC_M(RC_A(ly, hy), 0.5);
      const double wx = RC_S(hx, lx), wy = RC_S(hy, ly);
      double sc = RC_M(wx > wy ? wx : wy, 0.5);
      if (!(sc > 0.0)) sc = 1.0;   // one point, or no correspondence
      s[side] = sc;
    }
    sp.np = np;
    sp.nl = nl;
    sp.c0x = c[0][0]; sp.c0y = c[0][1]; sp.s0 = s[0]; sp.i0 = __drcp_rn(s[0]);
    sp.c1x = c[1][0]; sp.c1y = c[1][1]; sp.s1 = s[1]; sp.i1 = __drcp_rn(s[1]);
  }
  __syncthreads();
}

// The two equation rows of correspondence d in normalised coordinates.
__device__ __forceinline__ void hg_rows(const HgStage& st, const HgPair& sp, int d, double* r0, double* r1) {
  if (d < sp.np) {
    const float4 q = st.pt[d];
    const double x = RC_M(RC_S(q.x, sp.c0x), sp.i0), y = RC_M(RC_S(q.y, sp.c0y), sp.i0);
    const double u = RC_M(RC_S(q.z, sp.c1x), sp.i1), v = RC_M(RC_S(q.w, sp.c1y), sp.i1);
    r0[0] = x; r0[1] = y; r0[2] = 1.0; r0[3] = 0.0; r0[4] = 0.0; r0[5] = 0.0;
    r0[6] = -RC_M(u, x); r0[7] = -RC_M(u, y); r0[8] = -u;
    r1[0] = 0.0; r1[1] = 0.0; r1[2] = 0.0; r1[3] = x; r1[4] = y; r1[5] = 1.0;
    r1[6] = -RC_M(v, x); r1[7] = -RC_M(v, y); r1[8] = -v;
  } else {
    const int i = d - sp.np;
    const float4 q = st.a[i], t = st.b[i];
    const double ua = RC_M(RC_S(t.x, sp.c1x), sp.i1), va = RC_M(RC_S(t.y, sp.c1y), sp.i1);
    const double ub = RC_M(RC_S(t.z, sp.c1x), sp.i1), vb = RC_M(RC_S(t.w, sp.c1y), sp.i1);
    const double la = RC_S(va, vb), lb = RC_S(ub, ua), lc = RC_S(RC_M(ua, vb), RC_M(ub, va));
    const double r = __drcp_rn(__dsqrt_rn(RC_A(RC_M(la, la), RC_M(lb, lb))));
    const double A = RC_M(la, r), B = RC_M(lb, r), C = RC_M(lc, r);
    double* rr[2] = {r0, r1};
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const double x = RC_M(RC_S(e ? q.z : q.x, sp.c0x), sp.i0), y = RC_M(RC_S(e ? q.w : q.y, sp.c0y), sp.i0);
      double* o = rr[e];
      o[0] = RC_M(A, x); o[1] = RC_M(A, y); o[2] = A;
      o[3] = RC_M(B, x); o[4] = RC_M(B, y); o[5] = B;
      o[6] = RC_M(C, x); o[7] = RC_M(C, y); o[8] = C;
    }
  }
}

// Normalised h (9) -> pixel H = T1^-1 H^ T0 / H33; false when |H33| < 1e-12 or a result is not finite.
__device__ __forceinline__ bool hg_to_pixels(const HgPair& sp, const double* h, double* H) {
  const double t0x = -RC_M(sp.c0x, sp.i0), t0y = -RC_M(sp.c0y, sp.i0);
  double M[9];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    M[3 * i] = RC_M(h[3 * i], sp.i0);
    M[3 * i + 1] = RC_M(h[3 * i + 1], sp.i0);
    M[3 * i + 2] = RC_A(RC_A(RC_M(h[3 * i], t0x), RC_M(h[3 * i + 1], t0y)), h[3 * i + 2]);
  }
  double G[9];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    G[j] = RC_A(RC_M(sp.s1, M[j]), RC_M(sp.c1x, M[6 + j]));
    G[3 + j] = RC_A(RC_M(sp.s1, M[3 + j]), RC_M(sp.c1y, M[6 + j]));
    G[6 + j] = M[6 + j];
  }
  if (!(fabs(G[8]) >= 1e-12)) return false;
  bool fin = true;
#pragma unroll
  for (int j = 0; j < 9; ++j) {
    H[j] = __ddiv_rn(G[j], G[8]);
    fin &= isfinite(H[j]);
  }
  return fin;
}

// Hypothesis k of pair p (pixel H), or false when it is rejected.
__device__ __noinline__ bool hg_hypothesis(const HgStage& st, const HgPair& sp, unsigned long long seed, int p, int k,
                                           double* H) {
  const int n = sp.np + sp.nl;
  int idx[4];
  if (!hg_draw<4>(seed, p, k, n, idx)) return false;
  double A[8][9];
  for (int q = 0; q < 4; ++q) {
    double r0[9], r1[9];
    hg_rows(st, sp, idx[q], r0, r1);
    for (int j = 0; j < 8; ++j) {
      A[2 * q][j] = r0[j];
      A[2 * q + 1][j] = r1[j];
    }
    A[2 * q][8] = -r0[8];
    A[2 * q + 1][8] = -r1[8];
  }
  for (int c = 0; c < 8; ++c) {
    int piv = c;
    double best = fabs(A[c][c]);
    for (int r = c + 1; r < 8; ++r)
      if (fabs(A[r][c]) > best) { best = fabs(A[r][c]); piv = r; }
    if (!(best >= 1e-12)) return false;
    if (piv != c)
      for (int j = 0; j < 9; ++j) { const double t = A[c][j]; A[c][j] = A[piv][j]; A[piv][j] = t; }
    for (int r = c + 1; r < 8; ++r) {
      const double f = __ddiv_rn(A[r][c], A[c][c]);
      for (int j = c + 1; j < 9; ++j) A[r][j] = RC_S(A[r][j], RC_M(f, A[c][j]));
    }
  }
  double h[9];
  h[8] = 1.0;
  for (int i = 7; i >= 0; --i) {
    double acc = A[i][8];
    for (int j = i + 1; j < 8; ++j) acc = RC_S(acc, RC_M(A[i][j], h[j]));
    h[i] = __ddiv_rn(acc, A[i][i]);
    if (!isfinite(h[i])) return false;
  }
  return hg_to_pixels(sp, h, H);
}

__device__ __forceinline__ bool hg_project(const double* H, double x, double y, double& px, double& py) {
  const double w = RC_A(RC_A(RC_M(H[6], x), RC_M(H[7], y)), H[8]);
  if (!(fabs(w) > HG_FLT_EPS)) return false;
  const double r = __drcp_rn(w);
  px = RC_M(RC_A(RC_A(RC_M(H[0], x), RC_M(H[1], y)), H[2]), r);
  py = RC_M(RC_A(RC_A(RC_M(H[3], x), RC_M(H[4], y)), H[5]), r);
  return true;
}

__device__ __forceinline__ bool hg_inlier(const HgStage& st, const HgPair& sp, const double* H, double t2, int d) {
  if (d < sp.np) {
    const float4 q = st.pt[d];
    double px, py;
    if (!hg_project(H, q.x, q.y, px, py)) return false;
    const double dx = RC_S(px, q.z), dy = RC_S(py, q.w);
    return RC_A(RC_M(dx, dx), RC_M(dy, dy)) < t2;
  }
  const int i = d - sp.np;
  const float4 q = st.a[i];
  const double la = st.l[3 * i], lb = st.l[3 * i + 1], lc = st.l[3 * i + 2];
  double ax, ay, bx, by;
  if (!hg_project(H, q.x, q.y, ax, ay) || !hg_project(H, q.z, q.w, bx, by)) return false;
  const double da = RC_A(RC_A(RC_M(la, ax), RC_M(lb, ay)), lc), db = RC_A(RC_A(RC_M(la, bx), RC_M(lb, by)), lc);
  const double ea = RC_M(da, da), eb = RC_M(db, db);
  return (ea > eb ? ea : eb) < t2;
}

__global__ void __launch_bounds__(HG_THREADS) homography_hyp_kernel(HomographyArgs a) {
  extern __shared__ __align__(16) unsigned char hg_smem[];
  __shared__ HgPair sp;
  __shared__ int warp_cnt[HG_THREADS / 32];
  __shared__ float red[HG_THREADS / 32 * 8];
  __shared__ unsigned long long wbest[HG_THREADS / 32];
  pdl_launch_dependents();
  pdl_wait();
  const int p = blockIdx.x;
  const HgStage st = hg_stage_ptrs(hg_smem, a.rows_p, a.rows_l);
  hg_stage_pair<HG_THREADS>(a, p, st, sp, warp_cnt, red);
  const int n = sp.np + sp.nl;
  if (n < 4) return;
  const int k = blockIdx.y * HG_THREADS + threadIdx.x;
  unsigned long long key = 0;
  double H[9];
  if (k < a.n_hyp && hg_hypothesis(st, sp, a.seed, p, k, H)) {
    unsigned cnt = 0;
    for (int d = 0; d < n; ++d) cnt += hg_inlier(st, sp, H, a.thresh2, d);
    key = ((unsigned long long)cnt << 32) | (unsigned long long)(~(unsigned)k);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long t = __shfl_xor_sync(0xffffffffu, key, o);
    key = t > key ? t : key;
  }
  if ((threadIdx.x & 31) == 0) wbest[threadIdx.x >> 5] = key;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < HG_THREADS / 32; ++i) key = wbest[i] > key ? wbest[i] : key;
    if (key) atomicMax(a.key + p, key);
  }
}

// Block-wide inlier flags of H into fl; returns (point inliers, line inliers) to every thread.
template <int NT>
__device__ __forceinline__ int2 hg_mark(const HgStage& st, const HgPair& sp, const double* H, double t2, uint8_t* fl,
                                        int2* red) {
  int cp = 0, cl = 0;
  const int n = sp.np + sp.nl;
  for (int d = threadIdx.x; d < n; d += NT) {
    const bool in = hg_inlier(st, sp, H, t2, d);
    fl[d] = in;
    if (d < sp.np) cp += in; else cl += in;
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

__global__ void __launch_bounds__(HG_REFIT_THREADS) homography_refit_kernel(HomographyArgs a) {
  constexpr int NT = HG_REFIT_THREADS, NW = NT / 32;
  extern __shared__ __align__(16) unsigned char hg_smem[];
  __shared__ HgPair sp;
  __shared__ int warp_cnt[NW];
  __shared__ float red[NW * 8];
  __shared__ int2 red2[NW];
  __shared__ double ata[NW][45];
  __shared__ double sH[2][9];
  __shared__ int s_ok[2];
  pdl_launch_dependents();
  pdl_wait();
  const int p = blockIdx.x;
  const HgStage st = hg_stage_ptrs(hg_smem, a.rows_p, a.rows_l);
  hg_stage_pair<NT>(a, p, st, sp, warp_cnt, red);
  const int n = sp.np + sp.nl;
  uint8_t* flh = reinterpret_cast<uint8_t*>(st.l + 3 * a.rows_l);
  uint8_t* flr = flh + (a.rows_p + a.rows_l);
  const unsigned long long key = a.key[p];
  const int k = (int)(~(unsigned)(key & 0xffffffffull));
  if (threadIdx.x == 0) {
    s_ok[0] = n >= 4 && key != 0 && hg_hypothesis(st, sp, a.seed, p, k, sH[0]);
    s_ok[1] = 0;
  }
  __syncthreads();
  const bool valid = s_ok[0];
  int2 cnt = make_int2(0, 0);
  const uint8_t* fl = flh;
  if (valid) {
    const int2 ch = hg_mark<NT>(st, sp, sH[0], a.thresh2, flh, red2);
    cnt = ch;
    if (ch.x + ch.y >= 4) {
      // A^T A over the hypothesis' inliers: thread t sums correspondences t, t + NT, ... in order, then a fixed tree
      double acc[45];
#pragma unroll
      for (int e = 0; e < 45; ++e) acc[e] = 0.0;
      for (int d = threadIdx.x; d < n; d += NT) {
        if (!flh[d]) continue;
        double r0[9], r1[9];
        hg_rows(st, sp, d, r0, r1);
        int e = 0;
#pragma unroll
        for (int i = 0; i < 9; ++i)
#pragma unroll
          for (int j = i; j < 9; ++j, ++e) acc[e] += r0[i] * r0[j] + r1[i] * r1[j];
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
        double M[81], h[9];
        int e = 0;
        for (int i = 0; i < 9; ++i)
          for (int j = i; j < 9; ++j, ++e) {
            double v = 0.0;
            for (int w = 0; w < NW; ++w) v += ata[w][e];
            M[9 * i + j] = v;
            M[9 * j + i] = v;
          }
        hg_smallest_eigvec(M, h);
        s_ok[1] = hg_to_pixels(sp, h, sH[1]);
      }
      __syncthreads();
      if (s_ok[1]) {
        const int2 cr = hg_mark<NT>(st, sp, sH[1], a.thresh2, flr, red2);
        if (cr.x + cr.y >= ch.x + ch.y) {
          cnt = cr;
          fl = flr;
        } else if (threadIdx.x == 0) {
          s_ok[1] = 0;
        }
      }
    }
  }
  __syncthreads();
  if (threadIdx.x < 9) a.H[9ll * p + threadIdx.x] = valid ? sH[s_ok[1]][threadIdx.x] : __longlong_as_double(0x7ff8000000000000ll);
  if (threadIdx.x == 0) {
    a.valid[p] = valid;
    a.n_inl_p[p] = cnt.x;
    a.n_inl_l[p] = cnt.y;
    a.hyp_index[p] = valid ? k : -1;
    a.hyp_inliers[p] = valid ? (int)(key >> 32) : 0;
  }
  // masks aligned with the match rows (0 for unmatched rows, unused kinds and invalid pairs)
  const int pb = a.cu_p[p], pe = a.cu_p[p + 1], lb = a.cu_l[p], le = a.cu_l[p + 1];
  if (a.rows_p && valid) {
    hg_compact<NT>(a.matches_p, pb, pe, a.n_pts1[p], warp_cnt, [&](int i, int, int ci) {
      a.inl_p[pb + i] = ci >= 0 ? fl[ci] : 0;
    });
  } else {
    for (int r = pb + threadIdx.x; r < pe; r += NT) a.inl_p[r] = 0;
  }
  if (a.rows_l && valid) {
    const int np = sp.np;
    hg_compact<NT>(a.matches_l, lb, le, a.n_segs1[p], warp_cnt, [&](int i, int, int ci) {
      a.inl_l[lb + i] = ci >= 0 ? fl[np + ci] : 0;
    });
  } else {
    for (int r = lb + threadIdx.x; r < le; r += NT) a.inl_l[r] = 0;
  }
}

}  // namespace ltr
