// RANSAC scaffolding shared by the homography (homography.cuh), essential-matrix (essential.cuh), fundamental-matrix
// (fundamental.cuh) and absolute-pose (absolute_pose.cuh) estimators: the counter-based sample hash, the row-ordered
// compaction of a pair's match rows into shared memory, the draw of one hypothesis' distinct correspondences
// (geometry.draw_samples restates it in numpy), and the fp64 solver pieces: the null basis of a minimal sample's epipolar rows (Householder QR), the Sturm-chain root
// finder (geometry.sturm_roots) and the cyclic Jacobi eigen-solvers of the refits and decompositions.
#pragma once
#include "common.cuh"
#include "rn_fp64.cuh"

namespace ltr {

constexpr int HG_MAX_DRAWS = 64;   // draws per hypothesis before it is rejected
constexpr int ESS_BISECT_STEPS = 100;
constexpr double ESS_RANK_EPS = 1e-10;    // a QR column norm at most this times the first rejects the sample
constexpr double ESS_ROOT_BOUND = 1e8;    // real roots are searched in [-B, B], B = min(Cauchy bound, this)
constexpr int RC_JACOBI3_SWEEPS = 30;
constexpr int RC_JACOBI9_SWEEPS = 32;

__device__ __forceinline__ unsigned long long hg_splitmix64(unsigned long long x) {
  unsigned long long z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// Row-ordered compaction of the rows [b, e) of a match array whose match m passes keep(m): f(local row, match, compact
// index or -1) for every row.  All threads of the block must call it.
template <int NT, typename K, typename F>
__device__ __forceinline__ int rc_compact_if(const int* __restrict__ match, int b, int e, int* warp_cnt, K keep, F f) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int base = 0;
  for (int r0 = b; r0 < e; r0 += NT) {
    const int r = r0 + threadIdx.x;
    const int m = r < e ? match[r] : -1;
    const bool ok = r < e && keep(m);
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) warp_cnt[w] = __popc(bal);
    __syncthreads();
    int off = base, tot = 0;
#pragma unroll
    for (int i = 0; i < NT / 32; ++i) {
      off += i < w ? warp_cnt[i] : 0;
      tot += warp_cnt[i];
    }
    if (r < e) f(r - b, m, ok ? off + __popc(bal & ((1u << lane) - 1u)) : -1);
    __syncthreads();
    base += tot;
  }
  return base;
}

// The matched rows (match in [0, n1)) of [b, e): rc_compact_if with that test.
template <int NT, typename F>
__device__ __forceinline__ int hg_compact(const int* __restrict__ match, int b, int e, int n1, int* warp_cnt, F f) {
  return rc_compact_if<NT>(match, b, e, warp_cnt, [n1](int m) { return m >= 0 && m < n1; }, f);
}

// The S distinct correspondence indices of hypothesis k of pair p among n: s = splitmix64(seed + splitmix64(p << 32 |
// k)), draw j = splitmix64(s + j) mod n, a duplicate redrawn with the next j; false after HG_MAX_DRAWS draws.
template <int S>
__device__ __forceinline__ bool hg_draw(unsigned long long seed, int p, int k, int n, int* idx) {
  const unsigned long long s = hg_splitmix64(seed + hg_splitmix64(((unsigned long long)(unsigned)p << 32) | (unsigned)k));
  int got = 0;
  for (int j = 0; j < HG_MAX_DRAWS && got < S; ++j) {
    const int v = (int)(hg_splitmix64(s + (unsigned long long)j) % (unsigned long long)n);
    bool dup = false;
    for (int q = 0; q < got; ++q) dup |= idx[q] == v;
    if (!dup) idx[got++] = v;
  }
  return got == S;
}

// Null basis of the S epipolar rows (x1 x0, x1 y0, x1, y1 x0, y1 y0, y1, x0, y0, 1) of q[c] = (x0, y0, x1, y1), S = 5
// (essential) or 7 (fundamental): the Householder QR of the 9 x S transpose (reflector c zeroes column c below the
// diagonal, alpha = -sign(M[c][c]) |column|), then basis vector b = Q e_(S + b) with e[i][b] its entry i.  Explicitly
// rounded fp64.  -> false for a rank-deficient sample (a column norm <= ESS_RANK_EPS times the first).
template <int S>
__device__ __forceinline__ bool rc_null_basis(const double4* q, double (*e)[9 - S]) {
  double M[9][S];
  for (int c = 0; c < S; ++c) {
    const double a0 = q[c].x, b0 = q[c].y, a1 = q[c].z, b1 = q[c].w;
    M[0][c] = RC_M(a1, a0); M[1][c] = RC_M(a1, b0); M[2][c] = a1;
    M[3][c] = RC_M(b1, a0); M[4][c] = RC_M(b1, b0); M[5][c] = b1;
    M[6][c] = a0; M[7][c] = b0; M[8][c] = 1.0;
  }
  double V[S][9], beta[S], nrm0 = 0.0;   // reflector c is V[c][c..8] (v_c = M[c][c] - alpha, then M[c+1..8][c])
  for (int c = 0; c < S; ++c) {
    double acc = 0.0;
    for (int i = c; i < 9; ++i) acc = RC_A(acc, RC_M(M[i][c], M[i][c]));
    const double nrm = __dsqrt_rn(acc);
    if (c == 0) {
      nrm0 = nrm;
      if (!(nrm > 0.0)) return false;
    } else if (!(nrm > RC_M(ESS_RANK_EPS, nrm0))) {
      return false;   // rank-deficient sample
    }
    const double alpha = M[c][c] >= 0.0 ? -nrm : nrm;
    for (int i = c + 1; i < 9; ++i) V[c][i] = M[i][c];
    V[c][c] = RC_S(M[c][c], alpha);
    double vtv = 0.0;
    for (int i = c; i < 9; ++i) vtv = RC_A(vtv, RC_M(V[c][i], V[c][i]));
    beta[c] = vtv > 0.0 ? RC_D(2.0, vtv) : 0.0;
    for (int j = c + 1; j < S; ++j) {
      double s = 0.0;
      for (int i = c; i < 9; ++i) s = RC_A(s, RC_M(V[c][i], M[i][j]));
      const double g = RC_M(s, beta[c]);
      for (int i = c; i < 9; ++i) M[i][j] = RC_S(M[i][j], RC_M(g, V[c][i]));
    }
  }
  for (int b = 0; b < 9 - S; ++b) {
    double y[9];
    for (int i = 0; i < 9; ++i) y[i] = i == S + b ? 1.0 : 0.0;
    for (int c = S - 1; c >= 0; --c) {
      double s = 0.0;
      for (int i = c; i < 9; ++i) s = RC_A(s, RC_M(V[c][i], y[i]));
      const double g = RC_M(s, beta[c]);
      for (int i = c; i < 9; ++i) y[i] = RC_S(y[i], RC_M(g, V[c][i]));
    }
    for (int i = 0; i < 9; ++i) e[i][b] = y[i];
  }
  return true;
}

// Polynomials in z, ascending coefficients: out (la + lb - 1) = x (la) * y (lb)
__device__ __forceinline__ void ess_pmul(const double* x, int la, const double* y, int lb, double* out) {
  for (int i = 0; i < la + lb - 1; ++i) out[i] = 0.0;
  for (int i = 0; i < la; ++i)
    for (int j = 0; j < lb; ++j) out[i + j] = RC_A(out[i + j], RC_M(x[i], y[j]));
}

__device__ __forceinline__ double ess_horner(const double* c, int deg, double x) {
  double v = c[deg];
  for (int i = deg - 1; i >= 0; --i) v = RC_A(RC_M(v, x), c[i]);
  return v;
}

__device__ __forceinline__ double ess_maxabs(const double* c, int n) {
  double m = 0.0;
  for (int i = 0; i < n; ++i) {
    const double v = fabs(c[i]);
    m = v > m ? v : m;
  }
  return m;
}

// Member k of the Sturm chain starts at chain + ESS_CHAIN_OFF(k) and has 11 - k coefficients: its degree is at most
// 10 - k (degrees strictly decrease along the chain), the coefficients above its degree are 0.
#define ESS_CHAIN_OFF(k) (11 * (k) - ((k) * ((k) - 1)) / 2)

// Degree of c (coefficients 0..top): the highest index with a non-zero coefficient, 0 for a constant.
__device__ __forceinline__ int ess_degree(const double* c, int top) {
  while (top > 0 && c[top] == 0.0) --top;
  return top;
}

__device__ __forceinline__ int ess_sign_changes(const double* chain, int len, double x) {
  int prev = 0, n = 0;
  for (int k = 0; k < len; ++k) {
    const double v = ess_horner(chain + ESS_CHAIN_OFF(k), 10 - k, x);
    const int s = (v > 0.0) - (v < 0.0);
    if (s != 0) {
      n += prev != 0 && s != prev;
      prev = s;
    }
  }
  return n;
}

// Real roots of the polynomial p (ascending, 11 coefficients, degree 1 to 10 once exact-zero leading coefficients are
// stripped) in [-B, B]: Sturm chain and bisection.  -> root count; 0 for a constant or a non-finite coefficient.
__device__ int ess_roots(const double* p, double* roots) {
  double chain[66];
  bool fin = true;
  for (int i = 0; i < 11; ++i) fin &= isfinite(p[i]);
  const double m = ess_maxabs(p, 11);
  if (!(fin && m > 0.0)) return 0;
  for (int i = 0; i < 11; ++i) chain[i] = RC_D(p[i], m);
  const int n = ess_degree(chain, 10);
  if (n == 0) return 0;
  double bound = 1.0;
  for (int i = 0; i < n; ++i) {
    const double v = RC_A(fabs(RC_D(chain[i], chain[n])), 1.0);
    bound = v > bound ? v : bound;
  }
  bound = bound < ESS_ROOT_BOUND ? bound : ESS_ROOT_BOUND;
  if (!(bound == bound)) return 0;
  double* d = chain + ESS_CHAIN_OFF(1);
  for (int i = 0; i < 10; ++i) d[i] = RC_M(chain[i + 1], (double)(i + 1));
  const double md = ess_maxabs(d, 10);   // > 0: d[n - 1] = n chain[n]
  for (int i = 0; i < 10; ++i) d[i] = RC_D(d[i], md);
  // Members len - 2 (A, degree da) and len - 1 (Bp, degree db < da) give the next member: the remainder of A / Bp by
  // long division, negated, stripped of exact-zero leading coefficients and divided by its largest |coefficient|.
  // The chain ends at a constant, or before a zero remainder (Bp is then the gcd of p and p').  Where every degree
  // drops by one this is the two-step division q1 = A[da] / lead, q0 = T[db] / lead.
  int len = 2, da = n, db = ess_degree(d, n - 1);
  while (db > 0) {
    const double* A = chain + ESS_CHAIN_OFF(len - 2);
    const double* Bp = chain + ESS_CHAIN_OFF(len - 1);
    double* r = chain + ESS_CHAIN_OFF(len);
    const double lead = Bp[db];
    double T[11];
    for (int i = 0; i <= da; ++i) T[i] = A[i];
    for (int j = da; j >= db; --j) {
      const double q = RC_D(T[j], lead);
      for (int i = 0; i < db; ++i) T[j - db + i] = RC_S(T[j - db + i], RC_M(q, Bp[i]));
    }
    for (int i = 0; i < db; ++i) r[i] = -T[i];
    const double mr = ess_maxabs(r, db);
    if (!(mr > 0.0)) break;
    for (int i = 0; i < db; ++i) r[i] = RC_D(r[i], mr);
    for (int i = db; i < 11 - len; ++i) r[i] = 0.0;
    da = db;
    db = ess_degree(r, db - 1);
    ++len;
  }
  const int v_lo = ess_sign_changes(chain, len, -bound);
  int count = v_lo - ess_sign_changes(chain, len, bound);
  count = count < 0 ? 0 : (count > 10 ? 10 : count);
  for (int i = 0; i < count; ++i) {
    double lo = -bound, hi = bound;
    for (int s = 0; s < ESS_BISECT_STEPS; ++s) {
      const double mid = RC_M(RC_A(lo, hi), 0.5);
      if (!(mid > lo && mid < hi)) break;   // converged: further steps change nothing
      if (v_lo - ess_sign_changes(chain, len, mid) > i) hi = mid; else lo = mid;
    }
    roots[i] = RC_M(RC_A(lo, hi), 0.5);
  }
  return count;
}

// Cyclic Jacobi eigen-decomposition of the symmetric 3 x 3 S (diagonalised in place; V accumulates the rotations and
// must start as the identity).
__device__ __forceinline__ void rc_jacobi3(double (*S)[3], double (*V)[3]) {
  const double fro = S[0][0] * S[0][0] + S[1][1] * S[1][1] + S[2][2] * S[2][2];
  for (int sweep = 0; sweep < RC_JACOBI3_SWEEPS; ++sweep) {
    const double off = S[0][1] * S[0][1] + S[0][2] * S[0][2] + S[1][2] * S[1][2];
    if (!(off > 1e-32 * fro)) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        const double apq = S[p][q];
        if (apq == 0.0) continue;
        const double theta = (S[q][q] - S[p][p]) / (2.0 * apq);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 3; ++k) {
          const double skp = S[k][p], skq = S[k][q];
          S[k][p] = c * skp - s * skq;
          S[k][q] = s * skp + c * skq;
        }
        for (int k = 0; k < 3; ++k) {
          const double spk = S[p][k], sqk = S[q][k];
          S[p][k] = c * spk - s * sqk;
          S[q][k] = s * spk + c * sqk;
        }
        for (int k = 0; k < 3; ++k) {
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - s * vkq;
          V[k][q] = s * vkp + c * vkq;
        }
      }
  }
}

// Eigenvector of the smallest eigenvalue of the symmetric 9x9 M (cyclic Jacobi; M is destroyed).
__device__ __noinline__ void hg_smallest_eigvec(double* M, double* h) {
  double V[81];
  for (int i = 0; i < 81; ++i) V[i] = (i % 10 == 0) ? 1.0 : 0.0;
  double fro = 0.0;
  for (int i = 0; i < 81; ++i) fro += M[i] * M[i];
  for (int sweep = 0; sweep < RC_JACOBI9_SWEEPS; ++sweep) {
    double off = 0.0;
    for (int i = 0; i < 9; ++i)
      for (int j = i + 1; j < 9; ++j) off += M[9 * i + j] * M[9 * i + j];
    if (!(off > 1e-32 * fro)) break;
    for (int p = 0; p < 8; ++p)
      for (int q = p + 1; q < 9; ++q) {
        const double apq = M[9 * p + q];
        if (apq == 0.0) continue;
        const double theta = (M[9 * q + q] - M[9 * p + p]) / (2.0 * apq);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 9; ++k) {
          const double mkp = M[9 * k + p], mkq = M[9 * k + q];
          M[9 * k + p] = c * mkp - s * mkq;
          M[9 * k + q] = s * mkp + c * mkq;
        }
        for (int k = 0; k < 9; ++k) {
          const double mpk = M[9 * p + k], mqk = M[9 * q + k];
          M[9 * p + k] = c * mpk - s * mqk;
          M[9 * q + k] = s * mpk + c * mqk;
        }
        for (int k = 0; k < 9; ++k) {
          const double vkp = V[9 * k + p], vkq = V[9 * k + q];
          V[9 * k + p] = c * vkp - s * vkq;
          V[9 * k + q] = s * vkp + c * vkq;
        }
      }
  }
  int m = 0;
  for (int i = 1; i < 9; ++i)
    if (M[10 * i] < M[10 * m]) m = i;
  for (int k = 0; k < 9; ++k) h[k] = V[9 * k + m];
}

#undef ESS_CHAIN_OFF

}  // namespace ltr
