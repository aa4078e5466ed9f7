// All-pairs descriptor distance + mutual nearest-neighbour matcher.
// Reference: get_dist_matrix (models/line_process.py:198-201), subline2keyline
// (models/line_transformer.py:277-282), nn_matcher_distmat / nn_matcher
// (models/nn_matcher.py:3-43).  Distances are computed with fp32 FMAs in a fixed k order
// (deterministic, fp32-accurate) so that argmin/threshold decisions track the reference's
// fp32 BLAS result to rounding noise; the argmin / threshold / mutual logic itself is
// integer-exact: first minimum wins (np.argmin), strict '<' threshold.
#pragma once
#include "common.cuh"

namespace ltr {

struct DistArgs {
  const float* d0; const float* d1;
  int layout;            // 0 rows [n,d], 1 channel-first [d,n]
  int d;
  const int* cu0; const int* cu1;  // sublines offsets per pair or nullptr
  int n0, n1;            // uniform sizes
  float* out;            // pair p at p*stride, row-major [n0_p, n1_p]
  long long stride;
};

constexpr int DK_BM = 64, DK_BN = 64, DK_BK = 16, DK_THREADS = 256;

// D[i][j] = max(0, 2 - 2 <a_i, b_j>)   (einsum + (2-2s).clip(0), line_process.py:199-200)
template <bool CF>
__global__ void __launch_bounds__(DK_THREADS) dist_kernel(DistArgs p) {
  __shared__ __align__(16) float As[DK_BK][DK_BM + 4];
  __shared__ __align__(16) float Bs[DK_BK][DK_BN + 4];
  pdl_launch_dependents();
  pdl_wait();
  const int pair = blockIdx.z;
  int b0, e0, b1, e1;
  image_range(p.cu0, p.n0, pair, b0, e0);
  image_range(p.cu1, p.n1, pair, b1, e1);
  const int M = e0 - b0, N = e1 - b1;
  const int m0 = blockIdx.x * DK_BM, n0 = blockIdx.y * DK_BN;
  if (m0 >= M || n0 >= N) return;
  const float* __restrict__ A = p.d0 + (long long)b0 * p.d;
  const float* __restrict__ B = p.d1 + (long long)b1 * p.d;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < p.d; k0 += DK_BK) {
    if (CF) {
      // [d, n] : element (i, k) at k*M + i ; coalesced along i
      for (int idx = tid; idx < DK_BK * DK_BM; idx += DK_THREADS) {
        int k = idx >> 6, i = idx & 63;
        As[k][i] = (m0 + i < M && k0 + k < p.d) ? A[(long long)(k0 + k) * M + m0 + i] : 0.f;
        Bs[k][i] = (n0 + i < N && k0 + k < p.d) ? B[(long long)(k0 + k) * N + n0 + i] : 0.f;
      }
    } else {
      // [n, d] : 64 rows x 16 k = 256 float4, one per thread
      int r = tid >> 2, kq = (tid & 3) * 4;
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
      if (m0 + r < M) a = *reinterpret_cast<const float4*>(A + (long long)(m0 + r) * p.d + k0 + kq);
      if (n0 + r < N) b = *reinterpret_cast<const float4*>(B + (long long)(n0 + r) * p.d + k0 + kq);
      As[kq + 0][r] = a.x; As[kq + 1][r] = a.y; As[kq + 2][r] = a.z; As[kq + 3][r] = a.w;
      Bs[kq + 0][r] = b.x; Bs[kq + 1][r] = b.y; Bs[kq + 2][r] = b.z; Bs[kq + 3][r] = b.w;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < DK_BK; ++k) {
      float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* __restrict__ O = p.out + (long long)pair * p.stride;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int r = m0 + ty * 4 + i;
    if (r >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int c = n0 + tx * 4 + j;
      if (c < N) O[(long long)r * N + c] = fmaxf(2.f - 2.f * acc[i][j], 0.f);
    }
  }
}

// Keyline distance = A0 @ D_sub @ A1^T with block-constant adjacency rows 1/n_sub
// (models/line_process.py:163-167, models/line_transformer.py:281).  sub_off are CSR offsets
// keyline -> sublines in GLOBAL subline numbering; cuk are keyline offsets per pair.
struct SegMeanArgs {
  const float* dist_sub; long long stride_sub;
  float* dist_key; long long stride_key;
  const int* cuk0; const int* cuk1;        // [n_pairs+1]
  const int* sub_off0; const int* sub_off1;  // [total keylines + 1]
  const int* img0; const int* img1;        // image pools: image of every pair's side [n_pairs], cuk over images;
                                           // nullptr: pair p is image p
};

__global__ void __launch_bounds__(256) segmean_kernel(SegMeanArgs p) {
  const int pair = blockIdx.z;
  const int im0 = p.img0 ? p.img0[pair] : pair, im1 = p.img1 ? p.img1[pair] : pair;
  const int kb0 = p.cuk0[im0], K0 = p.cuk0[im0 + 1] - kb0;
  const int kb1 = p.cuk1[im1], K1 = p.cuk1[im1 + 1] - kb1;
  const int sb0 = p.sub_off0[kb0], sb1 = p.sub_off1[kb1];
  const int N1 = p.sub_off1[kb1 + K1] - sb1;
  const int b = blockIdx.x * 32 + (threadIdx.x & 31);
  const int a = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (a >= K0 || b >= K1) return;
  const int i0 = p.sub_off0[kb0 + a] - sb0, i1 = p.sub_off0[kb0 + a + 1] - sb0;
  const int j0 = p.sub_off1[kb1 + b] - sb1, j1 = p.sub_off1[kb1 + b + 1] - sb1;
  const float wa = 1.f / (float)(i1 - i0), wb = 1.f / (float)(j1 - j0);
  const float* __restrict__ D = p.dist_sub + (long long)pair * p.stride_sub;
  float acc = 0.f;
  for (int j = j0; j < j1; ++j) {
    float t = 0.f;
    for (int i = i0; i < i1; ++i) t = fmaf(wa, D[(long long)i * N1 + j], t);
    acc = fmaf(t, wb, acc);
  }
  p.dist_key[(long long)pair * p.stride_key + (long long)a * K1 + b] = acc;
}

// np.argmin order on clipped distances: a NaN compares as the minimum (np.argmin returns the FIRST NaN of
// a row; its score NaN then fails the strict `< thr`, nn_matcher.py:15-18), otherwise plain `<`.
__device__ __forceinline__ bool nn_less(float a, int ia, float b, int ib) {
  const bool an = a != a, bn = b != b;
  if (an || bn) return an && (!bn || ia < ib);
  return a < b || (a == b && ia < ib);
}

struct NNArgs {
  const float* dist; long long stride;
  const int* cuk0; const int* cuk1;  // keyline offsets per pair or nullptr (uniform)
  int n0, n1;
  float thr; int mutual;
  int* matches0; float* scores0; int* nn1; int* counts;
};

// idx = argmin(d, axis=1), score = d[i, idx]   (nn_matcher.py:13-16); one warp per row.
__global__ void __launch_bounds__(256) row_argmin_kernel(NNArgs p) {
  const int pair = blockIdx.y;
  pdl_launch_dependents();
  pdl_wait();
  if (blockIdx.x == 0 && threadIdx.x == 0) p.counts[pair] = 0;   // mutual_kernel (a later launch) accumulates into it
  int b0, e0, b1, e1;
  image_range(p.cuk0, p.n0, pair, b0, e0);
  image_range(p.cuk1, p.n1, pair, b1, e1);
  const int K0 = e0 - b0, K1 = e1 - b1;
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= K0) return;
  const float* __restrict__ D = p.dist + (long long)pair * p.stride + (long long)row * K1;
  float best = INFINITY; int bi = 0x7fffffff;
  for (int j = lane; j < K1; j += 32) {
    float v = D[j];
    v = v < 0.f ? 0.f : v;       // .clip(min=0), nn_matcher.py:12; a NaN stays NaN, as with np.clip
    if (nn_less(v, j, best, bi)) { best = v; bi = j; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, best, o);
    int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (nn_less(ov, oi, best, bi)) { best = ov; bi = oi; }
  }
  if (lane == 0) {
    p.matches0[b0 + row] = (K1 > 0) ? bi : -1;
    p.scores0[b0 + row] = best;
  }
}

// idx2 = argmin(d, axis=0)  (nn_matcher.py:21); block = 32 columns x 8 row groups.
__global__ void __launch_bounds__(256) col_argmin_kernel(NNArgs p) {
  __shared__ float sv[8][33];
  __shared__ int si[8][33];
  pdl_launch_dependents();
  pdl_wait();
  const int pair = blockIdx.y;
  int b0, e0, b1, e1;
  image_range(p.cuk0, p.n0, pair, b0, e0);
  image_range(p.cuk1, p.n1, pair, b1, e1);
  const int K0 = e0 - b0, K1 = e1 - b1;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + tx;
  if (blockIdx.x * 32 >= K1) return;
  const float* __restrict__ D = p.dist + (long long)pair * p.stride;
  float best = INFINITY; int bi = 0x7fffffff;
  if (col < K1) {
    for (int i = ty; i < K0; i += 8) {
      float v = D[(long long)i * K1 + col];
      v = v < 0.f ? 0.f : v;     // NaN-preserving clip
      if (nn_less(v, i, best, bi)) { best = v; bi = i; }
    }
  }
  sv[ty][tx] = best; si[ty][tx] = bi;
  __syncthreads();
  if (ty == 0 && col < K1) {
#pragma unroll
    for (int r = 1; r < 8; ++r) {
      float ov = sv[r][tx]; int oi = si[r][tx];
      if (nn_less(ov, oi, best, bi)) { best = ov; bi = oi; }
    }
    p.nn1[b1 + col] = (K0 > 0) ? bi : -1;
  }
}

// keep = score < thr [and i == idx2[idx[i]]]  (nn_matcher.py:18-23); counts per pair.
__global__ void __launch_bounds__(256) mutual_kernel(NNArgs p) {
  pdl_launch_dependents();
  pdl_wait();
  const int pair = blockIdx.y;
  int b0, e0, b1, e1;
  image_range(p.cuk0, p.n0, pair, b0, e0);
  image_range(p.cuk1, p.n1, pair, b1, e1);
  const int K0 = e0 - b0;
  const int i = blockIdx.x * 256 + threadIdx.x;
  bool keep = false;
  if (i < K0) {
    int j = p.matches0[b0 + i];
    keep = j >= 0 && p.scores0[b0 + i] < p.thr;
    if (keep && p.mutual) keep = (p.nn1[b1 + j] == i);
    if (!keep) p.matches0[b0 + i] = -1;
  }
  unsigned m = __ballot_sync(0xffffffffu, keep);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(&p.counts[pair], __popc(m));
}

}  // namespace ltr
