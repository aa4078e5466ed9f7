// RANSAC scaffolding shared by the homography (homography.cuh) and essential-matrix (essential.cuh) estimators: the
// counter-based sample hash, the row-ordered compaction of a pair's match rows into shared memory, and the draw of
// one hypothesis' distinct correspondences (geometry.draw_samples restates it in numpy).
#pragma once
#include "common.cuh"

namespace ltr {

constexpr int HG_MAX_DRAWS = 64;   // draws per hypothesis before it is rejected

__device__ __forceinline__ unsigned long long hg_splitmix64(unsigned long long x) {
  unsigned long long z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// Row-ordered compaction of the matched rows [b, e) of a match array: f(local row, match, compact index or -1) for
// every row.  All threads of the block must call it.
template <int NT, typename F>
__device__ __forceinline__ int hg_compact(const int* __restrict__ match, int b, int e, int n1, int* warp_cnt, F f) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int base = 0;
  for (int r0 = b; r0 < e; r0 += NT) {
    const int r = r0 + threadIdx.x;
    const int m = r < e ? match[r] : -1;
    const bool ok = r < e && m >= 0 && m < n1;
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

}  // namespace ltr
