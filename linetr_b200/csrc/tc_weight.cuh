// Split-bf16 weight images for the tensor-core kernels (gemm_img.cuh, token_fused.cuh).
//
// Precision: every fp32 operand is split x = hi + lo (both bf16) and three MMAs are issued per
// k-step, hi*hi + lo*hi + hi*lo, accumulated in fp32 - ~2^-17 relative operand error instead of
// bf16's 2^-9 (single-pass TF32 already misses the 1e-3 descriptor bar, SURVEY.md 0 fact 9).
#pragma once
#include <cstring>
#include "common.cuh"
#include "ptx_sm90.cuh"

namespace ltr {

// W [N, K] packed for the engine: bf16 hi and lo images, tiled as [K/64][N/8] atoms of
// 8 rows x 64 k (1024 bytes, 128B swizzle) so that any (n0, kb) tile of BN rows is one
// contiguous BN*128-byte range (one bulk copy).
struct TcWeight {
  const __nv_bfloat16* hi = nullptr;
  const __nv_bfloat16* lo = nullptr;
  int N = 0, K = 0;
};

// ---------------------------------------------------------------- host-side weight packing
inline uint16_t f32_to_bf16_rn(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  u += 0x7FFFu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
inline float bf16_to_f32(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
// W: [N, K] row-major (double).  hi/lo: N*K uint16 each, engine tile layout.
inline void pack_tc_weight(const double* W, int N, int K, uint16_t* hi, uint16_t* lo) {
  for (int n = 0; n < N; ++n)
    for (int k = 0; k < K; ++k) {
      const float w = (float)W[(size_t)n * K + k];
      const uint16_t h = f32_to_bf16_rn(w);
      const uint16_t l = f32_to_bf16_rn(w - bf16_to_f32(h));
      const size_t atom = (size_t)(k / 64) * (N / 8) + n / 8;
      const size_t idx = atom * 512 + ptx::sw128_offset(n & 7, k & 63) / 2;
      hi[idx] = h;
      lo[idx] = l;
    }
}

}  // namespace ltr
