// Split-bf16 activation image: the operand format of the tensor-core GEMM engine.
// See gemm_img.cuh for the layout description.
#pragma once
#include "ptx_sm90.cuh"

namespace ltr {

struct ActImg {
  __nv_bfloat16* hi = nullptr;
  __nv_bfloat16* lo = nullptr;
  int kblocks = 0;  // K/64 tiles per 128-row block
};
constexpr int IMG_TILE_ELEMS = 128 * 64;  // 16 KB of bf16 per tile and plane

// element index (in bf16 units, same for both planes) of activation element (row, k)
__device__ __forceinline__ size_t img_index(const ActImg& a, int row, int k) {
  return ((size_t)(row >> 7) * a.kblocks + (k >> 6)) * IMG_TILE_ELEMS + ptx::sw128_offset(row & 127, k & 63) / 2;
}
__device__ __forceinline__ void img_store1(const ActImg& a, int row, int k, float v) {
  __nv_bfloat16 h, l;
  ptx::split_bf16(v, h, l);
  const size_t i = img_index(a, row, k);
  a.hi[i] = h;
  a.lo[i] = l;
}
// 4 consecutive k (k % 4 == 0): one 8-byte store per plane
__device__ __forceinline__ void img_store4(const ActImg& a, int row, int k, float v0, float v1, float v2, float v3) {
  uint2 h, l;
  ptx::split2_bf16(v0, v1, h.x, l.x);
  ptx::split2_bf16(v2, v3, h.y, l.y);
  const size_t i = img_index(a, row, k);
  *reinterpret_cast<uint2*>(a.hi + i) = h;
  *reinterpret_cast<uint2*>(a.lo + i) = l;
}
// 8 consecutive k (k % 8 == 0): one 16-byte store per plane
__device__ __forceinline__ void img_store8(const ActImg& a, int row, int k, const float (&v)[8]) {
  uint4 h, l;
  ptx::split8_bf16(v, h, l);
  const size_t i = img_index(a, row, k);
  *reinterpret_cast<uint4*>(a.hi + i) = h;
  *reinterpret_cast<uint4*>(a.lo + i) = l;
}

}  // namespace ltr
