// Homography image pairs: image 1 of every pair (OpenCV's fixed-point warpPerspective, INTER_LINEAR,
// BORDER_CONSTANT 0) and the homography builder's eroded valid mask, one CTA per output tile.
//
// Per output pixel (x, y) of pair p with inverse map M (image 1 -> image 0):
//   the columns go in blocks of bw = min(1024 / min(16, height), width) (cv2's remap block); for x = xb + j,
//   X0 = M0*xb + M1*y + M2 (likewise Y0, W0), w = W0 + M6*j, w = w ? 32/w : 0,
//   X = rint(clamp((X0 + M0*j) * w, INT_MIN, INT_MAX)) (likewise Y), all in round-to-nearest fp64 without FMA
//   contraction: this operation order is part of the contract (cv2 evaluates it so, and other orders change bits).
//   Cell (X >> 5, Y >> 5), sub-pixel (X & 31, Y & 31); the four neighbours weigh (32-fx)(32-fy)*32, fx(32-fy)*32,
//   (32-fx)fy*32, fx*fy*32 (sum 32768); neighbours outside the image are 0; grey = (sum w_i p_i + 16384) >> 15.
//   The pre-erosion mask is 1 iff some in-image neighbour with a nonzero weight has a nonzero colour channel (the
//   float colour warp is then not exactly 0); the mask is its 5 x 5 erosion, pixels outside the image counting as 1.
// The CTA computes the pre-erosion mask on its tile plus a 2-pixel halo in shared memory, erodes it there and
// writes grey and mask once.  Nothing else is written to device memory.
#pragma once
#include <climits>

#include "common.cuh"

namespace ltr {

constexpr int WP_TW = 64, WP_TH = 32, WP_HALO = 2, WP_THREADS = 256;
constexpr int WP_RW = WP_TW + 2 * WP_HALO, WP_RH = WP_TH + 2 * WP_HALO;   // tile + halo
constexpr int WP_MAX_SIDE = 32767;   // cv2's remap keeps source cells in int16

struct WarpArgs {
  const uint8_t* gray;      // [n_images, h, w]
  const uint8_t* colour;    // [n_images, h, w, c]
  const int32_t* src_index; // [n_pairs]
  const double* inv_maps;   // [n_pairs, 9]
  uint8_t* warped;          // [n_pairs, h, w]
  uint8_t* mask;            // [n_pairs, h, w]
  int n_images, h, w, c, bw, tiles_x, tiles_per_pair;
};

// Fixed-point source position (X, Y) of output pixel (x, y), in 1/32 pixel.
__device__ __forceinline__ void wp_position(const double* m, int x, int y, int bw, int& X, int& Y) {
  const int j = x % bw;
  const double xb = (double)(x - j), yd = (double)y, jd = (double)j;
  const double X0 = __dadd_rn(__dadd_rn(__dmul_rn(m[0], xb), __dmul_rn(m[1], yd)), m[2]);
  const double Y0 = __dadd_rn(__dadd_rn(__dmul_rn(m[3], xb), __dmul_rn(m[4], yd)), m[5]);
  const double W0 = __dadd_rn(__dadd_rn(__dmul_rn(m[6], xb), __dmul_rn(m[7], yd)), m[8]);
  double w = __dadd_rn(W0, __dmul_rn(m[6], jd));
  w = w != 0.0 ? __ddiv_rn(32.0, w) : 0.0;
  const double fx = __dmul_rn(__dadd_rn(X0, __dmul_rn(m[0], jd)), w);
  const double fy = __dmul_rn(__dadd_rn(Y0, __dmul_rn(m[3], jd)), w);
  X = __double2int_rn(fmin(fmax(fx, (double)INT_MIN), (double)INT_MAX));
  Y = __double2int_rn(fmin(fmax(fy, (double)INT_MIN), (double)INT_MAX));
}

__global__ void __launch_bounds__(WP_THREADS) warp_pairs_kernel(WarpArgs a) {
  __shared__ uint8_t pre[WP_RH][WP_RW];   // pre-erosion mask of tile + halo (1 outside the image)
  __shared__ uint8_t rmin[WP_RH][WP_TW];  // its 5-wide row minimum
  __shared__ double m[9];
  const int pair = blockIdx.x / a.tiles_per_pair, t = blockIdx.x % a.tiles_per_pair;
  const int x0 = (t % a.tiles_x) * WP_TW, y0 = (t / a.tiles_x) * WP_TH;
  const int h = a.h, w = a.w, c = a.c;
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x < 9) m[threadIdx.x] = a.inv_maps[(size_t)pair * 9 + threadIdx.x];
  const int src = a.src_index[pair];
  const bool src_ok = (unsigned)src < (unsigned)a.n_images;   // the host validated it; a bad copy warps nothing
  const size_t plane = (size_t)h * w;
  const uint8_t* g = a.gray + (src_ok ? (size_t)src : 0) * plane;
  const uint8_t* col = a.colour + (src_ok ? (size_t)src : 0) * plane * c;
  uint8_t* out = a.warped + (size_t)pair * plane;
  __syncthreads();

  for (int i = threadIdx.x; i < WP_RH * WP_RW; i += WP_THREADS) {
    const int ry = i / WP_RW, rx = i - ry * WP_RW;
    const int y = y0 - WP_HALO + ry, x = x0 - WP_HALO + rx;
    uint8_t valid = 1;
    if (y >= 0 && y < h && x >= 0 && x < w) {
      const bool inner = rx >= WP_HALO && rx < WP_HALO + WP_TW && ry >= WP_HALO && ry < WP_HALO + WP_TH;
      int acc = 16384;
      bool nz = false;
      if (src_ok) {
        int X, Y;
        wp_position(m, x, y, a.bw, X, Y);
        const int sx = X >> 5, sy = Y >> 5, fx = X & 31, fy = Y & 31;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int dy = k >> 1, dx = k & 1;
          const int r = sy + dy, cc = sx + dx;
          if ((unsigned)r < (unsigned)h && (unsigned)cc < (unsigned)w) {
            const int wt = (dy ? fy : 32 - fy) * (dx ? fx : 32 - fx) * 32;
            const size_t o = (size_t)r * w + cc;
            if (inner) acc += wt * (int)__ldg(g + o);
            if (wt != 0 && !nz) {
              const uint8_t* p = col + o * c;
              nz = c == 3 ? (__ldg(p) | __ldg(p + 1) | __ldg(p + 2)) != 0 : __ldg(p) != 0;
            }
          }
        }
      }
      if (inner) out[(size_t)y * w + x] = (uint8_t)min(acc >> 15, 255);
      valid = nz ? 1 : 0;
    }
    pre[ry][rx] = valid;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < WP_RH * WP_TW; i += WP_THREADS) {
    const int ry = i / WP_TW, cx = i - ry * WP_TW;
    rmin[ry][cx] = pre[ry][cx] & pre[ry][cx + 1] & pre[ry][cx + 2] & pre[ry][cx + 3] & pre[ry][cx + 4];
  }
  __syncthreads();
  uint8_t* mk = a.mask + (size_t)pair * plane;
  for (int i = threadIdx.x; i < WP_TH * WP_TW; i += WP_THREADS) {
    const int oy = i / WP_TW, ox = i - oy * WP_TW;
    const int y = y0 + oy, x = x0 + ox;
    if (y < h && x < w)
      mk[(size_t)y * w + x] = rmin[oy][ox] & rmin[oy + 1][ox] & rmin[oy + 2][ox] & rmin[oy + 3][ox] & rmin[oy + 4][ox];
  }
}

}  // namespace ltr
