// Photometric augmentation of the homography dataset builder for a batch of uint8 images (DESIGN.md "Photometric
// augmentation"; the numpy model is linetr_b200/photometric.py).  Four launches per batch:
//   photo_stage1_kernel   brightness -> contrast -> Gaussian noise -> impulse noise -> 3 x 3 motion blur, one
//                         64 x 16 tile per CTA; the tile's 1-pixel halo is recomputed pointwise (the noise is a
//                         counter-based function of the pixel), so no second pass is needed.  Writes stage-1 bytes.
//   photo_ellipse_kernel  one CTA per shade ellipse: cv2.ellipse's fixed-point polygon, its 8-connected outline and
//                         its convex scan fill, written as 255 into a zeroed uint8 mask.
//   photo_blur_row_kernel the Gaussian's row pass, mask -> fp32, 8 rows x 128 columns per CTA.
//   photo_blur_col_kernel the column pass, 128 rows x 32 columns per CTA, fused with the shade's multiply, clip and
//                         the reference's float32/float64 chain ending in truncation; writes the output.
// Every floating-point step is explicitly rounded in the model's order (no contraction): the blur's sums are
// acc = fl32(acc + fl32(tap * v)) for taps k = 0.., the motion blur's are fp32 FMAs in row-major kernel order.
#pragma once
#include "common.cuh"

namespace ltr {

constexpr int PH_NPARAM = 28, PH_MAX_KSIZE = 149, PH_KPAD = 152;   // taps padded with zeros to a multiple of 4
constexpr int PH_P_BRIGHT = 0, PH_P_CONTRAST = 3, PH_P_NOISE = 6, PH_P_SPECKLE = 9, PH_P_BLUR = 12, PH_P_KERNEL = 13,
              PH_P_SHADE = 22, PH_P_TRANSPARENCY = 23, PH_P_KSIZE = 24, PH_P_KEY_LO = 25, PH_P_KEY_HI = 26,
              PH_P_N_ELLIPSES = 27;
constexpr int PS_TW = 64, PS_TH = 16, PS_THREADS = 256;
constexpr int PE_THREADS = 128, PE_MAXV = 80, PE_MAXSPAN = 96;
constexpr int PR_W = 128, PR_ROWS = 8, PR_LEN = PR_W + PH_KPAD + 8;          // row pass tile, smem row length
constexpr int PC_W = 32, PC_H = 128, PC_Q = 16, PC_LEN = PC_H + PH_KPAD + 8;  // column pass tile, rows per thread
constexpr int PH_XY_SHIFT = 16;
constexpr long long PH_XY_HALF = 1LL << (PH_XY_SHIFT - 1);

struct PhotoArgs {
  const uint8_t* in;       // [n, h, w]
  uint8_t* out;            // [n, h, w] (may equal in)
  const double* params;    // [n, PH_NPARAM]
  const int32_t* ellipses; // [n, max_ellipses, 5] (ax, ay, x, y, angle)
  const float* taps;       // [n, PH_MAX_KSIZE]
  uint8_t* stage1;         // workspace [n, h, w]
  uint8_t* mask;           // workspace [n, h, w], zeroed before photo_ellipse_kernel
  float* rowblur;          // workspace [n, h, w]
  int h, w, max_ellipses;
};

__device__ __forceinline__ int ph_reflect101(int i, int n) {
  if (n == 1) return 0;
  const int p = 2 * (n - 1);
  i %= p;
  if (i < 0) i += p;
  return i >= n ? p - i : i;
}

// Philox4x64-10 (Salmon et al. 2011; numpy.random.Philox's block function), counter c under key (k0, k1).
__device__ __forceinline__ void ph_philox(unsigned long long c[4], unsigned long long k0, unsigned long long k1) {
  const unsigned long long M0 = 0xD2E7470EE14C6C93ULL, M1 = 0xCA5A826395121157ULL;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += 0x9E3779B97F4A7C15ULL; k1 += 0xBB67AE8584CAA73BULL; }
    const unsigned long long lo0 = M0 * c[0], hi0 = __umul64hi(M0, c[0]);
    const unsigned long long lo1 = M1 * c[2], hi1 = __umul64hi(M1, c[2]);
    const unsigned long long n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
    c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
  }
}

__device__ __forceinline__ double ph_uniform(unsigned long long v) { return (double)(v >> 11) * 0x1.0p-53; }

__device__ __forceinline__ int ph_clamp255(int v) { return min(max(v, 0), 255); }

// Steps 1-4 of the contract for the pixel with linear index pix and value a.
__device__ int ph_pointwise(int a, const double* P, unsigned long long pix, unsigned long long key) {
  const int nb = (int)P[PH_P_BRIGHT], nc = (int)P[PH_P_CONTRAST], ng = (int)P[PH_P_NOISE], ns = (int)P[PH_P_SPECKLE];
  for (int r = 0; r < nb; ++r) a = ph_clamp255(a + (int)P[PH_P_BRIGHT + 1 + r]);
  for (int r = 0; r < nc; ++r) {
    const float al = (float)P[PH_P_CONTRAST + 1 + r];
    const float t = __fadd_rn(127.5f, __fmul_rn(al, __fsub_rn((float)a, 127.5f)));
    a = (int)fminf(fmaxf(t, 0.f), 255.f);
  }
  const int nr = max(ng, ns);
  if (nr == 0) return a;
  unsigned long long wd[2][4];
  for (int r = 0; r < nr; ++r) {
    wd[r][0] = pix; wd[r][1] = (unsigned long long)r; wd[r][2] = 0; wd[r][3] = 0;
    ph_philox(wd[r], key, 0ULL);
  }
  for (int r = 0; r < ng; ++r) {
    const double u1 = __dmul_rn((double)(wd[r][0] >> 11) + 1.0, 0x1.0p-53), u2 = ph_uniform(wd[r][1]);
    const double z = __dmul_rn(__dsqrt_rn(__dmul_rn(-2.0, log(u1))), cos(__dmul_rn(2.0 * 3.141592653589793, u2)));
    const double v = fmin(fmax(rint(__dmul_rn(P[PH_P_NOISE + 1 + r], z)), -255.0), 255.0);
    a = ph_clamp255(a + (int)v);
  }
  for (int r = 0; r < ns; ++r) {
    if (ph_uniform(wd[r][2]) < P[PH_P_SPECKLE + 1 + r]) {
      const double s = sin(__dmul_rn(1.5707963267948966, ph_uniform(wd[r][3])));
      a = ph_clamp255((int)rint(__dmul_rn(255.0, __dmul_rn(s, s))));
    }
  }
  return a;
}

__global__ void __launch_bounds__(PS_THREADS) photo_stage1_kernel(PhotoArgs a) {
  __shared__ float pw[PS_TH + 2][PS_TW + 2];
  __shared__ double P[PH_NPARAM];
  const int img = blockIdx.z, x0 = blockIdx.x * PS_TW, y0 = blockIdx.y * PS_TH, h = a.h, w = a.w;
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x < PH_NPARAM) P[threadIdx.x] = a.params[(size_t)img * PH_NPARAM + threadIdx.x];
  __syncthreads();
  const bool blur = P[PH_P_BLUR] != 0.0;
  const unsigned long long key = (unsigned long long)P[PH_P_KEY_LO] | ((unsigned long long)P[PH_P_KEY_HI] << 32);
  const size_t plane = (size_t)h * w;
  const uint8_t* src = a.in + (size_t)img * plane;
  for (int i = threadIdx.x; i < (PS_TH + 2) * (PS_TW + 2); i += PS_THREADS) {
    const int ry = i / (PS_TW + 2), rx = i - ry * (PS_TW + 2);
    const int y = y0 - 1 + ry, x = x0 - 1 + rx;
    const bool inner = ry >= 1 && ry <= PS_TH && rx >= 1 && rx <= PS_TW;
    if ((!blur && !inner) || y > h || x > w) continue;   // only y == h / x == w are read past the image
    const int gy = ph_reflect101(y, h), gx = ph_reflect101(x, w);
    const size_t o = (size_t)gy * w + gx;
    pw[ry][rx] = (float)ph_pointwise(src[o], P, (unsigned long long)o, key);
  }
  __syncthreads();
  uint8_t* dst = a.stage1 + (size_t)img * plane;
  for (int i = threadIdx.x; i < PS_TH * PS_TW; i += PS_THREADS) {
    const int oy = i / PS_TW, ox = i - oy * PS_TW, y = y0 + oy, x = x0 + ox;
    if (y >= h || x >= w) continue;
    int v;
    if (blur) {
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < 9; ++k) s = __fmaf_rn(pw[oy + k / 3][ox + k % 3], (float)P[PH_P_KERNEL + k], s);
      v = ph_clamp255((int)rintf(s));
    } else {
      v = (int)pw[oy + 1][ox + 1];
    }
    dst[(size_t)y * w + x] = (uint8_t)v;
  }
}

// cv2's drawing sine table: sin(i degrees) rounded to 7 decimals, as float.  No entry lies within 1e-6 of a rounding
// tie (tests/test_photometric.py), so the last bits of the device sine cannot change it.
__device__ __forceinline__ float ph_sin_table(int i) {
  const double s = sin(__dmul_rn((double)i, 3.141592653589793 / 180.0));
  return (float)__ddiv_rn(rint(__dmul_rn(s, 1e7)), 1e7);
}

// cv2's 8-connected fixed-point line from (x1, y1) to (x2, y2), value 255, clipped to the image.
__device__ void ph_line(uint8_t* m, int h, int w, long long x1, long long y1, long long x2, long long y2) {
  long long dx = x2 - x1, dy = y2 - y1;
  auto put = [&](long long x, long long y) {
    if (x >= 0 && x < w && y >= 0 && y < h) m[(size_t)y * w + x] = 255;
  };
  put((x2 + PH_XY_HALF) >> PH_XY_SHIFT, (y2 + PH_XY_HALF) >> PH_XY_SHIFT);
  if (llabs(dx) > llabs(dy)) {
    if (dx < 0) { long long t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; dy = -dy; }
    const long long step = (dy * 65536) / (llabs(dx) | 1), ecount = (x2 - x1) >> PH_XY_SHIFT;
    const long long x = (x1 + PH_XY_HALF) >> PH_XY_SHIFT, yy = y1 + PH_XY_HALF;
    for (long long k = 0; k <= ecount; ++k) put(x + k, (yy + k * step) >> PH_XY_SHIFT);
  } else {
    if (dy < 0) { long long t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; dx = -dx; }
    const long long step = (dx * 65536) / (llabs(dy) | 1), ecount = (y2 - y1) >> PH_XY_SHIFT;
    const long long xx = x1 + PH_XY_HALF, y = (y1 + PH_XY_HALF) >> PH_XY_SHIFT;
    for (long long k = 0; k <= ecount; ++k) put((xx + k * step) >> PH_XY_SHIFT, y + k);
  }
}

__global__ void __launch_bounds__(PE_THREADS) photo_ellipse_kernel(PhotoArgs a) {
  __shared__ long long vx[PE_MAXV], vy[PE_MAXV];
  __shared__ long long sp[PE_MAXSPAN][6];   // (y0, y1, x_left_chain, dx, x_right_chain, dx) at row y0
  __shared__ int s_nv, s_nsp;
  const int img = blockIdx.y, e = blockIdx.x, h = a.h, w = a.w;
  pdl_launch_dependents();
  pdl_wait();
  const double* P = a.params + (size_t)img * PH_NPARAM;
  if (P[PH_P_SHADE] == 0.0 || e >= (int)P[PH_P_N_ELLIPSES]) return;
  const int32_t* el = a.ellipses + ((size_t)img * a.max_ellipses + e) * 5;
  const int ax = el[0], ay = el[1], cx = el[2], cy = el[3];
  const int mr = max(ax, ay);
  // outside sample_photometric's bounds (the contract) an ellipse is not drawn
  if (ax < 0 || ay < 0 || cx < mr || cx + mr >= w || cy < mr || cy + mr >= h) return;
  int ang = el[4] % 360;
  if (ang < 0) ang += 360;
  const int step = mr < 3 ? 90 : mr < 10 ? 30 : mr < 15 ? 18 : 5;
  const int nraw = 360 / step + 1;
  if ((int)threadIdx.x < nraw) {
    const int t = min((int)threadIdx.x * step, 360);
    const double alpha = ph_sin_table(450 - ang), beta = ph_sin_table(ang);
    const double px = __dmul_rn((double)((long long)ax << PH_XY_SHIFT), (double)ph_sin_table(450 - t));
    const double py = __dmul_rn((double)((long long)ay << PH_XY_SHIFT), (double)ph_sin_table(t));
    const double X = __dsub_rn(__dadd_rn((double)((long long)cx << PH_XY_SHIFT), __dmul_rn(px, alpha)), __dmul_rn(py, beta));
    const double Y = __dadd_rn(__dadd_rn((double)((long long)cy << PH_XY_SHIFT), __dmul_rn(px, beta)), __dmul_rn(py, alpha));
    const long long qx = __double2ll_rn(__dmul_rn(X, 1.0 / 65536)) << PH_XY_SHIFT;
    const long long qy = __double2ll_rn(__dmul_rn(Y, 1.0 / 65536)) << PH_XY_SHIFT;
    vx[threadIdx.x] = qx + __double2ll_rn(__dsub_rn(X, (double)qx));
    vy[threadIdx.x] = qy + __double2ll_rn(__dsub_rn(Y, (double)qy));
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int n = 1;   // drop consecutive duplicates
    for (int i = 1; i < nraw; ++i)
      if (vx[i] != vx[n - 1] || vy[i] != vy[n - 1]) { vx[n] = vx[i]; vy[n] = vy[i]; ++n; }
    if (n == 1) {
      vx[0] = vx[1] = (long long)cx << PH_XY_SHIFT;
      vy[0] = vy[1] = (long long)cy << PH_XY_SHIFT;
      n = 2;
    }
    s_nv = n;
    // the spans of cv2's convex scan fill: two edge chains walk from the top vertex, sharing one vertex budget
    int nsp = 0;
    long long xmin = vx[0], xmax = vx[0];
    int imin = 0;
    for (int i = 1; i < n; ++i) {
      if (vy[i] < vy[imin]) imin = i;
      xmin = min(xmin, vx[i]);
      xmax = max(xmax, vx[i]);
    }
    if (n >= 3 && ((xmax + PH_XY_HALF) >> PH_XY_SHIFT) >= 0 && ((xmin + PH_XY_HALF) >> PH_XY_SHIFT) < w) {
      long long ymax = vy[0];
      for (int i = 1; i < n; ++i) ymax = max(ymax, vy[i]);
      const long long ymin = (vy[imin] + PH_XY_HALF) >> PH_XY_SHIFT;
      ymax = min((ymax + PH_XY_HALF) >> PH_XY_SHIFT, (long long)h - 1);
      int edges = n, idx[2] = {imin, imin};
      const int di[2] = {1, n - 1};
      long long ye[2] = {ymin, ymin}, ex[2] = {0, 0}, edx[2] = {0, 0};
      long long y = ymin;
      while (y <= ymax && nsp < PE_MAXSPAN) {
        for (int c = 0; c < 2; ++c) {
          if (y < ye[c]) continue;
          int i0 = idx[c], i1 = (i0 + di[c]) % n;
          while (true) {
            if (--edges < 0) break;
            const long long ty = (vy[i1] + PH_XY_HALF) >> PH_XY_SHIFT;
            if (ty > y) {
              ye[c] = ty; ex[c] = vx[i0]; idx[c] = i1;
              edx[c] = ((vx[i1] - vx[i0]) * 2 + (ty - y)) / (2 * (ty - y));
              break;
            }
            i0 = i1;
            i1 = (i1 + di[c]) % n;
          }
        }
        if (edges < 0) break;
        const long long y1 = min(min(ye[0], ye[1]), ymax + 1);
        sp[nsp][0] = y; sp[nsp][1] = y1; sp[nsp][2] = ex[0]; sp[nsp][3] = edx[0]; sp[nsp][4] = ex[1]; sp[nsp][5] = edx[1];
        ++nsp;
        ex[0] += edx[0] * (y1 - y);
        ex[1] += edx[1] * (y1 - y);
        y = y1;
      }
    }
    s_nsp = nsp;
  }
  __syncthreads();
  uint8_t* m = a.mask + (size_t)img * h * w;
  const int n = s_nv, nsp = s_nsp;
  for (int j = threadIdx.x; j < n; j += PE_THREADS) {
    const int p = j == 0 ? n - 1 : j - 1;
    ph_line(m, h, w, vx[p], vy[p], vx[j], vy[j]);
  }
  if (nsp == 0) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long ybeg = max(sp[0][0], 0LL), yend = sp[nsp - 1][1];
  int s = 0;
  for (long long y = ybeg + warp; y < yend; y += PE_THREADS / 32) {
    while (y >= sp[s][1]) ++s;
    long long l = sp[s][2] + (y - sp[s][0]) * sp[s][3], r = sp[s][4] + (y - sp[s][0]) * sp[s][5];
    if (l > r) { const long long t = l; l = r; r = t; }
    const long long x1 = (l + PH_XY_HALF) >> PH_XY_SHIFT, x2 = (r + PH_XY_HALF) >> PH_XY_SHIFT;
    if (x2 < 0 || x1 >= w) continue;
    for (long long x = max(x1, 0LL) + lane; x <= min(x2, (long long)w - 1); x += 32) m[(size_t)y * w + x] = 255;
  }
}

__device__ __forceinline__ void ph_load_taps(float* t, const PhotoArgs& a, int img, int ks) {
  for (int k = threadIdx.x; k < PH_KPAD; k += blockDim.x) t[k] = k < ks ? a.taps[(size_t)img * PH_MAX_KSIZE + k] : 0.f;
}

__global__ void __launch_bounds__(PR_ROWS * 32) photo_blur_row_kernel(PhotoArgs a) {
  __shared__ __align__(16) float s[PR_ROWS][PR_LEN];
  __shared__ float taps[PH_KPAD];
  const int img = blockIdx.z, x0 = blockIdx.x * PR_W, yb = blockIdx.y * PR_ROWS, h = a.h, w = a.w;
  pdl_launch_dependents();
  pdl_wait();
  const double* P = a.params + (size_t)img * PH_NPARAM;
  if (P[PH_P_SHADE] == 0.0) return;
  const int ks = (int)P[PH_P_KSIZE], R = ks / 2, kp = (ks + 3) & ~3;
  ph_load_taps(taps, a, img, ks);
  const uint8_t* m = a.mask + (size_t)img * h * w;
  for (int i = threadIdx.x; i < PR_ROWS * PR_LEN; i += PR_ROWS * 32) {
    const int r = i / PR_LEN, j = i - r * PR_LEN, y = yb + r;
    float v = 0.f;
    if (y < h && j < PR_W + 2 * R) v = (float)m[(size_t)y * w + ph_reflect101(x0 - R + j, w)];
    s[r][j] = v;
  }
  __syncthreads();
  const int r = threadIdx.x >> 5, b = (threadIdx.x & 31) * 4, y = yb + r;
  if (y >= h) return;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  float4 lo = *reinterpret_cast<const float4*>(&s[r][b]), hi = *reinterpret_cast<const float4*>(&s[r][b + 4]);
  for (int k = 0; k < kp; k += 4) {
    const float v[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const float t = taps[k + kk];
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[q] = __fadd_rn(acc[q], __fmul_rn(t, v[q + kk]));
    }
    lo = hi;
    hi = *reinterpret_cast<const float4*>(&s[r][b + k + 8]);
  }
  float* dst = a.rowblur + ((size_t)img * h + y) * w;
#pragma unroll
  for (int q = 0; q < 4; ++q)
    if (x0 + b + q < w) dst[x0 + b + q] = acc[q];
}

// The reference's chain from a stage-1 byte and the blurred mask to the output byte (see the header comment).
__device__ __forceinline__ uint8_t ph_shade(int a, float m, float t) {
  const float x = __fmul_rn(__fdiv_rn((float)a, 255.f), 255.f);
  const float s = __fmul_rn(x, __fsub_rn(1.f, __fdiv_rn(__fmul_rn(t, m), 255.f)));
  const float c = fminf(fmaxf(s, 0.f), 255.f);
  return (uint8_t)(int)__dmul_rn((double)__fdiv_rn(c, 255.f), 255.0);
}

__global__ void __launch_bounds__(PC_W * (PC_H / PC_Q)) photo_blur_col_kernel(PhotoArgs a) {
  __shared__ float s[PC_LEN][PC_W];
  __shared__ float taps[PH_KPAD];
  const int img = blockIdx.z, x0 = blockIdx.x * PC_W, y0 = blockIdx.y * PC_H, h = a.h, w = a.w;
  const int tx = threadIdx.x % PC_W, b = (threadIdx.x / PC_W) * PC_Q, x = x0 + tx;
  pdl_launch_dependents();
  pdl_wait();
  const double* P = a.params + (size_t)img * PH_NPARAM;
  const size_t plane = (size_t)h * w;
  const uint8_t* s1 = a.stage1 + (size_t)img * plane;
  uint8_t* out = a.out + (size_t)img * plane;
  if (P[PH_P_SHADE] == 0.0) {
    for (int q = 0; q < PC_Q; ++q)
      if (y0 + b + q < h && x < w) out[(size_t)(y0 + b + q) * w + x] = s1[(size_t)(y0 + b + q) * w + x];
    return;
  }
  const int ks = (int)P[PH_P_KSIZE], R = ks / 2, kp = (ks + 3) & ~3;
  ph_load_taps(taps, a, img, ks);
  const float* rb = a.rowblur + (size_t)img * plane;
  for (int i = threadIdx.x; i < PC_LEN * PC_W; i += blockDim.x) {
    const int rr = i / PC_W, c = i - rr * PC_W;
    float v = 0.f;
    if (x0 + c < w && rr < PC_H + 2 * R) v = rb[(size_t)ph_reflect101(y0 - R + rr, h) * w + x0 + c];
    s[rr][c] = v;
  }
  __syncthreads();
  if (x >= w || y0 + b >= h) return;
  float acc[PC_Q];
#pragma unroll
  for (int q = 0; q < PC_Q; ++q) acc[q] = 0.f;
  for (int k = 0; k < kp; k += 4) {
    float v[PC_Q + 3];
#pragma unroll
    for (int j = 0; j < PC_Q + 3; ++j) v[j] = s[b + k + j][tx];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const float t = taps[k + kk];
#pragma unroll
      for (int q = 0; q < PC_Q; ++q) acc[q] = __fadd_rn(acc[q], __fmul_rn(t, v[q + kk]));
    }
  }
  const float t = (float)P[PH_P_TRANSPARENCY];
#pragma unroll
  for (int q = 0; q < PC_Q; ++q) {
    const int y = y0 + b + q;
    if (y < h) out[(size_t)y * w + x] = ph_shade(s1[(size_t)y * w + x], acc[q], t);
  }
}

}  // namespace ltr
