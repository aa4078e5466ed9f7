// Line-signature attention on tensor cores (sm_90a): softmax(q k^T) v over the L_i lines of ONE
// image, per head, no mask (attention(), models/line_transformer.py:132-136; 1/8 is folded into
// W_q and the heads are head-major, see ltr_create).
//
// CTA = (128-query tile, head, image), 256 threads = two warpgroups of 64 query rows each; the
// accumulators live in registers (wgmma fragment: a thread holds two rows, a quad of threads a row).
// Per key tile of 128 lines:
//   * q, k, v arrive as the split-bf16 tile image the qkv GEMM epilogue wrote (k-block h = q of head h,
//     4 + h = k, 8 + h = v).  Images of the batch are not 128-row aligned in the row space, so the
//     operand tiles are assembled from 16-byte chunks with cp.async (re-swizzled for the new row
//     phase, rows past the image zero-filled) - no conversion, no registers, all copies in flight;
//     v lands behind the S MMA.  V is staged exactly like K ([keys x 64 dims]) and consumed as an
//     MN-major B operand - no transpose anywhere.
//   * S = Q K^T      wgmma (M64 N128 K64 per warpgroup, 3 split products)
//   * p = exp(s - m), row sums in registers; P written as the A operand of the second MMA
//     (re-using the Q/K shared memory, which is dead once S is complete)
//   * O += P V       wgmma (M64 N64 K128 per warpgroup), accumulated in registers across key tiles
// Images with more than 128 lines run a first pass that only computes the row maxima (S is
// recomputed in the second pass - QK^T is 1/3 of the work and far from the bottleneck), so no
// rescaling of the accumulator is ever needed.  Output: columns [out_k0, out_k0+256) of a split-bf16
// activation image (the second half of the signature MLP input; the `merge` projection is folded into W1).
#pragma once
#include <cstdlib>
#include <cstring>
#include "act_img.cuh"
#include "common.cuh"
#include "ptx_sm90.cuh"

namespace ltr {

struct SigAttnSmem {
  static constexpr int QK = 64 * 1024;   // Q hi/lo + K hi/lo (4 x 16 KB); later P hi/lo (2 x 32 KB)
  static constexpr int V = 32 * 1024;    // V hi/lo: [128 keys x 64 d] each
  static constexpr int OFF_BAR = QK + V;
  static constexpr int TOTAL = OFF_BAR + 64 + 1024;
};

// the S accumulator of one warpgroup (64 rows x 128 keys) from the staged Q and K tiles
__device__ __forceinline__ void attn_qk(float (&d)[64], uint32_t qh, uint32_t ql, uint32_t kh, uint32_t kl) {
  ptx::wg_fence_regs(d);
  ptx::wg_fence();
#pragma unroll
  for (int k16 = 0; k16 < 4; ++k16) {
    const uint32_t ko = k16 * 32;
    ptx::wgmma_ss_n128(d, ptx::make_sw128_kmajor_desc(ql + ko, 1024), ptx::make_sw128_kmajor_desc(kh + ko, 1024), k16 != 0);
    ptx::wgmma_ss_n128(d, ptx::make_sw128_kmajor_desc(qh + ko, 1024), ptx::make_sw128_kmajor_desc(kl + ko, 1024), 1);
    ptx::wgmma_ss_n128(d, ptx::make_sw128_kmajor_desc(qh + ko, 1024), ptx::make_sw128_kmajor_desc(kh + ko, 1024), 1);
  }
  ptx::wg_commit();
  ptx::wg_wait<0>();
  ptx::wg_fence_regs(d);
}

__global__ void __launch_bounds__(256) sig_attention_tc_kernel(ActImg qkv, ActImg out, int out_k0,
                                                                const int* __restrict__ cu, int lpi) {
  using S = SigAttnSmem;
  // Uniform batches know their line range without touching memory; for var-len batches `cu` is read
  // only AFTER griddepcontrol.wait (nothing a preceding kernel on the stream wrote is guaranteed
  // visible before it - several kernels of the chain can be resident ahead of their wait at once).
  int lb = blockIdx.z * lpi, le = lb + lpi;
  int L = lpi;
  const int q0 = blockIdx.x * 128;
  if (!cu && q0 >= L) return;
  const int h = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;
  const int row_a = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // query rows row_a and row_a + 8 of this thread
  const int cq = 2 * (lane & 3);                                 // first of the thread's two columns per 8-column group
  if (tid == 0) LTR_DBG_STAMP(30);
  pdl_launch_dependents();

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t raw = ptx::smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw & 1023u)) & 1023u);
  uint8_t* q_hi = smem;                 // [128 x 64]
  uint8_t* q_lo = smem + 16384;
  uint8_t* k_hi = smem + 32768;         // [128 keys x 64]
  uint8_t* k_lo = smem + 49152;
  uint8_t* p_hi = smem;                 // [2 k-blocks][128 x 64 keys]  (aliases q/k)
  uint8_t* p_lo = smem + 32768;
  uint8_t* v_hi = smem + S::QK;         // [128 keys x 64 d]
  uint8_t* v_lo = v_hi + 16384;
  uint64_t* ld_qk = reinterpret_cast<uint64_t*>(smem + S::OFF_BAR);   // TMA path: q and k tiles landed
  uint64_t* ld_v = ld_qk + 1;                                         // TMA path: v tile landed

  if (tid == 0) {
    ptx::mbar_init(ld_qk, 1);
    ptx::mbar_init(ld_v, 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();   // qkv of this layer is complete; the previous reader of the output image is done
  if (tid == 0) LTR_DBG_STAMP(31);
  if (cu) {
    lb = cu[blockIdx.z]; le = cu[blockIdx.z + 1];
    L = le - lb;
    if (q0 >= L) return;   // uniform per CTA
  }

  // [128 rows x 64] operand tile (hi and lo plane) <- rows row0.. of this image, k-block kb of the qkv image:
  // chunk f = tid + 256 i -> row f/8, 16-byte chunk f%8 (8 lanes read one 128-byte image line)
  auto stage_tile = [&](int row0, int kb, uint8_t* hi, uint8_t* lo) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int f = tid + 256 * i, r = f >> 3, c = f & 7;
      const bool ok = row0 + r < L;
      const int gr = lb + row0 + r;
      const size_t src = ok ? ((size_t)(gr >> 7) * qkv.kblocks + kb) * (IMG_TILE_ELEMS * 2) + ptx::sw128_offset(gr & 127, c * 8) : 0;
      const uint32_t dst = ptx::sw128_offset(r, c * 8);
      ptx::cp_async16(hi + dst, reinterpret_cast<const uint8_t*>(qkv.hi) + src, ok ? 16u : 0u);
      ptx::cp_async16(lo + dst, reinterpret_cast<const uint8_t*>(qkv.lo) + src, ok ? 16u : 0u);
    }
  };
  const uint32_t qh = ptx::smem_u32(q_hi) + wg * 8192, ql = ptx::smem_u32(q_lo) + wg * 8192;
  const uint32_t kh = ptx::smem_u32(k_hi), kl = ptx::smem_u32(k_lo);
  // row maxima of this thread's two rows over the valid key columns of S (a quad shares a row)
  auto row_max = [&](const float (&sd)[64], int kn, float& m0, float& m1) {
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e)
        if (8 * j + cq + e < kn) {
          m0 = fmaxf(m0, sd[4 * j + e]);
          m1 = fmaxf(m1, sd[4 * j + 2 + e]);
        }
#pragma unroll
    for (int o = 1; o < 4; o <<= 1) {
      m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, o));
      m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, o));
    }
  };

  const int n_kt = (L + 127) / 128;
  // An image of exactly 128 lines that starts on a 128-row tile of the qkv image (every uniform L = 128 batch): its
  // q, k, v operand tiles ARE tiles of that image - six 16 KB bulk copies (TMA) by one thread instead of 24 cp.async
  // per thread; v still lands behind the S MMA.  Single key tile: the shared memory is written exactly once.
  const bool tma = L == 128 && ((lb & 127) == 0);
  float m0 = -INFINITY, m1 = -INFINITY;
  float sd[64];
  if (n_kt > 1) {
    // ---- pass 1: row maxima over all key tiles
    for (int kt = 0; kt < n_kt; ++kt) {
      const int k0 = kt * 128, kn = min(128, L - k0);
      stage_tile(q0, h, q_hi, q_lo);
      stage_tile(k0, 4 + h, k_hi, k_lo);
      ptx::cp_async_wait_all();
      ptx::fence_proxy_async_smem();
      __syncthreads();
      attn_qk(sd, qh, ql, kh, kl);
      row_max(sd, kn, m0, m1);
      __syncthreads();
    }
  }
  float l0 = 0.f, l1 = 0.f;
  float od[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) od[i] = 0.f;
  constexpr float LOG2E = 1.4426950408889634f;
  for (int kt = 0; kt < n_kt; ++kt) {
    const int k0 = kt * 128, kn = min(128, L - k0);
    if (tid == 0) LTR_DBG_STAMP(32);
    if (tma) {
      if (tid == 0) {
        const size_t t0 = (size_t)(lb >> 7) * qkv.kblocks * IMG_TILE_ELEMS;
        const size_t tq = t0 + (size_t)h * IMG_TILE_ELEMS, tk = t0 + (size_t)(4 + h) * IMG_TILE_ELEMS, tv = t0 + (size_t)(8 + h) * IMG_TILE_ELEMS;
        ptx::mbar_arrive_expect_tx(ld_qk, 4 * 16384);
        ptx::bulk_g2s(q_hi, qkv.hi + tq, 16384, ld_qk);
        ptx::bulk_g2s(q_lo, qkv.lo + tq, 16384, ld_qk);
        ptx::bulk_g2s(k_hi, qkv.hi + tk, 16384, ld_qk);
        ptx::bulk_g2s(k_lo, qkv.lo + tk, 16384, ld_qk);
        ptx::mbar_arrive_expect_tx(ld_v, 2 * 16384);
        ptx::bulk_g2s(v_hi, qkv.hi + tv, 16384, ld_v);
        ptx::bulk_g2s(v_lo, qkv.lo + tv, 16384, ld_v);
      }
      ptx::mbar_wait(ld_qk, 0);
    } else {
      stage_tile(q0, h, q_hi, q_lo);
      stage_tile(k0, 4 + h, k_hi, k_lo);
      ptx::cp_async_commit();
      stage_tile(k0, 8 + h, v_hi, v_lo);
      ptx::cp_async_commit();
      ptx::cp_async_wait_group<1>();   // q and k have landed; v is still in flight behind the S MMA
      ptx::fence_proxy_async_smem();
    }
    __syncthreads();
    attn_qk(sd, qh, ql, kh, kl);
    if (tid == 0) LTR_DBG_STAMP(35);
    if (n_kt == 1) row_max(sd, kn, m0, m1);
    __syncthreads();   // both warpgroups are done reading Q / K: P may overwrite them
    // p = exp(s - m) -> P operand: key column c of row r at k-block c / 64 of the P tile
    const float mb0 = m0 * LOG2E, mb1 = m1 * LOG2E;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int c = 8 * j + cq;
      const bool v0 = c < kn, v1 = c + 1 < kn;
      const float p00 = v0 ? ptx::ex2_approx(fmaf(sd[4 * j], LOG2E, -mb0)) : 0.f;
      const float p01 = v1 ? ptx::ex2_approx(fmaf(sd[4 * j + 1], LOG2E, -mb0)) : 0.f;
      const float p10 = v0 ? ptx::ex2_approx(fmaf(sd[4 * j + 2], LOG2E, -mb1)) : 0.f;
      const float p11 = v1 ? ptx::ex2_approx(fmaf(sd[4 * j + 3], LOG2E, -mb1)) : 0.f;
      l0 += p00 + p01;
      l1 += p10 + p11;
      uint32_t hh, ll;
      const uint32_t off0 = (c >> 6) * 16384 + ptx::sw128_offset(row_a, c & 63);
      const uint32_t off1 = (c >> 6) * 16384 + ptx::sw128_offset(row_a + 8, c & 63);
      ptx::split2_bf16(p00, p01, hh, ll);
      *reinterpret_cast<uint32_t*>(p_hi + off0) = hh;
      *reinterpret_cast<uint32_t*>(p_lo + off0) = ll;
      ptx::split2_bf16(p10, p11, hh, ll);
      *reinterpret_cast<uint32_t*>(p_hi + off1) = hh;
      *reinterpret_cast<uint32_t*>(p_lo + off1) = ll;
    }
    if (tma) ptx::mbar_wait(ld_v, 0);
    else ptx::cp_async_wait_group<0>();   // v
    ptx::fence_proxy_async_smem();
    __syncthreads();
    {   // O += P V    (B = V as an MN-major operand: [K = keys][N = 64 dims])
      const uint32_t ph = ptx::smem_u32(p_hi) + wg * 8192, pl = ptx::smem_u32(p_lo) + wg * 8192;
      const uint32_t vh = ptx::smem_u32(v_hi), vl = ptx::smem_u32(v_lo);
      ptx::wg_fence_regs(od);
      ptx::wg_fence();
#pragma unroll
      for (int kb = 0; kb < 2; ++kb) {
#pragma unroll
        for (int k16 = 0; k16 < 4; ++k16) {
          const uint32_t pa = kb * 16384 + k16 * 32;          // A: 16 keys = 32 bytes along K
          const uint32_t va = (kb * 4 + k16) * 2048;          // B: 16 key rows of 128 bytes
          ptx::wgmma_ss_n64_tb(od, ptx::make_sw128_kmajor_desc(pl + pa, 1024), ptx::make_sw128_mnmajor_desc(vh + va, 1024, 1024), 1);
          ptx::wgmma_ss_n64_tb(od, ptx::make_sw128_kmajor_desc(ph + pa, 1024), ptx::make_sw128_mnmajor_desc(vl + va, 1024, 1024), 1);
          ptx::wgmma_ss_n64_tb(od, ptx::make_sw128_kmajor_desc(ph + pa, 1024), ptx::make_sw128_mnmajor_desc(vh + va, 1024, 1024), 1);
        }
      }
      ptx::wg_commit();
      ptx::wg_wait<0>();
      ptx::wg_fence_regs(od);
    }
    __syncthreads();   // P, V shared memory may be overwritten by the next key tile
    if (tid == 0) LTR_DBG_STAMP(37);
  }
  // ---- epilogue: o / l -> image (this thread: rows row_a, row_a + 8, dims 8 j + cq, + 1)
  {
#pragma unroll
    for (int o = 1; o < 4; o <<= 1) {
      l0 += __shfl_xor_sync(0xffffffffu, l0, o);
      l1 += __shfl_xor_sync(0xffffffffu, l1, o);
    }
    const float inv0 = 1.f / l0, inv1 = 1.f / l1;
    if (tma) {
      // aligned 128-line image: this CTA's output (128 rows x 64 head dims) is ONE k-block tile of the output image -
      // stage hi / lo planes in tile layout (the P operand's memory is dead: the PV MMAs have completed) and store each
      // with one 16 KB bulk copy
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        uint32_t hh, ll;
        ptx::split2_bf16(od[4 * j] * inv0, od[4 * j + 1] * inv0, hh, ll);
        *reinterpret_cast<uint32_t*>(smem + ptx::sw128_offset(row_a, 8 * j + cq)) = hh;
        *reinterpret_cast<uint32_t*>(smem + 16384 + ptx::sw128_offset(row_a, 8 * j + cq)) = ll;
        ptx::split2_bf16(od[4 * j + 2] * inv1, od[4 * j + 3] * inv1, hh, ll);
        *reinterpret_cast<uint32_t*>(smem + ptx::sw128_offset(row_a + 8, 8 * j + cq)) = hh;
        *reinterpret_cast<uint32_t*>(smem + 16384 + ptx::sw128_offset(row_a + 8, 8 * j + cq)) = ll;
      }
      ptx::fence_proxy_async_smem();
      __syncthreads();
      if (tid == 0) {
        const size_t toff = ((size_t)(lb >> 7) * out.kblocks + (out_k0 >> 6) + h) * IMG_TILE_ELEMS;
        ptx::bulk_s2g(out.hi + toff, smem, 16384);
        ptx::bulk_s2g(out.lo + toff, smem + 16384, 16384);
        ptx::bulk_commit();
        // the copies only have to be done READING this CTA's shared memory before it exits; their global writes are
        // complete (and visible to the next kernel behind griddepcontrol.wait) when the grid is
        ptx::bulk_wait_read_all();
      }
    } else {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int r = row_a + 8 * e;
        if (q0 + r >= L) continue;
        const float inv = e ? inv1 : inv0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          uint32_t hh, ll;
          ptx::split2_bf16(od[4 * j + 2 * e] * inv, od[4 * j + 2 * e + 1] * inv, hh, ll);
          const size_t i = img_index(out, lb + q0 + r, out_k0 + h * 64 + 8 * j + cq);
          *reinterpret_cast<uint32_t*>(out.hi + i) = hh;
          *reinterpret_cast<uint32_t*>(out.lo + i) = ll;
        }
      }
    }
  }
  if (tid == 0) LTR_DBG_STAMP(38);
}

// ------------------------------------------------------------------ uniform batches of 128-line images
// Image i is exactly tile i of the qkv image, so one (image, head) unit is six 16 KB bulk copies and one 128-query tile.
// One persistent CTA per SM walks its images (b, b + grid, ...) and all four heads of each, 384 threads:
//   * a producer warpgroup (one lane issues the copies) fills a two-stage ring, so head h + 1 - or the next image's
//     head 0 - lands while head h computes; q and k complete on full_qk, v on full_v (S does not wait for v);
//   * two consumer warpgroups of 64 query rows each run S -> softmax -> PV on their own: the split P is the register A
//     fragment of the PV wgmma (the S accumulator layout is the A-fragment layout), so nothing is written to shared
//     memory and there is no barrier across warpgroups.  A stage is released (8 warp arrivals on empty) as soon as
//     its PV MMAs have completed;
//   * each consumer warp stages its 16 output rows x 64 head dims - one contiguous 2 KB piece of the output tile per
//     plane - and bulk-stores them itself.
// Per element this is the instruction sequence of sig_attention_tc_kernel's single-key-tile path (same MMA products in
// the same order, same softmax and split), so the output is bit-identical to it.
struct SigAttnPipeSmem {
  static constexpr int TILE = 16384;             // [128 x 64] bf16, one plane
  static constexpr int STAGE = 6 * TILE;         // q hi/lo, k hi/lo, v hi/lo
  static constexpr int STAGES = 2;
  static constexpr int STG_WARP = 2 * 2048;      // 16 rows x 64 dims, hi and lo
  static constexpr int OFF_STG = STAGES * STAGE;
  static constexpr int OFF_BAR = OFF_STG + 8 * STG_WARP;
  static constexpr int TOTAL = OFF_BAR + 64 + 1024;   // + alignment slack
};

__global__ void __launch_bounds__(384, 1) sig_attention_pipe_kernel(ActImg qkv, ActImg out, int out_k0, int n_images) {
  using S = SigAttnPipeSmem;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t raw = ptx::smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S::OFF_BAR);
  uint64_t* full_qk = bars;        // [2] q and k of the stage have landed
  uint64_t* full_v = bars + 2;     // [2] v of the stage has landed
  uint64_t* empty = bars + 4;      // [2] the stage's MMAs are done (8 consumer warps)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  pdl_launch_dependents();
  if (tid == 0) {
    for (int s = 0; s < S::STAGES; ++s) {
      ptx::mbar_init(&full_qk[s], 1);
      ptx::mbar_init(&full_v[s], 1);
      ptx::mbar_init(&empty[s], 8);
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ---------------------------------------------------------------- TMA producer
    ptx::setmaxnreg_dec<40>();
    if (warp == 8 && lane == 0) {
      pdl_wait();   // qkv of this layer is complete
      uint32_t it = 0;
      for (int img = blockIdx.x; img < n_images; img += gridDim.x)
        for (int h = 0; h < 4; ++h, ++it) {
          const int s = it & 1;
          ptx::mbar_wait(&empty[s], ((it >> 1) & 1) ^ 1);
          uint8_t* st = smem + s * S::STAGE;
          const size_t t0 = (size_t)img * qkv.kblocks * IMG_TILE_ELEMS;
          const size_t tq = t0 + (size_t)h * IMG_TILE_ELEMS, tk = t0 + (size_t)(4 + h) * IMG_TILE_ELEMS,
                       tv = t0 + (size_t)(8 + h) * IMG_TILE_ELEMS;
          ptx::mbar_arrive_expect_tx(&full_qk[s], 4 * S::TILE);
          ptx::bulk_g2s(st, qkv.hi + tq, S::TILE, &full_qk[s]);
          ptx::bulk_g2s(st + S::TILE, qkv.lo + tq, S::TILE, &full_qk[s]);
          ptx::bulk_g2s(st + 2 * S::TILE, qkv.hi + tk, S::TILE, &full_qk[s]);
          ptx::bulk_g2s(st + 3 * S::TILE, qkv.lo + tk, S::TILE, &full_qk[s]);
          ptx::mbar_arrive_expect_tx(&full_v[s], 2 * S::TILE);
          ptx::bulk_g2s(st + 4 * S::TILE, qkv.hi + tv, S::TILE, &full_v[s]);
          ptx::bulk_g2s(st + 5 * S::TILE, qkv.lo + tv, S::TILE, &full_v[s]);
        }
    }
  } else {
    // ---------------------------------------------------------------- consumers (2 warpgroups x 64 query rows)
    ptx::setmaxnreg_inc<232>();
    pdl_wait();   // the previous kernel may still read the output image's columns this kernel writes
    const int wg = warp >> 2;
    const int r0 = lane >> 2, cq = 2 * (lane & 3);   // rows 16 warp + r0 and + 8 of the tile, columns 8 j + cq, + 1
    uint8_t* stg = smem + S::OFF_STG + warp * S::STG_WARP;   // hi plane, lo plane 2 KB on
    constexpr float LOG2E = 1.4426950408889634f;
    uint32_t it = 0;
    for (int img = blockIdx.x; img < n_images; img += gridDim.x)
      for (int h = 0; h < 4; ++h, ++it) {
        const int s = it & 1;
        const uint32_t par = (it >> 1) & 1;
        const uint32_t sb = ptx::smem_u32(smem + s * S::STAGE);
        float sd[64];
        ptx::mbar_wait(&full_qk[s], par);
        attn_qk(sd, sb + wg * 8192, sb + S::TILE + wg * 8192, sb + 2 * S::TILE, sb + 3 * S::TILE);
        float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            m0 = fmaxf(m0, sd[4 * j + e]);
            m1 = fmaxf(m1, sd[4 * j + 2 + e]);
          }
#pragma unroll
        for (int o = 1; o < 4; o <<= 1) {
          m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, o));
          m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, o));
        }
        // p = exp(s - m) -> A fragments of the PV MMA: K = 16 step kk takes the accumulator groups 2 kk (a[0], a[1])
        // and 2 kk + 1 (a[2], a[3]), rows r0 and r0 + 8 each
        float l0 = 0.f, l1 = 0.f;
        uint32_t ah[8][4], al[8][4];
        const float mb0 = m0 * LOG2E, mb1 = m1 * LOG2E;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float p00 = ptx::ex2_approx(fmaf(sd[4 * j], LOG2E, -mb0));
          const float p01 = ptx::ex2_approx(fmaf(sd[4 * j + 1], LOG2E, -mb0));
          const float p10 = ptx::ex2_approx(fmaf(sd[4 * j + 2], LOG2E, -mb1));
          const float p11 = ptx::ex2_approx(fmaf(sd[4 * j + 3], LOG2E, -mb1));
          l0 += p00 + p01;
          l1 += p10 + p11;
          ptx::split2_bf16(p00, p01, ah[j >> 1][2 * (j & 1)], al[j >> 1][2 * (j & 1)]);
          ptx::split2_bf16(p10, p11, ah[j >> 1][2 * (j & 1) + 1], al[j >> 1][2 * (j & 1) + 1]);
        }
        // O = P V    (B = V as an MN-major operand: [K = keys][N = 64 dims], 16 key rows of 128 bytes per K step)
        // The accumulator starts from +0 held in registers, as in sig_attention_tc_kernel.  With a literal 0 ptxas drops
        // the C input of the first MMA, which would turn an output whose products are all -0 into -0 instead of +0.
        const float zero = 0.f * l0;   // l0 >= 1
        float od[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) od[i] = zero;
        const uint32_t vh = sb + 4 * S::TILE, vl = sb + 5 * S::TILE;
        ptx::mbar_wait(&full_v[s], par);
        ptx::wg_fence_regs(od);
        ptx::wg_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
          const uint32_t va = kk * 2048;
          ptx::wgmma_rs_n64_tb(od, al[kk], ptx::make_sw128_mnmajor_desc(vh + va, 1024, 1024), 1);
          ptx::wgmma_rs_n64_tb(od, ah[kk], ptx::make_sw128_mnmajor_desc(vl + va, 1024, 1024), 1);
          ptx::wgmma_rs_n64_tb(od, ah[kk], ptx::make_sw128_mnmajor_desc(vh + va, 1024, 1024), 1);
        }
        ptx::wg_commit();
        ptx::wg_wait<0>();
        ptx::wg_fence_regs(od);
        if (lane == 0) ptx::mbar_arrive(&empty[s]);   // this warpgroup is done reading the stage
        // ---- o / l -> this warp's 16 rows of output tile (img, out_k0 / 64 + h)
#pragma unroll
        for (int o = 1; o < 4; o <<= 1) {
          l0 += __shfl_xor_sync(0xffffffffu, l0, o);
          l1 += __shfl_xor_sync(0xffffffffu, l1, o);
        }
        const float inv0 = 1.f / l0, inv1 = 1.f / l1;
        if (lane == 0) ptx::bulk_wait_read_all();   // the previous head's store is done reading the staging block
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          uint32_t hh, ll;
          ptx::split2_bf16(od[4 * j] * inv0, od[4 * j + 1] * inv0, hh, ll);
          *reinterpret_cast<uint32_t*>(stg + ptx::sw128_offset(r0, 8 * j + cq)) = hh;
          *reinterpret_cast<uint32_t*>(stg + 2048 + ptx::sw128_offset(r0, 8 * j + cq)) = ll;
          ptx::split2_bf16(od[4 * j + 2] * inv1, od[4 * j + 3] * inv1, hh, ll);
          *reinterpret_cast<uint32_t*>(stg + ptx::sw128_offset(r0 + 8, 8 * j + cq)) = hh;
          *reinterpret_cast<uint32_t*>(stg + 2048 + ptx::sw128_offset(r0 + 8, 8 * j + cq)) = ll;
        }
        ptx::fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) {
          // rows 16 warp .. + 15 of a SWIZZLE_128B tile are its bytes [2048 warp, 2048 warp + 2048)
          const size_t toff = ((size_t)img * out.kblocks + (out_k0 >> 6) + h) * IMG_TILE_ELEMS + (size_t)warp * 1024;
          ptx::bulk_s2g(out.hi + toff, stg, 2048);
          ptx::bulk_s2g(out.lo + toff, stg + 2048, 2048);
          ptx::bulk_commit();
        }
      }
    if (lane == 0) ptx::bulk_wait<0>();   // the staging stays allocated, and the writes done, until the stores complete
  }
}

// LTR_ATTN_PIPE=0 keeps every batch on sig_attention_tc_kernel (A/B runs and the bit-identity tests); read at every
// call so that one process can run both kernels.
inline bool attn_pipe_enabled() {
  const char* e = std::getenv("LTR_ATTN_PIPE");
  return !(e && std::strcmp(e, "0") == 0);
}

inline int launch_sig_attention_tc(ActImg qkv, ActImg out, int out_k0, const int* cu, int lpi, int max_l,
                                   int n_images, cudaStream_t s) {
  if (max_l <= 0 || n_images <= 0) return 0;
  if (!cu && lpi == 128 && attn_pipe_enabled()) {
    const int grid = std::min(n_images, device_sm_count());
    return launch(KC_SIG_ATTN, true, sig_attention_pipe_kernel, dim3(grid), dim3(384), SigAttnPipeSmem::TOTAL, s, qkv, out,
                  out_k0, n_images);
  }
  dim3 grid(cdiv(max_l, 128), 4, n_images);
  return launch(KC_SIG_ATTN, true, sig_attention_tc_kernel, grid, dim3(256), SigAttnSmem::TOTAL, s, qkv, out, out_k0, cu, lpi);
}

}  // namespace ltr
