// Fused token stage of the line-descriptor forward (sm_90a, wgmma + TMA).
//
// One persistent CTA per SM walks tiles of LPT = floor(128 / T) whole lines (LPT*T <= 128 token
// rows).  Per tile, entirely on chip:
//   P0  3 -> 32 (+ReLU) on CUDA cores                                        -> h32  (registers, split-bf16)
//   L2  32 -> 64 (+ReLU)    wgmma (N = 64, two K steps)                      -> h64
//   L3  64 -> 128 (+ReLU)   wgmma                                            -> h128
//   L4  128 -> 256 (+ReLU)  wgmma, two n-blocks of 128                       -> h256
//   L5  256 -> 256          wgmma, epilogue adds the sampled descriptors     -> x = desc + wpe (fp32, smem)
//   CLS pooling: folded CLS-query scores x.u_h, softmax over the T tokens + CLS per head,
//       z_h = sum_n p_h[n] x[n]                                               -> z image (global)
// Replaces WordPositionalEncoder (models/line_transformer.py:61-73), `desc + pos` and the CLS
// concat (:117-121) and the attention part of MultiHeadAttention restricted to the CLS query row
// (models/line_attention.py:13-21,55-63), i.e. what a narrow-MLP kernel, two GEMM launches and a
// pooling kernel would do through global memory.  Only `desc` (the mandatory HBM read, one
// SWIZZLE_128B tensor-map TMA per 32-column block of the tile), the weights (L2 resident, streamed
// by 1-D TMA through a 2-slot ring) and the pooled z leave/enter the SM.
//
// The activations never touch shared memory: every layer is a register-A wgmma, and the accumulator
// fragment of a layer (after bias, ReLU and the split into packed bf16 hi / lo pairs) is exactly the A
// fragment of the next layer.  The 128 KB of shared memory beside the weight ring are the descriptor /
// x tile alone: the next tile's descriptors are requested the moment the pooling of this tile has read x.
//
// Warp roles: warps 0-7 = two warpgroups of 64 token rows (MMA, epilogues, softmax and pooling),
// warps 8-11 = producer warpgroup (its first lane streams the weights by TMA; it hands its registers to the
// workers with setmaxnreg: 128 x 40 + 256 x 232 <= 64 K).
#pragma once
#include <cuda.h>   // CUtensorMap (types only; the encoder is fetched through cudaGetDriverEntryPoint)
#include "act_img.cuh"
#include "common.cuh"
#include "tc_weight.cuh"
#include "ptx_sm90.cuh"

namespace ltr {

struct TokenFusedArgs {
  const float* pnt;    // [R*T, 2]
  const float* score;  // [R*T]
  const float* desc;   // [R*T, 256]
  // first layer (fp32, BN folded): w1 [32,3]; b2 [64] is the bias of the second
  const float *w1, *b1, *b2;
  TcWeight W2, W3, W4, W5;  // [64,64 (K 32 zero-padded)], [128,64], [256,128], [256,256] packed split-bf16
  const float *b3, *b4, *b5;
  const float* U;      // [4,256] folded CLS query u_h = W_k,h^T q_h / 8 (ltr_create)
  const float* s_cls;  // [4]
  const float* cls;    // [256]
  ActImg z;            // out: image of [R, 1024]
  int R, T, lpt, n_tiles;
  float cx, cy, scale;
};

struct TokenFusedSmem {
  static constexpr int ACT = 128 * 1024;   // the descriptor / x tile (fp32); the activations live in registers
  static constexpr int SLOT = 32 * 1024;   // one W tile [128 n x 64 k] hi + lo
  static constexpr int NSLOT = 2;
  static constexpr int OFF_RING = ACT;
  static constexpr int OFF_W1 = OFF_RING + NSLOT * SLOT;   // 96 floats
  static constexpr int OFF_B1 = OFF_W1 + 96 * 4;           // 32
  static constexpr int OFF_B2 = OFF_B1 + 32 * 4;           // 64
  static constexpr int OFF_B3 = OFF_B2 + 64 * 4;           // 128
  static constexpr int OFF_B4 = OFF_B3 + 128 * 4;          // 256
  static constexpr int OFF_B5 = OFF_B4 + 256 * 4;          // 256
  static constexpr int OFF_U = OFF_B5 + 256 * 4;           // 1024
  static constexpr int OFF_CLS = OFF_U + 1024 * 4;         // 256
  static constexpr int OFF_SC = OFF_CLS + 256 * 4;         // partial scores [2][128][4]
  static constexpr int OFF_P = OFF_SC + 2 * 128 * 4 * 4;   // softmax scratch (see below)
  static constexpr int OFF_BAR = OFF_P + (512 + 512 + 512) * 4;   // exps [128][4], 1/sum [<=512], CLS exp [<=512]
  static constexpr int TOTAL = OFF_BAR + 128 + 1024;       // + alignment slack
};

// x tile: 8 column blocks of [128 rows x 32 fp32 (128 B)], each row's eight
// 16-byte chunks XOR-swizzled by row & 7 - the layout a SWIZZLE_128B tensor-map box load produces.
// Conflict-free for a thread per channel quad (pooling).
__device__ __forceinline__ int xs_index(int row, int col) {
  return (col >> 5) * 4096 + row * 32 + (((((col >> 2) & 7) ^ (row & 7)) << 2) | (col & 3));
}

// relu(acc + bias) of a warpgroup accumulator fragment (N = 2 NR columns) -> split-bf16 A fragments of the next layer,
// K = 16 steps KK0 .. KK0 + NR / 8 (a K = 16 step of A takes the columns of two 8-column accumulator groups)
template <int KK0, int NR, int NK>
__device__ __forceinline__ void acc_to_afrag(const float (&d)[NR], const float* bias, int cq, uint32_t (&ah)[NK][4], uint32_t (&al)[NK][4]) {
#pragma unroll
  for (int kk = 0; kk < NR / 8; ++kk)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int jj = 2 * kk + (e >> 1), hr = (e & 1) * 2, c = 8 * jj + cq;
      const float v0 = fmaxf(d[4 * jj + hr] + bias[c], 0.f), v1 = fmaxf(d[4 * jj + hr + 1] + bias[c + 1], 0.f);
      ptx::split2_bf16(v0, v1, ah[KK0 + kk][e], al[KK0 + kk][e]);
    }
}

// One W slot (64 k) of a layer: A fragments KA0 .. KA0 + NK16 - 1, three split products per K = 16 step
template <int KA0, int NK16, int NR, int NK>
__device__ __forceinline__ void slot_mma(float (&d)[NR], const uint32_t (&ah)[NK][4], const uint32_t (&al)[NK][4], uint32_t w_hi,
                                         bool first) {
  ptx::wg_fence_regs(d);
  ptx::wg_fence();
#pragma unroll
  for (int k16 = 0; k16 < NK16; ++k16) {
    const uint64_t dwh = ptx::make_sw128_kmajor_desc(w_hi + k16 * 32, 1024);
    const uint64_t dwl = ptx::make_sw128_kmajor_desc(w_hi + 16384 + k16 * 32, 1024);
    if constexpr (NR == 32) {
      ptx::wgmma_rs_n64(d, al[KA0 + k16], dwh, (first && k16 == 0) ? 0u : 1u);
      ptx::wgmma_rs_n64(d, ah[KA0 + k16], dwl, 1);
      ptx::wgmma_rs_n64(d, ah[KA0 + k16], dwh, 1);
    } else {
      ptx::wgmma_rs_n128(d, al[KA0 + k16], dwh, (first && k16 == 0) ? 0u : 1u);
      ptx::wgmma_rs_n128(d, ah[KA0 + k16], dwl, 1);
      ptx::wgmma_rs_n128(d, ah[KA0 + k16], dwh, 1);
    }
  }
  ptx::wg_commit();
  ptx::wg_wait<0>();
  ptx::wg_fence_regs(d);
}

__global__ void __launch_bounds__(384, 1) token_fused_kernel(TokenFusedArgs p, const __grid_constant__ CUtensorMap desc_map) {
  using S = TokenFusedSmem;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t raw = ptx::smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw & 1023u)) & 1023u);
  uint8_t* act = smem;
  float* sW1 = reinterpret_cast<float*>(smem + S::OFF_W1);
  float* sB1 = reinterpret_cast<float*>(smem + S::OFF_B1);
  float* sB2 = reinterpret_cast<float*>(smem + S::OFF_B2);
  float* sB3 = reinterpret_cast<float*>(smem + S::OFF_B3);
  float* sB4 = reinterpret_cast<float*>(smem + S::OFF_B4);
  float* sB5 = reinterpret_cast<float*>(smem + S::OFF_B5);
  float* sU = reinterpret_cast<float*>(smem + S::OFF_U);
  float* sCls = reinterpret_cast<float*>(smem + S::OFF_CLS);
  float* sSc = reinterpret_cast<float*>(smem + S::OFF_SC);
  float* sP = reinterpret_cast<float*>(smem + S::OFF_P);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S::OFF_BAR);
  uint64_t* full = bars;            // [2] W slot filled (TMA tx)
  uint64_t* empty = bars + 2;       // [2] W slot consumed (8 consumer warps)
  uint64_t* dbar = bars + 4;        // [4] descriptor columns {32 s .. 32 s + 32} u {128 + 32 s ..} of the tile have landed
  uint64_t* x_free = bars + 8;      // workers -> descriptor request: the pooling has read the x tile (256 arrivals)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  pdl_launch_dependents();

  for (int i = tid; i < 96; i += blockDim.x) sW1[i] = p.w1[i];
  for (int i = tid; i < 32; i += blockDim.x) sB1[i] = p.b1[i];
  for (int i = tid; i < 64; i += blockDim.x) sB2[i] = p.b2[i];
  for (int i = tid; i < 128; i += blockDim.x) sB3[i] = p.b3[i];
  for (int i = tid; i < 256; i += blockDim.x) { sB4[i] = p.b4[i]; sB5[i] = p.b5[i]; sCls[i] = p.cls[i]; }
  for (int i = tid; i < 1024; i += blockDim.x) sU[i] = p.U[i];
  if (tid == 0) {
    for (int s = 0; s < 2; ++s) { ptx::mbar_init(&full[s], 1); ptx::mbar_init(&empty[s], 8); }
    for (int i = 0; i < 4; ++i) ptx::mbar_init(&dbar[i], 1);
    ptx::mbar_init(x_free, 256);
    ptx::prefetch_tensormap(&desc_map);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();   // z (output image) may still be read by the previous launch sequence

  if (warp >= 8) {
    // ---------------------------------------------------------------- W producer: 14 slots per tile
    ptx::setmaxnreg_dec<40>();
    uint32_t it = 0;
    auto push = [&](const TcWeight& W, int nb, int kb) {
      const int s = it & 1;
      const uint32_t ph = (it >> 1) & 1;
      ptx::mbar_wait(&empty[s], ph ^ 1);
      uint8_t* dst = smem + S::OFF_RING + s * S::SLOT;
      const size_t off = ((size_t)kb * (W.N / 8) + (size_t)nb * 16) * 1024;
      const uint32_t bytes = (uint32_t)min(128, W.N - nb * 128) * 128u;   // rows of this n-block x 128 B, per plane
      ptx::mbar_arrive_expect_tx(&full[s], 2 * bytes);
      ptx::bulk_g2s(dst, reinterpret_cast<const uint8_t*>(W.hi) + off, bytes, &full[s]);
      ptx::bulk_g2s(dst + 16384, reinterpret_cast<const uint8_t*>(W.lo) + off, bytes, &full[s]);
      ++it;
    };
    if (warp == 8 && lane == 0) {
      for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        push(p.W2, 0, 0);
        push(p.W3, 0, 0);
        for (int nb = 0; nb < 2; ++nb)
          for (int kb = 0; kb < 2; ++kb) push(p.W4, nb, kb);
        for (int nb = 0; nb < 2; ++nb)
          for (int kb = 0; kb < 4; ++kb) push(p.W5, nb, kb);
      }
    }
  } else {
    // ---------------------------------------------------------------- workers (2 warpgroups x 64 token rows)
    // Every layer is a register-A wgmma: the accumulator fragment of one layer, after bias + ReLU and the split into
    // bf16 hi / lo, is exactly the A fragment of the next, so the activations never leave the registers.
    ptx::setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int row_a = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // token rows row_a and row_a + 8 of the tile
    const int cq = 2 * (lane & 3);
    const int wt = tid;                // 0..255
    const int rows_used = p.lpt * p.T;
    uint32_t dph = 0, it = 0;
    auto worker_sync = [&]() { asm volatile("bar.sync 1, 256;" ::: "memory"); };
    auto slot_wait = [&]() -> uint32_t {
      ptx::mbar_wait(&full[it & 1], (it >> 1) & 1);
      return ptx::smem_u32(smem + S::OFF_RING + (it & 1) * S::SLOT);
    };
    auto slot_release = [&]() {
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&empty[it & 1]);
      ++it;
    };
    const float scls0 = p.s_cls[0], scls1 = p.s_cls[1], scls2 = p.s_cls[2], scls3 = p.s_cls[3];
    // ---- Softmax and pooling of a tile are DEFERRED into the next tile's MMA phases: they need only shared memory
    //      (the tile's partial scores and its x tile), while the workers would otherwise idle behind L2, L3, the first
    //      n-blocks of L4 and L5 (8.8 k of a 26.6 k-cycle tile in the clock64 trace).  The x tile is handed back for the
    //      next descriptors (x_free) as soon as the last deferred line has been pooled, during L5's first n-block.
    float* xs = reinterpret_cast<float*>(act);
    float* sInv = sP + 512;     // [4*lpt] 1/sum;   sP + 1024 .. : [4*lpt] CLS weight e0
    int prev_line0 = 0;
    bool have_prev = false;
    // The tile's sampled descriptors ([128 token rows x 256] fp32 - the one mandatory HBM stream of this stage) land in
    // the x tile, four groups of two 32-column SWIZZLE_128B boxes (group s = blocks s and 4 + s, the order the L5 epilogue
    // walks them).  Requested by worker thread 0: for the first tile at once, later the moment all 256 workers have
    // handed the x tile back (x_free) - a wait its warp has to sit out anyway before it can touch the new descriptors.
    uint32_t nx = 0;
    auto request_desc = [&](int t) {
      float* xs_t = reinterpret_cast<float*>(act);
      const int tok0 = (int)((long long)t * p.lpt * p.T);
      for (int sgrp = 0; sgrp < 4; ++sgrp) {
        ptx::mbar_arrive_expect_tx(&dbar[sgrp], 2 * 16384);
        ptx::tma_load_2d(xs_t + sgrp * 4096, &desc_map, sgrp * 32, tok0, &dbar[sgrp]);
        ptx::tma_load_2d(xs_t + (4 + sgrp) * 4096, &desc_map, (4 + sgrp) * 32, tok0, &dbar[sgrp]);
      }
    };
    if (wt == 0 && (int)blockIdx.x < p.n_tiles) request_desc(blockIdx.x);
    // softmax over the T tokens + CLS of every (line, head).  Thread = (token row, head pair): it scans the scores of
    // its row's line (both column halves, 2 x 8 B per token) for the maximum - redundantly per row, which costs T
    // cheap iterations instead of a barrier and a pass by 4 * lpt threads - and stores its own exp; after one barrier
    // the first row of every line sums the line's exps -> 1/sum and the CLS weight.  sP keeps UNNORMALISED exps; the
    // pooling multiplies by 1/sum once per output.
    auto softmax_prev = [&]() {
      const int srow = wt & 127, h2 = (wt >> 7) * 2;
      const bool live = srow < rows_used;
      const int ln = live ? srow / p.T : 0, rb = ln * p.T;
      const float c0 = h2 ? scls2 : scls0, c1 = h2 ? scls3 : scls1;
      float m0 = c0, m1 = c1;
      if (live) {
        for (int n = 0; n < p.T; ++n) {
          const float2 a = *reinterpret_cast<const float2*>(&sSc[(rb + n) * 4 + h2]);
          const float2 b = *reinterpret_cast<const float2*>(&sSc[(128 + rb + n) * 4 + h2]);
          m0 = fmaxf(m0, a.x + b.x);
          m1 = fmaxf(m1, a.y + b.y);
        }
        const float2 a = *reinterpret_cast<const float2*>(&sSc[srow * 4 + h2]);
        const float2 b = *reinterpret_cast<const float2*>(&sSc[(128 + srow) * 4 + h2]);
        *reinterpret_cast<float2*>(&sP[srow * 4 + h2]) = make_float2(expf(a.x + b.x - m0), expf(a.y + b.y - m1));
      }
      worker_sync();
      if (live && srow == rb) {
        const float e0 = expf(c0 - m0), e1 = expf(c1 - m1);
        float s0 = e0, s1 = e1;
        for (int n = 0; n < p.T; ++n) {
          const float2 e = *reinterpret_cast<const float2*>(&sP[(rb + n) * 4 + h2]);
          s0 += e.x;
          s1 += e.y;
        }
        *reinterpret_cast<float2*>(&sInv[ln * 4 + h2]) = make_float2(1.f / s0, 1.f / s1);
        *reinterpret_cast<float2*>(&sP[1024 + ln * 4 + h2]) = make_float2(e0, e1);
      }
      worker_sync();
    };
    // pooling: z_h[c] = (e0 * cls[c] + sum_n e[n] x[n][c]) / sum.  Thread = (4 channels, every fourth line), all four
    // heads: one 16-byte x read and one 16-byte read of the four heads' weights feed 16 FMAs, and the x tile is read
    // ONCE per tile (a head pair per thread read it twice: 256 KB of the SM's shared-memory bandwidth per tile).
    // Lines [first, first + count) of this thread's line sequence lg, lg + 4, ...
    auto pool_prev = [&](int first, int count) {
      const int cq = wt & 63, lg = wt >> 6;
      const float4 cv = *reinterpret_cast<const float4*>(&sCls[cq * 4]);
      for (int k = first; k < first + count; ++k) {
        const int ln = lg + 4 * k;
        if (ln >= p.lpt) break;
        const int gl = prev_line0 + ln;
        if (gl >= p.R) break;
        const float4 pc = *reinterpret_cast<const float4*>(&sP[1024 + ln * 4]);
        float z[4][4];
        const float pcv[4] = {pc.x, pc.y, pc.z, pc.w};
#pragma unroll
        for (int h = 0; h < 4; ++h) { z[h][0] = pcv[h] * cv.x; z[h][1] = pcv[h] * cv.y; z[h][2] = pcv[h] * cv.z; z[h][3] = pcv[h] * cv.w; }
        const int rb = ln * p.T;
#pragma unroll 3
        for (int n = 0; n < p.T; ++n) {
          const float4 xv = *reinterpret_cast<const float4*>(&xs[xs_index(rb + n, cq * 4)]);
          const float4 pr = *reinterpret_cast<const float4*>(&sP[(rb + n) * 4]);
          const float prv[4] = {pr.x, pr.y, pr.z, pr.w};
#pragma unroll
          for (int h = 0; h < 4; ++h) {
            const float2 pp = make_float2(prv[h], prv[h]);
            z[h][0] = fmaf(pp.x, xv.x, z[h][0]); z[h][1] = fmaf(pp.y, xv.y, z[h][1]);
            z[h][2] = fmaf(pp.x, xv.z, z[h][2]); z[h][3] = fmaf(pp.y, xv.w, z[h][3]);
          }
        }
        const float4 iv = *reinterpret_cast<const float4*>(&sInv[ln * 4]);
        const float ivv[4] = {iv.x, iv.y, iv.z, iv.w};
#pragma unroll
        for (int h = 0; h < 4; ++h)
          img_store4(p.z, gl, h * 256 + cq * 4, z[h][0] * ivv[h], z[h][1] * ivv[h], z[h][2] * ivv[h], z[h][3] * ivv[h]);
      }
    };
    for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
      const int line0 = tile * p.lpt;
      // ---- P0: first layer 3 -> 32 (+ReLU) on CUDA cores, straight into the A fragments of L2 (K = 32)
      uint32_t a32h[2][4], a32l[2][4];
      {
        const long long tk0 = (long long)tile * p.lpt * p.T;
        float x0[2], x1[2], x2[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int r = row_a + 8 * e;
          x0[e] = x1[e] = x2[e] = 0.f;
          if (r < rows_used && tk0 + r < (long long)p.R * p.T) {
            const long long tk = tk0 + r;
            x0[e] = (p.pnt[2 * tk] - p.cx) / p.scale;
            x1[e] = (p.pnt[2 * tk + 1] - p.cy) / p.scale;
            x2[e] = p.score[tk];
          }
        }
#pragma unroll
        for (int kk = 0; kk < 2; ++kk)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int r = e & 1, n = 16 * kk + 8 * (e >> 1) + cq;
            const float a = fmaxf(fmaf(sW1[n * 3 + 2], x2[r], fmaf(sW1[n * 3 + 1], x1[r], fmaf(sW1[n * 3], x0[r], sB1[n]))), 0.f);
            const float b = fmaxf(fmaf(sW1[n * 3 + 5], x2[r], fmaf(sW1[n * 3 + 4], x1[r], fmaf(sW1[n * 3 + 3], x0[r], sB1[n + 1]))), 0.f);
            ptx::split2_bf16(a, b, a32h[kk][e], a32l[kk][e]);
          }
      }
      if (have_prev) softmax_prev();
      // ---- L2: 32 -> 64 (the k-block's upper half is zero padding)
      uint32_t a64h[4][4], a64l[4][4];
      {
        float d[32];
        const uint32_t w = slot_wait();
        slot_mma<0, 2>(d, a32h, a32l, w, true);
        slot_release();
        acc_to_afrag<0>(d, sB2, cq, a64h, a64l);
      }
      if (have_prev) pool_prev(0, 1);
      // ---- L3: 64 -> 128
      uint32_t a128h[8][4], a128l[8][4];
      {
        float d[64];
        const uint32_t w = slot_wait();
        slot_mma<0, 4>(d, a64h, a64l, w, true);
        slot_release();
        acc_to_afrag<0>(d, sB3, cq, a128h, a128l);
      }
      if (have_prev) pool_prev(1, 1);
      // ---- L4: 128 -> 256, two n-blocks of 128
      uint32_t a256h[16][4], a256l[16][4];
#pragma unroll
      for (int nb = 0; nb < 2; ++nb) {
        float d[64];
        uint32_t w = slot_wait();
        slot_mma<0, 4>(d, a128h, a128l, w, true);
        slot_release();
        w = slot_wait();
        slot_mma<4, 4>(d, a128h, a128l, w, false);
        slot_release();
        if (nb == 0) acc_to_afrag<0>(d, sB4, cq, a256h, a256l);
        else acc_to_afrag<8>(d, sB4 + 128, cq, a256h, a256l);
      }
      if (have_prev) {                  // the rest of the pooling, then the x tile is free for this tile's descriptors
        pool_prev(2, 1 << 30);
        ptx::fence_proxy_async_smem();  // this thread's generic accesses to the x tile before the TMA writes that follow
        ptx::mbar_arrive(x_free);
        if (wt == 0) {
          ptx::mbar_wait(x_free, nx++ & 1);
          request_desc(tile);
        }
      }
      // ---- L5: 256 -> 256; x = acc + b5 + desc -> fp32, in place in the x tile (where the TMA put desc);
      //      partial CLS scores x . u_h of this thread's two rows
      float sc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
      for (int nb = 0; nb < 2; ++nb) {
        float d[64];
#pragma unroll
        for (int kb = 0; kb < 4; ++kb) {
          const uint32_t w = slot_wait();
          if (kb == 0) slot_mma<0, 4>(d, a256h, a256l, w, true);
          if (kb == 1) slot_mma<4, 4>(d, a256h, a256l, w, false);
          if (kb == 2) slot_mma<8, 4>(d, a256h, a256l, w, false);
          if (kb == 3) slot_mma<12, 4>(d, a256h, a256l, w, false);
          slot_release();
        }
        if (nb == 0)
          for (int g = 0; g < 4; ++g) ptx::mbar_wait(&dbar[g], dph);   // the tile's descriptors have landed
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int n = nb * 128 + 8 * j + cq;
          const float2 b = *reinterpret_cast<const float2*>(&sB5[n]);
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float2* xp = reinterpret_cast<float2*>(&xs[xs_index(row_a + 8 * e, n)]);
            const float2 dv = *xp;
            const float2 x = make_float2(d[4 * j + 2 * e] + b.x + dv.x, d[4 * j + 2 * e + 1] + b.y + dv.y);
            *xp = x;
#pragma unroll
            for (int hh = 0; hh < 4; ++hh) {
              const float2 u = *reinterpret_cast<const float2*>(&sU[hh * 256 + n]);
              sc[e][hh] = fmaf(x.x, u.x, fmaf(x.y, u.y, sc[e][hh]));
            }
          }
        }
      }
      dph ^= 1;
#pragma unroll
      for (int e = 0; e < 2; ++e)
#pragma unroll
        for (int hh = 0; hh < 4; ++hh) {
          sc[e][hh] += __shfl_xor_sync(0xffffffffu, sc[e][hh], 1);
          sc[e][hh] += __shfl_xor_sync(0xffffffffu, sc[e][hh], 2);
        }
      if ((lane & 3) == 0) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int r = row_a + 8 * e;
          *reinterpret_cast<float4*>(&sSc[r * 4]) = make_float4(sc[e][0], sc[e][1], sc[e][2], sc[e][3]);
          *reinterpret_cast<float4*>(&sSc[(128 + r) * 4]) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
      worker_sync();
      // softmax + pooling of THIS tile run inside the next tile (or after the loop for the last one)
      prev_line0 = line0;
      have_prev = true;
    }
    if (have_prev) {   // drain: the CTA's last tile
      softmax_prev();
      pool_prev(0, 1 << 30);
    }
  }
}

// cuTensorMapEncodeTiled through the runtime (no link against libcuda)
typedef CUresult (*TensorMapEncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                           const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                           CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline TensorMapEncodeTiledFn tensor_map_encoder() {
  static TensorMapEncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<TensorMapEncodeTiledFn>(p);
  }
  return fn;
}

inline int launch_token_fused(TokenFusedArgs a, cudaStream_t s) {
  if (a.R <= 0) return 0;
  if (a.T < 1 || a.T > 128) return set_error(-1, "token_fused: T must be in 1..128");
  if ((long long)a.R * a.T >= (1ll << 31)) return set_error(-1, "token_fused: more than 2^31 tokens in one call");
  if (reinterpret_cast<uintptr_t>(a.desc) % 16) return set_error(-1, "token_fused: desc_sublines must be 16-byte aligned");
  a.lpt = 128 / a.T;
  a.n_tiles = cdiv(a.R, a.lpt);
  // tensor map of the sampled descriptors viewed as [R*T rows, 256] fp32; box = 32 columns (128 B) x 128 rows
  TensorMapEncodeTiledFn enc = tensor_map_encoder();
  if (!enc) return set_error(-1, "token_fused: cuTensorMapEncodeTiled is not available from this driver");
  CUtensorMap map;
  const cuuint64_t gdim[2] = {256, (cuuint64_t)a.R * a.T};
  const cuuint64_t gstride[1] = {256 * sizeof(float)};
  const cuuint32_t box[2] = {32, 128};
  const cuuint32_t estride[2] = {1, 1};
  const CUresult cr = enc(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(a.desc), gdim, gstride, box, estride,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) return set_error(-1, "token_fused: cuTensorMapEncodeTiled failed (" + std::to_string((int)cr) + ")");
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (sms <= 0) sms = 132;
  const int grid = a.n_tiles < sms ? a.n_tiles : sms;
  return launch(KC_TOKEN_FUSED, true, token_fused_kernel, dim3(grid), dim3(384), TokenFusedSmem::TOTAL, s, a, map);
}

}  // namespace ltr
