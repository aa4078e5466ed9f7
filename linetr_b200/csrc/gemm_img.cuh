// Persistent tensor-core GEMM for sm_90a whose operands travel as split-bf16 "tile images".
//
//   Y = act(X W^T + b) (+ R),   X given as an activation image, Y written as fp32 rows and/or
//   as the activation image the next layer consumes.
//
// Activation image (ActImg) of a row-major activation [M, K]: two planes (bf16 hi, bf16 lo with
// x ~= hi + lo), each a sequence of 16 KB tiles [m_tile = row/128][k_block = k/64] holding
// 128 rows x 64 k in the K-major SWIZZLE_128B layout wgmma reads.  A tile is therefore ONE
// contiguous cp.async.bulk (TMA) transfer and needs no CUDA-core work on the consumer side.
// Weights use the same trick (TcWeight, tc_weight.cuh).
//
// The main loop is pure TMA + wgmma:  warp 8 (of a producer warpgroup) streams A and W tiles through an mbarrier ring,
// two consumer warpgroups (64 rows each) issue 3 MMAs per k-step (lo*hi + hi*lo + hi*hi, fp32
// accumulate in registers), then apply bias / activation / residual and write fp32 rows and/or the
// split-bf16 image of the result.  A plain tile that writes only an image does that on the
// accumulator fragment and bulk-stores each warp's rows (epi_frag_tile); the others stage the
// accumulator through shared memory so that a thread owns one row of 32 columns.  CTAs are
// persistent (one per SM) and walk the tile list round-robin; the producer fetches the next
// tile's k-blocks while the epilogue runs.
#pragma once
#include "common.cuh"
#include "tc_weight.cuh"
#include "act_img.cuh"
#include "ptx_sm90.cuh"

namespace ltr {

struct GemmImgArgs {
  ActImg A; int a_kb0;       // contract k-blocks [a_kb0 + nb*a_kb_nb, ... + W.K/64) of A for n-block nb
  int a_kb_nb;               // 0 for a plain GEMM; K/64 for a block-diagonal one (each n-block reads its own K slice)
  TcWeight W;
  const float* bias;
  const float* R; int ldr;   // fp32 residual (added after the activation) or nullptr
  ActImg Rimg; int r_kb0;    // OR: residual read from a split-bf16 image (hi + lo), k-block offset
  float* C; int ldc;         // fp32 output or nullptr
  ActImg O; int o_kb0;       // image output (O.hi == nullptr: none); column n -> k-block o_kb0 + n/64
  int M, act;
  // row-normalising epilogue (BN = 256 = N only, one tile spans whole rows):
  //   NORM_LAYER: y = LayerNorm(acc + bias (+ R | Rimg)) * ng + nbeta (+ nadd | NaddImg)      (models/line_attention.py:51-53,73-75)
  //   NORM_L2:    y = (acc + bias) / max(||.||_2, 1e-12)                      (models/line_transformer.py:246)
  int norm; float eps;
  const float* ng; const float* nbeta;
  const float* nadd; int ldadd;   // fp32 rows added AFTER the normalisation or nullptr
  ActImg NaddImg; int nadd_kb0;   // OR: the same addend read from a split-bf16 image
  int m_tiles, n_blks;
};

enum Act : int { ACT_NONE = 0, ACT_RELU = 1, ACT_GELU = 2 };
enum { NORM_NONE = 0, NORM_LAYER = 1, NORM_L2 = 2 };

// GELU(x) = x * Phi(x) with the erf form the reference uses (F.gelu default, models/line_attention.py:92).
// erfc(u) = P(t) exp(-u^2), t = 1 / (1 + 0.3275911 u)  (Abramowitz-Stegun 7.1.26, |error| <= 1.5e-7 - the
// size of an fp32 rounding of erf itself) costs 2 SFU ops + ~12 FMAs; erff() is ~35 instructions per value
// and made the 256 -> 1024 FFN epilogue twice as long as its main loop.  Written with erfc on both
// sides of zero so that the negative tail has no 1 - erf cancellation.
__device__ __forceinline__ float gelu_erf(float x) {
  const float u = fabsf(x) * 0.70710678118654752440f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, u, 1.f)));
  float pl = fmaf(1.061405429f, t, -1.453152027f);
  pl = fmaf(pl, t, 1.421413741f);
  pl = fmaf(pl, t, -0.284496736f);
  pl = fmaf(pl, t, 0.254829592f);
  pl *= t;
  const float g = 0.5f * x * pl * ptx::ex2_approx(u * u * -1.4426950408889634f);   // 0.5 x erfc(|x| / sqrt 2)
  return x < 0.f ? g : x - g;
}

// two values at once (the epilogues work on column pairs)
__device__ __forceinline__ float2 gelu_erf2(float2 x) { return make_float2(gelu_erf(x.x), gelu_erf(x.y)); }

// ---------------------------------------------------------------- epilogue building blocks
// One epilogue warp owns 32 accumulator rows (row0 .. row0+31, lane = row) and works on 32-column
// chunks `acc[32]` starting at global column `nbase`.  Global traffic goes through the warp's 4 KB
// staging tile so that each load/store instruction touches whole 32-byte sectors of a few rows.

// acc += X[row0 + lane][nbase .. nbase+32) for fp32 rows X (coalesced read of the 32 x 32 tile)
__device__ __forceinline__ void epi_add_rows_f32(const float* __restrict__ X, int ldx, int row0, int nbase, int M, int lane,
                                                 float* stg, float (&acc)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int rl = i * 4 + (lane >> 3), c4 = lane & 7;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row0 + rl < M) v = *reinterpret_cast<const float4*>(X + (long long)(row0 + rl) * ldx + nbase + c4 * 4);
    *reinterpret_cast<float4*>(&stg[rl * 32 + ((c4 ^ (rl & 7)) << 2)]) = v;
  }
  __syncwarp();
#pragma unroll
  for (int c4 = 0; c4 < 8; ++c4) {
    const float4 v = *reinterpret_cast<const float4*>(&stg[lane * 32 + ((c4 ^ (lane & 7)) << 2)]);
    acc[c4 * 4] += v.x; acc[c4 * 4 + 1] += v.y; acc[c4 * 4 + 2] += v.z; acc[c4 * 4 + 3] += v.w;
  }
  __syncwarp();
}

// C[row0 + lane][nbase .. nbase+32) = acc.  Eight lanes store one row's 128 contiguous bytes (4 rows per instruction),
// so every 16-byte store instruction writes whole 32-byte sectors: with one lane writing 32 bytes as two 16-byte
// stores, each instruction wrote half sectors and needed twice the L2 write requests.
__device__ __forceinline__ void epi_store_rows_f32(float* __restrict__ C, int ldc, int row0, int nbase, int M, int lane,
                                                   float* stg, const float (&acc)[32]) {
#pragma unroll
  for (int c4 = 0; c4 < 8; ++c4)
    *reinterpret_cast<float4*>(&stg[lane * 32 + ((c4 ^ (lane & 7)) << 2)]) =
        make_float4(acc[c4 * 4], acc[c4 * 4 + 1], acc[c4 * 4 + 2], acc[c4 * 4 + 3]);
  __syncwarp();
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int rl = i * 4 + (lane >> 3), c4 = lane & 7;
    const float4 v = *reinterpret_cast<const float4*>(&stg[rl * 32 + ((c4 ^ (rl & 7)) << 2)]);
    if (row0 + rl < M) *reinterpret_cast<float4*>(C + (long long)(row0 + rl) * ldc + nbase + c4 * 4) = v;
  }
  __syncwarp();
}

// image O, m-tile mt, k-block kb0 + nbase/64: columns nbase .. nbase+32 of rows q*32 + lane <- split-bf16(acc)
__device__ __forceinline__ void epi_store_image(const ActImg& O, int kb0, int mt, int nbase, int q, int row0, int M, int lane,
                                                uint8_t* stgb, const float (&acc)[32]) {
  // staging: plane [32 rows][4 chunks of 16 B], chunk slot swizzled by (row>>1)&3
#pragma unroll
  for (int cc = 0; cc < 4; ++cc) {
    uint4 h, l;
    ptx::split8_bf16(&acc[cc * 8], h, l);
    const int slot = (lane * 4 + (cc ^ ((lane >> 1) & 3))) * 16;
    *reinterpret_cast<uint4*>(stgb + slot) = h;
    *reinterpret_cast<uint4*>(stgb + 2048 + slot) = l;
  }
  __syncwarp();
  const int kb_out = kb0 + (nbase >> 6);
  const size_t toff = ((size_t)mt * O.kblocks + kb_out) * IMG_TILE_ELEMS;
  uint8_t* ohi = reinterpret_cast<uint8_t*>(O.hi + toff);
  uint8_t* olo = reinterpret_cast<uint8_t*>(O.lo + toff);
  const int gch0 = (nbase & 63) >> 3;   // first 16-byte chunk of these 32 columns inside the 64-wide k-block
  // the 4 chunks of a row form one aligned 64-byte group of its 128-byte tile line; four lanes store a row's group
  // (8 rows per instruction and plane), so every 16-byte store instruction writes whole 32-byte sectors
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int rl = i * 8 + (lane >> 2), phys = lane & 3;    // phys: physical chunk (0..3) inside the 64-byte group
    const int r_in = q * 32 + rl;
    // physical chunk index inside the group = (gch0 + cc) ^ (r_in & 7) restricted to the group's 2 low bits
    const int base_phys = (gch0 ^ (r_in & 7)) & 4;          // which 64-byte half of the 128-byte line
    const int cc = phys ^ (r_in & 3);                       // logical chunk stored there (low two bits of the XOR)
    const int slot = (rl * 4 + (cc ^ ((rl >> 1) & 3))) * 16;
    const uint4 vh = *reinterpret_cast<const uint4*>(stgb + slot);
    const uint4 vl = *reinterpret_cast<const uint4*>(stgb + 2048 + slot);
    if (row0 + rl < M) {
      const uint32_t off = (r_in >> 3) * 1024u + (r_in & 7u) * 128u + (uint32_t)(base_phys + phys) * 16u;
      *reinterpret_cast<uint4*>(ohi + off) = vh;
      *reinterpret_cast<uint4*>(olo + off) = vl;
    }
  }
  __syncwarp();
}

// acc += X[rows q*32 + lane of m-tile mt][columns nbase .. nbase+32) for a split-bf16 image X (k-block kb0 + nbase/64):
// coalesced 16-byte chunk loads -> staging -> own row; bf16 -> fp32 is a 16-bit shift
__device__ __forceinline__ void epi_add_rows_img(const ActImg& X, int kb0, int mt, int nbase, int q, int row0, int M, int lane,
                                                 uint8_t* stgb, float (&acc)[32]) {
  const size_t rtoff = ((size_t)mt * X.kblocks + kb0 + (nbase >> 6)) * IMG_TILE_ELEMS;
  const uint8_t* rhi = reinterpret_cast<const uint8_t*>(X.hi + rtoff);
  const uint8_t* rlo = reinterpret_cast<const uint8_t*>(X.lo + rtoff);
  const int gch0r = (nbase & 63) >> 3;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int rl = i * 8 + (lane >> 2), cc = lane & 3;
    uint4 vh = make_uint4(0u, 0u, 0u, 0u), vl = vh;
    if (row0 + rl < M) {
      const uint32_t off = ptx::sw128_offset(q * 32 + rl, (gch0r + cc) * 8);
      vh = *reinterpret_cast<const uint4*>(rhi + off);
      vl = *reinterpret_cast<const uint4*>(rlo + off);
    }
    const int slot = (rl * 4 + (cc ^ ((rl >> 1) & 3))) * 16;
    *reinterpret_cast<uint4*>(stgb + slot) = vh;
    *reinterpret_cast<uint4*>(stgb + 2048 + slot) = vl;
  }
  __syncwarp();
#pragma unroll
  for (int cc = 0; cc < 4; ++cc) {
    const int slot = (lane * 4 + (cc ^ ((lane >> 1) & 3))) * 16;
    const uint4 vh = *reinterpret_cast<const uint4*>(stgb + slot);
    const uint4 vl = *reinterpret_cast<const uint4*>(stgb + 2048 + slot);
    const uint32_t wh[4] = {vh.x, vh.y, vh.z, vh.w}, wl[4] = {vl.x, vl.y, vl.z, vl.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      acc[cc * 8 + 2 * e] += __uint_as_float(wh[e] << 16) + __uint_as_float(wl[e] << 16);
      acc[cc * 8 + 2 * e + 1] += __uint_as_float(wh[e] & 0xFFFF0000u) + __uint_as_float(wl[e] & 0xFFFF0000u);
    }
  }
  __syncwarp();
}


template <int BN>
struct GemmImgCfg {
  static constexpr int A_TILE = 16384;            // one plane of a 128x64 bf16 tile
  static constexpr int W_TILE = BN * 128;         // one plane of a BN x 64 bf16 tile
  static constexpr int STAGE = 2 * A_TILE + 2 * W_TILE;
  static constexpr int STAGES = BN >= 256 ? 2 : (BN >= 128 ? 3 : 4);
  static constexpr int STG_WARP = 4096;           // per epilogue warp: 32 rows x 32 fp32 (or 2 x [32 x 64 B] bf16)
  static constexpr int OFF_STG = STAGES * STAGE;
  static constexpr int OFF_BAR = OFF_STG + 8 * STG_WARP;
  static constexpr int OFF_XCH = OFF_BAR + 256;                     // row-norm partial sums [2][128] fp32 (BN = 256 only)
  static constexpr int XCH = BN == 256 ? 2048 : 0;
  // the dynamic window is declared __align__(1024) (no static shared memory in this kernel, so it starts
  // at the CTA's 1 KB-aligned window base); the in-kernel round-up is then a no-op and the slack below
  // is never consumed - it only keeps the carve-up valid should a toolchain ever place the window at a
  // smaller alignment (BN = 256 has 768 B left under the 227 KB CTA limit)
  static constexpr int SMEM = OFF_XCH + XCH + (BN == 256 ? 768 : 1024);
  static_assert(SMEM <= 232448, "gemm_img: shared memory budget (227 KB per CTA)");
  // 2 consumer warpgroups (MMA + epilogue) and a producer warpgroup whose first warp issues the TMA copies; the
  // producer gives its registers to the consumers (setmaxnreg: 128 x 40 + 256 x 232 <= 64 K), which hold a 64 x BN
  // fp32 accumulator fragment (128 registers at BN = 256) plus the epilogue's working set
  static constexpr int THREADS = 384;
};

// barrier over the 8 consumer warps only (the producer warpgroup never joins it)
__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// Chained GEMMs (gemm_chain_kernel): this warp has stored its part of one 64-column output k-block; order the stores
// before the TMA reads of the next op (generic -> async proxy fence in every lane, then the warp's arrival on the
// k-block's barrier, a release that the producer thread of the same CTA acquires before it issues the copy) and count
// the warp (8 arrivals = the whole 128 x 64 block is written).  CTA scope is enough: writer and TMA issuer share the CTA.
// A device-scope __threadfence() here cost ~4 % of a chained signature layer on H100 and is not needed.
// The epilogues publish a chunk after the NEXT chunk's arithmetic, when its stores have long been issued.
// `ready` == nullptr: no consumer, nothing to do.
__device__ __forceinline__ void publish_kblock(uint64_t* ready, int kb, int lane) {
  if (!ready) return;
  ptx::fence_proxy_async_global();
  __syncwarp();
  if (lane == 0) ptx::mbar_arrive(&ready[kb]);
}

// Columns [64 chunk, 64 chunk + 64) of a consumer warpgroup's accumulator fragment (64 rows x N, see ptx::wg_*) ->
// the eight 32 x 32 fp32 staging blocks of the tile (block 4 * column half + q holds rows 32 q .. 32 q + 31, chunk
// columns 32 * column half ..; a row's float4 groups XOR-swizzled by row & 7, the layout epi_add_rows_f32 reads).
// row_a = first accumulator row of this thread inside the 128-row tile.
template <int NR>
__device__ __forceinline__ void stage_acc64(const float (&d)[NR], int chunk, float* stg_all, int row_a, int lane) {
#pragma unroll
  for (int j = 0; j < NR / 4; ++j) {
    if ((j >> 3) != chunk) continue;
    const int c = (j & 7) * 8 + 2 * (lane & 3), ch = c >> 5, cl = c & 31;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row_a + 8 * h, rl = r & 31;
      float* blk = stg_all + (ch * 4 + (r >> 5)) * 1024;
      *reinterpret_cast<float2*>(&blk[rl * 32 + ((((cl >> 2) ^ (rl & 7))) << 2) + (cl & 3)]) = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
    }
  }
}
// this warp's staging block -> acc[32] (lane = row)
__device__ __forceinline__ void load_stage(const float* stg, int lane, float (&acc)[32]) {
#pragma unroll
  for (int c4 = 0; c4 < 8; ++c4) {
    const float4 v = *reinterpret_cast<const float4*>(&stg[lane * 32 + ((c4 ^ (lane & 7)) << 2)]);
    acc[c4 * 4] = v.x; acc[c4 * 4 + 1] = v.y; acc[c4 * 4 + 2] = v.z; acc[c4 * 4 + 3] = v.w;
  }
  __syncwarp();
}

// v, opaque to the compiler: what a staged epilogue derives from it (stage_acc64's sixteen staging addresses) is formed
// per chunk.  Hoisted out of the tile loop, those addresses stayed live through the whole chained kernel, next to the
// fragment epilogue's working set, and were spilled.
__device__ __forceinline__ int opaque(int v) {
  asm volatile("" : "+r"(v));
  return v;
}

// Row-normalising epilogue of one 128 x 256 tile (see GemmImgArgs::norm).  A row's 256 columns sit in two
// threads (column halves of every 64-column chunk, different warps); partial sums are exchanged through `xch`.
// The accumulator stays in registers and is staged again for every pass.  ready: see publish_kblock.
template <int NR>
__device__ __forceinline__ void epi_norm_tile(const GemmImgArgs& p, const float (&d)[NR], int mt, int q, int half, int lane,
                                              int row_a, float* stg_all, float* stg, uint8_t* stgb, float* xch,
                                              uint64_t* ready = nullptr) {
  if (lane == 0) ptx::bulk_wait_read_all();   // a chain's fragment epilogues may still be bulk-storing from the staging
  const int row0 = mt * 128 + q * 32, r_in = q * 32 + lane;
  auto chunk = [&](int ch, float (&v)[32]) {
    epi_bar();
    stage_acc64(d, ch, stg_all, opaque(row_a), lane);
    epi_bar();
    load_stage(stg, lane, v);
    const int c0 = ch * 64 + half * 32;
    if (p.bias) {
#pragma unroll
      for (int j = 0; j < 32; j += 4) {
        const float4 b = *reinterpret_cast<const float4*>(p.bias + c0 + j);
        v[j] += b.x; v[j + 1] += b.y; v[j + 2] += b.z; v[j + 3] += b.w;
      }
    }
    if (p.R) epi_add_rows_f32(p.R, p.ldr, row0, c0, p.M, lane, stg, v);
    if (p.Rimg.hi) epi_add_rows_img(p.Rimg, p.r_kb0, mt, c0, q, row0, p.M, lane, stgb, v);
  };
  float mean = 0.f, scale;
  if (p.norm == NORM_LAYER) {
    float s = 0.f;
#pragma unroll 1
    for (int ch = 0; ch < 4; ++ch) {
      float v[32];
      chunk(ch, v);
#pragma unroll
      for (int j = 0; j < 32; ++j) s += v[j];
    }
    xch[half * 128 + r_in] = s;
    epi_bar();
    mean = (s + xch[(half ^ 1) * 128 + r_in]) * (1.f / 256.f);
    float ss = 0.f;
#pragma unroll 1
    for (int ch = 0; ch < 4; ++ch) {
      float v[32];
      chunk(ch, v);
#pragma unroll
      for (int j = 0; j < 32; ++j) { const float dv = v[j] - mean; ss = fmaf(dv, dv, ss); }
    }
    xch[256 + half * 128 + r_in] = ss;
    epi_bar();
    ss += xch[256 + (half ^ 1) * 128 + r_in];
    scale = 1.f / sqrtf(ss * (1.f / 256.f) + p.eps);
  } else {
    float ss = 0.f;
#pragma unroll 1
    for (int ch = 0; ch < 4; ++ch) {
      float v[32];
      chunk(ch, v);
#pragma unroll
      for (int j = 0; j < 32; ++j) ss = fmaf(v[j], v[j], ss);
    }
    xch[half * 128 + r_in] = ss;
    epi_bar();
    ss += xch[(half ^ 1) * 128 + r_in];
    scale = 1.f / fmaxf(sqrtf(ss), 1e-12f);
  }
#pragma unroll 1
  for (int ch = 0; ch < 4; ++ch) {
    float v[32];
    chunk(ch, v);
    const int c0 = ch * 64 + half * 32;
    if (p.norm == NORM_LAYER) {
#pragma unroll
      for (int j = 0; j < 32; j += 4) {
        const float4 g = *reinterpret_cast<const float4*>(p.ng + c0 + j);
        const float4 b = *reinterpret_cast<const float4*>(p.nbeta + c0 + j);
        v[j] = (v[j] - mean) * scale * g.x + b.x;
        v[j + 1] = (v[j + 1] - mean) * scale * g.y + b.y;
        v[j + 2] = (v[j + 2] - mean) * scale * g.z + b.z;
        v[j + 3] = (v[j + 3] - mean) * scale * g.w + b.w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] *= scale;
    }
    if (p.nadd) epi_add_rows_f32(p.nadd, p.ldadd, row0, c0, p.M, lane, stg, v);
    if (p.NaddImg.hi) epi_add_rows_img(p.NaddImg, p.nadd_kb0, mt, c0, q, row0, p.M, lane, stgb, v);
    if (ch > 0) publish_kblock(ready, ch - 1, lane);   // one chunk late: its stores have drained by now
    if (p.C) epi_store_rows_f32(p.C, p.ldc, row0, c0, p.M, lane, stg, v);
    if (p.O.hi) epi_store_image(p.O, p.o_kb0, mt, c0, q, row0, p.M, lane, stgb, v);
  }
  publish_kblock(ready, 3, lane);
}

// Plain epilogue of one 128 x BN tile: this warp's 32 rows x one half of every 64-column chunk:
// bias -> activation -> residual (fp32 rows or split-bf16 image) -> fp32 rows and/or image output.
// An in-place residual (Rimg == O, same k-blocks: mlp2's x += delta) is race-free: an element is read
// (epi_add_rows_img) and written back (epi_store_image) by the same warp within the same chunk.
template <int BN, int NR>
__device__ __forceinline__ void epi_plain_tile(const GemmImgArgs& p, const float (&d)[NR], int mt, int nb, int q, int half, int lane,
                                               int row_a, float* stg_all, float* stg, uint8_t* stgb, uint64_t* ready = nullptr) {
  if (lane == 0) ptx::bulk_wait_read_all();   // a chain's fragment epilogues may still be bulk-storing from the staging
  const int row0 = mt * 128 + q * 32;   // first row of this warp
#pragma unroll 1
  for (int ch = 0; ch < BN / 64; ++ch) {
    float acc[32];
    epi_bar();
    stage_acc64(d, ch, stg_all, opaque(row_a), lane);
    epi_bar();
    load_stage(stg, lane, acc);
    const int nbase = nb * BN + ch * 64 + half * 32;
    if (p.bias) {
#pragma unroll
      for (int j = 0; j < 32; j += 4) {
        const float4 b = *reinterpret_cast<const float4*>(p.bias + nbase + j);
        acc[j] += b.x; acc[j + 1] += b.y; acc[j + 2] += b.z; acc[j + 3] += b.w;
      }
    }
    // the activation is uniform per launch: branch ONCE per chunk (an if-converted erff per
    // element costs ~40 instructions even when ReLU/identity is selected)
    if (p.act == ACT_RELU) {
#pragma unroll
      for (int j = 0; j < 32; ++j) acc[j] = fmaxf(acc[j], 0.f);
    } else if (p.act == ACT_GELU) {
#pragma unroll
      for (int j = 0; j < 32; j += 2) {
        const float2 g = gelu_erf2(make_float2(acc[j], acc[j + 1]));
        acc[j] = g.x; acc[j + 1] = g.y;
      }
    }
    if (p.R) epi_add_rows_f32(p.R, p.ldr, row0, nbase, p.M, lane, stg, acc);
    if (p.Rimg.hi) epi_add_rows_img(p.Rimg, p.r_kb0, mt, nbase, q, row0, p.M, lane, stgb, acc);
    if (ch > 0) publish_kblock(ready, nb * (BN / 64) + ch - 1, lane);   // one chunk late: its stores have drained by now
    if (p.C) epi_store_rows_f32(p.C, p.ldc, row0, nbase, p.M, lane, stg, acc);
    if (p.O.hi) epi_store_image(p.O, p.o_kb0, mt, nbase, q, row0, p.M, lane, stgb, acc);
  }
  publish_kblock(ready, nb * (BN / 64) + BN / 64 - 1, lane);
}

// ---------------------------------------------------------------- fragment epilogue: plain tiles that write only an image
// Warp q of consumer warpgroup wg holds tile rows frow + lane / 4 + {0, 8}, frow = 64 wg + 16 q (ptx::wg_*), and row r
// of an image tile is the 128-byte line at byte 128 r.  So the warp's 16 rows of one 64-column chunk are one contiguous
// 2 KB piece of each plane's tile: the warp splits its fragment into its 4 KB staging block (hi piece, then lo piece, in
// the tile's own SWIZZLE_128B layout) and lane 0 writes each piece with one bulk copy.  No barrier spans warps, and no
// lane waits for its global stores.  Every element gets the staged path's operations in its order (acc + bias,
// activation, acc + (hi + lo) of the residual, split), so the image is bit-identical to the split of its fp32 rows.
// Ordering (all of it lane 0's bulk groups and the warp's residual mbarrier):
//  - the staging block is rewritten only after the previous bulk store has read it (wait_group.read 0, then the warp
//    syncs, or the residual load issued after that wait has landed);
//  - chained GEMMs: output k-block kb is published once its stores have completed: wait_group 1 after the next
//    chunk's commit, wait_group 0 after the tile's last one (publish_bulk);
//  - an image residual (mlp2's in-place x += delta) is bulk-loaded into the staging block: chunk 0 before the tile's
//    main loop (epi_frag_prefetch), chunk c + 1 once chunk c's store has read the block.  A lane reads the residual
//    words at the positions it then overwrites with its output, and a chunk's store is issued after its residual
//    has landed, so an in-place update reads the old values.
__host__ __device__ __forceinline__ bool epi_frag(const GemmImgArgs& p) { return p.norm == NORM_NONE && p.O.hi && !p.C && !p.R; }

// bytes of the warp's 16-row piece (first tile row frow) that lie above row M; rows >= M stay unwritten
__device__ __forceinline__ uint32_t frag_piece_bytes(int M, int mt, int frow) {
  return 128u * (uint32_t)min(max(M - (mt * 128 + frow), 0), 16);
}

// lane 0: this warp's piece of residual k-block r_kb0 + kb -> its staging block, completing on rbar
__device__ __forceinline__ void frag_load_res(const GemmImgArgs& p, int mt, int kb, int frow, uint32_t bytes, uint8_t* stgb,
                                              uint64_t* rbar) {
  const size_t toff = ((size_t)mt * p.Rimg.kblocks + p.r_kb0 + kb) * IMG_TILE_ELEMS;
  ptx::mbar_arrive_expect_tx(rbar, 2 * bytes);
  ptx::bulk_g2s(stgb, reinterpret_cast<const uint8_t*>(p.Rimg.hi + toff) + 128 * frow, bytes, rbar);
  ptx::bulk_g2s(stgb + 2048, reinterpret_cast<const uint8_t*>(p.Rimg.lo + toff) + 128 * frow, bytes, rbar);
}

// before a fragment tile's main loop: start loading its first chunk's residual, once the staging block is free
__device__ __forceinline__ void epi_frag_prefetch(const GemmImgArgs& p, int mt, int kb0, int frow, int lane, uint8_t* stgb,
                                                  uint64_t* rbar) {
  if (lane != 0 || !p.Rimg.hi) return;
  const uint32_t bytes = frag_piece_bytes(p.M, mt, frow);
  if (!bytes) return;
  ptx::bulk_wait_read_all();
  frag_load_res(p, mt, kb0, frow, bytes, stgb, rbar);
}

// Chained GEMMs, lane 0: all but its newest N bulk groups have completed, and with them every store of output k-block
// kb; fence them to the async proxy (the next op's TMA reads) and count the warp on kb_ready[kb] (as publish_kblock).
template <int N>
__device__ __forceinline__ void publish_bulk(uint64_t* ready, int kb) {
  ptx::bulk_wait<N>();
  ptx::fence_proxy_async_global();
  ptx::mbar_arrive(&ready[kb]);
}

// The fragment epilogue of one 128 x BN tile for this warp (d is consumed in place).  ph0: parity of the residual
// barrier's phase that completes with this tile's first load.  The barrier completes one phase per load, a tile issues
// BN / 64 loads when its piece has rows below M and none otherwise, and the m-tile never decreases along a CTA's walk,
// so tiles without loads come last: after tl tiles, ph0 = (tl BN / 64) & 1, which is 0 for BN = 256 whatever the walk.
// ready: chained GEMMs publish k-blocks up to the tile's second-to-last one here; the caller publishes the last one
// (publish_bulk<0>).
template <int BN, int NR>
__device__ __forceinline__ void epi_frag_tile(const GemmImgArgs& p, float (&d)[NR], int mt, int nb, int frow, int lane,
                                              uint8_t* stgb, uint64_t* rbar, uint32_t ph0, uint64_t* ready) {
  constexpr int NCH = BN / 64;
  const uint32_t bytes = frag_piece_bytes(p.M, mt, frow);
  const bool res = p.Rimg.hi && bytes;
  const int r8 = lane >> 2, cq = 2 * (lane & 3);   // fragment row mod 8 (also its swizzle key), first column of a pair
  // word of (row r8, columns 8 j + cq) in the hi piece: 128 r8 + 16 (j ^ r8) + 2 cq = sbase ^ 16 j (the staging block is
  // 4 KB aligned, so the fields occupy disjoint bits); row r8 + 8 is 1024 bytes further, the lo piece 2048
  const uint32_t sbase = ptx::smem_u32(stgb) + 144u * r8 + 2u * cq;
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const int kb = nb * NCH + c;
    if (p.bias) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 b = *reinterpret_cast<const float2*>(p.bias + kb * 64 + 8 * j + cq);
        const int e = 32 * c + 4 * j;
        d[e] += b.x; d[e + 1] += b.y; d[e + 2] += b.x; d[e + 3] += b.y;
      }
    }
    // the activation is uniform per op: branch once per chunk
    if (p.act == ACT_RELU) {
#pragma unroll
      for (int e = 32 * c; e < 32 * c + 32; ++e) d[e] = fmaxf(d[e], 0.f);
    } else if (p.act == ACT_GELU) {
#pragma unroll
      for (int e = 32 * c; e < 32 * c + 32; e += 2) {
        const float2 g = gelu_erf2(make_float2(d[e], d[e + 1]));
        d[e] = g.x; d[e + 1] = g.y;
      }
    }
    if (res) {
      ptx::mbar_wait(rbar, (ph0 + c) & 1);
    } else {
      if (lane == 0) ptx::bulk_wait_read_all();
      __syncwarp();
    }
    // opaque to the compiler, so that the eight addresses below are formed per chunk: hoisted out of the tile loop, they
    // stayed live through the whole kernel and were spilled
    uint32_t sb = sbase;
    asm volatile("" : "+r"(sb));
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        // the 32 lanes of one (j, h) write 32 distinct banks: word lane & 3 of 16-byte chunk j ^ r8 (8 distinct r8)
        const uint32_t wh = (sb ^ (16u * j)) + 1024u * h, wl = wh + 2048u;
        const int e = 32 * c + 4 * j + 2 * h;
        float a = d[e], b = d[e + 1];
        if (res) {
          const uint32_t rh = ptx::ld_shared_u32(wh), rl = ptx::ld_shared_u32(wl);
          a += __uint_as_float(rh << 16) + __uint_as_float(rl << 16);
          b += __uint_as_float(rh & 0xFFFF0000u) + __uint_as_float(rl & 0xFFFF0000u);
        }
        uint32_t hi, lo;
        ptx::split2_bf16(a, b, hi, lo);
        ptx::st_shared_u32(wh, hi);
        ptx::st_shared_u32(wl, lo);
      }
    ptx::fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
      if (bytes) {
        const size_t toff = ((size_t)mt * p.O.kblocks + p.o_kb0 + kb) * IMG_TILE_ELEMS;
        ptx::bulk_s2g(reinterpret_cast<uint8_t*>(p.O.hi + toff) + 128 * frow, stgb, bytes);
        ptx::bulk_s2g(reinterpret_cast<uint8_t*>(p.O.lo + toff) + 128 * frow, stgb + 2048, bytes);
      }
      ptx::bulk_commit();
      if (ready && c > 0) publish_bulk<1>(ready, kb - 1);
      if (res && c + 1 < NCH) {
        ptx::bulk_wait_read_all();
        frag_load_res(p, mt, kb + 1, frow, bytes, stgb, rbar);
      }
    }
  }
}

// One k-block (64 deep) of a warpgroup's 64 x BN accumulator: three split products per K = 16 step
// (lo*hi + hi*lo + hi*hi).  a_hi / a_lo: this warpgroup's 64 rows of the A tile planes; w_hi / w_lo: the W tile planes.
template <int BN>
__device__ __forceinline__ void mma_kblock(float (&d)[BN / 2], uint32_t a_hi, uint32_t a_lo, uint32_t w_hi, uint32_t w_lo, bool first) {
#pragma unroll
  for (int k16 = 0; k16 < 4; ++k16) {
    const uint32_t ko = k16 * 32;
    const uint64_t dah = ptx::make_sw128_kmajor_desc(a_hi + ko, 1024);
    const uint64_t dal = ptx::make_sw128_kmajor_desc(a_lo + ko, 1024);
    const uint64_t dwh = ptx::make_sw128_kmajor_desc(w_hi + ko, 1024);
    const uint64_t dwl = ptx::make_sw128_kmajor_desc(w_lo + ko, 1024);
    const uint32_t acc = (first && k16 == 0) ? 0u : 1u;
    if constexpr (BN == 64) {
      ptx::wgmma_ss_n64(d, dal, dwh, acc); ptx::wgmma_ss_n64(d, dah, dwl, 1); ptx::wgmma_ss_n64(d, dah, dwh, 1);
    } else if constexpr (BN == 128) {
      ptx::wgmma_ss_n128(d, dal, dwh, acc); ptx::wgmma_ss_n128(d, dah, dwl, 1); ptx::wgmma_ss_n128(d, dah, dwh, 1);
    } else {
      ptx::wgmma_ss_n256(d, dal, dwh, acc); ptx::wgmma_ss_n256(d, dah, dwl, 1); ptx::wgmma_ss_n256(d, dah, dwh, 1);
    }
  }
}

// FRAG: the launch's op takes the fragment epilogue (epi_frag, chosen on the host).  The two epilogues are separate
// instantiations so that neither one's registers are allocated around the other's: in one kernel, the staged
// epilogue's hoisted staging addresses and the fragment epilogue together spilled into the main loop.
template <int BN, bool FRAG>
__global__ void __launch_bounds__(384, 1) gemm_img_kernel(GemmImgArgs p) {
  using Cfg = GemmImgCfg<BN>;
  static_assert((2 * Cfg::STAGES + 8) * 8 <= Cfg::OFF_XCH - Cfg::OFF_BAR, "gemm_img: barrier area");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t raw = ptx::smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::STAGES;
  uint64_t* res_bar = bars + 2 * Cfg::STAGES;   // one per consumer warp (epi_frag_tile's residual loads)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nk = p.W.K / 64;
  const int n_tiles = p.m_tiles * p.n_blks;
  // Only CTA 0 reads the debug-trace switch, once: a global load at every stamp sits on each CTA's critical path.
  const bool trace = blockIdx.x == 0 && g_dbg_on;
  pdl_launch_dependents();

  if (tid == 0) {
    for (int s = 0; s < Cfg::STAGES; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], 8);
    }
    for (int w = 0; w < 8; ++w) ptx::mbar_init(&res_bar[w], 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();   // the previous kernel's outputs (A image, residual) are complete and visible from here on

  if (warp >= 8) {
    // ---------------------------------------------------------------- TMA producer
    ptx::setmaxnreg_dec<40>();
    if (warp == 8 && lane == 0) {
      const uint8_t* whi = reinterpret_cast<const uint8_t*>(p.W.hi);
      const uint8_t* wlo = reinterpret_cast<const uint8_t*>(p.W.lo);
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int mt = tile / p.n_blks, nb = tile - mt * p.n_blks;
        for (int kb = 0; kb < nk; ++kb, ++it) {
          const int s = it % Cfg::STAGES;
          const uint32_t ph = (it / Cfg::STAGES) & 1;
          ptx::mbar_wait(&empty[s], ph ^ 1);
          if (trace && it < 4) LTR_DBG_STAMP(it * 16 + 6);
          uint8_t* st = smem + s * Cfg::STAGE;
          const size_t aoff = ((size_t)mt * p.A.kblocks + p.a_kb0 + nb * p.a_kb_nb + kb) * IMG_TILE_ELEMS;
          const size_t woff = ((size_t)kb * (p.W.N / 8) + (size_t)nb * (BN / 8)) * 1024;
          ptx::mbar_arrive_expect_tx(&full[s], Cfg::STAGE);
          ptx::bulk_g2s(st, p.A.hi + aoff, Cfg::A_TILE, &full[s]);
          ptx::bulk_g2s(st + Cfg::A_TILE, p.A.lo + aoff, Cfg::A_TILE, &full[s]);
          ptx::bulk_g2s(st + 2 * Cfg::A_TILE, whi + woff, Cfg::W_TILE, &full[s]);
          ptx::bulk_g2s(st + 2 * Cfg::A_TILE + Cfg::W_TILE, wlo + woff, Cfg::W_TILE, &full[s]);
        }
      }
    }
  } else {
    // ---------------------------------------------------------------- consumers (2 warpgroups x 64 rows)
    // Main loop: wgmma with the accumulator in registers, one k-block in flight behind the one being issued.
    // Epilogue: image-only plain tiles work on the fragment and bulk-store each warp's rows (epi_frag_tile).
    // Otherwise 64-column chunks of the accumulator go through the staging blocks so that a thread owns one
    // row (lane = row) of 32 columns; global traffic then goes through the warp's 4 KB block so that every
    // global load/store instruction touches whole 32-byte sectors of a few rows.
    ptx::setmaxnreg_inc<232>();
    const int wg = warp >> 2, q = warp & 3, half = warp >> 2;
    const int row_a = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int frow = 16 * warp;   // first tile row of the warp's fragment (64 wg + 16 q)
    float* stg_all = reinterpret_cast<float*>(smem + Cfg::OFF_STG);
    float* stg = stg_all + warp * (Cfg::STG_WARP / 4);
    uint8_t* stgb = reinterpret_cast<uint8_t*>(stg);
    uint32_t it = 0, tl = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tl) {
      const int mt = tile / p.n_blks, nb = tile - mt * p.n_blks;
      float d[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
      if constexpr (FRAG) epi_frag_prefetch(p, mt, nb * (BN / 64), frow, lane, stgb, &res_bar[warp]);
      if (trace && tl < 4 && tid == 0) LTR_DBG_STAMP(tl * 16 + 0);
      for (int kb = 0; kb < nk; ++kb, ++it) {
        const int s = it % Cfg::STAGES;
        ptx::mbar_wait(&full[s], (it / Cfg::STAGES) & 1);
        const uint32_t a_hi = ptx::smem_u32(smem + s * Cfg::STAGE) + wg * 8192;
        const uint32_t w_hi = ptx::smem_u32(smem + s * Cfg::STAGE + 2 * Cfg::A_TILE);
        ptx::wg_fence_regs(d);
        ptx::wg_fence();
        mma_kblock<BN>(d, a_hi, a_hi + Cfg::A_TILE, w_hi, w_hi + Cfg::W_TILE, kb == 0);
        ptx::wg_commit();
        ptx::wg_wait<1>();
        ptx::wg_fence_regs(d);
        if (kb > 0 && lane == 0) ptx::mbar_arrive(&empty[(it - 1) % Cfg::STAGES]);
      }
      ptx::wg_wait<0>();
      ptx::wg_fence_regs(d);
      if (lane == 0) ptx::mbar_arrive(&empty[(it - 1) % Cfg::STAGES]);
      if (trace && tl < 4 && tid == 0) LTR_DBG_STAMP(tl * 16 + 2);
      if constexpr (FRAG) {
        epi_frag_tile<BN>(p, d, mt, nb, frow, lane, stgb, &res_bar[warp], (tl * (BN / 64)) & 1, nullptr);
      } else {
        if constexpr (BN == 256) {
          if (p.norm != NORM_NONE) {
            epi_norm_tile(p, d, mt, q, half, lane, row_a, stg_all, stg, stgb, reinterpret_cast<float*>(smem + Cfg::OFF_XCH));
            continue;
          }
        }
        epi_plain_tile<BN>(p, d, mt, nb, q, half, lane, row_a, stg_all, stg, stgb);
      }
      if (trace && tl < 4 && tid == 0) LTR_DBG_STAMP(tl * 16 + 5);
    }
    if constexpr (FRAG) {
      if (lane == 0) ptx::bulk_wait<0>();   // the staging stays allocated, and the writes done, until the stores complete
    }
  }
}

template <int BN, bool FRAG>
static int launch_gemm_img_bn(GemmImgArgs a, cudaStream_t s) {
  using Cfg = GemmImgCfg<BN>;
  a.m_tiles = cdiv(a.M, 128);
  a.n_blks = a.W.N / BN;
  const int tiles = a.m_tiles * a.n_blks;
  const int grid = tiles < device_sm_count() ? tiles : device_sm_count();
  return launch(KC_LINEAR, true, gemm_img_kernel<BN, FRAG>, dim3(grid), dim3(Cfg::THREADS), Cfg::SMEM, s, a);
}

// bn_hint: 0 = choose (256 when N % 256 == 0 and that still gives >= 1 tile per SM, else 128)
inline int launch_gemm_img(const GemmImgArgs& a, cudaStream_t s, int bn_hint = 0) {
  if (a.M <= 0) return 0;
  if (a.W.K % 64 || a.W.N % 64 || (a.C && a.ldc % 8) || (a.R && a.ldr % 4))
    return set_error(-1, "gemm_img: K%64, N%64, ldc%8, ldr%4 required");
  {   // operand / output k-block ranges must lie inside their images (a wrong d_inner would otherwise alias tiles silently)
    const int nblk = a.a_kb_nb ? a.W.N / 64 : 1;   // block-diagonal: 64-wide n-blocks, each with its own K slice
    if (a.a_kb0 < 0 || a.a_kb0 + (nblk - 1) * a.a_kb_nb + a.W.K / 64 > a.A.kblocks)
      return set_error(-1, "gemm_img: A k-block range exceeds the activation image");
    if (a.O.hi && (a.o_kb0 < 0 || a.o_kb0 + a.W.N / 64 > a.O.kblocks))
      return set_error(-1, "gemm_img: output columns exceed the output image");
    if (a.Rimg.hi && (a.r_kb0 < 0 || a.r_kb0 + a.W.N / 64 > a.Rimg.kblocks))
      return set_error(-1, "gemm_img: residual columns exceed the residual image");
  }
  if (a.norm != NORM_NONE) {
    if (a.W.N != 256 || a.act != ACT_NONE || (a.nadd && a.ldadd % 4) || (a.norm == NORM_LAYER && (!a.ng || !a.nbeta)) ||
        (a.R && a.Rimg.hi) || (a.nadd && a.NaddImg.hi) ||
        (a.NaddImg.hi && (a.nadd_kb0 < 0 || a.nadd_kb0 + 4 > a.NaddImg.kblocks)))
      return set_error(-1, "gemm_img: the row-norm epilogue needs N == 256, no activation, fp32 residual");
    return launch_gemm_img_bn<256, false>(a, s);
  }
  const bool frag = epi_frag(a);
  if (bn_hint == 64 || a.W.N % 128) return frag ? launch_gemm_img_bn<64, true>(a, s) : launch_gemm_img_bn<64, false>(a, s);
  int bn = bn_hint;
  if (!bn) {
    bn = 128;
    if (a.W.N % 256 == 0 && (long long)cdiv(a.M, 128) * (a.W.N / 256) >= device_sm_count()) bn = 256;
  }
  if (bn == 256 && a.W.N % 256 == 0) return frag ? launch_gemm_img_bn<256, true>(a, s) : launch_gemm_img_bn<256, false>(a, s);
  return frag ? launch_gemm_img_bn<128, true>(a, s) : launch_gemm_img_bn<128, false>(a, s);
}

// ---------------------------------------------------------------- chained GEMMs (one launch, several row-local layers)
// Layers whose every output row depends only on the same row of the previous layer's output run back to back in ONE
// persistent launch: CTA b owns m-tiles b, b + grid, ... and walks through all n-blocks of op 0, then of op 1, ... for
// each of them, with the main loop, epilogues and TMA / mbarrier ring of gemm_img_kernel<256> (same tile arithmetic, so
// the results are bit-identical to one launch per op).  What a chain saves over separate launches: the ring fill, the
// idle SMs of the last wave and the grid-wide wait at every op boundary.
// Dependency between consecutive ops, inside the CTA: op o+1 reads A k-block kb of its m-tile (TMA) only after all 8
// epilogue warps have stored - and fenced to the async proxy - output columns [64 kb, 64 kb + 64) of op o for that
// m-tile (`kb_ready[kb]`, 8 arrivals; publish_kblock).  One barrier per k-block rather than per op lets the producer
// load op o+1's first k-blocks while the epilogue still writes the later ones.  Each arrival phase of kb_ready[kb] is
// waited for exactly once, in order: op o+1 reads exactly the k-blocks op o writes (gemm_chain_check), the last op of
// the chain publishes nothing, and op o+1 cannot reach its epilogue (its next publication) before the producer has
// loaded - so waited for - all its A k-blocks.  W tiles depend on nothing; the first ones are requested before
// pdl_wait.  BN = 256 only.
constexpr int CHAIN_MAX_OPS = 4;
constexpr int CHAIN_MAX_KB = 16;   // output k-blocks of an op that feeds the next one (N <= 1024)
// k-block timeline of CTA 0 in g_dbg_trace when armed (ltr_debug_trace_arm; tools/gemm_chain_trace.py reads it).
// k-block it < CHAIN_TRACE_KB of the CTA's walk: slot 3*it = producer has issued the k-block's loads (its empty-wait
// ended), 3*it + 1 = the consumers' first thread sees its stage landed (full-wait returned), 3*it + 2 = its MMAs are
// done (wgmma.wait_group 0).  Tile o * 4 + nb of the first m-tile: slot CHAIN_TRACE_EPI + o * 4 + nb = its epilogue
// is done (an epilogue starts at its last k-block's 3*it + 2; a fragment epilogue is done when the first thread's warp
// has committed its last bulk store, before the wait that publishes that k-block).  CHAIN_TRACE_T0 / + 1: producer / consumers past
// pdl_wait.  Off (the default), a stamp costs its thread an `it` compare and, in the window, a load of g_dbg_on.
constexpr int CHAIN_TRACE_KB = 36;
constexpr int CHAIN_TRACE_EPI = 3 * CHAIN_TRACE_KB;
constexpr int CHAIN_TRACE_T0 = CHAIN_TRACE_EPI + CHAIN_MAX_OPS * 4;
static_assert(CHAIN_TRACE_T0 + 2 <= 128, "gemm_chain: trace slots");
struct GemmChainArgs {
  GemmImgArgs op[CHAIN_MAX_OPS];
  int n_ops, m_tiles;
};

__global__ void __launch_bounds__(384, 1) gemm_chain_kernel(const __grid_constant__ GemmChainArgs c) {
  constexpr int BN = 256;
  using Cfg = GemmImgCfg<BN>;
  static_assert((2 * Cfg::STAGES + CHAIN_MAX_KB + 8) * 8 <= Cfg::OFF_XCH - Cfg::OFF_BAR, "gemm_chain: barrier area");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t raw = ptx::smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::STAGES;
  uint64_t* kb_ready = bars + 2 * Cfg::STAGES;
  uint64_t* res_bar = kb_ready + CHAIN_MAX_KB;   // one per consumer warp (epi_frag_tile's residual loads)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  pdl_launch_dependents();

  if (tid == 0) {
    for (int s = 0; s < Cfg::STAGES; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], 8);
    }
    for (int k = 0; k < CHAIN_MAX_KB; ++k) ptx::mbar_init(&kb_ready[k], 8);
    for (int w = 0; w < 8; ++w) ptx::mbar_init(&res_bar[w], 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ---------------------------------------------------------------- TMA producer
    ptx::setmaxnreg_dec<40>();
    if (warp == 8 && lane == 0) {
      // the first STAGES k-blocks of op 0 go to fresh slots: their W tiles are requested before pdl_wait
      const int npre = (int)blockIdx.x < c.m_tiles ? min(Cfg::STAGES, c.op[0].W.K / 64) : 0;
      for (int kb = 0; kb < npre; ++kb) {
        const size_t woff = (size_t)kb * (c.op[0].W.N / 8) * 1024;
        uint8_t* st = smem + kb * Cfg::STAGE;
        ptx::mbar_arrive_expect_tx(&full[kb], Cfg::STAGE);
        ptx::bulk_g2s(st + 2 * Cfg::A_TILE, reinterpret_cast<const uint8_t*>(c.op[0].W.hi) + woff, Cfg::W_TILE, &full[kb]);
        ptx::bulk_g2s(st + 2 * Cfg::A_TILE + Cfg::W_TILE, reinterpret_cast<const uint8_t*>(c.op[0].W.lo) + woff, Cfg::W_TILE, &full[kb]);
      }
      pdl_wait();   // the previous kernel's outputs (op 0's A image, residuals, addends) are complete from here on
      LTR_DBG_STAMP(CHAIN_TRACE_T0);
      uint32_t it = 0, ph = 0;   // ph bit kb: parity of the next kb_ready[kb] phase to wait for
      for (int mt = blockIdx.x; mt < c.m_tiles; mt += gridDim.x)
        for (int o = 0; o < c.n_ops; ++o) {
          const GemmImgArgs& p = c.op[o];
          const int nk = p.W.K / 64;
          const uint8_t* whi = reinterpret_cast<const uint8_t*>(p.W.hi);
          const uint8_t* wlo = reinterpret_cast<const uint8_t*>(p.W.lo);
          for (int nb = 0; nb < p.n_blks; ++nb)
            for (int kb = 0; kb < nk; ++kb, ++it) {
              const int s = it % Cfg::STAGES;
              uint8_t* st = smem + s * Cfg::STAGE;
              if (it >= (uint32_t)npre) {
                ptx::mbar_wait(&empty[s], ((it / Cfg::STAGES) & 1) ^ 1);
                const size_t woff = ((size_t)kb * (p.W.N / 8) + (size_t)nb * (BN / 8)) * 1024;
                ptx::mbar_arrive_expect_tx(&full[s], Cfg::STAGE);
                ptx::bulk_g2s(st + 2 * Cfg::A_TILE, whi + woff, Cfg::W_TILE, &full[s]);
                ptx::bulk_g2s(st + 2 * Cfg::A_TILE + Cfg::W_TILE, wlo + woff, Cfg::W_TILE, &full[s]);
              }
              if (it < CHAIN_TRACE_KB) LTR_DBG_STAMP(3 * it);
              if (o > 0 && nb == 0) {   // A k-block kb = output k-block kb of op o-1 for this m-tile
                ptx::mbar_wait(&kb_ready[kb], (ph >> kb) & 1);
                ph ^= 1u << kb;
              }
              const size_t aoff = ((size_t)mt * p.A.kblocks + p.a_kb0 + kb) * IMG_TILE_ELEMS;
              ptx::bulk_g2s(st, p.A.hi + aoff, Cfg::A_TILE, &full[s]);
              ptx::bulk_g2s(st + Cfg::A_TILE, p.A.lo + aoff, Cfg::A_TILE, &full[s]);
            }
        }
    }
  } else {
    // ---------------------------------------------------------------- consumers (2 warpgroups x 64 rows), as gemm_img_kernel
    // except for the stage release (below)
    ptx::setmaxnreg_inc<232>();
    pdl_wait();   // residual / addend images of op 0 may come from the previous kernel
    if (tid == 0) LTR_DBG_STAMP(CHAIN_TRACE_T0 + 1);
    const int wg = warp >> 2, q = warp & 3, half = warp >> 2;
    const int row_a = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int frow = 16 * warp;   // first tile row of the warp's fragment (64 wg + 16 q)
    float* stg_all = reinterpret_cast<float*>(smem + Cfg::OFF_STG);
    float* stg = stg_all + warp * (Cfg::STG_WARP / 4);
    uint8_t* stgb = reinterpret_cast<uint8_t*>(stg);
    float* xch = reinterpret_cast<float*>(smem + Cfg::OFF_XCH);
    uint32_t it = 0;
    for (int mt = blockIdx.x; mt < c.m_tiles; mt += gridDim.x)
      for (int o = 0; o < c.n_ops; ++o) {
        const GemmImgArgs& p = c.op[o];
        const int nk = p.W.K / 64;
        const bool frag = epi_frag(p);
        uint64_t* ready = o + 1 < c.n_ops ? kb_ready : nullptr;
        for (int nb = 0; nb < p.n_blks; ++nb) {
          float d[BN / 2];
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
          if (frag) epi_frag_prefetch(p, mt, nb * (BN / 64), frow, lane, stgb, &res_bar[warp]);
          for (int kb = 0; kb < nk; ++kb, ++it) {
            const int s = it % Cfg::STAGES;
            ptx::mbar_wait(&full[s], (it / Cfg::STAGES) & 1);
            if (it < CHAIN_TRACE_KB && tid == 0) LTR_DBG_STAMP(3 * it + 1);
            const uint32_t a_hi = ptx::smem_u32(smem + s * Cfg::STAGE) + wg * 8192;
            const uint32_t w_hi = ptx::smem_u32(smem + s * Cfg::STAGE + 2 * Cfg::A_TILE);
            ptx::wg_fence_regs(d);
            ptx::wg_fence();
            mma_kblock<BN>(d, a_hi, a_hi + Cfg::A_TILE, w_hi, w_hi + Cfg::W_TILE, kb == 0);
            ptx::wg_commit();
            // Release the stage as soon as its own MMAs are done, before waiting for the next one.  With two stages,
            // keeping one k-block of MMAs in flight (wait_group 1) released stage it-1 only after full[it] had
            // arrived, so the refill of a stage started only when the previous load had landed: one 96 KB load in
            // flight at a time, and a k-block took a whole load latency (~4.4 us on H100 against ~1.6 us of MMA).
            ptx::wg_wait<0>();
            ptx::wg_fence_regs(d);
            if (lane == 0) ptx::mbar_arrive(&empty[s]);
            if (it < CHAIN_TRACE_KB && tid == 0) LTR_DBG_STAMP(3 * it + 2);
          }
          if (p.norm != NORM_NONE)
            epi_norm_tile(p, d, mt, q, half, lane, row_a, stg_all, stg, stgb, xch, ready);
          else if (frag)
            epi_frag_tile<BN>(p, d, mt, nb, frow, lane, stgb, &res_bar[warp], 0, ready);
          else
            epi_plain_tile<BN>(p, d, mt, nb, q, half, lane, row_a, stg_all, stg, stgb, ready);
          if (mt == (int)blockIdx.x && nb < 4 && tid == 0) LTR_DBG_STAMP(CHAIN_TRACE_EPI + o * 4 + nb);
          if (frag && ready && lane == 0) publish_bulk<0>(ready, nb * (BN / 64) + BN / 64 - 1);
        }
      }
    if (lane == 0) ptx::bulk_wait<0>();   // the staging stays allocated, and the writes done, until the stores complete
  }
}

// nullptr if ops[0 .. n_ops) can run as one gemm_chain_kernel launch, else why not.  Every op: BN = 256 tiles (N % 256),
// a plain A operand (no block-diagonal slices), k-block ranges inside their images; op i > 0 must read exactly the
// image k-blocks op i-1 writes (the row-local hand-over the kernel's dependencies are built on).
inline const char* gemm_chain_check(const GemmImgArgs* ops, int n_ops) {
  if (n_ops < 1 || n_ops > CHAIN_MAX_OPS) return "gemm_chain: 1..4 ops";
  for (int i = 0; i < n_ops; ++i) {
    const GemmImgArgs& a = ops[i];
    if (a.M != ops[0].M || a.W.K <= 0 || a.W.K % 64 || a.W.N <= 0 || a.W.N % 256 || a.a_kb_nb || !a.A.hi ||
        (a.C && a.ldc % 8) || (a.R && a.ldr % 4))
      return "gemm_chain: ops need equal M, K % 64, N % 256, a plain A image, ldc % 8, ldr % 4";
    if (a.a_kb0 < 0 || a.a_kb0 + a.W.K / 64 > a.A.kblocks || (a.O.hi && (a.o_kb0 < 0 || a.o_kb0 + a.W.N / 64 > a.O.kblocks)) ||
        (a.Rimg.hi && (a.r_kb0 < 0 || a.r_kb0 + a.W.N / 64 > a.Rimg.kblocks)))
      return "gemm_chain: a k-block range exceeds its image";
    if ((a.R && a.Rimg.hi) || (a.nadd && a.NaddImg.hi))
      return "gemm_chain: residual or addend given twice";
    if (a.norm != NORM_NONE &&
        (a.W.N != 256 || a.act != ACT_NONE || (a.nadd && a.ldadd % 4) || (a.norm == NORM_LAYER && (!a.ng || !a.nbeta)) ||
         (a.NaddImg.hi && (a.nadd_kb0 < 0 || a.nadd_kb0 + 4 > a.NaddImg.kblocks))))
      return "gemm_chain: the row-norm epilogue needs N == 256, no activation, ldadd % 4, LayerNorm parameters";
    if (i == 0) continue;
    const GemmImgArgs& prev = ops[i - 1];
    if (!prev.O.hi || a.A.hi != prev.O.hi || a.A.lo != prev.O.lo || a.A.kblocks != prev.O.kblocks)
      return "gemm_chain: op i must read the image op i-1 writes (row-local chain)";
    if (a.a_kb0 != prev.o_kb0 || a.W.K != prev.W.N)
      return "gemm_chain: op i must read exactly the k-blocks op i-1 writes";
    if (prev.W.N / 64 > CHAIN_MAX_KB) return "gemm_chain: an op that feeds the next one may write at most 16 k-blocks";
  }
  return nullptr;
}

inline int launch_gemm_chain(const GemmImgArgs* ops, int n_ops, cudaStream_t s) {
  if (const char* why = gemm_chain_check(ops, n_ops)) return set_error(-1, why);
  if (ops[0].M <= 0) return 0;
  GemmChainArgs c{};
  c.n_ops = n_ops;
  c.m_tiles = cdiv(ops[0].M, 128);
  for (int i = 0; i < n_ops; ++i) {
    c.op[i] = ops[i];
    c.op[i].m_tiles = c.m_tiles;
    c.op[i].n_blks = ops[i].W.N / 256;
  }
  using Cfg = GemmImgCfg<256>;
  const int grid = c.m_tiles < device_sm_count() ? c.m_tiles : device_sm_count();
  return launch(KC_LINEAR, true, gemm_chain_kernel, dim3(grid), dim3(Cfg::THREADS), Cfg::SMEM, s, c);
}

// ---------------------------------------------------------------- image <-> fp32 helpers
// fp32 rows [M, K] (ld) -> image k-blocks [kb0, kb0 + K/64); one thread per 8 consecutive k.
__global__ void __launch_bounds__(256) to_image_kernel(const float* __restrict__ x, int ld, int M, int K, ActImg o, int kb0) {
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  const int k8 = K / 8;
  if (idx >= (long long)M * k8) return;
  const int row = (int)(idx / k8), k = (int)(idx % k8) * 8;
  const float4 a = *reinterpret_cast<const float4*>(x + (long long)row * ld + k);
  const float4 b = *reinterpret_cast<const float4*>(x + (long long)row * ld + k + 4);
  const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  uint4 h, l;
  ptx::split8_bf16(v, h, l);
  const size_t toff = ((size_t)(row >> 7) * o.kblocks + kb0 + (k >> 6)) * IMG_TILE_ELEMS;
  const uint32_t off = ptx::sw128_offset(row & 127, k & 63);
  *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(o.hi + toff) + off) = h;
  *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(o.lo + toff) + off) = l;
}

// image k-blocks [kb0, kb0 + K/64) -> fp32 rows (hi + lo); test helper.
__global__ void __launch_bounds__(256) from_image_kernel(ActImg a, int kb0, float* __restrict__ y, int ld, int M, int K) {
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= (long long)M * K) return;
  const int row = (int)(idx / K), k = (int)(idx % K);
  const size_t toff = ((size_t)(row >> 7) * a.kblocks + kb0 + (k >> 6)) * IMG_TILE_ELEMS;
  const uint32_t off = ptx::sw128_offset(row & 127, k & 63) / 2;
  y[(long long)row * ld + k] = __bfloat162float(a.hi[toff + off]) + __bfloat162float(a.lo[toff + off]);
}

}  // namespace ltr
