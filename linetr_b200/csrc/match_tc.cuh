// Tensor-core descriptor matcher (K3): all-pairs distance D = 2 - 2 <a_i, b_j> on wgmma with the
// row-argmin fused into the epilogue, for BOTH directions (side 0 rows vs side 1 and side 1 rows vs
// side 0 - the second one is the column argmin the mutual check needs), an exact fp32 re-check pass
// (match_exact_kernel) for the decisions the tensor-core arithmetic cannot make safely, and a tail kernel
// that applies threshold + mutual check + per-pair counts.
//
// Reference: get_dist_matrix (models/line_process.py:198-201: einsum('bdn,bdm->bnm'), (2 - 2 s).clip(0)),
// nn_matcher / nn_matcher_distmat (models/nn_matcher.py:3-43: argmin axis 1, strict '<' threshold,
// argmin axis 0, mutual check), and - distance mode 1 - the training-side matcher
// evaluations/matcher.py:51-102 (||a||^2 + ||b||^2 - 2 ab).
//
// Precision contract.  The contraction is a 3-term split-bf16 product (hi*hi + lo*hi + hi*lo, fp32
// accumulate in registers): ~1e-5 absolute on a distance of unit descriptors, growing with |a| |b|.  Match
// indices must be bit-exact, so every row whose best and second-best distance are closer than a margin eps,
// or whose best distance lies within eps of the threshold, is recomputed by match_exact_kernel with fp32 FMAs in
// ascending k order (the arithmetic of the round-1 FFMA matcher the golden vectors were pinned with) before
// any decision is taken.  Exact ties therefore resolve to the lowest index exactly as np.argmin does.
// eps = MATCH_EPS in distance mode 0 (unit descriptors) and MATCH_EPS * max(1, |a_i| * max_j |b_j|) in mode 1
// (j over the pair's other side).  The exact distance of lines a, b is
//     acc = 0; for k = 0..255: acc = fmaf(a_k, b_k, acc)
//     mode 0: max(0, 2 - 2 acc)      mode 1: max(0, (sq(a) + sq(b)) - 2 acc)
// with sq(x) the same ascending-k fmaf chain of x_k * x_k (desc_tiles_kernel, both layouts).
//
// Operands are "descriptor tile images": the split-bf16 activation-image format of gemm_img.cuh
// (planes hi / lo, 16 KB tiles [row/128][k/64] of 128 rows x 64 k, K-major SWIZZLE_128B), 4 k-blocks
// per 128-row tile.  Either the encoder's final GEMM writes them (pairs whose first line is 128-aligned
// in the batch - every uniform batch with L % 128 == 0) or desc_tiles_kernel builds pair-aligned tiles
// from fp32 descriptors (rows [n, 256] or channel-first [256, n]).
#pragma once
#include "act_img.cuh"
#include "common.cuh"
#include "gemm_img.cuh"
#include "ptx_sm90.cuh"

namespace ltr {

constexpr float MATCH_EPS = 1e-4f;
constexpr int MT_D = 256;                         // descriptor dimension the tensor-core matcher is built for
constexpr int MT_KB = MT_D / 64;                  // k-blocks per tile row
constexpr int MT_TILE = 16384;                    // one plane of a 128 x 64 bf16 tile
constexpr int MT_A_BYTES = MT_KB * 2 * MT_TILE;   // resident A: 4 k-blocks x (hi + lo) = 128 KB
constexpr int MT_STAGE = 2 * MT_TILE;             // B ring stage: one k-block, hi + lo
constexpr int MT_STAGES = 2;
constexpr int MT_OFF_B = MT_A_BYTES;
constexpr int MT_OFF_STG = MT_OFF_B + MT_STAGES * MT_STAGE;   // accumulator staging: 8 blocks of 32 x 32 fp32
constexpr int MT_OFF_BAR = MT_OFF_STG + 8 * 4096;
constexpr int MT_OFF_XCH = MT_OFF_BAR + 256;      // half-merge exchange: 3 x 128 x 4 B
constexpr int MT_SMEM = MT_OFF_XCH + 1536 + 1024; // + alignment slack (<= 227 KB)
constexpr int MT_THREADS = 288;                   // 2 consumer warpgroups (MMA + epilogue), TMA warp
static_assert(MT_SMEM <= 232448, "match_tc: shared memory budget");

// One side of a batch of pairs.
struct MatchSide {
  ActImg img;            // descriptor tile image (kblocks = 4)
  const int* cu;         // [n_pairs + 1] line offsets or nullptr (uniform n); indexed: [n_images + 1] of the pool
  int n;                 // lines per pair when cu == nullptr
  int tile_mode;         // 0: pair p starts at tile p * tmax (pair-aligned scratch tiles)
                         // 1: pair p starts at tile (tile_row0 + first line of p) / 128 (encoder image, aligned pairs)
                         // 2: pair p starts at tile tile_off[pimg[p]] (image-aligned pool, ltr_image_tiles)
  int tile_row0;         // mode 1: row of this side's first line inside the image
  int tmax;              // row tiles per pair (grid sizing; tile stride in mode 0)
  const float* sq;       // mode-1 distance only: squared norms, indexed like the lines (cu / p * n)
  uint2* slot;           // out: per line {bits(best distance), best index | ambiguous << 31}; nullptr = not needed
  const int* pimg;       // indexed: image of every pair [n_pairs] (nullptr: pair p is image p)
  const int* tile_off;   // mode 2: first tile of every image [n_images + 1]
  const int* out_off;    // indexed: first slot of every pair [n_pairs + 1] (one image line takes part in many pairs)
};

struct MatchTcArgs {
  MatchSide s[2];
  int dist_mode;         // 0: 2 - 2 s (unit descriptors, nn_matcher.py:37-38)   1: |a|^2 + |b|^2 - 2 s (evaluations/matcher.py:66-70)
  float thr;             // match threshold (distance mode 1: side-0 rows near it are flagged ambiguous here)
  float* dist;           // optional dense output of side 0 vs side 1, pair p at p * dist_stride, row-major [n0_p, n1_p]
  long long dist_stride;
  int* counts;           // zeroed here (the tail kernel accumulates into it)
  int* done;             // tail-kernel block counter (last-block detection), zeroed here
  int n_pairs;
};

// image of a pair's side: itself unless the side indexes an image pool
__device__ __forceinline__ int side_image(const MatchSide& s, int pair) { return s.pimg ? s.pimg[pair] : pair; }
__device__ __forceinline__ void side_range(const MatchSide& s, int im, int& b, int& e) { image_range(s.cu, s.n, im, b, e); }
__device__ __forceinline__ int side_tile0(const MatchSide& s, int pair, int im, int b) {
  return s.tile_mode == 2 ? s.tile_off[im] : s.tile_mode ? (s.tile_row0 + b) >> 7 : pair * s.tmax;
}

__device__ __forceinline__ void mt_epi_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// grid = (tmax0 + tmax1, n_pairs): CTA x < tmax0 handles row block x of side 0 against all of side 1,
// the others row block x - tmax0 of side 1 against all of side 0.
__global__ void __launch_bounds__(MT_THREADS, 1) match_tc_kernel(MatchTcArgs p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t raw = ptx::smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + MT_OFF_BAR);
  uint64_t* full = bars;                   // [STAGES] B stage landed
  uint64_t* empty = bars + MT_STAGES;      // [STAGES] B stage consumed
  uint64_t* a_full = bars + 2 * MT_STAGES; // [1] resident A landed
  float* xch = reinterpret_cast<float*>(smem + MT_OFF_XCH);
  float* stg_all = reinterpret_cast<float*>(smem + MT_OFF_STG);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int pair = blockIdx.y;
  const int side = (int)blockIdx.x >= p.s[0].tmax ? 1 : 0;
  const int rb = side ? (int)blockIdx.x - p.s[0].tmax : (int)blockIdx.x;
  const MatchSide& SA = p.s[side];
  const MatchSide& SB = p.s[side ^ 1];
  pdl_launch_dependents();

  if (tid == 0) {
    for (int s = 0; s < MT_STAGES; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], 8);
    }
    ptx::mbar_init(a_full, 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();   // descriptors / tile images of the producing kernel are complete from here on

  const int ia = side_image(SA, pair), ib = side_image(SB, pair);
  int ba, ea, bb, eb;
  side_range(SA, ia, ba, ea);
  side_range(SB, ib, bb, eb);
  const int na = ea - ba, nb = eb - bb;
  if (p.counts && blockIdx.x == 0 && tid == 0) p.counts[pair] = 0;
  if (p.done && blockIdx.x == 0 && pair == 0 && tid == 0) *p.done = 0;
  const bool active = rb * 128 < na && nb > 0;   // uniform per CTA
  const int n_ct = active ? (nb + 127) >> 7 : 0;

  if (warp == 8) {
    // ---------------------------------------------------------------- TMA producer
    if (lane == 0 && active) {
      const size_t ta = (size_t)(side_tile0(SA, pair, ia, ba) + rb) * MT_KB;
      ptx::mbar_arrive_expect_tx(a_full, MT_A_BYTES);
#pragma unroll
      for (int kb = 0; kb < MT_KB; ++kb) {
        ptx::bulk_g2s(smem + kb * 2 * MT_TILE, SA.img.hi + (ta + kb) * IMG_TILE_ELEMS, MT_TILE, a_full);
        ptx::bulk_g2s(smem + kb * 2 * MT_TILE + MT_TILE, SA.img.lo + (ta + kb) * IMG_TILE_ELEMS, MT_TILE, a_full);
      }
      const size_t tb0 = (size_t)side_tile0(SB, pair, ib, bb) * MT_KB;
      uint32_t it = 0;
      for (int ct = 0; ct < n_ct; ++ct)
        for (int kb = 0; kb < MT_KB; ++kb, ++it) {
          const int s = it % MT_STAGES;
          const uint32_t ph = (it / MT_STAGES) & 1;
          ptx::mbar_wait(&empty[s], ph ^ 1);
          uint8_t* st = smem + MT_OFF_B + s * MT_STAGE;
          const size_t toff = (tb0 + (size_t)ct * MT_KB + kb) * IMG_TILE_ELEMS;
          ptx::mbar_arrive_expect_tx(&full[s], MT_STAGE);
          ptx::bulk_g2s(st, SB.img.hi + toff, MT_TILE, &full[s]);
          ptx::bulk_g2s(st + MT_TILE, SB.img.lo + toff, MT_TILE, &full[s]);
        }
    }
  } else {
    // ---------------------------------------------------------------- consumers (2 warpgroups x 64 rows)
    // wgmma per 128-column tile of side B (accumulator in registers), then the tile goes through the staging
    // blocks in 64-column chunks: thread = row (lane) x one 32-column half of each chunk; running best /
    // second-best over all column tiles stay in registers.
    const int wg = warp >> 2, q = warp & 3, half = warp >> 2;
    const int row_a = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    float* stg = stg_all + warp * 1024;
    const int r_in = q * 32 + lane;
    const int row = rb * 128 + r_in;             // line of side A inside the pair
    const bool valid_row = row < na;
    float best = INFINITY, second = INFINITY;
    int bidx = 0x7fffffff;
    const float sqa = (p.dist_mode == 1 && valid_row) ? SA.sq[ba + row] : 0.f;
    float* drow = (p.dist && side == 0 && valid_row) ? p.dist + (long long)pair * p.dist_stride + (long long)row * nb : nullptr;
    const bool dvec = drow && (nb % 8 == 0) && (p.dist_stride % 8 == 0) && ((reinterpret_cast<uintptr_t>(p.dist) & 31) == 0);
    // distance mode 1: the largest squared norm of side B, for the margin of this row (see eps below)
    float sqb_max = 0.f;
    if (p.dist_mode == 1 && active) {
      for (int j = tid; j < nb; j += 256) sqb_max = fmaxf(sqb_max, SB.sq[bb + j]);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sqb_max = fmaxf(sqb_max, __shfl_xor_sync(0xffffffffu, sqb_max, o));
      if (lane == 0) xch[warp] = sqb_max;
      mt_epi_bar();
#pragma unroll
      for (int w = 0; w < 8; ++w) sqb_max = fmaxf(sqb_max, xch[w]);
      mt_epi_bar();   // xch is reused by the half merge
    }
    if (active) ptx::mbar_wait(a_full, 0);
    uint32_t it = 0;
    for (int ct = 0; ct < n_ct; ++ct) {
      float d[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) d[i] = 0.f;
      for (int kb = 0; kb < MT_KB; ++kb, ++it) {
        const int s = it % MT_STAGES;
        ptx::mbar_wait(&full[s], (it / MT_STAGES) & 1);
        const uint32_t a_hi = ptx::smem_u32(smem + kb * 2 * MT_TILE) + wg * 8192, a_lo = a_hi + MT_TILE;
        const uint32_t b_hi = ptx::smem_u32(smem + MT_OFF_B + s * MT_STAGE), b_lo = b_hi + MT_TILE;
        ptx::wg_fence_regs(d);
        ptx::wg_fence();
#pragma unroll
        for (int k16 = 0; k16 < 4; ++k16) {
          const uint32_t ko = k16 * 32;
          const uint64_t dah = ptx::make_sw128_kmajor_desc(a_hi + ko, 1024);
          const uint64_t dal = ptx::make_sw128_kmajor_desc(a_lo + ko, 1024);
          const uint64_t dbh = ptx::make_sw128_kmajor_desc(b_hi + ko, 1024);
          const uint64_t dbl = ptx::make_sw128_kmajor_desc(b_lo + ko, 1024);
          ptx::wgmma_ss_n128(d, dal, dbh, (kb | k16) != 0);
          ptx::wgmma_ss_n128(d, dah, dbl, 1);
          ptx::wgmma_ss_n128(d, dah, dbh, 1);
        }
        ptx::wg_commit();
        ptx::wg_wait<1>();
        ptx::wg_fence_regs(d);
        if (kb > 0 && lane == 0) ptx::mbar_arrive(&empty[(it - 1) % MT_STAGES]);
      }
      ptx::wg_wait<0>();
      ptx::wg_fence_regs(d);
      if (lane == 0) ptx::mbar_arrive(&empty[(it - 1) % MT_STAGES]);
#pragma unroll 1
      for (int ch = 0; ch < 2; ++ch) {
        float acc[32];
        mt_epi_bar();
        stage_acc64(d, ch, stg_all, row_a, lane);
        mt_epi_bar();
        load_stage(stg, lane, acc);
        const int j0 = ct * 128 + ch * 64 + half * 32;   // first column (line of side B) of this chunk
        if (j0 >= nb) continue;                  // whole chunk is padding
        if (p.dist_mode == 1) {
#pragma unroll
          for (int j = 0; j < 32; j += 4) {
            float4 sb = make_float4(0.f, 0.f, 0.f, 0.f);
            if (j0 + j + 3 < nb) {
              sb.x = SB.sq[bb + j0 + j]; sb.y = SB.sq[bb + j0 + j + 1]; sb.z = SB.sq[bb + j0 + j + 2]; sb.w = SB.sq[bb + j0 + j + 3];
            } else {
              if (j0 + j < nb) sb.x = SB.sq[bb + j0 + j];
              if (j0 + j + 1 < nb) sb.y = SB.sq[bb + j0 + j + 1];
              if (j0 + j + 2 < nb) sb.z = SB.sq[bb + j0 + j + 2];
            }
            acc[j] = fmaxf((sqa + sb.x) - 2.f * acc[j], 0.f);
            acc[j + 1] = fmaxf((sqa + sb.y) - 2.f * acc[j + 1], 0.f);
            acc[j + 2] = fmaxf((sqa + sb.z) - 2.f * acc[j + 2], 0.f);
            acc[j + 3] = fmaxf((sqa + sb.w) - 2.f * acc[j + 3], 0.f);
          }
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j) acc[j] = fmaxf(fmaf(-2.f, acc[j], 2.f), 0.f);
        }
        if (j0 + 32 <= nb) {
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const float v = acc[j];
            if (v < best) { second = best; best = v; bidx = j0 + j; }
            else if (v < second) second = v;
          }
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const float v = (j0 + j < nb) ? acc[j] : INFINITY;
            if (v < best) { second = best; best = v; bidx = j0 + j; }
            else if (v < second) second = v;
          }
        }
        if (drow) {
          if (dvec && j0 + 32 <= nb) {
#pragma unroll
            for (int j = 0; j < 32; j += 8) {
              const uint4 a = make_uint4(__float_as_uint(acc[j]), __float_as_uint(acc[j + 1]), __float_as_uint(acc[j + 2]), __float_as_uint(acc[j + 3]));
              const uint4 b = make_uint4(__float_as_uint(acc[j + 4]), __float_as_uint(acc[j + 5]), __float_as_uint(acc[j + 6]), __float_as_uint(acc[j + 7]));
              ptx::st_global_256(drow + j0 + j, a, b);
            }
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (j0 + j < nb) drow[j0 + j] = acc[j];
          }
        }
      }
    }
    // merge the two column halves of every row (lexicographic (value, index): first minimum wins)
    if (half == 1) {
      xch[r_in] = best;
      xch[128 + r_in] = second;
      reinterpret_cast<int*>(xch)[256 + r_in] = bidx;
    }
    mt_epi_bar();
    if (half == 0 && valid_row) {
      const float ob = xch[r_in], os = xch[128 + r_in];
      const int oi = reinterpret_cast<int*>(xch)[256 + r_in];
      if (ob < best || (ob == best && oi < bidx)) { second = fminf(best, os); best = ob; bidx = oi; }
      else second = fminf(second, ob);
      // Margin below which the tensor-core value cannot decide: MATCH_EPS for unit descriptors (mode 0).  In mode 1
      // the product error grows with |a| |b|, so the margin is MATCH_EPS * max(1, |a_i| * max_j |b_j|), and it also
      // covers the distance to the threshold on side 0 (the tail's own MATCH_EPS check is then never the tighter one).
      bool amb = !(second - best >= MATCH_EPS);   // also true for NaN
      if (p.dist_mode == 1) {
        const float eps = MATCH_EPS * fmaxf(1.f, sqrtf(sqa * sqb_max));
        amb = !(second - best >= eps) || (side == 0 && !(fabsf(best - p.thr) >= eps));
      }
      if (SA.slot) {
        const int sbase = SA.pimg ? SA.out_off[pair] : ba;   // slots are per (pair, line) when images are shared
        SA.slot[sbase + row] = make_uint2(__float_as_uint(best), (uint32_t)bidx | (amb ? 0x80000000u : 0u));
      }
    }
  }
}

// ---------------------------------------------------------------- fp32 descriptors -> pair- or image-aligned tile images
struct DescTilesArgs {
  const float* d[2];     // fp32 descriptors of side 0 / 1
  int layout;            // 0 rows [n, 256] per line; 1 channel-first [256, n_p] per pair (pair p at 256 * first line)
  const int* cu[2]; int n[2];
  ActImg img[2]; int tmax[2];
  float* sq[2];          // optional squared norms per line (distance mode 1) or nullptr
  const int* tile_off[2];  // image-aligned pool (ltr_image_tiles): "pair" p is image p, its ceil(n_p / 128) tiles
                           // start at tile_off[p]; nullptr: pair-aligned, pair p at tile p * tmax
};

// Squared norm of one line for distance mode 1: a single ascending-k fmaf chain, s = fmaf(x_k, x_k, s) for
// k = 0..255 - the order of the exact pass's dot products, and the same in both descriptor layouts, so the same
// descriptors get the same bits wherever they come from.  x_k is at x[k * stride].
__device__ __forceinline__ float sq_chain(const float* __restrict__ x, size_t stride) {
  float s = 0.f;
#pragma unroll 8
  for (int k = 0; k < MT_D; ++k) s = fmaf(x[k * stride], x[k * stride], s);
  return s;
}

// grid = (max(tmax0, tmax1) * 4, n_pairs, 2): block = 32 lines of one tile; 256 threads.
__global__ void __launch_bounds__(256) desc_tiles_kernel(DescTilesArgs p) {
  pdl_launch_dependents();
  pdl_wait();
  const int side = blockIdx.z, pair = blockIdx.y;
  const int tile = blockIdx.x >> 2, sub = blockIdx.x & 3;
  if (tile >= p.tmax[side]) return;
  int b, e;
  image_range(p.cu[side], p.n[side], pair, b, e);
  const int n = e - b;
  if (p.tile_off[side] && tile * 128 >= n) return;   // an image owns only the tiles its lines need
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* __restrict__ src = p.d[side];
  const ActImg& img = p.img[side];
  const size_t t0 = ((p.tile_off[side] ? (size_t)p.tile_off[side][pair] : (size_t)pair * p.tmax[side]) + tile) * MT_KB;
  uint8_t* hi = reinterpret_cast<uint8_t*>(img.hi);
  uint8_t* lo = reinterpret_cast<uint8_t*>(img.lo);
  if (p.layout == 0) {
    // warp -> 4 consecutive lines, lane -> 8 consecutive k
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r_in = sub * 32 + warp * 4 + i, r = tile * 128 + r_in;
      float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (r < n) {
        const float4 a = *reinterpret_cast<const float4*>(src + (size_t)(b + r) * MT_D + lane * 8);
        const float4 c = *reinterpret_cast<const float4*>(src + (size_t)(b + r) * MT_D + lane * 8 + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = c.x; v[5] = c.y; v[6] = c.z; v[7] = c.w;
      }
      uint4 h, l;
      ptx::split8_bf16(v, h, l);
      const size_t off = (t0 + (lane >> 3)) * (size_t)MT_TILE + ptx::sw128_offset(r_in, (lane & 7) * 8);
      *reinterpret_cast<uint4*>(hi + off) = h;
      *reinterpret_cast<uint4*>(lo + off) = l;
    }
    if (p.sq[side] && lane < 4) {   // lanes 0-3: the 4 lines this warp just converted
      const int r = tile * 128 + sub * 32 + warp * 4 + lane;
      if (r < n) p.sq[side][b + r] = sq_chain(src + (size_t)(b + r) * MT_D, 1);
    }
  } else {
    // lane -> line, warp -> groups of 8 consecutive k (4 groups per warp): loads coalesced along lines
    const int r_in = sub * 32 + lane, r = tile * 128 + r_in;
    const float* __restrict__ base = src + (size_t)b * MT_D;   // [256, n] of this pair
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const int k0 = (g * 8 + warp) * 8;
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = (r < n) ? base[(size_t)(k0 + j) * n + r] : 0.f;
      uint4 h, l;
      ptx::split8_bf16(v, h, l);
      const size_t off = (t0 + (k0 >> 6)) * (size_t)MT_TILE + ptx::sw128_offset(r_in, k0 & 63);
      *reinterpret_cast<uint4*>(hi + off) = h;
      *reinterpret_cast<uint4*>(lo + off) = l;
    }
    if (p.sq[side] && warp == 0 && r < n) p.sq[side][b + r] = sq_chain(base + r, n);   // coalesced along lines
  }
}

// ---------------------------------------------------------------- exact re-check of the flagged lines
// Slot word y after match_exact_kernel: bit 31 ambiguous (tensor-core result, not trusted), bit 30 decided exactly.
// An exact slot holds the index in bits 0-29, all ones when no column had a distance below infinity (index
// 0x7fffffff, as np.argmin never returns it); line counts per pair stay below 2^30 (run_match checks it).
constexpr uint32_t SLOT_AMBIGUOUS = 0x80000000u, SLOT_EXACT = 0x40000000u;
__device__ __forceinline__ int slot_index(uint32_t y) {
  const uint32_t i = y & 0x3fffffffu;
  return i == 0x3fffffffu ? 0x7fffffff : (int)i;
}

struct MatchExactArgs {
  const float* d[2]; int layout;   // the fp32 descriptors the tiles were made from
  const int* cu[2]; int n[2];
  const float* sq[2];              // distance mode 1
  int dist_mode;
  uint2* slot[2];                  // read (flags), and the flagged lines' slots rewritten
  float thr; int mutual;
  const int* pimg[2]; const int* out_off[2];   // indexed mode, as in MatchTailArgs
};

// The exact distance of two lines from their ascending-k fmaf chain acc (see the header), before the clip at 0.
__device__ __forceinline__ float exact_dist_raw(float acc, float sqa, float sqb, int dist_mode) {
  return dist_mode == 1 ? (sqa + sqb) - 2.f * acc : 2.f - 2.f * acc;
}
// ... and clipped, shared by every exact matcher path.
__device__ __forceinline__ float exact_dist(float acc, float sqa, float sqb, int dist_mode) {
  return fmaxf(exact_dist_raw(acc, sqa, sqb, dist_mode), 0.f);
}

constexpr int MX_WIN = 256;                 // lines of one side a CTA scans for flags per window (one per thread)
constexpr int MX_R = 32;                    // flagged rows per group: 4 row blocks of 8 rows
constexpr int MX_C = 64;                    // columns of the other side per staged chunk
constexpr int MX_BLD = MX_C + 1;            // padded k-row of the chunk: transposing stores hit 32 banks
constexpr int MX_OFF_B = MT_D * MX_R * 4;   // As [256][32] k-major, then Bs [256][65]
constexpr int MX_SMEM = MX_OFF_B + MT_D * MX_BLD * 4;

// The exact FMA tiling (match_exact_kernel, triplet_mine_kernel), 256 threads.  A group of up to 32 rows of side a sits
// k-major in As [k][MX_R]; chunks of 64 lines of side b go k-major into Bs [k][MX_BLD]; thread (rb = tid / 64,
// c = tid % 64) runs the 8 fmaf chains of rows rb * 8 .. + 7 against column c.
//
// Row r of side a (lines [ba, ba + na)) into column `lane` of As: lane -> row, warps split k in float4 steps.
__device__ __forceinline__ void mx_stage_row(float* As, const float* __restrict__ A, int layout, int ba, int na, int r,
                                             int lane, int warp) {
  if (layout == 0) {
    const float4* __restrict__ x = reinterpret_cast<const float4*>(A + (size_t)(ba + r) * MT_D);
    for (int k4 = warp; k4 < MT_D / 4; k4 += 8) {
      const float4 v = x[k4];
      As[(4 * k4) * MX_R + lane] = v.x; As[(4 * k4 + 1) * MX_R + lane] = v.y;
      As[(4 * k4 + 2) * MX_R + lane] = v.z; As[(4 * k4 + 3) * MX_R + lane] = v.w;
    }
  } else {
    const float* __restrict__ x = A + (size_t)ba * MT_D + r;
    for (int k = warp; k < MT_D; k += 8) As[k * MX_R + lane] = x[(size_t)k * na];
  }
}

// Lines j0 .. j0 + 63 of side b (lines [bb, bb + nb)) into Bs, zeros past nb.
__device__ __forceinline__ void mx_stage_chunk(float* Bs, const float* __restrict__ B, int layout, int bb, int nb, int j0,
                                               int tid, int rb, int c) {
  if (layout == 0) {
    // 8 lanes read one line's 128 B run of float4s (coalesced), 4 lines per warp; padded transpose into Bs
    for (int e = tid; e < MX_C * (MT_D / 4); e += 256) {
      const int cc = (e >> 3) & (MX_C - 1), k4 = ((e >> 9) << 3) | (e & 7);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (j0 + cc < nb) v = reinterpret_cast<const float4*>(B + (size_t)(bb + j0 + cc) * MT_D)[k4];
      Bs[(4 * k4) * MX_BLD + cc] = v.x; Bs[(4 * k4 + 1) * MX_BLD + cc] = v.y;
      Bs[(4 * k4 + 2) * MX_BLD + cc] = v.z; Bs[(4 * k4 + 3) * MX_BLD + cc] = v.w;
    }
  } else {
    const float* __restrict__ y = B + (size_t)bb * MT_D + j0 + c;
    const bool col = j0 + c < nb;
    for (int k = rb; k < MT_D; k += 4) Bs[k * MX_BLD + c] = col ? y[(size_t)k * nb] : 0.f;
  }
}

// acc[i] = ascending-k fmaf chain of row rb * 8 + i of As with column c of Bs (rows read as broadcast LDS.128).
__device__ __forceinline__ void mx_dot8(const float* As, const float* Bs, int rb, int c, float acc[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  const float4* __restrict__ a4 = reinterpret_cast<const float4*>(As) + rb * 2;
#pragma unroll 8
  for (int k = 0; k < MT_D; ++k) {
    const float4 x0 = a4[k * (MX_R / 4)], x1 = a4[k * (MX_R / 4) + 1];
    const float y = Bs[k * MX_BLD + c];
    acc[0] = fmaf(x0.x, y, acc[0]); acc[1] = fmaf(x0.y, y, acc[1]);
    acc[2] = fmaf(x0.z, y, acc[2]); acc[3] = fmaf(x0.w, y, acc[3]);
    acc[4] = fmaf(x1.x, y, acc[4]); acc[5] = fmaf(x1.y, y, acc[5]);
    acc[6] = fmaf(x1.z, y, acc[6]); acc[7] = fmaf(x1.w, y, acc[7]);
  }
}

// grid = (n_pairs, 2 sides, S), 256 threads.  CTA (pair, side, z) scans the windows w = z, z + S, ... of MX_WIN lines
// of its side, compacts the lines whose slot cannot be trusted (side 0: ambiguous or within MATCH_EPS of the
// threshold; side 1: ambiguous, only when mutual) and recomputes each with fp32 FMAs in ascending k against every
// line of the other side.  Groups of 32 rows sit k-major in shared memory; the other side streams through in
// 64-column chunks.  Thread = 8 rows (broadcast LDS.128) x 1 column, 8 independent fmaf chains; each thread keeps a
// running first-minimum over its columns in ascending j, then the 64 column threads of a row merge lexicographically.
__global__ void __launch_bounds__(256) match_exact_kernel(MatchExactArgs p) {
  extern __shared__ __align__(16) float mx_smem[];
  float* As = mx_smem;                      // [k][MX_R]
  float* Bs = mx_smem + MT_D * MX_R;        // [k][MX_BLD]
  __shared__ int list[MX_WIN];
  __shared__ int wcount[8];
  __shared__ float xb[MX_R];
  __shared__ int xi[MX_R];
  pdl_launch_dependents();
  const int pair = blockIdx.x, sa = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (sa == 1 && !p.mutual) return;
  pdl_wait();
  // side a = the lines re-checked here, side b = the other side (selects, not indexing: the params stay in constant bank)
  const int* pimg_a = sa ? p.pimg[1] : p.pimg[0];
  const int* pimg_b = sa ? p.pimg[0] : p.pimg[1];
  const int* oo_a = sa ? p.out_off[1] : p.out_off[0];
  int ba, ea, bb, eb;
  image_range(sa ? p.cu[1] : p.cu[0], sa ? p.n[1] : p.n[0], pimg_a ? pimg_a[pair] : pair, ba, ea);
  image_range(sa ? p.cu[0] : p.cu[1], sa ? p.n[0] : p.n[1], pimg_b ? pimg_b[pair] : pair, bb, eb);
  const int na = ea - ba, nb = eb - bb;
  if (na == 0 || nb == 0) return;           // match_tc_kernel wrote no slots for this pair
  uint2* slot = (sa ? p.slot[1] : p.slot[0]) + (oo_a ? oo_a[pair] : ba);
  const float* __restrict__ A = sa ? p.d[1] : p.d[0];
  const float* __restrict__ B = sa ? p.d[0] : p.d[1];
  const float* __restrict__ sq_a = sa ? p.sq[1] : p.sq[0];
  const float* __restrict__ sq_b = sa ? p.sq[0] : p.sq[1];
  const int rb = tid >> 6, c = tid & 63;    // row block (rows rb * 8 .. + 7 of a group), column in the chunk
  for (int w0 = blockIdx.z * MX_WIN; w0 < na; w0 += gridDim.z * MX_WIN) {
    // ---- compact the flagged lines of the window (ballot + prefix over the warps)
    bool flag = false;
    if (w0 + tid < na) {
      const uint2 s = slot[w0 + tid];
      flag = (s.y & SLOT_AMBIGUOUS) != 0;
      if (sa == 0) flag = flag || !(fabsf(__uint_as_float(s.x) - p.thr) >= MATCH_EPS);
    }
    const unsigned fb = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) wcount[warp] = __popc(fb);
    __syncthreads();
    int pre = 0, nf = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      pre += q < warp ? wcount[q] : 0;
      nf += wcount[q];
    }
    if (flag) list[pre + __popc(fb & ((1u << lane) - 1u))] = w0 + tid;
    __syncthreads();
    for (int g0 = 0; g0 < nf; g0 += MX_R) {
      const int nr = min(MX_R, nf - g0);
      // ---- stage the group's rows k-major (stores conflict-free)
      if (lane < nr) mx_stage_row(As, A, p.layout, ba, na, list[g0 + lane], lane, warp);
      float sqa[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int gi = rb * 8 + i;
        sqa[i] = (p.dist_mode == 1 && gi < nr) ? sq_a[ba + list[g0 + gi]] : 0.f;
      }
      float best[8];
      int bidx[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) { best[i] = INFINITY; bidx[i] = 0x7fffffff; }
      for (int j0 = 0; j0 < nb; j0 += MX_C) {
        __syncthreads();   // As staged / the previous chunk consumed
        // ---- stage columns j0 .. j0 + 63 of the other side k-major (zeros past nb)
        mx_stage_chunk(Bs, B, p.layout, bb, nb, j0, tid, rb, c);
        __syncthreads();
        if (rb * 8 < nr) {
          float acc[8];
          mx_dot8(As, Bs, rb, c, acc);
          const int j = j0 + c;
          if (j < nb) {
            const float sqb = p.dist_mode == 1 ? sq_b[bb + j] : 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float v = exact_dist(acc[i], sqa[i], sqb, p.dist_mode);
              if (v < best[i]) { best[i] = v; bidx[i] = j; }
            }
          }
        }
      }
      // ---- merge the 64 column threads of every row: 32 lanes by shuffles, then the two warps of a row block
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const float ov = __shfl_xor_sync(0xffffffffu, best[i], o);
          const int oi = __shfl_xor_sync(0xffffffffu, bidx[i], o);
          if (ov < best[i] || (ov == best[i] && oi < bidx[i])) { best[i] = ov; bidx[i] = oi; }
        }
      }
      if ((warp & 1) && lane == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) { xb[rb * 8 + i] = best[i]; xi[rb * 8 + i] = bidx[i]; }
      }
      __syncthreads();
      if (!(warp & 1) && lane < 8 && rb * 8 + lane < nr) {
        float v = best[0];
        int idx = bidx[0];
#pragma unroll
        for (int i = 1; i < 8; ++i)
          if (lane == i) { v = best[i]; idx = bidx[i]; }
        const float ov = xb[rb * 8 + lane];
        const int oi = xi[rb * 8 + lane];
        if (ov < v || (ov == v && oi < idx)) { v = ov; idx = oi; }
        slot[list[g0 + rb * 8 + lane]] = make_uint2(__float_as_uint(v), (uint32_t)idx | SLOT_EXACT);
      }
    }
    __syncthreads();   // list / wcount / xb are rewritten by the next window
  }
}

// ---------------------------------------------------------------- tail: threshold, mutual, counts
struct MatchTailArgs {
  const int* cu[2]; int n[2];
  const uint2* slot[2];
  float thr; int mutual;
  int* matches0; float* scores0; int* nn1; int* counts;
  int max0;                        // max lines of side 0 per pair (row part of the grid)
  // indexed mode (image pools): cu[s] are image offsets, pimg[s][pair] the image of a pair's side, and slots /
  // outputs of the pair start at out_off[s][pair]; nullptr: pair p is image p and its outputs start at cu[s][p]
  const int* pimg[2]; const int* out_off[2];
  // multi-GPU publication of `counts` (LtrPeerGather): symmetric buffer = counts[SLOTS][world][n_pairs] | flags[SLOTS][world]
  int* done;                       // block counter for last-block detection
  int* mc_base; int* const* peer_bases;
  int rank, world, gslot, epoch, n_pairs;
};

constexpr int GATHER_SLOTS = 8;   // = LTR_GATHER_SLOTS
__device__ __forceinline__ void multimem_st_u32(int* mc_addr, int v) {
  asm volatile("multimem.st.relaxed.sys.global.u32 [%0], %1;" ::"l"(mc_addr), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_acquire_sys(const int* p) {
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// grid = (ceil((max0 + max1) / 256), n_pairs), 256 threads, one line per thread: items below max0 decide side-0
// lines (matches0 / scores0 / counts), the others publish nn1 (argmin over axis 0).  Every slot holds a result
// that can be trusted as it stands: match_exact_kernel has already re-taken the ones match_tc_kernel flagged.
__global__ void __launch_bounds__(256) match_tail_kernel(MatchTailArgs p) {
  __shared__ int n_keep;
  pdl_launch_dependents();
  pdl_wait();
  const int pair = blockIdx.y, tid = threadIdx.x, lane = tid & 31;
  int b0, e0, b1, e1;
  image_range(p.cu[0], p.n[0], p.pimg[0] ? p.pimg[0][pair] : pair, b0, e0);
  image_range(p.cu[1], p.n[1], p.pimg[1] ? p.pimg[1][pair] : pair, b1, e1);
  const int n0 = e0 - b0, n1 = e1 - b1;
  const int o0 = p.out_off[0] ? p.out_off[0][pair] : b0, o1 = p.out_off[1] ? p.out_off[1][pair] : b1;
  if (tid == 0) n_keep = 0;
  __syncthreads();
  const int w = blockIdx.x * 256 + tid;
  bool keep = false;
  if (w < p.max0) {
    const int i = w;
    if (i < n0) {
      if (n1 == 0) {
        p.matches0[o0 + i] = -1;
        p.scores0[o0 + i] = INFINITY;
      } else {
        const uint2 s = p.slot[0][o0 + i];
        const float v = __uint_as_float(s.x);
        const int idx = slot_index(s.y);
        keep = v < p.thr;   // strict '<' (nn_matcher.py:18)
        if (keep && p.mutual) keep = slot_index(p.slot[1][o1 + idx].y) == i;
        p.matches0[o0 + i] = keep ? idx : -1;
        p.scores0[o0 + i] = v;
      }
    }
  } else if (p.mutual) {
    const int j = w - p.max0;
    if (j < n1) p.nn1[o1 + j] = n0 == 0 ? -1 : slot_index(p.slot[1][o1 + j].y);
  }
  const unsigned kb = __ballot_sync(0xffffffffu, keep);
  if (lane == 0 && kb) atomicAdd(&n_keep, __popc(kb));
  __syncthreads();
  if (tid == 0 && n_keep) atomicAdd(&p.counts[pair], n_keep);
  if (p.world > 1) {
    // ---- fused collective: the LAST block of the grid publishes this rank's counts to every rank over NVLink ----
    __shared__ int is_last;
    if (tid == 0) {
      __threadfence();
      is_last = atomicAdd(p.done, 1) == (int)(gridDim.x * gridDim.y) - 1;
    }
    __syncthreads();
    if (is_last) {
      __threadfence();
      const long long cnt_off = ((long long)p.gslot * p.world + p.rank) * p.n_pairs;
      const long long flag_off = (long long)GATHER_SLOTS * p.world * p.n_pairs + (long long)p.gslot * p.world + p.rank;
      for (int i = tid; i < p.n_pairs; i += 256) {
        const int v = __ldcg(p.counts + i);
        if (p.mc_base) multimem_st_u32(p.mc_base + cnt_off + i, v);
        else
          for (int r = 0; r < p.world; ++r) p.peer_bases[r][cnt_off + i] = v;
      }
      __threadfence_system();
      __syncthreads();
      if (tid == 0) {
        if (p.mc_base) multimem_st_u32(p.mc_base + flag_off, p.epoch);
        else
          for (int r = 0; r < p.world; ++r) *reinterpret_cast<volatile int*>(p.peer_bases[r] + flag_off) = p.epoch;
        __threadfence_system();
      }
    }
  }
}

// one block: wait until every rank's flag of the slot reached `epoch`, then copy the gathered counts out
__global__ void __launch_bounds__(256) gather_wait_kernel(const int* base, int world, int n_pairs, int slot, int epoch, int* out) {
  pdl_launch_dependents();
  pdl_wait();
  const int* flags = base + (long long)GATHER_SLOTS * world * n_pairs + (long long)slot * world;
  if ((int)threadIdx.x < world) {
    const long long t0 = clock64();
    while (ld_acquire_sys(flags + threadIdx.x) < epoch)
      if (clock64() - t0 > 20000000000LL) __trap();   // ~10 s: a rank died - fail loudly instead of hanging
  }
  __syncthreads();
  const int* src = base + (long long)slot * world * n_pairs;
  for (int i = threadIdx.x; i < world * n_pairs; i += 256) out[i] = __ldcv(src + i);
}

}  // namespace ltr
