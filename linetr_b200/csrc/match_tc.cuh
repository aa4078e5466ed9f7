// Tensor-core descriptor matcher (K3): all-pairs distance D = 2 - 2 <a_i, b_j> on wgmma with the
// row-argmin fused into the epilogue, for BOTH directions (side 0 rows vs side 1 and side 1 rows vs
// side 0 - the second one is the column argmin the mutual check needs), a tail kernel that applies
// threshold + mutual check + per-pair counts, and an exact fp32 re-check for decisions the
// tensor-core arithmetic cannot make safely.
//
// Reference: get_dist_matrix (models/line_process.py:198-201: einsum('bdn,bdm->bnm'), (2 - 2 s).clip(0)),
// nn_matcher / nn_matcher_distmat (models/nn_matcher.py:3-43: argmin axis 1, strict '<' threshold,
// argmin axis 0, mutual check), and - distance mode 1 - the training-side matcher
// evaluations/matcher.py:51-102 (||a||^2 + ||b||^2 - 2 ab).
//
// Precision contract.  The contraction is a 3-term split-bf16 product (hi*hi + lo*hi + hi*lo, fp32
// accumulate in registers): ~1e-5 absolute on a distance of unit descriptors, growing with |a| |b|.  Match
// indices must be bit-exact, so every row whose best and second-best distance are closer than a margin eps,
// or whose best distance lies within eps of the threshold, is recomputed by the tail kernel with fp32 FMAs in
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
// k = 0..255 - the order of exact_row's dot products, and the same in both descriptor layouts, so the same
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

// ---------------------------------------------------------------- tail: exact re-check, threshold, mutual, counts
struct MatchTailArgs {
  const float* d[2]; int layout;   // the fp32 descriptors the tiles were made from (exact re-check)
  const int* cu[2]; int n[2];
  const float* sq[2];              // distance mode 1
  int dist_mode;
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

// Exact fp32 distances of line `r` of side `sa` to every line of the other side (ascending-k fmaf chain,
// the arithmetic of the round-1 FFMA matcher), first-minimum argmin over them; whole warp.
__device__ __forceinline__ void exact_row(const MatchTailArgs& p, int sa, int pair_b_a, int na, int r, int pair_b_b, int nb,
                                          float* xrow, int lane, float& best, int& bidx) {
  const int sb = sa ^ 1;
  const float* __restrict__ A = p.d[sa];
  const float* __restrict__ B = p.d[sb];
  // stage the row in shared memory (per-warp 1 KB)
  if (p.layout == 0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) xrow[i * 32 + lane] = A[(size_t)(pair_b_a + r) * MT_D + i * 32 + lane];
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) xrow[i * 32 + lane] = A[(size_t)pair_b_a * MT_D + (size_t)(i * 32 + lane) * na + r];
  }
  __syncwarp();
  const float sqa = p.dist_mode == 1 ? p.sq[sa][pair_b_a + r] : 0.f;
  best = INFINITY; bidx = 0x7fffffff;
  for (int j = lane; j < nb; j += 32) {
    float acc = 0.f;
    if (p.layout == 0) {
      const float4* __restrict__ y = reinterpret_cast<const float4*>(B + (size_t)(pair_b_b + j) * MT_D);
#pragma unroll 8
      for (int k = 0; k < MT_D / 4; ++k) {
        const float4 b = y[k];
        acc = fmaf(xrow[4 * k], b.x, acc);
        acc = fmaf(xrow[4 * k + 1], b.y, acc);
        acc = fmaf(xrow[4 * k + 2], b.z, acc);
        acc = fmaf(xrow[4 * k + 3], b.w, acc);
      }
    } else {
      const float* __restrict__ y = B + (size_t)pair_b_b * MT_D + j;
#pragma unroll 8
      for (int k = 0; k < MT_D; ++k) acc = fmaf(xrow[k], y[(size_t)k * nb], acc);
    }
    const float v = p.dist_mode == 1 ? fmaxf((sqa + p.sq[sb][pair_b_b + j]) - 2.f * acc, 0.f) : fmaxf(2.f - 2.f * acc, 0.f);
    if (v < best) { best = v; bidx = j; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
    if (ov < best || (ov == best && oi < bidx)) { best = ov; bidx = oi; }
  }
  __syncwarp();
}

// One decision (warp-cooperative; used for the lines whose slots are flagged ambiguous): side-0 line i ->
// matches0 / scores0 (returns keep), or side-1 line j -> nn1.  b0 / b1: first descriptor row of each side,
// o0 / o1: first slot / output of each side (equal unless images are shared between pairs).
__device__ __forceinline__ bool tail_decide_row(const MatchTailArgs& p, int i, int b0, int o0, int n0, int b1, int o1, int n1,
                                                float* xrow, int lane, bool force_exact) {
  const uint2 s = p.slot[0][o0 + i];
  float v = __uint_as_float(s.x);
  int idx = (int)(s.y & 0x7fffffffu);
  if (force_exact || (s.y >> 31) || !(fabsf(v - p.thr) >= MATCH_EPS)) exact_row(p, 0, b0, n0, i, b1, n1, xrow, lane, v, idx);
  bool keep = v < p.thr;   // strict '<' (nn_matcher.py:18)
  if (keep && p.mutual) {
    const uint2 t = p.slot[1][o1 + idx];
    int back = (int)(t.y & 0x7fffffffu);
    if (t.y >> 31) {
      float bv;
      exact_row(p, 1, b1, n1, idx, b0, n0, xrow, lane, bv, back);
    }
    keep = back == i;
  }
  if (lane == 0) {
    p.matches0[o0 + i] = keep ? idx : -1;
    p.scores0[o0 + i] = v;
  }
  return keep;
}

// grid = (ceil((max0 + max1) / 256), n_pairs), 256 threads, one line per THREAD on the fast path: items below
// max0 decide side-0 lines (matches0 / scores0 / counts), the others publish nn1 (argmin over axis 0).
// Lines whose tensor-core result cannot be trusted (ambiguous slot, score next to the threshold, or an
// ambiguous partner column) go to a shared work list that the block's 8 warps then process
// cooperatively with exact fp32 arithmetic.
__global__ void __launch_bounds__(256) match_tail_kernel(MatchTailArgs p) {
  __shared__ float xrows[8][MT_D];
  __shared__ int work[256];
  __shared__ int n_work, n_keep;
  pdl_launch_dependents();
  pdl_wait();
  const int pair = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  int b0, e0, b1, e1;
  image_range(p.cu[0], p.n[0], p.pimg[0] ? p.pimg[0][pair] : pair, b0, e0);
  image_range(p.cu[1], p.n[1], p.pimg[1] ? p.pimg[1][pair] : pair, b1, e1);
  const int n0 = e0 - b0, n1 = e1 - b1;
  const int o0 = p.out_off[0] ? p.out_off[0][pair] : b0, o1 = p.out_off[1] ? p.out_off[1][pair] : b1;
  if (tid == 0) { n_work = 0; n_keep = 0; }
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
        const int idx = (int)(s.y & 0x7fffffffu);
        bool hard = (s.y >> 31) || !(fabsf(v - p.thr) >= MATCH_EPS);
        if (!hard) {
          keep = v < p.thr;
          if (keep && p.mutual) {
            const uint2 t = p.slot[1][o1 + idx];
            if (t.y >> 31) { hard = true; keep = false; }
            else keep = (int)(t.y & 0x7fffffffu) == i;
          }
        }
        if (hard) work[atomicAdd(&n_work, 1)] = w;
        else { p.matches0[o0 + i] = keep ? idx : -1; p.scores0[o0 + i] = v; }
      }
    }
  } else if (p.mutual) {
    const int j = w - p.max0;
    if (j < n1) {
      if (n0 == 0) p.nn1[o1 + j] = -1;
      else {
        const uint2 t = p.slot[1][o1 + j];
        if (t.y >> 31) work[atomicAdd(&n_work, 1)] = w;
        else p.nn1[o1 + j] = (int)(t.y & 0x7fffffffu);
      }
    }
  }
  const unsigned kb = __ballot_sync(0xffffffffu, keep);
  if (lane == 0 && kb) atomicAdd(&n_keep, __popc(kb));
  __syncthreads();
  for (int e = warp; e < n_work; e += 8) {     // exact path, one work item per warp at a time
    const int ww = work[e];
    if (ww < p.max0) {
      if (tail_decide_row(p, ww, b0, o0, n0, b1, o1, n1, xrows[warp], lane, false) && lane == 0) atomicAdd(&n_keep, 1);
    } else {
      const int j = ww - p.max0;
      float bv; int back;
      exact_row(p, 1, b1, n1, j, b0, n0, xrows[warp], lane, bv, back);
      if (lane == 0) p.nn1[o1 + j] = back;
    }
  }
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
