// Semi-hard triplet loss of the reference's validation step, forward value only.
// Reference: descriptor_loss.compute_distances + forward (evaluations/criteria.py:35-192), as train.py:198-240
// (run_epochs('val')) calls it, and Evaluate_PR.calc_TFPN (evaluations/evaluate_pr.py:10-22) of the matcher's
// predictions against the same assignment.
//
// Per pair, d[i, j] = 2 - 2 <a_i, b_j> is the exact path's fp32 distance (ascending-k fmaf chain, exact_dist_raw) NOT
// clipped at 0.  The anchors are every side-0 line i (candidates d[i, :]) and then every side-1 line j (candidates
// d[:, j]), the reference's cat((X, X^T), 1).  For an anchor:
//   match    = (double)v > match_thr, unmatch = (double)v <= unmatch_thr, v its assignment entry;
//   pos      = max of d over the match candidates; the anchor has a positive iff pos > 0 (the reference's
//              max over match ? d : d*0, then > 0);
//   u        = unmatch ? d : 10000.f (the reference's literal: matched and in-between entries take part as 10000);
//   neg      = min of u over pos < u < pos + 0.5f; the anchor is valid iff that window is not empty.
// Every decision is taken on fp32 values that are bit-identical to a host fmaf model, so no margin is needed.
#pragma once
#include "common.cuh"
#include "line_gt.cuh"
#include "match_tc.cuh"

namespace ltr {

constexpr float TRIPLET_FAR = 10000.0f;     // criteria.py:95 max_dist
constexpr float TRIPLET_MARGIN = 0.5f;      // criteria.py:102
constexpr float TRIPLET_LOSS_MARGIN = 1.0f; // criteria.py:183

struct TripletArgs {
  const float* d[2]; int layout;   // descriptors of side 0 / side 1 (LTR_LAYOUT_*)
  const int* cu[2]; int n[2];      // line offsets [n_pairs + 1] or nullptr (uniform n)
  const float* assign; long long assign_stride; int assign_ld;   // ld 0: n1 of the pair
  double match_thr, unmatch_thr;
  const int* pred0;                // optional [S0]: local side-1 index or -1
  float* pos; float* neg; int* state;   // [S0 + S1] anchors
  int* tfpn;                       // [n_pairs, 4], zeroed by the caller, when pred0
};

// First anchor of pair p: side 0 then side 1 of every pair, pair-major.
__device__ __forceinline__ long long triplet_anchor0(const int* cu0, const int* cu1, int n0, int n1, int p) {
  return cu0 ? (long long)cu0[p] + cu1[p] : (long long)p * (n0 + n1);
}

// grid = (n_pairs, 2 sides, S), 256 threads.  CTA (pair, side, z) takes the anchors of its side 32 at a time (windows
// z, z + S, ...), k-major in shared memory, and streams the other side through in 64-column chunks with
// match_exact_kernel's tiling (thread = 8 anchors x 1 column, 8 independent fmaf chains).  Phase 1 takes the max over
// the match candidates (chunks without one are skipped), phase 2 the min over the semi-hard window.  Max and min are
// order-independent, so the result does not depend on the tiling.  With pred0, side-0 CTAs also count the
// Evaluate_PR row terms of their anchors (from the assignment alone).  Shared memory (MX_SMEM) allows two CTAs per SM;
// the launch bound caps registers at 128 to match (without it ptxas picks 80 and spills).
__global__ void __launch_bounds__(256, 2) triplet_mine_kernel(TripletArgs p) {
  extern __shared__ __align__(16) float mx_smem[];
  float* As = mx_smem;                      // [k][MX_R]
  float* Bs = mx_smem + MT_D * MX_R;        // [k][MX_BLD]
  __shared__ float xb[2][MX_R];
  __shared__ float s_pos[MX_R];
  __shared__ int s_red[3][8];
  pdl_launch_dependents();
  const int pair = blockIdx.x, sa = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  pdl_wait();
  int b0, e0, b1, e1;
  image_range(p.cu[0], p.n[0], pair, b0, e0);
  image_range(p.cu[1], p.n[1], pair, b1, e1);
  const int n0 = e0 - b0, n1 = e1 - b1;
  const int ba = sa ? b1 : b0, na = sa ? n1 : n0;
  const int bb = sa ? b0 : b1, nb = sa ? n0 : n1;
  const float* __restrict__ A = sa ? p.d[1] : p.d[0];
  const float* __restrict__ B = sa ? p.d[0] : p.d[1];
  const float* __restrict__ G = p.assign + (long long)pair * p.assign_stride;
  const long long ld = p.assign_ld ? p.assign_ld : n1;
  // entry (anchor r, candidate j) of the assignment: [r][j] for side-0 anchors, [j][r] for side-1 anchors
  const long long sr = sa ? 1 : ld, sc = sa ? ld : 1;
  const long long out0 = triplet_anchor0(p.cu[0], p.cu[1], p.n[0], p.n[1], pair) + (sa ? n0 : 0);
  const int rb = tid >> 6, c = tid & 63;    // row block (anchors rb * 8 .. + 7 of a group), column in the chunk
  int n_tp = 0, n_pos = 0, n_tn = 0;        // side 0 with pred0: TP, positive and TN rows of this thread

  for (int g0 = blockIdx.z * MX_R; g0 < na; g0 += gridDim.z * MX_R) {
    const int nr = min(MX_R, na - g0);
    __syncthreads();   // the previous group's readers are done with As / s_pos
    if (lane < nr) mx_stage_row(As, A, p.layout, ba, na, g0 + lane, lane, warp);
    float pv[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) pv[i] = -INFINITY;
    // ---- phase 1: positives
    for (int j0 = 0; j0 < nb; j0 += MX_C) {
      const int j = j0 + c;
      unsigned mm = 0;   // bit i: (anchor rb*8+i, column j) is a match
      if (j < nb) {
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (rb * 8 + i < nr) mm |= ((double)G[(g0 + rb * 8 + i) * sr + j * sc] > p.match_thr) << i;
      }
      if (!__syncthreads_or(mm)) continue;   // also: As staged / the previous chunk consumed
      mx_stage_chunk(Bs, B, p.layout, bb, nb, j0, tid, rb, c);
      __syncthreads();
      if (mm) {
        float acc[8];
        mx_dot8(As, Bs, rb, c, acc);
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (mm >> i & 1) pv[i] = fmaxf(pv[i], exact_dist_raw(acc[i], 0.f, 0.f, 0));
      }
    }
    // max over the 64 column threads of every anchor: 32 lanes by shuffles, then the two warps of a row block
#pragma unroll
    for (int i = 0; i < 8; ++i) pv[i] = warp_max(pv[i]);
    if ((warp & 1) && lane == 0) {
#pragma unroll
      for (int i = 0; i < 8; ++i) xb[0][rb * 8 + i] = pv[i];
    }
    __syncthreads();
    if (!(warp & 1) && lane == 0) {
#pragma unroll
      for (int i = 0; i < 8; ++i) s_pos[rb * 8 + i] = fmaxf(pv[i], xb[0][rb * 8 + i]);
    }
    __syncthreads();
    // ---- phase 2: negatives in the semi-hard window (pos, pos + 0.5f); an anchor without a positive has none
    float lo[8], hi[8], nv[8];
    bool want = false;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      lo[i] = s_pos[rb * 8 + i];
      hi[i] = lo[i] + TRIPLET_MARGIN;
      nv[i] = INFINITY;
      want |= rb * 8 + i < nr && lo[i] > 0.f;
    }
    for (int j0 = 0; j0 < nb; j0 += MX_C) {
      const int j = j0 + c;
      unsigned um = 0;   // bit i: (anchor rb*8+i, column j) is an unmatch, u = d; other entries u = 10000
      if (j < nb && want) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          if (rb * 8 + i < nr && lo[i] > 0.f) {
            if ((double)G[(g0 + rb * 8 + i) * sr + j * sc] <= p.unmatch_thr) um |= 1u << i;
            else if (lo[i] < TRIPLET_FAR && TRIPLET_FAR < hi[i]) nv[i] = fminf(nv[i], TRIPLET_FAR);
          }
        }
      }
      if (!__syncthreads_or(um)) continue;
      mx_stage_chunk(Bs, B, p.layout, bb, nb, j0, tid, rb, c);
      __syncthreads();
      if (um) {
        float acc[8];
        mx_dot8(As, Bs, rb, c, acc);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float u = exact_dist_raw(acc[i], 0.f, 0.f, 0);
          if ((um >> i & 1) && lo[i] < u && u < hi[i]) nv[i] = fminf(nv[i], u);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) nv[i] = -warp_max(-nv[i]);
    if ((warp & 1) && lane == 0) {
#pragma unroll
      for (int i = 0; i < 8; ++i) xb[1][rb * 8 + i] = nv[i];
    }
    __syncthreads();
    if (!(warp & 1) && lane < 8 && rb * 8 + lane < nr) {
      float pos = lo[0], neg = nv[0];
#pragma unroll
      for (int i = 1; i < 8; ++i)
        if (lane == i) { pos = lo[i]; neg = nv[i]; }
      neg = fminf(neg, xb[1][rb * 8 + lane]);
      const int st = !(pos > 0.f) ? 0 : neg < INFINITY ? 2 : 1;
      const long long a = out0 + g0 + rb * 8 + lane;
      p.pos[a] = st ? pos : __int_as_float(0x7fffffff);
      p.neg[a] = st == 2 ? neg : __int_as_float(0x7fffffff);
      p.state[a] = st;
    }
    // ---- Evaluate_PR row terms of side-0 anchors: warp w takes rows w, w + 8, ... of the group, lanes over columns
    if (sa == 0 && p.pred0) {
      for (int r = warp; r < nr; r += 8) {
        const int i = g0 + r;
        int pred = p.pred0[b0 + i];
        if (pred < 0 || pred >= n1) pred = -1;
        bool any_gt = false, tp = false;
        int neither = 0;
        for (int j = lane; j < n1; j += 32) {
          const bool g = (double)G[i * ld + j] > p.match_thr;
          any_gt |= g;
          if (j == pred) tp = g;
          else neither += !g;
        }
        any_gt = __any_sync(0xffffffffu, any_gt);
        tp = __any_sync(0xffffffffu, tp);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) neither += __shfl_xor_sync(0xffffffffu, neither, o);
        if (lane == 0) tfpn_row(any_gt, tp, neither, n0, n_tp, n_pos, n_tn);
      }
    }
  }
  if (sa == 0 && p.pred0) {
    if (lane == 0) {
      s_red[0][warp] = n_tp;
      s_red[1][warp] = n_pos;
      s_red[2][warp] = n_tn;
    }
    __syncthreads();
    if (tid == 0) {
      int tp = 0, pos = 0, tn = 0, rows = 0;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        tp += s_red[0][q];
        pos += s_red[1][q];
        tn += s_red[2][q];
      }
      for (int g0 = blockIdx.z * MX_R; g0 < na; g0 += gridDim.z * MX_R) rows += min(MX_R, na - g0);
      tfpn_add(p.tfpn + 4 * pair, rows, pos, tp, tn);
    }
  }
}

struct TripletReduceArgs {
  const int* cu[2]; int n[2];
  const int* group_off;            // [n_groups + 1] pair offsets or nullptr (one group of n_pairs)
  int n_pairs;
  const float* pos; const float* neg; const int* state;
  float* loss; float* hardest_pos; float* hardest_neg; int* n_valid;   // [n_groups]
};

// grid = n_groups, 256 threads.  The anchors of a group are a contiguous range; thread t sums the anchors t, t + 256, ...
// of it (counted from the group's first anchor) in fp64, then a fixed tree merges the threads: the same group gives the
// same bits in any call.  loss = float(sum relu((pos - neg) + 1) / n_valid), computed per anchor in fp32 as the
// reference does; hardest_pos = max pos, hardest_neg = min neg; all three NaN when no anchor is valid.
__global__ void __launch_bounds__(256) triplet_reduce_kernel(TripletReduceArgs p) {
  __shared__ double s_sum[256];
  __shared__ float s_hp[256], s_hn[256];
  __shared__ int s_nv[256];
  pdl_launch_dependents();
  pdl_wait();
  const int g = blockIdx.x, t = threadIdx.x;
  const int p0 = p.group_off ? p.group_off[g] : 0, p1 = p.group_off ? p.group_off[g + 1] : p.n_pairs;
  const long long a0 = triplet_anchor0(p.cu[0], p.cu[1], p.n[0], p.n[1], p0);
  const long long a1 = triplet_anchor0(p.cu[0], p.cu[1], p.n[0], p.n[1], p1);
  double sum = 0.0;
  float hp = -INFINITY, hn = INFINITY;
  int nv = 0;
  for (long long a = a0 + t; a < a1; a += 256) {
    if (p.state[a] != 2) continue;
    const float ps = p.pos[a], ng = p.neg[a];
    sum += (double)fmaxf(__fadd_rn(__fsub_rn(ps, ng), TRIPLET_LOSS_MARGIN), 0.f);
    hp = fmaxf(hp, ps);
    hn = fminf(hn, ng);
    ++nv;
  }
  s_sum[t] = sum; s_hp[t] = hp; s_hn[t] = hn; s_nv[t] = nv;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (t < o) {
      s_sum[t] += s_sum[t + o];
      s_hp[t] = fmaxf(s_hp[t], s_hp[t + o]);
      s_hn[t] = fminf(s_hn[t], s_hn[t + o]);
      s_nv[t] += s_nv[t + o];
    }
    __syncthreads();
  }
  if (t == 0) {
    const int n = s_nv[0];
    const float nan = __int_as_float(0x7fffffff);
    p.loss[g] = n ? (float)(s_sum[0] / (double)n) : nan;
    p.hardest_pos[g] = n ? s_hp[0] : nan;
    p.hardest_neg[g] = n ? s_hn[0] : nan;
    p.n_valid[g] = n;
  }
}

}  // namespace ltr
