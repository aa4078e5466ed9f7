// Image retrieval (DESIGN.md "Image retrieval"): spherical k-means vocabularies over an image set's point and line
// descriptors, intra-normalised VLAD global descriptors, and the exact top-k database images of every query.
//
// - rt_bucket_kernel groups rows by cluster, stably (ascending row order inside every (segment, cluster)): per image
//   for VLAD, over the whole set for the centroid update.  rt_cluster_sum, the one fp64 sum of a cluster's rows (or of
//   their residuals to the centroid) in that order, serves both the centroid update and VLAD.
// - rt_kmeans_kernel: every centroid becomes the normalised sum of its rows (an empty cluster keeps its centroid).
//   The assignment step is the descriptor matcher (ltr_match_indexed against the vocabulary as a one-image pool).
// - rt_vlad_kernel: the intra-normalised VLAD of one image per CTA, written as fp32 rows and as the split-bf16 tile
//   image (act_img.cuh, kblocks = D / 64) the screening contracts.
// - rt_screen_kernel: wgmma over 128 x 128 query x database tiles (3-term split-bf16 product, operands streamed
//   through a TMA / mbarrier ring); per query row the tile's top-k candidates and the best score the tile dropped.
// - rt_merge_kernel: one CTA per query; the k-th screened score s_k, the exact fp64 rescoring of every candidate with
//   a screened score >= s_k - 2 rt_eps(D), and a full exact pass over the database when a tile dropped a score there.
// Every fp64 operation is an explicitly rounded intrinsic (rn_fp64.cuh), so linetr_b200/retrieval.py gives every bit.
#pragma once
#include "act_img.cuh"
#include "common.cuh"
#include "ptx_sm90.cuh"
#include "rn_fp64.cuh"

namespace ltr {

constexpr int RT_DL = 256;                // dimension of a local (point or line) descriptor
constexpr int RT_MAX_CLUSTERS = 256;      // = LTR_RT_MAX_CLUSTERS
constexpr int RT_MAX_K = 64;              // = LTR_RT_MAX_K
// = LTR_RT_EPS(D): bound on |screened - exact| score of descriptors of norm <= 1 (DESIGN.md): the split terms plus
// the fp32 accumulation over 3 D / 16 wgmma steps, which grows with D.
__host__ __device__ constexpr double rt_eps(int D) { return 1e-4 + 3e-8 * D; }

// ---------------------------------------------------------------- rows of one part
// x: rows [R, 256] (layout 0) or per image channel-first [256, n_i] blocks back to back (layout 1, image i at
// 256 * cu[i]); cu [n_images + 1] row offsets.
struct RtRows {
  const float* x;
  const int* cu;
  int layout;
  int n_images;
};

// Element 0 of row g (of image img, or found from cu when img < 0) and the stride between its elements.
__device__ __forceinline__ const float* rt_row(const RtRows& r, int img, int g, size_t& stride) {
  if (r.layout == 0) {
    stride = 1;
    return r.x + (size_t)g * RT_DL;
  }
  if (img < 0) img = rc_segment(r.cu, r.n_images, g);
  const int b = r.cu[img];
  stride = (size_t)(r.cu[img + 1] - b);
  return r.x + (size_t)b * RT_DL + (g - b);
}

// Component k of sum over the slots [sb, se) of perm, in slot order, of x_g (cent == nullptr) or x_g - cent, fp64.
__device__ __forceinline__ double rt_cluster_sum(const RtRows& r, const int* __restrict__ perm, int sb, int se, int img,
                                                 const float* cent, int k) {
  const double ck = cent ? (double)cent[k] : 0.0;
  double acc = 0.0;
  for (int s = sb; s < se; ++s) {
    size_t st;
    const float* x = rt_row(r, img, perm[s], st);
    const double v = (double)x[k * st];
    acc = RC_A(acc, cent ? RC_S(v, ck) : v);
  }
  return acc;
}

// Sum of one fp64 value per thread of a 256-thread CTA: xor butterfly in every warp, then the warps' lane 0 in warp
// order (_posed.block_sum(terms [256, 1], 256)).  Every thread gets the result; red is 8 doubles of shared memory.
__device__ __forceinline__ double rt_block_sum256(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = RC_A(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int w = 0; w < 8; ++w) s = RC_A(s, red[w]);
  return s;
}

// ---------------------------------------------------------------- stable bucketing by cluster
struct RtBucketArgs {
  const int* assign;     // [n_rows] cluster of every row; rows outside [0, K) belong to no cluster
  const int* seg;        // [n_seg + 1] row offsets of the segments (images), or nullptr: one segment of n_rows
  int n_seg, n_rows, K;
  int* cstart;           // out [n_seg * K + 1]: first slot of every (segment, cluster), then the end
  int* perm;             // out: the rows by (segment, cluster), ascending inside each
  const float* scores;   // optional [n_rows]: the matcher's distances, summed into cost (one segment only)
  double* cost;
};

constexpr int RT_BUCKET_THREADS = 1024;

// grid = n_seg, 1024 threads.  Chunks of 1024 rows in order: a row's slot is the cluster's running base, plus the
// counts of the earlier warps of the chunk, plus its rank among the equal lanes of its warp (__match_any_sync).
__global__ void __launch_bounds__(RT_BUCKET_THREADS) rt_bucket_kernel(RtBucketArgs a) {
  __shared__ int wcnt[32 * RT_MAX_CLUSTERS];
  __shared__ int base[RT_MAX_CLUSTERS];
  __shared__ double red[32];
  pdl_launch_dependents();
  pdl_wait();
  const int s = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, K = a.K;
  const int b = a.seg ? a.seg[s] : 0, e = a.seg ? a.seg[s + 1] : a.n_rows;
  for (int c = tid; c < K; c += RT_BUCKET_THREADS) base[c] = 0;
  __syncthreads();
  for (int r = b + tid; r < e; r += RT_BUCKET_THREADS) {
    const int c = a.assign[r];
    if (c >= 0 && c < K) atomicAdd(&base[c], 1);
  }
  __syncthreads();
  if (tid == 0) {
    int run = b;
    for (int c = 0; c < K; ++c) {
      const int t = base[c];
      base[c] = run;
      a.cstart[s * K + c] = run;
      run += t;
    }
    if (s == a.n_seg - 1) a.cstart[a.n_seg * K] = run;
  }
  for (int r0 = b; r0 < e; r0 += RT_BUCKET_THREADS) {
    for (int i = tid; i < 32 * K; i += RT_BUCKET_THREADS) wcnt[(i / K) * RT_MAX_CLUSTERS + i % K] = 0;
    __syncthreads();
    const int r = r0 + tid;
    int c = r < e ? a.assign[r] : -1;
    if (c >= K) c = -1;
    const unsigned peers = __match_any_sync(0xffffffffu, c);
    const int rank = __popc(peers & ((1u << lane) - 1u));
    if (c >= 0 && rank == 0) wcnt[warp * RT_MAX_CLUSTERS + c] = __popc(peers);
    __syncthreads();
    for (int cc = tid; cc < K; cc += RT_BUCKET_THREADS) {
      int run = base[cc];
      for (int w = 0; w < 32; ++w) {
        const int t = wcnt[w * RT_MAX_CLUSTERS + cc];
        wcnt[w * RT_MAX_CLUSTERS + cc] = run;
        run += t;
      }
      base[cc] = run;
    }
    __syncthreads();
    if (c >= 0) a.perm[wcnt[warp * RT_MAX_CLUSTERS + c] + rank] = r;
    __syncthreads();
  }
  if (a.cost) {   // k-means cost: per thread its rows in order, then the warps in order (a statistic, not a model output)
    double v = 0.0;
    for (int r = b + tid; r < e; r += RT_BUCKET_THREADS) v = RC_A(v, (double)a.scores[r]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = RC_A(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (lane == 0) red[warp] = v;
    __syncthreads();
    if (tid == 0) {
      double t = 0.0;
      for (int w = 0; w < 32; ++w) t = RC_A(t, red[w]);
      *a.cost = t;
    }
  }
}

// ---------------------------------------------------------------- centroid update
struct RtKmeansArgs {
  RtRows rows;
  int K;
  const int* cstart; const int* perm;   // rt_bucket_kernel over the whole set
  const int* init_rows;                 // [K] or nullptr: centroid c = row init_rows[c] (the initial vocabulary)
  const float* cent_in;                 // [K, 256] the current centroids (an empty cluster keeps its own)
  float* cent;                          // out [K, 256] (may be cent_in)
  float* cent_cf;                       // out [256, K]: the same, channel-first (the matcher's point layout)
  ActImg img;                           // out: tile image of the centroids (kblocks = 4)
  int* counts;                          // out [K]: rows per cluster
};

// grid = K, 256 threads (thread = component).
__global__ void __launch_bounds__(256) rt_kmeans_kernel(RtKmeansArgs a) {
  __shared__ double red[8];
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.x, k = threadIdx.x;
  float v;
  if (a.init_rows) {
    size_t st;
    const float* x = rt_row(a.rows, -1, a.init_rows[c], st);
    v = x[k * st];
    if (k == 0) a.counts[c] = 0;
  } else {
    const int sb = a.cstart[c], se = a.cstart[c + 1];
    v = a.cent_in[c * RT_DL + k];
    if (se > sb) {
      const double s = rt_cluster_sum(a.rows, a.perm, sb, se, -1, nullptr, k);
      const double n2 = rt_block_sum256(RC_M(s, s), red);
      if (n2 > 0.0) v = __double2float_rn(RC_D(s, __dsqrt_rn(n2)));   // a sum of norm 0 keeps the centroid too
    }
    if (k == 0) a.counts[c] = se - sb;
  }
  a.cent[c * RT_DL + k] = v;
  a.cent_cf[(size_t)k * a.K + c] = v;
  img_store1(a.img, c, k, v);
}

// ---------------------------------------------------------------- VLAD
struct RtPart {
  RtRows rows;
  int K;
  const float* cent;          // [K, 256]
  const int* cstart;          // rt_bucket_kernel per image: [n_images * K + 1]
  const int* perm;
  double sw;                  // sqrt(w_part)
  int col0;                   // first column of the part in the descriptor
};

struct RtVladArgs {
  RtPart part[2];
  int n_images, D;
  float* desc;                // out [n_images, D]
  ActImg img;                 // out: tile image, kblocks = D / 64, rows up to the next multiple of 128 zero
};

// v_c / |v_c| of cluster c of image i (0 for an empty cluster or a residual sum of norm 0), component k.
__device__ __forceinline__ double rt_vlad_unit(const RtPart& p, int i, int c, int k, double* red) {
  const int sb = p.cstart[i * p.K + c], se = p.cstart[i * p.K + c + 1];
  if (se == sb) return 0.0;   // uniform per CTA
  const double v = rt_cluster_sum(p.rows, p.perm, sb, se, i, p.cent + c * RT_DL, k);
  const double n2 = rt_block_sum256(RC_M(v, v), red);
  return n2 > 0.0 ? RC_D(v, __dsqrt_rn(n2)) : 0.0;
}

// grid = n_images rounded up to 128, 256 threads (thread = component of a cluster).  Each part twice over its
// clusters: once for the part's norm (per thread the squares in ascending cluster order, then rt_block_sum256), once
// to write (v_c / |v_c|) / |part| * sqrt(w).
__global__ void __launch_bounds__(256) rt_vlad_kernel(RtVladArgs a) {
  __shared__ double red[8];
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x, k = threadIdx.x;
  if (i >= a.n_images) {   // padding row of the last tile
    for (int col = k; col < a.D; col += 256) img_store1(a.img, i, col, 0.f);
    return;
  }
  for (int pi = 0; pi < 2; ++pi) {
    const RtPart& p = a.part[pi];
    double sq = 0.0;
    for (int c = 0; c < p.K; ++c) {
      const double u = rt_vlad_unit(p, i, c, k, red);
      sq = RC_A(sq, RC_M(u, u));
    }
    const double pn = __dsqrt_rn(rt_block_sum256(sq, red));
    for (int c = 0; c < p.K; ++c) {
      const double u = rt_vlad_unit(p, i, c, k, red);
      const float o = pn > 0.0 ? __double2float_rn(RC_M(RC_D(u, pn), p.sw)) : 0.f;
      const int col = p.col0 + c * RT_DL + k;
      a.desc[(size_t)i * a.D + col] = o;
      img_store1(a.img, i, col, o);
    }
  }
}

// ---------------------------------------------------------------- tile image of fp32 rows [n, D]
// grid = n rounded up to 128, 256 threads; padding rows are written 0.
__global__ void __launch_bounds__(256) rt_tiles_kernel(const float* __restrict__ x, int n, int D, ActImg img) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x;
  for (int col = threadIdx.x; col < D; col += 256) img_store1(img, i, col, i < n ? x[(size_t)i * D + col] : 0.f);
}

// ---------------------------------------------------------------- screening: wgmma over query x database tiles
constexpr int RT_TILE = 16384;                    // one plane of a 128 x 64 bf16 tile
constexpr int RT_STAGE = 4 * RT_TILE;             // one k-block of A and B, hi + lo
constexpr int RT_STAGES = 3;
constexpr int RT_OFF_BAR = RT_STAGES * RT_STAGE;
constexpr int RT_SLD = 129;                       // padded row of the epilogue's score tile (over the ring)
constexpr int RT_SMEM = RT_OFF_BAR + 64 + 1024;   // + barriers + alignment slack
constexpr int RT_THREADS = 288;                   // 2 consumer warpgroups (64 query rows each) + 1 TMA warp
static_assert(128 * RT_SLD * 4 <= RT_OFF_BAR, "rt_screen: the score tile fits over the ring");
static_assert(RT_SMEM <= 232448, "rt_screen: shared memory budget");

struct RtScreenArgs {
  ActImg q, db;               // tile images (kblocks = D / 64)
  int Q, N, kb, k, exclude_self, n_tiles;
  float* cand_score;          // [Q, n_tiles, k]: per query and database tile the top-k screened scores, -inf past them
  int* cand_idx;              // ... and their database indices, -1 past them
  float* drop;                // [Q, n_tiles]: the best screened score the tile did not keep, -inf if none
  int* n_full;                // zeroed here for rt_merge_kernel
};

__device__ __forceinline__ void rt_epi_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// grid = (database tiles, query tiles).
__global__ void __launch_bounds__(RT_THREADS, 1) rt_screen_kernel(RtScreenArgs p) {
  extern __shared__ __align__(1024) uint8_t rt_smem_raw[];
  const uint32_t raw = ptx::smem_u32(rt_smem_raw);
  uint8_t* smem = rt_smem_raw + ((1024u - (raw & 1023u)) & 1023u);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + RT_OFF_BAR);
  uint64_t* empty = full + RT_STAGES;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tn = blockIdx.x, tq = blockIdx.y;
  pdl_launch_dependents();
  if (tid == 0) {
    for (int s = 0; s < RT_STAGES; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], 8);
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  if (tid == 0 && tn == 0 && tq == 0 && p.n_full) *p.n_full = 0;
  if (warp == 8) {
    if (lane == 0) {
      for (int kb = 0; kb < p.kb; ++kb) {
        const int s = kb % RT_STAGES;
        ptx::mbar_wait(&empty[s], ((kb / RT_STAGES) & 1) ^ 1);
        uint8_t* st = smem + s * RT_STAGE;
        const size_t ta = ((size_t)tq * p.kb + kb) * IMG_TILE_ELEMS, tb = ((size_t)tn * p.kb + kb) * IMG_TILE_ELEMS;
        ptx::mbar_arrive_expect_tx(&full[s], RT_STAGE);
        ptx::bulk_g2s(st, p.q.hi + ta, RT_TILE, &full[s]);
        ptx::bulk_g2s(st + RT_TILE, p.q.lo + ta, RT_TILE, &full[s]);
        ptx::bulk_g2s(st + 2 * RT_TILE, p.db.hi + tb, RT_TILE, &full[s]);
        ptx::bulk_g2s(st + 3 * RT_TILE, p.db.lo + tb, RT_TILE, &full[s]);
      }
    }
    return;
  }
  const int wg = warp >> 2;
  float d[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) d[i] = 0.f;
  for (int kb = 0; kb < p.kb; ++kb) {
    const int s = kb % RT_STAGES;
    ptx::mbar_wait(&full[s], (kb / RT_STAGES) & 1);
    const uint32_t a_hi = ptx::smem_u32(smem + s * RT_STAGE) + wg * 8192, a_lo = a_hi + RT_TILE;
    const uint32_t b_hi = ptx::smem_u32(smem + s * RT_STAGE + 2 * RT_TILE), b_lo = b_hi + RT_TILE;
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
    if (kb > 0 && lane == 0) ptx::mbar_arrive(&empty[(kb - 1) % RT_STAGES]);
  }
  ptx::wg_wait<0>();
  ptx::wg_fence_regs(d);
  rt_epi_bar();   // both warpgroups' MMAs are complete: the ring becomes the score tile
  float* S = reinterpret_cast<float*>(smem);
  {
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      S[r0 * RT_SLD + 8 * j + c0] = d[4 * j];
      S[r0 * RT_SLD + 8 * j + c0 + 1] = d[4 * j + 1];
      S[(r0 + 8) * RT_SLD + 8 * j + c0] = d[4 * j + 2];
      S[(r0 + 8) * RT_SLD + 8 * j + c0 + 1] = d[4 * j + 3];
    }
  }
  rt_epi_bar();
  // per row: k + 1 rounds of a warp argmax (ties to the lower column) over the valid columns
  for (int r = warp; r < 128; r += 8) {
    const int qi = tq * 128 + r;
    if (qi >= p.Q) break;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int col = tn * 128 + 32 * j + lane;
      const bool ok = col < p.N && !(p.exclude_self && col == qi);
      v[j] = ok ? S[r * RT_SLD + 32 * j + lane] : -INFINITY;
    }
    const size_t o = ((size_t)qi * p.n_tiles + tn) * p.k;
    for (int t = 0; t <= p.k; ++t) {
      float bv = -INFINITY;
      int bc = INT_MAX;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (v[j] > bv) { bv = v[j]; bc = 32 * j + lane; }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, off);
        const int oc = __shfl_xor_sync(0xffffffffu, bc, off);
        if (ov > bv || (ov == bv && oc < bc)) { bv = ov; bc = oc; }
      }
      if (t == p.k) {
        if (lane == 0) p.drop[(size_t)qi * p.n_tiles + tn] = bv;
      } else if (lane == 0) {
        p.cand_score[o + t] = bv;
        p.cand_idx[o + t] = bc == INT_MAX ? -1 : tn * 128 + bc;
      }
      if (bc != INT_MAX && (bc & 31) == lane) v[bc >> 5] = -INFINITY;
    }
  }
}

// ---------------------------------------------------------------- merge, exact rescoring, full pass
constexpr int RT_MERGE_THREADS = 256;

struct RtMergeArgs {
  const float* q; const float* db;   // fp32 rows [Q, D], [N, D]
  int Q, N, D, k, exclude_self, n_tiles;
  const float* cand_score; const int* cand_idx; const float* drop;
  int* idx;                          // out [Q, k], -1 past the candidates
  double* score;                     // out [Q, k], NaN past the candidates
  int* n_full;                       // out: queries that took the full exact pass
};

// The exact score of two fp32 rows: lane l sums the products of components l, l + 32, ... in ascending order (each
// product is exact in fp64), then the xor butterfly (_posed.block_sum(products, 32)).
__device__ __forceinline__ double rt_exact_dot(const float* __restrict__ a, const float* __restrict__ b, int D, int lane) {
  double acc = 0.0;
  for (int k = lane; k < D; k += 32) acc = RC_A(acc, RC_M((double)a[k], (double)b[k]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc = RC_A(acc, __shfl_xor_sync(0xffffffffu, acc, o));
  return acc;
}

__device__ __forceinline__ uint32_t rt_key(float f) {   // order-preserving: larger float, larger key
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// grid = Q, 256 threads.
__global__ void __launch_bounds__(RT_MERGE_THREADS) rt_merge_kernel(RtMergeArgs p) {
  __shared__ int hist[256];
  __shared__ int wcnt[8];
  __shared__ int list[RT_MERGE_THREADS];
  __shared__ double lsc[RT_MERGE_THREADS];
  __shared__ int top_i[2][RT_MAX_K];
  __shared__ double top_s[2][RT_MAX_K];
  __shared__ uint32_t sel[2];   // prefix of the k-th largest key, the count still wanted
  pdl_launch_dependents();
  pdl_wait();
  const int qi = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, K = p.k;
  const int nc = p.n_tiles * K;
  const float* cs = p.cand_score + (size_t)qi * nc;
  const int* ci = p.cand_idx + (size_t)qi * nc;
  // ---- the k-th largest screened score: 8-bit radix select over the valid candidates
  int nv = 0;
  for (int j = tid; j < nc; j += RT_MERGE_THREADS) nv += ci[j] >= 0;
  for (int o = 16; o > 0; o >>= 1) nv += __shfl_xor_sync(0xffffffffu, nv, o);
  if (lane == 0) wcnt[warp] = nv;
  __syncthreads();
  nv = 0;
  for (int w = 0; w < 8; ++w) nv += wcnt[w];
  __syncthreads();   // wcnt is rewritten by the compaction below
  double thr = -INFINITY;
  bool flag = false;
  if (nv >= K) {
    if (tid == 0) { sel[0] = 0; sel[1] = (uint32_t)K; }
    uint32_t mask = 0;
    for (int sh = 24; sh >= 0; sh -= 8) {
      hist[tid] = 0;
      __syncthreads();
      const uint32_t pre = sel[0];
      for (int j = tid; j < nc; j += RT_MERGE_THREADS) {
        if (ci[j] < 0) continue;
        const uint32_t key = rt_key(cs[j]);
        if ((key & mask) == pre) atomicAdd(&hist[(key >> sh) & 255u], 1);
      }
      __syncthreads();
      if (tid == 0) {
        uint32_t want = sel[1], cum = 0;
        for (int dg = 255; dg >= 0; --dg) {
          if (cum + (uint32_t)hist[dg] >= want) { sel[0] = pre | ((uint32_t)dg << sh); sel[1] = want - cum; break; }
          cum += (uint32_t)hist[dg];
        }
      }
      mask |= 255u << sh;
      __syncthreads();
    }
    const uint32_t key = sel[0];
    const float sk = __uint_as_float((key & 0x80000000u) ? (key & 0x7fffffffu) : ~key);
    thr = RC_S((double)sk, 2.0 * rt_eps(p.D));
    bool f = false;
    for (int t = tid; t < p.n_tiles; t += RT_MERGE_THREADS) f |= (double)p.drop[(size_t)qi * p.n_tiles + t] >= thr;
    flag = __syncthreads_or(f);
  }
  // ---- exact scores of the kept candidates (or of the whole database), merged into the running top-k by rank
  int cur = 0, m_top = 0;
  const float* qrow = p.q + (size_t)qi * p.D;
  const int n_src = flag ? p.N : nc;
  for (int j0 = 0; j0 < n_src; j0 += RT_MERGE_THREADS) {
    const int j = j0 + tid;
    int id = -1;
    if (j < n_src) {
      if (flag) id = (p.exclude_self && j == qi) ? -1 : j;
      else id = (ci[j] >= 0 && (double)cs[j] >= thr) ? ci[j] : -1;
    }
    const unsigned b = __ballot_sync(0xffffffffu, id >= 0);
    if (lane == 0) wcnt[warp] = __popc(b);
    __syncthreads();
    int pre = 0, m = 0;
    for (int w = 0; w < 8; ++w) { pre += w < warp ? wcnt[w] : 0; m += wcnt[w]; }
    if (id >= 0) list[pre + __popc(b & ((1u << lane) - 1u))] = id;
    __syncthreads();
    for (int e = warp; e < m; e += 8) {
      const double v = rt_exact_dot(qrow, p.db + (size_t)list[e] * p.D, p.D, lane);
      if (lane == 0) lsc[e] = v;
    }
    __syncthreads();
    const int tot = m_top + m;
    for (int e = tid; e < tot; e += RT_MERGE_THREADS) {
      const double s = e < m_top ? top_s[cur][e] : lsc[e - m_top];
      const int ix = e < m_top ? top_i[cur][e] : list[e - m_top];
      int rank = 0;
      for (int f = 0; f < tot; ++f) {
        const double sf = f < m_top ? top_s[cur][f] : lsc[f - m_top];
        const int xf = f < m_top ? top_i[cur][f] : list[f - m_top];
        rank += (sf > s) || (sf == s && xf < ix);
      }
      if (rank < K) { top_s[cur ^ 1][rank] = s; top_i[cur ^ 1][rank] = ix; }
    }
    m_top = min(K, tot);
    cur ^= 1;
    __syncthreads();
  }
  for (int t = tid; t < K; t += RT_MERGE_THREADS) {
    p.idx[(size_t)qi * K + t] = t < m_top ? top_i[cur][t] : -1;
    p.score[(size_t)qi * K + t] = t < m_top ? top_s[cur][t] : __longlong_as_double(0x7ff8000000000000LL);
  }
  if (tid == 0 && flag) atomicAdd(p.n_full, 1);
}

}  // namespace ltr
