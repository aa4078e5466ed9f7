/*
 * linetr_b200 - C ABI of the H100-native LineTR line-descriptor + NN-matcher hot path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch types, no exceptions.
 * Every entry point replaces a piece of the reference's Python call surface (paths are
 * relative to the reference checkout, yosungho/LineTR):
 *
 *   ltr_create / ltr_destroy   <- LineTransformer.__init__ + load_state_dict
 *                                 (models/line_transformer.py:203-223): takes the raw
 *                                 checkpoint tensors by their state-dict names, folds the
 *                                 eval-mode BatchNorms, repacks heads, uploads to the GPU.
 *   ltr_encode                 <- LineTransformer.forward (models/line_transformer.py:225-249)
 *                                 = normalize_keylines (:22-38) + KeylineEncoder.forward
 *                                 (:107-130, models/line_attention.py:42-94) +
 *                                 SelfAttentionalLayer.forward (:176-183) + final_proj +
 *                                 F.normalize (:245-246).
 *   ltr_match                  <- get_dist_matrix (models/line_process.py:198-201) +
 *                                 LineTransformer.subline2keyline (models/line_transformer.py:277-282)
 *                                 + nn_matcher_distmat (models/nn_matcher.py:3-31); with
 *                                 descriptors as input it is nn_matcher (models/nn_matcher.py:33-43).
 *   ltr_match_distmat          <- nn_matcher_distmat on a caller-supplied distance matrix.
 *   ltr_image_tiles +          <- Matching.forward with a side already in `data` (models/matching.py:20-60):
 *   ltr_match_indexed             images encoded once, matched in any number of pairs.
 *   ltr_line_gt                <- mat_assign_sublines of the homography dataset builder
 *                                 (dataloaders/build_homography_dataset.py:210-234) + Evaluate_PR.calc_TFPN
 *                                 (evaluations/evaluate_pr.py:10-22) for a batch of pairs.
 *   ltr_triplet_loss           <- descriptor_loss.forward (evaluations/criteria.py:35-192) of the validation step
 *                                 (train.py:198-240) + Evaluate_PR.calc_TFPN, for groups of pairs.
 *   ltr_homography             <- cv2.findHomography(RANSAC) per pair, as the reference's geometry helpers
 *                                 (models/utils.py:291-412) verify matches, with line matches as well as points.
 *   ltr_essential              <- estimate_pose (models/utils.py:291-315): cv2.findEssentialMat(RANSAC) +
 *                                 cv2.recoverPose per pair, batched.
 *   ltr_fundamental            <- cv2.findFundamentalMat(FM_RANSAC) per pair, batched, for pairs without intrinsics,
 *                                 with an epipolar check of the line matches.
 *   ltr_absolute_pose          <- cv2.solvePnPRansac per query, batched, with the line matches scored and refined too
 *                                 (PL-Loc's localization step).
 *   ltr_triangulate            <- cv2.triangulatePoints per pair, batched over every image of a posed set, multi-view
 *                                 with outlier rejection, and for the key lines' end points too.
 *   ltr_warp_pairs             <- cv2.warpPerspective of the grey and colour images + the eroded valid mask of the
 *                                 homography dataset builder (dataloaders/build_homography_dataset.py:164-184).
 *   ltr_photometric            <- imgPhotometric of the homography dataset builder (ImgAugTransform +
 *                                 customizedTransform.additive_shade, dataloaders/utils/photometric.py).
 *
 * Conventions: return 0 on success, a negative LTR_E_* code on failure (message via
 * ltr_last_error(), thread-local).  All device pointers are caller-owned and must live on
 * the device the model was created on.  Calls are asynchronous with respect to the host
 * and ordered on the given CUDA stream (pass the cudaStream_t as void*; NULL = default
 * stream).  There is no CPU fallback: every function fails if no CUDA device is usable.
 */
#ifndef LINETR_B200_H_
#define LINETR_B200_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LTR_ABI_VERSION 4

#define LTR_OK 0
#define LTR_E_INVALID (-1)   /* bad argument / missing checkpoint tensor / shape mismatch */
#define LTR_E_CUDA (-2)      /* CUDA runtime error (no device, launch failure, OOM) */
#define LTR_E_WORKSPACE (-3) /* caller workspace too small */
#define LTR_E_UNSUPPORTED (-4)

typedef struct LtrModel LtrModel;

/* One checkpoint tensor, fp32, host memory, in the reference state-dict layout
 * (SURVEY.md 8a "State-dict contract"); `name` is the state-dict key. */
typedef struct {
  const char* name;
  const float* data;
  int64_t numel;
} LtrTensor;

typedef struct {
  int32_t d_model;        /* 256  (config 'descriptor_dim') */
  int32_t n_heads;        /* 4    (config 'n_heads') */
  int32_t d_inner;        /* 1024 (config 'd_inner') */
  int32_t n_desc_layers;  /* config 'n_line_descriptive_layers'; only the LAST layer is live
                             in the reference (line_transformer.py:123-125 never chains) */
  int32_t n_sig_layers;   /* 7 (line_transformer.py:213) */
} LtrConfig;

/* Tokenised lines of a batch of images, rows of all images concatenated.
 * Image i owns lines [cu_lines[i], cu_lines[i+1]).  For a uniform batch [B, L, ...] pass
 * cu_lines_host = cu_lines_dev = NULL and lines_per_image = L.
 * The token mask ('mask_sublines') is deliberately absent: in the reference it masks
 * query rows of which only the always-valid CLS row is consumed (models/line_attention.py:
 * 15-16,62-63; models/line_transformer.py:128), so it cannot change the output. */
typedef struct {
  const float* sublines;  /* [n_lines, 2, 2] end points, pixels */
  const float* resp;      /* [n_lines, 1] */
  const float* angle;     /* [n_lines, 2] */
  const float* pnt;       /* [n_lines, n_tokens, 2] token positions, pixels */
  const float* desc;      /* [n_lines, n_tokens, d_model] sampled descriptors */
  const float* score;     /* [n_lines, n_tokens, 1] */
  const int32_t* cu_lines_host; /* [n_images + 1] or NULL (uniform) */
  const int32_t* cu_lines_dev;  /* device copy of the same, or NULL (uniform) */
  int32_t n_images;
  int32_t n_lines;         /* total lines over all images */
  int32_t n_tokens;        /* T (config 'max_tokens'), 1..128 */
  int32_t lines_per_image; /* used when cu_lines_* are NULL */
  float image_width;       /* LineTransformer.image_shape (ctor-time, :206,238) */
  float image_height;
} LtrEncodeInput;

/* Bytes of device scratch ltr_encode needs for this problem size. */
int64_t ltr_encode_workspace_bytes(const LtrModel* m, int32_t n_images, int32_t n_lines,
                                   int32_t n_tokens);

int ltr_create(const LtrTensor* tensors, int32_t n_tensors, const LtrConfig* cfg,
               int32_t device, LtrModel** out);
void ltr_destroy(LtrModel* m);

/* Outputs of ltr_encode (device, caller-owned; any of them may be NULL).
 * desc_cf:    unit-norm descriptors channel-first, image i at offset d_model*cu_lines[i],
 *             element (c, l) at c*L_i + l - for a uniform batch exactly the reference's
 *             line_desc [B, d_model, L].
 * desc_rows:  the same descriptors row-major [n_lines, d_model] (matcher layout).
 * desc_tiles: the same descriptors as the split-bf16 "tile image" the tensor-core matcher
 *             contracts (ltr_desc_tiles_bytes(n_lines) bytes, opaque): hand it to ltr_match
 *             (LtrMatchInput.tiles0/1) and the matcher skips its own fp32 -> tile conversion.
 *             Needs desc_rows != NULL and desc_cf == NULL (it is written by the same fused
 *             projection + L2-normalisation launch as desc_rows). */
typedef struct {
  float* desc_cf;
  float* desc_rows;
  void* desc_tiles;
} LtrEncodeOutput;

int64_t ltr_desc_tiles_bytes(int32_t n_lines);

int ltr_encode(LtrModel* m, const LtrEncodeInput* in, const LtrEncodeOutput* out,
               void* workspace, int64_t workspace_bytes, void* stream);

#define LTR_LAYOUT_ROWS 0          /* [n, d] */
#define LTR_LAYOUT_CHANNEL_FIRST 1 /* [d, n] per image */

/* A batch of independent image pairs.  Side s of pair p owns sublines
 * [cu_s[p], cu_s[p+1]) (uniform: p*n_s .. (p+1)*n_s when cu_s == NULL).
 * Keyline merging (LineTransformer.subline2keyline): the adjacency of
 * models/line_process.py:163-167 is block-constant with weight 1/n_sub over contiguous
 * sublines, so it is passed as CSR offsets: keyline g (global numbering over the whole
 * batch) owns sublines [sub_off_s[g], sub_off_s[g+1]) in global subline numbering and pair
 * p owns keylines [cuk_s[p], cuk_s[p+1]).  With sub_off0 == sub_off1 == NULL every subline
 * is its own keyline (A = I) and no merging pass runs. */
typedef struct {
  const float* desc0;
  const float* desc1;
  int32_t layout;          /* LTR_LAYOUT_* of desc0/desc1 */
  int32_t d;               /* descriptor dim, multiple of 16 (others: LTR_E_UNSUPPORTED, from
                              ltr_match_workspace_bytes too) */
  int32_t n_pairs;         /* at most 65535 (the pair is a grid dimension); more: LTR_E_UNSUPPORTED, from
                              ltr_match_workspace_bytes too - split the pairs into calls */
  int32_t n0, n1;          /* sublines per image when cu0/cu1 are NULL */
  const int32_t* cu0;      /* device [n_pairs+1] or NULL */
  const int32_t* cu1;
  const int32_t* sub_off0; /* device [total keylines side 0 + 1] or NULL */
  const int32_t* sub_off1;
  const int32_t* cuk0;     /* device [n_pairs+1] keyline offsets, required iff sub_off0 != NULL */
  const int32_t* cuk1;
  int32_t max_n0, max_n1;  /* max sublines per image on each side (grid sizing; var-len only) */
  int32_t max_k0, max_k1;  /* max keylines per image on each side (keyline merging only; max_k0 above
                              8 * 65535: LTR_E_UNSUPPORTED) */
  int64_t dist_pair_stride; /* elements between consecutive pairs' matrices in `dist_key`;
                               0 = max_k0*max_k1 (or max_n0*max_n1 without merging) */
  float nn_thresh;         /* strict '<' (models/nn_matcher.py:18) */
  int32_t mutual;
  int32_t total_n0, total_n1; /* total sublines per side (required with cu0/cu1; 0 = n_pairs*n0/n1) */
  int32_t dist_mode;       /* 0: 2 - 2<a,b> (unit descriptors; models/nn_matcher.py:37-38,
                              models/line_process.py:199-200); 1: |a|^2 + |b|^2 - 2<a,b>
                              (evaluations/matcher.py:66-70); mode 1 needs d == 256, no merging */
  /* Optional: descriptor tile images written by ltr_encode (LtrEncodeOutput.desc_tiles) for the SAME
   * descriptors as desc0/desc1.  Usable when d == 256, the batch is uniform (cu0 == cu1 == NULL),
   * n0 % 128 == 0, n1 % 128 == 0 and tiles_row0_s % 128 == 0; tiles_lines_s = the n_lines the image
   * was produced for, tiles_row0_s = row of this side's first line inside it (both sides may live in
   * one image: one ltr_encode over 2P images).  NULL = the matcher converts desc0/desc1 itself. */
  const void* tiles0;
  const void* tiles1;
  int32_t tiles_lines0, tiles_lines1;
  int32_t tiles_row0_0, tiles_row0_1;
} LtrMatchInput;

/* Multi-GPU: the path's ONE collective - every rank learns the per-pair match counts of all ranks - fused
 * into the matcher's tail kernel.  The caller owns a SYMMETRIC int32 buffer (same size on every rank, peer
 * mapped over NVLink, e.g. torch.distributed._symmetric_memory) laid out as
 *     counts[LTR_GATHER_SLOTS][world][n_pairs]  followed by  flags[LTR_GATHER_SLOTS][world].
 * The last thread block of the tail kernel stores this rank's n_pairs counts into row `rank` of slot `slot`
 * of EVERY rank's buffer - one multimem.st per element through the NVSwitch multicast address when `mc_base`
 * is given, else plain stores through the `world` peer pointers - and then publishes flags[slot][rank] =
 * epoch the same way.  No NCCL kernel, no extra launch on the producing side; ltr_gather_wait (one tiny
 * block) waits for the `world` flags of a slot and copies the gathered counts out.  A rank may run at most
 * LTR_GATHER_SLOTS - 2 steps ahead of its own ltr_gather_wait calls. */
#define LTR_GATHER_SLOTS 8
typedef struct {
  void* mc_base;               /* multicast address of the symmetric buffer or NULL */
  void* const* peer_bases;     /* device array [world]: address of the buffer on every rank (used if !mc_base) */
  int32_t rank, world;
  int32_t slot;                /* 0 .. LTR_GATHER_SLOTS-1 */
  int32_t epoch;               /* > 0, increasing per use of a slot */
} LtrPeerGather;

/* Waits (on the stream) until flags[slot][0..world) of the LOCAL symmetric buffer have all reached `epoch`, then
 * copies counts[slot] (world * n_pairs int32) to `out`. */
int ltr_gather_wait(const void* local_base, int32_t world, int32_t n_pairs, int32_t slot, int32_t epoch,
                    int32_t* out, int32_t device, void* stream);

/* Outputs (device).  Keyline k of side 0 lives at index cuk0[p]+k (cu0[p]+k without
 * merging, p*n0+k for a uniform batch); likewise side 1.
 * matches0[k] = index (local to the pair) of the matched keyline in side 1, or -1;
 * scores0[k]  = distance to the nearest neighbour;
 * nn1[k1]     = nearest side-0 keyline of every side-1 keyline (only written if mutual);
 * counts[p]   = number of matches of pair p;
 * dist_key    = keyline distance matrices, pair p at p*dist_pair_stride, row-major
 *               [K0_p, K1_p] (Matching's 'matching_scores_l');
 * dist_sub    = scratch for subline distances [n_pairs, max_n0*max_n1], merging only.
 * workspace   = device scratch of ltr_match_workspace_bytes(in) bytes (tile images, per-line
 *               argmin slots).
 * dist_key may be NULL when there is no key-line merging and d == 256: the distance matrix is
 * then never materialised (row argmin lives in the epilogue of the tensor-core contraction).
 * matches0 == NULL (with scores0, nn1, counts) computes dist_key only (get_dist_matrix). */
typedef struct {
  int32_t* matches0;
  float* scores0;
  int32_t* nn1;
  int32_t* counts;
  float* dist_key;
  float* dist_sub;
  void* workspace;
  int64_t workspace_bytes;
  const LtrPeerGather* gather;   /* optional (d == 256, no merging): publish `counts` to all ranks, see above */
} LtrMatchOutput;

int64_t ltr_match_workspace_bytes(const LtrMatchInput* in);

int ltr_match(const LtrMatchInput* in, const LtrMatchOutput* out, int32_t device, void* stream);

/* Image sets: encode each image once, then match any list of pairs between two image pools.
 *
 * An image-aligned tile image holds the descriptors of a pool of images in the split-bf16 format the
 * tensor-core matcher contracts (the format of LtrEncodeOutput.desc_tiles): image i occupies the
 * ceil(L_i / 128) 128-row tiles starting at tile tile_off[i], where tile_off is the prefix sum of
 * ceil(L_i / 128) (tile_off[0] = 0, n_tiles = tile_off[n_images]); rows past L_i in an image's last tile are
 * zero.  ltr_image_tiles_bytes(n_images, cu_host) = n_tiles * 128 KB (cu_host: HOST [n_images+1] line
 * offsets).  ltr_image_tiles builds it in one launch: desc is the pool's fp32 descriptors, either rows
 * [cu[n_images], 256] (LTR_LAYOUT_ROWS) or channel-first [256, L_i] per image, image i at 256 * cu[i]
 * (LTR_LAYOUT_CHANNEL_FIRST, the layout of SuperPoint's point descriptors); cu_dev and tile_off_dev are device
 * copies of the offsets, max_n = max L_i, out is 16-byte aligned. */
int64_t ltr_image_tiles_bytes(int32_t n_images, const int32_t* cu_host);
int ltr_image_tiles(const float* desc, int32_t layout, const int32_t* cu_dev, const int32_t* tile_off_dev, int32_t n_images,
                    int32_t max_n, int32_t n_tiles, void* out, int32_t device, void* stream);

/* Pair list over two image pools for ltr_match_indexed (device arrays unless noted).  Pair p matches image
 * img0[p] of pool 0 against image img1[p] of pool 1.  img0 / img1 are NOT range-checked on the device: every
 * entry must lie in [0, n_images) of its pool (validate on the host before the call).  out_off0 / out_off1
 * [n_pairs+1] are the per-pair output offsets: prefix sums over the pairs of the side-0 / side-1 key-line counts
 * (line counts without key-line merging; point counts for points); total_out0 / total_out1 = out_off0[n_pairs] /
 * out_off1[n_pairs] (host values: scratch sizing). */
typedef struct {
  const int32_t* img0;
  const int32_t* img1;
  const void* tiles0;        /* image-aligned tile image of pool 0 (ltr_image_tiles) */
  const void* tiles1;
  const int32_t* tile_off0;  /* [n_images0 + 1] */
  const int32_t* tile_off1;
  int32_t n_tiles0, n_tiles1;
  const int32_t* out_off0;
  const int32_t* out_off1;
  int32_t total_out0, total_out1;
} LtrPairIndex;

/* ltr_match over a pair list.  In this mode desc0/desc1, cu0/cu1 (required), cuk0/cuk1 and sub_off0/sub_off1
 * describe the IMAGES of pool 0 and pool 1 (the two pools may be the same arrays), max_n* / max_k* bound the
 * images' line / key-line counts and total_n0/total_n1 are the pools' line counts; n0, n1, tiles* of
 * LtrMatchInput are ignored.  Outputs are per pair: matches0 / scores0 of pair p at out_off0[p] + k, nn1 at
 * out_off1[p] + j, counts[p], dist_key at p * dist_pair_stride, dist_sub at p * max_n0 * max_n1.
 * Supported: d == 256, dist_mode 0, with or without key-line merging; dist_mode 1 and `gather` return
 * LTR_E_UNSUPPORTED. */
int64_t ltr_match_indexed_workspace_bytes(const LtrMatchInput* in, const LtrPairIndex* idx);
int ltr_match_indexed(const LtrMatchInput* in, const LtrPairIndex* idx, const LtrMatchOutput* out, int32_t device,
                      void* stream);

/* nn_matcher_distmat on caller-supplied distance matrices (device, row-major [n0, n1],
 * pair p at p*dist_pair_stride, 0 = n0*n1); negative entries are clipped to 0 as the
 * reference does (models/nn_matcher.py:12).  At most 65535 pairs (more: LTR_E_UNSUPPORTED). */
int ltr_match_distmat(const float* dist, int32_t n_pairs, int32_t n0, int32_t n1,
                      int64_t dist_pair_stride, float nn_thresh, int32_t mutual,
                      int32_t* matches0, float* scores0, int32_t* nn1, int32_t* counts,
                      int32_t device, void* stream);

/* LineTransformer.subline2keyline alone: dist_key[p] = A0_p @ dist_sub[p] @ A1_p^T with the
 * adjacencies given as CSR offsets (see LtrMatchInput).  dist_sub: pair p at p*stride_sub,
 * row-major [S0_p, S1_p]; dist_key: pair p at p*stride_key, row-major [K0_p, K1_p].  At most
 * 65535 pairs and max_k0 <= 8 * 65535 (more: LTR_E_UNSUPPORTED). */
int ltr_merge_sublines(const float* dist_sub, int64_t stride_sub, int32_t n_pairs,
                       const int32_t* cuk0, const int32_t* cuk1, const int32_t* sub_off0,
                       const int32_t* sub_off1, int32_t max_k0, int32_t max_k1, float* dist_key,
                       int64_t stride_key, int32_t device, void* stream);

/* GPU line tokenizer - the step that feeds ltr_encode (reference line_tokenizer +
 * sample_descriptors, models/line_process.py:86-196), over many images in one call.  The host supplies
 * per key line (device arrays): start point, end point before and after the in-place clip to
 * (W-0.6, H-0.6) [K,2] float64, detector length [K] float64, angle code [K,2] float32, n_tok =
 * ceil(length / token_distance) [K], first subline index sub0 [K+1], the key line of every subline [S]
 * and the image of every key line line_image [K].  Key lines of all images are concatenated, image by
 * image, and sub0 / sub2line use global subline numbering.
 * images [n_images] and cu_sublines [n_images+1] are HOST arrays read during the call only: image i
 * owns output rows [cu_sublines[i], cu_sublines[i+1]) of the packed outputs (the LineBatch layout)
 * and is tokenised with its own token_distance and sampled from its own maps, whose sizes may
 * differ between images; a batch equals per-image calls bit for bit.  An image without key lines is
 * an empty range; its maps may be NULL (and so may the outputs of a batch without any key line).
 * Outputs (device, fp32) in the tokenizer's layout: sublines [S,2,2], pnt [S,T,2], mask [S,T+1,1],
 * resp [S,1], angle [S,2], desc [S,T,256] (bilinear grid_sample of the image's dense_desc
 * [256,desc_h,desc_w] + L2 normalisation), score [S,T,1] (its dense_score [score_h,score_w] at the
 * rounded token position).
 * n_tokens must be 1..128 (the encoder's limit) and desc_channels 256.  Nothing synchronises. */
typedef struct {
  const float* dense_desc;     /* device [256, desc_h, desc_w] */
  const float* dense_score;    /* device [score_h, score_w] */
  double token_distance;
  int32_t desc_h, desc_w;
  int32_t score_h, score_w;
} LtrTokenizeImage;

typedef struct {
  const double* sp;
  const double* ep;
  const double* ep_clipped;
  const double* length;
  const float* angle;
  const int32_t* n_tok;
  const int32_t* sub0;
  const int32_t* sub2line;
  const int32_t* line_image;
  int32_t n_images, n_keylines, n_sublines, n_tokens;
  int32_t desc_channels;
  int32_t align_corners;
  const LtrTokenizeImage* images;   /* host [n_images] */
  const int32_t* cu_sublines;       /* host [n_images+1] */
} LtrTokenizeBatchInput;

int ltr_tokenize_batch(const LtrTokenizeBatchInput* in, float* sublines, float* pnt, float* mask, float* resp,
                       float* angle, float* desc, float* score, int32_t device, void* stream);

/* Homography ground truth for line matches, and precision/recall counts of predicted matches, for a batch of
 * pairs.  Per pair this is the homography dataset builder's mat_assign_sublines
 * (dataloaders/build_homography_dataset.py:210-234): find_line_matches (dataloaders/utils/util_lines.py:67-114) of
 * side 0 against side 1 projected into image 0 and of side 1 against side 0 projected into image 1, the mutual AND,
 * calculate_line_overlaps (:116-171) both ways on the mutual entries, then their element-wise max.  Counts follow
 * Evaluate_PR.calc_TFPN (evaluations/evaluate_pr.py:10-22).
 *
 * Side s of pair p owns segments [cu_s[p], cu_s[p+1]) of segs_s ([S, 2, 2] fp32 pixels, start xy then end xy).
 * homography[p] maps image 0 to image 1 and homography_inv[p] is its inverse (computed by the caller; the library
 * never inverts a matrix).  proj0 = segs0 mapped by H and proj1 = segs1 mapped by H^-1 follow
 * cv2.perspectiveTransform: in fp64, w = x*m6 + y*m7 + m8, the point is ((x*m0 + y*m1 + m2) * (1/w), ...) rounded
 * to fp32 if |w| > FLT_EPSILON, else (0, 0).  A caller may pass proj0 / proj1 itself (e.g. the projections a dataset
 * stored); the kernel then skips its own.
 *
 * Arithmetic reproduces the reference's numpy float32 scalars: every + - * / sqrt is an IEEE fp32 operation in the
 * reference's order, so distances, lengths and overlap ratios are bit-identical for the same projections.  Literal
 * behaviours kept on purpose:
 *   - the angle is degrees(atan2(dx, dy)) (x and y swapped) and the difference is |a1 - a0| % 180, so anti-parallel
 *     lines just past 180 degrees pass and lines at ~179 degrees fail;
 *   - a zero-length segment gives a 0/0 = NaN point-line distance, which fails every comparison, so the "both
 *     endpoints far" skip does not fire;
 *   - all comparisons are the reference's strict < / > (overlap: both end points inside -> len1/len0, one inside ->
 *     the distance ratio, neither -> 1 if max distance <= len0 + len1);
 *   - TN counts rows whose number of columns with neither a prediction nor ground truth equals the number of ROWS
 *     (shape[0]); this differs from "all columns" for non-square pairs only.
 * The one deliberate difference: the angle is computed in fp64 (atan2, * 180/pi, fmod) where numpy's float32
 * arctan2 / degrees are not correctly rounded, so the angle decision can differ from the reference's only where
 * its |ang_diff - thres_angdiff| (or |a1 - a0| against 180 / 360) is within about 1e-3 degrees.
 * Inputs must be finite. */
typedef struct {
  const float* segs0;            /* device [S0, 2, 2] */
  const float* segs1;            /* device [S1, 2, 2] */
  const int32_t* cu0;            /* device [n_pairs + 1] */
  const int32_t* cu1;
  const double* homography;      /* device [n_pairs, 3, 3], image 0 -> image 1 */
  const double* homography_inv;  /* device [n_pairs, 3, 3] */
  const float* proj0;            /* optional device [S0, 2, 2]: segs0 mapped by H (NULL: computed) */
  const float* proj1;            /* optional device [S1, 2, 2]: segs1 mapped by H^-1 */
  const int32_t* pred0;          /* optional device [S0]: predicted match of every side-0 segment, local index into
                                    side 1, or -1 (values outside [0, n1_p) count as no prediction) */
  int32_t n_pairs;
  int32_t max_n0, max_n1;        /* bounds of every pair's segment counts (grid sizing) */
  float thres_reprojected;       /* pixels (confs/homography.yaml: 3) */
  double thres_angdiff;          /* degrees (2) */
  double min_overlap_ratio;      /* n_gt counts entries > this (0.3) */
} LtrLineGtInput;

/* Outputs (device, caller-owned).  assign (optional): mat_assign_sublines of pair p as fp32 row-major [n0_p, n1_p]
 * at p * assign_stride (values 0, 1 or fp32 ratios, so lossless), assign_stride >= max_n0 * max_n1.  n_gt [n_pairs]
 * (required): entries > min_overlap_ratio, the length of the builder's lmatches.  tfpn [n_pairs, 4] (required iff
 * pred0): TP, FP, FN, TN with score_gt = assign > 0.  With assign == NULL no dense matrix is written: the counts-only
 * mode for large evaluations. */
typedef struct {
  float* assign;
  int64_t assign_stride;
  int32_t* n_gt;
  int32_t* tfpn;
} LtrLineGtOutput;

/* Asynchronous on `stream`; never synchronises. */
int ltr_line_gt(const LtrLineGtInput* in, const LtrLineGtOutput* out, int32_t device, void* stream);

/* Semi-hard triplet loss of the validation step, forward value only: descriptor_loss.compute_distances + forward
 * (evaluations/criteria.py:35-192) for a batch of pairs, and optionally Evaluate_PR.calc_TFPN
 * (evaluations/evaluate_pr.py:10-22) of predicted matches against the same assignment.
 *
 * Per pair, d[i, j] = 2 - 2 <a_i, b_j> with <a_i, b_j> one ascending-k fmaf chain (the matcher's exact fp32 path), NOT
 * clipped.  With v = the pair's assignment entry (i, j): match iff (double)v > match_thr, unmatch iff
 * (double)v <= unmatch_thr.  Anchors: every side-0 line i (candidates d[i, :]), then every side-1 line j (candidates
 * d[:, j]).  pos = max of d over the anchor's match candidates; the anchor has a positive iff pos > 0.  u = d on unmatch
 * candidates and the literal 10000.f on the others; neg = min of u over pos < u < pos + 0.5f (strict, fp32 sum); the
 * anchor is valid iff that window is not empty.  Per group: n_valid, loss = float(sum of relu((pos - neg) + 1.f) in fp64
 * over the valid anchors, in a fixed order / n_valid), hardest_pos = max pos, hardest_neg = min neg; all three NaN
 * when n_valid == 0.  The reference requires n0 == n1 per pair; this call does not.
 *
 * Thresholds: match_thr = (double)0.3f, unmatch_thr = 0 reproduce torch's float32 comparisons of
 * `mat_assign_sublines` (an entry exactly 0.3f is not a match); match_thr = unmatch_thr = 0.3 on the builder's raw
 * overlaps reproduce the 0/1 matrix train.py builds from `lmatches`. */
typedef struct {
  const float* desc0;            /* device, LTR_LAYOUT_ROWS [S0, 256] or channel-first [256, n0_p] per pair at 256*cu0[p] */
  const float* desc1;
  int32_t layout;
  int32_t d;                     /* must be 256 (others: LTR_E_UNSUPPORTED) */
  int32_t n_pairs;
  int32_t n0, n1;                /* lines per pair when cu0/cu1 are NULL */
  const int32_t* cu0;            /* device [n_pairs + 1] or NULL (uniform) */
  const int32_t* cu1;
  int32_t max_n0, max_n1;        /* bounds of every pair's line counts (var-len only) */
  const float* assign;           /* device fp32, pair p at p * assign_stride, row i at i * assign_ld (0: n1 of the pair),
                                    so [b, n0+1, n1+1] with its dustbin row / column is read in place */
  int64_t assign_stride;
  int32_t assign_ld;
  double match_thr;
  double unmatch_thr;
  const int32_t* pred0;          /* optional device [S0]: predicted side-1 index (local) of every side-0 line, or -1
                                    (values outside [0, n1_p) count as no prediction) */
  int32_t n_groups;              /* groups are contiguous pair ranges [group_off[g], group_off[g+1]) */
  const int32_t* group_off;      /* device [n_groups + 1] or NULL: one group of all pairs (n_groups must be 1) */
} LtrTripletInput;

/* Outputs (device, caller-owned).  Per anchor [S0 + S1]: side-0 line i of pair p at cu0[p] + cu1[p] + i, side-1 line j
 * at cu0[p+1] + cu1[p] + j; pos (NaN without a positive), neg (NaN unless valid), state (0 no positive, 1 positive but
 * empty window, 2 valid).  Per group: loss, hardest_pos, hardest_neg, n_valid.  tfpn [n_pairs, 4] (required iff
 * pred0): TP, FP, FN, TN with ground truth = the match class. */
typedef struct {
  float* pos;
  float* neg;
  int32_t* state;
  float* loss;
  float* hardest_pos;
  float* hardest_neg;
  int32_t* n_valid;
  int32_t* tfpn;
} LtrTripletOutput;

/* Asynchronous on `stream`; never synchronises.  n_pairs == 0 writes nothing. */
int ltr_triplet_loss(const LtrTripletInput* in, const LtrTripletOutput* out, int32_t device, void* stream);

/* RANSAC homographies (image 0 -> image 1) from point and line matches, for a batch of image pairs.  The reference
 * verifies matches with one cv2.findHomography per pair, points only (models/utils.py:291-412 works the same way for
 * poses); this is the project's own estimator, DESIGN.md "Homography estimation" states the model:
 *   - correspondences of pair p: every matched side-0 keypoint row (match in [0, n_pts1[p])) in row order, then every
 *     matched side-0 segment row in row order; each kind only when its switch is on;
 *   - per pair and side, coordinates are normalised by the centre and half the larger extent of that side's bounding
 *     box (points and segment end points);
 *   - hypothesis k draws 4 distinct correspondences with the counter-based hash
 *       s = splitmix64(seed + splitmix64((uint64)p << 32 | k)),  draw j = splitmix64(s + j) mod n,  j = 0, 1, ...
 *     (a duplicate is redrawn with the next j; after 64 draws the hypothesis is rejected) and solves the 8 equations
 *     (two DLT rows per point, l1^T H a0 = l1^T H b0 = 0 per line, l1 the unit-normal line through s1) with h33 = 1 by
 *     fp64 Gaussian elimination with partial pivoting; a pivot below 1e-12, a non-finite result or |H33| < 1e-12
 *     rejects it;
 *   - residuals are fp64 pixels in image 1: point |pi(H x0) - x1|^2, line the larger squared distance of pi(H a0),
 *     pi(H b0) to the line through s1; a projected |w| <= FLT_EPSILON makes an outlier; inlier iff residual <
 *     thresh^2;
 *   - the winner has the most inliers, the lowest k on a tie; it is refitted by least squares over its inliers
 *     (smallest eigenvector of A^T A, cyclic Jacobi) and the refit is kept iff it has at least as many inliers.
 * A pair with fewer than 4 correspondences or no accepted hypothesis is invalid: H is NaN and no row is an inlier.
 *
 * Capacity: one pair's correspondences are staged in shared memory, 18 bytes per keypoint row and 58 per segment row,
 * counted over max_rows_p / max_rows_l of the kinds in use, at most 200 KiB: e.g. 8192 keypoints with 900 segments,
 * 11377 keypoints alone or 3531 segments alone.  Beyond that the call returns LTR_E_UNSUPPORTED before any launch.
 * Coordinates must be finite. */
typedef struct {
  const float* pts0;              /* device [*, 2] keypoint pool of side 0 */
  const float* pts1;              /* device [*, 2] keypoint pool of side 1 */
  const int32_t* pts_off0;        /* device [n_pairs]: pair p's side-0 keypoints start at pts0 row pts_off0[p] */
  const int32_t* pts_off1;        /* device [n_pairs] */
  const int32_t* n_pts1;          /* device [n_pairs]: side-1 keypoints of pair p */
  const int32_t* matches_p;       /* device: local side-1 index or -1 per side-0 keypoint row */
  const int32_t* cu_p;            /* device [n_pairs + 1]: pair p owns matches_p rows [cu_p[p], cu_p[p+1]) */
  const float* segs0;             /* device [*, 2, 2] segment pools (start xy, end xy) */
  const float* segs1;
  const int32_t* seg_off0;        /* device [n_pairs] */
  const int32_t* seg_off1;
  const int32_t* n_segs1;         /* device [n_pairs] */
  const int32_t* matches_l;       /* device: local side-1 index or -1 per side-0 segment row */
  const int32_t* cu_l;            /* device [n_pairs + 1] */
  int32_t n_pairs;
  int32_t max_rows_p, max_rows_l; /* bounds of every pair's match rows (cu_p / cu_l differences); they size the
                                     shared-memory staging, and a pair whose rows exceed them is invalid */
  double thresh;                  /* pixels (3: OpenCV's default) */
  int32_t n_hypotheses;           /* >= 1 (2048) */
  uint64_t seed;
  int32_t use_points, use_lines;  /* 0 / 1: which kinds of correspondence are used */
} LtrHomographyInput;

/* Outputs (device, caller-owned).  key [n_pairs] is workspace (winning (count << 32) | ~k, 0 = none). */
typedef struct {
  double* H;                      /* [n_pairs, 3, 3] */
  uint8_t* valid;                 /* [n_pairs] */
  uint8_t* inliers_p;             /* aligned with matches_p (0 for unmatched rows and unused kinds) */
  uint8_t* inliers_l;             /* aligned with matches_l */
  int32_t* n_inliers_p;           /* [n_pairs] */
  int32_t* n_inliers_l;
  int32_t* hypothesis;            /* [n_pairs] winning hypothesis index, -1 when invalid */
  int32_t* hypothesis_inliers;    /* [n_pairs] its inlier count */
  uint64_t* key;
} LtrHomographyOutput;

/* Asynchronous on `stream`; never synchronises.  n_pairs == 0 writes nothing. */
int ltr_homography(const LtrHomographyInput* in, const LtrHomographyOutput* out, int32_t device, void* stream);

/* Relative pose of calibrated image pairs <- estimate_pose (models/utils.py:291-315): cv2.findEssentialMat(RANSAC) +
 * cv2.recoverPose per pair on the CPU.  Five-point RANSAC essential matrices and the pose, for a batch of pairs; DESIGN.md
 * "Relative pose" states the model:
 *   - correspondences of pair p: every matched side-0 keypoint row (match in [0, n_pts1[p])) in row order with its
 *     partner, in normalised coordinates x = (k - c) / f per axis (K0[p] for side 0, K1[p] for side 1; fp64, correctly
 *     rounded division);
 *   - threshold as the reference: f_mean = (((K0[0,0] + K1[1,1]) + K0[0,0]) + K1[1,1]) / 4, t_n = thresh / f_mean; an
 *     inlier has Sampson error (x1^T E x0)^2 / ((E x0)_0^2 + (E x0)_1^2 + (E^T x1)_0^2 + (E^T x1)_1^2) < t_n^2,
 *     evaluated as (x1^T E x0)^2 < t_n^2 * (the denominator);
 *   - hypothesis k draws 5 distinct correspondences with ltr_homography's hash and redraw rule and solves them with
 *     Nister's five-point method (QR null space, 10 x 20 Gauss-Jordan, degree-10 determinant, Sturm chain and
 *     bisection) in explicitly rounded fp64: up to 10 solutions j (real root j in ascending order);
 *   - the winner has the most inliers, then the lowest k, then the lowest j; no refit;
 *   - E is scaled to unit Frobenius norm with its largest-magnitude entry positive; of its four (R, t) candidates the
 *     one with the most inliers of depth in (0, dist_thresh) in both cameras wins; |t| = 1.  X1 = R X0 + t.
 * A pair with fewer than 5 correspondences, no finite solution, or more match rows than max_rows_p is invalid: E, R and
 * t are NaN, no row is an inlier, hypothesis is -1.
 *
 * Capacity: one pair's correspondences are staged in shared memory, 33 bytes per keypoint row over max_rows_p, at most
 * 200 KiB (6206 rows).  Beyond that the call returns LTR_E_UNSUPPORTED before any launch.  Coordinates and K must be
 * finite, with fx, fy > 0. */
typedef struct {
  const float* pts0;              /* device [*, 2] keypoint pool of side 0 */
  const float* pts1;              /* device [*, 2] keypoint pool of side 1 */
  const int32_t* pts_off0;        /* device [n_pairs]: pair p's side-0 keypoints start at pts0 row pts_off0[p] */
  const int32_t* pts_off1;        /* device [n_pairs] */
  const int32_t* n_pts1;          /* device [n_pairs]: side-1 keypoints of pair p */
  const int32_t* matches_p;       /* device: local side-1 index or -1 per side-0 keypoint row */
  const int32_t* cu_p;            /* device [n_pairs + 1]: pair p owns matches_p rows [cu_p[p], cu_p[p+1]) */
  const double* K0;               /* device [n_pairs, 3, 3] intrinsics of side 0 */
  const double* K1;               /* device [n_pairs, 3, 3] intrinsics of side 1 */
  int32_t n_pairs;
  int32_t max_rows_p;             /* bound of every pair's match rows; sizes the staging, a pair over it is invalid */
  double thresh;                  /* pixels (the reference's evaluation passes 1) */
  double dist_thresh;             /* cheirality depth limit in units of |t| (1e9, as the reference's recoverPose) */
  int32_t n_hypotheses;           /* >= 1 (1024) */
  uint64_t seed;
} LtrEssentialInput;

/* Outputs (device, caller-owned).  key [n_pairs] is workspace (winning (count << 32) | ~(10 k + j), 0 = none). */
typedef struct {
  double* E;                      /* [n_pairs, 3, 3] essential matrix, x1^T E x0 = 0 in normalised coordinates */
  double* R;                      /* [n_pairs, 3, 3] */
  double* t;                      /* [n_pairs, 3] unit */
  uint8_t* valid;                 /* [n_pairs] */
  uint8_t* inliers_p;             /* aligned with matches_p (0 for unmatched rows) */
  int32_t* n_inliers;             /* [n_pairs] */
  int32_t* n_cheirality;          /* [n_pairs] inliers in front of both cameras under (R, t) */
  int32_t* hypothesis;            /* [n_pairs] 10 k + j of the winning solution, -1 when invalid */
  int32_t* hypothesis_inliers;    /* [n_pairs] its inlier count */
  uint64_t* key;
} LtrEssentialOutput;

/* Asynchronous on `stream`; never synchronises.  Errors (LTR_E_INVALID for bad arguments, LTR_E_UNSUPPORTED over
 * capacity) come before any launch.  n_pairs == 0 writes nothing. */
int ltr_essential(const LtrEssentialInput* in, const LtrEssentialOutput* out, int32_t device, void* stream);

/* Fundamental matrices of uncalibrated image pairs, as one cv2.findFundamentalMat(FM_RANSAC) per pair would verify
 * them, plus an epipolar check of the line matches; DESIGN.md "Fundamental matrices" states the model:
 *   - F maps image 0 to image 1: x1^T F x0 = 0 in pixels;
 *   - correspondences of pair p: every matched side-0 keypoint row (match in [0, n_pts1[p])) in row order with its
 *     partner; per side, coordinates are normalised by the centre and half the larger extent of that side's bounding
 *     box (as ltr_homography's points);
 *   - hypothesis k draws 7 distinct correspondences with ltr_homography's hash and redraw rule and solves them with the
 *     seven-point method (QR null space F1, F2, the cubic det(F2 + a (F1 - F2)), its real roots by a Sturm chain and
 *     bisection) in explicitly rounded fp64: up to 3 solutions j (real root j in ascending order; the solution at
 *     a = infinity is not returned), denormalised and scaled to unit Frobenius norm, largest |entry| positive;
 *   - inlier iff cv2's FM error, max((x1^T F x0)^2 / |(F x0)_xy|^2, (x1^T F x0)^2 / |(F^T x1)_xy|^2), is below
 *     thresh^2, evaluated without the division; a zero line normal makes an outlier;
 *   - the winner has the most inliers, then the lowest k, then the lowest j; with at least 8 inliers it is refitted by
 *     the normalised eight-point method over them (smallest eigenvector of A^T A, rank 2 through the SVD), and the
 *     refit is kept iff it has at least as many inliers;
 *   - line check (lines_consistent, aligned with matches_l): for a matched key-line pair s0 = (a0, b0), s1 = (a1, b1),
 *     the epipolar lines F a0, F b0 cut the line through s1 at positions ta, tb (a1 at 0, b1 at 1); the overlap ratio
 *     is |[min, max] n [0, 1]| / min(max - min, 1); the same with F^T on s0.  A side whose intersection has |w| <=
 *     FLT_EPSILON |X|, or whose two positions coincide, cannot reject.  Consistent iff no side's ratio is below
 *     min_overlap.  Lines take no part in the fit.
 * A pair with fewer than 7 correspondences, no finite solution, or more match rows than max_rows_p is invalid: F is NaN,
 * no row is an inlier or consistent, hypothesis is -1.  A planar scene is degenerate for F: use ltr_homography there.
 *
 * Capacity: one pair's correspondences are staged in shared memory, 18 bytes per keypoint row over max_rows_p, at most
 * 200 KiB (11377 rows).  Beyond that the call returns LTR_E_UNSUPPORTED before any launch.  Line rows are read from
 * global memory and have no bound.  Coordinates must be finite. */
typedef struct {
  const float* pts0;              /* device [*, 2] keypoint pool of side 0 */
  const float* pts1;              /* device [*, 2] keypoint pool of side 1 */
  const int32_t* pts_off0;        /* device [n_pairs]: pair p's side-0 keypoints start at pts0 row pts_off0[p] */
  const int32_t* pts_off1;        /* device [n_pairs] */
  const int32_t* n_pts1;          /* device [n_pairs]: side-1 keypoints of pair p */
  const int32_t* matches_p;       /* device: local side-1 index or -1 per side-0 keypoint row */
  const int32_t* cu_p;            /* device [n_pairs + 1]: pair p owns matches_p rows [cu_p[p], cu_p[p+1]) */
  const float* segs0;             /* device [*, 2, 2] segment pools (start xy, end xy) */
  const float* segs1;
  const int32_t* seg_off0;        /* device [n_pairs]: pair p's side-0 segments start at segs0 row seg_off0[p] */
  const int32_t* seg_off1;
  const int32_t* n_segs1;         /* device [n_pairs] */
  const int32_t* matches_l;       /* device: local side-1 index or -1 per side-0 segment row */
  const int32_t* cu_l;            /* device [n_pairs + 1] */
  int32_t n_pairs;
  int32_t max_rows_p;             /* bound of every pair's keypoint match rows; sizes the staging, a pair over it is
                                     invalid */
  int32_t max_rows_l;             /* bound of every pair's segment match rows (0: no line matches) */
  double thresh;                  /* pixels (3: OpenCV's default) */
  double min_overlap;             /* in [0, 1] (0.5) */
  int32_t n_hypotheses;           /* >= 1 (2048) */
  uint64_t seed;
} LtrFundamentalInput;

/* Outputs (device, caller-owned).  key [n_pairs] is workspace (winning (count << 32) | ~(3 k + j), 0 = none). */
typedef struct {
  double* F;                      /* [n_pairs, 3, 3] x1^T F x0 = 0 in pixels, unit Frobenius norm */
  uint8_t* valid;                 /* [n_pairs] */
  uint8_t* refit;                 /* [n_pairs] 1 where F is the eight-point refit */
  uint8_t* inliers_p;             /* aligned with matches_p (0 for unmatched rows) */
  uint8_t* lines_consistent;      /* aligned with matches_l (0 for unmatched rows and invalid pairs) */
  int32_t* n_inliers;             /* [n_pairs] */
  int32_t* n_lines_consistent;    /* [n_pairs] */
  int32_t* hypothesis;            /* [n_pairs] 3 k + j of the winning solution, -1 when invalid */
  int32_t* hypothesis_inliers;    /* [n_pairs] its inlier count */
  uint64_t* key;
} LtrFundamentalOutput;

/* Asynchronous on `stream`; never synchronises.  Errors (LTR_E_INVALID for bad arguments, LTR_E_UNSUPPORTED over
 * capacity) come before any launch.  n_pairs == 0 writes nothing. */
int ltr_fundamental(const LtrFundamentalInput* in, const LtrFundamentalOutput* out, int32_t device, void* stream);

/* Absolute pose of query images, as cv2.solvePnPRansac per query would localize them from 2D-3D point matches, with
 * the line matches scored and refined too; DESIGN.md "Absolute pose" states the model:
 *   - side 0 is the query, side 1 a database image with 3D: X1 rows (fp64 [*, 3]) are aligned with pair p's side-1
 *     keypoints from x_off1[p], L1 rows (fp64 [*, 2, 3], the two end points) with its side-1 segments from l_off1[p];
 *     a row with a non-finite coordinate has no 3D.  The pose maps world to query camera: X_cam = R X + t;
 *   - group g is the run of pairs [groups[g], groups[g+1]), which share one side-0 (query) image; its correspondences
 *     are its pairs' point rows in pair and row order (a side-0 keypoint row with a match in [0, n_x1[p]) whose 3D is
 *     finite), then, with use_lines, its line rows (a side-0 segment row with a match in [0, n_l1[p]) whose two end
 *     points are finite); query pixels are normalised as ((x - cx) / fx, (y - cy) / fy) with K0[g] (skew ignored);
 *   - world coordinates are shifted by the midpoint c of the bounding box of the group's staged 3D coordinates;
 *   - hypothesis k draws 3 distinct point rows with ltr_homography's hash and redraw rule (pair index = group index) and
 *     solves them with Grunert's P3P in explicitly rounded fp64: the quartic in the distance ratio, its real roots by
 *     a Sturm chain and bisection, positive distances only, R from the triads of the camera and world points,
 *     t = P1 - R X1.  Up to 4 solutions j (real root j in ascending order); a sample whose world points are collinear
 *     (cross-product norm <= 1e-10 times the product of the edge lengths) has none;
 *   - a point is an inlier iff its depth is > 0 and its reprojection error through K0 is below thresh pixels; a line
 *     iff both end points have depth > 0 and lie within thresh pixels of the infinite line through the query segment;
 *     without use_lines only points are scored.  Lines never take part in sampling;
 *   - the winner has the most inliers (points plus lines), then the lowest k, then the lowest j.  With at least 3
 *     inliers it is refined by Levenberg-Marquardt over them (20 steps, R <- cay(w) R, t <- t + dt, damping 1e-3 times
 *     0.1 after a step that lowers the cost and 10 after one that does not), kept iff it has at least as many inliers.
 * A group with fewer than 3 point rows, no finite solution, or more match rows than max_rows_p / max_rows_l is
 * invalid: R and t are NaN, no row is an inlier, hypothesis is -1.
 *
 * Capacity: one group's correspondences are staged in shared memory, 32 bytes per keypoint row over max_rows_p and 64
 * per segment row over max_rows_l (with use_lines), at most 200 KiB.  Beyond that the call returns LTR_E_UNSUPPORTED
 * before any launch.  K0 must be finite with fx, fy > 0. */
typedef struct {
  const float* pts0;              /* device [*, 2] query keypoint pool */
  const int32_t* pts_off0;        /* device [n_pairs]: pair p's query keypoints start at pts0 row pts_off0[p] */
  const int32_t* matches_p;       /* device: local side-1 index or -1 per query keypoint row */
  const int32_t* cu_p;            /* device [n_pairs + 1]: pair p owns matches_p rows [cu_p[p], cu_p[p+1]) */
  const double* X1;               /* device [*, 3] world points of the database keypoints */
  const int32_t* x_off1;          /* device [n_pairs]: pair p's side-1 rows start at X1 row x_off1[p] */
  const int32_t* n_x1;            /* device [n_pairs]: side-1 keypoints of pair p */
  const float* segs0;             /* device [*, 2, 2] query segment pool (start xy, end xy) */
  const int32_t* seg_off0;        /* device [n_pairs] */
  const int32_t* matches_l;       /* device: local side-1 index or -1 per query segment row */
  const int32_t* cu_l;            /* device [n_pairs + 1] */
  const double* L1;               /* device [*, 2, 3] world end points of the database segments */
  const int32_t* l_off1;          /* device [n_pairs] */
  const int32_t* n_l1;            /* device [n_pairs] */
  const int32_t* groups;          /* device [n_groups + 1]: pair offsets, non-decreasing from 0 to n_pairs */
  const double* K0;               /* device [n_groups, 3, 3] query intrinsics */
  int32_t n_pairs;
  int32_t n_groups;
  int32_t max_rows_p;             /* bound of every group's keypoint match rows; sizes the staging, a group over it is
                                     invalid */
  int32_t max_rows_l;             /* bound of every group's segment match rows */
  double thresh;                  /* pixels (8: cv2.solvePnPRansac's default) */
  int32_t n_hypotheses;           /* >= 1 (1024) */
  uint64_t seed;
  int32_t use_lines;              /* 0: score points only */
} LtrAbsPoseInput;

/* Outputs (device, caller-owned).  key [n_groups] is workspace (winning (count << 32) | ~(4 k + j), 0 = none). */
typedef struct {
  double* R;                      /* [n_groups, 3, 3] world -> query camera */
  double* t;                      /* [n_groups, 3] */
  uint8_t* valid;                 /* [n_groups] */
  uint8_t* refit;                 /* [n_groups] 1 where the pose is the Levenberg-Marquardt refit */
  uint8_t* inliers_p;             /* aligned with matches_p (0 for rows without a correspondence) */
  uint8_t* inliers_l;             /* aligned with matches_l (0 for rows without a correspondence, and without use_lines) */
  int32_t* n_inliers_p;           /* [n_groups] */
  int32_t* n_inliers_l;           /* [n_groups] */
  int32_t* hypothesis;            /* [n_groups] 4 k + j of the winning solution, -1 when invalid */
  int32_t* hypothesis_inliers;    /* [n_groups] its inlier count (points and lines) */
  uint64_t* key;
} LtrAbsPoseOutput;

/* Asynchronous on `stream`; never synchronises.  Errors (LTR_E_INVALID for bad arguments, LTR_E_UNSUPPORTED over
 * capacity) come before any launch.  n_groups == 0 writes nothing.  Writes the masks of the rows of pairs in
 * [groups[0], groups[n_groups]). */
int ltr_absolute_pose(const LtrAbsPoseInput* in, const LtrAbsPoseOutput* out, int32_t device, void* stream);

/* ltr_absolute_pose with line hypotheses too: n_line_hypotheses (0 to 2^21) hypotheses for each of three minimal
 * solvers that use line matches, next to the n_hypotheses P3P ones and competing for the same winner (DESIGN.md
 * "Absolute pose"):
 *   - solver s = 0 P2P1L (2 point rows, 1 line row), 1 P1P2L (1 point, 2 lines), 2 P3L (3 lines); it draws its point
 *     rows with seed + 2 s + 1 and its line rows with seed + 2 s + 2, and runs only in groups with that many rows;
 *   - a line row constrains the pose by both world end points lying on the plane through the camera centre and the
 *     query segment; each solver reduces its six constraints to two equations in the two angles of R' = Rz(a) Rx(b)
 *     between a world and a camera triad, and up to 8 solutions j (real root j of a degree-8 polynomial in tan(b / 2),
 *     ascending; b = pi is not found);
 *   - hypothesis k of solver s has index 4 n_hypotheses + 8 (s n_line_hypotheses + k) + j; ties still go to the
 *     lowest index, so P3P wins equal counts.  A group without point rows can be valid.
 * Samples degenerate for their solver have no solution: |j1 x j2| <= 1e-10 for P2P1L's two unit bearings, |n1 . j1|
 * <= 1e-10 |n1| for P1P2L (the point on line 1), |n1 . (n2 x n3)| <= 1e-10 |n1| |n2| |n3| for P3L (concurrent query
 * lines).  With n_line_hypotheses > 0, n_hypotheses may be 0 and use_lines is required (LTR_E_INVALID otherwise);
 * with 0 this is ltr_absolute_pose, the same bits. */
int ltr_absolute_pose_lines(const LtrAbsPoseInput* in, const LtrAbsPoseOutput* out, int32_t n_line_hypotheses,
                            int32_t device, void* stream);

/* Triangulation of posed images: a world point for every keypoint and two world end points for every key line of every
 * image, from the pair matches of the set (ltr_match_indexed / match_set); DESIGN.md "Triangulation" states the model:
 *   - image i has intrinsics K[i] (zero skew: fx, fy, cx, cy are read) and the world -> camera pose X_cam = R[i] X +
 *     t[i], centre C = -R^T t.  A row of image a (the anchor) is lifted along its own ray by its depth s,
 *     X = C_a + s R_a^T K_a^-1 (x, y, 1): a keypoint's ray, or each end point's ray of a key line;
 *   - observations: every pair that contains a gives at most one partner row, in the order of views[view_off[a] ..
 *     view_off[a+1]) (pair << 1 | side of a; pair order): matches_*[cu_*[p] + k] when a is side 0 of pair p, the
 *     lowest side-0 row that matched k when a is side 1 (found by an atomicMin scatter into inv_*); a match outside
 *     [0, rows of the partner) is no observation;
 *   - residuals in pixels: a point's reprojection error into the partner; an end point's signed distance of its
 *     projection to the infinite line through the partner segment (the partner's back-projected plane);
 *   - candidates: each observation's two-view depth (a point's least-squares root of its two residual numerators, an
 *     end point's plane intersection), kept iff depth > 0 and the triangulation angle >= min_angle degrees (a point:
 *     the angle between the two rays at X; a key line: between each end point's ray and the partner plane);
 *   - support: an observation supports a depth iff its own depth is > 0 and its residual is <= thresh (a key line at
 *     both end points).  The winner has the most supporters, ties to the lowest observation;
 *   - refit: 5 one-dimensional Gauss-Newton steps over the supporters' residuals (a key line's end points separately),
 *     kept iff its depth is > 0 and it has at least as many supporters;
 *   - valid iff 1 + supporters >= min_views: n_views = 1 + supporters, else NaN coordinates and n_views = 0.
 * Every operation is explicitly rounded fp64 in a fixed order.
 *
 * Capacity: at most LTR_TRI_MAX_VIEWS pairs per image (max_views), else LTR_E_UNSUPPORTED before any launch.  Pairs
 * must be distinct unordered pairs of two different images (checked by the caller: the kernels take them as given). */
#define LTR_TRI_MAX_VIEWS 64
typedef struct {
  const float* kpts;              /* device [*, 2] keypoints, image i's rows from kp_off[i] */
  const int32_t* kp_off;          /* device [n_images + 1] */
  const float* segs;              /* device [*, 2, 2] key lines (start xy, end xy), image i's rows from seg_off[i] */
  const int32_t* seg_off;         /* device [n_images + 1] */
  const double* K;                /* device [n_images, 3, 3] */
  const double* R;                /* device [n_images, 3, 3] world -> camera */
  const double* t;                /* device [n_images, 3] */
  const int32_t* pairs;           /* device [n_pairs, 2] image indices */
  const int32_t* matches_p;       /* device: local side-1 keypoint index or -1 per side-0 keypoint row */
  const int32_t* cu_p;            /* device [n_pairs + 1]: pair p owns matches_p rows [cu_p[p], cu_p[p+1]), as many as
                                     image pairs[p][0] has keypoints */
  const int32_t* matches_l;       /* device: the same for key lines */
  const int32_t* cu_l;            /* device [n_pairs + 1] */
  const int32_t* views;           /* device: image i's observations [view_off[i], view_off[i+1]), pair << 1 | side */
  const int32_t* view_off;        /* device [n_images + 1] */
  const int32_t* block_off;       /* device [2 n_images + 1]: prefix sum of ceil(rows / 128) over the images'
                                     keypoints, then over their key lines */
  const int32_t* inv_off_p;       /* device [n_pairs + 1]: prefix sum of the keypoint counts of images pairs[p][1] */
  const int32_t* inv_off_l;       /* device [n_pairs + 1]: the same for key lines */
  int32_t n_images;
  int32_t n_pairs;
  int32_t total_p;                /* cu_p[n_pairs] (host value) */
  int32_t total_l;                /* cu_l[n_pairs] */
  int32_t n_inv_p;                /* inv_off_p[n_pairs] */
  int32_t n_inv_l;                /* inv_off_l[n_pairs] */
  int32_t n_blocks;               /* block_off[2 n_images] */
  int32_t max_views;              /* the largest view_off[i+1] - view_off[i], at most LTR_TRI_MAX_VIEWS */
  double thresh;                  /* pixels (4) */
  double min_angle;               /* degrees in [0, 90) (1.5) */
  int32_t min_views;              /* >= 1 (2) */
} LtrTriangulateInput;

/* Outputs (device, caller-owned), aligned with kpts / segs.  inv_p [n_inv_p] / inv_l [n_inv_l] int32 are workspace. */
typedef struct {
  double* points3d;               /* [*, 3] */
  double* lines3d;                /* [*, 2, 3] */
  int32_t* n_views_p;             /* [*] */
  int32_t* n_views_l;             /* [*] */
  int32_t* inv_p;
  int32_t* inv_l;
} LtrTriangulateOutput;

/* Asynchronous on `stream`; never synchronises.  Errors (LTR_E_INVALID for bad arguments, LTR_E_UNSUPPORTED over
 * capacity) come before any launch.  Two launches: the scatter of the side-1 index, then one thread per row. */
int ltr_triangulate(const LtrTriangulateInput* in, const LtrTriangulateOutput* out, int32_t device, void* stream);

/* Tracks of posed images: the pair matches that agree with the poses join the rows of all images into point and line
 * tracks, and each track gets one world point or world line; DESIGN.md "Tracks" states the model:
 *   - nodes: image i's keypoint k is point node kp_off[i] + k, its key line k line node seg_off[i] + k (two graphs);
 *   - edges: a match row of pair p = (i, j) whose match m lies in [0, rows of j) and agrees with F[p], the pixel
 *     fundamental matrix of the poses (x_j^T F x_i = 0, computed by the caller): a point under cv2's FM error below
 *     epi_thresh, a key line under the epipolar overlap check of ltr_fundamental with min_overlap;
 *   - tracks: connected components of >= 2 nodes (lock-free union-find, each labelled by its minimum node), numbered in
 *     ascending order of that node; a track's observations obs[track_off[t] .. track_off[t+1]) ascend by node;
 *   - candidates (tracks of at most LTR_TRK_MAX_OBS observations): every pair (i, j), i < j in track order, gives
 *     ltr_triangulate's two-view estimate along observation i's ray(s) from j (depth > 0, triangulation angle >=
 *     min_angle);
 *   - support: observation q supports a world point iff its depth is > 0 and its reprojection error is <= thresh (a key
 *     line: the distance of both world end points to q's infinite line).  The winner has the most supporters, ties to
 *     the lowest i * LTR_TRK_MAX_OBS + j;
 *   - refit: 5 Gauss-Newton steps on the 3D point (a key line: each of the anchor's world end points, with the anchor's
 *     own pixel residuals and the supporters' line distances) over the winner's supporters, kept iff every supporter
 *     keeps depth > 0 and the supporter count does not fall; the inliers are the supporters of the kept estimate;
 *   - status: LTR_TRK_OK iff inliers >= min_views; LTR_TRK_TOO_LONG (more than LTR_TRK_MAX_OBS observations),
 *     LTR_TRK_NO_CANDIDATE, LTR_TRK_TOO_FEW give NaN coordinates.  An inlier row of a valid track gets its track's point
 *     (a key line: the points of the track's line closest to its own two end-point rays) and n_views = inliers; every
 *     other row NaN and 0.
 * Every operation is explicitly rounded fp64 in a fixed order, so the outputs do not depend on the atomics' order. */
#define LTR_TRK_MAX_OBS 64
#define LTR_TRK_OK 0
#define LTR_TRK_TOO_LONG 1
#define LTR_TRK_NO_CANDIDATE 2
#define LTR_TRK_TOO_FEW 3
typedef struct {
  const float* kpts;              /* device [n_kp, 2] keypoints, image i's rows from kp_off[i] */
  const int32_t* kp_off;          /* device [n_images + 1] */
  const float* segs;              /* device [n_kl, 2, 2] key lines (start xy, end xy), image i's rows from seg_off[i] */
  const int32_t* seg_off;         /* device [n_images + 1] */
  const double* K;                /* device [n_images, 3, 3] */
  const double* R;                /* device [n_images, 3, 3] world -> camera */
  const double* t;                /* device [n_images, 3] */
  const double* F;                /* device [n_pairs, 3, 3] pixel fundamental matrix of pair p, image pairs[p][0] -> 1 */
  const int32_t* pairs;           /* device [n_pairs, 2] image indices */
  const int32_t* matches_p;       /* device: local side-1 keypoint index or -1 per side-0 keypoint row */
  const int32_t* cu_p;            /* device [n_pairs + 1] */
  const int32_t* matches_l;       /* device: the same for key lines */
  const int32_t* cu_l;            /* device [n_pairs + 1] */
  int32_t n_images;
  int32_t n_pairs;
  int32_t total_p;                /* cu_p[n_pairs] (host value) */
  int32_t total_l;                /* cu_l[n_pairs] */
  int32_t n_kp;                   /* kp_off[n_images] (host value) */
  int32_t n_kl;                   /* seg_off[n_images] */
  double thresh;                  /* pixels (4) */
  double min_angle;               /* degrees in [0, 90) (1.5) */
  int32_t min_views;              /* >= 1 (2) */
  double epi_thresh;              /* pixels (4) */
  double min_overlap;             /* (0.5) */
} LtrTracksInput;

/* Outputs (device, caller-owned).  T_p = max(n_kp / 2, 1) and T_l = max(n_kl / 2, 1) bound the track counts; entries
 * of tracks at or past *n_tracks_* are not written.  workspace: int32 [5 (n_kp + n_kl)]. */
typedef struct {
  int32_t* track_p;               /* [n_kp] track of each keypoint row, -1 for none */
  int32_t* track_l;               /* [n_kl] */
  int32_t* n_tracks_p;            /* [1] */
  int32_t* n_tracks_l;            /* [1] */
  int32_t* track_off_p;           /* [T_p + 1] */
  int32_t* track_off_l;           /* [T_l + 1] */
  int32_t* obs_p;                 /* [n_kp] keypoint rows of track t: obs_p[track_off_p[t] .. track_off_p[t+1]) */
  int32_t* obs_l;                 /* [n_kl] */
  double* points3d;               /* [T_p, 3] */
  double* lines3d;                /* [T_l, 2, 3] the anchor observation's two world end points */
  int32_t* n_obs_p;               /* [T_p] */
  int32_t* n_obs_l;               /* [T_l] */
  int32_t* n_inliers_p;           /* [T_p] */
  int32_t* n_inliers_l;           /* [T_l] */
  int32_t* n_images_p;            /* [T_p] distinct images among the observations */
  int32_t* n_images_l;            /* [T_l] */
  int32_t* status_p;              /* [T_p] LTR_TRK_* */
  int32_t* status_l;              /* [T_l] */
  uint8_t* inlier_p;              /* [n_kp] 1 for a supporter of its track's kept estimate */
  uint8_t* inlier_l;              /* [n_kl] */
  double* row_points3d;           /* [n_kp, 3] */
  double* row_lines3d;            /* [n_kl, 2, 3] */
  int32_t* n_views_p;             /* [n_kp] */
  int32_t* n_views_l;             /* [n_kl] */
  int32_t* workspace;
} LtrTracksOutput;

/* Asynchronous on `stream`; never synchronises.  Errors (LTR_E_INVALID for bad arguments) come before any launch.  Six
 * launches: initialisation, edges and unions, path compression, the prefix sum over the roots, the observation slots,
 * then one persistent grid over the tracks up to the device track count. */
int ltr_tracks(const LtrTracksInput* in, const LtrTracksOutput* out, int32_t device, void* stream);

/* Bundle adjustment of a posed image set over the tracks of ltr_tracks: the camera poses, the world points of the
 * point tracks and the world lines of the line tracks refined together; DESIGN.md "Bundle adjustment" states the model:
 *   - participation: a track takes part (LTR_BA_IN) iff its ltr_tracks status is LTR_TRK_OK, its inlier rows lie in
 *     distinct images (else LTR_BA_SAME_IMAGE) and every pivot of the Cholesky of its undamped initial landmark block is
 *     > 1e-12 times its diagonal entry (else LTR_BA_DEGENERATE); any other track is LTR_BA_NOT_VALID.  Its inlier rows
 *     are its residual blocks;
 *   - residuals (pixels): a point row's two reprojection errors, a key-line row the signed distances n . P / P_z of the
 *     track's two world end points to the row's infinite line; the cost is their sum of squares;
 *   - parameters: camera R <- cay(w) R, C <- C + dC (t = -R C); point 3 DoF; line 4 DoF, each end point moving in the
 *     plane orthogonal to the line's direction;
 *   - gauge: images with fixed[i] != 0 keep their input bits; with n_fixed == 1, the lowest free image k with a
 *     participating row also holds its centre coordinate hold[k] (the caller's choice: the first-largest |C_k - C_f|);
 *   - solver: Levenberg-Marquardt (A + lambda diag A, lambda from 1e-3, x0.1 after an accepted step, x10 after a
 *     rejected one) with a Schur complement onto the cameras, a dense Cholesky of the reduced camera matrix in one CTA;
 *     a step is accepted iff every factorization succeeds, every participating depth stays > 0 and the cost falls; the
 *     adjustment stops after an accepted step with relative decrease <= ftol, when lambda > 1e32 or after max_iters
 *     iterations.
 * Every operation is explicitly rounded fp64 in a fixed order, so two calls give the same bits. */
#define LTR_BA_MAX_IMAGES 128
#define LTR_BA_MAX_ITERS 1000
#define LTR_BA_IN 0
#define LTR_BA_NOT_VALID 1
#define LTR_BA_SAME_IMAGE 2
#define LTR_BA_DEGENERATE 3
#define LTR_BA_STOP_ITERS 0
#define LTR_BA_STOP_FTOL 1
#define LTR_BA_STOP_LAMBDA 2
#define LTR_BA_STATS 8
typedef struct {
  const float* kpts;              /* device [n_kp, 2], as ltr_tracks */
  const int32_t* kp_off;          /* device [n_images + 1] */
  const float* segs;              /* device [n_kl, 2, 2] */
  const int32_t* seg_off;         /* device [n_images + 1] */
  const double* K;                /* device [n_images, 3, 3] */
  const double* R;                /* device [n_images, 3, 3] world -> camera */
  const double* t;                /* device [n_images, 3] */
  const int32_t* hold;            /* device [n_images] the held centre coordinate (0..2) of each image (n_fixed == 1) */
  const int32_t* fixed;           /* device [n_images] 1 = the pose is held */
  const int32_t* n_tracks_p;      /* device [1]: the ltr_tracks outputs of the same set */
  const int32_t* n_tracks_l;
  const int32_t* track_off_p;
  const int32_t* track_off_l;
  const int32_t* obs_p;
  const int32_t* obs_l;
  const int32_t* status_p;        /* LTR_TRK_* */
  const int32_t* status_l;
  const uint8_t* inlier_p;
  const uint8_t* inlier_l;
  const int32_t* track_p;
  const int32_t* track_l;
  const int32_t* n_views_p;
  const int32_t* n_views_l;
  const double* points3d;         /* [t_p, 3] */
  const double* lines3d;          /* [t_l, 2, 3] */
  int32_t n_images;               /* <= LTR_BA_MAX_IMAGES */
  int32_t n_fixed;                /* >= 1: images with fixed[i] != 0 */
  int32_t n_kp;                   /* kp_off[n_images] (host value) */
  int32_t n_kl;                   /* seg_off[n_images] */
  int32_t t_p;                    /* the ltr_tracks bounds max(n_kp / 2, 1), max(n_kl / 2, 1) */
  int32_t t_l;
  int32_t max_iters;              /* in [0, LTR_BA_MAX_ITERS] (50): 5 launches each are enqueued, whatever the stop */
  double ftol;                    /* finite, >= 0 (1e-10) */
} LtrBundleInput;

/* Outputs (device, caller-owned).  Entries of tracks at or past *n_tracks_* are not written.  stats fp64
 * [LTR_BA_STATS]: initial cost, final cost, final lambda, iterations, accepted steps, stop reason (LTR_BA_STOP_*),
 * participating observations, participating tracks.  workspace: LTR_BA_WORKSPACE_BYTES(n_images, n_kp, n_kl, t_p, t_l)
 * bytes, 8-byte aligned. */
#define LTR_BA_WORKSPACE_BYTES(n, n_kp, n_kl, t_p, t_l)                                                            \
  (8 * (64 * ((int64_t)(n_kp) + (n_kl)) + 40 * ((int64_t)(t_p) + (t_l)) + 36 * (int64_t)(n) * (n) + 60 * (int64_t)(n) + \
        16) +                                                                                                        \
   4 * (2 * ((int64_t)(n_kp) + (n_kl)) + 4 * ((int64_t)(t_p) + (t_l)) + 7 * (int64_t)(n) + 24) + (int64_t)(n))
typedef struct {
  double* R;                      /* [n_images, 3, 3]: the input bits for an image whose pose did not move */
  double* t;                      /* [n_images, 3] */
  double* points3d;               /* [t_p, 3]: refined for LTR_BA_IN tracks, the input otherwise */
  double* lines3d;                /* [t_l, 2, 3] */
  int32_t* status_p;              /* [t_p] LTR_BA_* */
  int32_t* status_l;              /* [t_l] */
  double* residual_p;             /* [n_kp] a participating row's reprojection error after the adjustment, else NaN */
  double* residual_l;             /* [n_kl] the larger end-point distance of a participating key-line row, else NaN */
  double* row_points3d;           /* [n_kp, 3] as ltr_tracks' rows, under the refined poses */
  double* row_lines3d;            /* [n_kl, 2, 3] */
  int32_t* n_views_p;             /* [n_kp] */
  int32_t* n_views_l;             /* [n_kl] */
  double* stats;                  /* [LTR_BA_STATS] */
  void* workspace;
} LtrBundleOutput;

/* Asynchronous on `stream`; never synchronises.  Errors come before any launch: LTR_E_INVALID for bad arguments,
 * LTR_E_UNSUPPORTED for more than LTR_BA_MAX_IMAGES images.  Three set-up launches, five per iteration (max_iters of
 * them; each returns at once after the stop) and one for the outputs. */
int ltr_bundle_adjust(const LtrBundleInput* in, const LtrBundleOutput* out, int32_t device, void* stream);

/* Global poses of an unposed image set from the relative poses of its pairs (rotation averaging, then BATA camera
 * positions); DESIGN.md "Global poses" states the model:
 *   - view graph: pair p is usable iff valid[p] and n_cheirality[p] >= min_inliers; the component of usable pairs with
 *     the most images (ties: the one holding the lowest image) is registered and anchor < 0 picks its lowest image;
 *     an anchor >= 0 registers its own component instead (the largest one when the caller checked it);
 *   - loop support of a usable pair (i, j): the third images k whose triangle |cayinv(R_ij^T R_kj R_ik)| <= rot_tan
 *     through usable pairs (cayinv(Q) = vee(Q - Q^T) / (1 + tr Q), |cayinv| = tan(theta / 2));
 *   - rotations: Prim's maximum spanning tree from the anchor on (support, n_cheirality, -p), chained, then IRLS on
 *     cayinv(R_j^T R_p R_i) with R_k <- R_k cay(w_k): LTR_GP_L1_ITERS L1 iterations, then Geman-McClure ones (scale
 *     LTR_GP_SIGMA_ROT) while the cost falls, up to rot_iters; a pair is a rotation outlier iff |cayinv| > rot_tan;
 *   - rigidity: images with fewer than two rotation-inlier pairs to kept images, or whose directions are all within
 *     LTR_GP_MIN_ANGLE of parallel, are dropped until none is (not the anchor, not below three images); the images
 *     still connected to the anchor are registered;
 *   - positions (BATA): C_anchor = 0, sum_p <dC_p, v_p> = E (v_p = -R_j^T t_p, E the pairs used), alternating C, the
 *     scales and Geman-McClure weights (scale LTR_GP_SIGMA_POS) up to pos_iters; a pair is a direction outlier iff not
 *     <dC_p, v_p> > dir_cos |dC_p|; t_k = -R_k C_k.
 * Both stages stop after an accepted step whose relative cost decrease is <= ftol.  Every operation is explicitly
 * rounded fp64 in a fixed order, so two calls give the same bits. */
#define LTR_GP_MAX_IMAGES 128
#define LTR_GP_MAX_ITERS 100000
#define LTR_GP_L1_ITERS 5
#define LTR_GP_L1_EPS 1e-9
#define LTR_GP_SIGMA_ROT 0.04366094290851206   /* tan(2.5 deg) */
#define LTR_GP_SIGMA_POS 0.1
#define LTR_GP_MIN_ANGLE 2                      /* degrees; the kernels compare against sin(2 deg) */
#define LTR_GP_EDGE_UNUSED 0                    /* not usable */
#define LTR_GP_EDGE_OUTSIDE 1                   /* usable, but an image is not registered */
#define LTR_GP_EDGE_ROT_OUTLIER 2
#define LTR_GP_EDGE_DIR_OUTLIER 3
#define LTR_GP_EDGE_INLIER 4
#define LTR_GP_STATS 7
typedef struct {
  const int32_t* pairs;           /* device [n_pairs, 2]: image i side 0, image j side 1; no self or repeated pair */
  const double* R;                /* device [n_pairs, 3, 3]: X_j = R_p X_i + t_p (ltr_essential) */
  const double* t;                /* device [n_pairs, 3] unit */
  const uint8_t* valid;           /* device [n_pairs] */
  const int32_t* n_cheirality;    /* device [n_pairs] */
  int32_t n_images;               /* in [1, LTR_GP_MAX_IMAGES] */
  int32_t n_pairs;                /* >= 0 */
  int32_t min_inliers;            /* (20) */
  int32_t anchor;                 /* < 0: the largest component's lowest image; else its own component is registered */
  int32_t rot_iters;              /* in [0, LTR_GP_MAX_ITERS] (100) */
  int32_t pos_iters;              /* in [0, LTR_GP_MAX_ITERS] (500) */
  double rot_tan;                 /* tan(rot_thresh / 2), finite > 0 */
  double dir_cos;                 /* cos(dir_thresh), finite */
  double ftol;                    /* finite, >= 0 (1e-12) */
} LtrGlobalPoseInput;

/* Outputs (device, caller-owned).  R [n_images, 3, 3] and t [n_images, 3] world -> camera, NaN for an image not
 * registered, exactly I and 0 for the anchor; registered uint8 [n_images]; per pair: edge_status int32 (LTR_GP_EDGE_*),
 * support int32 (-1 for a pair not usable), rot_residual fp64 (the final |cayinv(R_j^T R_p R_i)| of the registered
 * component's pairs, NaN elsewhere), dir_cos fp64 (<dC_p, v_p> / |dC_p| of the pairs of the position solve, NaN
 * elsewhere); stats fp64 [LTR_GP_STATS]: rotation iterations and final cost, position iterations and final cost,
 * images registered, inlier pairs, anchor.  workspace: LTR_GP_WORKSPACE_BYTES(n_images, n_pairs) bytes, 8-byte
 * aligned. */
#define LTR_GP_WORKSPACE_BYTES(n, n_pairs) \
  (8 * (16 * (int64_t)(n_pairs) + 24 * (int64_t)(n)) + 4 * (2 * (int64_t)(n) * (n) + 8 * (int64_t)(n) + 16))
typedef struct {
  double* R;
  double* t;
  uint8_t* registered;
  int32_t* edge_status;
  int32_t* support;
  double* rot_residual;
  double* dir_cos;
  double* stats;
  void* workspace;
} LtrGlobalPoseOutput;

/* Asynchronous on `stream`; never synchronises.  Errors come before any launch: LTR_E_INVALID for bad arguments,
 * LTR_E_UNSUPPORTED for more than LTR_GP_MAX_IMAGES images.  Three launches: the view graph (one CTA), the loop support
 * (one CTA per pair; not launched without pairs) and one persistent CTA for the tree, both iterative stages and the
 * outputs. */
int ltr_global_poses(const LtrGlobalPoseInput* in, const LtrGlobalPoseOutput* out, int32_t device, void* stream);

/* Image retrieval (DESIGN.md "Image retrieval"; linetr_b200/retrieval.py is the numpy model of every output bit).
 * Local descriptors are 256-dim fp32 rows of a part (points or lines): layout LTR_LAYOUT_ROWS [n_rows, 256], or
 * LTR_LAYOUT_CHANNEL_FIRST [256, n_i] blocks back to back (image i at 256 * cu[i]); cu [n_images + 1] row offsets.
 * A vocabulary part holds K <= LTR_RT_MAX_CLUSTERS unit fp32 centroids [K, 256]; a global descriptor has
 * D = 256 (K_p + K_l) components.  fp64 is explicitly rounded throughout; two calls give the same bits. */
#define LTR_RT_MAX_CLUSTERS 256
#define LTR_RT_MAX_K 64
/* bound on |screened - exact| score of descriptors of norm <= 1 at dimension D (DESIGN.md "Image retrieval") */
#define LTR_RT_EPS(D) (1e-4 + 3e-8 * (double)(D))

/* One step of spherical k-means over all rows of a part.  With init_rows (device [K]): centroid c = row init_rows[c].
 * Otherwise assign (device [n_rows], each in [0, K), the matcher's nearest centroid) groups the rows, and centroid c
 * becomes fl32(s / sqrt(|s|^2)) for s the fp64 sum of its rows in ascending row order; a cluster without rows (or
 * with |s| = 0) keeps centroids_in[c].  scores (device [n_rows], optional): the matcher's distances, summed into
 * out.cost. */
#define LTR_RT_KMEANS_WORKSPACE_BYTES(n_rows, K) (4 * ((int64_t)(n_rows) + (K) + 1))
typedef struct {
  const float* desc;
  const int32_t* cu;              /* device [n_images + 1] */
  int32_t layout;
  int32_t n_images;
  int32_t n_rows;                 /* = cu[n_images] */
  int32_t K;                      /* in [1, LTR_RT_MAX_CLUSTERS] */
  const float* centroids_in;      /* device [K, 256] */
  const int32_t* assign;
  const float* scores;
  const int32_t* init_rows;
} LtrKmeansInput;

/* centroids [K, 256] (may be centroids_in), centroids_cf [256, K], tiles: the centroids' descriptor tile image
 * (kblocks 4, ceil(K / 128) tiles of 2 x 16 KB; rows past K are not written), counts [K] rows per cluster (0 with
 * init_rows), cost fp64 [1] (written when scores is given), workspace LTR_RT_KMEANS_WORKSPACE_BYTES. */
typedef struct {
  float* centroids;
  float* centroids_cf;
  void* tiles;
  int32_t* counts;
  double* cost;
  void* workspace;
  int64_t workspace_bytes;
} LtrKmeansOutput;

/* Errors before any launch: LTR_E_INVALID for a null pointer, a bad layout or count, n_rows < K with init_rows;
 * LTR_E_UNSUPPORTED for K outside [1, LTR_RT_MAX_CLUSTERS]; LTR_E_WORKSPACE for a short workspace.  Two launches
 * (bucketing, centroids) or one with init_rows; asynchronous on `stream`, never synchronises. */
int ltr_kmeans_update(const LtrKmeansInput* in, const LtrKmeansOutput* out, int32_t device, void* stream);

/* Intra-normalised VLAD of n_images images: per part with K clusters, v_c = sum (x - c) over the image's rows
 * assigned to c (ascending row order, fp64); each v_c of norm > 0 divided by its norm (others 0); the part divided by
 * its norm (when > 0) and multiplied by sqrt(w).  The descriptor is [points part, lines part]. */
#define LTR_RT_VLAD_WORKSPACE_BYTES(n_images, rows_p, rows_l, k_p, k_l) \
  (4 * ((int64_t)(rows_p) + (rows_l) + (int64_t)(n_images) * ((k_p) + (k_l)) + 2))
typedef struct {
  const float* desc_p;
  const int32_t* cu_p;
  int32_t layout_p;
  int32_t rows_p;
  const int32_t* assign_p;        /* device [rows_p] in [0, k_p) */
  const float* centroids_p;       /* device [k_p, 256] */
  int32_t k_p;
  double w_p;                     /* finite, >= 0 */
  const float* desc_l;
  const int32_t* cu_l;
  int32_t layout_l;
  int32_t rows_l;
  const int32_t* assign_l;
  const float* centroids_l;
  int32_t k_l;
  double w_l;
  int32_t n_images;               /* >= 1 */
} LtrVladInput;

/* desc [n_images, D] fp32; tiles: its tile image (kblocks D / 64, ceil(n_images / 128) row tiles, padding rows 0). */
typedef struct {
  float* desc;
  void* tiles;
  void* workspace;
  int64_t workspace_bytes;
} LtrVladOutput;

/* Errors before any launch: LTR_E_INVALID for a null pointer, a bad layout, count or weight; LTR_E_UNSUPPORTED for
 * k_p or k_l outside [1, LTR_RT_MAX_CLUSTERS]; LTR_E_WORKSPACE for a short workspace.  Three launches. */
int ltr_vlad(const LtrVladInput* in, const LtrVladOutput* out, int32_t device, void* stream);

/* Top-k database images of every query by the exact score: the fp64 sum of the products of the fp32 components,
 * lane l of a warp summing components l, l + 32, ... in ascending order, then the xor butterfly 16, 8, 4, 2, 1.
 * Sorted by score descending, ties to the lower index; exclude_self skips database index q for query q.  The GPU
 * screens with a split-bf16 tensor-core product and rescores exactly every candidate within 2 LTR_RT_EPS(D) of the k-th
 * screened score; a query whose tiles may have dropped a candidate there takes an exact pass over all N. */
#define LTR_RT_WORKSPACE_BYTES(Q, N, k) ((int64_t)(Q) * (((int64_t)(N) + 127) / 128) * (8 * (int64_t)(k) + 4))
typedef struct {
  const float* q;                 /* device [Q, D] */
  const void* q_tiles;            /* their tile image (kblocks D / 64) */
  const float* db;                /* device [N, D] */
  const void* db_tiles;
  int32_t Q;                      /* >= 1 */
  int32_t N;                      /* >= 1 */
  int32_t D;                      /* a positive multiple of 64, <= 2 * 256 * LTR_RT_MAX_CLUSTERS */
  int32_t k;                      /* in [1, LTR_RT_MAX_K] */
  int32_t exclude_self;
} LtrRetrieveInput;

/* idx [Q, k] int32 (-1 past the candidates), score [Q, k] fp64 (NaN there), n_full [1] int32: queries that took the
 * full exact pass; workspace LTR_RT_WORKSPACE_BYTES(Q, N, k) bytes. */
typedef struct {
  int32_t* idx;
  double* score;
  int32_t* n_full;
  void* workspace;
  int64_t workspace_bytes;
} LtrRetrieveOutput;

/* Errors before any launch: LTR_E_INVALID for a null pointer or a bad count; LTR_E_UNSUPPORTED for k or D out of range,
 * more than 65535 query tiles; LTR_E_WORKSPACE for a short workspace.  Two launches (screening, merge). */
int ltr_retrieve(const LtrRetrieveInput* in, const LtrRetrieveOutput* out, int32_t device, void* stream);

/* The descriptor tile image of fp32 rows x [n, D] (device; D a positive multiple of 64): kblocks D / 64,
 * ceil(n / 128) row tiles, padding rows 0; LTR_RT_TILES_BYTES(n, D) bytes.  What ltr_retrieve takes for descriptors
 * that do not come from ltr_vlad.  Errors before any launch: LTR_E_INVALID for n < 1, a bad D or a null pointer. */
#define LTR_RT_TILES_BYTES(n, D) (4 * (((int64_t)(n) + 127) / 128) * 128 * (int64_t)(D))
int ltr_rt_tiles(const float* x, int32_t n, int32_t D, void* tiles, int32_t device, void* stream);

/* Homography image pairs <- the warp and valid mask of the homography dataset builder
 * (dataloaders/build_homography_dataset.py:164-184): cv2.warpPerspective of the grey image, and the mask that is 0 where
 * the warped colour image is 0 in every channel, eroded with a 5 x 5 kernel of ones.
 *
 * gray [n_images, height, width] and colour [n_images, height, width, channels] uint8 (device; channels 1 or 3: pass
 * the grey image for grey-only data).  Pair p warps source image src_index[p] with inv_maps[p] (device fp64 [n_pairs,
 * 9], row-major M = inv(H), H mapping image 0 to image 1); src_index_host is the same array in host memory, checked
 * against n_images before any launch.  Outputs (device): warped and mask [n_pairs, height, width] uint8, mask 1 = valid.
 *
 * The warp is OpenCV's fixed-point INTER_LINEAR with BORDER_CONSTANT 0, bit for bit: with bw = min(1024 /
 * min(16, height), width) and output column x = xb + j of the column block xb = x - x % bw, row y:
 *   X0 = M0*xb + M1*y + M2, Y0 = M3*xb + M4*y + M5, W0 = M6*xb + M7*y + M8   (fp64, round to nearest, no FMA)
 *   w = W0 + M6*j;  w = w != 0 ? 32 / w : 0;  X = rint(clamp((X0 + M0*j) * w)), Y = rint(clamp((Y0 + M3*j) * w))
 *   cell (X >> 5, Y >> 5), sub-pixel (fx, fy) = (X & 31, Y & 31); neighbours (0,0) (0,1) (1,0) (1,1) weigh
 *   (32-fx)(32-fy)*32, fx(32-fy)*32, (32-fx)fy*32, fx*fy*32; outside the image they are 0;
 *   pixel = (sum of weight * value + 16384) >> 15.
 * Before the erosion a pixel is valid iff an in-image neighbour with a nonzero weight has a nonzero channel; the 5 x 5
 * erosion counts pixels outside the image as valid.
 *
 * Errors before any launch: LTR_E_INVALID for n_images < 1, n_pairs < 0, a null pointer or a src_index outside
 * [0, n_images); LTR_E_UNSUPPORTED for a side outside [1, 32767] or channels other than 1 and 3.  n_pairs == 0 writes
 * nothing.  Writes only warped and mask; asynchronous on `stream`, never synchronises. */
int ltr_warp_pairs(const uint8_t* gray, const uint8_t* colour, int32_t n_images, int32_t height, int32_t width,
                   int32_t channels, const int32_t* src_index_host, const int32_t* src_index, const double* inv_maps,
                   int32_t n_pairs, uint8_t* warped, uint8_t* mask, int32_t device, void* stream);

/* Photometric augmentation <- imgPhotometric of the homography dataset builder
 * (dataloaders/build_homography_dataset.py:105-121, dataloaders/utils/photometric.py) for the yaml's primitives, on
 * n_images uint8 images [n_images, height, width] (device).  `out` may equal `in` (in place).
 *
 * Per image, params[i * LTR_PHOTOMETRIC_PARAMS + slot] (fp64; params_host is the same array in host memory, checked
 * before any launch):
 *    0- 2  brightness: application count (0-2), integer delta of application 0, of application 1
 *    3- 5  contrast: count, float32 alpha 0, alpha 1        6- 8  Gaussian noise: count, stddev 0, stddev 1
 *    9-11  impulse noise: count, p 0, p 1                   12    motion blur on (1) / off (0)
 *   13-21  the 3 x 3 float32 motion-blur kernel, row-major  22    shade on / off
 *   23     transparency (used as float32)   24  odd Gaussian kernel size <= 149   25, 26  noise key low / high 32 bits
 *   27     number of shade ellipses (<= max_ellipses)
 * ellipses [n_images, max_ellipses, 5] int32 (device): ax, ay, x, y, integer angle in degrees, each inside the image as
 * sample_photometric draws them (max(ax, ay) <= x < width - max(ax, ay), likewise y); others are not drawn.
 * taps [n_images, 149] float32 (device): the first ksize are the image's Gaussian taps.
 *
 * The arithmetic (DESIGN.md "Photometric augmentation"; linetr_b200/photometric.py is its numpy model):
 *   brightness a = clip(a + d); contrast a = trunc(clip(fl32(127.5 + fl32(alpha * fl32(a - 127.5)))));
 *   Gaussian noise a = clip(a + clip(rint(s * z), -255, 255)); impulse noise a = rint(255 sin^2(pi u / 2)) where
 *   u' < p; z, u, u' from Philox4x64-10 with key (key, 0) and counter (y * width + x, application, 0, 0);
 *   motion blur: fp32 FMAs over the kernel in row-major order from 0, BORDER_REFLECT_101, rint and saturate;
 *   shade: cv2.ellipse's filled ellipses into a 0/255 mask, the separable fp32 Gaussian (rows, then columns, each
 *   acc = fl32(acc + fl32(tap_k * v_k)), BORDER_REFLECT_101 reflected as often as needed), then
 *   out = trunc(double(fl32(clip(fl32(x * fl32(1 - fl32(fl32(t * m) / 255))), 0, 255) / 255)) * 255) with
 *   x = fl32(fl32(a / 255) * 255).  Without the shade, out is the stage-1 byte.
 *
 * workspace: device, at least LTR_PHOTOMETRIC_WORKSPACE_BYTES(n_images, height, width) bytes, 256-byte aligned.
 * Errors before any launch: LTR_E_INVALID for a negative count, a null pointer, n_params != LTR_PHOTOMETRIC_PARAMS or
 * a parameter outside the ranges above; LTR_E_UNSUPPORTED for a side outside [1, 32767] or more than 65535 images;
 * LTR_E_WORKSPACE for a short workspace.  n_images == 0 writes nothing.  Writes out and the workspace; asynchronous on
 * `stream`, never synchronises. */
#define LTR_PHOTOMETRIC_PARAMS 28
#define LTR_PHOTOMETRIC_MAX_KSIZE 149
#define LTR_PHOTOMETRIC_WORKSPACE_BYTES(n, h, w) ((int64_t)(n) * (h) * (w) * 6 + 512)
int ltr_photometric(const uint8_t* in, uint8_t* out, int32_t n_images, int32_t height, int32_t width,
                    const double* params_host, const double* params, int32_t n_params, const int32_t* ellipses,
                    int32_t max_ellipses, const float* taps, void* workspace, int64_t workspace_bytes, int32_t device,
                    void* stream);

/* Row-major linear layer Y = act(X W^T + b) (+ R) on the tensor-core engine (gemm_img.cuh:
 * persistent, TMA-fed split-bf16 tile images, wgmma), exported so the engine can be unit-tested in
 * isolation; act: 0 none, 1 relu, 2 gelu(erf).  x is converted to a split-bf16 tile image, the GEMM writes fp32 rows into `y` (may be NULL) and - when
 * `y_from_image` is given - also the split-bf16 image of the result, which is converted back
 * to fp32 rows [m, n] there so that both outputs can be checked.  n % 64 == 0, k % 64 == 0;
 * bn_hint: 0 (auto), 64, 128 or 256.  Synchronous; unit-test hook only. */
int ltr_linear_img(const float* x, int32_t ldx, const float* w_host, const float* bias,
                   const float* res, int32_t ldr, float* y, int32_t ldy, float* y_from_image,
                   int32_t m, int32_t n, int32_t k, int32_t act, int32_t bn_hint, int32_t device,
                   void* stream);

/* ltr_linear_img with the row-normalising epilogue the encoder uses (n = 256 fixed): norm = 1:
 * y = LayerNorm(x W^T + b (+ res); eps) * gamma + beta (+ add)   - MultiHeadAttention / FeedForward
 * tails, models/line_attention.py:51-53,73-75, plus the `klines_pos +` of models/line_transformer.py:128;
 * norm = 2: y = (x W^T + b) / max(||.||_2, 1e-12)               - final_proj + F.normalize,
 * models/line_transformer.py:245-246.  Synchronous; unit-test hook only. */
int ltr_linear_img_norm(const float* x, int32_t ldx, const float* w_host, const float* bias,
                        const float* res, int32_t ldr, int32_t norm, float eps, const float* gamma,
                        const float* beta, const float* add, int32_t ldadd, float* y, int32_t ldy,
                        float* y_from_image, int32_t m, int32_t k, int32_t device, void* stream);

/* Instrumentation.  Kernel launches issued by this library since the last reset: one count per kernel
 * launch, those of the debug hooks (include/linetr_b200_debug.h) included.  A launch that fails is not
 * counted. */
int64_t ltr_launch_count(void);
void ltr_reset_launch_count(void);
/* Per-kernel-class device timing with CUDA events on the launching stream, one event pair around each
 * kernel launch.  ltr_profile_begin() arms it; ltr_profile_end() synchronises, fills `names` (pointers to
 * static strings), `ms` (summed elapsed per class) and `launches` (one per kernel launch issued, debug
 * hooks included, in class "debug" unless they run a production kernel; failed launches are not counted),
 * returns the class count. */
void ltr_profile_begin(void);
int ltr_profile_end(const char** names, float* ms, int32_t* launches, int32_t max_classes);

const char* ltr_last_error(void);
int ltr_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* LINETR_B200_H_ */
