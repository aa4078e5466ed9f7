/*
 * linetr_b200 - debug / micro-benchmark hooks of the CUDA library.  NOT part of the drop-in
 * boundary (include/linetr_b200.h); used by tools/ and the engine unit tests only.
 */
#ifndef LINETR_B200_DEBUG_H_
#define LINETR_B200_DEBUG_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Micro-benchmark of the image-operand GEMM engine (zero-filled operands, timing only):
 * average device milliseconds per launch.  out_mode: 0 fp32 rows, 1 image, 2 both. */
float ltr_gemm_bench(int32_t m, int32_t n, int32_t k, int32_t bn_hint, int32_t out_mode, int32_t iters,
                     int32_t device);

/* One signature layer's row-local GEMMs (mlp1 ReLU -> mlp2 + x -> qkv) at m rows, zero-filled operands:
 * average device milliseconds per layer as one chained launch (chained != 0) or three launches.
 * -1 on failure. */
float ltr_gemm_chain_bench(int32_t m, int32_t chained, int32_t iters, int32_t device);

/* Kernels instrumented with LTR_DBG_STAMP store clock64 stamps of their first CTA into a
 * 128-slot device array while tracing is armed.  gemm_img_kernel (as ltr_gemm_bench launches it)
 * stamps the first 4 tiles of CTA 0, 16 slots per tile, slot 16 * i + j: j = 0 consumers start tile i,
 * 2 its MMAs are done, 5 its epilogue is done; j = 6 the producer got a ring slot for its i-th k-block
 * (counted across tiles).  gemm_chain_kernel's layout is CHAIN_TRACE_* in csrc/gemm_img.cuh. */
void ltr_debug_trace_arm(int32_t on);
int ltr_debug_trace_read(unsigned long long* out128);

/* Where ltr_encode leaves each stage's activation in `workspace` (the pointer given to ltr_encode) for a batch of
 * n_lines lines, so that tests can read every stage's real inputs and outputs after an encode.  Slot i of hi / lo /
 * kblocks: 0 z, 1 ctx, 2 l128, 3 l256, 4 lpos, 5 y1i, 6 g, 7 xm, 8 hm, 9 qkv: split-bf16 activation images (hi and lo
 * planes, kblocks 64-wide k-blocks per 128-row block); 10 yf: fp32 rows [n_lines, 256] in hi, lo = NULL, kblocks 0.
 * Returns 0, or LTR_E_INVALID on a null argument. */
/* ltr_linear_img with its residual read from a split-bf16 image: res [m, n] (device, row stride n) is split into an
 * image first, and the GEMM adds hi + lo of it after the activation, as mlp2's x += delta does.  y_from_image given:
 * the output image is written in place over the residual image (y must be NULL), then read back as hi + lo.  Else y
 * gets the fp32 rows.  Test hook of the two image-residual epilogues. */
int ltr_debug_linear_img_res(const float* x, int32_t ldx, const float* w_host, const float* bias, const float* res,
                             float* y, float* y_from_image, int32_t m, int32_t n, int32_t k, int32_t act,
                             int32_t bn_hint, int32_t device, void* stream);

int ltr_debug_encode_images(const struct LtrModel* model, int32_t n_lines, void* workspace, void* hi[11], void* lo[11],
                            int32_t kblocks[11]);

/* `launches` back-to-back signature-attention launches as ltr_encode issues them for n_images images of 128 lines
 * (uniform batch): qkv image (12 k-blocks per 128-row block, hi / lo planes, device) -> columns 256..511 of an
 * 8-k-block output image.  The kernel is chosen as an encode chooses it, LTR_ATTN_PIPE included.  Returns 0, LTR_E_INVALID on a
 * bad argument, or the launch error. */
int ltr_debug_sig_attention(const void* qkv_hi, const void* qkv_lo, void* out_hi, void* out_lo, int32_t n_images,
                            int32_t launches, void* stream);

/* The relative-pose estimator's fp64 root finder on its own, one thread per polynomial: poly [n, 11] ascending
 * coefficients (device) -> roots [n, 10] ascending, NaN past the count, and count [n] (device).  The estimator's own
 * __device__ function (Sturm chain and bisection). */
int ltr_debug_sturm_roots(const double* poly, int32_t n, double* roots, int32_t* count, int32_t device, void* stream);

/* The estimator's five-point solver on its own, one thread per sample: q [n, 5, 4] normalised correspondences
 * (a0, b0, a1, b1; device) -> E [n, 10, 9] row-major, root_index [n, 10] (the real root each solution came from) and
 * n_solutions [n] (device); entries past n_solutions are NaN / -1.  The same compiled function the estimator runs. */
int ltr_debug_essential_solve(const double* q, int32_t n, double* E, int32_t* root_index, int32_t* n_solutions,
                              int32_t device, void* stream);

/* The fundamental-matrix estimator's seven-point solver on its own, one thread per sample: q [n, 7, 4] normalised
 * correspondences (x0, y0, x1, y1; device) -> F [n, 3, 9] normalised F^ row-major, root_index [n, 3] (the real root of
 * the cubic each solution came from) and n_solutions [n] (device); entries past n_solutions are NaN / -1.  The same
 * compiled function the estimator runs. */
int ltr_debug_fundamental_solve(const double* q, int32_t n, double* F, int32_t* root_index, int32_t* n_solutions,
                                int32_t device, void* stream);

/* The absolute-pose estimator's P3P solver on its own, one thread per sample: j [n, 3, 3] unit bearings and X [n, 3, 3]
 * world points of the sample's three points (device) -> R [n, 4, 9] row-major, t [n, 4, 3] (X_cam = R X + t),
 * root_index [n, 4] (the real root of the quartic each pose came from) and n_solutions [n] (device); entries past
 * n_solutions are NaN / -1.  The same compiled function the estimator runs. */
int ltr_debug_p3p(const double* j, const double* X, int32_t n, double* R, double* t, int32_t* root_index,
                  int32_t* n_solutions, int32_t device, void* stream);

/* The absolute-pose estimator's line solvers on their own, one thread per sample of solver 0 (P2P1L), 1 (P1P2L) or 2
 * (P3L): j and X [count, 2 - solver, 3] unit bearings and world points of the sample's points (NULL for P3L), n
 * [count, solver + 1, 3] camera-ray normals of its query lines and E [count, solver + 1, 2, 3] the world end points
 * of its lines (device) -> R [count, 8, 9] row-major, t [count, 8, 3] (X_cam = R X + t), root_index [count, 8] (the
 * real root of the degree-8 polynomial each pose came from) and n_solutions [count] (device); entries past
 * n_solutions are NaN / -1.  The same compiled function the estimator runs. */
int ltr_debug_line_pose(int32_t solver, const double* j, const double* X, const double* n, const double* E, int32_t count,
                        double* R, double* t, int32_t* root_index, int32_t* n_solutions, int32_t device, void* stream);

/* The fundamental-matrix estimator's line check on its own, one thread per key-line pair: F [n, 9] pixel F (row-major,
 * fp64), s0 / s1 [n, 4] the matched segments (a, b; fp32) -> r1 [n] (the overlap ratio in image 1), r0 [n] (in
 * image 0; NaN where the side cannot reject) and ok [n] (1 iff consistent at min_overlap in [0, 1]; device).  The same
 * compiled functions the fit kernel runs. */
int ltr_debug_fundamental_lines(const double* F, const float* s0, const float* s1, int32_t n, double min_overlap,
                                double* r1, double* r0, uint8_t* ok, int32_t device, void* stream);

/* The pose stages' dense SPD solver (rc_cholesky_solve) on its own, one 1024-thread CTA per system, the instantiation
 * ba_solve_kernel and gp_solve_kernel run: A [n, m, ld] (its lower triangle read, L written over it) and the
 * right-hand sides x [n, m, k] (device), solved in place; ok [n] (device) is 1, or 0 at the first pivot that is not
 * > 0, with x untouched.  shared = 1 copies A (m <= 127) and x into dynamic shared memory first, as gp_solve_kernel
 * keeps them; shared = 0 works in place in global memory with leading dimension ld, as ba_solve_kernel does.  Returns
 * 0, or LTR_E_INVALID before any launch unless 0 <= m <= 1024 (<= 127 when shared), 1 <= k <= 6, ld >= m, shared
 * is 0 or 1, and (n > 0) ok and (m > 0) A and x are given. */
int ltr_debug_cholesky_solve(double* A, int32_t n, int32_t m, int32_t ld, double* x, int32_t k, int32_t shared,
                             uint8_t* ok, int32_t device, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LINETR_B200_DEBUG_H_ */
