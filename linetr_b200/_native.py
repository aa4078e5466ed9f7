"""ctypes binding of the C-ABI CUDA library (include/linetr_b200.h).

There is no fallback: if the shared library has not been built
(`python -c "import __graft_entry__ as g; g.build()"` or tools/build_native.sh)
importing the compute entry points raises, and every call raises on a non-zero return code.
"""
from __future__ import annotations

import ctypes as C
import os

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "liblinetr_b200.so")
_lib = None

c_float_p = C.POINTER(C.c_float)
c_int32_p = C.POINTER(C.c_int32)

LAYOUT_ROWS = 0
LAYOUT_CHANNEL_FIRST = 1

# slots of ltr_debug_encode_images, in order
ENCODE_IMAGES = ("z", "ctx", "l128", "l256", "lpos", "y1i", "g", "xm", "hm", "qkv", "yf")
ABI_VERSION = 4
PHOTOMETRIC_PARAMS = 28      # LTR_PHOTOMETRIC_PARAMS
PHOTOMETRIC_MAX_KSIZE = 149  # LTR_PHOTOMETRIC_MAX_KSIZE
TRI_MAX_VIEWS = 64           # LTR_TRI_MAX_VIEWS
TRK_MAX_OBS = 64             # LTR_TRK_MAX_OBS
TRK_OK, TRK_TOO_LONG, TRK_NO_CANDIDATE, TRK_TOO_FEW = 0, 1, 2, 3   # LTR_TRK_OK .. LTR_TRK_TOO_FEW
BA_MAX_IMAGES = 128          # LTR_BA_MAX_IMAGES
BA_MAX_ITERS = 1000          # LTR_BA_MAX_ITERS
BA_IN, BA_NOT_VALID, BA_SAME_IMAGE, BA_DEGENERATE = 0, 1, 2, 3     # LTR_BA_IN .. LTR_BA_DEGENERATE
BA_STOP_ITERS, BA_STOP_FTOL, BA_STOP_LAMBDA = 0, 1, 2              # LTR_BA_STOP_ITERS .. LTR_BA_STOP_LAMBDA
BA_STATS = 8                 # LTR_BA_STATS
GP_MAX_IMAGES = 128          # LTR_GP_MAX_IMAGES
GP_EDGE_UNUSED, GP_EDGE_OUTSIDE, GP_EDGE_ROT_OUTLIER, GP_EDGE_DIR_OUTLIER, GP_EDGE_INLIER = 0, 1, 2, 3, 4   # LTR_GP_EDGE_*
GP_STATS = 7                 # LTR_GP_STATS
RT_MAX_CLUSTERS = 256        # LTR_RT_MAX_CLUSTERS
RT_MAX_K = 64                # LTR_RT_MAX_K


def ba_workspace_bytes(n_images, n_kp, n_kl, t_p, t_l) -> int:
    """LTR_BA_WORKSPACE_BYTES(n_images, n_kp, n_kl, t_p, t_l)."""
    n, rows, trk = int(n_images), int(n_kp) + int(n_kl), int(t_p) + int(t_l)
    return 8 * (64 * rows + 40 * trk + 36 * n * n + 60 * n + 16) + 4 * (2 * rows + 4 * trk + 7 * n + 24) + n


def gp_workspace_bytes(n_images, n_pairs) -> int:
    """LTR_GP_WORKSPACE_BYTES(n_images, n_pairs)."""
    n, P = int(n_images), int(n_pairs)
    return 8 * (16 * P + 24 * n) + 4 * (2 * n * n + 8 * n + 16)


def rt_kmeans_workspace_bytes(n_rows, K) -> int:
    """LTR_RT_KMEANS_WORKSPACE_BYTES(n_rows, K)."""
    return 4 * (int(n_rows) + int(K) + 1)


def rt_vlad_workspace_bytes(n_images, rows_p, rows_l, k_p, k_l) -> int:
    """LTR_RT_VLAD_WORKSPACE_BYTES(n_images, rows_p, rows_l, k_p, k_l)."""
    return 4 * (int(rows_p) + int(rows_l) + int(n_images) * (int(k_p) + int(k_l)) + 2)


def rt_eps(D) -> float:
    """LTR_RT_EPS(D)."""
    return 1e-4 + 3e-8 * float(D)


def rt_workspace_bytes(Q, N, k) -> int:
    """LTR_RT_WORKSPACE_BYTES(Q, N, k)."""
    return int(Q) * ((int(N) + 127) // 128) * (8 * int(k) + 4)


def photometric_workspace_bytes(n, h, w) -> int:
    """LTR_PHOTOMETRIC_WORKSPACE_BYTES(n, h, w)."""
    return int(n) * int(h) * int(w) * 6 + 512


class LtrError(RuntimeError):
    pass


class _Tag:
    """A `[const] T*` field of a struct mirror: ctypes passes it as C.c_void_p, `_typed` records T."""

    def __init__(self, pointee):
        self.pointee = pointee


F32P, F64P, I32P, U8P, U64P = (_Tag(t) for t in (C.c_float, C.c_double, C.c_int32, C.c_uint8, C.c_uint64))


def _typed(fields):
    """(_fields_, _pointees_) of a struct mirror from its fields with tagged pointers: every field the header declares
    `[const] T*` (T float, double, int32_t, uint8_t or uint64_t) is a tag, and goes into _fields_ as C.c_void_p, so
    it takes an address as an int or None; _pointees_ {field: ctypes T} is what tests/test_abi.py holds to the header
    and _ops.call_struct holds a tensor's dtype to."""
    return ([(nm, C.c_void_p if isinstance(t, _Tag) else t) for nm, t in fields],
            {nm: t.pointee for nm, t in fields if isinstance(t, _Tag)})


class LtrTensor(C.Structure):
    _fields_, _pointees_ = _typed([
        ("name", C.c_char_p), ("data", F32P), ("numel", C.c_int64)])


class LtrConfig(C.Structure):
    _fields_ = [("d_model", C.c_int32), ("n_heads", C.c_int32), ("d_inner", C.c_int32),
                ("n_desc_layers", C.c_int32), ("n_sig_layers", C.c_int32)]


class LtrEncodeInput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("sublines", F32P), ("resp", F32P), ("angle", F32P), ("pnt", F32P), ("desc", F32P), ("score", F32P),
        ("cu_lines_host", I32P), ("cu_lines_dev", I32P), ("n_images", C.c_int32), ("n_lines", C.c_int32),
        ("n_tokens", C.c_int32), ("lines_per_image", C.c_int32), ("image_width", C.c_float),
        ("image_height", C.c_float)])


class LtrEncodeOutput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("desc_cf", F32P), ("desc_rows", F32P), ("desc_tiles", C.c_void_p)])


class LtrMatchInput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("desc0", F32P), ("desc1", F32P), ("layout", C.c_int32), ("d", C.c_int32), ("n_pairs", C.c_int32),
        ("n0", C.c_int32), ("n1", C.c_int32), ("cu0", I32P), ("cu1", I32P), ("sub_off0", I32P), ("sub_off1", I32P),
        ("cuk0", I32P), ("cuk1", I32P), ("max_n0", C.c_int32), ("max_n1", C.c_int32), ("max_k0", C.c_int32),
        ("max_k1", C.c_int32), ("dist_pair_stride", C.c_int64), ("nn_thresh", C.c_float), ("mutual", C.c_int32),
        ("total_n0", C.c_int32), ("total_n1", C.c_int32), ("dist_mode", C.c_int32), ("tiles0", C.c_void_p),
        ("tiles1", C.c_void_p), ("tiles_lines0", C.c_int32), ("tiles_lines1", C.c_int32), ("tiles_row0_0", C.c_int32),
        ("tiles_row0_1", C.c_int32)])


class LtrPairIndex(C.Structure):
    _fields_, _pointees_ = _typed([
        ("img0", I32P), ("img1", I32P), ("tiles0", C.c_void_p), ("tiles1", C.c_void_p), ("tile_off0", I32P),
        ("tile_off1", I32P), ("n_tiles0", C.c_int32), ("n_tiles1", C.c_int32), ("out_off0", I32P), ("out_off1", I32P),
        ("total_out0", C.c_int32), ("total_out1", C.c_int32)])


GATHER_SLOTS = 8


class LtrPeerGather(C.Structure):
    _fields_ = [("mc_base", C.c_void_p), ("peer_bases", C.c_void_p), ("rank", C.c_int32), ("world", C.c_int32),
                ("slot", C.c_int32), ("epoch", C.c_int32)]


class LtrMatchOutput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("matches0", I32P), ("scores0", F32P), ("nn1", I32P), ("counts", I32P), ("dist_key", F32P), ("dist_sub", F32P),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64), ("gather", C.POINTER(LtrPeerGather))])


class LtrTokenizeImage(C.Structure):
    _fields_, _pointees_ = _typed([
        ("dense_desc", F32P), ("dense_score", F32P), ("token_distance", C.c_double), ("desc_h", C.c_int32),
        ("desc_w", C.c_int32), ("score_h", C.c_int32), ("score_w", C.c_int32)])


class LtrTokenizeBatchInput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("sp", F64P), ("ep", F64P), ("ep_clipped", F64P), ("length", F64P), ("angle", F32P), ("n_tok", I32P),
        ("sub0", I32P), ("sub2line", I32P), ("line_image", I32P), ("n_images", C.c_int32), ("n_keylines", C.c_int32),
        ("n_sublines", C.c_int32), ("n_tokens", C.c_int32), ("desc_channels", C.c_int32), ("align_corners", C.c_int32),
        ("images", C.POINTER(LtrTokenizeImage)), ("cu_sublines", c_int32_p)])


class LtrLineGtInput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("segs0", F32P), ("segs1", F32P), ("cu0", I32P), ("cu1", I32P), ("homography", F64P), ("homography_inv", F64P),
        ("proj0", F32P), ("proj1", F32P), ("pred0", I32P), ("n_pairs", C.c_int32), ("max_n0", C.c_int32),
        ("max_n1", C.c_int32), ("thres_reprojected", C.c_float), ("thres_angdiff", C.c_double),
        ("min_overlap_ratio", C.c_double)])


class LtrLineGtOutput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("assign", F32P), ("assign_stride", C.c_int64), ("n_gt", I32P), ("tfpn", I32P)])


class LtrTripletInput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("desc0", F32P), ("desc1", F32P), ("layout", C.c_int32), ("d", C.c_int32), ("n_pairs", C.c_int32),
        ("n0", C.c_int32), ("n1", C.c_int32), ("cu0", I32P), ("cu1", I32P), ("max_n0", C.c_int32),
        ("max_n1", C.c_int32), ("assign", F32P), ("assign_stride", C.c_int64), ("assign_ld", C.c_int32),
        ("match_thr", C.c_double), ("unmatch_thr", C.c_double), ("pred0", I32P), ("n_groups", C.c_int32),
        ("group_off", I32P)])


class LtrTripletOutput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("pos", F32P), ("neg", F32P), ("state", I32P), ("loss", F32P), ("hardest_pos", F32P), ("hardest_neg", F32P),
        ("n_valid", I32P), ("tfpn", I32P)])


class LtrHomographyInput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("pts0", F32P), ("pts1", F32P), ("pts_off0", I32P), ("pts_off1", I32P), ("n_pts1", I32P), ("matches_p", I32P),
        ("cu_p", I32P), ("segs0", F32P), ("segs1", F32P), ("seg_off0", I32P), ("seg_off1", I32P), ("n_segs1", I32P),
        ("matches_l", I32P), ("cu_l", I32P), ("n_pairs", C.c_int32), ("max_rows_p", C.c_int32),
        ("max_rows_l", C.c_int32), ("thresh", C.c_double), ("n_hypotheses", C.c_int32), ("seed", C.c_uint64),
        ("use_points", C.c_int32), ("use_lines", C.c_int32)])


class LtrHomographyOutput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("H", F64P), ("valid", U8P), ("inliers_p", U8P), ("inliers_l", U8P), ("n_inliers_p", I32P),
        ("n_inliers_l", I32P), ("hypothesis", I32P), ("hypothesis_inliers", I32P), ("key", U64P)])


class LtrEssentialInput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("pts0", F32P), ("pts1", F32P), ("pts_off0", I32P), ("pts_off1", I32P), ("n_pts1", I32P), ("matches_p", I32P),
        ("cu_p", I32P), ("K0", F64P), ("K1", F64P), ("n_pairs", C.c_int32), ("max_rows_p", C.c_int32),
        ("thresh", C.c_double), ("dist_thresh", C.c_double), ("n_hypotheses", C.c_int32), ("seed", C.c_uint64)])


class LtrEssentialOutput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("E", F64P), ("R", F64P), ("t", F64P), ("valid", U8P), ("inliers_p", U8P), ("n_inliers", I32P),
        ("n_cheirality", I32P), ("hypothesis", I32P), ("hypothesis_inliers", I32P), ("key", U64P)])


class LtrFundamentalInput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("pts0", F32P), ("pts1", F32P), ("pts_off0", I32P), ("pts_off1", I32P), ("n_pts1", I32P), ("matches_p", I32P),
        ("cu_p", I32P), ("segs0", F32P), ("segs1", F32P), ("seg_off0", I32P), ("seg_off1", I32P), ("n_segs1", I32P),
        ("matches_l", I32P), ("cu_l", I32P), ("n_pairs", C.c_int32), ("max_rows_p", C.c_int32),
        ("max_rows_l", C.c_int32), ("thresh", C.c_double), ("min_overlap", C.c_double), ("n_hypotheses", C.c_int32),
        ("seed", C.c_uint64)])


class LtrFundamentalOutput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("F", F64P), ("valid", U8P), ("refit", U8P), ("inliers_p", U8P), ("lines_consistent", U8P), ("n_inliers", I32P),
        ("n_lines_consistent", I32P), ("hypothesis", I32P), ("hypothesis_inliers", I32P), ("key", U64P)])


class LtrAbsPoseInput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("pts0", F32P), ("pts_off0", I32P), ("matches_p", I32P), ("cu_p", I32P), ("X1", F64P), ("x_off1", I32P),
        ("n_x1", I32P), ("segs0", F32P), ("seg_off0", I32P), ("matches_l", I32P), ("cu_l", I32P), ("L1", F64P),
        ("l_off1", I32P), ("n_l1", I32P), ("groups", I32P), ("K0", F64P), ("n_pairs", C.c_int32),
        ("n_groups", C.c_int32), ("max_rows_p", C.c_int32), ("max_rows_l", C.c_int32), ("thresh", C.c_double),
        ("n_hypotheses", C.c_int32), ("seed", C.c_uint64), ("use_lines", C.c_int32)])


class LtrAbsPoseOutput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("R", F64P), ("t", F64P), ("valid", U8P), ("refit", U8P), ("inliers_p", U8P), ("inliers_l", U8P),
        ("n_inliers_p", I32P), ("n_inliers_l", I32P), ("hypothesis", I32P), ("hypothesis_inliers", I32P),
        ("key", U64P)])


class LtrTriangulateInput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("kpts", F32P), ("kp_off", I32P), ("segs", F32P), ("seg_off", I32P), ("K", F64P), ("R", F64P), ("t", F64P),
        ("pairs", I32P), ("matches_p", I32P), ("cu_p", I32P), ("matches_l", I32P), ("cu_l", I32P), ("views", I32P),
        ("view_off", I32P), ("block_off", I32P), ("inv_off_p", I32P), ("inv_off_l", I32P), ("n_images", C.c_int32),
        ("n_pairs", C.c_int32), ("total_p", C.c_int32), ("total_l", C.c_int32), ("n_inv_p", C.c_int32),
        ("n_inv_l", C.c_int32), ("n_blocks", C.c_int32), ("max_views", C.c_int32), ("thresh", C.c_double),
        ("min_angle", C.c_double), ("min_views", C.c_int32)])


class LtrTriangulateOutput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("points3d", F64P), ("lines3d", F64P), ("n_views_p", I32P), ("n_views_l", I32P), ("inv_p", I32P),
        ("inv_l", I32P)])


class LtrTracksInput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("kpts", F32P), ("kp_off", I32P), ("segs", F32P), ("seg_off", I32P), ("K", F64P), ("R", F64P), ("t", F64P),
        ("F", F64P), ("pairs", I32P), ("matches_p", I32P), ("cu_p", I32P), ("matches_l", I32P), ("cu_l", I32P),
        ("n_images", C.c_int32), ("n_pairs", C.c_int32), ("total_p", C.c_int32), ("total_l", C.c_int32),
        ("n_kp", C.c_int32), ("n_kl", C.c_int32), ("thresh", C.c_double), ("min_angle", C.c_double),
        ("min_views", C.c_int32), ("epi_thresh", C.c_double), ("min_overlap", C.c_double)])


class LtrTracksOutput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("track_p", I32P), ("track_l", I32P), ("n_tracks_p", I32P), ("n_tracks_l", I32P), ("track_off_p", I32P),
        ("track_off_l", I32P), ("obs_p", I32P), ("obs_l", I32P), ("points3d", F64P), ("lines3d", F64P),
        ("n_obs_p", I32P), ("n_obs_l", I32P), ("n_inliers_p", I32P), ("n_inliers_l", I32P), ("n_images_p", I32P),
        ("n_images_l", I32P), ("status_p", I32P), ("status_l", I32P), ("inlier_p", U8P), ("inlier_l", U8P),
        ("row_points3d", F64P), ("row_lines3d", F64P), ("n_views_p", I32P), ("n_views_l", I32P), ("workspace", I32P)])


class LtrBundleInput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("kpts", F32P), ("kp_off", I32P), ("segs", F32P), ("seg_off", I32P), ("K", F64P), ("R", F64P), ("t", F64P),
        ("hold", I32P), ("fixed", I32P), ("n_tracks_p", I32P), ("n_tracks_l", I32P), ("track_off_p", I32P),
        ("track_off_l", I32P), ("obs_p", I32P), ("obs_l", I32P), ("status_p", I32P), ("status_l", I32P),
        ("inlier_p", U8P), ("inlier_l", U8P), ("track_p", I32P), ("track_l", I32P), ("n_views_p", I32P),
        ("n_views_l", I32P), ("points3d", F64P), ("lines3d", F64P), ("n_images", C.c_int32), ("n_fixed", C.c_int32),
        ("n_kp", C.c_int32), ("n_kl", C.c_int32), ("t_p", C.c_int32), ("t_l", C.c_int32), ("max_iters", C.c_int32),
        ("ftol", C.c_double)])


class LtrBundleOutput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("R", F64P), ("t", F64P), ("points3d", F64P), ("lines3d", F64P), ("status_p", I32P), ("status_l", I32P),
        ("residual_p", F64P), ("residual_l", F64P), ("row_points3d", F64P), ("row_lines3d", F64P), ("n_views_p", I32P),
        ("n_views_l", I32P), ("stats", F64P), ("workspace", C.c_void_p)])


class LtrGlobalPoseInput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("pairs", I32P), ("R", F64P), ("t", F64P), ("valid", U8P), ("n_cheirality", I32P), ("n_images", C.c_int32),
        ("n_pairs", C.c_int32), ("min_inliers", C.c_int32), ("anchor", C.c_int32), ("rot_iters", C.c_int32),
        ("pos_iters", C.c_int32), ("rot_tan", C.c_double), ("dir_cos", C.c_double), ("ftol", C.c_double)])


class LtrGlobalPoseOutput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("R", F64P), ("t", F64P), ("registered", U8P), ("edge_status", I32P), ("support", I32P), ("rot_residual", F64P),
        ("dir_cos", F64P), ("stats", F64P), ("workspace", C.c_void_p)])


class LtrKmeansInput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("desc", F32P), ("cu", I32P), ("layout", C.c_int32), ("n_images", C.c_int32), ("n_rows", C.c_int32),
        ("K", C.c_int32), ("centroids_in", F32P), ("assign", I32P), ("scores", F32P), ("init_rows", I32P)])


class LtrKmeansOutput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("centroids", F32P), ("centroids_cf", F32P), ("tiles", C.c_void_p), ("counts", I32P), ("cost", F64P),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64)])


class LtrVladInput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("desc_p", F32P), ("cu_p", I32P), ("layout_p", C.c_int32), ("rows_p", C.c_int32), ("assign_p", I32P),
        ("centroids_p", F32P), ("k_p", C.c_int32), ("w_p", C.c_double), ("desc_l", F32P), ("cu_l", I32P),
        ("layout_l", C.c_int32), ("rows_l", C.c_int32), ("assign_l", I32P), ("centroids_l", F32P), ("k_l", C.c_int32),
        ("w_l", C.c_double), ("n_images", C.c_int32)])


class LtrVladOutput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("desc", F32P), ("tiles", C.c_void_p), ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64)])


class LtrRetrieveInput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("q", F32P), ("q_tiles", C.c_void_p), ("db", F32P), ("db_tiles", C.c_void_p), ("Q", C.c_int32),
        ("N", C.c_int32), ("D", C.c_int32), ("k", C.c_int32), ("exclude_self", C.c_int32)])


class LtrRetrieveOutput(C.Structure):
    _fields_, _pointees_ = _typed([
        ("idx", I32P), ("score", F64P), ("n_full", I32P), ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64)])


_P, _I32, _I64, _F32, _ptr = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.POINTER
# {name: (restype, argtypes)} of every function include/linetr_b200.h declares (tests check the library exports all
# of them, and each entry against its C prototype)
PROTOTYPES = {
    "ltr_abi_version": (C.c_int, []),
    "ltr_last_error": (C.c_char_p, []),
    "ltr_create": (C.c_int, [_ptr(LtrTensor), _I32, _ptr(LtrConfig), _I32, _ptr(_P)]),
    "ltr_destroy": (None, [_P]),
    "ltr_encode_workspace_bytes": (_I64, [_P, _I32, _I32, _I32]),
    "ltr_desc_tiles_bytes": (_I64, [_I32]),
    "ltr_encode": (C.c_int, [_P, _ptr(LtrEncodeInput), _ptr(LtrEncodeOutput), _P, _I64, _P]),
    "ltr_match_workspace_bytes": (_I64, [_ptr(LtrMatchInput)]),
    "ltr_match": (C.c_int, [_ptr(LtrMatchInput), _ptr(LtrMatchOutput), _I32, _P]),
    "ltr_gather_wait": (C.c_int, [_P, _I32, _I32, _I32, _I32, _P, _I32, _P]),
    "ltr_image_tiles_bytes": (_I64, [_I32, c_int32_p]),
    "ltr_image_tiles": (C.c_int, [_P, _I32, _P, _P, _I32, _I32, _I32, _P, _I32, _P]),
    "ltr_match_indexed_workspace_bytes": (_I64, [_ptr(LtrMatchInput), _ptr(LtrPairIndex)]),
    "ltr_match_indexed": (C.c_int, [_ptr(LtrMatchInput), _ptr(LtrPairIndex), _ptr(LtrMatchOutput), _I32, _P]),
    "ltr_match_distmat": (C.c_int, [_P, _I32, _I32, _I32, _I64, _F32, _I32, _P, _P, _P, _P, _I32, _P]),
    "ltr_merge_sublines": (C.c_int, [_P, _I64, _I32, _P, _P, _P, _P, _I32, _I32, _P, _I64, _I32, _P]),
    "ltr_tokenize_batch": (C.c_int, [_ptr(LtrTokenizeBatchInput)] + [_P] * 7 + [_I32, _P]),
    "ltr_line_gt": (C.c_int, [_ptr(LtrLineGtInput), _ptr(LtrLineGtOutput), _I32, _P]),
    "ltr_triplet_loss": (C.c_int, [_ptr(LtrTripletInput), _ptr(LtrTripletOutput), _I32, _P]),
    "ltr_homography": (C.c_int, [_ptr(LtrHomographyInput), _ptr(LtrHomographyOutput), _I32, _P]),
    "ltr_essential": (C.c_int, [_ptr(LtrEssentialInput), _ptr(LtrEssentialOutput), _I32, _P]),
    "ltr_fundamental": (C.c_int, [_ptr(LtrFundamentalInput), _ptr(LtrFundamentalOutput), _I32, _P]),
    "ltr_absolute_pose": (C.c_int, [_ptr(LtrAbsPoseInput), _ptr(LtrAbsPoseOutput), _I32, _P]),
    "ltr_absolute_pose_lines": (C.c_int, [_ptr(LtrAbsPoseInput), _ptr(LtrAbsPoseOutput), _I32, _I32, _P]),
    "ltr_triangulate": (C.c_int, [_ptr(LtrTriangulateInput), _ptr(LtrTriangulateOutput), _I32, _P]),
    "ltr_tracks": (C.c_int, [_ptr(LtrTracksInput), _ptr(LtrTracksOutput), _I32, _P]),
    "ltr_bundle_adjust": (C.c_int, [_ptr(LtrBundleInput), _ptr(LtrBundleOutput), _I32, _P]),
    "ltr_global_poses": (C.c_int, [_ptr(LtrGlobalPoseInput), _ptr(LtrGlobalPoseOutput), _I32, _P]),
    "ltr_kmeans_update": (C.c_int, [_ptr(LtrKmeansInput), _ptr(LtrKmeansOutput), _I32, _P]),
    "ltr_vlad": (C.c_int, [_ptr(LtrVladInput), _ptr(LtrVladOutput), _I32, _P]),
    "ltr_retrieve": (C.c_int, [_ptr(LtrRetrieveInput), _ptr(LtrRetrieveOutput), _I32, _P]),
    "ltr_rt_tiles": (C.c_int, [_P, _I32, _I32, _P, _I32, _P]),
    "ltr_warp_pairs": (C.c_int, [_P, _P] + [_I32] * 4 + [c_int32_p, _P, _P, _I32, _P, _P, _I32, _P]),
    "ltr_photometric": (C.c_int, [_P, _P] + [_I32] * 3 + [_P, _P, _I32, _P, _I32, _P, _P, _I64, _I32, _P]),
    "ltr_linear_img": (C.c_int, [_P, _I32, _P, _P, _P, _I32, _P, _I32, _P] + [_I32] * 6 + [_P]),
    "ltr_linear_img_norm": (C.c_int, [_P, _I32, _P, _P, _P, _I32, _I32, _F32, _P, _P, _P, _I32, _P, _I32, _P, _I32,
                                      _I32, _I32, _P]),
    "ltr_launch_count": (_I64, []),
    "ltr_reset_launch_count": (None, []),
    "ltr_profile_begin": (None, []),
    "ltr_profile_end": (C.c_int, [_ptr(C.c_char_p), c_float_p, c_int32_p, _I32]),
}
# include/linetr_b200_debug.h (micro-benchmark / tracing hooks; not part of the drop-in boundary)
DEBUG_PROTOTYPES = {
    "ltr_gemm_bench": (_F32, [_I32] * 7),
    "ltr_gemm_chain_bench": (_F32, [_I32] * 4),
    "ltr_debug_trace_arm": (None, [_I32]),
    "ltr_debug_trace_read": (C.c_int, [_ptr(C.c_uint64)]),
    "ltr_debug_linear_img_res": (C.c_int, [_P, _I32, _P, _P, _P, _P, _P] + [_I32] * 6 + [_P]),
    "ltr_debug_encode_images": (C.c_int, [_P, _I32, _P, _ptr(_P), _ptr(_P), c_int32_p]),
    "ltr_debug_sig_attention": (C.c_int, [_P, _P, _P, _P, _I32, _I32, _P]),
    "ltr_debug_sturm_roots": (C.c_int, [_P, _I32, _P, _P, _I32, _P]),
    "ltr_debug_essential_solve": (C.c_int, [_P, _I32, _P, _P, _P, _I32, _P]),
    "ltr_debug_fundamental_solve": (C.c_int, [_P, _I32, _P, _P, _P, _I32, _P]),
    "ltr_debug_p3p": (C.c_int, [_P, _P, _I32, _P, _P, _P, _P, _I32, _P]),
    "ltr_debug_line_pose": (C.c_int, [_I32, _P, _P, _P, _P, _I32, _P, _P, _P, _P, _I32, _P]),
    "ltr_debug_fundamental_lines": (C.c_int, [_P, _P, _P, _I32, C.c_double, _P, _P, _P, _I32, _P]),
    "ltr_debug_cholesky_solve": (C.c_int, [_P, _I32, _I32, _I32, _P, _I32, _I32, _P, _I32, _P]),
}
EXPORTED_SYMBOLS = tuple(PROTOTYPES)
DEBUG_SYMBOLS = tuple(DEBUG_PROTOTYPES)


def lib_path() -> str:
    return _LIB_PATH


def load():
    """Load the shared library (once).  Raises LtrError if it is missing - no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise LtrError(
            f"linetr_b200: native CUDA library not built ({_LIB_PATH}); run tools/build_native.sh "
            "or __graft_entry__.build().  There is no CPU/PyTorch fallback.")
    lib = C.CDLL(_LIB_PATH)
    missing = [s for s in EXPORTED_SYMBOLS if not hasattr(lib, s)]
    if missing:
        raise LtrError(f"linetr_b200: the native library predates this binding (missing {', '.join(missing)}); rebuild it")
    for name, (restype, argtypes) in {**PROTOTYPES, **DEBUG_PROTOTYPES}.items():
        f = getattr(lib, name)
        f.restype, f.argtypes = restype, argtypes
    if lib.ltr_abi_version() != ABI_VERSION:
        raise LtrError("linetr_b200: ABI version mismatch between _native.py and the shared library")
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc != 0:
        msg = load().ltr_last_error()
        raise LtrError(f"{what} failed (code {rc}): {msg.decode() if msg else ''}")


def encode_images(model_ptr, n_lines: int, workspace_ptr: int) -> dict:
    """ltr_debug_encode_images: {name: (hi address, lo address, kblocks)} of the activations ltr_encode leaves in a
    workspace (names ENCODE_IMAGES; 'yf' is fp32 rows with lo = 0, kblocks = 0)."""
    hi, lo, kb = (C.c_void_p * 11)(), (C.c_void_p * 11)(), (C.c_int32 * 11)()
    check(load().ltr_debug_encode_images(model_ptr, int(n_lines), C.c_void_p(workspace_ptr), hi, lo, kb),
          "ltr_debug_encode_images")
    return {n: (hi[i] or 0, lo[i] or 0, int(kb[i])) for i, n in enumerate(ENCODE_IMAGES)}


def launch_count() -> int:
    return int(load().ltr_launch_count())


def reset_launch_count():
    load().ltr_reset_launch_count()


def profile_begin():
    load().ltr_profile_begin()


def profile_end():
    """-> {kernel_class: (ms_total, launches)} since profile_begin(); synchronises the device."""
    n = 32
    names = (C.c_char_p * n)()
    ms = (C.c_float * n)()
    cnt = (C.c_int32 * n)()
    k = load().ltr_profile_end(names, ms, cnt, n)
    return {names[i].decode(): (float(ms[i]), int(cnt[i])) for i in range(k)}
