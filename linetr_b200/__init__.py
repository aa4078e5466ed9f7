"""linetr_b200 - H100-native LineTR line-descriptor forward + mutual-NN matcher.

Drop-in names (same call surface as yosungho/LineTR `models/`):
    LineTransformer, get_dist_matrix, nn_matcher, nn_matcher_distmat
Batched front-end:
    PairEngine, LineBatch, ImagePairMatches, ImageSet, exhaustive_pairs
Match quality against homography ground truth (eval_homography):
    line_assignment, get_precision_recall, homography_ground_truth, score_line_matches
The validation step's descriptor loss and metrics (eval_criteria; drop-in eval_criteria.descriptor_loss):
    triplet_loss, validation_metrics
Geometric verification (geometry): RANSAC homographies from line and point matches, batched on the GPU, and the
homography-estimation metric:
    estimate_homographies, homography_corner_error
Relative pose (geometry): five-point RANSAC essential matrices and the pose of calibrated pairs, batched on the GPU, and
the reference's pose metrics:
    estimate_poses, compute_epipolar_error, compute_pose_error, pose_auc, pose_errors
Fundamental matrices (geometry): seven-point RANSAC with an eight-point refit for uncalibrated pairs, and an epipolar
check of the line matches, batched on the GPU:
    estimate_fundamentals
Visual localization (localization): the absolute pose of query images from 2D-3D point and line matches (P3P RANSAC
and a Levenberg-Marquardt refit), batched on the GPU, and the localization metrics:
    estimate_absolute_poses, absolute_pose_errors, localization_recall, lift_to_3d
Triangulation (triangulation): world points of every keypoint and world end points of every key line of posed images
from their pair matches (multi-view, with outlier rejection and a Gauss-Newton refit), batched on the GPU:
    triangulate, TriangulationResult
Tracks (tracks): the pair matches that agree with the poses joined into point and line tracks across a posed image
set, and one robust multi-view world point or world line per track, batched on the GPU:
    triangulate_tracks, TrackResult
Bundle adjustment (bundle): the poses of a posed image set and the world points and lines of its tracks refined
together (Levenberg-Marquardt with a Schur complement onto the cameras), on the GPU:
    bundle_adjust, BundleResult
Image retrieval (retrieval): a spherical k-means vocabulary over an image set's point and line descriptors, VLAD
global descriptors and the exact top-k database images of every query, as pair lists, on the GPU:
    Vocabulary, train_vocabulary, global_descriptors, retrieve, retrieval_pairs
Homography image pairs (homography_pairs): sampled homographies, warped images and valid masks, batched on the GPU:
    sample_homographies, warp_pairs, homography_pairs, apply_valid_masks
Photometric augmentation (photometric): the homography builder's brightness, contrast, noise, motion blur and shade,
batched on the GPU, and pairs built from augmented images:
    sample_photometric, photometric_augment, photometric_homography_pairs
`install_as_reference_models()` registers this package's modules under the reference's
module names (`models.line_transformer`, `models.nn_matcher`, `models.line_process`) so that
the reference's own `models/matching.py` / `match_line_pairs.py` run unchanged on top of it.
"""
from __future__ import annotations

import sys
import types

__version__ = "0.1.0"

_LAZY = {
    "LineTransformer": ("line_transformer", "LineTransformer"),
    "get_dist_matrix": ("line_process", "get_dist_matrix"),
    "nn_matcher": ("nn_matcher", "nn_matcher"),
    "nn_matcher_distmat": ("nn_matcher", "nn_matcher_distmat"),
    "PairEngine": ("engine", "PairEngine"),
    "LineBatch": ("engine", "LineBatch"),
    "ImagePairMatches": ("engine", "ImagePairMatches"),
    "ImageSet": ("engine", "ImageSet"),
    "exhaustive_pairs": ("engine", "exhaustive_pairs"),
    "line_assignment": ("eval_homography", "line_assignment"),
    "get_precision_recall": ("eval_homography", "get_precision_recall"),
    "homography_ground_truth": ("eval_homography", "homography_ground_truth"),
    "score_line_matches": ("eval_homography", "score_line_matches"),
    "triplet_loss": ("eval_criteria", "triplet_loss"),
    "validation_metrics": ("eval_criteria", "validation_metrics"),
    "estimate_homographies": ("geometry", "estimate_homographies"),
    "homography_corner_error": ("geometry", "homography_corner_error"),
    "estimate_poses": ("geometry", "estimate_poses"),
    "compute_epipolar_error": ("geometry", "compute_epipolar_error"),
    "compute_pose_error": ("geometry", "compute_pose_error"),
    "pose_auc": ("geometry", "pose_auc"),
    "pose_errors": ("geometry", "pose_errors"),
    "estimate_fundamentals": ("geometry", "estimate_fundamentals"),
    "estimate_absolute_poses": ("localization", "estimate_absolute_poses"),
    "AbsolutePoseResult": ("localization", "AbsolutePoseResult"),
    "absolute_pose_errors": ("localization", "absolute_pose_errors"),
    "localization_recall": ("localization", "localization_recall"),
    "lift_to_3d": ("localization", "lift_to_3d"),
    "triangulate": ("triangulation", "triangulate"),
    "TriangulationResult": ("triangulation", "TriangulationResult"),
    "triangulate_tracks": ("tracks", "triangulate_tracks"),
    "TrackResult": ("tracks", "TrackResult"),
    "bundle_adjust": ("bundle", "bundle_adjust"),
    "BundleResult": ("bundle", "BundleResult"),
    "global_poses": ("global_poses", "global_poses"),
    "GlobalPoseResult": ("global_poses", "GlobalPoseResult"),
    "registered_set": ("global_poses", "registered_set"),
    "Vocabulary": ("retrieval", "Vocabulary"),
    "train_vocabulary": ("retrieval", "train_vocabulary"),
    "global_descriptors": ("retrieval", "global_descriptors"),
    "GlobalDescriptors": ("retrieval", "GlobalDescriptors"),
    "retrieve": ("retrieval", "retrieve"),
    "Retrieval": ("retrieval", "Retrieval"),
    "retrieval_pairs": ("retrieval", "retrieval_pairs"),
    "sample_homographies": ("homography_pairs", "sample_homographies"),
    "warp_pairs": ("homography_pairs", "warp_pairs"),
    "homography_pairs": ("homography_pairs", "homography_pairs"),
    "apply_valid_masks": ("homography_pairs", "apply_valid_masks"),
    "sample_photometric": ("photometric", "sample_photometric"),
    "photometric_augment": ("photometric", "photometric_augment"),
    "photometric_homography_pairs": ("photometric", "photometric_homography_pairs"),
}


def __getattr__(name):
    if name in _LAZY:
        import importlib
        mod, attr = _LAZY[name]
        return getattr(importlib.import_module(f"{__name__}.{mod}"), attr)
    raise AttributeError(name)


def install_as_reference_models(package: str = "models"):
    """Make `from models.line_transformer import LineTransformer, get_dist_matrix` and
    `from models.nn_matcher import nn_matcher, nn_matcher_distmat` (reference
    models/matching.py:5-6) resolve to this package.  Call before importing `models.matching`
    from a reference checkout; the remaining reference modules (superpoint, line_detector,
    matching) are left untouched."""
    from . import line_process, line_transformer, nn_matcher as nnm
    if package not in sys.modules:
        try:
            __import__(package)
        except Exception:
            pkg = types.ModuleType(package)
            pkg.__path__ = []
            sys.modules[package] = pkg
    sys.modules[f"{package}.line_transformer"] = line_transformer
    sys.modules[f"{package}.nn_matcher"] = nnm
    sys.modules[f"{package}.line_process"] = line_process
    pkg = sys.modules[package]
    pkg.line_transformer, pkg.nn_matcher, pkg.line_process = line_transformer, nnm, line_process
