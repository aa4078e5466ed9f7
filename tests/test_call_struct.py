"""_ops.call_struct, the one host path into the C-ABI entry points that take an input and an output struct: it refuses a
missing scalar field, an unknown field, a CPU tensor, a tensor of another dtype than the field's pointee or on
another device, and a workspace below the entry's size, all before any launch."""
import pytest
import torch

from linetr_b200 import _native as N, _ops

HOMOGRAPHY_SCALARS = dict(n_pairs=1, max_rows_p=4, max_rows_l=0, thresh=3.0, n_hypotheses=16, seed=0, use_points=True,
                          use_lines=False)


def test_missing_scalar_field_is_named():
    scalars = {k: v for k, v in HOMOGRAPHY_SCALARS.items() if k != "use_lines"}
    with pytest.raises(N.LtrError, match=r"homography: LtrHomographyInput\.use_lines is not given"):
        _ops.call_struct("ltr_homography", scalars, {})


def test_unknown_field_is_refused():
    with pytest.raises(N.LtrError, match=r"homography: LtrHomographyOutput has no field \['inliers'\]"):
        _ops.call_struct("ltr_homography", HOMOGRAPHY_SCALARS, {"inliers": None})


def test_cpu_tensor_has_no_fallback():
    with pytest.raises(N.LtrError, match=r"'pts0' is on cpu; .*no CPU fallback"):
        _ops.call_struct("ltr_homography", {**HOMOGRAPHY_SCALARS, "pts0": torch.zeros((4, 2))}, {})
    with pytest.raises(N.LtrError, match=r"'H' is on cpu; .*no CPU fallback"):
        _ops.call_struct("ltr_homography", HOMOGRAPHY_SCALARS, {"H": torch.zeros((1, 3, 3), dtype=torch.float64)})


@pytest.mark.gpu
def test_dtype_layout_and_workspace_are_checked():
    dev = torch.device("cuda", 0)
    H = torch.empty((1, 3, 3), dtype=torch.float64, device=dev)
    N.reset_launch_count()
    with pytest.raises(N.LtrError, match=r"homography: 'H' must be a contiguous torch.float64 tensor on cuda:0"):
        _ops.call_struct("ltr_homography", HOMOGRAPHY_SCALARS, {"H": H.float()})
    with pytest.raises(N.LtrError, match=r"homography: 'valid' must be a contiguous torch.uint8 tensor on cuda:0"):
        _ops.call_struct("ltr_homography", HOMOGRAPHY_SCALARS,
                         {"H": H, "valid": torch.empty((2, 2), dtype=torch.uint8, device=dev).t()})
    with pytest.raises(N.LtrError, match=r"homography: 'pts0' must be a contiguous torch.float32 tensor on cuda:0"):
        _ops.call_struct("ltr_homography", {**HOMOGRAPHY_SCALARS, "pts0": torch.empty((4, 2), dtype=torch.float64,
                                                                                      device=dev)}, {"H": H})
    with pytest.raises(N.LtrError, match=r"global_poses: the workspace holds 8 bytes, 16 needed"):
        _ops.call_struct("ltr_global_poses", dict(n_images=1, n_pairs=0, min_inliers=20, anchor=-1, rot_iters=0,
                                                  pos_iters=0, rot_tan=0.1, dir_cos=0.9, ftol=0.0),
                         {"workspace": torch.empty(1, dtype=torch.float64, device=dev)}, workspace_bytes=16)
    assert N.launch_count() == 0
