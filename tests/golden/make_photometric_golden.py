"""Writes tests/golden/photometric.npz: the homography builder's additive shade and the OpenCV filters the photometric
contract is pinned to.  Build container only (needs the reference checkout and cv2):

    python tests/golden/make_photometric_golden.py

- shade/<case>: the UNMODIFIED reference `customizedTransform` (dataloaders/utils/photometric.py, imported with a stub
  `imgaug` module, which it does not use for the shade) applied with the yaml's additive_shade parameters after
  np.random.seed(seed), in the builder's chain (build_homography_dataset.py:115-121, :157): stage-1 bytes a ->
  float32 a / 255 -> customizedTransform -> float64 -> * 255 -> astype(uint8).  The ellipse, transparency and kernel
  size draws are recorded by replaying the same np.random sequence.  Keys: input, ellipses (ax, ay, x, y, rint(angle)),
  angle (the raw draws), transparency, ksize, output.
- filter2d/<k>: cv2.filter2D(image, -1, kernel) (BORDER_REFLECT_101) of uint8 images with 3 x 3 float32 kernels.
- blur/<case>: cv2.GaussianBlur(mask, (ksize, ksize), 0) of float32 0/255 masks, with kernel sizes the builder draws.
Inputs are stored with the outputs, so the GPU tests need neither cv2 nor the reference.
"""
import os
import sys
import types

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("LINETR_REFERENCE", "/root/reference")
sys.path.insert(0, ROOT)
from linetr_b200 import photometric as PH, synthetic as syn   # noqa: E402

SHADE = {"transparency_range": [-0.5, 0.5], "kernel_size_range": [100, 150]}
# (name, seed, height, width)
SHADE_CASES = [("vga", 11, 480, 640), ("qvga", 13, 120, 160), ("ragged", 14, 37, 70),
               ("short", 15, 9, 150), ("tiny", 16, 1, 7)]
BLUR_CASES = [("qvga", 120, 160, 125), ("ragged", 37, 70, 101), ("short", 9, 150, 149),
              ("tiny", 1, 7, 101)]


def reference_transform():
    stub = types.ModuleType("imgaug")
    stub.augmenters = types.ModuleType("imgaug.augmenters")
    sys.modules.setdefault("imgaug", stub)
    sys.modules.setdefault("imgaug.augmenters", stub.augmenters)
    sys.path.insert(0, os.path.join(REF, "dataloaders", "utils"))
    import photometric as ref   # the reference's module
    return ref.customizedTransform()


def replay(seed, h, w, nb_ellipses=20):
    """The draws of _py_additive_shade after np.random.seed(seed), made by the same np.random calls."""
    np.random.seed(seed)
    min_dim = min(h, w) / 4
    ell, ang = [], []
    for _ in range(nb_ellipses):
        ax = int(max(np.random.rand() * min_dim, min_dim / 5))
        ay = int(max(np.random.rand() * min_dim, min_dim / 5))
        mr = max(ax, ay)
        x = np.random.randint(mr, w - mr)
        y = np.random.randint(mr, h - mr)
        a = np.random.rand() * 90
        ell.append((ax, ay, x, y, int(np.rint(a))))
        ang.append(a)
    t = np.random.uniform(*SHADE["transparency_range"])
    k = np.random.randint(*SHADE["kernel_size_range"])
    return np.array(ell, np.int32), np.array(ang), t, k + (k % 2 == 0)


def main():
    cus = reference_transform()
    conf = {"photometric": {"params": {"additive_shade": SHADE}}}
    out = {}
    for name, seed, h, w in SHADE_CASES:
        gray, _ = syn.make_warp_images(seed, 1, h, w)
        a = gray[0]
        ell, ang, t, k = replay(seed, h, w)
        np.random.seed(seed)
        img = cus(a[..., None].astype(np.float32) / 255, **conf)
        batch = np.empty((1, 1, h, w))
        batch[0] = img.squeeze()
        res = (batch[0][0] * 255).astype("uint8")
        out.update({f"shade/{name}/input": a, f"shade/{name}/ellipses": ell, f"shade/{name}/angle": ang,
                    f"shade/{name}/transparency": np.float64(t), f"shade/{name}/ksize": np.int32(k),
                    f"shade/{name}/output": res})
    rng = np.random.default_rng(20261016)
    for j, (h, w) in enumerate([(120, 160), (37, 70), (9, 150), (1, 7), (3, 1)]):
        img = rng.integers(0, 256, (h, w)).astype(np.uint8)
        kern = PH.motion_blur_kernel(rng.uniform(0, 360), rng.uniform(-1, 1))
        out.update({f"filter2d/{j}/input": img, f"filter2d/{j}/kernel": kern,
                    f"filter2d/{j}/output": cv2.filter2D(img, -1, kern)})
    for name, h, w, k in BLUR_CASES:
        m = PH.ellipse_mask((h, w), PH.sample_photometric(1, (h, w), rng, additive_shade=SHADE)["ellipses"][0])
        out.update({f"blur/{name}/input": m, f"blur/{name}/ksize": np.int32(k),
                    f"blur/{name}/output": cv2.GaussianBlur(m.astype(np.float32), (k, k), 0)})
    path = os.path.join(HERE, "photometric.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
