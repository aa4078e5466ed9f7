"""Writes tests/golden/homography_pairs.npz: image 1 of homography pairs and its valid mask, computed with OpenCV the
way the reference's homography dataset builder computes them (dataloaders/build_homography_dataset.py:164-184):
cv2.warpPerspective of the grey image, and the float32 colour warp == 0 in every channel, eroded with a 5 x 5 kernel of
ones.  Inputs are seeded synthetic images (`synthetic.make_warp_images`) and sampled homographies; they are stored
with the outputs, so the GPU tests need neither cv2 nor this script.  Keys per case c: c/gray, c/colour, c/src_index,
c/H, c/warped, c/mask.

    python tests/golden/make_homography_pairs_golden.py
"""
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from linetr_b200 import homography_pairs as HP, synthetic as syn   # noqa: E402

# (name, n source images, height, width, pairs per image, sample_homographies parameters)
CASES = [
    ("small", 3, 96, 120, 3, dict()),
    ("wide", 1, 120, 200, 3, dict(allow_artifacts=True, translation_overflow=0.1)),
    ("ragged", 2, 37, 70, 2, dict(allow_artifacts=True, translation_overflow=0.3)),
    ("short", 1, 9, 150, 3, dict(allow_artifacts=True)),
]


def builder_pair(gray, colour, H):
    h, w = gray.shape
    warped = cv2.warpPerspective(gray, H, (w, h))
    wc = cv2.warpPerspective(colour.astype(np.float32), H, (w, h))
    mask = np.ones_like(gray)
    mask[(wc == 0).all(-1)] = 0
    return warped, cv2.erode(mask, np.ones((5, 5), np.uint8))


def main():
    rng = np.random.default_rng(20261016)
    out = {}
    for k, (name, n, h, w, per, params) in enumerate(CASES):
        gray, colour = syn.make_warp_images(100 + k, n, h, w)
        H, _ = HP.sample_homographies(n * per, (h, w), rng, **params)
        src = np.arange(n * per, dtype=np.int32) // per
        pairs = [builder_pair(gray[s], colour[s], Hp) for s, Hp in zip(src, H)]
        out.update({f"{name}/gray": gray, f"{name}/colour": colour, f"{name}/src_index": src, f"{name}/H": H,
                    f"{name}/warped": np.stack([p[0] for p in pairs]), f"{name}/mask": np.stack([p[1] for p in pairs])})
    path = os.path.join(ROOT, "tests", "golden", "homography_pairs.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
