"""Stage, from a checkout of the original LineTR project, what the parity tests run against into the
git-ignored directory oracle/_ref/reference/: its `models` package with the shipped checkpoints
(LineTR_weight.pth, superpoint_v1.pth) and the bundled image pairs of assets/input_pairs.txt.

Nothing here is committed; build() runs `stage()` when a checkout is available (LINETR_REFERENCE, default
/root/reference), so that the staged copy travels with the working tree to machines that have no checkout.
"""
import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
STAGE_DIR = os.path.join(HERE, "_ref", "reference")


def reference_checkout():
    return os.environ.get("LINETR_REFERENCE", "/root/reference")


def stage(ref_dir=None) -> bool:
    """Copy models/ and the image pairs; returns False when no checkout is available.  Idempotent."""
    ref_dir = ref_dir or reference_checkout()
    if not os.path.isfile(os.path.join(ref_dir, "models", "weights", "LineTR_weight.pth")):
        return False
    models = os.path.join(STAGE_DIR, "models")
    if not os.path.isdir(models):
        tmp = models + ".tmp"
        shutil.rmtree(tmp, ignore_errors=True)
        shutil.copytree(os.path.join(ref_dir, "models"), tmp, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
        os.replace(tmp, models)
    assets = os.path.join(STAGE_DIR, "assets")
    os.makedirs(assets, exist_ok=True)
    with open(os.path.join(ref_dir, "assets", "input_pairs.txt")) as f:
        names = ["input_pairs.txt"] + [n for line in f for n in line.split()[:2]]
    for n in names:
        if not os.path.exists(os.path.join(assets, n)):
            shutil.copyfile(os.path.join(ref_dir, "assets", n), os.path.join(assets, n))
    return True


if __name__ == "__main__":
    print("staged" if stage() else "no reference checkout found", STAGE_DIR)
