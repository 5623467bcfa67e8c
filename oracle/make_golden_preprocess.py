"""Generate tests/golden/preprocess.npz with the REFERENCE's own load_and_preprocess_images.

TEST INFRASTRUCTURE.  Run where the reference checkout is present:  python -m oracle.make_golden_preprocess
`util/load_img_folder.py` is loaded unmodified from the checkout and run on seeded synthetic PNG files written by
`images_for(case, folder)`.  PNG is lossless, so PIL decodes the same pixels everywhere and no source image is stored; the tests
regenerate the files from the same seeds.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import tempfile

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.ref_loader import REFERENCE_ROOT  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "preprocess.npz")
CASES = {  # name: (image_size, [(height, width, PIL mode), ...], seed)
    "landscape_odd": (64, [(75, 133, "RGB")], 1),   # left = 29
    "portrait": (64, [(150, 97, "RGB")], 2),        # top = 26
    "identity": (64, [(64, 91, "RGB")], 3),         # side == image_size: an exact copy
    "upsample": (64, [(57, 40, "RGB")], 4),         # side < image_size
    "rgba": (64, [(90, 120, "RGBA")], 5),
    "grey": (64, [(100, 80, "L")], 6),
    "mixed": (64, [(75, 133, "RGB"), (57, 40, "RGB"), (120, 120, "RGB"), (90, 61, "L")], 7),
    "full": (224, [(300, 401, "RGB")], 8),
}


def frames_for(shapes, seed, channels=3):
    """Seeded uint8 [H,W,channels] frames: a smooth gradient plus noise, so that the resize sees both."""
    rng = np.random.default_rng(seed)
    out = []
    for h, w in shapes:
        yy, xx = np.mgrid[0:h, 0:w]
        base = (255.0 * (0.5 + 0.25 * np.sin(yy / 17.0 + 1.3 * np.arange(channels)[:, None, None]) * np.cos(xx / 23.0))).transpose(1, 2, 0)
        noisy = base + rng.normal(0.0, 40.0, size=(h, w, channels))
        out.append(np.clip(np.rint(noisy), 0, 255).astype(np.uint8))
    return out


def images_for(case, folder):
    """Write the case's PNG files into `folder`; returns their paths in frame order (names sort in that order)."""
    _, specs, seed = CASES[case]
    paths = []
    for k, (h, w, mode) in enumerate(specs):
        ch = {"RGB": 3, "RGBA": 4, "L": 1}[mode]
        px = frames_for([(h, w)], seed * 100 + k, ch)[0]
        path = os.path.join(folder, f"{case}_{k:02d}.png")
        Image.fromarray(px[..., 0] if mode == "L" else px, mode).save(path)
        paths.append(path)
    return paths


def reference_function():
    path = os.path.join(REFERENCE_ROOT, "pose_diffusion", "util", "load_img_folder.py")
    spec = importlib.util.spec_from_file_location("ref_load_img_folder", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.load_and_preprocess_images


def main():
    # ATen picks its scalar resize loop for 3-channel images on one thread and its vectorised loop otherwise; the two differ by an
    # ulp here and there.  One thread makes the fixture independent of the machine's core count.
    torch.set_num_threads(1)
    ref = reference_function()
    out = {}
    with tempfile.TemporaryDirectory() as folder:
        for case, (size, _, _) in CASES.items():
            paths = images_for(case, folder)
            images, info = ref(image_size=size, image_paths=list(paths))
            out[f"{case}_images"] = images.numpy()
            out[f"{case}_bboxes"] = info["bboxes_xyxy"]
            out[f"{case}_scales"] = info["resized_scales"]
            out[f"{case}_size"] = np.asarray(info["size"], dtype=np.int64)
            print(case, images.shape, info["bboxes_xyxy"].tolist(), info["size"])
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
