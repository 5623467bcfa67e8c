"""`load_and_preprocess_images` with the reference's signature and returns (util/load_img_folder.py).

Frames are decoded with PIL exactly as the reference decodes them (`np.array(Image.open(p).convert("RGB"))`), on a thread pool;
the centre crop, the uint8 -> float32 conversion and the bilinear resize run on the GPU (pdb_images_preprocess_host), which
uploads only the crop rows the resize reads.  The one visible difference: `images` is returned on the GPU (`device`, default
the current CUDA device), so the callers' `.to(device)` is a no-op.  There is no CPU fallback.
"""
from __future__ import annotations

import os
from concurrent.futures import ThreadPoolExecutor
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch
from PIL import Image

from . import _native

IMAGE_EXTENSIONS = (".png", ".jpg", ".jpeg")


def list_images(folder_path) -> List[str]:
    """Files of `folder_path` whose lower-cased name ends in .png / .jpg / .jpeg (unsorted, as os.listdir gives them)."""
    return [os.path.join(folder_path, f) for f in os.listdir(folder_path) if f.lower().endswith(IMAGE_EXTENSIONS)]


def decode_image(path) -> np.ndarray:
    """HWC uint8 RGB pixels of one file, as the reference's _load_image reads them before its float conversion."""
    with Image.open(path) as pil_im:
        return np.array(pil_im.convert("RGB"))


def center_crop_geometry(shapes: Sequence[Tuple[int, int]], image_size: int):
    """Square centre crops of frames of (h, w) -> (crops [n,3] int32 {top, left, side}, image_info) as the reference builds
    image_info: bboxes_xyxy int64 [n,4] = [left, top, left+side, top+side], resized_scales float64 [n] = image_size / side, and
    size = (side, side) of the LAST frame.  Raises the reference's ValueError for a side <= 1."""
    crops, bboxes, scales = [], [], []
    min_hw = None
    for h, w in shapes:
        min_hw = min(int(h), int(w))
        top, left = (int(h) - min_hw) // 2, (int(w) - min_hw) // 2
        if min_hw <= 1:
            raise ValueError("squashed image!! The bounding box contains no pixels.")
        crops.append((top, left, min_hw))
        bboxes.append(np.array([left, top, left + min_hw, top + min_hw], dtype=np.int64))
        scales.append(image_size / min_hw)
    if not crops:
        raise ValueError("need at least one array to stack")
    info = {"size": (min_hw, min_hw), "bboxes_xyxy": np.stack(bboxes), "resized_scales": np.stack(scales)}
    return np.asarray(crops, dtype=np.int32), info


def load_and_preprocess_images(folder_path=None, image_size: int = 224, image_paths=None, mode: str = "bilinear",
                               device=None) -> Tuple[torch.Tensor, Dict]:
    """-> (images float32 [n,3,image_size,image_size] on `device`, image_info).  Sorts a given `image_paths` in place, like the
    reference.  Only mode="bilinear" is implemented."""
    if image_paths is None:
        image_paths = list_images(folder_path)
    image_paths.sort()
    if mode != "bilinear":
        raise NotImplementedError(f"mode={mode!r}: only the default 'bilinear' preprocessing is implemented")
    if not image_paths:
        raise ValueError("need at least one array to stack")
    with ThreadPoolExecutor(max_workers=min(len(image_paths), os.cpu_count() or 1)) as pool:
        frames = list(pool.map(decode_image, image_paths))
    crops, info = center_crop_geometry([f.shape[:2] for f in frames], image_size)
    ctx = _native.Context.get("cuda" if device is None else device)  # NativeError without a CUDA device
    return ctx.preprocess_images(frames, crops, image_size), info
