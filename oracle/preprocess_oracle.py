"""CPU oracle of load_and_preprocess_images after decoding (TEST INFRASTRUCTURE).

Restates the reference's float conversion, centre crop and `F.interpolate(..., mode="bilinear", align_corners=False)` on decoded
uint8 HWC frames, in the reference's order of operations (numpy float32 / 255, crop as a view, ATen's CPU resize).  It is the
arbiter at sizes the golden file does not hold and on machines without the reference checkout.
"""
from __future__ import annotations

from typing import Sequence

import numpy as np
import torch
import torch.nn.functional as F


def preprocess(frames: Sequence[np.ndarray], image_size: int):
    """uint8 [H,W,3] frames -> (images float32 [n,3,S,S] CPU tensor, bboxes_xyxy int64 [n,4], resized_scales float64 [n])."""
    images, bboxes, scales = [], [], []
    for frame in frames:
        im = frame.transpose((2, 0, 1)).astype(np.float32) / 255.0
        h, w = im.shape[1:]
        side = min(h, w)
        top, left = (h - side) // 2, (w - side) // 2
        crop = im[:, top: top + side, left: left + side]
        out = F.interpolate(torch.from_numpy(crop)[None], size=(image_size, image_size), mode="bilinear", align_corners=False)[0]
        images.append(out.numpy())
        bboxes.append(np.array([left, top, left + side, top + side], dtype=np.int64))
        scales.append(image_size / side)
    return torch.from_numpy(np.stack(images)), np.stack(bboxes), np.stack(scales)
