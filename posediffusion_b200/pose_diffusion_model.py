"""`PoseDiffusionModel` facade with the reference's constructor / forward signature
(models/pose_diffusion_model.py:35-142): the sampling branch, and the training branch (training=True) with a frozen
image feature extractor or precomputed features.

Hydra is not a dependency: the `_target_` strings of cfgs/default.yaml are resolved against this package
(`models.Denoiser`, `models.GaussianDiffusion`, `models.TransformerEncoderWrapper`,
`models.MultiScaleImageFeatureExtractor`).  Features may also be passed precomputed as forward(z=...).
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.nn as nn

from .camera_transform import camera_to_pose_encoding, pose_encoding_to_camera
from .denoiser import Denoiser, TransformerEncoderWrapper
from .gaussian_diffuser import GaussianDiffusion
from .image_feature_extractor import MultiScaleImageFeatureExtractor

_TARGETS = {"Denoiser": Denoiser, "GaussianDiffusion": GaussianDiffusion, "TransformerEncoderWrapper": TransformerEncoderWrapper,
            "MultiScaleImageFeatureExtractor": MultiScaleImageFeatureExtractor}


def instantiate(cfg, **overrides):
    """`hydra.utils.instantiate(cfg, _recursive_=False)` for the handful of targets on this path."""
    if cfg is None or isinstance(cfg, nn.Module):
        return cfg
    spec = dict(cfg)
    name = spec.pop("_target_").rsplit(".", 1)[-1]
    if name not in _TARGETS:
        raise NotImplementedError(f"_target_ {name} is outside the native sampling hot path")
    spec.update(overrides)
    return _TARGETS[name](**spec)


class PoseDiffusionModel(nn.Module):
    def __init__(self, pose_encoding_type: str, IMAGE_FEATURE_EXTRACTOR: Optional[Dict], DIFFUSER: Dict, DENOISER: Dict):
        super().__init__()
        self.pose_encoding_type = pose_encoding_type
        try:
            self.image_feature_extractor = instantiate(IMAGE_FEATURE_EXTRACTOR)
        except NotImplementedError:
            self.image_feature_extractor = None  # features must then be passed as z=...
        self.diffuser = instantiate(DIFFUSER)
        denoiser = instantiate(DENOISER)
        self.diffuser.model = denoiser
        self.target_dim = denoiser.target_dim
        self.apply(self._init_weights)

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            nn.init.trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def forward(self, image: Optional[torch.Tensor] = None, gt_cameras=None, sequence_name: Optional[List[str]] = None,
                cond_fn=None, cond_start_step=0, training=True, batch_repeat=-1, z: Optional[torch.Tensor] = None):
        if z is None:
            if self.image_feature_extractor is None or image is None:
                raise ValueError("no image feature extractor configured: pass precomputed features as z=[B,N,384]")
            if training and any(p.requires_grad for p in self.image_feature_extractor.parameters()):
                raise NotImplementedError(
                    "training with a trainable image feature extractor needs the DINO ViT backward, which is not built: "
                    "construct MultiScaleImageFeatureExtractor with freeze=True or pass precomputed features as z=")
            b, n = image.shape[:2]
            z = self.image_feature_extractor(image.reshape(b * n, *image.shape[2:])).reshape(b, n, -1)
        if training:  # models/pose_diffusion_model.py:111-126
            batch_num = z.shape[0]
            pose_encoding = camera_to_pose_encoding(gt_cameras, pose_encoding_type=self.pose_encoding_type)
            if batch_repeat > 0:
                pose_encoding = pose_encoding.reshape(batch_num * batch_repeat, -1, self.target_dim)
                z = z.repeat(batch_repeat, 1, 1)
            else:
                pose_encoding = pose_encoding.reshape(batch_num, -1, self.target_dim)
            diffusion_results = self.diffuser(pose_encoding, z=z)
            diffusion_results["pred_cameras"] = pose_encoding_to_camera(
                diffusion_results["x_0_pred"].detach(), pose_encoding_type=self.pose_encoding_type
            )
            return diffusion_results
        B, N, _ = z.shape
        pose_encoding, _trajectory = self.diffuser.sample(
            shape=[B, N, self.target_dim], z=z, cond_fn=cond_fn, cond_start_step=cond_start_step
        )
        pred_cameras = pose_encoding_to_camera(pose_encoding, pose_encoding_type=self.pose_encoding_type)
        return {"pred_cameras": pred_cameras, "z": z}
