"""Pose encoding -> cameras, after the sampling loop (reference: util/camera_transform.py:64-105).

pytorch3d is not a dependency of this package: `PerspectiveCameras` below is a plain container with the
attributes the reference's callers read (R, T, focal_length, principal_point, device, len()).  The conversion itself
runs in the native library (pdb_pose_to_camera); there is no CPU path.
"""
from __future__ import annotations

import torch

from . import _native


class PerspectiveCameras:
    def __init__(self, focal_length, R, T, principal_point=None, device=None):
        self.focal_length, self.R, self.T = focal_length, R, T
        self.principal_point = torch.zeros_like(focal_length) if principal_point is None else principal_point
        self.device = R.device if device is None else device

    def __len__(self):
        return self.R.shape[0]


def pose_encoding_to_camera(
    pose_encoding: torch.Tensor,
    pose_encoding_type: str = "absT_quaR_logFL",
    log_focal_length_bias: float = 1.8,
    min_focal_length: float = 0.1,
    max_focal_length: float = 20,
    return_dict: bool = False,
):
    if pose_encoding_type != "absT_quaR_logFL":
        raise ValueError(f"Unknown pose encoding {pose_encoding_type}")
    if not pose_encoding.is_cuda:
        raise _native.NativeError("pose_encoding must be a CUDA tensor (posediffusion_b200 has no CPU fallback)")
    ctx = _native.Context.get(pose_encoding.device)
    R, T, fl = ctx.pose_to_camera(pose_encoding, log_focal_length_bias, min_focal_length, max_focal_length)
    if return_dict:
        return {"focal_length": fl, "R": R, "T": T}
    return PerspectiveCameras(focal_length=fl, R=R, T=T, device=R.device)


def camera_to_pose_encoding(
    camera,
    pose_encoding_type: str = "absT_quaR_logFL",
    log_focal_length_bias: float = 1.8,
    min_focal_length: float = 0.1,
    max_focal_length: float = 20,
):
    """Cameras (anything with R [...,3,3], T [...,3], focal_length [...,2], e.g. pytorch3d PerspectiveCameras) -> pose encoding
    [..., 9] (reference: util/camera_transform.py:108-129), computed by pdb_camera_to_pose.  The quaternion is pytorch3d's
    matrix_to_quaternion with its real part made non-negative (standardize_quaternion; DESIGN.md, Training)."""
    if pose_encoding_type != "absT_quaR_logFL":
        raise ValueError(f"Unknown pose encoding {pose_encoding_type}")
    if not camera.R.is_cuda:
        raise _native.NativeError("camera tensors must be on a CUDA device (posediffusion_b200 has no CPU fallback)")
    ctx = _native.Context.get(camera.R.device)
    return ctx.camera_to_pose(camera.R, camera.T, camera.focal_length, log_focal_length_bias, min_focal_length, max_focal_length)
