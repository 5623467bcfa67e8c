"""Synthetic inputs for the sampling hot path (bench + tests).

There is no network for the Co3D checkpoint, DINO weights or hloc matches, so both
the native path and the CPU oracle run on: random-init denoiser weights with the
reference's initialisation law (trunc-normal sigma=0.02 Linear weights, zero biases,
unit LayerNorm; reference pose_diffusion_model.py:67-74), z ~ N(0,1) of DINO ViT-S/16
CLS shape [B,N,384], pre-drawn Gaussian noise, and 2D correspondences in the
reference's `matches_dict` format (demo.py:79-89): kp1/kp2 float64 [M_tot,2] pixel
coordinates in the 224^2 crop, i12 int64 [M_tot,2], grouped contiguously by pair.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import numpy as np
import torch

TARGET_DIM = 9
Z_DIM = 384
D_MODEL = 512
N_HEAD = 4
D_FF = 1024
N_LAYERS = 8
MLP_HIDDEN = 128
T_EMB_IN = 256
T_EMB_OUT = 128
N_HARMONIC = 10
POSE_EMB_DIM = TARGET_DIM * (2 * N_HARMONIC + 1)  # 189
FIRST_IN = POSE_EMB_DIM + T_EMB_OUT + Z_DIM + 1  # 702


def default_ggs_cfg() -> Dict:
    """cfgs/default.yaml:6-13 (+ pose_encoding_type added by demo.py:87)."""
    return dict(
        enable=True,
        start_step=10,
        learning_rate=0.01,
        iter_num=100,
        sampson_max=10,
        min_matches=10,
        alpha=0.0001,
        pose_encoding_type="absT_quaR_logFL",
    )


def denoiser_param_shapes() -> Dict[str, Tuple[int, ...]]:
    """Reference checkpoint layout below `diffuser.model.` (SURVEY.md §8b)."""
    shapes: Dict[str, Tuple[int, ...]] = {
        "time_embed.linear.0.weight": (T_EMB_OUT, T_EMB_IN),
        "time_embed.linear.0.bias": (T_EMB_OUT,),
        "time_embed.linear.2.weight": (T_EMB_OUT, T_EMB_OUT),
        "time_embed.linear.2.bias": (T_EMB_OUT,),
        "_first.weight": (D_MODEL, FIRST_IN),
        "_first.bias": (D_MODEL,),
    }
    for layer in range(N_LAYERS):
        p = f"_trunk.layers.{layer}."
        shapes[p + "self_attn.in_proj_weight"] = (3 * D_MODEL, D_MODEL)
        shapes[p + "self_attn.in_proj_bias"] = (3 * D_MODEL,)
        shapes[p + "self_attn.out_proj.weight"] = (D_MODEL, D_MODEL)
        shapes[p + "self_attn.out_proj.bias"] = (D_MODEL,)
        shapes[p + "linear1.weight"] = (D_FF, D_MODEL)
        shapes[p + "linear1.bias"] = (D_FF,)
        shapes[p + "linear2.weight"] = (D_MODEL, D_FF)
        shapes[p + "linear2.bias"] = (D_MODEL,)
        shapes[p + "norm1.weight"] = (D_MODEL,)
        shapes[p + "norm1.bias"] = (D_MODEL,)
        shapes[p + "norm2.weight"] = (D_MODEL,)
        shapes[p + "norm2.bias"] = (D_MODEL,)
    shapes["_last.0.weight"] = (MLP_HIDDEN, D_MODEL)
    shapes["_last.0.bias"] = (MLP_HIDDEN,)
    shapes["_last.1.weight"] = (MLP_HIDDEN,)
    shapes["_last.1.bias"] = (MLP_HIDDEN,)
    shapes["_last.3.weight"] = (TARGET_DIM, MLP_HIDDEN)
    shapes["_last.3.bias"] = (TARGET_DIM,)
    return shapes


def random_denoiser_state(seed: int = 0, bias_std: float = 0.0) -> Dict[str, torch.Tensor]:
    """Random-init denoiser weights (fp32, CPU) keyed like the reference state_dict.

    `bias_std > 0` perturbs biases / LayerNorm affine terms too, so that parity tests
    exercise every parameter (the reference init leaves them at 0 / 1).
    """
    gen = torch.Generator().manual_seed(seed)
    state: Dict[str, torch.Tensor] = {}
    for name, shape in denoiser_param_shapes().items():
        is_norm = ".norm" in name or name.startswith("_last.1.")
        if name.endswith("weight") and len(shape) == 2:
            w = torch.empty(shape, dtype=torch.float32)
            torch.nn.init.trunc_normal_(w, std=0.02, generator=gen)
            state[name] = w
        elif is_norm and name.endswith("weight"):
            state[name] = 1.0 + bias_std * torch.randn(shape, generator=gen)
        else:
            state[name] = bias_std * torch.randn(shape, generator=gen)
    return state


def random_features(batch: int, frames: int, seed: int = 0) -> torch.Tensor:
    gen = torch.Generator().manual_seed(1000 + seed)
    return torch.randn(batch, frames, Z_DIM, generator=gen)


def predraw_noise(batch: int, frames: int, timesteps: int = 100, seed: int = 0) -> torch.Tensor:
    """[timesteps+1, B, N, 9]: draw 0 = x_T, draw 1+k = noise of the k-th loop iteration
    (t = timesteps-1-k).  Guided steps and t=0 ignore their slot (reference draws nothing
    there, gaussian_diffuser.py:270-278)."""
    gen = torch.Generator().manual_seed(2000 + seed)
    return torch.randn(timesteps + 1, batch, frames, TARGET_DIM, generator=gen)


def ordered_pairs(frames: int, ordered: bool = True) -> np.ndarray:
    pairs = [(a, b) for a in range(frames) for b in range(frames) if (a != b if ordered else a < b)]
    return np.asarray(pairs, dtype=np.int64).reshape(-1, 2)


def uniform_matches(frames: int, per_pair: int, seed: int = 0, ordered: bool = True, image_size: int = 224) -> Dict:
    """Uniform-random correspondences for every (ordered) pair, `per_pair` rows each
    (BASELINE.md §3): almost all are geometrically inconsistent, ~0.7 % pass s < 10."""
    rng = np.random.default_rng(3000 + seed)
    pairs = ordered_pairs(frames, ordered)
    total = len(pairs) * per_pair
    return {
        "kp1": rng.uniform(0.0, image_size, size=(total, 2)),
        "kp2": rng.uniform(0.0, image_size, size=(total, 2)),
        "i12": np.repeat(pairs, per_pair, axis=0),
        "img_shape": (frames, 3, image_size, image_size),
    }


def _quat_to_rot(q: np.ndarray) -> np.ndarray:
    w, x, y, z = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    s2 = 2.0 / (q * q).sum(-1)
    m = np.stack(
        [
            1 - s2 * (y * y + z * z), s2 * (x * y - z * w), s2 * (x * z + y * w),
            s2 * (x * y + z * w), 1 - s2 * (x * x + z * z), s2 * (y * z - x * w),
            s2 * (x * z - y * w), s2 * (y * z + x * w), 1 - s2 * (x * x + y * y),
        ],
        axis=-1,
    )
    return m.reshape(q.shape[:-1] + (3, 3))


def scene_matches(
    frames: int,
    per_pair: int,
    seed: int = 0,
    ordered: bool = True,
    image_size: int = 224,
    pixel_noise: float = 1.0,
    pose_noise: float = 0.02,
    ragged: bool = False,
) -> Tuple[Dict, np.ndarray, np.ndarray]:
    """Geometry-consistent scene: random 3D points seen by cameras on a ring, projected
    with the PyTorch3D NDC convention the reference assumes (X_cam = X R + T,
    u = W/2 - s f X/Z, v = H/2 - s f Y/Z, s = min(H,W)/2).

    Returns (matches_dict, gt_pose [N,9], start_pose [N,9]) with start = gt + pose_noise*N(0,1);
    most matches are valid at the start pose (Sampson < 10).  `ragged` draws a different
    match count per pair (0..2*per_pair), as hloc does.
    """
    rng = np.random.default_rng(4000 + seed)
    half = image_size / 2.0
    quat = rng.normal(size=(frames, 4))
    quat[:, 0] = np.abs(quat[:, 0]) + 2.0  # rotations of moderate angle
    quat /= np.linalg.norm(quat, axis=1, keepdims=True)
    rot = _quat_to_rot(quat)
    trans = np.concatenate([rng.normal(scale=0.3, size=(frames, 2)), 6.0 + rng.normal(scale=0.3, size=(frames, 1))], 1)
    log_fl = rng.normal(scale=0.05, size=(1, 2)).repeat(frames, 0)  # shared focal (GGS averages it)
    focal = np.exp(log_fl + 1.8)
    gt_pose = np.concatenate([trans, quat, log_fl], axis=1)

    pairs = ordered_pairs(frames, ordered)
    kp1, kp2, i12 = [], [], []
    for a, b in pairs:
        count = int(rng.integers(0, 2 * per_pair + 1)) if ragged else per_pair
        if count == 0:
            continue
        pts = rng.normal(scale=0.8, size=(count, 3))
        uv = []
        for cam in (a, b):
            xc = pts @ rot[cam] + trans[cam]
            u = half - half * focal[cam, 0] * xc[:, 0] / xc[:, 2]
            v = half - half * focal[cam, 1] * xc[:, 1] / xc[:, 2]
            uv.append(np.stack([u, v], 1) + rng.normal(scale=pixel_noise, size=(count, 2)))
        kp1.append(uv[0])
        kp2.append(uv[1])
        i12.append(np.tile(np.array([[a, b]], dtype=np.int64), (count, 1)))
    matches = {
        "kp1": np.concatenate(kp1, 0),
        "kp2": np.concatenate(kp2, 0),
        "i12": np.concatenate(i12, 0),
        "img_shape": (frames, 3, image_size, image_size),
    }
    start = gt_pose + pose_noise * rng.normal(size=gt_pose.shape)
    return matches, gt_pose.astype(np.float32), start.astype(np.float32)
