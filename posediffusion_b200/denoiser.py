"""`Denoiser` with the reference's constructor, parameter names and state_dict layout
(models/denoiser.py:22-98), whose forward runs the hand-written sm_90a kernels.

The torch modules below only HOLD the parameters (so real checkpoints load with strict=True and
`.to(device)` works); no torch operator runs in `forward`.  The kernels are compiled for the checkpoint
architecture of cfgs/default.yaml:25-35 (d_model 512, 4 heads, FFN 1024, 8 pre-norm layers, ReLU).
"""
from __future__ import annotations

from typing import Dict, List

import torch
import torch.nn as nn

from . import _native
from .synthetic import denoiser_param_shapes


def _cfg_get(cfg, key, default=None):
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


def TransformerEncoderWrapper(
    d_model: int,
    nhead: int,
    num_encoder_layers: int,
    dim_feedforward: int = 2048,
    dropout: float = 0.1,
    norm_first: bool = True,
    batch_first: bool = True,
):
    """Parameter container with torch's key layout (`layers.{i}.self_attn.in_proj_weight`, ...)."""
    layer = nn.TransformerEncoderLayer(
        d_model=d_model, nhead=nhead, dim_feedforward=dim_feedforward, dropout=dropout,
        batch_first=batch_first, norm_first=norm_first,
    )
    return nn.TransformerEncoder(layer, num_encoder_layers, enable_nested_tensor=False)


class TimeStepEmbedding(nn.Module):
    """Holds `linear.0/2` of the timestep MLP (util/embedding.py:13-37); evaluated once per weight load
    into a 100-row table by the native library."""

    def __init__(self, dim: int = 256):
        super().__init__()
        self.dim, self.out_dim = dim, dim // 2
        self.linear = nn.Sequential(nn.Linear(dim, dim // 2), nn.SiLU(), nn.Linear(dim // 2, dim // 2))


class Denoiser(nn.Module):
    def __init__(self, TRANSFORMER: Dict, target_dim: int = 9, pivot_cam_onehot: bool = True, z_dim: int = 384,
                 mlp_hidden_dim: int = 128):
        super().__init__()
        arch = dict(
            d_model=_cfg_get(TRANSFORMER, "d_model"), nhead=_cfg_get(TRANSFORMER, "nhead"),
            dim_feedforward=_cfg_get(TRANSFORMER, "dim_feedforward", 2048),
            num_encoder_layers=_cfg_get(TRANSFORMER, "num_encoder_layers"),
            norm_first=_cfg_get(TRANSFORMER, "norm_first", True), batch_first=_cfg_get(TRANSFORMER, "batch_first", True),
        )
        want = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, norm_first=True, batch_first=True)
        if arch != want or target_dim != 9 or not pivot_cam_onehot or z_dim != 384 or mlp_hidden_dim != 128:
            raise NotImplementedError(
                f"the sm_90a kernels are built for the checkpoint architecture {want} with target_dim=9, z_dim=384, "
                f"mlp_hidden_dim=128, pivot_cam_onehot=True; got {arch}"
            )
        self.pivot_cam_onehot = pivot_cam_onehot
        self.target_dim = target_dim
        self.time_embed = TimeStepEmbedding()
        first_dim = self.time_embed.out_dim + target_dim * 21 + z_dim + 1
        self._first = nn.Linear(first_dim, arch["d_model"])
        self._trunk = TransformerEncoderWrapper(dropout=_cfg_get(TRANSFORMER, "dropout", 0.1), **arch)
        self._last = nn.Sequential(
            nn.Linear(arch["d_model"], mlp_hidden_dim), nn.LayerNorm(mlp_hidden_dim), nn.ReLU(inplace=True),
            nn.Linear(mlp_hidden_dim, target_dim),
        )
        self._native_token = _native.module_token()  # identity for the context's weight cache (never reused, unlike id())
        self._native_epoch = 0

    # ---- native weight sync -------------------------------------------------------------------------
    def ordered_parameters(self) -> List[torch.Tensor]:
        state = dict(self.named_parameters())
        return [state[name] for name in denoiser_param_shapes()]

    def native_context(self) -> "_native.Context":
        """Context on the parameters' device with this module's current weights loaded."""
        params = self.ordered_parameters()
        device = params[0].device
        if device.type != "cuda":
            raise _native.NativeError("Denoiser parameters are on the CPU: call .to('cuda') (no CPU fallback)")
        ctx = _native.Context.get(device)
        key = (self._native_token, self._native_epoch, tuple((p.data_ptr(), p._version) for p in params))
        if ctx.weights_key != key:
            ctx.load_denoiser(params)
            ctx.weights_key = key
        return ctx

    def invalidate_native_weights(self) -> None:
        """Force a re-upload at the next call (needed after editing parameters through `.data`, which does not bump `_version`)."""
        self._native_epoch += 1

    def forward(self, x: torch.Tensor, t: torch.Tensor, z: torch.Tensor) -> torch.Tensor:
        """x [B,N,9], t [B] (all entries equal, as the sampler passes them), z [B,N,384] -> eps [B,N,9]."""
        ctx = self.native_context()
        t_host = t.reshape(-1)
        step = int(t_host[0]) if t_host.numel() else 0
        if t_host.numel() > 1 and not bool((t_host == t_host[0]).all()):
            raise NotImplementedError("per-sample timesteps are a training feature; the sampler uses one t per batch")
        return ctx.denoiser_forward(x.contiguous().float(), step, z.contiguous().float())
