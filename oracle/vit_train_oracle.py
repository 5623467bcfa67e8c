"""Float64 gradients of the image feature extractor -- TEST INFRASTRUCTURE.

d(sum(g * z)) / d(the 150 DINO ViT-S/16 tensors) by torch autograd through the evaluator of oracle/vit_f64.py, with LayerNorm
applied explicitly as the training path does.  `tf32=True` rounds the operands of every matrix product, in the forward and in both
backward products (oracle.train_oracle._Matmul): the projections and the patch embedding truncate, as the wgmma engine reads
fp32, and the two attention products round to nearest, as the attention kernel's cvt.rna does.  Tests derive their tolerances
from the distance between the rounded and the exact run.
"""
from __future__ import annotations

from typing import Dict, Sequence

import torch
import torch.nn.functional as F

from oracle.dino_vit import EMBED, HEADS
from oracle.train_oracle import _Matmul
from oracle.vit_f64 import VitF64


class _VitGrad(VitF64):
    """VitF64 over parameters that require grad; `mode` is None (exact) or "tf32"."""

    def __init__(self, params: Dict[str, torch.Tensor], dtype, device="cpu"):
        self.dtype = dtype
        self.device = torch.device(device)
        self.p = params
        self.folded = {}

    def linear(self, x, w, b, mode):
        return _Matmul.apply(x, w.transpose(0, 1), "trunc" if mode else None) + b

    def ln_linear(self, x, l, which, mode):
        pre = f"blocks.{l}."
        lin, norm = ("attn.qkv", "norm1") if which == "qkv" else ("mlp.fc1", "norm2")
        y = F.layer_norm(x, (EMBED,), self.p[pre + norm + ".weight"], self.p[pre + norm + ".bias"], 1e-6)
        return self.linear(y, self.p[pre + lin + ".weight"], self.p[pre + lin + ".bias"], mode)

    def attention(self, qkv, mode):
        B, L, _ = qkv.shape
        q, k, v = qkv.reshape(B, L, 3, HEADS, EMBED // HEADS).permute(2, 0, 3, 1, 4)
        rn = "rn" if mode else None
        p = _Matmul.apply(q * 0.125, k.transpose(-2, -1), rn).softmax(dim=-1)
        return _Matmul.apply(p, v, rn).transpose(1, 2).reshape(B, L, EMBED)


def features_and_grads(state: Dict[str, torch.Tensor], image_rgb: torch.Tensor, scale_factors: Sequence[float], grad_z: torch.Tensor,
                       tf32: bool = False, dtype: torch.dtype = torch.float64, device="cpu"):
    """(z [n,384], {name: d(sum(grad_z * z)) / d tensor}) on `device` (default the CPU), in float64 unless `dtype` says otherwise."""
    params = {k: v.detach().to(device, dtype).requires_grad_(True) for k, v in state.items()}
    z = _VitGrad(params, dtype, device).features(image_rgb, scale_factors, "tf32" if tf32 else None)
    grads = torch.autograd.grad((z * grad_z.to(device, dtype)).sum(), list(params.values()))
    return z.detach(), dict(zip(params, grads))


def features_and_grads_chunked(state: Dict[str, torch.Tensor], image_rgb: torch.Tensor, scale_factors: Sequence[float],
                               grad_z: torch.Tensor, tf32: bool = False, chunk: int = 32, dtype: torch.dtype = torch.float64,
                               device="cpu"):
    """features_and_grads() of a large batch, `chunk` images at a time: (z [n,384], gradients summed over chunks in `dtype`),
    both on the CPU.  Every image is its own sequence, so the chunks' z are the batch's and the gradients add up."""
    zs, total = [], None
    for i in range(0, image_rgb.shape[0], chunk):
        z, g = features_and_grads(state, image_rgb[i:i + chunk], scale_factors, grad_z[i:i + chunk], tf32, dtype, device)
        zs.append(z.cpu())
        g = {k: v.cpu() for k, v in g.items()}
        total = g if total is None else {k: total[k] + g[k] for k in g}
    return torch.cat(zs), total
