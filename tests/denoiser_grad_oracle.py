"""Float64 restatement of the reference's Denoiser.forward under autograd -- TEST INFRASTRUCTURE.

`denoiser_eps` is oracle/train_oracle.py's forward() from the feed row onwards, started at a given pose x instead of q_sample's
x_t (models/denoiser.py:53-76 with injected dropout masks); it reuses that module's TF32 operand emulation (`tf32=`) and its
mask layout.  When x requires grad the harmonic features are evaluated in `dtype` so that dL/dx flows through them; otherwise
they are the float32 features forward() uses, so that denoiser_eps(x = x_t) reproduces forward()["eps"] exactly.
`eps_and_grads` adds d sum(grad_eps * eps) / d (parameters, x, z).
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence

import torch
import torch.nn.functional as F

from oracle.pose_oracle import harmonic_features, timestep_features
from oracle.train_oracle import D_MODEL, HEADS, LAYERS, _drop, _linear, dropout_masks

N_HARMONIC = 10


def denoiser_eps(params: Dict[str, torch.Tensor], x, t, z, masks=None, p: float = 0.0, tf32: Optional[str] = None,
                 dtype: torch.dtype = torch.float64, device="cpu") -> torch.Tensor:
    """params: the 108 denoiser tensors by state_dict name (in `dtype` on `device`, may require grad); x [B,N,9], t [B] int,
    z [B,N,384] -> eps [B,N,9].  masks as in oracle.train_oracle.forward."""
    P, dt = params, dtype
    B, N, _ = x.shape
    tl = t.long().cpu()
    tf = timestep_features(tl).to(device, dt)
    u1 = tf @ P["time_embed.linear.0.weight"].T + P["time_embed.linear.0.bias"]
    temb = F.silu(u1) @ P["time_embed.linear.2.weight"].T + P["time_embed.linear.2.bias"]
    pivot = torch.zeros(B, N, 1, dtype=dt, device=device)
    pivot[:, 0] = 1.0
    if x.requires_grad:
        xd = x.to(device, dt)
        octaves = 2.0 ** torch.arange(N_HARMONIC, dtype=dt, device=device)
        arg = (xd[..., None] * octaves).reshape(B, N, -1)
        harm = torch.cat([arg.sin(), arg.cos(), xd], dim=-1)
    else:
        harm = harmonic_features(x.detach().float().cpu()).to(device, dt)
    feed = torch.cat([harm, temb[:, None, :].expand(B, N, -1), z.to(device, dt), pivot], dim=-1)
    h = _linear(feed, P["_first.weight"], P["_first.bias"], tf32)
    scale = 1.0 / math.sqrt(D_MODEL // HEADS)
    for l in range(LAYERS):
        pre = f"_trunk.layers.{l}."
        a1 = F.layer_norm(h, (D_MODEL,), P[pre + "norm1.weight"], P[pre + "norm1.bias"], 1e-5)
        qkv = _linear(a1, P[pre + "self_attn.in_proj_weight"], P[pre + "self_attn.in_proj_bias"], tf32)
        q, k, v = (m.reshape(B, N, HEADS, -1).transpose(1, 2) for m in qkv.split(D_MODEL, dim=-1))
        probs = torch.softmax((q @ k.transpose(-1, -2)) * scale, dim=-1)
        att = (_drop(probs, masks, (l, 0), p) @ v).transpose(1, 2).reshape(B, N, D_MODEL)
        y = _linear(att, P[pre + "self_attn.out_proj.weight"], P[pre + "self_attn.out_proj.bias"], tf32)
        h = h + _drop(y, masks, (l, 1), p)
        a2 = F.layer_norm(h, (D_MODEL,), P[pre + "norm2.weight"], P[pre + "norm2.bias"], 1e-5)
        f = _drop(torch.relu(_linear(a2, P[pre + "linear1.weight"], P[pre + "linear1.bias"], tf32)), masks, (l, 2), p)
        h = h + _drop(_linear(f, P[pre + "linear2.weight"], P[pre + "linear2.bias"], tf32), masks, (l, 3), p)
    u = _linear(h, P["_last.0.weight"], P["_last.0.bias"], tf32)
    r = torch.relu(F.layer_norm(u, (u.shape[-1],), P["_last.1.weight"], P["_last.1.bias"], 1e-5))
    return r @ P["_last.3.weight"].T + P["_last.3.bias"]


def eps_and_grads(state: Dict[str, torch.Tensor], x, t, z, grad_eps, masks=None, p: float = 0.0, tf32: Optional[str] = None,
                  names: Optional[Sequence[str]] = None, dtype: torch.dtype = torch.float64, device="cpu", seed: Optional[int] = None):
    """(eps, {name: dL/d param}, dL/dx, dL/dz) of L = sum(grad_eps * eps), all detached on the CPU.  With p > 0 and `seed` (and
    no `masks`), the masks are the kernels' Philox masks of the whole batch."""
    params = {k: v.detach().to(device, dtype).requires_grad_(True) for k, v in state.items()}
    if masks is None and p > 0:
        masks = dropout_masks(seed, 0, x.shape[0], x.shape[1], p)
    xx = x.detach().to(device, dtype).requires_grad_(True)
    zz = z.detach().to(device, dtype).requires_grad_(True)
    eps = denoiser_eps(params, xx, t, zz, masks, p, tf32, dtype, device)
    names = list(names or params)
    g = torch.autograd.grad((eps * grad_eps.to(device, dtype)).sum(), [params[n] for n in names] + [xx, zz], allow_unused=True)
    grads = {n: (gi if gi is not None else torch.zeros_like(params[n])).detach().cpu() for n, gi in zip(names, g[:-2])}
    return eps.detach().cpu(), grads, g[-2].detach().cpu(), g[-1].detach().cpu()
