"""Float64 restatement of the reference's training step -- TEST INFRASTRUCTURE.

GaussianDiffusion.p_losses (models/gaussian_diffuser.py:211-216, 308-341) around Denoiser.forward (models/denoiser.py:53-76) with
nn.TransformerEncoderLayer's pre-norm layer written out (self-attention, dropout on the attention weights, after the out-projection,
after the ReLU and after linear2), so that dropout masks can be injected instead of drawn.  The backward is torch autograd in
float64.  `tf32="trunc"` or `"rn"` rounds every operand of the projections (forward and both backward products) to TF32 the way
the tensor-core engine reads them, truncating or rounding to nearest; attention, LayerNorm, the time MLP and `_last.3` stay
unrounded, as they run on the CUDA cores.  Tests derive their tolerances from the distance between the rounded and the exact run.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from oracle.pose_oracle import diffusion_schedule, harmonic_features, timestep_features

D_MODEL, HEADS, LAYERS = 512, 4, 8


def tf32_round(x: torch.Tensor, mode: Optional[str]) -> torch.Tensor:
    """x as the tensor cores read it: float32, then 13 low mantissa bits dropped ("trunc") or rounded to nearest ("rn")."""
    if mode is None:
        return x
    bits = x.detach().to(torch.float32).contiguous().view(torch.int32)
    if mode == "rn":
        bits = bits + 0x1000
    elif mode != "trunc":
        raise ValueError(f"unknown TF32 rounding {mode!r}")
    bits = bits & -8192  # ~0x1FFF
    return bits.view(torch.float32).to(x.dtype)


class _Matmul(torch.autograd.Function):
    """a @ b with TF32-rounded operands in the forward and in both backward products."""

    @staticmethod
    def forward(ctx, a, b, mode):
        ctx.save_for_backward(a, b)
        ctx.mode = mode
        return tf32_round(a, mode) @ tf32_round(b, mode)

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        r = lambda v: tf32_round(v, ctx.mode)  # noqa: E731
        return r(g) @ r(b).transpose(-1, -2), r(a).transpose(-1, -2) @ r(g), None


def _linear(x, w, b, mode):
    return _Matmul.apply(x, w.transpose(0, 1), mode) + b


def _drop(x, masks, key, p):
    if masks is None:
        return x
    return x * masks[key].to(x.dtype) / (1.0 - p)


def forward(params: Dict[str, torch.Tensor], x_start, t, noise, z, loss_type: str = "l1", masks: Optional[Dict[Tuple[int, int], torch.Tensor]] = None,
            p: float = 0.0, tf32: Optional[str] = None, dtype: torch.dtype = torch.float64) -> Dict[str, torch.Tensor]:
    """params: the 108 denoiser tensors by state_dict name (float64, may require grad); x_start / noise [B,N,9], t [B] int, z [B,N,384].
    masks[(layer, site)]: keep masks, site 0 [B,4,N,N], sites 1 and 3 [B,N,512], site 2 [B,N,1024]."""
    P = params
    dt = dtype
    sched = {k: v.to(dt) for k, v in diffusion_schedule().items()}
    B, N, _ = x_start.shape
    tl = t.long().cpu()
    col = lambda name: sched[name][tl].view(B, 1, 1)  # noqa: E731
    x_start, noise, z = x_start.to(dt), noise.to(dt), z.to(dt)
    x_t = col("sqrt_alphas_cumprod") * x_start + col("sqrt_one_minus_alphas_cumprod") * noise
    tf = timestep_features(tl).to(dt)
    u1 = tf @ P["time_embed.linear.0.weight"].T + P["time_embed.linear.0.bias"]
    temb = F.silu(u1) @ P["time_embed.linear.2.weight"].T + P["time_embed.linear.2.bias"]
    pivot = torch.zeros(B, N, 1, dtype=dt)
    pivot[:, 0] = 1.0
    feed = torch.cat([harmonic_features(x_t.float()).to(dt), temb[:, None, :].expand(B, N, -1), z, pivot], dim=-1)
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
    eps = r @ P["_last.3.weight"].T + P["_last.3.bias"]
    x0 = col("sqrt_recip_alphas_cumprod") * x_t - col("sqrt_recipm1_alphas_cumprod") * eps
    if loss_type == "l1":
        loss = (eps - noise).abs()
    elif loss_type == "l2":
        loss = (eps - noise) ** 2
    else:
        raise ValueError(f"invalid loss type {loss_type}")
    return {"x_t": x_t, "eps": eps, "x_0_pred": x0, "loss": loss}


def loss_and_grads(state: Dict[str, torch.Tensor], x_start, t, noise, z, grad_loss, grad_x0=None, loss_type: str = "l1", masks=None,
                   p: float = 0.0, tf32: Optional[str] = None, names: Optional[Sequence[str]] = None,
                   dtype: torch.dtype = torch.float64):
    """forward() plus d(sum(grad_loss * loss) + sum(grad_x0 * x_0_pred)) / d params on the CPU, in float64 unless `dtype` says
    otherwise (float32 gives the distance an fp32 evaluation of the same step has from float64)."""
    params = {k: v.detach().to("cpu", dtype).requires_grad_(True) for k, v in state.items()}
    out = forward(params, x_start.cpu(), t.cpu(), noise.cpu(), z.cpu(), loss_type, masks, p, tf32, dtype)
    total = (out["loss"] * grad_loss.cpu().to(dtype)).sum()
    if grad_x0 is not None:
        total = total + (out["x_0_pred"] * grad_x0.cpu().to(dtype)).sum()
    names = list(names or params)
    grads = torch.autograd.grad(total, [params[n] for n in names], allow_unused=True)
    return {k: v.detach() for k, v in out.items()}, {n: (g if g is not None else torch.zeros_like(params[n])) for n, g in zip(names, grads)}


def matrix_to_quaternion(matrix: torch.Tensor) -> torch.Tensor:
    """pytorch3d's matrix_to_quaternion followed by standardize_quaternion (real part >= 0), the convention the package's
    camera_to_pose_encoding implements (DESIGN.md, Training)."""
    m = matrix.reshape(matrix.shape[:-2] + (9,))
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = m.unbind(-1)
    arg = torch.stack([1.0 + m00 + m11 + m22, 1.0 + m00 - m11 - m22, 1.0 - m00 + m11 - m22, 1.0 - m00 - m11 + m22], dim=-1)
    q_abs = torch.where(arg > 0, arg.clamp(min=0).sqrt(), torch.zeros_like(arg))
    cand = torch.stack([
        torch.stack([q_abs[..., 0] ** 2, m21 - m12, m02 - m20, m10 - m01], dim=-1),
        torch.stack([m21 - m12, q_abs[..., 1] ** 2, m10 + m01, m02 + m20], dim=-1),
        torch.stack([m02 - m20, m10 + m01, q_abs[..., 2] ** 2, m12 + m21], dim=-1),
        torch.stack([m10 - m01, m20 + m02, m21 + m12, q_abs[..., 3] ** 2], dim=-1),
    ], dim=-2)
    cand = cand / (2.0 * q_abs[..., None].clamp(min=0.1))
    idx = q_abs.argmax(dim=-1)
    out = torch.gather(cand, -2, idx[..., None, None].expand(idx.shape + (1, 4)))[..., 0, :]
    return torch.where(out[..., 0:1] < 0, -out, out)


def camera_to_pose_encoding(R, T, focal, log_focal_length_bias=1.8, min_focal_length=0.1, max_focal_length=20):
    """util/camera_transform.py:108-129 on plain tensors."""
    return torch.cat([T, matrix_to_quaternion(R), torch.log(torch.clamp(focal, min=min_focal_length, max=max_focal_length))
                      - log_focal_length_bias], dim=-1)
