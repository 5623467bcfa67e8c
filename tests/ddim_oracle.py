"""DDIM (Song et al. 2021, eq. 12) restated on the oracle denoiser -- TEST INFRASTRUCTURE.

The fewer-step sampler of `GaussianDiffusion.ddim_sample` / `pdb_sample_loop_ddim`, written out independently of the library:
the step times and coefficients from their float64 formulas, `ddim_sample_loop` in fp32 on `oracle.pose_oracle`'s denoiser with
the same `cond_fn` tail as `po.p_sample_loop`, and `ddim_step_f64`, one DDIM step in float64 with the fp32 oracle's distance d32
for `oracle.denoiser_f64.bound`.
"""
from __future__ import annotations

import math
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np
import torch

from oracle import pose_oracle as po

T = 100


def ddim_times(k: int, g: int) -> List[int]:
    """tau_0 .. tau_k = (g - 1) + floor(j (T - g) / k): tau_k = 99, tau_0 = g - 1 (-1 = x0)."""
    return [(g - 1) + (j * (T - g)) // k for j in range(k + 1)]


def alphas_cumprod_f64(beta_1: float = 1e-4, beta_T: float = 0.1) -> np.ndarray:
    beta = torch.linspace(beta_1, beta_T, T, dtype=torch.float64)
    return torch.cumprod(1.0 - beta, 0).numpy()


def ddim_coef_f64(t: int, s: int, eta: float, abar: np.ndarray) -> Dict[str, float]:
    """x_s = c1 (a x_t - b eps) + c2 x_t + sigma noise, abar_{-1} = 1."""
    at = float(abar[t])
    as_ = 1.0 if s < 0 else float(abar[s])
    sigma = eta * math.sqrt((1.0 - as_) / (1.0 - at)) * math.sqrt(1.0 - at / as_)
    c2 = math.sqrt(1.0 - as_ - sigma * sigma) / math.sqrt(1.0 - at)
    c1 = math.sqrt(as_) - c2 * math.sqrt(at)
    return {"a": math.sqrt(1.0 / at), "b": math.sqrt(1.0 / at - 1.0), "c1": c1, "c2": c2, "sigma": sigma}


def prefix_steps(k: int, g: int, eta: float) -> List[Tuple[int, int, Dict[str, float]]]:
    """(t, s, float64 coefficients) of the k unguided DDIM steps, in the order they run."""
    tau, abar = ddim_times(k, g), alphas_cumprod_f64()
    return [(tau[j], tau[j - 1], ddim_coef_f64(tau[j], tau[j - 1], eta, abar)) for j in range(k, 0, -1)]


def _f32(c: Dict[str, float]) -> Dict[str, torch.Tensor]:
    return {n: torch.tensor(v, dtype=torch.float64).float() for n, v in c.items()}


@torch.no_grad()
def ddim_step(net, x: torch.Tensor, t: int, z: torch.Tensor, coef: Dict[str, float], noise: Optional[torch.Tensor]):
    """One fp32 DDIM step on the float32-rounded coefficients: (x_s, x0)."""
    c = _f32(coef)
    eps = net(x, torch.full((x.shape[0],), t, dtype=torch.long), z)
    x0 = c["a"] * x - c["b"] * eps
    out = c["c1"] * x0 + c["c2"] * x
    if noise is not None and coef["sigma"] > 0:
        out = out + c["sigma"] * noise
    return out, x0


@torch.no_grad()
def ddim_sample_loop(net, sched, z: torch.Tensor, draws: torch.Tensor, k: int, eta: float, cond_fn: Optional[Callable] = None,
                     cond_start_step: int = 0):
    """draws[0] = x_T, draws[1 + i] = noise of prefix step i (eta > 0).  The guided tail t = g-1 .. 0 (g = cond_start_step when
    cond_fn is given) is po.p_sample's.  Returns (pose, trail [1 + k + g, B, N, 9])."""
    g = max(0, min(int(cond_start_step), T)) if cond_fn is not None else 0
    pose = draws[0].clone()
    trail = [pose.clone()]
    for i, (t, _s, coef) in enumerate(prefix_steps(k, g, eta)):
        pose, _ = ddim_step(net, pose, t, z, coef, draws[1 + i] if eta > 0 else None)
        trail.append(pose.clone())
    for t in reversed(range(g)):
        pose, _ = po.p_sample(net, sched, pose, t, z, None, cond_fn, g)
        trail.append(pose.clone())
    return pose, torch.stack(trail)


@torch.no_grad()
def ddim_step_f64(den, x: torch.Tensor, t: int, s: int, eta: float, z: torch.Tensor, noise: Optional[torch.Tensor]):
    """One DDIM step t -> s in float64 on the float32-rounded coefficients (den: oracle.denoiser_f64.DenoiserF64), and the fp32
    oracle's distance from it: (x_s f64, x0 f64, d32 of x_s, d32 of x0)."""
    coef = ddim_coef_f64(t, s, eta, alphas_cumprod_f64())
    c = {n: v.double() for n, v in _f32(coef).items()}
    x, z = x.detach().cpu(), z.detach().cpu()
    steps = torch.full((x.shape[0],), int(t), dtype=torch.long)
    out = []
    for net, dt in ((den.net64, torch.float64), (den.net32, torch.float32)):
        xd = x.to(dt)
        eps = net(xd, steps, z.to(dt))
        x0 = c["a"].to(dt) * xd - c["b"].to(dt) * eps
        xs = c["c1"].to(dt) * x0 + c["c2"].to(dt) * xd
        if noise is not None and coef["sigma"] > 0:
            xs = xs + c["sigma"].to(dt) * noise.detach().cpu().to(dt)
        out.append((xs, x0))
    (xs64, x064), (xs32, x032) = out
    return xs64, x064, (xs32.double() - xs64).abs().max().item(), (x032.double() - x064).abs().max().item()
