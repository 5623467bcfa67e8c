"""Float64 evaluation of the denoiser and of one DDPM step -- TEST INFRASTRUCTURE.

The arbiter for the fp32 kernels: `po.build_denoiser(state).double()` is the reference's network evaluated in float64.  The
sinusoidal timestep features stay what the reference computes, float32 (`po.timestep_features`; the library tabulates the same
float32 values), and are widened to float64 before the time MLP.  That happens in a wrapper installed on the one network
instance, not by patching `pose_oracle`.

`noise_f64` also evaluates the fp32 oracle: d32 = max |eps_fp32 - eps_f64| is the reference's own rounding noise at that shape
and the scale of the bound `4 * d32 + 1e-6` the device tests apply (DESIGN.md section 2).
"""
from __future__ import annotations

from typing import Dict, Tuple

import torch
import torch.nn as nn

from . import pose_oracle as po


class _TimeEmbedF64(nn.Module):
    """time_embed of OracleDenoiser with the float32 features cast to float64 (the MLP itself runs in float64)."""

    def __init__(self, linear: nn.Sequential):
        super().__init__()
        self.linear = linear

    def forward(self, t):
        return self.linear(po.timestep_features(t).double())


class DenoiserF64:
    """The fp32 oracle and its float64 twin over the same weights."""

    def __init__(self, state: Dict[str, torch.Tensor]):
        self.net32 = po.build_denoiser(state)
        self.net64 = po.build_denoiser(state).double()
        self.net64.time_embed = _TimeEmbedF64(self.net64.time_embed.linear)
        self.sched = po.diffusion_schedule()  # float32 buffers, as the reference and the library hold them

    @torch.no_grad()
    def noise_f64(self, x: torch.Tensor, t: int, z: torch.Tensor) -> Tuple[torch.Tensor, float]:
        """(eps in float64, d32) for x [B,N,9], one timestep t for the whole batch, z [B,N,384] (CPU tensors)."""
        x, z = x.detach().cpu(), z.detach().cpu()
        steps = torch.full((x.shape[0],), int(t), dtype=torch.long)
        eps64 = self.net64(x.double(), steps, z.double())
        eps32 = self.net32(x.float(), steps, z.float())
        return eps64, (eps32.double() - eps64).abs().max().item()

    @torch.no_grad()
    def p_sample_f64(self, x: torch.Tensor, t: int, z: torch.Tensor, noise) -> Tuple[torch.Tensor, torch.Tensor, float, float]:
        """po.p_sample (unguided) restated in float64 on the float32 schedule values: (x_{t-1}, x0, d32 of x_{t-1}, d32 of x0).
        No noise at t = 0."""
        x, z = x.detach().cpu(), z.detach().cpu()
        steps = torch.full((x.shape[0],), int(t), dtype=torch.long)
        out = []
        for net, dt in ((self.net64, torch.float64), (self.net32, torch.float32)):
            xd = x.to(dt)
            eps = net(xd, steps, z.to(dt))
            c = {k: self.sched[k][t].to(dt) for k in ("sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod",
                                                         "posterior_mean_coef1", "posterior_mean_coef2")}
            x0 = c["sqrt_recip_alphas_cumprod"] * xd - c["sqrt_recipm1_alphas_cumprod"] * eps
            pred = c["posterior_mean_coef1"] * x0 + c["posterior_mean_coef2"] * xd
            if t > 0:
                sigma = (0.5 * self.sched["posterior_log_variance_clipped"][t]).exp().to(dt)
                pred = pred + sigma * noise.detach().cpu().to(dt)
            out.append((pred, x0))
        (pred64, x064), (pred32, x032) = out
        return pred64, x064, (pred32.double() - pred64).abs().max().item(), (x032.double() - x064).abs().max().item()


def bound(d32: float, scale: float = 1.0) -> float:
    """max |device - float64| allowed for the fp32 engine: four times the fp32 oracle's own distance, plus 1e-6 of the output's
    magnitude (at least 1: eps is O(0.1..1))."""
    return 4.0 * d32 + 1e-6 * max(1.0, scale)
