"""Guided DDIM jumps restated on the oracle -- TEST INFRASTRUCTURE, next to tests/ddim_oracle.py.

`GaussianDiffusion.ddim_sample(..., guided_steps=g')` / `pdb_sample_loop_ddim_guided` take the guided tail over timesteps g-1 .. 0
in g' DDIM jumps: jump times from their integer formula, coefficients from `ddim_oracle.ddim_coef_f64`, and one jump in float64 with
the fp32 oracle's distance d32 (`guided_jump_f64`).  A guided jump adds no noise; cond_fn (GGS) then runs on its mean.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import torch

import ddim_oracle as dd


def guided_times(g: int, gs: int) -> List[int]:
    """tau'_0 .. tau'_{g'} = floor(j g / g') - 1: tau'_{g'} = g - 1 (where the prefix lands), tau'_0 = -1 (x0)."""
    return [(j * g) // gs - 1 for j in range(gs + 1)]


def guided_jumps(g: int, gs: int, eta: float) -> List[Tuple[int, int, Dict[str, float]]]:
    """(t, s, float64 coefficients) of the g' guided jumps, in the order they run."""
    tau, abar = guided_times(g, gs), dd.alphas_cumprod_f64()
    return [(tau[j], tau[j - 1], dd.ddim_coef_f64(tau[j], tau[j - 1], eta, abar)) for j in range(gs, 0, -1)]


@torch.no_grad()
def guided_jump_f64(den, x: torch.Tensor, t: int, s: int, eta: float, z: torch.Tensor):
    """The pre-guidance mean of one guided jump t -> s in float64 on the float32-rounded coefficients, and the fp32 oracle's
    distance from it: (mean f64, d32)."""
    mean, _x0, d32, _ = dd.ddim_step_f64(den, x, t, s, eta, z, None)
    return mean, d32
