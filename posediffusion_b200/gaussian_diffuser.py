"""`GaussianDiffusion` sampler with the reference's surface (models/gaussian_diffuser.py:75-306):
same constructor, the same 13 persistent schedule buffers, `.model` attached after construction,
`sample` / `p_sample_loop` / `p_sample`, and the training methods `q_sample` / `p_losses` / `forward` (:211-216, :308-341),
whose loss and gradients come from the native training kernels (csrc/api_train.cu).

`p_sample_loop` runs the whole loop natively (one persistent denoiser launch for the unguided prefix, then
denoiser + GGS launches per guided step) when `cond_fn` is None or a `partial(geometry_guided_sampling, ...)`
of this package; any other callable falls back to a Python loop around the native single-step kernel --
still CUDA-only.  Gaussian draws come from torch's generator on the sampler's device in the reference's
order (one `randn(shape)` then one `randn_like` per unguided step with t > 0, :289, :278).
"""
from __future__ import annotations

from functools import partial
from typing import Callable, Optional

import torch
import torch.nn.functional as F
from torch import nn

from . import _native
from .geometry_guided_sampling import format_log, geometry_guided_sampling, packed_matches


class GaussianDiffusion(nn.Module):
    def __init__(self, timesteps=100, sampling_timesteps=None, beta_1=0.0001, beta_T=0.1, loss_type="l1",
                 objective="pred_noise", beta_schedule="custom", p2_loss_weight_gamma=0.0, p2_loss_weight_k=1):
        super().__init__()
        assert objective in {"pred_noise", "pred_x0"}, "objective must be either pred_noise or pred_x0"
        self.timesteps, self.sampling_timesteps = timesteps, sampling_timesteps
        self.beta_1, self.beta_T = beta_1, beta_T
        self.loss_type, self.objective, self.beta_schedule = loss_type, objective, beta_schedule
        self.p2_loss_weight_gamma, self.p2_loss_weight_k = p2_loss_weight_gamma, p2_loss_weight_k
        if beta_schedule == "custom":  # the released configuration (cfgs/default.yaml); models/gaussian_diffuser.py:66-69
            betas = torch.linspace(beta_1, beta_T, timesteps, dtype=torch.float64)
        elif beta_schedule in ("linear", "cosine"):
            # the reference also offers these (:62-65); no released checkpoint uses them and the sm_90a sampler tabulates
            # the custom schedule only -- refuse at construction instead of building buffers nothing can run
            raise NotImplementedError(f"beta_schedule={beta_schedule!r}: only the released 'custom' schedule is built")
        else:
            raise ValueError(f"unknown beta schedule {beta_schedule}")
        self.num_timesteps = int(betas.shape[0])
        self.sampling_timesteps = timesteps if sampling_timesteps is None else sampling_timesteps
        assert self.sampling_timesteps <= timesteps
        abar = torch.cumprod(1.0 - betas, dim=0)
        abar_prev = F.pad(abar[:-1], (1, 0), value=1.0)
        post_var = betas * (1.0 - abar_prev) / (1.0 - abar)
        table = {  # float64 -> float32 persistent buffers, same names as the reference checkpoint
            "betas": betas,
            "alphas_cumprod": abar,
            "alphas_cumprod_prev": abar_prev,
            "sqrt_alphas_cumprod": abar.sqrt(),
            "sqrt_one_minus_alphas_cumprod": (1.0 - abar).sqrt(),
            "log_one_minus_alphas_cumprod": (1.0 - abar).log(),
            "sqrt_recip_alphas_cumprod": (1.0 / abar).sqrt(),
            "sqrt_recipm1_alphas_cumprod": (1.0 / abar - 1).sqrt(),
            "posterior_variance": post_var,
            "posterior_log_variance_clipped": post_var.clamp(min=1e-20).log(),
            "posterior_mean_coef1": betas * abar_prev.sqrt() / (1.0 - abar),
            "posterior_mean_coef2": (1.0 - abar_prev) * (1.0 - betas).sqrt() / (1.0 - abar),
            "p2_loss_weight": (p2_loss_weight_k + abar / (1 - abar)) ** -p2_loss_weight_gamma,
        }
        for name, value in table.items():
            self.register_buffer(name, value.to(torch.float32))
        self.model = None  # attached by PoseDiffusionModel (pose_diffusion_model.py:61)
        self.last_ggs_stats = None

    # ---- native eligibility -----------------------------------------------------------------------------
    def _native_ok(self) -> bool:
        from .denoiser import Denoiser

        return (
            isinstance(self.model, Denoiser)
            and self.objective == "pred_noise"
            and self.beta_schedule == "custom"
            and self.num_timesteps == _native.NUM_TIMESTEPS
            and abs(self.beta_1 - 1e-4) < 1e-12
            and abs(self.beta_T - 0.1) < 1e-12
        )

    def _require_native(self):
        if not self._native_ok():
            raise NotImplementedError(
                "the sm_90a sampler is built for the released configuration: Denoiser model, objective='pred_noise', "
                "beta_schedule='custom' (beta 1e-4..0.1), 100 timesteps"
            )

    def draw_noise(self, shape, device, guided_below: int) -> torch.Tensor:
        """[T+1, B, N, 9] Gaussian draws consumed in the reference's order on `device`'s generator."""
        T = self.num_timesteps
        draws = torch.zeros(T + 1, *shape, device=device)
        draws[0] = torch.randn(shape, device=device)
        for k, t in enumerate(reversed(range(T))):
            if t > 0 and t >= guided_below:
                draws[1 + k] = torch.randn(shape, device=device)
        return draws

    # ---- reference API ---------------------------------------------------------------------------------
    @torch.no_grad()
    def p_sample(self, x: torch.Tensor, t: int, z: torch.Tensor, x_self_cond=None, clip_denoised=False, cond_fn=None,
                 cond_start_step=0):
        if clip_denoised:
            raise NotImplementedError("We don't clip the output because pose does not have a clear bound.")
        self._require_native()
        ctx = self.model.native_context()
        guided = cond_fn is not None and t < cond_start_step
        noise = None if (guided or t == 0) else torch.randn_like(x)
        pred, mean, x0 = ctx.p_sample(x.contiguous().float(), int(t), z.contiguous().float(), noise)
        if guided:
            pred = cond_fn(mean, t)
        return pred, x0

    @torch.no_grad()
    def p_sample_loop(self, shape, z: torch.Tensor, cond_fn: Optional[Callable] = None, cond_start_step: int = 0,
                      draws: Optional[torch.Tensor] = None):
        self._require_native()
        device = self.betas.device
        ctx = self.model.native_context()
        z = z.contiguous().float()
        fused = cond_fn is None or (
            isinstance(cond_fn, partial) and cond_fn.func is geometry_guided_sampling and not cond_fn.args
            and set(cond_fn.keywords) == {"matches_dict", "GGS_cfg"}
        )
        guided_below = cond_start_step if cond_fn is not None else 0
        if draws is None:
            draws = self.draw_noise(tuple(shape), device, guided_below)
        if fused:
            problems = cfg = None
            if cond_fn is not None:
                cfg = cond_fn.keywords["GGS_cfg"]
                problems = packed_matches(ctx, cond_fn.keywords["matches_dict"])
            pose, trail, stats = ctx.sample_loop(z, draws.contiguous(), problems, cfg, cond_start_step)
            self.last_ggs_stats = stats
            if stats is not None and bool(cfg.get("verbose", True)):
                rows = _native.stats_to_numpy(stats).reshape(-1, shape[0])
                for i, per_step in enumerate(rows):
                    for row in per_step:
                        print("\n".join(format_log(min(cond_start_step, self.num_timesteps) - 1 - i, row)))
            return pose, trail
        # generic cond_fn: Python loop around the native step
        pose = draws[0].clone()
        trail = [pose.unsqueeze(0)]
        for k, t in enumerate(reversed(range(self.num_timesteps))):
            guided = t < cond_start_step
            noise = None if (guided or t == 0) else draws[1 + k]
            pred, mean, _ = ctx.p_sample(pose, t, z, noise)
            pose = cond_fn(mean, t) if guided else pred
            trail.append(pose.unsqueeze(0))
        return pose, torch.cat(trail)

    @torch.no_grad()
    def sample(self, shape, z, cond_fn=None, cond_start_step=0):
        return self.p_sample_loop(shape, z=z, cond_fn=cond_fn, cond_start_step=cond_start_step)

    # ---- training (models/gaussian_diffuser.py:211-216, 308-341) ------------------------------------------
    def _extract(self, a: torch.Tensor, t: torch.Tensor, x_shape) -> torch.Tensor:
        return a.gather(-1, t).reshape(t.shape[0], *((1,) * (len(x_shape) - 1)))

    def q_sample(self, x_start: torch.Tensor, t: torch.Tensor, noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        """x_t = sqrt(abar_t) x_start + sqrt(1 - abar_t) noise.  p_losses evaluates the same inside its first kernel."""
        noise = torch.randn_like(x_start) if noise is None else noise
        return (self._extract(self.sqrt_alphas_cumprod, t, x_start.shape) * x_start
                + self._extract(self.sqrt_one_minus_alphas_cumprod, t, x_start.shape) * noise)

    @property
    def loss_fn(self):
        if self.loss_type == "l1":
            return F.l1_loss
        elif self.loss_type == "l2":
            return F.mse_loss
        raise ValueError(f"invalid loss type {self.loss_type}")

    def p_losses(self, x_start: torch.Tensor, t: torch.Tensor, z: torch.Tensor = None, noise: Optional[torch.Tensor] = None):
        """The diffusion loss of the denoiser in one native forward (q_sample, Denoiser, x_0 prediction, element-wise loss) whose
        backward returns the 108 denoiser parameter gradients.  Dropout follows the denoiser's train()/eval() mode; its masks come
        from one 64-bit seed drawn after the noise on the device generator."""
        self.loss_fn  # noqa: B018 -- ValueError for an unknown loss type, as the reference raises it
        if self.objective != "pred_noise":
            raise NotImplementedError("objective='pred_x0' is not built: the native denoiser is trained for 'pred_noise'")
        self._require_native()
        if z is None:
            raise ValueError("p_losses needs the image features z [B,N,384]")
        noise = torch.randn_like(x_start) if noise is None else noise
        den = self.model
        p = den.dropout_p if den.training else 0.0
        seed = torch.randint(0, 2**63 - 1, (1,), device=x_start.device)  # read with the timestep check: one synchronisation
        loss, x_0_pred, x_t = den.train_step_forward(x_start, t, noise, z, p, seed, self.loss_type)
        return {"loss": loss, "noise": noise, "x_0_pred": x_0_pred, "x_t": x_t, "t": t}

    def forward(self, pose: torch.Tensor, z: torch.Tensor = None, *args, **kwargs):
        b = len(pose)
        t = torch.randint(0, self.num_timesteps, (b,), device=pose.device).long()
        return self.p_losses(pose, t, z=z, *args, **kwargs)
