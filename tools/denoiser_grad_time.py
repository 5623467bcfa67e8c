#!/usr/bin/env python
"""Time forward + backward through the differentiable Denoiser.forward (Denoiser.enable_autograd) at the released recipe's shapes.

    python tools/denoiser_grad_time.py [--steps 10] [--warmup 3] [--repeat 90] [--out FILE] [--no-reference]

Shapes are sequences x frames before batch_repeat (cfgs/default_train.yaml repeats every batch 90 times).  Timed per shape, in one
process on one GPU, with CUDA events after warm-up (tools/train_step_time.py's method), in train() mode (dropout 0.1):
  native_all        eps = Denoiser(x, t, z), backward of sum(g * eps) into all 108 parameters and x;
  native_dx         the same with every parameter frozen: dL/dx only (the input-gradient chain, no weight-gradient GEMMs);
  native_p_losses   GaussianDiffusion.p_losses + loss.mean().backward() (the fused training step, for comparison);
  reference_fp32 / reference_tf32   the reference's own models.Denoiser (oracle/_ref, installed by build()) under torch autograd,
                    into all parameters and x, with allow_tf32 off / on.
Printed per run: median and range of the step time and the peak memory allocated; the card's name, power limit and maximum SM
clock are read in the same call.  Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from train_step_time import card, time_steps  # noqa: E402

SHAPES = [(51, 10), (10, 50)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeat", type=int, default=90)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("denoiser_grad_time needs a CUDA device")
    import posediffusion_b200 as pdb
    from posediffusion_b200 import synthetic as syn

    dev = torch.device("cuda:0")
    state = syn.random_denoiser_state(0, 0.02)
    cfg = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)
    den = pdb.Denoiser(TRANSFORMER=cfg)
    den.load_state_dict(state)
    den = den.to(dev).train().enable_autograd()
    dif = pdb.GaussianDiffusion()
    dif.model = den
    dif = dif.to(dev).train()
    rden = None
    if not args.no_reference:
        from oracle import ref_loader

        ref = ref_loader.load_reference()
        rden = ref.Denoiser(TRANSFORMER=ref.to_attr(ref_loader.TRANSFORMER_CFG))
        rden.load_state_dict(state)
        rden = rden.to(dev).train()
    name = card()
    lines = []
    for seqs, frames in SHAPES:
        B = seqs * args.repeat
        g = torch.Generator(device=dev).manual_seed(seqs)
        x = torch.randn(B, frames, 9, device=dev, generator=g)
        z = torch.randn(B, frames, 384, device=dev, generator=g)
        ge = torch.randn(B, frames, 9, device=dev, generator=g)
        t = torch.randint(0, 100, (B,), device=dev, generator=g)

        def through(model, params_trainable):
            params = list(model.parameters())

            def step():
                for p in params:
                    p.requires_grad_(params_trainable)
                    p.grad = None
                xx = x.detach().requires_grad_(True)
                (model(xx, t, z) * ge).sum().backward()

            return step

        def p_losses_step():
            for p in den.parameters():
                p.requires_grad_(True)
                p.grad = None
            dif.p_losses(x, t, z)["loss"].mean().backward()

        runs = [("native_all", through(den, True), None), ("native_dx", through(den, False), None),
                ("native_p_losses", p_losses_step, None)]
        if rden is not None:
            runs += [("reference_fp32", through(rden, True), False), ("reference_tf32", through(rden, True), True)]
        for label, step, tf32 in runs:
            torch.backends.cuda.matmul.allow_tf32 = bool(tf32)
            torch.backends.cudnn.allow_tf32 = bool(tf32)
            torch.cuda.empty_cache()
            times, peak = time_steps(step, args.steps, args.warmup)
            med = times[len(times) // 2]
            rec = {"impl": label, "sequences": B, "frames": frames, "tokens": B * frames, "ms_median": round(med, 3),
                   "ms_min": round(times[0], 3), "ms_max": round(times[-1], 3), "runs": len(times), "warmup": args.warmup,
                   "peak_mem_gib": round(peak / 2**30, 2), "card": name}
            lines.append(rec)
            print(json.dumps(rec), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            for rec in lines:
                fh.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
