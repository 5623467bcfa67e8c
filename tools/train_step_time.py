#!/usr/bin/env python
"""Time one training step (GaussianDiffusion.p_losses forward + loss.mean().backward()) at the released recipe's shapes.

    python tools/train_step_time.py [--steps 10] [--warmup 3] [--repeat 90] [--out FILE]

cfgs/default_train.yaml draws 3..51 frames per sequence and repeats every batch 90 times (batch_repeat); at max_images 512 the
shapes below carry about 46 000 tokens per step.  For each shape the native path (this package) and the reference's own modules
(oracle/_ref, installed by build(); torch autograd, fp32 with allow_tf32 off and on) are timed with CUDA events after warm-up, on
the same GPU, in one process.  Printed per run: median and range of the step time, tokens/s, achieved TFLOP/s from the
shape-derived count below and its share of the 495 TFLOP/s dense-TF32 data-sheet figure of the H100 SXM, and the peak memory
allocated.  The card's name and power limit are read in the same call.  Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SHAPES = [(51, 10), (10, 50), (170, 3)]  # sequences x frames before batch_repeat
TF32_PEAK = 495e12


def forward_flop_per_token(frames: int) -> float:
    """Multiply-adds x 2 of the denoiser forward per token: projections, attention scores and P.V, _last, the t-MLP per sequence."""
    proj = 702 * 512 + 8 * (512 * 1536 + 512 * 512 + 512 * 1024 + 1024 * 512) + 512 * 128 + 128 * 9
    attn = 8 * 2 * frames * 512
    tmlp = (256 * 128 + 128 * 128) / frames
    return 2.0 * (proj + attn + tmlp)


def step_flop(seqs: int, frames: int) -> float:
    return 3.0 * forward_flop_per_token(frames) * seqs * frames  # backward = two products per forward product


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def time_steps(step, steps: int, warmup: int):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times, torch.cuda.max_memory_allocated()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeat", type=int, default=90)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_step_time needs a CUDA device")
    import posediffusion_b200 as pdb
    from posediffusion_b200 import synthetic as syn

    dev = torch.device("cuda:0")
    state = syn.random_denoiser_state(0, 0.02)
    cfg = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)
    impls = {}
    den = pdb.Denoiser(TRANSFORMER=cfg)
    den.load_state_dict(state)
    dif = pdb.GaussianDiffusion()
    dif.model = den
    impls["native"] = (dif.to(dev).train(), None)
    if not args.no_reference:
        from oracle import ref_loader

        ref = ref_loader.load_reference()
        rden = ref.Denoiser(TRANSFORMER=ref.to_attr(ref_loader.TRANSFORMER_CFG))
        rden.load_state_dict(state)
        rdif = ref.GaussianDiffusion(beta_schedule="custom")
        rdif.model = rden
        rdif = rdif.to(dev).train()
        impls["reference_fp32"] = (rdif, False)
        impls["reference_tf32"] = (rdif, True)
    name = card()
    lines = []
    for seqs, frames in SHAPES:
        B = seqs * args.repeat
        g = torch.Generator(device=dev).manual_seed(seqs)
        pose = torch.randn(B, frames, 9, device=dev, generator=g) * 0.5
        z = torch.randn(B, frames, 384, device=dev, generator=g)
        for label, (model, tf32) in impls.items():
            if tf32 is not None:
                torch.backends.cuda.matmul.allow_tf32 = tf32
                torch.backends.cudnn.allow_tf32 = tf32
            params = [p for p in model.parameters() if p.requires_grad]

            def step():
                for p in params:
                    p.grad = None
                model(pose, z=z)["loss"].mean().backward()

            torch.cuda.empty_cache()
            times, peak = time_steps(step, args.steps, args.warmup)
            med = times[len(times) // 2]
            flop = step_flop(B, frames)
            rec = {"impl": label, "sequences": B, "frames": frames, "tokens": B * frames, "ms_median": round(med, 3),
                   "ms_min": round(times[0], 3), "ms_max": round(times[-1], 3), "steps": len(times),
                   "tokens_per_s": round(B * frames / (med * 1e-3)), "tflop_per_step": round(flop / 1e12, 3),
                   "tflop_per_s": round(flop / (med * 1e-3) / 1e12, 2), "share_of_tf32_datasheet": round(flop / (med * 1e-3) / TF32_PEAK, 4),
                   "peak_mem_gib": round(peak / 2**30, 2), "card": name}
            if label == "native":
                from posediffusion_b200 import _native

                rec["workspace_gib"] = round(_native.train_workspace_bytes(B, frames) / 2**30, 2)
            print(json.dumps(rec), flush=True)
            lines.append(rec)
        torch.backends.cuda.matmul.allow_tf32 = False
    if args.out:
        with open(args.out, "w") as fh:
            for rec in lines:
                fh.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
