#!/usr/bin/env python
"""Time the image backbone's training step (multi-scale DINO ViT-S/16 forward + backward) and the whole released step.

    python tools/vit_train_time.py [--steps 10] [--warmup 3] [--out FILE]

cfgs/default_train.yaml fine-tunes the backbone (`freeze: False`) on up to 512 images of 224^2 per step at scales (1, 1/2, 1/3):
264 tokens per image.  For 512, 200 and 30 images the native path (this package) and oracle/dino_vit.py under torch autograd
(fp32 with allow_tf32 off and on) are timed on the same GPU in one process: median and range of the step time after warm-up, each
step ending in a synchronise, tokens/s, achieved TFLOP/s from the shape-derived count below, and the peak memory allocated.
Then the whole released step through PoseDiffusionModel: 51 sequences x 10 frames through the backbone, repeated 90 times
through the denoiser.  The card's name, power limit and maximum SM clock are read in the same call.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

IMAGES = [512, 200, 30]
SCALES = (1, 1 / 2, 1 / 3)
TOKENS = (197, 50, 17)  # per 224^2 image at SCALES


def step_flop(n_images: int) -> float:
    """Multiply-adds x 2 of the forward (patch embedding, the four projections and both attention products of 12 blocks), times
    three: the backward is two products per forward product."""
    fwd = 0.0
    for L in TOKENS:
        per_token = 12 * (384 * 1152 + 384 * 384 + 2 * 384 * 1536 + 2 * L * 384)
        fwd += 2.0 * n_images * (L * per_token + (L - 1) * 768 * 384)
    return 3.0 * fwd


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
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        step()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    times.sort()
    return times, torch.cuda.max_memory_allocated()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-torch", action="store_true")
    ap.add_argument("--images", type=int, nargs="*", default=IMAGES)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vit_train_time needs a CUDA device")
    import posediffusion_b200 as pdb
    from oracle.dino_vit import RESNET_MEAN, RESNET_STD, DinoViTSmall16, randomize
    from posediffusion_b200 import _native
    from posediffusion_b200 import synthetic as syn

    dev = torch.device("cuda:0")
    vit = randomize(DinoViTSmall16(), 0)
    ext = pdb.MultiScaleImageFeatureExtractor(freeze=False)
    ext._net.load_state_dict(vit.state_dict())
    ext = ext.to(dev)
    vit = vit.to(dev)
    mean, std = torch.tensor(RESNET_MEAN, device=dev).view(1, 3, 1, 1), torch.tensor(RESNET_STD, device=dev).view(1, 3, 1, 1)

    def torch_features(img):
        normed = (img - mean) / std
        total = None
        for f in SCALES:
            feat = vit(normed if f == 1 else F.interpolate(normed, scale_factor=f, mode="bilinear", align_corners=False))
            total = feat if total is None else total + feat
        return total / len(SCALES)

    name = card()
    lines = []

    def report(rec):
        rec["card"] = name
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    arms = [("native", None)] + ([] if args.no_torch else [("torch_fp32", False), ("torch_tf32", True)])
    for n in args.images:
        img = torch.rand(n, 3, 224, 224, device=dev, generator=torch.Generator(device=dev).manual_seed(n))
        g = torch.randn(n, 384, device=dev, generator=torch.Generator(device=dev).manual_seed(n + 1))
        for label, tf32 in arms:
            if tf32 is not None:
                torch.backends.cuda.matmul.allow_tf32 = tf32
                torch.backends.cudnn.allow_tf32 = tf32
            module, fn = (ext, ext) if label == "native" else (vit, torch_features)

            def step():
                for p in module.parameters():
                    p.grad = None
                fn(img).backward(g)

            torch.cuda.empty_cache()
            tokens, flop = n * sum(TOKENS), step_flop(n)
            try:
                times, peak = time_steps(step, args.steps, args.warmup)
            except torch.OutOfMemoryError:
                module.zero_grad(set_to_none=True)
                report({"impl": label, "images": n, "tokens": tokens, "result": "out of memory"})
                continue
            med = times[len(times) // 2]
            rec = {"impl": label, "images": n, "tokens": tokens, "ms_median": round(med, 2), "ms_min": round(times[0], 2),
                   "ms_max": round(times[-1], 2), "steps": len(times), "tokens_per_s": round(tokens / (med * 1e-3)),
                   "tflop_per_step": round(flop / 1e12, 3), "tflop_per_s": round(flop / (med * 1e-3) / 1e12, 2),
                   "peak_mem_gib": round(peak / 2**30, 2)}
            if label == "native":
                rec["workspace_gib"] = round(_native.vit_train_workspace_bytes(n, 224, 224, SCALES) / 2**30, 2)
            report(rec)
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.allow_tf32 = False
        del img, g

    # the whole released step: backbone on 51 x 10 images, denoiser on the features repeated 90 times
    cfg_t = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)
    model = pdb.PoseDiffusionModel(
        pose_encoding_type="absT_quaR_logFL",
        IMAGE_FEATURE_EXTRACTOR=dict(_target_="models.MultiScaleImageFeatureExtractor", freeze=False),
        DIFFUSER=dict(_target_="models.GaussianDiffusion", beta_schedule="custom"),
        DENOISER=dict(_target_="models.Denoiser", TRANSFORMER=cfg_t, target_dim=9, pivot_cam_onehot=True, z_dim=384, mlp_hidden_dim=128))
    model.image_feature_extractor._net.load_state_dict(vit.state_dict())
    model.diffuser.model.load_state_dict(syn.random_denoiser_state(0, 0.02))
    model = model.to(dev).train()
    seqs, frames, repeat = 51, 10, 90
    gen = torch.Generator(device=dev).manual_seed(3)
    image = torch.rand(seqs, frames, 3, 224, 224, device=dev, generator=gen)
    count = seqs * repeat * frames
    eye = torch.eye(3, device=dev).expand(count, 3, 3).contiguous()
    cams = SimpleNamespace(R=eye, T=torch.randn(count, 3, device=dev, generator=gen), focal_length=1.5 + torch.rand(count, 2, device=dev, generator=gen))

    def full_step():
        for p in model.parameters():
            p.grad = None
        model(image=image, gt_cameras=cams, training=True, batch_repeat=repeat)["loss"].mean().backward()

    torch.cuda.empty_cache()
    times, peak = time_steps(full_step, args.steps, args.warmup)
    med = times[len(times) // 2]
    report({"impl": "native_full_step", "images": seqs * frames, "denoiser_tokens": count, "ms_median": round(med, 2),
            "ms_min": round(times[0], 2), "ms_max": round(times[-1], 2), "steps": len(times), "peak_mem_gib": round(peak / 2**30, 2)})
    if args.out:
        with open(args.out, "w") as fh:
            for rec in lines:
                fh.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
