#!/usr/bin/env python
"""Write the outputs of both native training paths and a digest of every gradient, at fixed seeds, to one .npz.

    python tools/train_grad_dump.py --out-dir DIR        # writes DIR/train_grads.npz
    python tools/train_grad_dump.py --compare A.npz B.npz

Gradients are reproducible run to run (fixed-order reductions, no split-K), so a change that only moves host code must leave
every array bit-identical: dump at both commits on the same GPU model and compare.  `--compare` needs no GPU and exits non-zero
unless both files hold the same names and numpy.array_equal holds for each.  Outputs are stored whole; a parameter gradient is
stored as the SHA-256 of its bytes (the denoiser's gradients alone are about 70 MB per case), so equal arrays still mean equal
bits.

Denoiser: (sequences, frames) = (2, 5), (3, 20), (51, 10), dropout 0.1, l1 and l2 loss: loss, x_0_pred, x_t, dL/dz and the 108
parameter gradients.  Backbone: 2 and 7 images of 224x224 at the default scales and 2 images of 224x232: z and the 150 parameter
gradients.
"""
from __future__ import annotations

import argparse
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

DENOISER_SHAPES = [(2, 5), (3, 20), (51, 10)]
BACKBONE_CASES = [(2, 224, 224), (7, 224, 224), (2, 224, 232)]
SCALES = (1, 1 / 2, 1 / 3)
TRANSFORMER = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)


def digest(t) -> np.ndarray:
    return np.frombuffer(hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).digest(), dtype=np.uint8)


def dump(out_dir: str) -> str:
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("train_grad_dump needs a CUDA device")
    import posediffusion_b200 as pdb
    from oracle.dino_vit import DinoViTSmall16, randomize
    from posediffusion_b200 import synthetic as syn

    dev = torch.device("cuda:0")
    arrays = {}
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    den.load_state_dict(syn.random_denoiser_state(3, 0.05), strict=True)
    den = den.to(dev).train()
    for B, N in DENOISER_SHAPES:
        for loss_type in ("l1", "l2"):
            g = torch.Generator().manual_seed(1000 * B + N)
            x, noise = torch.randn(B, N, 9, generator=g) * 0.5, torch.randn(B, N, 9, generator=g)
            t = torch.randint(0, 100, (B,), generator=g)
            gl, gx = torch.randn(B, N, 9, generator=g), torch.randn(B, N, 9, generator=g)
            z = syn.random_features(B, N, B + N).to(dev).requires_grad_(True)
            den.zero_grad(set_to_none=True)
            loss, x0, x_t = den.train_step_forward(x.to(dev), t.to(dev), noise.to(dev), z, 0.1, 0x1234_5678_9ABC, loss_type)
            torch.autograd.backward([loss, x0], [gl.to(dev), gx.to(dev)])
            key = f"denoiser_{B}x{N}_{loss_type}"
            for name, v in (("loss", loss), ("x0", x0), ("x_t", x_t), ("dz", z.grad)):
                arrays[f"{key}/{name}"] = v.detach().cpu().numpy()
            for name, p in den.named_parameters():
                arrays[f"{key}/grad_sha256:{name}"] = digest(p.grad)
    ext = pdb.MultiScaleImageFeatureExtractor(freeze=False, scale_factors=SCALES)
    ext._net.load_state_dict(randomize(DinoViTSmall16(), 11).state_dict(), strict=True)
    ext = ext.to(dev)
    for n, h, w in BACKBONE_CASES:
        img = torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(n + w))
        gz = torch.randn(n, 384, generator=torch.Generator().manual_seed(7))
        ext.zero_grad(set_to_none=True)
        z = ext(img.to(dev))
        z.backward(gz.to(dev))
        key = f"backbone_{n}x{h}x{w}"
        arrays[f"{key}/z"] = z.detach().cpu().numpy()
        for name, p in ext._net.named_parameters():
            arrays[f"{key}/grad_sha256:{name}"] = digest(p.grad)
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "train_grads.npz")
    np.savez(path, **arrays)
    print(f"{path}: {len(arrays)} arrays on {torch.cuda.get_device_name(0)}")
    return path


def compare(a_path: str, b_path: str) -> int:
    a, b = np.load(a_path), np.load(b_path)
    names = sorted(set(a.files) | set(b.files))
    bad = [k for k in names if k not in a.files or k not in b.files or not np.array_equal(a[k], b[k])]
    for k in bad:
        print("differs:", k)
    print(f"{len(names) - len(bad)} of {len(names)} arrays bit-identical")
    return 1 if bad else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=None)
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"))
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    if not args.out_dir:
        ap.error("--out-dir or --compare")
    dump(args.out_dir)


if __name__ == "__main__":
    main()
